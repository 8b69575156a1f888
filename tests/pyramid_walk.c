/* pyramid_walk.c — plain-C restatement of the input downscaling of --pyramid_level (APP/main.cc:299-303,
 * 946-981), which the reference runs on the CPU inside its upload loop. TEST INFRASTRUCTURE: the checker of
 * k_downscale_depth_median* / k_downscale_color (csrc/preprocess.cu), written from the documented semantics
 * (include/surfel_b200.h) in the style of oracle/cpu_walk.c. Built by tests/pyramid_walk.py. */
#include <math.h>
#include <stdint.h>
#include <string.h>

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;

/* Image<u16>::DownscaleUsingMedianWhileExcluding (libvis image.h:1003-1050): output pixel (x, y) covers
 * input columns [W x / w, W (x + 1) / w) and rows [H y / h, H (y + 1) / h) (u32 arithmetic); values equal
 * to value_to_ignore are dropped; none left -> value_to_ignore; odd count -> sorted[n / 2]; even count ->
 * sorted[n / 2 - 1] if it is strictly closer to the float average (float sum / count) than sorted[n / 2],
 * else sorted[n / 2]. Blocks of up to 16 x 16 pixels; tightly packed rasters. */
void cw_downscale_median_excluding(u16 value_to_ignore, int in_width, int in_height, const u16* in, int out_width,
                                   int out_height, u16* out) {
  u16 values[256];
  for (u32 y = 0; y < (u32)out_height; ++y) {
    for (u32 x = 0; x < (u32)out_width; ++x) {
      const u32 x0 = ((u32)in_width * x) / (u32)out_width, x1 = ((u32)in_width * (x + 1)) / (u32)out_width;
      const u32 y0 = ((u32)in_height * y) / (u32)out_height, y1 = ((u32)in_height * (y + 1)) / (u32)out_height;
      int n = 0;
      float sum = 0.f;
      for (u32 yy = y0; yy < y1; ++yy) {
        for (u32 xx = x0; xx < x1; ++xx) {
          const u16 v = in[(size_t)yy * in_width + xx];
          if (v == value_to_ignore || n >= 256) continue;
          /* insertion into the sorted prefix */
          int i = n++;
          while (i > 0 && values[i - 1] > v) { values[i] = values[i - 1]; --i; }
          values[i] = v;
          sum += (float)v;
        }
      }
      u16 result = value_to_ignore;
      if (n > 0) {
        if (n % 2 == 1) {
          result = values[n / 2];
        } else {
          const float average = sum / (float)n;
          const u16 low = values[n / 2 - 1], high = values[n / 2];
          result = fabsf(average - (float)low) < fabsf(average - (float)high) ? low : high;
        }
      }
      out[(size_t)y * out_width + x] = result;
    }
  }
}

/* ImagePyramid(color, levels) (libvis image_cache.h:205-282): `levels` successive halvings of packed
 * 8-bit RGB, each Image<Vec3u8>::DownscaleToHalfSize (image.h:929-948): per channel a/4 + b/4 + c/4 + d/4
 * with every quarter truncated. Every level needs even sizes (the caller checks). `scratch` holds
 * width * height bytes (the intermediate levels one after the other: 3/4 + 3/16 + ... < 1 of that);
 * out is (width >> levels) x (height >> levels) x 3. levels == 0 copies. */
void cw_color_image_pyramid(int levels, int width, int height, const u8* in, u8* scratch, u8* out) {
  if (levels == 0) {
    memcpy(out, in, (size_t)width * height * 3);
    return;
  }
  const u8* src = in;
  int w = width, h = height;
  size_t offset = 0;
  for (int level = 1; level <= levels; ++level) {
    const int ow = w / 2, oh = h / 2;
    u8* dst = level == levels ? out : scratch + offset;
    offset += (size_t)ow * oh * 3;
    for (int y = 0; y < oh; ++y) {
      const u8* upper = src + (size_t)(2 * y) * w * 3;
      const u8* lower = src + (size_t)(2 * y + 1) * w * 3;
      for (int x = 0; x < ow; ++x) {
        for (int c = 0; c < 3; ++c) {
          dst[((size_t)y * ow + x) * 3 + c] =
              (u8)(upper[6 * x + c] / 4 + upper[6 * x + 3 + c] / 4 + lower[6 * x + c] / 4 + lower[6 * x + 3 + c] / 4);
        }
      }
    }
    src = dst;
    w = ow;
    h = oh;
  }
}
