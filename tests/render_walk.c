/* render_walk.c — plain-C restatement of sm_render_surfels (include/surfel_b200.h, "rendering the surfel cloud").
 * TEST INFRASTRUCTURE: the checker of k_render_splat / k_render_large / k_render_resolve (csrc/render.cu), written
 * from the documented semantics. fp32 throughout, no contraction (built with -ffp-contract=off), fmaf where the
 * library's helpers use an FMA, and FTZ / DAZ set in MXCSR for the duration of the call to match -ftz=true.
 * Each surfel tests its own screen rectangle, computed here in double with a wide margin: any superset of the
 * covered pixels gives the same images. Built by tests/render_walk.py. */
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <xmmintrin.h>

typedef uint8_t u8;
typedef uint32_t u32;
typedef uint64_t u64;

enum { ROW_SMOOTH_X = 3, ROW_RADIUS_SQUARED = 7, ROW_NORMAL_X = 8, ROW_COLOR = 24 };

static float transform_row(const float* r, float px, float py, float pz) {
  float t = py * r[1];
  t = fmaf(px, r[0], t);
  t = fmaf(pz, r[2], t);
  return t + r[3];
}
static float rotate_row(const float* r, float px, float py, float pz) {
  float t = py * r[1];
  t = fmaf(px, r[0], t);
  return fmaf(pz, r[2], t);
}
static float dot3(float ax, float ay, float az, float bx, float by, float bz) {
  return fmaf(az, bz, fmaf(ax, bx, ay * by));
}
static float ray_coord(int p, float c, float f) { return (((float)p + 0.5f) - c) / f; }

/* Pixels of one axis that a hit point within `reach` of the centre can project to, with two pixels of margin. */
static int axis_range(double c, double cz, double reach, double f, double cc, int size, int* p0, int* p1) {
  const double z_lo = cz - reach, z_hi = cz + reach, lo = c - reach, hi = c + reach;
  const double d_min = lo >= 0 ? lo / z_hi : lo / z_lo, d_max = hi >= 0 ? hi / z_lo : hi / z_hi;
  double q0 = f * d_min + cc - 0.5, q1 = f * d_max + cc - 0.5;
  if (f < 0) { const double q = q0; q0 = q1; q1 = q; }
  q0 = floor(q0) - 2;
  q1 = ceil(q1) + 2;
  if (q0 < 0) q0 = 0;
  if (q1 > size - 1) q1 = size - 1;
  if (!(q0 <= q1)) return 0;
  *p0 = (int)q0;
  *p1 = (int)q1;
  return 1;
}

/* rows: [25][stride] float32 (rows 3-5 = the smooth position, as sm_dump_state returns them), slots [0, n).
 * T: view_T_global, 3x4 row-major. Outputs: tightly packed [height][width](x3); keys: width * height scratch. */
void rw_render(const float* rows, u64 stride, u32 n, int width, int height, float fx, float fy, float cx, float cy,
               float near_depth, float far_depth, const float* T, float* depth, u8* color, float* normal, u32* index,
               u64* keys) {
  const unsigned saved_csr = _mm_getcsr();
  _mm_setcsr(saved_csr | 0x8040u); /* FTZ | DAZ */
  const size_t P = (size_t)width * height;
  for (size_t k = 0; k < P; ++k) keys[k] = ~0ull;
#define ROW(r, i) rows[(size_t)(r) * stride + (i)]
  for (u32 i = 0; i < n; ++i) {
    const float radius_squared = ROW(ROW_RADIUS_SQUARED, i);
    if (!(radius_squared > 0.f)) continue;
    const float sx = ROW(ROW_SMOOTH_X, i), sy = ROW(ROW_SMOOTH_X + 1, i), sz = ROW(ROW_SMOOTH_X + 2, i);
    const float c[3] = {transform_row(T, sx, sy, sz), transform_row(T + 4, sx, sy, sz), transform_row(T + 8, sx, sy, sz)};
    if (!(near_depth <= c[2] && c[2] <= far_depth)) continue;
    const float nx = ROW(ROW_NORMAL_X, i), ny = ROW(ROW_NORMAL_X + 1, i), nz = ROW(ROW_NORMAL_X + 2, i);
    const float m[3] = {rotate_row(T, nx, ny, nz), rotate_row(T + 4, nx, ny, nz), rotate_row(T + 8, nx, ny, nz)};
    const float num = dot3(m[0], m[1], m[2], c[0], c[1], c[2]);
    int x0 = 0, x1 = width - 1, y0 = 0, y1 = height - 1;
    const double reach = sqrt((double)radius_squared) * 1.01 + 1e-4 * (fabs(c[0]) + fabs(c[1]) + fabs(c[2]));
    if (c[2] - reach > 0) {
      if (!axis_range(c[0], c[2], reach, fx, cx, width, &x0, &x1) || !axis_range(c[1], c[2], reach, fy, cy, height, &y0, &y1))
        continue;
    }
    for (int py = y0; py <= y1; ++py) {
      const float dy = ray_coord(py, cy, fy);
      for (int px = x0; px <= x1; ++px) {
        const float dx = ray_coord(px, cx, fx);
        const float den = dot3(m[0], m[1], m[2], dx, dy, 1.0f);
        if (den == 0.f) continue;
        const float t = num / den;
        if (!(t > 0.f) || !isfinite(t)) continue;
        const float ex = t * dx - c[0], ey = t * dy - c[1], ez = t - c[2];
        if (!(fmaf(ez, ez, fmaf(ex, ex, ey * ey)) <= radius_squared)) continue;
        u32 bits;
        memcpy(&bits, &t, 4);
        const u64 key = ((u64)bits << 32) | i;
        u64* slot = keys + (size_t)py * width + px;
        if (key < *slot) *slot = key;
      }
    }
  }
  for (size_t k = 0; k < P; ++k) {
    float d = 0.f, mm[3] = {0.f, 0.f, 0.f};
    u32 idx = 0xFFFFFFFFu, rgb = 0;
    if (keys[k] != ~0ull) {
      idx = (u32)keys[k];
      const u32 bits = (u32)(keys[k] >> 32);
      memcpy(&d, &bits, 4);
      memcpy(&rgb, &ROW(ROW_COLOR, idx), 4);
      const float nx = ROW(ROW_NORMAL_X, idx), ny = ROW(ROW_NORMAL_X + 1, idx), nz = ROW(ROW_NORMAL_X + 2, idx);
      mm[0] = rotate_row(T, nx, ny, nz);
      mm[1] = rotate_row(T + 4, nx, ny, nz);
      mm[2] = rotate_row(T + 8, nx, ny, nz);
    }
    depth[k] = d;
    index[k] = idx;
    color[3 * k] = rgb & 0xFFu;
    color[3 * k + 1] = (rgb >> 8) & 0xFFu;
    color[3 * k + 2] = (rgb >> 16) & 0xFFu;
    memcpy(normal + 3 * k, mm, sizeof(mm));
  }
#undef ROW
  _mm_setcsr(saved_csr);
}
