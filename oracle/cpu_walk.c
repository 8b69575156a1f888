/* oracle/cpu_walk.c — TEST INFRASTRUCTURE, not product code.
 *
 * Plain-C CPU restatement ("port") of the per-pixel depth filter chain and of the
 * per-surfel min-depth + association loop of puzzlepaint/surfelmeshing. The reference
 * ships NO CPU implementation of this path (SURVEY.md §8c/§8d); this walk exists
 *   (1) as the reported CPU baseline of bench.py (`cpu_baseline`, kind "port"), and
 *   (2) as a sequential-semantics cross-check of the oracle/product in tests/.
 * It follows, function by function (APP = applications/surfel_meshing/src/surfel_meshing):
 *   cw_bilateral   APP/cuda_depth_processing.cu:50-118
 *   cw_outlier     APP/cuda_depth_processing.cu:168-227 (all inliers) / :337-397 (>= required)
 *   cw_erode       APP/cuda_depth_processing.cu:514-538, :589-607
 *   cw_normals     APP/cuda_depth_processing.cu:642-718
 *   cw_radii       APP/cuda_depth_processing.cu:765-837
 *   cw_preprocess  APP/main.cc:1015-1191 (the five stages in sequence)
 *   cw_associate   APP/cuda_surfel_reconstruction_kernels.cu:1466-1557 (min depth),
 *                  :1586-1808 (association)
 * Parity status: "parity unpinned" by reference tests (the reference has none for this
 * path); pinned against the reference's own kernels run on the GPU (tests/golden/, produced
 * by tests/golden/make_golden.py through oracle/_ref/libsurfel_ref.so). IEEE division,
 * expf and sqrtf replace the GPU's approximate MUFU ops, so u16 results may differ from the
 * GPU by 1 LSB on a small fraction of pixels (tolerance stated in tests/test_cpu_walk.py).
 *
 * Only tests/, __graft_entry__ and bench.py's cpu_baseline leg may load this library.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef uint8_t u8;

#define CW_INVALID 0xFFFFFFFFu

int cw_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

void cw_set_threads(int n) {
#ifdef _OPENMP
  if (n > 0) omp_set_num_threads(n);
#else
  (void)n;
#endif
}

/* ---- a1 ------------------------------------------------------------------------------- */
void cw_bilateral(float sigma_xy, float sigma_value_factor, u16 value_to_ignore, float radius_factor, u16 max_depth,
                  float depth_valid_region_radius, int W, int H, const u16* in, u16* out) {
  const int radius = (int)(radius_factor * sigma_xy + 0.5f);
  const int radius_squared = radius * radius;
  const float denom_xy = 2.0f * sigma_xy * sigma_xy;
  const float valid_r2 = depth_valid_region_radius * depth_valid_region_radius;
#pragma omp parallel for schedule(dynamic, 4)
  for (int y = 0; y < H; ++y) {
    for (int x = 0; x < W; ++x) {
      const int hx = x - W / 2, hy = y - H / 2;
      const float center_distance_squared = (float)(hx * hx + hy * hy);
      if (center_distance_squared > valid_r2) { out[y * W + x] = value_to_ignore; continue; }
      const u16 center_value = in[y * W + x];
      if (center_value == value_to_ignore || center_value > max_depth) { out[y * W + x] = value_to_ignore; continue; }
      const float adapted_sigma_value = center_value * sigma_value_factor;
      const float adapted_denom_value = 2.0f * adapted_sigma_value * adapted_sigma_value;
      float sum = 0, weight = 0;
      const int min_y = y - radius < 0 ? 0 : y - radius, max_y = y + radius > H - 1 ? H - 1 : y + radius;
      const int min_x = x - radius < 0 ? 0 : x - radius, max_x = x + radius > W - 1 ? W - 1 : x + radius;
      for (int sy = min_y; sy <= max_y; ++sy) {
        const int dy = sy - y;
        for (int sx = min_x; sx <= max_x; ++sx) {
          const int dx = sx - x;
          const int grid_distance_squared = dx * dx + dy * dy;
          if (grid_distance_squared > radius_squared) continue;
          const u16 sample = in[sy * W + sx];
          if (sample == value_to_ignore) continue;
          float value_distance_squared = (float)(center_value - sample);
          value_distance_squared *= value_distance_squared;
          const float w = expf(-grid_distance_squared / denom_xy + -value_distance_squared / adapted_denom_value);
          sum += w * sample;
          weight += w;
        }
      }
      out[y * W + x] = (weight == 0) ? value_to_ignore : (u16)(sum / weight + 0.5f);
    }
  }
}

/* ---- a2 ------------------------------------------------------------------------------- */
void cw_outlier(int other_count, int required_count, float tolerance, float fx, float fy, float cx, float cy, int W,
                int H, const u16* in, const u16* const* other_depths, const float* others_TR_reference, u16* out) {
  const float max_tol = 1 + tolerance, min_tol = 1 - tolerance;
  const float fx_inv = 1.0f / fx, fy_inv = 1.0f / fy;
  const float cx_inv = -(cx - 0.5f) / fx, cy_inv = -(cy - 0.5f) / fy;
  const int all = (required_count < 0 || required_count == other_count);
#pragma omp parallel for schedule(dynamic, 4)
  for (int y = 0; y < H; ++y) {
    for (int x = 0; x < W; ++x) {
      const u16 depth_value = in[y * W + x];
      if (depth_value == 0) { out[y * W + x] = 0; continue; }
      const float px = depth_value * (fx_inv * x + cx_inv), py = depth_value * (fy_inv * y + cy_inv), pz = depth_value;
      int ok_count = 0, ok = 1;
      for (int k = 0; k < other_count; ++k) {
        const float* m = others_TR_reference + 12 * k;
        const float ox = m[0] * px + m[1] * py + m[2] * pz + m[3];
        const float oy = m[4] * px + m[5] * py + m[6] * pz + m[7];
        const float oz = m[8] * px + m[9] * py + m[10] * pz + m[11];
        int good = 0;
        if (oz > 0) {
          const int ix = (int)(fx * (ox / oz) + cx), iy = (int)(fy * (oy / oz) + cy);
          if (ix >= 0 && iy >= 0 && ix < W && iy < H) {
            const u16 od = other_depths[k][iy * W + ix];
            if (!(od <= 0 || od > max_tol * oz || od < min_tol * oz)) good = 1;
          }
        }
        if (good) ++ok_count;
        else if (all) { ok = 0; break; }
      }
      out[y * W + x] = all ? (ok ? depth_value : 0) : (ok_count >= required_count ? depth_value : 0);
    }
  }
}

/* ---- a3 ------------------------------------------------------------------------------- */
void cw_erode(int radius, int W, int H, const u16* in, u16* out) {
#pragma omp parallel for
  for (int y = 0; y < H; ++y) {
    for (int x = 0; x < W; ++x) {
      const int border = radius == 0 ? 1 : radius;
      if (x < border || y < border || x >= W - border || y >= H - border) { out[y * W + x] = 0; continue; }
      int all_valid = 1;
      for (int dy = y - radius; dy <= y + radius; ++dy)
        for (int dx = x - radius; dx <= x + radius; ++dx)
          if (in[dy * W + dx] == 0) all_valid = 0;
      out[y * W + x] = all_valid ? in[y * W + x] : 0;
    }
  }
}

/* ---- a4 ------------------------------------------------------------------------------- */
void cw_normals(float observation_angle_threshold_deg, float depth_scaling, float fx, float fy, float cx, float cy,
                int W, int H, const u16* in, u16* out, float* normals /* 2 per pixel */) {
  const float thr = -1 * cosf(M_PI / 180.f * observation_angle_threshold_deg);
  const float ids = 1.0f / depth_scaling;
  const float fx_inv = 1.0f / fx, fy_inv = 1.0f / fy;
  const float cx_inv = -(cx - 0.5f) / fx, cy_inv = -(cy - 0.5f) / fy;
#pragma omp parallel for
  for (int y = 0; y < H; ++y) {
    for (int x = 0; x < W; ++x) {
      const int p = y * W + x;
      normals[2 * p] = 0; normals[2 * p + 1] = 0; out[p] = 0;
      if (in[p] == 0 || x < 1 || y < 1 || x >= W - 1 || y >= H - 1) continue;
      const u16 r = in[p + 1], l = in[p - 1], b = in[p + W], t = in[p - W];
      if (r == 0 || l == 0 || b == 0 || t == 0) continue;
      const float ld = ids * l, td = ids * t, rd = ids * r, bd = ids * b;
      const float lp[3] = {ld * (fx_inv * (x - 1) + cx_inv), ld * (fy_inv * y + cy_inv), ld};
      const float tp[3] = {td * (fx_inv * x + cx_inv), td * (fy_inv * (y - 1) + cy_inv), td};
      const float rp[3] = {rd * (fx_inv * (x + 1) + cx_inv), rd * (fy_inv * y + cy_inv), rd};
      const float bp[3] = {bd * (fx_inv * x + cx_inv), bd * (fy_inv * (y + 1) + cy_inv), bd};
      const float a[3] = {rp[0] - lp[0], rp[1] - lp[1], rp[2] - lp[2]};
      const float c[3] = {tp[0] - bp[0], tp[1] - bp[1], tp[2] - bp[2]};
      float n[3] = {a[1] * c[2] - c[1] * a[2], c[0] * a[2] - a[0] * c[2], a[0] * c[1] - c[0] * a[1]};
      const float length = sqrtf(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
      if (!(length > 1e-6f)) { n[0] = 0; n[1] = 0; n[2] = -1; }
      else { const float inv = ((fy_inv < 0) ? -1.0f : 1.0f) / length; n[0] *= inv; n[1] *= inv; n[2] *= inv; }
      normals[2 * p] = n[0]; normals[2 * p + 1] = n[1];
      float v[3] = {fx_inv * x + cx_inv, fy_inv * y + cy_inv, 1};
      const float inv_dir = 1.0f / sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
      const float dot = inv_dir * v[0] * n[0] + inv_dir * v[1] * n[1] + inv_dir * v[2] * n[2];
      out[p] = (dot >= thr) ? 0 : in[p];
    }
  }
}

/* ---- a5 ------------------------------------------------------------------------------- */
void cw_radii(float point_radius_extension_factor, float point_radius_clamp_factor, float depth_scaling, float fx,
              float fy, float cx, float cy, int W, int H, const u16* in, float* radius, u16* out) {
  const float ext2 = point_radius_extension_factor * point_radius_extension_factor;
  const float clamp_term = point_radius_clamp_factor * point_radius_clamp_factor * sqrtf(2) * sqrtf(2);
  const float ids = 1.0f / depth_scaling;
  const float fx_inv = 1.0f / fx, fy_inv = 1.0f / fy;
  const float cx_inv = -(cx - 0.5f) / fx, cy_inv = -(cy - 0.5f) / fy;
#pragma omp parallel for
  for (int y = 0; y < H; ++y) {
    for (int x = 0; x < W; ++x) {
      const int p = y * W + x;
      if (in[p] == 0) { out[p] = 0; continue; }
      const float depth = ids * in[p];
      const float lp[3] = {depth * (fx_inv * x + cx_inv), depth * (fy_inv * y + cy_inv), depth};
      int neighbor_count = 0;
      float radius_squared = 0, min_d2 = INFINITY;
      for (int dy = y - 1; dy <= y + 1; ++dy) {
        for (int dx = x - 1; dx <= x + 1; ++dx) {
          if (dx < 0 || dy < 0 || dx >= W || dy >= H) continue;
          const float dd = ids * in[dy * W + dx];
          if ((dx == x && dy == y) || dd <= 0) continue;
          ++neighbor_count;
          const float o[3] = {dd * (fx_inv * dx + cx_inv) - lp[0], dd * (fy_inv * dy + cy_inv) - lp[1], dd - lp[2]};
          const float d2 = o[0] * o[0] + o[1] * o[1] + o[2] * o[2];
          if (d2 > radius_squared) radius_squared = d2;
          if (d2 < min_d2) min_d2 = d2;
        }
      }
      radius_squared *= ext2;
      const float clamp = clamp_term * min_d2;
      if (radius_squared > clamp) radius_squared = clamp;
      radius[p] = radius_squared;
      out[p] = (neighbor_count < 8) ? 0 : in[p];
    }
  }
}

/* ---- f2: MedianFilterAndDensifyDepthMap (APP/main.cc:207-252), one iteration ---------------
 * 3x3 window clipped to the image, zeros excluded; with >= 2 valid values the output is their
 * median (even count: the middle element closer to the float average, the upper one on a tie),
 * otherwise the input pixel. Fills holes that have >= 2 valid neighbours. */
void cw_median_filter_and_densify(int W, int H, const u16* in, u16* out) {
#pragma omp parallel for schedule(static)
  for (int y = 0; y < H; ++y) {
    for (int x = 0; x < W; ++x) {
      u16 values[9];
      int n = 0;
      const int dy_end = (H - 1 < y + 1) ? H - 1 : y + 1;
      for (int dy = (y - 1 > 0) ? y - 1 : 0; dy <= dy_end; ++dy) {
        const int dx_end = (W - 1 < x + 1) ? W - 1 : x + 1;
        for (int dx = (x - 1 > 0) ? x - 1 : 0; dx <= dx_end; ++dx) {
          if (in[dy * W + dx] != 0) values[n++] = in[dy * W + dx];
        }
      }
      if (n >= 2) {
        for (int i = 1; i < n; ++i) { /* insertion sort = std::sort on <= 9 keys */
          const u16 v = values[i];
          int j = i - 1;
          while (j >= 0 && values[j] > v) { values[j + 1] = values[j]; --j; }
          values[j + 1] = v;
        }
        if (n % 2 == 0) {
          float sum = 0;
          for (int i = 0; i < n; ++i) sum += values[i];
          const float average = sum / n;
          const float prev_diff = fabsf(values[n / 2 - 1] - average);
          const float next_diff = fabsf(values[n / 2] - average);
          out[y * W + x] = (prev_diff < next_diff) ? values[n / 2 - 1] : values[n / 2];
        } else {
          out[y * W + x] = values[n / 2];
        }
      } else {
        out[y * W + x] = in[y * W + x];
      }
    }
  }
}

/* ---- a16: the five stages of APP/main.cc:1015-1191 ------------------------------------- */
typedef struct cw_preprocess_params {
  float depth_scaling, max_depth, depth_valid_region_radius, bilateral_filter_sigma_xy, bilateral_filter_radius_factor,
      bilateral_filter_sigma_depth_factor;
  int32_t outlier_filtering_frame_count, outlier_filtering_required_inliers;
  float outlier_filtering_depth_tolerance_factor;
  int32_t depth_erosion_radius;
  float observation_angle_threshold_deg, point_radius_extension_factor, point_radius_clamp_factor;
} cw_preprocess_params; /* same layout as sm_preprocess_params */

void cw_preprocess(const cw_preprocess_params* p, float fx, float fy, float cx, float cy, int W, int H, const u16* raw,
                   const u16* const* other_depths, const float* others_TR_reference, u16* scratch_A, u16* scratch_B,
                   u16* out_depth, float* out_normals, float* out_radius) {
  cw_bilateral(p->bilateral_filter_sigma_xy, p->bilateral_filter_sigma_depth_factor, 0,
               p->bilateral_filter_radius_factor, (u16)(p->depth_scaling * p->max_depth),
               p->depth_valid_region_radius, W, H, raw, scratch_A);
  cw_outlier(p->outlier_filtering_frame_count, p->outlier_filtering_required_inliers,
             p->outlier_filtering_depth_tolerance_factor, fx, fy, cx, cy, W, H, scratch_A, other_depths,
             others_TR_reference, scratch_B);
  cw_erode(p->depth_erosion_radius, W, H, scratch_B, scratch_A);
  cw_normals(p->observation_angle_threshold_deg, p->depth_scaling, fx, fy, cx, cy, W, H, scratch_A, scratch_B,
             out_normals);
  cw_radii(p->point_radius_extension_factor, p->point_radius_clamp_factor, p->depth_scaling, fx, fy, cx, cy, W, H,
           scratch_B, out_radius, out_depth);
}

/* ---- a7 + a8 --------------------------------------------------------------------------- */
static inline int cw_project(const float* T, float fx, float fy, float cx, float cy, int W, int H, float X, float Y,
                             float Z, float* lp, float* u, float* v, int* px, int* py) {
  lp[0] = T[0] * X + T[1] * Y + T[2] * Z + T[3];
  lp[1] = T[4] * X + T[5] * Y + T[6] * Z + T[7];
  lp[2] = T[8] * X + T[9] * Y + T[10] * Z + T[11];
  if (lp[2] <= 0) return 0;
  *u = fx * (lp[0] / lp[2]) + cx;
  *v = fy * (lp[1] / lp[2]) + cy;
  *px = (int)*u;
  *py = (int)*v;
  return !(*u < 0 || *v < 0 || *px < 0 || *py < 0 || *px >= W || *py >= H);
}

static inline int cw_secondary(float u, float v, int px, int py, int W, int H, int* ox, int* oy) {
  const float xf = u - px, yf = v - py;
  if (xf < yf) {
    if (xf < 1 - yf) { if (px > 1) { *ox = px - 1; *oy = py; return 1; } return 0; }
    if (py < H - 1) { *ox = px; *oy = py + 1; return 1; }
    return 0;
  }
  if (xf < 1 - yf) { if (py > 0) { *ox = px; *oy = py - 1; return 1; } return 0; }
  if (px < W - 1) { *ox = px + 1; *oy = py; return 1; }
  return 0;
}

/* surfels: the 25-row SoA (row stride `stride` floats). Rasters are W*H, tightly packed.
 * supporting_surfels receives the canonical winner (primary association before secondary,
 * then lowest index). The walk over surfels is sequential per thread; min-depth uses an
 * atomic min on the int-punned float exactly like the reference. */
static void cw_associate_impl(const float* surfels, size_t stride, u32 surfel_count, u32 frame_index, int active_window, float fx,
                  float fy, float cx, float cy, const float* local_T_global, float sensor_noise_factor,
                  float normal_compatibility_threshold_deg, float depth_scaling, int W, int H, const u16* depth,
                  const float* normals, u32* supporting_surfels, u32* supporting_surfel_counts,
                  float* supporting_surfel_depth_sums, u32* conflicting_surfels, float* first_surfel_depth,
                  u32* event_pixel, u32* event_key, u64 max_events, u64* event_count) {
  const float cos_thr = cosf(M_PI / 180.0f * normal_compatibility_threshold_deg);
  const float corr = 1.0f / depth_scaling;
  const size_t P = (size_t)W * H;
  const u32* stamps = (const u32*)(surfels + 18 * stride);
  for (size_t i = 0; i < P; ++i) {
    supporting_surfels[i] = CW_INVALID; supporting_surfel_counts[i] = 0; supporting_surfel_depth_sums[i] = 0;
    conflicting_surfels[i] = CW_INVALID; first_surfel_depth[i] = INFINITY;
  }
  int32_t* first_i = (int32_t*)first_surfel_depth;
#pragma omp parallel for schedule(static, 4096)
  for (u32 i = 0; i < surfel_count; ++i) {
    if (!((int)stamps[i] > (int)(frame_index - (u32)active_window))) continue;
    float lp[3], u, v; int px, py, ox, oy;
    if (!cw_project(local_T_global, fx, fy, cx, cy, W, H, surfels[i], surfels[stride + i], surfels[2 * stride + i], lp,
                    &u, &v, &px, &py)) continue;
    int32_t zi; memcpy(&zi, &lp[2], 4);
    int n_pix = 1, xs[2] = {px, 0}, ys[2] = {py, 0};
    if (cw_secondary(u, v, px, py, W, H, &ox, &oy)) { xs[1] = ox; ys[1] = oy; n_pix = 2; }
    for (int k = 0; k < n_pix; ++k) {
      int32_t* addr = &first_i[ys[k] * W + xs[k]];
      int32_t old = __atomic_load_n(addr, __ATOMIC_RELAXED);
      while (zi < old && !__atomic_compare_exchange_n(addr, &old, zi, 1, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
    }
  }
#pragma omp parallel for schedule(static, 4096)
  for (u32 i = 0; i < surfel_count; ++i) {
    if (!((int)stamps[i] > (int)(frame_index - (u32)active_window))) continue;
    float lp[3], u, v; int px, py, ox, oy;
    if (!cw_project(local_T_global, fx, fy, cx, cy, W, H, surfels[i], surfels[stride + i], surfels[2 * stride + i], lp,
                    &u, &v, &px, &py)) continue;
    int n_pix = 1, xs[2] = {px, 0}, ys[2] = {py, 0};
    if (cw_secondary(u, v, px, py, W, H, &ox, &oy)) { xs[1] = ox; ys[1] = oy; n_pix = 2; }
    for (int k = 0; k < n_pix; ++k) {
      const int p = ys[k] * W + xs[k];
      const float measurement_depth = corr * depth[p];
      if (measurement_depth <= 0) continue;
      const float first = first_surfel_depth[p];
      if (first < (1 - sensor_noise_factor) * measurement_depth) {
        if (first == lp[2]) conflicting_surfels[p] = i;
        continue;
      }
      if (lp[2] > (1 + sensor_noise_factor) * measurement_depth) continue;
      const float dist = sqrtf(lp[0] * lp[0] + lp[1] * lp[1] + lp[2] * lp[2]);
      const float gn[3] = {surfels[8 * stride + i], surfels[9 * stride + i], surfels[10 * stride + i]};
      const float* T = local_T_global;
      const float ln[3] = {T[0] * gn[0] + T[1] * gn[1] + T[2] * gn[2], T[4] * gn[0] + T[5] * gn[1] + T[6] * gn[2],
                           T[8] * gn[0] + T[9] * gn[1] + T[10] * gn[2]};
      if ((1.0f / dist) * (lp[0] * ln[0] + lp[1] * ln[1] + lp[2] * ln[2]) > 0) continue;
      if (measurement_depth < lp[2]) {
        const float nx = normals[2 * p], ny = normals[2 * p + 1];
        const float t = 1 - nx * nx - ny * ny;
        const float nz = -sqrtf(t > 0 ? t : 0);
        if (ln[0] * nx + ln[1] * ny + ln[2] * nz < cos_thr) continue;
      }
      if (surfels[7 * stride + i] <= 0) continue;
      const u32 key = i | (k ? 0x80000000u : 0u);
      if (event_count) { /* every association that reaches the atomicCAS of kernels.cu:1688 */
        const u64 e = __atomic_fetch_add(event_count, 1ull, __ATOMIC_RELAXED);
        if (e < max_events) { event_pixel[e] = (u32)p; event_key[e] = key; }
      }
      u32 old = __atomic_load_n(&supporting_surfels[p], __ATOMIC_RELAXED);
      while (key < old && !__atomic_compare_exchange_n(&supporting_surfels[p], &old, key, 1, __ATOMIC_RELAXED,
                                                       __ATOMIC_RELAXED)) {}
      __atomic_fetch_add(&supporting_surfel_counts[p], 1u, __ATOMIC_RELAXED);
#pragma omp atomic
      supporting_surfel_depth_sums[p] += lp[2];
    }
  }
  for (size_t i = 0; i < P; ++i)
    if (supporting_surfels[i] != CW_INVALID) supporting_surfels[i] &= 0x7FFFFFFFu;
}

void cw_associate(const float* surfels, size_t stride, u32 surfel_count, u32 frame_index, int active_window, float fx,
                  float fy, float cx, float cy, const float* local_T_global, float sensor_noise_factor,
                  float normal_compatibility_threshold_deg, float depth_scaling, int W, int H, const u16* depth,
                  const float* normals, u32* supporting_surfels, u32* supporting_surfel_counts,
                  float* supporting_surfel_depth_sums, u32* conflicting_surfels, float* first_surfel_depth) {
  cw_associate_impl(surfels, stride, surfel_count, frame_index, active_window, fx, fy, cx, cy, local_T_global,
                    sensor_noise_factor, normal_compatibility_threshold_deg, depth_scaling, W, H, depth, normals,
                    supporting_surfels, supporting_surfel_counts, supporting_surfel_depth_sums, conflicting_surfels,
                    first_surfel_depth, 0, 0, 0, 0);
}

/* The same walk, also listing every (pixel, surfel) association that reaches the reference's
 * atomicCAS (kernels.cu:1688): event_key = surfel index | 0x80000000 for a secondary-pixel
 * association. The supporter SET of a pixel = the events with that pixel; the reference's winner
 * is whichever of them arrives first. *event_count receives the number of events (may exceed
 * max_events: then only the first max_events were stored). Order of the events is arbitrary. */
void cw_associate_events(const float* surfels, size_t stride, u32 surfel_count, u32 frame_index, int active_window,
                         float fx, float fy, float cx, float cy, const float* local_T_global,
                         float sensor_noise_factor, float normal_compatibility_threshold_deg, float depth_scaling, int W,
                         int H, const u16* depth, const float* normals, u32* supporting_surfels,
                         u32* supporting_surfel_counts, float* supporting_surfel_depth_sums, u32* conflicting_surfels,
                         float* first_surfel_depth, u32* event_pixel, u32* event_key, u64 max_events, u64* event_count) {
  *event_count = 0;
  cw_associate_impl(surfels, stride, surfel_count, frame_index, active_window, fx, fy, cx, cy, local_T_global,
                    sensor_noise_factor, normal_compatibility_threshold_deg, depth_scaling, W, H, depth, normals,
                    supporting_surfels, supporting_surfel_counts, supporting_surfel_depth_sums, conflicting_surfels,
                    first_surfel_depth, event_pixel, event_key, max_events, event_count);
}
