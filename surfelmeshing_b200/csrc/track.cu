// track.cu — sm_track_frame / sm_track_linearize (DESIGN.md section 5.6): the live depth map tracked against a model
// view by projective point-to-plane ICP, coarse to fine, with every Gauss-Newton iteration on the device. The
// per-pixel rules are in include/surfel_b200.h.
//
// One frame on the caller's stream, one host synchronisation at the end:
//   bilateral filter + depth cutoff of the raw map       (StageBilateral, the kernel of the pre-processing)
//   levels 1..L-1: k_downscale_depth_median of level 0   (StageDownscaleMedian, the path of "pyramid_level")
//   model view: RenderSurfels at the handle's camera     (SM_TRACK_CLOUD; the previous frame's view otherwise)
//   k_track_live_view  level-0 depth and normals, kept as the model view of the next SM_TRACK_PREVIOUS_FRAME call
//   per level, coarse to fine, per iteration:
//     k_track_linearize  resident grid, grid-stride over the live pixels: fp32 per-pixel terms, fp64 sums in
//                        registers, warp shuffles and a block reduction into one partial row per block (no atomics)
//     k_track_solve      one block: sums the rows in block order, Cholesky, SE(3) exponential, pose update in fp64
// Both iteration kernels return at once when the frame is lost or the level has converged (TrackState), so the
// launch count does not depend on the data.

#include <cmath>
#include <string>

#include "sm_handle.cuh"

namespace smb {

namespace {

#define SM_CUDA(call)                                                                                   \
  do {                                                                                                  \
    const cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) return SetError(SM_ERR_CUDA, (std::string(#call) + ": " + cudaGetErrorString(e_)).c_str()); \
  } while (0)

constexpr int kLinearizeBlock = 256;
constexpr int kLinearizeWarps = kLinearizeBlock / 32;
constexpr int kSolveBlock = 256;
constexpr int kSolveChunks = 8;   // the solve sums the partial rows in 8 chunks of consecutive blocks
// Terms of one partial row: the upper triangle of J^T J (21, row by row), J^T r (6), sum r^2, inliers, valid pixels.
constexpr int kTerms = 30;
constexpr int kSystemTerms = 27;
constexpr int kTermR2 = 27, kTermInliers = 28, kTermValid = 29;
constexpr int kMaxLevels = 4;
// Depth range of the model render (metres).
constexpr float kModelNear = 0.1f, kModelFar = 100.f;

}  // namespace

// Device-resident tracker state: the pose being refined and the flags the iteration kernels read.
struct TrackState {
  float pose[12];        // model_T_live, 3x4 row-major
  int lost;              // a pivot <= 0, a non-finite step or too few inliers
  int done_level;        // the level whose step fell below the convergence thresholds (-1: none yet)
  int iterations;        // Gauss-Newton steps applied
  u32 inliers, valid;    // level 0, last linearisation
  float rms;             // level 0, last linearisation: sqrt(sum r^2 / inliers)
  double system[kTerms]; // sums of the last linearisation
};

namespace {

struct LinearizeArgs {
  int level;
  int width, height;              // live image
  float fx, fy, cx, cy;           // live intrinsics (pixel-corner)
  float inv_depth_scaling;
  const u16* live; size_t live_pitch;
  int model_width, model_height;
  float mfx, mfy, mcx, mcy;
  const float* model_depth; size_t model_depth_pitch;
  const float* model_normal; size_t model_normal_pitch;
  float max_distance_squared;
  float cos_max_angle;
  TrackState* state;
  double* partials;               // [gridDim.x][kTerms]
};

struct LiveViewArgs {
  int width, height;
  float fx, fy, cx, cy;
  float inv_depth_scaling;
  const u16* live; size_t live_pitch;
  float* depth; size_t depth_pitch;
  float* normal; size_t normal_pitch;
};

struct SolveArgs {
  int level;
  int solve;                      // 0: only sum the partial rows into state->system
  int blocks;                     // partial rows
  const double* partials;
  TrackState* state;
  float min_inlier_fraction;
  float convergence_rotation, convergence_translation;
};

// ((p + 0.5) - c) / f, IEEE division: the pixel-centre ray of sm_render_surfels.
__device__ __forceinline__ float ray_coord(int p, float c, float f) { return __fdiv_rn(fsub(fadd(i2f(p), 0.5f), c), f); }

// a.x*b.x + a.y*b.y + a.z*b.z as ((a.x*b.x + a.y*b.y) + a.z*b.z), every product and sum rounded.
__device__ __forceinline__ float dot_rn(float3 a, float3 b) {
  return fadd(fadd(fmul(a.x, b.x), fmul(a.y, b.y)), fmul(a.z, b.z));
}
__device__ __forceinline__ float3 cross_rn(float3 a, float3 b) {
  return make_float3(fsub(fmul(a.y, b.z), fmul(a.z, b.y)), fsub(fmul(a.z, b.x), fmul(a.x, b.z)),
                     fsub(fmul(a.x, b.y), fmul(a.y, b.x)));
}
__device__ __forceinline__ float3 sub_rn(float3 a, float3 b) { return make_float3(fsub(a.x, b.x), fsub(a.y, b.y), fsub(a.z, b.z)); }
// n / sqrt(n . n) with IEEE sqrt and division; false if n . n is not finite and > 0.
__device__ __forceinline__ bool normalize_rn(float3* n) {
  const float len2 = dot_rn(*n, *n);
  if (!(len2 > 0.f) || !isfinite(len2)) return false;
  const float inv = __fdiv_rn(1.f, __fsqrt_rn(len2));
  *n = make_float3(fmul(n->x, inv), fmul(n->y, inv), fmul(n->z, inv));
  return true;
}
// Row of a rigid transform: ((r.x*p.x + r.y*p.y) + r.z*p.z) + r.w.
__device__ __forceinline__ float3 rigid_point(const float* T, float3 p) {
  return make_float3(fadd(dot_rn(make_float3(T[0], T[1], T[2]), p), T[3]),
                     fadd(dot_rn(make_float3(T[4], T[5], T[6]), p), T[7]),
                     fadd(dot_rn(make_float3(T[8], T[9], T[10]), p), T[11]));
}
__device__ __forceinline__ float3 rigid_vector(const float* T, float3 v) {
  return make_float3(dot_rn(make_float3(T[0], T[1], T[2]), v), dot_rn(make_float3(T[4], T[5], T[6]), v),
                     dot_rn(make_float3(T[8], T[9], T[10]), v));
}

__device__ __forceinline__ float3 live_point(const u16* live, size_t pitch, float inv_scale, float fx, float fy, float cx,
                                             float cy, int x, int y, u16 d) {
  const float z = fmul(u2f(d), inv_scale);
  return make_float3(fmul(z, ray_coord(x, cx, fx)), fmul(z, ray_coord(y, cy, fy)), z);
}

// Steps 1-2 of the header: the live point and its unit normal, false for a border pixel, a zero among the five
// depths or a degenerate normal.
__device__ __forceinline__ bool live_point_normal(const u16* live, size_t pitch, int width, int height, float inv_scale,
                                                  float fx, float fy, float cx, float cy, int x, int y, float3* p,
                                                  float3* n) {
  if (x <= 0 || y <= 0 || x >= width - 1 || y >= height - 1) return false;
  const u16* row = row_ptr(live, pitch, y);
  const u16 dc = row[x], dl = row[x - 1], dr = row[x + 1];
  const u16 du = row_ptr(live, pitch, y - 1)[x], dd = row_ptr(live, pitch, y + 1)[x];
  if (dc == 0 || dl == 0 || dr == 0 || du == 0 || dd == 0) return false;
  *p = live_point(live, pitch, inv_scale, fx, fy, cx, cy, x, y, dc);
  const float3 pl = live_point(live, pitch, inv_scale, fx, fy, cx, cy, x - 1, y, dl);
  const float3 pr = live_point(live, pitch, inv_scale, fx, fy, cx, cy, x + 1, y, dr);
  const float3 pu = live_point(live, pitch, inv_scale, fx, fy, cx, cy, x, y - 1, du);
  const float3 pd = live_point(live, pitch, inv_scale, fx, fy, cx, cy, x, y + 1, dd);
  *n = cross_rn(sub_rn(pd, pu), sub_rn(pr, pl));   // faces the camera
  return normalize_rn(n);
}

__global__ void __launch_bounds__(256) k_track_live_view(LiveViewArgs a) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= a.width) return;
  float3 p, n;
  const bool ok = live_point_normal(a.live, a.live_pitch, a.width, a.height, a.inv_depth_scaling, a.fx, a.fy, a.cx, a.cy, x,
                                    y, &p, &n);
  row_ptr(a.depth, a.depth_pitch, y)[x] = ok ? p.z : 0.f;
  float* o = row_ptr(a.normal, a.normal_pitch, y) + 3 * static_cast<size_t>(x);
  o[0] = ok ? n.x : 0.f; o[1] = ok ? n.y : 0.f; o[2] = ok ? n.z : 0.f;
}

__global__ void __launch_bounds__(kLinearizeBlock) k_track_linearize(LinearizeArgs a) {
  const TrackState* s = a.state;
  if (s->lost || s->done_level == a.level) return;
  float T[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) T[k] = s->pose[k];
  double acc[kTerms];
#pragma unroll
  for (int k = 0; k < kTerms; ++k) acc[k] = 0.0;
  const u32 pixels = static_cast<u32>(a.width) * static_cast<u32>(a.height);
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < pixels; i += gridDim.x * blockDim.x) {
    const int x = static_cast<int>(i % static_cast<u32>(a.width)), y = static_cast<int>(i / static_cast<u32>(a.width));
    float3 p, n;
    if (!live_point_normal(a.live, a.live_pitch, a.width, a.height, a.inv_depth_scaling, a.fx, a.fy, a.cx, a.cy, x, y, &p,
                           &n))
      continue;
    acc[kTermValid] += 1.0;
    const float3 pm = rigid_point(T, p);
    const float3 nl = rigid_vector(T, n);
    if (!(pm.z > 0.f)) continue;
    const float u = fadd(fmul(a.mfx, __fdiv_rn(pm.x, pm.z)), a.mcx);
    const float v = fadd(fmul(a.mfy, __fdiv_rn(pm.y, pm.z)), a.mcy);
    if (!(u >= 0.f && u < i2f(a.model_width) && v >= 0.f && v < i2f(a.model_height))) continue;
    const int ix = static_cast<int>(u), iy = static_cast<int>(v);
    const float dm = row_ptr(a.model_depth, a.model_depth_pitch, iy)[ix];
    if (!(dm > 0.f) || !isfinite(dm)) continue;
    const float* mn = row_ptr(a.model_normal, a.model_normal_pitch, iy) + 3 * static_cast<size_t>(ix);
    float3 nm = make_float3(mn[0], mn[1], mn[2]);
    if (!normalize_rn(&nm)) continue;
    const float3 q = make_float3(fmul(dm, ray_coord(ix, a.mcx, a.mfx)), fmul(dm, ray_coord(iy, a.mcy, a.mfy)), dm);
    if (dot_rn(nm, q) > 0.f) nm = make_float3(-nm.x, -nm.y, -nm.z);
    const float3 e = sub_rn(pm, q);
    if (!(dot_rn(e, e) <= a.max_distance_squared)) continue;
    if (!(dot_rn(nl, nm) >= a.cos_max_angle)) continue;
    const float r = dot_rn(nm, e);
    const float3 c = cross_rn(pm, nm);
    const double J[6] = {c.x, c.y, c.z, nm.x, nm.y, nm.z};
    int k = 0;
#pragma unroll
    for (int row = 0; row < 6; ++row) {
#pragma unroll
      for (int col = row; col < 6; ++col) acc[k++] += J[row] * J[col];
    }
    const double rd = r;
#pragma unroll
    for (int row = 0; row < 6; ++row) acc[21 + row] += J[row] * rd;
    acc[kTermR2] += rd * rd;
    acc[kTermInliers] += 1.0;
  }
  __shared__ double warp_sums[kLinearizeWarps][kTerms];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kTerms; ++k) {
    double v = acc[k];
#pragma unroll
    for (int offset = 16; offset > 0; offset >>= 1) v += __shfl_down_sync(0xffffffffu, v, offset);
    if (lane == 0) warp_sums[warp][k] = v;
  }
  __syncthreads();
  if (threadIdx.x < kTerms) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < kLinearizeWarps; ++w) v += warp_sums[w][threadIdx.x];
    a.partials[static_cast<size_t>(blockIdx.x) * kTerms + threadIdx.x] = v;
  }
}

// exp(xi) . T for xi = (omega, v) and T = state pose, in fp64 (Rodrigues for the rotation, the left Jacobian for the
// translation), rounded to fp32 once.
__device__ void apply_increment(TrackState* s, const double xi[6]) {
  const double wx = xi[0], wy = xi[1], wz = xi[2];
  const double theta2 = wx * wx + wy * wy + wz * wz, theta = sqrt(theta2);
  double A, B, Cc;   // sin t / t, (1 - cos t) / t^2, (t - sin t) / t^3
  if (theta < 1e-4) {
    A = 1.0 - theta2 / 6.0;
    B = 0.5 - theta2 / 24.0;
    Cc = 1.0 / 6.0 - theta2 / 120.0;
  } else {
    const double sn = sin(theta), cs = cos(theta);
    A = sn / theta;
    B = (1.0 - cs) / theta2;
    Cc = (theta - sn) / (theta2 * theta);
  }
  const double K[3][3] = {{0.0, -wz, wy}, {wz, 0.0, -wx}, {-wy, wx, 0.0}};
  double K2[3][3], R[3][3], V[3][3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) K2[i][j] = K[i][0] * K[0][j] + K[i][1] * K[1][j] + K[i][2] * K[2][j];
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double I = i == j ? 1.0 : 0.0;
      R[i][j] = I + A * K[i][j] + B * K2[i][j];
      V[i][j] = I + B * K[i][j] + Cc * K2[i][j];
    }
  }
  double t[3], P[12];
#pragma unroll
  for (int i = 0; i < 3; ++i) t[i] = V[i][0] * xi[3] + V[i][1] * xi[4] + V[i][2] * xi[5];
#pragma unroll
  for (int k = 0; k < 12; ++k) P[k] = s->pose[k];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double v = R[i][0] * P[j] + R[i][1] * P[4 + j] + R[i][2] * P[8 + j];
      if (j == 3) v += t[i];
      s->pose[4 * i + j] = static_cast<float>(v);
    }
  }
}

__global__ void __launch_bounds__(kSolveBlock) k_track_solve(SolveArgs a) {
  TrackState* s = a.state;
  if (s->lost || s->done_level == a.level) return;
  // Fixed-order sum of the partial rows: thread (chunk, term) adds the rows of its chunk in row order, then one
  // thread per term adds the chunk sums in chunk order.
  __shared__ double chunk_sum[kSolveChunks][kTerms];
  __shared__ double sum[kTerms];
  if (threadIdx.x < kSolveChunks * kTerms) {
    const int term = threadIdx.x % kTerms, chunk = threadIdx.x / kTerms;
    const int per_chunk = (a.blocks + kSolveChunks - 1) / kSolveChunks;
    const int b1 = min(a.blocks, (chunk + 1) * per_chunk);
    double v = 0.0;
    for (int b = chunk * per_chunk; b < b1; ++b) v += a.partials[static_cast<size_t>(b) * kTerms + term];
    chunk_sum[chunk][term] = v;
  }
  __syncthreads();
  if (threadIdx.x < kTerms) {
    double v = 0.0;
#pragma unroll
    for (int c = 0; c < kSolveChunks; ++c) v += chunk_sum[c][threadIdx.x];
    sum[threadIdx.x] = v;
    s->system[threadIdx.x] = v;
  }
  __syncthreads();
  if (threadIdx.x != 0 || !a.solve) return;
  const double inliers = sum[kTermInliers], valid = sum[kTermValid];
  if (a.level == 0) {
    s->inliers = static_cast<u32>(inliers);
    s->valid = static_cast<u32>(valid);
    s->rms = inliers > 0.0 ? static_cast<float>(sqrt(sum[kTermR2] / inliers)) : 0.f;
  }
  if (inliers < static_cast<double>(a.min_inlier_fraction) * valid) { s->lost = 1; return; }
  double H[6][6], L[6][6], g[6];
  int k = 0;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
#pragma unroll
    for (int j = i; j < 6; ++j) { H[i][j] = sum[k]; H[j][i] = sum[k]; ++k; }
    g[i] = sum[21 + i];
  }
  // Cholesky H = L L^T
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    double d = H[j][j];
#pragma unroll
    for (int m = 0; m < j; ++m) d -= L[j][m] * L[j][m];
    if (!(d > 0.0)) { s->lost = 1; return; }
    L[j][j] = sqrt(d);
#pragma unroll
    for (int i = j + 1; i < 6; ++i) {
      double v = H[i][j];
#pragma unroll
      for (int m = 0; m < j; ++m) v -= L[i][m] * L[j][m];
      L[i][j] = v / L[j][j];
    }
  }
  // H xi = -g: forward then back substitution
  double y[6], xi[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    double v = -g[i];
#pragma unroll
    for (int m = 0; m < i; ++m) v -= L[i][m] * y[m];
    y[i] = v / L[i][i];
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    double v = y[i];
#pragma unroll
    for (int m = i + 1; m < 6; ++m) v -= L[m][i] * xi[m];
    xi[i] = v / L[i][i];
  }
  bool finite = true;
#pragma unroll
  for (int i = 0; i < 6; ++i) finite = finite && isfinite(xi[i]);
  if (!finite) { s->lost = 1; return; }
  apply_increment(s, xi);
  s->iterations += 1;
  const double w2 = xi[0] * xi[0] + xi[1] * xi[1] + xi[2] * xi[2], v2 = xi[3] * xi[3] + xi[4] * xi[4] + xi[5] * xi[5];
  if (sqrt(w2) < a.convergence_rotation && sqrt(v2) < a.convergence_translation) s->done_level = a.level;
}

bool Finite(float v) { return std::isfinite(v); }

// Size and intrinsics of Camera.scaled(level) of the handle's camera (libvis Camera::Scaled(1 / 2^level)).
struct LevelCamera { int width, height; float fx, fy, cx, cy; };
LevelCamera ScaledCamera(const sm_reconstruction* r, int level) {
  const float factor = 1.0f / static_cast<float>(1 << level);
  LevelCamera c;
  c.width = static_cast<int>(static_cast<double>(factor) * r->d.width + 0.5);
  c.height = static_cast<int>(static_cast<double>(factor) * r->d.height + 0.5);
  c.fx = r->fx * factor; c.fy = r->fy * factor; c.cx = r->cx * factor; c.cy = r->cy * factor;
  return c;
}
bool LevelUsable(const sm_reconstruction* r, int level) {
  if (level < 0 || level >= kMaxLevels) return false;
  const LevelCamera c = ScaledCamera(r, level);
  return c.width >= 3 && c.height >= 3;
}

// Checks of the sm_track_params fields that both calls use.
const char* CheckTrackParams(const sm_track_params& tp) {
  if (!(Finite(tp.max_point_distance) && tp.max_point_distance > 0.f)) return "max_point_distance must be finite and > 0";
  if (!(Finite(tp.max_normal_angle_deg) && tp.max_normal_angle_deg >= 0.f && tp.max_normal_angle_deg <= 180.f))
    return "max_normal_angle_deg must be in [0, 180]";
  if (!(Finite(tp.min_inlier_fraction) && tp.min_inlier_fraction >= 0.f && tp.min_inlier_fraction <= 1.f))
    return "min_inlier_fraction must be in [0, 1]";
  if (!(Finite(tp.convergence_rotation) && tp.convergence_rotation >= 0.f && Finite(tp.convergence_translation) &&
        tp.convergence_translation >= 0.f))
    return "the convergence thresholds must be finite and >= 0";
  return nullptr;
}

// Replaces the 3x3 part of a 3x4 pose by its nearest rotation (polar decomposition, Newton iteration
// R <- (R + R^-T) / 2 in fp64). Poses that went through fp32 are a few ulp off SO(3); the inverse below is a
// transpose and the Gauss-Newton update only multiplies from the left, so without this projection that scale and
// shear would be carried into every later pose of a chain of calls and grow frame by frame. False for a
// non-finite or non-positive determinant (a reflection or a singular matrix).
bool ProjectToRigid(double* T) {
  for (int it = 0; it < 8; ++it) {
    const double a = T[0], b = T[1], c = T[2], d = T[4], e = T[5], f = T[6], g = T[8], h = T[9], i = T[10];
    const double C00 = e * i - f * h, C01 = f * g - d * i, C02 = d * h - e * g;   // cofactors: R^-T = C / det
    const double C10 = c * h - b * i, C11 = a * i - c * g, C12 = b * g - a * h;
    const double C20 = b * f - c * e, C21 = c * d - a * f, C22 = a * e - b * d;
    const double det = a * C00 + b * C01 + c * C02;
    if (!(det > 0.0) || !std::isfinite(det)) return false;
    const double s = 0.5 / det;
    T[0] = 0.5 * a + s * C00; T[1] = 0.5 * b + s * C01; T[2] = 0.5 * c + s * C02;
    T[4] = 0.5 * d + s * C10; T[5] = 0.5 * e + s * C11; T[6] = 0.5 * f + s * C12;
    T[8] = 0.5 * g + s * C20; T[9] = 0.5 * h + s * C21; T[10] = 0.5 * i + s * C22;
  }
  return true;
}

void InvertRigid(const double* m, double* out) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) out[4 * i + j] = m[4 * j + i];
    out[4 * i + 3] = -(m[i] * m[3] + m[4 + i] * m[7] + m[8 + i] * m[11]);
  }
}
void ComposeRigid(const double* a, const double* b, double* out) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 4; ++j) {
      double v = a[4 * i] * b[j] + a[4 * i + 1] * b[4 + j] + a[4 * i + 2] * b[8 + j];
      if (j == 3) v += a[4 * i + 3];
      out[4 * i + j] = v;
    }
  }
}

// All scratch, the device state last: a non-null track_state means every buffer exists. A failed allocation frees
// what was allocated, so the next call starts over.
int AllocateTrackBuffers(sm_reconstruction* r) {
  const int status = ResidentBlocks(k_track_linearize, kLinearizeBlock, r->sm_count, &r->track_blocks);
  if (status != SM_OK) return status;
  SM_CUDA(cudaMalloc(&r->track_partials, sizeof(double) * kTerms * r->track_blocks));
  SM_CUDA(cudaMallocHost(&r->track_host_state, sizeof(TrackState)));
  const size_t W = static_cast<size_t>(r->d.width), H = static_cast<size_t>(r->d.height);
  for (int l = 0; l < kMaxLevels; ++l) {
    if (!LevelUsable(r, l)) break;
    const LevelCamera c = ScaledCamera(r, l);
    SM_CUDA(cudaMallocPitch(&r->track_level[l], &r->track_level_pitch[l], sizeof(u16) * c.width, c.height));
  }
  SM_CUDA(cudaMallocPitch(&r->track_model_depth, &r->track_model_depth_pitch, sizeof(float) * W, H));
  SM_CUDA(cudaMallocPitch(&r->track_model_normal, &r->track_model_normal_pitch, 3 * sizeof(float) * W, H));
  for (int k = 0; k < 2; ++k) {
    SM_CUDA(cudaMallocPitch(&r->track_view_depth[k], &r->track_view_depth_pitch[k], sizeof(float) * W, H));
    SM_CUDA(cudaMallocPitch(&r->track_view_normal[k], &r->track_view_normal_pitch[k], 3 * sizeof(float) * W, H));
  }
  SM_CUDA(cudaMalloc(&r->track_state, sizeof(TrackState)));
  return SM_OK;
}

int EnsureTrackBuffers(sm_reconstruction* r) {
  if (r->track_state != nullptr) return SM_OK;
  const int status = AllocateTrackBuffers(r);
  if (status != SM_OK) FreeTrackBuffers(r);
  return status;
}

LinearizeArgs MakeLinearizeArgs(const sm_reconstruction* r, const sm_track_params& tp, float depth_scaling, int level,
                                const u16* live, size_t live_pitch, const float* model_depth, size_t model_depth_pitch,
                                const float* model_normal, size_t model_normal_pitch) {
  const LevelCamera c = ScaledCamera(r, level);
  LinearizeArgs a;
  a.level = level;
  a.width = c.width; a.height = c.height;
  a.fx = c.fx; a.fy = c.fy; a.cx = c.cx; a.cy = c.cy;
  a.inv_depth_scaling = 1.0f / depth_scaling;
  a.live = live; a.live_pitch = live_pitch;
  a.model_width = r->d.width; a.model_height = r->d.height;
  a.mfx = r->fx; a.mfy = r->fy; a.mcx = r->cx; a.mcy = r->cy;
  a.model_depth = model_depth; a.model_depth_pitch = model_depth_pitch;
  a.model_normal = model_normal; a.model_normal_pitch = model_normal_pitch;
  a.max_distance_squared = tp.max_point_distance * tp.max_point_distance;
  a.cos_max_angle = static_cast<float>(std::cos(static_cast<double>(tp.max_normal_angle_deg) * M_PI / 180.0));
  a.state = r->track_state;
  a.partials = r->track_partials;
  return a;
}

SolveArgs MakeSolveArgs(const sm_reconstruction* r, const sm_track_params& tp, int level, bool solve) {
  SolveArgs s;
  s.level = level;
  s.solve = solve ? 1 : 0;
  s.blocks = r->track_blocks;
  s.partials = r->track_partials;
  s.state = r->track_state;
  s.min_inlier_fraction = tp.min_inlier_fraction;
  s.convergence_rotation = tp.convergence_rotation;
  s.convergence_translation = tp.convergence_translation;
  return s;
}

void LaunchIteration(sm_reconstruction* r, cudaStream_t stream, const LinearizeArgs& la, const SolveArgs& sa) {
  { LaunchScope scope(stream, KID_TRACK_LINEARIZE); LaunchKernel(k_track_linearize, dim3(r->track_blocks), dim3(kLinearizeBlock), 0, stream, la); }
  { LaunchScope scope(stream, KID_TRACK_SOLVE); LaunchKernel(k_track_solve, dim3(1), dim3(kSolveBlock), 0, stream, sa); }
}

// Uploads a fresh state with `pose` as model_T_live.
int UploadState(sm_reconstruction* r, cudaStream_t stream, const float* pose) {
  TrackState* h = r->track_host_state;
  memset(h, 0, sizeof(TrackState));
  for (int k = 0; k < 12; ++k) h->pose[k] = pose[k];
  h->done_level = -1;
  SM_CUDA(cudaMemcpyAsync(r->track_state, h, sizeof(TrackState), cudaMemcpyHostToDevice, stream));
  return SM_OK;
}

int DownloadState(sm_reconstruction* r, cudaStream_t stream) {
  SM_CUDA(cudaMemcpyAsync(r->track_host_state, r->track_state, sizeof(TrackState), cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaStreamSynchronize(stream));
  return SM_OK;
}

}  // namespace

int TrackFrame(sm_reconstruction* r, cudaStream_t stream, const sm_track_params& tp, const sm_preprocess_params& pp,
               const u16* depth, size_t depth_pitch, const float* guess, float* pose_out, sm_track_result* result) {
  auto bad = [](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (std::string("sm_track_frame: ") + why).c_str()); };
  if (depth_pitch < sizeof(u16) * static_cast<size_t>(r->d.width)) return bad("depth_pitch is below the row size");
  if (tp.levels < 1 || tp.levels > kMaxLevels) return bad("levels must be in [1, 4]");
  for (int l = 0; l < kMaxLevels; ++l) if (tp.iterations[l] < 0) return bad("iterations must be >= 0");
  if (!LevelUsable(r, tp.levels - 1)) return bad("the coarsest level is smaller than 3 x 3 pixels");
  if (const char* why = CheckTrackParams(tp)) return bad(why);
  if (tp.model_source != SM_TRACK_CLOUD && tp.model_source != SM_TRACK_PREVIOUS_FRAME) return bad("unknown model_source");
  if (tp.model_source == SM_TRACK_PREVIOUS_FRAME && !r->track_has_previous)
    return bad("SM_TRACK_PREVIOUS_FRAME needs an earlier sm_track_frame call on this handle");
  for (int k = 0; k < 12; ++k) if (!Finite(guess[k])) return bad("global_T_guess must be finite");
  if (!(Finite(pp.depth_scaling) && pp.depth_scaling > 0.f)) return bad("depth_scaling must be finite and > 0");
  if (!Finite(pp.max_depth) || !Finite(pp.depth_valid_region_radius) || !Finite(pp.bilateral_filter_sigma_xy) ||
      !Finite(pp.bilateral_filter_radius_factor) || !Finite(pp.bilateral_filter_sigma_depth_factor))
    return bad("the pre-processing parameters must be finite");
  if (BilateralRadius(pp) < 0) return bad("the bilateral filter radius must be >= 0");
  // poses first: a guess whose inverse or starting model_T_live is not finite in fp32 is refused before any launch
  double guess_d[12], model_T_global[12], global_T_model[12], init[12];
  for (int k = 0; k < 12; ++k) {
    guess_d[k] = guess[k];
    global_T_model[k] = tp.model_source == SM_TRACK_CLOUD ? guess_d[k] : r->track_previous_pose[k];
  }
  if (!ProjectToRigid(guess_d)) return bad("the rotation of global_T_guess must have a positive determinant");
  if (tp.model_source == SM_TRACK_CLOUD) {
    for (int k = 0; k < 12; ++k) global_T_model[k] = guess_d[k];
  } else if (!ProjectToRigid(global_T_model)) {
    return bad("the pose of the previous frame is not a rigid transform");
  }
  InvertRigid(global_T_model, model_T_global);
  ComposeRigid(model_T_global, guess_d, init);
  float view_f[12], init_f[12];
  for (int k = 0; k < 12; ++k) {
    view_f[k] = static_cast<float>(model_T_global[k]);
    init_f[k] = static_cast<float>(init[k]);
    if (!Finite(view_f[k]) || !Finite(init_f[k])) return bad("global_T_guess is too large for an fp32 pose");
  }
  int status = EnsureTrackBuffers(r);
  if (status != SM_OK) return status;
  r->last_stream = stream;
  const int W = r->d.width, H = r->d.height;

  // 1. live pyramid
  status = StageBilateral(stream, pp.bilateral_filter_sigma_xy, pp.bilateral_filter_sigma_depth_factor, 0,
                          pp.bilateral_filter_radius_factor, static_cast<u16>(pp.depth_scaling * pp.max_depth),
                          pp.depth_valid_region_radius, W, H, depth, depth_pitch, r->track_level[0], r->track_level_pitch[0]);
  if (status != SM_OK) return status;
  for (int l = 1; l < tp.levels; ++l) {
    const LevelCamera c = ScaledCamera(r, l);
    status = StageDownscaleMedian(stream, 0, W, H, r->track_level[0], r->track_level_pitch[0], c.width, c.height,
                                  r->track_level[l], r->track_level_pitch[l]);
    if (status != SM_OK) return status;
  }

  // 2. model view and the initial model_T_live
  const float* model_depth = r->track_model_depth;
  const float* model_normal = r->track_model_normal;
  size_t model_depth_pitch = r->track_model_depth_pitch, model_normal_pitch = r->track_model_normal_pitch;
  if (tp.model_source == SM_TRACK_CLOUD) {
    sm_render_params rp;
    rp.width = W; rp.height = H; rp.fx = r->fx; rp.fy = r->fy; rp.cx = r->cx; rp.cy = r->cy;
    rp.near_depth = kModelNear; rp.far_depth = kModelFar;
    status = RenderSurfels(r, stream, rp, view_f, r->track_model_depth, r->track_model_depth_pitch, nullptr, 0,
                           r->track_model_normal, r->track_model_normal_pitch, nullptr, 0);
    if (status != SM_OK) return status;
  } else {
    model_depth = r->track_view_depth[r->track_previous];
    model_normal = r->track_view_normal[r->track_previous];
    model_depth_pitch = r->track_view_depth_pitch[r->track_previous];
    model_normal_pitch = r->track_view_normal_pitch[r->track_previous];
  }
  status = UploadState(r, stream, init_f);
  if (status != SM_OK) return status;

  // 3. this frame's level-0 view, the model of the next SM_TRACK_PREVIOUS_FRAME call
  const int view = r->track_has_previous ? 1 - r->track_previous : 0;
  {
    LiveViewArgs v;
    const LevelCamera c = ScaledCamera(r, 0);
    v.width = c.width; v.height = c.height;
    v.fx = c.fx; v.fy = c.fy; v.cx = c.cx; v.cy = c.cy;
    v.inv_depth_scaling = 1.0f / pp.depth_scaling;
    v.live = r->track_level[0]; v.live_pitch = r->track_level_pitch[0];
    v.depth = r->track_view_depth[view]; v.depth_pitch = r->track_view_depth_pitch[view];
    v.normal = r->track_view_normal[view]; v.normal_pitch = r->track_view_normal_pitch[view];
    LaunchScope scope(stream, KID_TRACK_LIVE_VIEW);
    LaunchKernel(k_track_live_view, dim3((W + 255) / 256, H), dim3(256), 0, stream, v);
  }

  // 4. Gauss-Newton, coarse to fine
  for (int l = tp.levels - 1; l >= 0; --l) {
    const LinearizeArgs la = MakeLinearizeArgs(r, tp, pp.depth_scaling, l, r->track_level[l], r->track_level_pitch[l],
                                               model_depth, model_depth_pitch, model_normal, model_normal_pitch);
    const SolveArgs sa = MakeSolveArgs(r, tp, l, true);
    for (int it = 0; it < tp.iterations[l]; ++it) LaunchIteration(r, stream, la, sa);
  }
  status = CheckLaunch("track frame");
  if (status != SM_OK) return status;

  // 5. one synchronisation, then the result
  status = DownloadState(r, stream);
  if (status != SM_OK) return status;
  const TrackState& h = *r->track_host_state;
  double out[12];
  if (h.lost) {
    for (int k = 0; k < 12; ++k) out[k] = guess[k];   // the caller's guess, unchanged
  } else {
    double refined[12];
    for (int k = 0; k < 12; ++k) refined[k] = h.pose[k];
    ComposeRigid(global_T_model, refined, out);
    ProjectToRigid(out);   // a few ulp off SO(3) at most; det > 0 as the product of two such matrices
  }
  for (int k = 0; k < 12; ++k) {
    pose_out[k] = static_cast<float>(out[k]);
    r->track_previous_pose[k] = pose_out[k];
  }
  r->track_previous = view;
  r->track_has_previous = true;
  if (result) {
    result->tracked = h.lost ? 0 : 1;
    result->iterations = h.iterations;
    result->inliers = h.inliers;
    result->valid_pixels = h.valid;
    result->rms_residual = h.rms;
  }
  return SM_OK;
}

int TrackLinearize(sm_reconstruction* r, cudaStream_t stream, const sm_track_params& tp, int level, float depth_scaling,
                   const u16* live, size_t live_pitch, const float* model_depth, size_t model_depth_pitch,
                   const float* model_normal, size_t model_normal_pitch, const float* model_T_live, double* out_system,
                   uint32_t* out_inliers) {
  auto bad = [](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (std::string("sm_track_linearize: ") + why).c_str()); };
  if (!LevelUsable(r, level)) return bad("level must be in [0, 3] with an image of at least 3 x 3 pixels");
  if (!(Finite(depth_scaling) && depth_scaling > 0.f)) return bad("depth_scaling must be finite and > 0");
  const LevelCamera c = ScaledCamera(r, level);
  const size_t W = static_cast<size_t>(r->d.width);
  if (live_pitch < sizeof(u16) * c.width || model_depth_pitch < sizeof(float) * W ||
      model_normal_pitch < 3 * sizeof(float) * W)
    return bad("a pitch is below the row size");
  if (const char* why = CheckTrackParams(tp)) return bad(why);
  for (int k = 0; k < 12; ++k) if (!Finite(model_T_live[k])) return bad("model_T_live must be finite");
  int status = EnsureTrackBuffers(r);
  if (status != SM_OK) return status;
  r->last_stream = stream;
  status = UploadState(r, stream, model_T_live);
  if (status != SM_OK) return status;
  const LinearizeArgs la = MakeLinearizeArgs(r, tp, depth_scaling, level, live, live_pitch, model_depth,
                                             model_depth_pitch, model_normal, model_normal_pitch);
  LaunchIteration(r, stream, la, MakeSolveArgs(r, tp, level, false));
  status = CheckLaunch("track linearize");
  if (status != SM_OK) return status;
  status = DownloadState(r, stream);
  if (status != SM_OK) return status;
  for (int k = 0; k < kSystemTerms; ++k) out_system[k] = r->track_host_state->system[k];
  *out_inliers = static_cast<uint32_t>(r->track_host_state->system[kTermInliers]);
  return SM_OK;
}

void FreeTrackBuffers(sm_reconstruction* r) {
  for (int l = 0; l < kMaxLevels; ++l) { cudaFree(r->track_level[l]); r->track_level[l] = nullptr; }
  cudaFree(r->track_model_depth); cudaFree(r->track_model_normal);
  r->track_model_depth = nullptr; r->track_model_normal = nullptr;
  for (int k = 0; k < 2; ++k) {
    cudaFree(r->track_view_depth[k]); cudaFree(r->track_view_normal[k]);
    r->track_view_depth[k] = nullptr; r->track_view_normal[k] = nullptr;
  }
  cudaFree(r->track_partials); cudaFree(r->track_state);
  if (r->track_host_state) cudaFreeHost(r->track_host_state);
  r->track_partials = nullptr;
  r->track_state = nullptr;
  r->track_host_state = nullptr;
}

}  // namespace smb
