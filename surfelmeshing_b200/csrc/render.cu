// render.cu — sm_render_surfels (DESIGN.md section 5.5): the surfel cloud drawn as oriented disks into any pinhole
// camera, with a z-buffer of 64-bit keys {bits of the depth, slot} whose minimum wins, so the images do not depend
// on the order in which the GPU does the work. The semantics, step by step, are in include/surfel_b200.h.
//
// Three launches on the caller's stream, no host synchronisation:
//   k_render_splat    grid-stride sweep over the slots [0, surfels_size()): one 16-byte regularisation record and
//                     rows 7-10 per slot; transforms the disk into the camera and bounds its pixels by a screen
//                     rectangle. A rectangle of at most kSmallSplatPixels pixels is tested by the slot's own
//                     thread (one 64-bit atomicMin per covered pixel); a larger one goes to the large-splat list
//                     (warp-aggregated append), so no thread walks an unbounded rectangle;
//   k_render_large    one block per listed slot strides over its rectangle (the list length stays on the device);
//   k_render_resolve  one thread per pixel decodes the winning key, gathers the winner's colour and normal, writes
//                     the outputs and puts the key back to "empty" for the next call (the raster is cleared once,
//                     when it is allocated); it also zeroes the list length.

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

#define SM_S(row, i) d.surfels[static_cast<size_t>(row) * d.stride + (i)]
#define SM_SU(row, i) reinterpret_cast<const u32*>(d.surfels)[static_cast<size_t>(row) * d.stride + (i)]

constexpr int kSplatBlock = 256;
constexpr int kLargeBlock = 256;
constexpr int kResolveBlock = 256;
// Rectangles up to this many pixels are tested by the sweep's own thread (DESIGN.md section 5.5).
constexpr long long kSmallSplatPixels = 64;
constexpr unsigned long long kEmptyKey = ~0ull;

struct RenderArgs {
  int count_slot;
  int width, height;
  float fx, fy, cx, cy;
  float near_depth, far_depth;
  Mat3x4 view_T_global;
  unsigned long long* keys;   // [height][width]
  u32* large_list;            // slots whose rectangle has more than kSmallSplatPixels pixels
  u32* large_count;
  float* depth; size_t depth_pitch;
  u8* color; size_t color_pitch;
  float* normal; size_t normal_pitch;
  u32* index; size_t index_pitch;
};

struct Splat {
  float3 c, m;            // camera-space centre and normal
  float num;              // dot3(m, c)
  float radius_squared;
  int x0, y0, x1, y1;     // pixel rectangle (inclusive), inside the image
};

// Ray coordinate of pixel p: ((p + 0.5) - c) / f with IEEE division.
__device__ __forceinline__ float ray_coord(int p, float c, float f) { return __fdiv_rn(fsub(fadd(i2f(p), 0.5f), c), f); }

// Pixels [*p0, *p1] of one image axis whose ray coordinate can lie in [lo / z, hi / z] for z in [z_lo, z_hi]
// (z_lo > 0), plus one pixel on each side for the rounding of the ray coordinate and of this bound, clamped to
// [0, size - 1]. False if none is inside the image. A NaN bound clamps to the image edge.
__device__ __forceinline__ bool axis_range(float lo, float hi, float z_lo, float z_hi, float f, float c, int size, int* p0,
                                           int* p1) {
  const float d_min = lo >= 0.f ? lo / z_hi : lo / z_lo;
  const float d_max = hi >= 0.f ? hi / z_lo : hi / z_hi;
  float q0 = f * d_min + (c - 0.5f), q1 = f * d_max + (c - 0.5f);   // pixel whose centre ray is d: f d + c - 0.5
  if (f < 0.f) { const float q = q0; q0 = q1; q1 = q; }
  q0 = floorf(q0) - 1.f;
  q1 = ceilf(q1) + 1.f;
  q0 = q0 > 0.f ? q0 : 0.f;
  const float last = static_cast<float>(size - 1);
  q1 = q1 < last ? q1 : last;
  if (!(q0 <= q1)) return false;
  *p0 = static_cast<int>(q0);
  *p1 = static_cast<int>(q1);
  return true;
}

// Steps 1-2 of the header and the screen rectangle. A pixel the coverage test accepts has its hit point
// h = t (dx, dy, 1) within `reach` of c: the disk radius plus a bound on the rounding of the fp32 test (a few ulp
// of |c| + r per component; 1e-5 relative is ~100 times that). So dx = h.x / h.z over that ball bounds the
// pixel. A ball that reaches the camera plane bounds nothing: the whole image.
__device__ __forceinline__ bool load_splat(const DeviceState& d, const RenderArgs& a, u32 i, Splat* s) {
  const float radius_squared = SM_S(SM_ROW_RADIUS_SQUARED, i);
  if (!(radius_squared > 0.f)) return false;
  const float4 p = d.smooth[i];
  const float3 c = transform_point(a.view_T_global, p.x, p.y, p.z);
  if (!(a.near_depth <= c.z && c.z <= a.far_depth)) return false;
  s->c = c;
  s->m = rotate_vec(a.view_T_global, SM_S(SM_ROW_NORMAL_X, i), SM_S(SM_ROW_NORMAL_Y, i), SM_S(SM_ROW_NORMAL_Z, i));
  s->num = dot3(s->m.x, s->m.y, s->m.z, c.x, c.y, c.z);
  s->radius_squared = radius_squared;
  const float reach = sqrtf(radius_squared) * 1.0001f + (fabsf(c.x) + fabsf(c.y) + fabsf(c.z)) * 1e-5f;
  const float z_lo = c.z - reach;
  if (!(z_lo > 0.f)) {
    s->x0 = 0; s->y0 = 0; s->x1 = a.width - 1; s->y1 = a.height - 1;
    return true;
  }
  const float z_hi = c.z + reach;
  return axis_range(c.x - reach, c.x + reach, z_lo, z_hi, a.fx, a.cx, a.width, &s->x0, &s->x1) &&
         axis_range(c.y - reach, c.y + reach, z_lo, z_hi, a.fy, a.cy, a.height, &s->y0, &s->y1);
}

// Step 3-4 for one pixel.
__device__ __forceinline__ void splat_pixel(const RenderArgs& a, const Splat& s, u32 i, int px, int py, float dy) {
  const float dx = ray_coord(px, a.cx, a.fx);
  const float den = dot3(s.m.x, s.m.y, s.m.z, dx, dy, 1.0f);
  if (den == 0.f) return;
  const float t = __fdiv_rn(s.num, den);
  if (!(t > 0.f) || !isfinite(t)) return;
  const float ex = fsub(fmul(t, dx), s.c.x), ey = fsub(fmul(t, dy), s.c.y), ez = fsub(t, s.c.z);
  if (!(squared_norm(ex, ey, ez) <= s.radius_squared)) return;
  const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(t)) << 32) | i;
  atomicMin(a.keys + static_cast<size_t>(py) * a.width + px, key);
}

__global__ void __launch_bounds__(kSplatBlock) k_render_splat(DeviceState d, RenderArgs a) {
  const u32 n = d.counters->surfel_count[a.count_slot];
  const int lane = threadIdx.x & 31;
  for (u32 base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
    const u32 i = base + threadIdx.x;
    Splat s;
    const bool drawn = i < n && load_splat(d, a, i, &s);
    const bool large =
        drawn && static_cast<long long>(s.x1 - s.x0 + 1) * (s.y1 - s.y0 + 1) > kSmallSplatPixels;
    const unsigned mask = __ballot_sync(0xffffffffu, large);
    if (mask) {
      u32 warp_base = 0;
      if (lane == 0) warp_base = atomicAdd(a.large_count, static_cast<u32>(__popc(mask)));
      warp_base = __shfl_sync(0xffffffffu, warp_base, 0);
      if (large) a.large_list[warp_base + __popc(mask & ((1u << lane) - 1u))] = i;   // < capacity: one entry per slot
    }
    if (!drawn || large) continue;
    for (int py = s.y0; py <= s.y1; ++py) {
      const float dy = ray_coord(py, a.cy, a.fy);
      for (int px = s.x0; px <= s.x1; ++px) splat_pixel(a, s, i, px, py, dy);
    }
  }
}

// One warp per listed slot. A rectangle at least 32 pixels wide is walked row by row with the lanes over the
// columns; a narrower one packs 32 / width rows into one pass of the warp.
__global__ void __launch_bounds__(kLargeBlock) k_render_large(DeviceState d, RenderArgs a) {
  const u32 count = *a.large_count;
  const int lane = threadIdx.x & 31;
  const u32 warps = gridDim.x * (kLargeBlock / 32);
  for (u32 k = blockIdx.x * (kLargeBlock / 32) + (threadIdx.x >> 5); k < count; k += warps) {
    const u32 i = a.large_list[k];
    Splat s;
    if (!load_splat(d, a, i, &s)) continue;   // not reached: the sweep listed the slot with the same result
    const int w = s.x1 - s.x0 + 1;
    const int rows = w >= 32 ? 1 : 32 / w;
    const int row = lane / (w >= 32 ? 32 : w), column = w >= 32 ? lane : lane % w;
    if (row >= rows) continue;
    for (int py = s.y0 + row; py <= s.y1; py += rows) {
      const float dy = ray_coord(py, a.cy, a.fy);
      for (int px = s.x0 + column; px <= s.x1; px += (w >= 32 ? 32 : w)) splat_pixel(a, s, i, px, py, dy);
    }
  }
}

__global__ void __launch_bounds__(kResolveBlock) k_render_resolve(DeviceState d, RenderArgs a) {
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *a.large_count = 0;   // k_render_large has finished
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= a.width) return;
  for (int py = blockIdx.y; py < a.height; py += gridDim.y) {
    unsigned long long* key_ptr = a.keys + static_cast<size_t>(py) * a.width + px;
    const unsigned long long key = *key_ptr;
    float depth = 0.f;
    u32 index = kInvalidIndex, rgb = 0;
    float3 m = make_float3(0.f, 0.f, 0.f);
    if (key != kEmptyKey) {
      *key_ptr = kEmptyKey;
      index = static_cast<u32>(key);
      depth = __uint_as_float(static_cast<u32>(key >> 32));
      if (a.color) rgb = SM_SU(SM_ROW_COLOR, index);
      if (a.normal)
        m = rotate_vec(a.view_T_global, SM_S(SM_ROW_NORMAL_X, index), SM_S(SM_ROW_NORMAL_Y, index),
                       SM_S(SM_ROW_NORMAL_Z, index));
    }
    if (a.depth) row_ptr(a.depth, a.depth_pitch, py)[px] = depth;
    if (a.index) row_ptr(a.index, a.index_pitch, py)[px] = index;
    if (a.color) {
      u8* o = row_ptr(a.color, a.color_pitch, py) + 3 * static_cast<size_t>(px);
      o[0] = rgb & 0xFFu; o[1] = (rgb >> 8) & 0xFFu; o[2] = (rgb >> 16) & 0xFFu;
    }
    if (a.normal) {
      float* o = row_ptr(a.normal, a.normal_pitch, py) + 3 * static_cast<size_t>(px);
      o[0] = m.x; o[1] = m.y; o[2] = m.z;
    }
  }
}

bool Finite(float v) { return std::isfinite(v); }

// The key raster grows to `pixels`; the list, its count and the grids are set up once.
int EnsureRenderBuffers(sm_reconstruction* r, cudaStream_t stream, size_t pixels) {
  if (r->render_large_list == nullptr) {
    SM_CUDA(cudaMalloc(&r->render_large_list, sizeof(u32) * r->d.stride));
    SM_CUDA(cudaMalloc(&r->render_large_count, sizeof(u32)));
    SM_CUDA(cudaMemsetAsync(r->render_large_count, 0, sizeof(u32), stream));
    int status = ResidentBlocks(k_render_splat, kSplatBlock, r->sm_count, &r->render_splat_blocks);
    if (status == SM_OK) status = ResidentBlocks(k_render_large, kLargeBlock, r->sm_count, &r->render_large_blocks);
    if (status != SM_OK) return status;
  }
  if (pixels > r->render_key_capacity) {
    cudaFree(r->render_keys);   // synchronises the device: an earlier render may still use it
    r->render_keys = nullptr;
    r->render_key_capacity = 0;
    SM_CUDA(cudaMalloc(&r->render_keys, sizeof(unsigned long long) * pixels));
    SM_CUDA(cudaMemsetAsync(r->render_keys, 0xFF, sizeof(unsigned long long) * pixels, stream));
    r->render_key_capacity = pixels;
  }
  return SM_OK;
}

}  // namespace

int RenderSurfels(sm_reconstruction* r, cudaStream_t stream, const sm_render_params& p, const float* view_T_global,
                  float* depth, size_t depth_pitch, uint8_t* color, size_t color_pitch, float* normal,
                  size_t normal_pitch, uint32_t* index, size_t index_pitch) {
  auto bad = [](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (std::string("sm_render_surfels: ") + why).c_str()); };
  if (p.width <= 0 || p.height <= 0) return bad("width and height must be > 0");
  if (!Finite(p.fx) || !Finite(p.fy) || p.fx == 0.f || p.fy == 0.f) return bad("fx and fy must be finite and non-zero");
  if (!Finite(p.cx) || !Finite(p.cy)) return bad("cx and cy must be finite");
  if (!(p.near_depth > 0.f) || !(p.far_depth > p.near_depth)) return bad("need 0 < near_depth < far_depth");
  for (int k = 0; k < 12; ++k) if (!Finite(view_T_global[k])) return bad("view_T_global must be finite");
  if (!depth && !color && !normal && !index) return bad("all outputs are NULL");
  const size_t w = static_cast<size_t>(p.width);
  if ((depth && depth_pitch < w * sizeof(float)) || (color && color_pitch < w * 3) ||
      (normal && normal_pitch < w * 3 * sizeof(float)) || (index && index_pitch < w * sizeof(u32)))
    return bad("a pitch is below the row size");
  const int status = EnsureRenderBuffers(r, stream, w * static_cast<size_t>(p.height));
  if (status != SM_OK) return status;
  RenderArgs a;
  a.count_slot = r->count_slot;
  a.width = p.width; a.height = p.height;
  a.fx = p.fx; a.fy = p.fy; a.cx = p.cx; a.cy = p.cy;
  a.near_depth = p.near_depth; a.far_depth = p.far_depth;
  a.view_T_global = MakeMat3x4(view_T_global);
  a.keys = r->render_keys;
  a.large_list = r->render_large_list;
  a.large_count = r->render_large_count;
  a.depth = depth; a.depth_pitch = depth_pitch;
  a.color = color; a.color_pitch = color_pitch;
  a.normal = normal; a.normal_pitch = normal_pitch;
  a.index = index; a.index_pitch = index_pitch;
  r->last_stream = stream;
  { LaunchScope scope(stream, KID_RENDER_SPLAT); LaunchKernel(k_render_splat, dim3(r->render_splat_blocks), dim3(kSplatBlock), 0, stream, r->d, a); }
  { LaunchScope scope(stream, KID_RENDER_LARGE); LaunchKernel(k_render_large, dim3(r->render_large_blocks), dim3(kLargeBlock), 0, stream, r->d, a); }
  const dim3 resolve_grid((p.width + kResolveBlock - 1) / kResolveBlock, p.height < 65535 ? p.height : 65535);
  { LaunchScope scope(stream, KID_RENDER_RESOLVE); LaunchKernel(k_render_resolve, resolve_grid, dim3(kResolveBlock), 0, stream, r->d, a); }
  return CheckLaunch("render surfels");
}

void FreeRenderBuffers(sm_reconstruction* r) {
  cudaFree(r->render_keys);
  cudaFree(r->render_large_list);
  cudaFree(r->render_large_count);
  r->render_keys = nullptr;
  r->render_large_list = nullptr;
  r->render_large_count = nullptr;
  r->render_key_capacity = 0;
}

}  // namespace smb
