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

// The scratch of sm_render_surfels and sm_render_mesh, created by the first render.
struct RenderScratch {
  // sm_render_surfels: the key raster (all keys "empty" between calls), the large-splat list (capacity slots) and
  // its count (zero between calls), resident grids
  unsigned long long* keys = nullptr; size_t key_capacity = 0;   // in pixels
  u32* large_list = nullptr;
  u32* large_count = nullptr;
  int splat_blocks = 0, large_blocks = 0;
  // sm_render_mesh, from the first mesh render: one bit per slot (the corners of the triangles drawn), the
  // large-triangle list (grown to the triangle count) and its count (zero between calls), resident grids
  u32* mesh_marks = nullptr;
  u32* mesh_large_list = nullptr; u32 mesh_large_capacity = 0;   // in triangles
  u32* mesh_large_count = nullptr;
  int mesh_mark_blocks = 0, mesh_tri_blocks = 0, mesh_large_blocks = 0;
  int mesh_splat_blocks = 0, mesh_splat_large_blocks = 0;
};

namespace {

#define SM_S(row, i) d.surfels[static_cast<size_t>(row) * d.stride + (i)]
#define SM_SU(row, i) reinterpret_cast<const u32*>(d.surfels)[static_cast<size_t>(row) * d.stride + (i)]

constexpr int kSplatBlock = 256;
constexpr int kLargeBlock = 256;
constexpr int kResolveBlock = 256;
// Rectangles up to this many pixels are tested by the sweep's own thread (DESIGN.md section 5.5).
constexpr long long kSmallSplatPixels = 64;
constexpr unsigned long long kEmptyKey = ~0ull;
// sm_render_mesh: the low word of a disk's key (T6), above every triangle index (< 2^31).
constexpr u32 kDiskTag = 0x80000000u;

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

// Step 3-4 for one pixel. The key's low word is the slot (sm_render_mesh: the slot with the disk tag).
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

// The body of k_render_large: one warp per listed slot. A rectangle at least 32 pixels wide is walked row by row
// with the lanes over the columns; a narrower one packs 32 / width rows into one pass of the warp.
template <bool kMesh>
__device__ __forceinline__ void splat_large(const DeviceState& d, const RenderArgs& a) {
  const u32 count = *a.large_count;
  const int lane = threadIdx.x & 31;
  const u32 warps = gridDim.x * (kLargeBlock / 32);
  for (u32 k = blockIdx.x * (kLargeBlock / 32) + (threadIdx.x >> 5); k < count; k += warps) {
    const u32 i = a.large_list[k];
    Splat s;
    if (!load_splat(d, a, i, &s)) continue;   // not reached: the sweep listed the slot with the same result
    const u32 key_low = kMesh ? (i | kDiskTag) : i;
    const int w = s.x1 - s.x0 + 1;
    const int rows = w >= 32 ? 1 : 32 / w;
    const int row = lane / (w >= 32 ? 32 : w), column = w >= 32 ? lane : lane % w;
    if (row >= rows) continue;
    for (int py = s.y0 + row; py <= s.y1; py += rows) {
      const float dy = ray_coord(py, a.cy, a.fy);
      for (int px = s.x0 + column; px <= s.x1; px += (w >= 32 ? 32 : w)) splat_pixel(a, s, key_low, px, py, dy);
    }
  }
}

__global__ void __launch_bounds__(kLargeBlock) k_render_large(DeviceState d, RenderArgs a) { splat_large<false>(d, a); }

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

// ---- sm_render_mesh (DESIGN.md section 5.9): rules T1-T7 of include/surfel_b200.h ----

constexpr int kMarkBlock = 256;
constexpr int kTriBlock = 256;
// Triangle rectangles up to this many pixels are tested by the sweep's own thread; larger ones go to the list.
constexpr long long kSmallTrianglePixels = 64;

struct MeshArgs {
  const u32* triangles;   // [triangle_count][3] slot indices
  u32 triangle_count;
  u32* marks;             // one bit per slot: a corner of a T1-valid triangle (SM_RENDER_UNMESHED_SURFELS only)
  u32* large_list;        // triangles whose rectangle has more than kSmallTrianglePixels pixels
  u32* large_count;
};

// T1 for triangle t: its three slots (in list order) if all are < n and present.
__device__ __forceinline__ bool triangle_corners(const DeviceState& d, const MeshArgs& m, u32 t, u32 n, u32 s[3]) {
  const u32* p = m.triangles + 3 * static_cast<size_t>(t);
  s[0] = p[0]; s[1] = p[1]; s[2] = p[2];
  for (int k = 0; k < 3; ++k)
    if (!(s[k] < n) || !(SM_S(SM_ROW_RADIUS_SQUARED, s[k]) > 0.f)) return false;
  return true;
}

// T3: the screen point of a camera-space corner. The one function every triangle uses, so a shared corner has the
// same (u, v) in each of them.
__device__ __forceinline__ float2 screen_point(const RenderArgs& a, float3 c) {
  return make_float2(fadd(fmul(a.fx, __fdiv_rn(c.x, c.z)), a.cx), fadd(fmul(a.fy, __fdiv_rn(c.y, c.z)), a.cy));
}

// Edge function of the edge from corner j to corner k (j the lower slot) at the point (x, y):
// (u_k - u_j) * (y - v_j) - (v_k - v_j) * (x - u_j), every operation rounded on its own.
__device__ __forceinline__ float edge_value(float uj, float vj, float uk, float vk, float x, float y) {
  return fsub(fmul(fsub(uk, uj), fsub(y, vj)), fmul(fsub(vk, vj), fsub(x, uj)));
}

struct Triangle {
  u32 s[3];          // slots, ascending
  float3 c[3];       // camera-space corners
  float u[3], v[3];  // screen points
  float area;        // D = edge_value(0 -> 1) at corner 2: twice the signed screen area
};

// T1-T3 for triangle t, its corners sorted by slot (so nothing below depends on the winding or the rotation).
__device__ __forceinline__ bool load_triangle(const DeviceState& d, const RenderArgs& a, const MeshArgs& m, u32 t,
                                              u32 n, Triangle* tr) {
  u32 s[3];
  if (!triangle_corners(d, m, t, n, s)) return false;
  u32 x;
  if (s[0] > s[1]) { x = s[0]; s[0] = s[1]; s[1] = x; }
  if (s[1] > s[2]) { x = s[1]; s[1] = s[2]; s[2] = x; }
  if (s[0] > s[1]) { x = s[0]; s[0] = s[1]; s[1] = x; }
  for (int k = 0; k < 3; ++k) {
    const float4 p = d.smooth[s[k]];
    const float3 c = transform_point(a.view_T_global, p.x, p.y, p.z);
    if (!(a.near_depth <= c.z && c.z <= a.far_depth)) return false;
    const float2 q = screen_point(a, c);
    tr->s[k] = s[k]; tr->c[k] = c; tr->u[k] = q.x; tr->v[k] = q.y;
  }
  tr->area = edge_value(tr->u[0], tr->v[0], tr->u[1], tr->v[1], tr->u[2], tr->v[2]);
  return tr->area != 0.f && isfinite(tr->area);
}

// T4: the three signed values at pixel (px, py), w[k] the one of the edge opposite corner k; true if covered.
__device__ __forceinline__ bool triangle_weights(const Triangle& tr, int px, int py, float w[3]) {
  const float x = fadd(i2f(px), 0.5f), y = fadd(i2f(py), 0.5f);
  w[0] = edge_value(tr.u[1], tr.v[1], tr.u[2], tr.v[2], x, y);
  w[1] = -edge_value(tr.u[0], tr.v[0], tr.u[2], tr.v[2], x, y);
  w[2] = edge_value(tr.u[0], tr.v[0], tr.u[1], tr.v[1], x, y);
  return tr.area > 0.f ? (w[0] >= 0.f && w[1] >= 0.f && w[2] >= 0.f) : (w[0] <= 0.f && w[1] <= 0.f && w[2] <= 0.f);
}

// T5: q[k] = (w[k] / D) / z_k and the perspective-correct depth 1 / ((q0 + q1) + q2).
__device__ __forceinline__ float triangle_depth(const Triangle& tr, const float w[3], float q[3]) {
  for (int k = 0; k < 3; ++k) q[k] = __fdiv_rn(__fdiv_rn(w[k], tr.area), tr.c[k].z);
  return __fdiv_rn(1.f, fadd(fadd(q[0], q[1]), q[2]));
}

__device__ __forceinline__ void triangle_pixel(const RenderArgs& a, const Triangle& tr, u32 t, int px, int py) {
  float w[3], q[3];
  if (!triangle_weights(tr, px, py, w)) return;
  const float z = triangle_depth(tr, w, q);
  if (!(z > 0.f) || !isfinite(z)) return;
  const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(z)) << 32) | t;
  atomicMin(a.keys + static_cast<size_t>(py) * a.width + px, key);
}

// Pixels [*p0, *p1] whose centres can lie in [lo, hi] on one axis, one pixel (plus a relative margin) wider on
// each side, clamped to the image. Coverage is decided by T4 alone; this only bounds the pixels tested.
__device__ __forceinline__ bool triangle_axis(float lo, float hi, int size, int* p0, int* p1) {
  const float pad = 1.f + (fabsf(lo) + fabsf(hi)) * 1e-6f;
  float q0 = floorf(lo - 0.5f - pad), q1 = ceilf(hi - 0.5f + pad);
  q0 = q0 > 0.f ? q0 : 0.f;
  const float last = static_cast<float>(size - 1);
  q1 = q1 < last ? q1 : last;
  if (!(q0 <= q1)) return false;
  *p0 = static_cast<int>(q0);
  *p1 = static_cast<int>(q1);
  return true;
}

__device__ __forceinline__ bool triangle_rect(const RenderArgs& a, const Triangle& tr, int* x0, int* y0, int* x1,
                                              int* y1) {
  const float u_lo = fminf(fminf(tr.u[0], tr.u[1]), tr.u[2]), u_hi = fmaxf(fmaxf(tr.u[0], tr.u[1]), tr.u[2]);
  const float v_lo = fminf(fminf(tr.v[0], tr.v[1]), tr.v[2]), v_hi = fmaxf(fmaxf(tr.v[0], tr.v[1]), tr.v[2]);
  return triangle_axis(u_lo, u_hi, a.width, x0, x1) && triangle_axis(v_lo, v_hi, a.height, y0, y1);
}

// T6 marking: one bit per corner of every T1-valid triangle.
__global__ void __launch_bounds__(kMarkBlock) k_mesh_render_mark(DeviceState d, RenderArgs a, MeshArgs m) {
  const u32 n = d.counters->surfel_count[a.count_slot];
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < m.triangle_count; t += gridDim.x * blockDim.x) {
    u32 s[3];
    if (!triangle_corners(d, m, t, n, s)) continue;
    for (int k = 0; k < 3; ++k) atomicOr(m.marks + (s[k] >> 5), 1u << (s[k] & 31));
  }
}

// Grid-stride sweep over the triangles: a small rectangle is tested by the thread itself, a larger one is listed
// (warp-aggregated append) for k_mesh_render_large.
__global__ void __launch_bounds__(kTriBlock) k_mesh_render_tri(DeviceState d, RenderArgs a, MeshArgs m) {
  const u32 n = d.counters->surfel_count[a.count_slot];
  const int lane = threadIdx.x & 31;
  for (u32 base = blockIdx.x * blockDim.x; base < m.triangle_count; base += gridDim.x * blockDim.x) {
    const u32 t = base + threadIdx.x;
    Triangle tr;
    int x0 = 0, y0 = 0, x1 = -1, y1 = -1;
    const bool drawn = t < m.triangle_count && load_triangle(d, a, m, t, n, &tr) && triangle_rect(a, tr, &x0, &y0, &x1, &y1);
    const bool large = drawn && static_cast<long long>(x1 - x0 + 1) * (y1 - y0 + 1) > kSmallTrianglePixels;
    const unsigned mask = __ballot_sync(0xffffffffu, large);
    if (mask) {
      u32 warp_base = 0;
      if (lane == 0) warp_base = atomicAdd(m.large_count, static_cast<u32>(__popc(mask)));
      warp_base = __shfl_sync(0xffffffffu, warp_base, 0);
      if (large) m.large_list[warp_base + __popc(mask & ((1u << lane) - 1u))] = t;   // < triangle_count entries
    }
    if (!drawn || large) continue;
    for (int py = y0; py <= y1; ++py)
      for (int px = x0; px <= x1; ++px) triangle_pixel(a, tr, t, px, py);
  }
}

// One warp per listed triangle, the lanes over the columns of its rectangle (bounded by the image).
__global__ void __launch_bounds__(kLargeBlock) k_mesh_render_large(DeviceState d, RenderArgs a, MeshArgs m) {
  const u32 n = d.counters->surfel_count[a.count_slot];
  const u32 count = *m.large_count;
  const int lane = threadIdx.x & 31;
  const u32 warps = gridDim.x * (kLargeBlock / 32);
  for (u32 k = blockIdx.x * (kLargeBlock / 32) + (threadIdx.x >> 5); k < count; k += warps) {
    const u32 t = m.large_list[k];
    Triangle tr;
    int x0, y0, x1, y1;
    // Not false: the sweep listed the triangle with the same result.
    if (!load_triangle(d, a, m, t, n, &tr) || !triangle_rect(a, tr, &x0, &y0, &x1, &y1)) continue;
    for (int py = y0; py <= y1; ++py)
      for (int px = x0 + lane; px <= x1; px += 32) triangle_pixel(a, tr, t, px, py);
  }
}

// T6: k_render_splat over the slots no T1-valid triangle names, with kDiskTag in the key. (The loop is k_render_splat's;
// sharing it through an inlined template changed k_render_splat's SASS, while load_splat and splat_pixel carry the
// rules.)
__global__ void __launch_bounds__(kSplatBlock) k_mesh_render_splat(DeviceState d, RenderArgs a, MeshArgs m) {
  const u32 n = d.counters->surfel_count[a.count_slot];
  const int lane = threadIdx.x & 31;
  for (u32 base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
    const u32 i = base + threadIdx.x;
    Splat s;
    const bool drawn = i < n && !((m.marks[i >> 5] >> (i & 31)) & 1u) && load_splat(d, a, i, &s);
    const bool large =
        drawn && static_cast<long long>(s.x1 - s.x0 + 1) * (s.y1 - s.y0 + 1) > kSmallSplatPixels;
    const unsigned mask = __ballot_sync(0xffffffffu, large);
    if (mask) {
      u32 warp_base = 0;
      if (lane == 0) warp_base = atomicAdd(a.large_count, static_cast<u32>(__popc(mask)));
      warp_base = __shfl_sync(0xffffffffu, warp_base, 0);
      if (large) a.large_list[warp_base + __popc(mask & ((1u << lane) - 1u))] = i;
    }
    if (!drawn || large) continue;
    for (int py = s.y0; py <= s.y1; ++py) {
      const float dy = ray_coord(py, a.cy, a.fy);
      for (int px = s.x0; px <= s.x1; ++px) splat_pixel(a, s, i | kDiskTag, px, py, dy);
    }
  }
}

__global__ void __launch_bounds__(kLargeBlock) k_mesh_render_splat_large(DeviceState d, RenderArgs a) {
  splat_large<true>(d, a);
}

// T7 colour channel: ((q0 c0 + q1 c1) + q2 c2) * z, rounded half up and clamped to 255.
__device__ __forceinline__ u32 blend_channel(const float q[3], const u32 rgb[3], int shift, float z) {
  float sum = fmul(q[0], u2f((rgb[0] >> shift) & 0xFFu));
  sum = fadd(sum, fmul(q[1], u2f((rgb[1] >> shift) & 0xFFu)));
  sum = fadd(sum, fmul(q[2], u2f((rgb[2] >> shift) & 0xFFu)));
  const float value = fadd(fmul(sum, z), 0.5f);
  return value >= 255.f ? 255u : static_cast<u32>(f2i_trunc(value));
}

// T7 normal: g = e1 x e2 with e1 = c1 - c0, e2 = c2 - c0 (corners in slot order), negated if g.c0 > 0, times
// 1 / sqrt(g.g); zero if g.g is not finite and > 0.
__device__ __forceinline__ float3 triangle_normal(const Triangle& tr) {
  const float3 e1 = make_float3(fsub(tr.c[1].x, tr.c[0].x), fsub(tr.c[1].y, tr.c[0].y), fsub(tr.c[1].z, tr.c[0].z));
  const float3 e2 = make_float3(fsub(tr.c[2].x, tr.c[0].x), fsub(tr.c[2].y, tr.c[0].y), fsub(tr.c[2].z, tr.c[0].z));
  float3 g = make_float3(fsub(fmul(e1.y, e2.z), fmul(e1.z, e2.y)), fsub(fmul(e1.z, e2.x), fmul(e1.x, e2.z)),
                         fsub(fmul(e1.x, e2.y), fmul(e1.y, e2.x)));
  const float facing = fadd(fadd(fmul(g.x, tr.c[0].x), fmul(g.y, tr.c[0].y)), fmul(g.z, tr.c[0].z));
  if (facing > 0.f) g = make_float3(-g.x, -g.y, -g.z);
  const float gg = fadd(fadd(fmul(g.x, g.x), fmul(g.y, g.y)), fmul(g.z, g.z));
  if (!(gg > 0.f) || !isfinite(gg)) return make_float3(0.f, 0.f, 0.f);
  const float inv = __fdiv_rn(1.f, __fsqrt_rn(gg));
  return make_float3(fmul(g.x, inv), fmul(g.y, inv), fmul(g.z, inv));
}

__global__ void __launch_bounds__(kResolveBlock) k_mesh_render_resolve(DeviceState d, RenderArgs a, MeshArgs m) {
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {   // the raster passes have finished
    *a.large_count = 0;
    *m.large_count = 0;
  }
  const int px = blockIdx.x * blockDim.x + threadIdx.x;
  if (px >= a.width) return;
  const u32 n = d.counters->surfel_count[a.count_slot];
  for (int py = blockIdx.y; py < a.height; py += gridDim.y) {
    unsigned long long* key_ptr = a.keys + static_cast<size_t>(py) * a.width + px;
    const unsigned long long key = *key_ptr;
    float depth = 0.f;
    u32 index = kInvalidIndex, rgb = 0;
    float3 nrm = make_float3(0.f, 0.f, 0.f);
    if (key != kEmptyKey) {
      *key_ptr = kEmptyKey;
      index = static_cast<u32>(key);
      depth = __uint_as_float(static_cast<u32>(key >> 32));
      if (index & kDiskTag) {
        const u32 i = index & ~kDiskTag;
        if (a.color) rgb = SM_SU(SM_ROW_COLOR, i);
        if (a.normal)
          nrm = rotate_vec(a.view_T_global, SM_S(SM_ROW_NORMAL_X, i), SM_S(SM_ROW_NORMAL_Y, i), SM_S(SM_ROW_NORMAL_Z, i));
      } else if (a.color || a.normal) {
        Triangle tr;
        load_triangle(d, a, m, index, n, &tr);   // true: the triangle proposed this key
        if (a.color) {
          float w[3], q[3];
          triangle_weights(tr, px, py, w);
          const float z = triangle_depth(tr, w, q);
          const u32 corner_rgb[3] = {SM_SU(SM_ROW_COLOR, tr.s[0]), SM_SU(SM_ROW_COLOR, tr.s[1]),
                                     SM_SU(SM_ROW_COLOR, tr.s[2])};
          rgb = blend_channel(q, corner_rgb, 0, z) | (blend_channel(q, corner_rgb, 8, z) << 8) |
                (blend_channel(q, corner_rgb, 16, z) << 16);
        }
        if (a.normal) nrm = triangle_normal(tr);
      }
    }
    if (a.depth) row_ptr(a.depth, a.depth_pitch, py)[px] = depth;
    if (a.index) row_ptr(a.index, a.index_pitch, py)[px] = index;
    if (a.color) {
      u8* o = row_ptr(a.color, a.color_pitch, py) + 3 * static_cast<size_t>(px);
      o[0] = rgb & 0xFFu; o[1] = (rgb >> 8) & 0xFFu; o[2] = (rgb >> 16) & 0xFFu;
    }
    if (a.normal) {
      float* o = row_ptr(a.normal, a.normal_pitch, py) + 3 * static_cast<size_t>(px);
      o[0] = nrm.x; o[1] = nrm.y; o[2] = nrm.z;
    }
  }
}

bool Finite(float v) { return std::isfinite(v); }

}  // namespace

const char* RenderCameraError(const sm_render_params& p, const float* view_T_global) {
  if (p.width <= 0 || p.height <= 0) return "width and height must be > 0";
  if (!Finite(p.fx) || !Finite(p.fy) || p.fx == 0.f || p.fy == 0.f) return "fx and fy must be finite and non-zero";
  if (!Finite(p.cx) || !Finite(p.cy)) return "cx and cy must be finite";
  if (!(p.near_depth > 0.f) || !(p.far_depth > p.near_depth)) return "need 0 < near_depth < far_depth";
  for (int k = 0; k < 12; ++k) if (!Finite(view_T_global[k])) return "view_T_global must be finite";
  return nullptr;
}

namespace {

// The key raster grows to `pixels`; the list, its count and the grids are set up once.
int EnsureRenderBuffers(sm_reconstruction* r, cudaStream_t stream, size_t pixels) {
  if (!r->render) r->render = new RenderScratch();
  RenderScratch& s = *r->render;
  if (s.large_list == nullptr) {
    SM_CUDA(cudaMalloc(&s.large_list, sizeof(u32) * r->d.stride));
    SM_CUDA(cudaMalloc(&s.large_count, sizeof(u32)));
    SM_CUDA(cudaMemsetAsync(s.large_count, 0, sizeof(u32), stream));
    int status = ResidentBlocks(k_render_splat, kSplatBlock, r->sm_count, &s.splat_blocks);
    if (status == SM_OK) status = ResidentBlocks(k_render_large, kLargeBlock, r->sm_count, &s.large_blocks);
    if (status != SM_OK) return status;
  }
  if (pixels > s.key_capacity) {
    cudaFree(s.keys);   // synchronises the device: an earlier render may still use it
    s.keys = nullptr;
    s.key_capacity = 0;
    SM_CUDA(cudaMalloc(&s.keys, sizeof(unsigned long long) * pixels));
    SM_CUDA(cudaMemsetAsync(s.keys, 0xFF, sizeof(unsigned long long) * pixels, stream));
    s.key_capacity = pixels;
  }
  return SM_OK;
}

// The argument checks of sm_render_surfels (also sm_render_mesh's) and the kernel arguments they allow.
int MakeRenderArgs(sm_reconstruction* r, cudaStream_t stream, const char* name, const sm_render_params& p,
                   const float* view_T_global, float* depth, size_t depth_pitch, uint8_t* color, size_t color_pitch,
                   float* normal, size_t normal_pitch, uint32_t* index, size_t index_pitch, RenderArgs* out) {
  auto bad = [name](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (std::string(name) + ": " + why).c_str()); };
  if (const char* why = RenderCameraError(p, view_T_global)) return bad(why);
  if (!depth && !color && !normal && !index) return bad("all outputs are NULL");
  const size_t w = static_cast<size_t>(p.width);
  if ((depth && depth_pitch < w * sizeof(float)) || (color && color_pitch < w * 3) ||
      (normal && normal_pitch < w * 3 * sizeof(float)) || (index && index_pitch < w * sizeof(u32)))
    return bad("a pitch is below the row size");
  RenderArgs& a = *out;
  a.count_slot = r->count_slot;
  a.width = p.width; a.height = p.height;
  a.fx = p.fx; a.fy = p.fy; a.cx = p.cx; a.cy = p.cy;
  a.near_depth = p.near_depth; a.far_depth = p.far_depth;
  a.view_T_global = MakeMat3x4(view_T_global);
  a.depth = depth; a.depth_pitch = depth_pitch;
  a.color = color; a.color_pitch = color_pitch;
  a.normal = normal; a.normal_pitch = normal_pitch;
  a.index = index; a.index_pitch = index_pitch;
  return SM_OK;
}

// sm_render_mesh's scratch beyond EnsureRenderBuffers': the triangle list grows to `triangles` entries; the slot
// bitmap (capacity bits), the list count and the grids are set up once.
int EnsureMeshRenderBuffers(sm_reconstruction* r, cudaStream_t stream, u32 triangles) {
  RenderScratch& s = *r->render;
  if (s.mesh_large_count == nullptr) {
    SM_CUDA(cudaMalloc(&s.mesh_marks, sizeof(u32) * ((r->d.stride + 31) / 32)));
    SM_CUDA(cudaMalloc(&s.mesh_large_count, sizeof(u32)));
    SM_CUDA(cudaMemsetAsync(s.mesh_large_count, 0, sizeof(u32), stream));
    int status = ResidentBlocks(k_mesh_render_mark, kMarkBlock, r->sm_count, &s.mesh_mark_blocks);
    if (status == SM_OK) status = ResidentBlocks(k_mesh_render_tri, kTriBlock, r->sm_count, &s.mesh_tri_blocks);
    if (status == SM_OK) status = ResidentBlocks(k_mesh_render_large, kLargeBlock, r->sm_count, &s.mesh_large_blocks);
    if (status == SM_OK) status = ResidentBlocks(k_mesh_render_splat, kSplatBlock, r->sm_count, &s.mesh_splat_blocks);
    if (status == SM_OK)
      status = ResidentBlocks(k_mesh_render_splat_large, kLargeBlock, r->sm_count, &s.mesh_splat_large_blocks);
    if (status != SM_OK) return status;
  }
  if (triangles > s.mesh_large_capacity) {
    cudaFree(s.mesh_large_list);   // synchronises the device: an earlier render may still use it
    s.mesh_large_list = nullptr;
    s.mesh_large_capacity = 0;
    SM_CUDA(cudaMalloc(&s.mesh_large_list, sizeof(u32) * triangles));
    s.mesh_large_capacity = triangles;
  }
  return SM_OK;
}

}  // namespace

int RenderSurfels(sm_reconstruction* r, cudaStream_t stream, const sm_render_params& p, const float* view_T_global,
                  float* depth, size_t depth_pitch, uint8_t* color, size_t color_pitch, float* normal,
                  size_t normal_pitch, uint32_t* index, size_t index_pitch) {
  RenderArgs a;
  int status = MakeRenderArgs(r, stream, "sm_render_surfels", p, view_T_global, depth, depth_pitch, color, color_pitch,
                              normal, normal_pitch, index, index_pitch, &a);
  if (status == SM_OK) status = EnsureRenderBuffers(r, stream, static_cast<size_t>(p.width) * static_cast<size_t>(p.height));
  if (status != SM_OK) return status;
  const RenderScratch& s = *r->render;
  a.keys = s.keys;
  a.large_list = s.large_list;
  a.large_count = s.large_count;
  r->last_stream = stream;
  { LaunchScope scope(stream, KID_RENDER_SPLAT); LaunchKernel(k_render_splat, dim3(s.splat_blocks), dim3(kSplatBlock), 0, stream, r->d, a); }
  { LaunchScope scope(stream, KID_RENDER_LARGE); LaunchKernel(k_render_large, dim3(s.large_blocks), dim3(kLargeBlock), 0, stream, r->d, a); }
  const dim3 resolve_grid((p.width + kResolveBlock - 1) / kResolveBlock, p.height < 65535 ? p.height : 65535);
  { LaunchScope scope(stream, KID_RENDER_RESOLVE); LaunchKernel(k_render_resolve, resolve_grid, dim3(kResolveBlock), 0, stream, r->d, a); }
  return CheckLaunch("render surfels");
}

int RenderMesh(sm_reconstruction* r, cudaStream_t stream, const sm_render_params& p, const float* view_T_global,
               const uint32_t* triangles, uint64_t triangle_count, int32_t flags, float* depth, size_t depth_pitch,
               uint8_t* color, size_t color_pitch, float* normal, size_t normal_pitch, uint32_t* index,
               size_t index_pitch) {
  RenderArgs a;
  int status = MakeRenderArgs(r, stream, "sm_render_mesh", p, view_T_global, depth, depth_pitch, color, color_pitch,
                              normal, normal_pitch, index, index_pitch, &a);
  if (status != SM_OK) return status;
  if (!triangles && triangle_count > 0)
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_render_mesh: triangles is NULL with a count > 0");
  if (triangle_count >= (1ull << 31)) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_render_mesh: triangle_count must be < 2^31");
  if (flags & ~SM_RENDER_UNMESHED_SURFELS) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_render_mesh: unknown flag bits");
  const bool disks = (flags & SM_RENDER_UNMESHED_SURFELS) != 0;
  status = EnsureRenderBuffers(r, stream, static_cast<size_t>(p.width) * static_cast<size_t>(p.height));
  if (status == SM_OK) status = EnsureMeshRenderBuffers(r, stream, static_cast<u32>(triangle_count));
  if (status != SM_OK) return status;
  const RenderScratch& s = *r->render;
  a.keys = s.keys;
  a.large_list = s.large_list;
  a.large_count = s.large_count;
  MeshArgs m;
  m.triangles = triangles;
  m.triangle_count = static_cast<u32>(triangle_count);
  m.marks = s.mesh_marks;
  m.large_list = s.mesh_large_list;
  m.large_count = s.mesh_large_count;
  r->last_stream = stream;
  auto grid = [](u32 items, int block, int resident) {
    const u32 blocks = (items + block - 1) / block;
    return dim3(blocks == 0 ? 1u : (blocks < static_cast<u32>(resident) ? blocks : static_cast<u32>(resident)));
  };
  if (disks) {
    SM_CUDA(cudaMemsetAsync(s.mesh_marks, 0, sizeof(u32) * ((r->d.stride + 31) / 32), stream));
    LaunchScope scope(stream, KID_MESH_RENDER_MARK);
    LaunchKernel(k_mesh_render_mark, grid(m.triangle_count, kMarkBlock, s.mesh_mark_blocks), dim3(kMarkBlock), 0,
                 stream, r->d, a, m);
  }
  { LaunchScope scope(stream, KID_MESH_RENDER_TRI); LaunchKernel(k_mesh_render_tri, grid(m.triangle_count, kTriBlock, s.mesh_tri_blocks), dim3(kTriBlock), 0, stream, r->d, a, m); }
  { LaunchScope scope(stream, KID_MESH_RENDER_LARGE); LaunchKernel(k_mesh_render_large, dim3(s.mesh_large_blocks), dim3(kLargeBlock), 0, stream, r->d, a, m); }
  if (disks) {
    { LaunchScope scope(stream, KID_MESH_RENDER_SPLAT); LaunchKernel(k_mesh_render_splat, dim3(s.mesh_splat_blocks), dim3(kSplatBlock), 0, stream, r->d, a, m); }
    { LaunchScope scope(stream, KID_MESH_RENDER_SPLAT_LARGE); LaunchKernel(k_mesh_render_splat_large, dim3(s.mesh_splat_large_blocks), dim3(kLargeBlock), 0, stream, r->d, a); }
  }
  const dim3 resolve_grid((p.width + kResolveBlock - 1) / kResolveBlock, p.height < 65535 ? p.height : 65535);
  { LaunchScope scope(stream, KID_MESH_RENDER_RESOLVE); LaunchKernel(k_mesh_render_resolve, resolve_grid, dim3(kResolveBlock), 0, stream, r->d, a, m); }
  return CheckLaunch("render mesh");
}

void FreeRenderBuffers(sm_reconstruction* r) {
  RenderScratch* s = r->render;
  if (!s) return;
  cudaFree(s->keys); cudaFree(s->large_list); cudaFree(s->large_count);
  cudaFree(s->mesh_marks); cudaFree(s->mesh_large_list); cudaFree(s->mesh_large_count);
  delete s;
  r->render = nullptr;
}

}  // namespace smb

using namespace smb;

extern "C" {

int sm_render_surfels(sm_reconstruction* r, void* stream, const sm_render_params* p, const float view_T_global[12],
                      float* depth, size_t depth_pitch, uint8_t* color, size_t color_pitch, float* normal,
                      size_t normal_pitch, uint32_t* index, size_t index_pitch) {
  if (!r || !p || !view_T_global) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_render_surfels: null argument");
  return RenderSurfels(r, static_cast<cudaStream_t>(stream), *p, view_T_global, depth, depth_pitch, color, color_pitch,
                       normal, normal_pitch, index, index_pitch);
}

int sm_render_mesh(sm_reconstruction* r, void* stream, const sm_render_params* p, const float view_T_global[12],
                   const uint32_t* triangles, uint64_t triangle_count, int32_t flags, float* depth, size_t depth_pitch,
                   uint8_t* color, size_t color_pitch, float* normal, size_t normal_pitch, uint32_t* index,
                   size_t index_pitch) {
  if (!r || !p || !view_T_global) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_render_mesh: null argument");
  return RenderMesh(r, static_cast<cudaStream_t>(stream), *p, view_T_global, triangles, triangle_count, flags, depth,
                    depth_pitch, color, color_pitch, normal, normal_pitch, index, index_pitch);
}

}  // extern "C"
