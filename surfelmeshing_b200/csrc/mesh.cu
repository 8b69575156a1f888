// mesh.cu — sm_triangulate (DESIGN.md section 5.7): the surfel cloud as an indexed triangle mesh. Every present
// slot builds its umbrella, the Delaunay neighbours of the slot in its tangent plane among its k-NN, and a
// triangle is output when the umbrellas of all three corners agree on it. The rules, step by step, are in
// include/surfel_b200.h.
//
// Launches on the caller's stream (the call synchronises three times: surfels_size(), the cell size of the
// index, the triangle count):
//   k_mesh_bound     largest radius^2 of the present slots (the cell size of the k-NN index);
//   (the k-NN index build of knn.cu over the smooth positions)
//   k_mesh_umbrella  one warp per slot: the k-NN query core of sm_knn_query, then the tangent-plane clipping with
//                    two candidates per lane; writes U(i) as {j, next(j)} pairs into the handle's scratch;
//   k_mesh_count     one thread per slot: checks its pairs against the other two umbrellas and the filters,
//                    counts the triangles it owns, the slots that are meshed and the boundary edges;
//   (the three-launch exclusive scan of knn.cu over the counts)
//   k_mesh_write     one thread per slot: writes its triangles at its scanned offset.

#include <cmath>
#include <cstring>
#include <string>

#include "sm_handle.cuh"
#include "sm_knn.cuh"

namespace smb {

struct MeshCounters {
  unsigned long long vertices_meshed;
  unsigned long long boundary_edges;
  unsigned long long umbrella_overflows;
  u32 max_radius_squared_bits;   // present radii are > 0: their bits order like the values
  u32 triangle_count;            // copied from the end of the scanned counts
};

namespace {

#define SM_CUDA(call)                                                                                   \
  do {                                                                                                  \
    const cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) return SetError(SM_ERR_CUDA, (std::string(#call) + ": " + cudaGetErrorString(e_)).c_str()); \
  } while (0)

constexpr int kUmbrellaBlock = 128;   // 4 slots per block, one warp each
constexpr int kEmitBlock = 256;
constexpr int kBoundBlock = 256;
constexpr int kUmbrella = SM_MESH_MAX_UMBRELLA;   // pairs per slot
constexpr u32 kNone = 0xFFFFFFFFu;

#define SM_S(row, i) a.rows[static_cast<size_t>(row) * a.stride + (i)]

struct MeshArgs {
  u32 n;                       // surfels_size()
  const float* rows;           // SoA, rows 3-5 = the mirror of the current smooth positions
  size_t stride;
  float radius_factor_squared;
  float cos_normal;            // neighbours with n_i . n_j below this are dropped
  float cos_triangle;          // an angle whose cosine is below this exceeds max_triangle_angle
  QueryArgs q;                 // the index (records, buckets, cell size); state NULL, 64 results
  uint2* umbrella;             // [n][kUmbrella]: {j, next(j)}
  u32* umbrella_count;         // [n]
  u32* counts;                 // [n + 1]: owned triangles, then (scanned) offsets
  uint3* triangles;
  MeshCounters* counters;
};

__device__ __forceinline__ float dot2(float ax, float ay, float bx, float by) { return fadd(fmul(ax, bx), fmul(ay, by)); }
__device__ __forceinline__ float cross2(float ax, float ay, float bx, float by) { return fsub(fmul(ax, by), fmul(ay, bx)); }
__device__ __forceinline__ float dot3p(float3 a, float3 b) { return fadd(fadd(fmul(a.x, b.x), fmul(a.y, b.y)), fmul(a.z, b.z)); }
__device__ __forceinline__ float3 sub3(float3 a, float3 b) { return make_float3(fsub(a.x, b.x), fsub(a.y, b.y), fsub(a.z, b.z)); }

__device__ __forceinline__ float3 position(const MeshArgs& a, u32 i) {
  return make_float3(SM_S(SM_ROW_SMOOTH_X, i), SM_S(SM_ROW_SMOOTH_Y, i), SM_S(SM_ROW_SMOOTH_Z, i));
}

// Rows 8-10 times 1 / sqrt(n . n) (IEEE); false unless n . n is finite and > 0.
__device__ __forceinline__ bool unit_normal(const MeshArgs& a, u32 i, float3* out) {
  const float3 n = make_float3(SM_S(SM_ROW_NORMAL_X, i), SM_S(SM_ROW_NORMAL_Y, i), SM_S(SM_ROW_NORMAL_Z, i));
  const float s = dot3p(n, n);
  if (!(s > 0.f) || !isfinite(s)) return false;
  const float inv = __fdiv_rn(1.f, __fsqrt_rn(s));
  *out = make_float3(fmul(n.x, inv), fmul(n.y, inv), fmul(n.z, inv));
  return true;
}

// Constraint k on the bisector of j, both projected: the bisector point m_j + (s / 2) perp(q_j) lies in k's
// half-plane iff s * c <= b, with c = cross(q_j, q_k) and b = |q_k|^2 - q_j . q_k.
__device__ __forceinline__ void constraint(float jx, float jy, float kx, float ky, float* c, float* b) {
  *c = cross2(jx, jy, kx, ky);
  *b = fsub(dot2(kx, ky, kx, ky), dot2(jx, jy, kx, ky));
}

__global__ void __launch_bounds__(kBoundBlock) k_mesh_bound(MeshArgs a) {
  u32 best = 0;
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const float r2 = SM_S(SM_ROW_RADIUS_SQUARED, i);
    if (r2 > 0.f && isfinite(r2)) best = max(best, __float_as_uint(r2));
  }
  best = __reduce_max_sync(kFullMask, best);
  if ((threadIdx.x & 31) == 0 && best) atomicMax(&a.counters->max_radius_squared_bits, best);
}

// One candidate (a k-NN rank) of the warp's slot.
struct Candidate {
  u32 index;
  bool valid;
  float qx, qy;
};

__device__ __forceinline__ float pick(int reg, float v0, float v1) { return reg ? v1 : v0; }

__global__ void __launch_bounds__(kUmbrellaBlock) k_mesh_umbrella(MeshArgs a) {
  __shared__ unsigned long long s_stage[kUmbrellaBlock / 32][kMaxResults];
  const int lane = threadIdx.x & 31;
  const u32 warps_per_grid = gridDim.x * (kUmbrellaBlock / 32);
  for (u32 i = blockIdx.x * (kUmbrellaBlock / 32) + (threadIdx.x >> 5); i < a.n; i += warps_per_grid) {
    const float r2 = SM_S(SM_ROW_RADIUS_SQUARED, i);
    float3 ni;
    if (!(r2 > 0.f) || !unit_normal(a, i, &ni)) {   // warp-uniform
      if (lane == 0) a.umbrella_count[i] = 0;
      continue;
    }
    const float3 pi = position(a, i);
    QueryState s{{kEmptyKey, kEmptyKey}, 0, true, kEmptyKey, s_stage[threadIdx.x >> 5]};
    warp_query(a.q, s, pi.x, pi.y, pi.z, fmul(r2, a.radius_factor_squared), lane);
    const int found = min(s.count, kMaxResults);

    // Tangent basis (Duff et al. 2017).
    const float sign = copysignf(1.f, ni.z);
    const float bf = __fdiv_rn(-1.f, fadd(sign, ni.z));
    const float bb = fmul(fmul(ni.x, ni.y), bf);
    const float3 u = make_float3(fadd(1.f, fmul(fmul(fmul(sign, ni.x), ni.x), bf)), fmul(sign, bb), -fmul(sign, ni.x));
    const float3 v = make_float3(bb, fadd(sign, fmul(fmul(ni.y, ni.y), bf)), -ni.y);

    // Rule 1-2: the candidates of ranks lane and lane + 32.
    Candidate c[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const unsigned long long key = r ? s.list.e1 : s.list.e0;
      const int rank = lane + 32 * r;
      c[r].index = static_cast<u32>(key);
      c[r].valid = rank < found && c[r].index != i;
      c[r].qx = 0.f; c[r].qy = 0.f;
      float3 nj;
      if (c[r].valid) c[r].valid = unit_normal(a, c[r].index, &nj) && dot3p(ni, nj) >= a.cos_normal;
      if (c[r].valid) {
        const float3 d = sub3(position(a, c[r].index), pi);
        c[r].qx = dot3p(d, u);
        c[r].qy = dot3p(d, v);
        c[r].valid = !(c[r].qx == 0.f && c[r].qy == 0.f);
      }
    }
    // Coincident projections: only the first in rank order stays.
    bool coincident[2] = {false, false};
    for (int src = 0; src < 64; ++src) {
      const int reg = src >> 5, from = src & 31;
      const bool kv = __shfl_sync(kFullMask, reg ? c[1].valid : c[0].valid, from);
      const float kx = __shfl_sync(kFullMask, pick(reg, c[0].qx, c[1].qx), from);
      const float ky = __shfl_sync(kFullMask, pick(reg, c[0].qy, c[1].qy), from);
#pragma unroll
      for (int r = 0; r < 2; ++r)
        if (kv && src < lane + 32 * r && kx == c[r].qx && ky == c[r].qy) coincident[r] = true;
    }
    c[0].valid = c[0].valid && !coincident[0];
    c[1].valid = c[1].valid && !coincident[1];

    // Rule 3: the interval [lo, hi] of each bisector, with the smallest slot index among the constraints that set
    // each end.
    float lo[2], hi[2];
    u32 lo_min[2] = {kNone, kNone}, hi_min[2] = {kNone, kNone};
    bool has_lo[2] = {false, false}, has_hi[2] = {false, false}, infeasible[2] = {false, false};
    lo[0] = lo[1] = hi[0] = hi[1] = 0.f;
    for (int src = 0; src < 64; ++src) {
      const int reg = src >> 5, from = src & 31;
      const bool kv = __shfl_sync(kFullMask, reg ? c[1].valid : c[0].valid, from);
      const u32 ki = __shfl_sync(kFullMask, reg ? c[1].index : c[0].index, from);
      const float kx = __shfl_sync(kFullMask, pick(reg, c[0].qx, c[1].qx), from);
      const float ky = __shfl_sync(kFullMask, pick(reg, c[0].qy, c[1].qy), from);
      if (!kv) continue;   // warp-uniform
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        if (!c[r].valid || src == lane + 32 * r) continue;
        float cc, b;
        constraint(c[r].qx, c[r].qy, kx, ky, &cc, &b);
        if (cc == 0.f) {
          if (b < 0.f) infeasible[r] = true;
          continue;
        }
        const float t = __fdiv_rn(b, cc);
        if (cc > 0.f) {
          if (!has_hi[r] || t < hi[r]) { hi[r] = t; hi_min[r] = ki; has_hi[r] = true; }
          else if (t == hi[r]) hi_min[r] = min(hi_min[r], ki);
        } else {
          if (!has_lo[r] || t > lo[r]) { lo[r] = t; lo_min[r] = ki; has_lo[r] = true; }
          else if (t == lo[r]) lo_min[r] = min(lo_min[r], ki);
        }
      }
    }
    bool kept[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      kept[r] = c[r].valid && !infeasible[r];
      if (kept[r] && has_lo[r] && has_hi[r] && !(lo[r] < hi[r]))
        kept[r] = lo[r] == hi[r] && min(i, c[r].index) < min(lo_min[r], hi_min[r]);
    }

    // next(j): among the kept constraints that set hi, the first counter-clockwise from j.
    u32 next[2] = {kNone, kNone};
    float bx[2] = {0.f, 0.f}, by[2] = {0.f, 0.f};
    for (int src = 0; src < 64; ++src) {
      const int reg = src >> 5, from = src & 31;
      const bool kk = __shfl_sync(kFullMask, reg ? kept[1] : kept[0], from);
      const u32 ki = __shfl_sync(kFullMask, reg ? c[1].index : c[0].index, from);
      const float kx = __shfl_sync(kFullMask, pick(reg, c[0].qx, c[1].qx), from);
      const float ky = __shfl_sync(kFullMask, pick(reg, c[0].qy, c[1].qy), from);
      if (!kk) continue;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        if (!kept[r] || !has_hi[r] || src == lane + 32 * r) continue;
        float cc, b;
        constraint(c[r].qx, c[r].qy, kx, ky, &cc, &b);
        if (!(cc > 0.f) || __fdiv_rn(b, cc) != hi[r]) continue;
        if (next[r] == kNone || cross2(kx, ky, bx[r], by[r]) > 0.f) { next[r] = ki; bx[r] = kx; by[r] = ky; }
      }
    }
    // Partial bijection: a slot named as next by two candidates is nobody's next.
    int predecessors[2] = {0, 0};
    for (int src = 0; src < 64; ++src) {
      const int reg = src >> 5, from = src & 31;
      const u32 kn = __shfl_sync(kFullMask, reg ? next[1] : next[0], from);
#pragma unroll
      for (int r = 0; r < 2; ++r) predecessors[r] += (kn != kNone && kn == next[r]) ? 1 : 0;
    }
    const bool pair0 = next[0] != kNone && predecessors[0] == 1;
    const bool pair1 = next[1] != kNone && predecessors[1] == 1;
    const unsigned b0 = __ballot_sync(kFullMask, pair0), b1 = __ballot_sync(kFullMask, pair1);
    const int total = __popc(b0) + __popc(b1);
    if (total > kUmbrella) {
      if (lane == 0) {
        a.umbrella_count[i] = 0;
        atomicAdd(&a.counters->umbrella_overflows, 1ull);
      }
      continue;
    }
    const unsigned below = (1u << lane) - 1u;
    uint2* row = a.umbrella + static_cast<size_t>(i) * kUmbrella;
    if (pair0) row[__popc(b0 & below)] = make_uint2(c[0].index, next[0]);
    if (pair1) row[__popc(b0) + __popc(b1 & below)] = make_uint2(c[1].index, next[1]);
    if (lane == 0) a.umbrella_count[i] = total;
  }
}

// {y, z} is a pair of U(x). A slot names each candidate at most once as the first of a pair.
__device__ __forceinline__ bool has_pair(const MeshArgs& a, u32 x, u32 y, u32 z) {
  const u32 count = a.umbrella_count[x];
  const uint2* row = a.umbrella + static_cast<size_t>(x) * kUmbrella;
  for (u32 t = 0; t < count; ++t) {
    const uint2 e = row[t];
    if (e.x == y) return e.y == z;
  }
  return false;
}

// The first pair of U(x) that starts with y: its second slot, or kNone.
__device__ __forceinline__ u32 successor(const MeshArgs& a, u32 x, u32 y) {
  const u32 count = a.umbrella_count[x];
  const uint2* row = a.umbrella + static_cast<size_t>(x) * kUmbrella;
  for (u32 t = 0; t < count; ++t) {
    const uint2 e = row[t];
    if (e.x == y) return e.y;
  }
  return kNone;
}

__device__ __forceinline__ bool angle_too_large(const MeshArgs& a, float3 e1, float3 e2) {
  const float d = dot3p(e1, e2);
  const float l = __fsqrt_rn(fmul(dot3p(e1, e1), dot3p(e2, e2)));
  return d < fmul(a.cos_triangle, l);
}

// Rule 4 for the triangle (i, x, y) where {x, y} is a pair of U(i): the other two umbrellas agree, and the
// filters hold, evaluated in the rotation that starts at the smallest index.
__device__ __forceinline__ bool triangle_ok(const MeshArgs& a, u32 i, u32 x, u32 y) {
  if (!has_pair(a, x, y, i) || !has_pair(a, y, i, x)) return false;
  u32 o = i, p = x, q = y;
  if (x < o && x < y) { o = x; p = y; q = i; }
  else if (y < o && y < x) { o = y; p = i; q = x; }
  float3 no;
  if (!unit_normal(a, o, &no)) return false;
  const float3 po = position(a, o), pp = position(a, p), pq = position(a, q);
  const float3 e1 = sub3(pp, po), e2 = sub3(pq, po);
  const float3 g = make_float3(fsub(fmul(e1.y, e2.z), fmul(e1.z, e2.y)), fsub(fmul(e1.z, e2.x), fmul(e1.x, e2.z)),
                               fsub(fmul(e1.x, e2.y), fmul(e1.y, e2.x)));
  if (!(dot3p(g, no) > 0.f)) return false;
  if (angle_too_large(a, e1, e2)) return false;
  if (angle_too_large(a, sub3(pq, pp), sub3(po, pp))) return false;
  if (angle_too_large(a, sub3(po, pq), sub3(pp, pq))) return false;
  return true;
}

__global__ void __launch_bounds__(kEmitBlock) k_mesh_count(MeshArgs a) {
  const int lane = threadIdx.x & 31;
  for (u32 base = blockIdx.x * blockDim.x; base < a.n; base += gridDim.x * blockDim.x) {
    const u32 i = base + threadIdx.x;
    u32 owned = 0, boundary = 0;
    bool meshed = false;
    if (i < a.n) {
      const u32 count = a.umbrella_count[i];
      const uint2* row = a.umbrella + static_cast<size_t>(i) * kUmbrella;
      for (u32 t = 0; t < count; ++t) {
        const uint2 e = row[t];
        if (!triangle_ok(a, i, e.x, e.y)) continue;
        meshed = true;
        if (i < e.x && i < e.y) ++owned;
        // The edge i -> e.x of this triangle; the reverse edge belongs to the triangle (e.x, i, successor).
        const u32 w = successor(a, e.x, i);
        if (w == kNone || !triangle_ok(a, e.x, i, w)) ++boundary;
      }
      a.counts[i] = owned;
    }
    const unsigned meshed_lanes = __ballot_sync(kFullMask, meshed);
    boundary = __reduce_add_sync(kFullMask, boundary);
    if (lane == 0) {
      if (meshed_lanes) atomicAdd(&a.counters->vertices_meshed, static_cast<unsigned long long>(__popc(meshed_lanes)));
      if (boundary) atomicAdd(&a.counters->boundary_edges, static_cast<unsigned long long>(boundary));
    }
  }
}

__global__ void __launch_bounds__(kEmitBlock) k_mesh_write(MeshArgs a) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    if (a.counts[i + 1] == a.counts[i]) continue;   // owns nothing
    u32 out = a.counts[i];
    const u32 count = a.umbrella_count[i];
    const uint2* row = a.umbrella + static_cast<size_t>(i) * kUmbrella;
    for (u32 t = 0; t < count; ++t) {
      const uint2 e = row[t];
      if (i < e.x && i < e.y && triangle_ok(a, i, e.x, e.y)) a.triangles[out++] = make_uint3(i, e.x, e.y);
    }
  }
}

void FreeMeshScratch(sm_reconstruction* r) {
  KnnDestroy(r->mesh_index);
  cudaFree(r->mesh_umbrella);
  cudaFree(r->mesh_umbrella_count);
  cudaFree(r->mesh_counts);
  cudaFree(r->mesh_scan_sums);
  r->mesh_index = nullptr;
  r->mesh_umbrella = nullptr;
  r->mesh_umbrella_count = nullptr;
  r->mesh_counts = nullptr;
  r->mesh_scan_sums = nullptr;
  r->mesh_slots = 0;
}

// Scratch for n slots (grown, never shrunk); the counters and the grids are set up once.
int EnsureMeshScratch(sm_reconstruction* r, u32 n) {
  if (!r->mesh_counters) {
    SM_CUDA(cudaMalloc(&r->mesh_counters, sizeof(MeshCounters)));
    SM_CUDA(cudaMallocHost(&r->mesh_host_counters, sizeof(MeshCounters)));
    int status = ResidentBlocks(k_mesh_umbrella, kUmbrellaBlock, r->sm_count, &r->mesh_umbrella_blocks);
    if (status == SM_OK) status = ResidentBlocks(k_mesh_count, kEmitBlock, r->sm_count, &r->mesh_emit_blocks);
    if (status != SM_OK) return status;
  }
  if (n <= r->mesh_slots) return SM_OK;
  FreeMeshScratch(r);   // cudaFree synchronises the device: an earlier call may still use the buffers
  const int status = KnnCreate(&r->mesh_index, n);
  if (status != SM_OK) return status;
  const u32 tiles = (n + 1 + kScanTile - 1) / kScanTile;
  SM_CUDA(cudaMalloc(&r->mesh_umbrella, sizeof(uint2) * kUmbrella * static_cast<size_t>(n)));
  SM_CUDA(cudaMalloc(&r->mesh_umbrella_count, sizeof(u32) * static_cast<size_t>(n)));
  SM_CUDA(cudaMalloc(&r->mesh_counts, sizeof(u32) * (static_cast<size_t>(n) + 1)));
  SM_CUDA(cudaMalloc(&r->mesh_scan_sums, sizeof(u32) * tiles));
  r->mesh_slots = n;
  return SM_OK;
}

}  // namespace

void FreeMeshBuffers(sm_reconstruction* r) {
  FreeMeshScratch(r);
  cudaFree(r->mesh_counters);
  if (r->mesh_host_counters) cudaFreeHost(r->mesh_host_counters);
  r->mesh_counters = nullptr;
  r->mesh_host_counters = nullptr;
}

int Triangulate(sm_reconstruction* r, cudaStream_t stream, const sm_mesh_params& p, uint32_t* triangles,
                uint64_t capacity, sm_mesh_stats* stats) {
  auto bad = [](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (std::string("sm_triangulate: ") + why).c_str()); };
  const float f = p.neighbor_radius_factor;
  const float f2 = f * f;
  if (!std::isfinite(f) || !(f > 0.f) || !std::isfinite(f2)) return bad("neighbor_radius_factor must be finite and > 0");
  auto angle_ok = [](float deg) { return std::isfinite(deg) && deg > 0.f && deg <= 180.f; };
  if (!angle_ok(p.max_angle_between_normals_deg) || !angle_ok(p.max_triangle_angle_deg))
    return bad("angles must be in (0, 180] degrees");
  if (!triangles && capacity > 0) return bad("triangles is NULL with a capacity > 0");
  *stats = sm_mesh_stats{};
  r->last_stream = stream;
  int status = FetchCounters(r, stream);
  if (status == SM_ERR_CUDA) return status;   // (a surfel-cap overflow of an earlier frame does not matter here)
  const u32 n = r->host_counters->surfel_count[r->count_slot];
  if (n == 0) return SM_OK;
  status = EnsureMeshScratch(r, n);
  if (status != SM_OK) return status;

  MeshArgs a{};
  a.n = n;
  a.rows = r->d.surfels;
  a.stride = r->d.stride;
  a.radius_factor_squared = f2;
  a.cos_normal = static_cast<float>(std::cos(static_cast<double>(p.max_angle_between_normals_deg) * (M_PI / 180.0)));
  a.cos_triangle = static_cast<float>(std::cos(static_cast<double>(p.max_triangle_angle_deg) * (M_PI / 180.0)));
  a.umbrella = r->mesh_umbrella;
  a.umbrella_count = r->mesh_umbrella_count;
  a.counts = r->mesh_counts;
  a.triangles = reinterpret_cast<uint3*>(triangles);
  a.counters = r->mesh_counters;
  status = MirrorRegRecords(stream, r->d, n, r->sm_count);   // rows 3-5 <- the current smooth positions
  if (status != SM_OK) return status;
  SM_CUDA(cudaMemsetAsync(r->mesh_counters, 0, sizeof(MeshCounters), stream));
  const int bound_blocks = static_cast<int>(std::min<u32>((n + kBoundBlock - 1) / kBoundBlock, 4u * r->sm_count));
  { LaunchScope scope(stream, KID_MESH_BOUND); LaunchKernel(k_mesh_bound, dim3(bound_blocks), dim3(kBoundBlock), 0, stream, a); }
  SM_CUDA(cudaMemcpyAsync(r->mesh_host_counters, r->mesh_counters, sizeof(MeshCounters), cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaStreamSynchronize(stream));
  float max_r2;
  std::memcpy(&max_r2, &r->mesh_host_counters->max_radius_squared_bits, sizeof(float));
  if (!(max_r2 > 0.f)) return SM_OK;   // no present slot
  // Cell size: twice the largest query radius, so that a query touches at most 3 cells per axis.
  const float cell_size = 2.f * std::sqrt(max_r2 * f2);
  const size_t st = r->d.stride;
  const float* s = r->d.surfels;
  status = KnnBuild(r->mesh_index, stream, n, s + SM_ROW_SMOOTH_X * st, s + SM_ROW_SMOOTH_Y * st,
                    s + SM_ROW_SMOOTH_Z * st, s + SM_ROW_RADIUS_SQUARED * st, nullptr, cell_size);
  if (status != SM_OK) return status;
  sm_knn_index* k = r->mesh_index;
  a.q = QueryArgs{};
  a.q.max_result_count = kMaxResults;
  a.q.radius_scale = 1.f;
  a.q.include_completed = 1;
  a.q.include_free = 1;
  a.q.inverse_cell_size = k->inverse_cell_size;
  a.q.mask = k->table_size - 1;
  a.q.bucket_start = k->bucket_start;
  a.q.records = k->records;
  const int umbrella_blocks =
      static_cast<int>(std::min<u32>((n + kUmbrellaBlock / 32 - 1) / (kUmbrellaBlock / 32), r->mesh_umbrella_blocks));
  const int emit_blocks = static_cast<int>(std::min<u32>((n + kEmitBlock - 1) / kEmitBlock, r->mesh_emit_blocks));
  { LaunchScope scope(stream, KID_MESH_UMBRELLA); LaunchKernel(k_mesh_umbrella, dim3(umbrella_blocks), dim3(kUmbrellaBlock), 0, stream, a); }
  SM_CUDA(cudaMemsetAsync(r->mesh_counts + n, 0, sizeof(u32), stream));
  { LaunchScope scope(stream, KID_MESH_COUNT); LaunchKernel(k_mesh_count, dim3(emit_blocks), dim3(kEmitBlock), 0, stream, a); }
  const u32 scan_n = n + 1;
  const u32 tiles = (scan_n + kScanTile - 1) / kScanTile;
  { LaunchScope scope(stream, KID_MESH_SCAN); k_knn_scan_tiles<<<tiles, kScanBlock, 0, stream>>>(r->mesh_counts, scan_n, r->mesh_scan_sums); }
  { LaunchScope scope(stream, KID_MESH_SCAN); k_knn_scan_sums<<<1, kScanBlock, 0, stream>>>(r->mesh_scan_sums, tiles); }
  { LaunchScope scope(stream, KID_MESH_SCAN); k_knn_scan_add<<<tiles, kScanBlock, 0, stream>>>(r->mesh_counts, scan_n, r->mesh_scan_sums); }
  SM_CUDA(cudaMemcpyAsync(&r->mesh_counters->triangle_count, r->mesh_counts + n, sizeof(u32), cudaMemcpyDeviceToDevice, stream));
  SM_CUDA(cudaMemcpyAsync(r->mesh_host_counters, r->mesh_counters, sizeof(MeshCounters), cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaStreamSynchronize(stream));
  const MeshCounters& h = *r->mesh_host_counters;
  stats->triangle_count = h.triangle_count;
  stats->vertices_meshed = h.vertices_meshed;
  stats->boundary_edges = h.boundary_edges;
  stats->umbrella_overflows = h.umbrella_overflows;
  if (capacity < stats->triangle_count) {
    return SetError(SM_ERR_CAPACITY, ("sm_triangulate: " + std::to_string(stats->triangle_count) +
                                      " triangles do not fit the capacity of " + std::to_string(capacity)).c_str());
  }
  if (stats->triangle_count > 0) {
    LaunchScope scope(stream, KID_MESH_WRITE);
    LaunchKernel(k_mesh_write, dim3(emit_blocks), dim3(kEmitBlock), 0, stream, a);
  }
  return CheckLaunch("triangulate");
}

}  // namespace smb
