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

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstring>
#include <string>
#include <vector>

#include "sm_handle.cuh"
#include "sm_knn.cuh"
#include "sm_mesh_edges.cuh"

namespace smb {

struct MeshCounters {
  unsigned long long vertices_meshed;
  unsigned long long boundary_edges;
  unsigned long long umbrella_overflows;
  u32 max_radius_squared_bits;   // present radii are > 0: their bits order like the values
  u32 triangle_count;            // copied from the end of the scanned counts
};

struct MeshLive;

// The scratch of sm_triangulate, allocated by the first call and grown to surfels_size(): the k-NN index over the
// smooth positions, the umbrellas ([slots][SM_MESH_MAX_UMBRELLA] pairs) and their lengths, the per-slot triangle
// counts (scanned in place into offsets) and the scan's tile sums; the device counters and their pinned mirror;
// resident grids. Also sm_mesh_update's persistent mesh, which shares only the index.
struct MeshScratch {
  sm_knn_index* index = nullptr;
  uint2* umbrella = nullptr;
  u32* umbrella_count = nullptr;
  u32* counts = nullptr;
  u32* scan_sums = nullptr;
  u32 slots = 0;
  CounterMirror<MeshCounters> counters;
  int umbrella_blocks = 0, emit_blocks = 0;
  MeshLive* live = nullptr;   // created by the first sm_mesh_update
};

namespace {

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

// Rules 1-3 for slot i, by one warp (`stage`: the warp's 64-key row in shared memory): writes U(i) and its length,
// 0 when U(i) overflowed. An overflow is counted in a.counters (sm_triangulate) or, with kSlotFlag, flagged in
// overflow[i], which is cleared otherwise (sm_mesh_update).
template <bool kSlotFlag>
__device__ __forceinline__ void build_umbrella(const MeshArgs& a, u32 i, int lane, unsigned long long* stage, u8* overflow) {
  {
    const float r2 = SM_S(SM_ROW_RADIUS_SQUARED, i);
    float3 ni;
    if (!(r2 > 0.f) || !unit_normal(a, i, &ni)) {   // warp-uniform
      if (lane == 0) {
        a.umbrella_count[i] = 0;
        if (kSlotFlag) overflow[i] = 0;
      }
      return;
    }
    const float3 pi = position(a, i);
    QueryState s{{kEmptyKey, kEmptyKey}, 0, true, kEmptyKey, stage};
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
        if (kSlotFlag) overflow[i] = 1;
        else atomicAdd(&a.counters->umbrella_overflows, 1ull);
      }
      return;
    }
    const unsigned below = (1u << lane) - 1u;
    uint2* row = a.umbrella + static_cast<size_t>(i) * kUmbrella;
    if (pair0) row[__popc(b0 & below)] = make_uint2(c[0].index, next[0]);
    if (pair1) row[__popc(b0) + __popc(b1 & below)] = make_uint2(c[1].index, next[1]);
    if (lane == 0) {
      a.umbrella_count[i] = total;
      if (kSlotFlag) overflow[i] = 0;
    }
  }
}

__global__ void __launch_bounds__(kUmbrellaBlock) k_mesh_umbrella(MeshArgs a) {
  __shared__ unsigned long long s_stage[kUmbrellaBlock / 32][kMaxResults];
  const int lane = threadIdx.x & 31;
  const u32 warps_per_grid = gridDim.x * (kUmbrellaBlock / 32);
  for (u32 i = blockIdx.x * (kUmbrellaBlock / 32) + (threadIdx.x >> 5); i < a.n; i += warps_per_grid) {
    build_umbrella<false>(a, i, lane, s_stage[threadIdx.x >> 5], nullptr);
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

// ---- sm_mesh_update (DESIGN.md section 5.8): the persistent mesh, brought up to date from what changed ----------

constexpr int kSnapshotWords = 7;   // bits of smooth x y z, radius^2, normal x y z at the previous update
// The rebuild walks the whole cloud, as k_mesh_umbrella does, once A holds more than this share of surfels_size().
// On an H100 (tools/mesh_update_probe.py, DESIGN.md 5.8) the list costs ~24.5 us per 1 000 umbrellas and the sweep
// ~19.2 us per 1 000 slots of the final bench cloud: they cross at |A| / n ~ 0.78.
constexpr u32 kSweepNumerator = 3, kSweepDenominator = 4;
// Every slot is in A and R, without marking, once |C| exceeds this share of surfels_size(). In a live session the
// regularisation window changes 28-66 % of the slots per frame, far past it; marking then cost 2-4 ms on top of an
// umbrella rebuild of most slots. Below it the marking costs <= ~0.5 ms on the bench cloud (DESIGN.md 5.8).
constexpr u32 kMarkNumerator = 1, kMarkDenominator = 16;

struct UpdateCounters {
  // sums of the per-slot words over the current mesh, kept from call to call
  unsigned long long vertices_meshed, boundary_edges, umbrella_overflows;
  // per call (cleared at its start)
  MeshCounters bound;   // k_mesh_bound's largest radius^2
  u32 changed, rebuilt, rechecked, full_sweep;
  u32 triangle_count, added, removed, unused;
};

struct UpdateArgs {
  u32 n_prev;                  // surfels_size() at the previous update (0 before the first)
  u32 n_max;                   // max(n, n_prev)
  int everything;              // every slot is in A and in R
  u32* snapshot;               // [slots][kSnapshotWords]
  u8* overflow;                // [slots] U(i) overflowed
  u32* word;                   // [slots] the slot's share of the stats: boundary edges | meshed << 16 | overflow << 17
  u8* in_a;                    // [slots]
  u8* in_r;                    // [slots]
  u32* rebuild_list;           // [slots] the slots of A, in no particular order
  float* points;               // [4][point_stride]: x, y, z, 1 (present) or -1 of the old and new position of C's slots
  u32 point_stride;
  QueryArgs changed;           // the index over `points`
  const u32* old_offsets;      // [n_prev + 1] the previous mesh, by owner
  const uint3* old_triangles;
  u32* new_offsets;            // [n_max + 1] owned triangles, then (scanned) offsets
  u32* added_offsets;          // [n_max + 1]
  u32* removed_offsets;        // [n_max + 1]
  uint3* new_triangles;
  uint3* added;
  uint3* removed;
  UpdateCounters* counters;
};

// The lane's place in a warp-aggregated append to *counter.
__device__ __forceinline__ u32 warp_append(bool take, u32* counter, int lane) {
  const unsigned m = __ballot_sync(kFullMask, take);
  u32 base = 0;
  if (lane == 0 && m) base = atomicAdd(counter, static_cast<u32>(__popc(m)));
  return __shfl_sync(kFullMask, base, 0) + __popc(m & ((1u << lane) - 1u));
}

// C: a slot that is or was present and whose inputs differ from the snapshot (every slot of [n_prev, n) differs).
// Refreshes the snapshot, flags C in in_a and appends the old and new position of each slot of C to `points`.
// A slot of [n_prev, n) that is not present gets an empty umbrella and a zero share of the stats here: neither
// the rebuild nor the recheck visits it.
__global__ void __launch_bounds__(kEmitBlock) k_mesh_changes(MeshArgs a, UpdateArgs u) {
  const int lane = threadIdx.x & 31;
  const int rows[kSnapshotWords] = {SM_ROW_SMOOTH_X, SM_ROW_SMOOTH_Y, SM_ROW_SMOOTH_Z, SM_ROW_RADIUS_SQUARED,
                                    SM_ROW_NORMAL_X, SM_ROW_NORMAL_Y, SM_ROW_NORMAL_Z};
  for (u32 base = blockIdx.x * blockDim.x; base < u.n_max; base += gridDim.x * blockDim.x) {
    const u32 i = base + threadIdx.x;
    bool changed = false, was = false, is = false;
    u32 cur[kSnapshotWords] = {}, old[kSnapshotWords] = {};
    if (i < u.n_max) {
      const bool now = i < a.n, then = i < u.n_prev;
      u32* snap = u.snapshot + static_cast<size_t>(i) * kSnapshotWords;
#pragma unroll
      for (int k = 0; k < kSnapshotWords; ++k) {
        if (now) cur[k] = __float_as_uint(SM_S(rows[k], i));
        if (then) old[k] = snap[k];
      }
      bool differ = !then || !now;
#pragma unroll
      for (int k = 0; k < kSnapshotWords; ++k) differ = differ || cur[k] != old[k];
      was = then && __uint_as_float(old[3]) > 0.f;
      is = now && __uint_as_float(cur[3]) > 0.f;
      changed = (was || is) && differ;
      if (now && differ) {
#pragma unroll
        for (int k = 0; k < kSnapshotWords; ++k) snap[k] = cur[k];
      }
      if (now && !then && !is) {
        a.umbrella_count[i] = 0;
        u.overflow[i] = 0;
        u.word[i] = 0;
      }
      if (now) u.in_a[i] = changed;
    }
    const u32 slot = warp_append(changed, &u.counters->changed, lane);
    if (changed && !u.everything) {
      const size_t st = u.point_stride;
      float* pt = u.points + 2 * static_cast<size_t>(slot);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        pt[k * st] = __uint_as_float(old[k]);
        pt[k * st + 1] = __uint_as_float(cur[k]);
      }
      pt[3 * st] = was ? 1.f : -1.f;
      pt[3 * st + 1] = is ? 1.f : -1.f;
    }
  }
}

// Whether some record of the index lies within radius_squared of p, by the test and the cell walk of warp_query.
__device__ __forceinline__ bool near_record(const QueryArgs& q, float px, float py, float pz, float radius_squared) {
  auto within = [&](const float4 record) {
    const float dx = fsub(record.x, px), dy = fsub(record.y, py), dz = fsub(record.z, pz);
    return fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz)) <= radius_squared;
  };
  const float reach = __fmul_ru(__fsqrt_ru(radius_squared), 1.00001f);
  const int x0 = cell_of(__fsub_rd(px, reach), q.inverse_cell_size), x1 = cell_of(__fadd_ru(px, reach), q.inverse_cell_size);
  const int y0 = cell_of(__fsub_rd(py, reach), q.inverse_cell_size), y1 = cell_of(__fadd_ru(py, reach), q.inverse_cell_size);
  const int z0 = cell_of(__fsub_rd(pz, reach), q.inverse_cell_size), z1 = cell_of(__fadd_ru(pz, reach), q.inverse_cell_size);
  const long long nx = static_cast<long long>(x1) - x0 + 1, ny = static_cast<long long>(y1) - y0 + 1,
                  nz = static_cast<long long>(z1) - z0 + 1;
  if (nx > kMaxCellsPerQuery || ny > kMaxCellsPerQuery || nz > kMaxCellsPerQuery || nx * ny * nz > kMaxCellsPerQuery ||
      x1 == INT_MAX || y1 == INT_MAX || z1 == INT_MAX) {
    const u32 end = q.bucket_start[q.mask + 1];
    for (u32 e = 0; e < end; ++e)
      if (within(q.records[e])) return true;
    return false;
  }
  for (int cz = z0; cz <= z1; ++cz) {
    for (int cy = y0; cy <= y1; ++cy) {
      for (int cx = x0; cx <= x1; ++cx) {
        const u32 bucket = bucket_of(cx, cy, cz, q.mask);
        for (u32 e = q.bucket_start[bucket]; e < q.bucket_start[bucket + 1]; ++e) {
          const float4 record = q.records[e];
          if (cell_of(record.x, q.inverse_cell_size) == cx && cell_of(record.y, q.inverse_cell_size) == cy &&
              cell_of(record.z, q.inverse_cell_size) == cz && within(record))
            return true;
        }
      }
    }
  }
  return false;
}

// A: C, plus every present slot whose ball (the query of rule 1) holds an old or new position of a slot of C.
__global__ void __launch_bounds__(kEmitBlock) k_mesh_mark(MeshArgs a, UpdateArgs u) {
  const int lane = threadIdx.x & 31;
  for (u32 base = blockIdx.x * blockDim.x; base < a.n; base += gridDim.x * blockDim.x) {
    const u32 i = base + threadIdx.x;
    bool in = false;
    if (i < a.n) {
      in = u.in_a[i] != 0;
      const float r2 = SM_S(SM_ROW_RADIUS_SQUARED, i);
      if (!in && r2 > 0.f) {
        const float3 p = position(a, i);
        in = near_record(u.changed, p.x, p.y, p.z, fmul(r2, a.radius_factor_squared));
        if (in) u.in_a[i] = 1;
      }
    }
    const u32 slot = warp_append(in, &u.counters->rebuilt, lane);
    if (in) u.rebuild_list[slot] = i;
  }
}

// R: A, plus every slot whose umbrella names a slot of A (a slot outside A has the same umbrella before and after).
__global__ void __launch_bounds__(kEmitBlock) k_mesh_owners(MeshArgs a, UpdateArgs u) {
  const int lane = threadIdx.x & 31;
  for (u32 base = blockIdx.x * blockDim.x; base < u.n_max; base += gridDim.x * blockDim.x) {
    const u32 o = base + threadIdx.x;
    bool in = false;
    if (o < u.n_max) {
      in = u.everything || u.in_a[o];
      if (!in) {
        const u32 count = a.umbrella_count[o];
        const uint2* row = a.umbrella + static_cast<size_t>(o) * kUmbrella;
        for (u32 t = 0; t < count && !in; ++t) {
          const uint2 e = row[t];
          in = u.in_a[e.x] || u.in_a[e.y];
        }
      }
      u.in_r[o] = in;
    }
    const unsigned m = __ballot_sync(kFullMask, in);
    if (lane == 0 && m) atomicAdd(&u.counters->rechecked, static_cast<u32>(__popc(m)));
  }
}

// The umbrellas of A from the list, or of every slot by the sweep once A is a large share of the cloud.
__global__ void __launch_bounds__(kUmbrellaBlock) k_mesh_umbrella_update(MeshArgs a, UpdateArgs u) {
  __shared__ unsigned long long s_stage[kUmbrellaBlock / 32][kMaxResults];
  const int lane = threadIdx.x & 31;
  const u32 listed = u.counters->rebuilt;
  const bool sweep = u.everything || static_cast<unsigned long long>(listed) * kSweepDenominator >
                                         static_cast<unsigned long long>(a.n) * kSweepNumerator;
  if (blockIdx.x == 0 && threadIdx.x == 0) u.counters->full_sweep = sweep;
  const u32 items = sweep ? a.n : listed;
  const u32 warps_per_grid = gridDim.x * (kUmbrellaBlock / 32);
  for (u32 k = blockIdx.x * (kUmbrellaBlock / 32) + (threadIdx.x >> 5); k < items; k += warps_per_grid)
    build_umbrella<true>(a, sweep ? k : u.rebuild_list[k], lane, s_stage[threadIdx.x >> 5], u.overflow);
}

// (o, t.y, t.z) of the previous mesh is in the new one.
__device__ __forceinline__ bool in_new_mesh(const MeshArgs& a, u32 o, uint3 t) {
  return o < a.n && successor(a, o, t.y) == t.z && triangle_ok(a, o, t.y, t.z);
}

// (o, x, y) is among the previous mesh's triangles of o, old_triangles[begin, end).
__device__ __forceinline__ bool in_old_mesh(const UpdateArgs& u, u32 begin, u32 end, u32 x, u32 y) {
  for (u32 t = begin; t < end; ++t) {
    const uint3 v = u.old_triangles[t];
    if (v.y == x && v.z == y) return true;
  }
  return false;
}

// One thread per owner o < n_max. Outside R, o keeps its triangles (counted, then copied). In R, the first pass
// counts o's new triangles, its added and removed ones and its share of the stats exactly as k_mesh_count does,
// and adds the change of that share to the totals; the second writes them at the scanned offsets.
template <bool kWrite>
__global__ void __launch_bounds__(kEmitBlock) k_mesh_recheck(MeshArgs a, UpdateArgs u) {
  const int lane = threadIdx.x & 31;
  for (u32 base = blockIdx.x * blockDim.x; base < u.n_max; base += gridDim.x * blockDim.x) {
    const u32 o = base + threadIdx.x;
    int d_meshed = 0, d_boundary = 0, d_overflow = 0;
    if (o < u.n_max) {
      const u32 begin = o < u.n_prev ? u.old_offsets[o] : 0u, end = o < u.n_prev ? u.old_offsets[o + 1] : 0u;
      const u32 count = o < a.n ? a.umbrella_count[o] : 0u;
      const uint2* row = a.umbrella + static_cast<size_t>(o) * kUmbrella;
      if (!u.in_r[o]) {
        if (!kWrite) {
          u.new_offsets[o] = end - begin;
          u.added_offsets[o] = 0;
          u.removed_offsets[o] = 0;
        } else {
          u32 out = u.new_offsets[o];
          for (u32 t = begin; t < end; ++t) u.new_triangles[out++] = u.old_triangles[t];
        }
      } else if (!kWrite) {
        u32 owned = 0, boundary = 0, added = 0, removed = 0;
        bool meshed = false;
        for (u32 t = 0; t < count; ++t) {
          const uint2 e = row[t];
          if (!triangle_ok(a, o, e.x, e.y)) continue;
          meshed = true;
          if (o < e.x && o < e.y) {
            ++owned;
            if (!in_old_mesh(u, begin, end, e.x, e.y)) ++added;
          }
          const u32 w = successor(a, e.x, o);
          if (w == kNone || !triangle_ok(a, e.x, o, w)) ++boundary;
        }
        for (u32 t = begin; t < end; ++t) removed += in_new_mesh(a, o, u.old_triangles[t]) ? 0u : 1u;
        const u32 word = boundary | (meshed ? 1u << 16 : 0u) | (o < a.n && u.overflow[o] ? 1u << 17 : 0u);
        const u32 before = o < u.n_prev ? u.word[o] : 0u;
        d_meshed = static_cast<int>((word >> 16) & 1u) - static_cast<int>((before >> 16) & 1u);
        d_boundary = static_cast<int>(word & 0xFFFFu) - static_cast<int>(before & 0xFFFFu);
        d_overflow = static_cast<int>(word >> 17) - static_cast<int>(before >> 17);
        u.word[o] = word;
        u.new_offsets[o] = owned;
        u.added_offsets[o] = added;
        u.removed_offsets[o] = removed;
      } else {
        u32 out = u.new_offsets[o], add = u.added_offsets[o], rem = u.removed_offsets[o];
        for (u32 t = 0; t < count; ++t) {
          const uint2 e = row[t];
          if (!(o < e.x && o < e.y) || !triangle_ok(a, o, e.x, e.y)) continue;
          const uint3 tri = make_uint3(o, e.x, e.y);
          u.new_triangles[out++] = tri;
          if (!in_old_mesh(u, begin, end, e.x, e.y)) u.added[add++] = tri;
        }
        for (u32 t = begin; t < end; ++t) {
          const uint3 v = u.old_triangles[t];
          if (!in_new_mesh(a, o, v)) u.removed[rem++] = v;
        }
      }
    }
    if (!kWrite) {
      d_meshed = __reduce_add_sync(kFullMask, d_meshed);
      d_boundary = __reduce_add_sync(kFullMask, d_boundary);
      d_overflow = __reduce_add_sync(kFullMask, d_overflow);
      if (lane == 0) {
        // two's complement: adding the sign-extended difference subtracts modulo 2^64
        if (d_meshed) atomicAdd(&u.counters->vertices_meshed, static_cast<unsigned long long>(static_cast<long long>(d_meshed)));
        if (d_boundary) atomicAdd(&u.counters->boundary_edges, static_cast<unsigned long long>(static_cast<long long>(d_boundary)));
        if (d_overflow) atomicAdd(&u.counters->umbrella_overflows, static_cast<unsigned long long>(static_cast<long long>(d_overflow)));
      }
    }
  }
}

void FreeSlotScratch(MeshScratch& m) {
  KnnDestroy(m.index);
  m.index = nullptr;
  FreeAndClear(m.umbrella, m.umbrella_count, m.counts, m.scan_sums);
  m.slots = 0;
}

// Scratch for n slots (grown, never shrunk); the grids and the counters are set up once. The counters come last: a
// first call that fails leaves them empty, and the next call sets everything up again.
int EnsureMeshScratch(sm_reconstruction* r, u32 n) {
  if (!r->mesh) r->mesh = new MeshScratch();
  MeshScratch& m = *r->mesh;
  if (!m.counters.device) {
    int status = ResidentBlocks(k_mesh_umbrella, kUmbrellaBlock, r->sm_count, &m.umbrella_blocks);
    if (status == SM_OK) status = ResidentBlocks(k_mesh_count, kEmitBlock, r->sm_count, &m.emit_blocks);
    if (status == SM_OK) status = CreateCounters(m.counters);
    if (status != SM_OK) return status;
  }
  if (n <= m.slots) return SM_OK;
  FreeSlotScratch(m);
  const int status = KnnCreate(&m.index, n);
  if (status != SM_OK) return status;
  SM_CUDA(cudaMalloc(&m.umbrella, sizeof(uint2) * kUmbrella * static_cast<size_t>(n)));
  SM_CUDA(cudaMalloc(&m.umbrella_count, sizeof(u32) * static_cast<size_t>(n)));
  SM_CUDA(cudaMalloc(&m.counts, sizeof(u32) * (static_cast<size_t>(n) + 1)));
  SM_CUDA(cudaMalloc(&m.scan_sums, sizeof(u32) * ScanTiles(n + 1)));
  m.slots = n;
  return SM_OK;
}

QueryArgs IndexQuery(const sm_knn_index* k) {
  QueryArgs q{};
  q.max_result_count = kMaxResults;
  q.radius_scale = 1.f;
  q.include_completed = 1;
  q.include_free = 1;
  q.inverse_cell_size = k->inverse_cell_size;
  q.mask = k->table_size - 1;
  q.bucket_start = k->bucket_start;
  q.records = k->records;
  return q;
}


// SM_OK, or SM_ERR_INVALID_ARGUMENT for parameters outside their documented ranges.
int CheckMeshParams(const sm_mesh_params& p, const char* who) {
  auto bad = [who](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (std::string(who) + ": " + why).c_str()); };
  const float f = p.neighbor_radius_factor;
  const float f2 = f * f;
  if (!std::isfinite(f) || !(f > 0.f) || !std::isfinite(f2)) return bad("neighbor_radius_factor must be finite and > 0");
  if (!AngleInRange(p.max_angle_between_normals_deg) || !AngleInRange(p.max_triangle_angle_deg))
    return bad("angles must be in (0, 180] degrees");
  return SM_OK;
}

}  // namespace

}  // namespace smb

using namespace smb;

extern "C" void sm_default_mesh_params(sm_mesh_params* p) {
  p->neighbor_radius_factor = 2.0f;
  p->max_angle_between_normals_deg = 90.0f;
  p->max_triangle_angle_deg = 170.0f;
}

extern "C" int sm_triangulate(sm_reconstruction* r, void* stream_v, const sm_mesh_params* params, uint32_t* triangles,
                              uint64_t capacity, sm_mesh_stats* stats) {
  if (!r || !params || !stats) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_triangulate: null argument");
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const sm_mesh_params& p = *params;
  const int checked = CheckMeshParams(p, "sm_triangulate");
  if (checked != SM_OK) return checked;
  if (!triangles && capacity > 0)
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_triangulate: triangles is NULL with a capacity > 0");
  const float f2 = p.neighbor_radius_factor * p.neighbor_radius_factor;
  *stats = sm_mesh_stats{};
  r->last_stream = stream;
  int status = FetchCounters(r, stream);
  if (status == SM_ERR_CUDA) return status;   // (a surfel-cap overflow of an earlier frame does not matter here)
  const u32 n = r->host_counters->surfel_count[r->count_slot];
  if (n == 0) return SM_OK;
  status = EnsureMeshScratch(r, n);
  if (status != SM_OK) return status;
  const MeshScratch& m = *r->mesh;

  MeshArgs a{};
  a.n = n;
  a.rows = r->d.surfels;
  a.stride = r->d.stride;
  a.radius_factor_squared = f2;
  a.cos_normal = CosDegrees(p.max_angle_between_normals_deg);
  a.cos_triangle = CosDegrees(p.max_triangle_angle_deg);
  a.umbrella = m.umbrella;
  a.umbrella_count = m.umbrella_count;
  a.counts = m.counts;
  a.triangles = reinterpret_cast<uint3*>(triangles);
  a.counters = m.counters.device;
  status = MirrorRegRecords(stream, r->d, n, r->sm_count);   // rows 3-5 <- the current smooth positions
  if (status != SM_OK) return status;
  SM_CUDA(cudaMemsetAsync(m.counters.device, 0, sizeof(MeshCounters), stream));
  const int bound_blocks = static_cast<int>(std::min<u32>((n + kBoundBlock - 1) / kBoundBlock, 4u * r->sm_count));
  { LaunchScope scope(stream, KID_MESH_BOUND); LaunchKernel(k_mesh_bound, dim3(bound_blocks), dim3(kBoundBlock), 0, stream, a); }
  status = ReadCounters(m.counters, stream);
  if (status != SM_OK) return status;
  const MeshCounters& h = *m.counters.host;
  float max_r2;
  std::memcpy(&max_r2, &h.max_radius_squared_bits, sizeof(float));
  if (!(max_r2 > 0.f)) return SM_OK;   // no present slot
  // Cell size: twice the largest query radius, so that a query touches at most 3 cells per axis.
  const float cell_size = 2.f * std::sqrt(max_r2 * f2);
  const size_t st = r->d.stride;
  const float* s = r->d.surfels;
  status = KnnBuild(m.index, stream, n, s + SM_ROW_SMOOTH_X * st, s + SM_ROW_SMOOTH_Y * st,
                    s + SM_ROW_SMOOTH_Z * st, s + SM_ROW_RADIUS_SQUARED * st, nullptr, cell_size);
  if (status != SM_OK) return status;
  a.q = IndexQuery(m.index);
  const int umbrella_blocks =
      static_cast<int>(std::min<u32>((n + kUmbrellaBlock / 32 - 1) / (kUmbrellaBlock / 32), m.umbrella_blocks));
  const int emit_blocks = static_cast<int>(std::min<u32>((n + kEmitBlock - 1) / kEmitBlock, m.emit_blocks));
  { LaunchScope scope(stream, KID_MESH_UMBRELLA); LaunchKernel(k_mesh_umbrella, dim3(umbrella_blocks), dim3(kUmbrellaBlock), 0, stream, a); }
  SM_CUDA(cudaMemsetAsync(m.counts + n, 0, sizeof(u32), stream));
  { LaunchScope scope(stream, KID_MESH_COUNT); LaunchKernel(k_mesh_count, dim3(emit_blocks), dim3(kEmitBlock), 0, stream, a); }
  ScanInPlace(stream, m.counts, n + 1, m.scan_sums, KID_MESH_SCAN);
  SM_CUDA(cudaMemcpyAsync(&m.counters.device->triangle_count, m.counts + n, sizeof(u32), cudaMemcpyDeviceToDevice, stream));
  status = ReadCounters(m.counters, stream);
  if (status != SM_OK) return status;
  stats->triangle_count = h.triangle_count;
  stats->vertices_meshed = h.vertices_meshed;
  stats->boundary_edges = h.boundary_edges;
  stats->umbrella_overflows = h.umbrella_overflows;
  if (capacity < stats->triangle_count) return TriangleCapacityError("sm_triangulate", stats->triangle_count, capacity);
  if (stats->triangle_count > 0) {
    LaunchScope scope(stream, KID_MESH_WRITE);
    LaunchKernel(k_mesh_write, dim3(emit_blocks), dim3(kEmitBlock), 0, stream, a);
  }
  return CheckLaunch("triangulate");
}

namespace smb {

// The persistent mesh of sm_mesh_update. Per-slot arrays hold `slots` entries and grow (keeping what the previous
// update left) with surfels_size(); the triangle arrays grow with the mesh and its deltas.
struct MeshLive {
  bool valid = false;          // an update completed and everything below describes its mesh
  u32 n_prev = 0;              // surfels_size() at that update
  sm_mesh_params params{};
  int current = 0;             // which of offsets[] / triangles[] holds that mesh
  u64 triangle_count = 0, added_count = 0, removed_count = 0;
  u32 slots = 0;
  // kept from one update to the next
  u32* snapshot = nullptr;                  // [slots][kSnapshotWords]
  uint2* umbrella = nullptr;                // [slots][SM_MESH_MAX_UMBRELLA]
  u32* umbrella_count = nullptr;            // [slots]
  u8* overflow = nullptr;                   // [slots]
  u32* word = nullptr;                      // [slots]
  u32* offsets[2] = {nullptr, nullptr};     // [slots + 1]
  uint3* triangles[2] = {nullptr, nullptr};
  u64 triangle_capacity[2] = {0, 0};
  uint3* added = nullptr; u64 added_capacity = 0;
  uint3* removed = nullptr; u64 removed_capacity = 0;
  CounterMirror<UpdateCounters> counters;
  // scratch of one update
  u8* in_a = nullptr;
  u8* in_r = nullptr;
  u32* rebuild_list = nullptr;
  u32* added_offsets = nullptr;             // [slots + 1]
  u32* removed_offsets = nullptr;           // [slots + 1]
  u32* scan_sums = nullptr;
  float* points = nullptr;                  // [4][2 slots]
  sm_knn_index* changed_index = nullptr;
  int umbrella_blocks = 0, emit_blocks = 0;
};

namespace {

void FreeLive(MeshLive* L) {
  if (!L) return;
  for (void* q : {static_cast<void*>(L->snapshot), static_cast<void*>(L->umbrella), static_cast<void*>(L->umbrella_count),
                  static_cast<void*>(L->overflow), static_cast<void*>(L->word), static_cast<void*>(L->offsets[0]),
                  static_cast<void*>(L->offsets[1]), static_cast<void*>(L->triangles[0]),
                  static_cast<void*>(L->triangles[1]), static_cast<void*>(L->added), static_cast<void*>(L->removed),
                  static_cast<void*>(L->in_a), static_cast<void*>(L->in_r), static_cast<void*>(L->rebuild_list),
                  static_cast<void*>(L->added_offsets), static_cast<void*>(L->removed_offsets),
                  static_cast<void*>(L->scan_sums), static_cast<void*>(L->points)})
    cudaFree(q);
  FreeCounters(L->counters);
  KnnDestroy(L->changed_index);
  delete L;
}

// Grows a set of buffers behind one synchronisation: each new buffer gets the first `keep` elements of the old one
// and zeros after them; the old buffers are freed (and the new ones take their place) only when every step
// succeeded, otherwise the new ones are freed and the old ones stay.
class Growth {
 public:
  explicit Growth(cudaStream_t stream) : stream_(stream) {}
  ~Growth() { for (const Item& it : items_) cudaFree(status_ == SM_OK && done_ ? it.old_buffer : it.buffer); }
  template <class T>
  void grow(T** target, size_t count, size_t keep) {
    if (status_ != SM_OK) return;
    void* q = nullptr;
    const size_t bytes = sizeof(T) * count, kept = *target ? sizeof(T) * keep : 0;
    cudaError_t e = cudaMalloc(&q, bytes);
    if (e == cudaSuccess && kept) e = cudaMemcpyAsync(q, *target, kept, cudaMemcpyDeviceToDevice, stream_);
    if (e == cudaSuccess && bytes > kept) e = cudaMemsetAsync(static_cast<char*>(q) + kept, 0, bytes - kept, stream_);
    if (q) items_.push_back({reinterpret_cast<void**>(target), q, *target});
    if (e != cudaSuccess) status_ = SetError(SM_ERR_CUDA, (std::string("growing the mesh buffers: ") + cudaGetErrorString(e)).c_str());
  }
  int finish() {
    if (status_ == SM_OK) {
      const cudaError_t e = cudaStreamSynchronize(stream_);
      if (e != cudaSuccess) status_ = SetError(SM_ERR_CUDA, (std::string("cudaStreamSynchronize: ") + cudaGetErrorString(e)).c_str());
    }
    if (status_ == SM_OK) {
      for (const Item& it : items_) *it.target = it.buffer;
      done_ = true;
    }
    return status_;
  }

 private:
  struct Item { void** target; void* buffer; void* old_buffer; };
  cudaStream_t stream_;
  std::vector<Item> items_;
  int status_ = SM_OK;
  bool done_ = false;
};

// The grids and the counters on the first call (the counters last, as in EnsureMeshScratch); per-slot arrays for
// `slots` slots (x 1.5 when they grow, behind one synchronisation).
int EnsureLive(MeshLive& L, cudaStream_t stream, u32 slots, int sm_count) {
  if (!L.counters.device) {
    int status = ResidentBlocks(k_mesh_umbrella_update, kUmbrellaBlock, sm_count, &L.umbrella_blocks);
    if (status == SM_OK) status = ResidentBlocks(k_mesh_recheck<false>, kEmitBlock, sm_count, &L.emit_blocks);
    if (status == SM_OK) status = CreateCounters(L.counters);
    if (status != SM_OK) return status;
    SM_CUDA(cudaMemset(L.counters.device, 0, sizeof(UpdateCounters)));
  }
  if (slots <= L.slots) return SM_OK;
  const size_t cap = std::max<size_t>(slots, static_cast<size_t>(L.slots) * 3 / 2);
  const size_t keep = L.n_prev;   // (0 unless the previous update completed)
  Growth g(stream);
  g.grow(&L.snapshot, cap * kSnapshotWords, keep * kSnapshotWords);
  g.grow(&L.umbrella, cap * kUmbrella, keep * kUmbrella);
  g.grow(&L.umbrella_count, cap, keep);
  g.grow(&L.overflow, cap, keep);
  g.grow(&L.word, cap, keep);
  g.grow(&L.offsets[L.current], cap + 1, keep ? keep + 1 : 0);
  g.grow(&L.offsets[L.current ^ 1], cap + 1, 0);
  g.grow(&L.in_a, cap, 0);
  g.grow(&L.in_r, cap, 0);
  g.grow(&L.rebuild_list, cap, 0);
  g.grow(&L.added_offsets, cap + 1, 0);
  g.grow(&L.removed_offsets, cap + 1, 0);
  g.grow(&L.scan_sums, ScanTiles(cap + 1), 0);
  g.grow(&L.points, 4 * 2 * cap, 0);
  const int status = g.finish();
  if (status != SM_OK) return status;
  L.slots = static_cast<u32>(cap);
  return SM_OK;
}

// A triangle buffer of at least `count` (x 1.5 when it grows); its content is not kept.
int EnsureTriangles(uint3** p, u64* capacity, u64 count) {
  if (count <= *capacity) return SM_OK;
  const u64 grown = GrownCapacity(count);
  FreeAndClear(*p);
  *capacity = 0;
  SM_CUDA(cudaMalloc(p, sizeof(uint3) * grown));
  *capacity = grown;
  return SM_OK;
}

int Grid(u32 items, int block, int resident) {
  return static_cast<int>(std::max<u32>(1u, std::min<u32>((items + block - 1) / block, static_cast<u32>(resident))));
}

}  // namespace

void FreeMeshBuffers(sm_reconstruction* r) {
  MeshScratch* m = r->mesh;
  if (!m) return;
  FreeSlotScratch(*m);
  FreeCounters(m->counters);
  FreeLive(m->live);
  delete m;
  r->mesh = nullptr;
}

}  // namespace smb

extern "C" int sm_mesh_update(sm_reconstruction* r, void* stream_v, const sm_mesh_params* params,
                              sm_mesh_update_stats* stats) {
  if (!r || !params || !stats) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_mesh_update: null argument");
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const sm_mesh_params& p = *params;
  int status = CheckMeshParams(p, "sm_mesh_update");
  if (status != SM_OK) return status;
  *stats = sm_mesh_update_stats{};
  r->last_stream = stream;
  status = FetchCounters(r, stream);
  if (status == SM_ERR_CUDA) return status;   // (a surfel-cap overflow of an earlier frame does not matter here)
  const u32 n = r->host_counters->surfel_count[r->count_slot];
  if (!r->mesh) r->mesh = new MeshScratch();
  MeshScratch& m = *r->mesh;
  if (!m.live) m.live = new MeshLive{};
  MeshLive& L = *m.live;
  const bool was_valid = L.valid;
  L.valid = false;   // until this update completes; a failed one is followed by a rebuild from an empty mesh
  if (!was_valid) L.n_prev = 0;
  const u32 n_prev = L.n_prev, n_max = std::max(n, n_prev);
  status = EnsureLive(L, stream, std::max(n_max, 1u), r->sm_count);
  if (status != SM_OK) return status;
  if (!was_valid) SM_CUDA(cudaMemsetAsync(L.counters.device, 0, sizeof(UpdateCounters), stream));
  bool everything = !was_valid || n < n_prev || std::memcmp(&p, &L.params, sizeof(p)) != 0;
  const int previous = L.current, next = previous ^ 1;

  const float f2 = p.neighbor_radius_factor * p.neighbor_radius_factor;
  MeshArgs a{};
  a.n = n;
  a.rows = r->d.surfels;
  a.stride = r->d.stride;
  a.radius_factor_squared = f2;
  a.cos_normal = CosDegrees(p.max_angle_between_normals_deg);
  a.cos_triangle = CosDegrees(p.max_triangle_angle_deg);
  a.umbrella = L.umbrella;
  a.umbrella_count = L.umbrella_count;
  a.counters = &L.counters.device->bound;
  UpdateArgs u{};
  u.n_prev = n_prev;
  u.n_max = n_max;
  u.everything = everything;
  u.snapshot = L.snapshot;
  u.overflow = L.overflow;
  u.word = L.word;
  u.in_a = L.in_a;
  u.in_r = L.in_r;
  u.rebuild_list = L.rebuild_list;
  u.points = L.points;
  u.point_stride = 2 * L.slots;
  u.old_offsets = L.offsets[previous];
  u.old_triangles = L.triangles[previous];
  u.new_offsets = L.offsets[next];
  u.added_offsets = L.added_offsets;
  u.removed_offsets = L.removed_offsets;
  u.counters = L.counters.device;

  const size_t per_call = offsetof(UpdateCounters, bound);
  SM_CUDA(cudaMemsetAsync(reinterpret_cast<char*>(L.counters.device) + per_call, 0, sizeof(UpdateCounters) - per_call, stream));
  if (n > 0) {
    status = MirrorRegRecords(stream, r->d, n, r->sm_count);   // rows 3-5 <- the current smooth positions
    if (status != SM_OK) return status;
    const int bound_blocks = static_cast<int>(std::min<u32>((n + kBoundBlock - 1) / kBoundBlock, 4u * r->sm_count));
    LaunchScope scope(stream, KID_MESH_BOUND);
    LaunchKernel(k_mesh_bound, dim3(bound_blocks), dim3(kBoundBlock), 0, stream, a);
  }
  if (n_max > 0) {
    LaunchScope scope(stream, KID_MESH_CHANGES);
    LaunchKernel(k_mesh_changes, dim3(Grid(n_max, kEmitBlock, L.emit_blocks)), dim3(kEmitBlock), 0, stream, a, u);
  }
  status = ReadCounters(L.counters, stream);
  if (status != SM_OK) return status;
  const u32 changed = L.counters.host->changed;
  float max_r2;
  std::memcpy(&max_r2, &L.counters.host->bound.max_radius_squared_bits, sizeof(float));
  if (!(max_r2 > 0.f)) everything = true;   // no present slot: every umbrella is empty, no query runs
  // Past this share of changed slots, marking A (an index over 2 |C| points and a query per slot) costs more than
  // the list can save: every slot is rebuilt, as sm_triangulate does.
  if (static_cast<unsigned long long>(changed) * kMarkDenominator > static_cast<unsigned long long>(n) * kMarkNumerator)
    everything = true;
  u.everything = everything;

  if (max_r2 > 0.f) {
    // The index of rule 1, as sm_triangulate builds it (the index object is shared: both calls rebuild it).
    if (!m.index || m.index->capacity < n) {
      KnnDestroy(m.index);
      m.index = nullptr;
      status = KnnCreate(&m.index, std::max(n + n / 2, m.slots));   // x 1.5: a session grows n
      if (status != SM_OK) return status;
    }
    const float cell_size = 2.f * std::sqrt(max_r2 * f2);
    const size_t st = r->d.stride;
    const float* rows = r->d.surfels;
    status = KnnBuild(m.index, stream, n, rows + SM_ROW_SMOOTH_X * st, rows + SM_ROW_SMOOTH_Y * st,
                      rows + SM_ROW_SMOOTH_Z * st, rows + SM_ROW_RADIUS_SQUARED * st, nullptr, cell_size);
    if (status != SM_OK) return status;
    a.q = IndexQuery(m.index);
    if (!everything && changed > 0) {
      // A from the small side: an index over the <= 2 |C| old and new positions, one existence query per present
      // slot with its own radius. A slot's work is bounded by the changed points near it, however large the
      // largest radius (which sets the cell size) is.
      const u32 points = 2 * changed;
      if (!L.changed_index || L.changed_index->capacity < points) {
        KnnDestroy(L.changed_index);
        L.changed_index = nullptr;
        status = KnnCreate(&L.changed_index, std::max(points, std::min(2 * L.slots, points * 2)));
        if (status != SM_OK) return status;
      }
      const size_t ps = u.point_stride;
      status = KnnBuild(L.changed_index, stream, points, L.points, L.points + ps, L.points + 2 * ps, L.points + 3 * ps,
                        nullptr, cell_size);
      if (status != SM_OK) return status;
      u.changed = IndexQuery(L.changed_index);
      LaunchScope scope(stream, KID_MESH_MARK);
      LaunchKernel(k_mesh_mark, dim3(Grid(n, kEmitBlock, L.emit_blocks)), dim3(kEmitBlock), 0, stream, a, u);
    }
  }
  const int emit_blocks = Grid(n_max, kEmitBlock, L.emit_blocks);
  {
    LaunchScope scope(stream, KID_MESH_OWNERS);
    LaunchKernel(k_mesh_owners, dim3(emit_blocks), dim3(kEmitBlock), 0, stream, a, u);
  }
  if (n > 0) {
    LaunchScope scope(stream, KID_MESH_UMBRELLA_UPDATE);
    LaunchKernel(k_mesh_umbrella_update, dim3(Grid(n, kUmbrellaBlock / 32, L.umbrella_blocks)), dim3(kUmbrellaBlock), 0,
                 stream, a, u);
  }
  for (u32* v : {u.new_offsets, u.added_offsets, u.removed_offsets})
    SM_CUDA(cudaMemsetAsync(v + n_max, 0, sizeof(u32), stream));
  {
    LaunchScope scope(stream, KID_MESH_RECHECK);
    LaunchKernel(k_mesh_recheck<false>, dim3(emit_blocks), dim3(kEmitBlock), 0, stream, a, u);
  }
  ScanInPlace(stream, u.new_offsets, n_max + 1, L.scan_sums, KID_MESH_SCAN);
  ScanInPlace(stream, u.added_offsets, n_max + 1, L.scan_sums, KID_MESH_SCAN);
  ScanInPlace(stream, u.removed_offsets, n_max + 1, L.scan_sums, KID_MESH_SCAN);
  SM_CUDA(cudaMemcpyAsync(&L.counters.device->triangle_count, u.new_offsets + n_max, sizeof(u32), cudaMemcpyDeviceToDevice, stream));
  SM_CUDA(cudaMemcpyAsync(&L.counters.device->added, u.added_offsets + n_max, sizeof(u32), cudaMemcpyDeviceToDevice, stream));
  SM_CUDA(cudaMemcpyAsync(&L.counters.device->removed, u.removed_offsets + n_max, sizeof(u32), cudaMemcpyDeviceToDevice, stream));
  status = ReadCounters(L.counters, stream);
  if (status != SM_OK) return status;
  const UpdateCounters h = *L.counters.host;
  status = EnsureTriangles(&L.triangles[next], &L.triangle_capacity[next], h.triangle_count);
  if (status == SM_OK) status = EnsureTriangles(&L.added, &L.added_capacity, h.added);
  if (status == SM_OK) status = EnsureTriangles(&L.removed, &L.removed_capacity, h.removed);
  if (status != SM_OK) return status;
  u.new_triangles = L.triangles[next];
  u.added = L.added;
  u.removed = L.removed;
  if (n_max > 0) {
    LaunchScope scope(stream, KID_MESH_RECHECK_WRITE);
    LaunchKernel(k_mesh_recheck<true>, dim3(emit_blocks), dim3(kEmitBlock), 0, stream, a, u);
  }
  status = CheckLaunch("mesh_update");
  if (status != SM_OK) return status;

  L.current = next;
  L.n_prev = n;
  L.params = p;
  L.triangle_count = h.triangle_count;
  L.added_count = h.added;
  L.removed_count = h.removed;
  L.valid = true;
  stats->mesh.triangle_count = h.triangle_count;
  stats->mesh.vertices_meshed = h.vertices_meshed;
  stats->mesh.boundary_edges = h.boundary_edges;
  stats->mesh.umbrella_overflows = h.umbrella_overflows;
  stats->slots_changed = h.changed;
  stats->umbrellas_rebuilt = everything ? n : h.rebuilt;
  stats->owners_rechecked = h.rechecked;
  stats->triangles_added = h.added;
  stats->triangles_removed = h.removed;
  stats->full_sweep = everything || h.full_sweep ? 1 : 0;
  return SM_OK;
}

namespace smb {

namespace {

// words[0] = 1 if a slot removed by sm_compact was present at the last update, words[1] = removed slots below n_prev.
__global__ void k_mesh_compact_check(const u32* map, const u32* snapshot, u32 n_prev, u32* words) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n_prev; i += gridDim.x * blockDim.x) {
    if (map[i] != kNone) continue;
    atomicAdd(words + 1, 1u);
    if (__uint_as_float(snapshot[static_cast<size_t>(i) * kSnapshotWords + 3]) > 0.f) words[0] = 1u;
  }
}

// Every corner of `count` triangles through the map (a removed slot, or one >= n, becomes kNone).
__global__ void k_mesh_compact_remap(u32* corners, u64 count, const u32* map, u32 n) {
  for (u64 i = blockIdx.x * static_cast<u64>(blockDim.x) + threadIdx.x; i < 3 * count;
       i += static_cast<u64>(gridDim.x) * blockDim.x) {
    const u32 v = corners[i];
    corners[i] = v < n ? map[v] : kNone;
  }
}

}  // namespace

int MeshCompact(sm_reconstruction* r, cudaStream_t stream, const u32* map, u32 n, u32* scratch, u32* words,
                u32* host_words, int* remapped) {
  *remapped = 0;
  MeshLive* L = r->mesh ? r->mesh->live : nullptr;
  if (!L || !L->valid) return SM_OK;
  const u32 n_prev = L->n_prev;
  const int blocks = 4 * r->sm_count;
  if (n_prev > n) { L->valid = false; return SM_OK; }   // (an sm_reset / sm_load_state since: a full rebuild anyway)
  if (n_prev > 0) {
    SM_CUDA(cudaMemsetAsync(words, 0, 2 * sizeof(u32), stream));
    { LaunchScope scope(stream, KID_COMPACT_MESH); LaunchKernel(k_mesh_compact_check, dim3(blocks), dim3(256), 0, stream, map, static_cast<const u32*>(L->snapshot), n_prev, words); }
    SM_CUDA(cudaMemcpyAsync(host_words, words, 2 * sizeof(u32), cudaMemcpyDeviceToHost, stream));
    SM_CUDA(cudaStreamSynchronize(stream));
    // A slot merged after the update is still a corner of the mesh, which names it: the next update rebuilds all.
    if (host_words[0]) { L->valid = false; return SM_OK; }
  } else {
    host_words[1] = 0;
  }
  const u32 kept = n_prev - host_words[1];
  const int sms = r->sm_count;
  int status = CompactWords(stream, sms, map, n_prev, kept, L->snapshot, kSnapshotWords, scratch, false);
  if (status == SM_OK) status = CompactWords(stream, sms, map, n_prev, kept, reinterpret_cast<u32*>(L->umbrella), 2 * kUmbrella, scratch, true);
  if (status == SM_OK) status = CompactWords(stream, sms, map, n_prev, kept, L->umbrella_count, 1, scratch, false);
  if (status == SM_OK) status = CompactWords(stream, sms, map, n_prev, kept, L->word, 1, scratch, false);
  if (status == SM_OK) status = CompactBytes(stream, sms, map, n_prev, kept, L->overflow, scratch);
  // offsets: the removed slots own no triangle, so the kept ones keep theirs, and the end moves down to `kept`
  u32* offsets = L->offsets[L->current];
  if (status == SM_OK) status = CompactWords(stream, sms, map, n_prev, kept, offsets, 1, scratch, false);
  if (status != SM_OK) return status;
  if (kept < n_prev) SM_CUDA(cudaMemcpyAsync(offsets + kept, offsets + n_prev, sizeof(u32), cudaMemcpyDeviceToDevice, stream));
  const struct { uint3* list; u64 count; } lists[3] = {
      {L->triangles[L->current], L->triangle_count}, {L->added, L->added_count}, {L->removed, L->removed_count}};
  for (const auto& t : lists) {
    if (t.count == 0) continue;
    LaunchScope scope(stream, KID_COMPACT_MESH);
    LaunchKernel(k_mesh_compact_remap, dim3(blocks), dim3(256), 0, stream, reinterpret_cast<u32*>(t.list), t.count, map, n);
  }
  status = CheckLaunch("compact: mesh");
  if (status != SM_OK) return status;
  L->n_prev = kept;
  *remapped = 1;
  return SM_OK;
}

}  // namespace smb

extern "C" int sm_mesh_read(sm_reconstruction* r, void* stream_v, int32_t which, uint32_t* triangles,
                            uint64_t capacity, uint64_t* count) {
  if (!r || !count) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_mesh_read: null argument");
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  auto bad = [](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (std::string("sm_mesh_read: ") + why).c_str()); };
  if (which != SM_MESH_ALL && which != SM_MESH_ADDED && which != SM_MESH_REMOVED) return bad("unknown `which`");
  if (!triangles && capacity > 0) return bad("triangles is NULL with a capacity > 0");
  const MeshLive* L = r->mesh ? r->mesh->live : nullptr;
  if (!L || !L->valid) return bad("no sm_mesh_update has completed on this handle");
  const uint3* src = which == SM_MESH_ALL ? L->triangles[L->current] : (which == SM_MESH_ADDED ? L->added : L->removed);
  const u64 size = which == SM_MESH_ALL ? L->triangle_count : (which == SM_MESH_ADDED ? L->added_count : L->removed_count);
  *count = size;
  if (capacity < size) return TriangleCapacityError("sm_mesh_read", size, capacity);
  r->last_stream = stream;
  if (size > 0) SM_CUDA(cudaMemcpyAsync(triangles, src, sizeof(uint3) * size, cudaMemcpyDeviceToDevice, stream));
  return SM_OK;
}
