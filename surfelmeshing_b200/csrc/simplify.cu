// simplify.cu — sm_mesh_simplify (DESIGN.md section 5.14): half-edge collapses ranked by plane quadrics, in rounds of
// collapses with disjoint closed neighbourhoods. The rules S1-S8, step by step, are in include/surfel_b200.h.
//
// Launches on the caller's stream:
//   k_simplify_edges       one thread per input triangle: the input checks of sm_mesh_fill_holes (sm_mesh_edges.cuh)
//                          and the copy into the working list;
//   k_simplify_boundary    one thread per directed edge: counts the edges whose reverse is absent;
//   (synchronisation: the input checks)
//   fans, at the start and after every round:
//     k_simplify_corners   one thread per input position: slot << 32 | position of each corner of a current triangle;
//     (CUB radix sort of the corners: each slot's triangles in ascending input position)
//     k_simplify_bounds    one thread per sorted corner: each slot's range, the list of slots, the marks cleared;
//   k_simplify_quadrics    one thread per listed slot: Q_i of S1 (once);
//   a round:
//     k_simplify_candidates  one thread per listed slot: the fan walk, the valid collapses and best(u) (S3), and
//                            the key into the marks of its closed neighbourhood (S4);
//     k_simplify_select      one thread per listed slot: selected iff it holds every mark of its neighbourhood;
//     (synchronisation: the selected count; in the budget round, a CUB radix sort of the selected keys)
//     k_simplify_apply       one thread per applied collapse (S6);
//   k_simplify_owners      one thread per sorted corner: 1 where the corner is its triangle's smallest slot;
//   (the three-launch exclusive scan of knn.cu over those flags: the order of S8; synchronisation: the end)
//   k_simplify_write       one thread per sorted corner: the owners write their rotated triangles.

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>

#include "sm_handle.cuh"
#include "sm_knn.cuh"
#include "sm_mesh_edges.cuh"

namespace smb {

namespace {

constexpr int kMaxValence = SM_MESH_MAX_VALENCE;
constexpr u32 kNone = 0xFFFFFFFFu;   // no slot; also every corner of a deleted triangle
constexpr u64 kNoKey = ~0ull;

}  // namespace

struct Quadric { double q[10]; };

struct SimplifyCounters {
  u32 errors;
  u32 boundary_edges;
  u32 corners;     // corner keys appended by k_simplify_corners
  u32 vertices;    // slots listed by k_simplify_bounds
  u32 selected;
  u32 pad;
  unsigned long long max_cost_bits;   // of a non-negative double: its bits order as its value
};

// The scratch of sm_mesh_simplify: per input triangle and per slot.
struct SimplifyScratch {
  CounterMirror<SimplifyCounters> counters;
  u64 triangle_capacity = 0;
  u64* edge_table = nullptr;      // a power of two >= 6 x triangle_capacity
  uint3* tri = nullptr;           // the working list by input position
  u64* corners = nullptr;         // 3 x: slot << 32 | position, unsorted
  u64* sorted = nullptr;          // 3 x: sorted
  u32* counts = nullptr;          // 3 x + 1: owner flags, then (scanned) output offsets
  u32* scan_sums = nullptr;
  u32 slot_capacity = 0;
  Quadric* quadric = nullptr;
  u32* begin = nullptr; u32* end = nullptr;   // a slot's range of sorted corners
  u64* mark = nullptr; u64* key = nullptr;
  u32* best = nullptr; double* cost = nullptr;
  u32* vertices = nullptr;        // the slots with a current triangle
  u64* selected = nullptr; u64* selected_sorted = nullptr;
  void* sort_temp = nullptr; size_t sort_temp_bytes = 0;
};

namespace {

struct SimplifyArgs {
  u32 n;                          // surfels_size()
  const float* rows;
  size_t stride;
  const uint3* input;
  u32 count;
  uint3* tri;
  u64* edge_table; u64 edge_mask;
  u64* corners; const u64* sorted; u32 corner_count;
  u32* begin; u32* end; u32* vertices;
  Quadric* quadric;
  u64* mark; u64* key; u32* best; double* cost;
  u64* selected; const u64* apply; u32 apply_count;
  u32* counts; uint3* out;
  float cos_normal, cos_triangle;
  double max_cost;
  SimplifyCounters* counters;
};

__device__ __forceinline__ u32 corner_slot(u64 key) { return static_cast<u32>(key >> 32); }
__device__ __forceinline__ u32 corner_position(u64 key) { return static_cast<u32>(key); }

// The other two corners of triangle c after slot u, in winding order.
__device__ __forceinline__ void after(uint3 c, u32 u, u32* a, u32* b) {
  if (c.x == u) { *a = c.y; *b = c.z; }
  else if (c.y == u) { *a = c.z; *b = c.x; }
  else { *a = c.x; *b = c.y; }
}

__device__ __forceinline__ double3 position_d(const SimplifyArgs& a, u32 i) {
  const float3 p = slot_position(a.rows, a.stride, i);
  return make_double3(p.x, p.y, p.z);
}

// S1: K_t of triangle c, added entry by entry to q.
__device__ __forceinline__ void add_plane(const SimplifyArgs& a, uint3 c, double* q) {
  const double3 pa = position_d(a, c.x), pb = position_d(a, c.y), pc = position_d(a, c.z);
  const double3 e1 = make_double3(__dsub_rn(pb.x, pa.x), __dsub_rn(pb.y, pa.y), __dsub_rn(pb.z, pa.z));
  const double3 e2 = make_double3(__dsub_rn(pc.x, pa.x), __dsub_rn(pc.y, pa.y), __dsub_rn(pc.z, pa.z));
  const double gx = __dsub_rn(__dmul_rn(e1.y, e2.z), __dmul_rn(e1.z, e2.y));
  const double gy = __dsub_rn(__dmul_rn(e1.z, e2.x), __dmul_rn(e1.x, e2.z));
  const double gz = __dsub_rn(__dmul_rn(e1.x, e2.y), __dmul_rn(e1.y, e2.x));
  const double gg = __dadd_rn(__dadd_rn(__dmul_rn(gx, gx), __dmul_rn(gy, gy)), __dmul_rn(gz, gz));
  if (!(gg > 0.0)) return;   // K_t = 0 (a sum that starts at +0 is never -0, so adding +0 changes no bit)
  const double s = __dsqrt_rn(gg);
  const double mx = __ddiv_rn(gx, s), my = __ddiv_rn(gy, s), mz = __ddiv_rn(gz, s);
  const double d = -__dadd_rn(__dadd_rn(__dmul_rn(mx, pa.x), __dmul_rn(my, pa.y)), __dmul_rn(mz, pa.z));
  const double k[10] = {__dmul_rn(mx, mx), __dmul_rn(mx, my), __dmul_rn(mx, mz), __dmul_rn(mx, d), __dmul_rn(my, my),
                        __dmul_rn(my, mz), __dmul_rn(my, d),  __dmul_rn(mz, mz), __dmul_rn(mz, d), __dmul_rn(d, d)};
#pragma unroll
  for (int j = 0; j < 10; ++j) q[j] = __dadd_rn(q[j], k[j]);
}

// S1: the cost E of quadric q at (x, y, z).
__device__ __forceinline__ double quadric_cost(const double* q, double x, double y, double z) {
  auto row = [&](double a, double b, double c, double w) {
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a, x), __dmul_rn(b, y)), __dmul_rn(c, z)), w);
  };
  const double r0 = row(q[0], q[1], q[2], q[3]);
  const double r1 = row(q[1], q[4], q[5], q[6]);
  const double r2 = row(q[2], q[5], q[7], q[8]);
  const double r3 = row(q[3], q[6], q[8], q[9]);
  return row(r0, r1, r2, r3);
}

// S3 (c): the geometric tests of the triangle (x0, x1, x2) (winding order).
__device__ bool triangle_ok(const SimplifyArgs& a, u32 x0, u32 x1, u32 x2) {
  float3 n0, n1, n2;
  if (!slot_unit_normal(a.rows, a.stride, x0, &n0) || !slot_unit_normal(a.rows, a.stride, x1, &n1) ||
      !slot_unit_normal(a.rows, a.stride, x2, &n2))
    return false;
  if (!(dot3p(n0, n1) >= a.cos_normal) || !(dot3p(n1, n2) >= a.cos_normal) || !(dot3p(n0, n2) >= a.cos_normal))
    return false;
  u32 o = x0, x = x1, y = x2;
  float3 no = n0, nx = n1, ny = n2;
  if (x1 < x0 && x1 < x2) { o = x1; x = x2; y = x0; no = n1; nx = n2; ny = n0; }
  else if (x2 < x0 && x2 < x1) { o = x2; x = x0; y = x1; no = n2; nx = n0; ny = n1; }
  const float3 po = slot_position(a.rows, a.stride, o), px = slot_position(a.rows, a.stride, x),
               py = slot_position(a.rows, a.stride, y);
  const float3 e1 = sub3(px, po), e2 = sub3(py, po);
  const float3 g = make_float3(fsub(fmul(e1.y, e2.z), fmul(e1.z, e2.y)), fsub(fmul(e1.z, e2.x), fmul(e1.x, e2.z)),
                               fsub(fmul(e1.x, e2.y), fmul(e1.y, e2.x)));
  if (!(dot3p(g, no) > 0.f) || !(dot3p(g, nx) > 0.f) || !(dot3p(g, ny) > 0.f)) return false;
  if (angle_too_large(a.cos_triangle, e1, e2)) return false;
  if (angle_too_large(a.cos_triangle, sub3(py, px), sub3(po, px))) return false;
  return !angle_too_large(a.cos_triangle, sub3(po, py), sub3(px, py));
}

__global__ void __launch_bounds__(kBlock) k_simplify_edges(SimplifyArgs a) {
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < a.count; t += gridDim.x * blockDim.x) {
    const uint3 c = a.input[t];
    const u32 error = check_and_insert_triangle(a.rows + static_cast<size_t>(SM_ROW_RADIUS_SQUARED) * a.stride, a.n,
                                                c, a.edge_table, a.edge_mask);
    if (error) atomicOr(&a.counters->errors, error);
    a.tri[t] = c;
  }
}

__global__ void __launch_bounds__(kBlock) k_simplify_boundary(SimplifyArgs a) {
  const u32 edges = 3 * a.count;
  for (u32 e = blockIdx.x * blockDim.x + threadIdx.x; e < edges; e += gridDim.x * blockDim.x) {
    const uint3 c = a.tri[e / 3];
    const int s = e % 3;
    const u32 x = s == 0 ? c.x : (s == 1 ? c.y : c.z);
    const u32 y = s == 0 ? c.y : (s == 1 ? c.z : c.x);
    if (table_find(a.edge_table, a.edge_mask, edge_key(y, x)) == ~0ull) atomicAdd(&a.counters->boundary_edges, 1u);
  }
}

__global__ void __launch_bounds__(kBlock) k_simplify_corners(SimplifyArgs a) {
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < a.count; t += gridDim.x * blockDim.x) {
    const uint3 c = a.tri[t];
    if (c.x == kNone) continue;
    const u32 at = atomicAdd(&a.counters->corners, 3u);
    a.corners[at] = (static_cast<u64>(c.x) << 32) | t;
    a.corners[at + 1] = (static_cast<u64>(c.y) << 32) | t;
    a.corners[at + 2] = (static_cast<u64>(c.z) << 32) | t;
  }
}

__global__ void __launch_bounds__(kBlock) k_simplify_bounds(SimplifyArgs a) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.corner_count; i += gridDim.x * blockDim.x) {
    const u32 s = corner_slot(a.sorted[i]);
    if (i == 0 || corner_slot(a.sorted[i - 1]) != s) {
      a.begin[s] = i;
      a.mark[s] = kNoKey;
      a.vertices[atomicAdd(&a.counters->vertices, 1u)] = s;
    }
    if (i + 1 == a.corner_count || corner_slot(a.sorted[i + 1]) != s) a.end[s] = i + 1;
  }
}

__global__ void __launch_bounds__(kBlock) k_simplify_quadrics(SimplifyArgs a) {
  const u32 V = a.counters->vertices;
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < V; i += gridDim.x * blockDim.x) {
    const u32 u = a.vertices[i];
    double q[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) q[j] = 0.0;
    for (u32 c = a.begin[u]; c < a.end[u]; ++c) add_plane(a, a.tri[corner_position(a.sorted[c])], q);
    Quadric& out = a.quadric[u];
#pragma unroll
    for (int j = 0; j < 10; ++j) out.q[j] = q[j];
  }
}

// S3 and S4's marks for every listed slot.
__global__ void __launch_bounds__(kBlock) k_simplify_candidates(SimplifyArgs a) {
  const u32 V = a.counters->vertices;
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < V; i += gridDim.x * blockDim.x) {
    const u32 u = a.vertices[i];
    a.key[u] = kNoKey;
    const u32 first = a.begin[u];
    const int d = static_cast<int>(a.end[u] - first);
    if (d < 3 || d > kMaxValence) continue;
    // The fan walk: (u, from[k], to[k]) in ascending input position; ring[j] in fan order from the first.
    u32 from[kMaxValence], to[kMaxValence], ring[kMaxValence];
    for (int k = 0; k < d; ++k) after(a.tri[corner_position(a.sorted[first + k])], u, &from[k], &to[k]);
    ring[0] = from[0];
    int cur = 0;
    bool fan = true;
    for (int s = 1; s < d && fan; ++s) {
      int next = -1;
      for (int k = 0; k < d; ++k) if (from[k] == to[cur]) next = k;
      fan = next > 0;   // none: a boundary vertex; the first triangle again: more than one fan
      if (fan) { ring[s] = from[next]; cur = next; }
    }
    if (!fan || to[cur] != from[0]) continue;

    double qu[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) qu[j] = a.quadric[u].q[j];
    double best_cost = 0.0;
    u32 best_v = kNone;
    for (int k = 0; k < d; ++k) {
      const u32 v = ring[k];
      // (d) first: a collapse that cannot become best(u) needs no other test
      double q[10];
#pragma unroll
      for (int j = 0; j < 10; ++j) q[j] = __dadd_rn(qu[j], a.quadric[v].q[j]);
      const double3 pv = position_d(a, v);
      const double e = quadric_cost(q, pv.x, pv.y, pv.z);
      if (!isfinite(e)) continue;
      const double cost = e > 0.0 ? e : 0.0;
      if (!(cost <= a.max_cost)) continue;
      if (best_v != kNone && !(cost < best_cost || (cost == best_cost && v < best_v))) continue;
      // (b), with deg(v) >= its triangle count
      const u32 vfirst = a.begin[v];
      const int cv = static_cast<int>(a.end[v] - vfirst);
      if (cv + d > kMaxValence + 4) continue;
      const u32 o1 = ring[(k + d - 1) % d], o2 = ring[(k + 1) % d];
      u32 vfrom[kMaxValence + 1], vto[kMaxValence + 1];
      bool ok = true;
      for (int j = 0; j < cv && ok; ++j) {
        after(a.tri[corner_position(a.sorted[vfirst + j])], v, &vfrom[j], &vto[j]);
        // (a): a neighbour of v other than u, o1 and o2 is no neighbour of u
        for (int side = 0; side < 2 && ok; ++side) {
          const u32 x = side ? vto[j] : vfrom[j];
          if (x == u || x == o1 || x == o2) continue;
          for (int m = 0; m < d; ++m) ok = ok && ring[m] != x;
        }
      }
      if (!ok) continue;
      int deg_v = cv;   // the from corners are distinct; add the to corners that are none of them
      for (int j = 0; j < cv; ++j) {
        bool seen = false;
        for (int m = 0; m < cv; ++m) seen = seen || vfrom[m] == vto[j];
        deg_v += seen ? 0 : 1;
      }
      if (d + deg_v - 4 > kMaxValence) continue;
      // (c): the triangles of u without v, given to v
      for (int j = 0; j < d && ok; ++j) {
        const int j1 = j + 1 == d ? 0 : j + 1;
        if (j == k || j1 == k) continue;
        const u32 x = ring[j], y = ring[j1];
        for (int m = 0; m < cv && ok; ++m)
          ok = !((vfrom[m] == x && vto[m] == y) || (vfrom[m] == y && vto[m] == x));
        ok = ok && triangle_ok(a, v, x, y);
      }
      if (!ok) continue;
      best_cost = cost;
      best_v = v;
    }
    if (best_v == kNone) continue;
    float f = __double2float_rn(best_cost);
    if (!(f >= FLT_MIN)) f = 0.f;
    const u64 key = (static_cast<u64>(__float_as_uint(f)) << 32) | u;
    a.key[u] = key;
    a.best[u] = best_v;
    a.cost[u] = best_cost;
    atomicMin(reinterpret_cast<unsigned long long*>(a.mark + u), key);
    for (int j = 0; j < d; ++j) atomicMin(reinterpret_cast<unsigned long long*>(a.mark + ring[j]), key);
  }
}

// S4: u is selected iff it holds the mark of every slot of its closed neighbourhood.
__global__ void __launch_bounds__(kBlock) k_simplify_select(SimplifyArgs a) {
  const u32 V = a.counters->vertices;
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < V; i += gridDim.x * blockDim.x) {
    const u32 u = a.vertices[i];
    const u64 key = a.key[u];
    if (key == kNoKey) continue;
    bool selected = true;
    for (u32 c = a.begin[u]; c < a.end[u] && selected; ++c) {
      const uint3 t = a.tri[corner_position(a.sorted[c])];
      selected = a.mark[t.x] == key && a.mark[t.y] == key && a.mark[t.z] == key;
    }
    if (selected) a.selected[atomicAdd(&a.counters->selected, 1u)] = key;
  }
}

// S6 for the first apply_count keys of `apply`.
__global__ void __launch_bounds__(kBlock) k_simplify_apply(SimplifyArgs a) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.apply_count; i += gridDim.x * blockDim.x) {
    const u32 u = static_cast<u32>(a.apply[i]);
    const u32 v = a.best[u];
    for (u32 c = a.begin[u]; c < a.end[u]; ++c) {
      const u32 t = corner_position(a.sorted[c]);
      uint3 tri = a.tri[t];
      if (tri.x == v || tri.y == v || tri.z == v) {
        tri = make_uint3(kNone, kNone, kNone);
      } else {
        tri.x = tri.x == u ? v : tri.x;
        tri.y = tri.y == u ? v : tri.y;
        tri.z = tri.z == u ? v : tri.z;
      }
      a.tri[t] = tri;
    }
    Quadric& qv = a.quadric[v];
    const Quadric& qu = a.quadric[u];
#pragma unroll
    for (int j = 0; j < 10; ++j) qv.q[j] = __dadd_rn(qv.q[j], qu.q[j]);
    atomicMax(&a.counters->max_cost_bits, static_cast<unsigned long long>(__double_as_longlong(a.cost[u])));
  }
}

__device__ __forceinline__ u32 smallest(uint3 c) { return min(c.x, min(c.y, c.z)); }

__global__ void __launch_bounds__(kBlock) k_simplify_owners(SimplifyArgs a) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.corner_count; i += gridDim.x * blockDim.x) {
    const u64 k = a.sorted[i];
    a.counts[i] = corner_slot(k) == smallest(a.tri[corner_position(k)]) ? 1u : 0u;
  }
}

__global__ void __launch_bounds__(kBlock) k_simplify_write(SimplifyArgs a) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.corner_count; i += gridDim.x * blockDim.x) {
    const u32 at = a.counts[i];
    if (a.counts[i + 1] == at) continue;
    const uint3 c = a.tri[corner_position(a.sorted[i])];
    const u32 o = corner_slot(a.sorted[i]);
    a.out[at] = o == c.x ? c : (o == c.y ? make_uint3(c.y, c.z, c.x) : make_uint3(c.z, c.x, c.y));
  }
}

void FreeTriangleScratch(SimplifyScratch& s) {
  FreeAndClear(s.edge_table, s.tri, s.corners, s.sorted, s.counts, s.scan_sums);
  s.triangle_capacity = 0;
}

// Per-triangle scratch for `count` triangles (x 1.5 when it grows).
int EnsureTriangleScratch(SimplifyScratch& s, u64 count) {
  if (count <= s.triangle_capacity) return SM_OK;
  const u64 cap = GrownCapacity(count);
  FreeTriangleScratch(s);
  SM_CUDA(cudaMalloc(&s.edge_table, sizeof(u64) * PowerOfTwoAtLeast(6 * cap)));
  SM_CUDA(cudaMalloc(&s.tri, sizeof(uint3) * cap));
  SM_CUDA(cudaMalloc(&s.corners, sizeof(u64) * 3 * cap));
  SM_CUDA(cudaMalloc(&s.sorted, sizeof(u64) * 3 * cap));
  SM_CUDA(cudaMalloc(&s.counts, sizeof(u32) * (3 * cap + 1)));
  SM_CUDA(cudaMalloc(&s.scan_sums, sizeof(u32) * ScanTiles(3 * cap + 1)));
  s.triangle_capacity = cap;
  return SM_OK;
}

void FreeSlotScratch(SimplifyScratch& s) {
  FreeAndClear(s.quadric, s.begin, s.end, s.mark, s.key, s.best, s.cost, s.vertices, s.selected, s.selected_sorted);
  s.slot_capacity = 0;
}

// Per-slot scratch for `n` slots (x 1.5 when it grows).
int EnsureSlotScratch(SimplifyScratch& s, u32 n) {
  if (n <= s.slot_capacity) return SM_OK;
  const u64 cap = GrownCapacity(n);
  FreeSlotScratch(s);
  SM_CUDA(cudaMalloc(&s.quadric, sizeof(Quadric) * cap));
  SM_CUDA(cudaMalloc(&s.begin, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.end, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.mark, sizeof(u64) * cap));
  SM_CUDA(cudaMalloc(&s.key, sizeof(u64) * cap));
  SM_CUDA(cudaMalloc(&s.best, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.cost, sizeof(double) * cap));
  SM_CUDA(cudaMalloc(&s.vertices, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.selected, sizeof(u64) * cap));
  SM_CUDA(cudaMalloc(&s.selected_sorted, sizeof(u64) * cap));
  s.slot_capacity = static_cast<u32>(cap);
  return SM_OK;
}

void FreeSortScratch(SimplifyScratch& s) {
  FreeAndClear(s.sort_temp);
  s.sort_temp_bytes = 0;
}

// The sort's scratch for the corners of triangle_capacity triangles and the keys of slot_capacity slots.
int EnsureSortScratch(SimplifyScratch& s) {
  size_t corners = 0, keys = 0;
  SM_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, corners, static_cast<const u64*>(nullptr), static_cast<u64*>(nullptr),
                                         static_cast<int>(3 * s.triangle_capacity)));
  SM_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, keys, static_cast<const u64*>(nullptr), static_cast<u64*>(nullptr),
                                         static_cast<int>(s.slot_capacity)));
  const size_t bytes = std::max(corners, keys);
  if (bytes <= s.sort_temp_bytes) return SM_OK;
  FreeSortScratch(s);
  SM_CUDA(cudaMalloc(&s.sort_temp, bytes));
  s.sort_temp_bytes = bytes;
  return SM_OK;
}

int BitsFor(u32 n) {
  int b = 0;
  while (b < 32 && (n >> b) != 0) ++b;
  return b;
}

int Stop(const sm_simplify_params& p, u64 triangles, u64 rounds) {
  if (p.target_triangles > 0 && triangles <= p.target_triangles) return SM_SIMPLIFY_STOP_TARGET;
  if (rounds >= static_cast<u64>(p.max_rounds)) return SM_SIMPLIFY_STOP_MAX_ROUNDS;
  return 0;
}

}  // namespace

void FreeSimplifyBuffers(sm_reconstruction* r) {
  SimplifyScratch* s = r->simplify;
  if (!s) return;
  FreeTriangleScratch(*s);
  FreeSlotScratch(*s);
  FreeSortScratch(*s);
  FreeCounters(s->counters);
  delete s;
  r->simplify = nullptr;
}

}  // namespace smb

using namespace smb;

extern "C" {

void sm_default_simplify_params(sm_simplify_params* p) {
  p->target_triangles = 0;
  p->max_cost = 1e-6;
  p->max_angle_between_normals_deg = 90.0f;
  p->max_triangle_angle_deg = 170.0f;
  p->max_rounds = 64;
  p->reserved = 0;
}

int sm_mesh_simplify(sm_reconstruction* r, void* stream_v, const sm_simplify_params* params, const uint32_t* triangles,
                     uint64_t count, uint32_t* out, uint64_t capacity, sm_simplify_stats* stats) {
  if (!r || !params || !stats) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_mesh_simplify: null argument");
  auto bad = [](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (std::string("sm_mesh_simplify: ") + why).c_str()); };
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const sm_simplify_params& p = *params;
  *stats = sm_simplify_stats{};
  if (!(p.max_cost >= 0.0)) return bad("max_cost must be >= 0");
  if (!AngleInRange(p.max_angle_between_normals_deg) || !AngleInRange(p.max_triangle_angle_deg))
    return bad("angles must be in (0, 180] degrees");
  if (p.max_rounds < 0 || p.max_rounds > SM_SIMPLIFY_MAX_ROUNDS) return bad("max_rounds must be in [0, SM_SIMPLIFY_MAX_ROUNDS]");
  if (const char* why = TriangleListError(triangles, count, !out && capacity > 0 ? "out is NULL with a capacity > 0" : nullptr))
    return bad(why);
  if (count > 0 && capacity > 0 && Overlap(triangles, 12 * count, out, Bytes(capacity, 12)))
    return bad("out overlaps triangles");
  r->last_stream = stream;
  int status = FetchCounters(r, stream);
  if (status == SM_ERR_CUDA) return status;   // (a surfel-cap overflow of an earlier frame does not matter here)
  if (count == 0) {
    stats->stop_reason = Stop(p, 0, 0) ? Stop(p, 0, 0) : SM_SIMPLIFY_STOP_CONVERGED;
    return SM_OK;
  }
  const u32 n = r->host_counters->surfel_count[r->count_slot];

  if (!r->simplify) {   // published only with its counters, so a failed first call is retried whole
    CounterMirror<SimplifyCounters> counters;
    status = CreateCounters(counters);
    if (status != SM_OK) return status;
    r->simplify = new SimplifyScratch();
    r->simplify->counters = counters;
  }
  SimplifyScratch& s = *r->simplify;
  status = EnsureTriangleScratch(s, count);
  if (status == SM_OK) status = EnsureSlotScratch(s, std::max<u32>(n, 1));
  if (status == SM_OK) status = EnsureSortScratch(s);
  if (status != SM_OK) return status;

  SimplifyArgs a{};
  a.n = n;
  a.rows = r->d.surfels;
  a.stride = r->d.stride;
  a.input = reinterpret_cast<const uint3*>(triangles);
  a.count = static_cast<u32>(count);
  a.tri = s.tri;
  const u64 edge_slots = PowerOfTwoAtLeast(6 * count);   // a call uses and clears only what its input needs
  a.edge_table = s.edge_table;
  a.edge_mask = edge_slots - 1;
  a.corners = s.corners;
  a.sorted = s.sorted;
  a.begin = s.begin; a.end = s.end; a.vertices = s.vertices;
  a.quadric = s.quadric;
  a.mark = s.mark; a.key = s.key; a.best = s.best; a.cost = s.cost;
  a.selected = s.selected;
  a.counts = s.counts;
  a.out = reinterpret_cast<uint3*>(out);
  a.cos_normal = CosDegrees(p.max_angle_between_normals_deg);
  a.cos_triangle = CosDegrees(p.max_triangle_angle_deg);
  a.max_cost = p.max_cost;
  a.counters = s.counters.device;
  if (n > 0) {
    status = MirrorRegRecords(stream, r->d, n, r->sm_count);   // rows 3-5 <- the current smooth positions
    if (status != SM_OK) return status;
  }
  SimplifyCounters* c = s.counters.device;
  const SimplifyCounters& h = *s.counters.host;
  SM_CUDA(cudaMemsetAsync(c, 0, sizeof(SimplifyCounters), stream));
  SM_CUDA(cudaMemsetAsync(s.edge_table, 0xFF, sizeof(u64) * edge_slots, stream));
  { LaunchScope scope(stream, KID_SIMPLIFY_EDGES); LaunchKernel(k_simplify_edges, dim3(Grid(count, r->sm_count)), dim3(kBlock), 0, stream, a); }
  { LaunchScope scope(stream, KID_SIMPLIFY_EDGES); LaunchKernel(k_simplify_boundary, dim3(Grid(3 * count, r->sm_count)), dim3(kBlock), 0, stream, a); }
  status = ReadCounters(s.counters, stream);
  if (status != SM_OK) return status;
  if (const char* why = MeshInputError(h.errors)) return bad(why);
  const u64 boundary_edges = h.boundary_edges;

  const int sort_bits = 32 + BitsFor(n - 1);
  u64 T = count;
  // The corners of the current triangles sorted by (slot, position), each slot's range and the slot list.
  auto fans = [&]() -> int {
    SM_CUDA(cudaMemsetAsync(&c->corners, 0, 2 * sizeof(u32), stream));   // corners, vertices
    { LaunchScope scope(stream, KID_SIMPLIFY_FANS); LaunchKernel(k_simplify_corners, dim3(Grid(count, r->sm_count)), dim3(kBlock), 0, stream, a); }
    {
      LaunchScope scope(stream, KID_SIMPLIFY_SORT);
      size_t temp = s.sort_temp_bytes;
      SM_CUDA(cub::DeviceRadixSort::SortKeys(s.sort_temp, temp, static_cast<const u64*>(s.corners), s.sorted,
                                             static_cast<int>(3 * T), 0, sort_bits, stream));
    }
    a.corner_count = static_cast<u32>(3 * T);
    { LaunchScope scope(stream, KID_SIMPLIFY_FANS); LaunchKernel(k_simplify_bounds, dim3(Grid(3 * T, r->sm_count)), dim3(kBlock), 0, stream, a); }
    return SM_OK;
  };
  const int vertex_grid = Grid(std::min<u64>(n, 3 * count), r->sm_count);
  status = fans();
  if (status != SM_OK) return status;
  { LaunchScope scope(stream, KID_SIMPLIFY_QUADRICS); LaunchKernel(k_simplify_quadrics, dim3(vertex_grid), dim3(kBlock), 0, stream, a); }

  u64 rounds = 0, collapses = 0, vertices_in = 0;
  bool have_vertices_in = false;
  int reason = 0;
  while (!(reason = Stop(p, T, rounds))) {
    SM_CUDA(cudaMemsetAsync(&c->selected, 0, sizeof(u32), stream));
    { LaunchScope scope(stream, KID_SIMPLIFY_CANDIDATES); LaunchKernel(k_simplify_candidates, dim3(vertex_grid), dim3(kBlock), 0, stream, a); }
    { LaunchScope scope(stream, KID_SIMPLIFY_SELECT); LaunchKernel(k_simplify_select, dim3(vertex_grid), dim3(kBlock), 0, stream, a); }
    status = ReadCounters(s.counters, stream);
    if (status != SM_OK) return status;
    if (!have_vertices_in) { vertices_in = h.vertices; have_vertices_in = true; }
    const u64 selected = h.selected;
    if (selected == 0) { reason = SM_SIMPLIFY_STOP_CONVERGED; break; }
    u64 apply = selected;
    a.apply = s.selected;
    const bool budget = p.target_triangles > 0 && 2 * selected > T - p.target_triangles;   // (T > target here)
    if (budget) {
      apply = (T - p.target_triangles + 1) / 2;
      LaunchScope scope(stream, KID_SIMPLIFY_SORT);
      size_t temp = s.sort_temp_bytes;
      SM_CUDA(cub::DeviceRadixSort::SortKeys(s.sort_temp, temp, static_cast<const u64*>(s.selected), s.selected_sorted,
                                             static_cast<int>(selected), 0, 64, stream));
      a.apply = s.selected_sorted;
    }
    a.apply_count = static_cast<u32>(apply);
    { LaunchScope scope(stream, KID_SIMPLIFY_APPLY); LaunchKernel(k_simplify_apply, dim3(Grid(apply, r->sm_count)), dim3(kBlock), 0, stream, a); }
    T -= 2 * apply;
    collapses += apply;
    ++rounds;
    status = fans();
    if (status != SM_OK) return status;
    if (budget) { reason = SM_SIMPLIFY_STOP_TARGET; break; }
  }

  // S8: the owner corners in (slot, position) order give the output order.
  { LaunchScope scope(stream, KID_SIMPLIFY_WRITE); LaunchKernel(k_simplify_owners, dim3(Grid(3 * T, r->sm_count)), dim3(kBlock), 0, stream, a); }
  SM_CUDA(cudaMemsetAsync(s.counts + 3 * T, 0, sizeof(u32), stream));
  ScanInPlace(stream, s.counts, static_cast<u32>(3 * T + 1), s.scan_sums, KID_SIMPLIFY_SCAN);
  status = ReadCounters(s.counters, stream);
  if (status != SM_OK) return status;
  stats->triangles_in = count;
  stats->triangles_out = T;
  stats->vertices_in = have_vertices_in ? vertices_in : h.vertices;
  stats->vertices_out = h.vertices;
  stats->collapses = collapses;
  stats->rounds = rounds;
  stats->boundary_edges = boundary_edges;
  std::memcpy(&stats->max_cost_applied, &h.max_cost_bits, sizeof(double));
  stats->stop_reason = reason;
  if (capacity < T) return TriangleCapacityError("sm_mesh_simplify", T, capacity);
  if (T > 0) {
    LaunchScope scope(stream, KID_SIMPLIFY_WRITE);
    LaunchKernel(k_simplify_write, dim3(Grid(3 * T, r->sm_count)), dim3(kBlock), 0, stream, a);
  }
  return CheckLaunch("simplify");
}

}  // extern "C"
