// holes.cu — sm_mesh_fill_holes (DESIGN.md section 5.12): the small boundary loops of a triangle mesh filled by a
// minimum-area triangulation. The rules H1-H7, step by step, are in include/surfel_b200.h.
//
// Launches on the caller's stream (the call synchronises three times: surfels_size(), the hole edge count and the
// input checks, the triangle count):
//   k_hole_edges     one thread per triangle: checks its corners and inserts its three directed edges into an
//                    open-addressed table of 64-bit keys (tail << 32 | head); an edge found there already is a
//                    duplicate;
//   k_hole_boundary  one thread per directed edge: looks its reverse up and appends the hole edges (H1);
//   (CUB radix sort of the hole edges: the order of H1, and each vertex's range of outgoing hole edges)
//   k_hole_walk      one thread per hole edge: follows successors (H2) for at most K steps, gives up as soon as
//                    it meets a smaller edge; the owner of a loop (H3) runs the dynamic programme of H5 in local
//                    memory, stores its loop and triangles and marks its diagonals in a table keyed by the
//                    unordered pair, with the smallest and largest owner that proposed each;
//   k_hole_conflict  one thread per hole edge: an owner whose diagonals were all proposed by it alone keeps its
//                    k - 2 triangles (H6), every other edge counts 0;
//   (the three-launch exclusive scan of knn.cu over the counts)
//   k_hole_write     one thread per hole edge: the owner writes its triangles at its scanned offset (H7).

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <string>

#include "sm_handle.cuh"
#include "sm_knn.cuh"
#include "sm_mesh_edges.cuh"

namespace smb {

namespace {

constexpr int kMaxHole = SM_MESH_MAX_HOLE;
constexpr u32 kNone = 0xFFFFFFFFu;

}  // namespace

struct HoleCounters {
  u32 errors;
  u32 hole_edges;
  unsigned long long loops_found, loops_rejected, loops_conflicting, loops_filled, filled_edges;
  u32 triangles;   // copied from the end of the scanned counts
};

// The scratch of sm_mesh_fill_holes: per input triangle (the edge table, the unsorted hole edges) and per hole edge.
struct HoleScratch {
  CounterMirror<HoleCounters> counters;
  u64* edge_table = nullptr; u64 edge_table_size = 0;   // a power of two >= 6 x triangle_capacity
  u64* unsorted = nullptr; u64 unsorted_capacity = 0;   // 3 x triangles
  u64 triangle_capacity = 0;
  u64* sorted = nullptr;
  void* sort_temp = nullptr; size_t sort_temp_bytes = 0;
  u32* loop_vertices = nullptr;   // [hole edge][kMaxHole]: L of the loop the edge owns
  u16* loop_triangles = nullptr;  // [hole edge][kMaxHole - 2]: i | j << 4 | m << 8
  u8* loop_length = nullptr;      // k of a loop the edge owns and that has a triangulation, else 0
  u32* counts = nullptr;          // [hole edges + 1]: triangles, then (scanned) offsets
  u32* scan_sums = nullptr;
  u64* diag_keys = nullptr; u32* diag_lo = nullptr; u32* diag_hi = nullptr; u64 diag_size = 0;   // >= 2 x hole_capacity
  u32 hole_capacity = 0;
};

namespace {

struct HoleArgs {
  u32 n;                       // surfels_size()
  const float* rows;
  size_t stride;
  const uint3* triangles;
  u32 count;
  int max_edges;               // K
  float cos_normal, cos_triangle;
  u64* edge_table; u64 edge_mask;
  u64* unsorted;
  const u64* sorted; u32 hole_edges;
  u32* loop_vertices; u16* loop_triangles; u8* loop_length;
  u32* counts;
  u64* diag_keys; u32* diag_lo; u32* diag_hi; u64 diag_mask;
  uint3* fill;
  HoleCounters* counters;
};

__device__ __forceinline__ float cross2(float2 a, float2 b) { return fsub(fmul(a.x, b.y), fmul(a.y, b.x)); }
__device__ __forceinline__ float dot2(float2 a, float2 b) { return fadd(fmul(a.x, b.x), fmul(a.y, b.y)); }

__device__ __forceinline__ float3 position(const HoleArgs& a, u32 i) { return slot_position(a.rows, a.stride, i); }

__device__ __forceinline__ bool unit_normal(const HoleArgs& a, u32 i, float3* out) {
  return slot_unit_normal(a.rows, a.stride, i, out);
}

__device__ __forceinline__ bool is_edge(const HoleArgs& a, u32 tail, u32 head) {
  return table_find(a.edge_table, a.edge_mask, edge_key(tail, head)) != ~0ull;
}

__global__ void __launch_bounds__(kBlock) k_hole_edges(HoleArgs a) {
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < a.count; t += gridDim.x * blockDim.x) {
    const u32 error = check_and_insert_triangle(a.rows + static_cast<size_t>(SM_ROW_RADIUS_SQUARED) * a.stride, a.n,
                                                a.triangles[t], a.edge_table, a.edge_mask);
    if (error) atomicOr(&a.counters->errors, error);
  }
}

// H1: the reverse of every input edge (a, b) whose reverse is not an input edge.
__global__ void __launch_bounds__(kBlock) k_hole_boundary(HoleArgs a) {
  const u32 edges = 3 * a.count;
  for (u32 e = blockIdx.x * blockDim.x + threadIdx.x; e < edges; e += gridDim.x * blockDim.x) {
    const uint3 c = a.triangles[e / 3];
    const int s = e % 3;
    const u32 x = s == 0 ? c.x : (s == 1 ? c.y : c.z);
    const u32 y = s == 0 ? c.y : (s == 1 ? c.z : c.x);
    if (!is_edge(a, y, x)) a.unsorted[atomicAdd(&a.counters->hole_edges, 1u)] = edge_key(y, x);
  }
}

// The first sorted hole edge >= key.
__device__ __forceinline__ u32 lower_bound(const HoleArgs& a, u64 key) {
  u32 lo = 0, hi = a.hole_edges;
  while (lo < hi) {
    const u32 mid = lo + (hi - lo) / 2;
    if (a.sorted[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// H2: 0 or 1 for the half of q_w around q_u, -1 when it has none.
__device__ __forceinline__ int half_of(float2 qu, float2 qw) {
  const float c = cross2(qu, qw);
  if (c < 0.f) return 0;
  if (c > 0.f || (c == 0.f && dot2(qu, qw) < 0.f)) return 1;
  return -1;   // (also when c is NaN)
}

// H2: the successor (a sorted index) of hole edge (u, v), or kNone.
__device__ u32 successor(const HoleArgs& a, u32 u, u32 v) {
  const u32 first = lower_bound(a, edge_key(v, 0));
  u32 end = first;
  while (end < a.hole_edges && tail_of(a.sorted[end]) == v) ++end;
  if (end == first) return kNone;
  if (end == first + 1) return first;
  float3 n;
  if (!unit_normal(a, v, &n)) return kNone;
  // Tangent basis of rule 2 (Duff et al. 2017).
  const float sign = copysignf(1.f, n.z);
  const float bf = __fdiv_rn(-1.f, fadd(sign, n.z));
  const float bb = fmul(fmul(n.x, n.y), bf);
  const float3 t = make_float3(fadd(1.f, fmul(fmul(fmul(sign, n.x), n.x), bf)), fmul(sign, bb), -fmul(sign, n.x));
  const float3 s = make_float3(bb, fadd(sign, fmul(fmul(n.y, n.y), bf)), -n.y);
  const float3 pv = position(a, v);
  auto project = [&](u32 x) {
    const float3 d = sub3(position(a, x), pv);
    return make_float2(dot3p(d, t), dot3p(d, s));
  };
  const float2 qu = project(u);
  // Pass 1: the candidate no earlier one comes after; pass 2: it comes before every other.
  u32 best = kNone;
  float2 qb = make_float2(0.f, 0.f);
  int hb = 0;
  for (u32 e = first; e < end; ++e) {
    const float2 q = project(head_of(a.sorted[e]));
    const int h = half_of(qu, q);
    if (h < 0) return kNone;
    if (best == kNone || h < hb || (h == hb && cross2(q, qb) < 0.f)) { best = e; qb = q; hb = h; }
  }
  for (u32 e = first; e < end; ++e) {
    if (e == best) continue;
    const float2 q = project(head_of(a.sorted[e]));
    const int h = half_of(qu, q);
    if (!(hb < h || (hb == h && cross2(qb, q) < 0.f))) return kNone;
  }
  return best;
}

// H4's geometric part for the triangle (x0, x1, x2) (loop order): its weight w, or +inf when it is invalid.
__device__ float triangle_weight(const HoleArgs& a, const u32* slot, const float3* p, const float3* n, int i0, int i1,
                                 int i2) {
  int o = i0, x = i1, y = i2;
  if (slot[i1] < slot[o] && slot[i1] < slot[i2]) { o = i1; x = i2; y = i0; }
  else if (slot[i2] < slot[o] && slot[i2] < slot[i1]) { o = i2; x = i0; y = i1; }
  const float3 e1 = sub3(p[x], p[o]), e2 = sub3(p[y], p[o]);
  const float3 g = make_float3(fsub(fmul(e1.y, e2.z), fmul(e1.z, e2.y)), fsub(fmul(e1.z, e2.x), fmul(e1.x, e2.z)),
                               fsub(fmul(e1.x, e2.y), fmul(e1.y, e2.x)));
  const float inf = __int_as_float(0x7F800000);
  if (!(dot3p(g, n[o]) > 0.f) || !(dot3p(g, n[x]) > 0.f) || !(dot3p(g, n[y]) > 0.f)) return inf;
  if (angle_too_large(a.cos_triangle, e1, e2)) return inf;
  if (angle_too_large(a.cos_triangle, sub3(p[y], p[x]), sub3(p[o], p[x]))) return inf;
  if (angle_too_large(a.cos_triangle, sub3(p[o], p[y]), sub3(p[x], p[y]))) return inf;
  return __fsqrt_rn(dot3p(g, g));
}

__device__ __forceinline__ u64 pair_key(u32 x, u32 y) { return x < y ? edge_key(x, y) : edge_key(y, x); }

// H3 and H5 for hole edge h: a thread that owns a loop with a triangulation stores it and marks its diagonals.
__global__ void __launch_bounds__(kBlock) k_hole_walk(HoleArgs a) {
  for (u32 h = blockIdx.x * blockDim.x + threadIdx.x; h < a.hole_edges; h += gridDim.x * blockDim.x) {
    a.loop_length[h] = 0;
    u32 L[kMaxHole + 1];
    const u64 key = a.sorted[h];
    L[0] = tail_of(key);
    L[1] = head_of(key);
    u32 cur = h;
    int k = 0;
    for (int s = 1; s <= a.max_edges; ++s) {
      const u32 next = successor(a, tail_of(a.sorted[cur]), head_of(a.sorted[cur]));
      if (next == kNone || next < h) break;   // an open chain, or an edge of the loop is smaller than h
      if (next == h) { k = s; break; }
      if (s == a.max_edges) break;
      L[s + 1] = head_of(a.sorted[next]);
      cur = next;
    }
    if (k < 3) continue;   // (k is 0, or at least 3: a hole edge's reverse is an input edge)
    bool distinct = true;
    for (int i = 1; i < k; ++i)
      for (int j = 0; j < i; ++j) distinct = distinct && L[i] != L[j];
    if (!distinct) continue;
    atomicAdd(&a.counters->loops_found, 1ull);

    float3 P[kMaxHole], N[kMaxHole];
    bool normal_ok = true;
    for (int i = 0; i < k; ++i) {
      P[i] = position(a, L[i]);
      normal_ok = unit_normal(a, L[i], &N[i]) && normal_ok;
    }
    // ok[i] bit m: the pair (i, m) may be a side of a triangle (normals, and a diagonal not an input edge).
    u32 ok[kMaxHole];
    for (int i = 0; i < k; ++i) {
      ok[i] = 0;
      for (int m = i + 1; m < k && normal_ok; ++m) {
        const bool loop_edge = m == i + 1 || (i == 0 && m == k - 1);
        bool pass = dot3p(N[i], N[m]) >= a.cos_normal;
        if (pass && !loop_edge) pass = !is_edge(a, L[i], L[m]) && !is_edge(a, L[m], L[i]);
        if (pass) ok[i] |= 1u << m;
      }
    }
    const float inf = __int_as_float(0x7F800000);
    float W[kMaxHole][kMaxHole];
    u8 J[kMaxHole][kMaxHole];
    for (int i = 0; i + 1 < k; ++i) W[i][i + 1] = 0.f;
    for (int d = 2; d < k; ++d) {
      for (int i = 0; i + d < k; ++i) {
        const int m = i + d;
        float best = inf;
        int bj = i + 1;
        if (ok[i] >> m & 1) {
          for (int j = i + 1; j < m; ++j) {
            if (!(ok[i] >> j & 1) || !(ok[j] >> m & 1)) continue;
            const float left = fadd(W[i][j], W[j][m]);
            if (!(left < inf)) continue;
            const float c = fadd(left, triangle_weight(a, L, P, N, i, j, m));
            if (c < best) { best = c; bj = j; }
          }
        }
        W[i][m] = best;
        J[i][m] = static_cast<u8>(bj);
      }
    }
    if (!(W[0][k - 1] < inf)) {
      atomicAdd(&a.counters->loops_rejected, 1ull);
      continue;
    }
    // The tree in pre-order; the diagonals into the table.
    u32* vertices = a.loop_vertices + static_cast<size_t>(h) * kMaxHole;
    u16* out = a.loop_triangles + static_cast<size_t>(h) * (kMaxHole - 2);
    for (int i = 0; i < k; ++i) vertices[i] = L[i];
    u8 stack[kMaxHole][2];
    int top = 0, written = 0;
    stack[top][0] = 0; stack[top][1] = static_cast<u8>(k - 1); ++top;
    while (top > 0) {
      --top;
      const int i = stack[top][0], m = stack[top][1];
      if (i != 0 || m != k - 1) {
        u64 slot;
        table_insert(a.diag_keys, a.diag_mask, pair_key(L[i], L[m]), &slot);
        atomicMin(a.diag_lo + slot, h);
        atomicMax(a.diag_hi + slot, h);
      }
      const int j = J[i][m];
      out[written++] = static_cast<u16>(i | j << 4 | m << 8);
      if (m - j >= 2) { stack[top][0] = static_cast<u8>(j); stack[top][1] = static_cast<u8>(m); ++top; }
      if (j - i >= 2) { stack[top][0] = static_cast<u8>(i); stack[top][1] = static_cast<u8>(j); ++top; }
    }
    a.loop_length[h] = static_cast<u8>(k);
  }
}

// H6: the triangle count of every hole edge (k - 2 for an owner whose diagonals nobody else proposed).
__global__ void __launch_bounds__(kBlock) k_hole_conflict(HoleArgs a) {
  for (u32 h = blockIdx.x * blockDim.x + threadIdx.x; h < a.hole_edges; h += gridDim.x * blockDim.x) {
    const int k = a.loop_length[h];
    u32 triangles = 0;
    if (k) {
      const u32* L = a.loop_vertices + static_cast<size_t>(h) * kMaxHole;
      const u16* tri = a.loop_triangles + static_cast<size_t>(h) * (kMaxHole - 2);
      bool alone = true;
      for (int t = 0; t < k - 2 && alone; ++t) {
        const int i = tri[t] & 15, m = tri[t] >> 8 & 15;   // every diagonal is the (i, m) of some node but the root
        if (t == 0) continue;
        const u64 slot = table_find(a.diag_keys, a.diag_mask, pair_key(L[i], L[m]));
        alone = a.diag_lo[slot] == a.diag_hi[slot];
      }
      if (alone) {
        triangles = k - 2;
        atomicAdd(&a.counters->loops_filled, 1ull);
        atomicAdd(&a.counters->filled_edges, static_cast<unsigned long long>(k));
      } else {
        atomicAdd(&a.counters->loops_conflicting, 1ull);
      }
    }
    a.counts[h] = triangles;
  }
}

__global__ void __launch_bounds__(kBlock) k_hole_write(HoleArgs a) {
  for (u32 h = blockIdx.x * blockDim.x + threadIdx.x; h < a.hole_edges; h += gridDim.x * blockDim.x) {
    u32 out = a.counts[h];
    const u32 end = a.counts[h + 1];
    const u32* L = a.loop_vertices + static_cast<size_t>(h) * kMaxHole;
    const u16* tri = a.loop_triangles + static_cast<size_t>(h) * (kMaxHole - 2);
    for (int t = 0; out < end; ++t, ++out) {
      const u32 x = L[tri[t] & 15], y = L[tri[t] >> 4 & 15], z = L[tri[t] >> 8 & 15];
      a.fill[out] = (x < y && x < z) ? make_uint3(x, y, z) : (y < z ? make_uint3(y, z, x) : make_uint3(z, x, y));
    }
  }
}

void FreeTriangleScratch(HoleScratch& s) {
  FreeAndClear(s.edge_table, s.unsorted);
  s.triangle_capacity = 0;
}

// Per-triangle scratch for `count` triangles (x 1.5 when it grows).
int EnsureTriangleScratch(HoleScratch& s, u64 count) {
  if (count <= s.triangle_capacity) return SM_OK;
  const u64 cap = GrownCapacity(count);
  FreeTriangleScratch(s);
  const u64 table = PowerOfTwoAtLeast(6 * cap);
  SM_CUDA(cudaMalloc(&s.edge_table, sizeof(u64) * table));
  SM_CUDA(cudaMalloc(&s.unsorted, sizeof(u64) * 3 * cap));
  s.edge_table_size = table;
  s.triangle_capacity = cap;
  return SM_OK;
}

void FreeHoleScratch(HoleScratch& s) {
  FreeAndClear(s.sorted, s.sort_temp, s.loop_vertices, s.loop_triangles, s.loop_length, s.counts, s.scan_sums,
               s.diag_keys, s.diag_lo, s.diag_hi);
  s.hole_capacity = 0;
}

// Per-hole-edge scratch for `edges` hole edges (x 1.5 when it grows).
int EnsureHoleScratch(HoleScratch& s, u32 edges) {
  if (edges <= s.hole_capacity) return SM_OK;
  const u64 cap = GrownCapacity(edges);
  FreeHoleScratch(s);
  size_t temp = 0;
  SM_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, temp, static_cast<const u64*>(nullptr), static_cast<u64*>(nullptr),
                                         static_cast<int>(cap)));
  const u64 diag = PowerOfTwoAtLeast(2 * cap);
  SM_CUDA(cudaMalloc(&s.sorted, sizeof(u64) * cap));
  SM_CUDA(cudaMalloc(&s.sort_temp, temp));
  SM_CUDA(cudaMalloc(&s.loop_vertices, sizeof(u32) * kMaxHole * cap));
  SM_CUDA(cudaMalloc(&s.loop_triangles, sizeof(u16) * (kMaxHole - 2) * cap));
  SM_CUDA(cudaMalloc(&s.loop_length, cap));
  SM_CUDA(cudaMalloc(&s.counts, sizeof(u32) * (cap + 1)));
  SM_CUDA(cudaMalloc(&s.scan_sums, sizeof(u32) * ScanTiles(cap + 1)));
  SM_CUDA(cudaMalloc(&s.diag_keys, sizeof(u64) * diag));
  SM_CUDA(cudaMalloc(&s.diag_lo, sizeof(u32) * diag));
  SM_CUDA(cudaMalloc(&s.diag_hi, sizeof(u32) * diag));
  s.sort_temp_bytes = temp;
  s.diag_size = diag;
  s.hole_capacity = static_cast<u32>(cap);
  return SM_OK;
}

}  // namespace

void FreeHoleBuffers(sm_reconstruction* r) {
  HoleScratch* s = r->holes;
  if (!s) return;
  FreeTriangleScratch(*s);
  FreeHoleScratch(*s);
  FreeCounters(s->counters);
  delete s;
  r->holes = nullptr;
}

}  // namespace smb

using namespace smb;

extern "C" {

void sm_default_hole_params(sm_hole_params* p) {
  p->max_hole_edges = 8;
  p->max_angle_between_normals_deg = 90.0f;
  p->max_triangle_angle_deg = 180.0f;
}

int sm_mesh_fill_holes(sm_reconstruction* r, void* stream_v, const sm_hole_params* params, const uint32_t* triangles,
                       uint64_t count, uint32_t* fill, uint64_t capacity, sm_hole_stats* stats) {
  if (!r || !params || !stats) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_mesh_fill_holes: null argument");
  auto bad = [](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (std::string("sm_mesh_fill_holes: ") + why).c_str()); };
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const sm_hole_params& p = *params;
  *stats = sm_hole_stats{};
  if (p.max_hole_edges < 3 || p.max_hole_edges > kMaxHole) return bad("max_hole_edges must be in [3, SM_MESH_MAX_HOLE]");
  if (!AngleInRange(p.max_angle_between_normals_deg) || !AngleInRange(p.max_triangle_angle_deg))
    return bad("angles must be in (0, 180] degrees");
  if (const char* why = TriangleListError(triangles, count, !fill && capacity > 0 ? "fill is NULL with a capacity > 0" : nullptr))
    return bad(why);
  r->last_stream = stream;
  int status = FetchCounters(r, stream);
  if (status == SM_ERR_CUDA) return status;   // (a surfel-cap overflow of an earlier frame does not matter here)
  if (count == 0) return SM_OK;
  const u32 n = r->host_counters->surfel_count[r->count_slot];

  if (!r->holes) {   // published only with its counters, so a failed first call is retried whole
    CounterMirror<HoleCounters> counters;
    status = CreateCounters(counters);
    if (status != SM_OK) return status;
    r->holes = new HoleScratch();
    r->holes->counters = counters;
  }
  HoleScratch& s = *r->holes;
  status = EnsureTriangleScratch(s, count);
  if (status != SM_OK) return status;

  HoleArgs a{};
  a.n = n;
  a.rows = r->d.surfels;
  a.stride = r->d.stride;
  a.triangles = reinterpret_cast<const uint3*>(triangles);
  a.count = static_cast<u32>(count);
  a.max_edges = p.max_hole_edges;
  a.cos_normal = CosDegrees(p.max_angle_between_normals_deg);
  a.cos_triangle = CosDegrees(p.max_triangle_angle_deg);
  // Each call uses (and clears) only the part of the tables its own input needs: a load of 1/4 to 1/2.
  const u64 edge_slots = PowerOfTwoAtLeast(6 * count);
  a.edge_table = s.edge_table;
  a.edge_mask = edge_slots - 1;
  a.unsorted = s.unsorted;
  a.fill = reinterpret_cast<uint3*>(fill);
  a.counters = s.counters.device;
  if (n > 0) {
    status = MirrorRegRecords(stream, r->d, n, r->sm_count);   // rows 3-5 <- the current smooth positions
    if (status != SM_OK) return status;
  }
  SM_CUDA(cudaMemsetAsync(s.counters.device, 0, sizeof(HoleCounters), stream));
  SM_CUDA(cudaMemsetAsync(s.edge_table, 0xFF, sizeof(u64) * edge_slots, stream));
  { LaunchScope scope(stream, KID_HOLE_EDGES); LaunchKernel(k_hole_edges, dim3(Grid(count, r->sm_count)), dim3(kBlock), 0, stream, a); }
  { LaunchScope scope(stream, KID_HOLE_BOUNDARY); LaunchKernel(k_hole_boundary, dim3(Grid(3 * count, r->sm_count)), dim3(kBlock), 0, stream, a); }
  status = ReadCounters(s.counters, stream);
  if (status != SM_OK) return status;
  const HoleCounters& c = *s.counters.host;
  if (const char* why = MeshInputError(c.errors)) return bad(why);
  const u32 H = c.hole_edges;
  stats->boundary_edges = H;
  stats->boundary_edges_after = H;
  if (H == 0) return CheckLaunch("fill holes");

  status = EnsureHoleScratch(s, H);
  if (status != SM_OK) return status;
  a.sorted = s.sorted;
  a.hole_edges = H;
  a.loop_vertices = s.loop_vertices;
  a.loop_triangles = s.loop_triangles;
  a.loop_length = s.loop_length;
  a.counts = s.counts;
  a.diag_keys = s.diag_keys;
  a.diag_lo = s.diag_lo;
  a.diag_hi = s.diag_hi;
  const u64 diag_slots = PowerOfTwoAtLeast(2 * static_cast<u64>(H));
  a.diag_mask = diag_slots - 1;
  {
    LaunchScope scope(stream, KID_HOLE_SORT);
    size_t temp = s.sort_temp_bytes;
    SM_CUDA(cub::DeviceRadixSort::SortKeys(s.sort_temp, temp, static_cast<const u64*>(s.unsorted), s.sorted,
                                           static_cast<int>(H), 0, 64, stream));
  }
  SM_CUDA(cudaMemsetAsync(s.diag_keys, 0xFF, sizeof(u64) * diag_slots, stream));
  SM_CUDA(cudaMemsetAsync(s.diag_lo, 0xFF, sizeof(u32) * diag_slots, stream));
  SM_CUDA(cudaMemsetAsync(s.diag_hi, 0, sizeof(u32) * diag_slots, stream));
  SM_CUDA(cudaMemsetAsync(s.counts + H, 0, sizeof(u32), stream));
  const int grid = Grid(H, r->sm_count);
  { LaunchScope scope(stream, KID_HOLE_WALK); LaunchKernel(k_hole_walk, dim3(grid), dim3(kBlock), 0, stream, a); }
  { LaunchScope scope(stream, KID_HOLE_CONFLICT); LaunchKernel(k_hole_conflict, dim3(grid), dim3(kBlock), 0, stream, a); }
  ScanInPlace(stream, s.counts, H + 1, s.scan_sums, KID_HOLE_SCAN);
  SM_CUDA(cudaMemcpyAsync(&s.counters.device->triangles, s.counts + H, sizeof(u32), cudaMemcpyDeviceToDevice, stream));
  status = ReadCounters(s.counters, stream);
  if (status != SM_OK) return status;
  stats->loops_found = c.loops_found;
  stats->loops_filled = c.loops_filled;
  stats->loops_rejected = c.loops_rejected;
  stats->loops_conflicting = c.loops_conflicting;
  stats->triangles_added = c.triangles;
  stats->boundary_edges_after = H - c.filled_edges;
  if (capacity < stats->triangles_added) return TriangleCapacityError("sm_mesh_fill_holes", stats->triangles_added, capacity);
  if (stats->triangles_added > 0) {
    LaunchScope scope(stream, KID_HOLE_WRITE);
    LaunchKernel(k_hole_write, dim3(grid), dim3(kBlock), 0, stream, a);
  }
  return CheckLaunch("fill holes");
}

}  // extern "C"
