// components.cu — sm_mesh_components (DESIGN.md section 5.16): the connected pieces of a triangle list (triangles that
// share an undirected edge), numbered by their smallest triangle position, each with its triangle count, area and
// bounds, and the triangles of the pieces the thresholds keep. The rules C1-C7 are in include/surfel_b200.h.
//
// Launches on the caller's stream:
//   k_cc_edges    one thread per triangle: the input checks (C1), its union-find parent set to itself, and its three
//                 undirected edge keys into the hash table, whose owner takes the smallest triangle position on it;
//   k_cc_hook     one thread per triangle: union with the owner of each of its edges (lock-free union-find with path
//                 halving, the larger root always linked under the smaller), so each root ends as its piece's
//                 smallest triangle position, the key of C3;
//   k_cc_number   one thread per triangle: its parent set to its root, 1 where it is a root;
//   (the three-launch exclusive scan of knn.cu over those flags: the numbers; synchronisation: the input checks and
//    the piece count)
//   k_cc_sums     one thread per triangle: count, Q (C4) and bounds (C5) into its piece with integer and ordered-int
//                 atomics, reduced within the warp first where all its lanes are one piece; each root names its piece's
//                 first triangle;
//   k_cc_largest  one thread per piece: the largest Q (and, when keep_largest limits, the sort keys);
//   k_cc_rank0    one thread per piece: the smallest number with the largest Q, the rank-0 piece;
//   (when keep_largest limits: CUB radix sort of (~Q, number); k_cc_rank marks the first keep_largest pieces)
//   k_cc_keep     one thread per piece: C6, the kept count and the rank-0 piece's stats;
//   k_cc_flags    one thread per triangle: 1 where its piece is kept;
//   (the scan again: the output positions; synchronisation: the end)
//   k_cc_write    one thread per triangle: out and labels;
//   k_cc_table    one thread per piece: the table.

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <string>

#include "sm_handle.cuh"
#include "sm_knn.cuh"
#include "sm_mesh_edges.cuh"

namespace smb {

namespace {

constexpr unsigned long long kMaxAreaUnits = 1ull << 36;   // C4's cap of q_t
constexpr unsigned kFullWarp = 0xFFFFFFFFu;

}  // namespace

struct ComponentCounters {
  u32 errors;
  u32 components;        // the root flags' total
  u32 triangles_out;     // the keep flags' total
  u32 kept;
  u32 largest;           // the number of the rank-0 piece
  u32 pad;
  unsigned long long max_q;
  unsigned long long largest_triangles, largest_q;
};

// The scratch of sm_mesh_components: per triangle and per piece.
struct ComponentScratch {
  CounterMirror<ComponentCounters> counters;
  u64 triangle_capacity = 0;
  u64* edge_keys = nullptr;       // a power of two >= 4 x triangle_capacity
  u32* edge_owner = nullptr;      // the smallest triangle position on the edge
  u32* parent = nullptr;          // union-find, then the root
  u32* roots = nullptr;           // + 1: root flags, then (scanned) the piece numbers
  u32* keep = nullptr;            // + 1: keep flags, then (scanned) the output positions
  u32* scan_sums = nullptr;
  u64 piece_capacity = 0;
  u32* count = nullptr;
  unsigned long long* q = nullptr;
  u32* lo = nullptr; u32* hi = nullptr;   // 3 x: the bounds as ordered ints
  u32* first = nullptr;
  u32* kept = nullptr;            // the rank marks, then C6
  u64* sort_keys = nullptr; u64* sorted_keys = nullptr;
  u32* sort_values = nullptr; u32* sorted_values = nullptr;
  void* sort_temp = nullptr; size_t sort_temp_bytes = 0;
};

namespace {

struct ComponentArgs {
  u32 n;                          // surfels_size()
  const float* radius_squared;    // row 7
  const float4* smooth;
  const uint3* input;
  u32 count;
  u64* edge_keys; u32* edge_owner; u64 edge_mask;
  u32* parent; u32* roots; u32* keep;
  u32 pieces;
  u32* count_of; unsigned long long* q; u32* lo; u32* hi; u32* first; u32* kept;
  u64* sort_keys; u32* sort_values; const u32* sorted_values;
  u32 rank_limit;                 // keep_largest when it limits (below the piece count), else 0
  unsigned long long min_triangles, min_q;
  uint3* out; int32_t* labels; sm_mesh_component* table;
  ComponentCounters* counters;
};

// IEEE totalOrder of floats as the order of u32 keys, and back.
__device__ __forceinline__ u32 ordered(float f) {
  const u32 b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float unordered(u32 k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

__device__ __forceinline__ float3 corner(const ComponentArgs& a, u32 i) {
  const float4 p = a.smooth[i];
  return make_float3(p.x, p.y, p.z);
}

// C4: q_t of the triangle with corners (pa, pb, pc).
__device__ __forceinline__ unsigned long long area_units(float3 pa, float3 pb, float3 pc) {
  const double ax = pa.x, ay = pa.y, az = pa.z;
  const double e1x = __dsub_rn(pb.x, ax), e1y = __dsub_rn(pb.y, ay), e1z = __dsub_rn(pb.z, az);
  const double e2x = __dsub_rn(pc.x, ax), e2y = __dsub_rn(pc.y, ay), e2z = __dsub_rn(pc.z, az);
  const double gx = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
  const double gy = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
  const double gz = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
  const double gg = __dadd_rn(__dadd_rn(__dmul_rn(gx, gx), __dmul_rn(gy, gy)), __dmul_rn(gz, gz));
  const double area = __dmul_rn(0.5, __dsqrt_rn(gg));
  if (!isfinite(area)) return 0;
  const double scaled = __dmul_rn(area, 0x1p30);
  return scaled >= 0x1p36 ? kMaxAreaUnits : __double2ull_rn(scaled);
}

// The root of x; halves the path it walks. Parents only ever move to a smaller position, so a stale read is still an
// ancestor, and the loads bypass L1 so that a spinning thread sees other threads' links.
__device__ __forceinline__ u32 find_root(u32* parent, u32 x) {
  u32 p = __ldcg(parent + x);
  while (p != x) {
    const u32 g = __ldcg(parent + p);
    if (g != p) atomicCAS(parent + x, p, g);
    x = g;
    p = __ldcg(parent + x);
  }
  return x;
}

__device__ __forceinline__ void unite(u32* parent, u32 a, u32 b) {
  while (true) {
    a = find_root(parent, a);
    b = find_root(parent, b);
    if (a == b) return;
    if (a < b) { const u32 t = a; a = b; b = t; }
    if (atomicCAS(parent + a, a, b) == a) return;   // else a gained a parent meanwhile: retry from the roots
  }
}

__device__ __forceinline__ u32 label_of(const ComponentArgs& a, u32 t) { return a.roots[a.parent[t]]; }

__global__ void __launch_bounds__(kBlock) k_cc_edges(ComponentArgs a) {
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < a.count; t += gridDim.x * blockDim.x) {
    const uint3 c = a.input[t];
    a.parent[t] = t;
    const u32 error = triangle_corner_errors(a.radius_squared, a.n, c);
    if (error) { atomicOr(&a.counters->errors, error); continue; }
    u64 slot;
    table_insert(a.edge_keys, a.edge_mask, undirected_edge_key(c.x, c.y), &slot);
    atomicMin(a.edge_owner + slot, t);
    table_insert(a.edge_keys, a.edge_mask, undirected_edge_key(c.y, c.z), &slot);
    atomicMin(a.edge_owner + slot, t);
    table_insert(a.edge_keys, a.edge_mask, undirected_edge_key(c.z, c.x), &slot);
    atomicMin(a.edge_owner + slot, t);
  }
}

__global__ void __launch_bounds__(kBlock) k_cc_hook(ComponentArgs a) {
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < a.count; t += gridDim.x * blockDim.x) {
    const uint3 c = a.input[t];
    // A triangle that fails C1 inserted nothing and the call fails; its keys may even equal the table's empty key
    // (two corners 0xFFFFFFFF), so it looks nothing up.
    if (triangle_corner_errors(a.radius_squared, a.n, c)) continue;
    const u64 keys[3] = {undirected_edge_key(c.x, c.y), undirected_edge_key(c.y, c.z), undirected_edge_key(c.z, c.x)};
#pragma unroll
    for (int e = 0; e < 3; ++e) {
      const u64 slot = table_find(a.edge_keys, a.edge_mask, keys[e]);   // present: k_cc_edges inserted it
      const u32 owner = a.edge_owner[slot];
      if (owner != t) unite(a.parent, t, owner);
    }
  }
}

__global__ void __launch_bounds__(kBlock) k_cc_number(ComponentArgs a) {
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < a.count; t += gridDim.x * blockDim.x) {
    const u32 r = find_root(a.parent, t);
    a.parent[t] = r;
    a.roots[t] = r == t ? 1u : 0u;
  }
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(kFullWarp, v, d);
  return v;
}

// C4 and C5 per piece. The loop strides by whole warps, so every lane of a warp runs the same iterations; a warp
// whose active lanes are all one piece adds its sums once (integer sums and min / max: the same bits).
__global__ void __launch_bounds__(kBlock) k_cc_sums(ComponentArgs a) {
  const u32 lane = threadIdx.x & 31;
  for (u32 base = blockIdx.x * blockDim.x + (threadIdx.x & ~31u); base < a.count; base += gridDim.x * blockDim.x) {
    const u32 t = base + lane;
    const bool active = t < a.count;
    u32 label = 0, count = 0;
    unsigned long long q = 0;
    u32 lo[3] = {~0u, ~0u, ~0u}, hi[3] = {0u, 0u, 0u};
    if (active) {
      const uint3 c = a.input[t];
      const u32 root = a.parent[t];
      label = a.roots[root];
      if (root == t) a.first[label] = t;
      const float3 pa = corner(a, c.x), pb = corner(a, c.y), pc = corner(a, c.z);
      q = area_units(pa, pb, pc);
      count = 1;
      lo[0] = min(ordered(pa.x), min(ordered(pb.x), ordered(pc.x)));
      lo[1] = min(ordered(pa.y), min(ordered(pb.y), ordered(pc.y)));
      lo[2] = min(ordered(pa.z), min(ordered(pb.z), ordered(pc.z)));
      hi[0] = max(ordered(pa.x), max(ordered(pb.x), ordered(pc.x)));
      hi[1] = max(ordered(pa.y), max(ordered(pb.y), ordered(pc.y)));
      hi[2] = max(ordered(pa.z), max(ordered(pb.z), ordered(pc.z)));
    }
    const u32 label0 = __shfl_sync(kFullWarp, label, 0);
    if (__all_sync(kFullWarp, !active || label == label0)) {
      count = __reduce_add_sync(kFullWarp, count);
      q = warp_sum(q);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        lo[k] = __reduce_min_sync(kFullWarp, lo[k]);
        hi[k] = __reduce_max_sync(kFullWarp, hi[k]);
      }
      if (lane != 0) continue;
    } else if (!active) {
      continue;
    }
    atomicAdd(a.count_of + label, count);
    atomicAdd(a.q + label, q);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      atomicMin(a.lo + 3 * static_cast<size_t>(label) + k, lo[k]);
      atomicMax(a.hi + 3 * static_cast<size_t>(label) + k, hi[k]);
    }
  }
}

__global__ void __launch_bounds__(kBlock) k_cc_largest(ComponentArgs a) {
  for (u32 p = blockIdx.x * blockDim.x + threadIdx.x; p < a.pieces; p += gridDim.x * blockDim.x) {
    const unsigned long long q = a.q[p];
    atomicMax(&a.counters->max_q, q);
    if (a.rank_limit) {
      a.sort_keys[p] = ~static_cast<u64>(q);
      a.sort_values[p] = p;
    }
  }
}

__global__ void __launch_bounds__(kBlock) k_cc_rank0(ComponentArgs a) {
  for (u32 p = blockIdx.x * blockDim.x + threadIdx.x; p < a.pieces; p += gridDim.x * blockDim.x)
    if (a.q[p] == a.counters->max_q) atomicMin(&a.counters->largest, p);
}

// The first rank_limit pieces of the stable sort by ~Q (numbers ascending within a Q): rank < keep_largest.
__global__ void __launch_bounds__(kBlock) k_cc_rank(ComponentArgs a) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.rank_limit; i += gridDim.x * blockDim.x)
    a.kept[a.sorted_values[i]] = 1u;
}

__global__ void __launch_bounds__(kBlock) k_cc_keep(ComponentArgs a) {
  for (u32 p = blockIdx.x * blockDim.x + threadIdx.x; p < a.pieces; p += gridDim.x * blockDim.x) {
    const u32 count = a.count_of[p];
    const unsigned long long q = a.q[p];
    const bool keep = count >= a.min_triangles && q >= a.min_q && (a.rank_limit == 0 || a.kept[p] != 0);
    a.kept[p] = keep ? 1u : 0u;
    if (keep) atomicAdd(&a.counters->kept, 1u);
    if (p == a.counters->largest) {
      a.counters->largest_triangles = count;
      a.counters->largest_q = q;
    }
  }
}

__global__ void __launch_bounds__(kBlock) k_cc_flags(ComponentArgs a) {
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < a.count; t += gridDim.x * blockDim.x)
    a.keep[t] = a.kept[label_of(a, t)];
}

__global__ void __launch_bounds__(kBlock) k_cc_write(ComponentArgs a) {
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < a.count; t += gridDim.x * blockDim.x) {
    if (a.labels) a.labels[t] = static_cast<int32_t>(label_of(a, t));
    const u32 at = a.keep[t];
    if (a.out && a.keep[t + 1] != at) a.out[at] = a.input[t];
  }
}

__global__ void __launch_bounds__(kBlock) k_cc_table(ComponentArgs a) {
  for (u32 p = blockIdx.x * blockDim.x + threadIdx.x; p < a.pieces; p += gridDim.x * blockDim.x) {
    sm_mesh_component e;
    e.triangles = a.count_of[p];
    e.area = __dmul_rn(__ull2double_rn(a.q[p]), 0x1p-30);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      e.lo[k] = unordered(a.lo[3 * static_cast<size_t>(p) + k]);
      e.hi[k] = unordered(a.hi[3 * static_cast<size_t>(p) + k]);
    }
    e.first_triangle = a.first[p];
    e.kept = static_cast<int32_t>(a.kept[p]);
    a.table[p] = e;
  }
}

void FreeTriangleScratch(ComponentScratch& s) {
  FreeAndClear(s.edge_keys, s.edge_owner, s.parent, s.roots, s.keep, s.scan_sums);
  s.triangle_capacity = 0;
}

// Per-triangle scratch for `count` triangles (x 1.5 when it grows).
int EnsureTriangleScratch(ComponentScratch& s, u64 count) {
  if (count <= s.triangle_capacity) return SM_OK;
  const u64 cap = GrownCapacity(count);
  FreeTriangleScratch(s);
  const u64 slots = PowerOfTwoAtLeast(4 * cap);
  SM_CUDA(cudaMalloc(&s.edge_keys, sizeof(u64) * slots));
  SM_CUDA(cudaMalloc(&s.edge_owner, sizeof(u32) * slots));
  SM_CUDA(cudaMalloc(&s.parent, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.roots, sizeof(u32) * (cap + 1)));
  SM_CUDA(cudaMalloc(&s.keep, sizeof(u32) * (cap + 1)));
  SM_CUDA(cudaMalloc(&s.scan_sums, sizeof(u32) * ScanTiles(cap + 1)));
  s.triangle_capacity = cap;
  return SM_OK;
}

void FreePieceScratch(ComponentScratch& s) {
  FreeAndClear(s.count, s.q, s.lo, s.hi, s.first, s.kept, s.sort_keys, s.sorted_keys, s.sort_values, s.sorted_values,
               s.sort_temp);
  s.sort_temp_bytes = 0;
  s.piece_capacity = 0;
}

// Per-piece scratch for `pieces` pieces (x 1.5 when it grows), with the rank sort's scratch.
int EnsurePieceScratch(ComponentScratch& s, u64 pieces) {
  if (pieces <= s.piece_capacity) return SM_OK;
  const u64 cap = GrownCapacity(pieces);
  FreePieceScratch(s);
  size_t temp = 0;
  SM_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, temp, static_cast<const u64*>(nullptr), static_cast<u64*>(nullptr),
                                          static_cast<const u32*>(nullptr), static_cast<u32*>(nullptr),
                                          static_cast<int>(cap)));
  SM_CUDA(cudaMalloc(&s.count, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.q, sizeof(unsigned long long) * cap));
  SM_CUDA(cudaMalloc(&s.lo, sizeof(u32) * 3 * cap));
  SM_CUDA(cudaMalloc(&s.hi, sizeof(u32) * 3 * cap));
  SM_CUDA(cudaMalloc(&s.first, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.kept, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.sort_keys, sizeof(u64) * cap));
  SM_CUDA(cudaMalloc(&s.sorted_keys, sizeof(u64) * cap));
  SM_CUDA(cudaMalloc(&s.sort_values, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.sorted_values, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.sort_temp, temp));
  s.sort_temp_bytes = temp;
  s.piece_capacity = cap;
  return SM_OK;
}

}  // namespace

void FreeComponentBuffers(sm_reconstruction* r) {
  ComponentScratch* s = r->components;
  if (!s) return;
  FreeTriangleScratch(*s);
  FreePieceScratch(*s);
  FreeCounters(s->counters);
  delete s;
  r->components = nullptr;
}

}  // namespace smb

using namespace smb;

extern "C" {

void sm_default_component_params(sm_component_params* p) {
  p->min_triangles = 10;
  p->min_area = 0.0;
  p->keep_largest = 0;
}

int sm_mesh_components(sm_reconstruction* r, void* stream_v, const sm_component_params* params,
                       const uint32_t* triangles, uint64_t count, uint32_t* out, uint64_t out_capacity, int32_t* labels,
                       sm_mesh_component* table, uint64_t table_capacity, sm_component_stats* stats) {
  if (!r || !params || !stats) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_mesh_components: null argument");
  auto bad = [](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (std::string("sm_mesh_components: ") + why).c_str()); };
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const sm_component_params& p = *params;
  *stats = sm_component_stats{};
  if (!(p.min_area >= 0.0) || !std::isfinite(p.min_area)) return bad("min_area must be finite and >= 0");
  const char* output_error = !out && out_capacity > 0 ? "out is NULL with a capacity > 0"
                             : (!table && table_capacity > 0 ? "table is NULL with a table_capacity > 0" : nullptr);
  if (const char* why = TriangleListError(triangles, count, output_error)) return bad(why);
  if (count > 0) {
    const u64 tri_bytes = 12 * count, out_bytes = Bytes(out_capacity, 12), label_bytes = 4 * count,
              table_bytes = Bytes(table_capacity, sizeof(sm_mesh_component));
    if (out && out_capacity > 0 && Overlap(triangles, tri_bytes, out, out_bytes)) return bad("out overlaps triangles");
    if (labels && Overlap(triangles, tri_bytes, labels, label_bytes)) return bad("labels overlaps triangles");
    if (table && table_capacity > 0 && Overlap(triangles, tri_bytes, table, table_bytes))
      return bad("table overlaps triangles");
    if (labels && out && out_capacity > 0 && Overlap(labels, label_bytes, out, out_bytes)) return bad("labels overlaps out");
    if (table && table_capacity > 0 && out && out_capacity > 0 && Overlap(table, table_bytes, out, out_bytes))
      return bad("table overlaps out");
    if (table && table_capacity > 0 && labels && Overlap(table, table_bytes, labels, label_bytes))
      return bad("table overlaps labels");
  }
  r->last_stream = stream;
  int status = FetchCounters(r, stream);
  if (status == SM_ERR_CUDA) return status;   // (a surfel-cap overflow of an earlier frame does not matter here)
  if (count == 0) return SM_OK;
  const u32 n = r->host_counters->surfel_count[r->count_slot];
  // C6's area bound in units of 2^-30 m^2; every Q is below 2^64, so a bound at or past it keeps nothing.
  const double min_units = std::nearbyint(p.min_area * 0x1p30);
  const unsigned long long min_q = min_units >= 0x1p64 ? UINT64_MAX : static_cast<unsigned long long>(min_units);

  if (!r->components) {   // published only with its counters, so a failed first call is retried whole
    CounterMirror<ComponentCounters> counters;
    status = CreateCounters(counters);
    if (status != SM_OK) return status;
    r->components = new ComponentScratch();
    r->components->counters = counters;
  }
  ComponentScratch& s = *r->components;
  status = EnsureTriangleScratch(s, count);
  if (status != SM_OK) return status;

  ComponentArgs a{};
  a.n = n;
  a.radius_squared = r->d.surfels + static_cast<size_t>(SM_ROW_RADIUS_SQUARED) * r->d.stride;
  a.smooth = r->d.smooth;
  a.input = reinterpret_cast<const uint3*>(triangles);
  a.count = static_cast<u32>(count);
  const u64 edge_slots = PowerOfTwoAtLeast(4 * count);   // a call uses and clears only what its input needs
  a.edge_keys = s.edge_keys;
  a.edge_owner = s.edge_owner;
  a.edge_mask = edge_slots - 1;
  a.parent = s.parent;
  a.roots = s.roots;
  a.keep = s.keep;
  a.min_triangles = p.min_triangles;
  a.min_q = min_q;
  a.counters = s.counters.device;
  ComponentCounters* c = s.counters.device;
  const ComponentCounters& h = *s.counters.host;
  const int grid = Grid(count, r->sm_count);
  SM_CUDA(cudaMemsetAsync(c, 0, sizeof(ComponentCounters), stream));
  SM_CUDA(cudaMemsetAsync(&c->largest, 0xFF, sizeof(u32), stream));
  SM_CUDA(cudaMemsetAsync(s.edge_keys, 0xFF, sizeof(u64) * edge_slots, stream));
  SM_CUDA(cudaMemsetAsync(s.edge_owner, 0xFF, sizeof(u32) * edge_slots, stream));
  { LaunchScope scope(stream, KID_COMPONENTS_EDGES); LaunchKernel(k_cc_edges, dim3(grid), dim3(kBlock), 0, stream, a); }
  { LaunchScope scope(stream, KID_COMPONENTS_HOOK); LaunchKernel(k_cc_hook, dim3(grid), dim3(kBlock), 0, stream, a); }
  { LaunchScope scope(stream, KID_COMPONENTS_NUMBER); LaunchKernel(k_cc_number, dim3(grid), dim3(kBlock), 0, stream, a); }
  SM_CUDA(cudaMemsetAsync(s.roots + count, 0, sizeof(u32), stream));
  ScanInPlace(stream, s.roots, a.count + 1, s.scan_sums, KID_COMPONENTS_SCAN);
  SM_CUDA(cudaMemcpyAsync(&c->components, s.roots + count, sizeof(u32), cudaMemcpyDeviceToDevice, stream));
  status = ReadCounters(s.counters, stream);
  if (status != SM_OK) return status;
  if (const char* why = MeshInputError(h.errors)) return bad(why);
  const u32 pieces = h.components;

  status = EnsurePieceScratch(s, pieces);
  if (status != SM_OK) return status;
  a.pieces = pieces;
  a.count_of = s.count; a.q = s.q; a.lo = s.lo; a.hi = s.hi; a.first = s.first; a.kept = s.kept;
  a.sort_keys = s.sort_keys; a.sort_values = s.sort_values; a.sorted_values = s.sorted_values;
  a.rank_limit = p.keep_largest > 0 && p.keep_largest < pieces ? static_cast<u32>(p.keep_largest) : 0;
  a.out = reinterpret_cast<uint3*>(out);
  a.labels = labels;
  a.table = table;
  const int piece_grid = Grid(pieces, r->sm_count);
  SM_CUDA(cudaMemsetAsync(s.count, 0, sizeof(u32) * pieces, stream));
  SM_CUDA(cudaMemsetAsync(s.q, 0, sizeof(unsigned long long) * pieces, stream));
  SM_CUDA(cudaMemsetAsync(s.lo, 0xFF, sizeof(u32) * 3 * pieces, stream));
  SM_CUDA(cudaMemsetAsync(s.hi, 0, sizeof(u32) * 3 * pieces, stream));
  SM_CUDA(cudaMemsetAsync(s.kept, 0, sizeof(u32) * pieces, stream));
  { LaunchScope scope(stream, KID_COMPONENTS_SUMS); LaunchKernel(k_cc_sums, dim3(grid), dim3(kBlock), 0, stream, a); }
  { LaunchScope scope(stream, KID_COMPONENTS_RANK); LaunchKernel(k_cc_largest, dim3(piece_grid), dim3(kBlock), 0, stream, a); }
  { LaunchScope scope(stream, KID_COMPONENTS_RANK); LaunchKernel(k_cc_rank0, dim3(piece_grid), dim3(kBlock), 0, stream, a); }
  if (a.rank_limit) {
    {
      LaunchScope scope(stream, KID_COMPONENTS_RANK);
      size_t temp = s.sort_temp_bytes;
      SM_CUDA(cub::DeviceRadixSort::SortPairs(s.sort_temp, temp, static_cast<const u64*>(s.sort_keys), s.sorted_keys,
                                              static_cast<const u32*>(s.sort_values), s.sorted_values,
                                              static_cast<int>(pieces), 0, 64, stream));
    }
    LaunchScope scope(stream, KID_COMPONENTS_RANK);
    LaunchKernel(k_cc_rank, dim3(Grid(a.rank_limit, r->sm_count)), dim3(kBlock), 0, stream, a);
  }
  { LaunchScope scope(stream, KID_COMPONENTS_RANK); LaunchKernel(k_cc_keep, dim3(piece_grid), dim3(kBlock), 0, stream, a); }
  { LaunchScope scope(stream, KID_COMPONENTS_WRITE); LaunchKernel(k_cc_flags, dim3(grid), dim3(kBlock), 0, stream, a); }
  SM_CUDA(cudaMemsetAsync(s.keep + count, 0, sizeof(u32), stream));
  ScanInPlace(stream, s.keep, a.count + 1, s.scan_sums, KID_COMPONENTS_SCAN);
  SM_CUDA(cudaMemcpyAsync(&c->triangles_out, s.keep + count, sizeof(u32), cudaMemcpyDeviceToDevice, stream));
  status = ReadCounters(s.counters, stream);
  if (status != SM_OK) return status;
  stats->triangles_in = count;
  stats->triangles_out = h.triangles_out;
  stats->components = pieces;
  stats->components_kept = h.kept;
  stats->largest_triangles = h.largest_triangles;
  stats->largest_area = std::ldexp(static_cast<double>(h.largest_q), -30);
  if (out_capacity < h.triangles_out) return TriangleCapacityError("sm_mesh_components", h.triangles_out, out_capacity);
  if (table && table_capacity < pieces) {
    return SetError(SM_ERR_CAPACITY, ("sm_mesh_components: " + std::to_string(pieces) +
                                      " pieces do not fit the table capacity of " + std::to_string(table_capacity)).c_str());
  }
  if (labels || h.triangles_out > 0) {
    LaunchScope scope(stream, KID_COMPONENTS_WRITE);
    LaunchKernel(k_cc_write, dim3(grid), dim3(kBlock), 0, stream, a);
  }
  if (table) { LaunchScope scope(stream, KID_COMPONENTS_WRITE); LaunchKernel(k_cc_table, dim3(piece_grid), dim3(kBlock), 0, stream, a); }
  return CheckLaunch("components");
}

}  // extern "C"
