// sm_mesh_edges.cuh — the edge hash table, the input checks and the fp32 corner geometry of a triangle list over the
// handle's slots, shared by holes.cu (sm_mesh_fill_holes), simplify.cu (sm_mesh_simplify), texture.cu
// (sm_mesh_texture) and components.cu (sm_mesh_components), and the host checks and scratch handling of those four
// calls and of mesh.cu (sm_triangulate, sm_mesh_update). The first two take an edge-manifold, consistently oriented
// list, refuse the same inputs and test new triangles by rule 4.
// The library is built without relocatable device code, so each translation unit compiles its own copy.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <string>

#include "sm_handle.cuh"
#include "sm_knn.cuh"

namespace smb {

namespace {

constexpr int kBlock = 256;   // the one-thread-per-item mesh kernels of holes.cu, simplify.cu, texture.cu, components.cu

// Below this, the 3 x count corners and edges index as u32 and x 1.5 of them still counts as the int of CUB's sort.
constexpr u64 kMaxMeshTriangles = 1ull << 28;

// Input errors found on the device (an atomicOr of these bits).
constexpr u32 kBadCorner = 1;      // index >= surfels_size(), or a slot that is not present
constexpr u32 kRepeatedCorner = 2;
constexpr u32 kDuplicateEdge = 4;

__device__ __forceinline__ u64 edge_key(u32 tail, u32 head) { return (static_cast<u64>(tail) << 32) | head; }
__device__ __forceinline__ u32 tail_of(u64 key) { return static_cast<u32>(key >> 32); }
__device__ __forceinline__ u32 head_of(u64 key) { return static_cast<u32>(key); }

// The key of the undirected edge {a, b}: the directed key from the smaller slot.
__device__ __forceinline__ u64 undirected_edge_key(u32 a, u32 b) { return a < b ? edge_key(a, b) : edge_key(b, a); }

// splitmix64's finaliser: the probe start of a key.
__device__ __forceinline__ u64 mix(u64 x) {
  x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull;
  x ^= x >> 27; x *= 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// Inserts key; false if it was there already.
__device__ __forceinline__ bool table_insert(u64* table, u64 mask, u64 key, u64* slot_out) {
  for (u64 slot = mix(key) & mask;; slot = (slot + 1) & mask) {
    const u64 old = atomicCAS(reinterpret_cast<unsigned long long*>(table + slot), kEmptyKey, key);
    if (old == kEmptyKey || old == key) { *slot_out = slot; return old == kEmptyKey; }
  }
}

// The slot of key, or ~0 when it is absent.
__device__ __forceinline__ u64 table_find(const u64* table, u64 mask, u64 key) {
  for (u64 slot = mix(key) & mask;; slot = (slot + 1) & mask) {
    const u64 k = table[slot];
    if (k == key) return slot;
    if (k == kEmptyKey) return ~0ull;
  }
}

// Checks triangle c of a list over slots [0, n) (row 7 = radius^2 of a slot, with `stride`) and inserts its three
// directed edges into the table. Returns the error bits it found; a triangle with a bad or repeated corner inserts
// nothing.
// The error bits of triangle c over slots [0, n) (row 7 = radius^2 of a slot): kBadCorner, kRepeatedCorner.
__device__ __forceinline__ u32 triangle_corner_errors(const float* radius_squared, u32 n, uint3 c) {
  u32 error = 0;
  for (int s = 0; s < 3; ++s) {
    const u32 i = s == 0 ? c.x : (s == 1 ? c.y : c.z);
    if (i >= n || !(radius_squared[i] > 0.f)) error |= kBadCorner;
  }
  if (c.x == c.y || c.y == c.z || c.z == c.x) error |= kRepeatedCorner;
  return error;
}

__device__ __forceinline__ u32 check_and_insert_triangle(const float* radius_squared, u32 n, uint3 c, u64* table,
                                                         u64 mask) {
  u32 error = triangle_corner_errors(radius_squared, n, c);
  if (!error) {
    u64 slot;
    if (!table_insert(table, mask, edge_key(c.x, c.y), &slot)) error |= kDuplicateEdge;
    if (!table_insert(table, mask, edge_key(c.y, c.z), &slot)) error |= kDuplicateEdge;
    if (!table_insert(table, mask, edge_key(c.z, c.x), &slot)) error |= kDuplicateEdge;
  }
  return error;
}

__device__ __forceinline__ float dot3p(float3 a, float3 b) { return fadd(fadd(fmul(a.x, b.x), fmul(a.y, b.y)), fmul(a.z, b.z)); }
__device__ __forceinline__ float3 sub3(float3 a, float3 b) { return make_float3(fsub(a.x, b.x), fsub(a.y, b.y), fsub(a.z, b.z)); }

// p_i: the smooth position (the rows 3-5 mirror) of slot i of a [row][stride] state.
__device__ __forceinline__ float3 slot_position(const float* rows, size_t stride, u32 i) {
  return make_float3(rows[SM_ROW_SMOOTH_X * stride + i], rows[SM_ROW_SMOOTH_Y * stride + i],
                     rows[SM_ROW_SMOOTH_Z * stride + i]);
}

// Rows 8-10 times 1 / sqrt(n . n) (IEEE); false unless n . n is finite and > 0 (sm_triangulate's unit normal).
__device__ __forceinline__ bool slot_unit_normal(const float* rows, size_t stride, u32 i, float3* out) {
  const float3 n = make_float3(rows[SM_ROW_NORMAL_X * stride + i], rows[SM_ROW_NORMAL_Y * stride + i],
                               rows[SM_ROW_NORMAL_Z * stride + i]);
  const float s = dot3p(n, n);
  if (!(s > 0.f) || !isfinite(s)) return false;
  const float inv = __fdiv_rn(1.f, __fsqrt_rn(s));
  *out = make_float3(fmul(n.x, inv), fmul(n.y, inv), fmul(n.z, inv));
  return true;
}

// Rule 4's angle test at one corner with edges (g, h).
__device__ __forceinline__ bool angle_too_large(float cos_triangle, float3 g, float3 h) {
  const float d = dot3p(g, h);
  const float l = __fsqrt_rn(fmul(dot3p(g, g), dot3p(h, h)));
  return d < fmul(cos_triangle, l);
}

inline u64 PowerOfTwoAtLeast(u64 v) {
  u64 p = 1;
  while (p < v) p <<= 1;
  return p;
}

// The message of the first error bit set, or nullptr.
inline const char* MeshInputError(u32 errors) {
  if (errors & kBadCorner) return "a corner is not a present slot below surfels_size()";
  if (errors & kRepeatedCorner) return "a triangle has a repeated corner";
  if (errors & kDuplicateEdge) return "a directed edge occurs twice (the input must be edge-manifold and consistently oriented)";
  return nullptr;
}

// An angle parameter of a mesh call in degrees: finite and in (0, 180].
inline bool AngleInRange(float deg) { return std::isfinite(deg) && deg > 0.f && deg <= 180.f; }

// The cosine the kernels compare against, through double.
inline float CosDegrees(float deg) { return static_cast<float>(std::cos(static_cast<double>(deg) * (M_PI / 180.0))); }

// Blocks of kBlock threads for one thread per item: at least one, at most 8 per SM (the kernels stride).
inline int Grid(u64 items, int sm_count) {
  return static_cast<int>(std::max<u64>(1, std::min<u64>((items + kBlock - 1) / kBlock, 8ull * sm_count)));
}

// The reason the input list of `count` triangles is refused, or nullptr. `output_error`, the caller's check of its
// output list (nullptr: it passed), is reported between the two checks.
inline const char* TriangleListError(const uint32_t* triangles, u64 count, const char* output_error = nullptr) {
  if (!triangles && count > 0) return "triangles is NULL with a count > 0";
  if (output_error) return output_error;
  if (count >= kMaxMeshTriangles) return "2^28 triangles or more";
  return nullptr;
}

// Whether the bytes [a, a + a_bytes) and [b, b + b_bytes) overlap. An end past the top of the address space is taken
// as the top, so a range of any length from the caller compares correctly.
inline bool Overlap(const void* a, u64 a_bytes, const void* b, u64 b_bytes) {
  const uintptr_t a0 = reinterpret_cast<uintptr_t>(a), b0 = reinterpret_cast<uintptr_t>(b);
  const uintptr_t a1 = a_bytes > UINTPTR_MAX - a0 ? UINTPTR_MAX : a0 + a_bytes;
  const uintptr_t b1 = b_bytes > UINTPTR_MAX - b0 ? UINTPTR_MAX : b0 + b_bytes;
  return a0 < b1 && b0 < a1;
}

// Bytes of `count` items of `size` bytes, saturated like the end of an address range.
inline u64 Bytes(u64 count, u64 size) { return count > UINT64_MAX / size ? UINT64_MAX : count * size; }

// The SM_ERR_CAPACITY of `who` when an output list of `capacity` triangles cannot take `count`.
inline int TriangleCapacityError(const char* who, u64 count, u64 capacity) {
  return SetError(SM_ERR_CAPACITY, (std::string(who) + ": " + std::to_string(count) +
                                    " triangles do not fit the capacity of " + std::to_string(capacity)).c_str());
}

// The capacity a group of scratch buffers grows to when `need` items do not fit: x 1.5, at least `floor`.
inline u64 GrownCapacity(u64 need, u64 floor = 1024) { return std::max<u64>(need + need / 2, floor); }

// Frees each buffer and sets it to NULL. cudaFree synchronises the device: an earlier call may still use them.
template <class... T>
void FreeAndClear(T*&... buffers) { ((cudaFree(buffers), buffers = nullptr), ...); }

// A call's device counter struct and its pinned host mirror.
template <class T>
struct CounterMirror {
  T* device = nullptr;
  T* host = nullptr;
};

// Both buffers or neither: on a failure nothing stays allocated and `c` stays empty, so the next call tries again.
template <class T>
int CreateCounters(CounterMirror<T>& c) {
  T* device = nullptr;
  T* host = nullptr;
  SM_CUDA(cudaMalloc(&device, sizeof(T)));
  if (const cudaError_t e = cudaMallocHost(&host, sizeof(T)); e != cudaSuccess) {
    cudaFree(device);
    return SetError(SM_ERR_CUDA, (std::string("cudaMallocHost: ") + cudaGetErrorString(e)).c_str());
  }
  c.device = device;
  c.host = host;
  return SM_OK;
}

template <class T>
void FreeCounters(CounterMirror<T>& c) {
  cudaFree(c.device);
  if (c.host) cudaFreeHost(c.host);
  c = CounterMirror<T>{};
}

// The first `bytes` of the device counters into the host mirror, then a synchronisation of the stream.
template <class T>
int ReadCounters(const CounterMirror<T>& c, cudaStream_t stream, size_t bytes = sizeof(T)) {
  SM_CUDA(cudaMemcpyAsync(c.host, c.device, bytes, cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaStreamSynchronize(stream));
  return SM_OK;
}

}  // namespace

}  // namespace smb
