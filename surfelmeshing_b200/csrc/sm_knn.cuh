// sm_knn.cuh — the k-NN index, its three-launch exclusive scan and the warp query core, shared by knn.cu (the
// sm_knn_* entry points) and mesh.cu (sm_triangulate); the mesh calls use the scan too. The library is built without
// relocatable device code, so the kernels and device functions live here and each translation unit compiles its own
// copy.
#pragma once

#include <climits>

#include "sm_handle.cuh"
#include "sm_math.cuh"

struct sm_knn_index {
  int device = 0;
  int sm_count = 0;
  smb::u32 capacity = 0;       // points the index can hold
  smb::u32 table_size = 0;     // buckets, a power of two
  smb::u32* bucket_start = nullptr;   // [table_size + 1]: counts, then (after the scan) first record of each bucket
  smb::u32* bucket_cursor = nullptr;  // [table_size]
  smb::u32* scan_sums = nullptr;      // one per scan tile
  smb::u32* point_bucket = nullptr;   // [capacity]
  float4* records = nullptr;          // [capacity]: x, y, z, index bits, grouped by bucket
  smb::u32 point_count = 0;           // points offered to the last build (indices are < this)
  float cell_size = 0.f;
  float inverse_cell_size = 0.f;
  bool built = false;
  // device staging of sm_knn_batch_host (grown on demand): 4 point rows, results
  smb::u32 batch_points = 0;
  int batch_k = 0;
  float* batch_rows = nullptr;             // [4][batch_points]: x, y, z, radius^2
  float* batch_distance_squared = nullptr; // [batch_points][batch_k]
  smb::u32* batch_index = nullptr;
  int* batch_count = nullptr;
  // pinned bounce buffers of the result download (two chunks in flight) and their events
  void* bounce[2] = {nullptr, nullptr};
  cudaEvent_t bounce_ready[2] = {nullptr, nullptr};
};

namespace smb {

// knn.cu: index lifetime and the batched build / query behind sm_knn_*.
int KnnCreate(sm_knn_index** out, u32 max_points);
void KnnDestroy(sm_knn_index* k);
int KnnBuild(sm_knn_index* k, cudaStream_t stream, u32 n, const float* x, const float* y, const float* z,
             const float* radius_squared, const u8* state, float cell_size);

namespace {

constexpr int kScanBlock = 1024;
constexpr int kScanPerThread = 4;
constexpr int kScanTile = kScanBlock * kScanPerThread;
constexpr int kMaxResults = 64;            // kMaxNeighbors / kMaxSurfelCount of the callers (surfel_meshing.cc:669,814)
constexpr u8 kStateFree = 0;               // Surfel::MeshingState, surfel.h:67-71
constexpr u8 kStateCompleted = 2;
constexpr u8 kStateAbsent = 255;           // slot holds no surfel
constexpr unsigned kFullMask = 0xFFFFFFFFu;
constexpr unsigned long long kEmptyKey = ~0ull;

__device__ __forceinline__ int cell_of(float v, float inverse_cell_size) {
  return __float2int_rd(fmul(v, inverse_cell_size));
}

__device__ __forceinline__ u32 bucket_of(int cx, int cy, int cz, u32 mask) {
  u32 h = static_cast<u32>(cx) * 73856093u ^ static_cast<u32>(cy) * 19349663u ^ static_cast<u32>(cz) * 83492791u;
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  return h & mask;
}

// Exclusive scan of `values[0, n)` in place, three launches: tile-local scan + tile sums, scan of the sums by
// one block, add-back. n is at most 2^27 + 1 (table of 2 x 64 M points), so there are at most 32 769 tile sums.
__global__ void __launch_bounds__(kScanBlock) k_knn_scan_tiles(u32* values, u32 n, u32* sums) {
  __shared__ u32 warp_totals[kScanBlock / 32];
  const u32 base = blockIdx.x * kScanTile + threadIdx.x * kScanPerThread;
  u32 v[kScanPerThread];
  u32 thread_total = 0;
#pragma unroll
  for (int k = 0; k < kScanPerThread; ++k) {
    v[k] = base + k < n ? values[base + k] : 0u;
    thread_total += v[k];
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  u32 inclusive = thread_total;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u32 up = __shfl_up_sync(kFullMask, inclusive, o);
    if (lane >= o) inclusive += up;
  }
  if (lane == 31) warp_totals[warp] = inclusive;
  __syncthreads();
  if (warp == 0) {
    u32 w = warp_totals[lane];
    u32 inc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u32 up = __shfl_up_sync(kFullMask, inc, o);
      if (lane >= o) inc += up;
    }
    warp_totals[lane] = inc - w;
    if (lane == 31) sums[blockIdx.x] = inc;
  }
  __syncthreads();
  u32 running = warp_totals[warp] + inclusive - thread_total;
#pragma unroll
  for (int k = 0; k < kScanPerThread; ++k) {
    if (base + k < n) values[base + k] = running;
    running += v[k];
  }
}

__global__ void __launch_bounds__(kScanBlock) k_knn_scan_sums(u32* sums, u32 tiles) {
  __shared__ u32 warp_totals[kScanBlock / 32];
  __shared__ u32 carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (u32 base = 0; base < tiles; base += kScanBlock) {
    const u32 i = base + threadIdx.x;
    const u32 v = i < tiles ? sums[i] : 0u;
    u32 inclusive = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u32 up = __shfl_up_sync(kFullMask, inclusive, o);
      if (lane >= o) inclusive += up;
    }
    if (lane == 31) warp_totals[warp] = inclusive;
    __syncthreads();
    if (warp == 0) {
      const u32 w = warp_totals[lane];
      u32 inc = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const u32 up = __shfl_up_sync(kFullMask, inc, o);
        if (lane >= o) inc += up;
      }
      warp_totals[lane] = inc - w;
    }
    __syncthreads();
    const u32 exclusive = carry + warp_totals[warp] + inclusive - v;
    if (i < tiles) sums[i] = exclusive;
    __syncthreads();
    if (threadIdx.x == kScanBlock - 1) carry = exclusive + v;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kScanBlock) k_knn_scan_add(u32* values, u32 n, const u32* sums) {
  const u32 offset = sums[blockIdx.x];
  const u32 base = blockIdx.x * kScanTile + threadIdx.x * kScanPerThread;
#pragma unroll
  for (int k = 0; k < kScanPerThread; ++k) {
    if (base + k < n) values[base + k] += offset;
  }
}

// The tiles of a scan over n values: the entries its tile sums take.
inline u32 ScanTiles(u64 n) { return static_cast<u32>((n + kScanTile - 1) / kScanTile); }

// The exclusive scan of values[0, n) in place, each of its launches in a LaunchScope of `id`.
inline void ScanInPlace(cudaStream_t stream, u32* values, u32 n, u32* sums, KernelId id) {
  const u32 tiles = ScanTiles(n);
  { LaunchScope scope(stream, id); k_knn_scan_tiles<<<tiles, kScanBlock, 0, stream>>>(values, n, sums); }
  { LaunchScope scope(stream, id); k_knn_scan_sums<<<1, kScanBlock, 0, stream>>>(sums, tiles); }
  { LaunchScope scope(stream, id); k_knn_scan_add<<<tiles, kScanBlock, 0, stream>>>(values, n, sums); }
}

struct QueryArgs {
  u32 query_count;
  const float* qx;
  const float* qy;
  const float* qz;
  const float* radius_squared;   // per query
  float radius_scale;            // the query radius^2 is radius_squared[q] * radius_scale (1 for sm_knn_query)
  const u8* state;               // optional, indexed by point index
  int include_completed;
  int include_free;
  int max_result_count;          // 1..64
  float inverse_cell_size;
  u32 mask;
  const u32* bucket_start;
  const float4* records;
  float* out_distance_squared;   // [query_count][max_result_count]
  u32* out_index;                // [query_count][max_result_count]
  int* out_count;                // [query_count]
};

// The warp's result list: rank g (0 = nearest) lives in lane g & 31, register g >> 5. Keys are
// {distance^2 bits, index}: non-negative floats order like their bit patterns, the index breaks ties.
struct WarpList {
  unsigned long long e0, e1;
  __device__ __forceinline__ void insert(unsigned long long key, int lane) {
    const int rank = __popc(__ballot_sync(kFullMask, e0 < key)) + __popc(__ballot_sync(kFullMask, e1 < key));
    const unsigned long long up0 = __shfl_up_sync(kFullMask, e0, 1);
    unsigned long long up1 = __shfl_up_sync(kFullMask, e1, 1);
    const unsigned long long last0 = __shfl_sync(kFullMask, e0, 31);
    if (lane == 0) up1 = last0;
    if (lane == rank) e0 = key; else if (lane > rank) e0 = up0;
    if (lane + 32 == rank) e1 = key; else if (lane + 32 > rank) e1 = up1;
  }
  __device__ __forceinline__ unsigned long long at(int rank) const {
    const unsigned long long a = __shfl_sync(kFullMask, e0, rank & 31);
    const unsigned long long b = __shfl_sync(kFullMask, e1, rank & 31);
    return rank < 32 ? a : b;
  }
  // Bitonic sort of the 64 keys (ascending over ranks 0..63; empty keys are the largest value and end up last).
  // kHalf: only e0 holds keys (e1 all empty): a 32-key network.
  template <bool kHalf>
  __device__ __forceinline__ void sort(int lane) {
#pragma unroll
    for (int k = 2; k <= (kHalf ? 32 : 64); k <<= 1) {
#pragma unroll
      for (int j = k >> 1; j >= 1; j >>= 1) {
        if (j == 32) {   // partner of rank g is g ^ 32: the other register of the same lane (k = 64: ascending)
          const unsigned long long lo = e0 < e1 ? e0 : e1, hi = e0 < e1 ? e1 : e0;
          e0 = lo; e1 = hi;
          continue;
        }
        const bool lower = (lane & j) == 0;
        {
          const bool ascending = (lane & k) == 0;   // k = 64: lane & 64 == 0
          const unsigned long long other = __shfl_xor_sync(kFullMask, e0, j);
          const bool take_min = lower == ascending;
          e0 = (take_min == (other < e0)) ? other : e0;
        }
        if (!kHalf) {
          const bool ascending = ((lane + 32) & k) == 0;
          const unsigned long long other = __shfl_xor_sync(kFullMask, e1, j);
          const bool take_min = lower == ascending;
          e1 = (take_min == (other < e1)) ? other : e1;
        }
      }
    }
  }
};

// Past this many cells per query the warp walks all records instead (bounded work for a radius far above the cell size).
constexpr long long kMaxCellsPerQuery = 1024;

// A query first APPENDS every record that passes the radius and state tests to a 64-key staging row in shared
// memory (one ballot and one store per batch of 32 records); most queries end with fewer than 64 candidates and
// sort them once at the end. Only when the row would overflow does the warp sort what it has into the register
// list and continue by insertion against the admission threshold.
struct QueryState {
  WarpList list;
  int count;                      // staged keys (staging) or list entries (sorted), <= 64
  bool staging;
  unsigned long long threshold;   // sorted mode: keys >= threshold cannot enter the first max_result_count ranks
  unsigned long long* stage;      // this warp's 64-key row in shared memory
};

__device__ __forceinline__ void leave_staging(const QueryArgs& a, QueryState& s, int lane) {
  __syncwarp();
  s.list.e0 = lane < s.count ? s.stage[lane] : kEmptyKey;
  s.list.e1 = lane + 32 < s.count ? s.stage[lane + 32] : kEmptyKey;
  if (s.count <= 32) s.list.sort<true>(lane); else s.list.sort<false>(lane);
  s.staging = false;
  if (s.count >= a.max_result_count) s.threshold = s.list.at(a.max_result_count - 1);
}

template <bool kCheckCell>
__device__ __forceinline__ void scan_records(const QueryArgs& a, QueryState& s, u32 begin, u32 end, int cx, int cy, int cz,
                                             float px, float py, float pz, float radius_squared, int lane) {
  for (u32 base = begin; base < end; base += 32) {
    const u32 e = base + lane;
    unsigned long long key = kEmptyKey;
    if (e < end) {
      const float4 record = a.records[e];
      // Several cells can share a bucket: a record counts only while its own cell is the one visited.
      if (!kCheckCell || (cell_of(record.x, a.inverse_cell_size) == cx && cell_of(record.y, a.inverse_cell_size) == cy &&
                          cell_of(record.z, a.inverse_cell_size) == cz)) {
        const float dx = fsub(record.x, px), dy = fsub(record.y, py), dz = fsub(record.z, pz);
        const float distance_squared = fadd(fadd(fmul(dx, dx), fmul(dy, dy)), fmul(dz, dz));
        if (distance_squared <= radius_squared) {
          const u32 index = __float_as_uint(record.w);
          bool wanted = true;
          if (a.state) {
            const u8 state = a.state[index];
            wanted = state != kStateAbsent && (a.include_completed || state != kStateCompleted) &&
                     (a.include_free || state != kStateFree);
          }
          if (wanted) key = (static_cast<unsigned long long>(__float_as_uint(distance_squared)) << 32) | index;
        }
      }
    }
    unsigned candidates = __ballot_sync(kFullMask, key < s.threshold);
    if (candidates == 0) continue;
    if (s.staging) {
      const int incoming = __popc(candidates);
      if (s.count + incoming <= kMaxResults) {
        if (key < s.threshold) s.stage[s.count + __popc(candidates & ((1u << lane) - 1u))] = key;
        s.count += incoming;
        continue;
      }
      leave_staging(a, s, lane);
      candidates = __ballot_sync(kFullMask, key < s.threshold);
    }
    while (candidates) {
      const int source = __ffs(candidates) - 1;
      candidates &= candidates - 1;
      const unsigned long long candidate = __shfl_sync(kFullMask, key, source);
      if (candidate < s.threshold) {   // the threshold may have dropped since the ballot
        s.list.insert(candidate, lane);
        s.count = min(s.count + 1, kMaxResults);
        if (s.count >= a.max_result_count) s.threshold = s.list.at(a.max_result_count - 1);
      }
    }
  }
}

// One query of the warp: every record within radius_squared of (px, py, pz) that passes the state filter, into
// s.list sorted by key (the first min(s.count, a.max_result_count) ranks are the answer). The staging row is
// free again when this returns.
__device__ __forceinline__ void warp_query(const QueryArgs& a, QueryState& s, float px, float py, float pz,
                                           float radius_squared, int lane) {
  if (radius_squared >= 0.f) {
    // Cells the ball can touch. Everything is rounded outwards: a record whose fp32 distance passes the
    // test lies inside [p - reach, p + reach] on every axis, and cell_of() is monotone.
    const float reach = __fmul_ru(__fsqrt_ru(radius_squared), 1.00001f);
    const int x0 = cell_of(__fsub_rd(px, reach), a.inverse_cell_size), x1 = cell_of(__fadd_ru(px, reach), a.inverse_cell_size);
    const int y0 = cell_of(__fsub_rd(py, reach), a.inverse_cell_size), y1 = cell_of(__fadd_ru(py, reach), a.inverse_cell_size);
    const int z0 = cell_of(__fsub_rd(pz, reach), a.inverse_cell_size), z1 = cell_of(__fadd_ru(pz, reach), a.inverse_cell_size);
    const long long nx = static_cast<long long>(x1) - x0 + 1, ny = static_cast<long long>(y1) - y0 + 1,
                    nz = static_cast<long long>(z1) - z0 + 1;
    // (also taken when a coordinate saturated: the cell loops below must not run into INT_MAX)
    if (nx > kMaxCellsPerQuery || ny > kMaxCellsPerQuery || nz > kMaxCellsPerQuery || nx * ny * nz > kMaxCellsPerQuery ||
        x1 == INT_MAX || y1 == INT_MAX || z1 == INT_MAX) {
      scan_records<false>(a, s, 0, a.bucket_start[a.mask + 1], 0, 0, 0, px, py, pz, radius_squared, lane);
    } else {
      for (int cz = z0; cz <= z1; ++cz) {
        for (int cy = y0; cy <= y1; ++cy) {
          for (int cx = x0; cx <= x1; ++cx) {
            const u32 bucket = bucket_of(cx, cy, cz, a.mask);
            scan_records<true>(a, s, a.bucket_start[bucket], a.bucket_start[bucket + 1], cx, cy, cz, px, py, pz,
                               radius_squared, lane);
          }
        }
      }
    }
  }
  if (s.staging) leave_staging(a, s, lane);
  __syncwarp();   // the staging row is reused by this warp's next query
}

}  // namespace

}  // namespace smb
