// knn.cu — batched radius-limited k-nearest-neighbour queries over the surfel cloud (SURVEY §8 f4).
//
// Reference: the CPU meshing thread asks CompressedOctree::FindNearestSurfelsWithinRadius
// (APP/octree.cc:313-470) for the <= 64 nearest surfels within a squared radius, once per surfel it
// triangulates (APP/surfel_meshing.cc:421, <false, true>: completed surfels excluded) and once per surfel it resets
// for remeshing (APP/surfel_meshing.cc:821, <true, false>: free surfels excluded). One query walks a lazily sorted
// compressed octree on one thread.
//
// Here the cloud is binned once per snapshot into a hashed uniform grid (counting sort by bucket: count, exclusive
// scan, scatter of {x, y, z, index} records, so that a cell is one contiguous run of 16-byte records) and queries run
// as a batch, one warp per query: the lanes stride over the records of the cells the search ball touches, and the
// warp keeps the best 64 {distance^2, index} keys sorted across its lanes (two per lane; an insertion is two ballots
// and two shuffles). Results are what the octree returns: ascending squared distance, `<= radius^2` inclusive, the
// meshing-state filter applied before the cap; equal distances, which the reference leaves to traversal order, are
// ordered by index. Squared distances are computed as ((dx*dx + dy*dy) + dz*dz) in fp32 without contraction, the
// order Eigen's squaredNorm() evaluates, so they agree bit for bit with the reference octree (oracle/_ref/
// liboctree_ref.so, built from the reference's octree.cc).

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>

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

namespace {

#define SM_CUDA(call)                                                                                   \
  do {                                                                                                  \
    const cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) return SetError(SM_ERR_CUDA, (std::string(#call) + ": " + cudaGetErrorString(e_)).c_str()); \
  } while (0)

constexpr int kBuildBlock = 256;
constexpr int kScanBlock = 1024;
constexpr int kScanPerThread = 4;
constexpr int kScanTile = kScanBlock * kScanPerThread;
constexpr int kQueryBlock = 128;           // 4 queries per block, one warp each
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

struct BuildArgs {
  u32 n;
  const float* x;
  const float* y;
  const float* z;
  const float* radius_squared;   // optional: points with radius^2 <= 0 are left out (merged surfels, kernels.cu:1987)
  const u8* state;               // optional: points with state 255 are left out
  float inverse_cell_size;
  u32 mask;
  u32* bucket_start;
  u32* bucket_cursor;
  u32* point_bucket;
  float4* records;
};

__device__ __forceinline__ bool point_present(const BuildArgs& a, u32 i) {
  if (a.radius_squared && !(a.radius_squared[i] > 0.f)) return false;
  if (a.state && a.state[i] == kStateAbsent) return false;
  return true;
}

__global__ void __launch_bounds__(kBuildBlock) k_knn_count(BuildArgs a) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    u32 bucket = 0xFFFFFFFFu;
    if (point_present(a, i)) {
      bucket = bucket_of(cell_of(a.x[i], a.inverse_cell_size), cell_of(a.y[i], a.inverse_cell_size),
                         cell_of(a.z[i], a.inverse_cell_size), a.mask);
      atomicAdd(&a.bucket_start[bucket], 1u);
    }
    a.point_bucket[i] = bucket;
  }
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

__global__ void __launch_bounds__(kBuildBlock) k_knn_scatter(BuildArgs a) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const u32 bucket = a.point_bucket[i];
    if (bucket == 0xFFFFFFFFu) continue;
    const u32 position = a.bucket_start[bucket] + atomicAdd(&a.bucket_cursor[bucket], 1u);
    a.records[position] = make_float4(a.x[i], a.y[i], a.z[i], __uint_as_float(i));
  }
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

__global__ void __launch_bounds__(kQueryBlock) k_knn_query(QueryArgs a) {
  __shared__ unsigned long long s_stage[kQueryBlock / 32][kMaxResults];
  const int lane = threadIdx.x & 31;
  const u32 warps_per_grid = gridDim.x * (kQueryBlock / 32);
  for (u32 q = blockIdx.x * (kQueryBlock / 32) + (threadIdx.x >> 5); q < a.query_count; q += warps_per_grid) {
    const float px = a.qx[q], py = a.qy[q], pz = a.qz[q];
    const float radius_squared = fmul(a.radius_squared[q], a.radius_scale);
    QueryState s{{kEmptyKey, kEmptyKey}, 0, true, kEmptyKey, s_stage[threadIdx.x >> 5]};
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
    const int found = min(s.count, a.max_result_count);
    const size_t out = static_cast<size_t>(q) * a.max_result_count;
    if (lane < a.max_result_count) {
      const bool valid = lane < found;
      a.out_distance_squared[out + lane] = valid ? __uint_as_float(static_cast<u32>(s.list.e0 >> 32)) : __int_as_float(0x7F800000);
      a.out_index[out + lane] = valid ? static_cast<u32>(s.list.e0) : 0xFFFFFFFFu;
    }
    if (lane + 32 < a.max_result_count) {
      const bool valid = lane + 32 < found;
      a.out_distance_squared[out + lane + 32] = valid ? __uint_as_float(static_cast<u32>(s.list.e1 >> 32)) : __int_as_float(0x7F800000);
      a.out_index[out + lane + 32] = valid ? static_cast<u32>(s.list.e1) : 0xFFFFFFFFu;
    }
    if (lane == 0) a.out_count[q] = found;
  }
}

u32 NextPowerOfTwo(u32 v) {
  u32 p = 1;
  while (p < v) p <<= 1;
  return p;
}

void FreeIndex(sm_knn_index* k) {
  cudaFree(k->bucket_start);
  cudaFree(k->bucket_cursor);
  cudaFree(k->scan_sums);
  cudaFree(k->point_bucket);
  cudaFree(k->records);
  cudaFree(k->batch_rows);
  cudaFree(k->batch_distance_squared);
  cudaFree(k->batch_index);
  cudaFree(k->batch_count);
  for (int i = 0; i < 2; ++i) {
    if (k->bounce[i]) cudaFreeHost(k->bounce[i]);
    if (k->bounce_ready[i]) cudaEventDestroy(k->bounce_ready[i]);
  }
  delete k;
}

int CreateIndex(sm_knn_index* k, u32 max_points) {
  SM_CUDA(cudaGetDevice(&k->device));
  SM_CUDA(cudaDeviceGetAttribute(&k->sm_count, cudaDevAttrMultiProcessorCount, k->device));
  k->capacity = max_points;
  k->table_size = NextPowerOfTwo(std::max<u32>(1024u, 2u * max_points));
  const u32 tiles = (k->table_size + 1 + kScanTile - 1) / kScanTile;
  SM_CUDA(cudaMalloc(&k->bucket_start, sizeof(u32) * (static_cast<size_t>(k->table_size) + 1)));
  SM_CUDA(cudaMalloc(&k->bucket_cursor, sizeof(u32) * static_cast<size_t>(k->table_size)));
  SM_CUDA(cudaMalloc(&k->scan_sums, sizeof(u32) * tiles));
  SM_CUDA(cudaMalloc(&k->point_bucket, sizeof(u32) * static_cast<size_t>(max_points)));
  SM_CUDA(cudaMalloc(&k->records, sizeof(float4) * static_cast<size_t>(max_points)));
  return SM_OK;
}

}  // namespace

int KnnBuild(sm_knn_index* k, cudaStream_t stream, u32 n, const float* x, const float* y, const float* z,
             const float* radius_squared, const u8* state, float cell_size) {
  if (n > k->capacity) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_build: more points than the index was created for");
  if (!(cell_size > 0.f)) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_build: cell_size must be positive");
  k->built = false;
  k->point_count = n;
  k->cell_size = cell_size;
  k->inverse_cell_size = 1.f / cell_size;
  SM_CUDA(cudaMemsetAsync(k->bucket_start, 0, sizeof(u32) * (static_cast<size_t>(k->table_size) + 1), stream));
  SM_CUDA(cudaMemsetAsync(k->bucket_cursor, 0, sizeof(u32) * static_cast<size_t>(k->table_size), stream));
  BuildArgs a{n, x, y, z, radius_squared, state, k->inverse_cell_size, k->table_size - 1, k->bucket_start,
              k->bucket_cursor, k->point_bucket, k->records};
  const u32 scan_n = k->table_size + 1;
  const u32 tiles = (scan_n + kScanTile - 1) / kScanTile;
  if (n > 0) {
    const int blocks = static_cast<int>(std::min<u32>((n + kBuildBlock - 1) / kBuildBlock, 8u * k->sm_count));
    k_knn_count<<<blocks, kBuildBlock, 0, stream>>>(a);
    k_knn_scan_tiles<<<tiles, kScanBlock, 0, stream>>>(k->bucket_start, scan_n, k->scan_sums);
    k_knn_scan_sums<<<1, kScanBlock, 0, stream>>>(k->scan_sums, tiles);
    k_knn_scan_add<<<tiles, kScanBlock, 0, stream>>>(k->bucket_start, scan_n, k->scan_sums);
    k_knn_scatter<<<blocks, kBuildBlock, 0, stream>>>(a);
  }
  SM_CUDA(cudaGetLastError());
  k->built = true;
  return SM_OK;
}

int KnnQuery(sm_knn_index* k, cudaStream_t stream, u32 query_count, const float* qx, const float* qy, const float* qz,
             const float* radius_squared, float radius_scale, const u8* state, int include_completed, int include_free,
             int max_result_count, float* out_distance_squared, u32* out_index, int* out_count) {
  if (!k->built) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_query: the index has not been built");
  if (max_result_count < 1 || max_result_count > kMaxResults) {
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_query: max_result_count must be in [1, 64]");
  }
  if (query_count == 0) return SM_OK;
  QueryArgs a{query_count, qx, qy, qz, radius_squared, radius_scale, state, include_completed, include_free, max_result_count,
              k->inverse_cell_size, k->table_size - 1, k->bucket_start, k->records, out_distance_squared, out_index,
              out_count};
  const u32 needed = (query_count + kQueryBlock / 32 - 1) / (kQueryBlock / 32);
  const int blocks = static_cast<int>(std::min<u32>(needed, 16u * k->sm_count));
  k_knn_query<<<blocks, kQueryBlock, 0, stream>>>(a);
  SM_CUDA(cudaGetLastError());
  return SM_OK;
}

// sm_knn_batch_host: one neighbour batch for a meshing iteration with host arrays on both sides.
int KnnBatchHost(sm_knn_index* k, cudaStream_t stream, u32 n, const float* x, const float* y, const float* z,
                 const float* radius_squared, float radius_factor_squared, float cell_size, int max_result_count,
                 float* out_distance_squared, u32* out_index, int* out_count) {
  if (n > k->capacity) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_batch_host: more points than the index was created for");
  if (max_result_count < 1 || max_result_count > kMaxResults) {
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_batch_host: max_result_count must be in [1, 64]");
  }
  if (!(radius_factor_squared > 0.f)) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_batch_host: radius_factor_squared must be positive");
  if (n == 0) return SM_OK;
  if (!(cell_size > 0.f)) {   // twice the largest query radius: a ball touches 8 cells
    float largest = 0.f;
    for (u32 i = 0; i < n; ++i) largest = std::max(largest, radius_squared[i]);
    if (!(largest > 0.f)) largest = 1.f;
    cell_size = 2.f * std::sqrt(largest * radius_factor_squared);
  }
  if (k->batch_points < n || k->batch_k < max_result_count) {
    SM_CUDA(cudaStreamSynchronize(stream));
    cudaFree(k->batch_rows); cudaFree(k->batch_distance_squared); cudaFree(k->batch_index); cudaFree(k->batch_count);
    k->batch_rows = nullptr; k->batch_distance_squared = nullptr; k->batch_index = nullptr; k->batch_count = nullptr;
    k->batch_points = 0;
    const size_t points = std::min<size_t>(k->capacity, std::max<size_t>(n, 1u << 16));
    const size_t width = static_cast<size_t>(std::max(max_result_count, k->batch_k));
    SM_CUDA(cudaMalloc(&k->batch_rows, sizeof(float) * 4 * points));
    SM_CUDA(cudaMalloc(&k->batch_distance_squared, sizeof(float) * width * points));
    SM_CUDA(cudaMalloc(&k->batch_index, sizeof(u32) * width * points));
    SM_CUDA(cudaMalloc(&k->batch_count, sizeof(int) * points));
    k->batch_points = static_cast<u32>(points);
    k->batch_k = static_cast<int>(width);
  }
  const size_t stride = k->batch_points;
  float* dx = k->batch_rows;
  float* dy = dx + stride;
  float* dz = dy + stride;
  float* dr = dz + stride;
  const size_t bytes = sizeof(float) * n;
  SM_CUDA(cudaMemcpyAsync(dx, x, bytes, cudaMemcpyHostToDevice, stream));
  SM_CUDA(cudaMemcpyAsync(dy, y, bytes, cudaMemcpyHostToDevice, stream));
  SM_CUDA(cudaMemcpyAsync(dz, z, bytes, cudaMemcpyHostToDevice, stream));
  SM_CUDA(cudaMemcpyAsync(dr, radius_squared, bytes, cudaMemcpyHostToDevice, stream));
  int status = KnnBuild(k, stream, n, dx, dy, dz, dr, nullptr, cell_size);
  if (status != SM_OK) return status;
  status = KnnQuery(k, stream, n, dx, dy, dz, dr, radius_factor_squared, nullptr, 1, 1, max_result_count,
                    k->batch_distance_squared, k->batch_index, k->batch_count);
  if (status != SM_OK) return status;
  // Results back through two pinned bounce buffers: the copy engine fills one chunk while the host moves the
  // previous one into the caller's (pageable) arrays - a direct copy into pageable memory runs at a few GB/s.
  constexpr u32 kChunk = 1u << 16;                                   // queries per chunk
  const size_t chunk_bytes = static_cast<size_t>(kChunk) * (kMaxResults * 8 + 4);
  for (int i = 0; i < 2; ++i) {
    if (!k->bounce[i]) SM_CUDA(cudaMallocHost(&k->bounce[i], chunk_bytes));
    if (!k->bounce_ready[i]) SM_CUDA(cudaEventCreateWithFlags(&k->bounce_ready[i], cudaEventDisableTiming));
  }
  const u32 chunks = (n + kChunk - 1) / kChunk;
  auto enqueue = [&](u32 c) -> int {
    const u32 first = c * kChunk, count = std::min(kChunk, n - first);
    const size_t row = static_cast<size_t>(count) * max_result_count;
    char* b = static_cast<char*>(k->bounce[c & 1]);
    SM_CUDA(cudaMemcpyAsync(b, k->batch_distance_squared + static_cast<size_t>(first) * max_result_count, sizeof(float) * row,
                            cudaMemcpyDeviceToHost, stream));
    SM_CUDA(cudaMemcpyAsync(b + sizeof(float) * row, k->batch_index + static_cast<size_t>(first) * max_result_count,
                            sizeof(u32) * row, cudaMemcpyDeviceToHost, stream));
    SM_CUDA(cudaMemcpyAsync(b + 2 * sizeof(float) * row, k->batch_count + first, sizeof(int) * count, cudaMemcpyDeviceToHost, stream));
    SM_CUDA(cudaEventRecord(k->bounce_ready[c & 1], stream));
    return SM_OK;
  };
  status = enqueue(0);
  if (status != SM_OK) return status;
  for (u32 c = 0; c < chunks; ++c) {
    if (c + 1 < chunks) {   // buffer (c + 1) & 1 was drained by the host in iteration c - 1
      status = enqueue(c + 1);
      if (status != SM_OK) return status;
    }
    SM_CUDA(cudaEventSynchronize(k->bounce_ready[c & 1]));
    const u32 first = c * kChunk, count = std::min(kChunk, n - first);
    const size_t row = static_cast<size_t>(count) * max_result_count;
    const char* b = static_cast<const char*>(k->bounce[c & 1]);
    std::memcpy(out_distance_squared + static_cast<size_t>(first) * max_result_count, b, sizeof(float) * row);
    std::memcpy(out_index + static_cast<size_t>(first) * max_result_count, b + sizeof(float) * row, sizeof(u32) * row);
    std::memcpy(out_count + first, b + 2 * sizeof(float) * row, sizeof(int) * count);
  }
  SM_CUDA(cudaStreamSynchronize(stream));
  return SM_OK;
}

}  // namespace smb

extern "C" {

int sm_knn_create(sm_knn_index** out, uint32_t max_points) {
  if (!out || max_points == 0 || max_points > (1u << 26)) {
    return smb::SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_create: need out and 1 <= max_points <= 2^26");
  }
  sm_knn_index* k = new sm_knn_index;
  const int status = smb::CreateIndex(k, max_points);
  if (status != SM_OK) {
    smb::FreeIndex(k);
    return status;
  }
  *out = k;
  return SM_OK;
}

void sm_knn_destroy(sm_knn_index* k) {
  if (k) smb::FreeIndex(k);
}

int sm_knn_build(sm_knn_index* k, void* stream, uint32_t point_count, const float* x, const float* y, const float* z,
                 const float* radius_squared, const uint8_t* state, float cell_size) {
  if (!k || (point_count && (!x || !y || !z))) return smb::SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_build: null argument");
  return smb::KnnBuild(k, static_cast<cudaStream_t>(stream), point_count, x, y, z, radius_squared, state, cell_size);
}

int sm_knn_build_from_reconstruction(sm_knn_index* k, sm_reconstruction* r, void* stream_v, float cell_size,
                                     uint32_t* out_point_count) {
  if (!k || !r) return smb::SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_build_from_reconstruction: null argument");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  uint32_t n = 0;
  const int status = sm_surfels_size(r, &n);
  if (status != SM_OK) return status;
  if (out_point_count) *out_point_count = n;
  // The positions the meshing thread sees are the smooth ones (TransferAllToCPU, cuda_surfel_reconstruction.cc:345-347),
  // read from their mirror in SoA rows 3-5.
  const size_t st = r->d.stride;
  const int mirrored = smb::MirrorRegRecords(stream, r->d, n, r->sm_count);
  if (mirrored != SM_OK) return mirrored;
  const float* s = r->d.surfels;
  return smb::KnnBuild(k, stream, n, s + SM_ROW_SMOOTH_X * st, s + SM_ROW_SMOOTH_Y * st, s + SM_ROW_SMOOTH_Z * st,
                       s + SM_ROW_RADIUS_SQUARED * st, nullptr, cell_size);
}

int sm_knn_query(sm_knn_index* k, void* stream, uint32_t query_count, const float* qx, const float* qy, const float* qz,
                 const float* radius_squared, const uint8_t* state, int32_t include_completed, int32_t include_free,
                 int32_t max_result_count, float* out_distance_squared, uint32_t* out_index, int32_t* out_count) {
  if (!k || (query_count && (!qx || !qy || !qz || !radius_squared || !out_distance_squared || !out_index || !out_count))) {
    return smb::SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_query: null argument");
  }
  return smb::KnnQuery(k, static_cast<cudaStream_t>(stream), query_count, qx, qy, qz, radius_squared, 1.0f, state,
                       include_completed, include_free, max_result_count, out_distance_squared, out_index, out_count);
}

int sm_knn_batch_host(sm_knn_index* k, void* stream, uint32_t point_count, const float* x, const float* y, const float* z,
                      const float* radius_squared, float radius_factor_squared, float cell_size, int32_t max_result_count,
                      float* out_distance_squared, uint32_t* out_index, int32_t* out_count) {
  if (!k || (point_count && (!x || !y || !z || !radius_squared || !out_distance_squared || !out_index || !out_count))) {
    return smb::SetError(SM_ERR_INVALID_ARGUMENT, "sm_knn_batch_host: null argument");
  }
  return smb::KnnBatchHost(k, static_cast<cudaStream_t>(stream), point_count, x, y, z, radius_squared, radius_factor_squared,
                           cell_size, max_result_count, out_distance_squared, out_index, out_count);
}

}  // extern "C"
