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
#include "sm_knn.cuh"
#include "sm_math.cuh"

namespace smb {

namespace {

#define SM_CUDA(call)                                                                                   \
  do {                                                                                                  \
    const cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) return SetError(SM_ERR_CUDA, (std::string(#call) + ": " + cudaGetErrorString(e_)).c_str()); \
  } while (0)

constexpr int kBuildBlock = 256;
constexpr int kQueryBlock = 128;           // 4 queries per block, one warp each

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

__global__ void __launch_bounds__(kBuildBlock) k_knn_scatter(BuildArgs a) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) {
    const u32 bucket = a.point_bucket[i];
    if (bucket == 0xFFFFFFFFu) continue;
    const u32 position = a.bucket_start[bucket] + atomicAdd(&a.bucket_cursor[bucket], 1u);
    a.records[position] = make_float4(a.x[i], a.y[i], a.z[i], __uint_as_float(i));
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
    warp_query(a, s, px, py, pz, radius_squared, lane);
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

int KnnCreate(sm_knn_index** out, u32 max_points) {
  sm_knn_index* k = new sm_knn_index;
  const int status = CreateIndex(k, max_points);
  if (status != SM_OK) {
    FreeIndex(k);
    return status;
  }
  *out = k;
  return SM_OK;
}

void KnnDestroy(sm_knn_index* k) {
  if (k) FreeIndex(k);
}

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
  return smb::KnnCreate(out, max_points);
}

void sm_knn_destroy(sm_knn_index* k) {
  smb::KnnDestroy(k);
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
