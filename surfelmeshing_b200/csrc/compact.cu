// compact.cu — sm_compact: reclaims the slots of merged surfels (include/surfel_b200.h, DESIGN.md section 5.13).
//
// The reference never frees the slot of a merged surfel (it marks it radius^2 = -1 and keeps sweeping it); this
// call removes those slots in place and keeps the order of the others:
//   k_compact_flags   1 per slot whose radius^2 is not below 0 (kept), into the row scratch
//   (CUB inclusive scan of the flags into the map)
//   k_compact_map     old_to_new[i] = scan[i] - 1 for a kept slot, SM_INVALID_SURFEL_INDEX for a removed one
//   k_compact_scatter one word of every kept record to its new slot in the row scratch (links remapped)
//   k_compact_store   the scratch back into the word's place
// Every SoA row goes through the one-row scratch (scatter, then store); the current regularisation records are
// scattered into the other record buffer and copied back, so both buffers hold the compacted records.

#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cstddef>
#include <string>
#include <type_traits>
#include <vector>

#include "sm_handle.cuh"

namespace smb {

struct CompactScratch {
  u32* map = nullptr;     // [capacity] old_to_new
  u32* row = nullptr;     // [capacity] the flags, then one word of every kept record
  u32 capacity = 0;
  void* scan_temp = nullptr; size_t scan_temp_bytes = 0;
  u32* words = nullptr;   // device: [0] kept slots, [1] dropped links, [2] [3] for the mesh (MeshCompact)
  u32* host = nullptr;    // pinned mirror of `words`
};

namespace {

constexpr int kCompactBlock = 256;

int Blocks(u32 n, int sm_count) {
  const u32 b = (n + kCompactBlock - 1) / kCompactBlock;
  return static_cast<int>(std::max<u32>(1u, std::min<u32>(b, static_cast<u32>(sm_count) * 8u)));
}

__global__ void __launch_bounds__(kCompactBlock) k_compact_flags(const float* radius_squared, u32 n, u32* flags) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    flags[i] = radius_squared[i] < 0.f ? 0u : 1u;   // the merge mark of k_integrate: radius^2 = -1
}

__global__ void __launch_bounds__(kCompactBlock) k_compact_map(const u32* flags, u32 n, u32* map, u32* kept) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const u32 inclusive = map[i];
    if (i == n - 1) *kept = inclusive;
    map[i] = flags[i] ? inclusive - 1u : kInvalidIndex;
  }
}

// dense[old_to_new[i]] = src[i * record_words + word] for every kept i < n. `remap`: the word names a slot, which is
// replaced by its new index (SM_INVALID_SURFEL_INDEX for a removed slot or one >= n, counted in *dropped unless it
// was SM_INVALID_SURFEL_INDEX already).
template <typename T>
__global__ void __launch_bounds__(kCompactBlock) k_compact_scatter(const T* src, u32 record_words, u32 word, const u32* map,
                                                                   u32 n, T* dense, bool remap, u32* dropped) {
  for (u32 base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
    const u32 i = base + threadIdx.x;
    bool drop = false;
    if (i < n) {
      const u32 k = map[i];
      if (k != kInvalidIndex) {
        T v = src[static_cast<size_t>(i) * record_words + word];
        if constexpr (std::is_same<T, u32>::value) {
          if (remap && v != kInvalidIndex) {
            const u32 to = v < n ? map[v] : kInvalidIndex;
            drop = to == kInvalidIndex;
            v = to;
          }
        }
        dense[k] = v;
      }
    }
    if (dropped) {
      const u32 count = __popc(__ballot_sync(0xffffffffu, drop));
      if ((threadIdx.x & 31) == 0 && count) atomicAdd(dropped, count);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kCompactBlock) k_compact_store(const T* dense, u32 kept, T* dst, u32 record_words, u32 word) {
  for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < kept; k += gridDim.x * blockDim.x)
    dst[static_cast<size_t>(k) * record_words + word] = dense[k];
}

template <typename T>
int CompactRecords(cudaStream_t stream, int sm_count, const u32* map, u32 n, u32 kept, T* base, u32 record_words,
                   T* scratch, bool remap, u32* dropped) {
  for (u32 w = 0; w < record_words; ++w) {
    {
      LaunchScope scope(stream, KID_COMPACT_SCATTER);
      LaunchKernel(k_compact_scatter<T>, dim3(Blocks(n, sm_count)), dim3(kCompactBlock), 0, stream, base, record_words, w,
                   map, n, scratch, remap, dropped);
    }
    if (kept > 0) {
      LaunchScope scope(stream, KID_COMPACT_STORE);
      LaunchKernel(k_compact_store<T>, dim3(Blocks(kept, sm_count)), dim3(kCompactBlock), 0, stream, scratch, kept, base,
                   record_words, w);
    }
  }
  return CheckLaunch("compact");
}

int EnsureCompactScratch(sm_reconstruction* r) {
  if (!r->compact) r->compact = new CompactScratch();
  CompactScratch& s = *r->compact;
  if (s.map) return SM_OK;
  const u32 cap = static_cast<u32>(r->d.stride);
  size_t temp = 0;
  SM_CUDA(cub::DeviceScan::InclusiveSum(nullptr, temp, static_cast<const u32*>(nullptr), static_cast<u32*>(nullptr),
                                        static_cast<int>(cap)));
  SM_CUDA(cudaMalloc(&s.words, 4 * sizeof(u32)));
  SM_CUDA(cudaMallocHost(&s.host, 4 * sizeof(u32)));
  SM_CUDA(cudaMalloc(&s.scan_temp, temp));
  s.scan_temp_bytes = temp;
  SM_CUDA(cudaMalloc(&s.row, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.map, sizeof(u32) * cap));
  s.capacity = cap;
  return SM_OK;
}

}  // namespace

int CompactWords(cudaStream_t stream, int sm_count, const u32* map, u32 n, u32 kept, u32* base, u32 record_words,
                 u32* scratch, bool remap) {
  return CompactRecords<u32>(stream, sm_count, map, n, kept, base, record_words, scratch, remap, nullptr);
}

int CompactBytes(cudaStream_t stream, int sm_count, const u32* map, u32 n, u32 kept, u8* base, u32* scratch) {
  return CompactRecords<u8>(stream, sm_count, map, n, kept, base, 1, reinterpret_cast<u8*>(scratch), false, nullptr);
}

void FreeCompactBuffers(sm_reconstruction* r) {
  CompactScratch* s = r->compact;
  if (!s) return;
  cudaFree(s->map); cudaFree(s->row); cudaFree(s->scan_temp); cudaFree(s->words);
  if (s->host) cudaFreeHost(s->host);
  delete s;
  r->compact = nullptr;
}

}  // namespace smb

using namespace smb;

extern "C" int sm_compact(sm_reconstruction* r, void* stream_v, uint32_t* old_to_new, uint64_t map_capacity,
                          sm_compact_stats* stats) {
  if (!r) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_compact: null handle");
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  r->last_stream = stream;
  int status = FetchCounters(r, stream);
  if (status == SM_ERR_CUDA) return status;   // (the sticky cap-overflow flag is no reason not to compact)
  const u32 n = r->host_counters->surfel_count[r->count_slot];
  // merged slots: what sm_surfel_count subtracts (in a frame-graph session, up to the newest integrated frame)
  const u32 merged = r->host_counters->merge_count;
  if (old_to_new && map_capacity < n) {
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_compact: map_capacity is below surfels_size()");
  }
  sm_compact_stats out{};
  out.slots_before = n;
  out.slots_after = n;
  if (merged == 0 || n == 0) {   // nothing to remove: no launch, no new state generation
    if (old_to_new && n > 0) {
      std::vector<u32> identity(n);
      for (u32 i = 0; i < n; ++i) identity[i] = i;
      SM_CUDA(cudaMemcpyAsync(old_to_new, identity.data(), sizeof(u32) * n, cudaMemcpyHostToDevice, stream));
      SM_CUDA(cudaStreamSynchronize(stream));
    }
    if (stats) *stats = out;
    return SM_OK;
  }
  status = EnsureCompactScratch(r);
  if (status != SM_OK) return status;
  CompactScratch& s = *r->compact;
  DeviceState& d = r->d;
  const int sms = r->sm_count;
  const size_t st = d.stride;
  u32* const rows = reinterpret_cast<u32*>(d.surfels);

  // the map
  SM_CUDA(cudaMemsetAsync(s.words, 0, 4 * sizeof(u32), stream));
  {
    LaunchScope scope(stream, KID_COMPACT_MAP);
    LaunchKernel(k_compact_flags, dim3(Blocks(n, sms)), dim3(kCompactBlock), 0, stream,
                 d.surfels + SM_ROW_RADIUS_SQUARED * st, n, s.row);
  }
  {
    LaunchScope scope(stream, KID_COMPACT_MAP);
    size_t temp = s.scan_temp_bytes;
    SM_CUDA(cub::DeviceScan::InclusiveSum(s.scan_temp, temp, static_cast<const u32*>(s.row), s.map, static_cast<int>(n),
                                          stream));
  }
  {
    LaunchScope scope(stream, KID_COMPACT_MAP);
    LaunchKernel(k_compact_map, dim3(Blocks(n, sms)), dim3(kCompactBlock), 0, stream, static_cast<const u32*>(s.row), n,
                 s.map, s.words);
  }
  SM_CUDA(cudaMemcpyAsync(s.host, s.words, sizeof(u32), cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaStreamSynchronize(stream));
  status = CheckLaunch("compact");
  if (status != SM_OK) return status;
  const u32 kept = s.host[0];
  if (old_to_new) SM_CUDA(cudaMemcpyAsync(old_to_new, s.map, sizeof(u32) * n, cudaMemcpyDeviceToDevice, stream));
  if (kept == n) {   // a merge count without merged slots (a loaded state): nothing changes
    SM_CUDA(cudaStreamSynchronize(stream));
    if (stats) *stats = out;
    return SM_OK;
  }
  {
    // every row of the SoA (the links of rows 19-22 remapped), through the row scratch
    for (int row = 0; row < SM_ROW_COUNT; ++row) {
      const bool link = row >= SM_ROW_NEIGHBOR0 && row < SM_ROW_NEIGHBOR0 + 4;
      status = CompactRecords<u32>(stream, sms, s.map, n, kept, rows + row * st, 1, s.row, link,
                                   link ? s.words + 1 : nullptr);
      if (status != SM_OK) return status;
    }
    // the current regularisation records into the other buffer, and back: both buffers hold them
    // (the gradient accumulators are zero between calls and stay so)
    {
      LaunchScope scope(stream, KID_COMPACT_SCATTER);
      LaunchKernel(k_compact_scatter<float4>, dim3(Blocks(n, sms)), dim3(kCompactBlock), 0, stream,
                   static_cast<const float4*>(d.smooth), 1u, 0u, static_cast<const u32*>(s.map), n, d.smooth_next,
                   false, static_cast<u32*>(nullptr));
    }
    if (kept > 0) SM_CUDA(cudaMemcpyAsync(d.smooth, d.smooth_next, sizeof(float4) * kept, cudaMemcpyDeviceToDevice, stream));
    status = CheckLaunch("compact");
    if (status != SM_OK) return status;
    d.reg_full_sweep = 1;   // as after sm_load_state
  }
  // surfels_size() = surfel_count() = kept, merge count 0 (the cap-overflow flag and the rest stay)
  for (int i = 0; i < kCountSlots; ++i) r->host_counters->surfel_count[i] = kept;
  r->host_counters->merge_count = 0;
  static_assert(offsetof(Counters, merge_count) == kCountSlots * sizeof(u32), "Counters layout");
  SM_CUDA(cudaMemcpyAsync(d.counters, r->host_counters, (kCountSlots + 1) * sizeof(u32), cudaMemcpyHostToDevice, stream));

  int mesh_remapped = 0;
  status = MeshCompact(r, stream, s.map, n, s.row, s.words + 2, s.host + 2, &mesh_remapped);
  if (status != SM_OK) return status;
  if (r->session) {
    status = SessionRefront(r, stream);   // the in-flight frame of a frame-graph session, on the new slots
    if (status != SM_OK) return status;
  }
  SM_CUDA(cudaMemcpyAsync(s.host + 1, s.words + 1, sizeof(u32), cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaStreamSynchronize(stream));
  r->state_generation = NextStateGeneration();   // tokens of earlier transfers no longer apply
  r->rasters_stale = true;                       // the rasters of the last Integrate name old slots
  out.slots_after = kept;
  out.merged_removed = n - kept;
  out.links_dropped = s.host[1];
  out.mesh_remapped = mesh_remapped;
  if (stats) *stats = out;
  return SM_OK;
}
