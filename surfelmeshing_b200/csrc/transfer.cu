// transfer.cu — hand-off of the surfel cloud to the CPU meshing thread (SURVEY §8 f1).
//
// Reference: CUDASurfelReconstruction::TransferAllToCPU (APP/cuda_surfel_reconstruction.cc:339-359)
// copies eight rows x surfels_size() floats into pageable arrays (CUDASurfelBuffersCPU,
// APP/cuda_surfels_cpu.h:40-73) every time, and the consumer (SurfelMeshing::IntegrateCUDABuffers,
// APP/surfel_meshing.cc:189-288) then compares every CPU surfel with the arrays.
//
// sm_transfer_all_to_cpu (api.cu) is that call 1:1. sm_transfer_delta_to_cpu below brings arrays
// that hold an EARLIER transfer up to date: one sweep selects the slots whose eight transferred
// attributes can have changed since that transfer, compacts {slot, smooth x y z, radius^2, normal,
// stamp} records into a device staging list (warp-aggregated reservation), one D2H copy moves the
// records into pinned memory and the host scatters them into the untouched CUDASurfelBuffersCPU
// layout. A slot can have changed if
//   * it did not exist at the earlier transfer (slot >= count then), or
//   * its last-update stamp is inside the regularisation window of any Integrate()/Regularize()
//     call since then (those calls move the smooth position of exactly the surfels with
//     stamp >= frame - window, kernels.cu:2132,2206; integration, replacement and creation set the
//     stamp to the frame index), or
//   * it was merged since then: k_integrate records the handle's operation epoch in the unused
//     row 14 of a surfel when it applies a merge (the merge itself resets the stamp to 0).
// This is a superset of the changed slots, so the arrays end up identical to a full transfer.

#include <algorithm>
#include <atomic>
#include <cstring>
#include <exception>
#include <string>
#include <thread>

#include "sm_handle.cuh"

namespace smb {

// The staging of sm_transfer_delta_to_cpu, created by the first delta transfer: the device record list (grown to
// surfels_size() in large steps) and its cursor, and the pinned host copy of the records.
struct TransferScratch {
  u32* index = nullptr; float* values = nullptr; u32* cursor = nullptr;
  u32 capacity = 0;
  u32* host = nullptr; size_t host_capacity = 0;   // in 32-bit words
};

namespace {

#define SM_S(row, i) d.surfels[static_cast<size_t>(row) * d.stride + (i)]
#define SM_SU(row, i) reinterpret_cast<u32*>(d.surfels)[static_cast<size_t>(row) * d.stride + (i)]

constexpr int kBlock = 256;

struct DeltaArgs {
  int count_slot;
  u32 count_at_token;     // surfels_size() at the earlier transfer
  int stamp_threshold;    // stamps >= this (signed compare, like the reference's window test) may have moved
  u32 epoch_at_token;     // merges recorded with a larger epoch happened since
  u32 capacity;           // records the staging list can hold
  u32* cursor;            // number of records written
  u32* index;             // [capacity]
  float* values;          // [8][capacity]: smooth x, y, z, radius^2, normal x, y, z, stamp (bits)
};

__global__ void __launch_bounds__(kBlock) k_delta_select(DeviceState d, DeltaArgs a) {
  const u32 n = d.counters->surfel_count[a.count_slot];
  const int lane = threadIdx.x & 31;
  for (u32 base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
    const u32 i = base + threadIdx.x;
    bool changed = false;
    u32 stamp = 0;
    float radius_squared = 0.f;
    if (i < n) {
      stamp = SM_SU(SM_ROW_LAST_UPDATE_STAMP, i);
      radius_squared = SM_S(SM_ROW_RADIUS_SQUARED, i);
      changed = i >= a.count_at_token || static_cast<int>(stamp) >= a.stamp_threshold ||
                (radius_squared < 0.f && SM_SU(kRowMergeEpoch, i) > a.epoch_at_token);
    }
    // warp-aggregated reservation: one atomic per warp, records of a warp stay in slot order
    const unsigned mask = __ballot_sync(0xffffffffu, changed);
    if (mask == 0) continue;
    u32 warp_base = 0;
    if (lane == 0) warp_base = atomicAdd(a.cursor, static_cast<u32>(__popc(mask)));
    warp_base = __shfl_sync(0xffffffffu, warp_base, 0);
    if (!changed) continue;
    const u32 k = warp_base + __popc(mask & ((1u << lane) - 1u));
    if (k >= a.capacity) continue;  // cannot happen: capacity >= surfels_size()
    a.index[k] = i;
    float* v = a.values + k;
    const size_t c = a.capacity;
    const float4 smooth = d.smooth[i];
    v[0 * c] = smooth.x;
    v[1 * c] = smooth.y;
    v[2 * c] = smooth.z;
    v[3 * c] = radius_squared;
    v[4 * c] = SM_S(SM_ROW_NORMAL_X, i);
    v[5 * c] = SM_S(SM_ROW_NORMAL_Y, i);
    v[6 * c] = SM_S(SM_ROW_NORMAL_Z, i);
    v[7 * c] = __uint_as_float(stamp);
  }
}

// ---------------------------------------------------------------------------------------------
// f3: visualisation buffers. The reference fills three CUDA-mapped OpenGL buffers with three sweeps
// over all slots (UpdateSurfelVertexBufferCUDAKernel<4 bools>, UpdateNeighborIndexBufferCUDAKernel,
// UpdateNormalVertexBufferCUDAKernel, kernels.cu:274-514); here ONE sweep reads every row once and
// writes whichever of the three (plain device) buffers the caller passes. Arithmetic as in the
// reference's compiled SASS: colour ramps are sat(fma) * 255.99 -> F2I.U32.TRUNC, the normal end point
// is fma(MUFU.SQRT(r^2), n, p).
// ---------------------------------------------------------------------------------------------
struct VizArgs {
  int count_slot;
  u32 frame_index;
  int active_window;
  u32 latest_triangulated_frame_index, latest_mesh_surfel_count;
  u32 point_size_in_floats;
  int mode;                 // 0 colour, 1 last-update age, 2 creation age, 3 radii, 4 normals
  float* vertex;            // [n][point_size_in_floats] or null
  u32* neighbor_index;      // [n][4][2] or null
  float* normal_vertex;     // [n][6] or null
};

__device__ __forceinline__ u32 pack_rgb(u32 r, u32 g, u32 b) { return (r & 0xFFu) | ((g & 0xFFu) << 8) | ((b & 0xFFu) << 16); }

__global__ void __launch_bounds__(kBlock) k_viz_buffers(DeviceState d, VizArgs a) {
  const u32 n = d.counters->surfel_count[a.count_slot];
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float4 smooth = d.smooth[i];
    const float sx = smooth.x, sy = smooth.y, sz = smooth.z;
    if (a.vertex) {
      // kernels.cu:287-351
      const u32 creation_stamp = SM_SU(SM_ROW_CREATION_STAMP, i);
      const bool output_vertex = creation_stamp <= a.latest_triangulated_frame_index || i >= a.latest_mesh_surfel_count;
      float* v = a.vertex + static_cast<size_t>(i) * a.point_size_in_floats;
      v[0] = output_vertex ? sx : __int_as_float(0x7fffffff);  // CUDART_NAN_F hides a replaced surfel's triangles
      v[1] = sy;
      v[2] = sz;
      u32 color;
      if (a.mode == 1 || a.mode == 2) {
        const u32 stamp = a.mode == 2 ? creation_stamp : SM_SU(SM_ROW_LAST_UPDATE_STAMP, i);
        const int age = static_cast<int>(a.frame_index - stamp);
        const int max_age = a.mode == 2 ? 3000 : a.active_window;
        if (age < 1) {
          color = pack_rgb(255, 80, 80);
        } else if (age > max_age) {
          color = pack_rgb(40, 40, 255);
        } else {
          const float blend = __saturatef(fmul(u2f(static_cast<u32>(age - 1)), frcp(u2f(static_cast<u32>(max_age - 1)))));
          const u32 intensity = 255u - (f2u_trunc(fmul(blend, 255.99f)) & 0xFFu);
          color = pack_rgb(intensity, intensity, intensity);
        }
      } else if (a.mode == 3) {
        const float radius = fsqrt_approx(SM_S(SM_ROW_RADIUS_SQUARED, i));
        const float blend = __saturatef(fmul(fadd(radius, -0.0005f), 105.26316070556640625f));  // 1 / (0.01 - 0.0005)
        const u32 red = f2u_trunc(fmul(blend, 255.99f)) & 0xFFu;
        color = pack_rgb(red, 255u - red, 80);
      } else if (a.mode == 4) {
        const u32 r8 = f2u_trunc(fmul(fadd(SM_S(SM_ROW_NORMAL_X, i), 1.0f), 127.99500274658203125f));
        const u32 g8 = f2u_trunc(fmul(fadd(SM_S(SM_ROW_NORMAL_Y, i), 1.0f), 127.99500274658203125f));
        const u32 b8 = f2u_trunc(fmul(fadd(SM_S(SM_ROW_NORMAL_Z, i), 1.0f), 127.99500274658203125f));
        color = pack_rgb(r8, g8, b8);
      } else {
        color = SM_SU(SM_ROW_COLOR, i);
      }
      v[3] = __uint_as_float(color);
    }
    if (a.neighbor_index) {
      // kernels.cu:434-449: line segments surfel -> neighbour (degenerate where there is none)
      uint4 lo, hi;
      const u32 n0 = SM_SU(SM_ROW_NEIGHBOR0 + 0, i), n1 = SM_SU(SM_ROW_NEIGHBOR0 + 1, i);
      const u32 n2 = SM_SU(SM_ROW_NEIGHBOR0 + 2, i), n3 = SM_SU(SM_ROW_NEIGHBOR0 + 3, i);
      lo = make_uint4(i, n0 == kInvalidIndex ? i : n0, i, n1 == kInvalidIndex ? i : n1);
      hi = make_uint4(i, n2 == kInvalidIndex ? i : n2, i, n3 == kInvalidIndex ? i : n3);
      uint4* out = reinterpret_cast<uint4*>(a.neighbor_index + static_cast<size_t>(i) * 8);  // 32 B per surfel: aligned
      out[0] = lo;
      out[1] = hi;
    }
    if (a.normal_vertex) {
      // kernels.cu:498-514
      const float radius = fsqrt_approx(SM_S(SM_ROW_RADIUS_SQUARED, i));
      float* o = a.normal_vertex + static_cast<size_t>(i) * 6;
      o[0] = sx; o[1] = sy; o[2] = sz;
      o[3] = ffma(radius, SM_S(SM_ROW_NORMAL_X, i), sx);
      o[4] = ffma(radius, SM_S(SM_ROW_NORMAL_Y, i), sy);
      o[5] = ffma(radius, SM_S(SM_ROW_NORMAL_Z, i), sz);
    }
  }
}

int FullTransfer(sm_reconstruction* r, cudaStream_t stream, u32 n, float* const out[7], uint32_t* stamp) {
  const size_t bytes = sizeof(float) * n;
  const float* s = r->d.surfels;
  const size_t st = r->d.stride;
  const int mirrored = MirrorRegRecords(stream, r->d, n, r->sm_count);   // rows 3-5 <- the current records
  if (mirrored != SM_OK) return mirrored;
  const float* src[7] = {s + SM_ROW_SMOOTH_X * st, s + SM_ROW_SMOOTH_Y * st, s + SM_ROW_SMOOTH_Z * st,
                         s + SM_ROW_RADIUS_SQUARED * st, s + SM_ROW_NORMAL_X * st, s + SM_ROW_NORMAL_Y * st,
                         s + SM_ROW_NORMAL_Z * st};
  for (int k = 0; k < 7; ++k) SM_CUDA(cudaMemcpyAsync(out[k], src[k], bytes, cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaMemcpyAsync(stamp, s + SM_ROW_LAST_UPDATE_STAMP * st, bytes, cudaMemcpyDeviceToHost, stream));
  return SM_OK;
}

}  // namespace

int UpdateVisualizationBuffers(sm_reconstruction* r, cudaStream_t stream, const sm_visualization_params& p, float* vertex,
                               uint32_t* neighbor_index, float* normal_vertex) {
  if (p.point_size_in_floats < 4 && vertex) return SetError(SM_ERR_INVALID_ARGUMENT, "point_size_in_floats < 4");
  if (neighbor_index && (reinterpret_cast<uintptr_t>(neighbor_index) & 15)) return SetError(SM_ERR_INVALID_ARGUMENT, "neighbor index buffer must be 16-byte aligned");
  VizArgs a;
  a.count_slot = r->count_slot;
  a.frame_index = p.frame_index;
  a.active_window = p.surfel_integration_active_window_size;
  a.latest_triangulated_frame_index = p.latest_triangulated_frame_index;
  a.latest_mesh_surfel_count = p.latest_mesh_surfel_count;
  a.point_size_in_floats = p.point_size_in_floats;
  // the reference's if / else-if chain (kernels.cu:404-414)
  a.mode = p.visualize_last_update_timestamp ? 1 : p.visualize_creation_timestamp ? 2 : p.visualize_radii ? 3 : p.visualize_normals ? 4 : 0;
  a.vertex = vertex; a.neighbor_index = neighbor_index; a.normal_vertex = normal_vertex;
  r->last_stream = stream;
  { LaunchScope scope(stream, KID_VIZ_BUFFERS); LaunchKernel(k_viz_buffers, dim3(r->sm_count * 8), dim3(kBlock), 0, stream, r->d, a); }
  return CheckLaunch("visualization buffers");
}

uint64_t NextStateGeneration() {
  // One counter for the whole process: a per-handle count would let a token filled from one handle (or from a
  // destroyed one) pass for another handle's cloud. 0 stays "never filled".
  static std::atomic<uint64_t> next{1};
  return next.fetch_add(1, std::memory_order_relaxed);
}

void RecordOperation(sm_reconstruction* r, int stamp_threshold) {
  ++r->op_epoch;
  r->op_history.push_back({r->op_epoch, stamp_threshold});
  if (r->op_history.size() > 8192) r->op_history.erase(r->op_history.begin(), r->op_history.begin() + 4096);
}

void FreeTransferBuffers(sm_reconstruction* r) {
  TransferScratch* s = r->transfer;
  if (!s) return;
  cudaFree(s->index); cudaFree(s->values); cudaFree(s->cursor);
  if (s->host) cudaFreeHost(s->host);
  delete s;
  r->transfer = nullptr;
}

int TransferDelta(sm_reconstruction* r, cudaStream_t stream, uint32_t frame_index, sm_transfer_token* token, float* x,
                  float* y, float* z, float* radius_squared, float* nx, float* ny, float* nz,
                  uint32_t* last_update_stamp, sm_transfer_stats* stats) {
  (void)frame_index;
  r->last_stream = stream;
  int status = FetchCounters(r, stream);
  if (status != SM_OK) return status;
  const u32 n = r->host_counters->surfel_count[r->count_slot];
  float* const out[7] = {x, y, z, radius_squared, nx, ny, nz};
  sm_transfer_stats st{};
  st.surfel_count = n;

  // Is the token usable? It must come from this handle's current cloud (no reset / load since) and
  // the operation history must reach back to it.
  bool full = token->generation != r->state_generation || token->epoch > r->op_epoch || token->surfel_count > n;
  int threshold = 0x7FFFFFFF;
  if (!full) {
    if (!r->op_history.empty() && r->op_history.front().epoch > token->epoch + 1) full = true;  // history was trimmed
    for (const auto& op : r->op_history)
      if (op.epoch > token->epoch) threshold = std::min(threshold, op.stamp_threshold);
  }
  if (!full && threshold <= 0) full = true;  // every stamp is inside a window: everything may have moved
  if (!full && n > 0) {
    if (!r->transfer) r->transfer = new TransferScratch();
    TransferScratch& s = *r->transfer;
    // staging list sized for the worst case (every slot changed), grown in large steps
    if (s.capacity < n) {
      SM_CUDA(cudaStreamSynchronize(stream));
      cudaFree(s.index); cudaFree(s.values);
      s.index = nullptr; s.values = nullptr;
      const size_t cap = std::min<size_t>(r->d.stride, std::max<size_t>(2 * static_cast<size_t>(n), 1u << 20));
      SM_CUDA(cudaMalloc(&s.index, sizeof(u32) * cap));
      SM_CUDA(cudaMalloc(&s.values, sizeof(float) * 8 * cap));
      s.capacity = static_cast<u32>(cap);
    }
    if (!s.cursor) SM_CUDA(cudaMalloc(&s.cursor, sizeof(u32)));
    SM_CUDA(cudaMemsetAsync(s.cursor, 0, sizeof(u32), stream));
    DeltaArgs a;
    a.count_slot = r->count_slot;
    a.count_at_token = static_cast<u32>(token->surfel_count);
    a.stamp_threshold = threshold;
    a.epoch_at_token = static_cast<u32>(token->epoch);
    a.capacity = s.capacity;
    a.cursor = s.cursor;
    a.index = s.index;
    a.values = s.values;
    { LaunchScope scope(stream, KID_DELTA_SELECT); LaunchKernel(k_delta_select, dim3(r->sm_count * 8), dim3(kBlock), 0, stream, r->d, a); }
    status = CheckLaunch("delta select");
    if (status != SM_OK) return status;
    u32 changed = 0;
    SM_CUDA(cudaMemcpyAsync(&changed, s.cursor, sizeof(u32), cudaMemcpyDeviceToHost, stream));
    SM_CUDA(cudaStreamSynchronize(stream));
    st.d2h_bytes += sizeof(u32);
    if (static_cast<size_t>(changed) * 9 > static_cast<size_t>(n) * 8) {
      full = true;  // the records (9 words each) would be more bytes than the eight rows
    } else if (changed > 0) {
      const size_t words = static_cast<size_t>(changed) * 9;
      if (s.host_capacity < words) {
        if (s.host) cudaFreeHost(s.host);
        s.host = nullptr;
        const size_t cap = std::max<size_t>(2 * words, 1u << 20);
        SM_CUDA(cudaMallocHost(&s.host, sizeof(u32) * cap));
        s.host_capacity = cap;
      }
      u32* host_index = s.host;
      float* host_values = reinterpret_cast<float*>(s.host + changed);
      SM_CUDA(cudaMemcpyAsync(host_index, s.index, sizeof(u32) * changed, cudaMemcpyDeviceToHost, stream));
      SM_CUDA(cudaMemcpy2DAsync(host_values, sizeof(float) * changed, s.values, sizeof(float) * s.capacity,
                                sizeof(float) * changed, 8, cudaMemcpyDeviceToHost, stream));
      SM_CUDA(cudaStreamSynchronize(stream));
      st.d2h_bytes += sizeof(u32) * words;
      // scatter into the CUDASurfelBuffersCPU arrays: the eight arrays are independent, four host threads take two
      // each once the list is long enough to pay for starting them
      u32* const dst_rows[8] = {reinterpret_cast<u32*>(x), reinterpret_cast<u32*>(y), reinterpret_cast<u32*>(z),
                                reinterpret_cast<u32*>(radius_squared), reinterpret_cast<u32*>(nx),
                                reinterpret_cast<u32*>(ny), reinterpret_cast<u32*>(nz), last_update_stamp};
      const u32* src_rows = reinterpret_cast<const u32*>(host_values);
      auto scatter_rows = [&](int first_row, int last_row) {
        for (int k = first_row; k < last_row; ++k) {
          const u32* v = src_rows + static_cast<size_t>(k) * changed;
          u32* dst = dst_rows[k];
          for (u32 j = 0; j < changed; ++j) dst[host_index[j]] = v[j];
        }
      };
      bool scattered = false;
      if (changed >= (1u << 16)) {
        std::thread workers[3];
        int started = 0;
        try {
          for (; started < 3; ++started) workers[started] = std::thread(scatter_rows, 2 * started + 2, 2 * started + 4);
        } catch (const std::exception&) {
          // no thread to be had (resource limit): the rows not handed out are done here
        }
        scatter_rows(0, 2);
        for (int t = 0; t < started; ++t) workers[t].join();
        if (started < 3) scatter_rows(2 * started + 2, 8);
        scattered = true;
      }
      if (!scattered) scatter_rows(0, 8);
    }
    st.changed_count = changed;
  }
  if (full) {
    if (n > 0) {
      status = FullTransfer(r, stream, n, out, last_update_stamp);
      if (status != SM_OK) return status;
      SM_CUDA(cudaStreamSynchronize(stream));
      st.d2h_bytes += static_cast<uint64_t>(n) * 8 * sizeof(float);
    }
    st.changed_count = n;
    st.full_transfer = 1;
  }
  token->generation = r->state_generation;
  token->epoch = r->op_epoch;
  token->surfel_count = n;
  if (stats) *stats = st;
  return SM_OK;
}

}  // namespace smb
