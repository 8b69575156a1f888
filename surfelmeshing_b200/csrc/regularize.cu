// regularize.cu — surfel regularisation for sm_90a (SURVEY §8 a14 + the second half of a12).
//
// Replaces RegularizeSurfelsCUDA (APP/cuda_surfel_reconstruction_kernels.cu:2099-2410: Clear,
// Accumulate, Step, Update = 4 sweeps over all slots) and
// UpdateNeighborsCUDARemoveReplacedNeighborsKernel (:1420-1437, a 5th sweep) by 2 sweeps:
//
//   k_reg_accumulate : [drop neighbour links to surfels with the detach flag] + Accumulate
//   k_reg_step       : gradient step (:2197-2290) from the current smooth buffer into the other one
//                      (= the reference's Update sweep, :2292-2308), accumulators reset to zero
//
// The gradient / weight accumulators (the reference's rows 11-13 and 23) live in one float4 record
// per slot (DeviceState::gradient) so that a neighbour contribution is one vector atomic.
// Invariant that makes the Clear sweep unnecessary: the records are zero between calls (new
// surfels are created with zeros, Accumulate only adds into surfels inside the regularisation
// window, and exactly those are reset by k_reg_step). The SoA rows 11-13 / 23 stay zero.
// Float atomics make the accumulated gradients order-dependent, as in the reference.
//
// Smooth positions live in 16-byte regularisation records {x, y, z, stamp | detach << 31}, double-buffered
// (DeviceState::smooth): a neighbour costs one gather (one 32-byte sector) in either sweep, where separate
// rows cost one sector per value.

#include <algorithm>

#include "sm_kernels.cuh"

namespace smb {

namespace {

#define SM_S(row, i) d.surfels[static_cast<size_t>(row) * d.stride + (i)]
#define SM_SU(row, i) reinterpret_cast<u32*>(d.surfels)[static_cast<size_t>(row) * d.stride + (i)]

constexpr int kBlock = 256;
// The two sweeps ask for a minimum of 1 resident block per SM: 64 and 56 registers, 4 blocks of 256 threads
// each. The explicit 1 is not the same as no minimum, which gives 60 and 46 registers. More resident warps
// cost spills: on an H100 at 400 W (tools/ab_probe.py, VGA stream, median of 5 passes) 6 blocks (40 registers,
// spills in both sweeps) ran 8 926 frames/s and 8 blocks (32 registers) 7 600, against 8 990-9 643 for 1.

struct RegParams {
  u32 frame_index;
  int window;                 // regularization_frame_window_size
  float radius_factor_squared;
  float regularizer_weight;
  int count_slot;
  int remove_below_slot;      // -1: no detach-flag pass
  int skip;                   // placeholder launch of the frame graph: return at once
  // k_reg_step writes smooth_next[i] only for a slot in the window or one that may differ between the two
  // buffers: int(stamp) >= t_prev (DeviceState::reg_t_prev), or every slot if full_sweep.
  int t_prev;
  int full_sweep;
};

// `stamp < frame_index - window` evaluated like the reference: the subtraction in u32, the
// comparison in int (kernels.cu:2132,2206).
__device__ __forceinline__ bool outside_window(u32 stamp, const RegParams& p) {
  return static_cast<int>(stamp) < static_cast<int>(p.frame_index - static_cast<u32>(p.window));
}

__global__ void __launch_bounds__(kBlock, 1) k_reg_accumulate(DeviceState d, RegParams p) {
  pdl_prologue();
  if (p.skip) return;
  const TimelineScope timeline_scope(d, p.frame_index, KID_REG_ACCUMULATE);
  const u32 n = d.counters->surfel_count[p.count_slot];
  const u32 n_remove = p.remove_below_slot >= 0 ? d.counters->surfel_count[p.remove_below_slot] : 0u;
  // The sweep is a chain of dependent gathers per surfel; the neighbour links (its first level)
  // are requested one round ahead, the first round's before the counts have arrived.
  const u32 step = gridDim.x * blockDim.x;
  u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  u32 nbr_ahead[4] = {kInvalidIndex, kInvalidIndex, kInvalidIndex, kInvalidIndex};
  if (i < d.stride) {
#pragma unroll
    for (int k = 0; k < 4; ++k) nbr_ahead[k] = SM_SU(SM_ROW_NEIGHBOR0 + k, i);
  }
  for (; i < n; i += step) {
    u32 nbr[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) nbr[k] = nbr_ahead[k];
    if (i + step < n) {
#pragma unroll
      for (int k = 0; k < 4; ++k) nbr_ahead[k] = SM_SU(SM_ROW_NEIGHBOR0 + k, i + step);
    }
    if ((nbr[0] & nbr[1] & nbr[2] & nbr[3]) == kInvalidIndex) continue;  // no neighbours at all

    // batch 1: the record of each neighbour (detach flag + stamp and smooth position in one 16-byte gather),
    // and this surfel's own attributes
    float4 rec[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const u32 q = nbr[k] != kInvalidIndex ? nbr[k] : i;
      rec[k] = d.smooth[q];
    }
    const float4 self = d.smooth[i];
    const float sx = self.x, sy = self.y, sz = self.z;
    const float nx = SM_S(SM_ROW_NORMAL_X, i), ny = SM_S(SM_ROW_NORMAL_Y, i), nz = SM_S(SM_ROW_NORMAL_Z, i);
    const float radius_squared = SM_S(SM_ROW_RADIUS_SQUARED, i);

    // UpdateNeighborsCUDARemoveReplacedNeighborsKernel (kernels.cu:1420-1437) for the slots
    // that existed before this frame, then the in-window count (kernels.cu:2125-2139).
    bool use[4];
    int neighbor_count = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const u32 meta = __float_as_uint(rec[k].w);
      if (i < n_remove && nbr[k] != kInvalidIndex && (meta & kMetaDetachBit)) {
        nbr[k] = kInvalidIndex;
        SM_SU(SM_ROW_NEIGHBOR0 + k, i) = kInvalidIndex;
      }
      use[k] = nbr[k] != kInvalidIndex && !outside_window(meta & ~kMetaDetachBit, p);
      neighbor_count += use[k] ? 1 : 0;
    }
    if (neighbor_count == 0) continue;

    const float max_distance_squared = fmul(radius_squared, p.radius_factor_squared);
    const float rcp_count = frcp(i2f(neighbor_count));
    const float factor = fmul(fadd(p.regularizer_weight, p.regularizer_weight), rcp_count);  // 2 * w / count
    const float weight_term = fmul(rcp_count, p.regularizer_weight);                         // w / count
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (!use[k]) continue;
      const u32 q = nbr[k];
      const float dx = fsub(rec[k].x, sx);
      const float dy = fsub(rec[k].y, sy);
      const float dz = fsub(rec[k].z, sz);
      const float f = fmul(factor, ffma(nz, dz, ffma(nx, dx, fmul(ny, dy))));
      // kernels.cu:2173-2176: four float atomicAdds; here one 16-byte vector atomic (sm_90+), the
      // same four fp32 additions in the same (arbitrary) arrival order
      atomicAdd(&d.gradient[q], make_float4(fmul(nx, f), fmul(ny, f), fmul(nz, f), weight_term));
      // If the neighbour is too far away, remove it (kernels.cu:2184-2192).
      if (squared_norm(dx, dy, dz) > max_distance_squared) SM_SU(SM_ROW_NEIGHBOR0 + k, i) = kInvalidIndex;
    }
  }
}

__global__ void __launch_bounds__(kBlock, 1) k_reg_step(DeviceState d, RegParams p) {
  pdl_prologue();
  if (p.skip) return;
  const TimelineScope timeline_scope(d, p.frame_index, KID_REG_STEP);
  const u32 n = d.counters->surfel_count[p.count_slot];
  // The stamp (first level of the gather chain) is requested one round ahead.
  const u32 step = gridDim.x * blockDim.x;
  u32 i = blockIdx.x * blockDim.x + threadIdx.x;
  u32 stamp_ahead = 0;
  if (i < d.stride) stamp_ahead = SM_SU(SM_ROW_LAST_UPDATE_STAMP, i);
  for (; i < n; i += step) {
    const u32 stamp = stamp_ahead;
    if (i + step < n) stamp_ahead = SM_SU(SM_ROW_LAST_UPDATE_STAMP, i + step);
    if (outside_window(stamp, p)) {
      // Not regularised (kernels.cu:2206): the smooth position carries over to the next buffer. It already
      // is there unless the previous sweep moved it (DeviceState::reg_t_prev; stamps below t_prev were below
      // that sweep's threshold too, and every other writer of smooth positions writes both buffers).
      if (p.full_sweep || static_cast<int>(stamp) >= p.t_prev) d.smooth_next[i] = d.smooth[i];
      continue;
    }
    u32 nbr[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) nbr[k] = SM_SU(SM_ROW_NEIGHBOR0 + k, i);
    const float4 self = d.smooth[i];
    const float sx = self.x, sy = self.y, sz = self.z;
    const float nx = SM_S(SM_ROW_NORMAL_X, i), ny = SM_S(SM_ROW_NORMAL_Y, i), nz = SM_S(SM_ROW_NORMAL_Z, i);
    // Data term (factor 2) + neighbour-induced terms.
    const float4 accumulated = d.gradient[i];
    float gx = ffma(fsub(sx, SM_S(SM_ROW_X, i)), 2.0f, accumulated.x);
    float gy = ffma(fsub(sy, SM_S(SM_ROW_Y, i)), 2.0f, accumulated.y);
    float gz = ffma(fsub(sz, SM_S(SM_ROW_Z, i)), 2.0f, accumulated.z);
    int neighbor_count = 0;
    float rx = 0.f, ry = 0.f, rz = 0.f;
    float4 rec[4];   // smooth positions of the neighbours: one 16-byte gather each
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const u32 q = nbr[k] != kInvalidIndex ? nbr[k] : i;
      rec[k] = d.smooth[q];
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (nbr[k] == kInvalidIndex) continue;
      ++neighbor_count;
      const float dx = fsub(rec[k].x, sx);
      const float dy = fsub(rec[k].y, sy);
      const float dz = fsub(rec[k].z, sz);
      const float normal_dot_difference = ffma(nz, dz, ffma(nx, dx, fmul(ny, dy)));
      rx = ffma(-nx, normal_dot_difference, rx);
      ry = ffma(-ny, normal_dot_difference, ry);
      rz = ffma(-nz, normal_dot_difference, rz);
    }
    if (neighbor_count > 0) {
      const float factor = fmul(fadd(p.regularizer_weight, p.regularizer_weight), frcp(i2f(neighbor_count)));
      gx = ffma(factor, rx, gx);
      gy = ffma(factor, ry, gy);
      gz = ffma(factor, rz, gz);
    }
    const float gradient_length = fsqrt_approx(ffma(gz, gz, ffma(gx, gx, fmul(gy, gy))));
    const float residual_terms_weight_sum = fadd(fadd(p.regularizer_weight, 1.0f), accumulated.w);
    float step_factor = fmul(frcp(residual_terms_weight_sum), 0.5f);
    const float max_step_length = fsqrt_approx(SM_S(SM_ROW_RADIUS_SQUARED, i));
    const float step_length = fmul(step_factor, gradient_length);
    if (step_length > max_step_length) step_factor = fmul(step_factor, fmul(max_step_length, frcp(step_length)));
    // The new smooth position goes to the other buffer (the neighbours still read the old one), with the
    // meta word carried over; this surfel's accumulator, read by nobody else in this sweep, is reset for
    // the next call.
    d.smooth_next[i] = make_float4(ffma(step_factor, -gx, sx), ffma(step_factor, -gy, sy), ffma(step_factor, -gz, sz), self.w);
    d.gradient[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// RegularizeSurfelsCUDACopyOnlyKernel (kernels.cu:2310-2327) [+ detach-flag pass].
__global__ void __launch_bounds__(kBlock) k_reg_copy_only(DeviceState d, RegParams p) {
  pdl_prologue();
  if (p.skip) return;
  const TimelineScope timeline_scope(d, p.frame_index, KID_REG_COPY_ONLY);
  const u32 n = d.counters->surfel_count[p.count_slot];
  const u32 n_remove = p.remove_below_slot >= 0 ? d.counters->surfel_count[p.remove_below_slot] : 0u;
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    if (i < n_remove) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const u32 q = SM_SU(SM_ROW_NEIGHBOR0 + k, i);
        if (q != kInvalidIndex && (SM_SU(SM_ROW_COLOR, q) >> 24) == 1u) SM_SU(SM_ROW_NEIGHBOR0 + k, i) = kInvalidIndex;
      }
    }
    if (outside_window(SM_SU(SM_ROW_LAST_UPDATE_STAMP, i), p)) continue;
    // both buffers (see RegParams::t_prev), meta word unchanged
    const float4 record = make_float4(SM_S(SM_ROW_X, i), SM_S(SM_ROW_Y, i), SM_S(SM_ROW_Z, i), d.smooth[i].w);
    d.smooth[i] = record;
    d.smooth_next[i] = record;
  }
}

}  // namespace

namespace {
__global__ void __launch_bounds__(kBlock) k_reg_pack(DeviceState d, u32 count) {
  pdl_prologue();
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
    const u32 flag = (SM_SU(SM_ROW_COLOR, i) >> 24) == 1u ? kMetaDetachBit : 0u;
    const u32 meta = (SM_SU(SM_ROW_LAST_UPDATE_STAMP, i) & ~kMetaDetachBit) | flag;
    const float4 record = make_float4(SM_S(SM_ROW_SMOOTH_X, i), SM_S(SM_ROW_SMOOTH_Y, i), SM_S(SM_ROW_SMOOTH_Z, i),
                                      __uint_as_float(meta));
    d.smooth[i] = record;
    d.smooth_next[i] = record;
  }
}

__global__ void __launch_bounds__(kBlock) k_reg_mirror(DeviceState d, u32 count) {
  pdl_prologue();
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
    const float4 record = d.smooth[i];
    SM_S(SM_ROW_SMOOTH_X, i) = record.x;
    SM_S(SM_ROW_SMOOTH_Y, i) = record.y;
    SM_S(SM_ROW_SMOOTH_Z, i) = record.z;
    SM_SU(kRowMeta, i) = __float_as_uint(record.w);
  }
}
}  // namespace

int PackRegRecords(cudaStream_t stream, const DeviceState& d, u32 count, int sm_count) {
  if (count == 0) return SM_OK;
  { LaunchScope scope(stream, KID_REG_PACK); LaunchKernel(k_reg_pack, dim3(sm_count * 4), dim3(kBlock), 0, stream, d, count); }
  return CheckLaunch("pack regularisation records");
}

int MirrorRegRecords(cudaStream_t stream, const DeviceState& d, u32 count, int sm_count) {
  if (count == 0) return SM_OK;
  { LaunchScope scope(stream, KID_REG_MIRROR); LaunchKernel(k_reg_mirror, dim3(sm_count * 4), dim3(kBlock), 0, stream, d, count); }
  return CheckLaunch("mirror regularisation records");
}

int DescribeRegularize(KernelLaunch* first, KernelLaunch* second, bool skip, const LaunchPlan& plan,
                       const DeviceState& d, bool disable_denoising, u32 frame_index,
                       float radius_factor_for_regularization_neighbors, float regularizer_weight,
                       int regularization_frame_window_size, int count_slot, int remove_replaced_below_slot) {
  RegParams p;
  p.frame_index = frame_index;
  p.window = regularization_frame_window_size;
  p.radius_factor_squared =
      radius_factor_for_regularization_neighbors * radius_factor_for_regularization_neighbors;  // kernels.cu:2379
  p.regularizer_weight = regularizer_weight;
  p.count_slot = count_slot;
  p.remove_below_slot = remove_replaced_below_slot;
  p.skip = skip ? 1 : 0;
  p.t_prev = d.reg_t_prev;
  p.full_sweep = d.reg_full_sweep;
  static_assert(sizeof(DeviceState) + sizeof(RegParams) + 32 <= sizeof(first->storage), "KernelLaunch::storage too small");
  if (disable_denoising) {
    first->Reset(reinterpret_cast<const void*>(k_reg_copy_only), dim3(plan.reg_copy), dim3(kBlock), 0, KID_REG_COPY_ONLY);
    first->Arg(d);
    first->Arg(p);
    return 1;
  }
  first->Reset(reinterpret_cast<const void*>(k_reg_accumulate), dim3(plan.reg_accumulate), dim3(kBlock), 0, KID_REG_ACCUMULATE);
  first->Arg(d);
  first->Arg(p);
  second->Reset(reinterpret_cast<const void*>(k_reg_step), dim3(plan.reg_step), dim3(kBlock), 0, KID_REG_STEP);
  second->Arg(d);
  second->Arg(p);
  return 2;
}

int RegularizeSurfels(cudaStream_t stream, DeviceState& d, bool disable_denoising, u32 frame_index,
                      float radius_factor_for_regularization_neighbors, float regularizer_weight,
                      int regularization_frame_window_size, int count_slot, int remove_replaced_below_slot,
                      const LaunchPlan& plan) {
  KernelLaunch first, second;
  const int n = DescribeRegularize(&first, &second, false, plan, d, disable_denoising, frame_index,
                                   radius_factor_for_regularization_neighbors, regularizer_weight,
                                   regularization_frame_window_size, count_slot, remove_replaced_below_slot);
  LaunchOnStream(stream, first, false);
  if (n == 1) return CheckLaunch("regularize (copy only)");
  LaunchOnStream(stream, second, true);
  // k_reg_step completed the other smooth buffer: it is the current one from here on
  float4* const filled = d.smooth_next;
  d.smooth_next = d.smooth;
  d.smooth = filled;
  NoteRegStep(d, frame_index, regularization_frame_window_size);
  return CheckLaunch("regularize");
}

// Per-device configuration: the shared-memory carve-out of every kernel of the file
// (kSharedMemoryCarveoutPercent) and grids = the blocks resident at once (ResidentBlocks).
int ConfigureRegularizeKernels(LaunchPlan* plan) {
  const int carveout_percent = kSharedMemoryCarveoutPercent;
  cudaFuncSetAttribute(k_reg_accumulate, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_reg_step, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_reg_copy_only, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaGetLastError();
  int status = ResidentBlocks(k_reg_accumulate, kBlock, plan->sm_count, &plan->reg_accumulate);
  if (status == SM_OK) status = ResidentBlocks(k_reg_step, kBlock, plan->sm_count, &plan->reg_step);
  if (status == SM_OK) status = ResidentBlocks(k_reg_copy_only, kBlock, plan->sm_count, &plan->reg_copy);
  return status;
}

}  // namespace smb
