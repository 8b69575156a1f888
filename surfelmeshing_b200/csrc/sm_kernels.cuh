// sm_kernels.cuh — declarations shared by the translation units of libsurfel_b200.so.
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include <string>

#include "../../include/surfel_b200.h"
#include "sm_math.cuh"

namespace smb {

// ---- error / bookkeeping (api.cu) ---------------------------------------------------------
int SetError(int code, const char* message);
int CheckLaunch(const char* what);   // cudaGetLastError() -> SM_OK / SM_ERR_CUDA
// A failed CUDA call returns SM_ERR_CUDA from the enclosing function, "<call>: <CUDA's message>" in sm_last_error().
#define SM_CUDA(call)                                                                                   \
  do {                                                                                                  \
    const cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) return smb::SetError(SM_ERR_CUDA, (std::string(#call) + ": " + cudaGetErrorString(e_)).c_str()); \
  } while (0)

// Every kernel launch of the library goes through a LaunchScope: it counts the launch
// (sm_kernel_launch_count) and, while sm_profile_kernels(1) is active, brackets it with CUDA
// events on the launching stream so that bench.py can report per-kernel durations measured
// live (never used inside a timed throughput region).
enum KernelId {
  KID_CLEAR = 0, KID_BILATERAL_OUTLIER, KID_BILATERAL_GENERIC, KID_OUTLIER, KID_ERODE_NORMALS_RADII, KID_ERODE,
  KID_NORMALS, KID_RADII, KID_PROJECT, KID_ASSOCIATE, KID_MERGE, KID_BLEND, KID_INTEGRATE, KID_UPDATE_NEIGHBORS,
  KID_NEW_SURFEL_SCAN, KID_CREATE_SURFELS, KID_REG_ACCUMULATE, KID_REG_STEP, KID_REG_COPY_ONLY,
  KID_EXPORT_VERTICES, KID_MEDIAN_DENSIFY, KID_DELTA_SELECT, KID_VIZ_BUFFERS, KID_DOWNSCALE_DEPTH, KID_DOWNSCALE_COLOR,
  KID_REG_MIRROR, KID_REG_PACK,
  // The kernels below this id have a column in the device timeline (DeviceState::timeline, [frame][column]); the
  // render kernels (render.cu), the tracking kernels (track.cu) and the meshing kernels (mesh.cu) run outside the
  // frame pipeline and have none.
  KID_TIMELINE_COUNT,
  KID_RENDER_SPLAT = KID_TIMELINE_COUNT, KID_RENDER_LARGE, KID_RENDER_RESOLVE,
  KID_TRACK_LIVE_VIEW, KID_TRACK_LINEARIZE, KID_TRACK_SOLVE,
  KID_MESH_BOUND, KID_MESH_UMBRELLA, KID_MESH_COUNT, KID_MESH_SCAN, KID_MESH_WRITE,
  KID_MESH_CHANGES, KID_MESH_MARK, KID_MESH_OWNERS, KID_MESH_UMBRELLA_UPDATE, KID_MESH_RECHECK, KID_MESH_RECHECK_WRITE,
  KID_MESH_RENDER_MARK, KID_MESH_RENDER_TRI, KID_MESH_RENDER_LARGE, KID_MESH_RENDER_SPLAT, KID_MESH_RENDER_SPLAT_LARGE,
  KID_MESH_RENDER_RESOLVE,
  KID_TRACK_INTENSITY_BASE, KID_TRACK_INTENSITY_DOWN, KID_TRACK_LINEARIZE_RGBD, KID_TRACK_SOLVE_RGBD,
  KID_RELOC_ENCODE, KID_RELOC_DISTANCE, KID_RELOC_SELECT,
  KID_HOLE_EDGES, KID_HOLE_BOUNDARY, KID_HOLE_SORT, KID_HOLE_WALK, KID_HOLE_CONFLICT, KID_HOLE_SCAN, KID_HOLE_WRITE,
  KID_COMPACT_MAP, KID_COMPACT_SCATTER, KID_COMPACT_STORE, KID_COMPACT_MESH,
  KID_SIMPLIFY_EDGES, KID_SIMPLIFY_FANS, KID_SIMPLIFY_SORT, KID_SIMPLIFY_QUADRICS, KID_SIMPLIFY_CANDIDATES,
  KID_SIMPLIFY_SELECT, KID_SIMPLIFY_APPLY, KID_SIMPLIFY_SCAN, KID_SIMPLIFY_WRITE,
  KID_TEXTURE_CLASSES, KID_TEXTURE_SORT, KID_TEXTURE_PLACE, KID_TEXTURE_UV, KID_TEXTURE_ACCUMULATE, KID_TEXTURE_RESOLVE,
  KID_TEXTURE_GAIN_SAMPLE, KID_TEXTURE_GAIN_COUNT, KID_TEXTURE_GAIN_POINTS, KID_TEXTURE_GAIN_VIEWS, KID_TEXTURE_GAIN_STEP,
  KID_COMPONENTS_EDGES, KID_COMPONENTS_HOOK, KID_COMPONENTS_NUMBER, KID_COMPONENTS_SCAN, KID_COMPONENTS_SUMS,
  KID_COMPONENTS_RANK, KID_COMPONENTS_WRITE,
  KID_COUNT
};
const char* KernelName(int id);
bool ProfilingEnabled();
class LaunchScope {
 public:
  LaunchScope(cudaStream_t stream, KernelId id);
  ~LaunchScope();
 private:
  cudaStream_t stream_;
  int slot_;
};

inline Mat3x4 MakeMat3x4(const float* m) {
  Mat3x4 r;
  r.r0 = make_float4(m[0], m[1], m[2], m[3]);
  r.r1 = make_float4(m[4], m[5], m[6], m[7]);
  r.r2 = make_float4(m[8], m[9], m[10], m[11]);
  return r;
}

// ---- device-side state shared by the Integrate kernels -------------------------------------

constexpr u32 kInvalidIndex = 0xFFFFFFFFu;   // APP/surfel.h:63, kernels.cu:74

// Rows 14-16 of the SoA ("accum", kernels.cuh:66-68) are never touched by the reference. Two of them
// carry bookkeeping here (sm_dump_state callers treat rows 11-16 and 23 as scratch):
//   row 14  operation epoch at which the surfel was merged (delta transfer, transfer.cu)
//   row 15  export mirror of the "meta" word of the regularisation record (DeviceState::smooth):
//           last-update stamp | detach flag << 31. Written only by MirrorRegRecords before a dump,
//           transfer or k-NN build; scratch otherwise.
// Stamps are frame indices < kFrameIndexLimit, which the entry points enforce: bit 31 of the meta word is free for
// the detach flag, and k_reg_accumulate's window test on the meta word equals the reference's on the whole stamp.
constexpr int kRowMergeEpoch = SM_ROW_ACCUM_X;
constexpr int kRowMeta = SM_ROW_ACCUM_Y;
constexpr u32 kMetaDetachBit = 0x80000000u;
constexpr u32 kFrameIndexLimit = 0x80000000u;

// The meta word (.w) of a regularisation record, stored on its own (4 bytes at offset 12 of the record).
__device__ __forceinline__ void store_reg_meta(float4* records, u32 i, u32 meta) {
  reinterpret_cast<u32*>(records + i)[3] = meta;
}
constexpr int kSegment = 1024;               // surfel slots per list segment (one block-iteration)
constexpr u32 kActiveBit = 0x80000000u;      // VisEntry.idx: surfel was active at projection time

// PixelAssoc.x while a frame is processed: the arrival key of the winning association. The
// reference lets the first atomicCAS win (kernels.cu:1688): which of several supporters of a pixel
// becomes its supporting surfel is a race. The product takes the minimum of a key that orders the
// associations the way the reference's race resolves ON AVERAGE (measured on an H100, tools/race_stats.py,
// DESIGN.md section 4) and is reproducible. Most significant first:
//   wave   slots are grouped into launch waves of W slots (the reference's 1024-thread blocks are
//          scheduled in slot order; of two supporters in different waves the earlier wave won
//          16 569 times out of 16 569);
//   late   set for a secondary-pixel association (a reference thread handles its primary pixel first:
//          inside a wave a secondary beat a primary in 2.9 % of the contests) - except for a
//          pseudo-random fraction `early` of them, which compete like primaries;
//   order  inside a wave: slot order for a pseudo-random fraction of the PIXELS (per frame), a per-frame
//          pseudo-random permutation of the slots for the others (the lower slot won 74 % of the
//          same-kind pairs, whatever their distance).
// W = 0 selects the plain rule of round 1: late (= secondary) first, then lowest slot index.
constexpr u32 kSecondaryBit = 0x80000000u;
struct TieBreak {
  u32 wave;             // W: slots per wave (0: plain rule)
  u32 lane_shift;       // log2 of the slots that keep their order inside the shuffled order (5: a warp of the reference; 0: none)
  u32 groups;           // W >> lane_shift
  u32 mul, mul_inv;     // perm(g) = (g * mul + add) mod groups, mul * mul_inv = 1 (mod groups)
  u32 add;              // per frame
  u32 salt;             // per frame, for the two draws
  u32 early_threshold;  // secondary association is NOT late iff hash(slot ^ salt) < early_threshold (slots of the first wave)
  u32 index_order_threshold;  // pixel uses slot order iff hash(pixel ^ ~salt) < index_order_threshold (first wave)
  u32 early_threshold_second;                              // the early threshold of the SECOND wave (partly filled at VGA sizes)
  u32 early_threshold_later, index_order_threshold_later;  // the same for the later waves: their blocks start one by one as
                                                           // earlier ones retire, so arrival follows the slot order more closely
                                                           // and a secondary association of an early block is ahead more often
  u32 wave_offset;      // 1: the wave boundaries sit at a per-pixel pseudo-random phase (whole groups) instead of at multiples of W
  u64 wave_reciprocal;  // floor((2^64 - 1) / W): division / modulo by W as a multiply (Barrett)
  u64 group_reciprocal; // the same for `groups`
};
// x / d and x % d for x < 2^62 without a hardware division (d is a run-time value, reciprocal = (2^64 - 1) / d).
__host__ __device__ __forceinline__ u64 tb_divide(u64 x, u32 d, u64 reciprocal, u32* remainder) {
#if defined(__CUDA_ARCH__)
  u64 q = __umul64hi(x, reciprocal);
#else
  u64 q = static_cast<u64>((static_cast<unsigned __int128>(x) * reciprocal) >> 64);
#endif
  u64 r = x - q * d;
  while (r >= d) { r -= d; ++q; }   // the truncated reciprocal leaves q at most 2 short
  *remainder = static_cast<u32>(r);
  return q;
}
__host__ __device__ __forceinline__ u32 tb_hash(u32 x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}
__host__ __device__ __forceinline__ bool tb_index_order(const TieBreak& t, u32 pixel, u32 wave_index) {
  return tb_hash(pixel ^ ~t.salt) < (wave_index == 0 ? t.index_order_threshold : t.index_order_threshold_later);
}
// Arrival key of a supporter: wave-major; inside a wave primary before (most) secondary associations; inside a
// kind either slot order or, per pixel, a shuffled order of the wave's warps in which the lanes of one warp keep
// their order (two lanes of one warp of the reference issue their compare-and-swap in lane order).
// Phase of the wave boundaries for one pixel, in slots (a whole number of groups). The blocks of the reference's
// launch do not start in lock step: two supporters d slots apart are ordered by slot with a probability that grows
// with d and reaches 1 at d = W. Cutting the slot axis into waves at a per-pixel random phase gives exactly that:
// the pair falls into different waves (ordered) with probability d / W and into one wave (shuffled) otherwise.
__host__ __device__ __forceinline__ u32 tb_phase(const TieBreak& t, u32 pixel) {
  if (!t.wave_offset) return 0u;
  u32 g;
  tb_divide(tb_hash(pixel ^ t.salt ^ 0x5bd1e995u), t.groups, t.group_reciprocal, &g);
  return g << t.lane_shift;
}
__host__ __device__ __forceinline__ u32 tb_encode(const TieBreak& t, u32 idx, bool secondary, u32 pixel) {
  if (t.wave == 0) return idx | (secondary ? kSecondaryBit : 0u);
  u32 r, rp;
  const u32 w = static_cast<u32>(tb_divide(static_cast<u64>(idx) + tb_phase(t, pixel), t.wave, t.wave_reciprocal, &r));
  if (tb_index_order(t, pixel, w)) {
    rp = r;
  } else {
    u32 gp;
    tb_divide(static_cast<u64>(r >> t.lane_shift) * t.mul + t.add, t.groups, t.group_reciprocal, &gp);
    rp = (gp << t.lane_shift) | (r & ((1u << t.lane_shift) - 1u));
  }
  const bool late = secondary && !(tb_hash(idx ^ t.salt) <
                                   (w == 0 ? t.early_threshold : (w == 1 ? t.early_threshold_second : t.early_threshold_later)));
  return w * (2u * t.wave) + (late ? t.wave : 0u) + rp;   // < 2^32 - 1: checked by SetTieBreakWave
}
__host__ __device__ __forceinline__ u32 supporting_index(const TieBreak& t, u32 key, u32 pixel) {
  if (key == kInvalidIndex) return kInvalidIndex;
  if (t.wave == 0) return key & ~kSecondaryBit;
  u32 rem;
  const u32 w2 = static_cast<u32>(tb_divide(key, t.wave, t.wave_reciprocal, &rem));   // key = (2 w + late) W + perm
  const u32 w = w2 >> 1;
  u32 r = rem;
  if (!tb_index_order(t, pixel, w)) {
    const u32 gp = rem >> t.lane_shift;
    const u32 shifted = gp >= t.add ? gp - t.add : gp + t.groups - t.add;
    u32 g;
    tb_divide(static_cast<u64>(shifted) * t.mul_inv, t.groups, t.group_reciprocal, &g);
    r = (g << t.lane_shift) | (rem & ((1u << t.lane_shift) - 1u));
  }
  return w * t.wave + r - tb_phase(t, pixel);
}

// Per-pixel association record (the reference keeps four separate rasters,
// APP/cuda_surfel_reconstruction.h:138-142): one 128-bit load/store per pixel.
//   x = supporting surfel, y = conflicting surfel, z = supporting count, w = depth sum (fp32 bits)
typedef uint4 PixelAssoc;

// Entry of the per-frame list of surfels that project into the image (z > 0, inside the
// image): surfel index (| kActiveBit) and camera-space position. Segment s owns list
// positions [s * kSegment, s * kSegment + seg_count[s]) and holds, in slot order, the visible
// surfels of slots [s * kSegment, (s + 1) * kSegment): the list needs no global atomic and
// is deterministic.
typedef uint4 VisEntry;

// surfel_count is a 3-slot history: frame f reads slot s (count before the frame), its scan
// writes slot (s + 1) % 3 (count after the frame) and its regularisation reads both. In the frame
// pipeline the scan of frame f + 1 (slot (s + 2) % 3) may run while the regularisation of frame f
// is still reading, which is why two slots are not enough.
constexpr int kCountSlots = 3;
struct Counters {
  u32 surfel_count[kCountSlots];
  u32 merge_count;
  u32 new_surfel_count;  // of the last frame
  u32 capacity_overflow; // sticky: a frame wanted more surfels than the cap (creation skipped)
  u32 scan_ticket;       // dynamic tile ids of the new-surfel scan
  u32 pad;
};

struct DeviceState {
  // surfel SoA: row r, surfel i -> surfels[r * stride + i]
  float* surfels;
  size_t stride;         // elements per row (multiple of 64)
  u32 capacity;
  int width, height;
  PixelAssoc* assoc;     // W*H
  float* first_depth;    // W*H
  u8* supported;         // W*H: 1 iff the pixel has a supporting surfel (assoc.x != invalid)
  VisEntry* vis;         // capacity (rounded up to kSegment)
  u32* seg_count;        // capacity / kSegment
  u8* merge_flag;        // per list position
  // Neighbour-update work list, filled by k_integrate: {slot, x | y << 16} of every surfel that passes the
  // gates of k_update_neighbors up to the occlusion test (x, y: its pixel after the integration), in
  // arbitrary order. Capacity as vis; the count is reset by k_project.
  uint2* upd_list;
  u32* upd_count;
  u8* new_flag;          // W*H
  u32* new_index;        // W*H
  u32* new_list;         // W*H: pixel (seq index) of the k-th new surfel
  unsigned long long* scan_state;  // per scan tile: status << 32 | value
  Counters* counters;
  // Regularisation gradient accumulators {gx, gy, gz, weight sum} per surfel slot: the reference's
  // rows 11-13 and 23 as one 16-byte record, so that a neighbour contribution is ONE vector
  // atomic instead of four. Zero between Regularize() calls (the SoA rows stay zero always).
  float4* gradient;
  // Regularisation records, double-buffered: one float4 per slot and buffer, {x, y, z} = the smooth position
  // (the reference's rows 3-5) and w = the bits of last_update_stamp | detach flag << 31 (the detach flag is
  // colour byte 3 == 1). Both regularisation sweeps gather, per neighbour, the in-window / detach gate and the
  // position in ONE 16-byte gather. `smooth` is the current buffer; k_reg_step reads it and writes the records
  // of `smooth_next` it has to (see reg_t_prev), then the two are swapped on the host (no separate update
  // sweep). SoA rows 3-5 and 15 are only an export mirror of the current buffer (MirrorRegRecords).
  // Invariants:
  //   * every writer of a smooth position or of the stamp / detach state writes BOTH buffers, .w included:
  //     merge application, stamping and replacement in k_integrate, k_create_surfels, k_reg_copy_only and
  //     the load-state pack; so .w is always equal in the two buffers;
  //   * k_reg_step writes the whole record of the next buffer and carries .w over from the current one.
  float4* smooth;
  float4* smooth_next;
  // Host-side bookkeeping of the two smooth buffers (regularize.cu). Invariant: a slot whose stamp is below
  // reg_t_prev holds the same smooth position in both buffers, unless reg_full_sweep is set (the second
  // buffer is undefined: after sm_create, sm_load_state, sm_reset). reg_t_prev is int(frame - window) of the
  // previous k_reg_step sweep, lowered to a frame index that k_integrate stamps below it.
  int reg_t_prev;
  int reg_full_sweep;
  // Device timeline (diagnostics, sm_timeline_enable): [frame % timeline_frames][kernel id]{first block start,
  // last block end} in %globaltimer nanoseconds; null when disabled.
  unsigned long long* timeline;
  u32 timeline_frames;
};

struct FrameParams {
  u32 frame_index;
  int count_slot;        // Counters::surfel_count slot holding the count before this frame
  int skip;              // != 0: the launch is a placeholder of the frame graph, the kernel returns at once
  u32 op_epoch;          // operation counter of the handle; recorded in row 14 of a surfel when it is merged (transfer.cu)
  TieBreak tb;           // supporting-surfel tie-break (see kSecondaryBit)
  int active_window;     // surfel_integration_active_window_size
  float fx, fy, cx, cy;
  float fx_inv, fy_inv, cx_inv, cy_inv;  // pixel-centre unprojection, kernels.cc:68-74
  float sensor_noise_factor;
  float cos_normal_compatibility_threshold;
  float max_surfel_confidence;
  float depth_scaling;
  float inv_depth_scaling;               // 1.0f / depth_scaling (depth_correction_factor)
  float radius_factor_squared;           // radius_factor_for_regularization_neighbors^2
  int blend_radius;
  Mat3x4 local_T_global;
  Mat3x4 global_T_local;
  // input rasters
  u16* depth; size_t depth_pitch;
  // The depth as it was before the measurement blending: read by the association and merge
  // gates (the reference runs them before BlendMeasurements). Equal to `depth` unless the
  // caller provides a separate copy so that merge and blend can run concurrently.
  const u16* depth_pre; size_t depth_pre_pitch;
  const float2* normals; size_t normals_pitch;
  const float* radius; size_t radius_pitch;
  const uchar3* color; size_t color_pitch;
};

// Programmatic dependent launch (sm_90+): every kernel starts with pdl_prologue(): it lets the NEXT
// kernel of the stream be scheduled early (launch_dependents) and then waits until the PREVIOUS
// kernel has completed and flushed its memory (wait). With the launch attribute set
// (LaunchConfig below) this overlaps launch latency / block scheduling of dependent kernels with
// the tail of their predecessor; without the attribute both instructions are no-ops.
__device__ __forceinline__ void pdl_prologue() {
#if defined(__CUDA_ARCH__)
  asm volatile("griddepcontrol.launch_dependents;");
  asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}
// Device timeline: the kernels stamp their own start / end (%globaltimer) so that the frame
// pipeline can be read as it really ran on the GPU (events and the profiler serialise it).
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
struct TimelineScope {
  unsigned long long* slot;
  __device__ __forceinline__ explicit TimelineScope(unsigned long long* s) : slot(s) { begin(); }
  __device__ __forceinline__ TimelineScope(const DeviceState& d, u32 frame, int kernel_id)
      : slot(d.timeline ? d.timeline + (static_cast<size_t>(frame % d.timeline_frames) * KID_TIMELINE_COUNT + kernel_id) * 2 : nullptr) {
    begin();
  }
  __device__ __forceinline__ void begin() {
    if (slot && threadIdx.x == 0 && blockIdx.x < 8 && blockIdx.y == 0) atomicMin(slot, globaltimer_ns());
  }
  __device__ __forceinline__ ~TimelineScope() {
    if (slot && threadIdx.x == 0) atomicMax(slot + 1, globaltimer_ns());
  }
};
// Host side: slot of (frame, kernel id) for kernels that do not take a DeviceState.
inline unsigned long long* TimelineSlot(const DeviceState& d, u32 frame, int kernel_id) {
  return d.timeline ? d.timeline + (static_cast<size_t>(frame % d.timeline_frames) * KID_TIMELINE_COUNT + kernel_id) * 2 : nullptr;
}

// Configuration of one stream launch. `dependent`: the kernel's producer is the previous kernel of the same stream,
// and the launch carries the programmatic-serialization attribute (sm_preprocess, sm_integrate and the serial mode
// of sm_stream_run; the nodes of the frame graph are not stream launches).
class LaunchConfig {
 public:
  LaunchConfig(dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool dependent) {
    attr_.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr_.val.programmaticStreamSerializationAllowed = 1;
    cfg_ = {};
    cfg_.gridDim = grid;
    cfg_.blockDim = block;
    cfg_.dynamicSmemBytes = smem;
    cfg_.stream = stream;
    cfg_.attrs = &attr_;
    cfg_.numAttrs = dependent ? 1 : 0;
  }
  LaunchConfig(const LaunchConfig&) = delete;
  LaunchConfig& operator=(const LaunchConfig&) = delete;
  const cudaLaunchConfig_t* get() const { return &cfg_; }

 private:
  cudaLaunchAttribute attr_;
  cudaLaunchConfig_t cfg_;
};

template <typename... KArgs, typename... Args>
inline void LaunchKernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                         Args&&... args) {
  cudaLaunchKernelEx(LaunchConfig(grid, block, smem, stream, false).get(), kernel, static_cast<KArgs>(args)...);
}

// One kernel launch with its by-value arguments packed into `storage`: what a stream launch and
// a kernel node of the frame graph (pipeline.cu) are both made from. The translation unit that
// owns a kernel fills the descriptor (Describe* functions below), so kernels and their argument
// structs stay file-local.
struct KernelLaunch {
  const void* func;
  dim3 grid, block;
  size_t smem;
  int kernel_id;                 // KernelId
  int arg_count;
  void* args[6];                 // point into storage
  alignas(64) unsigned char storage[2304];
  size_t used;
  void Reset(const void* f, dim3 g, dim3 b, size_t shared, int id) {
    func = f; grid = g; block = b; smem = shared; kernel_id = id; arg_count = 0; used = 0;
  }
  template <typename T>
  void Arg(const T& v) {
    used = (used + alignof(T) - 1) / alignof(T) * alignof(T);
    static_assert(alignof(T) <= 64, "argument alignment");
    memcpy(storage + used, &v, sizeof(T));   // used + sizeof(T) <= sizeof(storage): checked by the static_asserts at the call sites
    args[arg_count++] = storage + used;
    used += sizeof(T);
  }
};
// Launches a described kernel on a stream (counts it, profiles it like LaunchKernel).
void LaunchOnStream(cudaStream_t stream, const KernelLaunch& k, bool dependent);

// Grid of a resident sweep: exactly the blocks of `kernel` that are resident at once (occupancy x SMs), so that
// every block is scheduled in the first wave and the per-block loops take care of longer lists.
template <typename Kernel>
inline int ResidentBlocks(Kernel kernel, int block, int sm_count, int* out) {
  int per_sm = 0;
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, 0);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return SetError(SM_ERR_CUDA, (std::string("cudaOccupancyMaxActiveBlocksPerMultiprocessor: ") + cudaGetErrorString(e)).c_str());
  }
  *out = (per_sm > 0 ? per_sm : 1) * sm_count;
  return SM_OK;
}

// Grid sizes of the list / sweep kernels (ResidentBlocks). Occupancy and function attributes are per
// device, so the plan lives in the handle (sm_create), not in statics.
struct LaunchPlan {
  int sm_count;
  int project, associate, merge, integrate, update_neighbors;
  int reg_accumulate, reg_step, reg_copy;
};
// Shared-memory carve-out of the pre-processing, Integrate() and regularisation kernels, in percent of the
// 228 KB of an SM. k_blend needs ~100 KB per block and everything else a few KB; left to the driver, the
// SMs keep switching between configurations and the gather kernels (integrate, update_neighbors,
// regularisation) slow down after a blend. 47 % selects the 132 KB configuration (an H100 SM offers 0, 8,
// 16, 32, 64, 100, 132, 164, 196 and 228 KB), the smallest that holds a blend block, and leaves 124 KB of
// L1 to the gathers.
constexpr int kSharedMemoryCarveoutPercent = 47;
// Per-device kernel configuration of the current device: the carve-out, k_blend's dynamic shared memory
// limit, the resident grids.
int ConfigurePreprocessKernels();
int ConfigureIntegrateKernels(LaunchPlan* plan);
int ConfigureRegularizeKernels(LaunchPlan* plan);

// ---- preprocess.cu --------------------------------------------------------------------------
// Opaque storage of a CUtensorMap (TMA descriptor; cuda.h stays out of this header).
struct alignas(64) TensorMapStorage { unsigned char bytes[128]; };
int MakeDepthTensorMap(TensorMapStorage* out, const u16* base, size_t pitch_bytes, int width, int height);
// `scratch_B_map`: TMA descriptor of scratch_B (MakeDepthTensorMap), the tail's input tile.
int PreprocessFused(cudaStream_t stream, const sm_preprocess_params& p, int width, int height, float fx, float fy,
                    float cx, float cy, const u16* raw, size_t raw_pitch, const u16* const* other_depths,
                    const size_t* other_pitches, const float* others_TR_reference, u16* scratch_B,
                    size_t scratch_B_pitch, u16* out_depth, size_t out_depth_pitch, float2* out_normals,
                    size_t out_normals_pitch, float* out_radius, size_t out_radius_pitch, uint4* clear_assoc,
                    float* clear_first_depth, u8* clear_supported, u16* out_depth_copy,
                    size_t out_depth_copy_pitch, unsigned long long* timeline_bilateral,
                    unsigned long long* timeline_tail, const TensorMapStorage& scratch_B_map);
// Bilateral filter radius (cuda_depth_processing.cu:135). Radius 6 has the fused bilateral + outlier kernel.
inline int BilateralRadius(const sm_preprocess_params& p) {
  return static_cast<int>(p.bilateral_filter_radius_factor * p.bilateral_filter_sigma_xy + 0.5f);
}
// The same launches as descriptors (frame graph): bilateral + outlier fused at radius 6 (`outlier` unused), else
// k_bilateral_generic and k_outlier in place on scratch_B; then the tail. `skip`: placeholder launches.
int DescribePreprocess(KernelLaunch* bilateral, KernelLaunch* outlier, KernelLaunch* tail, bool skip,
                       const sm_preprocess_params& p, int width, int height, float fx, float fy, float cx, float cy,
                       const u16* raw, size_t raw_pitch, const u16* const* other_depths, const size_t* other_pitches,
                       const float* others_TR_reference, u16* scratch_B, size_t scratch_B_pitch, u16* out_depth,
                       size_t out_depth_pitch, float2* out_normals, size_t out_normals_pitch, float* out_radius,
                       size_t out_radius_pitch, uint4* clear_assoc, float* clear_first_depth, u8* clear_supported,
                       u16* out_depth_copy, size_t out_depth_copy_pitch, unsigned long long* timeline_bilateral,
                       unsigned long long* timeline_tail, const TensorMapStorage& scratch_B_map);
int StageBilateral(cudaStream_t stream, float sigma_xy, float sigma_value_factor, u16 value_to_ignore,
                   float radius_factor, u16 max_depth, float depth_valid_region_radius, int width, int height,
                   const u16* in, size_t in_pitch, u16* out, size_t out_pitch);
int StageMedianDensify(cudaStream_t stream, int iterations, int width, int height, const u16* in, size_t in_pitch,
                       u16* out, size_t out_pitch, u16* scratch, size_t scratch_pitch);
// The input downscaling of --pyramid_level: median depth blocks of up to 16 x 16 pixels, and `levels`
// (0-4) colour halvings of packed uchar3 in one launch (levels == 0 copies).
int StageDownscaleMedian(cudaStream_t stream, u16 value_to_ignore, int in_width, int in_height, const u16* in,
                         size_t in_pitch, int out_width, int out_height, u16* out, size_t out_pitch);
int StageColorPyramid(cudaStream_t stream, int levels, int width, int height, const u8* in, size_t in_pitch, u8* out,
                      size_t out_pitch);

// ---- integrate.cu ---------------------------------------------------------------------------
struct IntegrateEvents {
  cudaEvent_t ev[14];
  bool enabled;
};
int IntegrateFrame(cudaStream_t stream, const DeviceState& d, const FrameParams& f, bool do_blending,
                   bool rasters_already_cleared, const LaunchPlan& plan, const IntegrateEvents* events);
// Kernels of one Integrate() as descriptors (stream launches and frame-graph nodes).
enum FrameKernel { FK_PROJECT = 0, FK_ASSOCIATE, FK_MERGE, FK_BLEND, FK_INTEGRATE, FK_UPDATE_NEIGHBORS, FK_SCAN, FK_CREATE,
                   FK_COUNT };
int DescribeFrameKernel(FrameKernel which, const LaunchPlan& plan, const DeviceState& d, const FrameParams& f,
                        KernelLaunch* out);
int ClearAssociationRasters(cudaStream_t stream, const DeviceState& d);

int ExportVertices(cudaStream_t stream, const DeviceState& d, int count_slot, int sm_count, float* position_buffer,
                   u8* color_buffer);

// ---- regularize.cu --------------------------------------------------------------------------
// `count_slot`: which Counters::surfel_count slot holds the surfel count to regularise.
// `remove_replaced_below`: if >= 0, slot of the surfel count below which neighbour links to
// surfels with the detach flag are dropped first (UpdateNeighborsCUDARemoveReplacedNeighbors
// fused into the first sweep); -1 = no removal.
// Bookkeeping of DeviceState::reg_t_prev on the host: after every k_reg_step sweep, and for every
// Integrate() (k_integrate stamps surfels with its frame index, which may lie below the last threshold).
inline void NoteRegStep(DeviceState& d, u32 frame_index, int window) {
  d.reg_t_prev = static_cast<int>(frame_index - static_cast<u32>(window));
  d.reg_full_sweep = 0;
}
inline void NoteIntegratedFrame(DeviceState& d, u32 frame_index) {
  if (static_cast<int>(frame_index) < d.reg_t_prev) d.reg_t_prev = static_cast<int>(frame_index);
}
// Packs both regularisation record buffers of slots [0, count) from SoA rows 3-5, the stamp row and the colour
// row's detach byte (after sm_load_state).
int PackRegRecords(cudaStream_t stream, const DeviceState& d, u32 count, int sm_count);
// Unpacks the current regularisation records of slots [0, count) into the export mirror: SoA rows 3-5 (smooth
// position) and row kRowMeta (.w). Runs on `stream` before the mirror is copied or read.
int MirrorRegRecords(cudaStream_t stream, const DeviceState& d, u32 count, int sm_count);
int RegularizeSurfels(cudaStream_t stream, DeviceState& d, bool disable_denoising, u32 frame_index,
                      float radius_factor_for_regularization_neighbors, float regularizer_weight,
                      int regularization_frame_window_size, int count_slot, int remove_replaced_below_slot,
                      const LaunchPlan& plan);
// One regularisation iteration as descriptors: `first` = k_reg_accumulate (or k_reg_copy_only when
// denoising is disabled, then *second is unused and the function returns 1), `second` = k_reg_step;
// returns the number of launches. Does NOT swap d.smooth / d.smooth_next (the caller does after a
// denoising iteration).
int DescribeRegularize(KernelLaunch* first, KernelLaunch* second, bool skip, const LaunchPlan& plan,
                       const DeviceState& d, bool disable_denoising, u32 frame_index,
                       float radius_factor_for_regularization_neighbors, float regularizer_weight,
                       int regularization_frame_window_size, int count_slot, int remove_replaced_below_slot);

}  // namespace smb
