// api.cu — C ABI of libsurfel_b200.so (include/surfel_b200.h): the handle that replaces
// class vis::CUDASurfelReconstruction (APP/cuda_surfel_reconstruction.{h,cc}), the host
// wrappers that replace APP/cuda_surfel_reconstruction_kernels.cc and the RGB-D stream
// runner that replaces the frame loop of APP/main.cc:885-1223.

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <limits>
#include <mutex>
#include <string>
#include <vector>

#include "sm_handle.cuh"

namespace smb {

namespace {
thread_local std::string g_last_error;
std::atomic<unsigned long long> g_launches{0};
}  // namespace

int SetError(int code, const char* message) {
  g_last_error = message ? message : "";
  return code;
}

int CheckLaunch(const char* what) {
  const cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return SM_OK;
  g_last_error = std::string(what) + ": " + cudaGetErrorString(e);
  return SM_ERR_CUDA;
}

namespace {
// Per-kernel profiling (sm_profile_kernels): event pairs recorded around every launch.
struct ProfileRecord { cudaEvent_t start, stop; int id; };
std::mutex g_profile_mutex;
bool g_profile_enabled = false;
std::vector<ProfileRecord> g_profile_records;
std::vector<cudaEvent_t> g_event_pool;

cudaEvent_t TakeEvent() {
  if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
}  // namespace

bool ProfilingEnabled() { return g_profile_enabled; }

void CountLaunches(unsigned long long n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
unsigned long long LaunchCount() { return g_launches.load(); }

// Launch of a described kernel (KernelLaunch, sm_kernels.cuh) on a stream.
void LaunchOnStream(cudaStream_t stream, const KernelLaunch& k, bool dependent) {
  LaunchScope scope(stream, static_cast<KernelId>(k.kernel_id));
  cudaLaunchKernelExC(LaunchConfig(k.grid, k.block, k.smem, stream, dependent).get(), k.func, const_cast<void**>(k.args));
}

// ---- supporting-surfel tie-break (sm_kernels.cuh, kSecondaryBit) ---------------------------------
namespace {
// x^-1 mod m for gcd(x, m) = 1 (extended Euclid).
u32 ModInverse(u32 x, u32 m) {
  long long t = 0, new_t = 1, r = m, new_r = x % m;
  while (new_r != 0) {
    const long long q = r / new_r;
    long long tmp = t - q * new_t; t = new_t; new_t = tmp;
    tmp = r - q * new_r; r = new_r; new_r = tmp;
  }
  if (t < 0) t += m;
  return static_cast<u32>(t);
}
}  // namespace

int SetTieBreakWave(TieBreakConfig* cfg, u32 wave, u32 capacity) {
  u32 lane_shift = cfg->lane_request;
  if (wave != 0) {
    // keys are ((slot + phase) / W) * 2 W + late * W + perm((slot + phase) % W) < 2^32 - 1, phase < W
    const unsigned long long top = (static_cast<unsigned long long>(capacity) / wave + 2) * 2ull * wave;
    if (wave < 2 || top >= 0xFFFFFFFFull) return SetError(SM_ERR_INVALID_ARGUMENT, "tiebreak_wave out of range for this surfel cap");
    if (lane_shift > 10) return SetError(SM_ERR_INVALID_ARGUMENT, "tiebreak_lanes must be a power of two <= 1024");
    if (wave % (1u << lane_shift) != 0 || (wave >> lane_shift) < 2) lane_shift = 0;   // the wave is not made of whole groups
    const u32 groups = wave >> lane_shift;
    const unsigned long long prime = 2654435761ull;  // > any wave, so gcd(prime % groups, groups) = 1
    cfg->mul = static_cast<u32>(prime % groups);
    if (cfg->mul == 0) cfg->mul = 1;
    cfg->mul_inv = ModInverse(cfg->mul, groups);
  }
  cfg->wave = wave;
  cfg->lane_shift = lane_shift;
  return SM_OK;
}

TieBreak MakeTieBreak(const TieBreakConfig& cfg, u32 frame_index) {
  TieBreak t{};
  t.wave = cfg.wave;
  if (cfg.wave == 0) return t;
  t.lane_shift = cfg.lane_shift;
  t.wave_offset = cfg.wave_offset;
  t.groups = cfg.wave >> cfg.lane_shift;
  t.mul = cfg.mul;
  t.mul_inv = cfg.mul_inv;
  t.wave_reciprocal = ~0ull / cfg.wave;
  t.group_reciprocal = ~0ull / t.groups;
  t.add = tb_hash(frame_index * 0x9E3779B9u + 0x7F4A7C15u) % t.groups;
  t.salt = tb_hash(frame_index ^ 0x85EBCA6Bu);
  auto threshold = [](double fraction) {
    const double scaled = fraction * 4294967296.0;
    return scaled <= 0 ? 0u : (scaled >= 4294967295.0 ? 0xFFFFFFFFu : static_cast<u32>(scaled));
  };
  t.early_threshold = threshold(cfg.early_fraction);
  t.index_order_threshold = threshold(cfg.index_order_fraction);
  const double later = cfg.early_fraction_later >= 0 ? cfg.early_fraction_later : cfg.early_fraction;
  t.early_threshold_later = threshold(later);
  t.early_threshold_second = threshold(cfg.early_fraction_second >= 0 ? cfg.early_fraction_second : later);
  t.index_order_threshold_later = threshold(cfg.index_order_fraction_later >= 0 ? cfg.index_order_fraction_later : cfg.index_order_fraction);
  return t;
}

const char* KernelName(int id) {
  static const char* names[KID_COUNT] = {
      "k_clear", "k_bilateral_outlier", "k_bilateral_generic", "k_outlier", "k_erode_normals_radii", "k_erode",
      "k_normals", "k_radii", "k_project", "k_associate", "k_merge", "k_blend", "k_integrate", "k_update_neighbors",
      "k_new_surfel_scan", "k_create_surfels", "k_reg_accumulate", "k_reg_step", "k_reg_copy_only",
      "k_export_vertices", "k_median_densify", "k_delta_select", "k_viz_buffers", "k_downscale_depth_median",
      "k_downscale_color", "k_reg_mirror", "k_reg_pack", "k_render_splat", "k_render_large", "k_render_resolve",
      "k_track_live_view", "k_track_linearize", "k_track_solve", "k_mesh_bound", "k_mesh_umbrella", "k_mesh_count",
      "k_mesh_scan", "k_mesh_write"};
  return (id >= 0 && id < KID_COUNT) ? names[id] : "?";
}

LaunchScope::LaunchScope(cudaStream_t stream, KernelId id) : stream_(stream), slot_(-1) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (g_profile_enabled) {
    std::lock_guard<std::mutex> lock(g_profile_mutex);
    ProfileRecord r{TakeEvent(), TakeEvent(), static_cast<int>(id)};
    cudaEventRecord(r.start, stream_);
    slot_ = static_cast<int>(g_profile_records.size());
    g_profile_records.push_back(r);
  }
}

LaunchScope::~LaunchScope() {
  if (slot_ >= 0) {
    std::lock_guard<std::mutex> lock(g_profile_mutex);
    cudaEventRecord(g_profile_records[slot_].stop, stream_);
  }
}

}  // namespace smb

using namespace smb;

#define SM_CUDA(call)                                                                        \
  do {                                                                                       \
    const cudaError_t e_ = (call);                                                           \
    if (e_ != cudaSuccess) {                                                                 \
      g_last_error = std::string(#call) + ": " + cudaGetErrorString(e_);                     \
      return SM_ERR_CUDA;                                                                    \
    }                                                                                        \
  } while (0)

namespace {
// Calls that would change what an open session builds on (sm_session_begin, include/surfel_b200.h).
int RejectInSession(const char* call) {
  return SetError(SM_ERR_INVALID_ARGUMENT, (std::string(call) + ": a stream session is open on this handle (sm_session_end first)").c_str());
}
}  // namespace

namespace smb {

int FetchCounters(sm_reconstruction* r, cudaStream_t stream) {
  SM_CUDA(cudaMemcpyAsync(r->host_counters, r->d.counters, sizeof(Counters), cudaMemcpyDeviceToHost, stream));
  if (r->reported_merge_count) {   // an open frame-graph session (pipeline.cu: SessionPush)
    SM_CUDA(cudaMemcpyAsync(&r->host_counters->merge_count, r->reported_merge_count, sizeof(u32), cudaMemcpyDeviceToHost,
                            stream));
  }
  SM_CUDA(cudaStreamSynchronize(stream));
  if (r->host_counters->capacity_overflow) {
    return SetError(SM_ERR_CAPACITY, "surfel cap exceeded: new surfels of at least one frame were dropped "
                                     "(the reference writes out of bounds here)");
  }
  return SM_OK;
}

FrameParams MakeFrameParams(const sm_reconstruction* r, u32 frame_index, int count_slot, const sm_integrate_params& p,
                            u16* depth, size_t depth_pitch, const u16* depth_pre, size_t depth_pre_pitch,
                            const float* normals, size_t normals_pitch, const float* radius, size_t radius_pitch,
                            const uint8_t* color, size_t color_pitch, const float* global_T_local,
                            const float* local_T_global) {
  FrameParams f;
  f.frame_index = frame_index;
  f.count_slot = count_slot;
  f.skip = 0;
  f.op_epoch = r->op_epoch;
  f.tb = MakeTieBreak(r->tiebreak, frame_index);
  f.active_window = p.surfel_integration_active_window_size;
  f.fx = r->fx; f.fy = r->fy; f.cx = r->cx; f.cy = r->cy;
  // Unprojection intrinsics for pixel center convention (kernels.cc:68-74).
  f.fx_inv = 1.0f / r->fx;
  f.fy_inv = 1.0f / r->fy;
  const float cx_pixel_center = r->cx - 0.5f;
  const float cy_pixel_center = r->cy - 0.5f;
  f.cx_inv = -cx_pixel_center / r->fx;
  f.cy_inv = -cy_pixel_center / r->fy;
  f.sensor_noise_factor = p.sensor_noise_factor;
  f.cos_normal_compatibility_threshold = cosf(M_PI / 180.0f * p.normal_compatibility_threshold_deg);  // kernels.cc:261
  f.max_surfel_confidence = p.max_surfel_confidence;
  f.inv_depth_scaling = 1.0f / p.depth_scaling;                 // cuda_surfel_reconstruction.cc:158
  f.depth_scaling = 1.0f / f.inv_depth_scaling;                 // kernels.cc:179: 1.0f / depth_correction_factor
  f.radius_factor_squared =
      p.radius_factor_for_regularization_neighbors * p.radius_factor_for_regularization_neighbors;
  f.blend_radius = p.measurement_blending_radius;
  f.local_T_global = MakeMat3x4(local_T_global);
  f.global_T_local = MakeMat3x4(global_T_local);
  f.depth = depth; f.depth_pitch = depth_pitch;
  f.depth_pre = depth_pre; f.depth_pre_pitch = depth_pre_pitch;
  f.normals = reinterpret_cast<const float2*>(normals); f.normals_pitch = normals_pitch;
  f.radius = radius; f.radius_pitch = radius_pitch;
  f.color = reinterpret_cast<const uchar3*>(color); f.color_pitch = color_pitch;
  return f;
}

// CUDASurfelReconstruction::Integrate (cuda_surfel_reconstruction.cc:112-320).
int IntegrateImpl(sm_reconstruction* r, cudaStream_t stream, u32 frame_index, const sm_integrate_params& p,
                  u16* depth, size_t depth_pitch, const float* normals, size_t normals_pitch, const float* radius,
                  size_t radius_pitch, const uint8_t* color, size_t color_pitch, const float* global_T_local,
                  const float* local_T_global) {
  r->last_stream = stream;
  RecordOperation(r, static_cast<int>(frame_index - static_cast<u32>(p.regularization_frame_window_size)));
  // The association / merge gates read the depth as it is before the blending, and the blending
  // reads that image while it writes the caller's buffer (k_blend): snapshot it first.
  const u16* depth_pre = depth;
  size_t depth_pre_pitch = depth_pitch;
  if (p.do_blending) {
    SM_CUDA(cudaMemcpy2DAsync(r->blend_src, r->blend_src_pitch, depth, depth_pitch, r->d.width * sizeof(u16),
                              r->d.height, cudaMemcpyDeviceToDevice, stream));
    depth_pre = r->blend_src;
    depth_pre_pitch = r->blend_src_pitch;
  }
  const FrameParams f = MakeFrameParams(r, frame_index, r->count_slot, p, depth, depth_pitch, depth_pre, depth_pre_pitch,
                                        normals, normals_pitch, radius, radius_pitch, color, color_pitch,
                                        global_T_local, local_T_global);
  r->last_tiebreak = f.tb;
  int status = IntegrateFrame(stream, r->d, f, p.do_blending != 0, r->rasters_cleared, r->plan, &r->events);
  r->rasters_cleared = false;
  if (status != SM_OK) return status;
  NoteIntegratedFrame(r->d, frame_index);
  const int old_slot = r->count_slot;
  r->count_slot = (r->count_slot + 1) % kCountSlots;  // k_new_surfel_scan wrote the next slot
  if (r->events.enabled) cudaEventRecord(r->events.ev[12], stream);
  // cuda_surfel_reconstruction.cc:295-317; the detach-flag pass of UpdateNeighborsCUDA
  // (kernels.cc:333-339) over the slots that existed before this frame rides on the first sweep.
  const int iterations = p.regularization_iterations_per_integration_iteration;
  if (iterations == 0) {
    status = RegularizeSurfels(stream, r->d, /*disable_denoising*/ true, frame_index,
                               p.radius_factor_for_regularization_neighbors, p.regularizer_weight,
                               p.regularization_frame_window_size, r->count_slot, old_slot, r->plan);
  } else {
    for (int i = 0; i < iterations && status == SM_OK; ++i) {
      status = RegularizeSurfels(stream, r->d, /*disable_denoising*/ false, frame_index,
                                 p.radius_factor_for_regularization_neighbors, p.regularizer_weight,
                                 p.regularization_frame_window_size, r->count_slot, i == 0 ? old_slot : -1, r->plan);
    }
  }
  if (r->events.enabled) cudaEventRecord(r->events.ev[13], stream);
  return status;
}

}  // namespace smb

namespace {

// Everything sm_create allocates; on failure the caller destroys the partially built handle.
int CreateImpl(sm_reconstruction* r, uint64_t max_surfel_count, int32_t width, int32_t height, float fx, float fy,
               float cx, float cy) {
  SM_CUDA(cudaGetDevice(&r->device));
  cudaDeviceProp prop;
  SM_CUDA(cudaGetDeviceProperties(&prop, r->device));
  r->sm_count = prop.multiProcessorCount;
  r->plan.sm_count = r->sm_count;
  {
    // The shared-memory carve-out (kSharedMemoryCarveoutPercent) of the pre-processing, Integrate() and
    // regularisation kernels, k_blend's shared memory limit and the resident grids. The render, tracking,
    // k-NN and transfer kernels keep the driver's carve-out. Function attributes and occupancy are per
    // device: configured for every handle.
    int status = ConfigurePreprocessKernels();
    if (status == SM_OK) status = ConfigureIntegrateKernels(&r->plan);
    if (status == SM_OK) status = ConfigureRegularizeKernels(&r->plan);
    if (status != SM_OK) return status;
  }
  r->fx = fx; r->fy = fy; r->cx = cx; r->cy = cy;
  DeviceState& d = r->d;
  d.width = width; d.height = height;
  d.capacity = static_cast<u32>(max_surfel_count);
  const size_t padded = (max_surfel_count + kSegment - 1) / kSegment * kSegment;
  d.stride = padded;
  const size_t P = static_cast<size_t>(width) * height;
  const size_t scan_tiles = (P + kSegment - 1) / kSegment;
  SM_CUDA(cudaMalloc(&d.surfels, sizeof(float) * SM_ROW_COUNT * d.stride));
  SM_CUDA(cudaMalloc(&d.gradient, sizeof(float4) * d.stride));
  SM_CUDA(cudaMalloc(&r->reg_records, sizeof(float4) * 2 * d.stride));
  d.smooth = r->reg_records;
  d.smooth_next = r->reg_records + d.stride;
  SM_CUDA(cudaMemset(d.gradient, 0, sizeof(float4) * d.stride));
  for (int i = 0; i < kSets; ++i) {
    SM_CUDA(cudaMalloc(&r->assoc_set[i], sizeof(PixelAssoc) * P));
    SM_CUDA(cudaMalloc(&r->first_depth_set[i], sizeof(float) * P));
    SM_CUDA(cudaMalloc(&r->supported_set[i], P));
    SM_CUDA(cudaMalloc(&r->vis_set[i], sizeof(VisEntry) * padded));
    SM_CUDA(cudaMalloc(&r->seg_count_set[i], sizeof(u32) * (padded / kSegment)));
    SM_CUDA(cudaMalloc(&r->merge_flag_set[i], padded));
    SM_CUDA(cudaMalloc(&r->upd_list_set[i], sizeof(uint2) * padded));
    SM_CUDA(cudaMalloc(&r->upd_count_set[i], sizeof(u32)));
  }
  d.assoc = r->assoc_set[0]; d.first_depth = r->first_depth_set[0]; d.supported = r->supported_set[0];
  d.vis = r->vis_set[0]; d.seg_count = r->seg_count_set[0]; d.merge_flag = r->merge_flag_set[0];
  d.upd_list = r->upd_list_set[0]; d.upd_count = r->upd_count_set[0];
  d.reg_t_prev = 0;
  d.reg_full_sweep = 1;  // smooth_next is undefined
  SM_CUDA(cudaMalloc(&d.new_list, sizeof(u32) * P));
  SM_CUDA(cudaMalloc(&d.new_flag, P));
  SM_CUDA(cudaMalloc(&d.new_index, sizeof(u32) * P));
  SM_CUDA(cudaMalloc(&d.scan_state, sizeof(unsigned long long) * scan_tiles));
  SM_CUDA(cudaMalloc(&d.counters, sizeof(Counters)));
  SM_CUDA(cudaMemset(d.counters, 0, sizeof(Counters)));
  d.timeline = nullptr;
  d.timeline_frames = 0;
  SM_CUDA(cudaMemset(d.new_flag, 0, P));
  SM_CUDA(cudaMemset(d.new_index, 0, sizeof(u32) * P));
  SM_CUDA(cudaMemset(d.scan_state, 0, sizeof(unsigned long long) * scan_tiles));
  SM_CUDA(cudaMallocHost(&r->host_counters, sizeof(Counters)));
  std::memset(r->host_counters, 0, sizeof(Counters));
  SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&r->scratch_B), &r->scratch_B_pitch, width * sizeof(u16), height));
  SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&r->blend_src), &r->blend_src_pitch, width * sizeof(u16), height));
  {
    // The pre-processing tail fills its input tile with one cp.async.bulk.tensor per block through this descriptor.
    const int status = MakeDepthTensorMap(&r->scratch_B_map, r->scratch_B, r->scratch_B_pitch, width, height);
    if (status != SM_OK) return status;
  }
  for (int i = 0; i < 14; ++i) SM_CUDA(cudaEventCreate(&r->events.ev[i]));
  r->events.enabled = false;
  // Supporting-surfel tie-break defaults (DESIGN.md section 4); sm_configure("tiebreak_*") changes them.
  {
    u32 wave = kDefaultTieBreakWave;
    // the keys of the default wave would not fit in 32 bits at this surfel cap: plain rule
    if ((static_cast<unsigned long long>(d.capacity) / wave + 2) * 2ull * wave >= 0xFFFFFFFFull) wave = 0;
    r->tiebreak.wave_offset = kDefaultTieBreakWaveOffset;
    r->tiebreak.lane_request = kDefaultTieBreakLaneShift;
    const int status = SetTieBreakWave(&r->tiebreak, wave, d.capacity);
    if (status != SM_OK) return status;
    r->tiebreak.early_fraction = kDefaultTieBreakEarlyFraction;
    r->tiebreak.index_order_fraction = kDefaultTieBreakIndexOrderFraction;
    r->tiebreak.early_fraction_later = kDefaultTieBreakEarlyFractionLater;
    r->tiebreak.index_order_fraction_later = kDefaultTieBreakIndexOrderFractionLater;
    r->tiebreak.early_fraction_second = kDefaultTieBreakEarlyFractionSecond;
  }
  const int status = ClearAssociationRasters(nullptr, d);
  if (status != SM_OK) return status;
  SM_CUDA(cudaDeviceSynchronize());
  return SM_OK;
}

}  // namespace

extern "C" {

void sm_default_integrate_params(sm_integrate_params* p) {
  // APP/main.cc:279-371.
  p->depth_scaling = 5000;
  p->sensor_noise_factor = 0.05f;
  p->max_surfel_confidence = 5.0f;
  p->regularizer_weight = 10.0f;
  p->regularization_frame_window_size = 30;
  p->do_blending = 1;
  p->measurement_blending_radius = 12;
  p->regularization_iterations_per_integration_iteration = 1;
  p->radius_factor_for_regularization_neighbors = 2;
  p->normal_compatibility_threshold_deg = 40;
  p->surfel_integration_active_window_size = std::numeric_limits<int>::max();
}

void sm_default_preprocess_params(sm_preprocess_params* p) {
  // APP/main.cc:415-478.
  p->depth_scaling = 5000;
  p->max_depth = 3.0f;
  p->depth_valid_region_radius = 333;
  p->bilateral_filter_sigma_xy = 3;
  p->bilateral_filter_radius_factor = 2.0f;
  p->bilateral_filter_sigma_depth_factor = 0.05;
  p->outlier_filtering_frame_count = 8;
  p->outlier_filtering_required_inliers = -1;
  p->outlier_filtering_depth_tolerance_factor = 0.02f;
  p->depth_erosion_radius = 2;
  p->observation_angle_threshold_deg = 85;
  p->point_radius_extension_factor = 1.5f;
  p->point_radius_clamp_factor = std::numeric_limits<float>::infinity();
}

const char* sm_last_error(void) { return g_last_error.c_str(); }
const char* sm_version(void) { return "surfel_b200 0.1 (sm_90a)"; }
uint64_t sm_kernel_launch_count(void) { return g_launches.load(); }

int sm_profile_kernels(int32_t enable) {
  std::lock_guard<std::mutex> lock(g_profile_mutex);
  g_profile_enabled = enable != 0;
  return SM_OK;
}

int32_t sm_profile_kernel_count(void) { return KID_COUNT; }
const char* sm_profile_kernel_name(int32_t id) { return KernelName(id); }

int sm_profile_report(double* total_ms, uint64_t* launches, int32_t n) {
  SM_CUDA(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lock(g_profile_mutex);
  for (int i = 0; i < n; ++i) { total_ms[i] = 0; launches[i] = 0; }
  for (const ProfileRecord& r : g_profile_records) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, r.start, r.stop) == cudaSuccess && r.id < n) {
      total_ms[r.id] += ms;
      launches[r.id] += 1;
    }
    g_event_pool.push_back(r.start);
    g_event_pool.push_back(r.stop);
  }
  g_profile_records.clear();
  return SM_OK;
}

int sm_create(sm_reconstruction** out, uint64_t max_surfel_count, int32_t width, int32_t height, float fx, float fy,
              float cx, float cy) {
  if (out) *out = nullptr;
  if (!out || width <= 0 || height <= 0 || max_surfel_count == 0 || max_surfel_count > 0x7FFFFFFFull - kSegment) {
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_create: bad argument");
  }
  sm_reconstruction* r = new sm_reconstruction();
  const int status = CreateImpl(r, max_surfel_count, width, height, fx, fy, cx, cy);
  if (status != SM_OK) {
    const std::string message = g_last_error;  // sm_destroy must not overwrite the cause
    sm_destroy(r);
    g_last_error = message;
    return status;
  }
  *out = r;
  return SM_OK;
}

int sm_destroy(sm_reconstruction* r) {
  if (!r) return SM_OK;
  if (r->session) SessionEnd(r, nullptr);   // drains the open session
  cudaDeviceSynchronize();
  cudaGetLastError();
  DestroyFrameGraph(r->graph);
  DeviceState& d = r->d;
  cudaFree(d.surfels); cudaFree(d.gradient); cudaFree(r->reg_records); cudaFree(d.new_list);
  for (int i = 0; i < kSets; ++i) {
    cudaFree(r->vis_set[i]); cudaFree(r->seg_count_set[i]); cudaFree(r->merge_flag_set[i]);
    cudaFree(r->upd_list_set[i]); cudaFree(r->upd_count_set[i]);
    cudaFree(r->assoc_set[i]); cudaFree(r->first_depth_set[i]); cudaFree(r->supported_set[i]);
    cudaFree(r->run_depth[i]); cudaFree(r->run_depth_pre[i]); cudaFree(r->run_normals[i]); cudaFree(r->run_radius[i]);
  }
  cudaFree(d.new_flag); cudaFree(d.new_index); cudaFree(d.scan_state); cudaFree(d.counters);
  cudaFree(d.timeline);
  if (r->host_counters) cudaFreeHost(r->host_counters);
  cudaFree(r->scratch_B);
  cudaFree(r->blend_src);
  cudaFree(r->median_stage[0]); cudaFree(r->median_stage[1]);
  cudaFree(r->pyramid_depth_stage); cudaFree(r->pyramid_color_stage);
  FreeTransferBuffers(r);
  FreeRenderBuffers(r);
  FreeTrackBuffers(r);
  FreeMeshBuffers(r);
  for (cudaStream_t st : {r->upload_stream, r->graph_stream})
    if (st) cudaStreamDestroy(st);
  for (cudaEvent_t e : {r->entry_event, r->upload_done, r->graph_exit})
    if (e) cudaEventDestroy(e);
  for (cudaEvent_t e : r->iteration_done) if (e) cudaEventDestroy(e);
  for (u16* b : r->ring_depth) cudaFree(b);
  for (uchar3* b : r->ring_color) cudaFree(b);
  for (int i = 0; i < 14; ++i) if (r->events.ev[i]) cudaEventDestroy(r->events.ev[i]);
  delete r;
  cudaGetLastError();
  return SM_OK;
}

int sm_reset(sm_reconstruction* r, void* stream) {
  if (r->session) return RejectInSession("sm_reset");
  SM_CUDA(cudaMemsetAsync(r->d.counters, 0, sizeof(Counters), static_cast<cudaStream_t>(stream)));
  r->count_slot = 0;
  r->rasters_cleared = false;
  r->last_stream = static_cast<cudaStream_t>(stream);
  ++r->state_generation;  // tokens of earlier transfers no longer apply
  r->op_history.clear();
  return SM_OK;
}

int sm_preprocess(sm_reconstruction* r, void* stream, const sm_preprocess_params* p, const uint16_t* raw_depth,
                  size_t raw_pitch, const uint16_t* const* other_depths, const size_t* other_pitches,
                  const float* others_TR_reference, uint16_t* out_depth, size_t out_depth_pitch, float* out_normals,
                  size_t out_normals_pitch, float* out_radius, size_t out_radius_pitch) {
  // the frame pipeline of a session pre-processes through the same scratch_B
  if (r->session) return RejectInSession("sm_preprocess");
  const int status = PreprocessFused(static_cast<cudaStream_t>(stream), *p, r->d.width, r->d.height, r->fx, r->fy,
                                     r->cx, r->cy, raw_depth, raw_pitch, other_depths, other_pitches,
                                     others_TR_reference, r->scratch_B, r->scratch_B_pitch, out_depth,
                                     out_depth_pitch, reinterpret_cast<float2*>(out_normals), out_normals_pitch,
                                     out_radius, out_radius_pitch, r->d.assoc, r->d.first_depth, r->d.supported, nullptr, 0,
                                     nullptr, nullptr, r->scratch_B_map);
  if (status == SM_OK) r->rasters_cleared = true;
  return status;
}

int sm_bilateral_filter_and_depth_cutoff(void* stream, float sigma_xy, float sigma_value_factor,
                                         uint16_t value_to_ignore, float radius_factor, uint16_t max_depth,
                                         float depth_valid_region_radius, int32_t width, int32_t height,
                                         const uint16_t* in_depth, size_t in_pitch, uint16_t* out_depth,
                                         size_t out_pitch) {
  return StageBilateral(static_cast<cudaStream_t>(stream), sigma_xy, sigma_value_factor, value_to_ignore,
                        radius_factor, max_depth, depth_valid_region_radius, width, height, in_depth, in_pitch,
                        out_depth, out_pitch);
}

int sm_outlier_depth_map_fusion(void* stream, int32_t other_count, int32_t required_count, float tolerance, float fx,
                                float fy, float cx, float cy, int32_t width, int32_t height, const uint16_t* in_depth,
                                size_t in_pitch, const uint16_t* const* other_depths, const size_t* other_pitches,
                                const float* others_TR_reference, uint16_t* out_depth, size_t out_pitch) {
  return StageOutlier(static_cast<cudaStream_t>(stream), other_count, required_count, tolerance, fx, fy, cx, cy,
                      width, height, in_depth, in_pitch, other_depths, other_pitches, others_TR_reference, out_depth,
                      out_pitch);
}

int sm_median_filter_and_densify_depth_map(void* stream, int32_t iterations, int32_t width, int32_t height,
                                           const uint16_t* in_depth, size_t in_pitch, uint16_t* out_depth,
                                           size_t out_pitch, uint16_t* scratch, size_t scratch_pitch) {
  return StageMedianDensify(static_cast<cudaStream_t>(stream), iterations, width, height, in_depth, in_pitch, out_depth,
                            out_pitch, scratch, scratch_pitch);
}

int sm_downscale_using_median_while_excluding(void* stream, uint16_t value_to_ignore, int32_t in_width,
                                              int32_t in_height, const uint16_t* in, size_t in_pitch,
                                              int32_t out_width, int32_t out_height, uint16_t* out,
                                              size_t out_pitch) {
  return StageDownscaleMedian(static_cast<cudaStream_t>(stream), value_to_ignore, in_width, in_height, in, in_pitch,
                              out_width, out_height, out, out_pitch);
}

int sm_color_image_pyramid(void* stream, int32_t levels, int32_t width, int32_t height, const uint8_t* in,
                           size_t in_pitch, uint8_t* out, size_t out_pitch) {
  return StageColorPyramid(static_cast<cudaStream_t>(stream), levels, width, height, in, in_pitch, out, out_pitch);
}

int sm_erode_depth_map(void* stream, int32_t radius, int32_t width, int32_t height, const uint16_t* in_depth,
                       size_t in_pitch, uint16_t* out_depth, size_t out_pitch) {
  return StageErode(static_cast<cudaStream_t>(stream), radius, width, height, in_depth, in_pitch, out_depth,
                    out_pitch);
}

int sm_compute_normals_and_drop_bad_pixels(void* stream, float observation_angle_threshold_deg, float depth_scaling,
                                           float fx, float fy, float cx, float cy, int32_t width, int32_t height,
                                           const uint16_t* in_depth, size_t in_pitch, uint16_t* out_depth,
                                           size_t out_pitch, float* out_normals, size_t normals_pitch) {
  return StageNormals(static_cast<cudaStream_t>(stream), observation_angle_threshold_deg, depth_scaling, fx, fy, cx,
                      cy, width, height, in_depth, in_pitch, out_depth, out_pitch,
                      reinterpret_cast<float2*>(out_normals), normals_pitch);
}

int sm_compute_point_radii_and_remove_isolated_pixels(void* stream, float point_radius_extension_factor,
                                                      float point_radius_clamp_factor, float depth_scaling, float fx,
                                                      float fy, float cx, float cy, int32_t width, int32_t height,
                                                      const uint16_t* in_depth, size_t in_pitch, float* out_radius,
                                                      size_t radius_pitch, uint16_t* out_depth, size_t out_pitch) {
  return StageRadii(static_cast<cudaStream_t>(stream), point_radius_extension_factor, point_radius_clamp_factor,
                    depth_scaling, fx, fy, cx, cy, width, height, in_depth, in_pitch, out_radius, radius_pitch,
                    out_depth, out_pitch);
}

int sm_integrate(sm_reconstruction* r, void* stream, uint32_t frame_index, const sm_integrate_params* p,
                 uint16_t* depth, size_t depth_pitch, const float* normals, size_t normals_pitch, const float* radius,
                 size_t radius_pitch, const uint8_t* color, size_t color_pitch, const float global_T_local[12],
                 const float local_T_global[12]) {
  if (r->session) return RejectInSession("sm_integrate");
  if (frame_index >= kFrameIndexLimit) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_integrate: frame_index must be below 2^31");
  return IntegrateImpl(r, static_cast<cudaStream_t>(stream), frame_index, *p, depth, depth_pitch, normals,
                       normals_pitch, radius, radius_pitch, color, color_pitch, global_T_local, local_T_global);
}

int sm_regularize(sm_reconstruction* r, void* stream, uint32_t frame_index, float regularizer_weight,
                  float radius_factor_for_regularization_neighbors, int32_t regularization_frame_window_size) {
  if (frame_index >= kFrameIndexLimit) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_regularize: frame_index must be below 2^31");
  r->last_stream = static_cast<cudaStream_t>(stream);
  RecordOperation(r, static_cast<int>(frame_index - static_cast<u32>(regularization_frame_window_size)));
  return RegularizeSurfels(static_cast<cudaStream_t>(stream), r->d, /*disable_denoising*/ false, frame_index,
                           radius_factor_for_regularization_neighbors, regularizer_weight,
                           regularization_frame_window_size, r->count_slot, -1, r->plan);
}

// The two count queries have no stream argument (cuda_surfel_reconstruction.h:125-128): they
// synchronise with the stream of the most recently submitted work.
int sm_surfel_count(sm_reconstruction* r, uint32_t* out) {
  const int status = FetchCounters(r, r->last_stream);
  *out = r->host_counters->surfel_count[r->count_slot] - r->host_counters->merge_count;
  return status;
}

int sm_surfels_size(sm_reconstruction* r, uint32_t* out) {
  const int status = FetchCounters(r, r->last_stream);
  *out = r->host_counters->surfel_count[r->count_slot];
  return status;
}

int sm_transfer_all_to_cpu(sm_reconstruction* r, void* stream_v, uint32_t /*frame_index*/, float* x, float* y,
                           float* z, float* radius_squared, float* nx, float* ny, float* nz,
                           uint32_t* last_update_stamp, uint64_t* out_count) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int status = FetchCounters(r, stream);
  const u32 n = r->host_counters->surfel_count[r->count_slot];
  if (out_count) *out_count = n;
  if (n == 0) return status;
  const size_t bytes = sizeof(float) * n;
  const float* s = r->d.surfels;
  const size_t st = r->d.stride;
  const int mirrored = MirrorRegRecords(stream, r->d, n, r->sm_count);   // rows 3-5 <- the current records
  if (mirrored != SM_OK) return mirrored;
  SM_CUDA(cudaMemcpyAsync(x, s + SM_ROW_SMOOTH_X * st, bytes, cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaMemcpyAsync(y, s + SM_ROW_SMOOTH_Y * st, bytes, cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaMemcpyAsync(z, s + SM_ROW_SMOOTH_Z * st, bytes, cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaMemcpyAsync(radius_squared, s + SM_ROW_RADIUS_SQUARED * st, bytes, cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaMemcpyAsync(nx, s + SM_ROW_NORMAL_X * st, bytes, cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaMemcpyAsync(ny, s + SM_ROW_NORMAL_Y * st, bytes, cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaMemcpyAsync(nz, s + SM_ROW_NORMAL_Z * st, bytes, cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaMemcpyAsync(last_update_stamp, s + SM_ROW_LAST_UPDATE_STAMP * st, bytes, cudaMemcpyDeviceToHost, stream));
  return status;
}

int sm_transfer_delta_to_cpu(sm_reconstruction* r, void* stream, uint32_t frame_index, sm_transfer_token* token,
                             float* x, float* y, float* z, float* radius_squared, float* nx, float* ny, float* nz,
                             uint32_t* last_update_stamp, sm_transfer_stats* stats) {
  if (!r || !token) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_transfer_delta_to_cpu: null argument");
  return TransferDelta(r, static_cast<cudaStream_t>(stream), frame_index, token, x, y, z, radius_squared, nx, ny, nz,
                       last_update_stamp, stats);
}

int sm_update_visualization_buffers(sm_reconstruction* r, void* stream, const sm_visualization_params* p,
                                    float* vertex_buffer, uint32_t* neighbor_index_buffer, float* normal_vertex_buffer) {
  if (!r || !p) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_update_visualization_buffers: null argument");
  return UpdateVisualizationBuffers(r, static_cast<cudaStream_t>(stream), *p, vertex_buffer, neighbor_index_buffer,
                                    normal_vertex_buffer);
}

int sm_render_surfels(sm_reconstruction* r, void* stream, const sm_render_params* p, const float view_T_global[12],
                      float* depth, size_t depth_pitch, uint8_t* color, size_t color_pitch, float* normal,
                      size_t normal_pitch, uint32_t* index, size_t index_pitch) {
  if (!r || !p || !view_T_global) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_render_surfels: null argument");
  return RenderSurfels(r, static_cast<cudaStream_t>(stream), *p, view_T_global, depth, depth_pitch, color, color_pitch,
                       normal, normal_pitch, index, index_pitch);
}

void sm_default_track_params(sm_track_params* p) {
  p->levels = 3;
  p->iterations[0] = 4; p->iterations[1] = 5; p->iterations[2] = 10; p->iterations[3] = 0;
  p->max_point_distance = 0.05f;
  p->max_normal_angle_deg = 20.0f;
  p->min_inlier_fraction = 0.1f;
  p->convergence_rotation = 1e-5f;
  p->convergence_translation = 1e-5f;
  p->model_source = SM_TRACK_CLOUD;
}

int sm_track_frame(sm_reconstruction* r, void* stream, const sm_track_params* tp, const sm_preprocess_params* pp,
                   const uint16_t* depth, size_t depth_pitch, const float global_T_guess[12], float global_T_out[12],
                   sm_track_result* result) {
  if (!r || !tp || !pp || !depth || !global_T_guess || !global_T_out || !result)
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_track_frame: null argument");
  return TrackFrame(r, static_cast<cudaStream_t>(stream), *tp, *pp, depth, depth_pitch, global_T_guess, global_T_out,
                    result);
}

int sm_track_linearize(sm_reconstruction* r, void* stream, const sm_track_params* tp, int32_t level,
                       float depth_scaling, const uint16_t* live_depth, size_t live_pitch, const float* model_depth,
                       size_t model_depth_pitch, const float* model_normal, size_t model_normal_pitch,
                       const float model_T_live[12], double out_system[27], uint32_t* out_inliers) {
  if (!r || !tp || !live_depth || !model_depth || !model_normal || !model_T_live || !out_system || !out_inliers)
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_track_linearize: null argument");
  return TrackLinearize(r, static_cast<cudaStream_t>(stream), *tp, level, depth_scaling, live_depth, live_pitch,
                        model_depth, model_depth_pitch, model_normal, model_normal_pitch, model_T_live, out_system,
                        out_inliers);
}

void sm_default_mesh_params(sm_mesh_params* p) {
  p->neighbor_radius_factor = 2.0f;
  p->max_angle_between_normals_deg = 90.0f;
  p->max_triangle_angle_deg = 170.0f;
}

int sm_triangulate(sm_reconstruction* r, void* stream, const sm_mesh_params* p, uint32_t* triangles, uint64_t capacity,
                   sm_mesh_stats* stats) {
  if (!r || !p || !stats) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_triangulate: null argument");
  return Triangulate(r, static_cast<cudaStream_t>(stream), *p, triangles, capacity, stats);
}

int sm_export_vertices(sm_reconstruction* r, void* stream, float* position_buffer, uint8_t* color_buffer) {
  return ExportVertices(static_cast<cudaStream_t>(stream), r->d, r->count_slot, r->sm_count, position_buffer,
                        color_buffer);
}

int sm_get_timings(sm_reconstruction* r, float out_ms[7]) {
  if (!r->events.enabled) return SetError(SM_ERR_INVALID_ARGUMENT, "timings are not enabled (sm_enable_timings)");
  SM_CUDA(cudaEventSynchronize(r->events.ev[13]));
  for (int i = 0; i < 7; ++i) SM_CUDA(cudaEventElapsedTime(&out_ms[i], r->events.ev[2 * i], r->events.ev[2 * i + 1]));
  return SM_OK;
}

int sm_enable_timings(sm_reconstruction* r, int32_t enable) {
  if (r->session) return RejectInSession("sm_enable_timings");
  r->events.enabled = enable != 0;
  return SM_OK;
}

int sm_dump_state(sm_reconstruction* r, void* stream_v, float* host_rows, uint64_t host_row_stride_elems,
                  uint32_t* surfels_size, uint32_t* merge_count) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int status = FetchCounters(r, stream);
  const u32 n = r->host_counters->surfel_count[r->count_slot];
  if (surfels_size) *surfels_size = n;
  if (merge_count) *merge_count = r->host_counters->merge_count;
  if (host_rows && n > host_row_stride_elems) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_dump_state: host rows shorter than surfels_size()");
  if (host_rows && n > 0) {
    // rows 3-5 and 15: the mirror of the current regularisation records (DeviceState::smooth)
    const int mirrored = MirrorRegRecords(stream, r->d, n, r->sm_count);
    if (mirrored != SM_OK) return mirrored;
    SM_CUDA(cudaMemcpy2DAsync(host_rows, host_row_stride_elems * sizeof(float), r->d.surfels,
                              r->d.stride * sizeof(float), n * sizeof(float), SM_ROW_COUNT, cudaMemcpyDeviceToHost,
                              stream));
    SM_CUDA(cudaStreamSynchronize(stream));
  }
  return status;
}

int sm_load_state(sm_reconstruction* r, void* stream_v, const float* host_rows, uint64_t host_row_stride_elems,
                  uint32_t surfels_size, uint32_t merge_count) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (r->session) return RejectInSession("sm_load_state");
  if (surfels_size > r->d.capacity) return SetError(SM_ERR_CAPACITY, "sm_load_state: state larger than the surfel cap");
  {
    const u32* stamps = reinterpret_cast<const u32*>(host_rows) + SM_ROW_LAST_UPDATE_STAMP * host_row_stride_elems;
    for (u32 i = 0; i < surfels_size; ++i) {
      if (stamps[i] >= kFrameIndexLimit) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_load_state: a last-update stamp is 2^31 or above");
    }
  }
  r->d.reg_full_sweep = 1;  // as after sm_create (both record buffers are packed below)
  if (surfels_size > 0) {
    SM_CUDA(cudaMemcpy2DAsync(r->d.surfels, r->d.stride * sizeof(float), host_rows,
                              host_row_stride_elems * sizeof(float), surfels_size * sizeof(float), SM_ROW_COUNT,
                              cudaMemcpyHostToDevice, stream));
    // Invariant of regularize.cu: gradient accumulators (and the SoA rows they replace) are zero between calls.
    SM_CUDA(cudaMemsetAsync(r->d.gradient, 0, surfels_size * sizeof(float4), stream));
    const int zero_rows[4] = {SM_ROW_GRADIENT_X, SM_ROW_GRADIENT_Y, SM_ROW_GRADIENT_Z, SM_ROW_GRADIENT_COUNT};
    for (int row : zero_rows) {
      SM_CUDA(cudaMemsetAsync(r->d.surfels + row * r->d.stride, 0, surfels_size * sizeof(float), stream));
    }
    // bookkeeping row the library keeps in the reference's unused row 14 (sm_kernels.cuh)
    SM_CUDA(cudaMemsetAsync(r->d.surfels + kRowMergeEpoch * r->d.stride, 0, surfels_size * sizeof(float), stream));
    // both regularisation record buffers from the loaded rows 3-5, stamps and colours
    const int status = PackRegRecords(stream, r->d, surfels_size, r->sm_count);
    if (status != SM_OK) return status;
  }
  Counters c{};
  for (int i = 0; i < kCountSlots; ++i) c.surfel_count[i] = surfels_size;
  c.merge_count = merge_count;
  *r->host_counters = c;
  SM_CUDA(cudaMemcpyAsync(r->d.counters, r->host_counters, sizeof(Counters), cudaMemcpyHostToDevice, stream));
  SM_CUDA(cudaStreamSynchronize(stream));
  r->count_slot = 0;
  r->last_stream = stream;
  ++r->state_generation;  // tokens of earlier transfers no longer apply
  r->op_history.clear();
  return SM_OK;
}

int sm_download_rasters(sm_reconstruction* r, void* stream_v, uint32_t* supporting_surfels,
                        uint32_t* supporting_surfel_counts, float* supporting_surfel_depth_sums,
                        uint32_t* conflicting_surfels, float* first_surfel_depth, uint8_t* new_surfel_flag_vector,
                        uint32_t* new_surfel_indices) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const size_t P = static_cast<size_t>(r->d.width) * r->d.height;
  std::vector<PixelAssoc> assoc(P);
  SM_CUDA(cudaMemcpyAsync(assoc.data(), r->d.assoc, sizeof(PixelAssoc) * P, cudaMemcpyDeviceToHost, stream));
  if (first_surfel_depth)
    SM_CUDA(cudaMemcpyAsync(first_surfel_depth, r->d.first_depth, sizeof(float) * P, cudaMemcpyDeviceToHost, stream));
  if (new_surfel_flag_vector)
    SM_CUDA(cudaMemcpyAsync(new_surfel_flag_vector, r->d.new_flag, P, cudaMemcpyDeviceToHost, stream));
  if (new_surfel_indices)
    SM_CUDA(cudaMemcpyAsync(new_surfel_indices, r->d.new_index, sizeof(u32) * P, cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaStreamSynchronize(stream));
  for (size_t i = 0; i < P; ++i) {
    if (supporting_surfels) supporting_surfels[i] = supporting_index(r->last_tiebreak, assoc[i].x, static_cast<u32>(i));
    if (conflicting_surfels) conflicting_surfels[i] = assoc[i].y;
    if (supporting_surfel_counts) supporting_surfel_counts[i] = assoc[i].z;
    if (supporting_surfel_depth_sums) std::memcpy(&supporting_surfel_depth_sums[i], &assoc[i].w, sizeof(float));
  }
  return SM_OK;
}

int sm_frame_counters(sm_reconstruction* r, void* stream_v, uint64_t out[4]) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int status = FetchCounters(r, stream);
  // The last Integrate() swept the slots that existed before its new surfels were appended.
  const u32 n_after = r->host_counters->surfel_count[r->count_slot];
  const u32 n_swept = n_after - r->host_counters->new_surfel_count;
  const size_t segments = (static_cast<size_t>(n_swept) + kSegment - 1) / kSegment;
  std::vector<u32> seg(segments);
  if (segments) SM_CUDA(cudaMemcpy(seg.data(), r->d.seg_count, sizeof(u32) * segments, cudaMemcpyDeviceToHost));
  uint64_t visible = 0;
  for (u32 c : seg) visible += c;
  const size_t P = static_cast<size_t>(r->d.width) * r->d.height;
  std::vector<PixelAssoc> assoc(P);
  SM_CUDA(cudaMemcpy(assoc.data(), r->d.assoc, sizeof(PixelAssoc) * P, cudaMemcpyDeviceToHost));
  uint64_t support = 0;
  for (const PixelAssoc& a : assoc) support += a.z;
  out[0] = n_swept; out[1] = visible; out[2] = support; out[3] = r->host_counters->new_surfel_count;
  return status;
}

int sm_timeline_enable(sm_reconstruction* r, int32_t frames) {
  if (r == nullptr || frames < 0) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_timeline_enable: bad arguments");
  if (r->session) return RejectInSession("sm_timeline_enable");
  SM_CUDA(cudaDeviceSynchronize());
  if (r->d.timeline) {
    cudaFree(r->d.timeline);
    r->d.timeline = nullptr;
    r->d.timeline_frames = 0;
  }
  if (frames == 0) return SM_OK;
  const size_t slots = static_cast<size_t>(frames) * KID_TIMELINE_COUNT;
  SM_CUDA(cudaMalloc(&r->d.timeline, slots * 2 * sizeof(unsigned long long)));
  std::vector<unsigned long long> init(slots * 2);
  for (size_t i = 0; i < slots; ++i) { init[2 * i] = ~0ull; init[2 * i + 1] = 0ull; }
  SM_CUDA(cudaMemcpy(r->d.timeline, init.data(), init.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice));
  r->d.timeline_frames = static_cast<u32>(frames);
  return SM_OK;
}

int sm_timeline_read(sm_reconstruction* r, uint64_t* out, int32_t frames) {
  if (r == nullptr || out == nullptr) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_timeline_read: bad arguments");
  if (r->d.timeline == nullptr || frames != static_cast<int32_t>(r->d.timeline_frames))
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_timeline_read: timeline not enabled with this frame count");
  SM_CUDA(cudaDeviceSynchronize());
  // Rows of sm_profile_kernel_count() columns; the kernels without a timeline column read "not launched".
  const size_t row = 2 * sizeof(uint64_t) * KID_COUNT, device_row = 2 * sizeof(uint64_t) * KID_TIMELINE_COUNT;
  for (int32_t f = 0; f < frames; ++f) {
    for (int k = KID_TIMELINE_COUNT; k < KID_COUNT; ++k) {
      out[(static_cast<size_t>(f) * KID_COUNT + k) * 2] = ~0ull;
      out[(static_cast<size_t>(f) * KID_COUNT + k) * 2 + 1] = 0ull;
    }
  }
  SM_CUDA(cudaMemcpy2D(out, row, r->d.timeline, device_row, device_row, frames, cudaMemcpyDeviceToHost));
  return SM_OK;
}

// The frame loop of APP/main.cc:885-1223 on a synthetic stream (pipeline.cu).
int sm_stream_run(sm_reconstruction* r, void* stream_v, const sm_stream_desc* s, const sm_preprocess_params* pp,
                  const sm_integrate_params* ip, int32_t first_frame, int32_t last_frame, sm_stream_stats* stats) {
  if (!r || !s || !pp || !ip) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_stream_run: null argument");
  if (r->session) return RejectInSession("sm_stream_run");
  return StreamRun(r, static_cast<cudaStream_t>(stream_v), s, pp, ip, first_frame, last_frame, stats);
}

int sm_outlier_filter_transforms(int32_t other_count, float depth_scaling, int32_t frame_count,
                                 const float* global_T_frame, const float* frame_T_global, int32_t frame, float* out) {
  if (!global_T_frame || !frame_T_global || !out) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_outlier_filter_transforms: null argument");
  if (other_count < 2 || other_count > 8 || other_count % 2 != 0)
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_outlier_filter_transforms: other_count must be 2, 4, 6 or 8");
  const int half = other_count / 2;
  if (frame < half || frame >= frame_count - half)
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_outlier_filter_transforms: the frame needs other_count/2 frames on both sides (main.cc:987-992)");
  const float* ref = global_T_frame + 12 * static_cast<size_t>(frame);
  for (int i = 0; i < half; ++i) {
    OutlierFilterTransform(depth_scaling, ref, frame_T_global + 12 * static_cast<size_t>(frame - (i + 1)), out + 12 * i);
    OutlierFilterTransform(depth_scaling, ref, frame_T_global + 12 * static_cast<size_t>(frame + (i + 1)), out + 12 * (half + i));
  }
  return SM_OK;
}

// An incremental session on the handle (pipeline.cu).
int sm_session_begin(sm_reconstruction* r, void* stream, const sm_preprocess_params* pp, const sm_integrate_params* ip,
                     int32_t frame_width, int32_t frame_height, uint32_t first_frame_index) {
  if (!r || !pp || !ip) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_begin: null argument");
  return SessionBegin(r, static_cast<cudaStream_t>(stream), pp, ip, frame_width, frame_height, first_frame_index);
}

int sm_session_push(sm_reconstruction* r, const uint16_t* depth, size_t depth_pitch, const uint8_t* color,
                    size_t color_pitch, int32_t frame_on_host, const float global_T_frame[12],
                    const float frame_T_global[12], sm_session_status* status) {
  if (!r) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_push: null argument");
  return SessionPush(r, depth, depth_pitch, color, color_pitch, frame_on_host != 0, global_T_frame, frame_T_global,
                     status);
}

int sm_session_end(sm_reconstruction* r, sm_stream_stats* stats) {
  if (!r) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_end: null argument");
  return SessionEnd(r, stats);
}

// Named tuning / experiment knobs of a handle (no counterpart in the reference):
//   "tiebreak_wave"            slots per launch wave of the modelled association race (0 = plain rule)
//   "tiebreak_early_fraction"  fraction of secondary-pixel associations that compete like primary ones
//   "tiebreak_index_order_fraction"  fraction of the pixels whose supporters are ordered by slot index inside a wave
//   "median_filter_and_densify_iterations"  sm_stream_run: MedianFilterAndDensifyDepthMap passes over every raw
//                              depth map on its way into the frame ring (APP/main.cc:435, 927-939; default 0)
//   "pyramid_level"            sm_stream_run: frames are 2^L times the handle's size and are downscaled on their
//                              way into the frame rings (APP/main.cc:299-303, 946-981; default 0)
int sm_configure(sm_reconstruction* r, const char* key, double value) {
  if (!r || !key) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_configure: null argument");
  if (r->session) return RejectInSession("sm_configure");
  const std::string k(key);
  if (k == "tiebreak_wave") {
    if (value < 0 || value > 2147483647.0) return SetError(SM_ERR_INVALID_ARGUMENT, "tiebreak_wave out of range");
    return SetTieBreakWave(&r->tiebreak, static_cast<u32>(value), r->d.capacity);
  }
  if (k == "tiebreak_early_fraction_later" || k == "tiebreak_index_order_fraction_later" || k == "tiebreak_early_fraction_second") {
    // < 0: follow the first wave (later) / the later waves (second)
    if (!(value <= 1.0)) return SetError(SM_ERR_INVALID_ARGUMENT, "tiebreak_*_later / _second must be <= 1 (negative: inherit)");
    (k == "tiebreak_early_fraction_later" ? r->tiebreak.early_fraction_later
     : k == "tiebreak_early_fraction_second" ? r->tiebreak.early_fraction_second : r->tiebreak.index_order_fraction_later) = value;
    return SM_OK;
  }
  if (k == "tiebreak_wave_offset") {   // 1: wave boundaries at a per-pixel random phase
    r->tiebreak.wave_offset = value != 0.0 ? 1u : 0u;
    return SM_OK;
  }
  if (k == "tiebreak_lanes") {   // slots that keep their order inside the shuffled order (1 = none, 32 = a warp)
    const u32 lanes = static_cast<u32>(value);
    if (value < 1 || value > 1024 || (lanes & (lanes - 1)) != 0) return SetError(SM_ERR_INVALID_ARGUMENT, "tiebreak_lanes must be a power of two in [1, 1024]");
    u32 shift = 0;
    while ((1u << shift) < lanes) ++shift;
    r->tiebreak.lane_request = shift;
    return SetTieBreakWave(&r->tiebreak, r->tiebreak.wave, r->d.capacity);
  }
  if (k == "tiebreak_early_fraction") {
    if (!(value >= 0.0 && value <= 1.0)) return SetError(SM_ERR_INVALID_ARGUMENT, "tiebreak_early_fraction must be in [0, 1]");
    r->tiebreak.early_fraction = value;
    return SM_OK;
  }
  if (k == "tiebreak_index_order_fraction") {
    if (!(value >= 0.0 && value <= 1.0)) return SetError(SM_ERR_INVALID_ARGUMENT, "tiebreak_index_order_fraction must be in [0, 1]");
    r->tiebreak.index_order_fraction = value;
    return SM_OK;
  }
  if (k == "median_filter_and_densify_iterations") {
    if (value < 0 || value > 16 || value != static_cast<int>(value)) return SetError(SM_ERR_INVALID_ARGUMENT, "median_filter_and_densify_iterations must be an integer in [0, 16]");
    r->median_iterations = static_cast<int>(value);
    return SM_OK;
  }
  if (k == "pyramid_level") {
    if (value < 0 || value > 4 || value != static_cast<int>(value)) return SetError(SM_ERR_INVALID_ARGUMENT, "pyramid_level must be an integer in [0, 4]");
    r->pyramid_level = static_cast<int>(value);
    return SM_OK;
  }
  return SetError(SM_ERR_INVALID_ARGUMENT, "sm_configure: unknown key");
}

}  // extern "C"
