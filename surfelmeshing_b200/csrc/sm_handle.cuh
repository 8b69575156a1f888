// sm_handle.cuh — the handle behind the C ABI (struct sm_reconstruction), shared by api.cu
// (entry points) and pipeline.cu (the RGB-D stream runner and its frame graph).
#pragma once

#include <vector>

#include "sm_kernels.cuh"

namespace smb {

constexpr int kSets = 3;  // buffer sets of the frame pipeline: frames f, f + 1, f + 2 are in flight

// Supporting-surfel tie-break configuration (sm_configure "tiebreak_*"; TieBreak in sm_kernels.cuh
// holds the per-frame values derived from it).
struct TieBreakConfig {
  u32 wave;              // slots per launch wave of the modelled race (0: plain "primary, then lowest index")
  double early_fraction; // fraction of secondary associations that compete like primary ones
  double index_order_fraction;  // fraction of the pixels that order the supporters of a wave by slot index
  double early_fraction_later, index_order_fraction_later;  // the same two for the waves after the first (< 0: same as the first)
  double early_fraction_second;  // early fraction of the second wave alone (< 0: same as the later waves)
  u32 wave_offset;       // 1: per-pixel random phase of the wave boundaries (sm_kernels.cuh: tb_phase)
  u32 lane_request;      // log2 of the slots that keep their order in the shuffled order (5: a warp of the reference)
  u32 lane_shift;        // what is in effect: lane_request, or 0 when the wave is not a multiple of it
  u32 mul, mul_inv;      // derived from wave and lane_shift
};
// Defaults (DESIGN.md section 4; tools/race_stats.py + tools/race_sets_fit.py on an H100: 641 k contested pixels of
// 31 teacher-forced frames of the 500-frame VGA stream): wave = the reference's AssociateSurfels launch wave on an
// H100 (1024-thread blocks, 31 registers -> 2 blocks x 132 SMs = 264 blocks of slots; the earlier wave won all
// 16 569 contests between two waves). Inside a wave and a kind the lower slot won 100 % of the pairs that sit in one
// warp, ~49 % across the warps of one block and 50 - 74 % across blocks (the warps of a wave in a shuffled order
// that keeps the lanes of a warp in order, and a share of the pixels in plain slot order); a secondary association
// beat a primary one of its wave 2.9 % of the time. Separate fractions for the first wave, the second (at VGA sizes
// only partly filled) and the later ones (1.5 % / 2 % / 4 % early secondaries, 25 % / 45 % / 45 % of the pixels in
// slot order) put the free-running totals of the 500-frame VGA stream within 0.12 % (merges) and 0.03 % (slots) of
// the reference's mean, less than half of its run-to-run spread.
constexpr u32 kDefaultTieBreakWave = 264 * 1024;
constexpr u32 kDefaultTieBreakLaneShift = 5;
constexpr u32 kDefaultTieBreakWaveOffset = 0;
constexpr double kDefaultTieBreakEarlyFraction = 0.015;
constexpr double kDefaultTieBreakIndexOrderFraction = 0.25;
constexpr double kDefaultTieBreakEarlyFractionLater = 0.04;
constexpr double kDefaultTieBreakIndexOrderFractionLater = 0.45;
constexpr double kDefaultTieBreakEarlyFractionSecond = 0.02;
TieBreak MakeTieBreak(const TieBreakConfig& cfg, u32 frame_index);
int SetTieBreakWave(TieBreakConfig* cfg, u32 wave, u32 capacity);   // uses cfg->lane_request

struct FrameGraph;  // pipeline.cu
void DestroyFrameGraph(FrameGraph* g);
struct StreamSession;  // pipeline.cu: an open sm_session_begin
void DestroySession(StreamSession* s);
struct TrackState;     // track.cu
struct MeshCounters;   // mesh.cu
struct MeshLive;       // mesh.cu: the persistent mesh of sm_mesh_update
struct HoleScratch;    // holes.cu: the buffers of sm_mesh_fill_holes

}  // namespace smb

struct sm_reconstruction {
  smb::DeviceState d{};
  int device = 0;
  int sm_count = 0;
  smb::LaunchPlan plan{};
  float fx = 0, fy = 0, cx = 0, cy = 0;
  int count_slot = 0;             // Counters::surfel_count slot holding the current count
  bool rasters_cleared = false;   // the fused pre-processing tail already reset the rasters
  smb::IntegrateEvents events{};
  smb::TieBreakConfig tiebreak{};
  smb::TieBreak last_tiebreak{};  // of the most recent frame (decodes the supporting raster, sm_download_rasters)
  // host mirror of the counters (pinned) for on-demand queries
  smb::Counters* host_counters = nullptr;
  // Stream of the most recently submitted work: the count queries, which have no stream argument,
  // synchronise with it (work on a non-blocking stream is not ordered with the NULL stream).
  cudaStream_t last_stream = nullptr;
  // pre-processing scratch (APP/main.cc filtered_depth_buffer_B)
  smb::u16* scratch_B = nullptr; size_t scratch_B_pitch = 0;
  smb::TensorMapStorage scratch_B_map{};   // TMA descriptor of scratch_B (tile fill of the pre-processing tail)
  // sm_integrate: snapshot of the depth before the measurement blending (k_blend reads the snapshot and
  // writes the caller's buffer: see the kernel)
  smb::u16* blend_src = nullptr; size_t blend_src_pitch = 0;
  // Association rasters / lists per buffer set: the pre-processing tail of a later frame resets one set
  // while Integrate() of an earlier frame still works on another (sm_stream_run).
  smb::PixelAssoc* assoc_set[smb::kSets] = {};
  float* first_depth_set[smb::kSets] = {};
  smb::u8* supported_set[smb::kSets] = {};
  smb::VisEntry* vis_set[smb::kSets] = {};
  smb::u32* seg_count_set[smb::kSets] = {};
  smb::u8* merge_flag_set[smb::kSets] = {};
  uint2* upd_list_set[smb::kSets] = {};
  smb::u32* upd_count_set[smb::kSets] = {};
  // stream-runner buffers (pre-processing outputs per buffer set)
  smb::u16* run_depth[smb::kSets] = {}; size_t run_depth_pitch = 0;
  float2* run_normals[smb::kSets] = {}; size_t run_normals_pitch = 0;
  float* run_radius[smb::kSets] = {}; size_t run_radius_pitch = 0;
  smb::u16* run_depth_pre[smb::kSets] = {};   // pre-blend copy of run_depth (merge runs next to blend)
  float4* reg_records = nullptr;  // [2][stride]: both regularisation record buffers (DeviceState::smooth / smooth_next)
  cudaEvent_t entry_event = nullptr;   // sm_stream_run / sm_session_begin: the start of the frame loop on the caller's stream
  // host-resident streams: raw-depth / colour rings filled by the upload stream
  std::vector<smb::u16*> ring_depth; size_t ring_depth_pitch = 0;
  std::vector<uchar3*> ring_color; size_t ring_color_pitch = 0;
  cudaStream_t upload_stream = nullptr;
  cudaEvent_t upload_done = nullptr;
  // MedianFilterAndDensifyDepthMap passes applied to every raw depth map entering the ring
  // (APP/main.cc:435 --median_filter_and_densify_iterations, default 0) and their staging buffers
  int median_iterations = 0;
  smb::u16* median_stage[2] = {nullptr, nullptr}; size_t median_stage_pitch = 0;
  // Input pyramid level (APP/main.cc:299-303 --pyramid_level, default 0): sm_stream_run takes frames of
  // 2^L times the handle's size and downscales them on the upload stream; host frames pass through
  // full-size staging buffers of pyramid_stage_width x pyramid_stage_height pixels.
  int pyramid_level = 0;
  smb::u16* pyramid_depth_stage = nullptr; size_t pyramid_depth_stage_pitch = 0;
  smb::u8* pyramid_color_stage = nullptr; size_t pyramid_color_stage_pitch = 0;
  int pyramid_stage_width = 0, pyramid_stage_height = 0;
  std::vector<cudaEvent_t> iteration_done;   // frame loop: one event per step slot (ring reuse)
  // delta transfer (transfer.cu): operation counter, per-operation regularisation thresholds, staging
  smb::u32 op_epoch = 0;
  uint64_t state_generation = 1;   // bumped by sm_reset / sm_load_state
  struct Operation { smb::u32 epoch; int stamp_threshold; };
  std::vector<Operation> op_history;
  smb::u32* delta_index = nullptr; float* delta_values = nullptr; smb::u32* delta_cursor = nullptr;
  smb::u32 delta_capacity = 0;
  smb::u32* delta_host = nullptr; size_t delta_host_capacity = 0;   // pinned, in 32-bit words
  // frame graph (pipeline.cu)
  cudaStream_t graph_stream = nullptr;
  cudaEvent_t graph_exit = nullptr;
  smb::FrameGraph* graph = nullptr;
  // incremental session (sm_session_begin .. sm_session_end); nullptr = none open
  smb::StreamSession* session = nullptr;
  // Set while a frame-graph session is open: a device copy of Counters::merge_count as of the newest integrated
  // frame, which FetchCounters reports instead (the front half of a step already counted the next frame's merges).
  const smb::u32* reported_merge_count = nullptr;
  // sm_render_surfels scratch (render.cu), allocated by the first render: the key raster (all keys "empty"
  // between calls), the large-splat list (capacity slots) and its count (zero between calls), resident grids.
  unsigned long long* render_keys = nullptr; size_t render_key_capacity = 0;   // in pixels
  smb::u32* render_large_list = nullptr;
  smb::u32* render_large_count = nullptr;
  int render_splat_blocks = 0, render_large_blocks = 0;
  // sm_render_mesh scratch (render.cu) beyond the above, allocated by the first mesh render: one bit per slot of
  // capacity (corners of the triangles drawn), the large-triangle list (grown to the triangle count) and its count
  // (zero between calls), resident grids.
  smb::u32* mesh_render_marks = nullptr;
  smb::u32* mesh_render_large_list = nullptr; smb::u32 mesh_render_large_capacity = 0;   // in triangles
  smb::u32* mesh_render_large_count = nullptr;
  int mesh_render_mark_blocks = 0, mesh_render_tri_blocks = 0, mesh_render_large_blocks = 0;
  int mesh_render_splat_blocks = 0, mesh_render_splat_large_blocks = 0;
  // sm_track_frame / sm_track_linearize scratch (track.cu), allocated by the first call: the filtered live pyramid,
  // the rendered model view, two level-0 views of tracked frames (depth, normals) of which track_previous is the
  // newest, the pose that call returned, the per-block partial rows and the device / pinned tracker state (allocated
  // last: non-null means every buffer exists).
  smb::u16* track_level[4] = {}; size_t track_level_pitch[4] = {};
  float* track_model_depth = nullptr; size_t track_model_depth_pitch = 0;
  float* track_model_normal = nullptr; size_t track_model_normal_pitch = 0;
  float* track_view_depth[2] = {}; size_t track_view_depth_pitch[2] = {};
  float* track_view_normal[2] = {}; size_t track_view_normal_pitch[2] = {};
  int track_previous = 0;
  bool track_has_previous = false;
  float track_previous_pose[12] = {};
  double* track_partials = nullptr;
  int track_blocks = 0;
  smb::TrackState* track_state = nullptr;
  smb::TrackState* track_host_state = nullptr;
  // sm_track_frame_rgbd / sm_track_linearize_rgbd scratch (track.cu), allocated by the first RGB-D call: the model
  // colour the render writes, the live and model intensity pyramids, the level-0 live intensity kept for the next
  // SM_TRACK_PREVIOUS_FRAME call (allocated last: non-null means every buffer exists), the partial rows of the RGB-D
  // linearisation's resident grid, and whether the previous tracking call was an RGB-D call.
  smb::u8* track_model_color = nullptr; size_t track_model_color_pitch = 0;
  float* track_live_intensity[4] = {}; size_t track_live_intensity_pitch[4] = {};
  float* track_model_intensity[4] = {}; size_t track_model_intensity_pitch[4] = {};
  double* track_rgbd_partials = nullptr;
  int track_rgbd_blocks = 0;
  float* track_kept_intensity = nullptr; size_t track_kept_intensity_pitch = 0;
  bool track_previous_rgbd = false;
  // sm_triangulate scratch (mesh.cu), allocated by the first call and grown to surfels_size(): the k-NN index over
  // the smooth positions, the umbrellas ([mesh_slots][SM_MESH_MAX_UMBRELLA] pairs) and their lengths, the per-slot
  // triangle counts (scanned in place into offsets) and the scan's tile sums; the device counters and their
  // pinned mirror; resident grids.
  sm_knn_index* mesh_index = nullptr;
  uint2* mesh_umbrella = nullptr;
  smb::u32* mesh_umbrella_count = nullptr;
  smb::u32* mesh_counts = nullptr;
  smb::u32* mesh_scan_sums = nullptr;
  smb::u32 mesh_slots = 0;
  smb::MeshCounters* mesh_counters = nullptr;
  smb::MeshCounters* mesh_host_counters = nullptr;
  int mesh_umbrella_blocks = 0, mesh_emit_blocks = 0;
  // sm_mesh_update's persistent mesh (mesh.cu), created by the first update; it shares only mesh_index.
  smb::MeshLive* mesh_live = nullptr;
  // sm_mesh_fill_holes scratch (holes.cu), created by the first call with more than zero triangles.
  smb::HoleScratch* holes = nullptr;
};

namespace smb {
// api.cu
int FetchCounters(sm_reconstruction* r, cudaStream_t stream);
FrameParams MakeFrameParams(const sm_reconstruction* r, u32 frame_index, int count_slot, const sm_integrate_params& p,
                            u16* depth, size_t depth_pitch, const u16* depth_pre, size_t depth_pre_pitch,
                            const float* normals, size_t normals_pitch, const float* radius, size_t radius_pitch,
                            const uint8_t* color, size_t color_pitch, const float* global_T_local,
                            const float* local_T_global);
int IntegrateImpl(sm_reconstruction* r, cudaStream_t stream, u32 frame_index, const sm_integrate_params& p, u16* depth,
                  size_t depth_pitch, const float* normals, size_t normals_pitch, const float* radius,
                  size_t radius_pitch, const uint8_t* color, size_t color_pitch, const float* global_T_local,
                  const float* local_T_global);
void CountLaunches(unsigned long long n);
unsigned long long LaunchCount();
// transfer.cu
void RecordOperation(sm_reconstruction* r, int stamp_threshold);   // one Integrate() / Regularize(): ++op_epoch
void FreeTransferBuffers(sm_reconstruction* r);
int TransferDelta(sm_reconstruction* r, cudaStream_t stream, uint32_t frame_index, sm_transfer_token* token, float* x,
                  float* y, float* z, float* radius_squared, float* nx, float* ny, float* nz,
                  uint32_t* last_update_stamp, sm_transfer_stats* stats);
int UpdateVisualizationBuffers(sm_reconstruction* r, cudaStream_t stream, const sm_visualization_params& p, float* vertex,
                               uint32_t* neighbor_index, float* normal_vertex);
// render.cu
int RenderSurfels(sm_reconstruction* r, cudaStream_t stream, const sm_render_params& p, const float* view_T_global,
                  float* depth, size_t depth_pitch, uint8_t* color, size_t color_pitch, float* normal,
                  size_t normal_pitch, uint32_t* index, size_t index_pitch);
int RenderMesh(sm_reconstruction* r, cudaStream_t stream, const sm_render_params& p, const float* view_T_global,
               const uint32_t* triangles, uint64_t triangle_count, int32_t flags, float* depth, size_t depth_pitch,
               uint8_t* color, size_t color_pitch, float* normal, size_t normal_pitch, uint32_t* index,
               size_t index_pitch);
void FreeRenderBuffers(sm_reconstruction* r);
// track.cu
int TrackFrame(sm_reconstruction* r, cudaStream_t stream, const sm_track_params& tp, const sm_preprocess_params& pp,
               const u16* depth, size_t depth_pitch, const float* guess, float* pose_out, sm_track_result* result);
int TrackLinearize(sm_reconstruction* r, cudaStream_t stream, const sm_track_params& tp, int level, float depth_scaling,
                   const u16* live, size_t live_pitch, const float* model_depth, size_t model_depth_pitch,
                   const float* model_normal, size_t model_normal_pitch, const float* model_T_live, double* out_system,
                   uint32_t* out_inliers);
// The photometric part of an RGB-D call (sm_track_frame_rgbd / sm_track_linearize_rgbd): the parameters, the raw
// live colour and, for the linearisation alone, the caller's model colour.
struct TrackColor {
  const sm_track_rgbd_params* params;
  const uint8_t* live; size_t live_pitch;
  const uint8_t* model; size_t model_pitch;
};
int TrackFrameRGBD(sm_reconstruction* r, cudaStream_t stream, const sm_track_params& tp, const sm_preprocess_params& pp,
                   const TrackColor& color, const u16* depth, size_t depth_pitch, const float* guess, float* pose_out,
                   sm_track_rgbd_result* result);
int TrackLinearizeRGBD(sm_reconstruction* r, cudaStream_t stream, const sm_track_params& tp, const TrackColor& color,
                       int level, float depth_scaling, const u16* live, size_t live_pitch, const float* model_depth,
                       size_t model_depth_pitch, const float* model_normal, size_t model_normal_pitch,
                       const float* model_T_live, double* out_system, double* out_sum_rc2, uint32_t* out_inliers,
                       uint32_t* out_photometric_inliers);
void FreeTrackBuffers(sm_reconstruction* r);
// mesh.cu
int Triangulate(sm_reconstruction* r, cudaStream_t stream, const sm_mesh_params& p, uint32_t* triangles,
                uint64_t capacity, sm_mesh_stats* stats);
void FreeMeshBuffers(sm_reconstruction* r);
int MeshUpdate(sm_reconstruction* r, cudaStream_t stream, const sm_mesh_params& p, sm_mesh_update_stats* stats);
int MeshRead(sm_reconstruction* r, cudaStream_t stream, int32_t which, uint32_t* triangles, uint64_t capacity,
             uint64_t* count);
// holes.cu
int FillHoles(sm_reconstruction* r, cudaStream_t stream, const sm_hole_params& p, const uint32_t* triangles,
              uint64_t count, uint32_t* fill, uint64_t capacity, sm_hole_stats* stats);
void FreeHoleBuffers(sm_reconstruction* r);
// pipeline.cu
int StreamRun(sm_reconstruction* r, cudaStream_t stream, const sm_stream_desc* s, const sm_preprocess_params* pp,
              const sm_integrate_params* ip, int first_frame, int last_frame, sm_stream_stats* stats);
int SessionBegin(sm_reconstruction* r, cudaStream_t stream, const sm_preprocess_params* pp,
                 const sm_integrate_params* ip, int width, int height, uint32_t first_frame_index);
int SessionPush(sm_reconstruction* r, const u16* depth, size_t depth_pitch, const uint8_t* color, size_t color_pitch,
                bool on_host, const float* global_T_frame, const float* frame_T_global, sm_session_status* status);
int SessionEnd(sm_reconstruction* r, sm_stream_stats* stats);
// out (3x4) = scale(other_T_global) . scale(global_T_ref) (sm_outlier_filter_transforms)
void OutlierFilterTransform(float depth_scaling, const float* global_T_ref, const float* other_T_global, float* out);
}  // namespace smb
