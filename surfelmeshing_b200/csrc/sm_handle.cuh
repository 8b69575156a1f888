// sm_handle.cuh — the handle behind the C ABI (struct sm_reconstruction), shared by api.cu, which
// creates it, and the files whose entry points work on it.
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

// One buffer set of the frame pipeline: association rasters, visible list, merge flags, neighbour-update list.
struct BufferSet {
  PixelAssoc* assoc = nullptr;
  float* first_depth = nullptr;
  u8* supported = nullptr;
  VisEntry* vis = nullptr;
  u32* seg_count = nullptr;
  u8* merge_flag = nullptr;
  uint2* upd_list = nullptr;
  u32* upd_count = nullptr;
};

// Points `d` at buffer set `s`.
inline void UseSet(DeviceState& d, const BufferSet& s) {
  d.assoc = s.assoc; d.first_depth = s.first_depth; d.supported = s.supported;
  d.vis = s.vis; d.seg_count = s.seg_count; d.merge_flag = s.merge_flag;
  d.upd_list = s.upd_list; d.upd_count = s.upd_count;
}

struct RunBuffers;       // pipeline.cu: the frame loop of sm_stream_run and of sessions
struct StreamSession;    // pipeline.cu: an open sm_session_begin
struct TransferScratch;  // transfer.cu: the staging of sm_transfer_delta_to_cpu
struct RenderScratch;    // render.cu: sm_render_surfels / sm_render_mesh
struct TrackScratch;     // track.cu: sm_track_frame* / sm_track_linearize*
struct MeshScratch;      // mesh.cu: sm_triangulate, and the persistent mesh of sm_mesh_update
struct HoleScratch;      // holes.cu: the buffers of sm_mesh_fill_holes
struct CompactScratch;   // compact.cu: the map and the row scratch of sm_compact
struct SimplifyScratch;  // simplify.cu: the buffers of sm_mesh_simplify
struct TextureScratch;   // texture.cu: the buffers of sm_mesh_texture
struct ComponentScratch;  // components.cu: the buffers of sm_mesh_components

}  // namespace smb

struct sm_reconstruction {
  smb::DeviceState d{};
  int device = 0;
  int sm_count = 0;
  smb::LaunchPlan plan{};
  float fx = 0, fy = 0, cx = 0, cy = 0;
  int count_slot = 0;             // Counters::surfel_count slot holding the current count
  bool rasters_cleared = false;   // the fused pre-processing tail already reset the rasters
  bool rasters_stale = false;     // sm_compact ran after the last Integrate: its rasters name old slots
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
  smb::BufferSet sets[smb::kSets];
  float4* reg_records = nullptr;  // [2][stride]: both regularisation record buffers (DeviceState::smooth / smooth_next)
  // MedianFilterAndDensifyDepthMap passes applied to every raw depth map entering the frame ring
  // (APP/main.cc:435 --median_filter_and_densify_iterations, default 0)
  int median_iterations = 0;
  // Input pyramid level (APP/main.cc:299-303 --pyramid_level, default 0): sm_stream_run takes frames of
  // 2^L times the handle's size and downscales them on the upload stream.
  int pyramid_level = 0;
  // delta transfer (transfer.cu): operation counter, per-operation regularisation thresholds
  smb::u32 op_epoch = 0;
  // Which cloud the handle holds: a fresh value of one process-wide counter at sm_create, sm_reset and
  // sm_load_state (NextStateGeneration), so a token can only match the cloud it was filled from.
  uint64_t state_generation = 0;
  struct Operation { smb::u32 epoch; int stamp_threshold; };
  std::vector<Operation> op_history;
  // incremental session (sm_session_begin .. sm_session_end); nullptr = none open
  smb::StreamSession* session = nullptr;
  // Set while a frame-graph session is open: a device copy of Counters::merge_count as of the newest integrated
  // frame, which FetchCounters reports instead (the front half of a step already counted the next frame's merges).
  const smb::u32* reported_merge_count = nullptr;
  // The scratch of each feature, created by its first call; nullptr = not yet. Its Free... releases it.
  smb::RunBuffers* run = nullptr;
  smb::TransferScratch* transfer = nullptr;
  smb::RenderScratch* render = nullptr;
  smb::TrackScratch* track = nullptr;
  smb::MeshScratch* mesh = nullptr;
  smb::HoleScratch* holes = nullptr;
  smb::CompactScratch* compact = nullptr;
  smb::SimplifyScratch* simplify = nullptr;
  smb::TextureScratch* texture = nullptr;
  smb::ComponentScratch* components = nullptr;
};

namespace smb {
// api.cu
// Calls that would change what an open session builds on (sm_session_begin, include/surfel_b200.h).
int RejectInSession(const char* call);
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
uint64_t NextStateGeneration();   // 1, 2, 3, ... across every handle of the process
void FreeTransferBuffers(sm_reconstruction* r);
// render.cu
int RenderSurfels(sm_reconstruction* r, cudaStream_t stream, const sm_render_params& p, const float* view_T_global,
                  float* depth, size_t depth_pitch, uint8_t* color, size_t color_pitch, float* normal,
                  size_t normal_pitch, uint32_t* index, size_t index_pitch);
int RenderMesh(sm_reconstruction* r, cudaStream_t stream, const sm_render_params& p, const float* view_T_global,
               const uint32_t* triangles, uint64_t triangle_count, int32_t flags, float* depth, size_t depth_pitch,
               uint8_t* color, size_t color_pitch, float* normal, size_t normal_pitch, uint32_t* index,
               size_t index_pitch);
void FreeRenderBuffers(sm_reconstruction* r);
// The camera and pose checks of sm_render_surfels and sm_render_mesh: the reason a camera is refused, or nullptr.
const char* RenderCameraError(const sm_render_params& p, const float* view_T_global);
// track.cu
int TrackFrame(sm_reconstruction* r, cudaStream_t stream, const sm_track_params& tp, const sm_preprocess_params& pp,
               const u16* depth, size_t depth_pitch, const float* guess, float* pose_out, sm_track_result* result);
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
void FreeTrackBuffers(sm_reconstruction* r);
// mesh.cu
void FreeMeshBuffers(sm_reconstruction* r);
// holes.cu
void FreeHoleBuffers(sm_reconstruction* r);
// compact.cu
void FreeCompactBuffers(sm_reconstruction* r);
// simplify.cu
void FreeSimplifyBuffers(sm_reconstruction* r);
// texture.cu
void FreeTextureBuffers(sm_reconstruction* r);
// components.cu
void FreeComponentBuffers(sm_reconstruction* r);
// In place: word w of record k' = word w of record i, old_to_new[i] = k' < kept, for every word of records of
// `record_words` 32-bit words (bytes) over slots [0, n), one word at a time through `scratch` (>= kept words).
// `remap`: the words name slots and are replaced by their new index (SM_INVALID_SURFEL_INDEX for a removed one).
int CompactWords(cudaStream_t stream, int sm_count, const u32* old_to_new, u32 n, u32 kept, u32* base,
                 u32 record_words, u32* scratch, bool remap);
int CompactBytes(cudaStream_t stream, int sm_count, const u32* old_to_new, u32 n, u32 kept, u8* base, u32* scratch);
// mesh.cu: carries the persistent mesh of sm_mesh_update over a compaction of slots [0, n) (`words`: 2 device
// words, `host_words` their pinned mirror); *remapped = 1 if it was carried over, 0 if there was none or it was
// dropped (the next update then rebuilds everything).
int MeshCompact(sm_reconstruction* r, cudaStream_t stream, const u32* old_to_new, u32 n, u32* scratch, u32* words,
                u32* host_words, int* remapped);
// pipeline.cu
int SessionEnd(sm_reconstruction* r, sm_stream_stats* stats);
void FreeRunBuffers(sm_reconstruction* r);
// After sm_compact in an open frame-graph session: runs the front half of the frame in flight again on `stream`
// (its association, merge decisions and blending named the old slots) and resets the reported merge count.
int SessionRefront(sm_reconstruction* r, cudaStream_t stream);
}  // namespace smb
