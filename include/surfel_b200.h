/*
 * surfel_b200.h — C ABI of libsurfel_b200.so, the Hopper-native (sm_90a)
 * replacement for the per-frame surfel reconstruction hot path of
 * puzzlepaint/surfelmeshing.
 *
 * Every entry point cites the reference interface it replaces (paths relative
 * to the reference tree; APP = applications/surfel_meshing/src/surfel_meshing).
 *
 * Conventions
 *  - Plain pointers and sizes only; `stream` is a cudaStream_t passed as void*.
 *  - Rasters are row-pitched device buffers (pitch in BYTES, as handed out by
 *    cudaMallocPitch / libvis CUDABuffer<T>, libvis/src/libvis/cuda/cuda_buffer_inl.h:36-48).
 *  - Rigid transforms are 3x4 row-major float[12] (= libvis CUDAMatrix3x4 rows,
 *    libvis/src/libvis/cuda/cuda_matrix.cuh:67-116).
 *  - Camera intrinsics are the reference's PinholeCamera4f::parameters()
 *    {fx, fy, cx, cy} in pixel-CORNER convention (cx_file + 0.5), APP/
 *    cuda_surfel_reconstruction_kernels.cc:63-74.
 *  - Every function returns SM_OK (0) or a negative SM_ERR_* code; the message is
 *    available from sm_last_error(). (Reference: no return values, CUDA errors
 *    abort through LOG(FATAL), libvis/src/libvis/cuda/cuda_util.h:35-49. The
 *    C++ adapter in surfel_b200_adapter.h maps non-zero to LOG(FATAL).)
 *  - There is NO CPU fallback: if the CUDA runtime or an sm_90 device is not
 *    available the calls fail with SM_ERR_CUDA.
 */
#ifndef SURFEL_B200_H_
#define SURFEL_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SM_OK 0
#define SM_ERR_CUDA (-1)
#define SM_ERR_INVALID_ARGUMENT (-2)
#define SM_ERR_CAPACITY (-3) /* surfel cap exceeded (reference: unchecked overflow) */

/* Row indices of the surfel SoA (row = attribute, column = surfel), identical
 * to APP/cuda_surfel_reconstruction_kernels.cuh:48-78. */
enum {
  SM_ROW_X = 0, SM_ROW_Y = 1, SM_ROW_Z = 2,
  SM_ROW_SMOOTH_X = 3, SM_ROW_SMOOTH_Y = 4, SM_ROW_SMOOTH_Z = 5,
  SM_ROW_CONFIDENCE = 6, SM_ROW_RADIUS_SQUARED = 7,
  SM_ROW_NORMAL_X = 8, SM_ROW_NORMAL_Y = 9, SM_ROW_NORMAL_Z = 10,
  SM_ROW_GRADIENT_X = 11, SM_ROW_GRADIENT_Y = 12, SM_ROW_GRADIENT_Z = 13,
  SM_ROW_ACCUM_X = 14, SM_ROW_ACCUM_Y = 15, SM_ROW_ACCUM_Z = 16,
  SM_ROW_CREATION_STAMP = 17, SM_ROW_LAST_UPDATE_STAMP = 18,
  SM_ROW_NEIGHBOR0 = 19, /* ..22 */
  SM_ROW_GRADIENT_COUNT = 23,
  SM_ROW_COLOR = 24,
  SM_ROW_COUNT = 25
};
#define SM_INVALID_SURFEL_INDEX 0xFFFFFFFFu /* APP/surfel.h:63, kernels.cu:74 */

/* Opaque handle: owns the surfel SoA, the scratch rasters, the compact index
 * lists and the timing events. Replaces class vis::CUDASurfelReconstruction,
 * APP/cuda_surfel_reconstruction.h:44-176. One handle per device/stream;
 * re-entrant per handle, no globals (the reference keeps a function-static
 * device buffer, APP/cuda_surfel_reconstruction_kernels.cc:479). */
typedef struct sm_reconstruction sm_reconstruction;

/* Arguments of CUDASurfelReconstruction::Integrate() that are not buffers,
 * APP/cuda_surfel_reconstruction.h:59-77; defaults APP/main.cc:279-371. */
typedef struct sm_integrate_params {
  float depth_scaling;                                       /* 5000 */
  float sensor_noise_factor;                                 /* 0.05 */
  float max_surfel_confidence;                               /* 5 */
  float regularizer_weight;                                  /* 10 */
  int32_t regularization_frame_window_size;                  /* 30 */
  int32_t do_blending;                                       /* 1 */
  int32_t measurement_blending_radius;                       /* 12 */
  int32_t regularization_iterations_per_integration_iteration; /* 1 */
  float radius_factor_for_regularization_neighbors;          /* 2 */
  float normal_compatibility_threshold_deg;                  /* 40 */
  int32_t surfel_integration_active_window_size;             /* INT_MAX */
} sm_integrate_params;

/* Arguments of the depth pre-processing call sequence APP/main.cc:1015-1191;
 * defaults APP/main.cc:415-478. */
typedef struct sm_preprocess_params {
  float depth_scaling;                          /* 5000 */
  float max_depth;                              /* 3 (metres) */
  float depth_valid_region_radius;              /* 333 (pixels) */
  float bilateral_filter_sigma_xy;              /* 3 */
  float bilateral_filter_radius_factor;         /* 2 */
  float bilateral_filter_sigma_depth_factor;    /* 0.05 */
  int32_t outlier_filtering_frame_count;        /* 8 (2,4,6,8) */
  int32_t outlier_filtering_required_inliers;   /* -1 = all */
  float outlier_filtering_depth_tolerance_factor; /* 0.02 */
  int32_t depth_erosion_radius;                 /* 2 (0..3) */
  float observation_angle_threshold_deg;        /* 85 */
  float point_radius_extension_factor;          /* 1.5 */
  float point_radius_clamp_factor;              /* +inf */
} sm_preprocess_params;

void sm_default_integrate_params(sm_integrate_params* p);
void sm_default_preprocess_params(sm_preprocess_params* p);

const char* sm_last_error(void);
/* Library/arch identification string, e.g. "surfel_b200 0.1 (sm_90a)". */
const char* sm_version(void);

/* ---- lifecycle ----------------------------------------------------------
 * sm_create replaces the CUDASurfelReconstruction constructor,
 * APP/cuda_surfel_reconstruction.cc:44-91 (max_surfel_count, camera; the three
 * GL resources and the render window are GUI-only and have no equivalent).
 * Uses the current CUDA device. */
int sm_create(sm_reconstruction** out, uint64_t max_surfel_count,
              int32_t width, int32_t height,
              float fx, float fy, float cx, float cy);
int sm_destroy(sm_reconstruction* r);
/* Empties the surfel cloud (surfel_count_ = merge_count_ = 0), stream-ordered. */
int sm_reset(sm_reconstruction* r, void* stream);

/* ---- depth pre-processing (SURVEY §8 a1-a5, a16) ------------------------
 * One call = the five launches of APP/main.cc:1015-1191:
 *   BilateralFilteringAndDepthCutoffCUDA  (APP/cuda_depth_processing.cu:120-158)
 *   OutlierDepthMapFusionCUDA<K+1,u16>    (:229-285 / :399-457)
 *   ErodeDepthMapCUDA | CopyWithoutBorder (:540-579 / :609-633)
 *   ComputeNormalsAndDropBadPixelsCUDA    (:720-762)
 *   ComputePointRadiiAndRemoveIsolatedPixelsCUDA (:839-883)
 * raw_depth: this frame's uploaded u16 depth. other_depths[k] /
 * other_pitches[k] / others_TR_reference[12*k..]: the K = outlier_filtering_
 * frame_count other RAW depth maps and (ref_T_global_scaled *
 * global_T_other_scaled)^-1 exactly as built at APP/main.cc:1039-1058 (host
 * arrays; device pointers inside). Outputs: out_depth (the reference's
 * filtered_depth_buffer_A handed to Integrate), out_normals (float2 per
 * pixel), out_radius (SQUARED radius per pixel; like the reference it is only
 * written where the normals stage kept a depth). */
int sm_preprocess(sm_reconstruction* r, void* stream,
                  const sm_preprocess_params* p,
                  const uint16_t* raw_depth, size_t raw_pitch,
                  const uint16_t* const* other_depths, const size_t* other_pitches,
                  const float* others_TR_reference,
                  uint16_t* out_depth, size_t out_depth_pitch,
                  float* out_normals, size_t out_normals_pitch,
                  float* out_radius, size_t out_radius_pitch);

/* The five stages individually (same kernels the fused call is built from);
 * these are what the vis::-named link shims forward to. */
int sm_bilateral_filter_and_depth_cutoff(
    void* stream, float sigma_xy, float sigma_value_factor, uint16_t value_to_ignore,
    float radius_factor, uint16_t max_depth, float depth_valid_region_radius,
    int32_t width, int32_t height,
    const uint16_t* in_depth, size_t in_pitch, uint16_t* out_depth, size_t out_pitch);
int sm_outlier_depth_map_fusion(
    void* stream, int32_t other_count, int32_t required_count /* -1 = all */,
    float tolerance, float fx, float fy, float cx, float cy,
    int32_t width, int32_t height,
    const uint16_t* in_depth, size_t in_pitch,
    const uint16_t* const* other_depths, const size_t* other_pitches,
    const float* others_TR_reference,
    uint16_t* out_depth, size_t out_pitch);
/* MedianFilterAndDensifyDepthMap(), APP/main.cc:207-252, which the reference runs on the CPU
 * inside its upload loop (main.cc:927-939): `iterations` passes (main.cc:435,
 * --median_filter_and_densify_iterations) of the 3x3 zero-excluding median that also fills
 * holes with >= 2 valid neighbours. Device buffers; `scratch` (same size) is needed for more
 * than one pass; the result is in out_depth. iterations == 0 copies. */
int sm_median_filter_and_densify_depth_map(
    void* stream, int32_t iterations, int32_t width, int32_t height,
    const uint16_t* in_depth, size_t in_pitch, uint16_t* out_depth, size_t out_pitch,
    uint16_t* scratch, size_t scratch_pitch);
/* The input downscaling of --pyramid_level (APP/main.cc:299-303), which the reference runs on the CPU
 * inside its upload loop (main.cc:946-981). Device buffers, pitches in bytes.
 * sm_downscale_using_median_while_excluding replaces Image<u16>::DownscaleUsingMedianWhileExcluding
 * (libvis image.h:1003-1050; main.cc:951-952): output pixel (x, y) is the median of the input block
 * [W x / out_width, W (x + 1) / out_width) x [H y / out_height, H (y + 1) / out_height) (integer
 * division) without the values equal to value_to_ignore, value_to_ignore if none is left; for an even
 * count the middle value closer to the float average, the upper one on a tie. Blocks up to 16 x 16.
 * sm_color_image_pyramid replaces ImagePyramid(color, levels) (libvis image_cache.h:205-282; main.cc:
 * 973-981): `levels` rounds of Image<Vec3u8>::DownscaleToHalfSize (image.h:929-948), a/4 + b/4 + c/4 +
 * d/4 per channel with each quarter truncated; out is (width >> levels) x (height >> levels) packed
 * uchar3; levels == 0 copies. Both return SM_ERR_INVALID_ARGUMENT for an empty output or one larger than
 * the input, blocks larger than 16 x 16, levels outside [0, 4] or a size that is odd at some level. */
int sm_downscale_using_median_while_excluding(void* stream, uint16_t value_to_ignore,
                                              int32_t in_width, int32_t in_height,
                                              const uint16_t* in, size_t in_pitch,
                                              int32_t out_width, int32_t out_height,
                                              uint16_t* out, size_t out_pitch);
int sm_color_image_pyramid(void* stream, int32_t levels, int32_t width, int32_t height,
                           const uint8_t* in, size_t in_pitch, uint8_t* out, size_t out_pitch);
int sm_erode_depth_map(void* stream, int32_t radius /* 0 = copy w/o border */,
                       int32_t width, int32_t height,
                       const uint16_t* in_depth, size_t in_pitch,
                       uint16_t* out_depth, size_t out_pitch);
int sm_compute_normals_and_drop_bad_pixels(
    void* stream, float observation_angle_threshold_deg, float depth_scaling,
    float fx, float fy, float cx, float cy, int32_t width, int32_t height,
    const uint16_t* in_depth, size_t in_pitch, uint16_t* out_depth, size_t out_pitch,
    float* out_normals, size_t normals_pitch);
int sm_compute_point_radii_and_remove_isolated_pixels(
    void* stream, float point_radius_extension_factor, float point_radius_clamp_factor,
    float depth_scaling, float fx, float fy, float cx, float cy,
    int32_t width, int32_t height,
    const uint16_t* in_depth, size_t in_pitch, float* out_radius, size_t radius_pitch,
    uint16_t* out_depth, size_t out_pitch);

/* ---- Integrate / Regularize (SURVEY §8 a6-a15) ---------------------------
 * sm_integrate replaces CUDASurfelReconstruction::Integrate(),
 * APP/cuda_surfel_reconstruction.cc:112-320. `depth` is in/out (blended in
 * place, :201-213); `color` is packed uchar3 rows. global_T_local and
 * local_T_global = global_T_local^-1 are both supplied so that both sides of
 * a parity test consume bit-identical matrices (the reference computes the
 * inverse with Sophus on the host, :144,:156,:181,:251).
 * Unlike the reference the call does NOT block the host (the reference
 * synchronises twice, cuda_surfel_reconstruction_kernels.cc:509 and
 * cuda_surfel_reconstruction.cc:290): counts stay device-resident and are
 * fetched by sm_surfel_count()/sm_surfels_size() on demand.
 *
 * Frame indices, and so last-update stamps, must stay below 2^31: the
 * window test int(stamp) >= int(frame_index - window) compares them as int,
 * and the regularisation records keep the detach flag in bit 31 of the
 * stamp. sm_integrate and sm_regularize return SM_ERR_INVALID_ARGUMENT, and
 * launch nothing, for frame_index >= 2^31; sm_load_state does the same for a
 * state with a last-update stamp >= 2^31. */
int sm_integrate(sm_reconstruction* r, void* stream, uint32_t frame_index,
                 const sm_integrate_params* p,
                 uint16_t* depth, size_t depth_pitch,
                 const float* normals, size_t normals_pitch,
                 const float* radius, size_t radius_pitch,
                 const uint8_t* color, size_t color_pitch,
                 const float global_T_local[12], const float local_T_global[12]);

/* Replaces CUDASurfelReconstruction::Regularize(), cuda_surfel_reconstruction.cc:322-337. */
int sm_regularize(sm_reconstruction* r, void* stream, uint32_t frame_index,
                  float regularizer_weight,
                  float radius_factor_for_regularization_neighbors,
                  int32_t regularization_frame_window_size);

/* surfel_count() = entries - merged, surfels_size() = entries in use
 * (cuda_surfel_reconstruction.h:125-128). Both synchronise with the stream of
 * the most recently submitted call on this handle and return the counters of
 * that call. */
int sm_surfel_count(sm_reconstruction* r, uint32_t* out);
int sm_surfels_size(sm_reconstruction* r, uint32_t* out);

/* Replaces TransferAllToCPU(), cuda_surfel_reconstruction.cc:339-359: fills the
 * eight CUDASurfelBuffersCPU arrays (APP/cuda_surfels_cpu.h:40-73: SMOOTH x,y,z,
 * radius^2, normal x,y,z, last-update stamp), surfels_size() entries each. The
 * host arrays may be pageable (as in the reference) or pinned. *out_count
 * receives surfels_size(). Stream-ordered; the caller synchronises the stream
 * before reading, as APP/main.cc:1261-1287 does. */
int sm_transfer_all_to_cpu(sm_reconstruction* r, void* stream, uint32_t frame_index,
                           float* x, float* y, float* z, float* radius_squared,
                           float* nx, float* ny, float* nz, uint32_t* last_update_stamp,
                           uint64_t* out_count);

/* Delta form of TransferAllToCPU (SURVEY section 8 f1). The reference copies all eight rows on
 * every transfer (cuda_surfel_reconstruction.cc:339-359; 160 MB at 5 M surfels, into pageable
 * memory) and its consumer then compares every CPU surfel with the arrays
 * (SurfelMeshing::IntegrateCUDABuffers, APP/surfel_meshing.cc:189-288). This call brings arrays
 * that hold an EARLIER transfer up to date: the slots whose transferred attributes can have
 * changed since then (new, integrated, regularised, merged) are compacted on the GPU, moved with
 * one copy through pinned staging and scattered into the untouched CUDASurfelBuffersCPU layout;
 * afterwards the arrays are identical to what sm_transfer_all_to_cpu would have produced.
 * `token` identifies the transfer that last filled THESE arrays (zero-initialise it for arrays
 * that were never filled: the call then does a full transfer) and is updated; with the
 * reference's write/read double buffer (cuda_surfels_cpu.h:83-124) keep one token per buffer.
 * After sm_reset / sm_load_state, or when most of the cloud changed, the call falls back to the
 * full transfer. Synchronises `stream`. */
typedef struct sm_transfer_token {
  uint64_t generation;    /* 0 = never */
  uint64_t epoch;
  uint64_t surfel_count;
} sm_transfer_token;
typedef struct sm_transfer_stats {
  uint64_t surfel_count;   /* surfels_size() */
  uint64_t changed_count;  /* records moved (= surfel_count for a full transfer) */
  uint64_t d2h_bytes;
  int32_t full_transfer;
  int32_t reserved;
} sm_transfer_stats;
int sm_transfer_delta_to_cpu(sm_reconstruction* r, void* stream, uint32_t frame_index,
                             sm_transfer_token* token,
                             float* x, float* y, float* z, float* radius_squared,
                             float* nx, float* ny, float* nz, uint32_t* last_update_stamp,
                             sm_transfer_stats* stats /* may be NULL */);

/* Replaces ExportVertices(), cuda_surfel_reconstruction.cc:405-410 /
 * kernels.cu:2412-2464: packed xyz (NaN for merged) and rgb, device buffers of
 * 3*surfels_size() elements each. */
int sm_export_vertices(sm_reconstruction* r, void* stream,
                       float* position_buffer, uint8_t* color_buffer);

/* Replaces UpdateVisualizationBuffers(), cuda_surfel_reconstruction.cc:361-403, and the three
 * kernels behind it (UpdateSurfelVertexBufferCUDA, UpdateNeighborIndexBufferCUDA,
 * UpdateNormalVertexBufferCUDA, kernels.cu:274-560) with one sweep. The reference writes CUDA-mapped
 * OpenGL buffers (cudaGraphicsResource_t); here the caller passes the mapped device pointers
 * (cudaGraphicsResourceGetMappedPointer) or any plain device buffers; a NULL pointer skips that
 * buffer, as the reference skips a null resource:
 *   vertex_buffer          surfels_size() x point_size_in_floats floats: x (NaN hides a surfel that
 *                          was replaced after the last triangulation), y, z, rgba bits
 *   neighbor_index_buffer  surfels_size() x 4 x {surfel, neighbour-or-surfel} u32 (16-byte aligned)
 *   normal_vertex_buffer   surfels_size() x {p, p + radius * normal} floats */
typedef struct sm_visualization_params {
  uint32_t frame_index;
  uint32_t latest_triangulated_frame_index;
  uint32_t latest_mesh_surfel_count;
  int32_t surfel_integration_active_window_size;
  uint32_t point_size_in_floats;               /* sizeof(Point3fC3u8) / sizeof(float) = 4 */
  int32_t visualize_last_update_timestamp;
  int32_t visualize_creation_timestamp;
  int32_t visualize_radii;
  int32_t visualize_normals;
} sm_visualization_params;
int sm_update_visualization_buffers(sm_reconstruction* r, void* stream, const sm_visualization_params* p,
                                    float* vertex_buffer, uint32_t* neighbor_index_buffer,
                                    float* normal_vertex_buffer);

/* ---- rendering the surfel cloud into any pinhole camera (DESIGN.md section 1 row f7, section 5.5) ----
 * The reference shows the cloud in its Qt/OpenGL render window, where a geometry shader draws each surfel of
 * the UpdateVisualizationBuffers vertex buffer as a splat (APP/surfel_meshing_render_window.cc:239-300,
 * 948-1003). sm_render_surfels draws it without a display: every surfel as an oriented disk, into a
 * deterministic z-buffer, from any camera and at any image size (independent of the handle's camera).
 *
 * Slots i in [0, surfels_size()) with radius_squared (row 7) > 0 are drawn (merged surfels, radius^2 < 0, are
 * not). The disk has centre s = the current SMOOTH position (what TransferAllToCPU, the viewer and the meshing
 * thread see), normal n = rows 8-10, squared radius row 7 and colour the low three bytes of row 24. Per
 * surfel, in fp32 with denormals flushed to zero, no contraction:
 *   1. c = view_T_global * s (per row: t = s.y*r.y; t = fma(s.x, r.x, t); t = fma(s.z, r.z, t); t + r.w) and
 *      m = R(view_T_global) * n (the same without + r.w).
 *   2. The surfel is skipped unless near_depth <= c.z <= far_depth.
 *   3. For pixel (px, py): dx = ((float(px) + 0.5f) - cx) / fx and dy = ((float(py) + 0.5f) - cy) / fy
 *      (IEEE division), the ray (dx, dy, 1); den = fma(m.z, 1, fma(m.x, dx, m.y*dy)) and
 *      num = fma(m.z, c.z, fma(m.x, c.x, m.y*c.y)); the pixel is skipped if den == 0; t = num / den (IEEE)
 *      must be finite and > 0; e = (t*dx - c.x, t*dy - c.y, t - c.z); the pixel is covered iff
 *      fma(e.z, e.z, fma(e.x, e.x, e.y*e.y)) <= radius^2. There is no back-face culling.
 *   4. A covered pixel proposes the key (bits(t) << 32) | i and keeps the smallest key: the nearest surfel
 *      wins, equal depths go to the lower slot, so the images do not depend on the order of the GPU's work.
 *   5. Outputs from the winning key: depth = t, index = i, colour = the low three bytes of row 24 (r, g, b),
 *      normal = m (camera frame, not re-normalised). Pixels without a covering surfel get 0 and
 *      SM_INVALID_SURFEL_INDEX.
 * Each surfel only tests the pixels of a screen rectangle that contains every pixel step 3 can accept (the
 * projection of its bounding sphere, rounded outwards); a sphere that reaches the camera plane tests the whole
 * image. Which pixels are covered is decided by step 3 alone.
 *
 * Outputs are device buffers of height rows, pitches in bytes, any of them NULL but not all: depth f32,
 * colour packed u8x3, normal f32x3, index u32. Bytes past a row's width x element size stay untouched.
 * Asynchronous on `stream`, no host synchronisation; surfels_size() is read on the device. The handle keeps
 * an 8-byte-per-pixel key raster and a list of large splats: the first call, and a call with a larger
 * image, allocate them (sm_create allocates nothing for rendering). Only reads the surfel state.
 * SM_ERR_INVALID_ARGUMENT (and no launch) for width or height <= 0, fx or fy zero or not finite, cx, cy or a
 * pose entry not finite, near_depth <= 0 or far_depth <= near_depth (either NaN included), a non-NULL output
 * whose pitch is below its row size, or all outputs NULL. */
typedef struct sm_render_params {
  int32_t width, height;        /* output image size */
  float fx, fy, cx, cy;         /* pinhole intrinsics, pixel-corner convention as sm_create */
  float near_depth, far_depth;  /* metres: a surfel is drawn iff near_depth <= its camera-space z <= far_depth */
} sm_render_params;
int sm_render_surfels(sm_reconstruction* r, void* stream, const sm_render_params* p,
                      const float view_T_global[12],     /* 3x4 row-major, global -> camera */
                      float* depth, size_t depth_pitch,
                      uint8_t* color, size_t color_pitch,
                      float* normal, size_t normal_pitch,
                      uint32_t* index, size_t index_pitch);

/* ---- camera tracking against the cloud (DESIGN.md section 1 row f8, section 5.6) ----------------------------
 * The reference reads every camera pose from a trajectory file (APP/main.cc:601-625) and has no tracker.
 * sm_track_frame estimates the pose of a depth map by projective point-to-plane ICP against a model view,
 * coarse to fine, with every Gauss-Newton iteration on the device. It only reads the surfel state.
 *
 * sm_track_frame, in order, on `stream`:
 *  1. Live images. Level 0 is the raw depth (u16, the handle's camera size) through the bilateral filter and depth
 *     cutoff of sm_bilateral_filter_and_depth_cutoff with pp's bilateral_filter_*, depth_scaling * max_depth and
 *     depth_valid_region_radius (the first pre-processing stage of the stream loop). Level l = 1..levels-1 is level
 *     0 downscaled as sm_downscale_using_median_while_excluding(0, ...) does, to the size of Camera.scaled(l):
 *     int(W / 2^l + 0.5) x int(H / 2^l + 0.5), intrinsics fx / 2^l, fy / 2^l, cx / 2^l, cy / 2^l (pixel corner).
 *  2. Model view at the handle's camera. SM_TRACK_CLOUD: sm_render_surfels from view_T_global = the fp64 inverse
 *     of global_T_guess rounded to fp32, depth range [0.1, 100] m, depth and normal only; the model pose is the
 *     guess. SM_TRACK_PREVIOUS_FRAME: the level-0 view (step 3) of this handle's previous sm_track_frame call;
 *     the model pose is the pose that call returned. Every level associates into this one full-size view.
 *     The starting model_T_live is inverse(model pose) * global_T_guess (fp64, rounded to fp32). Before that, the
 *     3x3 parts of the guess and of the model pose are replaced by their nearest rotations (polar decomposition in
 *     fp64), and so is the returned pose: fp32 poses are a few ulp off SO(3), and a chain of calls that feeds each
 *     returned pose into the next guess would otherwise carry that scale and shear forward and amplify it.
 *  3. The level-0 view of this frame is kept for the next call: per pixel z and n of rule L below (0 where L
 *     rejects the pixel).
 *  4. For level = levels-1 down to 0, iterations[level] times: linearise (rules L and M below), then solve.
 *  5. One synchronisation; then global_T_out = model pose * model_T_live (fp64, rounded to fp32), or
 *     global_T_guess if the frame is lost. Synchronous, like sm_knn_batch_host; every SM_OK call keeps its view
 *     and its returned pose as the "previous frame".
 *
 * Per live pixel (x, y) of a level of size w x h and intrinsics fx, fy, cx, cy, in fp32 with every product, sum
 * and quotient rounded on its own (no fma), IEEE division and square root; a.b = (a.x*b.x + a.y*b.y) + a.z*b.z:
 *  L1. The pixel is skipped at the border (x = 0, y = 0, x = w-1, y = h-1) and if any of the depths at (x, y),
 *      (x+-1, y), (x, y+-1) is 0. Otherwise valid_pixels counts it.
 *  L2. P(u, v) = z * (((u + 0.5) - cx) / fx, ((v + 0.5) - cy) / fy, 1) with z = depth * (1 / depth_scaling)
 *      (the reciprocal rounded once); p = P(x, y). a = P(x+1, y) - P(x-1, y), b = P(x, y+1) - P(x, y-1);
 *      n = b x a (per component (b.y*a.z) - (b.z*a.y) etc.: faces the camera), then n = n * (1 / sqrt(n.n));
 *      the pixel is skipped (and not counted) unless n.n is finite and > 0.
 *  M1. With T = model_T_live (device memory, rows r): p' = ((r.x*p.x + r.y*p.y) + r.z*p.z) + r.w per row, n' the
 *      same without r.w. The pixel is an outlier unless p'.z > 0.
 *  M2. u = fmx * (p'.x / p'.z) + mcx, v likewise (the model camera = the handle's camera); outlier unless
 *      0 <= u < W and 0 <= v < H; (ix, iy) = (int(u), int(v)).
 *  M3. d = model depth at (ix, iy): outlier unless finite and > 0. m = model normal at (ix, iy) normalised as in
 *      L2 (outlier if that fails); q = d * (((ix + 0.5) - mcx) / mfx, ((iy + 0.5) - mcy) / mfy, 1); m = -m if
 *      m.q > 0 (the renderer draws both faces of a disk).
 *  M4. e = p' - q. Inlier iff e.e <= max_point_distance^2 (fp32) and n'.m >= cos(max_normal_angle_deg)
 *      (evaluated in double, rounded to fp32).
 *  M5. r = m.e, J = (p' x m, m) (cross product as in L2) for the increment xi = (omega, v) applied as
 *      T <- exp(xi) T in the model camera frame. The 21 products J_i J_j (i <= j, row by row), the 6 J_i r,
 *      r^2 and the inlier and valid counts are formed and summed in fp64 (fixed per-thread, warp-shuffle and
 *      block orders, one partial row per block, no atomics: a call reproduces bit for bit).
 * Solve (one block, fp64): the partial rows are summed in block order. The frame is lost if inliers <
 * min_inlier_fraction * valid_pixels, a Cholesky pivot of J^T J is <= 0 or the step is not finite; otherwise
 * xi = -(J^T J)^-1 J^T r, T <- exp(xi) T (Rodrigues, the SE(3) left Jacobian for the translation), rounded to fp32.
 * |omega| < convergence_rotation and |v| < convergence_translation end the level; the remaining iterations of a
 * level that converged, and all after a loss, return at once (the launch count does not depend on the data).
 * result: tracked (0 = lost, global_T_out = global_T_guess), iterations = steps applied, inliers / valid_pixels /
 * rms_residual = sqrt(sum r^2 / inliers) of the last level-0 linearisation. A lost frame still returns SM_OK.
 *
 * sm_track_linearize runs one linearisation (rules L and M) on caller images, synchronously: live_depth is the
 * filtered u16 image of Camera.scaled(level) of the handle's camera; model_depth (f32) and model_normal (f32x3)
 * are at the handle's camera size. out_system = the 21 J^T J sums then the 6 J^T r sums; out_inliers = inliers.
 *
 * Scratch (the live pyramid, the model view, two level-0 views, one partial row per resident block of the
 * linearisation, the state) is allocated by the first call; sm_create allocates nothing for tracking.
 * SM_ERR_INVALID_ARGUMENT, with no launch, for NULL pointers, a pitch below the row size, levels outside [1, 4],
 * a negative iterations entry, a non-finite pose, a guess whose 3x3 part has a determinant <= 0, a non-finite threshold (max_point_distance <= 0, max_normal_angle_deg
 * outside [0, 180], min_inlier_fraction outside [0, 1], a negative convergence threshold, depth_scaling <= 0),
 * SM_TRACK_PREVIOUS_FRAME without an earlier sm_track_frame call on the handle, or a level whose image is smaller
 * than 3 x 3 pixels. */
#define SM_TRACK_CLOUD 0
#define SM_TRACK_PREVIOUS_FRAME 1
typedef struct sm_track_params {
  int32_t levels;                  /* live-depth pyramid levels, 1..4 (3) */
  int32_t iterations[4];           /* Gauss-Newton iterations per level, finest first ({4, 5, 10, 0}) */
  float max_point_distance;        /* metres, correspondence gate (0.05) */
  float max_normal_angle_deg;      /* live vs model normal gate (20) */
  float min_inlier_fraction;       /* of the level's valid live pixels; below it the frame is lost (0.1) */
  float convergence_rotation;      /* rad (1e-5) */
  float convergence_translation;   /* metres (1e-5) */
  int32_t model_source;            /* SM_TRACK_CLOUD or SM_TRACK_PREVIOUS_FRAME (SM_TRACK_CLOUD) */
} sm_track_params;
typedef struct sm_track_result {
  int32_t tracked;                 /* 0 = lost: global_T_out = global_T_guess */
  int32_t iterations;              /* Gauss-Newton steps applied, all levels */
  uint32_t inliers, valid_pixels;  /* level 0, last linearisation */
  float rms_residual;              /* metres, level 0, last linearisation */
} sm_track_result;
/* Host only, no device needed. */
void sm_default_track_params(sm_track_params* p);
int sm_track_frame(sm_reconstruction* r, void* stream, const sm_track_params* tp, const sm_preprocess_params* pp,
                   const uint16_t* depth, size_t depth_pitch,   /* raw u16, device, the handle's camera size */
                   const float global_T_guess[12], float global_T_out[12], sm_track_result* result);
int sm_track_linearize(sm_reconstruction* r, void* stream, const sm_track_params* tp, int32_t level,
                       float depth_scaling,
                       const uint16_t* live_depth, size_t live_pitch,   /* filtered level image, device */
                       const float* model_depth, size_t model_depth_pitch,
                       const float* model_normal, size_t model_normal_pitch,
                       const float model_T_live[12], double out_system[27], uint32_t* out_inliers);

/* ---- triangulating the surfel cloud (DESIGN.md section 1 row f9, section 5.7) ---------------------------------
 * The reference's meshing thread grows its mesh by advancing triangle fronts one surfel at a time
 * (APP/surfel_meshing.cc:667-752), which is sequential by construction. sm_triangulate meshes the whole current
 * cloud at once with a different, local rule: every slot proposes the triangles of its umbrella, and a triangle is
 * output when its three corners propose it alike. Only reads the surfel state.
 *
 * Slots i in [0, surfels_size()) with radius_squared (row 7) > 0 take part ("present"). Slot i has position p_i =
 * its current SMOOTH position, radius^2 r_i^2 and normal n_i = rows 8-10 times 1 / sqrt(n.n) (IEEE square root and
 * division); a slot whose n.n is not finite and > 0 has no umbrella and is nobody's neighbour. In fp32 with
 * denormals flushed to zero and no contraction, a.b = (a.x*b.x + a.y*b.y) + a.z*b.z, 2D a.b = a.x*b.x + a.y*b.y,
 * cross(a, b) = a.x*b.y - a.y*b.x, each product, sum and quotient rounded on its own; f2 = f * f with
 * f = neighbor_radius_factor, cos_n and cos_t = cos(angle in radians) of the two angle parameters, evaluated in
 * double and rounded to float:
 *  1. Neighbours. The <= 64 nearest present slots j with (d^2, j) ascending, d^2 = ((dx*dx + dy*dy) + dz*dz) <=
 *     r_i^2 * f2 (what sm_knn_query returns), i itself dropped wherever it ranks; then every j with n_i.n_j < cos_n.
 *  2. Tangent plane. sign = copysign(1, n.z), a = -1 / (sign + n.z), b = (n.x * n.y) * a,
 *     u = (1 + ((sign * n.x) * n.x) * a, sign * b, -(sign * n.x)), v = (b, sign + (n.y * n.y) * a, -n.y)
 *     (Duff et al. 2017: u x v = n). q_j = ((p_j - p_i).u, (p_j - p_i).v). A neighbour with q_j = (0, 0), or with
 *     the same q as a neighbour of lower rank, is dropped.
 *  3. Umbrella. On the bisector of j, parametrised by s (the point q_j / 2 + (s / 2) (-q_j.y, q_j.x)), every
 *     other neighbour k sets c = cross(q_j, q_k), b = q_k.q_k - q_j.q_k. c == 0: j is dropped if b < 0, else k sets
 *     nothing. c > 0: an upper end t = b / c; c < 0: a lower end t = b / c. hi = the smallest upper end, lo = the
 *     largest lower end, each with the smallest slot index among the neighbours that set it (hi_min, lo_min).
 *     j is kept iff it has no lower or no upper end, or lo < hi, or lo == hi (bisectors through one point:
 *     cocircular neighbours) and min(i, j) < min(lo_min, hi_min), so that the four slots of a cocircular quad
 *     agree on its diagonal. next(j) = among the kept k with c > 0 and b / c == hi, the first counter-clockwise
 *     from j (k replaces the current choice m iff cross(q_k, q_m) > 0, k in rank order); none if j has no upper
 *     end (an open cell: a boundary). A slot that is next(j) of two or more j is nobody's next. U(i) = the pairs
 *     {j, next(j)} in the rank order of j. A slot with more than SM_MESH_MAX_UMBRELLA pairs has an empty umbrella
 *     and counts as an umbrella overflow.
 *  4. Triangles. For {a, b} in U(i), the triangle (i, a, b) is output iff {b, i} is in U(a), {i, a} is in U(b),
 *     and, in the rotation (o, x, y) that starts at o = min(i, a, b): with e1 = p_x - p_o, e2 = p_y - p_o, the
 *     geometric normal (e1.y*e2.z - e1.z*e2.y, e1.z*e2.x - e1.x*e2.z, e1.x*e2.y - e1.y*e2.x) has g.n_o > 0, and
 *     at each corner (o: e1, e2; x: p_y - p_x, p_o - p_x; y: p_o - p_y, p_x - p_y) with edges (g, h) it is not
 *     true that g.h < cos_t * sqrt((g.g) * (h.h)). It is written once, by o, as (o, x, y): counter-clockwise
 *     about n_o. A directed edge lies in at most one output triangle, so the mesh is edge-manifold and
 *     consistently oriented.
 *  5. Order: by owner slot, then by the owner's umbrella order.
 * stats: triangle_count (set also when the capacity is too small), vertices_meshed = present slots that are a
 * corner of an output triangle, boundary_edges = edges in exactly one output triangle, umbrella_overflows.
 *
 * triangles is a DEVICE buffer of 3 x capacity uint32 (may be NULL with capacity 0: a count query). If capacity <
 * triangle_count the call returns SM_ERR_CAPACITY with stats filled and nothing written. The call synchronises
 * `stream` three times (surfels_size(), the largest radius, the triangle count); on return the triangles are
 * written by work enqueued on `stream`, ordered before anything the caller enqueues there next. The k-NN index uses
 * cells of 2 * sqrt(max r_i^2 * f2) (a query touches at most 3 cells per axis; one slot with a huge radius makes
 * every query walk more records, never a different answer). Scratch (the index, SM_MESH_MAX_UMBRELLA pairs and a
 * few words per slot) belongs to the handle, is allocated by the first call and grows to surfels_size(); sm_create
 * allocates nothing for meshing. SM_ERR_INVALID_ARGUMENT, with no launch, for NULL params or stats, triangles NULL
 * with capacity > 0, a neighbor_radius_factor that is not finite and > 0 (or whose square overflows), or an angle
 * that is not in (0, 180]. */
#define SM_MESH_MAX_UMBRELLA 16
typedef struct sm_mesh_params {
  float neighbor_radius_factor;          /* 2   (main.cc max_neighbor_search_range_increase_factor) */
  float max_angle_between_normals_deg;   /* 90  (main.cc default) */
  float max_triangle_angle_deg;          /* 170 (main.cc default) */
} sm_mesh_params;
typedef struct sm_mesh_stats {
  uint64_t triangle_count;    /* always set, also when capacity was too small */
  uint64_t vertices_meshed;   /* present slots with >= 1 output triangle */
  uint64_t boundary_edges;    /* edges in exactly one output triangle */
  uint64_t umbrella_overflows;
} sm_mesh_stats;
/* Host only, no device needed. */
void sm_default_mesh_params(sm_mesh_params* p);
int sm_triangulate(sm_reconstruction* r, void* stream, const sm_mesh_params* p,
                   uint32_t* triangles /* device, 3 x capacity */, uint64_t capacity, sm_mesh_stats* stats);

/* ---- radius-limited k-nearest-neighbour queries for the meshing thread (SURVEY section 8 f4) ----
 * Replaces CompressedOctree::FindNearestSurfelsWithinRadius<include_completed_surfels, include_free_surfels>
 * (octree.h:471, octree.cc:313-470; callers surfel_meshing.cc:421 <false, true> and :821 <true, false>) for a BATCH of
 * queries against one snapshot of the cloud: per query the <= max_result_count (<= 64) nearest points with
 * squared distance <= radius_squared, ascending, the meshing-state filter applied before the cap, exactly what
 * the octree returns (equal distances, which the octree leaves to its traversal order, come out by ascending
 * index). All pointers are DEVICE pointers; the calls are asynchronous on `stream`. An index lives on the CUDA device that
 * was current at sm_knn_create; that device must be current for every later call on it (as for a reconstruction handle).
 *
 *   sm_knn_create   index for up to max_points points (<= 2^26)
 *   sm_knn_build    bins points [0, point_count) into a hashed uniform grid of `cell_size` (choose it near the
 *                   largest query radius: a query visits the (2 r / cell_size + 1)^3 cells its ball touches).
 *                   A point is left out if radius_squared (optional) is <= 0 at its index (merged surfels,
 *                   kernels.cu:1987) or state (optional) is 255 there.
 *   sm_knn_build_from_reconstruction   the same over the handle's current surfels: smooth positions (what
 *                   TransferAllToCPU hands to the meshing thread, cuda_surfel_reconstruction.cc:345-347) of
 *                   all slots with radius_squared > 0.
 *   sm_knn_query    state (optional, one byte per point index: 0 free, 1 front, 2 completed, 255 absent; Surfel::
 *                   MeshingState, surfel.h:67-71) is read at query time, so one index serves both callers.
 *                   Outputs: [query_count][max_result_count] squared distances (+inf past the count) and indices
 *                   (0xFFFFFFFF past the count), [query_count] counts. */
typedef struct sm_knn_index sm_knn_index;
int sm_knn_create(sm_knn_index** out, uint32_t max_points);
void sm_knn_destroy(sm_knn_index* k);
int sm_knn_build(sm_knn_index* k, void* stream, uint32_t point_count, const float* x, const float* y, const float* z,
                 const float* radius_squared /* may be NULL */, const uint8_t* state /* may be NULL */, float cell_size);
int sm_knn_build_from_reconstruction(sm_knn_index* k, sm_reconstruction* r, void* stream, float cell_size,
                                     uint32_t* out_point_count /* may be NULL */);
int sm_knn_query(sm_knn_index* k, void* stream, uint32_t query_count, const float* qx, const float* qy, const float* qz,
                 const float* radius_squared, const uint8_t* state /* may be NULL */, int32_t include_completed_surfels,
                 int32_t include_free_surfels, int32_t max_result_count, float* out_distance_squared,
                 uint32_t* out_index, int32_t* out_count);
/* One neighbour batch for a meshing iteration with HOST arrays on both sides (the CUDASurfelBuffersCPU arrays of the
 * last TransferAllToCPU, cuda_surfels_cpu.h:40-73): uploads x, y, z, radius_squared [point_count], indexes the points with
 * radius_squared > 0, asks for every point its <= max_result_count nearest members within radius_factor_squared *
 * radius_squared[i] (all meshing states; max_neighbor_search_range_increase_factor^2 covers every radius
 * TriangulateSurfel can ask for, surfel_meshing.cc:323-413) and writes the [point_count][max_result_count] rows and
 * [point_count] counts to host memory (count 0 for points that are not indexed). cell_size <= 0: twice the largest
 * query radius. Synchronous; the device staging lives in the index and is reused. */
int sm_knn_batch_host(sm_knn_index* k, void* stream, uint32_t point_count, const float* x, const float* y, const float* z,
                      const float* radius_squared, float radius_factor_squared, float cell_size, int32_t max_result_count,
                      float* out_distance_squared, uint32_t* out_index, int32_t* out_count);

/* Replaces GetTimings(), cuda_surfel_reconstruction.cc:412-429 (milliseconds of
 * the last Integrate: data association, merging, blending, integration,
 * neighbour update, new-surfel creation, regularisation). */
int sm_get_timings(sm_reconstruction* r, float out_ms[7]);
/* Event timing costs a few microseconds per frame; off by default. */
int sm_enable_timings(sm_reconstruction* r, int32_t enable);

/* ---- state access for parity tests / checkpointing ----------------------
 * The reference has no save/load (SURVEY §5); these move the 25-row SoA and
 * the two counters. rows: SM_ROW_COUNT x surfels_size floats, row-major. */
int sm_dump_state(sm_reconstruction* r, void* stream, float* host_rows,
                  uint64_t host_row_stride_elems, uint32_t* surfels_size, uint32_t* merge_count);
int sm_load_state(sm_reconstruction* r, void* stream, const float* host_rows,
                  uint64_t host_row_stride_elems, uint32_t surfels_size, uint32_t merge_count);

/* Scratch rasters of the last Integrate, de-interleaved into the reference's
 * per-pixel buffers (cuda_surfel_reconstruction.h:133-144), tightly packed
 * W*H host arrays; any pointer may be NULL. */
int sm_download_rasters(sm_reconstruction* r, void* stream,
                        uint32_t* supporting_surfels, uint32_t* supporting_surfel_counts,
                        float* supporting_surfel_depth_sums, uint32_t* conflicting_surfels,
                        float* first_surfel_depth, uint8_t* new_surfel_flag_vector,
                        uint32_t* new_surfel_indices);

/* ---- RGB-D stream runner (the frame loop of APP/main.cc:885-1223) ---------
 * Runs preprocess + Integrate over frames [first_frame, last_frame) of a
 * stream whose other-frame transforms were precomputed by the caller. With
 * frames_on_host != 0 the depth/colour pointers are (pinned) host memory and
 * each raw depth map / colour image is uploaded once on an internal copy
 * stream, overlapped with compute, exactly like the reference's upload_stream
 * (APP/main.cc:902-995); otherwise they are device-resident.
 * The call never synchronises with the host inside the loop and overlaps the
 * kernels of three consecutive frames (one instantiated CUDA graph per frame
 * step on an internal stream, DESIGN.md section 5); `stream` only brackets the call: work enqueued on it
 * before the call is complete before the first frame starts, work enqueued
 * after the call sees all frames integrated. The call itself returns after
 * one synchronisation at the end (to fetch the counters for `stats`). With
 * sm_enable_timings(r, 1) or sm_profile_kernels(1) the frames run one kernel
 * after the other on `stream`. */
typedef struct sm_stream_desc {
  int32_t width, height, frame_count;
  int32_t frames_on_host;
  const uint16_t* depth;         /* frame_count x H x W, tightly packed */
  const uint8_t* color;          /* frame_count x H x W x 3 */
  const float* global_T_frame;   /* frame_count x 12, host */
  const float* frame_T_global;   /* frame_count x 12, host */
  const float* others_TR_reference; /* frame_count x K x 12, host (K = outlier_filtering_frame_count) */
} sm_stream_desc;

typedef struct sm_stream_stats {
  uint32_t frames_integrated;
  uint32_t surfels_size;      /* entries in use after the last frame */
  uint32_t surfel_count;      /* entries - merged */
  uint64_t kernel_launches;   /* kernels this library launched during the call */
  uint64_t h2d_bytes;         /* bytes uploaded inside the call */
  uint64_t d2h_bytes;         /* bytes downloaded inside the call */
  double host_enqueue_ms;     /* host time spent enqueuing the frames (before the final synchronisation) */
} sm_stream_stats;

int sm_stream_run(sm_reconstruction* r, void* stream, const sm_stream_desc* s,
                  const sm_preprocess_params* pp, const sm_integrate_params* ip,
                  int32_t first_frame, int32_t last_frame, sm_stream_stats* stats);

/* The K = other_count outlier-filter transforms of reference frame `frame` (APP/main.cc:1039-1058) from
 * per-frame poses (frame_count x 12 each, host): out[k] for the other frame o = frame - (k + 1) (k < K/2)
 * or frame + (k - K/2 + 1) (k >= K/2), the layout sm_preprocess and sm_stream_desc.others_TR_reference
 * take. Host only, no device needed. With A = frame_T_global[o] and B = global_T_frame[frame], both with
 * their translation column multiplied by depth_scaling, out[k] = A . B, which equals the reference's
 * (ref_T_global_scaled . global_T_other_scaled)^-1 without an explicit inverse. Every value is converted
 * to double and every entry is evaluated as
 *     m[r][c] = ((A[r][0] * B[0][c] + A[r][1] * B[1][c]) + A[r][2] * B[2][c])            (c < 3)
 *     m[r][3] = (((A[r][0] * B[0][3] + A[r][1] * B[1][3]) + A[r][2] * B[2][3]) + A[r][3])
 * (A[r][3] = double(frame_T_global[o][4 r + 3]) * double(depth_scaling), likewise B[k][3]), then rounded to
 * float once. SM_ERR_INVALID_ARGUMENT for other_count not in {2, 4, 6, 8}, NULL pointers, or a frame without
 * K/2 neighbours on both sides in [0, frame_count). */
int sm_outlier_filter_transforms(int32_t other_count, float depth_scaling, int32_t frame_count,
                                 const float* global_T_frame, const float* frame_T_global,
                                 int32_t frame, float* out /* other_count x 12 */);

/* ---- incremental stream sessions (the frame loop of APP/main.cc:885-1293, one frame per call) ----------
 * A session runs the same pipeline as sm_stream_run on frames that arrive one at a time. The k-th pushed
 * frame has frame index first_frame_index + k (first_frame_index + frames pushed < 2^30); frame_width x
 * frame_height is the sensor size, as sm_stream_desc.width/height (the handle's size, or 2^L times it with
 * "pyramid_level" L). A frame is integrated once its K/2 successors were pushed (K = pp's
 * outlier_filtering_frame_count, 2, 4, 6 or 8); the first K/2 and the last K/2 frames of a session are never
 * integrated (main.cc:987-992). The session computes frame f's outlier-filter transforms, as
 * sm_outlier_filter_transforms does, from the pushed poses when frame f + K/2 arrives (pp.depth_scaling).
 *
 * In frame-graph mode pushing frame p launches the step {integrate p - K/2 - 2, associate p - K/2 - 1,
 * pre-process p - K/2}, so status.last_integrated_frame becomes p - K/2 - 2; sm_session_end launches the
 * remaining steps. The session runs serially on `stream` wherever sm_stream_run does (sm_enable_timings,
 * sm_profile_kernels); a push of frame p then integrates p - K/2.
 *
 * Frames: with frame_on_host != 0, depth / colour are host memory, pageable or pinned. The push copies them
 * into pinned staging owned by the library before it returns (main.cc:942-944, 974-976), so the caller may
 * reuse the buffers at once; it blocks only while that staging slot's previous frame is still being
 * uploaded. Otherwise they are device memory: they are copied (or downscaled / median-filtered, as in
 * sm_stream_run) into the library's rings after the work enqueued on `stream`
 * before the push, and `stream` waits for that copy, so work the caller enqueues on `stream` after the push
 * may overwrite them. depth is u16 rows, colour packed u8x3 rows, pitches in bytes.
 *
 * Between pushes, calls on `stream` see the state after status.last_integrated_frame, and the next push's
 * work waits for them: the hand-off calls (sm_transfer_all_to_cpu, sm_transfer_delta_to_cpu,
 * sm_update_visualization_buffers, sm_export_vertices, sm_dump_state, sm_download_rasters,
 * sm_frame_counters, sm_knn_build_from_reconstruction, sm_render_surfels, sm_track_frame, sm_track_linearize,
 * sm_triangulate, sm_surfel_count / sm_surfels_size) and
 * sm_regularize, which main.cc calls between frames (:1573-1579). In frame-graph mode the step a push
 * launches has also decided the merges of the next frame (k_merge runs in the step's front half), which
 * that frame's Integrate() applies in the next step. The device merge counter then already includes them, so
 * the push snapshots it first, and while the session is open the count queries report the snapshot:
 * sm_surfel_count and sm_dump_state's merge_count are those after Integrate(last_integrated_frame), as
 * in the reference (sm_export_vertices' non-NaN count == sm_surfel_count, main.cc:150).
 *
 * While a session is open, sm_integrate, sm_preprocess, sm_stream_run, sm_reset, sm_load_state,
 * sm_configure, sm_enable_timings, sm_timeline_enable and a second sm_session_begin return
 * SM_ERR_INVALID_ARGUMENT and leave the handle unchanged; so do sm_session_push / sm_session_end without
 * one. A push with bad arguments (NULL pointers, a pitch below the row size) returns
 * SM_ERR_INVALID_ARGUMENT without consuming the frame; the session stays open. A CUDA error drains the
 * device and closes the session. sm_destroy ends an open session first.
 *
 * sm_session_end fills `stats` as sm_stream_run does, for the whole session: frames_integrated,
 * surfels_size / surfel_count after it, the kernel launches since sm_session_begin, h2d_bytes = the
 * sensor-size depth and colour bytes of every host frame pushed (0 for device frames), d2h_bytes = the
 * counters fetched at the end, host_enqueue_ms = host time inside begin, the pushes and end. */
typedef struct sm_session_status {
  uint32_t frames_pushed;          /* since sm_session_begin */
  uint32_t frames_integrated;      /* since sm_session_begin */
  int64_t last_integrated_frame;   /* frame index of the newest integrated frame, -1 = none yet */
} sm_session_status;

int sm_session_begin(sm_reconstruction* r, void* stream, const sm_preprocess_params* pp,
                     const sm_integrate_params* ip, int32_t frame_width, int32_t frame_height,
                     uint32_t first_frame_index);
int sm_session_push(sm_reconstruction* r, const uint16_t* depth, size_t depth_pitch,
                    const uint8_t* color, size_t color_pitch, int32_t frame_on_host,
                    const float global_T_frame[12], const float frame_T_global[12],
                    sm_session_status* status /* may be NULL */);
int sm_session_end(sm_reconstruction* r, sm_stream_stats* stats /* may be NULL */);

/* Named tuning knobs of a handle (no counterpart in the reference). Keys:
 *   "tiebreak_wave" (slots per launch wave of the reference's association kernel; 0 = the plain rule "primary-pixel
 *   association before secondary, then lowest index"), "tiebreak_lanes" (consecutive slots that keep their order: a
 *   warp), "tiebreak_early_fraction" / "tiebreak_index_order_fraction" (first wave), "tiebreak_early_fraction_second"
 *   (second wave), "tiebreak_early_fraction_later" / "tiebreak_index_order_fraction_later" (later waves; negative =
 *   inherit), "tiebreak_wave_offset" (measurement hook): the reproducible rule that picks the supporting surfel of a
 *   pixel with several supporters, where the reference lets the first atomicCAS win
 *   (APP/cuda_surfel_reconstruction_kernels.cu:1688); DESIGN.md section 4 has the measurements behind the defaults.
 *   "median_filter_and_densify_iterations": sm_stream_run applies that many
 *   MedianFilterAndDensifyDepthMap passes (APP/main.cc:207-252, 927-939) to every raw depth map
 *   as it enters the device-side frame ring (default 0, as in the reference).
 *   "pyramid_level" (integer in [0, 4], default 0, APP/main.cc:299-303 --pyramid_level L): sm_stream_run
 *   reconstructs at 1 / 2^L of the sensor resolution. sm_stream_desc.width/height and the depth/colour frames
 *   are then the sensor's, width and height must be divisible by 2^L and (width >> L, height >> L) must be the
 *   handle's size (create the handle with the camera scaled by 1 / 2^L, libvis Camera::Scaled); every raw
 *   depth map and colour image is downscaled on the upload stream as sm_downscale_using_median_while_excluding
 *   and sm_color_image_pyramid do (host frames through full-size staging, device frames in place;
 *   stats.h2d_bytes counts the full-size uploads). Like the reference (main.cc:946-949) a level above 0
 *   cannot be combined with median_filter_and_densify_iterations > 0: sm_stream_run then returns
 *   SM_ERR_INVALID_ARGUMENT, whatever the order of the sm_configure calls. */
int sm_configure(sm_reconstruction* r, const char* key, double value);

/* Number of kernel launches issued by this library since load (all handles). */
uint64_t sm_kernel_launch_count(void);

/* Per-kernel device timing for the roofline report of bench.py: while enabled, every kernel
 * launch of the library is bracketed by CUDA events on its launching stream.
 * sm_profile_report synchronises the device and returns, per kernel id, the accumulated
 * elapsed milliseconds and the launch count since the last report. Never enabled inside a
 * timed throughput region (the extra events serialise the launches). */
int sm_profile_kernels(int32_t enable);
int32_t sm_profile_kernel_count(void);
const char* sm_profile_kernel_name(int32_t id);
int sm_profile_report(double* total_ms, uint64_t* launches, int32_t n);

/* Work counters of the last Integrate(): surfel slots swept (N), surfels that projected
 * into the image (V), sum of the supporting counts (S), new surfels (M). Synchronises. */
int sm_frame_counters(sm_reconstruction* r, void* stream, uint64_t out[4]);

/* Diagnostics: device timeline. After sm_timeline_enable(r, frames) every kernel of the frame
 * pipeline stamps the start of its first block and the end of its last warp (%globaltimer,
 * nanoseconds) into slot [frame_index % frames][kernel id]; this shows the pipeline as it runs on
 * the GPU (events and profilers serialise it). sm_timeline_read copies frames x
 * sm_profile_kernel_count() x {start, end} values (start = UINT64_MAX: not launched).
 * frames = 0 disables and frees the buffer. No counterpart in the reference. */
int sm_timeline_enable(sm_reconstruction* r, int32_t frames);
int sm_timeline_read(sm_reconstruction* r, uint64_t* out, int32_t frames);

#ifdef __cplusplus
}
#endif
#endif  /* SURFEL_B200_H_ */
