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
 * full transfer. Every sm_create, sm_reset and sm_load_state takes a fresh generation from one
 * process-wide counter, so a token filled from another handle, or from a destroyed one, also
 * gets the full transfer. Synchronises `stream`. */
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

/* ---- rendering the triangle mesh into any pinhole camera (DESIGN.md section 1 row f11, section 5.9) ----------
 * The reference's viewer draws its mesh over the visualisation vertex buffer with per-vertex colours, and keeps
 * drawing the surfels the mesh does not cover yet as splats (APP/surfel_meshing_render_window.cc:239-359,
 * --hide_new_surfel_splats off by default). sm_render_mesh draws a caller's triangle list over the handle's current
 * cloud without a display, into the deterministic z-buffer of sm_render_surfels: same params, camera convention,
 * output layouts and argument checks. triangles (DEVICE, 3 x triangle_count slot indices) may come from
 * sm_triangulate or sm_mesh_read(SM_MESH_ALL), or be any list: it may be stale against the cloud.
 *
 * n = surfels_size(). In fp32 with denormals flushed to zero and no contraction, every product, sum and quotient
 * rounded on its own (IEEE division and square root), for triangle t = (a, b, c):
 *  T1. Corners. t is drawn only if a, b and c are all < n and have radius^2 (row 7) > 0; a triangle naming a merged
 *      slot or a slot past the end is skipped (not an error). Its corners s_0 < s_1 < s_2 are a, b, c sorted by
 *      slot, so nothing below depends on the winding or the rotation of t. A corner's vertex is its current SMOOTH
 *      position, its colour the low three bytes (r, g, b) of row 24.
 *  T2. Camera. c_k = view_T_global * vertex_k as in rule 1 of sm_render_surfels. t is skipped unless every corner
 *      has near_depth <= c_k.z <= far_depth. There is no clipping: a triangle crossing the near plane is dropped.
 *  T3. Screen. (u_k, v_k) = (fx * (c_k.x / c_k.z) + cx, fy * (c_k.y / c_k.z) + cy): the pixel-corner convention,
 *      pixel (px, py) has its centre at (float(px) + 0.5, float(py) + 0.5). One function computes it, so a
 *      corner shared by several triangles has the same bits in each. With the edge function of corners j < k
 *        E_jk(x, y) = (u_k - u_j) * (y - v_j) - (v_k - v_j) * (x - u_j)
 *      (always evaluated from the lower slot), D = E_01(u_2, v_2) is twice the signed screen area; t is skipped
 *      if D == 0 or D is not finite.
 *  T4. Coverage. At a pixel centre (x, y): w_0 = E_12(x, y), w_1 = -E_02(x, y), w_2 = E_01(x, y) (w_k belongs to
 *      the edge opposite corner k; a triangle that runs an edge the other way negates its value, which is exact).
 *      The pixel is covered iff w_0, w_1, w_2 >= 0 (D > 0) or all <= 0 (D < 0): edges are inclusive and there is
 *      no back-face culling. Two triangles that share an edge compute its value alike, so no pixel centre between
 *      them is left uncovered; a centre on the shared edge is proposed by both, and the key decides.
 *  T5. Depth. q_k = (w_k / D) / c_k.z and z = 1 / ((q_0 + q_1) + q_2) (perspective-correct); the pixel is skipped
 *      unless z is finite and > 0. It proposes the key (bits(z) << 32) | t, and the smallest key wins.
 *  T6. Surfels the mesh leaves out (flags & SM_RENDER_UNMESHED_SURFELS, what the reference's viewer shows by
 *      default). A slot < n that is a corner of no T1-valid triangle of the list is drawn as a disk by rules 1-4
 *      of sm_render_surfels, with (bits(t) << 32) | (0x80000000 | slot) as its key: at equal depth a triangle
 *      beats a disk.
 *  T7. Outputs of the winning key. Triangle: depth = z, index = t, and with q_k and z of T5 at that pixel,
 *      colour channel ch = the u8 of (((q_0 * C_0 + q_1 * C_1) + q_2 * C_2) * z) + 0.5, truncated, 255 if that
 *      sum is >= 255 (C_k = float(channel ch of corner k)); normal = g * (1 / sqrt(g.g)) with e1 = c_1 - c_0,
 *      e2 = c_2 - c_0, g = (e1.y*e2.z - e1.z*e2.y, e1.z*e2.x - e1.x*e2.z, e1.x*e2.y - e1.y*e2.x) negated if
 *      g.c_0 > 0 (so it faces the camera), a.b = (a.x*b.x + a.y*b.y) + a.z*b.z, and (0, 0, 0) unless g.g is finite
 *      and > 0. Disk: depth, colour and normal as sm_render_surfels gives them, index = 0x80000000 | slot. Empty
 *      pixel: 0 / 0 / 0 / SM_INVALID_SURFEL_INDEX.
 * Each triangle tests the pixels of its screen rectangle (the bounds of its corners, rounded outwards by at least
 * one pixel); which pixels are covered is decided by T4 alone.
 *
 * Asynchronous on `stream`, no host synchronisation; surfels_size() is read on the device. Only reads the surfel
 * state and the triangles. Scratch: the key raster of sm_render_surfels, a list of large triangles grown to
 * triangle_count (4 bytes per triangle; growing it synchronises the device once) and one bit per slot of the
 * handle's capacity, allocated by the first call (sm_create allocates nothing for rendering) and freed by
 * sm_destroy. SM_ERR_INVALID_ARGUMENT, with no launch, for everything sm_render_surfels rejects, triangles NULL
 * with triangle_count > 0, triangle_count >= 2^31 and flag bits other than SM_RENDER_UNMESHED_SURFELS. A count of 0
 * is legal: with the flag it gives sm_render_surfels' image, the index with its high bit set. */
#define SM_RENDER_UNMESHED_SURFELS 1
int sm_render_mesh(sm_reconstruction* r, void* stream, const sm_render_params* p,
                   const float view_T_global[12],      /* 3x4 row-major, global -> camera */
                   const uint32_t* triangles /* device, 3 x triangle_count slot indices */, uint64_t triangle_count,
                   int32_t flags,
                   float* depth, size_t depth_pitch,
                   uint8_t* color, size_t color_pitch,
                   float* normal, size_t normal_pitch,
                   uint32_t* index, size_t index_pitch);

/* ---- rendering the textured triangle mesh (DESIGN.md section 5.17) ---------------------------------------------
 * sm_render_mesh with the colour of its triangles read from a texture atlas, such as the atlas and uv that
 * sm_mesh_texture makes for the same list: to look at a textured mesh from new cameras, compare it with held-out
 * frames or hand its images to something that consumes them. Same raster, rules T1-T7 and outputs; in the same
 * arithmetic (fp32, denormals flushed to zero, no contraction, each operation rounded on its own):
 *  T8. Textured colour, for a pixel whose winning key is a triangle t (every other output, and every disk or empty
 *      pixel, is what sm_render_mesh gives for the same arguments). With s_0 < s_1 < s_2 t's corners sorted by slot
 *      (T1), UV_k = (uv[6t + 2j], uv[6t + 2j + 1]) with j the list position of the corner whose slot is s_k, so
 *      rotating or re-winding t together with its uv leaves the image unchanged. With q_k and z of T5 at the pixel,
 *      U = ((q_0 * U_0 + q_1 * U_1) + q_2 * U_2) * z, and V alike. If U or V is not finite the pixel takes T7's
 *      colour. Otherwise U and V are clamped to [0, 1], x = U * float(W) - 0.5, y = V * float(H) - 0.5, x0 = floor(x),
 *      fx = x - x0, y0 = floor(y), fy = y - y0, and texel (i, j) is read with i clamped to [0, W - 1] and j to
 *      [0, H - 1]. Per channel, with V_ab the texel (x0 + a, y0 + b) as a float, sample = top + fy * (bot - top),
 *      top = V_00 + fx * (V_10 - V_00), bot = V_01 + fx * (V_11 - V_01) (X6's form), and the colour is the u8 of
 *      sample + 0.5, truncated, 255 if that is >= 255. The lookup is done in software: the 8-bit weights of hardware
 *      texture filtering cannot meet this rule.
 * atlas is a DEVICE buffer of packed u8x3 texels (r, g, b), W = atlas_width by H = atlas_height, atlas_pitch bytes
 * per row; uv (DEVICE, 6 x triangle_count floats) holds per triangle and per corner in list order the (u, v) of
 * sm_mesh_texture's uv output, v = 0 at row 0. Asynchronous on `stream`, no host synchronisation; only reads the
 * surfel state, the triangles, uv and the atlas; the same scratch and launches as sm_render_mesh.
 * SM_ERR_INVALID_ARGUMENT, with no launch, for everything sm_render_mesh rejects, color NULL, uv or atlas NULL with
 * triangle_count > 0, atlas_width or atlas_height outside [1, SM_TEXTURE_MAX_ATLAS_SIDE] with triangle_count > 0,
 * atlas_pitch below 3 x atlas_width, and an output that overlaps the atlas or uv. An empty list with a 0 x 0 atlas
 * is legal. */
int sm_render_mesh_textured(sm_reconstruction* r, void* stream, const sm_render_params* p,
                            const float view_T_global[12],      /* 3x4 row-major, global -> camera */
                            const uint32_t* triangles /* device, 3 x triangle_count */, uint64_t triangle_count,
                            int32_t flags,
                            const float* uv,          /* device, 6 x triangle_count: sm_mesh_texture's uv output */
                            const uint8_t* atlas, size_t atlas_pitch, int32_t atlas_width, int32_t atlas_height,
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

/* ---- camera tracking with colour (DESIGN.md section 1 row f12, section 5.10) ----------------------------------
 * Point-to-plane ICP cannot see motion that slides along the surfaces in view: a single plane fixes 3 of the 6
 * degrees of freedom, two planes or a corridor leave one translation free, and J^T J is then singular up to
 * rounding. sm_track_frame_rgbd tracks a depth map and its registered colour image by minimising
 *     E(T) = sum_icp r^2 + lambda^2 sum_photo r_c^2,
 * the residual r_c aligning the model's intensity to the live intensity through the live depth (as ElasticFusion's
 * joint ICP + RGB tracker and DVO do). Everything not written below is sm_track_frame: steps 1-5, rules L and M,
 * the solve, the loss rule (depth inliers against min_inlier_fraction of the valid pixels), the convergence test,
 * the pose bookkeeping and every argument check. Only reads the surfel state.
 *
 * Per-pixel rules, fp32 with every product, sum and quotient rounded on its own (no fma, IEEE division):
 *  P1. Intensity of a u8x3 pixel (r, g, b): I = ((0.299f * r) + (0.587f * g)) + (0.114f * b).
 *  P2. Live pyramid. Level 0 is P1 of the raw colour. Level l has the size w x h of Camera.scaled(l) and is built
 *      from level l-1 of size w' x h': with a = (2x, 2y), b = (min(2x+1, w'-1), 2y), c = (2x, min(2y+1, h'-1)),
 *      d = (min(2x+1, w'-1), min(2y+1, h'-1)), I_l(x, y) = ((I(a) + I(b)) + (I(c) + I(d))) * 0.25f.
 *      (2x <= w'-1 and 2y <= h'-1 hold for every size Camera.scaled produces.)
 *  P3. Model pyramid, at the model camera Camera.scaled(l) of the handle's camera. Level 0: P1 of the model colour
 *      where the model depth is finite and > 0, NaN elsewhere; levels >= 1 as in P2 (a NaN child makes its parent
 *      NaN). Model colour: SM_TRACK_CLOUD: the colour output of the sm_render_surfels call of step 2 (rendered
 *      together with depth and normal); SM_TRACK_PREVIOUS_FRAME: the level-0 live intensity kept by this handle's
 *      previous sm_track_frame_rgbd call, with that call's kept depth (step 3) as the model depth.
 *  P4. Photometric sample, only for a pixel that is a depth inlier (passes M1-M4), with p' = T p of M1 and the
 *      level-l model camera (fx_l, fy_l, cx_l, cy_l, size w_l x h_l):
 *        u = fx_l * (p'.x / p'.z) + cx_l, v likewise; s = u - 0.5, t = v - 0.5; a photometric outlier unless
 *        0 <= s < w_l - 1 and 0 <= t < h_l - 1 (the right-hand sides exact small integers);
 *        i = int(s), j = int(t), a = s - i, b = t - j; I00, I10, I01, I11 = model level l at (i, j), (i+1, j),
 *        (i, j+1), (i+1, j+1), all four finite or the pixel is a photometric outlier;
 *        Im = ((1-a)*I00 + a*I10) * (1-b) + ((1-a)*I01 + a*I11) * b;
 *        gx = (1-b)*(I10-I00) + b*(I11-I01), gy = (1-a)*(I01-I00) + a*(I11-I10)  (the analytic gradient of the
 *        bilinear patch, so the Jacobian is the exact derivative inside a cell);
 *        r_c = Im - I_live_l(x, y). A photometric inlier needs |r_c| <= max_intensity_residual and
 *        gx*gx + gy*gy >= g2, g2 = min_gradient * min_gradient rounded to fp32.
 *  P5. Jacobian for the increment of M5 (T <- exp(xi) T, xi = (omega, v)): ga = gx * fx_l, gb = gy * fy_l,
 *      iz = 1 / p'.z, w = (ga * iz, gb * iz, -(((ga * p'.x + gb * p'.y) * iz) * iz)), J_c = (p' x w, w) with the
 *      cross product of L2.
 *  P6. Sums. With L2 = double(lambda) * double(lambda), the 21 L2 * (J_ci * J_cj) and the 6 L2 * (J_ci * r_c) are
 *      formed in fp64 and added, after the pixel's depth terms, into the same per-thread sums as M5's; r_c^2 and the
 *      photometric inlier count are two more sums. The solve and everything after it are those of sm_track_frame.
 *  P7. photometric_weight == 0 runs sm_track_frame's own linearisation and solve: pose and result.depth are
 *      sm_track_frame's bit for bit. The call still renders the model colour, builds the pyramids and keeps the
 *      level-0 intensity, so a following SM_TRACK_PREVIOUS_FRAME call has its model.
 * result: depth exactly as sm_track_frame reports it; photometric_inliers and rms_intensity = sqrt(sum r_c^2 /
 * photometric_inliers) (0 without inliers) of the last level-0 linearisation (both 0 when the frame was lost
 * before level 0, and with photometric_weight == 0).
 *
 * sm_track_linearize_rgbd runs one linearisation on caller images, synchronously: sm_track_linearize's arguments,
 * plus rp, the raw live colour and the model colour (packed u8x3, both at the handle's camera size); it builds
 * levels 0..level of both pyramids from them (P2, P3 with model_depth as the model depth) and returns the 27
 * combined sums (P6), out_sum_rc2 = sum r_c^2, out_inliers = the depth inliers and out_photometric_inliers.
 *
 * Scratch (the render's colour image, both intensity pyramids in fp32 and one kept level-0 intensity) is allocated
 * by the first RGB-D call; sm_create allocates nothing for it and sm_destroy frees it. A depth-only sm_track_frame
 * between RGB-D calls keeps working as before; it leaves no kept intensity, so the next RGB-D call may not use
 * SM_TRACK_PREVIOUS_FRAME. SM_ERR_INVALID_ARGUMENT, with no launch, for everything sm_track_frame (or
 * sm_track_linearize) rejects, plus a NULL colour or rp, a colour pitch below 3 x width, a negative or non-finite
 * photometric_weight, max_intensity_residual or min_gradient, and SM_TRACK_PREVIOUS_FRAME when the handle's
 * previous sm_track_frame / sm_track_frame_rgbd call was not an RGB-D call. */
typedef struct sm_track_rgbd_params {
  float photometric_weight;        /* lambda, metres per intensity unit; 0 = the depth-only system (1e-4) */
  float max_intensity_residual;    /* |r_c| gate, intensity units on the 0..255 scale (40) */
  float min_gradient;              /* |grad I| gate, intensity units per pixel (2) */
} sm_track_rgbd_params;
typedef struct sm_track_rgbd_result {
  sm_track_result depth;           /* exactly as sm_track_frame reports it */
  uint32_t photometric_inliers;    /* level 0, last linearisation */
  float rms_intensity;             /* sqrt(sum r_c^2 / photometric_inliers), level 0, last linearisation */
} sm_track_rgbd_result;
/* Host only, no device needed. */
void sm_default_track_rgbd_params(sm_track_rgbd_params* p);
int sm_track_frame_rgbd(sm_reconstruction* r, void* stream, const sm_track_params* tp, const sm_preprocess_params* pp,
                        const sm_track_rgbd_params* rp,
                        const uint16_t* depth, size_t depth_pitch,   /* raw u16, device, the handle's camera size */
                        const uint8_t* color, size_t color_pitch,    /* packed u8x3 (r, g, b), registered to depth */
                        const float global_T_guess[12], float global_T_out[12], sm_track_rgbd_result* result);
int sm_track_linearize_rgbd(sm_reconstruction* r, void* stream, const sm_track_params* tp,
                            const sm_track_rgbd_params* rp, int32_t level, float depth_scaling,
                            const uint16_t* live_depth, size_t live_pitch,   /* filtered level image, device */
                            const uint8_t* live_color, size_t live_color_pitch,   /* raw u8x3, handle size */
                            const float* model_depth, size_t model_depth_pitch,
                            const float* model_normal, size_t model_normal_pitch,
                            const uint8_t* model_color, size_t model_color_pitch,   /* u8x3, handle size */
                            const float model_T_live[12], double out_system[27], double* out_sum_rc2,
                            uint32_t* out_inliers, uint32_t* out_photometric_inliers);

/* ---- relocalisation: a keyframe database of random-fern codes (DESIGN.md section 1 row f13, section 5.11) --------
 * A tracker that tracks against its own model has a small basin: a lost camera does not come back by itself. As in
 * ElasticFusion (Glocker et al., "Real-Time RGB-D Camera Relocalization via Randomized Ferns for Keyframe Encoding",
 * TVCG 2015), a frame is reduced to `ferns` 4-bit codes, keyframes are stored by code, a lost frame is matched to
 * its nearest keyframes by block Hamming distance and tracking is restarted from their poses. The database is an
 * object of its own (like sm_knn_index), bound to the device and the camera size of the handle it was created from;
 * it is created on the current device, which must be the handle's.
 * Every rule below is integer or fp64 arithmetic, so codes, distances and decisions are exact.
 *  F1. Fern image. L = level in [1, 4]; w = int(W / 2^L + 0.5), h = int(H / 2^L + 0.5) (Camera.scaled(L) of the
 *      handle's W x H camera). Depth D: the raw u16 depth downscaled to w x h by sm_downscale_using_median_while_excluding
 *      (0, ...). Colour: the input block of pixel (x, y) is [W x / w, W (x + 1) / w) x [H y / h, H (y + 1) / h) (integer
 *      division, the median's block); each channel is (S + n / 2) / n in integers, S the sum over the block's n pixels
 *      of the raw packed u8x3 colour. sm_keyframe_db_create rejects a level whose blocks exceed 16 x 16 pixels.
 *  F2. Fern tables, drawn once at creation by splitmix64 from `seed` (state += 0x9E3779B97F4A7C15; z = state;
 *      z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9; z = (z ^ (z >> 27)) * 0x94D049BB133111EB; next = z ^ (z >> 31)),
 *      for f = 0 .. ferns-1 in order, six draws per fern: x = (next >> 32) % w, y = (next >> 32) % h, then the
 *      thresholds t_R, t_G, t_B = next >> 56 each, then t_D = min_depth + (max_depth - min_depth) *
 *      ((next >> 11) * 2^-53) in fp64 (metres; min_depth and max_depth converted to double first). ferns is a multiple
 *      of 8 in [8, 2048].
 *  F3. Code. Nibble f: bit0 = R >= t_R, bit1 = G >= t_G, bit2 = B >= t_B, bit3 = (D > 0 and double(D) >= t_D *
 *      double(depth_scaling)), with (R, G, B, D) the fern image at (x_f, y_f). Fern f is the nibble at bits
 *      4 (f % 8) of 32-bit word f / 8; a code is ferns / 8 words.
 *  F4. Distance between two codes: the number of ferns whose nibbles differ (block Hamming distance).
 *  F5. Query: the distances to every stored keyframe; the keys (distance << 32 | index) in ascending order, the first
 *      `candidates` (at most 8) of them, without those with double(distance) > double(max_query_fraction) * ferns.
 *  F6. Add: the frame's code and its global_T_frame are appended as keyframe `count` when the database is empty, when
 *      force != 0, or when its smallest distance to a stored keyframe d satisfies double(d) > double(add_fraction) *
 *      ferns. A frame that would be appended to a database holding `capacity` keyframes is not, and `full` is set.
 *      Nothing is ever evicted.
 *  F7. Relocalise: the query (F5) with the call's params; then, for each candidate in order, sm_track_frame (or
 *      sm_track_frame_rgbd when rp != NULL) against the cloud (params.track with model_source = SM_TRACK_CLOUD)
 *      from the keyframe's pose, with the call's pp (and rp). The first candidate whose call reports tracked,
 *      double(inliers) >= double(accept_inlier_fraction) * double(valid_pixels) and rms_residual <= accept_rms is
 *      accepted: global_T_out is that call's pose bit for bit, result.relocalised = 1 and result.keyframe / rank /
 *      distance / track name the candidate and that call's result. Otherwise relocalised = 0, keyframe = rank = -1,
 *      global_T_out is NaN and result.track is the last attempt's (zero without attempts). attempts = the tracking
 *      calls made (0 for an empty database or no candidate within the query bound).
 *      The handle's "previous frame" (SM_TRACK_PREVIOUS_FRAME) afterwards is that of the last attempt, as for any
 *      tracking call: this frame, with the accepted pose when one was accepted, otherwise the pose the last attempt
 *      returned (its guess if it was lost). Without attempts it is left as it was. Only reads the surfel state.
 *
 * Kernels (one stream, a fixed launch count): a frame is encoded by the median downscale and k_reloc_encode; add and
 * query run k_reloc_distance (one warp per keyframe) and k_reloc_select (one block: the top candidates, and for add
 * the F6 decision and the append on the device), then one synchronisation. sm_relocalise adds one tracking call's
 * launches per attempt. sm_keyframe_db_create uploads the tables and allocates every buffer (codes for `capacity`
 * keyframes, the fern image, one code, the distances, the selection result); no later call allocates. Calls on one
 * database are serialised by the caller.
 *
 * sm_keyframe_db_encode writes the code (F3) of a frame to out_codes (device, ferns / 8 words), asynchronously on
 * `stream`. sm_keyframe_db_add (F6) and sm_keyframe_db_query (F5; out_index / out_distance hold `candidates`
 * entries, *found are filled) are synchronous. sm_keyframe_db_read copies keyframe `index`'s pose (host, 12 floats)
 * and / or code (host, ferns / 8 words); either may be NULL. sm_relocalise params: NULL uses the database's own;
 * otherwise its level, ferns, seed, min_depth, max_depth and capacity must equal the database's.
 * SM_ERR_INVALID_ARGUMENT, with no launch, for NULL pointers, a pitch below the row size, params outside their
 * ranges (below), depth_scaling not finite and > 0, a non-finite global_T_frame, an index >= count, and a database
 * created from a handle of another camera size or device than `r`. Everything is allowed while a stream session is
 * open on `r` (like sm_track_frame; the database reads no surfel state except through the tracking calls).
 * Ranges: level 1..4 with blocks <= 16 x 16, ferns % 8 == 0 in [8, 2048], 0 <= min_depth < max_depth finite,
 * capacity in [1, 2^20], add_fraction and max_query_fraction finite in [0, 1], candidates 1..8,
 * accept_inlier_fraction finite in [0, 1], accept_rms finite and >= 0, track as sm_track_frame checks it. */
#define SM_RELOC_MAX_CANDIDATES 8
typedef struct sm_reloc_params {
  int32_t level;                   /* fern image level, 1..4 (3) */
  int32_t ferns;                   /* multiple of 8 in [8, 2048] (512) */
  uint64_t seed;                   /* splitmix64 seed of the fern tables (20150401) */
  float min_depth, max_depth;      /* metres, range of the depth thresholds (0.3, 4.0) */
  uint32_t capacity;               /* keyframes (4096) */
  float add_fraction;              /* F6 (0.2) */
  int32_t candidates;              /* F5, 1..8 (1) */
  float max_query_fraction;        /* F5 (0.4) */
  sm_track_params track;           /* F7: the tracking calls (sm_default_track_params, max_point_distance 0.1) */
  float accept_inlier_fraction;    /* F7 (0.7) */
  float accept_rms;                /* metres, F7 (0.01) */
} sm_reloc_params;
typedef struct sm_reloc_result {
  int32_t relocalised;             /* 1 = global_T_out is the accepted pose; 0 = NaN */
  int32_t attempts;                /* tracking calls made */
  int32_t keyframe;                /* accepted keyframe, -1 */
  int32_t rank;                    /* its rank among the candidates, -1 */
  uint32_t distance;               /* its distance (F4), 0 */
  sm_track_result track;           /* the accepted call's; the last attempt's when none was accepted */
} sm_reloc_result;
typedef struct sm_keyframe_db sm_keyframe_db;
/* Host only, no device needed. */
void sm_default_reloc_params(sm_reloc_params* p);
int sm_keyframe_db_create(sm_keyframe_db** out, sm_reconstruction* r, const sm_reloc_params* params);
void sm_keyframe_db_destroy(sm_keyframe_db* db);
int sm_keyframe_db_reset(sm_keyframe_db* db);
int sm_keyframe_db_count(sm_keyframe_db* db, uint32_t* out);
int sm_keyframe_db_encode(sm_keyframe_db* db, void* stream, const uint16_t* depth, size_t depth_pitch,
                          const uint8_t* color, size_t color_pitch, float depth_scaling, uint32_t* out_codes);
int sm_keyframe_db_add(sm_keyframe_db* db, void* stream, const uint16_t* depth, size_t depth_pitch,
                       const uint8_t* color, size_t color_pitch, float depth_scaling, const float global_T_frame[12],
                       int32_t force, int32_t* out_index /* -1: not appended */, int32_t* out_full);
int sm_keyframe_db_query(sm_keyframe_db* db, void* stream, const uint16_t* depth, size_t depth_pitch,
                         const uint8_t* color, size_t color_pitch, float depth_scaling, int32_t* out_index,
                         uint32_t* out_distance, int32_t* out_found);
int sm_keyframe_db_read(sm_keyframe_db* db, uint32_t index, float pose[12] /* may be NULL */,
                        uint32_t* codes /* may be NULL */);
int sm_relocalise(sm_reconstruction* r, sm_keyframe_db* db, void* stream, const sm_reloc_params* params,
                  const sm_preprocess_params* pp, const sm_track_rgbd_params* rp /* NULL: depth only */,
                  const uint16_t* depth, size_t depth_pitch, const uint8_t* color, size_t color_pitch,
                  float global_T_out[12], sm_reloc_result* result);

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

/* ---- keeping the mesh up to date (DESIGN.md section 1 row f10, section 5.8) ----------------------------------
 * The reference's meshing thread remeshes only the surfels that changed (APP/surfel_meshing.cc:189-288).
 * sm_mesh_update keeps a persistent mesh in the handle and brings it up to date with the current cloud, rebuilding
 * only the umbrellas a change can reach. Afterwards:
 *  1. Full mesh. sm_mesh_read(SM_MESH_ALL) gives exactly what sm_triangulate with the same params returns on this
 *     state (triangles, their order, and stats->mesh == its four stats), after any sequence of calls between
 *     updates (sm_integrate, sm_regularize, session pushes, sm_stream_run, sm_load_state, sm_reset).
 *  2. Delta. As sets of ordered triples (o, x, y): removed = previous mesh - new mesh, added = new - previous,
 *     where the previous mesh is that of this handle's last completed update (empty before the first one, and
 *     after an update that failed). Each list is ordered by owner slot, then by that owner's umbrella order (the
 *     old umbrella for removed, the new one for added).
 *  3. Read-only: only reads the surfel state (apart from the smooth-position mirror into rows 3-5 that
 *     sm_triangulate also writes).
 *  4. Independent of sm_triangulate, which has buffers of its own (both rebuild the one k-NN index object).
 * What is recomputed, step by step (n = surfels_size(), n_prev = surfels_size() at the previous update; a slot's
 * inputs are the bits of its smooth x y z, radius^2 and normal x y z, kept as a snapshot of 28 bytes per slot):
 *  a. C (changed): the slots that are or were present and whose inputs differ from the snapshot; every present
 *     slot of [n_prev, n) is in C. C does not depend on what caused the change.
 *  b. A (umbrellas rebuilt): C, plus every present slot i whose ball holds the old position (of a slot present
 *     then) or the new position (of a slot present now) of some slot of C, by rule 1's own fp32 test
 *     ((dx*dx + dy*dy) + dz*dz) <= r_i^2 * f2. A slot outside A has the same ball with the same slots inside it,
 *     so the same umbrella.
 *  c. R (owners rechecked): A, plus every slot whose umbrella names a slot of A in either place of a pair. A slot
 *     outside R owns the same triangles and has the same share of the stats (meshed, boundary edges of its
 *     triangles, overflow), all of which read only its umbrella, the umbrellas it names and their inputs.
 *  d. Everything: every slot is in A and in R when the params differ from the previous update's, when n < n_prev
 *     (after sm_reset), before the first update, after a failed one, and when C holds more than 1/16 of the slots
 *     (marking A would then cost more than it saves). Slots of [n, n_prev) then own nothing.
 *  e. The umbrellas of A are rebuilt from a list of A, or by a sweep over all slots when A holds more than three
 *     quarters of them (stats->full_sweep); both give the same umbrellas. The stats are kept as sums of per-slot
 *     shares.
 * stats: mesh = the whole mesh after the update; slots_changed = |C|, umbrellas_rebuilt = |A| (n when everything
 * is rebuilt), owners_rechecked = |R|, triangles_added / triangles_removed = the lengths of the two lists.
 * The call synchronises `stream` three times (surfels_size(), the largest radius and |C|, the mesh and delta
 * sizes), plus once, with cudaFree's device synchronisations, in a call whose buffers grow (by x 1.5). Memory (allocated by the first update, grown with surfels_size() and the mesh, freed by sm_destroy;
 * sm_create allocates nothing for meshing): 173 bytes per slot kept between updates (snapshot 28, umbrella
 * SM_MESH_MAX_UMBRELLA x 8 + 4, 5 bytes of per-slot stats, 8 of offsets), 46 bytes per slot of scratch, 24 bytes per
 * triangle (the previous and the current mesh), 12 per added or removed triangle, and an index over the changed
 * positions. SM_ERR_INVALID_ARGUMENT, with no launch, for NULL arguments and for params sm_triangulate rejects.
 *
 * sm_mesh_read copies one of the lists of the last completed update into `triangles` (DEVICE, 3 x capacity
 * uint32; may be NULL with capacity 0: a count query) with work enqueued on `stream`, and sets *count. If capacity
 * < *count it returns SM_ERR_CAPACITY and writes nothing; SM_ERR_INVALID_ARGUMENT for an unknown `which`, NULL
 * count, or when no update has completed on this handle. */
typedef struct sm_mesh_update_stats {
  sm_mesh_stats mesh;            /* the whole mesh after the update (== sm_triangulate's stats) */
  uint64_t slots_changed;        /* |C| */
  uint64_t umbrellas_rebuilt;    /* |A| */
  uint64_t owners_rechecked;     /* |R| */
  uint64_t triangles_added, triangles_removed;
  int32_t full_sweep;            /* 1 when the umbrellas were rebuilt by the plain sweep */
  int32_t reserved;
} sm_mesh_update_stats;
int sm_mesh_update(sm_reconstruction* r, void* stream, const sm_mesh_params* p, sm_mesh_update_stats* stats);
#define SM_MESH_ALL 0
#define SM_MESH_ADDED 1
#define SM_MESH_REMOVED 2
int sm_mesh_read(sm_reconstruction* r, void* stream, int32_t which, uint32_t* triangles /* device, 3 x capacity */,
                 uint64_t capacity, uint64_t* count);

/* ---- closing the small holes of a triangle mesh (DESIGN.md section 1 row f14, section 5.12) -------------------
 * sm_triangulate and sm_mesh_update output a triangle only when the umbrellas of its three corners agree on it;
 * where neighbouring tangent planes disagree (usually about the diagonal of a quad) they leave a hole. The
 * reference's front-advancing mesher closes such holes as it goes (APP/surfel_meshing.cc:368-393, 1870-1944).
 * sm_mesh_fill_holes closes the small ones afterwards: it takes an edge-manifold, consistently oriented triangle
 * list over the handle's slots (the output of either call, or any list a caller builds) and returns the triangles
 * that fill its closable boundary loops. It writes only the new triangles; the caller appends them to its list.
 * Positions are read from the rows 3-5 mirror of the smooth positions, which the call refreshes as sm_triangulate
 * does; nothing else of the surfel state is written.
 *
 * p_i, n_i (rows 8-10 normalised), the fp32 conventions and rule 2's tangent basis are those of sm_triangulate;
 * cos_n and cos_t come from the two angles of sm_hole_params the same way. An edge is an ordered pair (a, b) of
 * slots; the triangle (o, x, y) has the edges (o, x), (x, y) and (y, o). K = max_hole_edges.
 *  H1. Hole edges. For each input edge (a, b) whose reverse (b, a) is not an input edge, (b, a) is a hole edge: the
 *      hole lies on its left, and a fill triangle contains it in that direction. Hole edges are ordered by
 *      (tail, head).
 *  H2. Successor. The successor of hole edge (u, v) is the hole edge leaving v if there is exactly one, none if
 *      there is none. With several (v is a pinch vertex): q_x = ((p_x - p_v).t, (p_x - p_v).s) in v's tangent basis
 *      (t, s) of rule 2, and each candidate (v, w) has the half h_w = 0 if cross(q_u, q_w) < 0, h_w = 1 if
 *      cross(q_u, q_w) > 0 or (cross(q_u, q_w) == 0 and q_u.q_w < 0), no half otherwise (a NaN cross product
 *      included). w comes before w' iff
 *      h_w < h_w', or h_w == h_w' and cross(q_w, q_w') < 0: the order is clockwise from q_u, the side on which the
 *      hole of (u, v) lies at v. The successor is the candidate that comes before every other one; there is none
 *      if n_v is not a unit normal, if a candidate has no half, or if no candidate comes before all the others
 *      (collinear candidates).
 *  H3. Loops. Following successors from a hole edge, if it comes back to that edge after k <= K edges whose k tails
 *      are distinct, those k edges form a loop (so every hole edge is in at most one loop). The owner of the loop
 *      is its smallest edge; L[0..k-1] are the tails of its edges in order, from the owner's tail.
 *      (L[i], L[i+1 mod k]) are its loop edges.
 *  H4. Validity. The triangle (L[i], L[j], L[m]), i < j < m, is valid iff: every edge of it that is not a loop edge
 *      is an input edge in neither direction; all three corners have unit normals with n_a.n_b >= cos_n for each
 *      pair; in the rotation (o, x, y) that starts at the smallest slot, rule 4's geometric normal g has g.n_c > 0
 *      at each corner c; and rule 4's angle test with cos_t holds at each corner. Its weight is w = sqrt(g.g).
 *  H5. Triangulation (minimum area). W(i, i+1) = 0; for m - i >= 2, W(i, m) = the minimum over i < j < m of
 *      ((W(i, j) + W(j, m)) + w(i, j, m)), an invalid triangle counting as +inf, and j*(i, m) = the smallest j that
 *      reaches it. The loop is rejected if W(0, k-1) is +inf; otherwise its triangles are (L[i], L[j*], L[m]) for
 *      the nodes (i, m) of the tree that starts at (0, k-1), where node (i, m) with m - i >= 2 has the children
 *      (i, j*) and (j*, m). Its diagonals are the unordered pairs {L[i], L[m]} of the nodes other than (0, k-1)
 *      with m - i >= 2.
 *  H6. Conflicts. A loop that is not rejected and shares a diagonal with another such loop is dropped, and so is
 *      that other loop (one symmetric round: loops_conflicting). The other loops are filled.
 *  H7. Output. The filled loops by owner edge, ascending; the triangles of a loop in the tree's pre-order (node
 *      (i, m), then the subtree of (i, j*), then that of (j*, m)); each triangle written in the rotation that
 *      starts at its smallest slot. Input and output together are edge-manifold and consistently oriented.
 * stats: boundary_edges = hole edges of the input; loops_found = loops of H3; loops_rejected, loops_conflicting,
 * loops_filled (the three add up to loops_found); triangles_added (set also when the capacity is too small);
 * boundary_edges_after = the boundary edges of input and fill together = boundary_edges minus the lengths of the
 * filled loops. All zero when the call fails for any other reason.
 *
 * fill is a DEVICE buffer of 3 x capacity uint32 (may be NULL with capacity 0: a count query); if capacity <
 * triangles_added the call returns SM_ERR_CAPACITY with the stats set and writes nothing. SM_ERR_INVALID_ARGUMENT,
 * with no launch, for NULL params or stats, triangles NULL with count > 0, fill NULL with capacity > 0, count >=
 * 2^28, max_hole_edges outside [3, SM_MESH_MAX_HOLE] or an angle outside (0, 180]; and, found on the device and
 * reported after the call's second synchronisation with nothing written, for a corner >= surfels_size() or whose
 * slot is not present (radius^2 > 0), a triangle with a repeated corner, or a directed edge that occurs twice.
 * The call synchronises `stream` three times (surfels_size(); the hole edge count and the input checks; the
 * triangle count), plus once, with cudaFree's device synchronisation, in a call whose buffers grow (by x 1.5); on
 * return the fill is written by work enqueued on `stream`. Memory (allocated by the first call, grown with the
 * input, freed by sm_destroy; sm_create allocates nothing for it): 72 to 120 bytes per triangle of capacity (a
 * directed-edge hash table, of which a call uses and clears the power of two >= 6 x count, and the unsorted hole
 * edges) and about 150 to 180 bytes per
 * hole edge of capacity (the sorted edges and the sort's scratch, the loop and its triangles, the count, the
 * diagonal table). */
#define SM_MESH_MAX_HOLE 16
typedef struct sm_hole_params {
  int32_t max_hole_edges;                /* 8; in [3, SM_MESH_MAX_HOLE] */
  float max_angle_between_normals_deg;   /* 90, as sm_mesh_params */
  float max_triangle_angle_deg;          /* 180 = no angle filter (the reference closes holes with pi,
                                            APP/surfel_meshing.cc:1874) */
} sm_hole_params;
typedef struct sm_hole_stats {
  uint64_t boundary_edges;         /* of the input mesh */
  uint64_t loops_found;            /* closed hole loops of <= max_hole_edges edges */
  uint64_t loops_filled;
  uint64_t loops_rejected;         /* no valid triangulation */
  uint64_t loops_conflicting;      /* a diagonal proposed by another loop too */
  uint64_t triangles_added;        /* always set, also when the capacity was too small */
  uint64_t boundary_edges_after;
} sm_hole_stats;
/* Host only, no device needed. */
void sm_default_hole_params(sm_hole_params* p);
int sm_mesh_fill_holes(sm_reconstruction* r, void* stream, const sm_hole_params* p,
                       const uint32_t* triangles /* device, 3 x count */, uint64_t count,
                       uint32_t* fill /* device, 3 x capacity; may be NULL with capacity 0 */, uint64_t capacity,
                       sm_hole_stats* stats);

/* ---- simplifying a triangle mesh (DESIGN.md section 1 row f16, section 5.14) ----------------------------------
 * The mesh of sm_triangulate has one vertex per meshed surfel, so flat walls and table tops are described by
 * thousands of triangles. sm_mesh_simplify removes vertices by half-edge collapses ranked by Garland-Heckbert plane
 * quadrics: a slot u is removed and its triangles are given to a neighbour v; no vertex moves, so every corner of the
 * output is still a slot of the handle (sm_render_mesh, sm_mesh_fill_holes, sm_compact's remap and the OBJ export
 * take it as they take the full mesh). It takes an edge-manifold, consistently oriented triangle list over the
 * handle's slots (as sm_mesh_fill_holes does) and returns a list over a subset of its slots. The collapses run in
 * rounds of collapses with disjoint closed neighbourhoods, so the result does not depend on thread order.
 * Positions are read from the rows 3-5 mirror of the smooth positions, which the call refreshes as sm_triangulate
 * does; nothing else of the surfel state, and not the persistent mesh of sm_mesh_update, is written.
 *
 * p_i, n_i (rows 8-10 normalised, "unit normal"), the fp32 conventions and rule 4 are those of sm_triangulate; cos_n
 * and cos_t come from the two angles of sm_simplify_params the same way. P_i = p_i converted to double. Quadric
 * arithmetic is IEEE double with every product, sum, quotient and square root rounded on its own, in the order
 * written: (a + b) + c means a + b first. Input triangle t = (a, b, c) keeps its input position t throughout.
 *  S1. Quadrics. e1 = P_b - P_a, e2 = P_c - P_a, g = (e1.y*e2.z - e1.z*e2.y, e1.z*e2.x - e1.x*e2.z,
 *      e1.x*e2.y - e1.y*e2.x), gg = (g.x*g.x + g.y*g.y) + g.z*g.z. If gg > 0: s = sqrt(gg), m = (g.x/s, g.y/s,
 *      g.z/s), d = -((m.x*P_a.x + m.y*P_a.y) + m.z*P_a.z), and K_t has the ten entries (k0..k9) = (m.x*m.x,
 *      m.x*m.y, m.x*m.z, m.x*d, m.y*m.y, m.y*m.z, m.y*d, m.z*m.z, m.z*d, d*d); otherwise K_t = 0. Q_i = ((0 + K_t1)
 *      + K_t2) + ..., entry by entry, over the input triangles t1 < t2 < ... that have corner i. The cost of
 *      quadric q at x = (x, y, z): r0 = ((q0*x + q1*y) + q2*z) + q3, r1 = ((q1*x + q4*y) + q5*z) + q6,
 *      r2 = ((q2*x + q5*y) + q7*z) + q8, r3 = ((q3*x + q6*y) + q8*z) + q9, E = ((r0*x + r1*y) + r2*z) + r3: the sum
 *      of squared distances (m^2) to the planes of the triangles q gathers.
 *  S2. Round state: the current list (each triangle with its input position). N(i) = the distinct slots that share
 *      a current triangle with i, deg(i) = |N(i)|. An edge of i is present in only one direction: i is a boundary
 *      vertex. No boundary vertex is ever removed, and no boundary edge changes.
 *  S3. Candidates. u is a candidate iff it is not a boundary vertex, its current triangles form one closed fan
 *      (following (u, a, b) -> the triangle (u, b, c) visits all of them before it comes back), and 3 <= deg(u) <=
 *      SM_MESH_MAX_VALENCE. Its ring r_0..r_{d-1} (d = deg(u)) is the fan order from the triangle of smallest input
 *      position, (u, r_j, r_{j+1 mod d}) being its triangles. A collapse u -> v = r_k, with o1 = r_{k-1 mod d} and
 *      o2 = r_{k+1 mod d} (the opposite corners of the two triangles on {u, v}), is valid iff:
 *      (a) link condition: N(u) and N(v) share exactly o1 and o2;
 *      (b) deg(u) + deg(v) - 4 <= SM_MESH_MAX_VALENCE;
 *      (c) every triangle (u, r_j, r_{j+1}) without v, with u replaced by v and the winding kept, passes H4's
 *          geometric tests (unit normals at its three corners, n_a.n_b >= cos_n for each pair, g.n_c > 0 at each
 *          corner for rule 4's g in the rotation that starts at its smallest slot, and rule 4's angle test with
 *          cos_t at each corner), and does not have the three slots of a current triangle (which stops a
 *          tetrahedron from collapsing further);
 *      (d) E = the cost of (Q_u + Q_v) (entry by entry) at P_v is finite and cost = (E > 0 ? E : +0) <= max_cost.
 *      best(u) = the valid v with the smallest (cost, v); key(u) = bits(f) << 32 | u, where f = float(cost)
 *      (round to nearest), taken as +0 when it is below the smallest normal float.
 *  S4. Independent selection. Every candidate with a best(u) takes the minimum of its key into mark[y] for each y of
 *      N[u] = {u} + N(u); u is selected iff mark[y] == key(u) for every y of N[u]. Two selected slots have
 *      disjoint closed neighbourhoods, so no selected collapse changes the validity, the cost or the result of
 *      another, and a round equals its collapses applied one after the other in any order.
 *  S5. Budget. With target_triangles > 0 and T - 2 s < target_triangles (T current triangles, s selected), only
 *      the ceil((T - target_triangles) / 2) selected slots of smallest key are collapsed, and the call stops. Every
 *      collapse removes exactly two triangles ({u, v} is an interior edge).
 *  S6. Apply u -> v: the two triangles on {u, v} are deleted, u is replaced by v in every other triangle of u, and
 *      Q_v = Q_v + Q_u entry by entry.
 *  S7. Rounds. Before each round: stop (SM_SIMPLIFY_STOP_TARGET) if target_triangles > 0 and T <= target_triangles;
 *      else stop (SM_SIMPLIFY_STOP_MAX_ROUNDS) if max_rounds rounds have been applied; else select (S3, S4), and
 *      stop (SM_SIMPLIFY_STOP_CONVERGED) if nothing is selected, else apply (S5, S6): one more round.
 *  S8. Output. Every current triangle rotated to start at its smallest slot, the winding kept; ordered by that slot,
 *      then by input position. The output is edge-manifold and consistently oriented, V - E + F, the boundary edges
 *      and the boundary loops are those of the input, and a triangle that changed is counter-clockwise about the
 *      normals of its three corners.
 * stats: triangles_in = count; triangles_out (set also when the capacity is too small); vertices_in / vertices_out
 * = the slots that are corners of the input / output; collapses; rounds (rounds applied); boundary_edges = directed
 * edges of the input whose reverse is not one (those of the output too); max_cost_applied = the largest cost of an
 * applied collapse (0 without one); stop_reason. All zero when the call fails for any other reason.
 *
 * out is a DEVICE buffer of 3 x capacity uint32 (may be NULL with capacity 0: a count query); triangles_out <=
 * count, so capacity = count always suffices; if capacity < triangles_out the call returns SM_ERR_CAPACITY with the
 * stats set and writes nothing. SM_ERR_INVALID_ARGUMENT, with no launch, for NULL params or stats, triangles NULL
 * with count > 0, out NULL with capacity > 0, out overlapping triangles (both as 3 x uint32 arrays of count and
 * capacity triangles), count >= 2^28, max_cost negative or NaN, an angle outside (0, 180] or max_rounds outside
 * [0, SM_SIMPLIFY_MAX_ROUNDS]; and, found on the device and reported after the call's second synchronisation with
 * nothing written, for the inputs sm_mesh_fill_holes refuses (a corner that is not a present slot below
 * surfels_size(), a repeated corner, a directed edge that occurs twice). The call synchronises `stream` on
 * surfels_size(), after the input checks, once per round (selected and triangle counts), and at the end, plus once,
 * with cudaFree's device synchronisation, in a call whose buffers grow (by x 1.5); on return the output is written
 * by work enqueued on `stream`. Memory (allocated by the first call, grown with the input and surfels_size(), freed
 * by sm_destroy; sm_create allocates nothing for it): 120 to 168 bytes per triangle of capacity (a directed-edge
 * hash table of which a call uses and clears the power of two >= 6 x count: 48 to 96; the working list: 12; the
 * corner keys unsorted and sorted: 48; the scan counts: 12), the radix sort's scratch (about 24 more per triangle)
 * and 136 bytes per slot (the quadric: 80; the fan range, the mark, the key, the best neighbour and its cost, the
 * slot list and the selected keys sorted and unsorted: 56). */
#define SM_MESH_MAX_VALENCE 32
#define SM_SIMPLIFY_MAX_ROUNDS 1024
#define SM_SIMPLIFY_STOP_TARGET 1      /* the triangle count reached target_triangles */
#define SM_SIMPLIFY_STOP_CONVERGED 2   /* no collapse was selected */
#define SM_SIMPLIFY_STOP_MAX_ROUNDS 3  /* max_rounds rounds were applied */
typedef struct sm_simplify_params {
  uint64_t target_triangles;             /* 0 = no count bound */
  double max_cost;                       /* 1e-6 m^2; >= 0 (+inf: no cost bound) */
  float max_angle_between_normals_deg;   /* 90, as sm_mesh_params */
  float max_triangle_angle_deg;          /* 170, as sm_mesh_params */
  int32_t max_rounds;                    /* 64; in [0, SM_SIMPLIFY_MAX_ROUNDS]; 0 = check and reorder only */
  int32_t reserved;                      /* 0 */
} sm_simplify_params;
typedef struct sm_simplify_stats {
  uint64_t triangles_in;
  uint64_t triangles_out;          /* always set, also when the capacity was too small */
  uint64_t vertices_in, vertices_out;
  uint64_t collapses;
  uint64_t rounds;
  uint64_t boundary_edges;         /* of the input, and of the output */
  double max_cost_applied;         /* m^2 */
  int32_t stop_reason;             /* SM_SIMPLIFY_STOP_* */
  int32_t reserved;
} sm_simplify_stats;
/* Host only, no device needed. */
void sm_default_simplify_params(sm_simplify_params* p);
int sm_mesh_simplify(sm_reconstruction* r, void* stream, const sm_simplify_params* p,
                     const uint32_t* triangles /* device, 3 x count */, uint64_t count,
                     uint32_t* out /* device, 3 x capacity; may be NULL with capacity 0 */, uint64_t capacity,
                     sm_simplify_stats* stats);

/* ---- texturing a triangle mesh from posed colour images (DESIGN.md section 1 row f17, section 5.15) ------------
 * The mesh calls carry one colour per vertex (row 24 of the corner's slot), so a simplified mesh loses the colour
 * detail between its vertices. sm_mesh_texture gives every triangle of a caller's list a patch of a texture atlas
 * and fills each texel from the colour images of caller-chosen views that see it: the visibility-weighted mean of
 * their bilinear samples, the corner colours where no view sees the texel. Any list of triangles over present slots
 * is accepted (manifoldness is not required), e.g. the output of sm_triangulate, sm_mesh_fill_holes or
 * sm_mesh_simplify. Positions are the current SMOOTH positions (what sm_render_mesh draws); the call only reads the
 * surfel state.
 *
 * fp32 with denormals flushed to zero and no contraction, every product, sum, quotient and square root rounded on
 * its own (IEEE), in the order written: (a + b) + c means a + b first; |d|^2 = (d.x*d.x + d.y*d.y) + d.z*d.z. p_i is
 * the smooth position of slot i; t is a triangle's position in the list; its corners k = 0, 1, 2 in list order.
 *  X1. Input. Every corner must be a present slot (radius^2 > 0) below surfels_size() and no triangle may repeat a
 *      corner. 0 triangles are legal.
 *  X2. Tile class. e_k = |p_(k+2) - p_(k+1)|^2 (indices mod 3) is the squared length of the edge opposite corner k;
 *      a = the first k with the largest e_k (in the order 0, 1, 2; a NaN is never larger), b = a + 1, c = a + 2
 *      (mod 3): the rotation of t that starts at a, winding kept. L = sqrt(max(e_c, e_b)) (the legs ab and ac). The
 *      tile side s is the smallest of 8, 16, ..., SM_TEXTURE_MAX_TILE with L <= float(s - 4) * texel_size; if none
 *      is, s = SM_TEXTURE_MAX_TILE and the triangle counts in tiles_clamped.
 *  X3. Layout. The triangles sorted by (s descending, t ascending); within one s, the 2j-th and (2j+1)-th share the
 *      j-th s x s square of that s, as its half 0 and half 1. The squares in that order (larger s first, then j) get
 *      running area offsets o (the sum of s^2 of the squares before); a square's origin (x0, y0) in texels is the
 *      Morton (Z-order) decode of o (x from the even bits, y from the odd ones). Every earlier square is at least as
 *      large, so o is a multiple of s^2 and the square is the aligned block of codes [o, o + s^2): squares never
 *      overlap. The atlas width W is the smallest power of two with W * W >= the total area, its height H the
 *      largest y0 + s (0 x 0 for an empty list).
 *  X4. UV. Texel (i, j) of a square is the atlas texel (x0 + i, y0 + j), its centre at (i + 0.5, j + 0.5) in square
 *      coordinates. Half 0 is the texels with i + j <= s - 1 and its triangle's (a, b, c) sit at (1, 1), (s - 3, 1),
 *      (1, s - 3); half 1 is those with i + j >= s, its (a, b, c) at (s - 1, s - 1), (3, s - 1), (s - 1, 3). A bilinear
 *      lookup (texel centres at integer + 0.5) at any point of a UV triangle reads only texels of its own half. The
 *      uv output holds, per triangle in list order and per corner in list order, (float(x0 + X) / float(W),
 *      float(y0 + Y) / float(H)) for the corner's (X, Y) above.
 *  X5. Texel point. For texel (i, j) of a half: x = float(i) + 0.5, y = float(j) + 0.5, q = float(s - 4); half 0:
 *      alpha = (x - 1) / q, beta = (y - 1) / q; half 1: alpha = (float(s - 1) - x) / q, beta = (float(s - 1) - y) / q.
 *      Clamp to the triangle: alpha = max(alpha, 0), beta = max(beta, 0), and if alpha + beta > 1: alpha =
 *      alpha / (alpha + beta), beta = 1 - alpha. X = (p_a + alpha * (p_b - p_a)) + beta * (p_c - p_a), per
 *      component. The geometric normal: e1 = p_b - p_a, e2 = p_c - p_a, g = (e1.y*e2.z - e1.z*e2.y,
 *      e1.z*e2.x - e1.x*e2.z, e1.x*e2.y - e1.y*e2.x), n = g * (1 / sqrt(|g|^2)); a triangle whose |g|^2 is not finite
 *      and > 0 has no normal and no view contributes to it.
 *  X6. One view's sample, views in array order. c = view_T_global * X and m = R(view_T_global) * n as in rule 1 of
 *      sm_render_surfels. The view contributes nothing unless near_depth <= c.z <= far_depth; with (u, v) = (fx *
 *      (c.x / c.z) + cx, fy * (c.y / c.z) + cy) (T3 of sm_render_mesh), px = u - 0.5, py = v - 0.5: unless 0 <= px <
 *      float(width - 1) and 0 <= py < float(height - 1) (the 2 x 2 bilinear footprint lies in the image); unless
 *      D > 0 and |D - c.z| <= depth_tolerance * c.z, D the depth that sm_render_mesh draws for the same triangle list
 *      and camera, without disks, at pixel (int(u), int(v)); unless cos_theta = -((m.x*c.x + m.y*c.y) + m.z*c.z) /
 *      sqrt(|c|^2) >= float(cos(max_view_angle_deg)) (computed in double). Then w = cos_theta / (c.z * c.z) and, with
 *      x0 = floor(px), fx = px - x0, y0 = floor(py), fy = py - y0 and V_xy the channel at pixel (x0 + x, y0 + y) as a
 *      float, the sample of a channel is top + fy * (bot - top), top = V_00 + fx * (V_10 - V_00), bot = V_01 + fx *
 *      (V_11 - V_01). Per texel S_ch = S_ch + w * sample_ch and S_w = S_w + w, from 0.
 *  X7. Resolve. If S_w > 0, channel ch = the u8 of S_ch / S_w + 0.5, truncated, 255 if it is >= 255. Otherwise
 *      (texels_fallback) the corner blend: with C_k = float(channel ch of row 24 of slot k), ((1 - alpha) - beta) * C_a
 *      + alpha * C_b, then + beta * C_c, + 0.5, truncated, 255 if >= 255. Atlas texels of no half (the empty half 1
 *      of a square whose s has an odd count, and every texel at or past the total area's last code) are 0.
 *  X8. Stats: triangles = count; atlas_width = W and atlas_height = H; texels = the texels of all halves used
 *      (s (s + 1) / 2 for half 0, s (s - 1) / 2 for half 1); texels_seen (S_w > 0) and texels_fallback (the rest);
 *      tiles_clamped; views_used = the views that contribute to at least one texel. The first five are set also on
 *      a layout query and on SM_ERR_CAPACITY (the last three 0); all are zero when the call fails otherwise.
 *
 * atlas is a DEVICE buffer of packed u8x3 texels (r, g, b) with atlas_pitch bytes per row and room for
 * atlas_capacity_width x atlas_capacity_height texels; only the W x H texels at its start are written (bytes past
 * 3 W of a row and rows past H stay untouched). atlas NULL with a 0 x 0 capacity is a layout query. If W >
 * max_atlas_side, or the capacity is smaller than W x H, the call returns SM_ERR_CAPACITY with the stats set and
 * writes nothing; a caller that hits max_atlas_side raises texel_size. uv (DEVICE, 6 x count floats, may be NULL) is
 * written together with the atlas. Each view's colour is a DEVICE u8x3 image of its camera's size, color_pitch bytes
 * per row. SM_ERR_INVALID_ARGUMENT, with no launch, for NULL params or stats, triangles NULL with count > 0, count >=
 * 2^28, views NULL with view_count > 0, view_count outside [0, SM_TEXTURE_MAX_VIEWS], a view camera or pose that
 * sm_render_mesh refuses, a view colour that is NULL or whose pitch is below 3 x width, texel_size not finite and
 * > 0, max_atlas_side outside [8, SM_TEXTURE_MAX_ATLAS_SIDE], max_view_angle_deg outside (0, 90], depth_tolerance
 * negative, NaN or infinite, atlas NULL with a capacity that is not 0 x 0, a negative capacity, atlas_pitch below 3
 * x atlas_capacity_width, or uv overlapping the triangles or the atlas; and, found on the device and reported after
 * the call's second synchronisation with nothing written, for a list that breaks X1.
 * The call synchronises `stream` three times (surfels_size(); the input checks and the layout; the end), plus once,
 * with cudaFree's device synchronisation, in a call whose buffers grow (by x 1.5); the per-view work is ordered on
 * `stream` without a host round trip. Memory (allocated by the first call, grown with the input, freed by
 * sm_destroy; sm_create allocates nothing for it): 24 bytes per triangle of capacity (sort keys in and out, the
 * tile records) plus the radix sort's scratch, 16 bytes per texel of the laid-out area (the float4 accumulators),
 * 4 bytes per pixel of the largest view (its depth) and sm_render_mesh's own scratch. */
#define SM_TEXTURE_MAX_TILE 512
#define SM_TEXTURE_MAX_VIEWS 1024
#define SM_TEXTURE_MAX_ATLAS_SIDE 32768
typedef struct sm_texture_params {
  float texel_size;            /* metres per texel; 0.004 (about one VGA pixel at 1.4 m) */
  int32_t max_atlas_side;      /* 16384; in [8, SM_TEXTURE_MAX_ATLAS_SIDE] */
  float max_view_angle_deg;    /* 75; in (0, 90]: views seeing a texel more obliquely do not contribute */
  float depth_tolerance;       /* 0.01, relative to the texel's camera depth; >= 0 */
} sm_texture_params;
typedef struct sm_texture_stats {
  uint64_t triangles;
  int32_t atlas_width, atlas_height;
  uint64_t texels;                 /* in the halves of all tiles */
  uint64_t texels_seen;            /* at least one view contributed */
  uint64_t texels_fallback;        /* no view contributed: the corner blend */
  uint64_t tiles_clamped;          /* triangles whose tile was capped at SM_TEXTURE_MAX_TILE */
  uint64_t views_used;             /* views that contributed to at least one texel */
} sm_texture_stats;
typedef struct sm_texture_view {
  sm_render_params camera;     /* size, intrinsics (pixel-corner convention), near/far: as sm_render_mesh */
  float view_T_global[12];     /* 3x4 row-major, global -> camera */
  const uint8_t* color;        /* DEVICE, packed u8x3 rows (r, g, b), as the stream frames */
  size_t color_pitch;
} sm_texture_view;
/* Host only, no device needed. */
void sm_default_texture_params(sm_texture_params* p);
int sm_mesh_texture(sm_reconstruction* r, void* stream, const sm_texture_params* p,
                    const uint32_t* triangles /* device, 3 x count */, uint64_t count,
                    const sm_texture_view* views /* host array */, int32_t view_count,
                    uint8_t* atlas /* device u8x3, pitched; NULL with 0 x 0 capacity = layout query */,
                    size_t atlas_pitch, int32_t atlas_capacity_width, int32_t atlas_capacity_height,
                    float* uv /* device, 6 x count: (u, v) per corner in the listed order, in [0, 1]; may be NULL */,
                    sm_texture_stats* stats);

/* ---- exposure compensation between the texture views (DESIGN.md section 1 row f20, section 5.18) ---------------
 * Cameras with auto-exposure and auto white balance give the views of one surface different brightness, and X6's
 * mean then shows patches whose edges follow the set of views. sm_mesh_texture_compensated fits one gain per view
 * and channel jointly over surface points the views share (Brown & Lowe 2007, gain compensation) and textures with
 * each view's samples scaled by its gains. Everything of sm_mesh_texture holds (arguments, checks, layout,
 * capacity protocol, X1-X8, the stats, read-only on the surfel state), with these rules added:
 *  G1. Sample points. P = min(count, floor(max_samples / view_count)), 0 without views. Point p in [0, P) lies on
 *      triangle t_p = floor(p * count / P) (u64): its corners in LIST order as (a, b, c) and alpha = beta =
 *      float(1/3) in X5's form give its position X and normal n (no X2 rotation, no clamp).
 *  G2. Samples. s_pv (3 channels) is X6's bilinear sample of view v at point p: the same depth raster, visibility,
 *      angle and footprint tests; the weight w is not used. The sample is absent if X6 rejects the view or any
 *      channel lies outside [min_level, max_level]. k_p = the present samples of p; p takes part in the fit iff
 *      k_p >= 2. n_v = the present samples of view v at such points; a view with n_v = 0 keeps gain 1.
 *  G3. Objective, per channel: E(g) = sum_p sum_(v in p) (g_v s_pv - m_p)^2 / sigma_noise^2 + sum_v n_v (g_v -
 *      1)^2 / sigma_gain^2, m_p = (1 / k_p) sum_(u in p) g_u s_pu. Its normal equations A g = b are, per view,
 *      (A x)_v = y_v(x) * cN + (n_v * cG) * x_v and b_v = n_v * cG with cN = 1 / (sigma_noise * sigma_noise),
 *      cG = 1 / (sigma_gain * sigma_gain) and y_v(x) = sum_p s_pv * (s_pv * x_v - m_p(x)).
 *  G4. Solve. fp64 from here on (samples and sigmas promoted; each product, sum, quotient and square root rounded
 *      alone), the three channels independently. m_p(x) = (sum over views in order of s_pv * x_v, from 0) / k_p.
 *      A column sum over points (y_v, and the data terms of G6) is a 32-ary tree: TREE(t_0 .. t_31) = t_0 after
 *      t_i = t_i + t_(i + off) for i < off, off = 16, 8, 4, 2, 1; level 1 is TREE of each 32 consecutive points
 *      (term 0 for a point past P, not in the fit or without a sample of v), level 2 the TREE of each 32
 *      consecutive level-1 sums (a block of 1024 points, 0 past the last); then, while more than one value is
 *      left, the TREE of each 32 consecutive values (0 past the last) replaces them. A sum over views (dot
 *      products) is TREE of the 32 TREEs of views 32w .. 32w + 31 (0 past view_count). Conjugate gradients from
 *      x = 1: r = b - A x, d = r, rr = r . r; each of `iterations` steps of a channel whose rr != 0: pAp = d . A d;
 *      if !(pAp > 0) the channel stops; else alpha = rr / pAp, x = x + alpha * d, r = r - alpha * (A d), rr' =
 *      r . r, beta = rr' / rr, d = r + beta * d, rr = rr'. The prior alone fixes the common scale only loosely
 *      (views that disagree for other reasons than exposure pull every gain down), so a view with n_v > 0 gets
 *      g = float(x / xbar) (every other view 1), xbar = (sum over views of n_v * x_v) / (sum over views of n_v) (two sums over views; xbar
 *      = 1 when the second is 0 or the quotient is not > 0): their n_v-weighted mean is 1 per channel.
 *  G5. Application. X6 with each channel's sample replaced by float(g_v,ch * sample_ch) before the product with w;
 *      X7 unchanged (the corner blend is not compensated). With iterations = 0 every gain is 1 and the atlas equals
 *      sm_mesh_texture's.
 *  G6. Stats: points = P, samples = sum of n_v, views_fitted = the views with n_v > 0; rms_before and rms_after =
 *      sqrt(D / (3 samples)) (0 without samples) at x = 1 and at x = the float gains, where D = (D_r + D_g) + D_b
 *      and D_ch = the sum over views of the G4 column sums of (s_pv * x_v - m_p(x))^2.
 * gains (HOST, 3 x view_count floats: r, g, b per view; may be NULL) and gain_stats are written only by a call that
 * fills the atlas (with count 0: every gain 1 and gain_stats zero); every other return leaves gains untouched and
 * gain_stats zero, and a layout query or SM_ERR_CAPACITY sets stats as sm_mesh_texture does. SM_ERR_INVALID_ARGUMENT
 * also for gp or gain_stats NULL, max_samples or iterations negative, sigma_noise or sigma_gain not finite and > 0,
 * min_level or max_level not finite, or min_level > max_level. The call renders every view twice (once to sample,
 * once to accumulate), adds one synchronisation (the gain read-back) and launches a number of kernels that depends
 * only on view_count, iterations and whether P > 0. Memory, on top of sm_mesh_texture's: 12 bytes per sample
 * (P x view_count, the sample matrix), 28 bytes per point (k_p and m_p), 24 bytes per view per 1024 points (the
 * level-2 column sums) and a fixed 88 KB of solver state. */
typedef struct sm_texture_gain_params {
  int32_t max_samples;     /* P x view_count entries of the sample matrix; 1 << 23 (96 MB at 12 bytes) */
  int32_t iterations;      /* conjugate-gradient steps; 0 = every gain 1; 32 */
  float sigma_noise;       /* grey levels; 10 (Brown & Lowe) */
  float sigma_gain;        /* the prior that fixes the common scale; 1 (Brown & Lowe's 0.1 undoes most of the
                              correction along a chain of views, 3 lets noisy views shrink the common scale:
                              DESIGN.md section 5.18) */
  float min_level, max_level;   /* 5, 250: a sample with any channel outside takes no part in the fit */
} sm_texture_gain_params;
typedef struct sm_texture_gain_stats {
  uint64_t points;         /* sample points P */
  uint64_t samples;        /* (point, view) samples in the fit */
  uint64_t views_fitted;   /* views with at least one such sample; every other view keeps gain 1 */
  double rms_before, rms_after;   /* grey levels, at gain 1 and at the fitted gains */
} sm_texture_gain_stats;
/* Host only, no device needed. */
void sm_default_texture_gain_params(sm_texture_gain_params* p);
int sm_mesh_texture_compensated(sm_reconstruction* r, void* stream, const sm_texture_params* p,
                                const sm_texture_gain_params* gp,
                                const uint32_t* triangles /* device, 3 x count */, uint64_t count,
                                const sm_texture_view* views /* host array */, int32_t view_count,
                                uint8_t* atlas, size_t atlas_pitch, int32_t atlas_capacity_width,
                                int32_t atlas_capacity_height, float* uv,
                                float* gains /* HOST, 3 x view_count; may be NULL */,
                                sm_texture_stats* stats, sm_texture_gain_stats* gain_stats);

/* ---- connected pieces of a triangle mesh (DESIGN.md section 1 row f18, section 5.16) ----------------------------
 * The surfel mesher leaves small floating pieces behind: a pair of surfels at a depth edge, or a few surfels the
 * normal gate cut off from their neighbours. sm_mesh_components splits a caller's triangle list into its connected
 * pieces, gives every triangle the number of its piece and every piece its size, area and bounds, and returns the
 * triangles of the pieces that pass the thresholds of sm_component_params (e.g. before sm_mesh_simplify and
 * sm_mesh_texture, so floaters take no part of the budget or the atlas). Positions are the current SMOOTH positions
 * (what sm_render_mesh draws); the call only reads the surfel state.
 *
 * t is a triangle's position in the list.
 *  C1. Input. Every corner must be a present slot (radius^2 > 0) below surfels_size() and no triangle may repeat a
 *      corner (X1 of sm_mesh_texture). Manifoldness is not required. 0 triangles are legal.
 *  C2. Adjacency. Triangles s and t are adjacent when they share an undirected edge {a, b}, in either winding and
 *      with any number of triangles on that edge. A piece is a class of the transitive closure of this relation: a
 *      triangle with no adjacent triangle is a piece of its own, and two pieces that touch only at a slot stay two.
 *  C3. Numbering. Pieces are numbered 0, 1, ... in the order of their smallest triangle position; labels[t] is the
 *      number of t's piece. Partition and numbering do not depend on thread order.
 *  C4. Area. P_i = the smooth position of slot i converted to double; e1, e2, g and gg as in S1 of sm_mesh_simplify
 *      (each double operation rounded on its own); a_t = 0.5 * sqrt(gg). q_t = rint(a_t * 2^30) (ties to even),
 *      capped at 2^36; q_t = 0 when a_t is not finite. A piece's area units Q = the integer sum of its q_t (below
 *      2^64 for count < 2^28), so any summation order gives the same bits. Its area is double(Q) * 2^-30 (m^2).
 *  C5. Bounds. A piece's lo / hi are the per-axis min / max of the fp32 smooth positions of its triangles' corners,
 *      compared in IEEE totalOrder (-0 < +0).
 *  C6. Keep. A piece is kept iff its triangle count >= min_triangles, Q >= rint(min_area * 2^30) (computed on the
 *      host in double), and keep_largest is 0 or its rank is below keep_largest; the rank orders all pieces by
 *      (Q descending, number ascending).
 *  C7. Output. The triangles of kept pieces, in input order, corners and winding unchanged. Stats: triangles_in =
 *      count, triangles_out, components, components_kept, and the triangle count and area of the rank-0 piece. All
 *      zero when the call fails for any reason other than capacity.
 *
 * out is a DEVICE buffer of 3 x out_capacity uint32 (may be NULL with out_capacity 0: a count query); labels (DEVICE,
 * count int32) and table (DEVICE, table_capacity entries, piece p at entry p) may be NULL. If out_capacity <
 * triangles_out, or table is not NULL and table_capacity < components, the call returns SM_ERR_CAPACITY with the
 * stats set and writes nothing; both counts are at most count, so capacities of count always suffice.
 * SM_ERR_INVALID_ARGUMENT, with no launch, for NULL params or stats, triangles NULL with count > 0, out NULL with
 * out_capacity > 0, table NULL with table_capacity > 0, count >= 2^28, min_area negative, NaN or infinite, or out,
 * labels or table overlapping the triangles or each other; and, found on the device and reported after the call's
 * second synchronisation with nothing written, for a list that breaks C1.
 * The call synchronises `stream` three times (surfels_size(); the input checks and the numbering; the end), plus
 * once, with cudaFree's device synchronisation, in a call whose buffers grow (by x 1.5); on return the output is
 * written by work enqueued on `stream`. Memory (allocated by the first call, grown with the input, freed by
 * sm_destroy; sm_create allocates nothing for it): 60 to 108 bytes per triangle of capacity (an undirected-edge hash
 * table of which a call uses and clears the power of two >= 4 x count slots, a u64 key and a u32 owner each: 48 to
 * 96; the union-find parents: 4; the root flags and the keep flags, each scanned: 8) and 68 bytes per piece (the
 * triangle count, the first triangle and the keep flag: 12; Q: 8; the ordered-int bounds: 24; the rank sort's keys
 * and values in and out: 24), plus the radix sort's scratch. */
typedef struct sm_component_params {
  uint64_t min_triangles;   /* 10; pieces with fewer triangles are dropped (0 and 1 keep every piece) */
  double min_area;          /* 0 m^2; finite, >= 0; pieces with less area are dropped */
  uint64_t keep_largest;    /* 0 = no limit; else only the keep_largest pieces of largest area can be kept */
} sm_component_params;
typedef struct sm_component_stats {
  uint64_t triangles_in, triangles_out;
  uint64_t components, components_kept;
  uint64_t largest_triangles;   /* of the rank-0 piece (0 for an empty list) */
  double largest_area;          /* m^2, of the rank-0 piece */
} sm_component_stats;
typedef struct sm_mesh_component {
  uint64_t triangles;
  double area;                  /* m^2: double(Q) * 2^-30 */
  float lo[3], hi[3];           /* smooth-position bounds of its corners */
  uint32_t first_triangle;      /* its smallest triangle position */
  int32_t kept;                 /* 1 if its triangles are in out */
} sm_mesh_component;
/* Host only, no device needed. */
void sm_default_component_params(sm_component_params* p);
int sm_mesh_components(sm_reconstruction* r, void* stream, const sm_component_params* p,
                       const uint32_t* triangles /* device, 3 x count */, uint64_t count,
                       uint32_t* out /* device, 3 x out_capacity; may be NULL with out_capacity 0 */,
                       uint64_t out_capacity,
                       int32_t* labels /* device, count; may be NULL */,
                       sm_mesh_component* table /* device, table_capacity; may be NULL with table_capacity 0 */,
                       uint64_t table_capacity, sm_component_stats* stats);

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
 * W*H host arrays; any pointer may be NULL. After sm_compact the rasters name
 * old slots: the call returns SM_ERR_INVALID_ARGUMENT until the next Integrate. */
int sm_download_rasters(sm_reconstruction* r, void* stream,
                        uint32_t* supporting_surfels, uint32_t* supporting_surfel_counts,
                        float* supporting_surfel_depth_sums, uint32_t* conflicting_surfels,
                        float* first_surfel_depth, uint8_t* new_surfel_flag_vector,
                        uint32_t* new_surfel_indices);

/* ---- reclaiming the slots of merged surfels (DESIGN.md section 1 row f15, section 5.13) ----------------------
 * A merge never frees its slot (like the reference, kernels.cu:1987: radius^2 = -1), so surfels_size() only grows
 * and a long session reaches the surfel cap with far fewer live surfels. sm_compact removes the merged slots in
 * place. It is never called by the library itself.
 *  1. Which slots go: slot i in [0, surfels_size()) is removed iff its radius^2 (row 7) < 0, the merge mark of
 *     Integrate(); every other slot is kept.
 *  2. Stable order: a kept slot moves from i to the number of kept slots below i. old_to_new[i] is that index, or
 *     SM_INVALID_SURFEL_INDEX for a removed slot.
 *  3. State after the call: every row sm_dump_state defines is the gather of the old rows through the map (rows
 *     11-16 and 23 are scratch), except that a neighbour link (rows 19-22) is replaced by the new index of the slot
 *     it names; a link that names a removed slot (or one >= surfels_size()) becomes SM_INVALID_SURFEL_INDEX and is
 *     counted in links_dropped. surfels_size() = surfel_count() = slots_after, the merge count is 0, both
 *     regularisation record buffers hold the gathered current records (as after sm_load_state), and the sticky
 *     cap-overflow flag stays as it is (the call itself does not report it).
 *  4. Nothing to remove: when the merge count (sm_dump_state's merge_count) is 0, or no slot carries the mark,
 *     the call launches no kernel and changes nothing; old_to_new, if given, is the identity. The delta-transfer
 *     token stays valid.
 *  5. Otherwise the handle takes a fresh state generation: the next sm_transfer_delta_to_cpu with an older token
 *     does a full transfer.
 *  6. Memory: allocated by the first call that removes something, freed by sm_destroy: the map and one row of
 *     scratch (8 bytes per slot of the cap), and CUB's scan storage. The SoA and the records are compacted in
 *     place.
 *  7. SM_ERR_INVALID_ARGUMENT, with no launch, for a NULL handle, or old_to_new non-NULL with map_capacity <
 *     surfels_size(). stats and old_to_new (DEVICE, surfels_size() entries) may be NULL.
 * What else names a slot:
 *  - The persistent mesh of sm_mesh_update is carried over when no slot it uses was removed, that is, when no
 *    surfel merged since the last update (compact right after sm_mesh_update): its snapshot, umbrellas, per-slot
 *    stats and the triangle lists are remapped (mesh_remapped = 1). sm_mesh_read(SM_MESH_ALL) then returns the
 *    remapped mesh and an update with no change in between reports slots_changed == 0 and empty deltas; a corner of
 *    the last update's removed list whose slot was removed reads SM_INVALID_SURFEL_INDEX. Otherwise the mesh is
 *    dropped (mesh_remapped = 0): sm_mesh_read fails and the next update rebuilds everything.
 *  - sm_download_rasters refuses until the next Integrate.
 *  - An open session: the call is allowed between pushes, on the session's stream. In frame-graph mode the front
 *    half of the frame in flight (projection, association, merge decisions, blending) runs again on the new slots,
 *    and the merge count the session reports becomes 0.
 *  - Outside the handle the caller must rebuild or remap (with old_to_new): sm_knn_index objects built from the
 *    reconstruction, triangle lists from sm_triangulate or sm_mesh_fill_holes, visualisation buffers and their
 *    latest_mesh_surfel_count, and CPU copies keyed by slot. The keyframe database holds poses and codes only.
 * The call synchronises `stream` (the counters; the map; the end), plus once more when a mesh is carried over. */
typedef struct sm_compact_stats {
  uint64_t slots_before;      /* surfels_size() before */
  uint64_t slots_after;       /* surfels_size() after == surfel_count() */
  uint64_t merged_removed;
  uint64_t links_dropped;     /* neighbour links (rows 19-22) of kept slots that named a removed slot */
  int32_t  mesh_remapped;     /* 1 if a persistent sm_mesh_update mesh existed and was carried over */
  int32_t  reserved;
} sm_compact_stats;
int sm_compact(sm_reconstruction* r, void* stream,
               uint32_t* old_to_new /* device, slots_before entries; may be NULL */, uint64_t map_capacity,
               sm_compact_stats* stats /* may be NULL */);

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
 * sm_frame_counters, sm_knn_build_from_reconstruction, sm_render_surfels, sm_render_mesh, sm_track_frame,
 * sm_track_linearize, sm_track_frame_rgbd, sm_track_linearize_rgbd, sm_relocalise,
 * sm_mesh_update, sm_mesh_read, sm_triangulate, sm_surfel_count / sm_surfels_size),
 * sm_compact, and sm_regularize, which main.cc calls between frames (:1573-1579). In frame-graph mode the step a push
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
