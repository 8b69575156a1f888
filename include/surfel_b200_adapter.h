// surfel_b200_adapter.h — header-only drop-in for vis::CUDASurfelReconstruction.
//
// Same public surface as the reference class
// (applications/surfel_meshing/src/surfel_meshing/cuda_surfel_reconstruction.h:44-176); every
// method forwards to the C ABI of libsurfel_b200.so (surfel_b200.h). Include this header INSTEAD of
// "surfel_meshing/cuda_surfel_reconstruction.h" in main.cc and drop cuda_surfel_reconstruction.cc /
// cuda_surfel_reconstruction_kernels.{cc,cu} from the SurfelMeshing target (INTEGRATION.md).
// It needs the reference's own libvis headers (Eigen, Sophus) and therefore only BUILDS inside the
// reference's tree; in this repository (no Eigen) it is syntax- and type-checked against minimal
// stand-ins of those headers (tests/stubs/, tests/test_adapter_syntax.py), with a translation unit that
// makes the calls main.cc makes.
//
// Define SURFEL_B200_DELTA_TRANSFER before including to let TransferAllToCPU() use
// sm_transfer_delta_to_cpu (one token per CUDASurfelBuffersCPU object): the same arrays, a fraction of
// the PCIe traffic; that variant synchronises the stream itself (main.cc:1261-1287 synchronises right
// after the call anyway).
#pragma once

#include <cuda_runtime.h>  // cudaGraphicsMapResources & co. are part of the generic interop API

#include <map>

#include <libvis/camera.h>
#include <libvis/cuda/cuda_buffer.h>
#include <libvis/libvis.h>
#include <libvis/logging.h>
#include <libvis/sophus.h>

#include "surfel_b200.h"
#include "surfel_meshing/cuda_surfels_cpu.h"

namespace vis {

class SurfelMeshingRenderWindow;

class CUDASurfelReconstruction {
 public:
  // The three GL resources serve UpdateVisualizationBuffers(); the render window only feeds debug
  // displays of the reference and is ignored.
  CUDASurfelReconstruction(usize max_surfel_count, const PinholeCamera4f& depth_camera,
                           cudaGraphicsResource_t vertex_buffer_resource,
                           cudaGraphicsResource_t neighbor_index_buffer_resource,
                           cudaGraphicsResource_t normal_vertex_buffer_resource,
                           const shared_ptr<SurfelMeshingRenderWindow>& /*render_window*/)
      : vertex_buffer_resource_(vertex_buffer_resource),
        neighbor_index_buffer_resource_(neighbor_index_buffer_resource),
        normal_vertex_buffer_resource_(normal_vertex_buffer_resource) {
    Check(sm_create(&handle_, max_surfel_count, depth_camera.width(), depth_camera.height(),
                    depth_camera.parameters()[0], depth_camera.parameters()[1], depth_camera.parameters()[2],
                    depth_camera.parameters()[3]));
    // The reference records its seven stage-event pairs on every Integrate() (cuda_surfel_reconstruction.cc:131-319).
    Check(sm_enable_timings(handle_, 1));
  }
  ~CUDASurfelReconstruction() { sm_destroy(handle_); }
  CUDASurfelReconstruction(const CUDASurfelReconstruction&) = delete;
  CUDASurfelReconstruction& operator=(const CUDASurfelReconstruction&) = delete;

  void Integrate(cudaStream_t stream, u32 frame_index, float depth_scaling, CUDABuffer<u16>* depth_buffer,
                 const CUDABuffer<float2>& normals_buffer, const CUDABuffer<float>& radius_buffer,
                 const CUDABuffer<Vec3u8>& color_buffer, const SE3f& global_T_local, float sensor_noise_factor,
                 float max_surfel_confidence, float regularizer_weight, int regularization_frame_window_size,
                 bool do_blending, int measurement_blending_radius,
                 int regularization_iterations_per_integration_iteration,
                 float radius_factor_for_regularization_neighbors, float normal_compatibility_threshold_deg,
                 int surfel_integration_active_window_size) {
    sm_integrate_params p;
    p.depth_scaling = depth_scaling;
    p.sensor_noise_factor = sensor_noise_factor;
    p.max_surfel_confidence = max_surfel_confidence;
    p.regularizer_weight = regularizer_weight;
    p.regularization_frame_window_size = regularization_frame_window_size;
    p.do_blending = do_blending ? 1 : 0;
    p.measurement_blending_radius = measurement_blending_radius;
    p.regularization_iterations_per_integration_iteration = regularization_iterations_per_integration_iteration;
    p.radius_factor_for_regularization_neighbors = radius_factor_for_regularization_neighbors;
    p.normal_compatibility_threshold_deg = normal_compatibility_threshold_deg;
    p.surfel_integration_active_window_size = surfel_integration_active_window_size;
    float g[12], l[12];
    ToRowMajor(global_T_local, g);
    ToRowMajor(global_T_local.inverse(), l);  // as cuda_surfel_reconstruction.cc:144
    Check(sm_integrate(handle_, stream, frame_index, &p, depth_buffer->ToCUDA().address(),
                       depth_buffer->ToCUDA().pitch(),
                       reinterpret_cast<const float*>(normals_buffer.ToCUDA().address()),
                       normals_buffer.ToCUDA().pitch(), radius_buffer.ToCUDA().address(),
                       radius_buffer.ToCUDA().pitch(),
                       reinterpret_cast<const uint8_t*>(color_buffer.ToCUDA().address()),
                       color_buffer.ToCUDA().pitch(), g, l));
  }

  void Regularize(cudaStream_t stream, u32 frame_index, float regularizer_weight,
                  float radius_factor_for_regularization_neighbors, int regularization_frame_window_size) {
    Check(sm_regularize(handle_, stream, frame_index, regularizer_weight, radius_factor_for_regularization_neighbors,
                        regularization_frame_window_size));
  }

  // The "buffers" object must be locked with LockWriteBuffers() when this is called.
  void TransferAllToCPU(cudaStream_t stream, u32 frame_index, CUDASurfelsCPU* buffers) {
    CUDASurfelBuffersCPU* b = buffers->write_buffers();
    b->frame_index = frame_index;
#ifdef SURFEL_B200_DELTA_TRANSFER
    sm_transfer_stats stats;
    Check(sm_transfer_delta_to_cpu(handle_, stream, frame_index, &transfer_tokens_[b], b->surfel_x_buffer,
                                   b->surfel_y_buffer, b->surfel_z_buffer, b->surfel_radius_squared_buffer,
                                   b->surfel_normal_x_buffer, b->surfel_normal_y_buffer, b->surfel_normal_z_buffer,
                                   b->surfel_last_update_stamp_buffer, &stats));
    b->surfel_count = stats.surfel_count;
#else
    uint64_t count = 0;
    Check(sm_transfer_all_to_cpu(handle_, stream, frame_index, b->surfel_x_buffer, b->surfel_y_buffer,
                                 b->surfel_z_buffer, b->surfel_radius_squared_buffer, b->surfel_normal_x_buffer,
                                 b->surfel_normal_y_buffer, b->surfel_normal_z_buffer,
                                 b->surfel_last_update_stamp_buffer, &count));
    b->surfel_count = count;
#endif
  }

  // cuda_surfel_reconstruction.cc:361-403: the three OpenGL buffers are mapped, filled by ONE sweep
  // (sm_update_visualization_buffers) and unmapped. Resources that are null are skipped, like there.
  void UpdateVisualizationBuffers(cudaStream_t stream, u32 frame_index, u32 latest_triangulated_frame_index,
                                  u32 latest_mesh_surfel_count, int surfel_integration_active_window_size,
                                  bool visualize_last_update_timestamp, bool visualize_creation_timestamp,
                                  bool visualize_radii, bool visualize_normals) {
    sm_visualization_params p;
    p.frame_index = frame_index;
    p.latest_triangulated_frame_index = latest_triangulated_frame_index;
    p.latest_mesh_surfel_count = latest_mesh_surfel_count;
    p.surfel_integration_active_window_size = surfel_integration_active_window_size;
    p.point_size_in_floats = 4;  // sizeof(Point3fC3u8) / sizeof(float)
    p.visualize_last_update_timestamp = visualize_last_update_timestamp;
    p.visualize_creation_timestamp = visualize_creation_timestamp;
    p.visualize_radii = visualize_radii;
    p.visualize_normals = visualize_normals;
    float* vertex = nullptr;
    uint32_t* neighbor_index = nullptr;
    float* normal_vertex = nullptr;
#ifndef SURFEL_B200_NO_GL_INTEROP
    cudaGraphicsResource_t resources[3];
    int count = 0;
    for (cudaGraphicsResource_t res : {vertex_buffer_resource_, neighbor_index_buffer_resource_, normal_vertex_buffer_resource_})
      if (res) resources[count++] = res;
    if (count == 0) return;
    CheckCuda(cudaGraphicsMapResources(count, resources, stream));
    size_t bytes = 0;
    if (vertex_buffer_resource_) CheckCuda(cudaGraphicsResourceGetMappedPointer(reinterpret_cast<void**>(&vertex), &bytes, vertex_buffer_resource_));
    if (neighbor_index_buffer_resource_) CheckCuda(cudaGraphicsResourceGetMappedPointer(reinterpret_cast<void**>(&neighbor_index), &bytes, neighbor_index_buffer_resource_));
    if (normal_vertex_buffer_resource_) CheckCuda(cudaGraphicsResourceGetMappedPointer(reinterpret_cast<void**>(&normal_vertex), &bytes, normal_vertex_buffer_resource_));
    Check(sm_update_visualization_buffers(handle_, stream, &p, vertex, neighbor_index, normal_vertex));
    CheckCuda(cudaGraphicsUnmapResources(count, resources, stream));
#else
    (void)stream; (void)p; (void)vertex; (void)neighbor_index; (void)normal_vertex;
#endif
  }

  void ExportVertices(cudaStream_t stream, CUDABuffer<float>* position_buffer, CUDABuffer<u8>* color_buffer) {
    Check(sm_export_vertices(handle_, stream, position_buffer->ToCUDA().address(), color_buffer->ToCUDA().address()));
  }

  void GetTimings(float* data_association, float* surfel_merging, float* measurement_blending, float* integration,
                  float* neighbor_update, float* new_surfel_creation, float* regularization) {
    float t[7] = {0, 0, 0, 0, 0, 0, 0};
    Check(sm_get_timings(handle_, t));  // of the last Integrate(); timings are on since construction
    *data_association = t[0]; *surfel_merging = t[1]; *measurement_blending = t[2]; *integration = t[3];
    *neighbor_update = t[4]; *new_surfel_creation = t[5]; *regularization = t[6];
  }

  inline u32 surfel_count() const { u32 v = 0; Check(sm_surfel_count(handle_, &v)); return v; }
  inline u32 surfels_size() const { u32 v = 0; Check(sm_surfels_size(handle_, &v)); return v; }

  // Extension (no counterpart in the reference): reclaims the slots of merged surfels (sm_compact). old_to_new
  // (device, surfels_size() entries, may be null) receives the new slot of every old one; a CPU meshing consumer
  // keyed by slot (SurfelMeshing::IntegrateCUDABuffers) must apply it or restart from a full transfer.
  sm_compact_stats Compact(cudaStream_t stream, u32* old_to_new = nullptr, uint64_t map_capacity = 0) {
    sm_compact_stats stats;
    Check(sm_compact(handle_, stream, old_to_new, map_capacity, &stats));
    return stats;
  }

  // Extension (no counterpart in the reference): a triangle list over the slots (device, 3 x count) simplified by
  // half-edge collapses (sm_mesh_simplify) into `out` (device, 3 x count suffices); every corner stays a slot.
  sm_simplify_stats SimplifyMesh(cudaStream_t stream, const u32* triangles, uint64_t count, u32* out,
                                 const sm_simplify_params* params = nullptr) {
    sm_simplify_params defaults;
    sm_default_simplify_params(&defaults);
    sm_simplify_stats stats;
    Check(sm_mesh_simplify(handle_, stream, params ? params : &defaults, triangles, count, out, count, &stats));
    return stats;
  }

  // Extension (no counterpart in the reference): the connected pieces of a triangle list over the slots (device, 3 x
  // count) (sm_mesh_components): the triangles of the kept pieces into `out` (device, 3 x count), each triangle's
  // piece number into `labels` (device, count, may be null) and the pieces into `table` (device, table_capacity
  // entries, may be null with 0).
  sm_component_stats MeshComponents(cudaStream_t stream, const u32* triangles, uint64_t count, u32* out,
                                    int32_t* labels = nullptr, sm_mesh_component* table = nullptr,
                                    uint64_t table_capacity = 0, const sm_component_params* params = nullptr) {
    sm_component_params defaults;
    sm_default_component_params(&defaults);
    sm_component_stats stats;
    Check(sm_mesh_components(handle_, stream, params ? params : &defaults, triangles, count, out, count, labels, table,
                             table_capacity, &stats));
    return stats;
  }

  // Extension (no counterpart in the reference): a texture atlas for a triangle list over the slots (device, 3 x
  // count) from posed colour views (sm_mesh_texture): `atlas` (device u8x3, atlas_pitch bytes per row, room for
  // capacity_width x capacity_height texels) and `uv` (device, 6 x count, may be null). A call with a null atlas and
  // a 0 x 0 capacity only lays the atlas out: the returned stats give its size.
  sm_texture_stats TextureMesh(cudaStream_t stream, const u32* triangles, uint64_t count, const sm_texture_view* views,
                               int view_count, u8* atlas, size_t atlas_pitch, int capacity_width, int capacity_height,
                               float* uv, const sm_texture_params* params = nullptr) {
    sm_texture_params defaults;
    sm_default_texture_params(&defaults);
    sm_texture_stats stats;
    const int status = sm_mesh_texture(handle_, stream, params ? params : &defaults, triangles, count, views,
                                       view_count, atlas, atlas_pitch, capacity_width, capacity_height, uv, &stats);
    if (!(status == SM_ERR_CAPACITY && atlas == nullptr)) Check(status);
    return stats;
  }

  // Extension: TextureMesh with one gain per view and channel fitted over the surface the views share, so that
  // views of different exposure and white balance give one even atlas (sm_mesh_texture_compensated). `gains` (host,
  // 3 x view_count, may be null) receives the fitted gains and `gain_stats` (may be null) the fit's statistics.
  sm_texture_stats TextureMeshCompensated(cudaStream_t stream, const u32* triangles, uint64_t count,
                                          const sm_texture_view* views, int view_count, u8* atlas, size_t atlas_pitch,
                                          int capacity_width, int capacity_height, float* uv, float* gains = nullptr,
                                          sm_texture_gain_stats* gain_stats = nullptr,
                                          const sm_texture_params* params = nullptr,
                                          const sm_texture_gain_params* gain_params = nullptr) {
    sm_texture_params defaults;
    sm_default_texture_params(&defaults);
    sm_texture_gain_params gain_defaults;
    sm_default_texture_gain_params(&gain_defaults);
    sm_texture_stats stats;
    sm_texture_gain_stats fit;
    const int status = sm_mesh_texture_compensated(handle_, stream, params ? params : &defaults,
                                                   gain_params ? gain_params : &gain_defaults, triangles, count, views,
                                                   view_count, atlas, atlas_pitch, capacity_width, capacity_height, uv,
                                                   gains, &stats, &fit);
    if (!(status == SM_ERR_CAPACITY && atlas == nullptr)) Check(status);
    if (gain_stats) *gain_stats = fit;
    return stats;
  }

 private:
  static void ToRowMajor(const SE3f& t, float* out) {
    const auto m = t.matrix3x4();
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 4; ++c) out[4 * r + c] = m(r, c);
  }
  // The reference aborts on any CUDA error (libvis/cuda/cuda_util.h:35-49).
  static void Check(int status) {
    if (status != SM_OK) LOG(FATAL) << "surfel_b200: " << sm_last_error();
  }
  static void CheckCuda(cudaError_t e) {
    if (e != cudaSuccess) LOG(FATAL) << "surfel_b200 adapter: " << cudaGetErrorString(e);
  }
  sm_reconstruction* handle_ = nullptr;
  cudaGraphicsResource_t vertex_buffer_resource_;
  cudaGraphicsResource_t neighbor_index_buffer_resource_;
  cudaGraphicsResource_t normal_vertex_buffer_resource_;
#ifdef SURFEL_B200_DELTA_TRANSFER
  std::map<const CUDASurfelBuffersCPU*, sm_transfer_token> transfer_tokens_;  // one per write / read buffer
#endif
};

}  // namespace vis
