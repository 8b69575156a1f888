// cuda_depth_processing_shims.cu — link-level drop-in for the reference's object
// applications/surfel_meshing/src/surfel_meshing/cuda_depth_processing.cu (SURVEY §8 b(3)).
//
// Defines the vis::-named host functions that file exports (declarations:
// APP/cuda_depth_processing.cuh:43-122, explicit instantiations APP/cuda_depth_processing.cu:287-334,
// :459-510, :573-587, :629-633) on top of the C ABI of libsurfel_b200.so. A maintainer of the
// reference replaces cuda_depth_processing.cu by this file in the SurfelMeshing target
// (applications/surfel_meshing/CMakeLists.txt:5-12) and links libsurfel_b200.so; main.cc:1015-1191 then
// runs the sm_90a kernels without a source change. Compiled against the reference's own headers, so
// a signature mismatch is a compile error; oracle/Makefile builds it into
// oracle/_ref/libsurfel_shimref.so (the reference's restated host glue + these shims) for
// tests/test_parity_gpu.py::test_vis_depth_processing_shims.
//
// Error convention of the reference (libvis/src/libvis/cuda/cuda_util.h:35-49): failures abort through
// LOG(FATAL); the C ABI's status codes are mapped onto that.

#include <cuda_runtime.h>

#include <libvis/libvis.h>
#include <libvis/cuda/cuda_buffer.cuh>
#include <libvis/cuda/cuda_matrix.cuh>
#include <libvis/logging.h>

#include "surfel_meshing/cuda_depth_processing.cuh"

#include "surfel_b200.h"

namespace vis {

namespace {
inline void CheckStatus(int status, const char* what) {
  if (status != SM_OK) {
    LOG(FATAL) << what << ": " << sm_last_error();
  }
}

template <int count>
void OutlierShim(cudaStream_t stream, int required_count, float tolerance, const CUDABuffer_<u16>& input_depth,
                 float depth_fx, float depth_fy, float depth_cx, float depth_cy, const CUDABuffer_<u16>** other_depths,
                 const CUDAMatrix3x4* others_TR_reference, CUDABuffer_<u16>* output_depth) {
  constexpr int kOthers = count - 1;
  const uint16_t* depths[kOthers];
  size_t pitches[kOthers];
  float mats[kOthers * 12];
  for (int i = 0; i < kOthers; ++i) {
    depths[i] = other_depths[i]->address();
    pitches[i] = other_depths[i]->pitch();
    const CUDAMatrix3x4& m = others_TR_reference[i];
    const float rows[12] = {m.row0.x, m.row0.y, m.row0.z, m.row0.w, m.row1.x, m.row1.y, m.row1.z, m.row1.w,
                            m.row2.x, m.row2.y, m.row2.z, m.row2.w};
    for (int k = 0; k < 12; ++k) mats[12 * i + k] = rows[k];
  }
  CheckStatus(sm_outlier_depth_map_fusion(stream, kOthers, required_count, tolerance, depth_fx, depth_fy, depth_cx,
                                          depth_cy, input_depth.width(), input_depth.height(), input_depth.address(),
                                          input_depth.pitch(), depths, pitches, mats, output_depth->address(),
                                          output_depth->pitch()),
              "OutlierDepthMapFusionCUDA");
}
}  // namespace

void BilateralFilteringAndDepthCutoffCUDA(cudaStream_t stream, float sigma_xy, float sigma_value_factor,
                                          u16 value_to_ignore, float radius_factor, u16 max_depth,
                                          float depth_valid_region_radius, const CUDABuffer_<u16>& input_depth,
                                          CUDABuffer_<u16>* output_depth) {
  CheckStatus(sm_bilateral_filter_and_depth_cutoff(stream, sigma_xy, sigma_value_factor, value_to_ignore, radius_factor,
                                                   max_depth, depth_valid_region_radius, input_depth.width(),
                                                   input_depth.height(), input_depth.address(), input_depth.pitch(),
                                                   output_depth->address(), output_depth->pitch()),
              "BilateralFilteringAndDepthCutoffCUDA");
}

template <int count, typename DepthT>
void OutlierDepthMapFusionCUDA(cudaStream_t stream, float tolerance, const CUDABuffer_<DepthT>& input_depth,
                               float depth_fx, float depth_fy, float depth_cx, float depth_cy,
                               const CUDABuffer_<DepthT>** other_depths, const CUDAMatrix3x4* others_TR_reference,
                               CUDABuffer_<u16>* output_depth) {
  OutlierShim<count>(stream, -1, tolerance, input_depth, depth_fx, depth_fy, depth_cx, depth_cy, other_depths,
                     others_TR_reference, output_depth);
}

template <int count, typename DepthT>
void OutlierDepthMapFusionCUDA(cudaStream_t stream, int required_count, float tolerance,
                               const CUDABuffer_<DepthT>& input_depth, float depth_fx, float depth_fy, float depth_cx,
                               float depth_cy, const CUDABuffer_<DepthT>** other_depths,
                               const CUDAMatrix3x4* others_TR_reference, CUDABuffer_<u16>* output_depth) {
  OutlierShim<count>(stream, required_count, tolerance, input_depth, depth_fx, depth_fy, depth_cx, depth_cy,
                     other_depths, others_TR_reference, output_depth);
}

#define SM_INSTANTIATE_OUTLIER(COUNT)                                                                                  \
  template void OutlierDepthMapFusionCUDA<COUNT, u16>(cudaStream_t, float, const CUDABuffer_<u16>&, float, float,     \
                                                      float, float, const CUDABuffer_<u16>**, const CUDAMatrix3x4*,    \
                                                      CUDABuffer_<u16>*);                                              \
  template void OutlierDepthMapFusionCUDA<COUNT, u16>(cudaStream_t, int, float, const CUDABuffer_<u16>&, float, float, \
                                                      float, float, const CUDABuffer_<u16>**, const CUDAMatrix3x4*,    \
                                                      CUDABuffer_<u16>*);
SM_INSTANTIATE_OUTLIER(9)
SM_INSTANTIATE_OUTLIER(7)
SM_INSTANTIATE_OUTLIER(5)
SM_INSTANTIATE_OUTLIER(3)
#undef SM_INSTANTIATE_OUTLIER

template <typename DepthT>
void ErodeDepthMapCUDA(cudaStream_t stream, int radius, const CUDABuffer_<DepthT>& input_depth,
                       CUDABuffer_<DepthT>* output_depth) {
  if (radius < 1 || radius > 3) LOG(FATAL) << "radius value of " << radius << " is not supported.";  // :569
  CheckStatus(sm_erode_depth_map(stream, radius, input_depth.width(), input_depth.height(), input_depth.address(),
                                 input_depth.pitch(), output_depth->address(), output_depth->pitch()),
              "ErodeDepthMapCUDA");
}
template void ErodeDepthMapCUDA<u16>(cudaStream_t, int, const CUDABuffer_<u16>&, CUDABuffer_<u16>*);

template <typename DepthT>
void CopyWithoutBorderCUDA(cudaStream_t stream, const CUDABuffer_<DepthT>& input_depth,
                           CUDABuffer_<DepthT>* output_depth) {
  CheckStatus(sm_erode_depth_map(stream, 0, input_depth.width(), input_depth.height(), input_depth.address(),
                                 input_depth.pitch(), output_depth->address(), output_depth->pitch()),
              "CopyWithoutBorderCUDA");
}
template void CopyWithoutBorderCUDA<u16>(cudaStream_t, const CUDABuffer_<u16>&, CUDABuffer_<u16>*);

void ComputeNormalsAndDropBadPixelsCUDA(cudaStream_t stream, float observation_angle_threshold_deg, float depth_scaling,
                                        float depth_fx, float depth_fy, float depth_cx, float depth_cy,
                                        const CUDABuffer_<u16>& in_depth, CUDABuffer_<u16>* out_depth,
                                        CUDABuffer_<float2>* out_normals) {
  CheckStatus(sm_compute_normals_and_drop_bad_pixels(stream, observation_angle_threshold_deg, depth_scaling, depth_fx,
                                                     depth_fy, depth_cx, depth_cy, in_depth.width(), in_depth.height(),
                                                     in_depth.address(), in_depth.pitch(), out_depth->address(),
                                                     out_depth->pitch(), reinterpret_cast<float*>(out_normals->address()),
                                                     out_normals->pitch()),
              "ComputeNormalsAndDropBadPixelsCUDA");
}

void ComputePointRadiiAndRemoveIsolatedPixelsCUDA(cudaStream_t stream, float point_radius_extension_factor,
                                                  float point_radius_clamp_factor, float depth_scaling, float depth_fx,
                                                  float depth_fy, float depth_cx, float depth_cy,
                                                  const CUDABuffer_<u16>& depth_buffer, CUDABuffer_<float>* radius_buffer,
                                                  CUDABuffer_<u16>* out_depth) {
  CheckStatus(sm_compute_point_radii_and_remove_isolated_pixels(
                  stream, point_radius_extension_factor, point_radius_clamp_factor, depth_scaling, depth_fx, depth_fy,
                  depth_cx, depth_cy, depth_buffer.width(), depth_buffer.height(), depth_buffer.address(),
                  depth_buffer.pitch(), radius_buffer->address(), radius_buffer->pitch(), out_depth->address(),
                  out_depth->pitch()),
              "ComputePointRadiiAndRemoveIsolatedPixelsCUDA");
}

}  // namespace vis
