// oracle/ref_driver.cu — TEST INFRASTRUCTURE, not product code.
//
// Eigen-/Qt-free driver around the UNMODIFIED reference kernels. The three
// reference translation units (APP/cuda_surfel_reconstruction_kernels.cu,
// APP/cuda_depth_processing.cu, libvis/src/libvis/cuda/cuda_buffer.cu, plus
// loguru.cpp) are compiled where they lie under the reference sources (REF) by
// oracle/Makefile and linked with this file into oracle/_ref/libsurfel_ref.so.
// Nothing from the reference is copied into the repository.
//
// The reference's host glue cannot be compiled here (Eigen/Sophus/Qt are absent),
// so this file restates it call for call (APP = applications/surfel_meshing/src/
// surfel_meshing):
//   * APP/cuda_surfel_reconstruction.cc:44-91,112-337,339-359,405-429  (class)
//   * APP/cuda_surfel_reconstruction_kernels.cc:37-511                  (wrappers)
//   * APP/main.cc:902-995,1015-1191                                     (frame loop)
// Poses enter as precomputed 3x4 float matrices so no Sophus is needed and both
// the oracle and the product consume bit-identical inputs.
//
// Exported C ABI: the same functions as include/surfel_b200.h with the prefix
// `smref_` instead of `sm_`. Only tests/, __graft_entry__.smoke() and
// bench.py's reference arm may load this library.

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
#include <string>
#include <vector>

#include <libvis/libvis.h>
#include <libvis/cuda/cuda_buffer.cuh>
#include <libvis/cuda/cuda_matrix.cuh>
#include <libvis/cuda/cuda_util.h>

#include "surfel_meshing/cuda_depth_processing.cuh"
#include "surfel_meshing/cuda_surfel_reconstruction_kernels.cuh"

#include "../include/surfel_b200.h"

using namespace vis;

namespace {

thread_local std::string g_error;

// Surfel::kInvalidIndex (APP/surfel.h:63) == kInvalidSurfelIndex (kernels.cu:74).
constexpr u32 kInvalidIndex = 0xFFFFFFFFu;

int Fail(int code, const std::string& msg) {
  g_error = msg;
  return code;
}

#define REF_CUDA(call)                                                              \
  do {                                                                              \
    cudaError_t e_ = (call);                                                        \
    if (e_ != cudaSuccess) {                                                        \
      return Fail(SM_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    }                                                                               \
  } while (0)

// Mirror of libvis CUDABuffer<T> (libvis/src/libvis/cuda/cuda_buffer_inl.h:36-48):
// a pitched 2-D allocation described by the POD CUDABuffer_<T>.
template <typename T>
struct PitchedBuffer {
  CUDABuffer_<T> b;
  PitchedBuffer() : b(nullptr, 0, 0, 0) {}
  cudaError_t Alloc(int height, int width) {
    T* ptr = nullptr;
    size_t pitch = 0;
    cudaError_t e = cudaMallocPitch(reinterpret_cast<void**>(&ptr), &pitch, width * sizeof(T), height);
    if (e != cudaSuccess) return e;
    b = CUDABuffer_<T>(ptr, height, width, pitch);
    return cudaSuccess;
  }
  void Free() {
    if (b.address()) cudaFree(b.address());
    b = CUDABuffer_<T>(nullptr, 0, 0, 0);
  }
};

CUDAMatrix3x4 ToMatrix(const float* m) {
  CUDAMatrix3x4 r;
  r.row0 = make_float4(m[0], m[1], m[2], m[3]);
  r.row1 = make_float4(m[4], m[5], m[6], m[7]);
  r.row2 = make_float4(m[8], m[9], m[10], m[11]);
  return r;
}

template <typename T>
CUDABuffer_<T> View(const T* ptr, int height, int width, size_t pitch) {
  return CUDABuffer_<T>(const_cast<T*>(ptr), height, width, pitch);
}

}  // namespace

// Restatement of class CUDASurfelReconstruction's state,
// APP/cuda_surfel_reconstruction.h:131-170.
struct smref_reconstruction {
  int width = 0, height = 0;
  float fx = 0, fy = 0, cx = 0, cy = 0;
  u32 surfel_count = 0;
  u32 merge_count = 0;
  usize max_surfel_count = 0;

  PitchedBuffer<float> surfels;
  PitchedBuffer<u8> distance_map;
  PitchedBuffer<float> surfel_depth_average_deltas;
  PitchedBuffer<u8> new_distance_map;
  PitchedBuffer<float> new_surfel_depth_average_deltas;
  PitchedBuffer<u32> supporting_surfels;
  PitchedBuffer<u32> supporting_surfel_counts;
  PitchedBuffer<float> supporting_surfel_depth_sums;
  PitchedBuffer<u32> conflicting_surfels;
  PitchedBuffer<float> first_surfel_depth;
  PitchedBuffer<u8> new_surfel_flag_vector;
  PitchedBuffer<u32> new_surfel_indices;
  PitchedBuffer<u32> num_merges_buffer;  // function-static in the reference (kernels.cc:479)

  void* new_surfels_temp_storage = nullptr;
  usize new_surfels_temp_storage_bytes = 0;

  // Pre-processing scratch (APP/main.cc filtered_depth_buffer_B) + stream runner state.
  PitchedBuffer<u16> filtered_depth_B;
  PitchedBuffer<u16> run_depth_A;
  PitchedBuffer<float2> run_normals;
  PitchedBuffer<float> run_radius;
  std::vector<PitchedBuffer<u16>> run_raw;   // ring of uploaded raw depth maps
  std::vector<PitchedBuffer<uchar3>> run_color;
  cudaStream_t upload_stream = nullptr;
  std::vector<cudaEvent_t> upload_events;

  cudaEvent_t ev[14] = {};
  bool timings = false;
  unsigned long long launches = 0;
};

namespace {

// ---- APP/cuda_surfel_reconstruction_kernels.cc restated ----------------------

struct Intrinsics {
  float fx, fy, cx, cy, fx_inv, fy_inv, cx_inv_pixel_center, cy_inv_pixel_center;
};

// kernels.cc:63-74 (identical at :236-247).
Intrinsics MakeIntrinsics(const smref_reconstruction* r) {
  Intrinsics k;
  k.fx = r->fx; k.fy = r->fy; k.cx = r->cx; k.cy = r->cy;
  k.fx_inv = 1.0f / k.fx;
  k.fy_inv = 1.0f / k.fy;
  const float cx_pixel_center = k.cx - 0.5f;
  const float cy_pixel_center = k.cy - 0.5f;
  k.cx_inv_pixel_center = -cx_pixel_center / k.fx;
  k.cy_inv_pixel_center = -cy_pixel_center / k.fy;
  return k;
}

// kernels.cc:37-146.
int CreateNewSurfels(smref_reconstruction* r, cudaStream_t stream, u32 frame_index,
                     const CUDAMatrix3x4& global_T_local, float depth_scaling,
                     float radius_factor, const CUDABuffer_<u16>& depth,
                     const CUDABuffer_<float2>& normals, const CUDABuffer_<float>& radius,
                     const CUDABuffer_<uchar3>& color, u32* new_surfel_count, u8* new_surfel_count_2) {
  const Intrinsics k = MakeIntrinsics(r);
  constexpr int kBlockWidth = 32, kBlockHeight = 32;
  dim3 grid_dim(GetBlockCount(depth.width(), kBlockWidth), GetBlockCount(depth.height(), kBlockHeight));
  dim3 block_dim(kBlockWidth, kBlockHeight);

  CallCreateNewSurfelsCUDASerializingKernel(stream, grid_dim, block_dim, depth, r->supporting_surfels.b,
                                            r->conflicting_surfels.b, r->new_surfel_flag_vector.b);
  const int num_items = depth.width() * depth.height();
  if (r->new_surfels_temp_storage_bytes == 0) {
    CallCUBExclusiveSum(r->new_surfels_temp_storage, r->new_surfels_temp_storage_bytes,
                        r->new_surfel_flag_vector.b.address(), r->new_surfel_indices.b.address(), num_items, stream);
    REF_CUDA(cudaMalloc(&r->new_surfels_temp_storage, r->new_surfels_temp_storage_bytes));
  }
  CallCUBExclusiveSum(r->new_surfels_temp_storage, r->new_surfels_temp_storage_bytes,
                      r->new_surfel_flag_vector.b.address(), r->new_surfel_indices.b.address(), num_items, stream);
  // DownloadPartAsync of the last index and the last flag (kernels.cc:116-125).
  REF_CUDA(cudaMemcpyAsync(new_surfel_count, r->new_surfel_indices.b.address() + (num_items - 1), sizeof(u32),
                           cudaMemcpyDeviceToHost, stream));
  REF_CUDA(cudaMemcpyAsync(new_surfel_count_2, r->new_surfel_flag_vector.b.address() + (num_items - 1), sizeof(u8),
                           cudaMemcpyDeviceToHost, stream));
  CallCreateNewSurfelsCUDACreationKernel(stream, grid_dim, block_dim, frame_index, 1.0f / depth_scaling, k.fx_inv,
                                         k.fy_inv, k.cx_inv_pixel_center, k.cy_inv_pixel_center, global_T_local, depth,
                                         normals, radius, color, r->supporting_surfels.b, r->new_surfel_flag_vector.b,
                                         r->new_surfel_indices.b, r->surfel_count, r->surfels.b,
                                         radius_factor * radius_factor);
  r->launches += 3;  // flag kernel, creation kernel, + CUB scan (counted as >=1 below)
  r->launches += 2;
  return SM_OK;
}

// kernels.cc:148-205.
void BlendMeasurements(smref_reconstruction* r, cudaStream_t stream, int measurement_blending_radius,
                       float depth_correction_factor, CUDABuffer_<u16> depth) {
  r->distance_map.b.Clear(0, stream);
  r->new_distance_map.b.Clear(0, stream);
  constexpr int kBlockWidth = 32, kBlockHeight = 32;
  dim3 grid_dim(GetBlockCount(r->supporting_surfels.b.width(), kBlockWidth),
                GetBlockCount(r->supporting_surfels.b.height(), kBlockHeight));
  dim3 block_dim(kBlockWidth, kBlockHeight);
  CallBlendMeasurementsCUDAStartKernel(stream, grid_dim, block_dim, 1.0f / depth_correction_factor, depth,
                                       r->supporting_surfels.b, r->supporting_surfel_counts.b,
                                       r->supporting_surfel_depth_sums.b, r->distance_map.b,
                                       r->surfel_depth_average_deltas.b, r->new_distance_map.b,
                                       r->new_surfel_depth_average_deltas.b);
  r->launches += 3;
  for (int iteration = 2; iteration < measurement_blending_radius; ++iteration) {
    CallBlendMeasurementsCUDAIterationKernel(stream, grid_dim, block_dim, iteration,
                                             1.0f / (measurement_blending_radius - 1.0f),
                                             1.0f / depth_correction_factor, depth, r->supporting_surfels.b,
                                             r->distance_map.b, r->surfel_depth_average_deltas.b,
                                             r->new_distance_map.b, r->new_surfel_depth_average_deltas.b);
    r->launches += 1;
  }
}

dim3 SurfelGrid(u32 surfel_count) { return dim3(GetBlockCount(surfel_count, 1024)); }

// cuda_surfel_reconstruction.cc:112-320.
int Integrate(smref_reconstruction* r, cudaStream_t stream, u32 frame_index, const sm_integrate_params& p,
              CUDABuffer_<u16> depth, CUDABuffer_<float2> normals, CUDABuffer_<float> radius,
              CUDABuffer_<uchar3> color, const CUDAMatrix3x4& global_T_local, const CUDAMatrix3x4& local_T_global) {
  const Intrinsics k = MakeIntrinsics(r);
  const float depth_correction_factor = 1.0f / p.depth_scaling;
  const float cos_normal_threshold = cosf(M_PI / 180.0f * p.normal_compatibility_threshold_deg);
  const dim3 block_dim(1024);

  if (r->timings) cudaEventRecord(r->ev[0], stream);
  r->supporting_surfels.b.Clear(kInvalidIndex, stream);
  r->supporting_surfel_counts.b.Clear(0, stream);
  r->supporting_surfel_depth_sums.b.Clear(0, stream);
  r->conflicting_surfels.b.Clear(kInvalidIndex, stream);
  r->first_surfel_depth.b.Clear(std::numeric_limits<float>::infinity(), stream);
  r->launches += 5;

  if (r->surfel_count > 0) {  // kernels.cc:356, :406
    CallRenderMinDepthCUDAKernel(stream, SurfelGrid(r->surfel_count), block_dim, frame_index,
                                 p.surfel_integration_active_window_size, k.fx, k.fy, k.cx, k.cy, local_T_global,
                                 r->surfel_count, r->surfels.b, r->first_surfel_depth.b);
    CallAssociateSurfelsCUDAKernel(stream, SurfelGrid(r->surfel_count), block_dim, frame_index,
                                   p.surfel_integration_active_window_size, k.fx, k.fy, k.cx, k.cy, local_T_global,
                                   p.sensor_noise_factor, cos_normal_threshold, r->surfel_count, r->surfels.b,
                                   depth_correction_factor, depth, normals, radius, r->supporting_surfels.b,
                                   r->supporting_surfel_counts.b, r->supporting_surfel_depth_sums.b,
                                   r->conflicting_surfels.b, r->first_surfel_depth.b);
    r->launches += 2;
  }
  if (r->timings) { cudaEventRecord(r->ev[1], stream); cudaEventRecord(r->ev[2], stream); }

  if (r->surfel_count > 0) {  // kernels.cc:442-511
    r->num_merges_buffer.b.Clear(0, stream);
    CallMergeSurfelsCUDAKernel(stream, dim3(GetBlockCount(r->surfel_count, kMergeBlockWidth)), dim3(kMergeBlockWidth),
                               k.fx, k.fy, k.cx, k.cy, local_T_global, p.sensor_noise_factor, cos_normal_threshold,
                               r->surfel_count, r->surfels.b, depth_correction_factor, depth, normals, radius,
                               r->supporting_surfels.b, r->supporting_surfel_counts.b,
                               r->supporting_surfel_depth_sums.b, r->conflicting_surfels.b, r->first_surfel_depth.b,
                               r->num_merges_buffer.b);
    r->launches += 2;
    u32 num_merges = 0;
    REF_CUDA(cudaMemcpyAsync(&num_merges, r->num_merges_buffer.b.address(), sizeof(u32), cudaMemcpyDeviceToHost, stream));
    REF_CUDA(cudaStreamSynchronize(stream));  // host sync #1 (kernels.cc:509)
    r->merge_count += num_merges;
  }
  if (r->timings) { cudaEventRecord(r->ev[3], stream); cudaEventRecord(r->ev[4], stream); }

  if (p.do_blending) {
    BlendMeasurements(r, stream, p.measurement_blending_radius, depth_correction_factor, depth);
  }
  if (r->timings) { cudaEventRecord(r->ev[5], stream); cudaEventRecord(r->ev[6], stream); }

  if (r->surfel_count > 0) {  // kernels.cc:207-277
    CallIntegrateMeasurementsCUDAKernel(stream, SurfelGrid(r->surfel_count), block_dim, frame_index,
                                        p.surfel_integration_active_window_size, p.max_surfel_confidence,
                                        p.sensor_noise_factor, cos_normal_threshold, 1.0f / p.depth_scaling, k.fx, k.fy,
                                        k.cx, k.cy, k.fx_inv, k.fy_inv, k.cx_inv_pixel_center, k.cy_inv_pixel_center,
                                        local_T_global, global_T_local, depth, normals, radius, color,
                                        r->supporting_surfels.b, r->supporting_surfel_counts.b,
                                        r->conflicting_surfels.b, r->first_surfel_depth.b, r->surfel_count,
                                        r->surfels.b);
    r->launches += 1;
  }
  if (r->timings) { cudaEventRecord(r->ev[7], stream); cudaEventRecord(r->ev[8], stream); }

  if (r->surfel_count > 0) {  // kernels.cc:279-340
    CallUpdateNeighborsCUDAKernel(stream, SurfelGrid(r->surfel_count), block_dim, frame_index,
                                  p.surfel_integration_active_window_size,
                                  p.radius_factor_for_regularization_neighbors * p.radius_factor_for_regularization_neighbors,
                                  r->supporting_surfels.b, k.fx, k.fy, k.cx, k.cy, local_T_global,
                                  p.sensor_noise_factor, depth_correction_factor, depth, radius,
                                  r->first_surfel_depth.b, r->surfel_count, r->surfels.b);
    CallUpdateNeighborsCUDARemoveReplacedNeighborsKernel(stream, SurfelGrid(r->surfel_count), block_dim, frame_index,
                                                         r->surfel_count, r->surfels.b);
    r->launches += 2;
  }
  if (r->timings) { cudaEventRecord(r->ev[9], stream); cudaEventRecord(r->ev[10], stream); }

  u32 new_surfel_count = 0;
  u8 new_surfel_count_2 = 0;
  int status = CreateNewSurfels(r, stream, frame_index, global_T_local, p.depth_scaling,
                                p.radius_factor_for_regularization_neighbors, depth, normals, radius, color,
                                &new_surfel_count, &new_surfel_count_2);
  if (status != SM_OK) return status;
  if (r->timings) cudaEventRecord(r->ev[11], stream);

  REF_CUDA(cudaStreamSynchronize(stream));  // host sync #2 (cuda_surfel_reconstruction.cc:290)
  r->surfel_count += new_surfel_count + new_surfel_count_2;
  if (r->surfel_count > r->max_surfel_count) {
    // The reference never checks the cap (SURVEY §5) and would write out of bounds;
    // the oracle reports it so that a test cannot silently run into UB.
    return Fail(SM_ERR_CAPACITY, "reference oracle: surfel cap exceeded (reference behaviour: unchecked overflow)");
  }

  if (r->timings) cudaEventRecord(r->ev[12], stream);
  if (p.regularization_iterations_per_integration_iteration == 0) {
    RegularizeSurfelsCUDA(stream, /*disable_denoising*/ true, frame_index,
                          p.radius_factor_for_regularization_neighbors, p.regularizer_weight,
                          p.regularization_frame_window_size, r->surfel_count, &r->surfels.b);
    r->launches += (r->surfel_count > 0) ? 1 : 0;
  } else {
    for (int i = 0; i < p.regularization_iterations_per_integration_iteration; ++i) {
      RegularizeSurfelsCUDA(stream, /*disable_denoising*/ false, frame_index,
                            p.radius_factor_for_regularization_neighbors, p.regularizer_weight,
                            p.regularization_frame_window_size, r->surfel_count, &r->surfels.b);
      r->launches += (r->surfel_count > 0) ? 4 : 0;
    }
  }
  if (r->timings) cudaEventRecord(r->ev[13], stream);
  REF_CUDA(cudaGetLastError());
  return SM_OK;
}

// APP/main.cc:1015-1191.
int Preprocess(smref_reconstruction* r, cudaStream_t stream, const sm_preprocess_params& p,
               const CUDABuffer_<u16>& raw, const CUDABuffer_<u16>* others, const CUDAMatrix3x4* others_TR_reference,
               CUDABuffer_<u16> A, CUDABuffer_<float2> normals, CUDABuffer_<float> radius) {
  CUDABuffer_<u16> B = r->filtered_depth_B.b;
  BilateralFilteringAndDepthCutoffCUDA(stream, p.bilateral_filter_sigma_xy, p.bilateral_filter_sigma_depth_factor,
                                       /*value_to_ignore*/ 0, p.bilateral_filter_radius_factor,
                                       p.depth_scaling * p.max_depth, p.depth_valid_region_radius, raw, &A);
  const int K = p.outlier_filtering_frame_count;
  std::vector<const CUDABuffer_<u16>*> other_ptrs(K);
  for (int i = 0; i < K; ++i) other_ptrs[i] = &others[i];
  const bool all = p.outlier_filtering_required_inliers == -1 || p.outlier_filtering_required_inliers == K;
#define REF_CALL_FUSION(n)                                                                                         \
  do {                                                                                                             \
    if (all)                                                                                                       \
      OutlierDepthMapFusionCUDA<n + 1, u16>(stream, p.outlier_filtering_depth_tolerance_factor, A, r->fx, r->fy,   \
                                            r->cx, r->cy, other_ptrs.data(), others_TR_reference, &B);             \
    else                                                                                                           \
      OutlierDepthMapFusionCUDA<n + 1, u16>(stream, p.outlier_filtering_required_inliers,                          \
                                            p.outlier_filtering_depth_tolerance_factor, A, r->fx, r->fy, r->cx,    \
                                            r->cy, other_ptrs.data(), others_TR_reference, &B);                    \
  } while (0)
  if (K == 2) REF_CALL_FUSION(2);
  else if (K == 4) REF_CALL_FUSION(4);
  else if (K == 6) REF_CALL_FUSION(6);
  else if (K == 8) REF_CALL_FUSION(8);
  else return Fail(SM_ERR_INVALID_ARGUMENT, "Unsupported value for outlier_filtering_frame_count");
#undef REF_CALL_FUSION
  if (p.depth_erosion_radius > 0) {
    if (p.depth_erosion_radius > 3) return Fail(SM_ERR_INVALID_ARGUMENT, "erosion radius not supported");
    ErodeDepthMapCUDA<u16>(stream, p.depth_erosion_radius, B, &A);
  } else {
    CopyWithoutBorderCUDA<u16>(stream, B, &A);
  }
  ComputeNormalsAndDropBadPixelsCUDA(stream, p.observation_angle_threshold_deg, p.depth_scaling, r->fx, r->fy, r->cx,
                                     r->cy, A, &B, &normals);
  ComputePointRadiiAndRemoveIsolatedPixelsCUDA(stream, p.point_radius_extension_factor, p.point_radius_clamp_factor,
                                               p.depth_scaling, r->fx, r->fy, r->cx, r->cy, B, &radius, &A);
  r->launches += 5;
  REF_CUDA(cudaGetLastError());
  return SM_OK;
}

}  // namespace

// ---- exported C ABI (prefix smref_) -------------------------------------------

extern "C" {

const char* smref_last_error(void) { return g_error.c_str(); }
const char* smref_version(void) { return "surfel_ref oracle (reference kernels rebuilt for sm_90a)"; }

int smref_create(smref_reconstruction** out, uint64_t max_surfel_count, int32_t width, int32_t height, float fx,
                 float fy, float cx, float cy) {
  if (!out || width <= 0 || height <= 0 || max_surfel_count == 0) return Fail(SM_ERR_INVALID_ARGUMENT, "bad argument");
  smref_reconstruction* r = new smref_reconstruction();
  r->width = width; r->height = height;
  r->fx = fx; r->fy = fy; r->cx = cx; r->cy = cy;
  r->max_surfel_count = max_surfel_count;
  // cuda_surfel_reconstruction.cc:59-72.
  REF_CUDA(r->surfels.Alloc(kSurfelAttributeCount, static_cast<int>(max_surfel_count)));
  REF_CUDA(r->distance_map.Alloc(height, width));
  REF_CUDA(r->surfel_depth_average_deltas.Alloc(height, width));
  REF_CUDA(r->new_distance_map.Alloc(height, width));
  REF_CUDA(r->new_surfel_depth_average_deltas.Alloc(height, width));
  REF_CUDA(r->supporting_surfels.Alloc(height, width));
  REF_CUDA(r->supporting_surfel_counts.Alloc(height, width));
  REF_CUDA(r->supporting_surfel_depth_sums.Alloc(height, width));
  REF_CUDA(r->conflicting_surfels.Alloc(height, width));
  REF_CUDA(r->first_surfel_depth.Alloc(height, width));
  REF_CUDA(r->new_surfel_flag_vector.Alloc(1, height * width));
  REF_CUDA(r->new_surfel_indices.Alloc(1, height * width));
  REF_CUDA(r->num_merges_buffer.Alloc(1, 1));
  REF_CUDA(r->filtered_depth_B.Alloc(height, width));
  for (int i = 0; i < 14; ++i) REF_CUDA(cudaEventCreate(&r->ev[i]));
  *out = r;
  return SM_OK;
}

int smref_destroy(smref_reconstruction* r) {
  if (!r) return SM_OK;
  cudaDeviceSynchronize();
  r->surfels.Free(); r->distance_map.Free(); r->surfel_depth_average_deltas.Free(); r->new_distance_map.Free();
  r->new_surfel_depth_average_deltas.Free(); r->supporting_surfels.Free(); r->supporting_surfel_counts.Free();
  r->supporting_surfel_depth_sums.Free(); r->conflicting_surfels.Free(); r->first_surfel_depth.Free();
  r->new_surfel_flag_vector.Free(); r->new_surfel_indices.Free(); r->num_merges_buffer.Free();
  r->filtered_depth_B.Free(); r->run_depth_A.Free(); r->run_normals.Free(); r->run_radius.Free();
  for (auto& b : r->run_raw) b.Free();
  for (auto& b : r->run_color) b.Free();
  for (auto e : r->upload_events) cudaEventDestroy(e);
  if (r->upload_stream) cudaStreamDestroy(r->upload_stream);
  cudaFree(r->new_surfels_temp_storage);
  for (int i = 0; i < 14; ++i) cudaEventDestroy(r->ev[i]);
  delete r;
  return SM_OK;
}

int smref_reset(smref_reconstruction* r, void* /*stream*/) {
  r->surfel_count = 0;
  r->merge_count = 0;
  return SM_OK;
}

int smref_preprocess(smref_reconstruction* r, void* stream, const sm_preprocess_params* p, const uint16_t* raw_depth,
                     size_t raw_pitch, const uint16_t* const* other_depths, const size_t* other_pitches,
                     const float* others_TR_reference, uint16_t* out_depth, size_t out_depth_pitch, float* out_normals,
                     size_t out_normals_pitch, float* out_radius, size_t out_radius_pitch) {
  const int K = p->outlier_filtering_frame_count;
  std::vector<CUDABuffer_<u16>> others(K);
  std::vector<CUDAMatrix3x4> transforms(K);
  for (int i = 0; i < K; ++i) {
    others[i] = View<u16>(other_depths[i], r->height, r->width, other_pitches[i]);
    transforms[i] = ToMatrix(others_TR_reference + 12 * i);
  }
  return Preprocess(r, static_cast<cudaStream_t>(stream), *p, View<u16>(raw_depth, r->height, r->width, raw_pitch),
                    others.data(), transforms.data(), View<u16>(out_depth, r->height, r->width, out_depth_pitch),
                    View<float2>(reinterpret_cast<float2*>(out_normals), r->height, r->width, out_normals_pitch),
                    View<float>(out_radius, r->height, r->width, out_radius_pitch));
}

int smref_bilateral_filter_and_depth_cutoff(void* stream, float sigma_xy, float sigma_value_factor,
                                            uint16_t value_to_ignore, float radius_factor, uint16_t max_depth,
                                            float depth_valid_region_radius, int32_t width, int32_t height,
                                            const uint16_t* in_depth, size_t in_pitch, uint16_t* out_depth,
                                            size_t out_pitch) {
  CUDABuffer_<u16> out = View<u16>(out_depth, height, width, out_pitch);
  BilateralFilteringAndDepthCutoffCUDA(static_cast<cudaStream_t>(stream), sigma_xy, sigma_value_factor, value_to_ignore,
                                       radius_factor, max_depth, depth_valid_region_radius,
                                       View<u16>(in_depth, height, width, in_pitch), &out);
  REF_CUDA(cudaGetLastError());
  return SM_OK;
}

int smref_outlier_depth_map_fusion(void* stream, int32_t other_count, int32_t required_count, float tolerance, float fx,
                                   float fy, float cx, float cy, int32_t width, int32_t height,
                                   const uint16_t* in_depth, size_t in_pitch, const uint16_t* const* other_depths,
                                   const size_t* other_pitches, const float* others_TR_reference, uint16_t* out_depth,
                                   size_t out_pitch) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int K = other_count;
  std::vector<CUDABuffer_<u16>> others(K);
  std::vector<const CUDABuffer_<u16>*> other_ptrs(K);
  std::vector<CUDAMatrix3x4> transforms(K);
  for (int i = 0; i < K; ++i) {
    others[i] = View<u16>(other_depths[i], height, width, other_pitches[i]);
    other_ptrs[i] = &others[i];
    transforms[i] = ToMatrix(others_TR_reference + 12 * i);
  }
  CUDABuffer_<u16> A = View<u16>(in_depth, height, width, in_pitch);
  CUDABuffer_<u16> B = View<u16>(out_depth, height, width, out_pitch);
  const bool all = required_count == -1 || required_count == K;
#define REF_CALL_FUSION(n)                                                                                            \
  do {                                                                                                                \
    if (all)                                                                                                          \
      OutlierDepthMapFusionCUDA<n + 1, u16>(s, tolerance, A, fx, fy, cx, cy, other_ptrs.data(), transforms.data(), &B); \
    else                                                                                                              \
      OutlierDepthMapFusionCUDA<n + 1, u16>(s, required_count, tolerance, A, fx, fy, cx, cy, other_ptrs.data(),       \
                                            transforms.data(), &B);                                                   \
  } while (0)
  if (K == 2) REF_CALL_FUSION(2);
  else if (K == 4) REF_CALL_FUSION(4);
  else if (K == 6) REF_CALL_FUSION(6);
  else if (K == 8) REF_CALL_FUSION(8);
  else return Fail(SM_ERR_INVALID_ARGUMENT, "Unsupported value for outlier_filtering_frame_count");
#undef REF_CALL_FUSION
  REF_CUDA(cudaGetLastError());
  return SM_OK;
}

int smref_erode_depth_map(void* stream, int32_t radius, int32_t width, int32_t height, const uint16_t* in_depth,
                          size_t in_pitch, uint16_t* out_depth, size_t out_pitch) {
  CUDABuffer_<u16> out = View<u16>(out_depth, height, width, out_pitch);
  if (radius > 0) {
    if (radius > 3) return Fail(SM_ERR_INVALID_ARGUMENT, "erosion radius not supported");
    ErodeDepthMapCUDA<u16>(static_cast<cudaStream_t>(stream), radius, View<u16>(in_depth, height, width, in_pitch), &out);
  } else {
    CopyWithoutBorderCUDA<u16>(static_cast<cudaStream_t>(stream), View<u16>(in_depth, height, width, in_pitch), &out);
  }
  REF_CUDA(cudaGetLastError());
  return SM_OK;
}

int smref_compute_normals_and_drop_bad_pixels(void* stream, float observation_angle_threshold_deg, float depth_scaling,
                                              float fx, float fy, float cx, float cy, int32_t width, int32_t height,
                                              const uint16_t* in_depth, size_t in_pitch, uint16_t* out_depth,
                                              size_t out_pitch, float* out_normals, size_t normals_pitch) {
  CUDABuffer_<u16> out = View<u16>(out_depth, height, width, out_pitch);
  CUDABuffer_<float2> normals = View<float2>(reinterpret_cast<float2*>(out_normals), height, width, normals_pitch);
  ComputeNormalsAndDropBadPixelsCUDA(static_cast<cudaStream_t>(stream), observation_angle_threshold_deg, depth_scaling,
                                     fx, fy, cx, cy, View<u16>(in_depth, height, width, in_pitch), &out, &normals);
  REF_CUDA(cudaGetLastError());
  return SM_OK;
}

int smref_compute_point_radii_and_remove_isolated_pixels(void* stream, float point_radius_extension_factor,
                                                         float point_radius_clamp_factor, float depth_scaling, float fx,
                                                         float fy, float cx, float cy, int32_t width, int32_t height,
                                                         const uint16_t* in_depth, size_t in_pitch, float* out_radius,
                                                         size_t radius_pitch, uint16_t* out_depth, size_t out_pitch) {
  CUDABuffer_<u16> out = View<u16>(out_depth, height, width, out_pitch);
  CUDABuffer_<float> radius = View<float>(out_radius, height, width, radius_pitch);
  ComputePointRadiiAndRemoveIsolatedPixelsCUDA(static_cast<cudaStream_t>(stream), point_radius_extension_factor,
                                               point_radius_clamp_factor, depth_scaling, fx, fy, cx, cy,
                                               View<u16>(in_depth, height, width, in_pitch), &radius, &out);
  REF_CUDA(cudaGetLastError());
  return SM_OK;
}

int smref_integrate(smref_reconstruction* r, void* stream, uint32_t frame_index, const sm_integrate_params* p,
                    uint16_t* depth, size_t depth_pitch, const float* normals, size_t normals_pitch,
                    const float* radius, size_t radius_pitch, const uint8_t* color, size_t color_pitch,
                    const float global_T_local[12], const float local_T_global[12]) {
  return Integrate(r, static_cast<cudaStream_t>(stream), frame_index, *p,
                   View<u16>(depth, r->height, r->width, depth_pitch),
                   View<float2>(reinterpret_cast<const float2*>(normals), r->height, r->width, normals_pitch),
                   View<float>(radius, r->height, r->width, radius_pitch),
                   View<uchar3>(reinterpret_cast<const uchar3*>(color), r->height, r->width, color_pitch),
                   ToMatrix(global_T_local), ToMatrix(local_T_global));
}

// cuda_surfel_reconstruction.cc:322-337.
int smref_regularize(smref_reconstruction* r, void* stream, uint32_t frame_index, float regularizer_weight,
                     float radius_factor_for_regularization_neighbors, int32_t regularization_frame_window_size) {
  RegularizeSurfelsCUDA(static_cast<cudaStream_t>(stream), /*disable_denoising*/ false, frame_index,
                        radius_factor_for_regularization_neighbors, regularizer_weight,
                        regularization_frame_window_size, r->surfel_count, &r->surfels.b);
  r->launches += (r->surfel_count > 0) ? 4 : 0;
  REF_CUDA(cudaGetLastError());
  return SM_OK;
}

int smref_surfel_count(smref_reconstruction* r, uint32_t* out) { *out = r->surfel_count - r->merge_count; return SM_OK; }
int smref_surfels_size(smref_reconstruction* r, uint32_t* out) { *out = r->surfel_count; return SM_OK; }

// cuda_surfel_reconstruction.cc:339-359.
int smref_transfer_all_to_cpu(smref_reconstruction* r, void* stream, uint32_t /*frame_index*/, float* x, float* y,
                              float* z, float* radius_squared, float* nx, float* ny, float* nz,
                              uint32_t* last_update_stamp, uint64_t* out_count) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t pitch = r->surfels.b.pitch();
  const size_t bytes = r->surfel_count * sizeof(float);
  const char* base = reinterpret_cast<const char*>(r->surfels.b.address());
  if (out_count) *out_count = r->surfel_count;
  if (bytes == 0) return SM_OK;
  REF_CUDA(cudaMemcpyAsync(x, base + kSurfelSmoothX * pitch, bytes, cudaMemcpyDeviceToHost, s));
  REF_CUDA(cudaMemcpyAsync(y, base + kSurfelSmoothY * pitch, bytes, cudaMemcpyDeviceToHost, s));
  REF_CUDA(cudaMemcpyAsync(z, base + kSurfelSmoothZ * pitch, bytes, cudaMemcpyDeviceToHost, s));
  REF_CUDA(cudaMemcpyAsync(radius_squared, base + kSurfelRadiusSquared * pitch, bytes, cudaMemcpyDeviceToHost, s));
  REF_CUDA(cudaMemcpyAsync(nx, base + kSurfelNormalX * pitch, bytes, cudaMemcpyDeviceToHost, s));
  REF_CUDA(cudaMemcpyAsync(ny, base + kSurfelNormalY * pitch, bytes, cudaMemcpyDeviceToHost, s));
  REF_CUDA(cudaMemcpyAsync(nz, base + kSurfelNormalZ * pitch, bytes, cudaMemcpyDeviceToHost, s));
  REF_CUDA(cudaMemcpyAsync(last_update_stamp, base + kSurfelLastUpdateStamp * pitch, bytes, cudaMemcpyDeviceToHost, s));
  return SM_OK;
}

// cuda_surfel_reconstruction.cc:405-410.
int smref_export_vertices(smref_reconstruction* r, void* stream, float* position_buffer, uint8_t* color_buffer) {
  CUDABuffer_<float> pos = View<float>(position_buffer, 1, 3 * r->surfel_count, 3 * r->surfel_count * sizeof(float));
  CUDABuffer_<u8> col = View<u8>(color_buffer, 1, 3 * r->surfel_count, 3 * r->surfel_count);
  ExportVerticesCUDA(static_cast<cudaStream_t>(stream), r->surfel_count, r->surfels.b, &pos, &col);
  REF_CUDA(cudaGetLastError());
  return SM_OK;
}

// cuda_surfel_reconstruction.cc:361-403: the reference writes CUDA-mapped OpenGL buffers. No GL here:
// oracle/Makefile redirects the three interop calls of the reference's object file
// (cudaGraphicsMapResources / ...GetMappedPointer / ...UnmapResources) to the stand-ins below, which
// treat the "resource" handle as a plain device pointer, so the reference's own wrappers and kernels
// (kernels.cu:274-560) run unmodified into device buffers.
extern "C" cudaError_t smref_gl_map_resources(int, cudaGraphicsResource_t*, cudaStream_t) { return cudaSuccess; }
extern "C" cudaError_t smref_gl_unmap_resources(int, cudaGraphicsResource_t*, cudaStream_t) { return cudaSuccess; }
extern "C" cudaError_t smref_gl_get_mapped_pointer(void** pointer, size_t* size, cudaGraphicsResource_t resource) {
  *pointer = reinterpret_cast<void*>(resource);
  if (size) *size = 0;
  return cudaSuccess;
}

int smref_update_visualization_buffers(smref_reconstruction* r, void* stream, const sm_visualization_params* p,
                                       float* vertex_buffer, uint32_t* neighbor_index_buffer,
                                       float* normal_vertex_buffer) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (vertex_buffer) {
    UpdateSurfelVertexBufferCUDA(s, p->frame_index, p->surfel_integration_active_window_size, r->surfel_count,
                                 r->surfels.b, p->latest_triangulated_frame_index, p->latest_mesh_surfel_count,
                                 reinterpret_cast<cudaGraphicsResource_t>(vertex_buffer), p->point_size_in_floats,
                                 p->visualize_last_update_timestamp != 0, p->visualize_creation_timestamp != 0,
                                 p->visualize_radii != 0, p->visualize_normals != 0);
  }
  if (neighbor_index_buffer) {
    UpdateNeighborIndexBufferCUDA(s, r->surfel_count, r->surfels.b,
                                  reinterpret_cast<cudaGraphicsResource_t>(neighbor_index_buffer));
  }
  if (normal_vertex_buffer) {
    UpdateNormalVertexBufferCUDA(s, r->surfel_count, r->surfels.b,
                                 reinterpret_cast<cudaGraphicsResource_t>(normal_vertex_buffer));
  }
  REF_CUDA(cudaGetLastError());
  return SM_OK;
}

// cuda_surfel_reconstruction.cc:412-429.
int smref_get_timings(smref_reconstruction* r, float out_ms[7]) {
  if (!r->timings) return Fail(SM_ERR_INVALID_ARGUMENT, "timings not enabled");
  REF_CUDA(cudaEventSynchronize(r->ev[13]));
  for (int i = 0; i < 7; ++i) REF_CUDA(cudaEventElapsedTime(&out_ms[i], r->ev[2 * i], r->ev[2 * i + 1]));
  return SM_OK;
}
int smref_enable_timings(smref_reconstruction* r, int32_t enable) { r->timings = enable != 0; return SM_OK; }

int smref_dump_state(smref_reconstruction* r, void* stream, float* host_rows, uint64_t host_row_stride_elems,
                     uint32_t* surfels_size, uint32_t* merge_count) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (surfels_size) *surfels_size = r->surfel_count;
  if (merge_count) *merge_count = r->merge_count;
  if (host_rows && r->surfel_count > 0) {
    REF_CUDA(cudaMemcpy2DAsync(host_rows, host_row_stride_elems * sizeof(float), r->surfels.b.address(),
                               r->surfels.b.pitch(), r->surfel_count * sizeof(float), kSurfelAttributeCount,
                               cudaMemcpyDeviceToHost, s));
  }
  REF_CUDA(cudaStreamSynchronize(s));
  return SM_OK;
}

int smref_load_state(smref_reconstruction* r, void* stream, const float* host_rows, uint64_t host_row_stride_elems,
                     uint32_t surfels_size, uint32_t merge_count) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (surfels_size > r->max_surfel_count) return Fail(SM_ERR_CAPACITY, "state larger than surfel cap");
  if (surfels_size > 0) {
    REF_CUDA(cudaMemcpy2DAsync(r->surfels.b.address(), r->surfels.b.pitch(), host_rows,
                               host_row_stride_elems * sizeof(float), surfels_size * sizeof(float),
                               kSurfelAttributeCount, cudaMemcpyHostToDevice, s));
  }
  REF_CUDA(cudaStreamSynchronize(s));
  r->surfel_count = surfels_size;
  r->merge_count = merge_count;
  return SM_OK;
}

int smref_download_rasters(smref_reconstruction* r, void* stream, uint32_t* supporting_surfels,
                           uint32_t* supporting_surfel_counts, float* supporting_surfel_depth_sums,
                           uint32_t* conflicting_surfels, float* first_surfel_depth, uint8_t* new_surfel_flag_vector,
                           uint32_t* new_surfel_indices) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int W = r->width, H = r->height;
#define REF_DL(dst, buf, T)                                                                                  \
  if (dst) REF_CUDA(cudaMemcpy2DAsync(dst, W * sizeof(T), buf.b.address(), buf.b.pitch(), W * sizeof(T), H, \
                                      cudaMemcpyDeviceToHost, s))
  REF_DL(supporting_surfels, r->supporting_surfels, u32);
  REF_DL(supporting_surfel_counts, r->supporting_surfel_counts, u32);
  REF_DL(supporting_surfel_depth_sums, r->supporting_surfel_depth_sums, float);
  REF_DL(conflicting_surfels, r->conflicting_surfels, u32);
  REF_DL(first_surfel_depth, r->first_surfel_depth, float);
#undef REF_DL
  if (new_surfel_flag_vector)
    REF_CUDA(cudaMemcpyAsync(new_surfel_flag_vector, r->new_surfel_flag_vector.b.address(), W * H, cudaMemcpyDeviceToHost, s));
  if (new_surfel_indices)
    REF_CUDA(cudaMemcpyAsync(new_surfel_indices, r->new_surfel_indices.b.address(), W * H * sizeof(u32), cudaMemcpyDeviceToHost, s));
  REF_CUDA(cudaStreamSynchronize(s));
  return SM_OK;
}

// The frame loop of APP/main.cc:885-1223 over a synthetic stream: upload of raw
// depth maps (kept in a ring, :905-968) and of the colour image (:971-984) on an
// upload stream, the five pre-processing launches, Integrate().
int smref_stream_run(smref_reconstruction* r, void* stream_v, const sm_stream_desc* s, const sm_preprocess_params* pp,
                     const sm_integrate_params* ip, int32_t first_frame, int32_t last_frame, sm_stream_stats* stats) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int W = r->width, H = r->height;
  if (s->width != W || s->height != H) return Fail(SM_ERR_INVALID_ARGUMENT, "stream size mismatch");
  const int K = pp->outlier_filtering_frame_count;
  const int half = K / 2;
  if (first_frame < half || last_frame > s->frame_count - half || first_frame > last_frame)
    return Fail(SM_ERR_INVALID_ARGUMENT, "frame range needs K/2 frames on both sides (main.cc:987-992)");
  const size_t depth_frame_elems = static_cast<size_t>(W) * H;
  const unsigned long long launches_before = r->launches;
  uint64_t h2d = 0, d2h = 0;

  if (!r->run_depth_A.b.address()) {
    REF_CUDA(r->run_depth_A.Alloc(H, W));
    REF_CUDA(r->run_normals.Alloc(H, W));
    REF_CUDA(r->run_radius.Alloc(H, W));
  }
  const int ring = K + 2;
  if (s->frames_on_host) {
    if (static_cast<int>(r->run_raw.size()) != ring) {
      for (auto& b : r->run_raw) b.Free();
      for (auto& b : r->run_color) b.Free();
      r->run_raw.assign(ring, PitchedBuffer<u16>());
      r->run_color.assign(2, PitchedBuffer<uchar3>());
      for (auto& b : r->run_raw) REF_CUDA(b.Alloc(H, W));
      for (auto& b : r->run_color) REF_CUDA(b.Alloc(H, W));
      for (auto e : r->upload_events) cudaEventDestroy(e);
      r->upload_events.assign(ring, nullptr);
      for (auto& e : r->upload_events) REF_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
      if (!r->upload_stream) REF_CUDA(cudaStreamCreateWithFlags(&r->upload_stream, cudaStreamNonBlocking));
    }
  }
  // frame_done_event[f % 2] marks the end of frame f's work; ring slots (K + 2 raw
  // depth maps, 2 colour images) written for frame f were last read by frame f - 2.
  cudaEvent_t color_event = nullptr, frame_done_event[2] = {nullptr, nullptr};
  if (s->frames_on_host) {
    REF_CUDA(cudaEventCreateWithFlags(&color_event, cudaEventDisableTiming));
    REF_CUDA(cudaEventCreateWithFlags(&frame_done_event[0], cudaEventDisableTiming));
    REF_CUDA(cudaEventCreateWithFlags(&frame_done_event[1], cudaEventDisableTiming));
  }

  auto raw_view = [&](int frame) -> CUDABuffer_<u16> {
    if (s->frames_on_host) return r->run_raw[frame % ring].b;
    return View<u16>(s->depth + depth_frame_elems * frame, H, W, W * sizeof(u16));
  };
  int uploaded_until = first_frame - half - 1;  // highest frame index already in the ring

  uint32_t integrated = 0;
  for (int frame = first_frame; frame < last_frame; ++frame) {
    CUDABuffer_<uchar3> color_view =
        View<uchar3>(reinterpret_cast<const uchar3*>(s->color + 3 * depth_frame_elems * frame), H, W, W * 3);
    if (s->frames_on_host) {
      if (frame >= first_frame + 2) REF_CUDA(cudaStreamWaitEvent(r->upload_stream, frame_done_event[frame % 2], 0));
      for (int f = uploaded_until + 1; f <= frame + half; ++f) {
        PitchedBuffer<u16>& dst = r->run_raw[f % ring];
        REF_CUDA(cudaMemcpy2DAsync(dst.b.address(), dst.b.pitch(), s->depth + depth_frame_elems * f, W * sizeof(u16),
                                   W * sizeof(u16), H, cudaMemcpyHostToDevice, r->upload_stream));
        h2d += depth_frame_elems * sizeof(u16);
      }
      uploaded_until = frame + half;
      PitchedBuffer<uchar3>& cdst = r->run_color[frame % 2];
      REF_CUDA(cudaMemcpy2DAsync(cdst.b.address(), cdst.b.pitch(), s->color + 3 * depth_frame_elems * frame, W * 3,
                                 W * 3, H, cudaMemcpyHostToDevice, r->upload_stream));
      h2d += depth_frame_elems * 3;
      REF_CUDA(cudaEventRecord(color_event, r->upload_stream));
      REF_CUDA(cudaStreamWaitEvent(stream, color_event, 0));  // main.cc:995
      color_view = cdst.b;
    }

    std::vector<CUDABuffer_<u16>> others(K);
    std::vector<CUDAMatrix3x4> transforms(K);
    for (int i = 0; i < half; ++i) {  // main.cc:1046-1059
      others[i] = raw_view(frame - (i + 1));
      others[half + i] = raw_view(frame + (i + 1));
    }
    for (int i = 0; i < K; ++i) transforms[i] = ToMatrix(s->others_TR_reference + (static_cast<size_t>(frame) * K + i) * 12);

    int status = Preprocess(r, stream, *pp, raw_view(frame), others.data(), transforms.data(), r->run_depth_A.b,
                            r->run_normals.b, r->run_radius.b);
    if (status != SM_OK) return status;
    status = Integrate(r, stream, static_cast<u32>(frame), *ip, r->run_depth_A.b, r->run_normals.b, r->run_radius.b,
                       color_view, ToMatrix(s->global_T_frame + 12 * frame), ToMatrix(s->frame_T_global + 12 * frame));
    if (status != SM_OK) return status;
    d2h += 4 + 4 + 1;  // merge count, last index, last flag
    if (s->frames_on_host) REF_CUDA(cudaEventRecord(frame_done_event[frame % 2], stream));
    ++integrated;
  }
  REF_CUDA(cudaStreamSynchronize(stream));
  if (color_event) cudaEventDestroy(color_event);
  if (frame_done_event[0]) cudaEventDestroy(frame_done_event[0]);
  if (frame_done_event[1]) cudaEventDestroy(frame_done_event[1]);
  if (stats) {
    stats->frames_integrated = integrated;
    stats->surfels_size = r->surfel_count;
    stats->surfel_count = r->surfel_count - r->merge_count;
    stats->kernel_launches = r->launches - launches_before;
    stats->h2d_bytes = h2d;
    stats->d2h_bytes = d2h;
    stats->host_enqueue_ms = 0;
  }
  return SM_OK;
}

}  // extern "C"
