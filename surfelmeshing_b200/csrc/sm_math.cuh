// sm_math.cuh — explicit fp32 arithmetic primitives.
//
// The reference is compiled with -use_fast_math (applications/surfel_meshing/
// CMakeLists.txt:24): ftz, div.approx (= x * MUFU.RCP(y)), sqrt.approx,
// ex2.approx and FMA contraction chosen by nvcc AND by ptxas (non-.rn mul/add
// pairs are fused at SASS level). Threshold tests and u16 roundings amplify a
// single differing ulp into different surfel counts, so the kernels in this
// directory are compiled with -ftz=true -fmad=false and spell every float
// operation out through the helpers below, in the operation order read from
// the reference's compiled SASS (SURVEY.md Appendix B; tools/sass_arith.sh).
// Nothing here is ever contracted or re-associated by the compiler.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace smb {

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }   // FMUL.FTZ
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }   // FADD.FTZ
__device__ __forceinline__ float fsub(float a, float b) { return __fadd_rn(a, -b); }  // FADD.FTZ a, -b
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }  // FFMA.FTZ

// MUFU.RCP / MUFU.SQRT / MUFU.RSQ / MUFU.EX2 (approx, ftz) — bare SFU ops, no fix-up code.
__device__ __forceinline__ float frcp(float a) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
  return r;
}
__device__ __forceinline__ float fsqrt_approx(float a) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
  return r;
}
__device__ __forceinline__ float frsqrt_approx(float a) {
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
  return r;
}
__device__ __forceinline__ float fex2_approx(float a) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(a));
  return r;
}
// a / b under -use_fast_math: FMUL(a, MUFU.RCP(b)).
__device__ __forceinline__ float fdiv_approx(float a, float b) { return fmul(a, frcp(b)); }

__device__ __forceinline__ int f2i_trunc(float a) { return __float2int_rz(a); }            // F2I.FTZ.TRUNC
__device__ __forceinline__ unsigned f2u_trunc(float a) { return __float2uint_rz(a); }      // F2I.FTZ.U32.TRUNC
__device__ __forceinline__ float i2f(int a) { return __int2float_rn(a); }
__device__ __forceinline__ float u2f(unsigned a) { return __uint2float_rn(a); }

// 3x4 rigid transform, rows as float4 (libvis/src/libvis/cuda/cuda_matrix.cuh:67-116).
struct Mat3x4 {
  float4 r0, r1, r2;
};

// One row of CUDAMatrix3x4::operator*: row.x*p.x + row.y*p.y + row.z*p.z + row.w as the
// reference's SASS evaluates it in RenderMinDepth/Associate/Merge/Integrate/UpdateNeighbors
// (SURVEY Appendix B): t = p.y*r.y; t = fma(p.x, r.x, t); t = fma(p.z, r.z, t); t = t + r.w.
__device__ __forceinline__ float transform_row(const float4& r, float px, float py, float pz) {
  float t = fmul(py, r.y);
  t = ffma(px, r.x, t);
  t = ffma(pz, r.z, t);
  return fadd(t, r.w);
}
// CUDAMatrix3x4::Rotate row: same without the translation.
__device__ __forceinline__ float rotate_row(const float4& r, float px, float py, float pz) {
  float t = fmul(py, r.y);
  t = ffma(px, r.x, t);
  return ffma(pz, r.z, t);
}
__device__ __forceinline__ float3 transform_point(const Mat3x4& m, float px, float py, float pz) {
  return make_float3(transform_row(m.r0, px, py, pz), transform_row(m.r1, px, py, pz),
                     transform_row(m.r2, px, py, pz));
}
__device__ __forceinline__ float3 rotate_vec(const Mat3x4& m, float px, float py, float pz) {
  return make_float3(rotate_row(m.r0, px, py, pz), rotate_row(m.r1, px, py, pz), rotate_row(m.r2, px, py, pz));
}

// x*x + y*y + z*z as nvcc contracts it: fma(z, z, fma(x, x, y*y)).
__device__ __forceinline__ float squared_norm(float x, float y, float z) {
  return ffma(z, z, ffma(x, x, fmul(y, y)));
}
// a.x*b.x + a.y*b.y + a.z*b.z: fma(a.z, b.z, fma(a.x, b.x, a.y*b.y)).
__device__ __forceinline__ float dot3(float ax, float ay, float az, float bx, float by, float bz) {
  return ffma(az, bz, ffma(ax, bx, fmul(ay, by)));
}

// Pitched raster access (pitch in bytes), like libvis CUDABuffer_<T>::operator().
template <typename T>
__device__ __forceinline__ T* row_ptr(T* base, size_t pitch, int y) {
  return reinterpret_cast<T*>(reinterpret_cast<char*>(base) + static_cast<size_t>(y) * pitch);
}
template <typename T>
__device__ __forceinline__ const T* row_ptr(const T* base, size_t pitch, int y) {
  return reinterpret_cast<const T*>(reinterpret_cast<const char*>(base) + static_cast<size_t>(y) * pitch);
}

// Ray coordinate of pixel p: ((p + 0.5) - c) / f with IEEE division. sm_render_surfels casts its rays through the
// pixel centres with it, and the tracker back-projects the live and the rendered model depth with the same rays.
__device__ __forceinline__ float ray_coord(int p, float c, float f) { return __fdiv_rn(fsub(fadd(i2f(p), 0.5f), c), f); }

}  // namespace smb
