// texture.cu — sm_mesh_texture (DESIGN.md section 5.15): a texture atlas for a triangle list, one square tile per pair
// of triangles, each texel the visibility-weighted mean of the caller's colour views. The rules X1-X8, step by step,
// are in include/surfel_b200.h.
//
// Launches on the caller's stream:
//   k_tex_classes     one thread per triangle: the input checks (X1) and the tile class (X2) as a sort key
//                     (class << 28 | t), the per-class counts and the clamped count;
//   (CUB radix sort of the keys: the order of X3)
//   k_tex_bases       one thread: each class's first sorted position and first area offset;
//   k_tex_place       one thread per sorted position: the square's Morton origin, a 16-byte tile record, the height;
//   (synchronisation: the input checks and the layout)
//   k_tex_uv          one thread per sorted position: the uv of X4;
//   per view, in array order:
//     sm_render_mesh's kernels: the view's depth (no disks) into the scratch raster;
//     k_tex_accumulate  one thread per texel code of the laid-out area: X5-X6 into its float4 accumulator;
//   k_tex_resolve     one thread per texel code: X7 into the atlas;
//   (synchronisation: the end).
// A texel code m is the Morton code of an atlas texel below the total area: the squares are aligned blocks of codes,
// so m names its class, its square and its texel (i, j) in it without a search, and the accumulators are indexed by m.
//
// sm_mesh_texture_compensated (DESIGN.md section 5.18, rules G1-G6) adds, after k_tex_uv and before the views'
// accumulation (whose k_tex_accumulate<true> scales each sample by the view's gains):
//   per view: sm_render_mesh's depth pass, then k_tex_gain_sample (one thread per sample point: G1-G2 into the
//     view's column of the [V][P] sample matrix);
//   k_tex_gain_count     one thread per point: k_p, n_v (warp-aggregated), and the solver state set to x = d = 1;
//   the data term at x = 1 and r = b - A 1, then per conjugate-gradient step three launches:
//     k_tex_gain_points  one thread per point: m_p of the step's vector;
//     k_tex_gain_views   one 1024-thread block per (1024 points, view): levels 1-2 of G4's column sums;
//     k_tex_gain_step    one 1024-thread block, a thread per view: the rest of the column sums, then the step;
//   then the float gains and the data term at them;
//   (synchronisation: the gain read-back after the end's).
// The launch count depends on view_count and iterations only; the gains never leave the device until the end.

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string>

#include "sm_handle.cuh"
#include "sm_mesh_edges.cuh"

namespace smb {

namespace {

constexpr int kClasses = 7;            // q = 0 .. 6: s = SM_TEXTURE_MAX_TILE >> q = 512 .. 8
constexpr int kMaxTileLog2 = 9;
constexpr u32 kTriangleBits = 28;      // count < 2^28 (kMaxMeshTriangles)
constexpr u32 kTriangleMask = (1u << kTriangleBits) - 1;
static_assert(SM_TEXTURE_MAX_TILE == 1 << kMaxTileLog2, "the classes run from SM_TEXTURE_MAX_TILE down to 8");

}  // namespace

// Class q's sorted positions [start[q], start[q + 1]) and texel codes [base[q], base[q + 1]).
struct TextureLayout {
  u32 start[kClasses + 1];
  u32 pad;
  unsigned long long base[kClasses + 1];
};

struct TextureCounters {
  u32 errors;
  u32 height;
  u32 clamped;
  u32 pad;
  u32 class_count[kClasses + 1];
  TextureLayout layout;
  unsigned long long seen, fallback;
  u32 view_used[SM_TEXTURE_MAX_VIEWS];
};

// The gain fit of sm_mesh_texture_compensated: what the host reads back first, then the solver's device state.
struct GainState {
  float gains[SM_TEXTURE_MAX_VIEWS][3];
  u32 view_samples[SM_TEXTURE_MAX_VIEWS];   // n_v
  double data[2];                           // D at x = 1 and at the float gains
  // (device only from here)
  double x[SM_TEXTURE_MAX_VIEWS][3], r[SM_TEXTURE_MAX_VIEWS][3], d[SM_TEXTURE_MAX_VIEWS][3];
  double rr[3];
  u32 done[3];
};

// The scratch of sm_mesh_texture: per triangle, per texel code and per pixel of the largest view.
struct TextureScratch {
  CounterMirror<TextureCounters> counters;
  u64 triangle_capacity = 0;
  u32* keys = nullptr;            // class << 28 | t, unsorted and sorted
  u32* sorted = nullptr;
  uint4* records = nullptr;       // by sorted position: t, x0, y0, s | half << 16 | a << 17
  void* sort_temp = nullptr; size_t sort_temp_bytes = 0;
  u64 texel_capacity = 0;
  float4* accum = nullptr;        // by texel code: sum of w * (r, g, b), sum of w
  size_t pixel_capacity = 0;
  float* depth = nullptr;         // one view's sm_render_mesh depth
  // sm_mesh_texture_compensated only (G1-G6)
  CounterMirror<GainState> gain;
  u64 sample_capacity = 0;
  float* samples = nullptr;       // [V][P] x (r, g, b), NaN when absent
  u64 point_capacity = 0;
  u32* fit_count = nullptr;       // per point: k_p, 0 when not in the fit
  double* mean = nullptr;         // per point: m_p per channel
  u64 block_capacity = 0;
  double* block_sums = nullptr;   // [V][ceil(P / 1024)] x 3: the level-2 column sums
};

namespace {

struct TextureArgs {
  u32 n;                          // surfels_size()
  const float* radius_squared;    // row 7
  const u32* color;               // row 24
  const float4* smooth;
  const u32* tri;                 // 3 x count
  u32 count;
  float texel_size;
  u32* keys; const u32* sorted; uint4* records;
  float4* accum;
  u32 area;                       // the laid-out area in texels (< 2^32 once the layout fits the atlas)
  float* uv; float atlas_w, atlas_h;
  u8* atlas; size_t atlas_pitch;
  TextureCounters* counters;
};

// One view of the accumulation pass.
struct TextureView {
  Mat3x4 T;
  float fx, fy, cx, cy, near_depth, far_depth;
  int width, height;
  const u8* color; size_t color_pitch;
  const float* depth; size_t depth_pitch;
  float cos_max, tolerance;
  u32* used;
};

__device__ __forceinline__ float3 position(const TextureArgs& a, u32 i) {
  const float4 p = a.smooth[i];
  return make_float3(p.x, p.y, p.z);
}

__device__ __forceinline__ float squared_length(float3 d) { return dot3p(d, d); }

// X1 and X2 for triangle t: the error bits, and otherwise its class q and the list index of corner a.
__device__ u32 classify(const TextureArgs& a, u32 t, int* q_out, int* a_out, bool* clamped) {
  const u32 c[3] = {a.tri[3 * static_cast<size_t>(t)], a.tri[3 * static_cast<size_t>(t) + 1],
                    a.tri[3 * static_cast<size_t>(t) + 2]};
  u32 error = 0;
  for (int k = 0; k < 3; ++k)
    if (c[k] >= a.n || !(a.radius_squared[c[k]] > 0.f)) error |= kBadCorner;
  if (c[0] == c[1] || c[1] == c[2] || c[2] == c[0]) error |= kRepeatedCorner;
  *q_out = kClasses - 1; *a_out = 0; *clamped = false;
  if (error) return error;
  const float3 p0 = position(a, c[0]), p1 = position(a, c[1]), p2 = position(a, c[2]);
  const float e[3] = {squared_length(sub3(p2, p1)), squared_length(sub3(p0, p2)), squared_length(sub3(p1, p0))};
  int k = 0;
  if (e[1] > e[k]) k = 1;
  if (e[2] > e[k]) k = 2;
  const float eb = e[(k + 1) % 3], ec = e[(k + 2) % 3];   // opposite b and c: the legs ac and ab
  const float L = __fsqrt_rn(ec > eb ? ec : eb);
  int s = 8, q = kClasses - 1;
  while (s < SM_TEXTURE_MAX_TILE && !(L <= fmul(u2f(s - 4), a.texel_size))) { s <<= 1; --q; }
  *clamped = !(L <= fmul(u2f(s - 4), a.texel_size));
  *q_out = q;
  *a_out = k;
  return 0;
}

__device__ __forceinline__ u32 compact_bits(unsigned long long v) {   // the even bits of v
  v &= 0x5555555555555555ull;
  v = (v | (v >> 1)) & 0x3333333333333333ull;
  v = (v | (v >> 2)) & 0x0F0F0F0F0F0F0F0Full;
  v = (v | (v >> 4)) & 0x00FF00FF00FF00FFull;
  v = (v | (v >> 8)) & 0x0000FFFF0000FFFFull;
  v = (v | (v >> 16)) & 0x00000000FFFFFFFFull;
  return static_cast<u32>(v);
}

__global__ void __launch_bounds__(kBlock) k_tex_classes(TextureArgs a) {
  __shared__ u32 counts[kClasses];
  __shared__ u32 clamped_count, errors;
  if (threadIdx.x < kClasses) counts[threadIdx.x] = 0;
  if (threadIdx.x == 0) { clamped_count = 0; errors = 0; }
  __syncthreads();
  for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < a.count; t += gridDim.x * blockDim.x) {
    int q, k;
    bool clamped;
    const u32 error = classify(a, t, &q, &k, &clamped);
    if (error) atomicOr(&errors, error);
    if (clamped) atomicAdd(&clamped_count, 1u);
    atomicAdd(&counts[q], 1u);
    a.keys[t] = (static_cast<u32>(q) << kTriangleBits) | t;
  }
  __syncthreads();
  if (threadIdx.x < kClasses && counts[threadIdx.x]) atomicAdd(&a.counters->class_count[threadIdx.x], counts[threadIdx.x]);
  if (threadIdx.x == 0) {
    if (clamped_count) atomicAdd(&a.counters->clamped, clamped_count);
    if (errors) atomicOr(&a.counters->errors, errors);
  }
}

__global__ void k_tex_bases(TextureCounters* c) {
  TextureLayout& l = c->layout;
  l.start[0] = 0;
  l.base[0] = 0;
  for (int q = 0; q < kClasses; ++q) {
    const unsigned long long side = SM_TEXTURE_MAX_TILE >> q;
    l.start[q + 1] = l.start[q] + c->class_count[q];
    l.base[q + 1] = l.base[q] + (c->class_count[q] + 1ull) / 2 * side * side;
  }
}

__global__ void __launch_bounds__(kBlock) k_tex_place(TextureArgs a) {
  const TextureLayout& l = a.counters->layout;
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.count; i += gridDim.x * blockDim.x) {
    const u32 key = a.sorted[i];
    const u32 t = key & kTriangleMask;
    const int q = static_cast<int>(key >> kTriangleBits);
    int q2, k;
    bool clamped;
    classify(a, t, &q2, &k, &clamped);   // the same class (and with an input error nothing is written)
    const u32 s = SM_TEXTURE_MAX_TILE >> q;
    const u32 r = i - l.start[q];
    const unsigned long long o = l.base[q] + static_cast<unsigned long long>(r >> 1) * s * s;
    const u32 x0 = compact_bits(o), y0 = compact_bits(o >> 1);
    a.records[i] = make_uint4(t, x0, y0, s | ((r & 1u) << 16) | (static_cast<u32>(k) << 17));
    if ((r & 1u) == 0) atomicMax(&a.counters->height, y0 + s);
  }
}

// X4: (X, Y) of the corner with role `role` (0 = a, 1 = b, 2 = c) in half `half` of an s x s square.
__device__ __forceinline__ void corner_uv(u32 s, u32 half, int role, u32* X, u32* Y) {
  if (half == 0) {
    *X = role == 1 ? s - 3 : 1;
    *Y = role == 2 ? s - 3 : 1;
  } else {
    *X = role == 1 ? 3 : s - 1;
    *Y = role == 2 ? 3 : s - 1;
  }
}

__global__ void __launch_bounds__(kBlock) k_tex_uv(TextureArgs a) {
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < a.count; i += gridDim.x * blockDim.x) {
    const uint4 rec = a.records[i];
    const u32 s = rec.w & 0xFFFFu, half = (rec.w >> 16) & 1u;
    const int k_a = static_cast<int>(rec.w >> 17);
    float* out = a.uv + 6 * static_cast<size_t>(rec.x);
    for (int k = 0; k < 3; ++k) {
      u32 X, Y;
      corner_uv(s, half, (k - k_a + 3) % 3, &X, &Y);
      out[2 * k] = __fdiv_rn(u2f(rec.y + X), a.atlas_w);
      out[2 * k + 1] = __fdiv_rn(u2f(rec.z + Y), a.atlas_h);
    }
  }
}

// Texel code m -> its tile record and (i, j) in the square; false for a texel of no half.
__device__ __forceinline__ bool texel_at(const TextureArgs& a, const TextureLayout& l, u32 m, uint4* rec, u32* i,
                                         u32* j) {
  int q = 0;
  while (q < kClasses - 1 && m >= l.base[q + 1]) ++q;
  const int shift = 2 * (kMaxTileLog2 - q);
  const u32 s = SM_TEXTURE_MAX_TILE >> q;
  const u32 local = m - static_cast<u32>(l.base[q]);
  const u32 within = local & ((1u << shift) - 1u);
  *i = compact_bits(within);
  *j = compact_bits(within >> 1);
  const u32 pos = l.start[q] + 2 * (local >> shift) + (*i + *j >= s ? 1u : 0u);
  if (pos >= l.start[q + 1]) return false;
  *rec = a.records[pos];
  return true;
}

struct TexelPoint {
  u32 corner[3];      // slots a, b, c
  float alpha, beta;
  float3 X;
  float3 n;
  bool has_normal;
};

// X5's position and normal at (alpha, beta) of the triangle p->corner (a, b, c).
__device__ __forceinline__ void point_on(const TextureArgs& a, float alpha, float beta, TexelPoint* p) {
  p->alpha = alpha;
  p->beta = beta;
  const float3 pa = position(a, p->corner[0]), pb = position(a, p->corner[1]), pc = position(a, p->corner[2]);
  const float3 e1 = sub3(pb, pa), e2 = sub3(pc, pa);
  p->X = make_float3(fadd(fadd(pa.x, fmul(alpha, e1.x)), fmul(beta, e2.x)),
                     fadd(fadd(pa.y, fmul(alpha, e1.y)), fmul(beta, e2.y)),
                     fadd(fadd(pa.z, fmul(alpha, e1.z)), fmul(beta, e2.z)));
  const float3 g = make_float3(fsub(fmul(e1.y, e2.z), fmul(e1.z, e2.y)), fsub(fmul(e1.z, e2.x), fmul(e1.x, e2.z)),
                               fsub(fmul(e1.x, e2.y), fmul(e1.y, e2.x)));
  const float gg = dot3p(g, g);
  p->has_normal = gg > 0.f && isfinite(gg);
  const float inv = p->has_normal ? __fdiv_rn(1.f, __fsqrt_rn(gg)) : 0.f;
  p->n = make_float3(fmul(g.x, inv), fmul(g.y, inv), fmul(g.z, inv));
}

// X5 for texel (i, j) of the tile `rec`.
__device__ __forceinline__ void texel_point(const TextureArgs& a, uint4 rec, u32 i, u32 j, TexelPoint* p) {
  const u32 s = rec.w & 0xFFFFu, half = (rec.w >> 16) & 1u;
  const u32 k_a = rec.w >> 17;
  const u32* tri = a.tri + 3 * static_cast<size_t>(rec.x);
  for (u32 k = 0; k < 3; ++k) p->corner[k] = tri[(k_a + k) % 3];
  const float x = fadd(u2f(i), 0.5f), y = fadd(u2f(j), 0.5f), q = u2f(s - 4);
  float alpha, beta;
  if (half == 0) {
    alpha = __fdiv_rn(fsub(x, 1.f), q);
    beta = __fdiv_rn(fsub(y, 1.f), q);
  } else {
    alpha = __fdiv_rn(fsub(u2f(s - 1), x), q);
    beta = __fdiv_rn(fsub(u2f(s - 1), y), q);
  }
  alpha = alpha > 0.f ? alpha : 0.f;
  beta = beta > 0.f ? beta : 0.f;
  const float sum = fadd(alpha, beta);
  if (sum > 1.f) {
    alpha = __fdiv_rn(alpha, sum);
    beta = fsub(1.f, alpha);
  }
  point_on(a, alpha, beta, p);
}

// X6: one view's weight and colour sample at the texel point; false if the view does not contribute.
__device__ __forceinline__ bool view_sample(const TextureView& v, const TexelPoint& p, float* w, float rgb[3]) {
  if (!p.has_normal) return false;
  const float3 c = transform_point(v.T, p.X.x, p.X.y, p.X.z);
  if (!(v.near_depth <= c.z && c.z <= v.far_depth)) return false;
  const float u = fadd(fmul(v.fx, __fdiv_rn(c.x, c.z)), v.cx), vv = fadd(fmul(v.fy, __fdiv_rn(c.y, c.z)), v.cy);
  const float px = fsub(u, 0.5f), py = fsub(vv, 0.5f);
  if (!(px >= 0.f && px < i2f(v.width - 1) && py >= 0.f && py < i2f(v.height - 1))) return false;
  const float D = row_ptr(v.depth, v.depth_pitch, f2i_trunc(vv))[f2i_trunc(u)];
  if (!(D > 0.f) || !(fabsf(fsub(D, c.z)) <= fmul(v.tolerance, c.z))) return false;
  const float3 m = rotate_vec(v.T, p.n.x, p.n.y, p.n.z);
  const float cos_theta = -__fdiv_rn(dot3p(m, c), __fsqrt_rn(dot3p(c, c)));
  if (!(cos_theta >= v.cos_max)) return false;
  *w = __fdiv_rn(cos_theta, fmul(c.z, c.z));
  const float xf = floorf(px), yf = floorf(py);
  const float fx = fsub(px, xf), fy = fsub(py, yf);
  const int x0 = f2i_trunc(xf), y0 = f2i_trunc(yf);
  const u8* r0 = row_ptr(v.color, v.color_pitch, y0) + 3 * x0;
  const u8* r1 = row_ptr(v.color, v.color_pitch, y0 + 1) + 3 * x0;
  for (int ch = 0; ch < 3; ++ch) {
    const float v00 = u2f(r0[ch]), v10 = u2f(r0[3 + ch]), v01 = u2f(r1[ch]), v11 = u2f(r1[3 + ch]);
    const float top = fadd(v00, fmul(fx, fsub(v10, v00)));
    const float bot = fadd(v01, fmul(fx, fsub(v11, v01)));
    rgb[ch] = fadd(top, fmul(fy, fsub(bot, top)));
  }
  return true;
}

// X6 into the accumulators; with kGain each sample channel is first scaled by the view's gain (G5).
template <bool kGain>
__global__ void __launch_bounds__(kBlock) k_tex_accumulate(TextureArgs a, TextureView v, const float* gain) {
  const TextureLayout& l = a.counters->layout;
  bool any = false;
  for (u32 m = blockIdx.x * blockDim.x + threadIdx.x; m < a.area; m += gridDim.x * blockDim.x) {
    uint4 rec;
    u32 i, j;
    if (!texel_at(a, l, m, &rec, &i, &j)) continue;
    TexelPoint p;
    texel_point(a, rec, i, j, &p);
    float w, rgb[3];
    if (!view_sample(v, p, &w, rgb)) continue;
    if constexpr (kGain) {
      for (int ch = 0; ch < 3; ++ch) rgb[ch] = fmul(gain[ch], rgb[ch]);
    }
    float4 s = a.accum[m];
    s.x = fadd(s.x, fmul(w, rgb[0]));
    s.y = fadd(s.y, fmul(w, rgb[1]));
    s.z = fadd(s.z, fmul(w, rgb[2]));
    s.w = fadd(s.w, w);
    a.accum[m] = s;
    any = true;
  }
  if (__any_sync(0xffffffffu, any) && (threadIdx.x & 31) == 0) *v.used = 1u;
}

__device__ __forceinline__ u32 to_u8(float value) { return value >= 255.f ? 255u : static_cast<u32>(f2i_trunc(value)); }

__global__ void __launch_bounds__(kBlock) k_tex_resolve(TextureArgs a) {
  const TextureLayout& l = a.counters->layout;
  u32 seen = 0, fallback = 0;
  for (u32 m = blockIdx.x * blockDim.x + threadIdx.x; m < a.area; m += gridDim.x * blockDim.x) {
    uint4 rec;
    u32 i, j;
    if (!texel_at(a, l, m, &rec, &i, &j)) continue;
    const float4 s = a.accum[m];
    u32 rgb[3];
    if (s.w > 0.f) {
      ++seen;
      rgb[0] = to_u8(fadd(__fdiv_rn(s.x, s.w), 0.5f));
      rgb[1] = to_u8(fadd(__fdiv_rn(s.y, s.w), 0.5f));
      rgb[2] = to_u8(fadd(__fdiv_rn(s.z, s.w), 0.5f));
    } else {
      ++fallback;
      TexelPoint p;
      texel_point(a, rec, i, j, &p);
      const float wa = fsub(fsub(1.f, p.alpha), p.beta);
      const u32 ca = a.color[p.corner[0]], cb = a.color[p.corner[1]], cc = a.color[p.corner[2]];
      for (int ch = 0; ch < 3; ++ch) {
        const int sh = 8 * ch;
        float sum = fmul(wa, u2f((ca >> sh) & 0xFFu));
        sum = fadd(sum, fmul(p.alpha, u2f((cb >> sh) & 0xFFu)));
        sum = fadd(sum, fmul(p.beta, u2f((cc >> sh) & 0xFFu)));
        rgb[ch] = to_u8(fadd(sum, 0.5f));
      }
    }
    u8* o = row_ptr(a.atlas, a.atlas_pitch, static_cast<int>(compact_bits(m >> 1))) + 3 * static_cast<size_t>(compact_bits(m));
    o[0] = static_cast<u8>(rgb[0]); o[1] = static_cast<u8>(rgb[1]); o[2] = static_cast<u8>(rgb[2]);
  }
  for (int off = 16; off > 0; off >>= 1) {
    seen += __shfl_down_sync(0xffffffffu, seen, off);
    fallback += __shfl_down_sync(0xffffffffu, fallback, off);
  }
  if ((threadIdx.x & 31) == 0) {
    if (seen) atomicAdd(&a.counters->seen, static_cast<unsigned long long>(seen));
    if (fallback) atomicAdd(&a.counters->fallback, static_cast<unsigned long long>(fallback));
  }
}

// ---- the gain fit of sm_mesh_texture_compensated (G1-G6) ----------------------------------------------------------

constexpr int kGainBlock = 1024;   // points per level-2 column sum; also the views of one k_tex_gain_step block
static_assert(SM_TEXTURE_MAX_VIEWS <= kGainBlock, "k_tex_gain_step holds one view per thread");

struct GainArgs {
  float* samples;          // [V][P] x 3
  u32* fit_count;          // [P]
  double* mean;            // [P] x 3
  double* block_sums;      // [V][blocks] x 3
  GainState* state;
  u32 points, views, blocks;
  float min_level, max_level;
  double cN, cG;           // 1 / sigma_noise^2, 1 / sigma_gain^2
};

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dadd_rn(a, -b); }

// TREE of G4 over the 32 lanes: the result in lane 0.
__device__ __forceinline__ double warp_tree(double t) {
  for (int off = 16; off > 0; off >>= 1) t = dadd(t, __shfl_down_sync(0xffffffffu, t, off));
  return t;
}

// G1 and G2: one thread per point writes view `view`'s column of the sample matrix.
__global__ void __launch_bounds__(kBlock) k_tex_gain_sample(TextureArgs a, TextureView v, GainArgs g, u32 view) {
  const float third = 1.f / 3.f;
  for (u32 p = blockIdx.x * blockDim.x + threadIdx.x; p < g.points; p += gridDim.x * blockDim.x) {
    const u64 t = static_cast<u64>(p) * a.count / g.points;
    TexelPoint pt;
    for (int k = 0; k < 3; ++k) pt.corner[k] = a.tri[3 * t + k];
    point_on(a, third, third, &pt);
    float w, rgb[3];
    bool present = view_sample(v, pt, &w, rgb);
    for (int ch = 0; ch < 3; ++ch) present = present && rgb[ch] >= g.min_level && rgb[ch] <= g.max_level;
    float* out = g.samples + 3 * (static_cast<size_t>(view) * g.points + p);
    for (int ch = 0; ch < 3; ++ch) out[ch] = present ? rgb[ch] : __int_as_float(0x7fc00000);
  }
}

// k_p per point (0 below two samples) and n_v per view; block 0 also sets x = d = 1 and clears the solver state.
__global__ void __launch_bounds__(kBlock) k_tex_gain_count(GainArgs g) {
  GainState* s = g.state;
  if (blockIdx.x == 0) {
    for (u32 i = threadIdx.x; i < 3 * SM_TEXTURE_MAX_VIEWS; i += blockDim.x) {
      (&s->x[0][0])[i] = 1.0;
      (&s->d[0][0])[i] = 1.0;
      (&s->r[0][0])[i] = 0.0;
    }
    if (threadIdx.x < 3) { s->rr[threadIdx.x] = 0.0; s->done[threadIdx.x] = 0; }
  }
  const u32 lane = threadIdx.x & 31;
  for (u32 base = blockIdx.x * blockDim.x; base < g.points; base += gridDim.x * blockDim.x) {
    const u32 p = base + threadIdx.x;
    const bool in = p < g.points;
    u32 k = 0;
    for (u32 v = 0; in && v < g.views; ++v) k += isnan(g.samples[3 * (static_cast<size_t>(v) * g.points + p)]) ? 0 : 1;
    const bool fit = k >= 2;
    if (in) g.fit_count[p] = fit ? k : 0;
    if (!__any_sync(0xffffffffu, fit)) continue;
    for (u32 v = 0; v < g.views; ++v) {
      const bool here = fit && !isnan(g.samples[3 * (static_cast<size_t>(v) * g.points + p)]);
      const u32 n = __popc(__ballot_sync(0xffffffffu, here));
      if (lane == 0 && n) atomicAdd(&s->view_samples[v], n);
    }
  }
}

// G4's point sweep: m_p of the vector `x` (x or d of the state) for every point in the fit.
__global__ void __launch_bounds__(kBlock) k_tex_gain_points(GainArgs g, const double* x) {
  for (u32 p = blockIdx.x * blockDim.x + threadIdx.x; p < g.points; p += gridDim.x * blockDim.x) {
    const u32 k = g.fit_count[p];
    if (k == 0) continue;
    double sum[3] = {0.0, 0.0, 0.0};
    for (u32 v = 0; v < g.views; ++v) {
      const float* sp = g.samples + 3 * (static_cast<size_t>(v) * g.points + p);
      const float s0 = sp[0];
      if (isnan(s0)) continue;
      const float sv[3] = {s0, sp[1], sp[2]};
      for (int ch = 0; ch < 3; ++ch) sum[ch] = dadd(sum[ch], dmul(static_cast<double>(sv[ch]), x[3 * v + ch]));
    }
    for (int ch = 0; ch < 3; ++ch) g.mean[3 * static_cast<size_t>(p) + ch] = __ddiv_rn(sum[ch], static_cast<double>(k));
  }
}

// G4's view sweep, levels 1 and 2: block (b, v) sums points [1024 b, 1024 b + 1024) of view v's column, of
// s (s x_v - m_p) (the product A x) or, with kSquares, of (s x_v - m_p)^2 (the data term of G6).
template <bool kSquares>
__global__ void __launch_bounds__(kGainBlock) k_tex_gain_views(GainArgs g, const double* x) {
  __shared__ double warp_sums[32][3];
  const u32 v = blockIdx.y, p = blockIdx.x * kGainBlock + threadIdx.x;
  double t[3] = {0.0, 0.0, 0.0};
  if (p < g.points && g.fit_count[p] != 0) {
    const float* sp = g.samples + 3 * (static_cast<size_t>(v) * g.points + p);
    const float s0 = sp[0];
    if (!isnan(s0)) {
      const float sv[3] = {s0, sp[1], sp[2]};
      for (int ch = 0; ch < 3; ++ch) {
        const double s = sv[ch];
        const double e = dsub(dmul(s, x[3 * v + ch]), g.mean[3 * static_cast<size_t>(p) + ch]);
        t[ch] = kSquares ? dmul(e, e) : dmul(s, e);
      }
    }
  }
  const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int ch = 0; ch < 3; ++ch) t[ch] = warp_tree(t[ch]);
  if (lane == 0) for (int ch = 0; ch < 3; ++ch) warp_sums[warp][ch] = t[ch];
  __syncthreads();
  if (warp == 0) {
    for (int ch = 0; ch < 3; ++ch) {
      const double b = warp_tree(warp_sums[lane][ch]);
      if (lane == 0) g.block_sums[3 * (static_cast<size_t>(v) * g.blocks + blockIdx.x) + ch] = b;
    }
  }
}

// The sum over views of G4 (0 past view_count) for the three channels, in every thread of the block.
__device__ __forceinline__ void views_tree(double t[3], double (*warp_sums)[3], double out[3]) {
  const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int ch = 0; ch < 3; ++ch) t[ch] = warp_tree(t[ch]);
  __syncthreads();   // (warp_sums may still be read from the previous call)
  if (lane == 0) for (int ch = 0; ch < 3; ++ch) warp_sums[warp][ch] = t[ch];
  __syncthreads();
  if (warp == 0)
    for (int ch = 0; ch < 3; ++ch) {
      const double s = warp_tree(warp_sums[lane][ch]);
      if (lane == 0) warp_sums[32][ch] = s;
    }
  __syncthreads();
  for (int ch = 0; ch < 3; ++ch) out[ch] = warp_sums[32][ch];
}

enum GainStep : int { kStepData0 = 0, kStepData1 = 1, kStepInit, kStepIterate, kStepFinish };

// One block of kGainBlock threads, thread v = view v: the rest of the column sums (levels 3 and up, one warp per
// view), then by `mode`: the data term D (into data[mode]), r = b - A x with d = r, one CG step, or the float gains
// with d = the gains (for the data term at the fitted gains).
__global__ void __launch_bounds__(kGainBlock) k_tex_gain_step(GainArgs g, int mode) {
  __shared__ double column[SM_TEXTURE_MAX_VIEWS][3];
  __shared__ double warp_sums[33][3];
  GainState* s = g.state;
  const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5, v = threadIdx.x;
  if (mode != kStepFinish) {
    for (u32 view = warp; view < g.views; view += kGainBlock / 32) {
      double* b = g.block_sums + 3 * static_cast<size_t>(view) * g.blocks;
      for (u32 n = g.blocks; n > 1; n = (n + 31) / 32) {
        for (u32 group = 0; 32 * group < n; ++group) {
          const u32 i = 32 * group + lane;
          for (int ch = 0; ch < 3; ++ch) {
            const double t = warp_tree(i < n ? b[3 * i + ch] : 0.0);
            __syncwarp();
            if (lane == 0) b[3 * group + ch] = t;
            __syncwarp();
          }
        }
      }
      if (lane == 0) for (int ch = 0; ch < 3; ++ch) column[view][ch] = b[ch];
    }
    __syncthreads();
  }
  const bool is_view = v < g.views;
  if (mode == kStepData0 || mode == kStepData1) {
    double t[3], D[3];
    for (int ch = 0; ch < 3; ++ch) t[ch] = is_view ? column[v][ch] : 0.0;
    views_tree(t, warp_sums, D);
    if (threadIdx.x == 0) s->data[mode] = dadd(dadd(D[0], D[1]), D[2]);
    return;
  }
  if (mode == kStepFinish) {   // the common scale: x over its n_v-weighted mean
    const double n = is_view ? static_cast<double>(s->view_samples[v]) : 0.0;
    double t[3], weighted[3], total[3];
    for (int ch = 0; ch < 3; ++ch) t[ch] = is_view ? dmul(n, s->x[v][ch]) : 0.0;
    views_tree(t, warp_sums, weighted);
    for (int ch = 0; ch < 3; ++ch) t[ch] = n;
    views_tree(t, warp_sums, total);
    if (is_view)
      for (int ch = 0; ch < 3; ++ch) {
        double mean = total[ch] > 0.0 ? __ddiv_rn(weighted[ch], total[ch]) : 1.0;
        if (!(mean > 0.0)) mean = 1.0;
        const float gain = n > 0.0 ? __double2float_rn(__ddiv_rn(s->x[v][ch], mean)) : 1.f;
        s->gains[v][ch] = gain;
        s->d[v][ch] = gain;
      }
    return;
  }
  const double nG = is_view ? dmul(static_cast<double>(s->view_samples[v]), g.cG) : 0.0;
  double Ad[3];
  for (int ch = 0; ch < 3; ++ch) Ad[ch] = is_view ? dadd(dmul(column[v][ch], g.cN), dmul(nG, s->d[v][ch])) : 0.0;
  if (mode == kStepInit) {
    double t[3], rr[3];
    for (int ch = 0; ch < 3; ++ch) {
      const double r = is_view ? dsub(nG, Ad[ch]) : 0.0;
      if (is_view) { s->r[v][ch] = r; s->d[v][ch] = r; }
      t[ch] = dmul(r, r);
    }
    views_tree(t, warp_sums, rr);
    if (threadIdx.x == 0)
      for (int ch = 0; ch < 3; ++ch) { s->rr[ch] = rr[ch]; s->done[ch] = !(rr[ch] != 0.0); }
    return;
  }
  // kStepIterate
  bool active[3];
  double rr[3], t[3], pAp[3], alpha[3];
  for (int ch = 0; ch < 3; ++ch) {
    rr[ch] = s->rr[ch];
    active[ch] = s->done[ch] == 0;
    t[ch] = is_view ? dmul(s->d[v][ch], Ad[ch]) : 0.0;
  }
  views_tree(t, warp_sums, pAp);
  for (int ch = 0; ch < 3; ++ch) {
    active[ch] = active[ch] && pAp[ch] > 0.0;
    alpha[ch] = active[ch] ? __ddiv_rn(rr[ch], pAp[ch]) : 0.0;
    double r = 0.0;
    if (is_view) {
      r = s->r[v][ch];
      if (active[ch]) {
        s->x[v][ch] = dadd(s->x[v][ch], dmul(alpha[ch], s->d[v][ch]));
        r = dsub(r, dmul(alpha[ch], Ad[ch]));
        s->r[v][ch] = r;
      }
    }
    t[ch] = dmul(r, r);
  }
  double rr_new[3];
  views_tree(t, warp_sums, rr_new);
  for (int ch = 0; ch < 3; ++ch) {
    if (!active[ch]) continue;
    const double beta = __ddiv_rn(rr_new[ch], rr[ch]);
    if (is_view) s->d[v][ch] = dadd(s->r[v][ch], dmul(beta, s->d[v][ch]));
  }
  __syncthreads();   // every thread has read rr and done
  if (threadIdx.x == 0)
    for (int ch = 0; ch < 3; ++ch) {
      if (active[ch]) s->rr[ch] = rr_new[ch];
      s->done[ch] = !active[ch] || !(rr_new[ch] != 0.0);
    }
}

void FreeTriangleScratch(TextureScratch& s) {
  FreeAndClear(s.keys, s.sorted, s.records, s.sort_temp);
  s.sort_temp_bytes = 0;
  s.triangle_capacity = 0;
}

// Per-triangle scratch for `count` triangles (x 1.5 when it grows).
int EnsureTriangleScratch(TextureScratch& s, u64 count) {
  if (count <= s.triangle_capacity) return SM_OK;
  const u64 cap = GrownCapacity(count);
  FreeTriangleScratch(s);
  size_t temp = 0;
  SM_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, temp, static_cast<const u32*>(nullptr), static_cast<u32*>(nullptr),
                                         static_cast<int>(cap)));
  SM_CUDA(cudaMalloc(&s.keys, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.sorted, sizeof(u32) * cap));
  SM_CUDA(cudaMalloc(&s.records, sizeof(uint4) * cap));
  SM_CUDA(cudaMalloc(&s.sort_temp, temp));
  s.sort_temp_bytes = temp;
  s.triangle_capacity = cap;
  return SM_OK;
}

void FreeTexelScratch(TextureScratch& s) {
  FreeAndClear(s.accum);
  s.texel_capacity = 0;
}

int EnsureTexelScratch(TextureScratch& s, u64 texels) {
  if (texels <= s.texel_capacity) return SM_OK;
  const u64 cap = GrownCapacity(texels, 1 << 16);
  FreeTexelScratch(s);
  SM_CUDA(cudaMalloc(&s.accum, sizeof(float4) * cap));
  s.texel_capacity = cap;
  return SM_OK;
}

void FreePixelScratch(TextureScratch& s) {
  FreeAndClear(s.depth);
  s.pixel_capacity = 0;
}

int EnsurePixelScratch(TextureScratch& s, size_t pixels) {
  if (pixels <= s.pixel_capacity) return SM_OK;
  FreePixelScratch(s);
  SM_CUDA(cudaMalloc(&s.depth, sizeof(float) * pixels));
  s.pixel_capacity = pixels;
  return SM_OK;
}

void FreeGainScratch(TextureScratch& s) {
  FreeAndClear(s.samples, s.fit_count, s.mean, s.block_sums);
  s.sample_capacity = s.point_capacity = s.block_capacity = 0;
}

// The sample matrix (P x V entries), the per-point vectors (P) and the level-2 column sums (V x blocks), each group
// grown by x 1.5 when it does not fit; the solver state once.
int EnsureGainScratch(TextureScratch& s, u64 entries, u64 points, u64 block_sums) {
  if (!s.gain.device) {
    const int status = CreateCounters(s.gain);
    if (status != SM_OK) return status;
  }
  if (entries > s.sample_capacity) {
    const u64 cap = GrownCapacity(entries, 1 << 16);
    FreeAndClear(s.samples);
    s.sample_capacity = 0;
    SM_CUDA(cudaMalloc(&s.samples, 3 * sizeof(float) * cap));
    s.sample_capacity = cap;
  }
  if (points > s.point_capacity) {
    const u64 cap = GrownCapacity(points);
    FreeAndClear(s.fit_count, s.mean);
    s.point_capacity = 0;
    SM_CUDA(cudaMalloc(&s.fit_count, sizeof(u32) * cap));
    SM_CUDA(cudaMalloc(&s.mean, 3 * sizeof(double) * cap));
    s.point_capacity = cap;
  }
  if (block_sums > s.block_capacity) {
    const u64 cap = GrownCapacity(block_sums);
    FreeAndClear(s.block_sums);
    s.block_capacity = 0;
    SM_CUDA(cudaMalloc(&s.block_sums, 3 * sizeof(double) * cap));
    s.block_capacity = cap;
  }
  return SM_OK;
}

}  // namespace

void FreeTextureBuffers(sm_reconstruction* r) {
  TextureScratch* s = r->texture;
  if (!s) return;
  FreeTriangleScratch(*s);
  FreeTexelScratch(*s);
  FreePixelScratch(*s);
  FreeGainScratch(*s);
  FreeCounters(s->counters);
  FreeCounters(s->gain);
  delete s;
  r->texture = nullptr;
}

namespace {

// sm_mesh_texture, and with `gp` set sm_mesh_texture_compensated; `who` names the call in its messages.
int Texture(const char* who, sm_reconstruction* r, void* stream_v, const sm_texture_params* params,
            const sm_texture_gain_params* gp, const uint32_t* triangles, uint64_t count, const sm_texture_view* views,
            int32_t view_count, uint8_t* atlas, size_t atlas_pitch, int32_t atlas_capacity_width,
            int32_t atlas_capacity_height, float* uv, float* gains, sm_texture_stats* stats,
            sm_texture_gain_stats* gain_stats) {
  const std::string prefix = std::string(who) + ": ";
  auto bad = [&prefix](const char* why) { return SetError(SM_ERR_INVALID_ARGUMENT, (prefix + why).c_str()); };
  if (!r || !params || !stats) return bad("null argument");
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const sm_texture_params& p = *params;
  *stats = sm_texture_stats{};
  if (gp) {
    if (!gain_stats) return bad("null argument");
    *gain_stats = sm_texture_gain_stats{};
    if (gp->max_samples < 0) return bad("max_samples must be >= 0");
    if (gp->iterations < 0) return bad("iterations must be >= 0");
    if (!std::isfinite(gp->sigma_noise) || !(gp->sigma_noise > 0.f)) return bad("sigma_noise must be finite and > 0");
    if (!std::isfinite(gp->sigma_gain) || !(gp->sigma_gain > 0.f)) return bad("sigma_gain must be finite and > 0");
    if (!std::isfinite(gp->min_level) || !std::isfinite(gp->max_level) || gp->min_level > gp->max_level)
      return bad("min_level and max_level must be finite with min_level <= max_level");
  }
  if (!std::isfinite(p.texel_size) || !(p.texel_size > 0.f)) return bad("texel_size must be finite and > 0");
  if (p.max_atlas_side < 8 || p.max_atlas_side > SM_TEXTURE_MAX_ATLAS_SIDE)
    return bad("max_atlas_side must be in [8, SM_TEXTURE_MAX_ATLAS_SIDE]");
  if (!(p.max_view_angle_deg > 0.f && p.max_view_angle_deg <= 90.f)) return bad("max_view_angle_deg must be in (0, 90]");
  if (!(p.depth_tolerance >= 0.f) || !std::isfinite(p.depth_tolerance)) return bad("depth_tolerance must be finite and >= 0");
  if (const char* why = TriangleListError(triangles, count)) return bad(why);
  if (view_count < 0 || view_count > SM_TEXTURE_MAX_VIEWS) return bad("view_count must be in [0, SM_TEXTURE_MAX_VIEWS]");
  if (!views && view_count > 0) return bad("views is NULL with a view_count > 0");
  size_t max_pixels = 1;
  for (int32_t k = 0; k < view_count; ++k) {
    const sm_texture_view& v = views[k];
    if (const char* why = RenderCameraError(v.camera, v.view_T_global))
      return bad((std::string("view ") + std::to_string(k) + ": " + why).c_str());
    if (!v.color) return bad((std::string("view ") + std::to_string(k) + ": color is NULL").c_str());
    if (v.color_pitch < 3 * static_cast<size_t>(v.camera.width))
      return bad((std::string("view ") + std::to_string(k) + ": color_pitch is below 3 x width").c_str());
    max_pixels = std::max(max_pixels, static_cast<size_t>(v.camera.width) * static_cast<size_t>(v.camera.height));
  }
  if (atlas_capacity_width < 0 || atlas_capacity_height < 0) return bad("the atlas capacity must be >= 0");
  const bool has_capacity = atlas_capacity_width > 0 || atlas_capacity_height > 0;
  if (!atlas && has_capacity) return bad("atlas is NULL with a capacity that is not 0 x 0");
  if (atlas && atlas_pitch < 3 * static_cast<size_t>(atlas_capacity_width)) return bad("atlas_pitch is below 3 x the capacity width");
  if (uv && count > 0) {
    if (Overlap(uv, 24 * count, triangles, 12 * count)) return bad("uv overlaps triangles");
    if (atlas && atlas_capacity_width > 0 && atlas_capacity_height > 0 &&
        Overlap(uv, 24 * count, atlas, atlas_pitch * (atlas_capacity_height - 1) + 3 * static_cast<u64>(atlas_capacity_width)))
      return bad("uv overlaps the atlas");
  }
  r->last_stream = stream;
  int status = FetchCounters(r, stream);
  if (status == SM_ERR_CUDA) return status;   // (a surfel-cap overflow of an earlier frame does not matter here)
  if (count == 0) {                           // a 0 x 0 atlas: nothing to write
    if (gains) std::fill(gains, gains + 3 * static_cast<size_t>(view_count), 1.f);
    return SM_OK;
  }
  const u32 n = r->host_counters->surfel_count[r->count_slot];

  if (!r->texture) {   // published only with its counters, so a failed first call is retried whole
    CounterMirror<TextureCounters> counters;
    status = CreateCounters(counters);
    if (status != SM_OK) return status;
    r->texture = new TextureScratch();
    r->texture->counters = counters;
  }
  TextureScratch& s = *r->texture;
  status = EnsureTriangleScratch(s, count);
  if (status != SM_OK) return status;

  TextureArgs a{};
  a.n = n;
  a.radius_squared = r->d.surfels + static_cast<size_t>(SM_ROW_RADIUS_SQUARED) * r->d.stride;
  a.color = reinterpret_cast<const u32*>(r->d.surfels) + static_cast<size_t>(SM_ROW_COLOR) * r->d.stride;
  a.smooth = r->d.smooth;
  a.tri = triangles;
  a.count = static_cast<u32>(count);
  a.texel_size = p.texel_size;
  a.keys = s.keys; a.sorted = s.sorted; a.records = s.records;
  a.counters = s.counters.device;
  TextureCounters* c = s.counters.device;
  const TextureCounters& h = *s.counters.host;
  const int grid = Grid(count, r->sm_count);
  SM_CUDA(cudaMemsetAsync(c, 0, sizeof(TextureCounters), stream));
  { LaunchScope scope(stream, KID_TEXTURE_CLASSES); LaunchKernel(k_tex_classes, dim3(grid), dim3(kBlock), 0, stream, a); }
  {
    LaunchScope scope(stream, KID_TEXTURE_SORT);
    size_t temp = s.sort_temp_bytes;
    SM_CUDA(cub::DeviceRadixSort::SortKeys(s.sort_temp, temp, static_cast<const u32*>(s.keys), s.sorted,
                                           static_cast<int>(count), 0, 31, stream));
  }
  { LaunchScope scope(stream, KID_TEXTURE_PLACE); LaunchKernel(k_tex_bases, dim3(1), dim3(1), 0, stream, c); }
  { LaunchScope scope(stream, KID_TEXTURE_PLACE); LaunchKernel(k_tex_place, dim3(grid), dim3(kBlock), 0, stream, a); }
  status = ReadCounters(s.counters, stream, offsetof(TextureCounters, seen));
  if (status != SM_OK) return status;
  if (const char* why = MeshInputError(h.errors)) return bad(why);

  const u64 area = h.layout.base[kClasses];
  u64 width = 1, texels = 0;
  while (width * width < area) width <<= 1;
  for (int q = 0; q < kClasses; ++q) {
    const u64 side = SM_TEXTURE_MAX_TILE >> q, k = h.class_count[q];
    texels += (k + 1) / 2 * (side * (side + 1) / 2) + k / 2 * (side * (side - 1) / 2);
  }
  stats->triangles = count;
  stats->atlas_width = static_cast<int32_t>(std::min<u64>(width, INT32_MAX));
  stats->atlas_height = static_cast<int32_t>(h.height);
  stats->texels = texels;
  stats->tiles_clamped = h.clamped;
  const u64 height = h.height;
  if (width > static_cast<u64>(p.max_atlas_side))
    return SetError(SM_ERR_CAPACITY, (prefix + "the atlas needs a side of " + std::to_string(width) +
                                      " texels, above max_atlas_side " + std::to_string(p.max_atlas_side) +
                                      "; raise texel_size").c_str());
  if (width > static_cast<u64>(atlas_capacity_width) || height > static_cast<u64>(atlas_capacity_height))
    return SetError(SM_ERR_CAPACITY, (prefix + "a " + std::to_string(width) + " x " + std::to_string(height) +
                                      " atlas does not fit the capacity of " + std::to_string(atlas_capacity_width) +
                                      " x " + std::to_string(atlas_capacity_height)).c_str());
  // From here on a failure leaves the stats zero.
  const sm_texture_stats layout = *stats;
  *stats = sm_texture_stats{};
  status = EnsureTexelScratch(s, area);
  if (status == SM_OK) status = EnsurePixelScratch(s, max_pixels);
  if (status != SM_OK) return status;
  // G1: the sample points
  const u64 points = gp && view_count > 0 ? std::min<u64>(count, static_cast<u64>(gp->max_samples) / view_count) : 0;
  const u64 blocks = (points + kGainBlock - 1) / kGainBlock;
  if (points > 0) {
    status = EnsureGainScratch(s, points * view_count, points, blocks * view_count);
    if (status != SM_OK) return status;
  }

  a.accum = s.accum;
  a.area = static_cast<u32>(area);   // width <= SM_TEXTURE_MAX_ATLAS_SIDE: area <= 2^30
  a.uv = uv;
  a.atlas_w = static_cast<float>(width);
  a.atlas_h = static_cast<float>(height);
  a.atlas = atlas;
  a.atlas_pitch = atlas_pitch;
  SM_CUDA(cudaMemset2DAsync(atlas, atlas_pitch, 0, 3 * width, height, stream));
  SM_CUDA(cudaMemsetAsync(s.accum, 0, sizeof(float4) * area, stream));
  if (uv) { LaunchScope scope(stream, KID_TEXTURE_UV); LaunchKernel(k_tex_uv, dim3(grid), dim3(kBlock), 0, stream, a); }
  const int texel_grid = Grid(area, r->sm_count);
  const float cos_max = CosDegrees(p.max_view_angle_deg);
  // View k's depth into the scratch raster, and its description for the kernels.
  auto render_view = [&](int32_t k, TextureView* v) {
    const sm_texture_view& view = views[k];
    const sm_render_params& cam = view.camera;
    const size_t depth_pitch = sizeof(float) * static_cast<size_t>(cam.width);
    v->T = MakeMat3x4(view.view_T_global);
    v->fx = cam.fx; v->fy = cam.fy; v->cx = cam.cx; v->cy = cam.cy;
    v->near_depth = cam.near_depth; v->far_depth = cam.far_depth;
    v->width = cam.width; v->height = cam.height;
    v->color = view.color; v->color_pitch = view.color_pitch;
    v->depth = s.depth; v->depth_pitch = depth_pitch;
    v->cos_max = cos_max;
    v->tolerance = p.depth_tolerance;
    v->used = c->view_used + k;
    return RenderMesh(r, stream, cam, view.view_T_global, triangles, count, 0, s.depth, depth_pitch, nullptr, 0,
                      nullptr, 0, nullptr, 0);
  };
  GainState* gs = s.gain.device;
  if (points > 0) {   // G2-G4 and the data terms of G6, all on `stream`
    GainArgs g{};
    g.samples = s.samples; g.fit_count = s.fit_count; g.mean = s.mean; g.block_sums = s.block_sums;
    g.state = gs;
    g.points = static_cast<u32>(points);   // points * view_count <= INT32_MAX
    g.views = static_cast<u32>(view_count);
    g.blocks = static_cast<u32>(blocks);
    g.min_level = gp->min_level; g.max_level = gp->max_level;
    const double sn = gp->sigma_noise, sg = gp->sigma_gain;
    g.cN = 1.0 / (sn * sn);
    g.cG = 1.0 / (sg * sg);
    const int point_grid = Grid(points, r->sm_count);
    const dim3 view_grid(static_cast<u32>(blocks), static_cast<u32>(view_count));
    SM_CUDA(cudaMemsetAsync(gs, 0, offsetof(GainState, x), stream));
    for (int32_t k = 0; k < view_count; ++k) {
      TextureView v;
      status = render_view(k, &v);
      if (status != SM_OK) return status;
      LaunchScope scope(stream, KID_TEXTURE_GAIN_SAMPLE);
      LaunchKernel(k_tex_gain_sample, dim3(point_grid), dim3(kBlock), 0, stream, a, v, g, static_cast<u32>(k));
    }
    { LaunchScope scope(stream, KID_TEXTURE_GAIN_COUNT); LaunchKernel(k_tex_gain_count, dim3(point_grid), dim3(kBlock), 0, stream, g); }
    auto sweep = [&](const double* x, bool squares, int mode) {
      if (x) { LaunchScope scope(stream, KID_TEXTURE_GAIN_POINTS); LaunchKernel(k_tex_gain_points, dim3(point_grid), dim3(kBlock), 0, stream, g, x); }
      {
        LaunchScope scope(stream, KID_TEXTURE_GAIN_VIEWS);
        const double* xv = x ? x : &gs->x[0][0];
        if (squares) LaunchKernel(k_tex_gain_views<true>, view_grid, dim3(kGainBlock), 0, stream, g, xv);
        else LaunchKernel(k_tex_gain_views<false>, view_grid, dim3(kGainBlock), 0, stream, g, xv);
      }
      LaunchScope scope(stream, KID_TEXTURE_GAIN_STEP);
      LaunchKernel(k_tex_gain_step, dim3(1), dim3(kGainBlock), 0, stream, g, mode);
    };
    sweep(&gs->x[0][0], true, kStepData0);   // D at x = 1
    sweep(nullptr, false, kStepInit);       // r = b - A 1 (the same m_p)
    for (int32_t it = 0; it < gp->iterations; ++it) sweep(&gs->d[0][0], false, kStepIterate);
    { LaunchScope scope(stream, KID_TEXTURE_GAIN_STEP); LaunchKernel(k_tex_gain_step, dim3(1), dim3(kGainBlock), 0, stream, g, static_cast<int>(kStepFinish)); }
    sweep(&gs->d[0][0], true, kStepData1);   // D at the float gains
  }
  for (int32_t k = 0; k < view_count; ++k) {
    TextureView v;
    status = render_view(k, &v);
    if (status != SM_OK) return status;
    LaunchScope scope(stream, KID_TEXTURE_ACCUMULATE);
    if (points > 0) LaunchKernel(k_tex_accumulate<true>, dim3(texel_grid), dim3(kBlock), 0, stream, a, v, &gs->gains[k][0]);
    else LaunchKernel(k_tex_accumulate<false>, dim3(texel_grid), dim3(kBlock), 0, stream, a, v, static_cast<const float*>(nullptr));
  }
  { LaunchScope scope(stream, KID_TEXTURE_RESOLVE); LaunchKernel(k_tex_resolve, dim3(texel_grid), dim3(kBlock), 0, stream, a); }
  status = ReadCounters(s.counters, stream);
  if (status == SM_OK && points > 0) status = ReadCounters(s.gain, stream, offsetof(GainState, x));
  if (status != SM_OK) return status;
  *stats = layout;
  stats->texels_seen = h.seen;
  stats->texels_fallback = h.fallback;
  for (int32_t k = 0; k < view_count; ++k) stats->views_used += h.view_used[k] ? 1 : 0;
  if (gp) {
    const GainState& hg = *s.gain.host;
    sm_texture_gain_stats out{};
    out.points = points;
    for (int32_t k = 0; points > 0 && k < view_count; ++k) {
      out.samples += hg.view_samples[k];
      out.views_fitted += hg.view_samples[k] ? 1 : 0;
    }
    if (out.samples > 0) {
      const double scale = 3.0 * static_cast<double>(out.samples);
      out.rms_before = std::sqrt(hg.data[0] / scale);
      out.rms_after = std::sqrt(hg.data[1] / scale);
    }
    *gain_stats = out;
    if (gains)
      for (int32_t k = 0; k < view_count; ++k)
        for (int ch = 0; ch < 3; ++ch) gains[3 * k + ch] = points > 0 ? hg.gains[k][ch] : 1.f;
  }
  return CheckLaunch("texture");
}

}  // namespace

}  // namespace smb

using namespace smb;

extern "C" {

void sm_default_texture_params(sm_texture_params* p) {
  p->texel_size = 0.004f;
  p->max_atlas_side = 16384;
  p->max_view_angle_deg = 75.0f;
  p->depth_tolerance = 0.01f;
}

void sm_default_texture_gain_params(sm_texture_gain_params* p) {
  p->max_samples = 1 << 23;
  p->iterations = 32;
  p->sigma_noise = 10.0f;
  p->sigma_gain = 1.0f;
  p->min_level = 5.0f;
  p->max_level = 250.0f;
}

int sm_mesh_texture(sm_reconstruction* r, void* stream, const sm_texture_params* params, const uint32_t* triangles,
                    uint64_t count, const sm_texture_view* views, int32_t view_count, uint8_t* atlas,
                    size_t atlas_pitch, int32_t atlas_capacity_width, int32_t atlas_capacity_height, float* uv,
                    sm_texture_stats* stats) {
  return Texture("sm_mesh_texture", r, stream, params, nullptr, triangles, count, views, view_count, atlas,
                 atlas_pitch, atlas_capacity_width, atlas_capacity_height, uv, nullptr, stats, nullptr);
}

int sm_mesh_texture_compensated(sm_reconstruction* r, void* stream, const sm_texture_params* params,
                                const sm_texture_gain_params* gp, const uint32_t* triangles, uint64_t count,
                                const sm_texture_view* views, int32_t view_count, uint8_t* atlas, size_t atlas_pitch,
                                int32_t atlas_capacity_width, int32_t atlas_capacity_height, float* uv, float* gains,
                                sm_texture_stats* stats, sm_texture_gain_stats* gain_stats) {
  if (!gp) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_mesh_texture_compensated: null argument");
  return Texture("sm_mesh_texture_compensated", r, stream, params, gp, triangles, count, views, view_count, atlas,
                 atlas_pitch, atlas_capacity_width, atlas_capacity_height, uv, gains, stats, gain_stats);
}

}  // extern "C"
