/* mesh_render_textured_walk.c — plain-C restatement of sm_render_mesh_textured (include/surfel_b200.h, rule T8).
 * TEST INFRASTRUCTURE: the checker of the T8 branch of k_mesh_render_resolve (csrc/render.cu), written from the
 * documented rule. The image is mesh_render_walk.c's (included below, with its triangle helpers); each pixel won by a
 * triangle then has its colour replaced by the atlas lookup, or keeps T7's colour when U or V is not finite. fp32
 * throughout, no contraction (built with -ffp-contract=off), FTZ / DAZ set in MXCSR for the duration of the call to
 * match -ftz=true. Built by tests/mesh_render_textured_walk.py. */
#include "mesh_render_walk.c"

/* T8 channel ch of the bilinear lookup between texels t00, t10 (one row) and t01, t11 (the next), X6's form. */
static u32 bilinear_channel(const u8* t00, const u8* t10, const u8* t01, const u8* t11, int ch, float fx, float fy) {
  const float v00 = (float)t00[ch], v10 = (float)t10[ch], v01 = (float)t01[ch], v11 = (float)t11[ch];
  const float top = v00 + fx * (v10 - v00);
  const float bot = v01 + fx * (v11 - v01);
  const float value = (top + fy * (bot - top)) + 0.5f;
  return value >= 255.f ? 255u : (u32)(int)value;
}

/* T8: the atlas colour of triangle t3 (list order; its uv [6]) at the pixel of T5's q and z; 0 if U or V is not
 * finite. */
static int texture_rgb(const Tri* tr, const u32* t3, const float* uv, const u8* atlas, int aw, int ah,
                       const float q[3], float z, u32* rgb) {
  float cu[3], cv[3];
  for (int k = 0; k < 3; ++k) {
    const int j = t3[0] == tr->s[k] ? 0 : (t3[1] == tr->s[k] ? 1 : 2);
    cu[k] = uv[2 * j];
    cv[k] = uv[2 * j + 1];
  }
  float u = ((q[0] * cu[0] + q[1] * cu[1]) + q[2] * cu[2]) * z;
  float v = ((q[0] * cv[0] + q[1] * cv[1]) + q[2] * cv[2]) * z;
  if (!isfinite(u) || !isfinite(v)) return 0;
  u = u < 0.f ? 0.f : (u > 1.f ? 1.f : u);
  v = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
  const float x = u * (float)aw - 0.5f, y = v * (float)ah - 0.5f;
  const float xf = floorf(x), yf = floorf(y);
  const float fx = x - xf, fy = y - yf;
  const int x0 = (int)xf, y0 = (int)yf;
  const int i0 = x0 < 0 ? 0 : x0, i1 = x0 + 1 > aw - 1 ? aw - 1 : x0 + 1;
  const int j0 = y0 < 0 ? 0 : y0, j1 = y0 + 1 > ah - 1 ? ah - 1 : y0 + 1;
  const u8* r0 = atlas + 3 * (size_t)j0 * aw;
  const u8* r1 = atlas + 3 * (size_t)j1 * aw;
  const u8 *t00 = r0 + 3 * i0, *t10 = r0 + 3 * i1, *t01 = r1 + 3 * i0, *t11 = r1 + 3 * i1;
  *rgb = bilinear_channel(t00, t10, t01, t11, 0, fx, fy) | (bilinear_channel(t00, t10, t01, t11, 1, fx, fy) << 8) |
         (bilinear_channel(t00, t10, t01, t11, 2, fx, fy) << 16);
  return 1;
}

/* mrw_render's arguments, then uv [count][6] and a tightly packed aw x ah u8x3 atlas (may be NULL with count 0),
 * before the outputs. */
void mrtw_render(const float* rows, u64 stride, u32 n, const u32* tris, u64 count, int flags, int width, int height,
                 float fx, float fy, float cx, float cy, float near_depth, float far_depth, const float* T,
                 const float* uv, const u8* atlas, int aw, int ah, float* depth, u8* color, float* normal, u32* index,
                 u64* keys, u64* stats) {
  mrw_render(rows, stride, n, tris, count, flags, width, height, fx, fy, cx, cy, near_depth, far_depth, T, depth, color,
             normal, index, keys, stats);
  if (!atlas) return;
  const unsigned saved_csr = _mm_getcsr();
  _mm_setcsr(saved_csr | 0x8040u); /* FTZ | DAZ; mrw_render restores the caller's MXCSR */
  const size_t P = (size_t)width * height;
  for (size_t k = 0; k < P; ++k) {
    const u32 t = index[k];
    if (t == 0xFFFFFFFFu || (t & DISK_TAG)) continue;
    Tri tr;
    load_tri(rows, stride, n, tris + 3 * (u64)t, T, fx, fy, cx, cy, near_depth, far_depth, &tr);
    float w[3], q[3];
    tri_weights(&tr, (int)(k % width), (int)(k / width), w);
    const float z = tri_depth(&tr, w, q);
    u32 rgb;
    if (!texture_rgb(&tr, tris + 3 * (u64)t, uv + 6 * (u64)t, atlas, aw, ah, q, z, &rgb)) continue;   /* T7's */
    color[3 * k] = rgb & 0xFFu;
    color[3 * k + 1] = (rgb >> 8) & 0xFFu;
    color[3 * k + 2] = (rgb >> 16) & 0xFFu;
  }
  _mm_setcsr(saved_csr);
}
