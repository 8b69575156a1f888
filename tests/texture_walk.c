/* texture_walk.c — plain-C restatement of sm_mesh_texture (include/surfel_b200.h, "texturing a triangle mesh", rules
 * X1-X8). TEST INFRASTRUCTURE: the checker of the k_tex_* kernels (csrc/texture.cu), written from the documented
 * rules, sequentially: the layout by a counting sort over the classes, then every tile's texels with the views in
 * array order. fp32 throughout, no contraction (built with -ffp-contract=off), fmaf where rule 1 of
 * sm_render_surfels uses an FMA, and FTZ / DAZ set in MXCSR for the duration of the call to match -ftz=true. The
 * visibility depth of each view comes from mesh_render_walk.c, the restatement of sm_render_mesh (included below).
 * Built by tests/texture_walk.py. */
#include "mesh_render_walk.c"

enum { MAX_TILE = 512, CLASSES = 7 };

static float sqlen(const float d[3]) { return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]; }

static void pos(const float* rows, u64 stride, u32 i, float p[3]) {
  for (int k = 0; k < 3; ++k) p[k] = rows[(size_t)(ROW_SMOOTH_X + k) * stride + i];
}

static u32 compact_bits(u64 v) {
  u32 out = 0;
  for (int b = 0; b < 32; ++b) out |= (u32)((v >> (2 * b)) & 1u) << b;
  return out;
}

/* X1 / X2: error bits, else the class q (s = 512 >> q), the list index of a and the clamp flag. */
static u32 classify(const float* rows, u64 stride, u32 n, const u32* c, float texel, int* q_out, int* a_out,
                    int* clamped) {
  u32 error = 0;
  for (int k = 0; k < 3; ++k)
    if (c[k] >= n || !(rows[(size_t)ROW_RADIUS_SQUARED * stride + c[k]] > 0.f)) error |= 1;
  if (c[0] == c[1] || c[1] == c[2] || c[2] == c[0]) error |= 2;
  *q_out = CLASSES - 1; *a_out = 0; *clamped = 0;
  if (error) return error;
  float p[3][3], d[3], e[3];
  for (int k = 0; k < 3; ++k) pos(rows, stride, c[k], p[k]);
  for (int k = 0; k < 3; ++k) {
    const float* from = p[(k + 1) % 3];
    const float* to = p[(k + 2) % 3];
    for (int x = 0; x < 3; ++x) d[x] = to[x] - from[x];
    e[k] = sqlen(d);
  }
  int a = 0;
  if (e[1] > e[a]) a = 1;
  if (e[2] > e[a]) a = 2;
  const float eb = e[(a + 1) % 3], ec = e[(a + 2) % 3];
  const float L = sqrtf(ec > eb ? ec : eb);
  int s = 8, q = CLASSES - 1;
  while (s < MAX_TILE && !(L <= (float)(s - 4) * texel)) { s <<= 1; --q; }
  *clamped = !(L <= (float)(s - 4) * texel);
  *q_out = q;
  *a_out = a;
  return 0;
}

static u32 to_u8(float v) { return v >= 255.f ? 255u : (u32)(int)v; }

/* rows: [25][stride] float32 (rows 3-5 = the smooth positions), slots [0, n); tris [count][3]. Views: size [V][2]
 * (width, height), cam [V][6] (fx, fy, cx, cy, near, far), T [V][12], color[V] tightly packed u8x3 images.
 * atlas: [H][W][3] for the W x H of a previous layout call (zeroed here), or NULL for the layout alone; uv [count][6]
 * or NULL. stats [8]: triangles, W, H, texels, texels_seen, texels_fallback, tiles_clamped, views_used. Returns the
 * input error bits (1: a bad corner, 2: a repeated corner), 0 when the list is valid. */
u32 txw_texture(const float* rows, u64 stride, u32 n, const u32* tris, u64 count, float texel, float cos_max,
                float tolerance, int view_count, const int* size, const float* cam, const float* T,
                const u8* const* color, u8* atlas, float* uv, u64* stats) {
  const unsigned saved_csr = _mm_getcsr();
  _mm_setcsr(saved_csr | 0x8040u); /* FTZ | DAZ */
  memset(stats, 0, 8 * sizeof(u64));
  u32 errors = 0;
  int* cls = (int*)malloc(sizeof(int) * (count ? count : 1));
  int* rot = (int*)malloc(sizeof(int) * (count ? count : 1));
  u32* order = (u32*)malloc(sizeof(u32) * (count ? count : 1));
  u64 class_count[CLASSES] = {0}, clamped = 0;
  for (u64 t = 0; t < count; ++t) {
    int c;
    errors |= classify(rows, stride, n, tris + 3 * t, texel, &cls[t], &rot[t], &c);
    clamped += c;
    class_count[cls[t]]++;
  }
  if (errors) goto done;
  /* X3 */
  u64 start[CLASSES + 1], base[CLASSES + 1], texels = 0;
  start[0] = 0; base[0] = 0;
  for (int q = 0; q < CLASSES; ++q) {
    const u64 s = MAX_TILE >> q, k = class_count[q];
    start[q + 1] = start[q] + k;
    base[q + 1] = base[q] + (k + 1) / 2 * s * s;
    texels += (k + 1) / 2 * (s * (s + 1) / 2) + k / 2 * (s * (s - 1) / 2);
  }
  {
    u64 at = 0;
    for (int q = 0; q < CLASSES; ++q)
      for (u64 t = 0; t < count; ++t)
        if (cls[t] == q) order[at++] = (u32)t;
  }
  u64 W = 0, H = 0;
  if (count) {
    W = 1;
    while (W * W < base[CLASSES]) W <<= 1;
  }
  for (u64 i = 0; i < count; ++i) {
    const int q = cls[order[i]];
    const u64 s = MAX_TILE >> q, r = i - start[q];
    const u64 o = base[q] + (r >> 1) * s * s;
    if ((r & 1) == 0 && compact_bits(o >> 1) + s > H) H = compact_bits(o >> 1) + s;
  }
  stats[0] = count; stats[1] = W; stats[2] = H; stats[3] = texels; stats[6] = clamped;
  if (!atlas) goto done;
  memset(atlas, 0, (size_t)(W * H * 3));
  /* the visibility depth of every view */
  float** depth = (float**)calloc(view_count ? view_count : 1, sizeof(float*));
  for (int v = 0; v < view_count; ++v) {
    const int w = size[2 * v], h = size[2 * v + 1];
    const size_t P = (size_t)w * h;
    depth[v] = (float*)malloc(sizeof(float) * P);
    u8* col = (u8*)malloc(3 * P);
    float* nrm = (float*)malloc(sizeof(float) * 3 * P);
    u32* idx = (u32*)malloc(sizeof(u32) * P);
    u64* keys = (u64*)malloc(sizeof(u64) * P);
    const float* c = cam + 6 * v;
    mrw_render(rows, stride, n, tris, count, 0, w, h, c[0], c[1], c[2], c[3], c[4], c[5], T + 12 * v, depth[v], col,
               nrm, idx, keys, NULL);
    _mm_setcsr(saved_csr | 0x8040u); /* mrw_render restores the caller's MXCSR */
    free(col); free(nrm); free(idx); free(keys);
  }
  int* used = (int*)calloc(view_count ? view_count : 1, sizeof(int));
  u64 seen = 0, fallback = 0;
  for (u64 i = 0; i < count; ++i) {
    const u32 t = order[i];
    const int q = cls[t], ka = rot[t];
    const u32 s = MAX_TILE >> q;
    const u64 r = i - start[q], half = r & 1;
    const u64 o = base[q] + (r >> 1) * (u64)s * s;
    const u32 x0 = compact_bits(o), y0 = compact_bits(o >> 1);
    const u32 corner[3] = {tris[3 * t + ka], tris[3 * t + (ka + 1) % 3], tris[3 * t + (ka + 2) % 3]};
    /* X4 */
    if (uv) {
      for (int k = 0; k < 3; ++k) {
        const int role = (k - ka + 3) % 3;
        u32 X, Y;
        if (half == 0) { X = role == 1 ? s - 3 : 1; Y = role == 2 ? s - 3 : 1; }
        else { X = role == 1 ? 3 : s - 1; Y = role == 2 ? 3 : s - 1; }
        uv[6 * t + 2 * k] = (float)(x0 + X) / (float)W;
        uv[6 * t + 2 * k + 1] = (float)(y0 + Y) / (float)H;
      }
    }
    float pa[3], pb[3], pc[3], e1[3], e2[3], g[3], nn[3];
    pos(rows, stride, corner[0], pa); pos(rows, stride, corner[1], pb); pos(rows, stride, corner[2], pc);
    for (int x = 0; x < 3; ++x) { e1[x] = pb[x] - pa[x]; e2[x] = pc[x] - pa[x]; }
    g[0] = e1[1] * e2[2] - e1[2] * e2[1];
    g[1] = e1[2] * e2[0] - e1[0] * e2[2];
    g[2] = e1[0] * e2[1] - e1[1] * e2[0];
    const float gg = sqlen(g);
    const int has_normal = gg > 0.f && isfinite(gg);
    const float inv = has_normal ? 1.f / sqrtf(gg) : 0.f;
    for (int x = 0; x < 3; ++x) nn[x] = g[x] * inv;
    u32 rgb_c[3];
    for (int k = 0; k < 3; ++k) memcpy(&rgb_c[k], &rows[(size_t)ROW_COLOR * stride + corner[k]], 4);
    for (u32 j = 0; j < s; ++j)
      for (u32 ii = 0; ii < s; ++ii) {
        if (half == 0 ? ii + j > s - 1 : ii + j < s) continue;
        /* X5 */
        const float x = (float)ii + 0.5f, y = (float)j + 0.5f, qf = (float)(s - 4);
        float alpha, beta;
        if (half == 0) { alpha = (x - 1.f) / qf; beta = (y - 1.f) / qf; }
        else { alpha = ((float)(s - 1) - x) / qf; beta = ((float)(s - 1) - y) / qf; }
        alpha = alpha > 0.f ? alpha : 0.f;
        beta = beta > 0.f ? beta : 0.f;
        const float sum = alpha + beta;
        if (sum > 1.f) { alpha = alpha / sum; beta = 1.f - alpha; }
        float X[3];
        for (int k = 0; k < 3; ++k) X[k] = (pa[k] + alpha * e1[k]) + beta * e2[k];
        /* X6 */
        float S[4] = {0.f, 0.f, 0.f, 0.f};
        for (int v = 0; v < view_count && has_normal; ++v) {
          const float* Tv = T + 12 * v;
          const float* cv = cam + 6 * v;
          const int w = size[2 * v], h = size[2 * v + 1];
          const float c[3] = {transform_row(Tv, X[0], X[1], X[2]), transform_row(Tv + 4, X[0], X[1], X[2]),
                              transform_row(Tv + 8, X[0], X[1], X[2])};
          if (!(cv[4] <= c[2] && c[2] <= cv[5])) continue;
          const float u = cv[0] * (c[0] / c[2]) + cv[2], vv = cv[1] * (c[1] / c[2]) + cv[3];
          const float px = u - 0.5f, py = vv - 0.5f;
          if (!(px >= 0.f && px < (float)(w - 1) && py >= 0.f && py < (float)(h - 1))) continue;
          const float D = depth[v][(size_t)(int)vv * w + (int)u];
          if (!(D > 0.f) || !(fabsf(D - c[2]) <= tolerance * c[2])) continue;
          const float m[3] = {rotate_row(Tv, nn[0], nn[1], nn[2]), rotate_row(Tv + 4, nn[0], nn[1], nn[2]),
                              rotate_row(Tv + 8, nn[0], nn[1], nn[2])};
          const float cos_theta = -(((m[0] * c[0] + m[1] * c[1]) + m[2] * c[2]) / sqrtf(sqlen(c)));
          if (!(cos_theta >= cos_max)) continue;
          const float wt = cos_theta / (c[2] * c[2]);
          const float xf = floorf(px), yf = floorf(py);
          const float fx = px - xf, fy = py - yf;
          const int xi = (int)xf, yi = (int)yf;
          const u8* r0 = color[v] + 3 * ((size_t)yi * w + xi);
          const u8* r1 = r0 + 3 * (size_t)w;
          for (int ch = 0; ch < 3; ++ch) {
            const float v00 = (float)r0[ch], v10 = (float)r0[3 + ch], v01 = (float)r1[ch], v11 = (float)r1[3 + ch];
            const float top = v00 + fx * (v10 - v00);
            const float bot = v01 + fx * (v11 - v01);
            S[ch] = S[ch] + wt * (top + fy * (bot - top));
          }
          S[3] = S[3] + wt;
          used[v] = 1;
        }
        /* X7 */
        u32 out[3];
        if (S[3] > 0.f) {
          ++seen;
          for (int ch = 0; ch < 3; ++ch) out[ch] = to_u8(S[ch] / S[3] + 0.5f);
        } else {
          ++fallback;
          const float wa = (1.f - alpha) - beta;
          for (int ch = 0; ch < 3; ++ch) {
            const int sh = 8 * ch;
            float b = wa * (float)((rgb_c[0] >> sh) & 0xFFu);
            b = b + alpha * (float)((rgb_c[1] >> sh) & 0xFFu);
            b = b + beta * (float)((rgb_c[2] >> sh) & 0xFFu);
            out[ch] = to_u8(b + 0.5f);
          }
        }
        u8* o8 = atlas + 3 * ((size_t)(y0 + j) * W + x0 + ii);
        o8[0] = (u8)out[0]; o8[1] = (u8)out[1]; o8[2] = (u8)out[2];
      }
  }
  stats[4] = seen;
  stats[5] = fallback;
  for (int v = 0; v < view_count; ++v) stats[7] += used[v];
  for (int v = 0; v < view_count; ++v) free(depth[v]);
  free(depth);
  free(used);
done:
  free(cls); free(rot); free(order);
  _mm_setcsr(saved_csr);
  return errors;
}
