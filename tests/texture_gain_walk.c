/* texture_gain_walk.c — plain-C restatement of sm_mesh_texture_compensated (include/surfel_b200.h, "exposure
 * compensation between the texture views", rules G1-G6 beside X1-X8). TEST INFRASTRUCTURE: the checker of the
 * k_tex_gain_* kernels and of k_tex_accumulate<true> (csrc/texture.cu), written from the documented rules,
 * sequentially. The layout, uv and stats come from texture_walk.c (included below), which restates
 * sm_mesh_texture; the sample matrix, the conjugate-gradient solve and the gained accumulation are restated here.
 * fp32 with FTZ / DAZ as texture_walk.c, and the fp64 solve with the caller's MXCSR (the device does not flush
 * doubles). Built by tests/texture_gain_walk.py with -ffp-contract=off. */
#include "texture_walk.c"

enum { GAIN_BLOCK = 1024, MAX_VIEWS = 1024 };

/* TREE of G4 over 32 values. */
static double tree32(const double* in) {
  double t[32];
  memcpy(t, in, sizeof(t));
  for (int off = 16; off > 0; off >>= 1)
    for (int i = 0; i < off; ++i) t[i] = t[i] + t[i + off];
  return t[0];
}

/* X6 of view v at point X with normal nn: 1 and (w, rgb) when the view contributes. */
static int x6(const float* Tv, const float* cv, int w, int h, const float* depth, const u8* color, float tolerance,
              float cos_max, const float X[3], const float nn[3], float* wt, float rgb[3]) {
  const float c[3] = {transform_row(Tv, X[0], X[1], X[2]), transform_row(Tv + 4, X[0], X[1], X[2]),
                      transform_row(Tv + 8, X[0], X[1], X[2])};
  if (!(cv[4] <= c[2] && c[2] <= cv[5])) return 0;
  const float u = cv[0] * (c[0] / c[2]) + cv[2], vv = cv[1] * (c[1] / c[2]) + cv[3];
  const float px = u - 0.5f, py = vv - 0.5f;
  if (!(px >= 0.f && px < (float)(w - 1) && py >= 0.f && py < (float)(h - 1))) return 0;
  const float D = depth[(size_t)(int)vv * w + (int)u];
  if (!(D > 0.f) || !(fabsf(D - c[2]) <= tolerance * c[2])) return 0;
  const float m[3] = {rotate_row(Tv, nn[0], nn[1], nn[2]), rotate_row(Tv + 4, nn[0], nn[1], nn[2]),
                      rotate_row(Tv + 8, nn[0], nn[1], nn[2])};
  const float cos_theta = -(((m[0] * c[0] + m[1] * c[1]) + m[2] * c[2]) / sqrtf(sqlen(c)));
  if (!(cos_theta >= cos_max)) return 0;
  *wt = cos_theta / (c[2] * c[2]);
  const float xf = floorf(px), yf = floorf(py);
  const float fx = px - xf, fy = py - yf;
  const int xi = (int)xf, yi = (int)yf;
  const u8* r0 = color + 3 * ((size_t)yi * w + xi);
  const u8* r1 = r0 + 3 * (size_t)w;
  for (int ch = 0; ch < 3; ++ch) {
    const float v00 = (float)r0[ch], v10 = (float)r0[3 + ch], v01 = (float)r1[ch], v11 = (float)r1[3 + ch];
    const float top = v00 + fx * (v10 - v00);
    const float bot = v01 + fx * (v11 - v01);
    rgb[ch] = top + fy * (bot - top);
  }
  return 1;
}

/* X5's position and normal at (alpha, beta) of the triangle with corners (a, b, c). */
static int point_on(const float* rows, u64 stride, const u32 corner[3], float alpha, float beta, float X[3],
                    float nn[3]) {
  float pa[3], pb[3], pc[3], e1[3], e2[3], g[3];
  pos(rows, stride, corner[0], pa); pos(rows, stride, corner[1], pb); pos(rows, stride, corner[2], pc);
  for (int x = 0; x < 3; ++x) { e1[x] = pb[x] - pa[x]; e2[x] = pc[x] - pa[x]; }
  for (int k = 0; k < 3; ++k) X[k] = (pa[k] + alpha * e1[k]) + beta * e2[k];
  g[0] = e1[1] * e2[2] - e1[2] * e2[1];
  g[1] = e1[2] * e2[0] - e1[0] * e2[2];
  g[2] = e1[0] * e2[1] - e1[1] * e2[0];
  const float gg = sqlen(g);
  const int has_normal = gg > 0.f && isfinite(gg);
  const float inv = has_normal ? 1.f / sqrtf(gg) : 0.f;
  for (int x = 0; x < 3; ++x) nn[x] = g[x] * inv;
  return has_normal;
}

typedef struct {
  const float* S;   /* [V][P][3], NaN when absent */
  const u32* k;     /* [P], 0 when not in the fit */
  u64 P, blocks;
  int V;
  double* mean;     /* [P][3] */
  double* blocks3;  /* [blocks][3] scratch */
} Fit;

/* G4's point sweep: m_p of x. */
static void means(const Fit* f, const double (*x)[3]) {
  for (u64 p = 0; p < f->P; ++p) {
    if (!f->k[p]) continue;
    double sum[3] = {0.0, 0.0, 0.0};
    for (int v = 0; v < f->V; ++v) {
      const float* s = f->S + 3 * ((size_t)v * f->P + p);
      if (isnan(s[0])) continue;
      for (int ch = 0; ch < 3; ++ch) sum[ch] = sum[ch] + (double)s[ch] * x[v][ch];
    }
    for (int ch = 0; ch < 3; ++ch) f->mean[3 * p + ch] = sum[ch] / (double)f->k[p];
  }
}

/* G4's column sum of view v: of s (s x_v - m_p), or with squares of (s x_v - m_p)^2. */
static void column(const Fit* f, int v, const double xv[3], int squares, double out[3]) {
  for (int ch = 0; ch < 3; ++ch) {
    double* b = f->blocks3;
    for (u64 blk = 0; blk < f->blocks; ++blk) {
      double ws[32];
      for (int w = 0; w < 32; ++w) {
        double t[32];
        for (int l = 0; l < 32; ++l) {
          const u64 p = blk * GAIN_BLOCK + 32 * w + l;
          t[l] = 0.0;
          if (p >= f->P || !f->k[p]) continue;
          const float* s = f->S + 3 * ((size_t)v * f->P + p);
          if (isnan(s[0])) continue;
          const double sv = s[ch];
          const double e = sv * xv[ch] - f->mean[3 * p + ch];
          t[l] = squares ? e * e : sv * e;
        }
        ws[w] = tree32(t);
      }
      b[blk] = tree32(ws);
    }
    for (u64 n = f->blocks; n > 1; n = (n + 31) / 32)
      for (u64 g = 0; 32 * g < n; ++g) {
        double t[32];
        for (int l = 0; l < 32; ++l) t[l] = 32 * g + l < n ? b[32 * g + l] : 0.0;
        b[g] = tree32(t);
      }
    out[ch] = b[0];
  }
}

/* The sum over views of G4: TREE of the TREEs of views 32w .. 32w + 31, 0 past view_count. */
static double views_tree(const double* t /* [MAX_VIEWS] */) {
  double ws[32];
  for (int w = 0; w < 32; ++w) ws[w] = tree32(t + 32 * w);
  return tree32(ws);
}

static void columns(const Fit* f, const double (*x)[3], int squares, double (*y)[3]) {
  for (int v = 0; v < f->V; ++v) column(f, v, x[v], squares, y[v]);
}

static double data_term(const Fit* f, const double (*x)[3], double (*y)[3]) {
  static double t[MAX_VIEWS];
  double D[3];
  means(f, x);
  columns(f, x, 1, y);
  for (int ch = 0; ch < 3; ++ch) {
    for (int v = 0; v < MAX_VIEWS; ++v) t[v] = v < f->V ? y[v][ch] : 0.0;
    D[ch] = views_tree(t);
  }
  return (D[0] + D[1]) + D[2];
}

/* The arguments of txw_texture, then the gain parameters. samples: [V][P][3] for P = min(count, max_samples / V)
 * (may be NULL); gains [V][3]; gain_stats [5]: points, samples, views_fitted, rms_before, rms_after. atlas NULL:
 * the layout alone (gains and gain_stats untouched). Returns txw_texture's error bits. */
u32 txg_texture(const float* rows, u64 stride, u32 n, const u32* tris, u64 count, float texel, float cos_max,
                float tolerance, int view_count, const int* size, const float* cam, const float* T,
                const u8* const* color, int max_samples, int iterations, float sigma_noise, float sigma_gain,
                float min_level, float max_level, u8* atlas, float* uv, u64* stats, float* gains, double* gain_stats,
                float* samples_out) {
  const u32 errors = txw_texture(rows, stride, n, tris, count, texel, cos_max, tolerance, view_count, size, cam, T,
                                 color, atlas, uv, stats);
  if (errors || !atlas) return errors;
  for (int i = 0; i < 5; ++i) gain_stats[i] = 0.0;
  for (int i = 0; i < 3 * view_count; ++i) gains[i] = 1.f;
  if (count == 0) return 0;
  const unsigned saved_csr = _mm_getcsr();
  _mm_setcsr(saved_csr | 0x8040u); /* FTZ | DAZ */
  const int V = view_count;
  float** depth = (float**)calloc(V ? V : 1, sizeof(float*));
  for (int v = 0; v < V; ++v) {
    const int w = size[2 * v], h = size[2 * v + 1];
    const size_t px = (size_t)w * h;
    depth[v] = (float*)malloc(sizeof(float) * px);
    u8* col = (u8*)malloc(3 * px);
    float* nrm = (float*)malloc(sizeof(float) * 3 * px);
    u32* idx = (u32*)malloc(sizeof(u32) * px);
    u64* keys = (u64*)malloc(sizeof(u64) * px);
    const float* c = cam + 6 * v;
    mrw_render(rows, stride, n, tris, count, 0, w, h, c[0], c[1], c[2], c[3], c[4], c[5], T + 12 * v, depth[v], col,
               nrm, idx, keys, NULL);
    _mm_setcsr(saved_csr | 0x8040u);
    free(col); free(nrm); free(idx); free(keys);
  }
  /* G1, G2 */
  const u64 P = V > 0 ? (count < (u64)max_samples / (u64)V ? count : (u64)max_samples / (u64)V) : 0;
  static double x[MAX_VIEWS][3], r[MAX_VIEWS][3], d[MAX_VIEWS][3], y[MAX_VIEWS][3];
  for (int v = 0; v < MAX_VIEWS; ++v)
    for (int ch = 0; ch < 3; ++ch) { x[v][ch] = 1.0; d[v][ch] = 1.0; r[v][ch] = 0.0; y[v][ch] = 0.0; }
  float* S = (float*)malloc(sizeof(float) * 3 * (P * V ? P * V : 1));
  u32* k = (u32*)calloc(P ? P : 1, sizeof(u32));
  u32 nv[MAX_VIEWS] = {0};
  const float third = 1.f / 3.f;
  for (u64 p = 0; p < P; ++p) {
    const u64 t = p * count / P;
    const u32 corner[3] = {tris[3 * t], tris[3 * t + 1], tris[3 * t + 2]};
    float X[3], nn[3];
    const int has_normal = point_on(rows, stride, corner, third, third, X, nn);
    for (int v = 0; v < V; ++v) {
      float wt, rgb[3];
      int present = has_normal && x6(T + 12 * v, cam + 6 * v, size[2 * v], size[2 * v + 1], depth[v], color[v],
                                     tolerance, cos_max, X, nn, &wt, rgb);
      for (int ch = 0; ch < 3; ++ch) present = present && rgb[ch] >= min_level && rgb[ch] <= max_level;
      for (int ch = 0; ch < 3; ++ch) S[3 * ((size_t)v * P + p) + ch] = present ? rgb[ch] : NAN;
    }
  }
  if (samples_out) memcpy(samples_out, S, sizeof(float) * 3 * P * V);
  for (u64 p = 0; p < P; ++p) {
    u32 kk = 0;
    for (int v = 0; v < V; ++v) kk += !isnan(S[3 * ((size_t)v * P + p)]);
    k[p] = kk >= 2 ? kk : 0;
    for (int v = 0; v < V && k[p]; ++v) nv[v] += !isnan(S[3 * ((size_t)v * P + p)]);
  }
  _mm_setcsr(saved_csr);   /* fp64 from here: no flushing */
  double data0 = 0.0, data1 = 0.0;
  u64 samples = 0, fitted = 0;
  for (int v = 0; v < V; ++v) { samples += nv[v]; fitted += nv[v] > 0; }
  if (P > 0) {
    Fit f;
    f.S = S; f.k = k; f.P = P; f.V = V;
    f.blocks = (P + GAIN_BLOCK - 1) / GAIN_BLOCK;
    f.mean = (double*)malloc(sizeof(double) * 3 * P);
    f.blocks3 = (double*)malloc(sizeof(double) * f.blocks);
    const double sn = sigma_noise, sg = sigma_gain;
    const double cN = 1.0 / (sn * sn), cG = 1.0 / (sg * sg);
    static double t[MAX_VIEWS];
    double rr[3];
    int done[3];
    /* D at x = 1; r = b - A 1 from the same means */
    data0 = data_term(&f, (const double (*)[3])x, y);
    columns(&f, (const double (*)[3])x, 0, y);
    for (int ch = 0; ch < 3; ++ch) {
      for (int v = 0; v < MAX_VIEWS; ++v) {
        t[v] = 0.0;
        if (v >= V) continue;
        const double nG = (double)nv[v] * cG;
        const double Ad = y[v][ch] * cN + nG * d[v][ch];
        r[v][ch] = nG - Ad;
        d[v][ch] = r[v][ch];
        t[v] = r[v][ch] * r[v][ch];
      }
      rr[ch] = views_tree(t);
      done[ch] = !(rr[ch] != 0.0);
    }
    for (int it = 0; it < iterations; ++it) {
      means(&f, (const double (*)[3])d);
      columns(&f, (const double (*)[3])d, 0, y);
      for (int ch = 0; ch < 3; ++ch) {
        static double Ad[MAX_VIEWS];
        for (int v = 0; v < MAX_VIEWS; ++v) {
          Ad[v] = v < V ? y[v][ch] * cN + ((double)nv[v] * cG) * d[v][ch] : 0.0;
          t[v] = v < V ? d[v][ch] * Ad[v] : 0.0;
        }
        const double pAp = views_tree(t);
        const int active = !done[ch] && pAp > 0.0;
        const double alpha = active ? rr[ch] / pAp : 0.0;
        for (int v = 0; v < MAX_VIEWS; ++v) {
          t[v] = 0.0;
          if (v >= V) continue;
          if (active) {
            x[v][ch] = x[v][ch] + alpha * d[v][ch];
            r[v][ch] = r[v][ch] - alpha * Ad[v];
          }
          t[v] = r[v][ch] * r[v][ch];
        }
        const double rr_new = views_tree(t);
        if (active) {
          const double beta = rr_new / rr[ch];
          for (int v = 0; v < V; ++v) d[v][ch] = r[v][ch] + beta * d[v][ch];
          rr[ch] = rr_new;
        }
        done[ch] = !active || !(rr_new != 0.0);
      }
    }
    for (int ch = 0; ch < 3; ++ch) {   /* the common scale: x over its n_v-weighted mean */
      for (int v = 0; v < MAX_VIEWS; ++v) t[v] = v < V ? (double)nv[v] * x[v][ch] : 0.0;
      const double weighted = views_tree(t);
      for (int v = 0; v < MAX_VIEWS; ++v) t[v] = v < V ? (double)nv[v] : 0.0;
      const double total = views_tree(t);
      double mean = total > 0.0 ? weighted / total : 1.0;
      if (!(mean > 0.0)) mean = 1.0;
      for (int v = 0; v < V; ++v) {
        gains[3 * v + ch] = nv[v] > 0 ? (float)(x[v][ch] / mean) : 1.f;
        d[v][ch] = (double)gains[3 * v + ch];
      }
    }
    data1 = data_term(&f, (const double (*)[3])d, y);
    free(f.mean); free(f.blocks3);
  }
  gain_stats[0] = (double)P;
  gain_stats[1] = (double)samples;
  gain_stats[2] = (double)fitted;
  if (samples > 0) {
    const double scale = 3.0 * (double)samples;
    gain_stats[3] = sqrt(data0 / scale);
    gain_stats[4] = sqrt(data1 / scale);
  }
  _mm_setcsr(saved_csr | 0x8040u);
  /* G5: X5-X7 again with the gained samples (the layout of X3 as texture_walk.c lays it out) */
  int* cls = (int*)malloc(sizeof(int) * count);
  int* rot = (int*)malloc(sizeof(int) * count);
  u32* order = (u32*)malloc(sizeof(u32) * count);
  u64 class_count[CLASSES] = {0};
  for (u64 t = 0; t < count; ++t) {
    int c;
    classify(rows, stride, n, tris + 3 * t, texel, &cls[t], &rot[t], &c);
    class_count[cls[t]]++;
  }
  u64 start[CLASSES + 1], base[CLASSES + 1];
  start[0] = 0; base[0] = 0;
  for (int q = 0; q < CLASSES; ++q) {
    const u64 s = MAX_TILE >> q;
    start[q + 1] = start[q] + class_count[q];
    base[q + 1] = base[q] + (class_count[q] + 1) / 2 * s * s;
  }
  {
    u64 at = 0;
    for (int q = 0; q < CLASSES; ++q)
      for (u64 t = 0; t < count; ++t)
        if (cls[t] == q) order[at++] = (u32)t;
  }
  const u64 W = stats[1];
  for (u64 i = 0; i < count; ++i) {
    const u32 t = order[i];
    const int q = cls[t], ka = rot[t];
    const u32 s = MAX_TILE >> q;
    const u64 rk = i - start[q], half = rk & 1;
    const u64 o = base[q] + (rk >> 1) * (u64)s * s;
    const u32 x0 = compact_bits(o), y0 = compact_bits(o >> 1);
    const u32 corner[3] = {tris[3 * t + ka], tris[3 * t + (ka + 1) % 3], tris[3 * t + (ka + 2) % 3]};
    for (u32 j = 0; j < s; ++j)
      for (u32 ii = 0; ii < s; ++ii) {
        if (half == 0 ? ii + j > s - 1 : ii + j < s) continue;
        const float xx = (float)ii + 0.5f, yy = (float)j + 0.5f, qf = (float)(s - 4);
        float alpha, beta;
        if (half == 0) { alpha = (xx - 1.f) / qf; beta = (yy - 1.f) / qf; }
        else { alpha = ((float)(s - 1) - xx) / qf; beta = ((float)(s - 1) - yy) / qf; }
        alpha = alpha > 0.f ? alpha : 0.f;
        beta = beta > 0.f ? beta : 0.f;
        const float sum = alpha + beta;
        if (sum > 1.f) { alpha = alpha / sum; beta = 1.f - alpha; }
        float X[3], nn[3];
        if (!point_on(rows, stride, corner, alpha, beta, X, nn)) continue;   /* the corner blend, as written */
        float Sacc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int v = 0; v < V; ++v) {
          float wt, rgb[3];
          if (!x6(T + 12 * v, cam + 6 * v, size[2 * v], size[2 * v + 1], depth[v], color[v], tolerance, cos_max, X,
                  nn, &wt, rgb))
            continue;
          for (int ch = 0; ch < 3; ++ch) Sacc[ch] = Sacc[ch] + wt * (gains[3 * v + ch] * rgb[ch]);
          Sacc[3] = Sacc[3] + wt;
        }
        if (!(Sacc[3] > 0.f)) continue;   /* the corner blend of texture_walk.c stands */
        u8* o8 = atlas + 3 * ((size_t)(y0 + j) * W + x0 + ii);
        for (int ch = 0; ch < 3; ++ch) o8[ch] = (u8)to_u8(Sacc[ch] / Sacc[3] + 0.5f);
      }
  }
  free(cls); free(rot); free(order);
  for (int v = 0; v < V; ++v) free(depth[v]);
  free(depth); free(S); free(k);
  _mm_setcsr(saved_csr);
  return 0;
}
