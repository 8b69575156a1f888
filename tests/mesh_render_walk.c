/* mesh_render_walk.c — plain-C restatement of sm_render_mesh (include/surfel_b200.h, "rendering the triangle
 * mesh", rules T1-T7). TEST INFRASTRUCTURE: the checker of the k_mesh_render_* kernels (csrc/render.cu), written
 * from the documented rules, sequentially: every triangle in list order, then every unmeshed disk, into a key
 * raster whose smallest key wins. fp32 throughout, no contraction (built with -ffp-contract=off), FTZ / DAZ set in
 * MXCSR for the duration of the call to match -ftz=true. The disk part is render_walk.c's (included below). Each
 * triangle tests its screen rectangle computed here in double with a two-pixel margin: any superset of the covered
 * pixels gives the same images. Built by tests/mesh_render_walk.py. */
#include "render_walk.c"

#include <stdlib.h>

enum { DISK_TAG = 0x80000000u };

typedef struct {
  u32 s[3];
  float c[3][3];
  float u[3], v[3];
  float area;
} Tri;

static float edge_value(float uj, float vj, float uk, float vk, float x, float y) {
  return (uk - uj) * (y - vj) - (vk - vj) * (x - uj);
}

/* T1-T3; 0 if the triangle is not drawn. */
static int load_tri(const float* rows, u64 stride, u32 n, const u32* t3, const float* T, float fx, float fy, float cx,
                    float cy, float near_depth, float far_depth, Tri* tr) {
#define ROW(r, i) rows[(size_t)(r) * stride + (i)]
  u32 s[3] = {t3[0], t3[1], t3[2]}, x;
  for (int k = 0; k < 3; ++k)
    if (!(s[k] < n) || !(ROW(ROW_RADIUS_SQUARED, s[k]) > 0.f)) return 0;
  if (s[0] > s[1]) { x = s[0]; s[0] = s[1]; s[1] = x; }
  if (s[1] > s[2]) { x = s[1]; s[1] = s[2]; s[2] = x; }
  if (s[0] > s[1]) { x = s[0]; s[0] = s[1]; s[1] = x; }
  for (int k = 0; k < 3; ++k) {
    const float px = ROW(ROW_SMOOTH_X, s[k]), py = ROW(ROW_SMOOTH_X + 1, s[k]), pz = ROW(ROW_SMOOTH_X + 2, s[k]);
    const float c0 = transform_row(T, px, py, pz), c1 = transform_row(T + 4, px, py, pz), c2 = transform_row(T + 8, px, py, pz);
    if (!(near_depth <= c2 && c2 <= far_depth)) return 0;
    tr->s[k] = s[k];
    tr->c[k][0] = c0; tr->c[k][1] = c1; tr->c[k][2] = c2;
    tr->u[k] = fx * (c0 / c2) + cx;
    tr->v[k] = fy * (c1 / c2) + cy;
  }
#undef ROW
  tr->area = edge_value(tr->u[0], tr->v[0], tr->u[1], tr->v[1], tr->u[2], tr->v[2]);
  return tr->area != 0.f && isfinite(tr->area);
}

/* T4. */
static int tri_weights(const Tri* tr, int px, int py, float w[3]) {
  const float x = (float)px + 0.5f, y = (float)py + 0.5f;
  w[0] = edge_value(tr->u[1], tr->v[1], tr->u[2], tr->v[2], x, y);
  w[1] = -edge_value(tr->u[0], tr->v[0], tr->u[2], tr->v[2], x, y);
  w[2] = edge_value(tr->u[0], tr->v[0], tr->u[1], tr->v[1], x, y);
  if (tr->area > 0.f) return w[0] >= 0.f && w[1] >= 0.f && w[2] >= 0.f;
  return w[0] <= 0.f && w[1] <= 0.f && w[2] <= 0.f;
}

/* T5. */
static float tri_depth(const Tri* tr, const float w[3], float q[3]) {
  for (int k = 0; k < 3; ++k) q[k] = (w[k] / tr->area) / tr->c[k][2];
  return 1.f / ((q[0] + q[1]) + q[2]);
}

static u32 blend_channel(const float q[3], const u32 rgb[3], int shift, float z) {
  float sum = q[0] * (float)((rgb[0] >> shift) & 0xFFu);
  sum = sum + q[1] * (float)((rgb[1] >> shift) & 0xFFu);
  sum = sum + q[2] * (float)((rgb[2] >> shift) & 0xFFu);
  const float value = sum * z + 0.5f;
  return value >= 255.f ? 255u : (u32)(int)value;
}

static void tri_normal(const Tri* tr, float out[3]) {
  const float* c0 = tr->c[0];
  const float e1[3] = {tr->c[1][0] - c0[0], tr->c[1][1] - c0[1], tr->c[1][2] - c0[2]};
  const float e2[3] = {tr->c[2][0] - c0[0], tr->c[2][1] - c0[1], tr->c[2][2] - c0[2]};
  float g[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
  const float facing = (g[0] * c0[0] + g[1] * c0[1]) + g[2] * c0[2];
  if (facing > 0.f) { g[0] = -g[0]; g[1] = -g[1]; g[2] = -g[2]; }
  const float gg = (g[0] * g[0] + g[1] * g[1]) + g[2] * g[2];
  if (!(gg > 0.f) || !isfinite(gg)) { out[0] = out[1] = out[2] = 0.f; return; }
  const float inv = 1.f / sqrtf(gg);
  out[0] = g[0] * inv; out[1] = g[1] * inv; out[2] = g[2] * inv;
}

static int clamp_axis(double lo, double hi, int size, int* p0, int* p1) {
  double q0 = floor(lo - 0.5) - 2, q1 = ceil(hi - 0.5) + 2;
  if (q0 < 0) q0 = 0;
  if (q1 > size - 1) q1 = size - 1;
  if (!(q0 <= q1)) return 0;
  *p0 = (int)q0;
  *p1 = (int)q1;
  return 1;
}

/* rows: [25][stride] float32 (rows 3-5 = smooth positions), slots [0, n). tris: [count][3]. flags: 1 = draw the
 * unmeshed surfels. Outputs tightly packed; keys: width * height scratch. stats (may be NULL): [0] triangles that
 * passed T1-T3 and cover at least one pixel centre, [1] disks drawn (T6 slots that pass rules 1-2), [2] marked
 * slots. */
void mrw_render(const float* rows, u64 stride, u32 n, const u32* tris, u64 count, int flags, int width, int height,
                float fx, float fy, float cx, float cy, float near_depth, float far_depth, const float* T, float* depth,
                u8* color, float* normal, u32* index, u64* keys, u64* stats) {
  const unsigned saved_csr = _mm_getcsr();
  _mm_setcsr(saved_csr | 0x8040u); /* FTZ | DAZ */
  const size_t P = (size_t)width * height;
  for (size_t k = 0; k < P; ++k) keys[k] = ~0ull;
  u64 drawn_tris = 0, drawn_disks = 0, marked = 0;
  u8* marks = (u8*)calloc(n ? n : 1, 1);
#define ROW(r, i) rows[(size_t)(r) * stride + (i)]
  for (u64 t = 0; t < count; ++t) {
    const u32* t3 = tris + 3 * t;
    int valid = 1;
    for (int k = 0; k < 3; ++k)
      if (!(t3[k] < n) || !(ROW(ROW_RADIUS_SQUARED, t3[k]) > 0.f)) valid = 0;
    if (valid)
      for (int k = 0; k < 3; ++k) marks[t3[k]] = 1;
    Tri tr;
    if (!load_tri(rows, stride, n, t3, T, fx, fy, cx, cy, near_depth, far_depth, &tr)) continue;
    double ulo = tr.u[0], uhi = tr.u[0], vlo = tr.v[0], vhi = tr.v[0];
    for (int k = 1; k < 3; ++k) {
      ulo = fmin(ulo, tr.u[k]); uhi = fmax(uhi, tr.u[k]);
      vlo = fmin(vlo, tr.v[k]); vhi = fmax(vhi, tr.v[k]);
    }
    int x0, x1, y0, y1, any = 0;
    if (!clamp_axis(ulo, uhi, width, &x0, &x1) || !clamp_axis(vlo, vhi, height, &y0, &y1)) continue;
    for (int py = y0; py <= y1; ++py)
      for (int px = x0; px <= x1; ++px) {
        float w[3], q[3];
        if (!tri_weights(&tr, px, py, w)) continue;
        any = 1;
        const float z = tri_depth(&tr, w, q);
        if (!(z > 0.f) || !isfinite(z)) continue;
        u32 bits;
        memcpy(&bits, &z, 4);
        const u64 key = ((u64)bits << 32) | (u32)t;
        u64* slot = keys + (size_t)py * width + px;
        if (key < *slot) *slot = key;
      }
    drawn_tris += any;
  }
  for (u32 i = 0; i < n; ++i) marked += marks[i];
  if (flags & 1) {
    for (u32 i = 0; i < n; ++i) {
      if (marks[i]) continue;
      const float radius_squared = ROW(ROW_RADIUS_SQUARED, i);
      if (!(radius_squared > 0.f)) continue;
      const float sx = ROW(ROW_SMOOTH_X, i), sy = ROW(ROW_SMOOTH_X + 1, i), sz = ROW(ROW_SMOOTH_X + 2, i);
      const float c[3] = {transform_row(T, sx, sy, sz), transform_row(T + 4, sx, sy, sz), transform_row(T + 8, sx, sy, sz)};
      if (!(near_depth <= c[2] && c[2] <= far_depth)) continue;
      ++drawn_disks;
      const float nx = ROW(ROW_NORMAL_X, i), ny = ROW(ROW_NORMAL_X + 1, i), nz = ROW(ROW_NORMAL_X + 2, i);
      const float m[3] = {rotate_row(T, nx, ny, nz), rotate_row(T + 4, nx, ny, nz), rotate_row(T + 8, nx, ny, nz)};
      const float num = dot3(m[0], m[1], m[2], c[0], c[1], c[2]);
      int x0 = 0, x1 = width - 1, y0 = 0, y1 = height - 1;
      const double reach = sqrt((double)radius_squared) * 1.01 + 1e-4 * (fabs(c[0]) + fabs(c[1]) + fabs(c[2]));
      if (c[2] - reach > 0) {
        if (!axis_range(c[0], c[2], reach, fx, cx, width, &x0, &x1) || !axis_range(c[1], c[2], reach, fy, cy, height, &y0, &y1))
          continue;
      }
      for (int py = y0; py <= y1; ++py) {
        const float dy = ray_coord(py, cy, fy);
        for (int px = x0; px <= x1; ++px) {
          const float dx = ray_coord(px, cx, fx);
          const float den = dot3(m[0], m[1], m[2], dx, dy, 1.0f);
          if (den == 0.f) continue;
          const float t = num / den;
          if (!(t > 0.f) || !isfinite(t)) continue;
          const float ex = t * dx - c[0], ey = t * dy - c[1], ez = t - c[2];
          if (!(fmaf(ez, ez, fmaf(ex, ex, ey * ey)) <= radius_squared)) continue;
          u32 bits;
          memcpy(&bits, &t, 4);
          const u64 key = ((u64)bits << 32) | (DISK_TAG | i);
          u64* slot = keys + (size_t)py * width + px;
          if (key < *slot) *slot = key;
        }
      }
    }
  }
  for (size_t k = 0; k < P; ++k) {
    float d = 0.f, mm[3] = {0.f, 0.f, 0.f};
    u32 idx = 0xFFFFFFFFu, rgb = 0;
    if (keys[k] != ~0ull) {
      idx = (u32)keys[k];
      const u32 bits = (u32)(keys[k] >> 32);
      memcpy(&d, &bits, 4);
      if (idx & DISK_TAG) {
        const u32 i = idx & ~(u32)DISK_TAG;
        memcpy(&rgb, &ROW(ROW_COLOR, i), 4);
        const float nx = ROW(ROW_NORMAL_X, i), ny = ROW(ROW_NORMAL_X + 1, i), nz = ROW(ROW_NORMAL_X + 2, i);
        mm[0] = rotate_row(T, nx, ny, nz);
        mm[1] = rotate_row(T + 4, nx, ny, nz);
        mm[2] = rotate_row(T + 8, nx, ny, nz);
      } else {
        Tri tr;
        load_tri(rows, stride, n, tris + 3 * (u64)idx, T, fx, fy, cx, cy, near_depth, far_depth, &tr);
        float w[3], q[3];
        tri_weights(&tr, (int)(k % width), (int)(k / width), w);
        const float z = tri_depth(&tr, w, q);
        u32 c3[3];
        for (int j = 0; j < 3; ++j) memcpy(&c3[j], &ROW(ROW_COLOR, tr.s[j]), 4);
        rgb = blend_channel(q, c3, 0, z) | (blend_channel(q, c3, 8, z) << 8) | (blend_channel(q, c3, 16, z) << 16);
        tri_normal(&tr, mm);
      }
    }
    depth[k] = d;
    index[k] = idx;
    color[3 * k] = rgb & 0xFFu;
    color[3 * k + 1] = (rgb >> 8) & 0xFFu;
    color[3 * k + 2] = (rgb >> 16) & 0xFFu;
    memcpy(normal + 3 * k, mm, sizeof(mm));
  }
#undef ROW
  free(marks);
  if (stats) { stats[0] = drawn_tris; stats[1] = drawn_disks; stats[2] = marked; }
  _mm_setcsr(saved_csr);
}
