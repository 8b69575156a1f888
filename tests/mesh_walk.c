/* mesh_walk.c — TEST INFRASTRUCTURE: a plain-C restatement of sm_triangulate (include/surfel_b200.h), one slot
 * after the other, with a brute-force k-NN. Built by tests/mesh_walk.py with -ffp-contract=off; every fp32
 * operation is rounded on its own, and denormals are flushed to zero (MXCSR FTZ | DAZ) as the kernels do. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <xmmintrin.h>

#define ROWS_SMOOTH_X 3
#define ROW_RADIUS_SQUARED 7
#define ROW_NORMAL_X 8
#define MAX_RESULTS 64
#define NONE 0xFFFFFFFFu

typedef struct {
  const float* rows;
  uint64_t stride;
  uint32_t n;
  uint32_t present_count;
  uint32_t* by_x;            /* present slots sorted by x (the brute-force search window) */
  int umbrella_cap;
  uint32_t* umbrella;        /* [n][cap][2] */
  uint32_t* umbrella_count;  /* [n] */
  float cos_triangle;
} Mesh;

static float at(const Mesh* m, int row, uint32_t i) { return m->rows[(uint64_t)row * m->stride + i]; }

static float dot3(const float* a, const float* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

static void position(const Mesh* m, uint32_t i, float* p) {
  for (int c = 0; c < 3; ++c) p[c] = at(m, ROWS_SMOOTH_X + c, i);
}

static int unit_normal(const Mesh* m, uint32_t i, float* out) {
  float n[3];
  for (int c = 0; c < 3; ++c) n[c] = at(m, ROW_NORMAL_X + c, i);
  const float s = dot3(n, n);
  if (!(s > 0.f) || !isfinite(s)) return 0;
  const float inv = 1.f / sqrtf(s);
  for (int c = 0; c < 3; ++c) out[c] = n[c] * inv;
  return 1;
}

static int present(const Mesh* m, uint32_t i) { return at(m, ROW_RADIUS_SQUARED, i) > 0.f; }

typedef struct { uint64_t key; } Key;
static int key_cmp(const void* a, const void* b) {
  const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
  return x < y ? -1 : (x > y ? 1 : 0);
}

static const Mesh* g_sort_mesh;
static int x_cmp(const void* a, const void* b) {
  const uint32_t i = *(const uint32_t*)a, j = *(const uint32_t*)b;
  const float xi = at(g_sort_mesh, ROWS_SMOOTH_X, i), xj = at(g_sort_mesh, ROWS_SMOOTH_X, j);
  return xi < xj ? -1 : (xi > xj ? 1 : (i < j ? -1 : (i > j)));
}

static uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* Rules 1-3 for slot i; writes U(i). Returns 1 if the umbrella overflowed. */
static int build_umbrella(Mesh* m, uint32_t i, float f2, float cos_normal, uint64_t* keys) {
  m->umbrella_count[i] = 0;
  const float r2 = at(m, ROW_RADIUS_SQUARED, i);
  float ni[3];
  if (!(r2 > 0.f) || !unit_normal(m, i, ni)) return 0;
  float pi[3];
  position(m, i, pi);
  const float radius_squared = r2 * f2;
  int found = 0;
  /* Every j that passes the fp32 test has fl(dx)^2 <= radius^2, so |x_j - x_i| lies inside this window; the
   * window only skips work, the test below decides. */
  const double window = sqrt((double)radius_squared) * 1.0001 + 1e-30;
  uint32_t first = 0, end = m->present_count;
  while (first < end) {
    const uint32_t mid = first + (end - first) / 2;
    if ((double)at(m, ROWS_SMOOTH_X, m->by_x[mid]) < (double)pi[0] - window) first = mid + 1; else end = mid;
  }
  for (uint32_t s = first; s < m->present_count; ++s) {
    const uint32_t j = m->by_x[s];
    if ((double)at(m, ROWS_SMOOTH_X, j) > (double)pi[0] + window) break;
    float pj[3];
    position(m, j, pj);
    const float dx = pj[0] - pi[0], dy = pj[1] - pi[1], dz = pj[2] - pi[2];
    const float d2 = (dx * dx + dy * dy) + dz * dz;
    if (d2 <= radius_squared) keys[found++] = ((uint64_t)fbits(d2) << 32) | j;
  }
  qsort(keys, found, sizeof(uint64_t), key_cmp);
  if (found > MAX_RESULTS) found = MAX_RESULTS;

  const float sign = copysignf(1.f, ni[2]);
  const float bf = -1.f / (sign + ni[2]);
  const float bb = (ni[0] * ni[1]) * bf;
  const float u[3] = {1.f + ((sign * ni[0]) * ni[0]) * bf, sign * bb, -(sign * ni[0])};
  const float v[3] = {bb, sign + (ni[1] * ni[1]) * bf, -ni[1]};

  uint32_t index[MAX_RESULTS];
  int valid[MAX_RESULTS];
  float qx[MAX_RESULTS], qy[MAX_RESULTS];
  for (int g = 0; g < MAX_RESULTS; ++g) {
    index[g] = g < found ? (uint32_t)keys[g] : NONE;
    valid[g] = g < found && index[g] != i;
    qx[g] = qy[g] = 0.f;
    float nj[3];
    if (valid[g]) valid[g] = unit_normal(m, index[g], nj) && dot3(ni, nj) >= cos_normal;
    if (valid[g]) {
      float pj[3];
      position(m, index[g], pj);
      const float d[3] = {pj[0] - pi[0], pj[1] - pi[1], pj[2] - pi[2]};
      qx[g] = dot3(d, u);
      qy[g] = dot3(d, v);
      valid[g] = !(qx[g] == 0.f && qy[g] == 0.f);
    }
  }
  int coincident[MAX_RESULTS] = {0};
  for (int g = 0; g < MAX_RESULTS; ++g)
    for (int k = 0; k < g; ++k)
      if (valid[k] && qx[k] == qx[g] && qy[k] == qy[g]) coincident[g] = 1;
  for (int g = 0; g < MAX_RESULTS; ++g) valid[g] = valid[g] && !coincident[g];

  float lo[MAX_RESULTS], hi[MAX_RESULTS];
  uint32_t lo_min[MAX_RESULTS], hi_min[MAX_RESULTS];
  int has_lo[MAX_RESULTS], has_hi[MAX_RESULTS], kept[MAX_RESULTS];
  for (int g = 0; g < MAX_RESULTS; ++g) {
    int infeasible = 0;
    has_lo[g] = has_hi[g] = 0;
    lo_min[g] = hi_min[g] = NONE;
    lo[g] = hi[g] = 0.f;
    for (int k = 0; k < MAX_RESULTS && valid[g]; ++k) {
      if (!valid[k] || k == g) continue;
      const float c = qx[g] * qy[k] - qy[g] * qx[k];
      const float b = (qx[k] * qx[k] + qy[k] * qy[k]) - (qx[g] * qx[k] + qy[g] * qy[k]);
      if (c == 0.f) {
        if (b < 0.f) infeasible = 1;
        continue;
      }
      const float t = b / c;
      if (c > 0.f) {
        if (!has_hi[g] || t < hi[g]) { hi[g] = t; hi_min[g] = index[k]; has_hi[g] = 1; }
        else if (t == hi[g] && index[k] < hi_min[g]) hi_min[g] = index[k];
      } else {
        if (!has_lo[g] || t > lo[g]) { lo[g] = t; lo_min[g] = index[k]; has_lo[g] = 1; }
        else if (t == lo[g] && index[k] < lo_min[g]) lo_min[g] = index[k];
      }
    }
    kept[g] = valid[g] && !infeasible;
    if (kept[g] && has_lo[g] && has_hi[g] && !(lo[g] < hi[g])) {
      const uint32_t a = i < index[g] ? i : index[g];
      const uint32_t b = lo_min[g] < hi_min[g] ? lo_min[g] : hi_min[g];
      kept[g] = lo[g] == hi[g] && a < b;
    }
  }
  uint32_t next[MAX_RESULTS];
  for (int g = 0; g < MAX_RESULTS; ++g) {
    next[g] = NONE;
    if (!kept[g] || !has_hi[g]) continue;
    float bx = 0.f, by = 0.f;
    for (int k = 0; k < MAX_RESULTS; ++k) {
      if (!kept[k] || k == g) continue;
      const float c = qx[g] * qy[k] - qy[g] * qx[k];
      const float b = (qx[k] * qx[k] + qy[k] * qy[k]) - (qx[g] * qx[k] + qy[g] * qy[k]);
      if (!(c > 0.f) || b / c != hi[g]) continue;
      if (next[g] == NONE || qx[k] * by - qy[k] * bx > 0.f) { next[g] = index[k]; bx = qx[k]; by = qy[k]; }
    }
  }
  int total = 0;
  uint32_t pairs[MAX_RESULTS][2];
  for (int g = 0; g < MAX_RESULTS; ++g) {
    if (next[g] == NONE) continue;
    int predecessors = 0;
    for (int k = 0; k < MAX_RESULTS; ++k) predecessors += next[k] == next[g];
    if (predecessors != 1) continue;
    pairs[total][0] = index[g];
    pairs[total][1] = next[g];
    ++total;
  }
  if (total > m->umbrella_cap) return 1;
  memcpy(m->umbrella + (uint64_t)i * m->umbrella_cap * 2, pairs, sizeof(uint32_t) * 2 * total);
  m->umbrella_count[i] = total;
  return 0;
}

static uint32_t successor(const Mesh* m, uint32_t x, uint32_t y) {
  const uint32_t* row = m->umbrella + (uint64_t)x * m->umbrella_cap * 2;
  for (uint32_t t = 0; t < m->umbrella_count[x]; ++t)
    if (row[2 * t] == y) return row[2 * t + 1];
  return NONE;
}

static int angle_too_large(const Mesh* m, const float* g, const float* h) {
  const float d = dot3(g, h);
  const float l = sqrtf(dot3(g, g) * dot3(h, h));
  return d < m->cos_triangle * l;
}

static void sub3(const float* a, const float* b, float* out) {
  for (int c = 0; c < 3; ++c) out[c] = a[c] - b[c];
}

static int triangle_ok(const Mesh* m, uint32_t i, uint32_t x, uint32_t y) {
  if (successor(m, x, y) != i || successor(m, y, i) != x) return 0;
  uint32_t o = i, p = x, q = y;
  if (x < o && x < y) { o = x; p = y; q = i; }
  else if (y < o && y < x) { o = y; p = i; q = x; }
  float no[3];
  if (!unit_normal(m, o, no)) return 0;
  float po[3], pp[3], pq[3], e1[3], e2[3], g[3], h[3];
  position(m, o, po);
  position(m, p, pp);
  position(m, q, pq);
  sub3(pp, po, e1);
  sub3(pq, po, e2);
  const float n[3] = {e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]};
  if (!(dot3(n, no) > 0.f)) return 0;
  if (angle_too_large(m, e1, e2)) return 0;
  sub3(pq, pp, g); sub3(po, pp, h);
  if (angle_too_large(m, g, h)) return 0;
  sub3(po, pq, g); sub3(pp, pq, h);
  if (angle_too_large(m, g, h)) return 0;
  return 1;
}

/* Returns the triangle count; writes up to `capacity` triangles and the four stats. umbrella / umbrella_count are
 * caller scratch of n x cap x 2 and n words (returned for inspection). */
uint64_t mw_triangulate(const float* rows, uint64_t stride, uint32_t n, float factor, float max_normal_deg,
                        float max_triangle_deg, int umbrella_cap, uint32_t* umbrella, uint32_t* umbrella_count,
                        uint32_t* triangles, uint64_t capacity, uint64_t* stats) {
  const unsigned int csr = _mm_getcsr();
  _mm_setcsr(csr | 0x8040);   /* FTZ | DAZ */
  Mesh m = {rows, stride, n, 0, NULL, umbrella_cap, umbrella, umbrella_count, 0.f};
  m.by_x = (uint32_t*)malloc(sizeof(uint32_t) * (n ? n : 1));
  for (uint32_t i = 0; i < n; ++i)
    if (present(&m, i) && isfinite(at(&m, ROWS_SMOOTH_X, i))) m.by_x[m.present_count++] = i;
  g_sort_mesh = &m;
  qsort(m.by_x, m.present_count, sizeof(uint32_t), x_cmp);
  const float f2 = factor * factor;
  const float cos_normal = (float)cos((double)max_normal_deg * (M_PI / 180.0));
  m.cos_triangle = (float)cos((double)max_triangle_deg * (M_PI / 180.0));
  uint64_t* keys = (uint64_t*)malloc(sizeof(uint64_t) * (n ? n : 1));
  uint64_t overflows = 0, meshed = 0, boundary = 0, count = 0;
  for (uint32_t i = 0; i < n; ++i) overflows += build_umbrella(&m, i, f2, cos_normal, keys);
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t* row = umbrella + (uint64_t)i * umbrella_cap * 2;
    int touched = 0;
    for (uint32_t t = 0; t < umbrella_count[i]; ++t) {
      const uint32_t a = row[2 * t], b = row[2 * t + 1];
      if (!triangle_ok(&m, i, a, b)) continue;
      touched = 1;
      if (i < a && i < b) {
        if (count < capacity) {
          triangles[3 * count] = i;
          triangles[3 * count + 1] = a;
          triangles[3 * count + 2] = b;
        }
        ++count;
      }
      const uint32_t w = successor(&m, a, i);
      if (w == NONE || !triangle_ok(&m, a, i, w)) ++boundary;
    }
    meshed += touched;
  }
  free(keys);
  free(m.by_x);
  stats[0] = count;
  stats[1] = meshed;
  stats[2] = boundary;
  stats[3] = overflows;
  _mm_setcsr(csr);
  return count;
}
