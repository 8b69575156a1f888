/* hole_walk.c — TEST INFRASTRUCTURE: a plain-C restatement of sm_mesh_fill_holes (rules H1-H7 of
 * include/surfel_b200.h), one step after the other, with sorted arrays where the kernels use hash tables. Built by
 * tests/hole_walk.py with -ffp-contract=off; every fp32 operation is rounded on its own, and denormals are flushed
 * to zero (MXCSR FTZ | DAZ) as the kernels do. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <xmmintrin.h>

#define ROWS_SMOOTH_X 3
#define ROW_RADIUS_SQUARED 7
#define ROW_NORMAL_X 8
#define MAX_HOLE 16
#define NONE 0xFFFFFFFFu

typedef struct {
  const float* rows;
  uint64_t stride;
  const uint64_t* edges; uint64_t edge_count;   /* input edges, sorted */
  const uint64_t* holes; uint32_t hole_count;   /* hole edges, sorted */
  float cos_normal, cos_triangle;
} Ctx;

static float at(const Ctx* c, int row, uint32_t i) { return c->rows[(uint64_t)row * c->stride + i]; }
static float dot3(const float* a, const float* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static void sub3(const float* a, const float* b, float* o) { for (int k = 0; k < 3; ++k) o[k] = a[k] - b[k]; }
static void position(const Ctx* c, uint32_t i, float* p) { for (int k = 0; k < 3; ++k) p[k] = at(c, ROWS_SMOOTH_X + k, i); }

static int unit_normal(const Ctx* c, uint32_t i, float* out) {
  float n[3];
  for (int k = 0; k < 3; ++k) n[k] = at(c, ROW_NORMAL_X + k, i);
  const float s = dot3(n, n);
  if (!(s > 0.f) || !isfinite(s)) return 0;
  const float inv = 1.f / sqrtf(s);
  for (int k = 0; k < 3; ++k) out[k] = n[k] * inv;
  return 1;
}

static uint64_t key(uint32_t tail, uint32_t head) { return ((uint64_t)tail << 32) | head; }

static int cmp_u64(const void* a, const void* b) {
  const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
  return x < y ? -1 : (x > y);
}

static uint64_t lower(const uint64_t* v, uint64_t n, uint64_t k) {
  uint64_t lo = 0, hi = n;
  while (lo < hi) { const uint64_t mid = lo + (hi - lo) / 2; if (v[mid] < k) lo = mid + 1; else hi = mid; }
  return lo;
}

static int is_edge(const Ctx* c, uint32_t a, uint32_t b) {
  const uint64_t k = key(a, b), i = lower(c->edges, c->edge_count, k);
  return i < c->edge_count && c->edges[i] == k;
}

static float cross2(const float* a, const float* b) { return a[0] * b[1] - a[1] * b[0]; }

static int half_of(const float* qu, const float* qw) {
  const float cr = cross2(qu, qw);
  if (cr < 0.f) return 0;
  if (cr > 0.f || (cr == 0.f && (qu[0] * qw[0] + qu[1] * qw[1]) < 0.f)) return 1;
  return -1;   /* also when cr is NaN */
}

/* w before w' (rule H2) */
static int before(int ha, const float* qa, int hb, const float* qb) { return ha < hb || (ha == hb && cross2(qa, qb) < 0.f); }

/* H2: the index of the successor of hole edge (u, v), or NONE. */
static uint32_t successor(const Ctx* c, uint32_t u, uint32_t v) {
  const uint32_t first = (uint32_t)lower(c->holes, c->hole_count, key(v, 0));
  uint32_t end = first;
  while (end < c->hole_count && (uint32_t)(c->holes[end] >> 32) == v) ++end;
  if (end == first) return NONE;
  if (end == first + 1) return first;
  float n[3];
  if (!unit_normal(c, v, n)) return NONE;
  const float sign = copysignf(1.f, n[2]);
  const float bf = -1.f / (sign + n[2]);
  const float bb = (n[0] * n[1]) * bf;
  const float t[3] = {1.f + ((sign * n[0]) * n[0]) * bf, sign * bb, -(sign * n[0])};
  const float s[3] = {bb, sign + (n[1] * n[1]) * bf, -n[1]};
  float pv[3], p[3], d[3];
  position(c, v, pv);
  float qu[2];
  position(c, u, p); sub3(p, pv, d);
  qu[0] = dot3(d, t); qu[1] = dot3(d, s);
  const uint32_t m = end - first;
  float (*q)[2] = (float (*)[2])malloc(sizeof(float) * 2 * m);
  int* h = (int*)malloc(sizeof(int) * m);
  uint32_t result = NONE;
  int defined = 1;
  for (uint32_t e = 0; e < m; ++e) {
    position(c, (uint32_t)c->holes[first + e], p); sub3(p, pv, d);
    q[e][0] = dot3(d, t); q[e][1] = dot3(d, s);
    h[e] = half_of(qu, q[e]);
    if (h[e] < 0) defined = 0;
  }
  for (uint32_t e = 0; e < m && defined && result == NONE; ++e) {
    int all = 1;
    for (uint32_t f = 0; f < m && all; ++f) if (f != e && !before(h[e], q[e], h[f], q[f])) all = 0;
    if (all) result = first + e;
  }
  free(q); free(h);
  return result;
}

static int angle_too_large(const Ctx* c, const float* g, const float* h) {
  const float d = dot3(g, h);
  const float l = sqrtf(dot3(g, g) * dot3(h, h));
  return d < c->cos_triangle * l;
}

/* H4 for (L[i], L[j], L[m]) of a loop of k; its weight, or +inf. */
static float weight(const Ctx* c, const uint32_t* L, int k, int i, int j, int m) {
  const int idx[3] = {i, j, m};
  const int pairs[3][2] = {{i, j}, {j, m}, {i, m}};
  for (int e = 0; e < 3; ++e) {
    const int a = pairs[e][0], b = pairs[e][1];
    const int loop_edge = b == a + 1 || (a == 0 && b == k - 1);
    if (!loop_edge && (is_edge(c, L[a], L[b]) || is_edge(c, L[b], L[a]))) return INFINITY;
  }
  float n[3][3], p[3][3];
  for (int e = 0; e < 3; ++e) {
    if (!unit_normal(c, L[idx[e]], n[e])) return INFINITY;
    position(c, L[idx[e]], p[e]);
  }
  if (!(dot3(n[0], n[1]) >= c->cos_normal) || !(dot3(n[1], n[2]) >= c->cos_normal) ||
      !(dot3(n[0], n[2]) >= c->cos_normal))
    return INFINITY;
  int o = 0;
  if (L[j] < L[i] && L[j] < L[m]) o = 1;
  else if (L[m] < L[i] && L[m] < L[j]) o = 2;
  const int x = (o + 1) % 3, y = (o + 2) % 3;
  float e1[3], e2[3], g[3], a[3], b[3];
  sub3(p[x], p[o], e1); sub3(p[y], p[o], e2);
  g[0] = e1[1] * e2[2] - e1[2] * e2[1];
  g[1] = e1[2] * e2[0] - e1[0] * e2[2];
  g[2] = e1[0] * e2[1] - e1[1] * e2[0];
  for (int e = 0; e < 3; ++e) if (!(dot3(g, n[e]) > 0.f)) return INFINITY;
  if (angle_too_large(c, e1, e2)) return INFINITY;
  sub3(p[y], p[x], a); sub3(p[o], p[x], b);
  if (angle_too_large(c, a, b)) return INFINITY;
  sub3(p[o], p[y], a); sub3(p[x], p[y], b);
  if (angle_too_large(c, a, b)) return INFINITY;
  return sqrtf(dot3(g, g));
}

typedef struct {
  uint32_t L[MAX_HOLE];
  int k;
  int tri[MAX_HOLE - 2][3];   /* loop positions, pre-order */
  int conflicting;
} Loop;

typedef struct { uint64_t key; uint32_t loop; } Diagonal;
static int cmp_diag(const void* a, const void* b) {
  const Diagonal *x = (const Diagonal*)a, *y = (const Diagonal*)b;
  return x->key < y->key ? -1 : (x->key > y->key ? 1 : (x->loop < y->loop ? -1 : (x->loop > y->loop)));
}

static uint64_t pair_key(uint32_t a, uint32_t b) { return a < b ? key(a, b) : key(b, a); }

/* Returns the fill's triangle count (writes up to `capacity` of them), or -1 / -2 / -3 for a bad corner, a repeated
 * corner, a duplicate directed edge. stats: the seven fields of sm_hole_stats. */
int64_t hw_fill_holes(const float* rows, uint64_t stride, uint32_t n, const uint32_t* tri, uint64_t count, int K,
                      float max_normal_deg, float max_triangle_deg, uint32_t* fill, uint64_t capacity,
                      uint64_t* stats) {
  const unsigned int csr = _mm_getcsr();
  _mm_setcsr(csr | 0x8040);   /* FTZ | DAZ */
  memset(stats, 0, 7 * sizeof(uint64_t));
  Ctx c = {rows, stride, NULL, 0, NULL, 0, 0.f, 0.f};
  c.cos_normal = (float)cos((double)max_normal_deg * (M_PI / 180.0));
  c.cos_triangle = (float)cos((double)max_triangle_deg * (M_PI / 180.0));
  int64_t result = 0;
  uint64_t* edges = (uint64_t*)malloc(sizeof(uint64_t) * (3 * count + 1));
  uint64_t* holes = (uint64_t*)malloc(sizeof(uint64_t) * (3 * count + 1));
  Loop* loops = NULL;
  Diagonal* diags = NULL;
  for (uint64_t t = 0; t < count; ++t) {
    const uint32_t* v = tri + 3 * t;
    for (int s = 0; s < 3; ++s)
      if (v[s] >= n || !(at(&c, ROW_RADIUS_SQUARED, v[s]) > 0.f)) { result = -1; goto done; }
    if (v[0] == v[1] || v[1] == v[2] || v[2] == v[0]) { result = -2; goto done; }
    edges[3 * t] = key(v[0], v[1]);
    edges[3 * t + 1] = key(v[1], v[2]);
    edges[3 * t + 2] = key(v[2], v[0]);
  }
  qsort(edges, 3 * count, sizeof(uint64_t), cmp_u64);
  for (uint64_t e = 1; e < 3 * count; ++e) if (edges[e] == edges[e - 1]) { result = -3; goto done; }
  c.edges = edges;
  c.edge_count = 3 * count;
  /* H1 */
  uint32_t H = 0;
  for (uint64_t e = 0; e < 3 * count; ++e) {
    const uint32_t a = (uint32_t)(edges[e] >> 32), b = (uint32_t)edges[e];
    if (!is_edge(&c, b, a)) holes[H++] = key(b, a);
  }
  qsort(holes, H, sizeof(uint64_t), cmp_u64);
  c.holes = holes;
  c.hole_count = H;
  stats[0] = H;
  loops = (Loop*)malloc(sizeof(Loop) * (H + 1));
  diags = (Diagonal*)malloc(sizeof(Diagonal) * (H + 1));
  uint32_t loop_count = 0, diag_count = 0;
  for (uint32_t h = 0; h < H; ++h) {
    /* H3: follow successors from h */
    Loop* lp = &loops[loop_count];
    uint32_t cur = h, smallest = h;
    int k = 0;
    for (int s = 1; s <= K; ++s) {
      lp->L[s - 1] = (uint32_t)(holes[cur] >> 32);
      const uint32_t next = successor(&c, (uint32_t)(holes[cur] >> 32), (uint32_t)holes[cur]);
      if (next == NONE) break;
      if (next == h) { k = s; break; }
      if (next < smallest) smallest = next;
      cur = next;
    }
    if (k == 0 || smallest != h) continue;
    int distinct = 1;
    for (int i = 0; i < k; ++i) for (int j = 0; j < i; ++j) if (lp->L[i] == lp->L[j]) distinct = 0;
    if (!distinct) continue;
    ++stats[1];
    /* H5 */
    float W[MAX_HOLE][MAX_HOLE];
    int J[MAX_HOLE][MAX_HOLE];
    for (int i = 0; i + 1 < k; ++i) W[i][i + 1] = 0.f;
    for (int d = 2; d < k; ++d)
      for (int i = 0; i + d < k; ++i) {
        const int m = i + d;
        float best = INFINITY;
        int bj = -1;
        for (int j = i + 1; j < m; ++j) {
          const float v = (W[i][j] + W[j][m]) + weight(&c, lp->L, k, i, j, m);
          if (v < best) { best = v; bj = j; }
        }
        W[i][m] = best;
        J[i][m] = bj;
      }
    if (!(W[0][k - 1] < INFINITY)) { ++stats[3]; continue; }
    lp->k = k;
    lp->conflicting = 0;
    int stack[MAX_HOLE][2], top = 0, written = 0;
    stack[top][0] = 0; stack[top][1] = k - 1; ++top;
    while (top > 0) {
      --top;
      const int i = stack[top][0], m = stack[top][1], j = J[i][m];
      if (i != 0 || m != k - 1) { diags[diag_count].key = pair_key(lp->L[i], lp->L[m]); diags[diag_count++].loop = loop_count; }
      lp->tri[written][0] = i; lp->tri[written][1] = j; lp->tri[written][2] = m; ++written;
      if (m - j >= 2) { stack[top][0] = j; stack[top][1] = m; ++top; }
      if (j - i >= 2) { stack[top][0] = i; stack[top][1] = j; ++top; }
    }
    ++loop_count;
  }
  /* H6 */
  qsort(diags, diag_count, sizeof(Diagonal), cmp_diag);
  for (uint32_t d = 1; d < diag_count; ++d)
    if (diags[d].key == diags[d - 1].key && diags[d].loop != diags[d - 1].loop)
      loops[diags[d].loop].conflicting = loops[diags[d - 1].loop].conflicting = 1;
  /* H7 (loops are already in owner order) */
  uint64_t out = 0, filled_edges = 0;
  for (uint32_t l = 0; l < loop_count; ++l) {
    const Loop* lp = &loops[l];
    if (lp->conflicting) { ++stats[4]; continue; }
    ++stats[2];
    filled_edges += lp->k;
    for (int t = 0; t < lp->k - 2; ++t, ++out) {
      const uint32_t x = lp->L[lp->tri[t][0]], y = lp->L[lp->tri[t][1]], z = lp->L[lp->tri[t][2]];
      uint32_t r[3] = {x, y, z};
      if (y < x && y < z) { r[0] = y; r[1] = z; r[2] = x; }
      else if (z < x && z < y) { r[0] = z; r[1] = x; r[2] = y; }
      if (out < capacity) memcpy(fill + 3 * out, r, sizeof(r));
    }
  }
  stats[5] = out;
  stats[6] = H - filled_edges;
  result = (int64_t)out;
done:
  if (result < 0) memset(stats, 0, 7 * sizeof(uint64_t));
  free(edges); free(holes); free(loops); free(diags);
  _mm_setcsr(csr);
  return result;
}
