/* simplify_walk.c — TEST INFRASTRUCTURE: a plain-C restatement of sm_mesh_simplify (rules S1-S8 of
 * include/surfel_b200.h), one collapse after the other, with per-slot incidence lists where the kernels sort corner
 * keys. Every round is applied twice, to two copies of the state: once in ascending and once in descending key
 * order, each collapse re-validated (same best neighbour, same cost) on the state the earlier ones left; the two
 * copies must end bit-equal (S4). Built by tests/simplify_walk.py with -ffp-contract=off; every fp32 and double
 * operation is rounded on its own. fp32 denormals are flushed to zero (MXCSR FTZ | DAZ) as the kernels do under
 * -ftz=true, which applies to fp32 operations (and fp32 inputs of conversions) only; since MXCSR's bits would flush
 * doubles too, the double arithmetic of S1, S3 (d) and S6 runs with them cleared (fp64_mode / fp32_mode). */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <xmmintrin.h>

#define ROWS_SMOOTH_X 3
#define ROW_RADIUS_SQUARED 7
#define ROW_NORMAL_X 8
#define MAX_VALENCE 32
#define NONE 0xFFFFFFFFu
#define STOP_TARGET 1
#define STOP_CONVERGED 2
#define STOP_MAX_ROUNDS 3

typedef struct {   /* sm_simplify_params */
  uint64_t target_triangles;
  double max_cost;
  float max_angle_between_normals_deg, max_triangle_angle_deg;
  int32_t max_rounds, reserved;
} Params;

typedef struct {   /* sm_simplify_stats */
  uint64_t triangles_in, triangles_out, vertices_in, vertices_out, collapses, rounds, boundary_edges;
  double max_cost_applied;
  int32_t stop_reason, reserved;
} Stats;

typedef struct { uint32_t* v; uint32_t n, cap; } List;   /* triangle positions, ascending */

typedef struct {
  uint32_t* tri;   /* [count][3], NONE: deleted */
  List* inc;       /* [n] */
  double* Q;       /* [n][10] */
} State;

typedef struct {
  const float* rows;
  uint64_t stride;
  uint32_t n, count;
  float cos_normal, cos_triangle;
  double max_cost;
} Ctx;

static void fp64_mode(void) { _mm_setcsr(_mm_getcsr() & ~0x8040u); }
static void fp32_mode(void) { _mm_setcsr(_mm_getcsr() | 0x8040u); }

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

static void list_insert(List* l, uint32_t t) {
  if (l->n == l->cap) {
    l->cap = l->cap ? 2 * l->cap : 8;
    l->v = (uint32_t*)realloc(l->v, sizeof(uint32_t) * l->cap);
  }
  uint32_t i = l->n;
  while (i > 0 && l->v[i - 1] > t) { l->v[i] = l->v[i - 1]; --i; }
  l->v[i] = t;
  ++l->n;
}

static void list_remove(List* l, uint32_t t) {
  uint32_t i = 0;
  while (i < l->n && l->v[i] != t) ++i;
  if (i == l->n) return;
  memmove(l->v + i, l->v + i + 1, sizeof(uint32_t) * (l->n - i - 1));
  --l->n;
}

/* the corners of triangle t after u, in winding order */
static void after(const uint32_t* c, uint32_t u, uint32_t* a, uint32_t* b) {
  if (c[0] == u) { *a = c[1]; *b = c[2]; }
  else if (c[1] == u) { *a = c[2]; *b = c[0]; }
  else { *a = c[0]; *b = c[1]; }
}

/* S1 */
static void add_plane(const Ctx* c, const uint32_t* t, double* q) {
  double P[3][3];
  for (int s = 0; s < 3; ++s)
    for (int k = 0; k < 3; ++k) P[s][k] = (double)at(c, ROWS_SMOOTH_X + k, t[s]);
  fp64_mode();
  double e1[3], e2[3];
  for (int k = 0; k < 3; ++k) { e1[k] = P[1][k] - P[0][k]; e2[k] = P[2][k] - P[0][k]; }
  const double gx = e1[1] * e2[2] - e1[2] * e2[1];
  const double gy = e1[2] * e2[0] - e1[0] * e2[2];
  const double gz = e1[0] * e2[1] - e1[1] * e2[0];
  const double gg = (gx * gx + gy * gy) + gz * gz;
  double k[10] = {0};
  if (gg > 0.0) {
    const double s = sqrt(gg);
    const double mx = gx / s, my = gy / s, mz = gz / s;
    const double d = -((mx * P[0][0] + my * P[0][1]) + mz * P[0][2]);
    const double kk[10] = {mx * mx, mx * my, mx * mz, mx * d, my * my, my * mz, my * d, mz * mz, mz * d, d * d};
    memcpy(k, kk, sizeof(k));
  }
  for (int j = 0; j < 10; ++j) q[j] = q[j] + k[j];
  fp32_mode();
}

static double row4(double a, double b, double c, double w, double x, double y, double z) {
  return ((a * x + b * y) + c * z) + w;
}

static double quadric_cost(const double* q, double x, double y, double z) {
  const double r0 = row4(q[0], q[1], q[2], q[3], x, y, z);
  const double r1 = row4(q[1], q[4], q[5], q[6], x, y, z);
  const double r2 = row4(q[2], q[5], q[7], q[8], x, y, z);
  const double r3 = row4(q[3], q[6], q[8], q[9], x, y, z);
  return row4(r0, r1, r2, r3, x, y, z);
}

static int angle_too_large(const Ctx* c, const float* g, const float* h) {
  const float d = dot3(g, h);
  const float l = sqrtf(dot3(g, g) * dot3(h, h));
  return d < c->cos_triangle * l;
}

/* S3 (c), geometric part, for the triangle (s[0], s[1], s[2]) */
static int triangle_ok(const Ctx* c, const uint32_t* s) {
  float n[3][3], p[3][3];
  for (int e = 0; e < 3; ++e) {
    if (!unit_normal(c, s[e], n[e])) return 0;
    position(c, s[e], p[e]);
  }
  if (!(dot3(n[0], n[1]) >= c->cos_normal) || !(dot3(n[1], n[2]) >= c->cos_normal) ||
      !(dot3(n[0], n[2]) >= c->cos_normal))
    return 0;
  int o = 0;
  if (s[1] < s[0] && s[1] < s[2]) o = 1;
  else if (s[2] < s[0] && s[2] < s[1]) o = 2;
  const int x = (o + 1) % 3, y = (o + 2) % 3;
  float e1[3], e2[3], g[3], a[3], b[3];
  sub3(p[x], p[o], e1); sub3(p[y], p[o], e2);
  g[0] = e1[1] * e2[2] - e1[2] * e2[1];
  g[1] = e1[2] * e2[0] - e1[0] * e2[2];
  g[2] = e1[0] * e2[1] - e1[1] * e2[0];
  for (int e = 0; e < 3; ++e) if (!(dot3(g, n[e]) > 0.f)) return 0;
  if (angle_too_large(c, e1, e2)) return 0;
  sub3(p[y], p[x], a); sub3(p[o], p[x], b);
  if (angle_too_large(c, a, b)) return 0;
  sub3(p[o], p[y], a); sub3(p[x], p[y], b);
  return !angle_too_large(c, a, b);
}

/* N(i) into out (distinct, any order); returns deg(i) */
static int neighbours(const State* S, uint32_t i, uint32_t* out, int cap) {
  int d = 0;
  const List* l = &S->inc[i];
  for (uint32_t k = 0; k < l->n; ++k) {
    const uint32_t* t = S->tri + 3 * (uint64_t)l->v[k];
    for (int s = 0; s < 3; ++s) {
      if (t[s] == i) continue;
      int seen = 0;
      for (int m = 0; m < d && !seen; ++m) seen = out[m] == t[s];
      if (!seen) { if (d < cap) out[d] = t[s]; ++d; }
    }
  }
  return d;
}

static int has_triangle(const State* S, uint32_t a, uint32_t b, uint32_t c) {
  const List* l = &S->inc[a];
  for (uint32_t k = 0; k < l->n; ++k) {
    const uint32_t* t = S->tri + 3 * (uint64_t)l->v[k];
    const int hb = t[0] == b || t[1] == b || t[2] == b, hc = t[0] == c || t[1] == c || t[2] == c;
    if (hb && hc) return 1;
  }
  return 0;
}

/* S3: 1 and (best v, cost) if u has a valid collapse */
static int candidate(const Ctx* c, const State* S, uint32_t u, uint32_t* best_v, double* best_cost) {
  const List* l = &S->inc[u];
  const int d = (int)l->n;
  if (d < 3 || d > MAX_VALENCE) return 0;
  uint32_t from[MAX_VALENCE], to[MAX_VALENCE], ring[MAX_VALENCE];
  for (int k = 0; k < d; ++k) after(S->tri + 3 * (uint64_t)l->v[k], u, &from[k], &to[k]);
  /* one closed fan: from (u, a, b) to (u, b, c) through all d triangles and back; then N(u) = the ring */
  int visited[MAX_VALENCE] = {0}, cur = 0;
  visited[0] = 1;
  ring[0] = from[0];
  for (int s = 1; s < d; ++s) {
    int next = -1;
    for (int k = 0; k < d; ++k) if (from[k] == to[cur]) next = k;
    if (next < 0 || visited[next]) return 0;
    visited[next] = 1;
    ring[s] = from[next];
    cur = next;
  }
  if (to[cur] != from[0]) return 0;
  uint32_t nu[2 * MAX_VALENCE];
  if (neighbours(S, u, nu, 2 * MAX_VALENCE) != d) return 0;   /* (cannot happen for one closed fan) */
  int found = 0;
  for (int k = 0; k < d; ++k) {
    const uint32_t v = ring[k], o1 = ring[(k + d - 1) % d], o2 = ring[(k + 1) % d];
    /* (a) */
    uint32_t nv[4 * MAX_VALENCE];
    const int dv = neighbours(S, v, nv, 4 * MAX_VALENCE);
    int common = 0, ok = 1;
    for (int m = 0; m < dv && m < 4 * MAX_VALENCE; ++m)
      for (int j = 0; j < d; ++j)
        if (nv[m] == ring[j]) { ++common; if (nv[m] != o1 && nv[m] != o2) ok = 0; }
    if (!ok || common != 2) continue;
    /* (b) */
    if (d + dv - 4 > MAX_VALENCE) continue;
    /* (c) */
    for (int j = 0; j < d && ok; ++j) {
      const uint32_t x = ring[j], y = ring[(j + 1) % d];
      if (x == v || y == v) continue;
      const uint32_t t[3] = {v, x, y};
      ok = triangle_ok(c, t) && !has_triangle(S, v, x, y);
    }
    if (!ok) continue;
    /* (d) */
    const double x = (double)at(c, ROWS_SMOOTH_X, v), y = (double)at(c, ROWS_SMOOTH_X + 1, v),
                 z = (double)at(c, ROWS_SMOOTH_X + 2, v);
    fp64_mode();
    double q[10];
    for (int j = 0; j < 10; ++j) q[j] = S->Q[10 * (uint64_t)u + j] + S->Q[10 * (uint64_t)v + j];
    const double e = quadric_cost(q, x, y, z);
    const double cost = e > 0.0 ? e : 0.0;
    const int better = isfinite(e) && cost <= c->max_cost &&
                       (!found || cost < *best_cost || (cost == *best_cost && v < *best_v));
    fp32_mode();
    if (better) {
      found = 1;
      *best_cost = cost;
      *best_v = v;
    }
  }
  return found;
}

static uint64_t make_key(double cost, uint32_t u) {
  float f = (float)cost;
  if (!(f >= FLT_MIN)) f = 0.f;
  uint32_t bits;
  memcpy(&bits, &f, 4);
  return ((uint64_t)bits << 32) | u;
}

/* S6 on S, after checking that u's best collapse on S is still (v, cost) */
static int apply(const Ctx* c, State* S, uint32_t u, uint32_t v, double cost) {
  uint32_t bv;
  double bc;
  if (!candidate(c, S, u, &bv, &bc) || bv != v || memcmp(&bc, &cost, sizeof(double)) != 0) return 0;
  List* l = &S->inc[u];
  const uint32_t n = l->n;
  uint32_t* mine = (uint32_t*)malloc(sizeof(uint32_t) * n);
  memcpy(mine, l->v, sizeof(uint32_t) * n);
  for (uint32_t k = 0; k < n; ++k) {
    uint32_t* t = S->tri + 3 * (uint64_t)mine[k];
    if (t[0] == v || t[1] == v || t[2] == v) {
      for (int s = 0; s < 3; ++s) list_remove(&S->inc[t[s]], mine[k]);
      t[0] = t[1] = t[2] = NONE;
    } else {
      for (int s = 0; s < 3; ++s) if (t[s] == u) t[s] = v;
      list_remove(&S->inc[u], mine[k]);
      list_insert(&S->inc[v], mine[k]);
    }
  }
  free(mine);
  fp64_mode();
  for (int j = 0; j < 10; ++j) S->Q[10 * (uint64_t)v + j] = S->Q[10 * (uint64_t)v + j] + S->Q[10 * (uint64_t)u + j];
  fp32_mode();
  return 1;
}

static void state_init(State* S, const uint32_t* tri, uint64_t count, uint32_t n) {
  S->tri = (uint32_t*)malloc(sizeof(uint32_t) * (3 * count + 1));
  memcpy(S->tri, tri, sizeof(uint32_t) * 3 * count);
  S->inc = (List*)calloc(n ? n : 1, sizeof(List));
  S->Q = (double*)calloc(10 * (uint64_t)(n ? n : 1), sizeof(double));
  for (uint64_t t = 0; t < count; ++t)
    for (int s = 0; s < 3; ++s) list_insert(&S->inc[tri[3 * t + s]], (uint32_t)t);
}

static void state_free(State* S, uint32_t n) {
  if (S->inc) for (uint32_t i = 0; i < n; ++i) free(S->inc[i].v);
  free(S->tri); free(S->inc); free(S->Q);
}

static int cmp_u64(const void* a, const void* b) {
  const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
  return x < y ? -1 : (x > y);
}

static uint64_t corner_slots(const State* S, uint32_t n) {
  uint64_t v = 0;
  for (uint32_t i = 0; i < n; ++i) v += S->inc[i].n > 0;
  return v;
}

/* Returns the output's triangle count (writes up to `capacity` of them), or -1 / -2 / -3 for a bad corner, a
 * repeated corner, a duplicate directed edge, or -4 when the two application orders of a round disagree (or a
 * collapse of a round stops being its slot's best). round_log (may be NULL): [max_rounds][2] = selected, applied.
 * last_selected (may be NULL, count entries): the keys selected by the last applied round, ascending; *last_count. */
int64_t sw_simplify(const float* rows, uint64_t stride, uint32_t n, const uint32_t* tri, uint64_t count,
                    const Params* p, uint32_t* out, uint64_t capacity, Stats* stats, uint64_t* round_log,
                    uint64_t* last_selected, uint64_t* last_count) {
  const unsigned int csr = _mm_getcsr();
  _mm_setcsr(csr | 0x8040);   /* FTZ | DAZ */
  memset(stats, 0, sizeof(Stats));
  if (last_count) *last_count = 0;
  Ctx c = {rows, stride, n, (uint32_t)count, 0.f, 0.f, p->max_cost};
  c.cos_normal = (float)cos((double)p->max_angle_between_normals_deg * (M_PI / 180.0));
  c.cos_triangle = (float)cos((double)p->max_triangle_angle_deg * (M_PI / 180.0));
  int64_t result = 0;
  uint64_t* edges = (uint64_t*)malloc(sizeof(uint64_t) * (3 * count + 1));
  State A = {0}, B = {0};
  uint64_t* keys = NULL;
  uint64_t* mark = NULL;
  uint32_t* best = NULL;
  double* cost = NULL;
  for (uint64_t t = 0; t < count; ++t)
    for (int s = 0; s < 3; ++s)
      if (tri[3 * t + s] >= n || !(at(&c, ROW_RADIUS_SQUARED, tri[3 * t + s]) > 0.f)) { result = -1; goto done; }
  for (uint64_t t = 0; t < count; ++t) {
    const uint32_t* v = tri + 3 * t;
    if (v[0] == v[1] || v[1] == v[2] || v[2] == v[0]) { result = -2; goto done; }
  }
  for (uint64_t t = 0; t < count; ++t) {
    const uint32_t* v = tri + 3 * t;
    for (int s = 0; s < 3; ++s) edges[3 * t + s] = ((uint64_t)v[s] << 32) | v[(s + 1) % 3];
  }
  qsort(edges, 3 * count, sizeof(uint64_t), cmp_u64);
  for (uint64_t e = 1; e < 3 * count; ++e) if (edges[e] == edges[e - 1]) { result = -3; goto done; }
  for (uint64_t e = 0; e < 3 * count; ++e) {
    const uint64_t rev = (edges[e] << 32) | (edges[e] >> 32);
    uint64_t lo = 0, hi = 3 * count;
    while (lo < hi) { const uint64_t mid = lo + (hi - lo) / 2; if (edges[mid] < rev) lo = mid + 1; else hi = mid; }
    if (lo == 3 * count || edges[lo] != rev) ++stats->boundary_edges;
  }
  stats->triangles_in = count;
  state_init(&A, tri, count, n);
  state_init(&B, tri, count, n);
  /* S1: the corners' lists are ascending input positions */
  for (uint32_t i = 0; i < n; ++i)
    for (uint32_t k = 0; k < A.inc[i].n; ++k) add_plane(&c, tri + 3 * (uint64_t)A.inc[i].v[k], A.Q + 10 * (uint64_t)i);
  memcpy(B.Q, A.Q, sizeof(double) * 10 * (uint64_t)(n ? n : 1));
  stats->vertices_in = corner_slots(&A, n);
  keys = (uint64_t*)malloc(sizeof(uint64_t) * (n + 1));
  mark = (uint64_t*)malloc(sizeof(uint64_t) * (n + 1));
  best = (uint32_t*)malloc(sizeof(uint32_t) * (n + 1));
  cost = (double*)malloc(sizeof(double) * (n + 1));
  uint64_t T = count;
  for (;;) {
    /* S7 */
    if (p->target_triangles > 0 && T <= p->target_triangles) { stats->stop_reason = STOP_TARGET; break; }
    if (stats->rounds >= (uint64_t)p->max_rounds) { stats->stop_reason = STOP_MAX_ROUNDS; break; }
    /* S3, S4 */
    for (uint32_t i = 0; i < n; ++i) mark[i] = ~0ull;
    for (uint32_t u = 0; u < n; ++u) {
      keys[u] = ~0ull;
      if (A.inc[u].n == 0 || !candidate(&c, &A, u, &best[u], &cost[u])) continue;
      keys[u] = make_key(cost[u], u);
      uint32_t nu[2 * MAX_VALENCE];
      const int d = neighbours(&A, u, nu, 2 * MAX_VALENCE);
      if (keys[u] < mark[u]) mark[u] = keys[u];
      for (int j = 0; j < d; ++j) if (keys[u] < mark[nu[j]]) mark[nu[j]] = keys[u];
    }
    uint64_t s = 0;
    for (uint32_t u = 0; u < n; ++u) {
      if (keys[u] == ~0ull) continue;
      uint32_t nu[2 * MAX_VALENCE];
      const int d = neighbours(&A, u, nu, 2 * MAX_VALENCE);
      int sel = mark[u] == keys[u];
      for (int j = 0; j < d; ++j) sel = sel && mark[nu[j]] == keys[u];
      if (sel) keys[s++] = keys[u];   /* (s <= u: the selected keys move to the front) */
    }
    if (s == 0) { stats->stop_reason = STOP_CONVERGED; break; }
    qsort(keys, s, sizeof(uint64_t), cmp_u64);
    /* S5 */
    uint64_t m = s;
    const int budget = p->target_triangles > 0 && T - 2 * s < p->target_triangles;
    if (budget) m = (T - p->target_triangles + 1) / 2;
    if (round_log) { round_log[2 * stats->rounds] = s; round_log[2 * stats->rounds + 1] = m; }
    if (last_selected) { memcpy(last_selected, keys, sizeof(uint64_t) * s); *last_count = s; }
    /* S6 in both orders */
    for (uint64_t i = 0; i < m; ++i) {
      const uint32_t u = (uint32_t)keys[i];
      if (!apply(&c, &A, u, best[u], cost[u])) { result = -4; goto done; }
      fp64_mode();
      if (cost[u] > stats->max_cost_applied) stats->max_cost_applied = cost[u];
      fp32_mode();
    }
    for (uint64_t i = m; i-- > 0;) {
      const uint32_t u = (uint32_t)keys[i];
      if (!apply(&c, &B, u, best[u], cost[u])) { result = -4; goto done; }
    }
    if (memcmp(A.tri, B.tri, sizeof(uint32_t) * 3 * count) != 0 ||
        memcmp(A.Q, B.Q, sizeof(double) * 10 * (uint64_t)n) != 0) { result = -4; goto done; }
    T -= 2 * m;
    stats->collapses += m;
    ++stats->rounds;
    if (budget) { stats->stop_reason = STOP_TARGET; break; }
  }
  /* S8 */
  {
    uint64_t* order = (uint64_t*)malloc(sizeof(uint64_t) * (T + 1));
    uint64_t k = 0;
    for (uint64_t t = 0; t < count; ++t) {
      const uint32_t* v = A.tri + 3 * t;
      if (v[0] == NONE) continue;
      const uint32_t o = v[0] < v[1] ? (v[0] < v[2] ? v[0] : v[2]) : (v[1] < v[2] ? v[1] : v[2]);
      order[k++] = ((uint64_t)o << 32) | t;
    }
    qsort(order, k, sizeof(uint64_t), cmp_u64);
    for (uint64_t i = 0; i < k && i < capacity; ++i) {
      const uint32_t* v = A.tri + 3 * (uint32_t)order[i];
      const uint32_t o = (uint32_t)(order[i] >> 32);
      const int r = v[0] == o ? 0 : (v[1] == o ? 1 : 2);
      for (int s = 0; s < 3; ++s) out[3 * i + s] = v[(r + s) % 3];
    }
    free(order);
    stats->triangles_out = k;
    stats->vertices_out = corner_slots(&A, n);
    result = (int64_t)k;
  }
done:
  if (result < 0) memset(stats, 0, sizeof(Stats));
  free(edges); free(keys); free(mark); free(best); free(cost);
  state_free(&A, n); state_free(&B, n);
  _mm_setcsr(csr);
  return result;
}
