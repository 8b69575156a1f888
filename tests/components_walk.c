/* components_walk.c — TEST INFRASTRUCTURE: a plain-C restatement of sm_mesh_components (rules C1-C7 of
 * include/surfel_b200.h) by a different algorithm from the kernels: the undirected edges of all triangles are sorted,
 * each run of one edge lists the triangles on it, and the pieces are flood-filled breadth-first, starting from each
 * triangle not yet reached in triangle order (so the numbers of C3 come out directly). Built by
 * tests/components_walk.py with -ffp-contract=off; every double operation is rounded on its own. The kernels run with
 * fp32 denormals flushed to zero (-ftz=true), which flushes an fp32 corner before its conversion to double. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ROWS_SMOOTH_X 3
#define ROW_RADIUS_SQUARED 7

typedef struct {   /* sm_component_params */
  uint64_t min_triangles;
  double min_area;
  uint64_t keep_largest;
} Params;

typedef struct {   /* sm_component_stats */
  uint64_t triangles_in, triangles_out, components, components_kept, largest_triangles;
  double largest_area;
} Stats;

typedef struct {   /* sm_mesh_component */
  uint64_t triangles;
  double area;
  float lo[3], hi[3];
  uint32_t first_triangle;
  int32_t kept;
} Component;

typedef struct { uint64_t key; uint32_t t; } Edge;

static int by_edge(const void* x, const void* y) {
  const Edge* a = (const Edge*)x;
  const Edge* b = (const Edge*)y;
  if (a->key != b->key) return a->key < b->key ? -1 : 1;
  return a->t < b->t ? -1 : (a->t > b->t);
}

/* totalOrder(a, b): a <= b in IEEE 754 totalOrder, by sign and magnitude. */
static int total_le(float a, float b) {
  uint32_t x, y;
  memcpy(&x, &a, 4);
  memcpy(&y, &b, 4);
  const int sx = x >> 31, sy = y >> 31;
  if (sx != sy) return sx;   /* negative <= positive */
  return sx ? (x >= y) : (x <= y);
}

static double widen(float f) {
  if (fpclassify(f) == FP_SUBNORMAL) f = copysignf(0.f, f);
  return (double)f;
}

/* C4: q_t. */
static uint64_t area_units(const float* pa, const float* pb, const float* pc) {
  double a[3], e1[3], e2[3];
  for (int k = 0; k < 3; ++k) {
    a[k] = widen(pa[k]);
    e1[k] = widen(pb[k]) - a[k];
    e2[k] = widen(pc[k]) - a[k];
  }
  const double gx = e1[1] * e2[2] - e1[2] * e2[1];
  const double gy = e1[2] * e2[0] - e1[0] * e2[2];
  const double gz = e1[0] * e2[1] - e1[1] * e2[0];
  const double gg = (gx * gx + gy * gy) + gz * gz;
  const double area = 0.5 * sqrt(gg);
  if (!isfinite(area)) return 0;
  const double scaled = area * 0x1p30;
  if (scaled >= 0x1p36) return 1ull << 36;
  return (uint64_t)nearbyint(scaled);
}

typedef struct { uint64_t q; uint32_t number; } Rank;

static int by_rank(const void* x, const void* y) {
  const Rank* a = (const Rank*)x;
  const Rank* b = (const Rank*)y;
  if (a->q != b->q) return a->q > b->q ? -1 : 1;
  return a->number < b->number ? -1 : (a->number > b->number);
}

/* Returns triangles_out, or -1 (a bad corner) / -2 (a repeated corner) with nothing written. out, labels and table
 * have room for `count` entries. */
int64_t cw_components(const float* rows, uint64_t stride, uint32_t n, const uint32_t* tri, uint64_t count,
                      const Params* p, uint32_t* out, int32_t* labels, Component* table, Stats* stats) {
  memset(stats, 0, sizeof(*stats));
  int bad = 0, repeated = 0;
  for (uint64_t t = 0; t < count; ++t) {
    const uint32_t* c = tri + 3 * t;
    for (int k = 0; k < 3; ++k)
      if (c[k] >= n || !(rows[ROW_RADIUS_SQUARED * stride + c[k]] > 0.f)) bad = 1;
    if (c[0] == c[1] || c[1] == c[2] || c[2] == c[0]) repeated = 1;
  }
  if (bad) return -1;
  if (repeated) return -2;
  if (count == 0) return 0;

  /* C2: the triangles on each undirected edge */
  Edge* edges = (Edge*)malloc(sizeof(Edge) * 3 * count);
  for (uint64_t t = 0; t < count; ++t)
    for (int k = 0; k < 3; ++k) {
      uint32_t a = tri[3 * t + k], b = tri[3 * t + (k + 1) % 3];
      if (a > b) { const uint32_t s = a; a = b; b = s; }
      edges[3 * t + k].key = ((uint64_t)a << 32) | b;
      edges[3 * t + k].t = (uint32_t)t;
    }
  qsort(edges, 3 * count, sizeof(Edge), by_edge);
  uint64_t* run_of = (uint64_t*)malloc(sizeof(uint64_t) * 3 * count);   /* by (t, k): its run's first sorted index */
  uint32_t* seen_k = (uint32_t*)calloc(count, sizeof(uint32_t));
  for (uint64_t i = 0, start = 0; i < 3 * count; ++i) {
    if (i > 0 && edges[i].key != edges[i - 1].key) start = i;
    const uint32_t t = edges[i].t;
    const uint64_t slot = 3 * (uint64_t)t + seen_k[t]++;   /* a triangle's own edges are distinct (no repeated corner) */
    run_of[slot] = start;
  }

  /* C3: breadth-first flood fill from each unreached triangle in triangle order */
  int32_t* label = (int32_t*)malloc(sizeof(int32_t) * count);
  for (uint64_t t = 0; t < count; ++t) label[t] = -1;
  uint32_t* queue = (uint32_t*)malloc(sizeof(uint32_t) * count);
  uint32_t pieces = 0;
  for (uint64_t s = 0; s < count; ++s) {
    if (label[s] >= 0) continue;
    uint64_t head = 0, tail = 0;
    label[s] = (int32_t)pieces;
    queue[tail++] = (uint32_t)s;
    while (head < tail) {
      const uint32_t t = queue[head++];
      for (int k = 0; k < 3; ++k) {
        const uint64_t start = run_of[3 * (uint64_t)t + k];
        for (uint64_t i = start; i < 3 * count && edges[i].key == edges[start].key; ++i) {
          const uint32_t u = edges[i].t;
          if (label[u] < 0) { label[u] = (int32_t)pieces; queue[tail++] = u; }
        }
      }
    }
    ++pieces;
  }

  /* C4, C5 */
  Component* comp = (Component*)calloc(pieces, sizeof(Component));
  uint64_t* Q = (uint64_t*)calloc(pieces, sizeof(uint64_t));
  for (uint64_t t = 0; t < count; ++t) {
    Component* e = comp + label[t];
    float P[3][3];
    for (int k = 0; k < 3; ++k)
      for (int d = 0; d < 3; ++d) P[k][d] = rows[(ROWS_SMOOTH_X + d) * stride + tri[3 * t + k]];
    if (e->triangles == 0) {
      e->first_triangle = (uint32_t)t;
      for (int d = 0; d < 3; ++d) { e->lo[d] = P[0][d]; e->hi[d] = P[0][d]; }
    }
    e->triangles += 1;
    Q[label[t]] += area_units(P[0], P[1], P[2]);
    for (int k = 0; k < 3; ++k)
      for (int d = 0; d < 3; ++d) {
        if (!total_le(e->lo[d], P[k][d])) e->lo[d] = P[k][d];
        if (!total_le(P[k][d], e->hi[d])) e->hi[d] = P[k][d];
      }
  }

  /* C6 */
  Rank* rank = (Rank*)malloc(sizeof(Rank) * pieces);
  for (uint32_t i = 0; i < pieces; ++i) { rank[i].q = Q[i]; rank[i].number = i; }
  qsort(rank, pieces, sizeof(Rank), by_rank);
  uint32_t* rank_of = (uint32_t*)malloc(sizeof(uint32_t) * pieces);
  for (uint32_t r = 0; r < pieces; ++r) rank_of[rank[r].number] = r;
  const double units = nearbyint(p->min_area * 0x1p30);
  const int none = !(units < 0x1p64);   /* every Q is below 2^64 */
  const uint64_t min_q = none ? 0 : (uint64_t)units;
  uint64_t kept = 0;
  for (uint32_t i = 0; i < pieces; ++i) {
    Component* e = comp + i;
    e->area = (double)Q[i] * 0x1p-30;
    e->kept = !none && e->triangles >= p->min_triangles && Q[i] >= min_q &&
              (p->keep_largest == 0 || rank_of[i] < p->keep_largest);
    kept += e->kept ? 1 : 0;
  }

  /* C7 */
  uint64_t written = 0;
  for (uint64_t t = 0; t < count; ++t) {
    labels[t] = label[t];
    if (comp[label[t]].kept) {
      memcpy(out + 3 * written, tri + 3 * t, 3 * sizeof(uint32_t));
      ++written;
    }
  }
  memcpy(table, comp, sizeof(Component) * pieces);
  stats->triangles_in = count;
  stats->triangles_out = written;
  stats->components = pieces;
  stats->components_kept = kept;
  stats->largest_triangles = comp[rank[0].number].triangles;
  stats->largest_area = comp[rank[0].number].area;
  free(edges); free(run_of); free(seen_k); free(label); free(queue); free(comp); free(Q); free(rank);
  free(rank_of);
  return (int64_t)written;
}
