// integrate_walk.c — TEST INFRASTRUCTURE: a sequential restatement of one Integrate() AFTER association.
//
// Given the state before the frame, the frame's rasters and the association rasters a run produced (supporting
// surfel, count, conflicting surfel, first depth), everything else the frame does is a plain function: merge flags,
// integrated / replaced / merged rows, neighbour links, new-surfel flags, indices and rows. This file states that
// function slot by slot from the reference (cuda_surfel_reconstruction_kernels.cu, "kernels.cu" below):
//
//   merge                    kernels.cu:1857-2043 (decisions on the state before the frame)
//   integrate or conflict    kernels.cu:741-982, per-surfel driver :1000-1142
//   neighbour update         kernels.cu:1197-1380, detach pass :1420-1437 over the slots that existed before
//   new-surfel flags         kernels.cu:90-111, creation :133-231
//
// It has no visible list, no gather levels, no update list and no short cuts: every slot walks every gate in the
// reference's order. Arithmetic: IEEE single operations in the order sm_math.cuh documents, built with
// -ffp-contract=off, denormals flushed as the kernels flush them. The SFU steps (rcp, rsqrt, sqrt) are replaced by
// correctly rounded results; tests/integrate_walk.py derives what that costs and how `clear` and the bounds are
// defined.
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

#define INVALID 0xFFFFFFFFu
#define EPS 1.1920929e-7f /* 2^-23 */

enum { ROW_X = 0, ROW_SX = 3, ROW_CONF = 6, ROW_R2 = 7, ROW_NX = 8, ROW_CREATED = 17, ROW_STAMP = 18, ROW_N0 = 19,
       ROW_COLOR = 24, ROW_COUNT = 25 };

// Named mutations: each is one subtle error of the kind a kernel rewrite makes.
enum {
  MUT_DROP_SECONDARY = 1 << 0,        // drop the secondary pixel when the primary cannot touch the surfel
  MUT_RATIO_GE = 1 << 1,              // >= for > at the 1.44 / 0.694 radius-ratio gates
  MUT_MERGE_ACTIVE_WINDOW = 1 << 2,   // test the active window in the merge
  MUT_SECOND_INTO_ORIGINAL = 1 << 3,  // integrate the second pixel into the original surfel state
  MUT_NO_DEPTH_REREAD = 1 << 4,       // keep the old pixel's depth when the surfel moved into another pixel
  MUT_FIRST_FARTHEST = 1 << 5,        // replace the LAST of several equally far slots (>= for >)
  MUT_KEEP_LINKS = 1 << 6,            // keep the old links after a replacement
  MUT_RAW_POSITIONS = 1 << 7,         // neighbours' raw instead of smooth positions at creation
  MUT_NO_DETACH = 1 << 8,             // forget the detach flag of a merged slot
  MUT_STALE_CANDIDATES = 1 << 9,      // neighbour update reads the candidates' positions from before the frame
};

// Branch counters; tests/integrate_walk.py reads the names from this list.
enum Branch {
  B_MEAS_ZERO, B_CONFLICT_FIRST_EQ, B_CONFLICT_FIRST_NE, B_OCCLUDED, B_BACKFACING, B_NORMAL_TEST_RUN, B_NORMAL_TEST_FAIL,
  B_RADIUS_NEG, B_RADIUS_ZERO, B_SEC_LEFT, B_SEC_DOWN, B_SEC_UP, B_SEC_RIGHT, B_SEC_BORDER, B_SEC_PX1_QUIRK,
  B_MERGE_SELF, B_MERGE_INVALID, B_MERGE_PARTNER_MERGED, B_MERGE_RATIO_HI_IN, B_MERGE_RATIO_HI_OUT, B_MERGE_RATIO_LO_IN,
  B_MERGE_RATIO_LO_OUT, B_MERGE_DISTANCE, B_MERGE_ANGLE, B_MERGE_OUTSIDE_WINDOW, B_MERGE_CHAIN, B_MERGED,
  B_CONF_DECREMENT, B_REPLACE, B_REPLACE_THEN_SECOND, B_INTEGRATE_ONCE, B_INTEGRATE_TWICE, B_COUNT_0, B_COUNT_1,
  B_COUNT_2, B_COUNT_3, B_COUNT_7, B_CLAMP, B_NO_CLAMP, B_COLOR_HALF, B_DETACH_CLEARED, B_RADIUS_MIN,
  B_CREATED_THIS_FRAME, B_INACTIVE,
  B_NU_MOVED_PIXEL, B_NU_CZ_NEG, B_NU_BORDER, B_NU_OCCLUDED, B_NU_BACKFACING, B_NU_SCALE, B_NU_SELF, B_NU_ALREADY,
  B_NU_SAME_TWICE, B_NU_FULL_TIE, B_NU_INVALID_SLOT, B_NU_COMPETE, B_NU_TOO_FAR, B_NU_DOT, B_NU_INSERT, B_NU_DETACHED,
  B_CR_BORDER, B_CR_SUPPORTED, B_CR_CONFLICT, B_CR_EXIST_IN, B_CR_EXIST_OUT, B_CR_NEW_IN, B_CR_NEW_OUT, B_CR_N0,
  B_CR_N1, B_CR_N2, B_CR_N3, B_CR_N4, B_CR_SMOOTH_FAR,
  B_NUM
};

enum { ST_UNCLEAR = 1, ST_LINKS_UNCLEAR = 2, ST_TOUCHED = 4, ST_REPLACED = 8, ST_INTEGRATED = 16, ST_MERGE_UNCLEAR = 32,
       ST_MERGE_CHAIN = 64 };

typedef struct {
  int32_t width, height;
  float fx, fy, cx, cy;
  float depth_scaling, sensor_noise_factor, max_surfel_confidence, radius_factor, normal_threshold_deg;
  int32_t active_window;
  u32 frame_index;
  float global_T_local[12], local_T_global[12];
  u32 mutations;
} iw_params;

typedef struct {
  const iw_params* p;
  float fx_inv, fy_inv, cx_inv, cy_inv, inv_depth_scaling, cos_threshold, radius_factor_squared;
  u64 n, stride;
  float* rows;             // [25, stride], state after the frame
  const float* before;     // [25, stride_before]
  u64 stride_before;
  const u16 *depth_pre, *depth;
  const float *normals, *radius;
  const u8* color;
  const u32 *supporting, *counts, *conflicting;
  const float* first;
  u8* status;
  float *pbound, *nbound, *cbound;
  u32 *color_lo, *color_hi;
  u64* branch;
} Walk;

#define R(row, i) w->rows[(u64)(row) * w->stride + (i)]
#define RU(row, i) ((u32*)w->rows)[(u64)(row) * w->stride + (i)]
#define R0(row, i) w->before[(u64)(row) * w->stride_before + (i)]
#define CNT(b) (w->branch[b]++)
#define MUT(m) (w->p->mutations & (m))

// ---- arithmetic (sm_math.cuh) ---------------------------------------------------------------------------------
static inline float ftz(float a) { return fabsf(a) < FLT_MIN ? copysignf(0.f, a) : a; }
static inline float fmul(float a, float b) { return ftz(ftz(a) * ftz(b)); }
static inline float fadd(float a, float b) { return ftz(ftz(a) + ftz(b)); }
static inline float fsub(float a, float b) { return fadd(a, -b); }
static inline float ffma(float a, float b, float c) { return ftz(fmaf(ftz(a), ftz(b), ftz(c))); }
static inline float frcp(float a) { return ftz((float)(1.0 / (double)ftz(a))); }
static inline float frsqrt(float a) { return ftz((float)(1.0 / sqrt((double)ftz(a)))); }
static inline float fsqrt(float a) { return ftz((float)sqrt((double)ftz(a))); }
static inline float u2f(u32 a) { return (float)a; }
static inline int f2i(float a) {
  if (!(a == a)) return 0;
  if (a >= 2147483648.f) return INT32_MAX;
  if (a <= -2147483648.f) return INT32_MIN;
  return (int)ftz(a);
}
static inline u32 f2u(float a) {
  if (!(a > 0.f)) return 0;
  if (a >= 4294967296.f) return 0xFFFFFFFFu;
  return (u32)ftz(a);
}
// v moved by k units in the last place (k = 0: v itself). A reciprocal of a power of two is exact on the SFU too.
static inline float nudge(float v, int k) {
  if (k == 0 || v == 0.f || !isfinite(v)) return v;
  u32 b;
  memcpy(&b, &v, 4);
  if ((b & 0x7FFFFFu) == 0 && k != 0) return v;
  b += (u32)k;
  memcpy(&v, &b, 4);
  return v;
}
static inline float trow(const float* m, int r, float x, float y, float z) {
  float t = fmul(y, m[4 * r + 1]);
  t = ffma(x, m[4 * r + 0], t);
  t = ffma(z, m[4 * r + 2], t);
  return fadd(t, m[4 * r + 3]);
}
static inline float rrow(const float* m, int r, float x, float y, float z) {
  float t = fmul(y, m[4 * r + 1]);
  t = ffma(x, m[4 * r + 0], t);
  return ffma(z, m[4 * r + 2], t);
}
static inline float sqnorm(float x, float y, float z) { return ffma(z, z, ffma(x, x, fmul(y, y))); }
static inline float dot3(float ax, float ay, float az, float bx, float by, float bz) {
  return ffma(az, bz, ffma(ax, bx, fmul(ay, by)));
}
static inline float fmax3(float a, float b, float c) { return fmaxf(fabsf(a), fmaxf(fabsf(b), fabsf(c))); }

static inline int is_active(u32 stamp, u32 frame, int window) { return (int)stamp > (int)(frame - (u32)window); }

// ---- projection (kernels.cu:1491-1549) ------------------------------------------------------------------------
typedef struct { int px, py, in_image, has2, ox, oy, side; } Proj;

static Proj project_k(const Walk* w, float x, float y, float z, int k) {
  const iw_params* p = w->p;
  Proj q;
  const float inv_z = nudge(frcp(z), k);
  const float u = ffma(fmul(x, inv_z), p->fx, p->cx), v = ffma(fmul(y, inv_z), p->fy, p->cy);
  q.px = f2i(u);
  q.py = f2i(v);
  q.in_image = !(u < 0.f || v < 0.f || q.px < 0 || q.py < 0 || q.px >= p->width || q.py >= p->height);
  q.has2 = 0; q.ox = q.px; q.oy = q.py; q.side = -1;
  if (!q.in_image) return q;
  const float xf = fsub(u, (float)q.px), yf = fsub(v, (float)q.py);
  if (xf < yf) {
    if (xf < fadd(-yf, 1.0f)) { q.side = 0; if (q.px > 1) { q.has2 = 1; q.ox = q.px - 1; } }      // note: > 1, not > 0
    else { q.side = 1; if (q.py < p->height - 1) { q.has2 = 1; q.oy = q.py + 1; } }
  } else {
    if (xf < fadd(-yf, 1.0f)) { q.side = 2; if (q.py > 0) { q.has2 = 1; q.oy = q.py - 1; } }
    else { q.side = 3; if (q.px < p->width - 1) { q.has2 = 1; q.ox = q.px + 1; } }
  }
  return q;
}

// The projection, and whether it is the same for every reciprocal within 2 ulp.
static Proj project(const Walk* w, float x, float y, float z, int* clear) {
  const Proj q = project_k(w, x, y, z, 0);
  for (int k = -2; k <= 2; ++k) {
    const Proj t = project_k(w, x, y, z, k);
    if (t.px != q.px || t.py != q.py || t.in_image != q.in_image || t.has2 != q.has2 || t.ox != q.ox || t.oy != q.oy) *clear = 0;
  }
  return q;
}

static inline float measurement_normal_z(float nx, float ny) { return fsqrt(fmaxf(0.f, ffma(-ny, ny, ffma(-nx, nx, 1.0f)))); }

// ---- merge (kernels.cu:1857-2043) -----------------------------------------------------------------------------
// Decided on the state before the frame. Returns 1 to merge; *clear = 0 if an SFU result within 2 ulp could change it.
static int consider_merge(Walk* w, u32 i, int* clear) {
  const iw_params* p = w->p;
  const float r2 = R0(ROW_R2, i);
  if (!(r2 >= 0.f)) { CNT(B_RADIUS_NEG); return 0; }
  if (MUT(MUT_MERGE_ACTIVE_WINDOW) && !is_active(((const u32*)w->before)[(u64)ROW_STAMP * w->stride_before + i], p->frame_index, p->active_window)) return 0;
  const float gx = R0(ROW_X, i), gy = R0(ROW_X + 1, i), gz = R0(ROW_X + 2, i);
  const float z = trow(p->local_T_global, 2, gx, gy, gz);
  if (!(z > 0.f)) return 0;
  const float x = trow(p->local_T_global, 0, gx, gy, gz), y = trow(p->local_T_global, 1, gx, gy, gz);
  const Proj q = project(w, x, y, z, clear);
  if (!q.in_image) return 0;
  const int pix = q.py * p->width + q.px;
  const float md = fmul(u2f(w->depth_pre[pix]), w->inv_depth_scaling);
  if (!(md > 0.f)) return 0;
  const float first = w->first[pix];
  if (first < fmul(md, fadd(-p->sensor_noise_factor, 1.0f))) return 0;
  if (z > fmul(fadd(p->sensor_noise_factor, 1.0f), md)) return 0;
  const float nx = R0(ROW_NX, i), ny = R0(ROW_NX + 1, i), nz = R0(ROW_NX + 2, i);
  const float lnx = rrow(p->local_T_global, 0, nx, ny, nz), lny = rrow(p->local_T_global, 1, nx, ny, nz),
              lnz = rrow(p->local_T_global, 2, nx, ny, nz);
  if (fmul(frsqrt(sqnorm(x, y, z)), ffma(z, lnz, ffma(x, lnx, fmul(y, lny)))) > 0.f) return 0;
  if (md < z) {
    const float mnx = w->normals[2 * pix], mny = w->normals[2 * pix + 1];
    const float s = measurement_normal_z(mnx, mny);
    const int fail = ffma(-lnz, s, ffma(lnx, mnx, fmul(lny, mny))) < w->cos_threshold;
    for (int k = -2; k <= 2; k += 4) {
      if ((ffma(-lnz, nudge(s, k), ffma(lnx, mnx, fmul(lny, mny))) < w->cos_threshold) != fail) *clear = 0;
    }
    if (fail) return 0;
  }
  const u32 other = w->supporting[pix];
  if (other == i) { CNT(B_MERGE_SELF); return 0; }
  if (other == INVALID) { CNT(B_MERGE_INVALID); return 0; }
  if (r2 == 0.f) CNT(B_RADIUS_ZERO);
  const float o2 = R0(ROW_R2, other);
  if (o2 < 0.f) CNT(B_MERGE_PARTNER_MERGED);
  const float hi = 1.4400000572204589844f, lo = 0.69444441795349121094f;
  const float rcp = frcp(o2);
  const float ratio = fmul(r2, rcp);
  for (int k = -2; k <= 2; ++k) {
    const float t = fmul(r2, nudge(rcp, k));
    if ((t > hi) != (ratio > hi) || (t < lo) != (ratio < lo) || (t >= hi) != (ratio >= hi) || (t <= lo) != (ratio <= lo)) *clear = 0;
  }
  const int ratio_out = MUT(MUT_RATIO_GE) ? (ratio >= hi || ratio <= lo) : (ratio > hi || ratio < lo);
  if (ratio > 1.f && fabsf(ratio - hi) < 0.03f) CNT(ratio_out ? B_MERGE_RATIO_HI_OUT : B_MERGE_RATIO_HI_IN);
  if (ratio < 1.f && fabsf(ratio - lo) < 0.015f) CNT(ratio_out ? B_MERGE_RATIO_LO_OUT : B_MERGE_RATIO_LO_IN);
  if (ratio_out) return 0;
  const float d2 = sqnorm(fsub(gx, R0(ROW_X, other)), fsub(gy, R0(ROW_X + 1, other)), fsub(gz, R0(ROW_X + 2, other)));
  if (d2 > fmul(fadd(r2, o2), 0.03125f)) { CNT(B_MERGE_DISTANCE); return 0; }
  if (dot3(nx, ny, nz, R0(ROW_NX, other), R0(ROW_NX + 1, other), R0(ROW_NX + 2, other)) < 0.93968999385833740234f) {
    CNT(B_MERGE_ANGLE);
    return 0;
  }
  if (!is_active(((const u32*)w->before)[(u64)ROW_STAMP * w->stride_before + i], p->frame_index, p->active_window)) CNT(B_MERGE_OUTSIDE_WINDOW);
  CNT(B_MERGED);
  return 1;
}

// ---- integrate or conflict (kernels.cu:741-982) ---------------------------------------------------------------
typedef struct {
  float x, y, z, conf, r2, nx, ny, nz, sx, sy, sz;
  u32 color, color_lo, color_hi, created;
  int replaced, touched, stamped, integrated, unclear;
  float pbound, nbound, cbound;
} Surfel;

static u32 blend_channel(float m, float weight, float conf, float old, float norm) {
  return f2u(ffma(norm, ffma(m, weight, fmul(conf, old)), 0.5f)) & 0xFFu;
}

static void integrate_or_conflict(Walk* w, u32 i, int x, int y, float cx, float cy, float cz, Surfel* s) {
  const iw_params* p = w->p;
  const int pix = y * p->width + x;
  const float md = fmul(u2f(w->depth[pix]), w->inv_depth_scaling);
  if (!(md > 0.f)) { CNT(B_MEAS_ZERO); return; }
  int integrate = 1, conflicting = 0;
  const float first = w->first[pix];
  if (first < fmul(md, fadd(-p->sensor_noise_factor, 1.0f))) {
    CNT(first == cz ? B_CONFLICT_FIRST_EQ : B_CONFLICT_FIRST_NE);
    if (first == cz && w->conflicting[pix] == i) conflicting = 1;
    integrate = 0;
  }
  if (!integrate && !conflicting) return;
  if (cz > fmul(fadd(p->sensor_noise_factor, 1.0f), md)) { if (integrate) CNT(B_OCCLUDED); integrate = 0; }
  if (!integrate && !conflicting) return;

  const float lx = fmul(md, ffma((float)x, w->fx_inv, w->cx_inv)), ly = fmul(md, ffma((float)y, w->fy_inv, w->cy_inv));
  const float* G = p->global_T_local;
  const float gx = trow(G, 0, lx, ly, md), gy = trow(G, 1, lx, ly, md), gz = trow(G, 2, lx, ly, md);
  const float mnx = w->normals[2 * pix], mny = w->normals[2 * pix + 1], mnz = -measurement_normal_z(mnx, mny);
  const float gnx = rrow(G, 0, mnx, mny, mnz), gny = rrow(G, 1, mnx, mny, mnz), gnz = rrow(G, 2, mnx, mny, mnz);

  if (conflicting) {
    const float conf = fadd(s->conf, -1.0f);
    if (s->cbound > 0.f && fabsf(conf) <= 4.f * s->cbound) s->unclear = 1;
    if (conf <= 0.f) {
      CNT(B_REPLACE);
      s->x = s->sx = gx; s->y = s->sy = gy; s->z = s->sz = gz;
      s->nx = gnx; s->ny = gny; s->nz = gnz;
      s->color = s->color_lo = s->color_hi = w->color[3 * pix] | (w->color[3 * pix + 1] << 8) | (w->color[3 * pix + 2] << 16) | (1u << 24);
      s->r2 = w->radius[pix];
      s->conf = 1.0f;
      s->created = p->frame_index;
      s->stamped = s->replaced = 1;
      s->pbound = s->cbound = 0.f;
      s->nbound = 4.f * EPS;  // the square root of the measurement normal
    } else {
      CNT(B_CONF_DECREMENT);
      s->conf = conf;
    }
    s->touched = 1;
  }
  if (!integrate) return;

  const float* L = p->local_T_global;
  const float lnx = rrow(L, 0, s->nx, s->ny, s->nz), lny = rrow(L, 1, s->nx, s->ny, s->nz), lnz = rrow(L, 2, s->nx, s->ny, s->nz);
  const float facing = ffma(cz, lnz, ffma(cx, lnx, fmul(cy, lny)));
  if (s->nbound > 0.f && fabsf(facing) <= 8.f * s->nbound * fmax3(cx, cy, cz)) s->unclear = 1;
  if (fmul(frsqrt(sqnorm(cx, cy, cz)), facing) > 0.f) { CNT(B_BACKFACING); return; }
  if (md < cz) {
    CNT(B_NORMAL_TEST_RUN);
    const float d = ffma(gnz, s->nz, ffma(gnx, s->nx, fmul(gny, s->ny)));
    if (fabsf(d - w->cos_threshold) <= 8.f * EPS + 4.f * s->nbound) s->unclear = 1;
    if (d < w->cos_threshold) { CNT(B_NORMAL_TEST_FAIL); return; }
  }
  if (s->r2 < 0.f) return;
  if (s->r2 == 0.f) CNT(B_RADIUS_ZERO);

  const u32 count = w->counts[pix];
  CNT(count == 0 ? B_COUNT_0 : count == 1 ? B_COUNT_1 : count == 2 ? B_COUNT_2 : count == 3 ? B_COUNT_3 : B_COUNT_7);
  const float weight = frcp(u2f(count > 1u ? count : 1u));
  if (!(s->created < p->frame_index)) { CNT(s->replaced ? B_REPLACE_THEN_SECOND : B_CREATED_THIS_FRAME); return; }
  const float conf = s->conf;
  const float cw = fadd(weight, conf);
  if (cw < p->max_surfel_confidence) { CNT(B_NO_CLAMP); s->conf = cw; } else { CNT(B_CLAMP); s->conf = p->max_surfel_confidence; }
  const float norm = frcp(cw);
  const float scale = fmaxf(fmax3(gx, gy, gz), fmax3(s->x, s->y, s->z));
  s->x = fmul(norm, ffma(gx, weight, fmul(conf, s->x)));
  s->y = fmul(norm, ffma(gy, weight, fmul(conf, s->y)));
  s->z = fmul(norm, ffma(gz, weight, fmul(conf, s->z)));
  const float nx = ffma(gnx, weight, fmul(conf, s->nx)), ny = ffma(gny, weight, fmul(conf, s->ny)),
              nz = ffma(gnz, weight, fmul(conf, s->nz));
  const float nn = frsqrt(ffma(nz, nz, ffma(nx, nx, fmul(ny, ny))));
  s->nx = fmul(nx, nn); s->ny = fmul(ny, nn); s->nz = fmul(nz, nn);
  if (w->radius[pix] < s->r2) CNT(B_RADIUS_MIN);
  s->r2 = fminf(s->r2, w->radius[pix]);
  if ((s->color >> 24) & 1u) CNT(B_DETACH_CLEARED);
  // colour: the emulated value, and the range it sweeps when weight and normalisation each move by up to 2 ulp
  u32 value = 0, lo = 0, hi = 0;
  for (int c = 0; c < 3; ++c) {
    const float m = u2f(w->color[3 * pix + c]);
    u32 clo = 255, chi = 0;
    for (u32 old = (s->color_lo >> (8 * c)) & 0xFFu; old <= ((s->color_hi >> (8 * c)) & 0xFFu); ++old) {
      for (int kw = -2; kw <= 2; kw += 2) for (int kn = -2; kn <= 2; kn += 2) {
        const u32 t = blend_channel(m, nudge(weight, kw), conf, u2f(old), nudge(norm, kn));
        if (t < clo) clo = t;
        if (t > chi) chi = t;
      }
    }
    const float old = u2f((s->color >> (8 * c)) & 0xFFu);
    value |= blend_channel(m, weight, conf, old, norm) << (8 * c);
    lo |= clo << (8 * c);
    hi |= chi << (8 * c);
    const double exact = ((double)m * weight + (double)conf * old) * norm;
    if (fabs(exact - floor(exact) - 0.5) < 1e-9) CNT(B_COLOR_HALF);
  }
  s->color = value; s->color_lo = lo; s->color_hi = hi;
  s->pbound += 8.f * EPS * scale;
  s->nbound += 16.f * EPS;
  s->cbound += 8.f * EPS * cw;
  s->stamped = s->touched = 1;
  s->integrated += 1;
}

static void integrate_slot(Walk* w, u32 i) {
  const iw_params* p = w->p;
  if (!is_active(RU(ROW_STAMP, i), p->frame_index, p->active_window)) { CNT(B_INACTIVE); return; }
  const float gx0 = R(ROW_X, i), gy0 = R(ROW_X + 1, i), gz0 = R(ROW_X + 2, i);
  const float z = trow(p->local_T_global, 2, gx0, gy0, gz0);
  if (!(z > 0.f)) return;
  const float x = trow(p->local_T_global, 0, gx0, gy0, gz0), y = trow(p->local_T_global, 1, gx0, gy0, gz0);
  int clear = 1;
  const Proj q = project(w, x, y, z, &clear);
  if (!q.in_image) return;
  if (R(ROW_R2, i) < 0.f) return;   // kernels.cu:1050
  const int side_branch[4] = {B_SEC_LEFT, B_SEC_DOWN, B_SEC_UP, B_SEC_RIGHT};
  CNT(side_branch[q.side]);
  if (!q.has2) CNT(q.side == 0 && q.px == 1 ? B_SEC_PX1_QUIRK : B_SEC_BORDER);
  Surfel s;
  memset(&s, 0, sizeof s);
  s.x = gx0; s.y = gy0; s.z = gz0;
  s.conf = R(ROW_CONF, i); s.r2 = R(ROW_R2, i);
  s.nx = R(ROW_NX, i); s.ny = R(ROW_NX + 1, i); s.nz = R(ROW_NX + 2, i);
  s.color = s.color_lo = s.color_hi = RU(ROW_COLOR, i);
  s.created = RU(ROW_CREATED, i);
  s.unclear = !clear;
  const Surfel original = s;
  integrate_or_conflict(w, i, q.px, q.py, x, y, z, &s);
  const int touched_by_primary = s.touched;
  if (q.has2 && !(MUT(MUT_DROP_SECONDARY) && !touched_by_primary)) {
    if (MUT(MUT_SECOND_INTO_ORIGINAL) && s.integrated) {
      Surfel t = original;
      integrate_or_conflict(w, i, q.ox, q.oy, x, y, z, &t);
      if (t.touched) s = t;
    } else {
      integrate_or_conflict(w, i, q.ox, q.oy, x, y, z, &s);
    }
  }
  if (s.integrated) CNT(s.integrated == 2 ? B_INTEGRATE_TWICE : B_INTEGRATE_ONCE);
  if (s.unclear) { w->status[i] |= ST_UNCLEAR; w->pbound[i] = INFINITY; }
  if (!s.touched) return;
  R(ROW_X, i) = s.x; R(ROW_X + 1, i) = s.y; R(ROW_X + 2, i) = s.z;
  R(ROW_CONF, i) = s.conf; R(ROW_R2, i) = s.r2;
  R(ROW_NX, i) = s.nx; R(ROW_NX + 1, i) = s.ny; R(ROW_NX + 2, i) = s.nz;
  RU(ROW_COLOR, i) = s.color;
  w->color_lo[i] = s.color_lo; w->color_hi[i] = s.color_hi;
  if (s.stamped) RU(ROW_STAMP, i) = p->frame_index;
  if (s.replaced) {
    RU(ROW_CREATED, i) = p->frame_index;
    R(ROW_SX, i) = s.sx; R(ROW_SX + 1, i) = s.sy; R(ROW_SX + 2, i) = s.sz;
    if (!MUT(MUT_KEEP_LINKS)) for (int k = 0; k < 4; ++k) RU(ROW_N0 + k, i) = INVALID;
  }
  w->status[i] |= ST_TOUCHED | (s.replaced ? ST_REPLACED : 0) | (s.integrated ? ST_INTEGRATED : 0);
  if (!s.unclear) w->pbound[i] = s.pbound;
  w->nbound[i] = s.nbound;
  w->cbound[i] = s.cbound;
}

// ---- neighbour update (kernels.cu:1197-1380) ------------------------------------------------------------------
// a > b, on values that carry an error of up to `tol`: *clear = 0 when the error could decide.
static inline int gt(float a, float b, float tol, int* clear) {
  if (tol > 0.f && !(fabsf(a - b) > tol)) *clear = 0;
  return a > b;
}

static void candidate_position(const Walk* w, u32 q, float* x, float* y, float* z) {
  if (w->p->mutations & MUT_STALE_CANDIDATES) { *x = w->before[(u64)ROW_X * w->stride_before + q]; *y = w->before[(u64)(ROW_X + 1) * w->stride_before + q]; *z = w->before[(u64)(ROW_X + 2) * w->stride_before + q]; return; }
  *x = w->rows[(u64)ROW_X * w->stride + q]; *y = w->rows[(u64)(ROW_X + 1) * w->stride + q]; *z = w->rows[(u64)(ROW_X + 2) * w->stride + q];
}

static void update_neighbors(Walk* w, u32 i, const u32* links_in, u32* links_out) {
  const iw_params* p = w->p;
  for (int k = 0; k < 4; ++k) links_out[k] = links_in[k];
  if (!is_active(RU(ROW_STAMP, i), p->frame_index, p->active_window)) return;
  const float gx = R(ROW_X, i), gy = R(ROW_X + 1, i), gz = R(ROW_X + 2, i);
  const float pb = w->pbound[i];
  int clear = 1;
  const float cz = trow(p->local_T_global, 2, gx, gy, gz);
  if (pb > 0.f && !(fabsf(cz) > 4.f * pb)) clear = 0;
  if (!(cz > 0.f)) { CNT(B_NU_CZ_NEG); goto done; }
  {
    const float cx = trow(p->local_T_global, 0, gx, gy, gz), cy = trow(p->local_T_global, 1, gx, gy, gz);
    const Proj q = project(w, cx, cy, cz, &clear);
    if (pb > 0.f) {  // a moved surfel: its pixel is only certain away from the pixel's edges
      const float inv = frcp(cz);
      const float u = ffma(fmul(cx, inv), p->fx, p->cx), v = ffma(fmul(cy, inv), p->fy, p->cy);
      const float tol = 8.f * pb * fmaxf(fabsf(p->fx), fabsf(p->fy)) * inv * (1.f + fabsf(cx * inv) + fabsf(cy * inv)) + 8.f * EPS * (fabsf(u) + fabsf(v));
      if (!(u - floorf(u) > tol && ceilf(u) - u > tol && v - floorf(v) > tol && ceilf(v) - v > tol)) clear = 0;
    }
    const int x = q.px, y = q.py;
    if (x < 1 || y < 1 || x >= p->width - 1 || y >= p->height - 1) { CNT(B_NU_BORDER); goto done; }
    int pix = y * p->width + x;
    if (w->status[i] & ST_TOUCHED) {
      const float ox = R0(ROW_X, i), oy = R0(ROW_X + 1, i), oz = R0(ROW_X + 2, i);
      const float z0 = trow(p->local_T_global, 2, ox, oy, oz);
      int dummy = 1;
      const Proj q0 = project(w, trow(p->local_T_global, 0, ox, oy, oz), trow(p->local_T_global, 1, ox, oy, oz), z0, &dummy);
      if (q0.px != x || q0.py != y) {
        CNT(B_NU_MOVED_PIXEL);
        if (MUT(MUT_NO_DEPTH_REREAD) && q0.in_image) pix = q0.py * p->width + q0.px;
      }
    }
    const float md = fmul(u2f(w->depth[pix]), w->inv_depth_scaling);
    pix = y * p->width + x;
    if (gt(cz, fmul(md, fadd(p->sensor_noise_factor, 1.0f)), 4.f * pb, &clear)) { CNT(B_NU_OCCLUDED); goto done; }
    const float nx = R(ROW_NX, i), ny = R(ROW_NX + 1, i), nz = R(ROW_NX + 2, i);
    const float lnx = rrow(p->local_T_global, 0, nx, ny, nz), lny = rrow(p->local_T_global, 1, nx, ny, nz),
                lnz = rrow(p->local_T_global, 2, nx, ny, nz);
    const float facing = ffma(cz, lnz, ffma(cx, lnx, fmul(cy, lny)));
    if ((w->nbound[i] > 0.f || pb > 0.f) && !(fabsf(facing) > 8.f * (w->nbound[i] * fmax3(cx, cy, cz) + pb))) clear = 0;
    if (fmul(frsqrt(sqnorm(cx, cy, cz)), facing) > 0.f) { CNT(B_NU_BACKFACING); goto done; }
    const float r2 = R(ROW_R2, i);
    if (r2 < 0.f) goto done;
    {
      const float rcp = frcp(r2), obs = w->radius[pix];
      const int out = fmul(obs, rcp) > 2.25f;
      for (int k = -2; k <= 2; ++k) if ((fmul(obs, nudge(rcp, k)) > 2.25f) != out) clear = 0;
      if (out) { CNT(B_NU_SCALE); goto done; }
    }
    float dist[4];
    u32 nbr[4];
    float qb_max = 0.f;
    int full = 1;
    for (int k = 0; k < 4; ++k) {
      nbr[k] = links_in[k];
      if (nbr[k] == INVALID) { dist[k] = INFINITY; full = 0; CNT(B_NU_INVALID_SLOT); continue; }
      float qx, qy, qz;
      candidate_position(w, nbr[k], &qx, &qy, &qz);
      dist[k] = sqnorm(fsub(gx, qx), fsub(gy, qy), fsub(gz, qz));
      qb_max = fmaxf(qb_max, w->pbound[nbr[k]]);
    }
    if (full && (dist[0] == dist[1] || dist[1] == dist[2] || dist[2] == dist[3] || dist[0] == dist[2] || dist[0] == dist[3] || dist[1] == dist[3])) CNT(B_NU_FULL_TIE);
    const float max_d2 = fmul(r2, w->radius_factor_squared);
    const int dxs[4] = {-1, 1, 0, 0}, dys[4] = {0, 0, -1, 1};
    u32 seen[4];
    int inserted = 0;
    for (int dir = 0; dir < 4; ++dir) {
      const u32 c = w->supporting[(y + dys[dir]) * p->width + x + dxs[dir]];
      seen[dir] = c;
      if (c == INVALID) continue;
      if (c == i) { CNT(B_NU_SELF); continue; }
      for (int e = 0; e < dir; ++e) if (seen[e] == c) { CNT(B_NU_SAME_TWICE); break; }
      float qx, qy, qz;
      candidate_position(w, c, &qx, &qy, &qz);
      const float d2 = sqnorm(fsub(qx, gx), fsub(qy, gy), fsub(qz, gz));
      const float err = pb + fmaxf(qb_max, w->pbound[c]);   // of a position difference
      const float tol = err > 0.f ? 8.f * err * (sqrtf(fmaxf(d2, max_d2)) + err) : 0.f;
      if (gt(d2, max_d2, tol, &clear)) { CNT(B_NU_TOO_FAR); continue; }
      const float nd = dot3(nx, ny, nz, w->rows[(u64)ROW_NX * w->stride + c], w->rows[(u64)(ROW_NX + 1) * w->stride + c], w->rows[(u64)(ROW_NX + 2) * w->stride + c]);
      if (!gt(nd, 0.f, 4.f * (w->nbound[i] + w->nbound[c]), &clear)) { CNT(B_NU_DOT); continue; }
      int best = -1;
      float best_d2 = -1.f;
      for (int k = 0; k < 4; ++k) {
        if (c == nbr[k]) { best = -1; CNT(B_NU_ALREADY); break; }
        const float tk = err > 0.f && isfinite(dist[k]) && isfinite(best_d2) ? 8.f * err * (sqrtf(fmaxf(dist[k], best_d2)) + err) : 0.f;
        const int farther = MUT(MUT_FIRST_FARTHEST) ? !gt(best_d2, dist[k], tk, &clear) : gt(dist[k], best_d2, tk, &clear);
        if (farther) { best = k; best_d2 = dist[k]; }
      }
      if (best >= 0) {
        const float tb = err > 0.f && isfinite(best_d2) ? 8.f * err * (sqrtf(fmaxf(d2, best_d2)) + err) : 0.f;
        if (gt(best_d2, d2, tb, &clear)) {
          if (inserted & (1 << best)) CNT(B_NU_COMPETE);
          nbr[best] = c; dist[best] = d2;
          inserted |= 1 << best;
          CNT(B_NU_INSERT);
        }
      }
    }
    for (int k = 0; k < 4; ++k) links_out[k] = nbr[k];
  }
done:
  if (!clear) w->status[i] |= ST_LINKS_UNCLEAR;
}

// ---- the frame ------------------------------------------------------------------------------------------------
// rows: [25, stride] with the state before the frame in the first n columns; on return the state after it (n_after
// columns). Returns n_after; counts = {n_after, merges of this frame, unclear merge decisions}.
u64 iw_integrate(const iw_params* p, u64 n, u64 stride, float* rows, const u16* depth_pre, const u16* depth,
                 const float* normals, const float* radius, const u8* color, const u32* supporting, const u32* counts,
                 const u32* conflicting, const float* first, u8* merge_flag, u8* new_flag, u32* new_index, u8* status,
                 float* pbound, float* nbound, float* cbound, u32* color_lo, u32* color_hi, u64* branch, u64* out_counts,
                 float* scratch_before) {
  Walk walk, *w = &walk;
  memset(w, 0, sizeof *w);
  w->p = p;
  // kernels.cc:68-74, cuda_surfel_reconstruction.cc:158, kernels.cc:261 (host expressions)
  w->fx_inv = 1.0f / p->fx; w->fy_inv = 1.0f / p->fy;
  w->cx_inv = -(p->cx - 0.5f) / p->fx; w->cy_inv = -(p->cy - 0.5f) / p->fy;
  w->inv_depth_scaling = 1.0f / p->depth_scaling;
  w->cos_threshold = cosf(M_PI / 180.0f * p->normal_threshold_deg);
  w->radius_factor_squared = p->radius_factor * p->radius_factor;
  w->n = n; w->stride = stride; w->rows = rows;
  w->before = scratch_before; w->stride_before = n ? n : 1;
  for (int r = 0; r < ROW_COUNT; ++r) memcpy(scratch_before + (u64)r * w->stride_before, rows + (u64)r * stride, n * sizeof(float));
  w->depth_pre = depth_pre; w->depth = depth; w->normals = normals; w->radius = radius; w->color = color;
  w->supporting = supporting; w->counts = counts; w->conflicting = conflicting; w->first = first;
  w->status = status; w->pbound = pbound; w->nbound = nbound; w->cbound = cbound; w->color_lo = color_lo; w->color_hi = color_hi;
  w->branch = branch;
  const int P = p->width * p->height;

  // merge: decisions on the state before the frame, then applied (kernels.cu:1986-1989)
  u64 merges = 0, unclear_merges = 0;
  for (u64 i = 0; i < n; ++i) {
    int clear = 1;
    merge_flag[i] = (u8)consider_merge(w, (u32)i, &clear);
    if (!clear) { status[i] |= ST_UNCLEAR | ST_MERGE_UNCLEAR; pbound[i] = INFINITY; ++unclear_merges; }
    merges += merge_flag[i];
  }
  for (u64 i = 0; i < n; ++i) {
    color_lo[i] = color_hi[i] = RU(ROW_COLOR, i);
    if (!merge_flag[i]) continue;
    RU(ROW_STAMP, i) = 0;
    R(ROW_R2, i) = -1.0f;
    if (!MUT(MUT_NO_DETACH)) RU(ROW_COLOR, i) = (RU(ROW_COLOR, i) & 0x00FFFFFFu) | (1u << 24);
    color_lo[i] = color_hi[i] = RU(ROW_COLOR, i);
  }
  // integration, each slot on its own rows
  for (u64 i = 0; i < n; ++i) integrate_slot(w, (u32)i);
  // neighbour update on the integrated state: a slot writes only its own links, so the pass is order-free
  for (u64 i = 0; i < n; ++i) {
    u32 in[4], out[4];
    for (int k = 0; k < 4; ++k) in[k] = RU(ROW_N0 + k, i);
    update_neighbors(w, (u32)i, in, out);
    for (int k = 0; k < 4; ++k) RU(ROW_N0 + k, i) = out[k];
  }
  // detach pass over the slots that existed before the frame (kernels.cu:1420-1437)
  for (u64 i = 0; i < n; ++i) {
    for (int k = 0; k < 4; ++k) {
      const u32 q = RU(ROW_N0 + k, i);
      if (q == INVALID) continue;
      if ((w->status[q] & ST_UNCLEAR) && !(w->status[i] & ST_UNCLEAR)) w->status[i] |= ST_LINKS_UNCLEAR;
      if ((RU(ROW_COLOR, q) >> 24) == 1u) { RU(ROW_N0 + k, i) = INVALID; CNT(B_NU_DETACHED); }
    }
  }
  // new-surfel flags and raster-order indices (kernels.cu:90-111; exclusive scan)
  u32 running = 0;
  for (int seq = 0; seq < P; ++seq) {
    const int y = seq / p->width, x = seq - y * p->width;
    const int interior = x >= 1 && y >= 1 && x < p->width - 1 && y < p->height - 1;
    u8 flag = 0;
    if (depth[seq] > 0) {
      if (!interior) CNT(B_CR_BORDER);
      else if (supporting[seq] != INVALID) CNT(B_CR_SUPPORTED);
      else if (conflicting[seq] != INVALID) CNT(B_CR_CONFLICT);
      else flag = 1;
    }
    new_flag[seq] = flag;
    new_index[seq] = running;
    running += flag;
  }
  const u64 n_after = n + running;
  if (n_after > stride) return n_after;   // the caller sized the rows too small
  // creation (kernels.cu:133-231)
  for (int seq = 0; seq < P; ++seq) {
    if (!new_flag[seq]) continue;
    const int y = seq / p->width, x = seq - y * p->width;
    const u64 i = n + new_index[seq];
    const float depth_m = fmul(u2f(depth[seq]), w->inv_depth_scaling);
    const float lx = fmul(depth_m, ffma((float)x, w->fx_inv, w->cx_inv)), ly = fmul(depth_m, ffma((float)y, w->fy_inv, w->cy_inv));
    const float* G = p->global_T_local;
    const float gx = trow(G, 0, lx, ly, depth_m), gy = trow(G, 1, lx, ly, depth_m), gz = trow(G, 2, lx, ly, depth_m);
    const float mnx = normals[2 * seq], mny = normals[2 * seq + 1], mnz = -measurement_normal_z(mnx, mny);
    const float r2 = radius[seq];
    const float max_d2 = fmul(r2, w->radius_factor_squared);
    const int dxs[4] = {-1, 1, 0, 0}, dys[4] = {0, 0, -1, 1};
    float sum_x = 0.f, sum_y = 0.f, sum_z = 0.f;
    int count_plus_1 = 1, clear = 1;
    for (int r = 0; r < ROW_COUNT; ++r) R(r, i) = 0.f;
    for (int dir = 0; dir < 4; ++dir) {
      const int nseq = (y + dys[dir]) * p->width + x + dxs[dir];
      u32 q = supporting[nseq];
      if (q != INVALID) {
        const float d2 = sqnorm(fsub(R(ROW_X, q), gx), fsub(R(ROW_X + 1, q), gy), fsub(R(ROW_X + 2, q), gz));
        const float err = pbound[q];
        if (gt(d2, max_d2, err > 0.f ? 8.f * err * (sqrtf(fmaxf(d2, max_d2)) + err) : 0.f, &clear)) {
          q = INVALID;
          CNT(B_CR_EXIST_OUT);
        } else {
          const int raw = MUT(MUT_RAW_POSITIONS) ? ROW_X : ROW_SX;
          const float qsx = R(raw, q), qsy = R(raw + 1, q), qsz = R(raw + 2, q);
          if (sqnorm(fsub(qsx, R(ROW_X, q)), fsub(qsy, R(ROW_X + 1, q)), fsub(qsz, R(ROW_X + 2, q))) > fmul(0.25f, max_d2)) CNT(B_CR_SMOOTH_FAR);
          sum_x = fadd(sum_x, qsx); sum_y = fadd(sum_y, qsy); sum_z = fadd(sum_z, qsz);
          ++count_plus_1;
          CNT(B_CR_EXIST_IN);
        }
      } else if (new_flag[nseq] == 1) {
        const float diff = ffma(-u2f(depth[nseq]), w->inv_depth_scaling, depth_m);
        if (!(fmul(diff, diff) > max_d2)) { q = (u32)(n + new_index[nseq]); CNT(B_CR_NEW_IN); } else CNT(B_CR_NEW_OUT);
      }
      RU(ROW_N0 + dir, i) = q;
    }
    CNT(B_CR_N0 + count_plus_1 - 1);
    R(ROW_X, i) = gx; R(ROW_X + 1, i) = gy; R(ROW_X + 2, i) = gz;
    R(ROW_NX, i) = rrow(G, 0, mnx, mny, mnz); R(ROW_NX + 1, i) = rrow(G, 1, mnx, mny, mnz); R(ROW_NX + 2, i) = rrow(G, 2, mnx, mny, mnz);
    RU(ROW_COLOR, i) = color[3 * seq] | (color[3 * seq + 1] << 8) | (color[3 * seq + 2] << 16);
    color_lo[i] = color_hi[i] = RU(ROW_COLOR, i);
    R(ROW_CONF, i) = 1.0f;
    RU(ROW_CREATED, i) = p->frame_index;
    RU(ROW_STAMP, i) = p->frame_index;
    R(ROW_R2, i) = r2;
    const float rcp = frcp((float)count_plus_1);
    R(ROW_SX, i) = fmul(fadd(gx, sum_x), rcp); R(ROW_SX + 1, i) = fmul(fadd(gy, sum_y), rcp); R(ROW_SX + 2, i) = fmul(fadd(gz, sum_z), rcp);
    status[i] = clear ? 0 : (ST_UNCLEAR | ST_LINKS_UNCLEAR);
    nbound[i] = 4.f * EPS;
    cbound[i] = 0.f;
    // the smooth mean passes through one reciprocal: 2 ulp of it plus the rounding of the product
    pbound[i] = count_plus_1 == 1 ? 0.f : 4.f * EPS * fmax3(R(ROW_SX, i), R(ROW_SX + 1, i), R(ROW_SX + 2, i));
  }
  // chains: a merges into b while b merges into c (the reference applies merges in place; see the Python module)
  for (u64 i = 0; i < n; ++i) {
    if (!merge_flag[i]) continue;
    const float gx = R0(ROW_X, i), gy = R0(ROW_X + 1, i), gz = R0(ROW_X + 2, i);
    const float z = trow(p->local_T_global, 2, gx, gy, gz);
    int dummy = 1;
    const Proj q = project(w, trow(p->local_T_global, 0, gx, gy, gz), trow(p->local_T_global, 1, gx, gy, gz), z, &dummy);
    const u32 other = supporting[q.py * p->width + q.px];
    if (other != INVALID && other < n && merge_flag[other]) { CNT(B_MERGE_CHAIN); status[i] |= ST_MERGE_CHAIN; }
  }
  out_counts[0] = n_after; out_counts[1] = merges; out_counts[2] = unclear_merges;
  return n_after;
}
