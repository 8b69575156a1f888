// integrate.cu — per-frame surfel reconstruction kernels for sm_90a (SURVEY §8 a6-a13).
//
// Replaces the ~36 launches and 2 host synchronisations of
// CUDASurfelReconstruction::Integrate() (APP/cuda_surfel_reconstruction.cc:112-291) by 9
// stream-ordered launches with device-resident counters:
//
//   k_clear          a6   5 CUDABuffer::Clear launches -> one 128-bit store per pixel
//   k_project        a7   RenderMinDepthCUDAKernel (kernels.cu:1466-1557): the only sweep over
//                         ALL surfel slots (2 slots/thread, 64-bit SoA loads); splats min depth
//                         and builds the segment-ordered list of surfels that project into the
//                         image (block-local ballot/scan compaction, no global atomic)
//   k_associate      a8   AssociateSurfelsCUDAKernel (:1586-1808) over the visible list
//   k_merge          a9   MergeSurfelsCUDAKernel (:1857-2052) over the visible list; decisions
//                         are taken on the pre-merge state and applied by k_integrate
//   k_blend          a10  BlendMeasurements Start + (radius-2) Iteration kernels (:563-708) as
//                         ONE kernel: every tile finds the level sets of the two rings with a
//                         bit-parallel breadth-first search in shared memory (halo radius - 1)
//                         and then walks them level by level with the reference's arithmetic
//   k_integrate      a11  IntegrateMeasurementsCUDAKernel (:741-1142) over the visible list; also
//                         evaluates the first gates of a12 and lists the surfels that pass them
//   k_update_neighbors a12 UpdateNeighborsCUDAKernel (:1197-1380) over that list
//   k_new_surfel_scan  a13 CreateNewSurfelsCUDASerializingKernel (:90-111) + the CUB exclusive
//                         scan (:2506-2520) fused: single-pass decoupled look-back scan in
//                         raster order (stable: the k-th flagged pixel owns slot N + k)
//   k_create_surfels   a13 CreateNewSurfelsCUDACreationKernel (:133-231)
//
// UpdateNeighborsCUDARemoveReplacedNeighborsKernel (:1420-1437) is folded into the first
// regularisation sweep (regularize.cu). Arithmetic follows the reference SASS (sm_math.cuh).
//
// Deterministic where the reference is not (SURVEY §7 hard part 1): the supporting surfel
// of a pixel is "primary-pixel association before secondary, then lowest index" (the
// reference: first atomicCAS wins), merge decisions read the pre-merge state. Both are legal
// outcomes of the reference.
//
// Host side at the end of the file: IntegrateFrame (one stream, stage events) and DescribeFrameKernel (the
// launches as descriptors, which the frame graph of pipeline.cu is built from).

#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include <cooperative_groups.h>

#include "sm_kernels.cuh"

namespace cg = cooperative_groups;

namespace smb {

namespace {

#define SM_S(row, i) d.surfels[static_cast<size_t>(row) * d.stride + (i)]
#define SM_SU(row, i) reinterpret_cast<u32*>(d.surfels)[static_cast<size_t>(row) * d.stride + (i)]

constexpr int kBlock = 256;

// IsSurfelActiveForIntegration (kernels.cu:77-87).
__device__ __forceinline__ bool is_active(u32 last_update_stamp, u32 frame_index, int window) {
  return static_cast<int>(last_update_stamp) > static_cast<int>(frame_index - static_cast<u32>(window));
}

struct Projection {
  float u, v;
  int px, py;
  bool in_image;
};

// kernels.cu:1491-1500 (identical in a7/a8/a9/a11): inv = RCP(z); u = fma(x*inv, fx, cx).
__device__ __forceinline__ Projection project(const FrameParams& f, int width, int height, float x, float y, float z) {
  Projection p;
  const float inv_z = frcp(z);
  p.u = ffma(fmul(x, inv_z), f.fx, f.cx);
  p.v = ffma(fmul(y, inv_z), f.fy, f.cy);
  p.px = f2i_trunc(p.u);
  p.py = f2i_trunc(p.v);
  p.in_image = !(p.u < 0.f || p.v < 0.f || p.px < 0 || p.py < 0 || p.px >= width || p.py >= height);
  return p;
}

// Secondary pixel by the sub-pixel triangle rule (kernels.cu:1506-1549; note `px > 1`).
__device__ __forceinline__ bool secondary_pixel(const Projection& p, int width, int height, int* ox, int* oy) {
  const float x_frac = fsub(p.u, i2f(p.px));
  const float y_frac = fsub(p.v, i2f(p.py));
  if (x_frac < y_frac) {
    if (x_frac < fadd(-y_frac, 1.0f)) {
      if (p.px > 1) { *ox = p.px - 1; *oy = p.py; return true; }
      return false;
    }
    if (p.py < height - 1) { *ox = p.px; *oy = p.py + 1; return true; }
    return false;
  }
  if (x_frac < fadd(-y_frac, 1.0f)) {
    if (p.py > 0) { *ox = p.px; *oy = p.py - 1; return true; }
    return false;
  }
  if (p.px < width - 1) { *ox = p.px + 1; *oy = p.py; return true; }
  return false;
}

// -z of the measurement normal: sqrt(max(0, 1 - nx^2 - ny^2)) (kernels.cu:172,811,1656).
__device__ __forceinline__ float normal_z_abs(float nx, float ny) {
  return fsqrt_approx(fmaxf(0.f, ffma(-ny, ny, ffma(-nx, nx, 1.0f))));
}

// (1/|p|) * dot(p, R*n) > 0 test shared by a8/a9/a11/a12; returns the rotated normal.
__device__ __forceinline__ float facing_dot(const FrameParams& f, float x, float y, float z, float nx, float ny,
                                            float nz, float3* local_normal) {
  const float rs = frsqrt_approx(squared_norm(x, y, z));
  *local_normal = rotate_vec(f.local_T_global, nx, ny, nz);
  return fmul(rs, ffma(z, local_normal->z, ffma(x, local_normal->x, fmul(y, local_normal->y))));
}

// Iterates the visible list with one entry per thread: a work item is one quarter (kBlock
// positions) of a list segment; `body(pos, entry)` runs for every occupied list position.
// The kernels built on this are chains of dependent gathers, so the chain is kept short: the
// first item's segment count and list entry are fetched before the surfel count has arrived
// (any position below the list capacity is readable; the count check discards stale ones), and
// the next item's are fetched before the current one is processed.
template <typename Body>
__device__ __forceinline__ void for_each_visible(const DeviceState& d, const u32* surfel_count, Body&& body) {
  constexpr u32 kItemsPerSegment = kSegment / kBlock;
  const u32 max_items = ((d.capacity + kSegment - 1) / kSegment) * kItemsPerSegment;
  const u32 n = *surfel_count;
  u32 item = blockIdx.x;
  u32 cnt = 0;
  VisEntry e = make_uint4(0u, 0u, 0u, 0u);
  if (item < max_items) {
    cnt = d.seg_count[item / kItemsPerSegment];
    e = d.vis[static_cast<size_t>(item) * kBlock + threadIdx.x];
  }
  const u32 items = ((n + kSegment - 1) / kSegment) * kItemsPerSegment;
  while (item < items) {
    const u32 next = item + gridDim.x;
    u32 cnt_next = 0;
    VisEntry e_next = e;
    if (next < items) {
      cnt_next = d.seg_count[next / kItemsPerSegment];
      e_next = d.vis[static_cast<size_t>(next) * kBlock + threadIdx.x];
    }
    const u32 k = (item % kItemsPerSegment) * kBlock + threadIdx.x;
    if (k < cnt) body(static_cast<size_t>(item) * kBlock + threadIdx.x, e);
    item = next;
    cnt = cnt_next;
    e = e_next;
  }
}

// ---------------------------------------------------------------------------------------
// a6: clear
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kBlock) k_clear(DeviceState d) {
  pdl_prologue();
  const int n = d.width * d.height;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    d.assoc[i] = make_uint4(kInvalidIndex, kInvalidIndex, 0u, 0u);
    d.first_depth[i] = __int_as_float(0x7f800000);
    d.supported[i] = 0;
  }
}

// ---------------------------------------------------------------------------------------
// a7: projection sweep + min-depth splat + visible list
// ---------------------------------------------------------------------------------------
constexpr int kProjectBlock = 512;  // 2 slots per thread, kSegment slots per block-iteration

__global__ void __launch_bounds__(kProjectBlock) k_project(DeviceState d, FrameParams f) {
  pdl_prologue();
  if (f.skip) return;
  const TimelineScope timeline_scope(d, f.frame_index, KID_PROJECT);
  __shared__ u32 warp_totals[kProjectBlock / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  if (blockIdx.x == 0) {
    // Reset the state of this frame's new-surfel scan and neighbour-update list (run after several kernel
    // boundaries).
    const int tiles = (d.width * d.height + kSegment - 1) / kSegment;
    for (int t = threadIdx.x; t < tiles; t += blockDim.x) d.scan_state[t] = 0ull;
    if (threadIdx.x == 0) { d.counters->scan_ticket = 0; *d.upd_count = 0; }
  }

  // The rows of the first segment are requested before the surfel count has arrived (slots up to
  // the row stride are readable; `i >= n` discards them), those of the next segment before the
  // current one is processed.
  struct SlotRows { float2 X, Y, Z; uint2 T; };
  auto fetch = [&](u32 seg) {
    SlotRows r;
    const size_t base = static_cast<size_t>(seg) * kSegment + threadIdx.x * 2;
    r.X = *reinterpret_cast<const float2*>(&SM_S(SM_ROW_X, base));
    r.Y = *reinterpret_cast<const float2*>(&SM_S(SM_ROW_Y, base));
    r.Z = *reinterpret_cast<const float2*>(&SM_S(SM_ROW_Z, base));
    r.T = *reinterpret_cast<const uint2*>(&SM_SU(SM_ROW_LAST_UPDATE_STAMP, base));
    return r;
  };
  SlotRows rows = {};
  if ((static_cast<size_t>(blockIdx.x) + 1) * kSegment <= d.stride) rows = fetch(blockIdx.x);
  const u32 n = d.counters->surfel_count[f.count_slot];
  for (u32 seg = blockIdx.x; static_cast<u64>(seg) * kSegment < n; seg += gridDim.x) {
    const u32 base = seg * kSegment + threadIdx.x * 2;
    const SlotRows cur = rows;
    if (static_cast<u64>(seg + gridDim.x) * kSegment < n) rows = fetch(seg + gridDim.x);
    VisEntry e[2];
    bool visible[2] = {false, false};
    u32 cnt = 0;
    if (base < n) {
      const float xs[2] = {cur.X.x, cur.X.y}, ys[2] = {cur.Y.x, cur.Y.y}, zs[2] = {cur.Z.x, cur.Z.y};
      const u32 ts[2] = {cur.T.x, cur.T.y};
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const u32 i = base + j;
        if (i >= n) break;
        const float z = transform_row(f.local_T_global.r2, xs[j], ys[j], zs[j]);
        if (!(z > 0.f)) continue;
        const float x = transform_row(f.local_T_global.r0, xs[j], ys[j], zs[j]);
        const float y = transform_row(f.local_T_global.r1, xs[j], ys[j], zs[j]);
        const Projection p = project(f, d.width, d.height, x, y, z);
        if (!p.in_image) continue;
        const bool active = is_active(ts[j], f.frame_index, f.active_window);
        e[j] = make_uint4(i | (active ? kActiveBit : 0u), __float_as_uint(x), __float_as_uint(y), __float_as_uint(z));
        visible[j] = true;
        ++cnt;
        if (active) {
          // RenderMinDepthAtPixel (kernels.cu:1458-1464): int-punned atomicMin, positive floats.
          atomicMin(reinterpret_cast<int*>(&d.first_depth[p.py * d.width + p.px]), __float_as_int(z));
          int ox, oy;
          if (secondary_pixel(p, d.width, d.height, &ox, &oy)) {
            atomicMin(reinterpret_cast<int*>(&d.first_depth[oy * d.width + ox]), __float_as_int(z));
          }
        }
      }
    }
    // Block-wide exclusive scan of cnt (slot order is preserved inside the segment).
    u32 incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const u32 t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    if (lane == 31) warp_totals[warp] = incl;
    __syncthreads();
    u32 warp_base = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kProjectBlock / 32; ++w) {
      const u32 t = warp_totals[w];
      if (w < warp) warp_base += t;
      total += t;
    }
    VisEntry* out = d.vis + static_cast<size_t>(seg) * kSegment + warp_base + (incl - cnt);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      if (visible[j]) *out++ = e[j];
    }
    if (threadIdx.x == 0) d.seg_count[seg] = total;
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------
// a8 / a9: association and merge gates
// ---------------------------------------------------------------------------------------

// What the association gates read from one pixel.
struct PixelGate {
  float measurement_depth;  // depth_correction_factor * depth
  float first;              // first_surfel_depth
  float2 normal;
};

// Association (kernels.cu:1603-1668) gathers in two levels. Level 1 loads the depth and min-depth of the
// (up to two) pixels: five entries out of six stop at the measurement / conflict / occlusion gates, which
// need nothing else. Level 2 loads the surfel's normal and radius and the pixels' normals only for the
// rest. The gates are pure predicates, so the order decides nothing; the conflicting-surfel entry is
// written where the reference writes it.
__global__ void __launch_bounds__(kBlock) k_associate(DeviceState d, FrameParams f) {
  pdl_prologue();
  if (f.skip) return;
  const TimelineScope timeline_scope(d, f.frame_index, KID_ASSOCIATE);
  for_each_visible(d, &d.counters->surfel_count[f.count_slot], [&](size_t, const VisEntry& e) {
    if (!(e.x & kActiveBit)) return;
    const u32 idx = e.x & ~kActiveBit;
    const float x = __uint_as_float(e.y), y = __uint_as_float(e.z), z = __uint_as_float(e.w);
    const Projection p = project(f, d.width, d.height, x, y, z);
    int ox = p.px, oy = p.py;
    const bool has2 = secondary_pixel(p, d.width, d.height, &ox, &oy);
    // level 1: measurement, conflict and occlusion gates (kernels.cu:1603-1632)
    PixelGate g0, g1;
    g0.measurement_depth = fmul(u2f(row_ptr(f.depth_pre, f.depth_pre_pitch, p.py)[p.px]), f.inv_depth_scaling);
    g1.measurement_depth = fmul(u2f(row_ptr(f.depth_pre, f.depth_pre_pitch, oy)[ox]), f.inv_depth_scaling);
    g0.first = d.first_depth[p.py * d.width + p.px];
    g1.first = d.first_depth[oy * d.width + ox];
    bool pass[2] = {true, has2};
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (!pass[k]) continue;
      const PixelGate& g = k == 0 ? g0 : g1;
      const int pp = k == 0 ? p.py * d.width + p.px : oy * d.width + ox;
      if (!(g.measurement_depth > 0.f)) { pass[k] = false; continue; }
      if (g.first < fmul(g.measurement_depth, fadd(-f.sensor_noise_factor, 1.0f))) {
        if (g.first == z) d.assoc[pp].y = idx;  // this surfel is conflicting
        pass[k] = false;
        continue;
      }
      if (z > fmul(fadd(f.sensor_noise_factor, 1.0f), g.measurement_depth)) pass[k] = false;  // occluded
    }
    if (!pass[0] && !pass[1]) return;
    // level 2: the surfel's normal and radius, the normals of the pixels that are left
    const float snx = SM_S(SM_ROW_NORMAL_X, idx), sny = SM_S(SM_ROW_NORMAL_Y, idx), snz = SM_S(SM_ROW_NORMAL_Z, idx);
    const float surfel_radius_squared = SM_S(SM_ROW_RADIUS_SQUARED, idx);
    g0.normal = row_ptr(f.normals, f.normals_pitch, pass[0] ? p.py : oy)[pass[0] ? p.px : ox];
    g1.normal = row_ptr(f.normals, f.normals_pitch, pass[1] ? oy : p.py)[pass[1] ? ox : p.px];
    float3 ln;
    const float dot_angle = facing_dot(f, x, y, z, snx, sny, snz, &ln);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      if (!pass[k]) continue;
      const int pp = k == 0 ? p.py * d.width + p.px : oy * d.width + ox;
      const PixelGate& g = k == 0 ? g0 : g1;
      if (dot_angle > 0.f) continue;  // kSurfelNormalToViewingDirThreshold = 0
      if (g.measurement_depth < z) {
        const float s = normal_z_abs(g.normal.x, g.normal.y);
        const float dot2 = ffma(-ln.z, s, ffma(ln.x, g.normal.x, fmul(ln.y, g.normal.y)));
        if (dot2 < f.cos_normal_compatibility_threshold) continue;
      }
      if (!(surfel_radius_squared > 0.f)) continue;
      PixelAssoc* a = &d.assoc[pp];
      // Reference: atomicCAS(INV -> idx), first come wins. Here: the minimum of a reproducible
      // arrival key (sm_kernels.cuh, kSecondaryBit) - one of the reference's legal outcomes.
      atomicMin(&a->x, tb_encode(f.tb, idx, k == 1, static_cast<u32>(pp)));
      atomicAdd(&a->z, 1u);
      atomicAdd(reinterpret_cast<float*>(&a->w), z);
      d.supported[pp] = 1;
    }
  });
}

// a9: merge decision (kernels.cu:1857-1992); applied by k_integrate.
// A surfel can only be merged if its primary pixel has a measurement that supports it AND that pixel's
// supporting surfel is another surfel - true for a small fraction of the list. The gates are pure
// predicates (the one side effect, the conflicting-surfel entry, comes first in the reference too), so
// they are evaluated cheapest first: level 1 gathers only the surfel's radius and the pixel's depth,
// min-depth and association record (4 gathers); the 14 row gathers of the surfel and of its merge
// partner are issued together as level 2, only for the candidates. (Gathering 11 values for every entry
// made this the longest kernel of the frame at BASELINE config 3.)
__global__ void __launch_bounds__(kBlock) k_merge(DeviceState d, FrameParams f) {
  pdl_prologue();
  if (f.skip) return;
  const TimelineScope timeline_scope(d, f.frame_index, KID_MERGE);
  u32 merged_by_thread = 0;
  for_each_visible(d, &d.counters->surfel_count[f.count_slot], [&](size_t pos, const VisEntry& e) {
    const u32 idx = e.x & ~kActiveBit;  // no active-window test here (kernels.cu:2016)
    const float x = __uint_as_float(e.y), y = __uint_as_float(e.z), z = __uint_as_float(e.w);
    const Projection p = project(f, d.width, d.height, x, y, z);
    const int pp = p.py * d.width + p.px;
    // level 1
    const float surfel_radius_squared = SM_S(SM_ROW_RADIUS_SQUARED, idx);
    const float measurement_depth = fmul(u2f(row_ptr(f.depth_pre, f.depth_pre_pitch, p.py)[p.px]), f.inv_depth_scaling);
    const float first = d.first_depth[pp];
    const u32 supporting_key = d.assoc[pp].x;
    bool merged = false;
    if (surfel_radius_squared >= 0.f && measurement_depth > 0.f) {
      if (first < fmul(measurement_depth, fadd(-f.sensor_noise_factor, 1.0f))) {
        if (first == z) d.assoc[pp].y = idx;  // this surfel is conflicting (kernels.cu:1885-1889)
      } else if (!(z > fmul(fadd(f.sensor_noise_factor, 1.0f), measurement_depth))) {  // not occluded
        const u32 q = supporting_index(f.tb, supporting_key, static_cast<u32>(pp));
        if (q != idx && q != kInvalidIndex) {
          // level 2: the remaining gates and the comparison with the supporting surfel (kernels.cu:1910-1984)
          const float snx = SM_S(SM_ROW_NORMAL_X, idx), sny = SM_S(SM_ROW_NORMAL_Y, idx), snz = SM_S(SM_ROW_NORMAL_Z, idx);
          const float gx = SM_S(SM_ROW_X, idx), gy = SM_S(SM_ROW_Y, idx), gz = SM_S(SM_ROW_Z, idx);
          const float2 pixel_normal = row_ptr(f.normals, f.normals_pitch, p.py)[p.px];
          const float other_radius_squared = SM_S(SM_ROW_RADIUS_SQUARED, q);
          const float qx = SM_S(SM_ROW_X, q), qy = SM_S(SM_ROW_Y, q), qz = SM_S(SM_ROW_Z, q);
          const float qnx = SM_S(SM_ROW_NORMAL_X, q), qny = SM_S(SM_ROW_NORMAL_Y, q), qnz = SM_S(SM_ROW_NORMAL_Z, q);
          float3 ln;
          const float dot_angle = facing_dot(f, x, y, z, snx, sny, snz, &ln);
          bool same_surface = !(dot_angle > 0.f);  // kSurfelNormalToViewingDirThreshold = 0
          if (same_surface && measurement_depth < z) {
            const float s = normal_z_abs(pixel_normal.x, pixel_normal.y);
            const float dot2 = ffma(-ln.z, s, ffma(ln.x, pixel_normal.x, fmul(ln.y, pixel_normal.y)));
            same_surface = !(dot2 < f.cos_normal_compatibility_threshold);
          }
          if (same_surface) {
            const float radius_diff = fmul(surfel_radius_squared, frcp(other_radius_squared));
            const float distance_squared = squared_norm(fsub(gx, qx), fsub(gy, qy), fsub(gz, qz));
            merged = !(radius_diff > 1.4400000572204589844f || radius_diff < 0.69444441795349121094f) &&
                     !(distance_squared > fmul(fadd(surfel_radius_squared, other_radius_squared), 0.03125f)) &&
                     !(dot3(snx, sny, snz, qnx, qny, qnz) < 0.93968999385833740234f);  // cos 20 deg
          }
        }
      }
    }
    d.merge_flag[pos] = merged ? 1 : 0;
    merged_by_thread += merged ? 1u : 0u;
  });
  // Block reduction of the merge count (reference: cub::BlockReduce + atomicAdd, :2045-2051).
  merged_by_thread = __reduce_add_sync(0xffffffffu, merged_by_thread);
  __shared__ u32 warp_sums[kBlock / 32];
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = merged_by_thread;
  __syncthreads();
  if (threadIdx.x == 0) {
    u32 total = 0;
    for (int w = 0; w < kBlock / 32; ++w) total += warp_sums[w];
    if (total > 0) atomicAdd(&d.counters->merge_count, total);
  }
}

// ---------------------------------------------------------------------------------------
// a10: measurement blending, all iterations in one kernel
// ---------------------------------------------------------------------------------------
// BlendMeasurementsCUDAStartKernel + (radius - 2) x IterationKernel (kernels.cu:563-708) grow two
// rings of pixels, level by level, from (a) the supported pixels that touch a pixel without depth
// ("measurement border", distance_map) and (b) the supported pixels that touch an unsupported
// pixel ("surfel border", new_distance_map); a pixel reached at level k takes the average delta
// of its 3x3 neighbours of level k - 1. Which pixel belongs to which level does not depend on the
// blended values, so one block per tile
//   1. loads the tile + halo and builds one bit per pixel for "no depth" / "unsupported" /
//      "supported",
//   2. finds the level sets with a bit-parallel breadth-first search (one thread per 32-pixel
//      word: 3x3 dilation of the previous level AND the still unassigned eligible pixels) and
//      compacts each level into a pixel list,
//   3. walks the lists level by level (one thread per pixel, one barrier per level) doing the
//      reference's float arithmetic; the search for level k + 1 runs beside the update of level k.
// Tile 32 x 40 (VGA: 20 x 12 = 240 tiles): with the halo of a radius-12 blend the region is 64 x 62 pixels,
// 61 KB of shared memory, so TWO blocks share an SM and all tiles of a VGA frame are resident at once
// (264 block slots on the 132 SMs of an H100);
// both bit rasters of a level search (2 x 124 words) take one pass of the 256 threads. The kernel is a
// chain of ~11 barrier-separated levels with little work each: what counts is how many tiles are in
// flight per SM, not the work per tile (round 1: 80 x 32 tiles, 1 block per SM, 120 blocks).
constexpr int kBlendTileW = 32, kBlendTileH = 40;
constexpr int kBlendBlock = 256;
constexpr int kMaxBlendRadius = 64;

__host__ __device__ inline int blend_halo_y(int radius) { return radius - 1 > 1 ? radius - 1 : 1; }  // (radius - 2) iterations + the 3x3 start stencil
__host__ __device__ inline int blend_halo_x(int radius) { return (blend_halo_y(radius) + 15) & ~15; }  // 16-pixel chunks stay aligned

// 3x3 dilation of a bit raster (rows of `wpr` words, bit b of word w = pixel 32 w + b) at word
// (y, w); rows / words outside the raster read as 0.
__device__ __forceinline__ u32 dilate_word(const u32* mask, int y, int w, int rh, int wpr) {
  u32 result = 0;
#pragma unroll
  for (int dy = -1; dy <= 1; ++dy) {
    const int r = y + dy;
    if (r < 0 || r >= rh) continue;
    const u32* row = mask + r * wpr;
    const u32 centre = row[w];
    const u32 left = w > 0 ? row[w - 1] : 0u;
    const u32 right = w < wpr - 1 ? row[w + 1] : 0u;
    result |= centre | (centre << 1) | (left >> 31) | (centre >> 1) | (right << 31);
  }
  return result;
}

// Appends the pixels of the set bits of `bits` (word w of row y) to a list; `take` lanes reserve
// `__popc(bits)` slots with one atomic per warp. Must be called by all 32 lanes.
__device__ __forceinline__ void append_word_pixels(u32 bits, int y, int w, u16* list, int list_base, int* counter, int lane) {
  const u32 count = __popc(bits);
  u32 inclusive = count;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u32 v = __shfl_up_sync(0xFFFFFFFFu, inclusive, o);
    if (lane >= o) inclusive += v;
  }
  const u32 warp_total = __shfl_sync(0xFFFFFFFFu, inclusive, 31);
  if (warp_total == 0) return;
  u32 warp_base = 0;
  if (lane == 31) warp_base = atomicAdd(counter, static_cast<int>(warp_total));
  warp_base = __shfl_sync(0xFFFFFFFFu, warp_base, 31);
  int out = list_base + static_cast<int>(warp_base + inclusive - count);
  while (bits) {
    const int b = __ffs(bits) - 1;
    bits &= bits - 1;
    list[out++] = static_cast<u16>((y << 8) | (w * 32 + b));
  }
}

__global__ void __launch_bounds__(kBlendBlock) k_blend(DeviceState d, FrameParams f) {
  pdl_prologue();
  if (f.skip) return;
  const TimelineScope timeline_scope(d, f.frame_index, KID_BLEND);
  extern __shared__ __align__(16) unsigned char blend_smem[];
  __shared__ int s_count[kMaxBlendRadius + 1][2];  // pixels per level and ring
  const int radius = f.blend_radius;
  const int halo_x = blend_halo_x(radius), halo_y = blend_halo_y(radius);
  const int rw = kBlendTileW + 2 * halo_x, rh = kBlendTileH + 2 * halo_y;  // rw is a multiple of 16
  const int rn = rw * rh;
  const int rn16 = (rn + 15) & ~15;
  const int wpr = (rw + 31) >> 5;   // mask words per region row
  const int nw = rh * wpr;          // words per bit raster
  float* s_delta = reinterpret_cast<float*>(blend_smem);    // ring 0 (distance_map) deltas
  float* s_ndelta = s_delta + rn16;                          // ring 1 (new_distance_map) deltas
  u16* s_depth = reinterpret_cast<u16*>(s_ndelta + rn16);   // working depth
  u16* s_front = s_depth + rn16;                             // [ring][rn16] pixel lists, level after level, entries (ly << 8) | lx
  u32* s_nodepth = reinterpret_cast<u32*>(s_front + 2 * rn16);  // bit rasters, nw words each
  u32* s_unsupported = s_nodepth + nw;
  u32* s_supported = s_unsupported + nw;
  u32* s_eligible = s_supported + nw;                        // [ring][nw]: pixels the ring may still grow into
  u32* s_level = s_eligible + 2 * nw;                        // [ring][3][nw]: level sets, plane = level % 3

  const int tile_x = blockIdx.x * kBlendTileW, tile_y = blockIdx.y * kBlendTileH;
  const int x0 = tile_x - halo_x, y0 = tile_y - halo_y;  // x0 is a multiple of 16
  const int lane = threadIdx.x & 31;

  for (int t = threadIdx.x; t < (kMaxBlendRadius + 1) * 2; t += kBlendBlock) (&s_count[0][0])[t] = 0;
  // Region load in 16-pixel chunks (two 128-bit depth loads + one of the support raster per
  // thread, all in flight together); rasters that are not 16-byte friendly take the scalar path.
  // Each chunk also yields 16 bits of the three class rasters.
  // The region (tile + halo) is read from the PRE-blend image f.depth_pre and only the tile interior
  // is written, to f.depth: a neighbouring tile's halo overlaps this interior, so reading and
  // writing the same raster would let a later-scheduled block see already blended depths.
  const bool vector_ok = (d.width & 15) == 0 && ((f.depth_pitch | f.depth_pre_pitch) & 15) == 0 &&
                         ((reinterpret_cast<uintptr_t>(f.depth) | reinterpret_cast<uintptr_t>(f.depth_pre)) & 15) == 0 &&
                         (reinterpret_cast<uintptr_t>(d.supported) & 15) == 0;
  const int chunks_per_row = wpr * 2;  // including the padding chunks right of the region
  for (int t = threadIdx.x; t < rh * chunks_per_row; t += kBlendBlock) {
    const int ly = t / chunks_per_row, chunk = t - ly * chunks_per_row;
    const int gy = y0 + ly, gx = x0 + chunk * 16;
    union { uint4 v[2]; u16 e[16]; } depth;
    union { uint4 v; u8 e[16]; } sup;
    depth.v[0] = depth.v[1] = sup.v = make_uint4(0u, 0u, 0u, 0u);
    const bool in_region = chunk * 16 < rw;
    if (in_region && gy >= 0 && gy < d.height) {
      const u16* depth_row = row_ptr(f.depth_pre, f.depth_pre_pitch, gy);
      const u8* sup_row = d.supported + static_cast<size_t>(gy) * d.width;
      if (vector_ok && gx >= 0 && gx + 16 <= d.width) {
        depth.v[0] = *reinterpret_cast<const uint4*>(depth_row + gx);
        depth.v[1] = *reinterpret_cast<const uint4*>(depth_row + gx + 8);
        sup.v = *reinterpret_cast<const uint4*>(sup_row + gx);
      } else {
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          if (gx + k >= 0 && gx + k < d.width) { depth.e[k] = depth_row[gx + k]; sup.e[k] = sup_row[gx + k]; }
        }
      }
    }
    u32 nodepth = 0, unsupported = 0, supported = 0;
    if (in_region) {
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        if (depth.e[k] == 0) nodepth |= 1u << k;
        else if (sup.e[k]) supported |= 1u << k;
        else unsupported |= 1u << k;
      }
      const int i = ly * rw + chunk * 16;
      *reinterpret_cast<uint4*>(s_depth + i) = depth.v[0];
      *reinterpret_cast<uint4*>(s_depth + i + 8) = depth.v[1];
    }
    reinterpret_cast<u16*>(s_nodepth)[t] = static_cast<u16>(nodepth);   // t = ly * 2 wpr + chunk: halfword index
    reinterpret_cast<u16*>(s_unsupported)[t] = static_cast<u16>(unsupported);
    reinterpret_cast<u16*>(s_supported)[t] = static_cast<u16>(supported);
  }
  __syncthreads();

  const float depth_scaling = f.depth_scaling;  // the reference passes 1 / depth_correction_factor (kernels.cc:179)
  const float rcp_scaling = frcp(depth_scaling);
  // pixels whose 3x3 stencil lies inside the region and that are interior image pixels
  const int lx_min = max(1, 1 - x0), lx_max = min(rw - 2, d.width - 2 - x0);
  const int ly_min = max(1, 1 - y0), ly_max = min(rh - 2, d.height - 2 - y0);

  // Start kernel (kernels.cu:563-615), classification: ring pixels (distance 1) are level 1.
  int begin0 = 0, begin1 = 0, end0 = 0, end1 = 0;  // list segment of the newest level, per ring
  for (int base = 0; base < nw; base += kBlendBlock) {
    const int t = base + threadIdx.x;
    u32 measurement_border = 0, surfel_border = 0;
    int y = 0, w = 0;
    if (t < nw) {
      y = t / wpr;
      w = t - y * wpr;
      u32 valid = 0;
      if (y >= ly_min && y <= ly_max) {
        const int lo = min(max(lx_min - 32 * w, 0), 32), hi = min(max(lx_max + 1 - 32 * w, 0), 32);
        const u32 below_hi = hi >= 32 ? 0xFFFFFFFFu : ((1u << hi) - 1u);
        const u32 below_lo = lo >= 32 ? 0xFFFFFFFFu : ((1u << lo) - 1u);
        valid = below_hi & ~below_lo;
      }
      const u32 supported = s_supported[t] & valid;
      measurement_border = supported & dilate_word(s_nodepth, y, w, rh, wpr);
      surfel_border = supported & dilate_word(s_unsupported, y, w, rh, wpr);
      s_level[(0 * 3 + 1) * nw + t] = measurement_border;
      s_level[(1 * 3 + 1) * nw + t] = surfel_border;
      s_eligible[t] = supported & ~measurement_border;  // distance_map == 255
      s_eligible[nw + t] = s_unsupported[t] & valid;    // new_distance_map == 0, has depth, unsupported
    }
    append_word_pixels(measurement_border, y, w, s_front, 0, &s_count[1][0], lane);
    append_word_pixels(surfel_border, y, w, s_front + rn16, 0, &s_count[1][1], lane);
  }
  __syncthreads();
  end0 = s_count[1][0];
  end1 = s_count[1][1];
  if (end0 == 0 && end1 == 0) return;  // no border ring reaches this tile: depth unchanged

  // One level of the breadth-first search for both rings (threads 0 .. 2 nw - 1, one word each).
  auto search_level = [&](int level) {
    const int previous_plane = (level - 1) % 3, plane = level % 3;
    for (int base = 0; base < 2 * nw; base += kBlendBlock) {
      const int t = base + threadIdx.x;
      u32 found = 0;
      int y = 0, w = 0, ring = 0;
      if (t < 2 * nw) {
        ring = t >= nw ? 1 : 0;
        const int word = t - ring * nw;
        y = word / wpr;
        w = word - y * wpr;
        const u32 eligible = s_eligible[t];
        found = eligible ? (eligible & dilate_word(s_level + (ring * 3 + previous_plane) * nw, y, w, rh, wpr)) : 0u;
        s_level[(ring * 3 + plane) * nw + word] = found;
        if (found) s_eligible[t] = eligible & ~found;
      }
      // (a warp never straddles the two rings unless nw is not a multiple of 32: append per ring)
      append_word_pixels(ring == 0 ? found : 0u, y, w, s_front, end0, &s_count[level][0], lane);
      append_word_pixels(ring == 1 ? found : 0u, y, w, s_front + rn16, end1, &s_count[level][1], lane);
    }
  };

  // Start kernel, values: the ring pixels fetch their association record and their depth as handed in
  // (the only global reads of the start step, all issued together; a pixel can sit on both rings, and
  // the ring-0 update rewrites the working depth, so the shared copy is not read here). The
  // reference's in-place write of the start kernel, flagged TODO at :610, can only matter if a
  // blended depth rounds to 0. The search for level 2 runs beside it.
  if (radius > 2) search_level(2);
  for (int t = threadIdx.x; t < end0 + end1; t += kBlendBlock) {
    const bool surfel_ring = t >= end0;
    const u32 q = surfel_ring ? s_front[rn16 + t - end0] : s_front[t];
    const int lx = static_cast<int>(q & 0xFFu), ly = static_cast<int>(q >> 8);
    const int i = ly * rw + lx;
    const PixelAssoc a = d.assoc[(y0 + ly) * d.width + x0 + lx];
    const float depth_f = u2f(row_ptr(f.depth_pre, f.depth_pre_pitch, y0 + ly)[x0 + lx]);
    const float sum = __uint_as_float(a.w);
    const float rcp_count = frcp(u2f(a.z));
    if (surfel_ring) {
      s_ndelta[i] = ffma(sum, rcp_count, -fmul(depth_f, rcp_scaling));
    } else {
      const float surfel_depth_average = fmul(sum, rcp_count);
      s_delta[i] = ffma(-depth_f, rcp_scaling, surfel_depth_average);
      s_depth[i] = static_cast<u16>(f2u_trunc(ffma(surfel_depth_average, depth_scaling, 0.5f)));
    }
  }
  __syncthreads();
  begin0 = end0; end0 += s_count[2][0];
  begin1 = end1; end1 += s_count[2][1];

  // Iteration kernels (kernels.cu:647-708), iteration = 2 .. radius - 1 (kernels.cc:190): the
  // pixels of level `iteration` take the average delta of their neighbours of level iteration - 1
  // (final since the previous barrier), one thread per pixel; the search for the next level runs
  // in the same barrier interval (it only touches the bit rasters).
  const float interpolation_factor_term = 1.0f / (radius - 1.0f);   // host expression, kernels.cc:196
  for (int iteration = 2; iteration < radius; ++iteration) {
    const int len0 = end0 - begin0, len1 = end1 - begin1;
    if (len0 + len1 == 0) break;  // both wavefronts died out
    if (iteration + 1 < radius) search_level(iteration + 1);
    const float scaled = fmul(ffma(-i2f(iteration - 1), interpolation_factor_term, 1.0f), depth_scaling);
    const int previous_plane = (iteration - 1) % 3;
    for (int t = threadIdx.x; t < len0 + len1; t += kBlendBlock) {
      const int ring = t >= len0 ? 1 : 0;
      const u32 q = ring == 0 ? s_front[begin0 + t] : s_front[rn16 + begin1 + t - len0];
      const int lx = static_cast<int>(q & 0xFFu), ly = static_cast<int>(q >> 8);
      const int i = ly * rw + lx;
      float* delta = ring == 0 ? s_delta : s_ndelta;
      // 3x3 bits of the previous level around the pixel (bit 3 * (wy + 1) + wx + 1)
      const u32* previous = s_level + (ring * 3 + previous_plane) * nw;
      const int first_bit = lx - 1, word = first_bit >> 5, shift = first_bit & 31;
      u32 taps = 0;
#pragma unroll
      for (int wy = -1; wy <= 1; ++wy) {
        const u32* row = previous + (ly + wy) * wpr;
        const u32 lo = row[word];
        const u32 hi = word + 1 < wpr ? row[word + 1] : 0u;
        taps |= (__funnelshift_r(lo, hi, shift) & 7u) << (3 * (wy + 1));
      }
      float neighbour_delta[9];
#pragma unroll
      for (int m = 0; m < 9; ++m) neighbour_delta[m] = ((taps >> m) & 1u) ? delta[i + (m / 3 - 1) * rw + (m % 3 - 1)] : 0.f;
      float delta_sum = 0.f;
#pragma unroll
      for (int m = 0; m < 9; ++m) {
        if ((taps >> m) & 1u) delta_sum = fadd(delta_sum, neighbour_delta[m]);
      }
      // taps != 0: the pixel was reached through a neighbour of the previous level
      const float avg = fmul(frcp(i2f(__popc(taps))), delta_sum);
      delta[i] = avg;
      s_depth[i] = static_cast<u16>(f2u_trunc(fadd(ffma(avg, scaled, 0.5f), u2f(s_depth[i]))));
    }
    __syncthreads();
    begin0 = end0; end0 += s_count[iteration + 1][0];
    begin1 = end1; end1 += s_count[iteration + 1][1];
  }

  // Write back the tile interior (f.depth holds the same values as f.depth_pre so far: tiles that no
  // ring reaches returned above and keep them).
  constexpr int kChunksPerTileRow = kBlendTileW / 8;
  for (int t = threadIdx.x; t < kBlendTileH * kChunksPerTileRow; t += kBlendBlock) {
    const int row = t / kChunksPerTileRow, chunk = t - row * kChunksPerTileRow;
    const int ly = row + halo_y, gy = y0 + ly;
    const int lx = halo_x + chunk * 8, gx = x0 + lx;
    if (gy >= d.height || gx >= d.width) continue;
    const int i = ly * rw + lx;
    union { uint4 v; u16 e[8]; } now;
    now.v = *reinterpret_cast<const uint4*>(s_depth + i);
    u16* out_row = row_ptr(f.depth, f.depth_pitch, gy);
    if (vector_ok && gx + 8 <= d.width) {
      *reinterpret_cast<uint4*>(out_row + gx) = now.v;
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (gx + k < d.width) out_row[gx + k] = now.e[k];
    }
  }
}

// ---------------------------------------------------------------------------------------
// a11: integration / conflict handling
// ---------------------------------------------------------------------------------------

// The attributes of one surfel that Integrate reads and writes, held in registers while its
// (up to two) pixels are processed; written back once.
struct SurfelState {
  float x, y, z, confidence, radius_squared, nx, ny, nz;
  float smooth_x, smooth_y, smooth_z;  // only set by a replacement
  u32 color, creation_stamp, last_update_stamp;
  bool replaced, dirty, stamped;
};

struct PixelMeasurement {
  float measurement_depth, first, radius_squared;
  float2 normal;
  u32 conflicting, count;
  u32 r, g, b;
};

// IntegrateOrConflictSurfel (kernels.cu:741-982) for one (surfel, pixel) pair. The
// reference serialises accesses to a surfel with a NaN spin-lock on its x coordinate; each
// surfel is owned by exactly one thread here (and there), so the lock is never contended.
__device__ __forceinline__ void integrate_or_conflict(const FrameParams& f, const PixelMeasurement& m, int x, int y,
                                                      u32 idx, float cx_, float cy_, float cz_, SurfelState& s) {
  if (!(m.measurement_depth > 0.f)) return;
  bool integrate = true, conflicting = false;
  if (m.first < fmul(m.measurement_depth, fadd(-f.sensor_noise_factor, 1.0f))) {
    if (m.first == cz_ && m.conflicting == idx) conflicting = true;
    integrate = false;
  }
  if (!integrate && !conflicting) return;
  if (cz_ > fmul(fadd(f.sensor_noise_factor, 1.0f), m.measurement_depth)) integrate = false;
  if (!integrate && !conflicting) return;

  // Read data (kernels.cu:804-814).
  const float lx = fmul(m.measurement_depth, ffma(i2f(x), f.fx_inv, f.cx_inv));
  const float ly = fmul(m.measurement_depth, ffma(i2f(y), f.fy_inv, f.cy_inv));
  const float3 g = transform_point(f.global_T_local, lx, ly, m.measurement_depth);
  const float3 gn = rotate_vec(f.global_T_local, m.normal.x, m.normal.y, -normal_z_abs(m.normal.x, m.normal.y));

  if (conflicting) {
    const float confidence = fadd(s.confidence, -1.0f);
    if (confidence <= 0.f) {
      // Delete the old surfel by replacing it with a new one (kernels.cu:828-854).
      s.x = g.x; s.y = g.y; s.z = g.z;
      s.smooth_x = g.x; s.smooth_y = g.y; s.smooth_z = g.z;
      s.nx = gn.x; s.ny = gn.y; s.nz = gn.z;
      s.color = m.r | (m.g << 8) | (m.b << 16) | (1u << 24);  // detach flag set
      s.radius_squared = m.radius_squared;
      s.confidence = 1.0f;
      s.creation_stamp = f.frame_index;
      s.stamped = true;
      s.replaced = true;
    } else {
      s.confidence = confidence;
    }
    s.dirty = true;
  }
  if (!integrate) return;

  float3 ln;
  if (facing_dot(f, cx_, cy_, cz_, s.nx, s.ny, s.nz, &ln) > 0.f) return;
  if (m.measurement_depth < cz_) {
    if (ffma(gn.z, s.nz, ffma(gn.x, s.nx, fmul(gn.y, s.ny))) < f.cos_normal_compatibility_threshold) return;
  }
  if (s.radius_squared < 0.f) return;

  // Integrate (kernels.cu:922-981).
  const float weight = frcp(u2f(max(1u, m.count)));
  if (s.creation_stamp < f.frame_index) {
    const float confidence = s.confidence;
    const float cw = fadd(weight, confidence);
    s.confidence = (cw < f.max_surfel_confidence) ? cw : f.max_surfel_confidence;
    const float normalization_factor = frcp(cw);
    // The reference's sm_90a SASS contracts all three coordinates as fma(g, w, c * s) (its sm_100a build
    // contracts x as fma(s, c, g * w) and y as fma(c, s, g * w)).
    s.x = fmul(normalization_factor, ffma(g.x, weight, fmul(confidence, s.x)));
    s.y = fmul(normalization_factor, ffma(g.y, weight, fmul(confidence, s.y)));
    s.z = fmul(normalization_factor, ffma(g.z, weight, fmul(confidence, s.z)));
    const float nx = ffma(gn.x, weight, fmul(confidence, s.nx));
    const float ny = ffma(gn.y, weight, fmul(confidence, s.ny));
    const float nz = ffma(gn.z, weight, fmul(confidence, s.nz));
    const float normal_normalization = frsqrt_approx(ffma(nz, nz, ffma(nx, nx, fmul(ny, ny))));
    s.nx = fmul(nx, normal_normalization);
    s.ny = fmul(ny, normal_normalization);
    s.nz = fmul(nz, normal_normalization);
    s.radius_squared = fminf(s.radius_squared, m.radius_squared);
    const u32 old_color = s.color;
    const u32 r = f2u_trunc(ffma(normalization_factor, ffma(u2f(m.r), weight, fmul(confidence, u2f(old_color & 0xFFu))), 0.5f));
    const u32 gr = f2u_trunc(ffma(normalization_factor, ffma(u2f(m.g), weight, fmul(confidence, u2f((old_color >> 8) & 0xFFu))), 0.5f));
    const u32 b = f2u_trunc(ffma(normalization_factor, ffma(u2f(m.b), weight, fmul(confidence, u2f((old_color >> 16) & 0xFFu))), 0.5f));
    s.color = (r & 0xFFu) | ((gr & 0xFFu) << 8) | ((b & 0xFFu) << 16);  // unsets the detach flag
    s.stamped = true;
    s.dirty = true;
  }
}

// The gates of integrate_or_conflict that only need the light per-pixel values (kernels.cu:757-800):
// can this pixel integrate into or conflict with the surfel at all?
__device__ __forceinline__ bool pixel_can_touch(const FrameParams& f, float measurement_depth, float first, u32 conflicting,
                                                u32 idx, float cz_) {
  if (!(measurement_depth > 0.f)) return false;
  if (first < fmul(measurement_depth, fadd(-f.sensor_noise_factor, 1.0f))) return first == cz_ && conflicting == idx;
  return !(cz_ > fmul(fadd(f.sensor_noise_factor, 1.0f), measurement_depth));
}

// One list entry of k_integrate. Returns whether the surfel goes on the neighbour-update list, with its
// pixel after the integration in (*ux, *uy).
// The entry is gathered in two levels. A light first batch (merge flag, radius, and per pixel the depth, the
// min-depth and the association record) decides whether either pixel can integrate into or conflict with
// the surfel; only then is the heavy batch (normal / radius / colour rasters, nine surfel rows) gathered.
// Only ~10 % of the listed surfels are changed by a frame, so the kernel moves a third of the bytes that
// one batch of everything the integration can need would (it was the longest kernel of BASELINE config 3),
// at the price of one more dependent level for the surfels that do integrate.
__device__ __forceinline__ bool integrate_entry(const DeviceState& d, const FrameParams& f, size_t pos, const VisEntry& e,
                                                int* ux, int* uy) {
    const u32 idx = e.x & ~kActiveBit;
    const float x = __uint_as_float(e.y), y = __uint_as_float(e.z), z = __uint_as_float(e.w);
    const Projection p = project(f, d.width, d.height, x, y, z);
    int ox = p.px, oy = p.py;
    const bool has2 = secondary_pixel(p, d.width, d.height, &ox, &oy);
    const u8 merged = d.merge_flag[pos];
    SurfelState s;
    PixelMeasurement m0, m1;
    // level 1: the merge decision, the radius and the light per-pixel values
    const int p0 = p.py * d.width + p.px, p1 = oy * d.width + ox;
    m0.measurement_depth = fmul(u2f(row_ptr(f.depth, f.depth_pitch, p.py)[p.px]), f.inv_depth_scaling);
    m1.measurement_depth = fmul(u2f(row_ptr(f.depth, f.depth_pitch, oy)[ox]), f.inv_depth_scaling);
    m0.first = d.first_depth[p0];
    m1.first = d.first_depth[p1];
    const PixelAssoc a0 = d.assoc[p0], a1 = d.assoc[p1];
    m0.conflicting = a0.y; m0.count = a0.z;
    m1.conflicting = a1.y; m1.count = a1.z;
    s.radius_squared = SM_S(SM_ROW_RADIUS_SQUARED, idx);
    s.last_update_stamp = 0;
    s.smooth_x = s.smooth_y = s.smooth_z = 0.f;
    s.replaced = false; s.dirty = false; s.stamped = false;
    if (merged) {
      // Apply the merge decided by k_merge (kernels.cu:1986-1989).
      SM_SU(SM_ROW_LAST_UPDATE_STAMP, idx) = 0;
      SM_S(SM_ROW_RADIUS_SQUARED, idx) = -1.0f;
      reinterpret_cast<u8*>(&SM_SU(SM_ROW_COLOR, idx))[3] = 1;
      SM_SU(kRowMergeEpoch, idx) = f.op_epoch;    // when it was merged (delta transfer)
      // Its stamp drops below every window: both record buffers have to hold its smooth position, and both
      // the new meta word (stamp 0, detach flag set; DeviceState::smooth).
      float4 record = d.smooth[idx];
      record.w = __uint_as_float(kMetaDetachBit);
      d.smooth[idx] = record;
      d.smooth_next[idx] = record;
      return false;
    }
    if (!(e.x & kActiveBit)) return false;
    if (s.radius_squared < 0.f) return false;  // kernels.cu:1050
    const bool touch0 = pixel_can_touch(f, m0.measurement_depth, m0.first, m0.conflicting, idx, z);
    const bool touch1 = has2 && pixel_can_touch(f, m1.measurement_depth, m1.first, m1.conflicting, idx, z);
    // level 2: the rest of the pixels that can touch the surfel, and the surfel
    if (touch0 || touch1) {
      const int qx0 = touch0 ? p.px : ox, qy0 = touch0 ? p.py : oy;   // unused pixel slots re-read a used one
      const int qx1 = touch1 ? ox : qx0, qy1 = touch1 ? oy : qy0;
      m0.normal = row_ptr(f.normals, f.normals_pitch, qy0)[qx0];
      m1.normal = row_ptr(f.normals, f.normals_pitch, qy1)[qx1];
      m0.radius_squared = row_ptr(f.radius, f.radius_pitch, qy0)[qx0];
      m1.radius_squared = row_ptr(f.radius, f.radius_pitch, qy1)[qx1];
      const uchar3 c0 = row_ptr(f.color, f.color_pitch, qy0)[qx0];
      const uchar3 c1 = row_ptr(f.color, f.color_pitch, qy1)[qx1];
      m0.r = c0.x; m0.g = c0.y; m0.b = c0.z;
      m1.r = c1.x; m1.g = c1.y; m1.b = c1.z;
      s.x = SM_S(SM_ROW_X, idx); s.y = SM_S(SM_ROW_Y, idx); s.z = SM_S(SM_ROW_Z, idx);
      s.confidence = SM_S(SM_ROW_CONFIDENCE, idx);
      s.nx = SM_S(SM_ROW_NORMAL_X, idx); s.ny = SM_S(SM_ROW_NORMAL_Y, idx); s.nz = SM_S(SM_ROW_NORMAL_Z, idx);
      s.color = SM_SU(SM_ROW_COLOR, idx);
      s.creation_stamp = SM_SU(SM_ROW_CREATION_STAMP, idx);
      if (touch0) integrate_or_conflict(f, m0, p.px, p.py, idx, x, y, z, s);
      if (touch1) integrate_or_conflict(f, m1, ox, oy, idx, x, y, z, s);
    }
    if (s.dirty) {
      SM_S(SM_ROW_X, idx) = s.x; SM_S(SM_ROW_Y, idx) = s.y; SM_S(SM_ROW_Z, idx) = s.z;
      SM_S(SM_ROW_CONFIDENCE, idx) = s.confidence;
      SM_S(SM_ROW_RADIUS_SQUARED, idx) = s.radius_squared;
      SM_S(SM_ROW_NORMAL_X, idx) = s.nx; SM_S(SM_ROW_NORMAL_Y, idx) = s.ny; SM_S(SM_ROW_NORMAL_Z, idx) = s.nz;
      SM_SU(SM_ROW_COLOR, idx) = s.color;
      if (s.stamped) {
        // every path that changes the colour's flag byte also stamps the surfel; the meta word goes to both
        // record buffers (DeviceState::smooth), with the new smooth position after a replacement
        SM_SU(SM_ROW_LAST_UPDATE_STAMP, idx) = f.frame_index;
        const u32 meta = f.frame_index | (((s.color >> 24) & 1u) ? kMetaDetachBit : 0u);
        if (s.replaced) {
          const float4 record = make_float4(s.smooth_x, s.smooth_y, s.smooth_z, __uint_as_float(meta));
          d.smooth[idx] = record;
          d.smooth_next[idx] = record;
        } else {
          store_reg_meta(d.smooth, idx, meta);
          store_reg_meta(d.smooth_next, idx, meta);
        }
      }
      if (s.replaced) {
        SM_SU(SM_ROW_CREATION_STAMP, idx) = f.frame_index;
#pragma unroll
        for (int i = 0; i < 4; ++i) SM_SU(SM_ROW_NEIGHBOR0 + i, idx) = kInvalidIndex;
      }
    }

    // The gates of the neighbour update (kernels.cu:1216-1262) up to the occlusion test, on the surfel as the
    // integration left it, with the arithmetic of k_update_neighbors: pure predicates, so their order is free.
    // Active: merged and inactive entries returned above; a stamped surfel's stamp is now the frame index.
    if (s.stamped && !is_active(f.frame_index, f.frame_index, f.active_window)) return false;
    if (s.radius_squared < 0.f) return false;
    // An unchanged surfel's list entry holds transform_row of its stored position (k_project, same pose),
    // and its pixel is the one of the entry, whose depth level 1 loaded.
    float cz_ = z;
    int px = p.px, py = p.py;
    if (s.dirty) {
      cz_ = transform_row(f.local_T_global.r2, s.x, s.y, s.z);
      if (!(cz_ > 0.f)) return false;
      const float cx_ = transform_row(f.local_T_global.r0, s.x, s.y, s.z);
      const float cy_ = transform_row(f.local_T_global.r1, s.x, s.y, s.z);
      const float inv_z = frcp(cz_);
      px = f2i_trunc(ffma(fmul(cx_, inv_z), f.fx, f.cx));
      py = f2i_trunc(ffma(fmul(cy_, inv_z), f.fy, f.cy));
    }
    constexpr int kBorder = 1;
    if (px < kBorder || py < kBorder || px >= d.width - kBorder || py >= d.height - kBorder) return false;
    float measurement_depth = m0.measurement_depth;
    if (px != p.px || py != p.py) {  // the surfel moved into another pixel
      measurement_depth = fmul(u2f(row_ptr(f.depth, f.depth_pitch, py)[px]), f.inv_depth_scaling);
    }
    if (cz_ > fmul(measurement_depth, fadd(f.sensor_noise_factor, 1.0f))) return false;  // occluded
    *ux = px;
    *uy = py;
    return true;
}

__global__ void __launch_bounds__(kBlock, 4) k_integrate(DeviceState d, FrameParams f) {
  pdl_prologue();
  if (f.skip) return;
  const TimelineScope timeline_scope(d, f.frame_index, KID_INTEGRATE);
  for_each_visible(d, &d.counters->surfel_count[f.count_slot], [&](size_t pos, const VisEntry& e) {
    int ux, uy;
    if (!integrate_entry(d, f, pos, e, &ux, &uy)) return;
    // Append to the neighbour-update list, one atomic per warp. The order does not matter: a listed surfel
    // only writes its own link row, and reads nothing that k_update_neighbors writes.
    const cg::coalesced_group g = cg::coalesced_threads();
    u32 base = 0;
    if (g.thread_rank() == 0) base = atomicAdd(d.upd_count, g.size());
    base = g.shfl(base, 0) + g.thread_rank();
    d.upd_list[base] = make_uint2(e.x & ~kActiveBit, static_cast<u32>(ux) | (static_cast<u32>(uy) << 16));
  });
}

// ---------------------------------------------------------------------------------------
// a12: neighbour update (kernels.cu:1197-1380)
// ---------------------------------------------------------------------------------------
// k_integrate evaluates the gates up to the occlusion test (active, not merged, radius, cz > 0, border,
// occlusion) and lists the surfels that pass, about one in ten of the visible ones. This is the rest for
// one listed surfel (x, y: its pixel after the integration).
__device__ __forceinline__ void update_neighbors_survivor(const DeviceState& d, const FrameParams& f, u32 idx, int x, int y) {
  const int kDirectionsX[4] = {-1, 1, 0, 0};
  const int kDirectionsY[4] = {0, 0, -1, 1};
  const float gx = SM_S(SM_ROW_X, idx), gy = SM_S(SM_ROW_Y, idx), gz = SM_S(SM_ROW_Z, idx);
  const float nx = SM_S(SM_ROW_NORMAL_X, idx), ny = SM_S(SM_ROW_NORMAL_Y, idx), nz = SM_S(SM_ROW_NORMAL_Z, idx);
  const float radius_squared = SM_S(SM_ROW_RADIUS_SQUARED, idx);
  u32 neighbor_surfel_indices[4];
#pragma unroll
  for (int m = 0; m < 4; ++m) neighbor_surfel_indices[m] = SM_SU(SM_ROW_NEIGHBOR0 + m, idx);
  const float observation_radius_squared = row_ptr(f.radius, f.radius_pitch, y)[x];
  u32 candidate[4];
#pragma unroll
  for (int direction = 0; direction < 4; ++direction) {
    const int candidate_pixel = (y + kDirectionsY[direction]) * d.width + x + kDirectionsX[direction];
    candidate[direction] = supporting_index(f.tb, d.assoc[candidate_pixel].x, static_cast<u32>(candidate_pixel));
  }
  const float cz_ = transform_row(f.local_T_global.r2, gx, gy, gz);
  const float cx_ = transform_row(f.local_T_global.r0, gx, gy, gz);
  const float cy_ = transform_row(f.local_T_global.r1, gx, gy, gz);
  float3 ln;
  if (facing_dot(f, cx_, cy_, cz_, nx, ny, nz, &ln) > 0.f) return;
  // kCheckScaleCompatibilityForNeighborAssignment, factor 1.5^2.
  if (fmul(observation_radius_squared, frcp(radius_squared)) > 2.25f) return;
  // A candidate that already is a neighbour is skipped (kernels.cu:1340-1346) and the list only
  // changes when some candidate is inserted: if every usable candidate is in the list as it
  // stands, nothing can happen (the steady state for most surfels) and the gathers below are
  // not needed.
  bool any_new = false;
#pragma unroll
  for (int direction = 0; direction < 4; ++direction) {
    const u32 q = candidate[direction];
    if (q == kInvalidIndex || q == idx) { candidate[direction] = kInvalidIndex; continue; }
    any_new |= q != neighbor_surfel_indices[0] && q != neighbor_surfel_indices[1] &&
               q != neighbor_surfel_indices[2] && q != neighbor_surfel_indices[3];
  }
  if (!any_new) return;

  // batch 3: the current neighbours' positions, positions and normals of the candidates
  float neighbor_distances_squared[4];
#pragma unroll
  for (int m = 0; m < 4; ++m) {
    const u32 q = neighbor_surfel_indices[m];
    if (q == kInvalidIndex) {
      neighbor_distances_squared[m] = __int_as_float(0x7f800000);
    } else {
      neighbor_distances_squared[m] = squared_norm(fsub(gx, SM_S(SM_ROW_X, q)), fsub(gy, SM_S(SM_ROW_Y, q)),
                                                   fsub(gz, SM_S(SM_ROW_Z, q)));
    }
  }
  const float max_distance_squared = fmul(radius_squared, f.radius_factor_squared);
  float cand_distance[4], cand_dot[4];
#pragma unroll
  for (int direction = 0; direction < 4; ++direction) {
    const u32 q = candidate[direction];
    if (q == kInvalidIndex) continue;
    cand_distance[direction] = squared_norm(fsub(SM_S(SM_ROW_X, q), gx), fsub(SM_S(SM_ROW_Y, q), gy),
                                            fsub(SM_S(SM_ROW_Z, q), gz));
    cand_dot[direction] = dot3(nx, ny, nz, SM_S(SM_ROW_NORMAL_X, q), SM_S(SM_ROW_NORMAL_Y, q), SM_S(SM_ROW_NORMAL_Z, q));
  }
  bool changed = false;
#pragma unroll
  for (int direction = 0; direction < 4; ++direction) {
    const u32 q = candidate[direction];
    if (q == kInvalidIndex) continue;
    const float distance_squared = cand_distance[direction];
    if (distance_squared > max_distance_squared) continue;
    if (cand_dot[direction] <= 0.f) continue;
    // Already a neighbour, or best (farthest) slot to replace.
    int best_n = -1;
    float best_distance_squared = -1.f;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      if (q == neighbor_surfel_indices[m]) { best_n = -1; break; }
      if (neighbor_distances_squared[m] > best_distance_squared) {
        best_n = m;
        best_distance_squared = neighbor_distances_squared[m];
      }
    }
    if (best_n >= 0 && distance_squared < best_distance_squared) {
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        if (m == best_n) { neighbor_surfel_indices[m] = q; neighbor_distances_squared[m] = distance_squared; }
      }
      changed = true;
    }
  }
  if (changed) {
#pragma unroll
    for (int m = 0; m < 4; ++m) SM_SU(SM_ROW_NEIGHBOR0 + m, idx) = neighbor_surfel_indices[m];
  }
}

__global__ void __launch_bounds__(kBlock) k_update_neighbors(DeviceState d, FrameParams f) {
  pdl_prologue();
  if (f.skip) return;
  const TimelineScope timeline_scope(d, f.frame_index, KID_UPDATE_NEIGHBORS);
  const u32 n = *d.upd_count;
  for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const uint2 w = d.upd_list[k];
    update_neighbors_survivor(d, f, w.x, static_cast<int>(w.y & 0xFFFFu), static_cast<int>(w.y >> 16));
  }
}

// ---------------------------------------------------------------------------------------
// a13: new-surfel flags + stable raster-order scan (single pass, decoupled look-back)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long load_scan_state(unsigned long long* p) { return atomicAdd(p, 0ull); }

__global__ void __launch_bounds__(kBlock) k_new_surfel_scan(DeviceState d, FrameParams f) {
  pdl_prologue();
  if (f.skip) return;
  const TimelineScope timeline_scope(d, f.frame_index, KID_NEW_SURFEL_SCAN);
  __shared__ u32 s_tile, s_prefix;
  __shared__ u32 warp_totals[kBlock / 32];
  const int total_pixels = d.width * d.height;
  const int tiles = (total_pixels + kSegment - 1) / kSegment;
  if (threadIdx.x == 0) s_tile = atomicAdd(&d.counters->scan_ticket, 1u);
  __syncthreads();
  const u32 tile = s_tile;
  if (tile >= static_cast<u32>(tiles)) return;

  const int base = tile * kSegment + threadIdx.x * 4;
  u32 flags[4];
  u32 cnt = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int seq = base + j;
    u32 flag = 0;
    if (seq < total_pixels) {
      const int y = seq / d.width, x = seq - y * d.width;
      constexpr int kBorder = 1;
      if (x >= kBorder && y >= kBorder && x < d.width - kBorder && y < d.height - kBorder &&
          row_ptr(f.depth, f.depth_pitch, y)[x] > 0 && !d.supported[seq]) {
        flag = (d.assoc[seq].y == kInvalidIndex) ? 1u : 0u;
      }
    }
    flags[j] = flag;
    cnt += flag;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  u32 incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const u32 t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) warp_totals[warp] = incl;
  __syncthreads();
  u32 warp_base = 0, block_total = 0;
#pragma unroll
  for (int w = 0; w < kBlock / 32; ++w) {
    const u32 t = warp_totals[w];
    if (w < warp) warp_base += t;
    block_total += t;
  }
  if (warp == 0) {
    // Publish this tile's aggregate, then look back 32 tiles at a time.
    if (lane == 0) atomicExch(&d.scan_state[tile], ((tile == 0 ? 2ull : 1ull) << 32) | block_total);
    u32 exclusive = 0;
    int window_end = static_cast<int>(tile) - 1;  // nearest preceding tile
    while (window_end >= 0) {
      const int t = window_end - lane;
      unsigned long long v = 2ull << 32;  // tiles before tile 0: inclusive prefix 0
      if (t >= 0) {
        do { v = load_scan_state(&d.scan_state[t]); } while ((v >> 32) == 0ull);
      }
      const unsigned inclusive_mask = __ballot_sync(0xffffffffu, (v >> 32) == 2ull);
      const int first_inclusive = __ffs(inclusive_mask) - 1;  // the closest tile that already has its prefix
      const u32 contribution = (first_inclusive < 0 || lane <= first_inclusive) ? static_cast<u32>(v) : 0u;
      exclusive += __reduce_add_sync(0xffffffffu, contribution);
      if (first_inclusive >= 0) break;
      window_end -= 32;
    }
    if (lane == 0) {
      if (tile != 0) atomicExch(&d.scan_state[tile], (2ull << 32) | (exclusive + block_total));
      s_prefix = exclusive;
      if (tile == static_cast<u32>(tiles) - 1) {
        // new_surfel_count = indices[P-1] + flag[P-1] (kernels.cc:116-125, cuda_surfel_reconstruction.cc:291).
        const u32 n_old = d.counters->surfel_count[f.count_slot];
        u32 new_count = exclusive + block_total;
        if (static_cast<u64>(n_old) + new_count > d.capacity) {
          d.counters->capacity_overflow = 1;  // the reference would write past the buffer here
          new_count = 0;
        }
        d.counters->new_surfel_count = new_count;
        d.counters->surfel_count[(f.count_slot + 1) % kCountSlots] = n_old + new_count;
      }
    }
  }
  __syncthreads();
  u32 running = s_prefix + warp_base + (incl - cnt);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int seq = base + j;
    if (seq < total_pixels) {
      d.new_flag[seq] = static_cast<u8>(flags[j]);
      d.new_index[seq] = running;
      if (flags[j]) d.new_list[running] = seq;  // compact list: the k-th new surfel comes from pixel new_list[k]
    }
    running += flags[j];
  }
}

// CreateNewSurfelsCUDACreationKernel (kernels.cu:133-231), one thread per NEW surfel.
__global__ void __launch_bounds__(kBlock) k_create_surfels(DeviceState d, FrameParams f) {
  pdl_prologue();
  if (f.skip) return;
  const TimelineScope timeline_scope(d, f.frame_index, KID_CREATE_SURFELS);
  const u32 new_count = d.counters->new_surfel_count;
  const u32 surfel_count = d.counters->surfel_count[f.count_slot];
  for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < new_count; k += gridDim.x * blockDim.x) {
    const int seq = d.new_list[k];
    const int y = seq / d.width, x = seq - y * d.width;
    const u32 idx = surfel_count + k;
    // batch 1: the pixel and its four neighbours
    const float depth = fmul(u2f(row_ptr(f.depth, f.depth_pitch, y)[x]), f.inv_depth_scaling);
    const float2 nm = row_ptr(f.normals, f.normals_pitch, y)[x];
    const uchar3 color = row_ptr(f.color, f.color_pitch, y)[x];
    const float radius_squared = row_ptr(f.radius, f.radius_pitch, y)[x];
    const int kDirectionsX[4] = {-1, 1, 0, 0};
    const int kDirectionsY[4] = {0, 0, -1, 1};
    u32 neighbor_index[4], neighbor_new_index[4];
    u8 neighbor_is_new[4];
    u16 neighbor_depth[4];
#pragma unroll
    for (int direction = 0; direction < 4; ++direction) {
      const int nx_ = x + kDirectionsX[direction], ny_ = y + kDirectionsY[direction];
      const int nseq = ny_ * d.width + nx_;
      neighbor_index[direction] = supporting_index(f.tb, d.assoc[nseq].x, static_cast<u32>(nseq));
      neighbor_is_new[direction] = d.new_flag[nseq];
      neighbor_new_index[direction] = d.new_index[nseq];
      neighbor_depth[direction] = row_ptr(f.depth, f.depth_pitch, ny_)[nx_];
    }
    const float lx = fmul(depth, ffma(i2f(x), f.fx_inv, f.cx_inv));
    const float ly = fmul(depth, ffma(u2f(y), f.fy_inv, f.cy_inv));
    const float3 g = transform_point(f.global_T_local, lx, ly, depth);
    const float3 gn = rotate_vec(f.global_T_local, nm.x, nm.y, -normal_z_abs(nm.x, nm.y));
    // batch 2: existing neighbours (kernels.cu:189-224)
    const float max_distance_squared = fmul(radius_squared, f.radius_factor_squared);
    float ndist[4], nsx[4], nsy[4], nsz[4];
#pragma unroll
    for (int direction = 0; direction < 4; ++direction) {
      const u32 q = neighbor_index[direction];
      if (q == kInvalidIndex) continue;
      ndist[direction] = squared_norm(fsub(SM_S(SM_ROW_X, q), g.x), fsub(SM_S(SM_ROW_Y, q), g.y), fsub(SM_S(SM_ROW_Z, q), g.z));
      const float4 record = d.smooth[q];   // smooth position: one 16-byte gather
      nsx[direction] = record.x;
      nsy[direction] = record.y;
      nsz[direction] = record.z;
    }
    float sum_x = 0.f, sum_y = 0.f, sum_z = 0.f;
    int existing_neighbor_count_plus_1 = 1;
#pragma unroll
    for (int direction = 0; direction < 4; ++direction) {
      u32 q = neighbor_index[direction];
      if (q != kInvalidIndex) {
        if (ndist[direction] > max_distance_squared) {
          q = kInvalidIndex;
        } else {
          sum_x = fadd(sum_x, nsx[direction]);
          sum_y = fadd(sum_y, nsy[direction]);
          sum_z = fadd(sum_z, nsz[direction]);
          ++existing_neighbor_count_plus_1;
        }
      } else if (neighbor_is_new[direction] == 1) {
        const float diff = ffma(-u2f(neighbor_depth[direction]), f.inv_depth_scaling, depth);
        if (!(fmul(diff, diff) > max_distance_squared)) q = surfel_count + neighbor_new_index[direction];
      }
      SM_SU(SM_ROW_NEIGHBOR0 + direction, idx) = q;
    }
    SM_S(SM_ROW_X, idx) = g.x; SM_S(SM_ROW_Y, idx) = g.y; SM_S(SM_ROW_Z, idx) = g.z;
    SM_S(SM_ROW_NORMAL_X, idx) = gn.x; SM_S(SM_ROW_NORMAL_Y, idx) = gn.y; SM_S(SM_ROW_NORMAL_Z, idx) = gn.z;
    SM_SU(SM_ROW_COLOR, idx) = color.x | (color.y << 8) | (color.z << 16);
    SM_S(SM_ROW_CONFIDENCE, idx) = 1.0f;
    SM_SU(SM_ROW_CREATION_STAMP, idx) = f.frame_index;
    SM_SU(SM_ROW_LAST_UPDATE_STAMP, idx) = f.frame_index;
    SM_S(SM_ROW_RADIUS_SQUARED, idx) = radius_squared;
    // The reference leaves rows 11-16 and 23 uninitialised; here rows 11-13 and 23 are always
    // zero and the regularisation accumulates in d.gradient, zero between calls (regularize.cu).
    SM_S(SM_ROW_GRADIENT_X, idx) = 0.f; SM_S(SM_ROW_GRADIENT_Y, idx) = 0.f; SM_S(SM_ROW_GRADIENT_Z, idx) = 0.f;
    SM_S(SM_ROW_GRADIENT_COUNT, idx) = 0.f;
    d.gradient[idx] = make_float4(0.f, 0.f, 0.f, 0.f);
    const float rcp_count = frcp(i2f(existing_neighbor_count_plus_1));
    const float sx = fmul(fadd(g.x, sum_x), rcp_count);
    const float sy = fmul(fadd(g.y, sum_y), rcp_count);
    const float sz = fmul(fadd(g.z, sum_z), rcp_count);
    // both record buffers (DeviceState::smooth): meta word = the stamp, detach flag clear
    const float4 record = make_float4(sx, sy, sz, __uint_as_float(f.frame_index));
    d.smooth[idx] = record;
    d.smooth_next[idx] = record;
  }
}

// ExportVerticesCUDAKernel (kernels.cu:2412-2433).
__global__ void __launch_bounds__(kBlock) k_export_vertices(DeviceState d, int count_slot, float* position_buffer,
                                                            u8* color_buffer) {
  pdl_prologue();
  const u32 n = d.counters->surfel_count[count_slot];
  for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const bool merged = SM_S(SM_ROW_RADIUS_SQUARED, i) < 0.f;
    const float nan = __int_as_float(0x7fffffff);
    const float4 smooth = d.smooth[i];
    position_buffer[3 * i + 0] = merged ? nan : smooth.x;
    position_buffer[3 * i + 1] = merged ? nan : smooth.y;
    position_buffer[3 * i + 2] = merged ? nan : smooth.z;
    const u32 c = SM_SU(SM_ROW_COLOR, i);
    color_buffer[3 * i + 0] = c & 0xFF;
    color_buffer[3 * i + 1] = (c >> 8) & 0xFF;
    color_buffer[3 * i + 2] = (c >> 16) & 0xFF;
  }
}

}  // namespace

namespace {
// Dynamic shared memory of k_blend: 14 B per region pixel + 11 bit rasters (see the kernel's carve-up).
size_t BlendSmemBytes(int radius) {
  const size_t rw = kBlendTileW + 2 * blend_halo_x(radius), rh = kBlendTileH + 2 * blend_halo_y(radius);
  const size_t rn16 = (rw * rh + 15) & ~static_cast<size_t>(15);
  const size_t mask_words = rh * ((rw + 31) / 32);
  return rn16 * 14 + mask_words * 11 * 4 + 16;
}
constexpr size_t kBlendSmemLimit = 224 * 1024;  // one region per block has to fit an SM
}  // namespace

int DescribeFrameKernel(FrameKernel which, const LaunchPlan& plan, const DeviceState& d, const FrameParams& f,
                        KernelLaunch* out) {
  static_assert(sizeof(DeviceState) + sizeof(FrameParams) + 32 <= sizeof(out->storage), "KernelLaunch::storage too small");
  const int scan_tiles = (d.width * d.height + kSegment - 1) / kSegment;
  switch (which) {
    case FK_PROJECT:
      out->Reset(reinterpret_cast<const void*>(k_project), dim3(plan.project), dim3(kProjectBlock), 0, KID_PROJECT);
      break;
    case FK_ASSOCIATE:
      out->Reset(reinterpret_cast<const void*>(k_associate), dim3(plan.associate), dim3(kBlock), 0, KID_ASSOCIATE);
      break;
    case FK_MERGE:
      out->Reset(reinterpret_cast<const void*>(k_merge), dim3(plan.merge), dim3(kBlock), 0, KID_MERGE);
      break;
    case FK_BLEND: {
      const size_t smem = BlendSmemBytes(f.blend_radius);
      if (f.blend_radius < 1 || f.blend_radius > kMaxBlendRadius || smem > kBlendSmemLimit)
        return SetError(SM_ERR_INVALID_ARGUMENT, "measurement_blending_radius too large for one tile region per SM");
      const dim3 pixel_tiles((d.width + kBlendTileW - 1) / kBlendTileW, (d.height + kBlendTileH - 1) / kBlendTileH);
      out->Reset(reinterpret_cast<const void*>(k_blend), pixel_tiles, dim3(kBlendBlock), smem, KID_BLEND);
      break;
    }
    case FK_INTEGRATE:
      out->Reset(reinterpret_cast<const void*>(k_integrate), dim3(plan.integrate), dim3(kBlock), 0, KID_INTEGRATE);
      break;
    case FK_UPDATE_NEIGHBORS:
      out->Reset(reinterpret_cast<const void*>(k_update_neighbors), dim3(plan.update_neighbors), dim3(kBlock), 0,
                 KID_UPDATE_NEIGHBORS);
      break;
    case FK_SCAN:
      out->Reset(reinterpret_cast<const void*>(k_new_surfel_scan), dim3(scan_tiles), dim3(kBlock), 0, KID_NEW_SURFEL_SCAN);
      break;
    case FK_CREATE:
      out->Reset(reinterpret_cast<const void*>(k_create_surfels), dim3(plan.sm_count * 2), dim3(kBlock), 0, KID_CREATE_SURFELS);
      break;
    default:
      return SetError(SM_ERR_INVALID_ARGUMENT, "DescribeFrameKernel");
  }
  out->Arg(d);
  out->Arg(f);
  return SM_OK;
}

namespace {
int LaunchFrameKernel(cudaStream_t stream, FrameKernel which, const LaunchPlan& plan, const DeviceState& d,
                      const FrameParams& f, bool dependent) {
  KernelLaunch k;
  const int status = DescribeFrameKernel(which, plan, d, f, &k);
  if (status != SM_OK) return status;
  LaunchOnStream(stream, k, dependent);
  return SM_OK;
}
}  // namespace

int ClearAssociationRasters(cudaStream_t stream, const DeviceState& d) {
  const int blocks = (d.width * d.height + kBlock * 4 - 1) / (kBlock * 4);
  { LaunchScope scope(stream, KID_CLEAR); LaunchKernel(k_clear, dim3(blocks), dim3(kBlock), 0, stream, d); }
  return CheckLaunch("clear");
}

int IntegrateFrame(cudaStream_t stream, const DeviceState& d, const FrameParams& f, bool do_blending,
                   bool rasters_already_cleared, const LaunchPlan& plan, const IntegrateEvents* events) {
  const bool timed = events && events->enabled;
  auto record = [&](int i) { if (timed) cudaEventRecord(events->ev[i], stream); };
  int status = SM_OK;
  auto launch = [&](FrameKernel which, bool dependent) {
    if (status == SM_OK) status = LaunchFrameKernel(stream, which, plan, d, f, dependent);
  };
  record(0);
  if (!rasters_already_cleared) {
    status = ClearAssociationRasters(stream, d);
    if (status != SM_OK) return status;
  }
  launch(FK_PROJECT, false);
  launch(FK_ASSOCIATE, true);
  record(1); record(2);
  launch(FK_MERGE, false);
  record(3); record(4);
  if (do_blending) launch(FK_BLEND, true);
  record(5); record(6);
  launch(FK_INTEGRATE, false);
  record(7); record(8);
  launch(FK_UPDATE_NEIGHBORS, false);
  record(9); record(10);
  launch(FK_SCAN, false);
  launch(FK_CREATE, false);
  record(11);
  if (status != SM_OK) return status;
  return CheckLaunch("integrate");
}

int ExportVertices(cudaStream_t stream, const DeviceState& d, int count_slot, int sm_count, float* position_buffer,
                   u8* color_buffer) {
  { LaunchScope scope(stream, KID_EXPORT_VERTICES); LaunchKernel(k_export_vertices, dim3(sm_count * 8), dim3(kBlock), 0, stream, d, count_slot, position_buffer, color_buffer); }
  return CheckLaunch("export vertices");
}

// Per-device configuration of the kernels of this file for the CURRENT device (called by
// sm_create for every handle: function attributes and occupancy are per device): the shared-memory
// carve-out (kSharedMemoryCarveoutPercent), k_blend's dynamic shared memory limit and the resident
// grids of the list kernels (ResidentBlocks).
int ConfigureIntegrateKernels(LaunchPlan* plan) {
  const int carveout_percent = kSharedMemoryCarveoutPercent;
  cudaFuncSetAttribute(k_clear, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_project, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_associate, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_merge, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_blend, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_integrate, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_update_neighbors, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_new_surfel_scan, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_create_surfels, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaFuncSetAttribute(k_export_vertices, cudaFuncAttributePreferredSharedMemoryCarveout, carveout_percent);
  cudaGetLastError();
  if (cudaFuncSetAttribute(k_blend, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kBlendSmemLimit)) != cudaSuccess) {
    return SetError(SM_ERR_CUDA, "cudaFuncSetAttribute(k_blend, MaxDynamicSharedMemorySize)");
  }
  const int sm_count = plan->sm_count;
  int status = ResidentBlocks(k_project, kProjectBlock, sm_count, &plan->project);
  if (status == SM_OK) status = ResidentBlocks(k_associate, kBlock, sm_count, &plan->associate);
  if (status == SM_OK) status = ResidentBlocks(k_merge, kBlock, sm_count, &plan->merge);
  if (status == SM_OK) status = ResidentBlocks(k_integrate, kBlock, sm_count, &plan->integrate);
  if (status == SM_OK) status = ResidentBlocks(k_update_neighbors, kBlock, sm_count, &plan->update_neighbors);
  return status;
}

}  // namespace smb
