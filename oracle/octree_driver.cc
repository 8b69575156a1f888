// TEST INFRASTRUCTURE (oracle).  C entry points around the reference's own CPU octree
// (applications/surfel_meshing/src/surfel_meshing/octree.{h,cc}, compiled unmodified from the reference sources (REF) by
// oracle/Makefile against oracle/eigen_shim) so that the GPU radius k-NN (SURVEY §8 f4) can be checked against
// CompressedOctree::FindNearestSurfelsWithinRadius (octree.cc:433-470) itself, plus a restatement of the brute-force
// checker the reference's own octree test uses (test/test_octree.cc:116-149).  Only tests/, smoke() and the
// cpu_baseline / reference legs of the probes may load this.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "surfel_meshing/octree.h"

namespace {

struct OctreeOracle {
  std::vector<vis::Surfel> surfels;
  vis::CompressedOctree* octree = nullptr;
};

template <bool kCompleted, bool kFree>
int Query(OctreeOracle* o, const vis::Vec3f& p, float r2, int k, float* d2, uint32_t* idx) {
  return o->octree->FindNearestSurfelsWithinRadius<kCompleted, kFree>(p, r2, k, d2, idx);
}

int QueryAny(OctreeOracle* o, int include_completed, int include_free, const vis::Vec3f& p, float r2, int k, float* d2,
             uint32_t* idx) {
  if (include_completed) {
    return include_free ? Query<true, true>(o, p, r2, k, d2, idx) : Query<true, false>(o, p, r2, k, d2, idx);
  }
  return include_free ? Query<false, true>(o, p, r2, k, d2, idx) : Query<false, false>(o, p, r2, k, d2, idx);
}

}  // namespace

extern "C" {

// state[i]: 0 free, 1 front, 2 completed (Surfel::MeshingState, surfel.h:67-71); 255 = the slot holds no surfel and
// is not inserted (what SurfelMeshing::IntegrateCUDABuffers does for merged / never-created slots).
void* smoct_create(int max_surfels_per_node, uint32_t n, const float* x, const float* y, const float* z,
                   const float* radius_squared, const uint8_t* state) {
  OctreeOracle* o = new OctreeOracle;
  o->surfels.reserve(n);
  for (uint32_t i = 0; i < n; ++i) {
    o->surfels.push_back(vis::Surfel(vis::Vec3f(x[i], y[i], z[i]), radius_squared ? radius_squared[i] : 1.f,
                                     vis::Vec3f(1, 0, 0), 0));
    if (state && state[i] != 255) o->surfels.back().SetMeshingState(static_cast<vis::Surfel::MeshingState>(state[i]));
  }
  o->octree = new vis::CompressedOctree(max_surfels_per_node, &o->surfels, nullptr);
  for (uint32_t i = 0; i < n; ++i) {
    if (state && state[i] == 255) continue;
    o->octree->AddSurfel(i, &o->surfels[i]);
  }
  return o;
}

void smoct_destroy(void* handle) {
  OctreeOracle* o = static_cast<OctreeOracle*>(handle);
  delete o->octree;
  delete o;
}

int smoct_query(void* handle, int include_completed, int include_free, float px, float py, float pz,
                float radius_squared, int max_result_count, float* d2, uint32_t* idx) {
  return QueryAny(static_cast<OctreeOracle*>(handle), include_completed, include_free, vis::Vec3f(px, py, pz),
                  radius_squared, max_result_count, d2, idx);
}

// The meshing thread's access pattern: one query after the other on one thread (the non-passive query re-sorts
// nodes lazily, octree.cc:455-460, so it is not thread safe).  Results of query q land at [q * max_result_count, ...).
void smoct_query_batch(void* handle, int include_completed, int include_free, uint32_t query_count, const float* qx,
                       const float* qy, const float* qz, const float* radius_squared, int max_result_count, float* d2,
                       uint32_t* idx, int32_t* counts) {
  OctreeOracle* o = static_cast<OctreeOracle*>(handle);
  for (uint32_t q = 0; q < query_count; ++q) {
    counts[q] = QueryAny(o, include_completed, include_free, vis::Vec3f(qx[q], qy[q], qz[q]), radius_squared[q],
                         max_result_count, d2 + size_t(q) * max_result_count, idx + size_t(q) * max_result_count);
  }
}

// Restatement of FindNearestSurfelsWithinRadiusBruteForce (test/test_octree.cc:116-149) with the state filter of
// octree.cc:329-334 and a total order (distance, then index) where the reference's std::sort leaves ties open.
int smoct_brute_force(uint32_t n, const float* x, const float* y, const float* z, const uint8_t* state,
                      int include_completed, int include_free, float px, float py, float pz, float radius_squared,
                      int max_result_count, float* d2, uint32_t* idx) {
  std::vector<std::pair<float, uint32_t>> found;
  for (uint32_t i = 0; i < n; ++i) {
    if (state) {
      if (state[i] == 255) continue;
      if (!include_completed && state[i] == 2) continue;
      if (!include_free && state[i] == 0) continue;
    }
    const float dx = x[i] - px, dy = y[i] - py, dz = z[i] - pz;
    const float distance_squared = (dx * dx + dy * dy) + dz * dz;
    if (distance_squared > radius_squared) continue;
    found.emplace_back(distance_squared, i);
  }
  std::sort(found.begin(), found.end());
  const int count = std::min<size_t>(found.size(), max_result_count);
  for (int i = 0; i < count; ++i) {
    d2[i] = found[i].first;
    idx[i] = found[i].second;
  }
  return count;
}

}  // extern "C"
