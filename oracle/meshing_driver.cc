// TEST INFRASTRUCTURE (oracle).  C entry points around the reference's own CPU meshing
// (applications/surfel_meshing/src/surfel_meshing/{surfel_meshing.cc,octree.cc}, compiled unmodified from
// the reference sources (REF) by oracle/Makefile against oracle/eigen_shim and oracle/libvis_stubs): BASELINE config 1, the
// pattern of the reference's triangulation test (test/test_triangulation.cc:57-98): fill CUDASurfelsCPU ->
// IntegrateCUDABuffers -> CheckRemeshing -> Triangulate.
//
// It also shows the binding a maintainer would add for the GPU neighbour search (SURVEY section 8 f4): the two
// octree queries of the meshing code (surfel_meshing.cc:421 <false, true>, :821 <true, false>) are redirected at
// object level (objcopy --redefine-sym on the compiled surfel_meshing.o, the source stays untouched) to the two
// functions below. They answer from a batch of sm_knn_query results when one was supplied for this meshing
// iteration and it provably contains the octree's answer, and call the octree otherwise:
//   * the batch holds, per surfel, its <= 64 nearest octree members within a radius that covers every radius
//     TriangulateSurfel can ask for (max_neighbor_search_range_increase_factor^2 x radius^2), computed for ALL
//     meshing states;
//   * the meshing state a query filters on changes while Triangulate() runs, so the filter (and the octree
//     membership) is applied to the batch entries at call time;
//   * if the batch row is full (64 entries) it may have cut candidates the filtered query still needs: fall back.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <mutex>
#include <vector>

#include "surfel_meshing/surfel_meshing.h"

namespace {

struct MeshingOracle {
  vis::SurfelMeshing* meshing = nullptr;
  // batch of GPU answers for the current iteration (empty: every query goes to the octree)
  uint32_t batch_points = 0;
  int batch_k = 0;
  std::vector<float> batch_d2;
  std::vector<uint32_t> batch_idx;
  std::vector<int32_t> batch_count;
  std::vector<float> batch_radius_squared;
  uint64_t served = 0, fallback = 0;
};

std::mutex g_registry_lock;
std::vector<MeshingOracle*> g_registry;

MeshingOracle* OwnerOf(const vis::CompressedOctree* octree) {
  std::lock_guard<std::mutex> lock(g_registry_lock);
  const char* p = reinterpret_cast<const char*>(octree);
  for (MeshingOracle* o : g_registry) {
    const char* base = reinterpret_cast<const char*>(o->meshing);
    if (p >= base && p < base + sizeof(vis::SurfelMeshing)) return o;
  }
  return nullptr;
}

// Returns -1 if the batch cannot answer.
template <bool kCompleted, bool kFree>
int FromBatch(MeshingOracle* o, const vis::Vec3f& position, float radius_squared, int max_result_count, float* d2,
              uint32_t* idx) {
  if (!o || o->batch_points == 0) return -1;
  const std::vector<vis::Surfel>& surfels = o->meshing->surfels();
  const char* first = reinterpret_cast<const char*>(surfels.data());
  const char* p = reinterpret_cast<const char*>(&position);
  if (p < first || p >= first + surfels.size() * sizeof(vis::Surfel)) return -1;   // not a surfel's own position
  const size_t i = (p - first) / sizeof(vis::Surfel);
  if (&surfels[i].position() != &position || i >= o->batch_points) return -1;
  if (radius_squared > o->batch_radius_squared[i]) return -1;                      // the batch does not reach that far
  const int n = o->batch_count[i];
  const float* bd = o->batch_d2.data() + i * o->batch_k;
  const uint32_t* bi = o->batch_idx.data() + i * o->batch_k;
  int out = 0;
  for (int j = 0; j < n && out < max_result_count; ++j) {
    if (bd[j] > radius_squared) break;
    const vis::Surfel& s = surfels[bi[j]];
    if (s.node() == nullptr) continue;                                             // not (any more) in the octree
    if (!kCompleted && s.meshing_state() == vis::Surfel::MeshingState::kCompleted) continue;
    if (!kFree && s.meshing_state() == vis::Surfel::MeshingState::kFree) continue;
    d2[out] = bd[j];
    idx[out] = bi[j];
    ++out;
  }
  if (out < max_result_count && n == o->batch_k && bd[n - 1] <= radius_squared) return -1;   // the row was cut short
  return out;
}

}  // namespace

// The redirected octree queries (same signature as the member functions, `this` first).
extern "C" int smmesh_query_triangulate(vis::CompressedOctree* self, const vis::Vec3f& position, float radius_squared,
                                        int max_result_count, float* d2, uint32_t* idx) {
  MeshingOracle* o = OwnerOf(self);
  const int n = FromBatch<false, true>(o, position, radius_squared, max_result_count, d2, idx);
  if (n >= 0) { ++o->served; return n; }
  if (o) ++o->fallback;
  return self->FindNearestSurfelsWithinRadius<false, true>(position, radius_squared, max_result_count, d2, idx);
}
extern "C" int smmesh_query_remesh(vis::CompressedOctree* self, const vis::Vec3f& position, float radius_squared,
                                   int max_result_count, float* d2, uint32_t* idx) {
  MeshingOracle* o = OwnerOf(self);
  const int n = FromBatch<true, false>(o, position, radius_squared, max_result_count, d2, idx);
  if (n >= 0) { ++o->served; return n; }
  if (o) ++o->fallback;
  return self->FindNearestSurfelsWithinRadius<true, false>(position, radius_squared, max_result_count, d2, idx);
}

extern "C" {

// Defaults of main.cc:374-400,481 (angles in radians).
void* smmesh_create(int max_surfels_per_node, float max_angle_between_normals, float min_triangle_angle,
                    float max_triangle_angle, float max_neighbor_search_range_increase_factor,
                    float long_edge_tolerance_factor, int regularization_frame_window_size) {
  MeshingOracle* o = new MeshingOracle;
  o->meshing = new vis::SurfelMeshing(max_surfels_per_node, max_angle_between_normals, min_triangle_angle,
                                      max_triangle_angle, max_neighbor_search_range_increase_factor,
                                      long_edge_tolerance_factor, regularization_frame_window_size, nullptr);
  std::lock_guard<std::mutex> lock(g_registry_lock);
  g_registry.push_back(o);
  return o;
}

void smmesh_destroy(void* handle) {
  MeshingOracle* o = static_cast<MeshingOracle*>(handle);
  {
    std::lock_guard<std::mutex> lock(g_registry_lock);
    g_registry.erase(std::remove(g_registry.begin(), g_registry.end(), o), g_registry.end());
  }
  delete o->meshing;
  delete o;
}

// One hand-off from the reconstruction: the arrays of CUDASurfelBuffersCPU (cuda_surfels_cpu.h:40-73) go through
// IntegrateCUDABuffers; CheckRemeshing and Triangulate follow as separate calls (test_triangulation.cc:92-97) so that
// a batch of GPU answers for the new positions can be supplied in between.
void smmesh_integrate(void* handle, uint32_t frame_index, uint32_t surfel_count, const float* x, const float* y,
                      const float* z, const float* radius_squared, const float* nx, const float* ny, const float* nz,
                      const uint32_t* last_update_stamp) {
  MeshingOracle* o = static_cast<MeshingOracle*>(handle);
  vis::CUDASurfelsCPU input(std::max<uint32_t>(surfel_count, 1));
  vis::CUDASurfelBuffersCPU* b = input.write_buffers();
  input.LockWriteBuffers();
  b->frame_index = frame_index;
  b->surfel_count = surfel_count;
  const size_t bytes = sizeof(float) * surfel_count;
  std::memcpy(b->surfel_x_buffer, x, bytes);
  std::memcpy(b->surfel_y_buffer, y, bytes);
  std::memcpy(b->surfel_z_buffer, z, bytes);
  std::memcpy(b->surfel_radius_squared_buffer, radius_squared, bytes);
  std::memcpy(b->surfel_normal_x_buffer, nx, bytes);
  std::memcpy(b->surfel_normal_y_buffer, ny, bytes);
  std::memcpy(b->surfel_normal_z_buffer, nz, bytes);
  std::memcpy(b->surfel_last_update_stamp_buffer, last_update_stamp, bytes);
  input.UnlockWriteBuffers();
  input.WaitForLockAndSwapBuffers();
  o->batch_points = 0;   // positions may have moved: a batch is valid for one iteration only
  o->meshing->IntegrateCUDABuffers(frame_index, input);
}

void smmesh_check_remeshing(void* handle) { static_cast<MeshingOracle*>(handle)->meshing->CheckRemeshing(); }

// GPU answers for this iteration: row i = the <= k nearest octree members of surfel i within batch_radius_squared[i]
// (all meshing states), ascending, as sm_knn_query returns them.
void smmesh_set_knn_batch(void* handle, uint32_t points, int k, const float* d2, const uint32_t* idx,
                          const int32_t* count, const float* batch_radius_squared) {
  MeshingOracle* o = static_cast<MeshingOracle*>(handle);
  o->batch_points = points;
  o->batch_k = k;
  o->batch_d2.assign(d2, d2 + size_t(points) * k);
  o->batch_idx.assign(idx, idx + size_t(points) * k);
  o->batch_count.assign(count, count + points);
  o->batch_radius_squared.assign(batch_radius_squared, batch_radius_squared + points);
}

void smmesh_triangulate(void* handle) { static_cast<MeshingOracle*>(handle)->meshing->Triangulate(); }

// RemeshTrianglesAt (public "such that it can be accessed from tests", surfel_meshing.h:107-112), then Triangulate:
// the second half of the reference's triangulation test.
void smmesh_remesh_at(void* handle, uint32_t surfel_index, float radius_factor_squared) {
  vis::SurfelMeshing* m = static_cast<MeshingOracle*>(handle)->meshing;
  vis::Surfel* s = const_cast<vis::Surfel*>(&m->surfels()[surfel_index]);
  m->RemeshTrianglesAt(s, radius_factor_squared * s->radius_squared());
}

uint64_t smmesh_triangle_count(void* handle) { return static_cast<MeshingOracle*>(handle)->meshing->triangle_count(); }

// Valid triangles as index triples, in storage order.
uint64_t smmesh_get_triangles(void* handle, uint32_t* out, uint64_t capacity) {
  vis::Mesh3fCu8 mesh;
  static_cast<MeshingOracle*>(handle)->meshing->ConvertToMesh3fCu8(&mesh, /*indices_only*/ true);
  const auto& t = mesh.triangles();
  const uint64_t n = std::min<uint64_t>(t.size(), capacity);
  for (uint64_t i = 0; i < n; ++i) {
    out[3 * i + 0] = t[i].index(0);
    out[3 * i + 1] = t[i].index(1);
    out[3 * i + 2] = t[i].index(2);
  }
  return t.size();
}

void smmesh_meshing_states(void* handle, uint8_t* out, uint32_t count) {
  const auto& s = static_cast<MeshingOracle*>(handle)->meshing->surfels();
  for (uint32_t i = 0; i < count && i < s.size(); ++i) {
    out[i] = s[i].node() == nullptr ? 255 : static_cast<uint8_t>(s[i].meshing_state());
  }
}

void smmesh_query_stats(void* handle, uint64_t* served, uint64_t* fallback) {
  MeshingOracle* o = static_cast<MeshingOracle*>(handle);
  *served = o->served;
  *fallback = o->fallback;
}

}  // extern "C"
