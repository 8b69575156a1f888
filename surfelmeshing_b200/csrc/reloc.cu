// reloc.cu — the keyframe database of random-fern codes and sm_relocalise (DESIGN.md section 5.11). The rules F1-F7
// are in include/surfel_b200.h.
//
// A frame, on the caller's stream:
//   k_downscale_depth_median   raw depth -> the w x h fern depth in db scratch (StageDownscaleMedian, rule F1)
//   k_reloc_encode             one thread per fern: its colour block means, the nibble (F3), packed by warp shuffles
// add / query, then one synchronisation:
//   k_reloc_distance           one warp per stored keyframe: XOR of the codes, nonzero nibbles by popc (F4)
//   k_reloc_select             one block: the smallest keys (distance << 32 | index) by `candidates` rounds of a
//                              block minimum (F5), and for add the F6 decision and the append of the code
// Every call launches the same kernels whatever the data; sm_relocalise adds one tracking call per attempt.

#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "sm_handle.cuh"

namespace smb {

namespace {

constexpr int kEncodeBlock = 256;
constexpr int kDistanceBlock = 256;
constexpr int kDistanceWarps = kDistanceBlock / 32;
constexpr int kSelectBlock = 1024;
constexpr int kMaxFerns = 2048;
constexpr u32 kMaxCapacity = 1u << 20;

struct Fern {
  u16 x, y;
  u8 r, g, b, pad;
  double depth;   // t_D in metres (F2)
};

// The selection result, device and pinned host (one copy per add / query).
struct Selection {
  u32 found;
  u32 index[SM_RELOC_MAX_CANDIDATES];
  u32 distance[SM_RELOC_MAX_CANDIDATES];
  int appended;   // add: the new keyframe's index, -1
  int full;       // add: a frame that would be appended found the database at capacity
};

struct EncodeArgs {
  int ferns;
  int width, height;              // the handle's camera (colour input)
  int fern_width, fern_height;    // w x h (F1)
  const Fern* table;
  const u16* depth; size_t depth_pitch;   // the median-downscaled depth, w x h
  const u8* color; size_t color_pitch;    // raw packed u8x3, W x H
  double depth_scaling;
  u32* code;
};

struct DistanceArgs {
  u32 count, words;
  const u32* code;
  const u32* codes;               // [capacity][words]
  u32* distance;
};

struct SelectArgs {
  u32 count, words, capacity;
  int rounds;                     // query: candidates; add: 1
  int add, force;
  double max_distance;            // query: max_query_fraction * ferns (F5); add: add_fraction * ferns (F6)
  const u32* distance;
  const u32* code;
  u32* codes;
  Selection* out;
};

__global__ void __launch_bounds__(kEncodeBlock) k_reloc_encode(EncodeArgs a) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  u32 nibble = 0;
  if (f < a.ferns) {
    const Fern fern = a.table[f];
    const int x = fern.x, y = fern.y;
    const int x0 = static_cast<int>(static_cast<long long>(a.width) * x / a.fern_width);
    const int x1 = static_cast<int>(static_cast<long long>(a.width) * (x + 1) / a.fern_width);
    const int y0 = static_cast<int>(static_cast<long long>(a.height) * y / a.fern_height);
    const int y1 = static_cast<int>(static_cast<long long>(a.height) * (y + 1) / a.fern_height);
    u32 s[3] = {0, 0, 0};
    for (int v = y0; v < y1; ++v) {
      const u8* row = row_ptr(a.color, a.color_pitch, v);
      for (int u = x0; u < x1; ++u) {
        s[0] += row[3 * u]; s[1] += row[3 * u + 1]; s[2] += row[3 * u + 2];
      }
    }
    const u32 n = static_cast<u32>((x1 - x0) * (y1 - y0));
    const u32 R = (s[0] + n / 2) / n, G = (s[1] + n / 2) / n, B = (s[2] + n / 2) / n;
    const u16 D = row_ptr(a.depth, a.depth_pitch, y)[x];
    nibble = (R >= fern.r ? 1u : 0u) | (G >= fern.g ? 2u : 0u) | (B >= fern.b ? 4u : 0u) |
             (D > 0 && static_cast<double>(D) >= fern.depth * a.depth_scaling ? 8u : 0u);
  }
  // eight consecutive ferns (lanes 8k .. 8k+7) make one word; ferns is a multiple of 8
  u32 word = nibble << (4 * (f & 7));
  word |= __shfl_xor_sync(0xffffffffu, word, 1);
  word |= __shfl_xor_sync(0xffffffffu, word, 2);
  word |= __shfl_xor_sync(0xffffffffu, word, 4);
  if (f < a.ferns && (f & 7) == 0) a.code[f >> 3] = word;
}

__global__ void __launch_bounds__(kDistanceBlock) k_reloc_distance(DistanceArgs a) {
  const u32 k = blockIdx.x * kDistanceWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (k >= a.count) return;
  const u32* other = a.codes + static_cast<size_t>(k) * a.words;
  u32 d = 0;
  for (u32 w = lane; w < a.words; w += 32) {
    const u32 x = a.code[w] ^ other[w];
    d += __popc((x | (x >> 1) | (x >> 2) | (x >> 3)) & 0x11111111u);
  }
#pragma unroll
  for (int offset = 16; offset > 0; offset >>= 1) d += __shfl_down_sync(0xffffffffu, d, offset);
  if (lane == 0) a.distance[k] = d;
}

__device__ __forceinline__ unsigned long long block_min(unsigned long long v) {
  __shared__ unsigned long long warp_min[kSelectBlock / 32];
#pragma unroll
  for (int offset = 16; offset > 0; offset >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, offset));
  if ((threadIdx.x & 31) == 0) warp_min[threadIdx.x >> 5] = v;
  __syncthreads();
  v = ~0ull;
  for (int w = 0; w < kSelectBlock / 32; ++w) v = min(v, warp_min[w]);
  __syncthreads();
  return v;
}

__global__ void __launch_bounds__(kSelectBlock) k_reloc_select(SelectArgs a) {
  __shared__ int append;
  // keys are unique (the index is part of the key): round r finds the smallest key above round r-1's
  unsigned long long last = 0;
  bool first = true;
  u32 found = 0, min_distance = 0;
  for (int r = 0; r < a.rounds; ++r) {
    unsigned long long best = ~0ull;
    for (u32 k = threadIdx.x; k < a.count; k += kSelectBlock) {
      const unsigned long long key = (static_cast<unsigned long long>(a.distance[k]) << 32) | k;
      if ((first || key > last) && key < best) best = key;
    }
    best = block_min(best);
    if (best == ~0ull) break;
    first = false;
    last = best;
    const u32 d = static_cast<u32>(best >> 32);
    if (r == 0) min_distance = d;
    if (!a.add && static_cast<double>(d) > a.max_distance) break;   // F5: later keys are no closer
    if (threadIdx.x == 0 && !a.add) {
      a.out->index[found] = static_cast<u32>(best & 0xffffffffu);
      a.out->distance[found] = d;
    }
    ++found;
  }
  if (threadIdx.x == 0) {
    a.out->found = a.add ? 0 : found;
    int appended = -1, full = 0;
    if (a.add && (a.count == 0 || a.force || static_cast<double>(min_distance) > a.max_distance)) {
      if (a.count >= a.capacity) full = 1;
      else appended = static_cast<int>(a.count);
    }
    a.out->appended = appended;
    a.out->full = full;
    append = appended;
  }
  __syncthreads();
  if (append >= 0) {
    u32* dst = a.codes + static_cast<size_t>(append) * a.words;
    for (u32 w = threadIdx.x; w < a.words; w += kSelectBlock) dst[w] = a.code[w];
  }
}

u64 SplitMix64(u64* state) {
  u64 z = (*state += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

bool Finite(float v) { return std::isfinite(v); }

// w x h of Camera.scaled(level) (F1).
int FernSize(int size, int level) {
  return static_cast<int>(static_cast<double>(1.0f / static_cast<float>(1 << level)) * size + 0.5);
}

}  // namespace

}  // namespace smb

struct sm_keyframe_db {
  int device = 0;
  int width = 0, height = 0;            // the handle's camera
  int fern_width = 0, fern_height = 0;  // F1
  sm_reloc_params params{};
  smb::u32 words = 0;                   // ferns / 8
  smb::u32 count = 0;
  std::vector<float> poses;             // [capacity][12], host
  smb::Fern* table = nullptr;           // [ferns]
  smb::u32* codes = nullptr;            // [capacity][words]
  smb::u16* fern_depth = nullptr; size_t fern_depth_pitch = 0;
  smb::u32* code = nullptr;             // [words]: the frame being added or queried
  smb::u32* distance = nullptr;         // [capacity]
  smb::Selection* selection = nullptr;
  smb::Selection* host_selection = nullptr;   // pinned
};

namespace smb {

namespace {

void FreeDatabase(sm_keyframe_db* db) {
  cudaFree(db->table); cudaFree(db->codes); cudaFree(db->fern_depth); cudaFree(db->code); cudaFree(db->distance);
  cudaFree(db->selection);
  if (db->host_selection) cudaFreeHost(db->host_selection);
  delete db;
}

// The range checks of the header; nullptr when params are usable for a camera of width x height.
const char* CheckRelocParams(const sm_reloc_params& p, int width, int height) {
  if (p.level < 1 || p.level > 4) return "level must be in [1, 4]";
  const int w = FernSize(width, p.level), h = FernSize(height, p.level);
  if (w < 1 || h < 1 || (width + w - 1) / w > 16 || (height + h - 1) / h > 16)
    return "the fern image's blocks exceed 16 x 16 pixels at this level";
  if (p.ferns < 8 || p.ferns > kMaxFerns || p.ferns % 8 != 0) return "ferns must be a multiple of 8 in [8, 2048]";
  if (!(Finite(p.min_depth) && Finite(p.max_depth) && p.min_depth >= 0.f && p.min_depth < p.max_depth))
    return "need finite 0 <= min_depth < max_depth";
  if (p.capacity < 1 || p.capacity > kMaxCapacity) return "capacity must be in [1, 2^20]";
  if (!(Finite(p.add_fraction) && p.add_fraction >= 0.f && p.add_fraction <= 1.f)) return "add_fraction must be in [0, 1]";
  if (p.candidates < 1 || p.candidates > SM_RELOC_MAX_CANDIDATES) return "candidates must be in [1, 8]";
  if (!(Finite(p.max_query_fraction) && p.max_query_fraction >= 0.f && p.max_query_fraction <= 1.f))
    return "max_query_fraction must be in [0, 1]";
  if (!(Finite(p.accept_inlier_fraction) && p.accept_inlier_fraction >= 0.f && p.accept_inlier_fraction <= 1.f))
    return "accept_inlier_fraction must be in [0, 1]";
  if (!(Finite(p.accept_rms) && p.accept_rms >= 0.f)) return "accept_rms must be finite and >= 0";
  const sm_track_params& t = p.track;
  if (t.levels < 1 || t.levels > 4) return "track.levels must be in [1, 4]";
  for (int l = 0; l < 4; ++l) if (t.iterations[l] < 0) return "track.iterations must be >= 0";
  if (!(Finite(t.max_point_distance) && t.max_point_distance > 0.f)) return "track.max_point_distance must be > 0";
  if (!(Finite(t.max_normal_angle_deg) && t.max_normal_angle_deg >= 0.f && t.max_normal_angle_deg <= 180.f))
    return "track.max_normal_angle_deg must be in [0, 180]";
  if (!(Finite(t.min_inlier_fraction) && t.min_inlier_fraction >= 0.f && t.min_inlier_fraction <= 1.f))
    return "track.min_inlier_fraction must be in [0, 1]";
  if (!(Finite(t.convergence_rotation) && t.convergence_rotation >= 0.f && Finite(t.convergence_translation) &&
        t.convergence_translation >= 0.f))
    return "track convergence thresholds must be finite and >= 0";
  return nullptr;
}

int Bad(const char* call, const char* why) {
  return SetError(SM_ERR_INVALID_ARGUMENT, (std::string(call) + ": " + why).c_str());
}

// Checks of a frame's arguments (before any launch).
const char* CheckFrame(const sm_keyframe_db* db, const u16* depth, size_t depth_pitch, const u8* color,
                       size_t color_pitch, float depth_scaling) {
  if (!depth || !color) return "null frame";
  if (depth_pitch < sizeof(u16) * static_cast<size_t>(db->width) || color_pitch < 3 * static_cast<size_t>(db->width))
    return "a pitch is below the row size";
  if (!(Finite(depth_scaling) && depth_scaling > 0.f)) return "depth_scaling must be finite and > 0";
  return nullptr;
}

// F1 + F3: the median downscale, then the encode into `out`.
int Encode(sm_keyframe_db* db, cudaStream_t stream, const u16* depth, size_t depth_pitch, const u8* color,
           size_t color_pitch, float depth_scaling, u32* out) {
  int status = StageDownscaleMedian(stream, 0, db->width, db->height, depth, depth_pitch, db->fern_width,
                                    db->fern_height, db->fern_depth, db->fern_depth_pitch);
  if (status != SM_OK) return status;
  EncodeArgs a;
  a.ferns = db->params.ferns;
  a.width = db->width; a.height = db->height;
  a.fern_width = db->fern_width; a.fern_height = db->fern_height;
  a.table = db->table;
  a.depth = db->fern_depth; a.depth_pitch = db->fern_depth_pitch;
  a.color = color; a.color_pitch = color_pitch;
  a.depth_scaling = static_cast<double>(depth_scaling);
  a.code = out;
  {
    LaunchScope scope(stream, KID_RELOC_ENCODE);
    LaunchKernel(k_reloc_encode, dim3((a.ferns + kEncodeBlock - 1) / kEncodeBlock), dim3(kEncodeBlock), 0, stream, a);
  }
  return CheckLaunch("keyframe encode");
}

// Encode, distances and selection, then one synchronisation; the result is in db->host_selection.
int Select(sm_keyframe_db* db, cudaStream_t stream, const u16* depth, size_t depth_pitch, const u8* color,
           size_t color_pitch, float depth_scaling, bool add, bool force, int candidates, double max_distance) {
  int status = Encode(db, stream, depth, depth_pitch, color, color_pitch, depth_scaling, db->code);
  if (status != SM_OK) return status;
  {
    DistanceArgs a{db->count, db->words, db->code, db->codes, db->distance};
    const u32 blocks = db->count ? (db->count + kDistanceWarps - 1) / kDistanceWarps : 1;
    LaunchScope scope(stream, KID_RELOC_DISTANCE);
    LaunchKernel(k_reloc_distance, dim3(blocks), dim3(kDistanceBlock), 0, stream, a);
  }
  {
    SelectArgs a;
    a.count = db->count; a.words = db->words; a.capacity = db->params.capacity;
    a.rounds = add ? 1 : candidates;
    a.add = add ? 1 : 0; a.force = force ? 1 : 0;
    a.max_distance = max_distance;
    a.distance = db->distance; a.code = db->code; a.codes = db->codes;
    a.out = db->selection;
    LaunchScope scope(stream, KID_RELOC_SELECT);
    LaunchKernel(k_reloc_select, dim3(1), dim3(kSelectBlock), 0, stream, a);
  }
  status = CheckLaunch("keyframe select");
  if (status != SM_OK) return status;
  SM_CUDA(cudaMemcpyAsync(db->host_selection, db->selection, sizeof(Selection), cudaMemcpyDeviceToHost, stream));
  SM_CUDA(cudaStreamSynchronize(stream));
  return SM_OK;
}

double QueryBound(const sm_reloc_params& p) {
  return static_cast<double>(p.max_query_fraction) * static_cast<double>(p.ferns);
}

int CreateDatabase(sm_keyframe_db* db, const sm_reconstruction* r, const sm_reloc_params& p) {
  db->device = r->device;
  db->width = r->d.width; db->height = r->d.height;
  db->fern_width = FernSize(db->width, p.level); db->fern_height = FernSize(db->height, p.level);
  db->params = p;
  db->words = static_cast<u32>(p.ferns / 8);
  std::vector<Fern> table(p.ferns);
  u64 state = p.seed;
  const double lo = p.min_depth, hi = p.max_depth;
  for (int f = 0; f < p.ferns; ++f) {
    Fern& t = table[f];
    t.x = static_cast<u16>((SplitMix64(&state) >> 32) % static_cast<u64>(db->fern_width));
    t.y = static_cast<u16>((SplitMix64(&state) >> 32) % static_cast<u64>(db->fern_height));
    t.r = static_cast<u8>(SplitMix64(&state) >> 56);
    t.g = static_cast<u8>(SplitMix64(&state) >> 56);
    t.b = static_cast<u8>(SplitMix64(&state) >> 56);
    t.pad = 0;
    t.depth = lo + (hi - lo) * (static_cast<double>(SplitMix64(&state) >> 11) * 0x1.0p-53);
  }
  int device = 0;
  SM_CUDA(cudaGetDevice(&device));
  if (device != r->device) return Bad("sm_keyframe_db_create", "the current device is not the handle's");
  db->poses.assign(static_cast<size_t>(p.capacity) * 12, 0.f);
  SM_CUDA(cudaMalloc(&db->table, sizeof(Fern) * table.size()));
  SM_CUDA(cudaMemcpy(db->table, table.data(), sizeof(Fern) * table.size(), cudaMemcpyHostToDevice));
  SM_CUDA(cudaMalloc(&db->codes, sizeof(u32) * db->words * static_cast<size_t>(p.capacity)));
  SM_CUDA(cudaMallocPitch(&db->fern_depth, &db->fern_depth_pitch, sizeof(u16) * db->fern_width, db->fern_height));
  SM_CUDA(cudaMalloc(&db->code, sizeof(u32) * db->words));
  SM_CUDA(cudaMalloc(&db->distance, sizeof(u32) * static_cast<size_t>(p.capacity)));
  SM_CUDA(cudaMalloc(&db->selection, sizeof(Selection)));
  SM_CUDA(cudaMallocHost(&db->host_selection, sizeof(Selection)));
  return SM_OK;
}

}  // namespace

}  // namespace smb

using namespace smb;

extern "C" {

void sm_default_reloc_params(sm_reloc_params* p) {
  p->level = 3;
  p->ferns = 512;
  p->seed = 20150401ull;
  p->min_depth = 0.3f;
  p->max_depth = 4.0f;
  p->capacity = 4096;
  p->add_fraction = 0.2f;
  p->candidates = 1;
  p->max_query_fraction = 0.4f;
  sm_default_track_params(&p->track);
  p->track.max_point_distance = 0.1f;
  p->accept_inlier_fraction = 0.7f;
  p->accept_rms = 0.01f;
}

int sm_keyframe_db_create(sm_keyframe_db** out, sm_reconstruction* r, const sm_reloc_params* params) {
  const char* call = "sm_keyframe_db_create";
  if (!out || !r || !params) return Bad(call, "null argument");
  if (const char* why = CheckRelocParams(*params, r->d.width, r->d.height)) return Bad(call, why);
  sm_keyframe_db* db = new sm_keyframe_db;
  const int status = CreateDatabase(db, r, *params);
  if (status != SM_OK) {
    FreeDatabase(db);
    return status;
  }
  *out = db;
  return SM_OK;
}

void sm_keyframe_db_destroy(sm_keyframe_db* db) {
  if (db) FreeDatabase(db);
}

int sm_keyframe_db_reset(sm_keyframe_db* db) {
  if (!db) return Bad("sm_keyframe_db_reset", "null argument");
  db->count = 0;
  return SM_OK;
}

int sm_keyframe_db_count(sm_keyframe_db* db, uint32_t* out) {
  if (!db || !out) return Bad("sm_keyframe_db_count", "null argument");
  *out = db->count;
  return SM_OK;
}

int sm_keyframe_db_encode(sm_keyframe_db* db, void* stream, const uint16_t* depth, size_t depth_pitch,
                          const uint8_t* color, size_t color_pitch, float depth_scaling, uint32_t* out_codes) {
  const char* call = "sm_keyframe_db_encode";
  if (!db || !out_codes) return Bad(call, "null argument");
  if (const char* why = CheckFrame(db, depth, depth_pitch, color, color_pitch, depth_scaling)) return Bad(call, why);
  return Encode(db, static_cast<cudaStream_t>(stream), depth, depth_pitch, color, color_pitch, depth_scaling, out_codes);
}

int sm_keyframe_db_add(sm_keyframe_db* db, void* stream, const uint16_t* depth, size_t depth_pitch,
                       const uint8_t* color, size_t color_pitch, float depth_scaling, const float global_T_frame[12],
                       int32_t force, int32_t* out_index, int32_t* out_full) {
  const char* call = "sm_keyframe_db_add";
  if (!db || !global_T_frame || !out_index || !out_full) return Bad(call, "null argument");
  if (const char* why = CheckFrame(db, depth, depth_pitch, color, color_pitch, depth_scaling)) return Bad(call, why);
  for (int k = 0; k < 12; ++k) if (!Finite(global_T_frame[k])) return Bad(call, "global_T_frame must be finite");
  const float* T = global_T_frame;   // a later guess of sm_relocalise: its rotation must have det > 0
  const double det = static_cast<double>(T[0]) * (static_cast<double>(T[5]) * T[10] - static_cast<double>(T[6]) * T[9]) -
                     static_cast<double>(T[1]) * (static_cast<double>(T[4]) * T[10] - static_cast<double>(T[6]) * T[8]) +
                     static_cast<double>(T[2]) * (static_cast<double>(T[4]) * T[9] - static_cast<double>(T[5]) * T[8]);
  if (!(det > 0.0)) return Bad(call, "the rotation of global_T_frame must have a positive determinant");
  const double bound = static_cast<double>(db->params.add_fraction) * static_cast<double>(db->params.ferns);
  const int status = Select(db, static_cast<cudaStream_t>(stream), depth, depth_pitch, color, color_pitch,
                            depth_scaling, true, force != 0, 1, bound);
  if (status != SM_OK) return status;
  const Selection& s = *db->host_selection;
  if (s.appended >= 0) {
    std::memcpy(&db->poses[static_cast<size_t>(s.appended) * 12], global_T_frame, sizeof(float) * 12);
    db->count = static_cast<u32>(s.appended) + 1;
  }
  *out_index = s.appended;
  *out_full = s.full;
  return SM_OK;
}

int sm_keyframe_db_query(sm_keyframe_db* db, void* stream, const uint16_t* depth, size_t depth_pitch,
                         const uint8_t* color, size_t color_pitch, float depth_scaling, int32_t* out_index,
                         uint32_t* out_distance, int32_t* out_found) {
  const char* call = "sm_keyframe_db_query";
  if (!db || !out_index || !out_distance || !out_found) return Bad(call, "null argument");
  if (const char* why = CheckFrame(db, depth, depth_pitch, color, color_pitch, depth_scaling)) return Bad(call, why);
  const int status = Select(db, static_cast<cudaStream_t>(stream), depth, depth_pitch, color, color_pitch,
                            depth_scaling, false, false, db->params.candidates, QueryBound(db->params));
  if (status != SM_OK) return status;
  const Selection& s = *db->host_selection;
  for (u32 i = 0; i < s.found; ++i) {
    out_index[i] = static_cast<int32_t>(s.index[i]);
    out_distance[i] = s.distance[i];
  }
  *out_found = static_cast<int32_t>(s.found);
  return SM_OK;
}

int sm_keyframe_db_read(sm_keyframe_db* db, uint32_t index, float pose[12], uint32_t* codes) {
  const char* call = "sm_keyframe_db_read";
  if (!db) return Bad(call, "null argument");
  if (index >= db->count) return Bad(call, "index must be below the keyframe count");
  if (pose) std::memcpy(pose, &db->poses[static_cast<size_t>(index) * 12], sizeof(float) * 12);
  if (codes) {
    const cudaError_t e = cudaMemcpy(codes, db->codes + static_cast<size_t>(index) * db->words, sizeof(u32) * db->words,
                                     cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return SetError(SM_ERR_CUDA, (std::string(call) + ": " + cudaGetErrorString(e)).c_str());
  }
  return SM_OK;
}

int sm_relocalise(sm_reconstruction* r, sm_keyframe_db* db, void* stream_v, const sm_reloc_params* params,
                  const sm_preprocess_params* pp, const sm_track_rgbd_params* rp, const uint16_t* depth,
                  size_t depth_pitch, const uint8_t* color, size_t color_pitch, float global_T_out[12],
                  sm_reloc_result* result) {
  const char* call = "sm_relocalise";
  if (!r || !db || !pp || !global_T_out || !result) return Bad(call, "null argument");
  if (db->width != r->d.width || db->height != r->d.height || db->device != r->device)
    return Bad(call, "the database was created from a handle of another camera size or device");
  const sm_reloc_params& p = params ? *params : db->params;
  if (const char* why = CheckRelocParams(p, r->d.width, r->d.height)) return Bad(call, why);
  const sm_reloc_params& q = db->params;
  if (p.level != q.level || p.ferns != q.ferns || p.seed != q.seed || p.min_depth != q.min_depth ||
      p.max_depth != q.max_depth || p.capacity != q.capacity)
    return Bad(call, "params must have the database's level, ferns, seed, depth range and capacity");
  if (const char* why = CheckFrame(db, depth, depth_pitch, color, color_pitch, pp->depth_scaling)) return Bad(call, why);
  // what the tracking calls would reject is rejected here, before the query launches anything
  sm_track_params tp = p.track;
  tp.model_source = SM_TRACK_CLOUD;
  if (!(Finite(pp->max_depth) && Finite(pp->depth_valid_region_radius) && Finite(pp->bilateral_filter_sigma_xy) &&
        Finite(pp->bilateral_filter_radius_factor) && Finite(pp->bilateral_filter_sigma_depth_factor)) ||
      BilateralRadius(*pp) < 0)
    return Bad(call, "the pre-processing parameters must be finite, with a bilateral radius >= 0");
  if (FernSize(r->d.width, tp.levels - 1) < 3 || FernSize(r->d.height, tp.levels - 1) < 3)
    return Bad(call, "the coarsest tracking level is smaller than 3 x 3 pixels");
  if (rp && !(Finite(rp->photometric_weight) && rp->photometric_weight >= 0.f && Finite(rp->max_intensity_residual) &&
              rp->max_intensity_residual >= 0.f && Finite(rp->min_gradient) && rp->min_gradient >= 0.f))
    return Bad(call, "the RGB-D params must be finite and >= 0");

  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int status = Select(db, stream, depth, depth_pitch, color, color_pitch, pp->depth_scaling, false, false,
                            p.candidates, QueryBound(p));
  if (status != SM_OK) return status;
  const Selection s = *db->host_selection;
  *result = sm_reloc_result{};
  result->keyframe = -1;
  result->rank = -1;
  for (int k = 0; k < 12; ++k) global_T_out[k] = std::nanf("");
  for (u32 i = 0; i < s.found; ++i) {
    const float* guess = &db->poses[static_cast<size_t>(s.index[i]) * 12];
    float pose[12];
    sm_track_result tr{};
    int st;
    if (rp) {
      sm_track_rgbd_result rr{};
      st = TrackFrameRGBD(r, stream, tp, *pp, TrackColor{rp, color, color_pitch, nullptr, 0}, depth, depth_pitch, guess,
                          pose, &rr);
      tr = rr.depth;
    } else {
      st = TrackFrame(r, stream, tp, *pp, depth, depth_pitch, guess, pose, &tr);
    }
    if (st != SM_OK) return st;
    result->attempts += 1;
    result->track = tr;
    if (tr.tracked &&
        static_cast<double>(tr.inliers) >= static_cast<double>(p.accept_inlier_fraction) *
                                               static_cast<double>(tr.valid_pixels) &&
        tr.rms_residual <= p.accept_rms) {
      std::memcpy(global_T_out, pose, sizeof(pose));
      result->relocalised = 1;
      result->keyframe = static_cast<int32_t>(s.index[i]);
      result->rank = static_cast<int32_t>(i);
      result->distance = s.distance[i];
      break;
    }
  }
  return SM_OK;
}

}  // extern "C"
