// pipeline.cu — the RGB-D stream runner behind sm_stream_run: the frame loop of APP/main.cc:885-1223
// (upload, the five pre-processing launches, CUDASurfelReconstruction::Integrate()) over a stream
// whose frames are resident in HBM or in pinned host memory.
//
// Three ways to run the same kernels:
//
//   frame graph (default)   one instantiated CUDA graph per steady-state step; a step holds the
//                           kernels of THREE consecutive frames that do not depend on each other:
//                             crit  (frame f)     integrate -> update_neighbors ┐
//                                                 scan ─┐ └-> create ───────────┴-> reg_accumulate -> reg_step
//                             front (frame f + 1) (create ->) project -> associate -> {merge | blend}
//                             pre   (frame f + 2) bilateral+outlier -> erode/normals/radii (+ raster clears)
//                           Per frame the host updates the kernel-node arguments of the executable
//                           graph (poses, raster pointers, count slot: by-value arguments, no device
//                           round trip) and launches it: 1 launch + 12 argument updates instead of 12
//                           launches + ~20 event records / waits; the hand-overs between the kernels
//                           are graph edges, the same-chain ones programmatic (griddepcontrol).
//   stream pipeline         SM_B200_GRAPH=0: the four-stream event pipeline of round 1
//                           (IntegrateFramePipelined, integrate.cu), kept for A/B measurements.
//   serial                  with sm_enable_timings / sm_profile_kernels: one kernel after the other on
//                           the caller's stream (stage events and per-kernel events need that).
//
// Three buffer sets (pre-processing outputs, association rasters, visible list) rotate with the
// frame index so that the three frames of a step never share a set.

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <string>

#include "sm_handle.cuh"

namespace smb {

namespace {

#define SM_CUDA(call)                                                                                   \
  do {                                                                                                  \
    const cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) return SetError(SM_ERR_CUDA, (std::string(#call) + ": " + cudaGetErrorString(e_)).c_str()); \
  } while (0)

constexpr int kDepthRing = 16;      // raw-depth frames resident at once (host-resident streams); >= K + 2 + slack
constexpr int kColorRing = 6;
constexpr int kIterationEvents = 32;

int EnvInt(const char* name, int fallback) {
  const char* e = std::getenv(name);
  return (e && e[0]) ? std::atoi(e) : fallback;
}

int EnsureRunBuffers(sm_reconstruction* r, bool on_host, bool depth_ring, bool color_ring, int source_width,
                     int source_height) {
  const int W = r->d.width, H = r->d.height;
  if (!r->run_depth[0]) {
    for (int i = 0; i < kSets; ++i) {
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&r->run_depth[i]), &r->run_depth_pitch, W * sizeof(u16), H));
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&r->run_depth_pre[i]), &r->run_depth_pitch, W * sizeof(u16), H));
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&r->run_normals[i]), &r->run_normals_pitch, W * sizeof(float2), H));
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&r->run_radius[i]), &r->run_radius_pitch, W * sizeof(float), H));
      SM_CUDA(cudaMemset2D(r->run_radius[i], r->run_radius_pitch, 0, W * sizeof(float), H));
    }
    for (int i = 0; i < 2; ++i) {
      SM_CUDA(cudaEventCreateWithFlags(&r->pipe.ev_create[i], cudaEventDisableTiming));
      SM_CUDA(cudaEventCreateWithFlags(&r->pipe.ev_update[i], cudaEventDisableTiming));
      SM_CUDA(cudaEventCreateWithFlags(&r->pre_done[i], cudaEventDisableTiming));
      SM_CUDA(cudaEventCreateWithFlags(&r->int_done[i], cudaEventDisableTiming));
    }
    SM_CUDA(cudaStreamCreateWithFlags(&r->pre_stream, cudaStreamNonBlocking));
    SM_CUDA(cudaStreamCreateWithFlags(&r->graph_stream, cudaStreamNonBlocking));
    SM_CUDA(cudaEventCreateWithFlags(&r->entry_event, cudaEventDisableTiming));
    SM_CUDA(cudaEventCreateWithFlags(&r->graph_exit, cudaEventDisableTiming));
    int least_priority = 0, greatest_priority = 0;
    SM_CUDA(cudaDeviceGetStreamPriorityRange(&least_priority, &greatest_priority));
    // SM_B200_PRIO (measurement hook of the stream pipeline): 0 (default) = no priorities, 1 = crit + side
    // high, 2 = front too.
    const int prio_mode = EnvInt("SM_B200_PRIO", 0);
    SM_CUDA(cudaStreamCreateWithPriority(&r->pipe.crit, cudaStreamNonBlocking, prio_mode >= 1 ? greatest_priority : least_priority));
    SM_CUDA(cudaStreamCreateWithPriority(&r->pipe.side, cudaStreamNonBlocking, prio_mode >= 1 ? greatest_priority : least_priority));
    SM_CUDA(cudaStreamCreateWithPriority(&r->pipe.front, cudaStreamNonBlocking, prio_mode >= 2 ? greatest_priority : least_priority));
    for (cudaEvent_t* e : {&r->pipe.ev_assoc, &r->pipe.ev_merge, &r->pipe.ev_blend, &r->pipe.ev_integrate,
                           &r->pipe.ev_reg}) {
      SM_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    }
  }
  if ((on_host || depth_ring) && !r->upload_stream) {
    SM_CUDA(cudaStreamCreateWithFlags(&r->upload_stream, cudaStreamNonBlocking));
    SM_CUDA(cudaEventCreateWithFlags(&r->upload_done, cudaEventDisableTiming));
    r->iteration_done.assign(kIterationEvents, nullptr);
    for (auto& e : r->iteration_done) SM_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  if (depth_ring && r->ring_depth.empty()) {
    r->ring_depth.assign(kDepthRing, nullptr);
    for (auto& b : r->ring_depth) {
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&b), &r->ring_depth_pitch, W * sizeof(u16), H));
    }
  }
  if (color_ring && r->ring_color.empty()) {
    r->ring_color.assign(kColorRing, nullptr);
    for (auto& b : r->ring_color) {
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&b), &r->ring_color_pitch, W * 3, H));
    }
  }
  // host frames at a pyramid level: full-size staging on the upload stream (one frame at a time)
  if (on_host && r->pyramid_level > 0 &&
      (r->pyramid_stage_width != source_width || r->pyramid_stage_height != source_height)) {
    SM_CUDA(cudaFree(r->pyramid_depth_stage));
    SM_CUDA(cudaFree(r->pyramid_color_stage));
    r->pyramid_depth_stage = nullptr;
    r->pyramid_color_stage = nullptr;
    r->pyramid_stage_width = r->pyramid_stage_height = 0;
    SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&r->pyramid_depth_stage), &r->pyramid_depth_stage_pitch,
                            source_width * sizeof(u16), source_height));
    SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&r->pyramid_color_stage), &r->pyramid_color_stage_pitch,
                            static_cast<size_t>(source_width) * 3, source_height));
    r->pyramid_stage_width = source_width;
    r->pyramid_stage_height = source_height;
  }
  if (r->median_iterations > 0 && !r->median_stage[0]) {
    for (int i = 0; i < 2; ++i) {
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&r->median_stage[i]), &r->median_stage_pitch, W * sizeof(u16), H));
    }
  }
  return SM_OK;
}

// Everything the three modes share about one call.
struct RunContext {
  sm_reconstruction* r;
  const sm_stream_desc* s;
  const sm_preprocess_params* pp;
  const sm_integrate_params* ip;
  int W, H, K, half, first, last;
  size_t frame_elems;
  int pyramid;            // input pyramid level: the stream's frames are (W << pyramid) x (H << pyramid)
  int source_W, source_H;
  size_t source_elems;    // pixels of one frame of the stream
  bool on_host;           // depth / colour frames are in (pinned) host memory
  bool depth_ring;        // raw depth maps pass through the device-side ring (host frames, median densify or pyramid)
  bool color_ring;        // colour images pass through the device-side ring (host frames or pyramid)
  int base_slot;          // Counters::surfel_count slot before the first frame
  uint64_t h2d = 0;

  int CountSlot(int frame) const { return (base_slot + (frame - first)) % kCountSlots; }
  const u16* Raw(int frame, size_t* pitch) const {
    if (depth_ring) { *pitch = r->ring_depth_pitch; return r->ring_depth[frame % kDepthRing]; }
    *pitch = W * sizeof(u16);
    return s->depth + frame_elems * frame;
  }
  const uint8_t* Color(int frame, size_t* pitch) const {
    if (color_ring) { *pitch = r->ring_color_pitch; return reinterpret_cast<const uint8_t*>(r->ring_color[frame % kColorRing]); }
    *pitch = static_cast<size_t>(W) * 3;
    return s->color + 3 * frame_elems * frame;
  }
  DeviceState SetState(int set) const {
    DeviceState d = r->d;
    d.assoc = r->assoc_set[set]; d.first_depth = r->first_depth_set[set]; d.supported = r->supported_set[set];
    d.vis = r->vis_set[set]; d.seg_count = r->seg_count_set[set]; d.merge_flag = r->merge_flag_set[set];
    d.upd_list = r->upd_list_set[set]; d.upd_count = r->upd_count_set[set];
    return d;
  }
  FrameParams Params(int frame, int set) const {
    size_t color_pitch;
    const uint8_t* color = Color(frame, &color_pitch);
    return MakeFrameParams(r, static_cast<u32>(frame), CountSlot(frame), *ip, r->run_depth[set], r->run_depth_pitch,
                           r->run_depth_pre[set], r->run_depth_pitch,
                           reinterpret_cast<const float*>(r->run_normals[set]), r->run_normals_pitch,
                           r->run_radius[set], r->run_radius_pitch, color, color_pitch, s->global_T_frame + 12 * frame,
                           s->frame_T_global + 12 * frame);
  }
  // Upload stream: raw depth map `frame` into its ring slot (main.cc:902-965), through the
  // MedianFilterAndDensifyDepthMap passes when configured (main.cc:927-939, there on the CPU).
  int EnqueueRawFrame(int frame) {
    u16* const slot = r->ring_depth[frame % kDepthRing];
    const u16* const src = s->depth + source_elems * frame;
    if (pyramid > 0) {
      // DownscaleUsingMedianWhileExcluding(0, W, H) of the full-size map (main.cc:951-952, there on the
      // CPU); host frames are uploaded full-size first, device frames are read in place
      const u16* full = src;
      size_t full_pitch = source_W * sizeof(u16);
      if (on_host) {
        SM_CUDA(cudaMemcpy2DAsync(r->pyramid_depth_stage, r->pyramid_depth_stage_pitch, src, full_pitch, full_pitch,
                                  source_H, cudaMemcpyHostToDevice, r->upload_stream));
        h2d += source_elems * sizeof(u16);
        full = r->pyramid_depth_stage;
        full_pitch = r->pyramid_depth_stage_pitch;
      }
      return StageDownscaleMedian(r->upload_stream, 0, source_W, source_H, full, full_pitch, W, H, slot,
                                  r->ring_depth_pitch);
    }
    const int n = r->median_iterations;
    u16* const target = n > 0 ? r->median_stage[0] : slot;
    const size_t target_pitch = n > 0 ? r->median_stage_pitch : r->ring_depth_pitch;
    SM_CUDA(cudaMemcpy2DAsync(target, target_pitch, src, W * sizeof(u16), W * sizeof(u16), H, cudaMemcpyDefault, r->upload_stream));
    if (on_host) h2d += frame_elems * sizeof(u16);
    if (n > 0) {
      return StageMedianDensify(r->upload_stream, n, W, H, r->median_stage[0], r->median_stage_pitch, slot,
                                r->ring_depth_pitch, r->median_stage[1], r->median_stage_pitch);
    }
    return SM_OK;
  }
  int EnqueueColorFrame(int frame) {
    if (pyramid > 0) {
      // ImagePyramid(color, pyramid) (main.cc:973-981, there on the CPU)
      const uint8_t* full = s->color + 3 * source_elems * frame;
      size_t full_pitch = static_cast<size_t>(source_W) * 3;
      if (on_host) {
        SM_CUDA(cudaMemcpy2DAsync(r->pyramid_color_stage, r->pyramid_color_stage_pitch, full, full_pitch, full_pitch,
                                  source_H, cudaMemcpyHostToDevice, r->upload_stream));
        h2d += source_elems * 3;
        full = r->pyramid_color_stage;
        full_pitch = r->pyramid_color_stage_pitch;
      }
      return StageColorPyramid(r->upload_stream, pyramid, source_W, source_H, full, full_pitch,
                               reinterpret_cast<u8*>(r->ring_color[frame % kColorRing]), r->ring_color_pitch);
    }
    SM_CUDA(cudaMemcpy2DAsync(r->ring_color[frame % kColorRing], r->ring_color_pitch, s->color + 3 * frame_elems * frame,
                              static_cast<size_t>(W) * 3, static_cast<size_t>(W) * 3, H, cudaMemcpyHostToDevice,
                              r->upload_stream));
    h2d += frame_elems * 3;
    return SM_OK;
  }
  void Others(int frame, const u16** others, size_t* pitches) const {  // main.cc:1046-1059
    for (int i = 0; i < half; ++i) {
      others[i] = Raw(frame - (i + 1), &pitches[i]);
      others[half + i] = Raw(frame + (i + 1), &pitches[half + i]);
    }
  }
};

// ---------------------------------------------------------------------------------------------
// serial mode / stream pipeline of round 1
// ---------------------------------------------------------------------------------------------
int RunStreams(RunContext& c, cudaStream_t stream, bool pipelined, uint32_t* integrated) {
  sm_reconstruction* r = c.r;
  const int W = c.W, H = c.H, half = c.half;
  r->pipe.have_frame = false;
  SM_CUDA(cudaEventRecord(r->entry_event, stream));
  for (cudaStream_t st : {r->pre_stream, r->pipe.crit, r->pipe.front, r->pipe.side}) {
    SM_CUDA(cudaStreamWaitEvent(st, r->entry_event, 0));
  }
  if (c.depth_ring) SM_CUDA(cudaStreamWaitEvent(r->upload_stream, r->entry_event, 0));
  int uploaded_until = c.first - half - 1;

  // Two-deep software pipeline: the pre-processing of frame f + 1 (pre_stream) runs while frame f
  // is integrated. Buffer set f & 1 holds frame f's pre-processing outputs and association rasters;
  // it is reused by frame f + 2 once Integrate(f) has finished.
  auto enqueue_preprocess = [&](int frame) -> int {
    const int set = frame & 1;
    const bool reuse = frame >= c.first + 2;
    if (c.depth_ring) {
      // Upload stream (main.cc:902-984): the new raw depth map(s) and this frame's colour image. The
      // rings are deep enough that the slots written now were last read two or more frames ago.
      if (reuse) {
        SM_CUDA(cudaStreamWaitEvent(r->upload_stream, r->pre_done[set], 0));
        SM_CUDA(cudaStreamWaitEvent(r->upload_stream, pipelined ? r->pipe.ev_create[set] : r->int_done[set], 0));
      }
      for (int f = uploaded_until + 1; f <= frame + half; ++f) {
        const int st = c.EnqueueRawFrame(f);
        if (st != SM_OK) return st;
      }
      uploaded_until = frame + half;
      if (c.color_ring) {
        const int st = c.EnqueueColorFrame(frame);
        if (st != SM_OK) return st;
      }
      SM_CUDA(cudaEventRecord(r->upload_done, r->upload_stream));
      SM_CUDA(cudaStreamWaitEvent(r->pre_stream, r->upload_done, 0));  // main.cc:995
    }
    if (reuse) {
      if (pipelined) {
        SM_CUDA(cudaStreamWaitEvent(r->pre_stream, r->pipe.ev_create[set], 0));
        SM_CUDA(cudaStreamWaitEvent(r->pre_stream, r->pipe.ev_update[set], 0));
      } else {
        SM_CUDA(cudaStreamWaitEvent(r->pre_stream, r->int_done[set], 0));
      }
    }
    const u16* others[8];
    size_t other_pitches[8];
    c.Others(frame, others, other_pitches);
    size_t raw_pitch;
    const u16* raw = c.Raw(frame, &raw_pitch);
    const int st = PreprocessFused(r->pre_stream, *c.pp, W, H, r->fx, r->fy, r->cx, r->cy, raw, raw_pitch, others,
                                   other_pitches, c.s->others_TR_reference + static_cast<size_t>(frame) * c.K * 12,
                                   r->scratch_B, r->scratch_B_pitch, r->run_depth[set], r->run_depth_pitch,
                                   r->run_normals[set], r->run_normals_pitch, r->run_radius[set], r->run_radius_pitch,
                                   r->assoc_set[set], r->first_depth_set[set], r->supported_set[set],
                                   pipelined ? r->run_depth_pre[set] : nullptr, r->run_depth_pitch,
                                   TimelineSlot(r->d, static_cast<u32>(frame), KID_BILATERAL_OUTLIER),
                                   TimelineSlot(r->d, static_cast<u32>(frame), KID_ERODE_NORMALS_RADII), r->ScratchBMap());
    if (st != SM_OK) return st;
    SM_CUDA(cudaEventRecord(r->pre_done[set], r->pre_stream));
    return SM_OK;
  };

  int status = SM_OK;
  if (c.first < c.last) {
    status = enqueue_preprocess(c.first);
    if (status != SM_OK) return status;
  }
  for (int frame = c.first; frame < c.last; ++frame) {
    const int set = frame & 1;
    if (frame + 1 < c.last) {
      status = enqueue_preprocess(frame + 1);
      if (status != SM_OK) return status;
    }
    SM_CUDA(cudaStreamWaitEvent(pipelined ? r->pipe.front : stream, r->pre_done[set], 0));
    r->d.assoc = r->assoc_set[set]; r->d.first_depth = r->first_depth_set[set]; r->d.supported = r->supported_set[set];
    r->d.vis = r->vis_set[set]; r->d.seg_count = r->seg_count_set[set]; r->d.merge_flag = r->merge_flag_set[set];
    r->d.upd_list = r->upd_list_set[set]; r->d.upd_count = r->upd_count_set[set];
    if (pipelined) {
      RecordOperation(r, static_cast<int>(static_cast<u32>(frame) - static_cast<u32>(c.ip->regularization_frame_window_size)));
      const FrameParams f = c.Params(frame, set);
      r->last_tiebreak = f.tb;
      RegularizeArgs reg;
      reg.iterations = c.ip->regularization_iterations_per_integration_iteration;
      reg.disable_denoising = reg.iterations == 0;
      reg.radius_factor = c.ip->radius_factor_for_regularization_neighbors;
      reg.regularizer_weight = c.ip->regularizer_weight;
      reg.window = c.ip->regularization_frame_window_size;
      status = IntegrateFramePipelined(r->pipe.front, &r->pipe, set, r->d, f, c.ip->do_blending != 0, reg, r->plan);
      if (status != SM_OK) return status;
      r->count_slot = (r->count_slot + 1) % kCountSlots;
    } else {
      r->rasters_cleared = true;
      size_t color_pitch;
      const uint8_t* color = c.Color(frame, &color_pitch);
      status = IntegrateImpl(r, stream, static_cast<u32>(frame), *c.ip, r->run_depth[set], r->run_depth_pitch,
                             reinterpret_cast<const float*>(r->run_normals[set]), r->run_normals_pitch,
                             r->run_radius[set], r->run_radius_pitch, color, color_pitch,
                             c.s->global_T_frame + 12 * frame, c.s->frame_T_global + 12 * frame);
      if (status != SM_OK) return status;
      SM_CUDA(cudaEventRecord(r->int_done[set], stream));
    }
    ++*integrated;
  }
  if (pipelined && r->pipe.have_frame) SM_CUDA(cudaStreamWaitEvent(stream, r->pipe.ev_reg, 0));  // join
  return SM_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// frame graph
// ---------------------------------------------------------------------------------------------
struct FrameGraph {
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  std::vector<cudaGraphNode_t> nodes;   // same order as the KernelLaunch list of a step
  std::vector<const void*> funcs;
  // what the graph was built for
  int blending = -1, reg_launches = -1, pdl = -1, prio = -1, order = -1;
  size_t blend_smem = 0;
  dim3 scan_grid;
};

void DestroyFrameGraph(FrameGraph* g) {
  if (!g) return;
  if (g->exec) cudaGraphExecDestroy(g->exec);
  if (g->graph) cudaGraphDestroy(g->graph);
  delete g;
}

namespace {

// Positions in the launch list of one step.
struct StepLayout {
  int integrate, scan, update, create, reg0, reg_count, project, project_tail /* -1: one projection kernel */, associate,
      merge, blend /* -1: none */, bilateral, tail, count;
};

StepLayout MakeLayout(bool blending, int reg_launches, bool split_project) {
  StepLayout l;
  int n = 0;
  l.integrate = n++; l.scan = n++; l.update = n++; l.create = n++;
  l.reg0 = n; l.reg_count = reg_launches; n += reg_launches;
  l.project = n++;
  l.project_tail = split_project ? n++ : -1;
  l.associate = n++; l.merge = n++;
  l.blend = blending ? n++ : -1;
  l.bilateral = n++; l.tail = n++;
  l.count = n;
  return l;
}

cudaKernelNodeParams NodeParams(const KernelLaunch& k) {
  cudaKernelNodeParams p = {};
  p.func = const_cast<void*>(k.func);
  p.gridDim = k.grid;
  p.blockDim = k.block;
  p.sharedMemBytes = static_cast<unsigned>(k.smem);
  p.kernelParams = const_cast<void**>(k.args);
  p.extra = nullptr;
  return p;
}

// Builds and instantiates the graph of one step from the launch list of its first use.
constexpr int kDefaultGraphOrder = 0;

int BuildFrameGraph(FrameGraph* g, const StepLayout& l, const std::vector<KernelLaunch>& launches, int pdl) {
  SM_CUDA(cudaGraphCreate(&g->graph, 0));
  g->nodes.assign(l.count, nullptr);
  g->funcs.assign(l.count, nullptr);
  for (int i = 0; i < l.count; ++i) {
    const cudaKernelNodeParams p = NodeParams(launches[i]);
    SM_CUDA(cudaGraphAddKernelNode(&g->nodes[i], g->graph, nullptr, 0, &p));
    g->funcs[i] = launches[i].func;
  }
  // SM_B200_GRAPH_PRIO (A/B hook): launch priorities of the nodes. 1 = the dependency chain that ends a
  // step (integrate -> create -> project -> associate -> blend) above everything else; 2 = additionally
  // the pre-processing of frame f + 2 below everything else.
  if (const int prio = EnvInt("SM_B200_GRAPH_PRIO", 0)) {
    int least = 0, greatest = 0;
    SM_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    auto set_priority = [&](int node, int priority) -> int {
      if (node < 0) return SM_OK;
      cudaKernelNodeAttrValue v = {};
      v.priority = priority;
      SM_CUDA(cudaGraphKernelNodeSetAttribute(g->nodes[node], cudaKernelNodeAttributePriority, &v));
      return SM_OK;
    };
    const int mid = (least + greatest) / 2;
    for (int i = 0; i < l.count; ++i) { const int st = set_priority(i, prio >= 2 ? mid : least); if (st != SM_OK) return st; }
    for (int node : {l.integrate, l.create, l.project, l.project_tail, l.associate, l.blend}) { const int st = set_priority(node, greatest); if (st != SM_OK) return st; }
    if (prio >= 2) for (int node : {l.bilateral, l.tail}) { const int st = set_priority(node, least); if (st != SM_OK) return st; }
  }
  std::vector<cudaGraphNode_t> from, to;
  std::vector<cudaGraphEdgeData> data;
  // `programmatic`: the consumer follows its only producer on the same chain and starts with
  // griddepcontrol.wait (pdl_prologue), so it may be scheduled while the producer drains.
  auto edge = [&](int a, int b, bool programmatic) {
    from.push_back(g->nodes[a]);
    to.push_back(g->nodes[b]);
    cudaGraphEdgeData e = {};
    if (pdl == 2 || (pdl == 1 && programmatic)) {
      e.from_port = cudaGraphKernelNodePortProgrammatic;
      e.type = cudaGraphDependencyTypeProgrammatic;
    }
    data.push_back(e);
  };
  // crit (frame f)
  edge(l.integrate, l.update, true);
  edge(l.integrate, l.create, false);
  edge(l.scan, l.create, false);
  if (l.reg_count > 0) {
    edge(l.update, l.reg0, false);
    edge(l.create, l.reg0, false);
    for (int i = 1; i < l.reg_count; ++i) edge(l.reg0 + i - 1, l.reg0 + i, true);
  }
  // front (frame f + 1): the projection needs this step's integration and, for the segments that hold
  // this step's new surfels, its creation kernel
  if (l.project_tail >= 0) {
    edge(l.integrate, l.project, false);
    edge(l.create, l.project_tail, false);
    edge(l.project, l.associate, false);
    edge(l.project_tail, l.associate, false);
  } else {
    edge(l.create, l.project, false);
    edge(l.project, l.associate, true);
  }
  edge(l.associate, l.merge, false);
  if (l.blend >= 0) edge(l.associate, l.blend, true);
  // pre (frame f + 2)
  edge(l.bilateral, l.tail, true);
  // SM_B200_GRAPH_ORDER (bit mask): ordering-only edges. The kernels of a step are launched with grids that fill
  // the register file, so whichever of two ready kernels gets the SMs first runs alone; these edges let the
  // chain that ends the step (integrate -> create -> project -> associate -> blend) go first where both are ready:
  //   1: create before update_neighbors      (both wait for integrate)
  //   2: associate(f + 1) before the regularisation of frame f
  //   4: merge(f + 1) before the regularisation of frame f
  //   8: project(f + 1) before update_neighbors(f)
  const int order = EnvInt("SM_B200_GRAPH_ORDER", kDefaultGraphOrder);
  if (order & 1) edge(l.create, l.update, false);
  if ((order & 2) && l.reg_count > 0) edge(l.associate, l.reg0, false);
  if ((order & 4) && l.reg_count > 0) edge(l.merge, l.reg0, false);
  if (order & 8) edge(l.project_tail >= 0 ? l.project_tail : l.project, l.update, false);
  SM_CUDA(cudaGraphAddDependencies_v2(g->graph, from.data(), to.data(), data.data(), from.size()));
  SM_CUDA(cudaGraphInstantiate(&g->exec, g->graph, 0));
  return SM_OK;
}

int RunGraph(RunContext& c, cudaStream_t stream, uint32_t* integrated) {
  sm_reconstruction* r = c.r;
  const int W = c.W, H = c.H, half = c.half;
  const bool blending = c.ip->do_blending != 0;
  const int iterations = c.ip->regularization_iterations_per_integration_iteration;
  const bool disable_denoising = iterations == 0;
  const int reg_launches = disable_denoising ? 1 : 2 * iterations;
  const bool split_project = EnvInt("SM_B200_SPLIT_PROJECT", 0) != 0;
  const StepLayout l = MakeLayout(blending, reg_launches, split_project);
  const int pdl = EnvInt("SM_B200_GRAPH_PDL", 0);
  std::vector<KernelLaunch> launches(l.count);

  cudaStream_t gs = r->graph_stream;
  SM_CUDA(cudaEventRecord(r->entry_event, stream));
  SM_CUDA(cudaStreamWaitEvent(gs, r->entry_event, 0));
  if (c.depth_ring) SM_CUDA(cudaStreamWaitEvent(r->upload_stream, r->entry_event, 0));
  int uploaded_until = c.first - half - 1;
  const int it0 = c.first - 2;

  // smooth-position double buffer as the host tracks it (swapped by every denoising iteration)
  float4* smooth = r->d.smooth;
  float4* smooth_next = r->d.smooth_next;

  auto active = [&](int frame) { return frame >= c.first && frame < c.last; };
  auto clamp_frame = [&](int frame) { return frame < c.first ? c.first : (frame >= c.last ? c.last - 1 : frame); };

  for (int it = it0; it < c.last; ++it) {
    const int crit = it, front = it + 1, pre = it + 2;
    // ---- uploads for the pre-processing of this step (host-resident streams) ----
    if (c.depth_ring && active(pre)) {
      for (int f = uploaded_until + 1; f <= pre + half; ++f) {
        // the slot held frame f - kDepthRing, last read by the pre-processing of frame f - kDepthRing + half
        const int last_reader_step = f - kDepthRing + half - 2;
        if (last_reader_step >= it0) SM_CUDA(cudaStreamWaitEvent(r->upload_stream, r->iteration_done[(last_reader_step - it0) % kIterationEvents], 0));
        const int st = c.EnqueueRawFrame(f);
        if (st != SM_OK) return st;
      }
      uploaded_until = pre + half;
      if (c.color_ring) {
        // the colour slot held frame pre - kColorRing, last read by the step that integrated it
        const int last_color_step = pre - kColorRing;
        if (last_color_step >= it0) SM_CUDA(cudaStreamWaitEvent(r->upload_stream, r->iteration_done[(last_color_step - it0) % kIterationEvents], 0));
        const int st = c.EnqueueColorFrame(pre);
        if (st != SM_OK) return st;
      }
      SM_CUDA(cudaEventRecord(r->upload_done, r->upload_stream));
      SM_CUDA(cudaStreamWaitEvent(gs, r->upload_done, 0));  // main.cc:995
    }

    // ---- arguments of the step ----
    int status = SM_OK;
    {  // crit: frame `crit`
      const int frame = clamp_frame(crit), set = frame % kSets;
      DeviceState d = c.SetState(set);
      d.smooth = smooth; d.smooth_next = smooth_next;
      if (active(crit)) RecordOperation(r, static_cast<int>(static_cast<u32>(frame) - static_cast<u32>(c.ip->regularization_frame_window_size)));
      FrameParams f = c.Params(frame, set);  // carries the operation epoch just recorded
      f.skip = active(crit) ? 0 : 1;
      if (active(crit)) r->last_tiebreak = f.tb;
      const FrameKernel kernels[4] = {FK_INTEGRATE, FK_SCAN, FK_UPDATE_NEIGHBORS, FK_CREATE};
      const int slots[4] = {l.integrate, l.scan, l.update, l.create};
      for (int i = 0; i < 4; ++i) {
        status = DescribeFrameKernel(kernels[i], r->plan, d, f, &launches[slots[i]]);
        if (status != SM_OK) return status;
      }
      const int old_slot = f.count_slot, new_slot = (f.count_slot + 1) % kCountSlots;
      if (active(crit)) NoteIntegratedFrame(d, static_cast<u32>(frame));
      for (int i = 0; i < (disable_denoising ? 1 : iterations); ++i) {
        KernelLaunch* first = &launches[l.reg0 + (disable_denoising ? 0 : 2 * i)];
        KernelLaunch* second = disable_denoising ? nullptr : first + 1;
        DescribeRegularize(first, second, !active(crit), r->plan, d, disable_denoising, static_cast<u32>(frame),
                           c.ip->radius_factor_for_regularization_neighbors, c.ip->regularizer_weight,
                           c.ip->regularization_frame_window_size, new_slot, i == 0 ? old_slot : -1);
        if (!disable_denoising && active(crit)) {  // k_reg_step fills the other smooth buffer
          float4* const filled = smooth_next;
          smooth_next = smooth;
          smooth = filled;
          d.smooth = smooth; d.smooth_next = smooth_next;
          NoteRegStep(d, static_cast<u32>(frame), c.ip->regularization_frame_window_size);
        }
      }
      r->d.reg_t_prev = d.reg_t_prev;   // the next step's SetState starts from here
      r->d.reg_full_sweep = d.reg_full_sweep;
      if (active(crit)) ++*integrated;
    }
    {  // front: frame `front`
      const int frame = clamp_frame(front), set = frame % kSets;
      const DeviceState d = c.SetState(set);
      FrameParams f = c.Params(frame, set);
      f.skip = active(front) ? 0 : 1;
      const FrameKernel kernels[5] = {split_project ? FK_PROJECT_MAIN : FK_PROJECT, FK_PROJECT_TAIL, FK_ASSOCIATE, FK_MERGE, FK_BLEND};
      const int slots[5] = {l.project, l.project_tail, l.associate, l.merge, l.blend};
      for (int i = 0; i < 5; ++i) {
        if (slots[i] < 0) continue;
        status = DescribeFrameKernel(kernels[i], r->plan, d, f, &launches[slots[i]]);
        if (status != SM_OK) return status;
      }
    }
    {  // pre: frame `pre`
      const int frame = clamp_frame(pre), set = frame % kSets;
      const u16* others[8];
      size_t other_pitches[8];
      c.Others(frame, others, other_pitches);
      size_t raw_pitch;
      const u16* raw = c.Raw(frame, &raw_pitch);
      status = DescribePreprocess(&launches[l.bilateral], &launches[l.tail], !active(pre), *c.pp, W, H, r->fx, r->fy,
                                  r->cx, r->cy, raw, raw_pitch, others, other_pitches,
                                  c.s->others_TR_reference + static_cast<size_t>(frame) * c.K * 12, r->scratch_B,
                                  r->scratch_B_pitch, r->run_depth[set], r->run_depth_pitch, r->run_normals[set],
                                  r->run_normals_pitch, r->run_radius[set], r->run_radius_pitch, r->assoc_set[set],
                                  r->first_depth_set[set], r->supported_set[set], r->run_depth_pre[set],
                                  r->run_depth_pitch, TimelineSlot(r->d, static_cast<u32>(frame), KID_BILATERAL_OUTLIER),
                                  TimelineSlot(r->d, static_cast<u32>(frame), KID_ERODE_NORMALS_RADII), r->ScratchBMap());
      if (status != SM_OK) return status;
    }

    // ---- (re)build on the first step or when the shape changed, else update the node arguments ----
    FrameGraph* g = r->graph;
    const int prio = EnvInt("SM_B200_GRAPH_PRIO", 0);
    const int order = EnvInt("SM_B200_GRAPH_ORDER", kDefaultGraphOrder);
    bool rebuild = g == nullptr || g->blending != (blending ? 1 : 0) || g->reg_launches != reg_launches || g->pdl != pdl ||
                   g->prio != prio || g->order != order || static_cast<int>(g->nodes.size()) != l.count;
    if (!rebuild) {
      for (int i = 0; i < l.count && !rebuild; ++i) rebuild = g->funcs[i] != launches[i].func;
      if (l.blend >= 0) rebuild = rebuild || g->blend_smem != launches[l.blend].smem;
    }
    if (rebuild) {
      if (g) { SM_CUDA(cudaStreamSynchronize(gs)); DestroyFrameGraph(g); r->graph = nullptr; }
      g = new FrameGraph();
      r->graph = g;
      g->blending = blending ? 1 : 0; g->reg_launches = reg_launches; g->pdl = pdl; g->prio = prio; g->order = order;
      g->blend_smem = l.blend >= 0 ? launches[l.blend].smem : 0;
      status = BuildFrameGraph(g, l, launches, pdl);
      if (status != SM_OK) return status;
    } else {
      for (int i = 0; i < l.count; ++i) {
        const cudaKernelNodeParams p = NodeParams(launches[i]);
        SM_CUDA(cudaGraphExecKernelNodeSetParams(g->exec, g->nodes[i], &p));
      }
    }
    SM_CUDA(cudaGraphLaunch(g->exec, gs));
    CountLaunches(static_cast<unsigned long long>(l.count));
    if (c.depth_ring) SM_CUDA(cudaEventRecord(r->iteration_done[(it - it0) % kIterationEvents], gs));
  }
  r->d.smooth = smooth;
  r->d.smooth_next = smooth_next;
  {  // the handle's rasters / lists are those of the last integrated frame (sm_download_rasters, sm_frame_counters)
    const DeviceState last_set = c.SetState((c.last - 1) % kSets);
    r->d.assoc = last_set.assoc; r->d.first_depth = last_set.first_depth; r->d.supported = last_set.supported;
    r->d.vis = last_set.vis; r->d.seg_count = last_set.seg_count; r->d.merge_flag = last_set.merge_flag;
    r->d.upd_list = last_set.upd_list; r->d.upd_count = last_set.upd_count;
  }
  r->count_slot = c.CountSlot(c.last);
  SM_CUDA(cudaEventRecord(r->graph_exit, gs));
  SM_CUDA(cudaStreamWaitEvent(stream, r->graph_exit, 0));
  return SM_OK;
}

}  // namespace

int StreamRun(sm_reconstruction* r, cudaStream_t stream, const sm_stream_desc* s, const sm_preprocess_params* pp,
              const sm_integrate_params* ip, int first_frame, int last_frame, sm_stream_stats* stats) {
  RunContext c;
  c.r = r; c.s = s; c.pp = pp; c.ip = ip;
  c.W = r->d.width; c.H = r->d.height;
  c.pyramid = r->pyramid_level;
  if (c.pyramid > 0) {
    // main.cc:946-949
    if (r->median_iterations > 0) {
      return SetError(SM_ERR_INVALID_ARGUMENT, "pyramid_level > 0 cannot be combined with median_filter_and_densify_iterations > 0");
    }
    const int step = 1 << c.pyramid;
    if (s->width <= 0 || s->height <= 0 || s->width % step != 0 || s->height % step != 0 ||
        (s->width >> c.pyramid) != c.W || (s->height >> c.pyramid) != c.H) {
      return SetError(SM_ERR_INVALID_ARGUMENT, "stream size must be the handle's size times 2^pyramid_level");
    }
  } else if (s->width != c.W || s->height != c.H) {
    return SetError(SM_ERR_INVALID_ARGUMENT, "stream size mismatch");
  }
  c.source_W = s->width; c.source_H = s->height;
  c.source_elems = static_cast<size_t>(c.source_W) * c.source_H;
  c.K = pp->outlier_filtering_frame_count;
  c.half = c.K / 2;
  if (c.K < 2 || c.K > 8 || first_frame < c.half || last_frame > s->frame_count - c.half || first_frame > last_frame) {
    return SetError(SM_ERR_INVALID_ARGUMENT,
                    "frame range needs outlier_filtering_frame_count/2 frames on both sides (main.cc:987-992)");
  }
  c.first = first_frame; c.last = last_frame;
  c.frame_elems = static_cast<size_t>(c.W) * c.H;
  c.on_host = s->frames_on_host != 0;
  c.depth_ring = c.on_host || r->median_iterations > 0 || c.pyramid > 0;
  c.color_ring = c.on_host || c.pyramid > 0;
  c.base_slot = r->count_slot;
  int status = EnsureRunBuffers(r, c.on_host, c.depth_ring, c.color_ring, c.source_W, c.source_H);
  if (status != SM_OK) return status;
  const unsigned long long launches_before = LaunchCount();
  const auto host_t0 = std::chrono::steady_clock::now();
  r->last_stream = stream;

  // Per-kernel profiling and stage timings need the kernels one after the other on one stream.
  const bool serial = r->events.enabled || ProfilingEnabled();
  const int radius = static_cast<int>(pp->bilateral_filter_radius_factor * pp->bilateral_filter_sigma_xy + 0.5f);
  const bool use_graph = !serial && EnvInt("SM_B200_GRAPH", 1) != 0 && radius == 6 && first_frame < last_frame;
  uint32_t integrated = 0;
  if (use_graph) {
    status = RunGraph(c, stream, &integrated);
    if (status != SM_OK) cudaStreamSynchronize(r->graph_stream);  // leave no work of a failed call in flight
  } else {
    status = RunStreams(c, stream, !serial, &integrated);
    if (status != SM_OK) cudaDeviceSynchronize();
  }
  if (status != SM_OK) return status;
  const double host_enqueue_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count();
  status = FetchCounters(r, stream);  // one 32-byte D2H + sync for the whole call
  if (stats) {
    stats->frames_integrated = integrated;
    stats->surfels_size = r->host_counters->surfel_count[r->count_slot];
    stats->surfel_count = stats->surfels_size - r->host_counters->merge_count;
    stats->kernel_launches = LaunchCount() - launches_before;
    stats->h2d_bytes = c.h2d;
    stats->d2h_bytes = sizeof(Counters);
    stats->host_enqueue_ms = host_enqueue_ms;
  }
  return status;
}

}  // namespace smb
