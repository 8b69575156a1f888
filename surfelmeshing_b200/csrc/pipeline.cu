// pipeline.cu — the RGB-D stream runner behind sm_stream_run: the frame loop of APP/main.cc:885-1223
// (upload, the five pre-processing launches, CUDASurfelReconstruction::Integrate()) over a stream
// whose frames are resident in HBM or in pinned host memory.
//
// Two ways to run the same kernels, both as one loop of steps (FrameLoop, Step):
//
//   frame graph (default)   one instantiated CUDA graph per steady-state step; a step holds the
//                           kernels of THREE consecutive frames that do not depend on each other:
//                             crit  (frame f)     integrate -> update_neighbors ┐
//                                                 scan ─┐ └-> create ───────────┴-> reg_accumulate -> reg_step
//                             front (frame f + 1) (create ->) project -> associate -> {merge | blend}
//                             pre   (frame f + 2) bilateral+outlier -> erode/normals/radii (+ raster clears)
//                                                 (bilateral -> outlier -> tail at a radius other than 6)
//                           Per frame the host updates the kernel-node arguments of the executable
//                           graph (poses, raster pointers, count slot: by-value arguments, no device
//                           round trip) and launches it: 1 launch + 12 argument updates instead of 12
//                           launches + ~20 event records / waits; the hand-overs between the kernels
//                           are graph edges.
//   serial                  with sm_enable_timings / sm_profile_kernels: step f pre-processes and integrates
//                           frame f, one kernel after the other on the caller's stream (stage events and
//                           per-kernel events need that).
//
// Three buffer sets (pre-processing outputs, association rasters, visible list) rotate with the
// frame index so that the three frames of a step never share a set.
//
// Incremental sessions (sm_session_begin / push / end) run the same steps one push at a time, and RunContext
// reads the frames either from the caller's arrays or from the session's rings (SessionFrames).

#include <algorithm>
#include <chrono>
#include <cstring>
#include <cstdio>
#include <string>

#include "sm_handle.cuh"

namespace smb {

struct FrameGraph;

// The frame loop's buffers, streams and events (sm_stream_run, sessions), created by the first call.
struct RunBuffers {
  // pre-processing outputs per buffer set
  u16* depth[kSets] = {}; size_t depth_pitch = 0;
  u16* depth_pre[kSets] = {};   // pre-blend copy of depth (merge runs next to blend)
  float2* normals[kSets] = {}; size_t normals_pitch = 0;
  float* radius[kSets] = {}; size_t radius_pitch = 0;
  cudaEvent_t entry_event = nullptr;   // the start of the frame loop on the caller's stream
  cudaStream_t graph_stream = nullptr;
  cudaEvent_t graph_exit = nullptr;
  FrameGraph* graph = nullptr;
  // host-resident streams: raw-depth / colour rings filled by the upload stream
  std::vector<u16*> ring_depth; size_t ring_depth_pitch = 0;
  std::vector<uchar3*> ring_color; size_t ring_color_pitch = 0;
  cudaStream_t upload_stream = nullptr;
  cudaEvent_t upload_done = nullptr;
  std::vector<cudaEvent_t> iteration_done;   // one event per step slot (ring reuse)
  // staging of the MedianFilterAndDensifyDepthMap passes (sm_reconstruction::median_iterations)
  u16* median_stage[2] = {nullptr, nullptr}; size_t median_stage_pitch = 0;
  // full-size staging of host frames at a pyramid level
  u16* pyramid_depth_stage = nullptr; size_t pyramid_depth_stage_pitch = 0;
  u8* pyramid_color_stage = nullptr; size_t pyramid_color_stage_pitch = 0;
  int pyramid_stage_width = 0, pyramid_stage_height = 0;
};

namespace {

constexpr int kDepthRing = 16;      // raw-depth frames resident at once (host-resident streams); >= K + 2 + slack
// Colour images resident at once. A session uploads frame p's image when p is pushed; the frame graph integrates
// it in the step that frame p + K/2 + 2 launches, so the slot must live K/2 + 3 frames (7 at K = 8).
constexpr int kColorRing = 8;
constexpr int kIterationEvents = 32;
// Session: poses and outlier-filter transforms of the newest frames. A push of frame p computes the transforms of
// frame p - K/2 (poses p - K .. p) and the step it launches integrates frame p - K/2 - 2: K + 1 frames, >= K + 3.
constexpr int kPoseRing = 16;
constexpr int kStagingSlots = 4;    // session: pinned staging of host frames (bounded run-ahead of the producer)

// Host-side frame source of a session: the pushed frames' poses and transforms in rings, and the frame
// being pushed (a device frame in place, or a host frame in pinned staging).
struct SessionFrames {
  float global_T_frame[kPoseRing][12];
  float frame_T_global[kPoseRing][12];
  float others_TR_reference[kPoseRing][8 * 12];
  const u16* depth = nullptr; size_t depth_pitch = 0;
  const uint8_t* color = nullptr; size_t color_pitch = 0;
};

int EnsureRunBuffers(sm_reconstruction* r, bool on_host, bool depth_ring, bool color_ring, int source_width,
                     int source_height) {
  const int W = r->d.width, H = r->d.height;
  if (!r->run) r->run = new RunBuffers();
  RunBuffers& b = *r->run;
  if (!b.depth[0]) {
    for (int i = 0; i < kSets; ++i) {
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&b.depth[i]), &b.depth_pitch, W * sizeof(u16), H));
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&b.depth_pre[i]), &b.depth_pitch, W * sizeof(u16), H));
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&b.normals[i]), &b.normals_pitch, W * sizeof(float2), H));
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&b.radius[i]), &b.radius_pitch, W * sizeof(float), H));
      SM_CUDA(cudaMemset2D(b.radius[i], b.radius_pitch, 0, W * sizeof(float), H));
    }
    SM_CUDA(cudaStreamCreateWithFlags(&b.graph_stream, cudaStreamNonBlocking));
    SM_CUDA(cudaEventCreateWithFlags(&b.entry_event, cudaEventDisableTiming));
    SM_CUDA(cudaEventCreateWithFlags(&b.graph_exit, cudaEventDisableTiming));
  }
  if ((on_host || depth_ring) && !b.upload_stream) {
    SM_CUDA(cudaStreamCreateWithFlags(&b.upload_stream, cudaStreamNonBlocking));
    SM_CUDA(cudaEventCreateWithFlags(&b.upload_done, cudaEventDisableTiming));
    b.iteration_done.assign(kIterationEvents, nullptr);
    for (auto& e : b.iteration_done) SM_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  if (depth_ring && b.ring_depth.empty()) {
    b.ring_depth.assign(kDepthRing, nullptr);
    for (auto& p : b.ring_depth) {
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&p), &b.ring_depth_pitch, W * sizeof(u16), H));
    }
  }
  if (color_ring && b.ring_color.empty()) {
    b.ring_color.assign(kColorRing, nullptr);
    for (auto& p : b.ring_color) {
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&p), &b.ring_color_pitch, W * 3, H));
    }
  }
  // host frames at a pyramid level: full-size staging on the upload stream (one frame at a time)
  if (on_host && r->pyramid_level > 0 &&
      (b.pyramid_stage_width != source_width || b.pyramid_stage_height != source_height)) {
    SM_CUDA(cudaFree(b.pyramid_depth_stage));
    SM_CUDA(cudaFree(b.pyramid_color_stage));
    b.pyramid_depth_stage = nullptr;
    b.pyramid_color_stage = nullptr;
    b.pyramid_stage_width = b.pyramid_stage_height = 0;
    SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&b.pyramid_depth_stage), &b.pyramid_depth_stage_pitch,
                            source_width * sizeof(u16), source_height));
    SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&b.pyramid_color_stage), &b.pyramid_color_stage_pitch,
                            static_cast<size_t>(source_width) * 3, source_height));
    b.pyramid_stage_width = source_width;
    b.pyramid_stage_height = source_height;
  }
  if (r->median_iterations > 0 && !b.median_stage[0]) {
    for (int i = 0; i < 2; ++i) {
      SM_CUDA(cudaMallocPitch(reinterpret_cast<void**>(&b.median_stage[i]), &b.median_stage_pitch, W * sizeof(u16), H));
    }
  }
  return SM_OK;
}

// Everything both modes share about one call (or one session).
struct RunContext {
  sm_reconstruction* r;
  const sm_stream_desc* s;        // sm_stream_run: the caller's arrays
  SessionFrames* ring = nullptr;  // session: the pushed frames (s is then unused)
  // Stream of the ring uploads: the upload stream, or (session, device frames) the stream the steps run on,
  // which waits for the caller's stream at every push anyway.
  cudaStream_t upload_override = nullptr;
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
  cudaStream_t Upload() const { return upload_override ? upload_override : r->run->upload_stream; }
  bool Active(int frame) const { return frame >= first && frame < last; }
  const float* GlobalT(int frame) const { return ring ? ring->global_T_frame[frame % kPoseRing] : s->global_T_frame + 12 * frame; }
  const float* FrameT(int frame) const { return ring ? ring->frame_T_global[frame % kPoseRing] : s->frame_T_global + 12 * frame; }
  const float* OthersTR(int frame) const {
    return ring ? ring->others_TR_reference[frame % kPoseRing] : s->others_TR_reference + static_cast<size_t>(frame) * K * 12;
  }
  // Source of the raw depth map / colour image `frame` on its way into the rings (sensor size).
  const u16* SourceDepth(int frame, size_t* pitch) const {
    if (ring) { *pitch = ring->depth_pitch; return ring->depth; }
    *pitch = source_W * sizeof(u16);
    return s->depth + source_elems * frame;
  }
  const uint8_t* SourceColor(int frame, size_t* pitch) const {
    if (ring) { *pitch = ring->color_pitch; return ring->color; }
    *pitch = static_cast<size_t>(source_W) * 3;
    return s->color + 3 * source_elems * frame;
  }
  const u16* Raw(int frame, size_t* pitch) const {
    if (depth_ring) { *pitch = r->run->ring_depth_pitch; return r->run->ring_depth[frame % kDepthRing]; }
    *pitch = W * sizeof(u16);
    return s->depth + frame_elems * frame;
  }
  const uint8_t* Color(int frame, size_t* pitch) const {
    if (color_ring) { *pitch = r->run->ring_color_pitch; return reinterpret_cast<const uint8_t*>(r->run->ring_color[frame % kColorRing]); }
    *pitch = static_cast<size_t>(W) * 3;
    return s->color + 3 * frame_elems * frame;
  }
  FrameParams Params(int frame, int set) const {
    size_t color_pitch;
    const uint8_t* color = Color(frame, &color_pitch);
    const RunBuffers& b = *r->run;
    return MakeFrameParams(r, static_cast<u32>(frame), CountSlot(frame), *ip, b.depth[set], b.depth_pitch,
                           b.depth_pre[set], b.depth_pitch, reinterpret_cast<const float*>(b.normals[set]),
                           b.normals_pitch, b.radius[set], b.radius_pitch, color, color_pitch, GlobalT(frame),
                           FrameT(frame));
  }
  // Upload stream: raw depth map `frame` into its ring slot (main.cc:902-965), through the
  // MedianFilterAndDensifyDepthMap passes when configured (main.cc:927-939, there on the CPU).
  int EnqueueRawFrame(int frame) {
    RunBuffers& b = *r->run;
    u16* const slot = b.ring_depth[frame % kDepthRing];
    size_t src_pitch;
    const u16* const src = SourceDepth(frame, &src_pitch);
    if (pyramid > 0) {
      // DownscaleUsingMedianWhileExcluding(0, W, H) of the full-size map (main.cc:951-952, there on the
      // CPU); host frames are uploaded full-size first, device frames are read in place
      const u16* full = src;
      size_t full_pitch = src_pitch;
      if (on_host) {
        SM_CUDA(cudaMemcpy2DAsync(b.pyramid_depth_stage, b.pyramid_depth_stage_pitch, src, src_pitch,
                                  source_W * sizeof(u16), source_H, cudaMemcpyHostToDevice, Upload()));
        h2d += source_elems * sizeof(u16);
        full = b.pyramid_depth_stage;
        full_pitch = b.pyramid_depth_stage_pitch;
      }
      return StageDownscaleMedian(Upload(), 0, source_W, source_H, full, full_pitch, W, H, slot,
                                  b.ring_depth_pitch);
    }
    const int n = r->median_iterations;
    u16* const target = n > 0 ? b.median_stage[0] : slot;
    const size_t target_pitch = n > 0 ? b.median_stage_pitch : b.ring_depth_pitch;
    SM_CUDA(cudaMemcpy2DAsync(target, target_pitch, src, src_pitch, W * sizeof(u16), H, cudaMemcpyDefault, Upload()));
    if (on_host) h2d += frame_elems * sizeof(u16);
    if (n > 0) {
      return StageMedianDensify(Upload(), n, W, H, b.median_stage[0], b.median_stage_pitch, slot,
                                b.ring_depth_pitch, b.median_stage[1], b.median_stage_pitch);
    }
    return SM_OK;
  }
  int EnqueueColorFrame(int frame) {
    RunBuffers& b = *r->run;
    size_t src_pitch;
    const uint8_t* const src = SourceColor(frame, &src_pitch);
    if (pyramid > 0) {
      // ImagePyramid(color, pyramid) (main.cc:973-981, there on the CPU)
      const uint8_t* full = src;
      size_t full_pitch = src_pitch;
      if (on_host) {
        SM_CUDA(cudaMemcpy2DAsync(b.pyramid_color_stage, b.pyramid_color_stage_pitch, src, src_pitch,
                                  static_cast<size_t>(source_W) * 3, source_H, cudaMemcpyHostToDevice, Upload()));
        h2d += source_elems * 3;
        full = b.pyramid_color_stage;
        full_pitch = b.pyramid_color_stage_pitch;
      }
      return StageColorPyramid(Upload(), pyramid, source_W, source_H, full, full_pitch,
                               reinterpret_cast<u8*>(b.ring_color[frame % kColorRing]), b.ring_color_pitch);
    }
    SM_CUDA(cudaMemcpy2DAsync(b.ring_color[frame % kColorRing], b.ring_color_pitch, src, src_pitch,
                              static_cast<size_t>(W) * 3, H, cudaMemcpyDefault, Upload()));
    if (on_host) h2d += frame_elems * 3;
    return SM_OK;
  }
  void Others(int frame, const u16** others, size_t* pitches) const {  // main.cc:1046-1059
    for (int i = 0; i < half; ++i) {
      others[i] = Raw(frame - (i + 1), &pitches[i]);
      others[half + i] = Raw(frame + (i + 1), &pitches[half + i]);
    }
  }
};

}  // namespace

// ---------------------------------------------------------------------------------------------
// frame graph
// ---------------------------------------------------------------------------------------------
struct FrameGraph {
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t exec = nullptr;
  std::vector<cudaGraphNode_t> nodes;   // same order as the KernelLaunch list of a step
  std::vector<const void*> funcs;       // with the node count: the layout the graph was built for
  size_t blend_smem = 0;
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
  int integrate, scan, update, create, reg0, reg_count, project, associate, merge, blend /* -1: none */, bilateral,
      outlier /* -1: fused into the bilateral kernel */, tail, count;
};

StepLayout MakeLayout(bool blending, int reg_launches, bool fused_outlier) {
  StepLayout l;
  int n = 0;
  l.integrate = n++; l.scan = n++; l.update = n++; l.create = n++;
  l.reg0 = n; l.reg_count = reg_launches; n += reg_launches;
  l.project = n++; l.associate = n++; l.merge = n++;
  l.blend = blending ? n++ : -1;
  l.bilateral = n++;
  l.outlier = fused_outlier ? -1 : n++;
  l.tail = n++;
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
int BuildFrameGraph(FrameGraph* g, const StepLayout& l, const std::vector<KernelLaunch>& launches) {
  SM_CUDA(cudaGraphCreate(&g->graph, 0));
  g->nodes.assign(l.count, nullptr);
  g->funcs.assign(l.count, nullptr);
  for (int i = 0; i < l.count; ++i) {
    const cudaKernelNodeParams p = NodeParams(launches[i]);
    SM_CUDA(cudaGraphAddKernelNode(&g->nodes[i], g->graph, nullptr, 0, &p));
    g->funcs[i] = launches[i].func;
  }
  g->blend_smem = l.blend >= 0 ? launches[l.blend].smem : 0;
  std::vector<cudaGraphNode_t> from, to;
  auto edge = [&](int a, int b) {
    from.push_back(g->nodes[a]);
    to.push_back(g->nodes[b]);
  };
  // crit (frame f)
  edge(l.integrate, l.update);
  edge(l.integrate, l.create);
  edge(l.scan, l.create);
  if (l.reg_count > 0) {
    edge(l.update, l.reg0);
    edge(l.create, l.reg0);
    for (int i = 1; i < l.reg_count; ++i) edge(l.reg0 + i - 1, l.reg0 + i);
  }
  // front (frame f + 1): the projection needs this step's integration and creation
  edge(l.create, l.project);
  edge(l.project, l.associate);
  edge(l.associate, l.merge);
  if (l.blend >= 0) edge(l.associate, l.blend);
  // pre (frame f + 2)
  if (l.outlier >= 0) {
    edge(l.bilateral, l.outlier);
    edge(l.outlier, l.tail);
  } else {
    edge(l.bilateral, l.tail);
  }
  SM_CUDA(cudaGraphAddDependencies(g->graph, from.data(), to.data(), from.size()));
  SM_CUDA(cudaGraphInstantiate(&g->exec, g->graph, 0));
  return SM_OK;
}

// State of the frame loop that lives from one step to the next (one sm_stream_run call, or one session). Step `it`
// integrates frame `it` and pre-processes frame `it + ahead`.
struct FrameLoop {
  bool graph = false;
  int ahead = 0;                 // 2 in the frame graph (crit it, front it + 1, pre it + 2), 0 in serial mode
  cudaStream_t work = nullptr;   // the stream the steps run on: the graph stream, or (serial) the caller's stream
  bool blending = false, disable_denoising = false;
  int iterations = 0, reg_launches = 0;
  StepLayout l{};
  std::vector<KernelLaunch> launches;
  int it0 = 0;                 // first step
  int uploaded_until = 0;      // newest raw depth map enqueued into the ring
  bool color_at_push = false;  // a session uploads each colour image when the frame is pushed
};

int BeginLoop(RunContext& c, cudaStream_t stream, bool graph, FrameLoop* g) {
  const RunBuffers& b = *c.r->run;
  g->graph = graph;
  g->ahead = graph ? 2 : 0;
  g->work = graph ? b.graph_stream : stream;
  if (graph) {
    g->blending = c.ip->do_blending != 0;
    g->iterations = c.ip->regularization_iterations_per_integration_iteration;
    g->disable_denoising = g->iterations == 0;
    g->reg_launches = g->disable_denoising ? 1 : 2 * g->iterations;
    g->l = MakeLayout(g->blending, g->reg_launches, BilateralRadius(*c.pp) == 6);
    g->launches.assign(g->l.count, KernelLaunch{});
  }
  g->it0 = c.first - g->ahead;
  g->uploaded_until = c.first - c.half - 1;
  SM_CUDA(cudaEventRecord(b.entry_event, stream));
  if (g->work != stream) SM_CUDA(cudaStreamWaitEvent(g->work, b.entry_event, 0));
  if (c.depth_ring) SM_CUDA(cudaStreamWaitEvent(b.upload_stream, b.entry_event, 0));
  return SM_OK;
}

// The ring uploads of both modes: a slot is rewritten once the step that last read it has finished
// (iteration_done, recorded on the loop's stream after every step).
int WaitForStep(RunContext& c, const FrameLoop& g, int step) {
  if (step >= g.it0) SM_CUDA(cudaStreamWaitEvent(c.Upload(), c.r->run->iteration_done[(step - g.it0) % kIterationEvents], 0));
  return SM_OK;
}

// Upload stream: raw depth maps up to frame `until` into the ring.
int UploadDepth(RunContext& c, FrameLoop& g, int until) {
  for (int f = g.uploaded_until + 1; f <= until; ++f) {
    // the slot held frame f - kDepthRing, last read by the pre-processing of frame f - kDepthRing + half
    int st = WaitForStep(c, g, f - kDepthRing + c.half - g.ahead);
    if (st == SM_OK) st = c.EnqueueRawFrame(f);
    if (st != SM_OK) return st;
  }
  if (until > g.uploaded_until) g.uploaded_until = until;
  return SM_OK;
}

// Upload stream: colour image `frame` into the ring.
int UploadColor(RunContext& c, FrameLoop& g, int frame) {
  // the colour slot held frame - kColorRing, last read by the step that integrated it
  const int st = WaitForStep(c, g, frame - kColorRing);
  return st != SM_OK ? st : c.EnqueueColorFrame(frame);
}

// Frame graph: crit = it, front = it + 1, pre = it + 2.
int GraphStep(RunContext& c, FrameLoop& g, int it, uint32_t* integrated) {
  sm_reconstruction* r = c.r;
  RunBuffers& b = *r->run;
  const int W = c.W, H = c.H;
  const StepLayout& l = g.l;
  std::vector<KernelLaunch>& launches = g.launches;
  const bool disable_denoising = g.disable_denoising;
  const int iterations = g.iterations;
  auto clamp_frame = [&](int frame) { return frame < c.first ? c.first : (frame >= c.last ? c.last - 1 : frame); };

  const int crit = it, front = it + 1, pre = it + 2;
  int status = SM_OK;
  {  // crit: frame `crit`
    const int frame = clamp_frame(crit), set = frame % kSets;
    DeviceState d = r->d;   // smooth / smooth_next as the handle holds them (a Regularize() swaps them)
    UseSet(d, r->sets[set]);
    if (c.Active(crit)) RecordOperation(r, static_cast<int>(static_cast<u32>(frame) - static_cast<u32>(c.ip->regularization_frame_window_size)));
    FrameParams f = c.Params(frame, set);  // carries the operation epoch just recorded
    f.skip = c.Active(crit) ? 0 : 1;
    if (c.Active(crit)) r->last_tiebreak = f.tb;
    const FrameKernel kernels[4] = {FK_INTEGRATE, FK_SCAN, FK_UPDATE_NEIGHBORS, FK_CREATE};
    const int slots[4] = {l.integrate, l.scan, l.update, l.create};
    for (int i = 0; i < 4; ++i) {
      status = DescribeFrameKernel(kernels[i], r->plan, d, f, &launches[slots[i]]);
      if (status != SM_OK) return status;
    }
    const int old_slot = f.count_slot, new_slot = (f.count_slot + 1) % kCountSlots;
    if (c.Active(crit)) NoteIntegratedFrame(d, static_cast<u32>(frame));
    for (int i = 0; i < (disable_denoising ? 1 : iterations); ++i) {
      KernelLaunch* first = &launches[l.reg0 + (disable_denoising ? 0 : 2 * i)];
      KernelLaunch* second = disable_denoising ? nullptr : first + 1;
      DescribeRegularize(first, second, !c.Active(crit), r->plan, d, disable_denoising, static_cast<u32>(frame),
                         c.ip->radius_factor_for_regularization_neighbors, c.ip->regularizer_weight,
                         c.ip->regularization_frame_window_size, new_slot, i == 0 ? old_slot : -1);
      if (!disable_denoising && c.Active(crit)) {  // k_reg_step fills the other smooth buffer
        float4* const filled = d.smooth_next;
        d.smooth_next = d.smooth;
        d.smooth = filled;
        NoteRegStep(d, static_cast<u32>(frame), c.ip->regularization_frame_window_size);
      }
    }
    r->d.smooth = d.smooth;           // the next step's state starts from here
    r->d.smooth_next = d.smooth_next;
    r->d.reg_t_prev = d.reg_t_prev;
    r->d.reg_full_sweep = d.reg_full_sweep;
    if (c.Active(crit)) {
      ++*integrated;
      // the handle's rasters / lists / count are those of the newest integrated frame (sm_download_rasters,
      // sm_frame_counters, sm_surfel_count, the hand-off calls between the pushes of a session)
      UseSet(r->d, r->sets[set]);
      r->count_slot = new_slot;
      r->rasters_stale = false;
    }
  }
  {  // front: frame `front`
    const int frame = clamp_frame(front), set = frame % kSets;
    DeviceState d = r->d;
    UseSet(d, r->sets[set]);
    FrameParams f = c.Params(frame, set);
    f.skip = c.Active(front) ? 0 : 1;
    const FrameKernel kernels[4] = {FK_PROJECT, FK_ASSOCIATE, FK_MERGE, FK_BLEND};
    const int slots[4] = {l.project, l.associate, l.merge, l.blend};
    for (int i = 0; i < 4; ++i) {
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
    const BufferSet& s = r->sets[set];
    status = DescribePreprocess(&launches[l.bilateral], l.outlier >= 0 ? &launches[l.outlier] : nullptr,
                                &launches[l.tail], !c.Active(pre), *c.pp, W, H, r->fx, r->fy, r->cx, r->cy, raw,
                                raw_pitch, others, other_pitches, c.OthersTR(frame), r->scratch_B, r->scratch_B_pitch,
                                b.depth[set], b.depth_pitch, b.normals[set], b.normals_pitch, b.radius[set],
                                b.radius_pitch, s.assoc, s.first_depth, s.supported, b.depth_pre[set], b.depth_pitch,
                                TimelineSlot(r->d, static_cast<u32>(frame), KID_BILATERAL_OUTLIER),
                                TimelineSlot(r->d, static_cast<u32>(frame), KID_ERODE_NORMALS_RADII), r->scratch_B_map);
    if (status != SM_OK) return status;
  }

  // ---- (re)build on the first step or when the layout changed, else update the node arguments ----
  FrameGraph* fg = b.graph;
  bool rebuild = fg == nullptr || static_cast<int>(fg->nodes.size()) != l.count;
  if (!rebuild) {
    for (int i = 0; i < l.count && !rebuild; ++i) rebuild = fg->funcs[i] != launches[i].func;
    if (l.blend >= 0) rebuild = rebuild || fg->blend_smem != launches[l.blend].smem;
  }
  if (rebuild) {
    if (fg) { SM_CUDA(cudaStreamSynchronize(g.work)); DestroyFrameGraph(fg); b.graph = nullptr; }
    fg = new FrameGraph();
    b.graph = fg;
    status = BuildFrameGraph(fg, l, launches);
    if (status != SM_OK) return status;
  } else {
    for (int i = 0; i < l.count; ++i) {
      const cudaKernelNodeParams p = NodeParams(launches[i]);
      SM_CUDA(cudaGraphExecKernelNodeSetParams(fg->exec, fg->nodes[i], &p));
    }
  }
  SM_CUDA(cudaGraphLaunch(fg->exec, g.work));
  CountLaunches(static_cast<unsigned long long>(l.count));
  return SM_OK;
}

// Serial mode: pre-processing and Integrate() of frame `it`, one kernel after the other.
int SerialStep(RunContext& c, FrameLoop& g, int it, uint32_t* integrated) {
  sm_reconstruction* r = c.r;
  const RunBuffers& b = *r->run;
  const int set = it % kSets;
  const BufferSet& s = r->sets[set];
  const u16* others[8];
  size_t other_pitches[8];
  c.Others(it, others, other_pitches);
  size_t raw_pitch;
  const u16* raw = c.Raw(it, &raw_pitch);
  int status = PreprocessFused(g.work, *c.pp, c.W, c.H, r->fx, r->fy, r->cx, r->cy, raw, raw_pitch, others,
                               other_pitches, c.OthersTR(it), r->scratch_B, r->scratch_B_pitch, b.depth[set],
                               b.depth_pitch, b.normals[set], b.normals_pitch, b.radius[set], b.radius_pitch, s.assoc,
                               s.first_depth, s.supported, nullptr, 0, TimelineSlot(r->d, static_cast<u32>(it), KID_BILATERAL_OUTLIER),
                               TimelineSlot(r->d, static_cast<u32>(it), KID_ERODE_NORMALS_RADII), r->scratch_B_map);
  if (status != SM_OK) return status;
  UseSet(r->d, s);
  r->rasters_cleared = true;
  size_t color_pitch;
  const uint8_t* color = c.Color(it, &color_pitch);
  status = IntegrateImpl(r, g.work, static_cast<u32>(it), *c.ip, b.depth[set], b.depth_pitch,
                         reinterpret_cast<const float*>(b.normals[set]), b.normals_pitch, b.radius[set],
                         b.radius_pitch, color, color_pitch, c.GlobalT(it), c.FrameT(it));
  if (status != SM_OK) return status;
  ++*integrated;
  return SM_OK;
}

// One step of the loop. Afterwards the handle's state (smooth record buffers, count slot, rasters, regularisation
// window) is that after frame `it` when it was integrated.
int Step(RunContext& c, FrameLoop& g, int it, uint32_t* integrated) {
  const RunBuffers& b = *c.r->run;
  const int pre = it + g.ahead;
  if (c.depth_ring && c.Active(pre)) {  // the frames the pre-processing of this step reads
    int st = UploadDepth(c, g, pre + c.half);
    if (st == SM_OK && c.color_ring && !g.color_at_push) st = UploadColor(c, g, pre);
    if (st != SM_OK) return st;
    if (c.Upload() != g.work) {
      SM_CUDA(cudaEventRecord(b.upload_done, c.Upload()));
      SM_CUDA(cudaStreamWaitEvent(g.work, b.upload_done, 0));  // main.cc:995
    }
  }
  const int status = g.graph ? GraphStep(c, g, it, integrated) : SerialStep(c, g, it, integrated);
  if (status != SM_OK) return status;
  if (c.depth_ring) SM_CUDA(cudaEventRecord(b.iteration_done[(it - g.it0) % kIterationEvents], g.work));
  return SM_OK;
}

// `stream` waits for everything the loop has launched so far.
int JoinLoop(sm_reconstruction* r, const FrameLoop& g, cudaStream_t stream) {
  if (g.work == stream) return SM_OK;
  SM_CUDA(cudaEventRecord(r->run->graph_exit, g.work));
  SM_CUDA(cudaStreamWaitEvent(stream, r->run->graph_exit, 0));
  return SM_OK;
}

}  // namespace

namespace {

// Sizes, pyramid level and K of a stream run or a session (main.cc:946-949, 987-992).
int SetupContext(RunContext& c, sm_reconstruction* r, const sm_preprocess_params* pp, const sm_integrate_params* ip,
                 int width, int height) {
  c.r = r; c.pp = pp; c.ip = ip;
  c.W = r->d.width; c.H = r->d.height;
  c.pyramid = r->pyramid_level;
  if (c.pyramid > 0) {
    // main.cc:946-949
    if (r->median_iterations > 0) {
      return SetError(SM_ERR_INVALID_ARGUMENT, "pyramid_level > 0 cannot be combined with median_filter_and_densify_iterations > 0");
    }
    const int step = 1 << c.pyramid;
    if (width <= 0 || height <= 0 || width % step != 0 || height % step != 0 ||
        (width >> c.pyramid) != c.W || (height >> c.pyramid) != c.H) {
      return SetError(SM_ERR_INVALID_ARGUMENT, "stream size must be the handle's size times 2^pyramid_level");
    }
  } else if (width != c.W || height != c.H) {
    return SetError(SM_ERR_INVALID_ARGUMENT, "stream size mismatch");
  }
  c.source_W = width; c.source_H = height;
  c.source_elems = static_cast<size_t>(c.source_W) * c.source_H;
  c.K = pp->outlier_filtering_frame_count;
  c.half = c.K / 2;
  c.frame_elems = static_cast<size_t>(c.W) * c.H;
  c.base_slot = r->count_slot;
  return SM_OK;
}

// The frame graph runs unless per-kernel profiling or stage timings need the kernels one after the other on one
// stream.
bool GraphAllowed(const sm_reconstruction* r) { return !r->events.enabled && !ProfilingEnabled(); }

int RunLoop(RunContext& c, cudaStream_t stream, uint32_t* integrated) {
  FrameLoop g;
  int status = BeginLoop(c, stream, GraphAllowed(c.r), &g);
  for (int it = g.it0; it < c.last && status == SM_OK; ++it) status = Step(c, g, it, integrated);
  if (status != SM_OK) return status;
  return JoinLoop(c.r, g, stream);
}

void FillStats(sm_reconstruction* r, uint32_t integrated, unsigned long long launches_before, uint64_t h2d,
               double host_enqueue_ms, sm_stream_stats* stats) {
  if (!stats) return;
  stats->frames_integrated = integrated;
  stats->surfels_size = r->host_counters->surfel_count[r->count_slot];
  stats->surfel_count = stats->surfels_size - r->host_counters->merge_count;
  stats->kernel_launches = LaunchCount() - launches_before;
  stats->h2d_bytes = h2d;
  stats->d2h_bytes = sizeof(Counters);
  stats->host_enqueue_ms = host_enqueue_ms;
}

double MillisecondsSince(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

}  // namespace

}  // namespace smb

using namespace smb;

// The frame loop of APP/main.cc:885-1223 on a synthetic stream.
extern "C" int sm_stream_run(sm_reconstruction* r, void* stream_v, const sm_stream_desc* s,
                             const sm_preprocess_params* pp, const sm_integrate_params* ip, int32_t first_frame,
                             int32_t last_frame, sm_stream_stats* stats) {
  if (!r || !s || !pp || !ip) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_stream_run: null argument");
  if (r->session) return RejectInSession("sm_stream_run");
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  RunContext c;
  c.s = s;
  int status = SetupContext(c, r, pp, ip, s->width, s->height);
  if (status != SM_OK) return status;
  if (c.K < 2 || c.K > 8 || first_frame < c.half || last_frame > s->frame_count - c.half || first_frame > last_frame) {
    return SetError(SM_ERR_INVALID_ARGUMENT,
                    "frame range needs outlier_filtering_frame_count/2 frames on both sides (main.cc:987-992)");
  }
  c.first = first_frame; c.last = last_frame;
  c.on_host = s->frames_on_host != 0;
  c.depth_ring = c.on_host || r->median_iterations > 0 || c.pyramid > 0;
  c.color_ring = c.on_host || c.pyramid > 0;
  status = EnsureRunBuffers(r, c.on_host, c.depth_ring, c.color_ring, c.source_W, c.source_H);
  if (status != SM_OK) return status;
  const unsigned long long launches_before = LaunchCount();
  const auto host_t0 = std::chrono::steady_clock::now();
  r->last_stream = stream;

  uint32_t integrated = 0;
  if (c.first < c.last) status = RunLoop(c, stream, &integrated);
  if (status != SM_OK) {
    cudaDeviceSynchronize();  // leave no work of a failed call in flight
    return status;
  }
  const double host_enqueue_ms = MillisecondsSince(host_t0);
  status = FetchCounters(r, stream);  // one 32-byte D2H + sync for the whole call
  FillStats(r, integrated, launches_before, c.h2d, host_enqueue_ms, stats);
  return status;
}

// ---------------------------------------------------------------------------------------------
// incremental sessions (sm_session_begin / push / end)
// ---------------------------------------------------------------------------------------------

namespace smb {

namespace {

void OutlierFilterTransform(float depth_scaling, const float* global_T_ref, const float* other_T_global, float* out) {
  // scale(other_T_global) . scale(global_T_ref), both 3x4 with an implicit last row (0 0 0 1); the
  // translations are multiplied by depth_scaling. Every product and sum in double, in the order the header gives.
  const double s = depth_scaling;
  for (int row = 0; row < 3; ++row) {
    const double a0 = other_T_global[4 * row + 0], a1 = other_T_global[4 * row + 1], a2 = other_T_global[4 * row + 2];
    const double a3 = static_cast<double>(other_T_global[4 * row + 3]) * s;
    for (int col = 0; col < 4; ++col) {
      double b0 = global_T_ref[col], b1 = global_T_ref[4 + col], b2 = global_T_ref[8 + col];
      if (col == 3) { b0 *= s; b1 *= s; b2 *= s; }
      double v = a0 * b0;
      v = v + a1 * b1;
      v = v + a2 * b2;
      if (col == 3) v = v + a3;
      out[4 * row + col] = static_cast<float>(v);
    }
  }
}

}  // namespace

struct StreamSession {
  RunContext c;
  SessionFrames frames;
  sm_preprocess_params pp;
  sm_integrate_params ip;
  cudaStream_t stream = nullptr;
  FrameLoop loop;
  int next_step = 0;         // the next step to launch
  uint32_t pushed = 0, integrated = 0;
  int64_t last_integrated = -1;
  unsigned long long launches_before = 0;
  double host_ms = 0;
  uint8_t* staging[kStagingSlots] = {};        // pinned: depth then colour of one sensor-size frame
  cudaEvent_t staging_free[kStagingSlots] = {};
  cudaEvent_t entry = nullptr;     // recorded on `stream` at every push
  cudaEvent_t uploaded = nullptr;  // recorded on the upload stream after a push's uploads
  u32* merge_count = nullptr;      // device: Counters::merge_count as of the newest integrated frame (frame graph)
};

namespace {

void FreeSession(StreamSession* ss) {
  if (!ss) return;
  for (int i = 0; i < kStagingSlots; ++i) {
    if (ss->staging[i]) cudaFreeHost(ss->staging[i]);
    if (ss->staging_free[i]) cudaEventDestroy(ss->staging_free[i]);
  }
  if (ss->entry) cudaEventDestroy(ss->entry);
  if (ss->uploaded) cudaEventDestroy(ss->uploaded);
  if (ss->merge_count) cudaFree(ss->merge_count);
  delete ss;
}

// A CUDA error inside a session: leave no work in flight and close it, as sm_stream_run's failure path does.
int AbortSession(sm_reconstruction* r, int status) {
  cudaDeviceSynchronize();
  r->reported_merge_count = nullptr;
  FreeSession(r->session);
  r->session = nullptr;
  return status;
}

constexpr int kMaxSessionFrameIndex = 1 << 30;   // frame indices stay far from int overflow in the ring arithmetic

}  // namespace

}  // namespace smb

// An incremental session on the handle.
extern "C" int sm_session_begin(sm_reconstruction* r, void* stream_v, const sm_preprocess_params* pp,
                                const sm_integrate_params* ip, int32_t width, int32_t height,
                                uint32_t first_frame_index) {
  if (!r || !pp || !ip) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_begin: null argument");
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (r->session) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_begin: a stream session is already open on this handle");
  const int K = pp->outlier_filtering_frame_count;
  if (K < 2 || K > 8 || K % 2 != 0) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_begin: outlier_filtering_frame_count must be 2, 4, 6 or 8");
  if (first_frame_index >= static_cast<uint32_t>(kMaxSessionFrameIndex)) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_begin: first_frame_index must be below 2^30");
  StreamSession* ss = new StreamSession();
  ss->pp = *pp;
  ss->ip = *ip;
  ss->stream = stream;
  RunContext& c = ss->c;
  c.ring = &ss->frames;
  int status = SetupContext(c, r, &ss->pp, &ss->ip, width, height);
  if (status != SM_OK) { FreeSession(ss); return status; }
  c.first = static_cast<int>(first_frame_index) + c.half;
  c.last = kMaxSessionFrameIndex + 16;   // open until sm_session_end
  c.depth_ring = c.color_ring = true;   // every pushed frame is copied into the device rings
  // on_host = true: the pyramid staging for host frames; set per push afterwards
  status = EnsureRunBuffers(r, true, true, true, c.source_W, c.source_H);
  if (status != SM_OK) { FreeSession(ss); return status; }
  const size_t staging_bytes = c.source_elems * (sizeof(u16) + 3);
  for (int i = 0; i < kStagingSlots; ++i) {
    if (cudaMallocHost(&ss->staging[i], staging_bytes) != cudaSuccess ||
        cudaEventCreateWithFlags(&ss->staging_free[i], cudaEventDisableTiming) != cudaSuccess) {
      FreeSession(ss);
      return SetError(SM_ERR_CUDA, "sm_session_begin: pinned staging allocation failed");
    }
  }
  if (cudaEventCreateWithFlags(&ss->entry, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&ss->uploaded, cudaEventDisableTiming) != cudaSuccess ||
      cudaMalloc(&ss->merge_count, sizeof(u32)) != cudaSuccess) {
    FreeSession(ss);
    return SetError(SM_ERR_CUDA, "sm_session_begin: event creation failed");
  }
  ss->launches_before = LaunchCount();
  const auto host_t0 = std::chrono::steady_clock::now();
  r->session = ss;
  r->last_stream = stream;
  status = BeginLoop(c, stream, GraphAllowed(r), &ss->loop);
  ss->loop.color_at_push = true;
  ss->next_step = ss->loop.it0;
  ss->host_ms += MillisecondsSince(host_t0);
  if (status != SM_OK) return AbortSession(r, status);
  return SM_OK;
}

extern "C" int sm_session_push(sm_reconstruction* r, const uint16_t* depth, size_t depth_pitch, const uint8_t* color,
                               size_t color_pitch, int32_t frame_on_host, const float global_T_frame[12],
                               const float frame_T_global[12], sm_session_status* out) {
  if (!r) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_push: null argument");
  const bool on_host = frame_on_host != 0;
  StreamSession* ss = r->session;
  if (!ss) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_push: no stream session is open on this handle (sm_session_begin)");
  RunContext& c = ss->c;
  if (!depth || !color || !global_T_frame || !frame_T_global) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_push: null argument");
  const size_t depth_row = static_cast<size_t>(c.source_W) * sizeof(u16), color_row = static_cast<size_t>(c.source_W) * 3;
  if (depth_pitch < depth_row || color_pitch < color_row) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_push: pitch below the row size of the session's frames");
  const int p = c.first - c.half + static_cast<int>(ss->pushed);   // frame index of this push
  if (p >= kMaxSessionFrameIndex) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_push: frame index would reach 2^30");
  const auto host_t0 = std::chrono::steady_clock::now();
  cudaStream_t stream = ss->stream;
  r->last_stream = stream;

  // poses, and the outlier-filter transforms of the frame that now has K/2 successors (main.cc:1039-1058)
  std::memcpy(ss->frames.global_T_frame[p % kPoseRing], global_T_frame, 12 * sizeof(float));
  std::memcpy(ss->frames.frame_T_global[p % kPoseRing], frame_T_global, 12 * sizeof(float));
  const int ref = p - c.half;
  if (ref >= c.first) {
    float* out_tr = ss->frames.others_TR_reference[ref % kPoseRing];
    for (int i = 0; i < c.half; ++i) {
      OutlierFilterTransform(ss->pp.depth_scaling, c.GlobalT(ref), c.FrameT(ref - (i + 1)), out_tr + 12 * i);
      OutlierFilterTransform(ss->pp.depth_scaling, c.GlobalT(ref), c.FrameT(ref + (i + 1)), out_tr + 12 * (c.half + i));
    }
  }

  int status = SM_OK;
  auto cuda = [&](cudaError_t e, const char* what) {
    if (e != cudaSuccess && status == SM_OK) status = SetError(SM_ERR_CUDA, (std::string(what) + ": " + cudaGetErrorString(e)).c_str());
  };
  FrameLoop& loop = ss->loop;
  const int step = p - c.half - loop.ahead;   // the step that pre-processes frame p - K/2
  if (loop.graph && step >= loop.it0) {
    // The front half of the step counts the merges of frame step + 1 (k_merge) before that frame is integrated
    // in the next step. merge_count now holds the merges of the frames up to `step`: what the count queries
    // report until the next push (sm_surfel_count, sm_dump_state; FetchCounters).
    cuda(cudaMemcpyAsync(ss->merge_count, &r->d.counters->merge_count, sizeof(u32), cudaMemcpyDeviceToDevice, stream),
         "cudaMemcpyAsync");
    r->reported_merge_count = ss->merge_count;
  }
  // work enqueued on `stream` since the last push (hand-off calls, sm_regularize) comes first
  cuda(cudaEventRecord(ss->entry, stream), "cudaEventRecord");
  if (loop.work != stream) cuda(cudaStreamWaitEvent(loop.work, ss->entry, 0), "cudaStreamWaitEvent");
  int slot = -1;
  if (on_host) {
    // main.cc:942-944, 974-976: into pinned staging, so that the caller can reuse its buffer at once; blocks
    // only while this slot's previous frame is still being uploaded
    slot = static_cast<int>(ss->pushed % kStagingSlots);
    cuda(cudaEventSynchronize(ss->staging_free[slot]), "cudaEventSynchronize");
    u16* staged_depth = reinterpret_cast<u16*>(ss->staging[slot]);
    uint8_t* staged_color = ss->staging[slot] + c.source_elems * sizeof(u16);
    for (int y = 0; y < c.source_H; ++y) {
      std::memcpy(staged_depth + static_cast<size_t>(y) * c.source_W, reinterpret_cast<const uint8_t*>(depth) + y * depth_pitch, depth_row);
      std::memcpy(staged_color + static_cast<size_t>(y) * color_row, color + y * color_pitch, color_row);
    }
    ss->frames.depth = staged_depth; ss->frames.depth_pitch = depth_row;
    ss->frames.color = staged_color; ss->frames.color_pitch = color_row;
  } else {
    // device frames: copied after the work the caller enqueued on `stream` that produced them, on the stream
    // the steps run on, which is or has just waited for `stream`
    ss->frames.depth = depth; ss->frames.depth_pitch = depth_pitch;
    ss->frames.color = color; ss->frames.color_pitch = color_pitch;
  }
  c.on_host = on_host;
  c.upload_override = on_host ? nullptr : loop.work;
  // after the previous push's uploads, which may have run on the other stream (pyramid / median staging is shared)
  cuda(cudaStreamWaitEvent(c.Upload(), ss->uploaded, 0), "cudaStreamWaitEvent");
  if (status == SM_OK) status = UploadDepth(c, loop, p);
  if (status == SM_OK) status = UploadColor(c, loop, p);
  cuda(cudaEventRecord(ss->uploaded, c.Upload()), "cudaEventRecord");
  if (on_host) {
    cuda(cudaEventRecord(ss->staging_free[slot], r->run->upload_stream), "cudaEventRecord");
  } else {
    cuda(cudaStreamWaitEvent(stream, ss->uploaded, 0), "cudaStreamWaitEvent");   // the caller may overwrite the frame now
  }
  if (status != SM_OK) return AbortSession(r, status);
  ++ss->pushed;

  // pushing frame p completes the inputs of frame p - K/2: its pre-processing runs now
  if (step >= loop.it0) {
    status = Step(c, loop, step, &ss->integrated);
    if (status == SM_OK) status = JoinLoop(r, loop, stream);
    ss->next_step = step + 1;
    if (c.Active(step)) ss->last_integrated = step;
  }
  if (status != SM_OK) return AbortSession(r, status);
  ss->host_ms += MillisecondsSince(host_t0);
  if (out) {
    out->frames_pushed = ss->pushed;
    out->frames_integrated = ss->integrated;
    out->last_integrated_frame = ss->last_integrated;
  }
  return SM_OK;
}

namespace smb {

int SessionEnd(sm_reconstruction* r, sm_stream_stats* stats) {
  StreamSession* ss = r->session;
  if (!ss) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_end: no stream session is open on this handle (sm_session_begin)");
  RunContext& c = ss->c;
  const auto host_t0 = std::chrono::steady_clock::now();
  cudaStream_t stream = ss->stream;
  r->last_stream = stream;
  // the last K/2 pushed frames are never integrated (main.cc:987-992)
  c.last = std::max(c.first, c.first - c.half + static_cast<int>(ss->pushed) - c.half);
  int status = SM_OK;
  FrameLoop& loop = ss->loop;
  if (c.last > c.first && ss->next_step < c.last) {
    // frame graph: the steps whose pre-processing part has no frame left (placeholder launches), as in RunLoop
    if (cudaEventRecord(ss->entry, stream) != cudaSuccess || cudaStreamWaitEvent(loop.work, ss->entry, 0) != cudaSuccess) {
      status = SetError(SM_ERR_CUDA, "sm_session_end: stream ordering failed");
    }
    for (int it = ss->next_step; it < c.last && status == SM_OK; ++it) status = Step(c, loop, it, &ss->integrated);
    if (status == SM_OK) status = JoinLoop(r, loop, stream);
    ss->last_integrated = c.last - 1;
  }
  if (status != SM_OK) return AbortSession(r, status);
  r->reported_merge_count = nullptr;   // the last step's front half has no frame: merge_count is exact again
  ss->host_ms += MillisecondsSince(host_t0);
  status = FetchCounters(r, stream);
  FillStats(r, ss->integrated, ss->launches_before, c.h2d, ss->host_ms, stats);
  cudaStreamSynchronize(r->run->upload_stream);   // the staging buffers are no longer read
  FreeSession(ss);
  r->session = nullptr;
  return status;
}

int SessionRefront(sm_reconstruction* r, cudaStream_t stream) {
  StreamSession* ss = r->session;
  if (!ss || !ss->loop.graph || ss->next_step <= ss->loop.it0) return SM_OK;   // serial mode: nothing in flight
  SM_CUDA(cudaMemsetAsync(ss->merge_count, 0, sizeof(u32), stream));   // merges up to the newest integrated frame
  RunContext& c = ss->c;
  const int frame = ss->next_step;   // the last push ran this frame's front half (GraphStep: front = it + 1)
  if (!c.Active(frame)) return SM_OK;
  const int set = frame % kSets;
  DeviceState d = r->d;
  UseSet(d, r->sets[set]);
  int status = ClearAssociationRasters(stream, d);
  if (status != SM_OK) return status;
  // k_blend reads the pre-blend copy and rewrites the frame's depth from it, so it can run again
  const FrameParams f = c.Params(frame, set);
  const FrameKernel kernels[4] = {FK_PROJECT, FK_ASSOCIATE, FK_MERGE, FK_BLEND};
  for (int i = 0; i < (ss->loop.blending ? 4 : 3); ++i) {
    KernelLaunch k;
    status = DescribeFrameKernel(kernels[i], r->plan, d, f, &k);
    if (status != SM_OK) return status;
    LaunchOnStream(stream, k, false);
  }
  return CheckLaunch("sm_compact: front half of the frame in flight");
}

void FreeRunBuffers(sm_reconstruction* r) {
  RunBuffers* b = r->run;
  if (!b) return;
  DestroyFrameGraph(b->graph);
  for (int i = 0; i < kSets; ++i) { cudaFree(b->depth[i]); cudaFree(b->depth_pre[i]); cudaFree(b->normals[i]); cudaFree(b->radius[i]); }
  for (u16* p : b->ring_depth) cudaFree(p);
  for (uchar3* p : b->ring_color) cudaFree(p);
  cudaFree(b->median_stage[0]); cudaFree(b->median_stage[1]);
  cudaFree(b->pyramid_depth_stage); cudaFree(b->pyramid_color_stage);
  for (cudaStream_t st : {b->upload_stream, b->graph_stream})
    if (st) cudaStreamDestroy(st);
  for (cudaEvent_t e : {b->entry_event, b->upload_done, b->graph_exit})
    if (e) cudaEventDestroy(e);
  for (cudaEvent_t e : b->iteration_done) if (e) cudaEventDestroy(e);
  delete b;
  r->run = nullptr;
}

}  // namespace smb

extern "C" {

int sm_session_end(sm_reconstruction* r, sm_stream_stats* stats) {
  if (!r) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_session_end: null argument");
  return SessionEnd(r, stats);
}

int sm_outlier_filter_transforms(int32_t other_count, float depth_scaling, int32_t frame_count,
                                 const float* global_T_frame, const float* frame_T_global, int32_t frame, float* out) {
  if (!global_T_frame || !frame_T_global || !out) return SetError(SM_ERR_INVALID_ARGUMENT, "sm_outlier_filter_transforms: null argument");
  if (other_count < 2 || other_count > 8 || other_count % 2 != 0)
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_outlier_filter_transforms: other_count must be 2, 4, 6 or 8");
  const int half = other_count / 2;
  if (frame < half || frame >= frame_count - half)
    return SetError(SM_ERR_INVALID_ARGUMENT, "sm_outlier_filter_transforms: the frame needs other_count/2 frames on both sides (main.cc:987-992)");
  const float* ref = global_T_frame + 12 * static_cast<size_t>(frame);
  for (int i = 0; i < half; ++i) {
    OutlierFilterTransform(depth_scaling, ref, frame_T_global + 12 * static_cast<size_t>(frame - (i + 1)), out + 12 * i);
    OutlierFilterTransform(depth_scaling, ref, frame_T_global + 12 * static_cast<size_t>(frame + (i + 1)), out + 12 * (half + i));
  }
  return SM_OK;
}

}  // extern "C"
