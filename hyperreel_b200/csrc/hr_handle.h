// Private definition of the opaque handle (shared by hr_api.cu and the weight packers).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <vector>

#include "hr_common.cuh"
#include "hr_mlp.cuh"

struct EventPair {
  cudaEvent_t a, b;
};

struct HostPipe {
  int64_t chunk = 0;
  cudaStream_t streams[3] = {nullptr, nullptr, nullptr};
  float* d_rays[3] = {nullptr, nullptr, nullptr};
  float* d_rgb[3] = {nullptr, nullptr, nullptr};
  void* d_ws[3] = {nullptr, nullptr, nullptr};
  int64_t ws_bytes = 0;
  // hr_render_host replays its whole copy/kernel pipeline as one CUDA graph while the call signature repeats
  cudaGraphExec_t graph = nullptr;
  const void* g_rays = nullptr;
  void* g_rgb = nullptr;
  int64_t g_n = 0, g_chunk = 0, g_launches = 0;
  cudaEvent_t fork_ev = nullptr, join_ev[3] = {nullptr, nullptr, nullptr};
};

// One sample net as hr_upload packs it: its configuration (a copy of the handle's with the net's own shape) and both packs.
struct SampleNet {
  hr_config cfg;
  hr::MlpSimtPack simt{};
  hr::MlpTcPack tc{};
  bool tc_ready = false;
  size_t tc_alloc_bytes = 0;  // current allocation behind tc.wpack / tc.bias (reused while the layout is unchanged)
  int tc_alloc_bias = 0;
};

// hr::GradTabs' buffers as a flat list (hr_api.cu: grad_bufs): their number, and the two read by name
constexpr int kGradTables = 14, kGradBasis = 12, kGradColorEmbedding = 13;

// every size of a workspace segment is rounded up to 256 bytes, so that every segment starts 256-byte aligned
static inline int64_t align256(int64_t bytes) { return (bytes + 255) / 256 * 256; }

struct hr_handle {
  hr_config cfg;
  hr::Derived dv;
  int device = 0;
  int num_sms = 148;
  bool uploaded = false;
  struct Slot { void* ptr; size_t bytes; };
  std::vector<Slot> slots;   // device allocations of packed parameters, in hr_upload's request order
  size_t slot_cursor = 0;
  hr::RenderTabs tabs{};
  // the net behind the final heads (net.cfg == cfg, or the point net of a cascaded pipeline evaluated on 8-float point rows)
  SampleNet net;
  // cascaded pipelines only: the first-stage ray net (cfg.pre_*), same kernels
  SampleNet pre;
  // gradient tables of the backward pass (hr_render_backward), packed like the forward tables; allocated on first use
  hr::GradTabs grads{};
  size_t g_sizes[kGradTables] = {0};  // element counts of grad_bufs' buffers (to notice a resized grid)
  int64_t launches = 0;
  bool timing = false;
  size_t timed_calls = 0;      // hr_render calls covered by ev_render / ev_mlp (a call may run several sub-batches)
  int64_t sub_rays = 0;        // rays per sub-batch of hr_render: 0 = 16 tile waves (default), < 0 = never split
  std::vector<EventPair> ev_render, ev_mlp, ev_bwd;
  HostPipe pipe;
};


// error plumbing shared with the packers (sets hr_last_error, returns 1)
int hr_fail(const char* fmt, ...);
