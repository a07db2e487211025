// gslam_b200/csrc/common.cuh — context, error plumbing and small device helpers shared by the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/gslam_b200.h"

struct OrbState;    // orb.cu
struct MatchState;  // match.cu

struct gb_ctx {
  int device = 0;
  int sm_count = 132;
  int max_smem_optin = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // gb_timer_*
  cudaEvent_t evs = nullptr, eve = nullptr;   // internal (gb_ba_result.gpu_ms)
  cudaEvent_t ev_x = nullptr;                 // gb_ctx_wait_for (cross-ctx ordering)
  std::recursive_mutex mu;
  std::string err;
  int64_t launches = 0;
  // pinned host staging (bump-allocated inside one API call, reset at its end)
  uint8_t* h_stage = nullptr;
  size_t h_stage_bytes = 0, h_stage_off = 0;
  int lock_depth = 0;
  // generic device scratch owned by subsystems
  OrbState* orb = nullptr;
  MatchState* match = nullptr;
  gb_features* tmp_q = nullptr;  // temporaries of the host-buffer match entry point
  gb_features* tmp_t = nullptr;
  gb_features* tmp_f = nullptr;  // temporary of the host-buffer extract entry point
  void* ba_arena = nullptr;      // grow-only slab reused by the host-buffer BA entry points (no cudaMalloc per call)
  size_t ba_arena_cap = 0;
  bool ba_arena_busy = false;
  gb_ba_graph* ba_cached = nullptr;  // the graph of the last gb_ba_solve, kept (with the arena) while the TOPOLOGY of the calls stays
  void* ba_cache_key = nullptr;      // the same: a sliding window re-solved with new estimates skips sorting / structure / plans
  void* pnp_scratch = nullptr;   // grow-only device scratch of gb_pnp_ransac (points, measurements, per-hypothesis results)
  size_t pnp_scratch_cap = 0;
};

struct gb_features {
  int capacity = 0;
  gb_keypoint* d_kps = nullptr;  // [capacity]
  uint8_t* d_desc = nullptr;     // [capacity*32], 32-byte rows
  int* d_count = nullptr;        // device-side keypoint count (written by extract)
  int* d_status = nullptr;       // device-side status word (0 ok, else required capacity)
  int h_count = -1;              // host copy (valid when >=0)
  int expect = 0;                // expected row count while h_count is unknown (nfeatures of the extraction in flight): tunes launches
  int32_t* d_best = nullptr;     // match outputs [capacity]
  int32_t* d_dist = nullptr;
  int32_t* d_dist2 = nullptr;
  int n_matched = 0;             // number of queries of the last match
};

void gb_set_error(gb_ctx* ctx, const char* fmt, ...);
int gb_stage_reserve(gb_ctx* ctx, size_t bytes);           // make sure the pinned staging holds >= bytes
void* gb_stage_alloc(gb_ctx* ctx, size_t bytes);           // bump-allocate from pinned staging (256-B aligned), or nullptr
int gb_dev_realloc(gb_ctx* ctx, void** p, size_t* cap, size_t bytes);  // grow-only device buffer

#define GB_CUDA(ctx, call)                                                                              \
  do {                                                                                                  \
    cudaError_t e_ = (call);                                                                            \
    if (e_ != cudaSuccess) {                                                                            \
      gb_set_error((ctx), "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_));         \
      return GB_ERR_CUDA;                                                                               \
    }                                                                                                   \
  } while (0)

#define GB_CHECK(expr)          \
  do {                          \
    int rc_ = (expr);           \
    if (rc_ != GB_OK) return rc_; \
  } while (0)

#define GB_LAUNCH_CHECK(ctx)                                                                            \
  do {                                                                                                  \
    (ctx)->launches++;                                                                                  \
    cudaError_t e_ = cudaGetLastError();                                                                \
    if (e_ != cudaSuccess) {                                                                            \
      gb_set_error((ctx), "%s:%d kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(e_));     \
      return GB_ERR_CUDA;                                                                               \
    }                                                                                                   \
  } while (0)

// ---- programmatic dependent launch (sm_90+): a kernel launched with gb_launch_pdl may be scheduled while its predecessor on
// the stream is still running; it must call gb_pdl_wait() before touching anything the predecessor wrote.  Calling
// gb_pdl_launch_dependents() first lets ITS successor start getting scheduled in turn.  Both are no-ops in a plain launch.
// What is hidden: the ~2-3 us launch + CTA-scheduling latency between short dependent kernels (40 launches per local-BA solve).
#ifdef __CUDACC__
__device__ __forceinline__ void gb_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void gb_pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KArgs, typename... Args>
static inline cudaError_t gb_launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
#endif

struct CtxLock {
  gb_ctx* c;
  explicit CtxLock(gb_ctx* ctx) : c(ctx) {
    c->mu.lock();
    if (c->lock_depth++ == 0) {
      cudaSetDevice(c->device);
      c->h_stage_off = 0;
    }
  }
  ~CtxLock() {
    c->lock_depth--;
    c->mu.unlock();
  }
};

static inline int gb_div_up(int a, int b) { return (a + b - 1) / b; }
