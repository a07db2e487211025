// gslam_b200/csrc/common.cuh — context, error plumbing and small device helpers shared by the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <initializer_list>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/gslam_b200.h"

struct OrbState;  // orb.cu
struct BaCache;   // ba.cu

// A grow-only buffer that one outermost API call on a ctx bump-allocates and CtxLock resets: the pinned staging, the device scratch.
struct GbBump {
  uint8_t* base = nullptr;
  size_t bytes = 0, off = 0;
};

struct gb_ctx {
  int device = 0;
  int sm_count = 132;
  int max_smem_optin = 0;
  cudaStream_t stream = nullptr;
  bool owns_stream = true;                    // false: `stream` belongs to another ctx (gb_ctx_create_on_stream)
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // gb_timer_*
  cudaEvent_t evs = nullptr, eve = nullptr;   // internal (gb_ba_result.gpu_ms, gb_dbg_popc_peak)
  cudaEvent_t ev_x = nullptr;                 // gb_ctx_wait_for (cross-ctx ordering)
  std::recursive_mutex mu;
  std::string err;
  int64_t launches = 0;
  GbBump stage;    // pinned host staging (gb_stage_take)
  GbBump scratch;  // device scratch (gb_scratch_take)
  int lock_depth = 0;
  // device state owned by subsystems
  OrbState* orb = nullptr;
  int match_last_plan[4] = {0, 0, 0, 0};  // qtiles, nsplit, chunk, stereo of the last match launch (gb_dbg_match_last_plan); 0s: none
  BaCache* ba_cache = nullptr;  // gb_ba_solve's topology cache: the graph it keeps between calls, in a buffer of its own
  int ba_last_paths = 0;        // gb_dbg_ba_paths bits of the graph the last gb_ba_solve / gb_ba_pnp solved (gb_dbg_ba_last_paths)
};

struct gb_features {
  int capacity = 0;
  void* d_slab = nullptr;        // the one device allocation holding every array below
  gb_keypoint* d_kps = nullptr;  // [capacity]
  uint8_t* d_desc = nullptr;     // [capacity*32], 32-byte rows
  int* d_count = nullptr;        // device-side keypoint count (written by extract)
  int* d_status = nullptr;       // device-side status word (0 ok, else required capacity)
  int* d_train_status = nullptr; // status word of the train set of the last match with this set as query (written by the match)
  // Split-merge tickets of the matches with this set as query, one per 128-row query tile, right after the four count words.
  // Zero between launches: zeroed with the count words when the set is made, and the merging CTA of a tile re-arms its ticket.
  // (Two contexts matching the same query set at once race on the tickets as they already do on d_best / d_dist / d_dist2.)
  unsigned int* d_tickets = nullptr;
  int h_count = -1;              // host copy (valid when >=0)
  int expect = 0;                // expected row count while h_count is unknown (nfeatures of the extraction in flight): tunes launches
  int32_t* d_best = nullptr;     // match outputs [capacity]
  int32_t* d_dist = nullptr;
  int32_t* d_dist2 = nullptr;
  int n_matched = 0;             // number of queries of the last match
};

void gb_set_error(gb_ctx* ctx, const char* fmt, ...);
// The {count, status} pair an extraction left in f->d_count, read back to the host as hc: on success sets f->h_count and *n to the
// count; else returns GB_ERR_CAPACITY with the reason in the error text and *n = the capacity the extraction needed (0: an
// internal overflow).
int gb_features_resolve(gb_ctx* ctx, gb_features* f, const int* hc, int* n);
// A ctx on `device` that enqueues on `stream`, which another ctx owns and must outlive it (gb_ctx_destroy leaves it alone).
int gb_ctx_create_on_stream(int device, cudaStream_t stream, gb_ctx** out);
// One buffer of a take from the ctx's pinned staging or device scratch: *p receives its address (nullptr when bytes == 0).
struct GbBuf {
  void** p;
  size_t bytes;
  template <typename T>
  GbBuf(T** p_, size_t bytes_) : p((void**)p_), bytes(bytes_) {}
};
// Takes `bufs` from the ctx's pinned staging, each 256-byte aligned, after what the outermost API call on the ctx has taken so far.
// When they do not fit, the staging is grown first: the stream is synchronised and the old buffer freed, so every pointer an earlier
// take of the same outermost call returned is dead.  Buffers that must be live at the same time are therefore taken in ONE call; a
// nested call may take again only once its caller is done with its own earlier buffers.  GB_ERR_CUDA when the staging cannot grow.
int gb_stage_take(gb_ctx* ctx, std::initializer_list<GbBuf> bufs);
// The same for the ctx's grow-only device scratch: the per-call working memory of the host-buffer entry points (their temporary feature
// sets and one-shot BA graphs among it), the matcher's split partials, the staged frames and the test hooks, so that the long-lived
// objects they read (maps, vocabularies) stay immutable after creation.  Two rules:
//  * Take together.  Buffers that must be live at the same time are taken in one call: growing the scratch synchronises the stream
//    and frees the old buffer, which kills every earlier take of the outermost call (bow_run takes the uploaded descriptors of
//    gb_bow_transform with its word, key and output buffers; gb_match_hamming its two feature sets with the partials).
//  * No scratch access before gb_pdl_wait().  The next call on the ctx reuses the same bytes, ordered behind this call's kernels only
//    by the stream, so a kernel launched with programmatic dependent launch must not read or write scratch before that wait
//    (remap_level0_kernel reads only the map's table before it, match_kernel touches nothing before it; every other kernel given
//    scratch is a plain launch).  And since the wait covers only the kernel's predecessor, every PDL kernel waits on every path.
//    One exception: the local-BA chain (ba_linearize_kernel .. ba_backsub_commit_kernel) reads the structure and measurements of a
//    graph before its wait, and gb_ba_pnp, gb_ba_solve_posegraph and an uncached gb_ba_solve place their graph here.  Those bytes are
//    written by the graph's H2D upload in the same call, ahead of a plain launch (ba_rt_kernel in gb_ba_graph_begin) that precedes the
//    chain, so no chain kernel overlaps their previous user; and each of those calls synchronises its stream before it returns, so
//    no later call overlaps the chain.
int gb_scratch_take(gb_ctx* ctx, std::initializer_list<GbBuf> bufs);
// Enqueues the copy of `rows` rows of `row_bytes` from src (pitch spitch) to device memory d_dst (pitch dpitch) on the ctx stream:
// device to device, pinned host memory directly, pageable host memory row by row through the pinned staging (one take).
int gb_upload_2d(gb_ctx* ctx, void* d_dst, size_t dpitch, const void* src, int src_is_device, size_t spitch, size_t row_bytes, int rows);
// A dense device copy of a frame (`height` rows of `row_bytes`): the frame itself when it is a device pointer with pitch == row_bytes,
// else a copy in the ctx's device scratch (one take, then gb_upload_2d).
int gb_stage_frame(gb_ctx* ctx, const uint8_t* img, int img_is_device, size_t row_bytes, int height, int pitch, const uint8_t** d_frame);

// ---- undistortion in front of the ORB extraction: what orb.cu needs of remap.cu ------------------------------------------------------
void gb_remap_geometry(const gb_remap* m, int* device, int* w_in, int* h_in, int* w_out, int* h_out);
// Enqueue the remap of the dense device frame d_src (w_in x h_in, 1 or 3 channels) as a GRAY w_out x h_out image at d_dst; d_dst and
// dst_pitch must be multiples of 4 and dst_pitch >= w_out rounded up to 4 (every word of a row is stored whole).  Reads the map only.
int gb_remap_enqueue_level0(gb_ctx* ctx, const gb_remap* m, const uint8_t* d_src, int channels, int rgb_order, uint8_t* d_dst, int dst_pitch);

// Function attributes are per-function, per-DEVICE state shared by every ctx on the device: gb_func_setup sets kernel `fn`'s
// dynamic shared-memory limit to `smem` bytes (GB_SMEM_OPTIN_MAX: the device's opt-in maximum less the kernel's static shared
// memory) and, when `nonportable_cluster` is given, permits cluster sizes above 8, reporting there whether that worked.  Each
// setting is made once per (device, function), under a lock, and a limit is never lowered: a value planned for one ctx's launch
// cannot shrink under another's.  Returns whether the limit is set.
constexpr int GB_SMEM_OPTIN_MAX = -1;
bool gb_func_setup(gb_ctx* ctx, const void* fn, int smem, bool* nonportable_cluster = nullptr);

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

// Layout of one device allocation, written as ONE list of declarations that is run twice: first to measure (base == nullptr),
// then to place the arrays at base.  put() declares an uploaded array and copies its host source, if it has one, into the pinned
// staging h at the array's offset; the puts come first, so [0, blob) is one contiguous upload.  take() declares device-only
// working memory after them.  Every array starts on a 256-byte boundary (kernels such as cta_copy_f64 rely on it).
struct Slab {
  uint8_t* base = nullptr;
  uint8_t* h = nullptr;  // host staging mirror of [0, blob)
  size_t off = 0, blob = 0;
  template <typename T>
  void take(T** p, size_t n) {
    off = (off + 255) & ~(size_t)255;
    if (base) *p = (T*)(base + off);
    off += std::max<size_t>(n, 1) * sizeof(T);
  }
  template <typename T>
  void put(T** p, size_t n, const std::remove_const_t<T>* src = nullptr) {
    take(p, n);
    blob = off;
    if (h && src && n) memcpy(h + ((const uint8_t*)*p - base), src, n * sizeof(T));
  }
  template <typename T>
  std::remove_const_t<T>* host(T* p) const { return (std::remove_const_t<T>*)(h + ((const uint8_t*)p - base)); }  // staging of a put array
};

// Places `layout` (a callable that declares its arrays on the Slab it is given) in ONE new device allocation: runs it to measure,
// allocates, runs it again to place the arrays there.  *base receives the allocation (cudaFree releases every array at once); the
// uploads of its puts are the caller's.
// Device memory is allocated in three places only: here (the one slab of a long-lived object: feature set, ORB state, remap table,
// vocabulary, BA graph), bump_grow (the ctx scratch, ctx.cu) and ba_cache_slab (the BA topology cache's buffer, ba.cu).
template <typename F>
int gb_slab_alloc(gb_ctx* ctx, void** base, F&& layout) {
  Slab sl;
  layout(sl);
  *base = nullptr;
  GB_CUDA(ctx, cudaMalloc(base, sl.off));
  sl = Slab{(uint8_t*)*base};
  layout(sl);
  return GB_OK;
}

// The same in ONE take of the ctx's device scratch (gb_scratch_take, and its rules): for the working memory of one call.
template <typename F>
int gb_scratch_slab(gb_ctx* ctx, F&& layout) {
  Slab sl;
  layout(sl);
  uint8_t* base;
  GB_CHECK(gb_scratch_take(ctx, {{&base, sl.off}}));
  sl = Slab{base};
  layout(sl);
  return GB_OK;
}

constexpr int kQPerCta = 128;  // match.cu: threads per CTA == query rows per CTA, one split-merge ticket per such query tile
// The arrays of a feature set of f->capacity rows: gb_features_create's allocation, and the temporaries of the host-buffer entry
// points in the scratch.  gb_features_words(capacity) words from d_count on are the four count words and the tickets.
void gb_features_layout(Slab& sl, gb_features* f);
static inline int gb_features_words(int capacity) { return 4 + (capacity + kQPerCta - 1) / kQPerCta; }

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

// Launch configuration of ONE thread-block cluster of `cluster` CTAs along x: for cudaLaunchKernelEx and
// cudaOccupancyMaxActiveClusters.  (cfg points into the object: not copyable.)
struct GbClusterConfig {
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute at[1];
  GbClusterConfig(int cluster, dim3 block, size_t smem, cudaStream_t stream) {
    cfg.gridDim = dim3(cluster); cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
  }
  GbClusterConfig(const GbClusterConfig&) = delete;
  GbClusterConfig& operator=(const GbClusterConfig&) = delete;
};

struct CtxLock {
  gb_ctx* c;
  explicit CtxLock(gb_ctx* ctx) : c(ctx) {
    c->mu.lock();
    if (c->lock_depth++ == 0) {
      cudaSetDevice(c->device);
      c->stage.off = c->scratch.off = 0;
    }
  }
  ~CtxLock() {
    c->lock_depth--;
    c->mu.unlock();
  }
};

// Releases a ctx that the calling thread holds exactly once (one CtxLock) for the scope of a host wait on the device, so that other
// threads can enqueue on it meanwhile (gb_ctx_wait_for from a tracking thread while the mapping thread waits for its solve).
// Nothing of the ctx's pinned staging or device scratch may be waited on or read across it: another thread's CtxLock restarts the bump
// allocation and a take may free and reallocate the buffer, so a pointer taken before the unlock is invalid after it.
struct CtxUnlock {
  gb_ctx* c;
  explicit CtxUnlock(gb_ctx* ctx) : c(ctx) {
    c->lock_depth--;
    c->mu.unlock();
  }
  ~CtxUnlock() {
    c->mu.lock();
    if (c->lock_depth++ == 0) cudaSetDevice(c->device);
  }
  CtxUnlock(const CtxUnlock&) = delete;
  CtxUnlock& operator=(const CtxUnlock&) = delete;
};

static inline int gb_div_up(int a, int b) { return (a + b - 1) / b; }
