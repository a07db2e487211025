// gslam_b200/csrc/ba_dist.cu — landmark-sharded multi-GPU global bundle adjustment UNDER the C-ABI
// (behind GSLAM::Optimizer::optimize(BundleGraph&), GSLAM/core/Optimizer.h:229, at BASELINE config 5: 500 cameras / 100k
// landmarks / 1M observations; SURVEY.md section 8e).
//
// Every rank holds ALL cameras and a contiguous shard of the landmarks with all their edges (ba.cu: ba_graph_create_impl with
// shard_world > 1; the covisibility block structure of the reduced camera matrix is derived from the WHOLE graph, so every rank's
// compact reduced system [Sb | g~ | diag U | cost] has the same layout).  One LM iteration:
//     sweep + Schur blocks of the shard            (O(observations / N), ba.cu)
//     all-reduce of the compact reduced system     (the path's one real exchange: f64 sum over NVLink; 14 MB at config 5
//                                                   instead of the 72 MB dense S of round 1)
//     block-CSR PCG, replicated                    (ba_pcg_bcsr.cu: persistent kernel, S resident in shared memory;
//                                                   bit-identical on every rank -> identical LM decisions, no broadcast)
//     back-substitution + candidate cost of the shard, all-reduce of ONE double, accept / reject
// The collective is NCCL, bound at run time with dlopen (the library loads and the single-GPU paths work without NCCL); two
// front ends share the engine: one process per GPU (gb_comm_create from a unique id the host distributes -- bench.py under
// torchrun) and one process driving N GPUs (gb_comm_create_all + gb_ba_solve_multi, one host thread per device -- what the
// libgslam_optimizer.so plugin uses when the svar option b200.devices lists several devices).  A loopback transport (test hook
// gb_dbg_comm_create_local) runs the same engine with several ranks on one device.
#include "ba_internal.cuh"

#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <thread>

namespace {

// ---- NCCL, bound at run time (minimal declarations; values are stable across NCCL 2.x) -----------------------------------------
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
constexpr int kNcclFloat64 = 8, kNcclSum = 0;

struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  ncclResult_t (*GetVersion)(int*) = nullptr;
  std::string err;
  bool ok = false;
};

NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);  // (a process that imported torch already holds torch's libnccl.so.2)
      if (api.handle) break;
    }
    if (!api.handle) { api.err = std::string("libnccl.so.2 not found: ") + dlerror(); return; }
    auto sym = [&](const char* s) { void* p = dlsym(api.handle, s); if (!p) api.err = std::string("NCCL symbol missing: ") + s; return p; };
    api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
    api.CommInitAll = (decltype(api.CommInitAll))sym("ncclCommInitAll");
    api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
    api.AllReduce = (decltype(api.AllReduce))sym("ncclAllReduce");
    api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
    api.GetVersion = (decltype(api.GetVersion))sym("ncclGetVersion");
    api.ok = api.err.empty();
  });
  return api;
}

// ---- loopback transport (test hook gb_dbg_comm_create_local): `world` ranks on ONE device whose contexts share one stream ------
// A host rendezvous per collective; the last rank to arrive enqueues one kernel that sums the buffers in rank order and writes the
// sum into every buffer, then releases the others.  So every rank gets the same bits (as with NCCL), no events are needed, and
// the ranks' kernels never run concurrently (one rank's cooperative-grid PCG never competes with another's for residency).
constexpr int kLoopbackMaxWorld = 16;
constexpr auto kLoopbackTimeout = std::chrono::seconds(120);

struct LoopbackBufs {
  double* p[kLoopbackMaxWorld];
};

__global__ void loopback_sum_kernel(LoopbackBufs b, int world, size_t n) {
  for (size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) {
    double s = b.p[0][k];
    for (int r = 1; r < world; ++r) s += b.p[r][k];
    for (int r = 0; r < world; ++r) b.p[r][k] = s;
  }
}

struct LoopbackGroup {
  int world = 0, live = 0;  // live: communicators of the group not destroyed yet
  cudaStream_t stream = nullptr;
  int sm_count = 0;
  std::mutex mu;
  std::condition_variable cv;
  unsigned long long gen = 0;  // collectives completed
  int arrived = 0;
  size_t n = 0;
  bool n_mismatch = false;
  LoopbackBufs bufs{};
  bool here[kLoopbackMaxWorld] = {};
  int rc = GB_OK;  // outcome of the last completed collective, and its message
  std::string err;
};

}  // namespace

struct gb_comm {
  gb_ctx* ctx = nullptr;
  ncclComm_t comm = nullptr;  // null when world == 1
  LoopbackGroup* loop = nullptr;  // the loopback transport instead of NCCL
  int rank = 0, world = 1;
};

static int loopback_allreduce(gb_comm* c, double* d_buf, size_t n) {
  LoopbackGroup& G = *c->loop;
  std::unique_lock<std::mutex> lk(G.mu);
  const unsigned long long gen = G.gen;
  if (G.arrived == 0) { G.n = n; G.n_mismatch = false; }
  else if (n != G.n) G.n_mismatch = true;
  G.bufs.p[c->rank] = d_buf;
  G.here[c->rank] = true;
  if (++G.arrived == G.world) {
    G.rc = GB_OK;
    G.err.clear();
    if (G.n_mismatch) {
      G.rc = GB_ERR_INVALID;
      G.err = "gb_comm (loopback): the ranks passed different lengths to one all-reduce";
    } else if (G.n > 0) {
      const int blocks = (int)std::min<size_t>((G.n + 255) / 256, (size_t)G.sm_count * 8);
      loopback_sum_kernel<<<blocks, 256, 0, G.stream>>>(G.bufs, G.world, G.n);
      c->ctx->launches++;
      const cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) { G.rc = GB_ERR_CUDA; G.err = std::string("gb_comm (loopback): sum kernel -> ") + cudaGetErrorString(e); }
    }
    G.arrived = 0;
    for (int r = 0; r < G.world; ++r) G.here[r] = false;
    ++G.gen;
    G.cv.notify_all();
  } else if (!G.cv.wait_for(lk, kLoopbackTimeout, [&] { return G.gen != gen; })) {
    std::string missing;
    for (int r = 0; r < G.world; ++r)
      if (!G.here[r]) missing += (missing.empty() ? "" : ", ") + std::to_string(r);
    G.here[c->rank] = false;  // (withdraw: a late rank must not complete a collective this rank left)
    --G.arrived;
    gb_set_error(c->ctx, "gb_comm (loopback): rank %d waited %d s at an all-reduce of %zu doubles; rank(s) %s never arrived", c->rank,
                 (int)kLoopbackTimeout.count(), n, missing.c_str());
    return GB_ERR_CUDA;
  }
  if (G.rc != GB_OK) gb_set_error(c->ctx, "%s", G.err.c_str());
  return G.rc;
}

#define GB_NCCL(ctx, call)                                                                              \
  do {                                                                                                  \
    ncclResult_t r_ = (call);                                                                           \
    if (r_ != 0) {                                                                                      \
      gb_set_error((ctx), "%s:%d %s -> %s", __FILE__, __LINE__, #call, nccl().GetErrorString(r_));      \
      return GB_ERR_CUDA;                                                                               \
    }                                                                                                   \
  } while (0)

extern "C" {

int gb_comm_unique_id(uint8_t* id128) {
  if (!id128) return GB_ERR_INVALID;
  NcclApi& n = nccl();
  if (!n.ok) { gb_set_error(nullptr, "gb_comm: %s", n.err.c_str()); return GB_ERR_NODEVICE; }
  ncclUniqueId id;
  static_assert(sizeof id == GB_COMM_ID_BYTES, "unique id size");
  GB_NCCL(nullptr, n.GetUniqueId(&id));
  memcpy(id128, &id, sizeof id);
  return GB_OK;
}

int gb_comm_create(gb_ctx* ctx, int world, int rank, const uint8_t* id128, gb_comm** out) {
  if (!ctx || !out || world < 1 || rank < 0 || rank >= world) return GB_ERR_INVALID;
  *out = nullptr;
  CtxLock lk(ctx);
  gb_comm* c = new gb_comm();
  c->ctx = ctx; c->rank = rank; c->world = world;
  if (world > 1) {
    NcclApi& n = nccl();
    if (!n.ok || !id128) { gb_set_error(ctx, "gb_comm: %s", n.ok ? "null unique id" : n.err.c_str()); delete c; return n.ok ? GB_ERR_INVALID : GB_ERR_NODEVICE; }
    ncclUniqueId id;
    memcpy(&id, id128, sizeof id);
    ncclResult_t r = n.CommInitRank(&c->comm, world, id, rank);
    if (r != 0) { gb_set_error(ctx, "ncclCommInitRank -> %s", n.GetErrorString(r)); delete c; return GB_ERR_CUDA; }
  }
  *out = c;
  return GB_OK;
}

int gb_comm_create_all(int n_dev, gb_ctx* const* ctxs, gb_comm** out) {
  if (n_dev < 1 || !ctxs || !out) return GB_ERR_INVALID;
  for (int i = 0; i < n_dev; ++i) { out[i] = nullptr; if (!ctxs[i]) return GB_ERR_INVALID; }
  std::vector<ncclComm_t> comms(n_dev, nullptr);
  if (n_dev > 1) {
    NcclApi& n = nccl();
    if (!n.ok) { gb_set_error(ctxs[0], "gb_comm: %s", n.err.c_str()); return GB_ERR_NODEVICE; }
    std::vector<int> devs(n_dev);
    for (int i = 0; i < n_dev; ++i) devs[i] = ctxs[i]->device;
    GB_NCCL(ctxs[0], n.CommInitAll(comms.data(), n_dev, devs.data()));
  }
  for (int i = 0; i < n_dev; ++i) {
    out[i] = new gb_comm();
    out[i]->ctx = ctxs[i]; out[i]->rank = i; out[i]->world = n_dev; out[i]->comm = comms[i];
  }
  return GB_OK;
}

int gb_comm_destroy(gb_comm* c) {
  if (!c) return GB_OK;
  if (c->loop) {
    bool last;
    {
      std::lock_guard<std::mutex> lk(c->loop->mu);
      last = --c->loop->live == 0;
    }
    if (last) delete c->loop;
  }
  if (c->comm) {
    CtxLock lk(c->ctx);
    cudaStreamSynchronize(c->ctx->stream);
    nccl().CommDestroy(c->comm);
  }
  delete c;
  return GB_OK;
}

int gb_comm_rank(const gb_comm* c) { return c ? c->rank : -1; }
int gb_comm_world(const gb_comm* c) { return c ? c->world : -1; }

int gb_comm_allreduce_sum_f64(gb_comm* c, double* d_buf, size_t n) {
  if (!c || !d_buf) return GB_ERR_INVALID;
  if (c->world == 1) return GB_OK;
  if (c->loop) {  // (n == 0 too: a collective every rank must reach)
    CtxLock lk(c->ctx);
    return loopback_allreduce(c, d_buf, n);
  }
  if (n == 0) return GB_OK;
  CtxLock lk(c->ctx);
  GB_NCCL(c->ctx, nccl().AllReduce(d_buf, d_buf, n, kNcclFloat64, kNcclSum, c->comm, c->ctx->stream));
  return GB_OK;
}

// ---- the sharded solve -----------------------------------------------------------------------------------------------------
int gb_ba_shard_create(gb_comm* c, const gb_ba_problem* full, gb_ba_graph** out) {
  if (!c || !full || !out) return GB_ERR_INVALID;
  return ba_graph_create_impl(c->ctx, full, out, false, c->rank, c->world);
}

int gb_ba_shard_range(const gb_ba_graph* g, int* lo, int* hi) {
  if (!g) return GB_ERR_INVALID;
  if (lo) *lo = g->shard_lo;
  if (hi) *hi = g->shard_hi;
  return GB_OK;
}

int gb_ba_shard_reduce_bytes(const gb_ba_graph* g, size_t* bytes) {
  if (!g || !bytes) return GB_ERR_INVALID;
  *bytes = g->rbuf_doubles * sizeof(double);
  return GB_OK;
}

int gb_ba_shard_solve(gb_comm* c, gb_ba_graph* g, const gb_ba_options* opt, gb_ba_result* res) {
  if (!c || !g) return GB_ERR_INVALID;
  gb_ctx* ctx = c->ctx;
  CtxLock lk(ctx);
  if (!g->pcg_bcsr || !g->rbuf) { gb_set_error(ctx, "gb_ba_shard_solve: the graph has no block-CSR reduced system"); return GB_ERR_INVALID; }
  if (g->shard_world != c->world || g->shard_rank != c->rank) { gb_set_error(ctx, "gb_ba_shard_solve: graph / communicator mismatch"); return GB_ERR_INVALID; }
  GB_CHECK(gb_ba_graph_begin(ctx, g, opt));
  GB_CUDA(ctx, cudaEventRecord(ctx->evs, ctx->stream));
  const bool poll = g->opt.function_tolerance > 0.0 || g->opt.verbose;
  for (int it = 0; it < g->opt.max_iterations; ++it) {
    GB_CHECK(ba_compact_iteration(ctx, g, c));
    if (poll) {  // every rank reads the same (reduced) scalars, so every rank stops at the same iteration
      BaScalars h;
      GB_CUDA(ctx, cudaMemcpyAsync(&h, g->d.sc, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
      GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
      if (g->opt.verbose && c->rank == 0)
        fprintf(stderr, "[gb_ba x%d] it %d cost %.12e lambda %.3e accepted %d pcg %d%s\n", c->world, it, h.cost, h.lambda, h.accepted, h.pcg_iters,
                h.stop ? " stop" : "");
      if (h.stop) break;
    }
  }
  GB_CUDA(ctx, cudaEventRecord(ctx->eve, ctx->stream));
  GB_CHECK(ba_graph_finish_impl(ctx, g, c, res));
  if (res) GB_CUDA(ctx, cudaEventElapsedTime(&res->gpu_ms, ctx->evs, ctx->eve));
  return GB_OK;
}

// One process, N GPUs: shard `pb` over the communicators' devices (one host thread per device), solve, write every camera
// (identical on all ranks; rank 0's copy) and each shard's landmarks back into the caller's arrays.
int gb_ba_solve_multi(int n_dev, gb_comm* const* comms, gb_ba_problem* pb, const gb_ba_options* opt, gb_ba_result* res) {
  if (n_dev < 1 || !comms || !pb) return GB_ERR_INVALID;
  for (int i = 0; i < n_dev; ++i)
    if (!comms[i] || comms[i]->world != n_dev || comms[i]->rank != i) return GB_ERR_INVALID;
  std::vector<int> rc(n_dev, GB_OK);
  std::vector<gb_ba_result> rr(n_dev);
  std::vector<std::vector<double>> poses(n_dev);
  auto worker = [&](int r) {
    gb_comm* c = comms[r];
    gb_ba_graph* g = nullptr;
    rc[r] = gb_ba_shard_create(c, pb, &g);
    // (a rank that failed BEFORE its first collective must not leave the others waiting inside NCCL: creation errors are
    //  argument errors, identical on every rank, so all ranks bail out together)
    if (rc[r] == GB_OK) rc[r] = gb_ba_shard_solve(c, g, opt, &rr[r]);
    if (rc[r] == GB_OK) {
      poses[r].resize((size_t)pb->n_cams * 7);
      const int lo = g->shard_lo, hi = g->shard_hi;
      rc[r] = gb_ba_graph_download(c->ctx, g, poses[r].data(), hi > lo ? pb->points + 3 * (size_t)lo : nullptr);
    }
    if (g) gb_ba_graph_destroy(c->ctx, g);
  };
  std::vector<std::thread> th;
  for (int r = 1; r < n_dev; ++r) th.emplace_back(worker, r);
  worker(0);
  for (auto& t : th) t.join();
  for (int r = 0; r < n_dev; ++r)
    if (rc[r] != GB_OK) {
      if (r > 0) gb_set_error(comms[0]->ctx, "rank %d: %s", r, gb_last_error(comms[r]->ctx));
      return rc[r];
    }
  if (pb->n_cams > 0) memcpy(pb->cam_pose_wc, poses[0].data(), (size_t)pb->n_cams * 56);
  if (res) {
    *res = rr[0];
    for (int r = 1; r < n_dev; ++r) res->gpu_ms = std::max(res->gpu_ms, rr[r].gpu_ms);
  }
  return GB_OK;
}

// ---- test hooks ---------------------------------------------------------------------------------------------------------------
// A loopback group of `world` ranks on base's device, for testing the sharded engine on one GPU: rank 0 runs on `base`, ranks
// 1..world-1 on new contexts that share base's stream (ctxs_out[r]; the caller destroys them before `base`).  Separate contexts are
// needed because gb_ba_shard_solve holds its ctx lock for the whole LM loop.  NCCL is not involved.
GB_API int gb_dbg_comm_create_local(gb_ctx* base, int world, gb_ctx** ctxs_out, gb_comm** comms_out) {
  if (!base || world < 1 || world > kLoopbackMaxWorld || !ctxs_out || !comms_out) return GB_ERR_INVALID;
  for (int r = 0; r < world; ++r) { ctxs_out[r] = nullptr; comms_out[r] = nullptr; }
  ctxs_out[0] = base;
  for (int r = 1; r < world; ++r) {
    const int rc = gb_ctx_create_on_stream(base->device, base->stream, &ctxs_out[r]);
    if (rc != GB_OK) {
      for (int k = 1; k < r; ++k) { gb_ctx_destroy(ctxs_out[k]); ctxs_out[k] = nullptr; }
      ctxs_out[0] = nullptr;
      return rc;
    }
  }
  LoopbackGroup* grp = new LoopbackGroup();
  grp->world = grp->live = world;
  grp->stream = base->stream;
  grp->sm_count = base->sm_count;
  for (int r = 0; r < world; ++r) {
    comms_out[r] = new gb_comm();
    comms_out[r]->ctx = ctxs_out[r]; comms_out[r]->rank = r; comms_out[r]->world = world; comms_out[r]->loop = grp;
  }
  return GB_OK;
}

// The compact reduced system of ONE LM iteration of a shard at its current estimate: begin, then the first half of the iteration
// (sweep, Schur complement of the shard's landmarks into rbuf) and, when `allreduce` is set, the all-reduce (a collective: every
// rank calls it).  S (6N x 6N, dense, undamped), g~, diag U (n6 each) and the cost, each where non-null.
GB_API int gb_dbg_ba_shard_reduced(gb_comm* c, gb_ba_graph* g, const gb_ba_options* opt, int allreduce, double* S, double* gt,
                                   double* diagU, double* cost) {
  if (!c || !g) return GB_ERR_INVALID;
  gb_ctx* ctx = c->ctx;
  CtxLock lk(ctx);
  if (!g->pcg_bcsr || !g->rbuf) { gb_set_error(ctx, "gb_dbg_ba_shard_reduced: the graph has no block-CSR reduced system"); return GB_ERR_INVALID; }
  if (g->shard_world != c->world || g->shard_rank != c->rank) { gb_set_error(ctx, "gb_dbg_ba_shard_reduced: graph / communicator mismatch"); return GB_ERR_INVALID; }
  GB_CHECK(gb_ba_graph_begin(ctx, g, opt));
  GB_CHECK(ba_compact_reduce(ctx, g, allreduce ? c : nullptr));
  const BaDev& d = g->d;
  const size_t n6 = d.n6, nnzb = d.s_nnzb;
  std::vector<double> rb(g->rbuf_doubles);
  std::vector<int> brow(nnzb), col(nnzb);
  GB_CUDA(ctx, cudaMemcpyAsync(rb.data(), g->rbuf, rb.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaMemcpyAsync(brow.data(), d.s_brow, nnzb * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaMemcpyAsync(col.data(), d.s_col, nnzb * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (S) {
    memset(S, 0, n6 * n6 * sizeof(double));
    for (size_t blk = 0; blk < nnzb; ++blk)
      for (int k = 0; k < 36; ++k) S[(6 * (size_t)brow[blk] + k / 6) * n6 + 6 * (size_t)col[blk] + k % 6] = rb[36 * blk + k];
  }
  const double* tail = rb.data() + 36 * nnzb;
  if (gt) memcpy(gt, tail, n6 * sizeof(double));
  if (diagU) memcpy(diagU, tail + n6, n6 * sizeof(double));
  if (cost) *cost = tail[2 * n6];
  return GB_OK;
}

}  // extern "C"
