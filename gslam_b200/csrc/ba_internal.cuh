// gslam_b200/csrc/ba_internal.cuh — host-side types and entry points shared by the bundle-adjustment translation units
// (ba.cu: graph upload, kernels of the sweep / Schur / local PCG paths; ba_pcg_bcsr.cu: the multi-CTA block-CSR PCG of large
// reduced systems; ba_dist.cu: the landmark-sharded multi-GPU solve and its communicator).  Not part of the C-ABI.
#pragma once
#include <vector>

#include "ba_device.cuh"
#include "common.cuh"

// host-made plans of graph creation, uploaded with the graph (ba_graph_create_impl lays them out)
struct BaSchurPlan {  // landmark-chunk Schur complement: BaDev::sp_*
  std::vector<int> pt0, order, nused, boff, bidx, coff, cidx;
  std::vector<unsigned short> mask;
  std::vector<uint8_t> slots;
};
struct BaPosePlan {  // pose-graph edges and their gather plans: BaDev::pe_* / pc_* / pp_*
  std::vector<int> ei, ej, pc_off, pc_ent, pp_off, pp_ij, pp_ent;
  std::vector<double> Zinv, info;
  size_t rec_doubles = 0;  // pe_H: staging records of every edge (zeroed at creation)
};

struct gb_ba_graph {
  BaDev d{};
  uint8_t* slab = nullptr;  // the device allocation of a BaPlace::own graph (else null): everything below
  double *pose_init = nullptr, *pts_init = nullptr, *pose_wc_out = nullptr;
  double* buf = nullptr;     // internal [S | gt | diagU | cost | pad]
  double* d_cost = nullptr;  // internal candidate cost
  size_t buf_doubles = 0;
  gb_ba_options opt{};
  std::vector<int> sorted_to_orig;  // sorted observation slot -> caller's edge index
  std::vector<int> cam_perm_h;      // host copy of cam_perm (camera-sorted slot -> sorted slot): refresh of a cached graph
  double* pose_wc_in = nullptr;     // device: the uploaded T_wc poses (blob), source of ba_prepare_kernel
  bool begun = false;
  // what a device-resident solve waits on without holding the ctx lock (made on its first call): the LM scalars' pinned host copy,
  // the solve's timing events and its completion event; `waiting` (read and written under the ctx lock) is set while a solve waits
  // unlocked on them, so that nothing else reuses or frees them meanwhile
  BaScalars* h_sc = nullptr;
  cudaEvent_t ev_s = nullptr, ev_e = nullptr, ev_done = nullptr;
  bool waiting = false;
  // PCG dispatch: single-CTA block-sparse kernel, else one-cluster kernel (pcg_cluster = 8/16), else generic multi-kernel
  bool pcg_sparse = false;
  size_t pcg_sparse_smem = 0;
  int pcg_max_row_blocks = 0;  // longest block row of S
  int sp_max_nused = 0;         // most slots any chunk of the landmark-chunk Schur plan uses (> 80: ba_schur_chunks_kernel runs a 2nd pass)
  int sweep_mode = 0;           // 0 = by size (ba_sweep.cu from 64k observations), 1 = ba.cu's latency-tuned kernel, 2 = ba_sweep.cu
  bool sweep_only = false;     // the last begin came from gb_ba_graph_sweep and nothing else ran since
  int pcg_nact = 0;            // cameras with at least one free dof (the sparse PCG kernel gives lanes to these only)
  int pcg_cluster = 0;
  size_t pcg_smem = 0;
  // multi-CTA block-CSR PCG (ba_pcg_bcsr.cu): plan made at graph creation when the block structure exists and the single-CTA
  // kernel does not apply
  bool pcg_bcsr = false;
  int bcsr_ctas = 0, bcsr_K = 0, bcsr_in_smem = 0, bcsr_max_cams = 0, bcsr_max_blocks = 0, bcsr_cluster = 0, bcsr_blk_stride = 37;
  size_t bcsr_smem = 0;
  unsigned short bcsr_need[16] = {0};  // cluster mode: bcsr_need[c] = CTAs that read the rows of u owned by CTA c
  const int* bcsr_cta_cam = nullptr;  // device [bcsr_ctas + 1]: first camera of each CTA's block-row range
  double* bcsr_part = nullptr;   // device [bcsr_ctas * 2]: per-CTA (gamma, delta) partials
  double* bcsr_u = nullptr;      // device [n6]: the published u = Minv r
  unsigned int* bcsr_bar = nullptr;  // device: grid barrier counter
  double* rbuf = nullptr;        // device: compact reduced system [Sb (nnzb*36) | g~ | diag U | cost | pad]
  size_t rbuf_doubles = 0;
  // direct solver (ba_chol.cu): skyline plan [first | rowoff | last] uploaded with the blob, when the skyline fits one SM
  bool chol_ok = false;
  const int* chol_plan = nullptr;
  int chol_blocks = 0;
  size_t chol_smem = 0;
  // room in the slab for what the test hooks switch on: a re-cut large-graph sweep plan (items, then team_off) of any split they
  // allow, and the PCG's clock stamps (BaDev::prof)
  int* sw_room = nullptr;
  long long* prof_room = nullptr;
  // landmark shard (multi-GPU global BA): this graph holds landmarks [shard_lo, shard_hi) of the caller's problem
  int shard_lo = 0, shard_hi = 0, shard_rank = 0, shard_world = 1;
};

// ---- ba.cu ------------------------------------------------------------------------------------------------------------------
// Where a graph's slab (its uploaded blob and working set) lives, one placement per lifetime:
//  own      a graph the caller holds (gb_ba_graph_create / _ex, gb_ba_shard_create): one allocation (gb_slab_alloc), which
//           gb_ba_graph_destroy frees;
//  cache    the graph gb_ba_solve keeps between calls: the topology cache's grow-only buffer, reused by the next graph it keeps;
//  scratch  a graph that a host-buffer call creates, solves and destroys within itself (gb_ba_pnp, gb_ba_solve_posegraph, an
//           uncached gb_ba_solve): one take of the ctx scratch (gb_scratch_slab), the call's last while the graph lives.
enum class BaPlace { own, cache, scratch };
// shard_world > 1: keep only the landmarks of `shard_rank` (contiguous range balanced by observation count) and their edges;
// all cameras and the GLOBAL covisibility block structure are kept, so that every rank's reduced system has the same layout.
int ba_graph_create_impl(gb_ctx* ctx, const gb_ba_problem* pb, gb_ba_graph** out, BaPlace place, int shard_rank, int shard_world,
                         const gb_pose_edges* pose_edges = nullptr);
// the first half of an LM iteration on the COMPACT reduced layout g->rbuf = [Sb | g~ | diag U | cost | pad] (g->rbuf_doubles
// doubles): sweep + Schur complement of this graph's landmarks into rbuf; a non-null `comm` then all-reduces it over the shards
int ba_compact_reduce(gb_ctx* ctx, gb_ba_graph* g, gb_comm* comm);
// a whole solve (gb_ba_graph_solve, the host-buffer solves, and with a non-null `comm` one rank of gb_ba_shard_solve): begin, the
// LM iterations, one synchronisation; T_wc poses / points into pose_out / pts_out where non-null
int ba_graph_solve_impl(gb_ctx* ctx, gb_ba_graph* g, gb_comm* comm, const gb_ba_options* opt, gb_ba_result* res, double* pose_out,
                        double* pts_out);
// test hooks: S (6N x 6N, dense) <- the block-CSR values `blocks` (36 per block of g's S structure, at block row s_brow and block
// column s_col), 0.0 elsewhere; synchronises the stream
int ba_download_S(gb_ctx* ctx, const gb_ba_graph* g, const double* blocks, double* S);

// ---- ba_pose.cu -------------------------------------------------------------------------------------------------------------
// pose-graph terms (SE3Edge / GPSEdge, Optimizer.h:127-148) on the stepwise dense-layout solver path
int ba_pose_validate(gb_ctx* ctx, const gb_ba_problem* pb, const gb_pose_edges* pe);
void ba_pose_plan(gb_ba_graph* g, const gb_pose_edges* pe, BaPosePlan& p);  // host-only: edges + gather plans, sets d.npe / d.pe_npairs
int ba_pose_linearize(gb_ctx* ctx, gb_ba_graph* g, cudaStream_t s);         // after the sweep: records -> U, g_c, cost terms
int ba_pose_offdiag(gb_ctx* ctx, gb_ba_graph* g, double* buf, cudaStream_t s);  // after the Schur complement: S_ij += J_i' Omega J_j
int ba_pose_cost(gb_ctx* ctx, gb_ba_graph* g, cudaStream_t s);              // candidate cost terms at pose_new

// ---- ba_sweep.cu ------------------------------------------------------------------------------------------------------------
// the bandwidth-tuned residual + Jacobian sweep of large graphs (persistent CTAs, pose table in shared memory, bulk-copied W tiles)
void ba_sweep_plan_host(int nc, int np, int cam_split, const std::vector<int>& cam_off, const std::vector<int>& pt_off, int n_teams,
                        std::vector<int>& items4, std::vector<int>& team_off);  // host-only: item records + per-team ranges
int ba_sweep_teams(const gb_ctx* ctx);  // the plan's n_teams on this ctx's device
int ba_sweep_launch(gb_ctx* ctx, const BaDev& d, cudaStream_t s, int which /* 3 whole, 1 cameras, 2 landmarks */);

// ---- ba_pcg_bcsr.cu ---------------------------------------------------------------------------------------------------------
// Host-only: decide whether / how the multi-CTA block-CSR PCG applies to `g` (sets pcg_bcsr and the scalar bcsr_* fields, fills
// cta_cam, the first camera of each CTA's block-row range).
void ba_pcg_bcsr_plan(gb_ctx* ctx, gb_ba_graph* g, const int* s_rowptr_host, const int* s_col_host, std::vector<int>& cta_cam);
// damp + block-Jacobi PCG on the reduced camera system held in `rbuf` + retraction of the cameras (pose_new, Rt_new, x)
int ba_pcg_bcsr_launch(gb_ctx* ctx, gb_ba_graph* g, const double* rbuf);

// ---- ba_chol.cu -------------------------------------------------------------------------------------------------------------
bool ba_chol_plan_host(gb_ctx* ctx, int nc, const int* s_rowptr, const int* s_col, std::vector<int>& plan3, int* nblocks, size_t* smem);
// block-skyline Cholesky solve of the damped reduced camera system in the dense-layout `buf` (+ g->d.Sb block values) + retraction
int ba_chol_launch(gb_ctx* ctx, gb_ba_graph* g, double* buf, bool pdl);

// host-buffer solve cache (ba.cu): free the graph gb_ba_solve kept on this ctx and the buffer it lives in (gb_ctx_destroy)
void ba_cache_free(gb_ctx* ctx);
