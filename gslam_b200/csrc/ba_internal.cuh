// gslam_b200/csrc/ba_internal.cuh — host-side types and entry points shared by the bundle-adjustment translation units
// (ba.cu: graph upload, kernels of the sweep / Schur / local PCG paths; ba_pcg_bcsr.cu: the multi-CTA block-CSR PCG of large
// reduced systems; ba_dist.cu: the landmark-sharded multi-GPU solve and its communicator).  Not part of the C-ABI.
#pragma once
#include <type_traits>
#include <vector>

#include "ba_device.cuh"
#include "common.cuh"

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
  uint8_t* slab = nullptr;  // one device allocation (or the ctx arena) holding everything below but the sweep plan
  size_t slab_bytes = 0;
  bool from_arena = false;
  double *pose_init = nullptr, *pts_init = nullptr, *pose_wc_out = nullptr;
  double* buf = nullptr;     // internal [S | gt | diagU | cost | pad]
  double* d_cost = nullptr;  // internal candidate cost
  size_t buf_doubles = 0;
  gb_ba_options opt{};
  std::vector<int> sorted_to_orig;  // sorted observation slot -> caller's edge index
  std::vector<int> cam_perm_h;      // host copy of cam_perm (camera-sorted slot -> sorted slot): refresh of a cached graph
  double* pose_wc_in = nullptr;     // device: the uploaded T_wc poses (blob), source of ba_prepare_kernel
  bool begun = false;
  // PCG dispatch: single-CTA block-sparse kernel, else one-cluster kernel (pcg_cluster = 8/16), else generic multi-kernel
  bool pcg_sparse = false;
  size_t pcg_sparse_smem = 0;
  int pcg_max_row_blocks = 0;  // longest block row of S
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
  void* sw_alloc = nullptr;      // device allocation holding the large-graph sweep's item plan (BaDev::sw_*), made on first use
  std::vector<int> pt_off_h, cam_off_h;  // host copies of pt_off / cam_off (the sweep plan is cut from them)
  // landmark shard (multi-GPU global BA): this graph holds landmarks [shard_lo, shard_hi) of the caller's problem
  int shard_lo = 0, shard_hi = 0, shard_rank = 0, shard_world = 1;
};

// ---- ba.cu ------------------------------------------------------------------------------------------------------------------
// shard_world > 1: keep only the landmarks of `shard_rank` (contiguous range balanced by observation count) and their edges;
// all cameras and the GLOBAL covisibility block structure are kept, so that every rank's reduced system has the same layout.
int ba_graph_create_impl(gb_ctx* ctx, const gb_ba_problem* pb, gb_ba_graph** out, bool use_arena, int shard_rank, int shard_world,
                         const gb_pose_edges* pose_edges = nullptr);
// one LM iteration on the COMPACT reduced layout g->rbuf = [Sb | g~ | diag U | cost | pad] (g->rbuf_doubles doubles): sweep (if
// needed) + Schur blocks, block-CSR PCG, back-substitution + candidate cost, LM accept / reject + install.  A non-null `comm`
// all-reduces the reduced system and the candidate cost of this landmark shard before they are used.
int ba_compact_iteration(gb_ctx* ctx, gb_ba_graph* g, gb_comm* comm);
// its two halves: ba_compact_reduce = sweep + Schur complement of this graph's landmarks into rbuf (+ the all-reduce);
// ba_compact_step = PCG, back-substitution + candidate cost (+ its all-reduce), LM accept / reject
int ba_compact_reduce(gb_ctx* ctx, gb_ba_graph* g, gb_comm* comm);
int ba_compact_step(gb_ctx* ctx, gb_ba_graph* g, gb_comm* comm);

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
void ba_sweep_plan_drop(gb_ba_graph* g);  // (cam_split changed / graph destroyed)
int ba_sweep_launch(gb_ctx* ctx, gb_ba_graph* g, const BaDev& d, cudaStream_t s, int which /* 3 whole, 1 cameras, 2 landmarks */);

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

// host-buffer solve cache (ba.cu): drop the graph gb_ba_solve kept from its previous call on this ctx
void ba_cache_drop(gb_ctx* ctx);
