// gslam_b200/csrc/ba.cu — bundle adjustment behind GSLAM::Optimizer::optimize / optimizePnP
// (GSLAM/core/Optimizer.h:202-207,229; graph PODs :106-172; OptimzeConfig :174-182).
//
// Generic stream-ordered path (any problem size; also the per-rank engine of the landmark-sharded global BA):
//   K6a ba_linearize_points : fused residual + 2x3/2x6 Jacobian sweep, one thread per landmark over its (point-sorted)
//                             observation segment -> V_j, g_p,j, W_k (6x3 per observation), per-landmark cost.  No J is
//                             ever materialised.
//   K6b ba_linearize_cams   : one CTA per camera over its (camera-sorted) observation list, recomputing the residual,
//                             fixed-tree block reduction -> U_i (6x6), g_c,i.  Deterministic (no atomics).
//   K7a ba_prepare_schur / ba_schur_blocks (or _chunks + _reduce, or _accum + ba_mirror) : damped V^-1,
//                             S = U - sum_j W V^-1 W', g~ = g_c - sum W V^-1 g_p.
//   K7b ba_damp / pcg_init / pcg_matvec / pcg_update / ba_retract : block-Jacobi PCG on the reduced camera system, convergence
//                             decided on device, candidate camera poses.
//   ba_backsub_cost / ba_reduce_cost / ba_commit_apply : back-substitution + candidate cost, LM accept/reject + install.
// All LM state lives in BaScalars on the device; kernels early-exit on its flags, so an iteration needs no host sync.  The LM rules
// themselves (decision, damping, preconditioner, retraction, V^-1) are the helpers of ba_device.cuh, shared by every solver path.
#include "ba_device.cuh"
#include "common.cuh"
#include "ba_internal.cuh"

#include <cooperative_groups.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>

using namespace ba;

// ======================================================================================================================
// kernels
// ======================================================================================================================
namespace {

constexpr int kMaxBlockCams = 2048;  // covisibility block structure of S is derived on the host up to this many cameras
constexpr int kPtThreads = 128;
constexpr int kCamThreads = 128;
constexpr int kRedThreads = 1024;

__global__ void ba_prepare_kernel(int nc, const double* __restrict__ pose_wc, double* __restrict__ pose_cw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  double in[7], out[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) in[k] = pose_wc[7 * i + k];
  se3_inverse(in, out);
#pragma unroll
  for (int k = 0; k < 7; ++k) pose_cw[7 * i + k] = out[k];
}

__global__ void ba_rt_kernel(int nc, const double* __restrict__ pose, double* __restrict__ Rt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  double q[4] = {pose[7 * i], pose[7 * i + 1], pose[7 * i + 2], pose[7 * i + 3]}, R[9];
  quat_to_R(q, R);
#pragma unroll
  for (int k = 0; k < 9; ++k) Rt[12 * i + k] = R[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) Rt[12 * i + 9 + k] = pose[7 * i + 4 + k];
}

// K6a: fused residual + Jacobian sweep, 8 lanes per landmark (lane k takes observations k, k+8, ... of the point-sorted
// segment), fixed xor-tree over the 8 lanes -> V_j, g_p,j, cost_j; every lane writes the W blocks of its own observations.
constexpr int kLpp = 8;
// The W blocks (144 B per observation) leave through a per-warp shared-memory tile: a lane's nine 16-byte pieces would hit 32
// half-written sectors per store instruction (144-byte lane stride); staged, the eight lanes of a landmark write its run of
// consecutive blocks as full 128-byte lines.  The loop is warp-uniform (max over the four landmarks of a warp) and the camera
// index / measurement of the NEXT round are requested before the current one is evaluated.
__device__ __forceinline__ void ba_linearize_points_body(const BaDev& g, int block) {
  __shared__ __align__(16) double s_w[kPtThreads / 32][32 * 18];
  const int gt = block * kPtThreads + threadIdx.x;
  const int jraw = gt / kLpp, sub = gt % kLpp, lane = threadIdx.x & 31;
  const bool valid = jraw < g.np;
  const int j = valid ? jraw : 0;
  // -- static graph structure first: under a programmatic dependent launch this runs while the predecessor kernel drains
  const bool pf = g.pfree[j] != 0;
  const int e0 = g.pt_off[j], e1 = valid ? g.pt_off[j + 1] : e0;
  int e = e0 + sub;
  bool act = e < e1;
  int i = act ? g.o_cam[e] : 0;
  double2 uv = act ? *reinterpret_cast<const double2*>(g.o_uv + 2 * (size_t)e) : make_double2(0.0, 0.0);
  gb_pdl_wait();
  if (g.sc->stop || !g.sc->need_linearize) return;
  // -- the estimate (written by the predecessor); an accepted-but-not-installed candidate is read from the candidate arrays
  //    and installed here (every reader of this launch takes the same branch, nobody reads what is being written)
  const double delta = g.sc->delta;
  const bool pend = g.sc->pending != 0;
  const double* PTS = pend ? g.pts_new : g.pts;
  const double* RT = pend ? g.Rt_new : g.Rt;
  const double p[3] = {PTS[3 * (size_t)j], PTS[3 * (size_t)j + 1], PTS[3 * (size_t)j + 2]};
  if (pend && valid && sub == 0) { g.pts[3 * (size_t)j] = p[0]; g.pts[3 * (size_t)j + 1] = p[1]; g.pts[3 * (size_t)j + 2] = p[2]; }
  double acc[10];  // V upper triangle (6), g_p (3), cost (1)
#pragma unroll
  for (int k = 0; k < 10; ++k) acc[k] = 0.0;
  const int rounds = __reduce_max_sync(0xffffffffu, (e1 - e0 + kLpp - 1) / kLpp);
  double* tile = s_w[threadIdx.x >> 5];
  double2* mine = reinterpret_cast<double2*>(tile + 18 * lane);                     // this lane's block in the tile
  const double2* run = reinterpret_cast<const double2*>(tile + 18 * (lane - sub));  // the landmark's eight blocks
  for (int rd = 0; rd < rounds; ++rd) {
    const int en = e + kLpp;
    const bool actn = en < e1;
    const int i_nx = actn ? g.o_cam[en] : 0;
    const double2 uv_nx = actn ? *reinterpret_cast<const double2*>(g.o_uv + 2 * (size_t)en) : make_double2(0.0, 0.0);
    bool have = false;
    if (act) {
      const double* Rt = RT + 12 * i;
      const ObsLin o = eval_obs(Rt, p, uv.x, uv.y, g.has_info ? g.o_info + 3 * (size_t)e : nullptr, delta);
      if (o.valid) {
        have = true;
        acc[9] += o.rho;
        double Jc[12], Jp[6], AJp[6];
        jac_cam(o, g.dof[i], Jc);
        jac_pt(o, Rt, pf, Jp);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          AJp[d] = o.A0 * Jp[d] + o.A1 * Jp[3 + d];
          AJp[3 + d] = o.A1 * Jp[d] + o.A2 * Jp[3 + d];
        }
        const double Ar0 = o.A0 * o.r0 + o.A1 * o.r1, Ar1 = o.A1 * o.r0 + o.A2 * o.r1;
        double wv[18];
#pragma unroll
        for (int a = 0; a < 6; ++a)
#pragma unroll
          for (int c = 0; c < 3; ++c) wv[a * 3 + c] = Jc[a] * AJp[c] + Jc[6 + a] * AJp[3 + c];
#pragma unroll
        for (int k = 0; k < 9; ++k) mine[k] = make_double2(wv[2 * k], wv[2 * k + 1]);
        int t = 0;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
#pragma unroll
          for (int c = a; c < 3; ++c) acc[t++] += Jp[a] * AJp[c] + Jp[3 + a] * AJp[3 + c];
          acc[6 + a] -= Jp[a] * Ar0 + Jp[3 + a] * Ar1;
        }
      }
    }
    if (!have) {  // behind the camera / no observation in this round: a zero block
#pragma unroll
      for (int k = 0; k < 9; ++k) mine[k] = make_double2(0.0, 0.0);
    }
    __syncwarp();
    {  // the landmark's run of (at most eight) consecutive blocks: 9 x 16-byte pieces each, copied by its eight lanes
      const int first = e0 + rd * kLpp;
      const int pieces = 9 * max(0, min(kLpp, e1 - first));
      double2* dst = reinterpret_cast<double2*>(g.W + 18 * (size_t)first);
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const int q = sub + kLpp * k;
        if (q < pieces) dst[q] = run[q];
      }
    }
    __syncwarp();
    e = en; act = actn; i = i_nx; uv = uv_nx;
  }
#pragma unroll
  for (int k = 0; k < 10; ++k) {
#pragma unroll
    for (int o = kLpp / 2; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o, kLpp);
  }
  if (valid && sub == 0) {
    double* V = g.V + 9 * (size_t)j;
    V[0] = acc[0]; V[1] = acc[1]; V[2] = acc[2];
    V[3] = acc[1]; V[4] = acc[3]; V[5] = acc[4];
    V[6] = acc[2]; V[7] = acc[4]; V[8] = acc[5];
    g.gp[3 * (size_t)j] = acc[6]; g.gp[3 * (size_t)j + 1] = acc[7]; g.gp[3 * (size_t)j + 2] = acc[8];
    g.cost_pt[j] = acc[9];
    // damped inverse right away (ba_prepare_schur_kernel redoes it only when a rejected step changed lambda)
    damped_vinv(V, pf && e1 > e0, g.sc->lambda, g.Vinv + 9 * (size_t)j);
  }
}

// K6b: cam_split CTAs per camera (each a contiguous slice of its camera-sorted observations); deterministic tree reduction of
// the 21 upper-triangular U entries + 6 gradient entries inside the CTA, then -- when a camera is split -- the LAST CTA of the
// camera to finish (per-camera ticket) folds the slices' partial sums in slice order.  Bit-reproducible run to run.
__device__ __forceinline__ void ba_linearize_cams_body(const BaDev& g, int cta) {
  const int K = g.cam_split, i = cta / K, slice = cta - i * K;
  // -- static graph structure first (see the landmark pass)
  const int dm = g.dof[i];
  const int c0 = g.cam_off[i], c1 = g.cam_off[i + 1];
  const int per = (c1 - c0 + K - 1) / K;
  const int s0 = min(c0 + slice * per, c1), s1 = min(s0 + per, c1);
  gb_pdl_wait();  // (prefetching the first observation here costs 40 registers: ptxas pipelines the whole loop body)
  if (g.sc->stop || !g.sc->need_linearize) return;
  const double delta = g.sc->delta;
  const bool pend = g.sc->pending != 0;  // (see the landmark pass)
  const double* PTS = pend ? g.pts_new : g.pts;
  const double* Rt = (pend ? g.Rt_new : g.Rt) + 12 * i;
  if (pend && slice == 0) {  // install this camera's accepted pose
    if (threadIdx.x < 12) g.Rt[12 * i + threadIdx.x] = g.Rt_new[12 * i + threadIdx.x];
    else if (threadIdx.x >= 32 && threadIdx.x < 39) g.pose[7 * i + threadIdx.x - 32] = g.pose_new[7 * i + threadIdx.x - 32];
  }
  double acc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0.0;
  for (int idx = s0 + threadIdx.x; idx < s1; idx += kCamThreads) {
    const int j = g.c_pt[idx];
    const double2 uv = *reinterpret_cast<const double2*>(g.c_uv + 2 * (size_t)idx);
    const double p[3] = {PTS[3 * (size_t)j], PTS[3 * (size_t)j + 1], PTS[3 * (size_t)j + 2]};
    const ObsLin o = eval_obs(Rt, p, uv.x, uv.y, g.has_info ? g.o_info + 3 * (size_t)g.cam_perm[idx] : nullptr, delta);
    if (!o.valid) continue;
    double Jc[12], AJc[12];
    jac_cam(o, dm, Jc);
#pragma unroll
    for (int d = 0; d < 6; ++d) {
      AJc[d] = o.A0 * Jc[d] + o.A1 * Jc[6 + d];
      AJc[6 + d] = o.A1 * Jc[d] + o.A2 * Jc[6 + d];
    }
    const double Ar0 = o.A0 * o.r0 + o.A1 * o.r1, Ar1 = o.A1 * o.r0 + o.A2 * o.r1;
    int t = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
#pragma unroll
      for (int b = a; b < 6; ++b) acc[t++] += Jc[a] * AJc[b] + Jc[6 + a] * AJc[6 + b];
    }
#pragma unroll
    for (int a = 0; a < 6; ++a) acc[21 + a] -= Jc[a] * Ar0 + Jc[6 + a] * Ar1;
  }
  // deterministic reduction: fixed shuffle tree inside each warp, then the 4 warp partials are summed in order
  __shared__ double s_red[kCamThreads / 32][27];
  __shared__ int s_last;
#pragma unroll
  for (int k = 0; k < 27; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_down_sync(0xffffffffu, acc[k], o);
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 27; ++k) s_red[threadIdx.x >> 5][k] = acc[k];
  }
  __syncthreads();
  if (threadIdx.x < 27) {
    double r = 0.0;
#pragma unroll
    for (int w = 0; w < kCamThreads / 32; ++w) r += s_red[w][threadIdx.x];
    s_red[0][threadIdx.x] = r;
    if (K > 1) g.cam_part[((size_t)i * K + slice) * 27 + threadIdx.x] = r;
  }
  if (K > 1) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&g.cam_ticket[i], 1u) == (unsigned)(K - 1)) ? 1 : 0;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    if (threadIdx.x < 27) {
      double r = 0.0;
      for (int k = 0; k < K; ++k) r += __ldcg(&g.cam_part[((size_t)i * K + k) * 27 + threadIdx.x]);
      s_red[0][threadIdx.x] = r;
    }
    if (threadIdx.x == 0) g.cam_ticket[i] = 0;
  }
  __syncthreads();
  if (threadIdx.x < 36) {
    const int a = threadIdx.x / 6, c = threadIdx.x % 6, lo = a < c ? a : c, hi = a < c ? c : a;
    const int t = lo * 6 - lo * (lo - 1) / 2 + (hi - lo);  // index of (lo,hi) in the packed upper triangle
    g.U[36 * i + threadIdx.x] = s_red[0][t];
  }
  if (threadIdx.x < 6) g.gc[6 * i + threadIdx.x] = s_red[0][21 + threadIdx.x];
}

// One launch for the whole sweep: the first `cam_blocks` CTAs run the camera pass (K6b: long serial slices, so they start
// first), the remaining CTAs the landmark pass (K6a); the two are independent.
static_assert(kPtThreads == kCamThreads, "the fused sweep launch uses one block size");
__global__ void __launch_bounds__(kPtThreads) ba_linearize_kernel(BaDev g, int cam_blocks) {
  gb_pdl_launch_dependents();  // (both bodies wait for the predecessor after their static prologue and test the LM flags there)
  if ((int)blockIdx.x < cam_blocks) ba_linearize_cams_body(g, blockIdx.x);
  else ba_linearize_points_body(g, blockIdx.x - cam_blocks);
}
// (the camera pass alone: used for the pose information matrix of optimizePnP)
__global__ void __launch_bounds__(kCamThreads) ba_linearize_cams_kernel(BaDev g) {
  ba_linearize_cams_body(g, blockIdx.x);
}

// Deterministic grid-wide sum: block b adds its contiguous slice of src (thread-strided, fixed block tree), the LAST block to finish
// (ticket) folds the gridDim partials in block order and writes scale * sum to out[0].  The order depends on the launch geometry
// only.  All threads of every block must call it; `part` holds >= gridDim doubles, `ticket` is left at 0.
constexpr int kRedPartials = 2048;
template <int NT>
__device__ __forceinline__ void grid_sum_to(const double* __restrict__ src, int n, double scale, double* __restrict__ part, unsigned int* ticket,
                                            double* __restrict__ out, double* s_part /* NT/32 + 1 */, int* s_flag) {
  const int per = (n + (int)gridDim.x - 1) / (int)gridDim.x;
  const int a = min((int)blockIdx.x * per, n), b = min(a + per, n);
  double v = 0.0;
  for (int k = a + (int)threadIdx.x; k < b; k += NT) v += src[k];
  const double t = block_sum<NT>(v, s_part);
  if (threadIdx.x == 0) {
    part[blockIdx.x] = t;
    __threadfence();
    *s_flag = (atomicAdd(ticket, 1u) == gridDim.x - 1) ? 1 : 0;
  }
  __syncthreads();
  if (!*s_flag) return;
  __threadfence();
  double w = 0.0;
  for (int k = threadIdx.x; k < (int)gridDim.x; k += NT) w += __ldcg(part + k);
  const double total = block_sum<NT>(w, s_part);
  if (threadIdx.x == 0) { out[0] = scale * total; *ticket = 0u; }
}

// out[0] = 0.5 * sum(src[0..n)) — any grid up to kRedPartials blocks, deterministic
__global__ void __launch_bounds__(kRedThreads) ba_reduce_cost_kernel(BaDev g, const double* __restrict__ src, int n, double* __restrict__ out) {
  if (g.sc->stop) return;
  __shared__ double s_part[kRedThreads / 32 + 1];
  __shared__ int s_flag;
  grid_sum_to<kRedThreads>(src, n, 0.5, g.red_part, g.red_ticket, out, s_part, &s_flag);
}

// one thread per observation e=(i,j): Y = W_e Vinv_j;  g~_i -= Y g_p,j;  S_{i,i'} -= Y W_f' for every f=(i',j)
__global__ void ba_schur_accum_kernel(BaDev g, double* __restrict__ buf) {
  if (g.sc->stop) return;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= g.no) return;
  const int j = g.o_pt[e], i = g.o_cam[e];
  if (!g.pfree[j]) return;
  const size_t n6 = g.n6;
  double Vi[9], Y[18];
#pragma unroll
  for (int k = 0; k < 9; ++k) Vi[k] = g.Vinv[9 * (size_t)j + k];
  const double* W = g.W + 18 * (size_t)e;
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    const double w0 = W[a * 3], w1 = W[a * 3 + 1], w2 = W[a * 3 + 2];
#pragma unroll
    for (int b = 0; b < 3; ++b) Y[a * 3 + b] = w0 * Vi[b] + w1 * Vi[3 + b] + w2 * Vi[6 + b];
  }
  const double g0 = g.gp[3 * (size_t)j], g1 = g.gp[3 * (size_t)j + 1], g2 = g.gp[3 * (size_t)j + 2];
  double* gt = buf + n6 * n6;
#pragma unroll
  for (int a = 0; a < 6; ++a) atomicAdd(&gt[6 * i + a], -(Y[a * 3] * g0 + Y[a * 3 + 1] * g1 + Y[a * 3 + 2] * g2));
  const int f0 = g.pt_off[j], f1 = g.pt_off[j + 1];
  for (int f = f0; f < f1; ++f) {
    const int i2 = g.o_cam[f];
    if (i2 < i) continue;  // S is symmetric: accumulate the upper block triangle only, ba_mirror_kernel fills the rest
    const double* W2 = g.W + 18 * (size_t)f;
    double w2[18];
#pragma unroll
    for (int k = 0; k < 18; ++k) w2[k] = W2[k];
    double* Sb = buf + (size_t)(6 * i) * n6 + 6 * i2;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int b = 0; b < 6; ++b)
        atomicAdd(&Sb[(size_t)a * n6 + b], -(Y[a * 3] * w2[b * 3] + Y[a * 3 + 1] * w2[b * 3 + 1] + Y[a * 3 + 2] * w2[b * 3 + 2]));
  }
}

// K7a (local BA): deterministic Schur complement, one warp per structurally non-zero UPPER block (i,i'), no atomics.
// The warp walks camera i's observation list (lanes stride it), looks up whether camera i' sees the same landmark, and
// accumulates Y W' (Y = W V^-1) in registers; a fixed shuffle tree reduces the 36 entries; the block and its transpose are
// written once.  The diagonal warps also produce g~_i = g_c,i - sum_j Y g_p,j and diag U.  Bit-reproducible run to run.
__global__ void __launch_bounds__(128) ba_schur_blocks_kernel(BaDev g, double* __restrict__ buf) {
  gb_pdl_launch_dependents();
  // one CTA (4 warps) per upper block: the warps split camera i's observation list, a fixed shuffle tree reduces inside each
  // warp and warp 0 adds the four partials in order
  __shared__ double s_part[4][42];
  const int wid = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int blk = g.s_upper[wid];
  const int i = g.s_brow[blk], i2 = g.s_col[blk];
  const bool diag = i == i2;
  // which edge pair (e, f) on which landmark: static graph structure -- the chain cam_perm -> o_pt -> pt_off -> o_cam of the
  // thread's first observation is walked BEFORE waiting for the predecessor kernel (programmatic dependent launch)
  auto find_pair = [&](int idx, int* e_out, int* j_out) -> int {
    const int e = g.cam_perm[idx];
    const int j = g.o_pt[e];
    *e_out = e; *j_out = j;
    if (!g.pfree[j]) return -1;
    if (diag) return e;
    const int f0 = g.pt_off[j], f1 = g.pt_off[j + 1];
    int f = -1;
    int cam8[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) cam8[t] = (f0 + t < f1) ? g.o_cam[f0 + t] : -1;  // independent loads
#pragma unroll
    for (int t = 7; t >= 0; --t) if (cam8[t] == i2) f = f0 + t;
    for (int t = f0 + 8; t < f1 && f < 0; ++t)
      if (g.o_cam[t] == i2) f = t;
    return f;
  };
  const int c0 = g.cam_off[i], c1 = g.cam_off[i + 1];
  int e_first = 0, j_first = 0, f_first = -1;
  if (c0 + (int)threadIdx.x < c1) f_first = find_pair(c0 + threadIdx.x, &e_first, &j_first);
  gb_pdl_wait();
  if (g.sc->stop) return;
  if (blockIdx.x == 0 && threadIdx.x == 0) g.sc->pending = 0;  // the sweep before this kernel has installed the candidate
  double acc[36], ga[6];
#pragma unroll
  for (int k = 0; k < 36; ++k) acc[k] = 0.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) ga[k] = 0.0;
#pragma unroll 1
  for (int idx = c0 + threadIdx.x; idx < c1; idx += 128) {
    int e = e_first, j = j_first, f = f_first;
    if (idx != c0 + (int)threadIdx.x) f = find_pair(idx, &e, &j);
    if (f < 0) continue;
    double Vi[9], Y[18];
#pragma unroll
    for (int k = 0; k < 9; ++k) Vi[k] = g.Vinv[9 * (size_t)j + k];
    const double* We = g.W + 18 * (size_t)e;
    const double* Wf = g.W + 18 * (size_t)f;
    double wf[18];
#pragma unroll
    for (int k = 0; k < 18; ++k) wf[k] = Wf[k];
#pragma unroll
    for (int a = 0; a < 6; ++a) {
      const double w0 = We[a * 3], w1 = We[a * 3 + 1], w2 = We[a * 3 + 2];
#pragma unroll
      for (int c = 0; c < 3; ++c) Y[a * 3 + c] = w0 * Vi[c] + w1 * Vi[3 + c] + w2 * Vi[6 + c];
    }
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int b = 0; b < 6; ++b) acc[a * 6 + b] += Y[a * 3] * wf[b * 3] + Y[a * 3 + 1] * wf[b * 3 + 1] + Y[a * 3 + 2] * wf[b * 3 + 2];
    if (diag) {
      const double g0 = g.gp[3 * (size_t)j], g1 = g.gp[3 * (size_t)j + 1], g2 = g.gp[3 * (size_t)j + 2];
#pragma unroll
      for (int a = 0; a < 6; ++a) ga[a] += Y[a * 3] * g0 + Y[a * 3 + 1] * g1 + Y[a * 3 + 2] * g2;
    }
  }
#pragma unroll
  for (int k = 0; k < 36; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_down_sync(0xffffffffu, acc[k], o);
  }
#pragma unroll
  for (int k = 0; k < 6; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ga[k] += __shfl_down_sync(0xffffffffu, ga[k], o);
  }
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < 36; ++k) s_part[warp][k] = acc[k];
#pragma unroll
    for (int k = 0; k < 6; ++k) s_part[warp][36 + k] = ga[k];
  }
  __syncthreads();
  if (threadIdx.x < 42) {
    const int k = threadIdx.x;
    const double sum = ((s_part[0][k] + s_part[1][k]) + s_part[2][k]) + s_part[3][k];
    if (k < 36) {
      const int a = k / 6, b = k - 6 * a;
      const double v = (diag ? g.U[36 * i + k] : 0.0) - sum;
      g.Sb[36 * (size_t)blk + k] = v;
      if (!diag) g.Sb[36 * (size_t)g.s_tidx[blk] + b * 6 + a] = v;
    } else if (diag) {
      const int a = k - 36;
      const size_t n6 = g.n6, nS = g.r_gt;
      buf[nS + 6 * i + a] = g.gc[6 * i + a] - sum;
      buf[nS + n6 + 6 * i + a] = g.U[36 * i + a * 7];
    }
  }
}

// ---- K7a (large graphs): Schur complement by LANDMARK CHUNKS -----------------------------------------------------------------------
// The block-gather kernel above walks, for every block (i,i'), camera i's whole observation list: fine for a 50-keyframe window,
// but at global-BA size (500 cameras x 2000 observations each, ~5000 upper blocks) it re-reads every W block ~10 times from L2
// (794 us per LM iteration at config 5).  Here the landmarks are cut (on the host, once per graph) into chunks of consecutive
// landmarks that together see at most 16 cameras; a CTA owns a chunk, thread s owns ONE block slot (la <= lb) of the chunk's
// 16 x 16 upper triangle and walks the chunk's landmarks in order, accumulating Y_a W_b' (Y = W V^-1) for the landmarks both
// cameras observe -- registers only, no atomics, fixed order.  Every W block is read once per slot that needs it and those reads
// hit L1 (the ~10 blocks of a landmark are shared by the whole CTA).  The per-chunk partial blocks go to a staging area and
// ba_schur_reduce_kernel folds them per block in ascending chunk order: bit-reproducible.
// Slots are numbered column-major over the upper triangle (slot = lb(lb+1)/2 + la) so that a chunk that only sees n cameras keeps
// its work in the first n(n+1)/2 threads and the remaining warps skip every landmark.
constexpr int kChunkCams = 16, kChunkSlots = kChunkCams * (kChunkCams + 1) / 2, kChunkThreads = 160, kChunkBatch = 4;
constexpr int kChunkMaxLm = 64;  // landmarks per chunk (host plan)

// v4 (v3 spent its issue slots on index arithmetic of the staging loops, idle lanes and DMUL+DADD around the DFMAs):
//  * the W blocks of a batch are staged EDGE-indexed: a landmark's blocks are contiguous in global memory, so staging is a plain
//    16-byte-granular copy; the slot threads find their two edges with one popcount each;
//  * thread t works the t-th slot the chunk really uses (host table), so a chunk over 10 cameras keeps exactly 55 lanes busy;
//  * batches of 4 landmarks per barrier pair (static shared memory stays under 48 KB: three CTAs per SM), the next batch's W
//    blocks in flight (cp.async) during the arithmetic;
//  * acc = fma(y0, w0, fma(y1, w1, fma(y2, w2, acc))): 108 DFMA per (landmark, slot), nothing else on the fp64 pipe.
//  * v6: TWO threads per slot (rows 0-2 / rows 3-5 of the 6x6 block): v5 kept 2 of a CTA's 5 warps busy in the accumulation and the
//    fp64 pipe mostly idle; halving the per-thread accumulator also frees registers for 4 CTAs / SM.
//    A chunk with more than 80 used slots (13+ cameras; the planner avoids it) is worked in passes of 80 slots.
constexpr int kChunkSlotsPerPass = kChunkThreads / 2;

__global__ void __launch_bounds__(kChunkThreads, 4) ba_schur_chunks_kernel(BaDev g) {
  if (g.sc->stop) return;
  __shared__ __align__(16) double sW[2][kChunkBatch][kChunkCams][18];  // [buffer][landmark of the batch][edge][6x3]
  __shared__ __align__(16) double sY[2][kChunkBatch][kChunkCams][18];
  __shared__ unsigned int s_mask[kChunkMaxLm];
  __shared__ int s_e0[kChunkMaxLm];
  __shared__ double s_vi[kChunkMaxLm][9];
  __shared__ double s_gp[kChunkMaxLm][3];
  const int t = threadIdx.x, chunk = blockIdx.x;
  const int nused = g.sp_nused[chunk];
  const int t0 = g.sp_pt0[chunk], nlm = min(g.sp_pt0[chunk + 1] - t0, kChunkMaxLm);
  for (int w = t; w < nlm * 12; w += kChunkThreads) {
    const int b = w / 12, k = w - 12 * b;
    const int j = g.sp_order[t0 + b];
    if (k < 9) s_vi[b][k] = g.Vinv[9 * (size_t)j + k];
    else s_gp[b][k - 9] = g.gp[3 * (size_t)j + k - 9];
    if (k == 0) { s_mask[b] = g.sp_mask[t0 + b]; s_e0[b] = g.pt_off[j]; }
  }
  __syncthreads();
  // staging: per batch landmark b, edges 0..d_b-1, nine 16-byte pieces each -- asynchronous global -> shared copies (cp.async /
  // LDGSTS: no registers in between; a register-staged prefetch was spilled to local memory by ptxas and stalled on the load it was
  // meant to hide), issued one batch ahead into the other buffer
  auto stage = [&](int tb, int bsel) {
    const int nb = min(kChunkBatch, nlm - tb);
    for (int w = t; w < nb * kChunkCams * 9; w += kChunkThreads) {
      const int b = w / (kChunkCams * 9), r = w - b * (kChunkCams * 9);
      if (r < 9 * __popc(s_mask[tb + b])) {
        const double2* src = reinterpret_cast<const double2*>(g.W + 18 * (size_t)s_e0[tb + b]) + r;
        const unsigned dst = (unsigned)__cvta_generic_to_shared(reinterpret_cast<double2*>(&sW[bsel][b][0][0]) + r);
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  const int half = t & 1;
  for (int pass = 0; pass * kChunkSlotsPerPass < nused; ++pass) {
    const int si = pass * kChunkSlotsPerPass + (t >> 1);
    const bool slot = si < nused;
    const int s = slot ? g.sp_slots[(size_t)chunk * kChunkSlots + si] : 0;
    int lb = 0;
    while (lb < kChunkCams - 1 && (lb + 1) * (lb + 2) / 2 <= s) ++lb;
    const int la = s - lb * (lb + 1) / 2;
    const unsigned int need = slot ? ((1u << la) | (1u << lb)) : 0xffffffffu, below_a = (1u << la) - 1u, below_b = (1u << lb) - 1u;
    double acc[18], ga[3];  // rows 3*half .. 3*half+2 of the slot's 6x6 block (and of g~ on the diagonal)
#pragma unroll
    for (int k = 0; k < 18; ++k) acc[k] = 0.0;
#pragma unroll
    for (int k = 0; k < 3; ++k) ga[k] = 0.0;
    __syncthreads();  // (a previous pass is done with the buffers)
    stage(0, 0);
    int buf = 0;
    for (int tb = 0; tb < nlm; tb += kChunkBatch, buf ^= 1) {
      const int nb = min(kChunkBatch, nlm - tb);
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncthreads();  // batch tb has landed in sW[buf]; everybody is done reading sW[buf ^ 1] / sY[buf ^ 1] (batch tb - 1)
      if (tb + kChunkBatch < nlm) stage(tb + kChunkBatch, buf ^ 1);  // in flight during the Y step and the accumulation below
      // Y = W V^-1 : one thread per (landmark, edge, row)
      for (int w = t; w < nb * kChunkCams * 6; w += kChunkThreads) {
        const int b = w / (kChunkCams * 6), r = w - b * (kChunkCams * 6), k = r / 6, a = r - 6 * k;
        if (k < __popc(s_mask[tb + b])) {
          const double* Vi = s_vi[tb + b];
          const double w0 = sW[buf][b][k][a * 3], w1 = sW[buf][b][k][a * 3 + 1], w2 = sW[buf][b][k][a * 3 + 2];
#pragma unroll
          for (int c = 0; c < 3; ++c) sY[buf][b][k][a * 3 + c] = w0 * Vi[c] + w1 * Vi[3 + c] + w2 * Vi[6 + c];
        }
      }
      __syncthreads();
      if (slot) {
        for (int b = 0; b < nb; ++b) {
          const unsigned int m = s_mask[tb + b];
          if ((m & need) != need) continue;
          const double* Yp = &sY[buf][b][__popc(m & below_a)][9 * half];
          const double2* W2 = reinterpret_cast<const double2*>(&sW[buf][b][__popc(m & below_b)][0]);
          double wb[18];
#pragma unroll
          for (int k = 0; k < 9; ++k) { const double2 v = W2[k]; wb[2 * k] = v.x; wb[2 * k + 1] = v.y; }
          const bool dg = la == lb;
          const double g0 = s_gp[tb + b][0], g1 = s_gp[tb + b][1], g2 = s_gp[tb + b][2];
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            const double y0 = Yp[a * 3], y1 = Yp[a * 3 + 1], y2 = Yp[a * 3 + 2];
#pragma unroll
            for (int c = 0; c < 6; ++c) acc[a * 6 + c] = fma(y0, wb[c * 3], fma(y1, wb[c * 3 + 1], fma(y2, wb[c * 3 + 2], acc[a * 6 + c])));
            if (dg) ga[a] = fma(y0, g0, fma(y1, g1, fma(y2, g2, ga[a])));
          }
        }
      }
    }
    if (slot) {
      double2* dst = reinterpret_cast<double2*>(g.sp_stageS + ((size_t)chunk * kChunkSlots + s) * 36 + 18 * half);
#pragma unroll
      for (int k = 0; k < 9; ++k) dst[k] = make_double2(acc[2 * k], acc[2 * k + 1]);
      if (la == lb) {
        double* dg = g.sp_stageG + ((size_t)chunk * kChunkCams + la) * 6 + 3 * half;
#pragma unroll
        for (int k = 0; k < 3; ++k) dg[k] = ga[k];
      }
    }
  }
}

// one 64-thread CTA per upper block: S_blk = [U_i on the diagonal] - sum of the chunk partials (ascending chunk order), written with
// its transpose; the diagonal CTAs also produce g~_i and diag U (same outputs as ba_schur_blocks_kernel)
__global__ void __launch_bounds__(64) ba_schur_reduce_kernel(BaDev g, double* __restrict__ buf) {
  if (g.sc->stop) return;
  const int u = blockIdx.x, k = threadIdx.x;
  const int blk = g.s_upper[u];
  const int i = g.s_brow[blk], i2 = g.s_col[blk];
  const bool diag = i == i2;
  if (k < 36) {
    double sum = 0.0;
    for (int t = g.sp_boff[u]; t < g.sp_boff[u + 1]; ++t) sum += g.sp_stageS[(size_t)g.sp_bidx[t] * 36 + k];
    const int a = k / 6, b = k - 6 * a;
    const double v = (diag ? g.U[36 * i + k] : 0.0) - sum;
    g.Sb[36 * (size_t)blk + k] = v;
    if (!diag) g.Sb[36 * (size_t)g.s_tidx[blk] + b * 6 + a] = v;
  } else if (diag && k < 42) {
    const int a = k - 36;
    double sum = 0.0;
    for (int t = g.sp_coff[i]; t < g.sp_coff[i + 1]; ++t) sum += g.sp_stageG[(size_t)g.sp_cidx[t] * 6 + a];
    const size_t n6 = g.n6;
    buf[g.r_gt + 6 * i + a] = g.gc[6 * i + a] - sum;
    buf[g.r_gt + n6 + 6 * i + a] = g.U[36 * i + a * 7];
  }
}

// scatter the block-CSR values into the dense S of `buf` (whose other entries ba_prepare_schur_kernel wrote)
__global__ void ba_densify_fill_kernel(BaDev g, double* __restrict__ buf) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= g.s_nnzb * 36) return;
  const int blk = w / 36, k = w - 36 * blk, a = k / 6, b = k - 6 * a;
  buf[(size_t)(6 * g.s_brow[blk] + a) * g.n6 + 6 * g.s_col[blk] + b] = g.Sb[w];
}

// lower block triangle <- transpose of the upper one (S_{i',i} = S_{i,i'}^T)
__global__ void ba_mirror_kernel(BaDev g, double* __restrict__ buf) {
  if (g.sc->stop) return;
  const size_t n6 = g.n6, nS = n6 * n6;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < nS; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t row = idx / n6, col = idx - row * n6;
    if (col / 6 < row / 6) buf[idx] = buf[col * n6 + row];
  }
}

// Marquardt damping of the camera blocks, reading the (possibly all-reduced) diag U; fixed dofs get a unit diagonal
__global__ void ba_damp_kernel(BaDev g, double* __restrict__ buf) {
  if (g.sc->stop) return;
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= g.n6) return;
  const size_t n6 = g.n6;
  const int i = d / 6, a = d % 6;
  double* s = buf + (size_t)d * n6 + d;
  *s = lm_damp(*s, buf[n6 * n6 + n6 + d], g.sc->lambda, (g.dof[i] >> a) & 1);
}

// ---- PCG ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kRedThreads) pcg_init_kernel(BaDev g, const double* __restrict__ buf) {
  if (g.sc->stop) return;
  const size_t n6 = g.n6;
  const double* S = buf;
  const double* gt = buf + n6 * n6;
  for (int i = threadIdx.x; i < g.nc; i += kRedThreads) {
    double M[36];
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int b = 0; b < 6; ++b) M[a * 6 + b] = S[(size_t)(6 * i + a) * n6 + 6 * i + b];
    block_jacobi_inverse(M, S + (size_t)(6 * i) * n6 + 6 * i, n6);
#pragma unroll
    for (int k = 0; k < 36; ++k) g.Minv[36 * (size_t)i + k] = M[k];
  }
  // Chronopoulos-Gear PCG (same recurrence as oracle/ba_ref.c::ba_pcg): u = Minv r is kept in g.z, w = S u in g.q, s = S p in g.sv
  for (int d = threadIdx.x; d < g.n6; d += kRedThreads) {
    g.x[d] = 0.0;
    g.r[d] = gt[d];
    g.p[d] = 0.0;
    g.sv[d] = 0.0;
  }
  __syncthreads();
  for (int d = threadIdx.x; d < g.n6; d += kRedThreads) {
    const int i = d / 6, a = d % 6;
    double s = 0.0;
#pragma unroll
    for (int b = 0; b < 6; ++b) s += g.Minv[36 * (size_t)i + a * 6 + b] * gt[6 * i + b];
    g.z[d] = s;
  }
  if (threadIdx.x == 0) {
    g.sc->pcg_first = 1;
    g.sc->pcg_k = 0;
    g.sc->pcg_done = 0;
  }
}

// w = S u : one warp per row, coalesced row reads, fixed shuffle tree
__global__ void __launch_bounds__(256) pcg_matvec_kernel(BaDev g, const double* __restrict__ buf) {
  if (g.sc->stop || g.sc->pcg_done) return;
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= g.n6) return;
  const double* Srow = buf + (size_t)row * g.n6;
  double s = 0.0;
  for (int c = lane; c < g.n6; c += 32) s += Srow[c] * g.z[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if (lane == 0) g.q[row] = s;
}

__global__ void __launch_bounds__(kRedThreads) pcg_update_kernel(BaDev g, int maxit) {
  if (g.sc->stop || g.sc->pcg_done) return;
  __shared__ double s_part[kRedThreads / 32 + 1];
  BaScalars* sc = g.sc;
  const double gamma_prev = sc->rz, gamma0_prev = sc->rz0, alpha_prev = sc->pcg_alpha, tol = sc->pcg_tol;
  const int first = sc->pcg_first, k = sc->pcg_k;
  double pa = 0.0, pb = 0.0;
  for (int d = threadIdx.x; d < g.n6; d += kRedThreads) {
    pa += g.r[d] * g.z[d];
    pb += g.q[d] * g.z[d];
  }
  const double gn = block_sum<kRedThreads>(pa, s_part);
  const double dl = block_sum<kRedThreads>(pb, s_part);
  double alpha, beta, gamma0 = gamma0_prev;
  if (first) {
    gamma0 = gn;
    if (!(gn > 0.0) || !(dl > 0.0)) {
      if (threadIdx.x == 0) sc->pcg_done = 1;
      return;
    }
    alpha = gn / dl;
    beta = 0.0;
  } else {
    if (!(gn > 0.0) || gn < tol * tol * gamma0) {  // convergence test of the previous update
      if (threadIdx.x == 0) sc->pcg_done = 1;
      return;
    }
    beta = gn / gamma_prev;
    const double den = dl - beta * gn / alpha_prev;
    if (!(den > 0.0)) {
      if (threadIdx.x == 0) sc->pcg_done = 1;
      return;
    }
    alpha = gn / den;
  }
  if (k >= maxit) {
    if (threadIdx.x == 0) sc->pcg_done = 1;
    return;
  }
  for (int d = threadIdx.x; d < g.n6; d += kRedThreads) {
    const double pd = g.z[d] + beta * g.p[d];
    const double sd = g.q[d] + beta * g.sv[d];
    g.p[d] = pd;
    g.sv[d] = sd;
    g.x[d] += alpha * pd;
    g.r[d] -= alpha * sd;
  }
  __syncthreads();
  for (int d = threadIdx.x; d < g.n6; d += kRedThreads) {
    const int i = d / 6, a = d % 6;
    double s = 0.0;
#pragma unroll
    for (int b = 0; b < 6; ++b) s += g.Minv[36 * (size_t)i + a * 6 + b] * g.r[6 * i + b];
    g.z[d] = s;
  }
  if (threadIdx.x == 0) {
    sc->rz = gn;
    sc->rz0 = gamma0;
    sc->pcg_alpha = alpha;
    sc->pcg_beta = beta;
    sc->pcg_first = 0;
    sc->pcg_k = k + 1;
    sc->pcg_iters++;
  }
}

__global__ void ba_retract_kernel(BaDev g) {
  if (g.sc->stop) return;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.nc) return;
  retract_camera(g, i, g.x + 6 * i);
}

// LM accept / reject AND the installation of an accepted candidate in one launch.  Every thread derives the decision from the two
// (possibly all-reduced) costs alone; only thread 0 of CTA 0 touches the LM scalars, so nobody reads what it writes.  Re-running it
// after a stop is harmless: the candidate arrays are frozen once `stop` is set.
__global__ void ba_commit_apply_kernel(BaDev g, const double* __restrict__ buf, const double* __restrict__ d_cost) {
  const size_t n6 = g.n6;
  const double cost = buf[g.r_gt + 2 * n6], cnew = d_cost[0];
  const bool ok = (blockIdx.x == 0 && threadIdx.x == 0 && !g.sc->stop) ? lm_decide(g.sc, cost, cnew) : lm_accepts(cost, cnew);
  if (!ok) return;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < g.nc * 7) g.pose[t] = g.pose_new[t];
  if (t < g.nc * 12) g.Rt[t] = g.Rt_new[t];
  if (t < g.np * 3) g.pts[t] = g.pts_new[t];
}

__global__ void ba_finalize_kernel(int nc, const double* __restrict__ pose_cw, double* __restrict__ pose_wc) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nc) return;
  double in[7], out[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) in[k] = pose_cw[7 * i + k];
  se3_inverse(in, out);
#pragma unroll
  for (int k = 0; k < 7; ++k) pose_wc[7 * i + k] = out[k];
}


// ---- fused helpers of the short-launch-chain path -------------------------------------------------------------------------
// buf <- [S = blockdiag(U) | gt = gc | diagU | cost]; Vinv for every landmark.  Single writer per entry (no memset needed).
__global__ void __launch_bounds__(256) ba_prepare_schur_kernel(BaDev g, double* __restrict__ buf, int dense) {
  if (g.sc->stop) return;
  __shared__ double s_part[256 / 32 + 1];
  const size_t n6 = g.n6, nS = n6 * n6;
  const size_t stride = (size_t)gridDim.x * blockDim.x, t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  // (the block-gather path writes S, g~ and diag U itself: ba_schur_blocks_kernel)
  for (size_t idx = t0; dense && idx < nS; idx += stride) {
    const int row = (int)(idx / n6), col = (int)(idx % n6);
    const int i = row / 6, i2 = col / 6;
    buf[idx] = (i == i2) ? g.U[36 * i + (row % 6) * 6 + (col % 6)] : 0.0;
  }
  for (size_t d = t0; dense && d < n6; d += stride) {
    buf[g.r_gt + d] = g.gc[d];
    buf[g.r_gt + n6 + d] = g.U[36 * (d / 6) + (d % 6) * 7];
  }
  const double lambda = g.sc->lambda;
  const bool fresh = g.sc->need_linearize != 0 && g.vinv_in_sweep != 0;  // the sweep of this iteration already produced Vinv with this lambda
  for (size_t j = t0; !fresh && j < (size_t)g.np; j += stride)
    damped_vinv(g.V + 9 * j, g.pfree[j] != 0 && g.pt_off[j + 1] > g.pt_off[j], lambda, g.Vinv + 9 * j);
  // deterministic cost reduction over the whole grid (every block adds a slice, the last one folds the partials in block order)
  __shared__ int s_flag;
  grid_sum_to<256>(g.cost_pt, g.np + g.npe, 0.5, g.red_part, g.red_ticket, buf + g.r_gt + 2 * n6, s_part, &s_flag);
}

// Back-substitution of landmark j followed by its robustified cost at the candidate estimate -> pts_new[j], cost_pt_new[j].  kLpp
// lanes per landmark: lane `sub` takes observations e0 + sub, e0 + sub + kLpp, ... of the landmark's segment [e0, e1); i_first is the
// camera of its first one (o_cam[e0 + sub]), which the caller may request early.
__device__ __forceinline__ void ba_backsub_cost(const BaDev& g, int j, bool valid, int sub, int e0, int e1, int i_first, double delta) {
  double b[3] = {0.0, 0.0, 0.0};
  for (int e = e0 + sub; e < e1; e += kLpp) {
    const int i = (e == e0 + sub) ? i_first : g.o_cam[e];
    const double* W = g.W + 18 * (size_t)e;
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
      for (int a = 0; a < 6; ++a) b[c] -= W[a * 3 + c] * g.x[6 * i + a];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
#pragma unroll
    for (int o = kLpp / 2; o > 0; o >>= 1) b[c] += __shfl_xor_sync(0xffffffffu, b[c], o, kLpp);
    b[c] += g.gp[3 * (size_t)j + c];
  }
  const double* Vi = g.Vinv + 9 * (size_t)j;
  double p[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) p[a] = g.pts[3 * (size_t)j + a] + Vi[a * 3] * b[0] + Vi[a * 3 + 1] * b[1] + Vi[a * 3 + 2] * b[2];
  double cost = 0.0;
  for (int e = e0 + sub; e < e1; e += kLpp) {
    const int i = (e == e0 + sub) ? i_first : g.o_cam[e];
    const ObsLin o = eval_obs(g.Rt_new + 12 * i, p, g.o_uv[2 * e], g.o_uv[2 * e + 1], g.has_info ? g.o_info + 3 * e : nullptr, delta);
    cost += o.rho;
  }
#pragma unroll
  for (int o = kLpp / 2; o > 0; o >>= 1) cost += __shfl_xor_sync(0xffffffffu, cost, o, kLpp);
  if (valid && sub == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) g.pts_new[3 * (size_t)j + a] = p[a];
    g.cost_pt_new[j] = cost;
  }
}

__global__ void __launch_bounds__(128) ba_backsub_cost_kernel(BaDev g) {
  if (g.sc->stop) return;
  const int gt = blockIdx.x * blockDim.x + threadIdx.x;
  const int jraw = gt / kLpp, sub = gt % kLpp;
  const bool valid = jraw < g.np;
  const int j = valid ? jraw : 0;
  const double delta = g.sc->delta;
  const int e0 = g.pt_off[j], e1 = valid ? g.pt_off[j + 1] : e0;
  ba_backsub_cost(g, j, valid, sub, e0, e1, (e0 + sub < e1) ? g.o_cam[e0 + sub] : 0, delta);
}

// Local-BA tail in ONE launch: back-substitution + candidate cost (8 lanes per landmark), then the LAST CTA to finish
// (atomic ticket) reduces both costs in a fixed order, takes the LM accept/reject decision, and either installs the candidate
// (accept) or refreshes the damped V^-1 with the new lambda (reject: the next iteration skips the sweep).  Replaces
// ba_prepare_schur + ba_backsub_cost + ba_reduce_cost + ba_commit_apply of the stepwise path.
constexpr int kTailThreads = 256;
// CTA-wide copy of n doubles (16-byte accesses; both pointers are slab-aligned)
__device__ __forceinline__ void cta_copy_f64(double* __restrict__ dst, const double* __restrict__ src, int n, int nthreads) {
  const int n2 = n >> 1;
  for (int t = threadIdx.x; t < n2; t += nthreads) reinterpret_cast<double2*>(dst)[t] = __ldcg(reinterpret_cast<const double2*>(src) + t);
  if ((n & 1) && threadIdx.x == 0) dst[n - 1] = __ldcg(src + n - 1);
}

__global__ void __launch_bounds__(kTailThreads) ba_backsub_commit_kernel(BaDev g, const double* __restrict__ buf) {
  gb_pdl_launch_dependents();
  BaScalars* sc = g.sc;
  __shared__ double s_part[kTailThreads / 32 + 1];
  __shared__ int s_flag;
  // static graph structure of this lane's first observation, requested before waiting for the PCG kernel
  const int gt = blockIdx.x * blockDim.x + threadIdx.x;
  const int jraw = gt / kLpp, sub = gt % kLpp;
  const bool valid = jraw < g.np;
  const int j = valid ? jraw : 0;
  const int e0 = g.pt_off[j], e1 = valid ? g.pt_off[j + 1] : e0;
  const int i_first = (e0 + sub < e1) ? g.o_cam[e0 + sub] : 0;
  gb_pdl_wait();
  if (sc->stop) return;
  ba_backsub_cost(g, j, valid, sub, e0, e1, i_first, sc->delta);
  // ---- the last CTA done: both costs, the LM decision, install or V^-1 refresh
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_flag = (atomicAdd(&sc->ticket, 1u) == gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (!s_flag) return;
  __threadfence();
  double v0 = 0.0, v1 = 0.0;
  for (int k = threadIdx.x; k < g.np; k += kTailThreads) {
    v0 += __ldcg(&g.cost_pt[k]);
    v1 += __ldcg(&g.cost_pt_new[k]);
  }
  const double cost = 0.5 * block_sum<kTailThreads>(v0, s_part);
  const double cnew = 0.5 * block_sum<kTailThreads>(v1, s_part);
  if (threadIdx.x == 0) {
    sc->ticket = 0;
    s_flag = lm_decide(sc, cost, cnew) ? 2 : 1;
  }
  __syncthreads();
  if (s_flag == 2) {  // accept: the next sweep reads the candidate arrays and installs them on the fly (no serial copy here)
    if (threadIdx.x == 0) sc->pending = 1;
  } else {  // reject: same linearisation, new lambda -> refresh the damped landmark inverses
    const double lambda = sc->lambda;
    for (int j = threadIdx.x; j < g.np; j += kTailThreads)
      damped_vinv(g.V + 9 * (size_t)j, g.pfree[j] != 0 && g.pt_off[j + 1] > g.pt_off[j], lambda, g.Vinv + 9 * (size_t)j);
  }
}

// end of a solve on the local path: install an accepted candidate the next sweep never came to pick up (single CTA: the flag is
// read by everybody before it is cleared)
__global__ void __launch_bounds__(1024) ba_install_pending_kernel(BaDev g) {
  gb_pdl_wait();
  __shared__ int s_p;
  if (threadIdx.x == 0) s_p = g.sc->pending;
  __syncthreads();
  if (!s_p) return;
  cta_copy_f64(g.pts, g.pts_new, g.np * 3, 1024);
  cta_copy_f64(g.Rt, g.Rt_new, g.nc * 12, 1024);
  cta_copy_f64(g.pose, g.pose_new, g.nc * 7, 1024);
  if (threadIdx.x == 0) g.sc->pending = 0;
}

// ---- K7b (local BA, sparse covisibility): block-Jacobi PCG in ONE CTA -------------------------------------------------------
// When the structurally non-zero 6x6 blocks of the reduced camera matrix fit one SM (sequential-SLAM windows: a band of
// co-visible keyframes) the whole solve needs no inter-CTA exchange.  What bounds an iteration on one SM is ISSUE, not memory:
// fp64 runs at 64 lanes/clk/SM (a warp DFMA every 2 clk per sub-partition, a DDIV ~10 clk of the SM's pipe), SHFL at one
// warp-instruction/clk/SM (tools/mb/microbench2.cu) -- so the kernel does nothing redundantly:
//  * EIGHT lanes per ACTIVE camera (fixed keyframes have identity rows and a zero right-hand side: they get no lanes).  A block
//    row of S (nb blocks = 6*nb columns) is split BY COLUMN over the eight lanes: lane l keeps columns l, l+8, ... (six
//    coefficients each) in registers for the whole solve, so a mat-vec is one shared-memory read of u and six DFMAs per column
//    (no lane repeats another's work) followed by a 3-stage transposing butterfly (6 exchanges) that leaves row r of the camera
//    in lane {0,1,2,-,3,4,5,-}[l] (lanes 3 and 7 duplicate rows 2 and 5).  Those lanes own element 6i+r of every CG vector;
//    u = Minv r exchanges the camera's six residuals through a warp-local shared-memory tile (a camera never straddles
//    warps: __syncwarp, no CTA barrier).
//  * (gamma, delta) are reduced packed into ONE butterfly per warp (a in lanes 0-15, b in lanes 16-31); EVERY warp then folds
//    the per-warp partials in warp order and runs the alpha/beta recurrences (one reciprocal) itself: identical operations on
//    identical operands, so every thread holds the same bits and takes the same stop decision without a broadcast.
//  * <= 48 active cameras run as 12 warps = 3 per sub-partition -> 168 registers per thread, enough for 7 columns per lane
//    (block rows of <= 9 blocks) without spilling; the wide variant (<= 80 cameras) keeps 5 columns.  Only graphs with a block
//    row longer than the register columns (LONG_ROWS, chosen on the host) read the rest from the shared-memory copy of S.
// An iteration = [partials | scalars, element-wise recurrences, u = Minv r | u published | register mat-vec], two barriers.
template <int THREADS, int KC, bool LONG_ROWS>
__global__ void __launch_bounds__(THREADS, 1) ba_pcg_sparse_kernel(BaDev g, double* __restrict__ buf, int maxit) {
  gb_pdl_launch_dependents();
  extern __shared__ __align__(16) double sm[];
  __shared__ double2 s_red[32];  // per-warp (gamma, delta) partials
  __shared__ int s_nact;
  constexpr int NW = THREADS / 32;
  static_assert(NW <= 32, "the fold handles at most 32 per-warp partials");
  const int n6 = g.n6, nc = g.nc, nnzb = g.s_nnzb, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long t_start = clock64();
  double* B = sm;                          // [nnzb][36] row-major blocks
  double* Minv = B + (size_t)nnzb * 36;    // [nc][36]
  double* vu = Minv + (size_t)nc * 36;     // u (mat-vec input), n6
  double* vx = vu + n6;                    // x (for the retraction), n6
  double* vr = vx + n6;                    // r (warp-local exchange for u = Minv r), n6
  int* rowptr = reinterpret_cast<int*>(vr + n6);  // [nc+1]
  int* col = rowptr + nc + 1;                     // [nnzb]
  int* act = col + nnzb;                          // [nc] active (not fully fixed) cameras, ascending
  const size_t nS = (size_t)n6 * n6;
  // static graph structure first: under a programmatic dependent launch this part overlaps the Schur kernel
  for (int k = tid; k <= nc; k += THREADS) rowptr[k] = g.s_rowptr[k];
  for (int k = tid; k < nnzb; k += THREADS) col[k] = g.s_col[k];
  for (int k = tid; k < n6; k += THREADS) { vu[k] = 0.0; vx[k] = 0.0; }
  if (warp == NW - 1) {  // stream compaction of the active cameras (ballot scan)
    int cnt = 0;
    for (int base = 0; base < nc; base += 32) {
      const int i = base + lane;
      const bool f = i < nc && g.dof[i] != 0;
      const unsigned m = __ballot_sync(0xffffffffu, f);
      if (f) act[cnt + __popc(m & ((1u << lane) - 1u))] = i;
      cnt += __popc(m);
    }
    if (lane == 0) s_nact = cnt;
  }
  gb_pdl_wait();
  if (g.sc->stop) return;
  const double lambda = g.sc->lambda, tol = g.sc->pcg_tol;
  // A. copy the block-CSR values of S (written by ba_schur_blocks_kernel) into shared memory (8 independent loads in
  //    flight per thread), then Marquardt damping on the 6N diagonal entries (written back so the damped system is observable)
  {
    const int n = nnzb * 36;
    int w = tid;
    for (; w + 7 * THREADS < n; w += 8 * THREADS) {
      double v[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = g.Sb[w + k * THREADS];
#pragma unroll
      for (int k = 0; k < 8; ++k) B[w + k * THREADS] = v[k];
    }
    for (; w < n; w += THREADS) B[w] = g.Sb[w];
  }
  __syncthreads();
  for (int d = tid; d < n6; d += THREADS) {
    const int i = d / 6, a = d - 6 * i;
    int dblk = rowptr[i];
    while (col[dblk] != i) ++dblk;  // the diagonal block is always present
    const int w = dblk * 36 + a * 7;
    const double v = lm_damp(B[w], buf[nS + n6 + d], lambda, (g.dof[i] >> a) & 1);
    B[w] = v;
    g.Sb[w] = v;
  }
  __syncthreads();
  // B. block-Jacobi preconditioner
  for (int i = tid; i < nc; i += THREADS) {
    int dblk = rowptr[i];
    while (col[dblk] != i) ++dblk;  // the diagonal block is always present
    double M[36];
#pragma unroll
    for (int k = 0; k < 36; ++k) M[k] = B[(size_t)dblk * 36 + k];
    block_jacobi_inverse(M, B + (size_t)dblk * 36, 6);
#pragma unroll
    for (int k = 0; k < 36; ++k) Minv[36 * i + k] = M[k];
  }
  __syncthreads();  // Minv complete
  // ---- thread roles
  const int l8 = tid & 7;
  const bool cam_ok = (tid >> 3) < s_nact;
  const int ci = cam_ok ? act[tid >> 3] : 0;
  const int row = (l8 >> 2) * 3 + ((l8 & 3) < 2 ? (l8 & 3) : 2);  // which row of the camera this lane ends up with
  const bool own = cam_ok && (l8 & 3) != 3;                       // lanes 3 / 7 duplicate rows 2 / 5
  const int d = 6 * ci + row;
  const int b0 = cam_ok ? rowptr[ci] : 0, b1 = cam_ok ? rowptr[ci + 1] : 0;
  const int ncols = 6 * (b1 - b0);
  // The mat-vec accumulates the camera's rows in a per-lane slot order chosen so that every butterfly exchange below sends and
  // keeps FIXED slots (no selects in the loop): slots 0-2 hold the half this lane keeps after the first exchange, slots 3-5
  // the same positions of the other half, and within a half lane {x0, x1, x2, x3} orders its rows {012, 102, 210, 201}.
  const bool hi = (l8 & 4) != 0, mid = (l8 & 2) != 0, odd = (l8 & 1) != 0;
  auto to_slots = [&](const double (&n)[6], double (&m)[6]) {  // one column, rows 0-5 -> slots 0-5
    const double k0 = hi ? n[3] : n[0], k1 = hi ? n[4] : n[1], k2 = hi ? n[5] : n[2];  // the half this lane keeps
    const double s0 = hi ? n[0] : n[3], s1 = hi ? n[1] : n[4], s2 = hi ? n[2] : n[5];  // the half it sends
    m[0] = mid ? k2 : (odd ? k1 : k0); m[1] = odd ? k0 : k1; m[2] = mid ? (odd ? k1 : k0) : k2;
    m[3] = mid ? s2 : (odd ? s1 : s0); m[4] = odd ? s0 : s1; m[5] = mid ? (odd ? s1 : s0) : s2;
  };
  // this lane's columns of the block row: coefficients in registers (absent columns: zeros, reading the camera's own u)
  double cf[KC][6];
  int pidx[KC];
#pragma unroll
  for (int k = 0; k < KC; ++k) {
    const int c = l8 + 8 * k;
    const bool ok = c < ncols;
    const int sblk = ok ? b0 + c / 6 : 0, a = ok ? c % 6 : 0;
    pidx[k] = ok ? 6 * col[sblk] + a : 6 * ci;
    double n[6];
#pragma unroll
    for (int r = 0; r < 6; ++r) n[r] = ok ? B[(size_t)sblk * 36 + r * 6 + a] : 0.0;
    to_slots(n, cf[k]);
  }
  double mrow[6];  // this lane's row of the camera's Minv block (constant over the solve)
#pragma unroll
  for (int b = 0; b < 6; ++b) mrow[b] = cam_ok ? Minv[36 * ci + row * 6 + b] : 0.0;
  // w_d = row d of S times u
  auto matvec = [&]() -> double {
    double pv[KC];
#pragma unroll
    for (int k = 0; k < KC; ++k) pv[k] = vu[pidx[k]];
    double y[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int k = 0; k < KC; ++k)
#pragma unroll
      for (int s = 0; s < 6; ++s) y[s] += cf[k][s] * pv[k];
    if constexpr (LONG_ROWS) {
      for (int c = l8 + 8 * KC; c < ncols; c += 8) {  // block rows longer than the register cache: shared-memory copy
        const int sblk = b0 + c / 6, a = c % 6;
        const double pc = vu[6 * col[sblk] + a];
        const double* Bc = B + (size_t)sblk * 36 + a;
        double n[6], m[6];
#pragma unroll
        for (int r = 0; r < 6; ++r) n[r] = Bc[r * 6];
        to_slots(n, m);
#pragma unroll
        for (int s = 0; s < 6; ++s) y[s] += m[s] * pc;
      }
    }
    // transposing butterfly over the 8 lanes of the camera: rows {0,1,2} go to lanes 0-3, rows {3,4,5} to lanes 4-7 ...
    double v[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) v[j] = y[j] + __shfl_xor_sync(0xffffffffu, y[3 + j], 4);
    // ... then rows {0,1} of the half to lanes x0/x1 (t0 = x0's row 0, x1's row 1; t1 = the other) and row 2 to lanes x2/x3 ...
    const double t0 = v[0] + __shfl_xor_sync(0xffffffffu, v[2], 2);
    const double t1 = v[1] + __shfl_xor_sync(0xffffffffu, v[1], 2);  // (meaningful in the !mid lanes only)
    // ... and the last exchange finishes the sums (the two `mid` lanes of a half both end with the third row)
    return t0 + __shfl_xor_sync(0xffffffffu, mid ? t0 : t1, 1);
  };
  // per-warp part of the fused deterministic reduction: lanes 0-15 fold a, lanes 16-31 fold b (ONE butterfly for both)
  auto warp_partials = [&](double a, double b) {
    const bool up = (lane & 16) != 0;
    double v = (up ? b : a) + __shfl_xor_sync(0xffffffffu, up ? a : b, 16);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s_red[warp].x = v;
    if (lane == 16) s_red[warp].y = v;
  };
  // u_d = (Minv r)_d: the camera's six residual entries are exchanged through shared memory INSIDE the warp (a camera never
  // straddles warps): 2 + 3 shared-memory wavefronts instead of 12 SHFLs
  auto precond = [&](double rd) -> double {
    if (own) vr[d] = rd;
    __syncwarp();
    const double2* rc = reinterpret_cast<const double2*>(vr + 6 * ci);
    const double2 q01 = rc[0], q23 = rc[1], q45 = rc[2];
    return ((mrow[0] * q01.x + mrow[1] * q01.y) + (mrow[2] * q23.x + mrow[3] * q23.y)) + (mrow[4] * q45.x + mrow[5] * q45.y);
  };
  // clock64 stamps of thread 0 (test hook gb_dbg_ba_pcg_profile): [7] setup cycles, then of iteration 3 [0] start, [1] scalars
  // done, [2] u = Minv r stored, [3] after barrier (2) and the mat-vec, [4] partials stored; [6] the loop's end
#define SP_STAMP(k) do { if (g.prof && tid == 0 && it == 3) g.prof[k] = clock64(); } while (0)
  if (g.prof && tid == 0) g.prof[7] = clock64() - t_start;
  // ---- Chronopoulos-Gear PCG (same recurrence as oracle/ba_ref.c::ba_pcg) ----
  double xd = 0.0, pd = 0.0, sd = 0.0, rd = 0.0, ud, wd;
  if (cam_ok) rd = buf[nS + d];
  ud = precond(rd);
  if (own) vu[d] = ud;
  __syncthreads();  // u published
  wd = matvec();
  warp_partials(own ? rd * ud : 0.0, own ? wd * ud : 0.0);
  // scalar recurrences: every thread runs them (same bits everywhere)
  const double tol2 = tol * tol;
  double gamma0 = 0.0, alpha_s = 0.0, beta_s = 0.0, inv_alpha = 0.0, inv_gamma = 0.0;
  int iters = 0;
  // Two barriers per iteration suffice.  s_red: a warp writes its partials of round `it` after barrier (2) of iteration it-1 and
  // every warp reads them after barrier (1) of iteration `it`; the next write comes after barrier (2) of iteration `it`, which no
  // warp passes before it has finished its fold.  vu: written before barrier (2), read by the mat-vec after it; the next write
  // comes after barrier (1) of the following iteration, which no warp passes before its mat-vec is done.  vr is warp-local
  // (__syncwarp inside precond) and is rewritten only after both barriers.
  for (int it = 0;; ++it) {
    SP_STAMP(0);
    __syncthreads();  // (1) the partials of round `it` are in s_red (round 0: the initial gamma, delta; round k: iteration k-1)
    double gn = 0.0, dl = 0.0;  // fixed-order fold of the per-warp partials (broadcast loads, two independent chains)
#pragma unroll
    for (int w = 0; w < NW; ++w) { const double2 t = s_red[w]; gn += t.x; dl += t.y; }
    // alpha = gn/den, 1/alpha = den/gn and 1/gn from ONE reciprocal: t = 1/(gn*den) (a DDIV is ~113 clk and three of them do
    // not overlap); the guarded fallback covers products outside the double range
    auto scalars = [&](double den) {
      const double t = __drcp_rn(gn * den);
      if (t > 0.0 && t < 1.0e300) {
        const double inv_gn = den * t, inv_den = gn * t;
        alpha_s = gn * inv_den; inv_alpha = den * inv_gn; inv_gamma = inv_gn;
      } else {
        alpha_s = gn / den; inv_alpha = den / gn; inv_gamma = 1.0 / gn;
      }
    };
    bool stop;
    if (it == 0) {
      gamma0 = gn;
      stop = !(gamma0 > 0.0) || !(dl > 0.0) || maxit <= 0;
      if (!stop) scalars(dl);
    } else {
      iters = it;
      stop = !(gn > 0.0) || gn < tol2 * gamma0;
      if (!stop) {
        // beta = gn/gamma, alpha = gn/(dl - beta*gn/alpha_prev) with the reciprocals of gamma and alpha carried along
        beta_s = gn * inv_gamma;
        const double den = dl - beta_s * (gn * inv_alpha);
        stop = !(den > 0.0);
        if (!stop) scalars(den);
      }
      stop = stop || it >= maxit;
    }
    SP_STAMP(1);
    if (stop) break;
    // element-wise recurrences, registers only (duplicate lanes compute duplicates)
    pd = ud + beta_s * pd;
    sd = wd + beta_s * sd;
    xd += alpha_s * pd;
    rd -= alpha_s * sd;
    ud = precond(rd);
    if (own) vu[d] = ud;
    SP_STAMP(2);
    __syncthreads();  // (2) u published
    wd = matvec();
    SP_STAMP(3);
    warp_partials(own ? rd * ud : 0.0, own ? wd * ud : 0.0);
    SP_STAMP(4);
  }
  if (g.prof && tid == 0) g.prof[6] = clock64();
  // publish the solution, the iteration count and the candidate camera poses
  if (own) vx[d] = xd;
  if (tid == 0) g.sc->pcg_iters += iters;
  __syncthreads();
  for (int k = tid; k < n6; k += THREADS) g.x[k] = vx[k];
  for (int i = tid; i < nc; i += THREADS) retract_camera(g, i, vx + 6 * i);
}
constexpr int kSpSmallCams = 48;     // active cameras of the 12-warp variant (168 registers, 7 register columns per lane)
constexpr int kSpMaxCams = 80;       // active cameras of the 20-warp variant (96 registers, 5 register columns per lane)
constexpr int kSpSmallCols = 7, kSpLargeCols = 5;
constexpr int kSpSmallThreads = 8 * kSpSmallCams, kSpLargeThreads = 8 * kSpMaxCams;
#define BA_SPARSE_SMALL(long_rows) ba_pcg_sparse_kernel<kSpSmallThreads, kSpSmallCols, long_rows>
#define BA_SPARSE_LARGE(long_rows) ba_pcg_sparse_kernel<kSpLargeThreads, kSpLargeCols, long_rows>

// ---- K7b (local BA): block-Jacobi PCG inside ONE thread-block cluster ------------------------------------------------------
// Each CTA of the cluster keeps a block-row slice of the (damped) reduced camera matrix S resident in its shared memory for the
// whole solve; per iteration it computes its rows of q = S p, scatters them into every CTA's shared memory through DSMEM, and
// after ONE cluster barrier every CTA redundantly (and bit-identically) performs the O(6N) vector part of CG.  q is
// double-buffered so a fast CTA can never overwrite data a slow one still reads.  No global-memory traffic inside the loop.
constexpr int kPcgThreads = 512;

__global__ void __launch_bounds__(kPcgThreads, 1) ba_pcg_cluster_kernel(BaDev g, double* __restrict__ buf, int maxit) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  if (g.sc->stop) return;  // uniform over the cluster
  extern __shared__ __align__(16) double sm[];
  const int C = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int n6 = g.n6, nc = g.nc, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cpc = (nc + C - 1) / C;
  const int c0 = min(rank * cpc, nc), c1 = min(c0 + cpc, nc);
  const int r0 = 6 * c0, nrows = 6 * (c1 - c0);
  double* S = sm;                          // [6*cpc][n6]
  double* Minv = S + (size_t)6 * cpc * n6; // [nc*36]
  double* qbuf = Minv + (size_t)nc * 36;   // [2][n6]
  double* vp = qbuf + 2 * (size_t)n6;      // p, r, z, x : [n6] each
  double* vr = vp + n6;
  double* vz = vr + n6;
  double* vx = vz + n6;
  const size_t nS = (size_t)n6 * n6;
  const double lambda = g.sc->lambda, tol = g.sc->pcg_tol;
  // A. slice of S -> shared memory, Marquardt damping on the diagonal (written back so the damped system is observable)
  for (int idx = tid; idx < nrows * n6; idx += kPcgThreads) {
    const int row = idx / n6, col = idx - row * n6, d = r0 + row;
    double v = buf[(size_t)d * n6 + col];
    if (col == d) {
      v = lm_damp(v, buf[nS + n6 + d], lambda, (g.dof[d / 6] >> (d % 6)) & 1);
      buf[(size_t)d * n6 + col] = v;
    }
    S[idx] = v;
  }
  __syncthreads();
  // B. block-Jacobi preconditioner: owners invert their 6x6 diagonal blocks, everyone gathers all of them
  if (tid < c1 - c0) {
    double M[36];
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int b = 0; b < 6; ++b) M[a * 6 + b] = S[(size_t)(6 * tid + a) * n6 + r0 + 6 * tid + b];
    block_jacobi_inverse(M, S + (size_t)(6 * tid) * n6 + r0 + 6 * tid, n6);
#pragma unroll
    for (int k = 0; k < 36; ++k) g.Minv[36 * (size_t)(c0 + tid) + k] = M[k];
  }
  __threadfence();
  cluster.sync();
  for (int k = tid; k < nc * 36; k += kPcgThreads) Minv[k] = __ldcg(&g.Minv[k]);
  for (int d = tid; d < n6; d += kPcgThreads) {
    vx[d] = 0.0;
    vr[d] = buf[nS + d];
  }
  __syncthreads();
  // From here on thread d < n6 owns vector element d (n6 <= kPcgThreads is guaranteed by the host-side dispatch).
  // Chronopoulos-Gear PCG (same recurrence as oracle/ba_ref.c::ba_pcg): vectors u (vp), s and r double-buffered, w arrives
  // from all CTAs through distributed shared memory into qbuf[parity].
  const bool own = tid < n6;
  const int ci = own ? tid / 6 : 0, ca = own ? tid - 6 * ci : 0;
  __shared__ double s_red[2][2 * (kPcgThreads / 32)];
  double* vu = vp;
  double* vs[2] = {vz, vx};                 // (vx is free: x lives in registers)
  double* vrr[2] = {vr, qbuf + 2 * (size_t)n6 + 4 * (size_t)n6};  // second r buffer sits after the four n6 vectors
  auto reduce2 = [&](double a, double b, int bufi, double* oa, double* ob) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_down_sync(0xffffffffu, a, o);
      b += __shfl_down_sync(0xffffffffu, b, o);
    }
    if (lane == 0) { s_red[bufi][2 * warp] = a; s_red[bufi][2 * warp + 1] = b; }
    __syncthreads();
    double pa[kPcgThreads / 32], pb[kPcgThreads / 32];
#pragma unroll
    for (int w = 0; w < kPcgThreads / 32; ++w) { pa[w] = s_red[bufi][2 * w]; pb[w] = s_red[bufi][2 * w + 1]; }
#pragma unroll
    for (int st = 1; st < kPcgThreads / 32; st <<= 1) {
#pragma unroll
      for (int w = 0; w + st < kPcgThreads / 32; w += 2 * st) { pa[w] += pa[w + st]; pb[w] += pb[w + st]; }
    }
    *oa = pa[0]; *ob = pb[0];
  };
  const int hl = tid & 15, grp = tid >> 4;  // 16 lanes per matrix row
  // rows of this CTA of w = S u, scattered into every CTA's wbuf through DSMEM
  auto matvec_scatter = [&](double* wbuf) {
    for (int row = grp; row < nrows; row += kPcgThreads / 16) {
      const double* Srow = S + (size_t)row * n6;
      double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
      int c = hl;
      for (; c + 48 < n6; c += 64) {
        s0 += Srow[c] * vu[c];
        s1 += Srow[c + 16] * vu[c + 16];
        s2 += Srow[c + 32] * vu[c + 32];
        s3 += Srow[c + 48] * vu[c + 48];
      }
      for (; c < n6; c += 16) s0 += Srow[c] * vu[c];
      double sv = (s0 + s1) + (s2 + s3);
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) sv += __shfl_xor_sync(0xffffffffu, sv, o, 16);  // a+b == b+a: all 16 lanes agree
      if (hl < C) cluster.map_shared_rank(wbuf, hl)[r0 + row] = sv;
    }
  };
  double xd = 0.0, pd = 0.0, sd = 0.0, rd = 0.0, ud = 0.0, wd = 0.0;
  if (own) {
    rd = vr[tid];
#pragma unroll
    for (int b = 0; b < 6; ++b) ud += Minv[36 * ci + ca * 6 + b] * vr[6 * ci + b];
    vs[0][tid] = 0.0;
  }
  __syncthreads();  // all reads of vr (as g~) done before anyone could overwrite; vu written next
  if (own) vu[tid] = ud;
  __syncthreads();
  matvec_scatter(qbuf);
  cluster.sync();
  if (own) wd = qbuf[tid];
  double gamma, delta;
  reduce2(rd * ud, wd * ud, 0, &gamma, &delta);
  const double gamma0 = gamma, tol2 = tol * tol;
  int iters = 0;
  double alpha = 0.0, beta = 0.0;
  bool done = !(gamma0 > 0.0) || !(delta > 0.0);
  if (!done) alpha = gamma / delta;
#define PCG_STAMP(k) do { if (g.prof && rank == 0 && tid == 0 && it == 3) g.prof[k] = clock64(); } while (0)
  for (int it = 0; it < maxit && !done; ++it) {
    PCG_STAMP(0);
    const int cur = it & 1, nxt = cur ^ 1;
    const double* wcur = qbuf + (size_t)cur * n6;  // w of the current u (iteration parity)
    double* wnxt = qbuf + (size_t)nxt * n6;
    if (own) {
      pd = ud + beta * pd;
      sd = wd + beta * sd;
      xd += alpha * pd;
      ud = 0.0;
#pragma unroll
      for (int b = 0; b < 6; ++b) {
        const double sb = wcur[6 * ci + b] + beta * vs[cur][6 * ci + b];
        const double rb = vrr[cur][6 * ci + b] - alpha * sb;
        if (b == ca) rd = rb;
        ud += Minv[36 * ci + ca * 6 + b] * rb;
      }
      vs[nxt][tid] = sd;
      vrr[nxt][tid] = rd;
      vu[tid] = ud;
    }
    __syncthreads();  // u (and s, r) published inside the CTA
    PCG_STAMP(1);
    matvec_scatter(wnxt);
    PCG_STAMP(2);
    cluster.sync();   // w of every CTA has landed in everybody's wnxt
    PCG_STAMP(3);
    if (own) wd = wnxt[tid];
    double gn, dl;
    reduce2(rd * ud, wd * ud, (it + 1) & 1, &gn, &dl);
    PCG_STAMP(4);
    ++iters;
    if (!(gn > 0.0) || gn < tol2 * gamma0) break;
    beta = gn / gamma;
    const double den = dl - beta * gn / alpha;
    if (!(den > 0.0)) break;
    alpha = gn / den;
    gamma = gn;
    PCG_STAMP(5);
  }
  __syncthreads();
  if (own) vx[tid] = xd;
  __syncthreads();
  // every CTA leaves the loop at the same iteration (bit-identical redundant arithmetic); make sure nobody exits while a
  // peer could still be storing into its shared memory
  cluster.sync();
  if (rank != 0) return;
  // D. CTA 0 publishes the solution, the iteration count and the candidate camera poses
  for (int d = tid; d < n6; d += kPcgThreads) g.x[d] = vx[d];
  if (tid == 0) g.sc->pcg_iters += iters;
  for (int i = tid; i < nc; i += kPcgThreads) retract_camera(g, i, vx + 6 * i);
}

}  // namespace

// ======================================================================================================================
// host side
// ======================================================================================================================

static size_t ba_buf_doubles(int nc) {
  const size_t n6 = 6 * (size_t)nc;
  return n6 * n6 + 2 * n6 + 8;
}

// a measurement's x and y are divided by its z (graph creation and the refresh of a cached graph)
static int ba_check_z(gb_ctx* ctx, const gb_ba_problem* pb, int k) {
  const double z = pb->obs_xyz[3 * (size_t)k + 2];
  if (!(z != 0.0) || !std::isfinite(z)) {
    gb_set_error(ctx, "gb_ba: edge %d has a zero/non-finite measurement z", k);
    return GB_ERR_INVALID;
  }
  return GB_OK;
}

// the measurements as the kernels read them: x/z, y/z in sorted edge order (uv) and in camera order (cuv), and the symmetrised 2x2
// information in sorted order (info, when the problem has it).  sorted_to_orig and cam_perm as in gb_ba_graph.
static void ba_fill_measurements(const gb_ba_problem* pb, const std::vector<int>& sorted_to_orig, const std::vector<int>& cam_perm, double* uv,
                                 double* cuv, double* info) {
  const size_t no = sorted_to_orig.size();
  for (size_t e = 0; e < no; ++e) {
    const int k = sorted_to_orig[e];
    const double* m = pb->obs_xyz + 3 * (size_t)k;
    uv[2 * e] = m[0] / m[2];
    uv[2 * e + 1] = m[1] / m[2];
    if (info) {
      const double* L = pb->obs_info + 4 * (size_t)k;
      info[3 * e] = L[0]; info[3 * e + 1] = 0.5 * (L[1] + L[2]); info[3 * e + 2] = L[3];
    }
  }
  for (size_t idx = 0; idx < no; ++idx) {
    const int e = cam_perm[idx];
    cuv[2 * idx] = uv[2 * e];
    cuv[2 * idx + 1] = uv[2 * e + 1];
  }
}

static int ba_validate(gb_ctx* ctx, const gb_ba_problem* pb) {
  if (!pb || pb->n_cams < 0 || pb->n_points < 0 || pb->n_obs < 0) {
    gb_set_error(ctx, "gb_ba: negative sizes");
    return GB_ERR_INVALID;
  }
  if ((pb->n_cams > 0 && !pb->cam_pose_wc) || (pb->n_points > 0 && !pb->points) ||
      (pb->n_obs > 0 && (!pb->obs_cam || !pb->obs_point || !pb->obs_xyz))) {
    gb_set_error(ctx, "gb_ba: null array");
    return GB_ERR_INVALID;
  }
  if (pb->n_cams > 20000) {
    gb_set_error(ctx, "gb_ba: %d cameras exceed the dense reduced-system limit (20000)", pb->n_cams);
    return GB_ERR_INVALID;
  }
  for (int k = 0; k < pb->n_obs; ++k) {
    if (pb->obs_cam[k] < 0 || pb->obs_cam[k] >= pb->n_cams || pb->obs_point[k] < 0 || pb->obs_point[k] >= pb->n_points) {
      gb_set_error(ctx, "gb_ba: edge %d references camera %d / point %d out of range", k, pb->obs_cam[k], pb->obs_point[k]);
      return GB_ERR_INVALID;
    }
    GB_CHECK(ba_check_z(ctx, pb, k));
  }
  return GB_OK;
}

// Can the reduced camera system be solved by the one-cluster PCG kernel?  Pick the cluster size (the largest of 16 and 8 that fits,
// at most max_cluster), remember the smem need.
static void ba_pick_pcg(gb_ctx* ctx, gb_ba_graph* g, int max_cluster = 16) {
  g->pcg_cluster = 0;
  g->pcg_sparse = false;
  const int nc = g->d.nc, n6 = g->d.n6;
  bool cluster16_ok = false;
  bool smem_ok = true;
  for (const void* f : {(const void*)BA_SPARSE_SMALL(false), (const void*)BA_SPARSE_SMALL(true), (const void*)BA_SPARSE_LARGE(false),
                        (const void*)BA_SPARSE_LARGE(true)})
    smem_ok = gb_func_setup(ctx, f, GB_SMEM_OPTIN_MAX) && smem_ok;
  smem_ok = gb_func_setup(ctx, (const void*)ba_pcg_cluster_kernel, GB_SMEM_OPTIN_MAX, &cluster16_ok) && smem_ok;
  if (nc > 0 && g->pcg_nact <= kSpMaxCams && g->d.s_nnzb > 0) {
    const size_t smem = ((size_t)g->d.s_nnzb * 36 + (size_t)nc * 36 + 3 * (size_t)n6) * sizeof(double) + (2 * (size_t)nc + 1 + g->d.s_nnzb) * sizeof(int) + 64;
    if (smem + 2048 <= (size_t)ctx->max_smem_optin && smem_ok) {
      g->pcg_sparse = true;
      g->pcg_sparse_smem = smem;
    }
  }
  if (nc <= 0 || n6 > kPcgThreads) return;  // the cluster kernel maps one thread per element of the 6N vectors
  const bool np_ok = smem_ok && cluster16_ok;
  const int sizes[2] = {16, 8};
  for (int t = 0; t < 2; ++t) {
    const int C = sizes[t];
    if ((C == 16 && !np_ok) || C > max_cluster) continue;
    const int cpc = (nc + C - 1) / C;
    const size_t smem = ((size_t)6 * cpc * n6 + (size_t)nc * 36 + 7 * (size_t)n6) * sizeof(double) + 64;
    if (smem + 2048 > (size_t)ctx->max_smem_optin || !smem_ok) continue;
    GbClusterConfig lc(C, dim3(kPcgThreads), smem, ctx->stream);
    int nclusters = 0;
    if (cudaOccupancyMaxActiveClusters(&nclusters, ba_pcg_cluster_kernel, &lc.cfg) != cudaSuccess || nclusters < 1) {
      cudaGetLastError();
      continue;
    }
    g->pcg_cluster = C;
    g->pcg_smem = smem;
    return;
  }
}


// GB_BA_TRACE=1: wall-clock stamps of the host-side phases of a host-buffer solve (stderr), for tools/e2e_breakdown.py
struct BaTrace {
  bool on;
  std::chrono::steady_clock::time_point t0;
  BaTrace() : on(getenv("GB_BA_TRACE") != nullptr), t0(std::chrono::steady_clock::now()) {}
  void stamp(const char* what) {
    if (!on) return;
    const auto t1 = std::chrono::steady_clock::now();
    fprintf(stderr, "[gb_ba trace] %-28s %8.1f us\n", what, std::chrono::duration<double, std::micro>(t1 - t0).count());
    t0 = t1;
  }
};

extern "C" {

void gb_ba_options_default(gb_ba_options* o) {
  if (!o) return;
  o->projection = 0;
  o->huber_delta = 0.01;    // OptimzeConfig::projectErrorHuberThreshold, Optimizer.h:177
  o->max_iterations = 500;  // OptimzeConfig::maxIterations, Optimizer.h:179
  o->verbose = 0;
  o->function_tolerance = 1e-6;
  o->lambda_init = 1e-4;
  o->pcg_max_iters = 50;
  o->pcg_tol = 1e-10;
  o->linear_solver = 0;
}

int gb_ba_graph_destroy(gb_ctx* ctx, gb_ba_graph* g) {
  if (!g) return GB_OK;
  if (ctx) {
    CtxLock lk(ctx);
    if (g->waiting) {  // another thread's solve of g is waiting on g's pinned scalars and events
      gb_set_error(ctx, "gb_ba_graph_destroy: a solve of this graph is still waiting for the device on another thread");
      return GB_ERR_INVALID;
    }
    if (g->slab) cudaStreamSynchronize(ctx->stream);
  }
  if (g->h_sc) cudaFreeHost(g->h_sc);
  for (cudaEvent_t ev : {g->ev_s, g->ev_e, g->ev_done})
    if (ev) cudaEventDestroy(ev);
  cudaFree(g->slab);
  delete g;
  return GB_OK;
}

int gb_ba_graph_create(gb_ctx* ctx, const gb_ba_problem* pb, gb_ba_graph** out) {
  return ba_graph_create_impl(ctx, pb, out, BaPlace::own, 0, 1);
}

// a BundleGraph with pose-graph terms (se3Graph / gpsGraph, Optimizer.h:163-168); `edges` may be NULL
int gb_ba_graph_create_ex(gb_ctx* ctx, const gb_ba_problem* pb, const gb_pose_edges* edges, gb_ba_graph** out) {
  return ba_graph_create_impl(ctx, pb, out, BaPlace::own, 0, 1, edges);
}

}  // extern "C"

// Landmark-chunk plan of the Schur complement (see ba_schur_chunks_kernel), host only: sets d.sp_nchunks and fills p.  Returns
// false when it does not apply (a landmark with more than 16 observers, no block structure): the block-gather kernel is used then.
static bool ba_schur_plan(gb_ctx* ctx, gb_ba_graph* g, int np, const std::vector<int>& pt_off, const std::vector<int>& scam, const uint8_t* pfree_host,
                          const std::vector<int>& s_rowptr, const std::vector<int>& s_col, const std::vector<int>& s_upper, BaSchurPlan& p) {
  BaDev& d = g->d;
  d.sp_nchunks = 0;
  if (np <= 0 || d.s_nnzb <= 0 || d.nc <= 0) return false;
  // landmarks in the order of the trajectory (first observing camera, then last, then id): consecutive landmarks then share
  // their cameras whatever order the caller numbered them in; fixed / unobserved landmarks contribute nothing and are left out
  std::vector<int>& ord = p.order;
  ord.reserve(np);
  for (int j = 0; j < np; ++j) {
    const int a = pt_off[j], b = pt_off[j + 1];
    if (b <= a || (pfree_host && !pfree_host[j])) continue;
    if (b - a > kChunkCams) return false;
    ord.push_back(j);
  }
  if (ord.empty()) return false;
  std::sort(ord.begin(), ord.end(), [&](int x, int y) {
    const int fx = scam[pt_off[x]], fy = scam[pt_off[y]];
    if (fx != fy) return fx < fy;
    const int lx = scam[pt_off[x + 1] - 1], ly = scam[pt_off[y + 1] - 1];
    if (lx != ly) return lx < ly;
    return x < y;
  });
  const int nl = (int)ord.size();
  const int lmax = std::min(kChunkMaxLm, std::max(8, nl / (4 * std::max(ctx->sm_count, 1))));
  std::vector<int> &ch_pt0 = p.pt0, ch_cams;  // ch_cams: 16 per chunk, ascending, -1 padded
  std::vector<unsigned short>& mask = p.mask;
  mask.assign((size_t)nl, 0);
  std::vector<int> cur, merged;  // sorted cameras of the open chunk
  int open_from = 0;
  auto close = [&](int upto) {
    ch_pt0.push_back(open_from);
    for (int k = 0; k < kChunkCams; ++k) ch_cams.push_back(k < (int)cur.size() ? cur[k] : -1);
    open_from = upto;
    cur.clear();
  };
  for (int t = 0; t < nl; ++t) {
    const int j = ord[t], a = pt_off[j], b = pt_off[j + 1];
    merged.clear();
    std::set_union(cur.begin(), cur.end(), scam.begin() + a, scam.begin() + b, std::back_inserter(merged));  // (edges are camera-sorted, no duplicates)
    // close when the camera set would overflow, the chunk is full, or -- so that most chunks keep ONE camera set and their slot
    // threads stay dense -- when the set would grow although the chunk already holds a fair number of landmarks
    // (12 cameras = 78 slots: one pass of the two-threads-per-slot kernel; only a landmark with 13..16 observers forces more)
    const int cam_cap = std::max(12, b - a);
    if ((int)merged.size() > std::min(kChunkCams, cam_cap) || t - open_from >= lmax || (merged.size() > cur.size() && !cur.empty() && t - open_from >= lmax / 4)) {
      close(t);
      merged.assign(scam.begin() + a, scam.begin() + b);
    }
    cur.swap(merged);
  }
  close(nl);
  ch_pt0.push_back(nl);
  const int nch = (int)ch_pt0.size() - 1;
  // masks + the slots each chunk really touches
  std::vector<std::vector<int>> blk_contrib(s_upper.size()), cam_contrib((size_t)d.nc);
  std::vector<int> upper_of((size_t)d.s_nnzb, -1);
  for (size_t u = 0; u < s_upper.size(); ++u) upper_of[s_upper[u]] = (int)u;
  std::vector<uint8_t> used(kChunkSlots), &slots = p.slots;
  std::vector<int>& nused = p.nused;
  slots.assign((size_t)nch * kChunkSlots, 0);
  nused.assign((size_t)nch, 0);
  for (int c = 0; c < nch; ++c) {
    const int* cams = &ch_cams[(size_t)c * kChunkCams];
    std::fill(used.begin(), used.end(), 0);
    for (int t = ch_pt0[c]; t < ch_pt0[c + 1]; ++t) {
      const int j = ord[t], a = pt_off[j], b = pt_off[j + 1];
      unsigned int m = 0;
      int l = 0;
      for (int e = a; e < b; ++e) {
        while (cams[l] != scam[e]) ++l;
        m |= 1u << l;
      }
      mask[t] = (unsigned short)m;
      for (int lb = 0; lb < kChunkCams; ++lb)
        if ((m >> lb) & 1)
          for (int la = 0; la <= lb; ++la)
            if ((m >> la) & 1) used[lb * (lb + 1) / 2 + la] = 1;
    }
    for (int lb = 0; lb < kChunkCams; ++lb)
      for (int la = 0; la <= lb; ++la) {
        if (!used[lb * (lb + 1) / 2 + la]) continue;
        const int i = cams[la], i2 = cams[lb];
        int t = s_rowptr[i];
        while (t < s_rowptr[i + 1] && s_col[t] != i2) ++t;
        if (t >= s_rowptr[i + 1]) return false;  // (cannot happen: the block structure covers every co-observed pair)
        blk_contrib[upper_of[t]].push_back(c * kChunkSlots + lb * (lb + 1) / 2 + la);
        if (la == lb) cam_contrib[i].push_back(c * kChunkCams + la);
        slots[(size_t)c * kChunkSlots + nused[c]++] = (uint8_t)(lb * (lb + 1) / 2 + la);
      }
  }
  std::vector<int> &boff = p.boff, &bidx = p.bidx, &coff = p.coff, &cidx = p.cidx;
  boff.assign(s_upper.size() + 1, 0);
  coff.assign((size_t)d.nc + 1, 0);
  for (size_t u = 0; u < s_upper.size(); ++u) { bidx.insert(bidx.end(), blk_contrib[u].begin(), blk_contrib[u].end()); boff[u + 1] = (int)bidx.size(); }
  for (int i = 0; i < d.nc; ++i) { cidx.insert(cidx.end(), cam_contrib[i].begin(), cam_contrib[i].end()); coff[i + 1] = (int)cidx.size(); }
  d.sp_nchunks = nch;
  return true;
}

// first landmark of rank r's shard: the first landmark whose edge prefix count reaches r/world of the edges (monotone in r)
static int ba_shard_bound(const std::vector<int>& pt_off, int n_obs, int n_points, int r, int world) {
  if (r <= 0) return 0;
  if (r >= world) return n_points;
  const double target = (double)n_obs * (double)r / (double)world;
  const int b = (int)(std::lower_bound(pt_off.begin(), pt_off.end(), target, [](int a, double t) { return (double)a < t; }) - pt_off.begin());
  return std::min(b, n_points);
}

// host-only test hook: the shard boundaries (world+1 entries) ba_graph_create_impl would use -- no device needed
extern "C" GB_API int gb_dbg_ba_shard_bounds(int n_points, int n_obs, const int32_t* obs_point, int world, int32_t* bounds) {
  if (n_points < 0 || n_obs < 0 || world < 1 || !bounds || (n_obs > 0 && !obs_point)) return GB_ERR_INVALID;
  std::vector<int> pt_off(n_points + 1, 0);
  for (int k = 0; k < n_obs; ++k) {
    if (obs_point[k] < 0 || obs_point[k] >= n_points) return GB_ERR_INVALID;
    pt_off[obs_point[k] + 1]++;
  }
  for (int j = 0; j < n_points; ++j) pt_off[j + 1] += pt_off[j];
  int prev = 0;
  for (int r = 0; r <= world; ++r) { prev = std::max(prev, ba_shard_bound(pt_off, n_obs, n_points, r, world)); bounds[r] = prev; }
  return GB_OK;
}

// places a graph in the topology cache's buffer (BaPlace::cache; defined with the cache, below)
template <typename F>
static int ba_cache_slab(gb_ctx* ctx, F&& layout);

// whether the graph's sweep is ba_sweep.cu's kernel, whose item plan is cut on the host
constexpr int kSweepLargeObs = 65536;
static bool ba_sweep_is_large(const gb_ba_graph* g) {
  return g->sweep_mode == 2 || (g->sweep_mode == 0 && g->d.no >= kSweepLargeObs);
}

int ba_graph_create_impl(gb_ctx* ctx, const gb_ba_problem* pb, gb_ba_graph** out, BaPlace place, int shard_rank, int shard_world,
                         const gb_pose_edges* pose_edges) {
  if (!ctx || !out) return GB_ERR_INVALID;
  *out = nullptr;
  CtxLock lk(ctx);
  BaTrace tr;
  GB_CHECK(ba_validate(ctx, pb));
  if (shard_world < 1 || shard_rank < 0 || shard_rank >= shard_world) return GB_ERR_INVALID;
  GB_CHECK(ba_pose_validate(ctx, pb, pose_edges));
  const int npe = pose_edges ? pose_edges->n_se3 + pose_edges->n_gps : 0;
  if (npe > 0 && shard_world > 1) { gb_set_error(ctx, "gb_ba: pose-graph terms are not sharded (single-GPU solve)"); return GB_ERR_INVALID; }
  tr.stamp("validate");
  const int nc = pb->n_cams, np_full = pb->n_points, no_full = pb->n_obs;
  gb_ba_graph* g = new gb_ba_graph();
  struct Guard {
    gb_ctx* c; gb_ba_graph* g; bool ok = false;
    ~Guard() { if (!ok) gb_ba_graph_destroy(c, g); }
  } guard{ctx, g};
  BaDev& d = g->d;

  // ---- host-side ordering over the WHOLE graph: stable counting sorts -> (point, camera) order -------------------------
  // (one histogram pass over both keys; `scam` keeps the camera of each sorted edge so that later passes stream it)
  std::vector<int> order, scam, pt_off;
  {
    std::vector<int> byc(no_full), cam_off_full(nc + 1, 0);
    order.resize(no_full); scam.resize(no_full); pt_off.assign(np_full + 1, 0);
    for (int k = 0; k < no_full; ++k) { cam_off_full[pb->obs_cam[k] + 1]++; pt_off[pb->obs_point[k] + 1]++; }
    for (int i = 0; i < nc; ++i) cam_off_full[i + 1] += cam_off_full[i];
    for (int j = 0; j < np_full; ++j) pt_off[j + 1] += pt_off[j];
    { std::vector<int> pos(cam_off_full.begin(), cam_off_full.end()); for (int k = 0; k < no_full; ++k) byc[pos[pb->obs_cam[k]]++] = k; }
    std::vector<int> pos(pt_off.begin(), pt_off.end() - 1);
    for (int t = 0; t < no_full; ++t) { const int k = byc[t]; const int e = pos[pb->obs_point[k]]++; order[e] = k; scam[e] = pb->obs_cam[k]; }
  }
  {  // duplicate (camera, point) edges would make the block-gather Schur complement drop their cross terms: reject them
    for (int e = 1; e < no_full; ++e)
      if (scam[e] == scam[e - 1] && pb->obs_point[order[e]] == pb->obs_point[order[e - 1]]) {
        gb_set_error(ctx, "gb_ba: edges %d and %d both connect camera %d and point %d (merge duplicate observations)", order[e - 1], order[e],
                     scam[e], pb->obs_point[order[e]]);
        return GB_ERR_INVALID;
      }
  }
  // ---- landmark shard: a contiguous landmark range balanced by observation count; since the edges are sorted by landmark the
  //      shard's edges are ONE contiguous slice [e_lo, e_hi) of the sorted order
  int lo = 0, hi = np_full;
  if (shard_world > 1) {
    lo = ba_shard_bound(pt_off, no_full, np_full, shard_rank, shard_world);
    hi = std::max(ba_shard_bound(pt_off, no_full, np_full, shard_rank + 1, shard_world), lo);
  }
  g->shard_lo = lo; g->shard_hi = hi; g->shard_rank = shard_rank; g->shard_world = shard_world;
  const int e_lo = pt_off[lo], e_hi = pt_off[hi];
  const int np = hi - lo, no = e_hi - e_lo;
  d.nc = nc; d.np = np; d.no = no; d.n6 = 6 * nc; d.has_info = pb->obs_info ? 1 : 0;
  d.vinv_in_sweep = 1;
  d.r_gt = (size_t)d.n6 * d.n6;  // dense layout unless a launch says otherwise (ba_compact_dev)
  g->buf_doubles = ba_buf_doubles(nc);
  // covisibility block structure of S over the WHOLE graph (every rank of a sharded solve must agree on the layout): block
  // (i,i') is structurally non-zero iff some landmark is seen by both cameras
  std::vector<int> s_rowptr(nc + 1, 0), s_col, s_brow;
  if (nc > 0 && nc <= kMaxBlockCams) {
    // one bit row per camera; a landmark ORs the bit mask of its observers into the row of each of them
    const int words = (nc + 63) / 64;
    std::vector<uint64_t> rows((size_t)nc * words, 0), mask(words);
    for (int i = 0; i < nc; ++i) rows[(size_t)i * words + (i >> 6)] |= 1ull << (i & 63);
    for (int j = 0; j < np_full; ++j) {
      const int a = pt_off[j], b = pt_off[j + 1];
      if (b - a < 2) continue;
      if (pb->point_free && !pb->point_free[j]) continue;  // a fixed landmark couples nothing
      int wlo = words, whi = -1;
      for (int e = a; e < b; ++e) { const int w = scam[e] >> 6; wlo = std::min(wlo, w); whi = std::max(whi, w); }
      for (int w = wlo; w <= whi; ++w) mask[w] = 0ull;
      for (int e = a; e < b; ++e) { const int i = scam[e]; mask[i >> 6] |= 1ull << (i & 63); }
      for (int e = a; e < b; ++e) {
        uint64_t* row = &rows[(size_t)scam[e] * words];
        for (int w = wlo; w <= whi; ++w) row[w] |= mask[w];
      }
    }
    for (int i = 0; i < nc; ++i) {
      for (int w = 0; w < words; ++w) {
        uint64_t m = rows[(size_t)i * words + w];
        while (m) {
          const int k = (w << 6) + __builtin_ctzll(m);
          m &= m - 1;
          s_col.push_back(k); s_brow.push_back(i);
        }
      }
      s_rowptr[i + 1] = (int)s_col.size();
    }
  }
  tr.stamp("counting sorts + covisibility");
  // ---- restrict to the shard ---------------------------------------------------------------------------------------------
  if (shard_world > 1) {
    std::vector<int> o2(order.begin() + e_lo, order.begin() + e_hi), c2(scam.begin() + e_lo, scam.begin() + e_hi), p2(np + 1);
    for (int j = 0; j <= np; ++j) p2[j] = pt_off[lo + j] - e_lo;
    order.swap(o2); scam.swap(c2); pt_off.swap(p2);
  }
  std::vector<int> cam_off(nc + 1, 0), cam_perm(no);
  for (int e = 0; e < no; ++e) cam_off[scam[e] + 1]++;
  for (int i = 0; i < nc; ++i) cam_off[i + 1] += cam_off[i];
  { std::vector<int> pos(cam_off.begin(), cam_off.end()); for (int e = 0; e < no; ++e) cam_perm[pos[scam[e]]++] = e; }

  d.s_nnzb = (int)s_col.size();
  std::vector<int> s_upper, s_tidx(s_col.size(), 0);
  for (int blk = 0; blk < (int)s_col.size(); ++blk) {
    const int i = s_brow[blk], i2 = s_col[blk];
    if (i2 >= i) s_upper.push_back(blk);
    int t = s_rowptr[i2];
    while (s_col[t] != i) ++t;  // the structure is symmetric
    s_tidx[blk] = t;
  }
  d.s_nupper = (int)s_upper.size();
  tr.stamp("covisibility block-CSR");
  {  // camera-pass split: ~256 observations per CTA, at most 16 CTAs per camera
    int max_obs = 0;
    for (int i = 0; i < nc; ++i) max_obs = std::max(max_obs, cam_off[i + 1] - cam_off[i]);
    // measured on the 1M-observation graph: 25 us unsplit, 31 / 38 / 54 us at 2 / 4 / 8 slices (the 27-value block reduction per
    // CTA outweighs the shorter serial slices) -> split only cameras that would otherwise run alone for a long time
    d.cam_split = std::min(16, std::max(1, max_obs / 8192));
  }

  // ---- plans: host only, from the host structure above --------------------------------------------------------------------
  std::vector<uint8_t> dof(nc), pfree(np);
  for (int i = 0; i < nc; ++i) dof[i] = pb->cam_dof ? (pb->cam_dof[i] & 63) : 63;
  for (int j = 0; j < np; ++j) pfree[j] = pb->point_free ? (pb->point_free[lo + j] ? 1 : 0) : 1;
  for (int i = 0; i < nc; ++i) g->pcg_nact += dof[i] != 0;
  for (int i = 0; i < nc && !s_col.empty(); ++i) g->pcg_max_row_blocks = std::max(g->pcg_max_row_blocks, s_rowptr[i + 1] - s_rowptr[i]);
  std::vector<int> chol_plan3;
  if (d.s_nnzb > 0) g->chol_ok = ba_chol_plan_host(ctx, nc, s_rowptr.data(), s_col.data(), chol_plan3, &g->chol_blocks, &g->chol_smem);
  const bool compact_only = shard_world > 1;  // a shard only ever sees the compact reduced layout: no dense 6N x 6N buffer
  g->rbuf_doubles = d.s_nnzb > 0 ? (size_t)d.s_nnzb * 36 + 2 * (size_t)d.n6 + 8 : 0;
  ba_pick_pcg(ctx, g);
  BaPosePlan pose;
  if (npe > 0) {  // pose-graph terms: the stepwise path on the dense reduced system (one-cluster / generic PCG)
    g->pcg_sparse = false;
    ba_pose_plan(g, pose_edges, pose);
  }
  std::vector<int> bcsr_cta_cam;
  BaSchurPlan schur;
  if (npe == 0 && (!g->pcg_sparse || compact_only) && d.s_nnzb > 0) {  // (a shard always runs on the compact block-CSR system)
    ba_pcg_bcsr_plan(ctx, g, s_rowptr.data(), s_col.data(), bcsr_cta_cam);
    if (!getenv("GB_BA_NO_SCHUR_CHUNKS")) ba_schur_plan(ctx, g, np, pt_off, scam, pfree.data(), s_rowptr, s_col, s_upper, schur);  // (optional: the block-gather kernel otherwise)
  }
  g->sp_max_nused = d.sp_nchunks > 0 ? *std::max_element(schur.nused.begin(), schur.nused.end()) : 0;
  if (compact_only && !g->pcg_bcsr) {
    gb_set_error(ctx, "gb_ba: the sharded solve needs the block-CSR reduced system (<= %d cameras)", kMaxBlockCams);
    return GB_ERR_INVALID;
  }
  std::vector<int> o_pt(no), c_pt(no);
  for (int e = 0; e < no; ++e) o_pt[e] = pb->obs_point[order[e]] - lo;
  for (int idx = 0; idx < no; ++idx) c_pt[idx] = o_pt[cam_perm[idx]];
  std::vector<int> sw_items, sw_team_off;
  const int sw_teams = ba_sweep_teams(ctx);
  if (ba_sweep_is_large(g)) {
    ba_sweep_plan_host(nc, np, d.cam_split, cam_off, pt_off, sw_teams, sw_items, sw_team_off);
    d.sw_nteams = sw_teams; d.sw_nitems = (int)(sw_items.size() / 4);
  }
  tr.stamp("plans");

  // ---- layout: one slab = [uploaded blob | working set] ----------------------------------------------------------------
  const size_t n6 = 6 * (size_t)nc;
  auto layout = [&](Slab& sl) {
    sl.put(&g->pose_wc_in, (size_t)nc * 7, pb->cam_pose_wc);  // T_wc as given: the source of ba_prepare_kernel
    sl.put(&g->pts_init, (size_t)np * 3, pb->points + 3 * (size_t)lo);
    sl.put(&d.dof, nc, dof.data()); sl.put(&d.pfree, np, pfree.data());
    sl.put(&d.o_cam, no, scam.data()); sl.put(&d.o_pt, no, o_pt.data());
    sl.put(&d.o_uv, 2 * (size_t)no);  // (the measurements: ba_fill_measurements)
    if (d.has_info) sl.put(&d.o_info, 3 * (size_t)no);
    sl.put(&d.c_pt, no, c_pt.data()); sl.put(&d.c_uv, 2 * (size_t)no);
    sl.put(&d.pt_off, pt_off.size(), pt_off.data()); sl.put(&d.cam_off, cam_off.size(), cam_off.data());
    sl.put(&d.cam_perm, no, cam_perm.data());
    sl.put(&d.s_rowptr, s_rowptr.size(), s_rowptr.data()); sl.put(&d.s_col, s_col.size(), s_col.data());
    sl.put(&d.s_brow, s_brow.size(), s_brow.data()); sl.put(&d.s_upper, s_upper.size(), s_upper.data());
    sl.put(&d.s_tidx, s_tidx.size(), s_tidx.data());
    sl.put(&g->chol_plan, chol_plan3.size(), chol_plan3.data());
    if (g->pcg_bcsr) sl.put(&g->bcsr_cta_cam, bcsr_cta_cam.size(), bcsr_cta_cam.data());
    if (d.sp_nchunks > 0) {
      sl.put(&d.sp_pt0, schur.pt0.size(), schur.pt0.data()); sl.put(&d.sp_order, schur.order.size(), schur.order.data());
      sl.put(&d.sp_mask, schur.mask.size(), schur.mask.data()); sl.put(&d.sp_nused, schur.nused.size(), schur.nused.data());
      sl.put(&d.sp_slots, schur.slots.size(), schur.slots.data());
      sl.put(&d.sp_boff, schur.boff.size(), schur.boff.data()); sl.put(&d.sp_bidx, schur.bidx.size(), schur.bidx.data());
      sl.put(&d.sp_coff, schur.coff.size(), schur.coff.data()); sl.put(&d.sp_cidx, schur.cidx.size(), schur.cidx.data());
    }
    if (npe > 0) {
      sl.put(&d.pe_i, pose.ei.size(), pose.ei.data()); sl.put(&d.pe_j, pose.ej.size(), pose.ej.data());
      sl.put(&d.pe_Zinv, pose.Zinv.size(), pose.Zinv.data()); sl.put(&d.pe_info, pose.info.size(), pose.info.data());
      sl.put(&d.pc_off, pose.pc_off.size(), pose.pc_off.data()); sl.put(&d.pc_ent, pose.pc_ent.size(), pose.pc_ent.data());
      sl.put(&d.pp_off, pose.pp_off.size(), pose.pp_off.data()); sl.put(&d.pp_ij, pose.pp_ij.size(), pose.pp_ij.data());
      sl.put(&d.pp_ent, pose.pp_ent.size(), pose.pp_ent.data());
    }
    if (d.sw_nteams > 0) { sl.put(&d.sw_items, sw_items.size(), sw_items.data()); sl.put(&d.sw_team_off, sw_team_off.size(), sw_team_off.data()); }
    sl.take(&g->pose_init, (size_t)nc * 7); sl.take(&g->pose_wc_out, (size_t)nc * 7);
    sl.take(&d.pose, (size_t)nc * 7); sl.take(&d.pose_new, (size_t)nc * 7);
    sl.take(&d.Rt, (size_t)nc * 12); sl.take(&d.Rt_new, (size_t)nc * 12);
    sl.take(&d.pts, (size_t)np * 3); sl.take(&d.pts_new, (size_t)np * 3);
    sl.take(&d.V, (size_t)np * 9); sl.take(&d.gp, (size_t)np * 3); sl.take(&d.Vinv, (size_t)np * 9);
    sl.take(&d.W, (size_t)no * 18); sl.take(&d.U, (size_t)nc * 36); sl.take(&d.gc, (size_t)nc * 6);
    sl.take(&d.cost_pt, (size_t)np + npe); sl.take(&d.cost_pt_new, (size_t)np + npe);
    sl.take(&d.cam_part, (size_t)nc * std::max(d.cam_split, 4) * 27); sl.take(&d.cam_ticket, (size_t)nc + 2);
    sl.take(&d.Minv, (size_t)nc * 36);
    sl.take(&d.Sb, (size_t)d.s_nnzb * 36);
    sl.take(&d.x, n6); sl.take(&d.r, n6); sl.take(&d.z, n6); sl.take(&d.p, n6); sl.take(&d.q, n6); sl.take(&d.sv, n6);
    sl.take(&d.sc, 1);
    sl.take(&d.red_part, (size_t)kRedPartials + 2);
    sl.take(&g->buf, compact_only ? 8 : g->buf_doubles);
    sl.take(&g->d_cost, 8);
    sl.take(&g->rbuf, g->rbuf_doubles);
    if (g->pcg_bcsr) { sl.take(&g->bcsr_part, 2 * (size_t)g->bcsr_ctas); sl.take(&g->bcsr_u, n6); sl.take(&g->bcsr_bar, 16); }
    if (d.sp_nchunks > 0) {
      sl.take(&d.sp_stageS, (size_t)d.sp_nchunks * kChunkSlots * 36);
      sl.take(&d.sp_stageG, (size_t)d.sp_nchunks * kChunkCams * 6);
    }
    if (npe > 0) sl.take(&d.pe_H, pose.rec_doubles);
    // the test hooks' room: a sweep plan of any split they allow (a landmark group holds at least one landmark), the PCG's stamps
    sl.take(&g->sw_room, 4 * ((size_t)nc * std::max(d.cam_split, 4) + np) + sw_teams + 1);
    sl.take(&g->prof_room, 8);
  };
  Slab placed;  // the layout as placed: its base and the size of its blob
  auto place_layout = [&](Slab& sl) { layout(sl); placed = sl; };
  if (place == BaPlace::own) GB_CHECK(gb_slab_alloc(ctx, (void**)&g->slab, place_layout));
  else if (place == BaPlace::cache) GB_CHECK(ba_cache_slab(ctx, place_layout));
  else GB_CHECK(gb_scratch_slab(ctx, place_layout));
  tr.stamp("slab");

  // ---- one pinned blob, one H2D ------------------------------------------------------------------------------------------
  uint8_t* h_blob;
  GB_CHECK(gb_stage_take(ctx, {{&h_blob, placed.blob}}));
  Slab real{placed.base, h_blob};
  layout(real);
  ba_fill_measurements(pb, order, cam_perm, real.host(d.o_uv), real.host(d.c_uv), d.has_info ? real.host(d.o_info) : nullptr);
  g->sorted_to_orig.swap(order);
  g->cam_perm_h.swap(cam_perm);
  tr.stamp("blob fill");
  GB_CUDA(ctx, cudaMemcpyAsync(real.base, real.h, real.blob, cudaMemcpyHostToDevice, ctx->stream));
  d.red_ticket = reinterpret_cast<unsigned int*>(d.red_part + kRedPartials);
  GB_CUDA(ctx, cudaMemsetAsync(d.red_ticket, 0, 16, ctx->stream));
  GB_CUDA(ctx, cudaMemsetAsync(d.cam_ticket, 0, ((size_t)nc + 2) * 4, ctx->stream));
  if (npe > 0) GB_CUDA(ctx, cudaMemsetAsync(d.pe_H, 0, pose.rec_doubles * 8, ctx->stream));
  if (nc > 0) {
    ba_prepare_kernel<<<gb_div_up(nc, 128), 128, 0, ctx->stream>>>(nc, g->pose_wc_in, g->pose_init);
    GB_LAUNCH_CHECK(ctx);
  }
  GB_CHECK(gb_ba_graph_reset(ctx, g));
  tr.stamp("enqueue H2D + prepare");
  // the pinned blob is reused by the next outermost call on this ctx: a graph handed to the caller must have consumed it; the
  // host-buffer paths (gb_ba_solve / gb_ba_solve_posegraph / gb_ba_pnp) synchronise in their own finish + download before they return
  if (place == BaPlace::own) GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  tr.stamp("sync");
  guard.ok = true;
  *out = g;
  return GB_OK;
}

extern "C" {

int gb_ba_graph_reset(gb_ctx* ctx, gb_ba_graph* g) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  BaDev& d = g->d;
  if (d.nc > 0) GB_CUDA(ctx, cudaMemcpyAsync(d.pose, g->pose_init, (size_t)d.nc * 56, cudaMemcpyDeviceToDevice, ctx->stream));
  if (d.np > 0) GB_CUDA(ctx, cudaMemcpyAsync(d.pts, g->pts_init, (size_t)d.np * 24, cudaMemcpyDeviceToDevice, ctx->stream));
  g->begun = false;
  return GB_OK;
}

int gb_ba_graph_reduce_size(gb_ctx* ctx, gb_ba_graph* g, size_t* n) {
  if (!ctx || !g || !n) return GB_ERR_INVALID;
  *n = g->buf_doubles;
  return GB_OK;
}

int gb_ba_graph_begin(gb_ctx* ctx, gb_ba_graph* g, const gb_ba_options* opt_in) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  gb_ba_options opt;
  if (opt_in) opt = *opt_in; else gb_ba_options_default(&opt);
  if (opt.projection != 0) {
    gb_set_error(ctx, "gb_ba: only PROJECTION_PINHOLE (Optimizer.h:59) is implemented");
    return GB_ERR_INVALID;
  }
  if (opt.max_iterations < 0 || opt.pcg_max_iters < 0) {
    gb_set_error(ctx, "gb_ba: max_iterations (%d) and pcg_max_iters (%d) must not be negative", opt.max_iterations, opt.pcg_max_iters);
    return GB_ERR_INVALID;
  }
  // (a NaN lambda never leaves NaN and a zero one never leaves a reject streak; a NaN tolerance never stops)
  if (!(std::isfinite(opt.lambda_init) && opt.lambda_init > 0.0)) {
    gb_set_error(ctx, "gb_ba: lambda_init must be finite and > 0 (got %g)", opt.lambda_init);
    return GB_ERR_INVALID;
  }
  if (std::isnan(opt.huber_delta) || std::isnan(opt.function_tolerance) || std::isnan(opt.pcg_tol)) {
    gb_set_error(ctx, "gb_ba: huber_delta, function_tolerance and pcg_tol must not be NaN");
    return GB_ERR_INVALID;
  }
  if (opt.linear_solver != 0 && opt.linear_solver != 1) { gb_set_error(ctx, "gb_ba: linear_solver must be 0 (PCG) or 1 (direct)"); return GB_ERR_INVALID; }
  if (opt.linear_solver == 1 && g->d.npe > 0) { gb_set_error(ctx, "gb_ba: graphs with pose-graph terms use linear_solver = 0 (PCG)"); return GB_ERR_INVALID; }
  if (opt.linear_solver == 1 && g->d.nc > 0 && (!g->chol_ok || g->shard_world > 1)) {
    gb_set_error(ctx, "gb_ba: the direct solver needs the block skyline of the reduced camera system to fit one SM's shared memory "
                      "(%d cameras here) and a single-GPU solve; use linear_solver = 0 (PCG)", g->d.nc);
    return GB_ERR_INVALID;
  }
  g->opt = opt;
  BaScalars h;
  memset(&h, 0, sizeof h);
  h.delta = opt.huber_delta; h.ftol = opt.function_tolerance; h.pcg_tol = opt.pcg_tol; h.lambda_init = opt.lambda_init;
  h.lambda = opt.lambda_init; h.nu = 2.0; h.need_linearize = 1;
  // kernel-argument-sized payload: no staging, no sync
  GB_CUDA(ctx, cudaMemcpyAsync(g->d.sc, &h, sizeof h, cudaMemcpyHostToDevice, ctx->stream));
  if (g->d.nc > 0) {
    ba_rt_kernel<<<gb_div_up(g->d.nc, 128), 128, 0, ctx->stream>>>(g->d.nc, g->d.pose, g->d.Rt);
    GB_LAUNCH_CHECK(ctx);
  }
  g->begun = true;
  g->sweep_only = false;
  return GB_OK;
}

// generic (any size) PCG: damp + init + max_iters x (matvec, update) + retract
static int ba_pcg_generic(gb_ctx* ctx, gb_ba_graph* g, double* buf) {
  BaDev& d = g->d;
  cudaStream_t s = ctx->stream;
  ba_damp_kernel<<<gb_div_up(d.n6, 128), 128, 0, s>>>(d, buf); GB_LAUNCH_CHECK(ctx);
  pcg_init_kernel<<<1, kRedThreads, 0, s>>>(d, buf); GB_LAUNCH_CHECK(ctx);
  for (int k = 0; k <= g->opt.pcg_max_iters; ++k) {  // one extra pair: the convergence test of update k runs in pair k+1
    pcg_matvec_kernel<<<gb_div_up(d.n6, 8), 256, 0, s>>>(d, buf); GB_LAUNCH_CHECK(ctx);
    pcg_update_kernel<<<1, kRedThreads, 0, s>>>(d, (int)g->opt.pcg_max_iters); GB_LAUNCH_CHECK(ctx);
  }
  ba_retract_kernel<<<gb_div_up(d.nc, 128), 128, 0, s>>>(d); GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}

// local-BA PCG: one thread-block cluster, S resident in shared memory, one cluster barrier per iteration
static int ba_pcg_cluster(gb_ctx* ctx, gb_ba_graph* g, double* buf) {
  GbClusterConfig lc(g->pcg_cluster, dim3(kPcgThreads), g->pcg_smem, ctx->stream);
  GB_CUDA(ctx, cudaLaunchKernelEx(&lc.cfg, ba_pcg_cluster_kernel, g->d, buf, (int)g->opt.pcg_max_iters));
  GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}

}  // extern "C"

// The residual + Jacobian sweep outside the local-BA launch chain: graphs with enough observations to fill the machine take the
// bandwidth-tuned persistent kernel (ba_sweep.cu), small ones the latency-tuned one above.  which: 3 whole, 1 cameras, 2 landmarks.
static int ba_launch_sweep(gb_ctx* ctx, gb_ba_graph* g, const BaDev& d, cudaStream_t s, int which) {
  if (ba_sweep_is_large(g)) return ba_sweep_launch(ctx, d, s, which);
  const int pt_blocks = (which & 2) ? gb_div_up(d.np * kLpp, kPtThreads) : 0, cam_blocks = (which & 1) ? d.nc * d.cam_split : 0;
  if (pt_blocks + cam_blocks > 0) { ba_linearize_kernel<<<pt_blocks + cam_blocks, kPtThreads, 0, s>>>(d, cam_blocks); GB_LAUNCH_CHECK(ctx); }
  return GB_OK;
}

// Sweep + Schur complement of g's landmarks into `buf`, on the layout `d` describes (g->d: the dense one, ba_compact_dev: the
// compact one).  `dense`: ba_prepare_schur_kernel also writes the dense S of buf.  The pose-graph terms, if any, go into U, g_c and
// the cost terms between the two.  With the covisibility block structure at hand (<= kMaxBlockCams = 2048 cameras) the S blocks
// are formed block by block without atomics (deterministic); without it this forms none (gb_ba_graph_reduce_local's atomic path).
static int ba_reduce(gb_ctx* ctx, gb_ba_graph* g, const BaDev& d, double* buf, bool dense) {
  cudaStream_t s = ctx->stream;
  GB_CHECK(ba_launch_sweep(ctx, g, d, s, 3));
  GB_CHECK(ba_pose_linearize(ctx, g, s));
  const size_t work = std::max<size_t>(dense ? (size_t)d.n6 * d.n6 : 0, (size_t)d.np);
  const int nblk = (int)std::min<size_t>(std::max<size_t>((work + 255) / 256, 1), (size_t)ctx->sm_count * 8);
  ba_prepare_schur_kernel<<<nblk, 256, 0, s>>>(d, buf, dense ? 1 : 0); GB_LAUNCH_CHECK(ctx);
  if (d.s_nnzb > 0 && d.nc > 0) {
    if (d.sp_nchunks > 0) {
      ba_schur_chunks_kernel<<<d.sp_nchunks, kChunkThreads, 0, s>>>(d); GB_LAUNCH_CHECK(ctx);
      ba_schur_reduce_kernel<<<d.s_nupper, 64, 0, s>>>(d, buf); GB_LAUNCH_CHECK(ctx);
    } else {
      ba_schur_blocks_kernel<<<d.s_nupper, 128, 0, s>>>(d, buf); GB_LAUNCH_CHECK(ctx);
    }
  }
  return GB_OK;
}

extern "C" {

int gb_ba_graph_sweep(gb_ctx* ctx, gb_ba_graph* g, double huber_delta) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  gb_ba_options o;
  gb_ba_options_default(&o);
  o.huber_delta = huber_delta;
  if (!g->begun || !g->sweep_only || g->opt.huber_delta != huber_delta) {  // (repeated sweeps re-use the scalars: nothing resets need_linearize)
    GB_CHECK(gb_ba_graph_begin(ctx, g, &o));
    g->sweep_only = true;
  }
  BaDev& d = g->d;
  GB_CHECK(ba_launch_sweep(ctx, g, d, ctx->stream, 3));
  return GB_OK;
}

int gb_ba_graph_reduce_local(gb_ctx* ctx, gb_ba_graph* g, double* buf) {
  if (!ctx || !g || !g->begun) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  BaDev& d = g->d;
  if (!buf) buf = g->buf;
  cudaStream_t s = ctx->stream;
  d.vinv_in_sweep = ba_sweep_is_large(g) ? 0 : 1;
  // The local-BA solver consumes the S blocks directly; every other consumer (one-cluster / generic PCG, the direct solver, a
  // caller's all-reduce) gets them scattered into the dense layout of `buf`.
  const bool have_blocks = d.s_nnzb > 0 && d.nc > 0;
  const bool csr_only = have_blocks && g->pcg_sparse && buf == g->buf;
  GB_CHECK(ba_reduce(ctx, g, d, buf, !csr_only));
  if (have_blocks) {
    if (!csr_only) { ba_densify_fill_kernel<<<gb_div_up(d.s_nnzb * 36, 256), 256, 0, s>>>(d, buf); GB_LAUNCH_CHECK(ctx); }
  } else if (d.no > 0 && d.nc > 0) {
    ba_schur_accum_kernel<<<gb_div_up(d.no, 128), 128, 0, s>>>(d, buf); GB_LAUNCH_CHECK(ctx);
    const int nblk = (int)std::min<size_t>(((size_t)d.n6 * d.n6 + 255) / 256, (size_t)ctx->sm_count * 8);
    ba_mirror_kernel<<<nblk, 256, 0, s>>>(d, buf); GB_LAUNCH_CHECK(ctx);
  }
  GB_CHECK(ba_pose_offdiag(ctx, g, buf, s));
  return GB_OK;
}

}  // extern "C"

static int ba_red_blocks(const gb_ctx* ctx, int n) { return std::max(1, std::min(std::min(ctx->sm_count, kRedPartials), (n + 8 * kRedThreads - 1) / (8 * kRedThreads))); }

// ---- one LM iteration on the COMPACT reduced layout rbuf = [Sb (nnzb x 36) | g~ | diag U | cost | pad] ------------------------------
// (large graphs on one GPU and every rank of the landmark-sharded solve: with a communicator, what the collective sums is the shard's
// contribution to the reduced system and to the candidate cost)
static BaDev ba_compact_dev(const gb_ba_graph* g) {
  BaDev d = g->d;
  d.Sb = g->rbuf;
  d.r_gt = (size_t)d.s_nnzb * 36;
  d.vinv_in_sweep = ba_sweep_is_large(g) ? 0 : 1;
  return d;
}

// The candidate tail of every LM iteration off the local-BA chain, after its linear solve: back-substitution of the landmarks, the
// candidate cost (pose-graph terms included) summed into d_cost and, with a communicator, all-reduced over the landmark shards ...
static int ba_candidate_cost(gb_ctx* ctx, gb_ba_graph* g, const BaDev& d, double* d_cost, gb_comm* comm) {
  cudaStream_t s = ctx->stream;
  if (d.np > 0) { ba_backsub_cost_kernel<<<gb_div_up(d.np * kLpp, 128), 128, 0, s>>>(d); GB_LAUNCH_CHECK(ctx); }
  GB_CHECK(ba_pose_cost(ctx, g, s));
  ba_reduce_cost_kernel<<<ba_red_blocks(ctx, d.np + d.npe), kRedThreads, 0, s>>>(d, d.cost_pt_new, d.np + d.npe, d_cost); GB_LAUNCH_CHECK(ctx);
  if (comm) GB_CHECK(gb_comm_allreduce_sum_f64(comm, d_cost, 1));
  return GB_OK;
}

// ... then the LM decision from the cost in `buf` (at d.r_gt + 2 n6) and d_cost, with the installation of an accepted candidate
static int ba_commit(gb_ctx* ctx, const BaDev& d, const double* buf, const double* d_cost) {
  const int n = std::max(std::max(d.nc * 12, d.np * 3), 1);
  ba_commit_apply_kernel<<<gb_div_up(n, 256), 256, 0, ctx->stream>>>(d, buf, d_cost); GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}

int ba_compact_reduce(gb_ctx* ctx, gb_ba_graph* g, gb_comm* comm) {
  GB_CHECK(ba_reduce(ctx, g, ba_compact_dev(g), g->rbuf, false));
  if (comm) GB_CHECK(gb_comm_allreduce_sum_f64(comm, g->rbuf, g->rbuf_doubles));
  return GB_OK;
}

// the second half of the iteration: block-CSR PCG, the candidate tail on the compact layout
static int ba_compact_step(gb_ctx* ctx, gb_ba_graph* g, gb_comm* comm) {
  const BaDev d = ba_compact_dev(g);
  GB_CHECK(ba_pcg_bcsr_launch(ctx, g, g->rbuf));
  GB_CHECK(ba_candidate_cost(ctx, g, d, g->d_cost, comm));
  return ba_commit(ctx, d, g->rbuf, g->d_cost);
}

// The costs of a solve come from its LM decisions (lm_decide); one that made none still reports the cost at its input estimate as
// both initial and final cost: a sweep, the pose-graph terms and the deterministic sum (all-reduced over the shards with a
// communicator) into the LM scalars.
static int ba_cost_at_input(gb_ctx* ctx, gb_ba_graph* g, gb_comm* comm) {
  const BaDev& d = g->d;
  cudaStream_t s = ctx->stream;
  GB_CHECK(ba_launch_sweep(ctx, g, d, s, 3));
  GB_CHECK(ba_pose_linearize(ctx, g, s));
  ba_reduce_cost_kernel<<<ba_red_blocks(ctx, d.np + d.npe), kRedThreads, 0, s>>>(d, d.cost_pt, d.np + d.npe, g->d_cost); GB_LAUNCH_CHECK(ctx);
  if (comm) GB_CHECK(gb_comm_allreduce_sum_f64(comm, g->d_cost, 1));
  GB_CUDA(ctx, cudaMemcpyAsync(&d.sc->initial_cost, g->d_cost, sizeof(double), cudaMemcpyDeviceToDevice, s));
  GB_CUDA(ctx, cudaMemcpyAsync(&d.sc->cost, g->d_cost, sizeof(double), cudaMemcpyDeviceToDevice, s));
  return GB_OK;
}

extern "C" {

// single-CTA block-sparse PCG, in the variant that fits the graph's active cameras and its longest block row of S (the
// shared-memory path for columns beyond the registers is compiled in only where a row needs it; pdl: programmatic dependent
// launch)
static void ba_pcg_sparse_variant(const gb_ba_graph* g, bool* small, bool* long_rows) {
  *small = g->pcg_nact <= kSpSmallCams;
  *long_rows = 6 * g->pcg_max_row_blocks > 8 * (*small ? kSpSmallCols : kSpLargeCols);
}

static int ba_pcg_sparse_launch(gb_ctx* ctx, gb_ba_graph* g, double* buf, bool pdl) {
  bool small, long_rows;
  ba_pcg_sparse_variant(g, &small, &long_rows);
  void (*kernel)(BaDev, double*, int) = small ? (long_rows ? BA_SPARSE_SMALL(true) : BA_SPARSE_SMALL(false))
                                              : (long_rows ? BA_SPARSE_LARGE(true) : BA_SPARSE_LARGE(false));
  const dim3 block(small ? kSpSmallThreads : kSpLargeThreads);
  const int maxit = (int)g->opt.pcg_max_iters;
  if (pdl) GB_CUDA(ctx, gb_launch_pdl(kernel, dim3(1), block, g->pcg_sparse_smem, ctx->stream, g->d, buf, maxit));
  else kernel<<<1, block, g->pcg_sparse_smem, ctx->stream>>>(g->d, buf, maxit);
  GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}

static int ba_pcg_dispatch(gb_ctx* ctx, gb_ba_graph* g, double* buf) {
  if (g->d.nc <= 0) return GB_OK;
  if (g->opt.linear_solver == 1) return ba_chol_launch(ctx, g, buf, false);
  if (g->pcg_sparse && buf == g->buf) return ba_pcg_sparse_launch(ctx, g, buf, false);
  if (g->pcg_cluster > 0) return ba_pcg_cluster(ctx, g, buf);
  return ba_pcg_generic(ctx, g, buf);
}

int gb_ba_graph_step(gb_ctx* ctx, gb_ba_graph* g, const double* buf_in, double* d_cost) {
  if (!ctx || !g || !g->begun) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  GB_CHECK(ba_pcg_dispatch(ctx, g, buf_in ? (double*)buf_in : g->buf));
  return ba_candidate_cost(ctx, g, g->d, d_cost ? d_cost : g->d_cost, nullptr);
}

int gb_ba_graph_commit(gb_ctx* ctx, gb_ba_graph* g, const double* buf_in, const double* d_cost) {
  if (!ctx || !g || !g->begun) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  return ba_commit(ctx, g->d, buf_in ? buf_in : g->buf, d_cost ? d_cost : g->d_cost);  // (dense layout: the cost sits at r_gt = n6 * n6)
}

static int ba_read_scalars(gb_ctx* ctx, gb_ba_graph* g, BaScalars* out) {
  GB_CUDA(ctx, cudaMemcpyAsync(out, g->d.sc, sizeof(BaScalars), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return GB_OK;
}

// res (all but gpu_ms, when given) <- the LM scalars at the end of a solve; a non-finite final cost is an error
static int ba_fill_result(gb_ctx* ctx, const BaScalars& h, gb_ba_result* res) {
  if (res) {
    res->initial_cost = h.initial_cost;
    res->final_cost = h.cost;
    res->iterations = h.iterations;
    res->accepted = h.accepted;
    res->pcg_iterations = h.pcg_iters;
    res->status = h.status;
    res->lambda_final = h.lambda;
  }
  if (!std::isfinite(h.cost)) {
    gb_set_error(ctx, "gb_ba: non-finite cost");
    return GB_ERR_NUMERIC;
  }
  return GB_OK;
}

// (the stepwise interface's caller ran the LM iterations, so whether any made a decision is read from the scalars)
int gb_ba_graph_finish(gb_ctx* ctx, gb_ba_graph* g, gb_ba_result* res) {
  if (!ctx || !g || !g->begun) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  BaScalars h;
  GB_CHECK(ba_read_scalars(ctx, g, &h));
  if (h.iterations == 0) {
    GB_CHECK(ba_cost_at_input(ctx, g, nullptr));
    GB_CHECK(ba_read_scalars(ctx, g, &h));
  }
  return ba_fill_result(ctx, h, res);
}

// local-BA fast path (block-CSR Schur + single-CTA PCG): 4 launches per LM iteration, for graphs whose estimate fits the
// single-CTA loops of its tail (ba_backsub_commit_kernel's last CTA, ba_install_pending_kernel)
static bool ba_takes_local4(const gb_ba_graph* g) {
  return g->d.npe == 0 && (size_t)g->d.np * 3 + (size_t)g->d.nc * 19 <= (size_t)1 << 16 && g->pcg_sparse && g->d.s_nnzb > 0 && g->d.nc > 0 &&
         g->d.np > 0;
}

// Enqueue the D2H copies of g's T_wc poses (finalized into g->pose_wc_out first) into hp and of its points into hx; a null
// buffer is skipped.
static int ba_enqueue_download(gb_ctx* ctx, gb_ba_graph* g, double* hp, double* hx) {
  const BaDev& d = g->d;
  if (hp) {
    ba_finalize_kernel<<<gb_div_up(d.nc, 128), 128, 0, ctx->stream>>>(d.nc, d.pose, g->pose_wc_out);
    GB_LAUNCH_CHECK(ctx);
    GB_CUDA(ctx, cudaMemcpyAsync(hp, g->pose_wc_out, (size_t)d.nc * 56, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (hx) GB_CUDA(ctx, cudaMemcpyAsync(hx, d.pts, (size_t)d.np * 24, cudaMemcpyDeviceToHost, ctx->stream));
  return GB_OK;
}

}  // extern "C"

// Whether g's LM iterations (and gb_dbg_ba_system) run on the compact reduced system: when the block-CSR PCG solves it and g is a
// landmark shard (`comm`; a shard of a small graph can have pcg_sparse set too) or too large for the local-BA chain
static bool ba_iterates_compact(const gb_ba_graph* g, const gb_comm* comm) {
  return g->pcg_bcsr && g->opt.linear_solver == 0 && (comm || !ba_takes_local4(g));
}

// LM loop of a whole solve, then ONE synchronisation for everything the host wants back: the LM scalars and, for the one-shot
// host-buffer paths, the final T_wc poses / points (pose_out / pts_out may be null).  With `comm`, g is this rank's landmark shard
// (gb_ba_shard_solve): every rank reaches the same collectives and reads the same all-reduced scalars, so all stop together.  A
// world-1 shard may take the direct solver (gb_ba_graph_begin refuses it at world > 1) and then iterates as gb_ba_graph_solve does.
int ba_graph_solve_impl(gb_ctx* ctx, gb_ba_graph* g, gb_comm* comm, const gb_ba_options* opt, gb_ba_result* res, double* pose_out,
                        double* pts_out) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  GB_CHECK(gb_ba_graph_begin(ctx, g, opt));
  // A device-resident solve (no host outputs, not nested in another call on this ctx) waits for the device WITHOUT the ctx lock,
  // on the graph's own pinned scalars and events: a tracking thread can then order its next frame after its match on this ctx
  // (gb_ctx_wait_for) while the mapping thread still waits for this solve, and the next solve finds that frame already handed over.
  // A second solve of g that another thread starts during that wait (g->waiting) takes the locked wait, leaving g's scalars and
  // events to the first.  A shard's solve always waits locked.
  const bool unlocked_wait = !comm && !pose_out && !pts_out && ctx->lock_depth == 1 && !g->waiting;
  if (unlocked_wait) {
    if (!g->h_sc) GB_CUDA(ctx, cudaMallocHost((void**)&g->h_sc, sizeof(BaScalars)));
    if (!g->ev_s) GB_CUDA(ctx, cudaEventCreate(&g->ev_s));
    if (!g->ev_e) GB_CUDA(ctx, cudaEventCreate(&g->ev_e));
    if (!g->ev_done) GB_CUDA(ctx, cudaEventCreateWithFlags(&g->ev_done, cudaEventDisableTiming));
  }
  cudaEvent_t ev_s = unlocked_wait ? g->ev_s : ctx->evs, ev_e = unlocked_wait ? g->ev_e : ctx->eve;
  GB_CUDA(ctx, cudaEventRecord(ev_s, ctx->stream));
  const bool poll = g->opt.function_tolerance > 0.0 || g->opt.verbose;
  const bool local4 = !comm && ba_takes_local4(g), compact = ba_iterates_compact(g, comm);
  for (int it = 0; it < g->opt.max_iterations; ++it) {
    if (local4) {
      BaDev& d = g->d;
      cudaStream_t s = ctx->stream;
      const int pt_blocks = gb_div_up(d.np * kLpp, kPtThreads), cam_blocks = d.nc * d.cam_split;
      // (programmatic dependent launches: each kernel is scheduled while its predecessor drains)
      GB_CUDA(ctx, gb_launch_pdl(ba_linearize_kernel, dim3(pt_blocks + cam_blocks), dim3(kPtThreads), 0, s, d, cam_blocks)); GB_LAUNCH_CHECK(ctx);
      GB_CUDA(ctx, gb_launch_pdl(ba_schur_blocks_kernel, dim3(d.s_nupper), dim3(128), 0, s, d, g->buf)); GB_LAUNCH_CHECK(ctx);
      if (g->opt.linear_solver == 1) GB_CHECK(ba_chol_launch(ctx, g, g->buf, true));
      else GB_CHECK(ba_pcg_sparse_launch(ctx, g, g->buf, true));
      GB_CUDA(ctx, gb_launch_pdl(ba_backsub_commit_kernel, dim3(gb_div_up(d.np * kLpp, kTailThreads)), dim3(kTailThreads), 0, s, d, (const double*)g->buf)); GB_LAUNCH_CHECK(ctx);
    } else if (compact) {  // compact block-CSR reduced system + the persistent multi-CTA PCG (+ the shards' all-reduces)
      GB_CHECK(ba_compact_reduce(ctx, g, comm));
      GB_CHECK(ba_compact_step(ctx, g, comm));
    } else {  // the stepwise interface on the dense reduced layout
      GB_CHECK(gb_ba_graph_reduce_local(ctx, g, nullptr));
      GB_CHECK(gb_ba_graph_step(ctx, g, nullptr, nullptr));
      GB_CHECK(gb_ba_graph_commit(ctx, g, nullptr, nullptr));
    }
    if (poll) {
      BaScalars h;
      GB_CHECK(ba_read_scalars(ctx, g, &h));
      if (g->opt.verbose && (!comm || gb_comm_rank(comm) == 0)) {
        char tag[24] = "[gb_ba]";
        if (comm) snprintf(tag, sizeof tag, "[gb_ba x%d]", gb_comm_world(comm));
        fprintf(stderr, "%s it %d cost %.12e lambda %.3e accepted %d pcg %d%s\n", tag, it, h.cost, h.lambda, h.accepted,
                h.pcg_iters, h.stop ? " stop" : "");
      }
      if (h.stop) break;
    }
  }
  if (local4) { ba_install_pending_kernel<<<1, 1024, 0, ctx->stream>>>(g->d); GB_LAUNCH_CHECK(ctx); }
  if (g->opt.max_iterations == 0) GB_CHECK(ba_cost_at_input(ctx, g, comm));  // (no LM decision: every iteration makes one)
  GB_CUDA(ctx, cudaEventRecord(ev_e, ctx->stream));
  BaDev& dd = g->d;
  const size_t bp = pose_out ? (size_t)dd.nc * 56 : 0, bx = pts_out ? (size_t)dd.np * 24 : 0;
  BaScalars* hs;
  double *hp, *hx;
  GB_CHECK(gb_stage_take(ctx, {{&hs, unlocked_wait ? 0 : sizeof(BaScalars)}, {&hp, bp}, {&hx, bx}}));
  if (unlocked_wait) hs = g->h_sc;
  GB_CUDA(ctx, cudaMemcpyAsync(hs, dd.sc, sizeof(BaScalars), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CHECK(ba_enqueue_download(ctx, g, hp, hx));
  if (unlocked_wait) {
    GB_CUDA(ctx, cudaEventRecord(g->ev_done, ctx->stream));
    cudaError_t done;
    g->waiting = true;
    {
      CtxUnlock ul(ctx);
      done = cudaEventSynchronize(g->ev_done);
    }
    g->waiting = false;
    GB_CUDA(ctx, done);
  } else {
    GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  if (res) GB_CUDA(ctx, cudaEventElapsedTime(&res->gpu_ms, ev_s, ev_e));
  GB_CHECK(ba_fill_result(ctx, *hs, res));
  if (hp) memcpy(pose_out, hp, bp);
  if (hx) memcpy(pts_out, hx, bx);
  return GB_OK;
}

extern "C" {

int gb_ba_graph_solve(gb_ctx* ctx, gb_ba_graph* g, const gb_ba_options* opt, gb_ba_result* res) {
  return ba_graph_solve_impl(ctx, g, nullptr, opt, res, nullptr, nullptr);
}

int gb_ba_graph_download(gb_ctx* ctx, gb_ba_graph* g, double* cam_pose_wc, double* points) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  const size_t bp = cam_pose_wc ? (size_t)g->d.nc * 56 : 0, bx = points ? (size_t)g->d.np * 24 : 0;
  double *hp, *hx;
  GB_CHECK(gb_stage_take(ctx, {{&hp, bp}, {&hx, bx}}));
  GB_CHECK(ba_enqueue_download(ctx, g, hp, hx));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (hp) memcpy(cam_pose_wc, hp, bp);
  if (hx) memcpy(points, hx, bx);
  return GB_OK;
}

}  // extern "C"

// ---- host-buffer solve with a topology cache ------------------------------------------------------------------------------------
// A SLAM's mapping thread re-solves a sliding window whose graph changes by one keyframe now and then but mostly only in its
// ESTIMATES.  gb_ba_solve keeps the graph of its previous call in a buffer of the cache's own (BaPlace::cache), which no other call
// on the ctx touches; when the next problem has the same cameras / landmarks / edges / masks (exact memcmp of the index arrays,
// ~10 us at the benchmark window) only poses, points and measurements are uploaded -- the ~165 us of sorting, covisibility
// structure, plans and blob fill are skipped.  A problem that misses the cache replaces the kept graph.
struct BaCache {
  gb_ba_graph* g = nullptr;  // the kept graph, if any
  uint8_t* buf = nullptr;    // the grow-only device buffer it lives in
  size_t cap = 0;
  // the topology of g
  int nc = 0, np = 0, no = 0;
  bool has_dof = false, has_pf = false, has_info = false;
  std::vector<int32_t> oc, op;
  std::vector<uint8_t> dof, pf;
  bool matches(const gb_ba_problem* pb) const {
    if (pb->n_cams != nc || pb->n_points != np || pb->n_obs != no) return false;
    if ((pb->cam_dof != nullptr) != has_dof || (pb->point_free != nullptr) != has_pf || (pb->obs_info != nullptr) != has_info) return false;
    if (no > 0 && (memcmp(oc.data(), pb->obs_cam, (size_t)no * 4) != 0 || memcmp(op.data(), pb->obs_point, (size_t)no * 4) != 0)) return false;
    if (has_dof && nc > 0 && memcmp(dof.data(), pb->cam_dof, nc) != 0) return false;
    if (has_pf && np > 0 && memcmp(pf.data(), pb->point_free, np) != 0) return false;
    return true;
  }
  void fill(const gb_ba_problem* pb) {
    nc = pb->n_cams; np = pb->n_points; no = pb->n_obs;
    has_dof = pb->cam_dof != nullptr; has_pf = pb->point_free != nullptr; has_info = pb->obs_info != nullptr;
    oc.assign(pb->obs_cam, pb->obs_cam + no); op.assign(pb->obs_point, pb->obs_point + no);
    if (has_dof) dof.assign(pb->cam_dof, pb->cam_dof + nc); else dof.clear();
    if (has_pf) pf.assign(pb->point_free, pb->point_free + np); else pf.clear();
  }
};

// BaPlace::cache, as gb_slab_alloc: places `layout` in the cache's buffer, which keeps no graph then.  The buffer grows with a
// quarter to spare (sliding windows grow a little at a time), after a synchronisation: nothing may be in flight from the old one.
template <typename F>
static int ba_cache_slab(gb_ctx* ctx, F&& layout) {
  if (!ctx->ba_cache) ctx->ba_cache = new BaCache();
  BaCache& c = *ctx->ba_cache;
  Slab sl;
  layout(sl);
  if (sl.off > c.cap) {
    GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    cudaFree(c.buf);
    c.buf = nullptr;
    c.cap = 0;
    GB_CUDA(ctx, cudaMalloc((void**)&c.buf, sl.off + sl.off / 4));
    c.cap = sl.off + sl.off / 4;
  }
  sl = Slab{c.buf};
  layout(sl);
  return GB_OK;
}

void ba_cache_free(gb_ctx* ctx) {
  if (!ctx->ba_cache) return;
  gb_ba_graph_destroy(ctx, ctx->ba_cache->g);
  cudaFree(ctx->ba_cache->buf);
  delete ctx->ba_cache;
  ctx->ba_cache = nullptr;
}

// new estimates / measurements into a cached graph of the same topology (one pinned blob, three H2D copies, no structure work)
static int ba_graph_refresh(gb_ctx* ctx, gb_ba_graph* g, const gb_ba_problem* pb) {
  BaDev& d = g->d;
  const int nc = d.nc, np = d.np, no = d.no;
  for (int k = 0; k < no; ++k) GB_CHECK(ba_check_z(ctx, pb, k));
  const size_t b_pose = (size_t)nc * 56, b_pts = (size_t)np * 24, b_uv = (size_t)no * 16, b_info = d.has_info ? (size_t)no * 24 : 0;
  double *h_pose, *h_pts, *h_uv, *h_cuv, *h_info;
  GB_CHECK(gb_stage_take(ctx, {{&h_pose, b_pose}, {&h_pts, b_pts}, {&h_uv, b_uv}, {&h_cuv, b_uv}, {&h_info, b_info}}));
  memcpy(h_pose, pb->cam_pose_wc, b_pose);
  memcpy(h_pts, pb->points, b_pts);
  ba_fill_measurements(pb, g->sorted_to_orig, g->cam_perm_h, h_uv, h_cuv, h_info);
  cudaStream_t s = ctx->stream;
  if (nc > 0) GB_CUDA(ctx, cudaMemcpyAsync(g->pose_wc_in, h_pose, b_pose, cudaMemcpyHostToDevice, s));
  if (np > 0) GB_CUDA(ctx, cudaMemcpyAsync(g->pts_init, h_pts, b_pts, cudaMemcpyHostToDevice, s));
  if (no > 0) {
    GB_CUDA(ctx, cudaMemcpyAsync((void*)d.o_uv, h_uv, b_uv, cudaMemcpyHostToDevice, s));
    GB_CUDA(ctx, cudaMemcpyAsync((void*)d.c_uv, h_cuv, b_uv, cudaMemcpyHostToDevice, s));
    if (h_info) GB_CUDA(ctx, cudaMemcpyAsync((void*)d.o_info, h_info, b_info, cudaMemcpyHostToDevice, s));
  }
  if (nc > 0) {
    ba_prepare_kernel<<<gb_div_up(nc, 128), 128, 0, s>>>(nc, g->pose_wc_in, g->pose_init);
    GB_LAUNCH_CHECK(ctx);
  }
  return gb_ba_graph_reset(ctx, g);
}

// the bits of gb_dbg_ba_paths (below)
static int ba_paths(const gb_ba_graph* g) {
  const BaDev& d = g->d;
  bool small, long_rows;
  ba_pcg_sparse_variant(g, &small, &long_rows);
  return (ba_takes_local4(g) ? 1 : 0) | (g->pcg_sparse ? 2 : 0) | (g->pcg_cluster > 0 ? 4 : 0) | (g->pcg_bcsr ? 8 : 0) |
         (g->pcg_bcsr && g->bcsr_cluster > 0 ? 16 : 0) | (d.sp_nchunks > 0 ? 32 : 0) | (ba_sweep_is_large(g) ? 64 : 0) |
         (d.s_nnzb == 0 && d.nc > 0 ? 128 : 0) | (g->chol_ok ? 256 : 0) | (d.cam_split > 1 ? 512 : 0) |
         (g->pcg_sparse && small ? 1024 : 0) | (g->pcg_sparse && long_rows ? 2048 : 0) |
         (d.sp_nchunks > 0 && g->sp_max_nused > kChunkSlotsPerPass ? 4096 : 0);
}

extern "C" int gb_ba_solve(gb_ctx* ctx, gb_ba_problem* pb, const gb_ba_options* opt, gb_ba_result* res) {
  if (!ctx || !pb) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  BaTrace tr;
  gb_ba_graph* g = nullptr;
  BaCache* c = ctx->ba_cache;
  const bool cacheable = pb->n_obs > 0 && pb->n_obs <= (1 << 22) && pb->obs_cam && pb->obs_point && pb->obs_xyz && pb->cam_pose_wc && pb->points &&
                         !getenv("GB_BA_NO_CACHE");
  if (cacheable && c && c->g && c->matches(pb)) {
    g = c->g;
    GB_CHECK(ba_graph_refresh(ctx, g, pb));
    tr.stamp("cached topology: refresh");
  } else {
    if (c) {
      gb_ba_graph_destroy(ctx, c->g);
      c->g = nullptr;
    }
    GB_CHECK(ba_graph_create_impl(ctx, pb, &g, cacheable ? BaPlace::cache : BaPlace::scratch, 0, 1));
    if (cacheable) {
      c = ctx->ba_cache;  // (made by the placement)
      c->fill(pb);
      c->g = g;
    }
  }
  const int rc = ba_graph_solve_impl(ctx, g, nullptr, opt, res, g->d.nc > 0 ? pb->cam_pose_wc : nullptr, g->d.np > 0 ? pb->points : nullptr);
  ctx->ba_last_paths = ba_paths(g);
  tr.stamp("solve + download (one sync)");
  if (!cacheable) gb_ba_graph_destroy(ctx, g);
  return rc;
}

// Optimizer::optimize(BundleGraph&) for graphs with SE3 / GPS edges (pose graph, or bundle adjustment + pose-graph terms)
extern "C" int gb_ba_solve_posegraph(gb_ctx* ctx, gb_ba_problem* pb, const gb_pose_edges* edges, const gb_ba_options* opt, gb_ba_result* res) {
  if (!ctx || !pb) return GB_ERR_INVALID;
  if (!edges || edges->n_se3 + edges->n_gps <= 0) return gb_ba_solve(ctx, pb, opt, res);
  CtxLock lk(ctx);
  gb_ba_graph* g = nullptr;
  GB_CHECK(ba_graph_create_impl(ctx, pb, &g, BaPlace::scratch, 0, 1, edges));
  const int rc = ba_graph_solve_impl(ctx, g, nullptr, opt, res, g->d.nc > 0 ? pb->cam_pose_wc : nullptr, g->d.np > 0 ? pb->points : nullptr);
  gb_ba_graph_destroy(ctx, g);
  return rc;
}

// Cuts the item plan of a graph that now takes the large-graph sweep into its room, after a test hook changed the split or the
// sweep.  The hooks run outside any solve, so its synchronisations cost nothing there.
static int ba_sweep_replan(gb_ctx* ctx, gb_ba_graph* g) {
  BaDev& d = g->d;
  if (!ba_sweep_is_large(g)) return GB_OK;
  std::vector<int> cam_off(d.nc + 1), pt_off(d.np + 1), plan, team_off;
  GB_CUDA(ctx, cudaMemcpyAsync(cam_off.data(), d.cam_off, cam_off.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaMemcpyAsync(pt_off.data(), d.pt_off, pt_off.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  ba_sweep_plan_host(d.nc, d.np, d.cam_split, cam_off, pt_off, ba_sweep_teams(ctx), plan, team_off);
  d.sw_nitems = (int)(plan.size() / 4);
  d.sw_nteams = (int)team_off.size() - 1;
  plan.insert(plan.end(), team_off.begin(), team_off.end());
  int* h;
  GB_CHECK(gb_stage_take(ctx, {{&h, plan.size() * 4}}));
  memcpy(h, plan.data(), plan.size() * 4);
  GB_CUDA(ctx, cudaMemcpyAsync(g->sw_room, h, plan.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  d.sw_items = g->sw_room;
  d.sw_team_off = g->sw_room + 4 * (size_t)d.sw_nitems;
  return GB_OK;
}

int ba_download_S(gb_ctx* ctx, const gb_ba_graph* g, const double* blocks, double* S) {
  const BaDev& d = g->d;
  const size_t n6 = d.n6, nnzb = d.s_nnzb;
  std::vector<double> sb(nnzb * 36);
  std::vector<int> brow(nnzb), col(nnzb);
  GB_CUDA(ctx, cudaMemcpyAsync(sb.data(), blocks, sb.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaMemcpyAsync(brow.data(), d.s_brow, nnzb * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaMemcpyAsync(col.data(), d.s_col, nnzb * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  memset(S, 0, n6 * n6 * sizeof(double));
  for (size_t blk = 0; blk < nnzb; ++blk)
    for (int k = 0; k < 36; ++k) S[(6 * (size_t)brow[blk] + k / 6) * n6 + 6 * (size_t)col[blk] + k % 6] = sb[36 * blk + k];
  return GB_OK;
}

extern "C" {

int gb_ba_pnp(gb_ctx* ctx, int n, const double* xyz, const double* xy1, double* pose_wc, int dof, double* info6x6,
              const gb_ba_options* opt, gb_ba_result* res) {
  if (!ctx || n < 0 || !pose_wc || (n > 0 && (!xyz || !xy1))) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  // optimizePnP == the same solver on a one-camera graph whose landmarks are all fixed (Optimizer.h:202-207)
  std::vector<double> pts(xyz, xyz + 3 * (size_t)n);
  std::vector<uint8_t> pf((size_t)n + 1, 0);
  std::vector<int32_t> oc((size_t)n + 1, 0), op((size_t)n + 1, 0);
  for (int k = 0; k < n; ++k) op[k] = k;
  uint8_t d = (uint8_t)(dof & 63);
  gb_ba_problem pb;
  memset(&pb, 0, sizeof pb);
  pb.n_cams = 1; pb.n_points = n; pb.n_obs = n;
  pb.cam_pose_wc = pose_wc; pb.cam_dof = &d; pb.points = pts.data(); pb.point_free = pf.data();
  pb.obs_cam = oc.data(); pb.obs_point = op.data(); pb.obs_xyz = xy1; pb.obs_info = nullptr;
  gb_ba_graph* g = nullptr;
  GB_CHECK(ba_graph_create_impl(ctx, &pb, &g, BaPlace::scratch, 0, 1));
  int rc = ba_graph_solve_impl(ctx, g, nullptr, opt, res, pose_wc, nullptr);
  ctx->ba_last_paths = ba_paths(g);
  if (rc == GB_OK && info6x6) {
    // information of the returned pose: U at the final estimate (re-linearise once; the graph holds the final state)
    BaScalars h;
    rc = ba_read_scalars(ctx, g, &h);
    if (rc == GB_OK) {
      h.stop = 0; h.need_linearize = 1;
      cudaMemcpyAsync(g->d.sc, &h, sizeof h, cudaMemcpyHostToDevice, ctx->stream);
      ba_linearize_cams_kernel<<<g->d.nc * g->d.cam_split, kCamThreads, 0, ctx->stream>>>(g->d);
      ctx->launches++;
      cudaMemcpyAsync(info6x6, g->d.U, 36 * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream);
      cudaError_t e = cudaStreamSynchronize(ctx->stream);
      if (e != cudaSuccess) { gb_set_error(ctx, "gb_ba_pnp info -> %s", cudaGetErrorString(e)); rc = GB_ERR_CUDA; }
    }
  }
  gb_ba_graph_destroy(ctx, g);
  return rc;
}

// ---- test hooks: expose the intermediates of one linearisation / reduced system in the CALLER's edge order -------------
GB_API int gb_dbg_ba_linearize(gb_ctx* ctx, gb_ba_graph* g, double delta, double* U, double* gc, double* V, double* gp,
                               double* W, double* cost) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  gb_ba_options o;
  gb_ba_options_default(&o);
  o.huber_delta = delta;
  GB_CHECK(gb_ba_graph_begin(ctx, g, &o));
  GB_CHECK(gb_ba_graph_reduce_local(ctx, g, nullptr));
  BaDev& d = g->d;
  const size_t n6 = d.n6;
  std::vector<double> Ws((size_t)d.no * 18 + 1);
  if (U) GB_CUDA(ctx, cudaMemcpyAsync(U, d.U, (size_t)d.nc * 36 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (gc) GB_CUDA(ctx, cudaMemcpyAsync(gc, d.gc, (size_t)d.nc * 6 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (V) GB_CUDA(ctx, cudaMemcpyAsync(V, d.V, (size_t)d.np * 9 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (gp) GB_CUDA(ctx, cudaMemcpyAsync(gp, d.gp, (size_t)d.np * 3 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (W) GB_CUDA(ctx, cudaMemcpyAsync(Ws.data(), d.W, (size_t)d.no * 18 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (cost) GB_CUDA(ctx, cudaMemcpyAsync(cost, g->buf + n6 * n6 + 2 * n6, 8, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (W)
    for (int e = 0; e < d.no; ++e) memcpy(W + 18 * (size_t)g->sorted_to_orig[e], Ws.data() + 18 * (size_t)e, 18 * 8);
  return GB_OK;
}

// mode: 0 = whatever gb_ba_graph_solve would use, 1 = force the generic multi-kernel PCG
GB_API int gb_dbg_ba_reduced(gb_ctx* ctx, gb_ba_graph* g, const gb_ba_options* opt, double* S, double* gt, double* dc,
                             int* pcg_iters) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  GB_CHECK(gb_ba_graph_begin(ctx, g, opt));
  GB_CHECK(gb_ba_graph_reduce_local(ctx, g, nullptr));
  GB_CHECK(gb_ba_graph_step(ctx, g, nullptr, nullptr));
  BaDev& d = g->d;
  const size_t n6 = d.n6;
  if (S && g->pcg_sparse && d.s_nnzb > 0 && d.nc > 0) GB_CHECK(ba_download_S(ctx, g, d.Sb, S));  // (the local-BA path keeps S as block-CSR)
  else if (S) GB_CUDA(ctx, cudaMemcpyAsync(S, g->buf, n6 * n6 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (gt) GB_CUDA(ctx, cudaMemcpyAsync(gt, g->buf + n6 * n6, n6 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (dc) GB_CUDA(ctx, cudaMemcpyAsync(dc, d.x, n6 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  BaScalars h;
  GB_CHECK(ba_read_scalars(ctx, g, &h));
  if (pcg_iters) *pcg_iters = h.pcg_iters;
  return GB_OK;
}

// The linear system one LM step of this graph would solve, and the answer of the solver that step would run: begin, the
// reduction onto the layout a solve uses (the compact block-CSR one when the multi-CTA block-CSR PCG solves it), then that
// solver alone -- single-CTA sparse, one-cluster, generic or block-CSR PCG, or the direct solver.  Out, each where non-null: S
// (6N x 6N dense, UNDAMPED, read before the solver damps its copy), g~ and diag U (n6 each), lambda (the damped system is S with
// lm_damp(S_dd, diagU_d, lambda) on its diagonal), the solution x (n6) and the PCG iterations (0 for the direct solver).
GB_API int gb_dbg_ba_system(gb_ctx* ctx, gb_ba_graph* g, const gb_ba_options* opt, double* S, double* gt, double* diagU,
                            double* lambda, double* x, int* pcg_iters) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  GB_CHECK(gb_ba_graph_begin(ctx, g, opt));
  const BaDev& d = g->d;
  const size_t n6 = d.n6, nnzb = d.s_nnzb;
  const bool compact = ba_iterates_compact(g, nullptr);
  // where S is read from: the compact buffer, the block-CSR values (the single-CTA PCG and the direct solver read only those), or
  // the dense layout (one-cluster / generic PCG, pose-graph coupling included)
  const bool dense_S = !compact && !(nnzb > 0 && (g->pcg_sparse || g->opt.linear_solver == 1));
  const double* tail = compact ? g->rbuf + nnzb * 36 : g->buf + n6 * n6;
  if (compact) GB_CHECK(ba_compact_reduce(ctx, g, nullptr));
  else GB_CHECK(gb_ba_graph_reduce_local(ctx, g, nullptr));
  if (S && dense_S) GB_CUDA(ctx, cudaMemcpyAsync(S, g->buf, n6 * n6 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  else if (S) GB_CHECK(ba_download_S(ctx, g, compact ? g->rbuf : d.Sb, S));
  if (gt) GB_CUDA(ctx, cudaMemcpyAsync(gt, tail, n6 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (diagU) GB_CUDA(ctx, cudaMemcpyAsync(diagU, tail + n6, n6 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // (the solver below damps S in place on some paths)
  if (compact) GB_CHECK(ba_pcg_bcsr_launch(ctx, g, g->rbuf));
  else GB_CHECK(ba_pcg_dispatch(ctx, g, g->buf));
  if (x) GB_CUDA(ctx, cudaMemcpyAsync(x, d.x, n6 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  BaScalars h;
  GB_CHECK(ba_read_scalars(ctx, g, &h));
  if (lambda) *lambda = h.lambda;
  if (pcg_iters) *pcg_iters = h.pcg_iters;
  return GB_OK;
}

// What the graph's last LM iteration left on the device, copied back without a launch, each where non-null: the camera step x (n6),
// the damped landmark inverses V~^-1 (np x 9: at the lambda of that iteration, or at the new one after a rejection on the local-BA
// chain, which refreshes them) and the candidate landmarks pts_new (np x 3).  Landmarks in the caller's order (of this shard).
GB_API int gb_dbg_ba_last_step(gb_ctx* ctx, gb_ba_graph* g, double* x, double* vinv, double* pts_new) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  const BaDev& d = g->d;
  if (x && d.n6 > 0) GB_CUDA(ctx, cudaMemcpyAsync(x, d.x, (size_t)d.n6 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (vinv && d.np > 0) GB_CUDA(ctx, cudaMemcpyAsync(vinv, d.Vinv, (size_t)d.np * 9 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (pts_new && d.np > 0) GB_CUDA(ctx, cudaMemcpyAsync(pts_new, d.pts_new, (size_t)d.np * 3 * 8, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return GB_OK;
}

// force (1) / release (0) the generic multi-kernel PCG on this graph — lets the tests cover both solver paths
// on: 0 = automatic dispatch, 1 = generic multi-kernel PCG, 2 = one-cluster DSMEM PCG (if it fits), 3 = single-CTA sparse,
// 4 = one-cluster DSMEM PCG in a cluster of 8 CTAs (the size taken where 16-CTA clusters are not available)
GB_API int gb_dbg_ba_force_generic_pcg(gb_ctx* ctx, gb_ba_graph* g, int on) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  ba_pick_pcg(ctx, g, on == 4 ? 8 : 16);
  if (g->d.npe > 0) g->pcg_sparse = false;  // (pose-graph terms live on the dense reduced system)
  if (on == 1) { g->pcg_cluster = 0; g->pcg_sparse = false; }
  if (on == 2 || on == 4) g->pcg_sparse = false;
  if (on == 3) g->pcg_cluster = 0;
  return GB_OK;
}

GB_API int gb_dbg_ba_pcg_sparse(gb_ctx* ctx, gb_ba_graph* g) { return (ctx && g) ? (g->pcg_sparse ? g->d.s_nnzb : 0) : -1; }

// force the camera-pass split (1..4 CTAs per camera; the partial-sum buffer always has room for 4): lets the tests cover the
// sliced path on small graphs
GB_API int gb_dbg_ba_set_cam_split(gb_ctx* ctx, gb_ba_graph* g, int split) {
  if (!ctx || !g || split < 1 || split > 4) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  g->d.cam_split = split;
  return ba_sweep_replan(ctx, g);  // (the large-graph sweep's items are cut per slice)
}

// one half of the sweep alone (which = 1: camera pass, 2: landmark pass, 3: both) -- timing experiments (tools/sweep_bench.py)
GB_API int gb_dbg_ba_sweep_part(gb_ctx* ctx, gb_ba_graph* g, int which) {
  if (!ctx || !g || !g->begun) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  BaDev& d = g->d;
  if (which < 1 || which > 3) return GB_ERR_INVALID;
  return ba_launch_sweep(ctx, g, d, ctx->stream, which);
}

// 0 = pick by size, 1 = the latency-tuned kernel of this file, 2 = the bandwidth-tuned kernel of ba_sweep.cu (tests cover both on
// the same graphs)
GB_API int gb_dbg_ba_set_sweep(gb_ctx* ctx, gb_ba_graph* g, int mode) {
  if (!ctx || !g || mode < 0 || mode > 2) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  g->sweep_mode = mode;
  return ba_sweep_replan(ctx, g);
}

GB_API int gb_dbg_ba_pcg_cluster_size(gb_ctx* ctx, gb_ba_graph* g) { return (ctx && g) ? g->pcg_cluster : -1; }

// What a solve of this graph would run, as it is planned now (after any of the hooks above), one bit per host-side decision:
//   1 local4: the 4-launch local-BA chain          2 pcg_sparse: single-CTA block-sparse PCG    4 one-cluster PCG (pcg_cluster > 0)
//   8 pcg_bcsr: compact block-CSR PCG               16 ... in one thread-block cluster (else as a cooperative grid)
//   32 landmark-chunk Schur plan (else block gather)   64 persistent large-graph sweep (ba_sweep.cu)
//   128 no block structure: dense Schur by fp64 atomics   256 chol_ok: the direct solver fits   512 camera pass sliced (cam_split > 1)
//   1024 ... the single-CTA sparse PCG in its 12-warp instantiation (<= kSpSmallCams active cameras; else the 20-warp one)
//   2048 ... in its variant for block rows longer than the register columns (shared-memory mat-vec tail)
//   4096 a chunk of the landmark-chunk Schur plan uses more than 80 slots: ba_schur_chunks_kernel runs its second slot pass
// Tests assert these bits so that a threshold change cannot quietly turn one path's test into a duplicate of another's.
GB_API int gb_dbg_ba_paths(gb_ctx* ctx, gb_ba_graph* g) { return (ctx && g) ? ba_paths(g) : -1; }

// gb_dbg_ba_paths of the last graph a host-buffer call (gb_ba_solve / gb_ba_pnp) solved on this ctx, taken after its solve
GB_API int gb_dbg_ba_last_paths(gb_ctx* ctx) { return ctx ? ctx->ba_last_paths : -1; }

// clock64 stamps of PCG iteration 3 on CTA 0 (8 values): enable, solve, then read
GB_API int gb_dbg_ba_pcg_profile(gb_ctx* ctx, gb_ba_graph* g, long long* out8) {
  if (!ctx || !g) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  if (!g->d.prof) {
    g->d.prof = g->prof_room;
    GB_CUDA(ctx, cudaMemsetAsync(g->d.prof, 0, 64, ctx->stream));
    return GB_OK;
  }
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  GB_CUDA(ctx, cudaMemcpy(out8, g->d.prof, 64, cudaMemcpyDeviceToHost));
  return GB_OK;
}

}  // extern "C"
