// gslam_b200/csrc/ba_pcg_bcsr.cu — block-Jacobi PCG on the reduced camera system of a LARGE bundle adjustment (global BA:
// hundreds of cameras), kept in covisibility block-CSR, solved by ONE persistent cooperative kernel.
// Behind GSLAM::Optimizer::optimize(BundleGraph&) (GSLAM/core/Optimizer.h:229); same Chronopoulos-Gear recurrence as the
// CPU checker (oracle/ba_ref.c::ba_pcg) and as the generic multi-kernel path it replaces (ba.cu: pcg_matvec / pcg_update).
//
// Why: at BASELINE config 5 (500 cameras / 100k landmarks / 1M observations) the dense S is 72 MB and one PCG iteration of the
// generic path is two launches that re-read it from HBM; the covisibility fill is ~20 %, so block-CSR S is ~14 MB -- 109 KB per SM
// when the block rows are dealt out over the 132 SMs, i.e. it FITS IN SHARED MEMORY for the whole solve.  What remains per
// iteration is latency: two grid barriers (the inner products; the publication of u = M^-1 r), a 24 KB read of u from L2 and
// ~12 k DFMA per CTA.  The same kernel runs replicated and bit-identically on every rank of the landmark-sharded solve (the
// all-reduced compact system is its input), so the ranks take identical LM decisions without any broadcast.
//
//   CTA c owns the contiguous block rows (cameras) [cta_cam[c], cta_cam[c+1]) -- balanced by block count on the host.
//   A local row (camera, component) is worked by K lanes (K = 2^k <= 32, chosen on the host so that rows * K fills the CTA):
//   lane `sub` takes blocks sub, sub+K, ... of the block row, 6 DFMA each, then a fixed xor tree over the K lanes.
//   Reductions are fixed-order everywhere (shuffle trees, per-warp partials summed in order, per-CTA partials summed in order by
//   every CTA): run-to-run and rank-to-rank bit-reproducible.
#include "ba_internal.cuh"

#include <cooperative_groups.h>

#include <algorithm>
#include <mutex>

using namespace ba;

namespace {

constexpr int kBcsrThreads = 512;
constexpr int kBlkStride = 38;  // doubles per 6x6 block in shared memory: 304 B keeps 16-byte alignment for LDS.128 and spreads the
                                // lanes of a camera (consecutive blocks) over distinct bank groups

struct BcsrArgs {
  const int* cta_cam;   // [G+1]
  double* part;         // [2G] per-CTA (gamma, delta)
  double* u_glob;       // [n6]
  unsigned int* bar;    // grid barrier counter (zeroed before the launch)
  int K, in_smem, maxit, max_cams, max_blocks, blk_stride;
  unsigned short need[16];  // CLUSTER: need[c] = which CTAs of the cluster read camera rows owned by CTA c (covisibility), self included
};

__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// All CTAs are co-resident (cooperative launch).  Monotonic ticket barrier: phase t completes when the counter reaches t*G.
__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int& target, unsigned int G) {
  __syncthreads();
  if (threadIdx.x == 0) {
    target += G;
    __threadfence();
    atomicAdd(bar, 1u);
    while (ld_acquire_u32(bar) < target) {}
    __threadfence();
  }
  __syncthreads();
}

// CLUSTER = true: the whole grid is ONE thread-block cluster (<= 16 CTAs, chosen on the host when S fits their shared memory):
// u and the per-CTA (gamma, delta) partials travel through distributed shared memory and the two barriers per iteration are
// hardware cluster barriers (~0.2 us) instead of a global-memory ticket barrier (one CTA per SM).
template <bool CLUSTER>
__global__ void __launch_bounds__(kBcsrThreads, 1) ba_pcg_bcsr_kernel(BaDev g, double* __restrict__ rbuf, BcsrArgs a) {
  namespace cg = cooperative_groups;
  if (g.sc->stop) return;  // uniform over the grid
  extern __shared__ __align__(16) double sm[];
  __shared__ double s_warp[2][kBcsrThreads / 32];
  __shared__ double s_scal[4];  // gamma, delta, alpha, beta (this iteration), broadcast
  __shared__ int s_go;
  __shared__ double s_cpart[2][16];  // CLUSTER: (gamma, delta) partials of every CTA of the cluster, written by the peers
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, G = gridDim.x, b = blockIdx.x;
  const int n6 = g.n6;
  const int cam0 = a.cta_cam[b], cam1 = a.cta_cam[b + 1], ncl = cam1 - cam0, rows = 6 * ncl;
  const int blk0 = g.s_rowptr[cam0], blk1 = g.s_rowptr[cam1], nb = blk1 - blk0;
  // ---- shared-memory carve-up (sizes from the host plan: max over CTAs) ----
  double* u_full = sm;                                         // [n6]
  double* vec = u_full + ((n6 + 1) & ~1);                      // r, p, s, x, w, u_own : 6 x [6*max_cams]
  const int vstride = 6 * a.max_cams;
  double *vr = vec, *vp = vec + vstride, *vs = vec + 2 * vstride, *vx = vec + 3 * vstride, *vw = vec + 4 * vstride, *vu = vec + 5 * vstride;
  double* Minv = vec + 6 * vstride;                            // [max_cams][36]
  double* Ssm = Minv + 36 * a.max_cams;                        // [max_blocks][37] when in_smem
  int* col = reinterpret_cast<int*>(Ssm + (a.in_smem ? (size_t)a.max_blocks * a.blk_stride : 0));  // [max_blocks]
  int* rp = col + a.max_blocks;                                // [max_cams + 1]
  const size_t r_gt = (size_t)g.s_nnzb * 36;
  const double lambda = g.sc->lambda, tol = g.sc->pcg_tol;

  // ---- A. block structure + values of the owned block rows ----
  for (int t = tid; t < nb; t += kBcsrThreads) col[t] = g.s_col[blk0 + t];
  for (int t = tid; t <= ncl; t += kBcsrThreads) rp[t] = g.s_rowptr[cam0 + t] - blk0;
  double* Sg = rbuf + (size_t)blk0 * 36;  // the owned blocks in global memory
  if (a.in_smem) {
    const int n = nb * 36;
    for (int t = tid; t < n; t += kBcsrThreads) Ssm[(t / 36) * a.blk_stride + (t % 36)] = __ldcg(Sg + t);
  }
  __syncthreads();
  const double* Sp = a.in_smem ? Ssm : Sg;
  const int bstride = a.in_smem ? a.blk_stride : 36;
  // ---- B. Marquardt damping of the diagonal (fixed dofs: unit diagonal), then the 6x6 block-Jacobi inverses ----
  for (int r = tid; r < rows; r += kBcsrThreads) {
    const int c = r / 6, comp = r - 6 * c, cam = cam0 + c;
    int diag = -1;
    for (int t = rp[c]; t < rp[c + 1]; ++t)
      if (col[t] == cam) diag = t;
    if (diag >= 0) {
      double* e = (a.in_smem ? Ssm + (size_t)diag * a.blk_stride : Sg + (size_t)diag * 36) + comp * 7;
      const double du = __ldcg(rbuf + r_gt + n6 + 6 * cam + comp);
      *e = lm_damp(*e, du, lambda, (g.dof[cam] >> comp) & 1);
    }
  }
  __syncthreads();
  for (int c = tid; c < ncl; c += kBcsrThreads) {
    const int cam = cam0 + c;
    int diag = rp[c];
    for (int t = rp[c]; t < rp[c + 1]; ++t)
      if (col[t] == cam) diag = t;
    const double* D = Sp + (size_t)diag * bstride;
    double M[36];
#pragma unroll
    for (int k = 0; k < 36; ++k) M[k] = D[k];
    block_jacobi_inverse(M, D, 6);
#pragma unroll
    for (int k = 0; k < 36; ++k) Minv[36 * c + k] = M[k];
  }
  for (int r = tid; r < rows; r += kBcsrThreads) {
    vr[r] = __ldcg(rbuf + r_gt + 6 * cam0 + r);
    vp[r] = 0.0; vs[r] = 0.0; vx[r] = 0.0;
  }
  __syncthreads();
  // u = Minv r for the owned rows, published for everybody
  auto apply_minv_publish = [&]() {
    for (int r = tid; r < rows; r += kBcsrThreads) {
      const int c = r / 6, comp = r - 6 * c;
      double s = 0.0;
#pragma unroll
      for (int k = 0; k < 6; ++k) s += Minv[36 * c + comp * 6 + k] * vr[6 * c + k];
      vu[r] = s;
      if (!CLUSTER) a.u_glob[6 * cam0 + r] = s;
    }
    if (CLUSTER) {  // push the owned rows into every CTA's copy of u (pairs of rows: 16-byte remote stores)
      __syncthreads();
      cg::cluster_group cluster = cg::this_cluster();
      const int pairs = rows >> 1;  // rows = 6 * cameras: even
      const unsigned int need = a.need[b];
      for (int t = tid; t < pairs * G; t += kBcsrThreads) {
        const int peer = t / pairs, q = t - peer * pairs;
        if (!((need >> peer) & 1u)) continue;  // that CTA has no block in these columns: it never reads them
        double* pu = cluster.map_shared_rank(u_full, peer);
        *reinterpret_cast<double2*>(pu + 6 * cam0 + 2 * q) = make_double2(vu[2 * q], vu[2 * q + 1]);
      }
    }
  };
  unsigned int target = 0;
  auto barrier = [&]() {
    if (CLUSTER) cg::this_cluster().sync();
    else grid_barrier(a.bar, target, G);
  };
  apply_minv_publish();
  barrier();
  // optional phase clocks (test hook gb_dbg_ba_pcg_profile): CTA 0 / thread 0 accumulates [setup, mat-vec + local dots, barrier 1,
  // scalars + recurrences + publication, barrier 2, total, iterations]
  const bool prof = g.prof != nullptr && b == 0 && tid == 0;
  long long pc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, t_prev = clock64();
  const long long t_begin = t_prev;
  auto stamp = [&](int k) { if (prof) { const long long t = clock64(); pc[k] += t - t_prev; t_prev = t; } };

  const int K = a.K, sub = tid & (K - 1), groups = kBcsrThreads / K;
  double gamma_prev = 0.0, gamma0 = 0.0, alpha_prev = 1.0;
  int k_it = 0;
  bool first = true;
  for (;;) {
    // ---- C. w = S u on the owned rows ----
    if (!CLUSTER) {
      for (int t = tid; t < n6; t += kBcsrThreads) u_full[t] = __ldcg(a.u_glob + t);
      __syncthreads();
    }
    // K lanes per CAMERA (K = 2^k <= 32): lane `sub` takes whole blocks sub, sub+K, ... of the block row -- the 36 coefficients and
    // the six entries of u with 16-byte shared-memory loads, 36 DFMA in six independent chains -- then a fixed xor tree over the K
    // lanes.  (One lane per ROW re-read u six times per block and moved 8 bytes per load: the mat-vec was shared-memory-bound.)
    double pg = 0.0, pd = 0.0;
    for (int cbase = 0; cbase < ncl; cbase += groups) {  // (uniform trip count: whole groups of K lanes share a camera)
      const int c = cbase + tid / K;
      double r0 = 0.0, r1 = 0.0, r2 = 0.0, r3 = 0.0, r4 = 0.0, r5 = 0.0;
      if (c < ncl) {
        for (int t = rp[c] + sub; t < rp[c + 1]; t += K) {
          const double2* B2 = reinterpret_cast<const double2*>(Sp + (size_t)t * bstride);
          const double2* U2 = reinterpret_cast<const double2*>(u_full + 6 * col[t]);
          const double2 ua = U2[0], ub = U2[1], uc = U2[2];
#define GB_ROW(acc, k)                                                                              \
          { const double2 s0 = B2[3 * (k)], s1 = B2[3 * (k) + 1], s2 = B2[3 * (k) + 2];              \
            acc = fma(s0.x, ua.x, fma(s0.y, ua.y, fma(s1.x, ub.x, fma(s1.y, ub.y, fma(s2.x, uc.x, fma(s2.y, uc.y, acc)))))); }
          GB_ROW(r0, 0) GB_ROW(r1, 1) GB_ROW(r2, 2) GB_ROW(r3, 3) GB_ROW(r4, 4) GB_ROW(r5, 5)
#undef GB_ROW
        }
      }
      for (int o = K >> 1; o > 0; o >>= 1) {
        r0 += __shfl_xor_sync(0xffffffffu, r0, o); r1 += __shfl_xor_sync(0xffffffffu, r1, o); r2 += __shfl_xor_sync(0xffffffffu, r2, o);
        r3 += __shfl_xor_sync(0xffffffffu, r3, o); r4 += __shfl_xor_sync(0xffffffffu, r4, o); r5 += __shfl_xor_sync(0xffffffffu, r5, o);
      }
      if (c < ncl && sub < 6) {  // (K >= 8 always holds here: lanes 0..5 of the camera publish one row each)
        const double v = sub == 0 ? r0 : sub == 1 ? r1 : sub == 2 ? r2 : sub == 3 ? r3 : sub == 4 ? r4 : r5;
        const int r = 6 * c + sub;
        vw[r] = v;
        pg += vr[r] * vu[r];
        pd += v * vu[r];
      }
    }
    stamp(5);  // (own mat-vec + lane reduction done)
    // ---- D. (gamma, delta): fixed tree inside the CTA, per-CTA partials folded in CTA order by everybody ----
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      pg += __shfl_down_sync(0xffffffffu, pg, o);
      pd += __shfl_down_sync(0xffffffffu, pd, o);
    }
    if (lane == 0) { s_warp[0][warp] = pg; s_warp[1][warp] = pd; }
    __syncthreads();
    stamp(6);  // (everybody's mat-vec done)
    if (CLUSTER) {
      if (tid < G) {  // thread p hands this CTA's partial pair to peer p
        double sg = 0.0, sd = 0.0;
#pragma unroll
        for (int w = 0; w < kBcsrThreads / 32; ++w) { sg += s_warp[0][w]; sd += s_warp[1][w]; }
        cg::cluster_group cluster = cg::this_cluster();
        double* pp = cluster.map_shared_rank(&s_cpart[0][0], tid);
        pp[b] = sg;
        pp[16 + b] = sd;
      }
    } else if (tid == 0) {
      double sg = 0.0, sd = 0.0;
#pragma unroll
      for (int w = 0; w < kBcsrThreads / 32; ++w) { sg += s_warp[0][w]; sd += s_warp[1][w]; }
      a.part[2 * b] = sg;
      a.part[2 * b + 1] = sd;
    }
    stamp(1);
    barrier();
    stamp(2);
    if (warp == 0) {
      double sg = 0.0, sd = 0.0;
      if (CLUSTER) {
        if (lane < G) { sg = s_cpart[0][lane]; sd = s_cpart[1][lane]; }
      } else {
        for (int c = lane; c < G; c += 32) { sg += __ldcg(a.part + 2 * c); sd += __ldcg(a.part + 2 * c + 1); }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        sg += __shfl_down_sync(0xffffffffu, sg, o);
        sd += __shfl_down_sync(0xffffffffu, sd, o);
      }
      if (lane == 0) { s_scal[0] = sg; s_scal[1] = sd; }
    }
    // lane 0 of warp 0 alone runs the scalar recurrences (three fp64 divisions cost ~340 clk of dependent latency AND fp64-pipe
    // time in every warp that repeats them); everybody reads (alpha, beta, verdict) after the barrier
    if (tid == 0) {
      const double gn = s_scal[0], dl = s_scal[1];
      double alpha = 0.0, beta = 0.0;
      int go = 1;
      if (first) {
        gamma0 = gn;
        if (!(gn > 0.0) || !(dl > 0.0)) go = 0;
        else alpha = gn / dl;
      } else {
        if (!(gn > 0.0) || gn < tol * tol * gamma0) go = 0;  // convergence test of the previous update
        else {
          beta = gn / gamma_prev;
          const double den = dl - beta * gn / alpha_prev;
          if (!(den > 0.0)) go = 0;
          else alpha = gn / den;
        }
      }
      if (k_it >= a.maxit) go = 0;
      gamma_prev = gn; alpha_prev = alpha;
      s_scal[2] = alpha; s_scal[3] = beta; s_go = go;
    }
    __syncthreads();
    if (!s_go) break;
    const double alpha = s_scal[2], beta = s_scal[3];
    // ---- E. element-wise recurrences on the owned rows, u = Minv r, publish ----
    for (int r = tid; r < rows; r += kBcsrThreads) {
      const double pn = vu[r] + beta * vp[r];
      const double sn = vw[r] + beta * vs[r];
      vp[r] = pn;
      vs[r] = sn;
      vx[r] += alpha * pn;
      vr[r] -= alpha * sn;
    }
    __syncthreads();
    apply_minv_publish();
    first = false; ++k_it;
    stamp(3);
    barrier();
    stamp(4);
  }
  if (prof) {
    g.prof[0] = pc[5]; g.prof[1] = pc[1]; g.prof[2] = pc[2]; g.prof[3] = pc[3]; g.prof[4] = pc[4]; g.prof[5] = clock64() - t_begin; g.prof[6] = k_it;
    g.prof[7] = pc[6];
  }
  // ---- F. solution + retraction of the owned cameras ----
  for (int r = tid; r < rows; r += kBcsrThreads) g.x[6 * cam0 + r] = vx[r];
  for (int c = tid; c < ncl; c += kBcsrThreads) retract_camera(g, cam0 + c, vx + 6 * c);
  if (b == 0 && tid == 0) g.sc->pcg_iters += k_it;
  if (CLUSTER) cg::this_cluster().sync();  // nobody leaves while a peer could still address its shared memory
}

size_t bcsr_smem_bytes(int n6, int max_cams, int max_blocks, bool in_smem, int blk_stride = kBlkStride) {
  size_t d = (size_t)((n6 + 1) & ~1) + 6 * (size_t)6 * max_cams + 36 * (size_t)max_cams + (in_smem ? (size_t)max_blocks * blk_stride : 0);
  return d * sizeof(double) + ((size_t)max_blocks + max_cams + 1) * sizeof(int) + 64;
}

}  // namespace

// contiguous camera ranges for G CTAs, balanced by block count, at least one camera each
static void bcsr_partition(int nc, int nnzb, const int* s_rowptr, int G, std::vector<int>& cta_cam, int* max_cams, int* max_blocks) {
  cta_cam.assign(G + 1, nc);
  int cam = 0;
  for (int c = 0; c < G; ++c) {
    cta_cam[c] = cam;
    const long long want = (long long)nnzb * (c + 1) / G;  // block count that should be covered after this CTA
    const int left_ctas = G - 1 - c;
    while (cam < nc - left_ctas && (s_rowptr[cam + 1] <= want || cam == cta_cam[c])) ++cam;
  }
  cta_cam[G] = nc;
  *max_cams = 1; *max_blocks = 1;
  for (int c = 0; c < G; ++c) {
    *max_cams = std::max(*max_cams, cta_cam[c + 1] - cta_cam[c]);
    *max_blocks = std::max(*max_blocks, s_rowptr[cta_cam[c + 1]] - s_rowptr[cta_cam[c]]);
  }
}

void ba_pcg_bcsr_plan(gb_ctx* ctx, gb_ba_graph* g, const int* s_rowptr, const int* s_col_host, std::vector<int>& cta_cam) {
  g->pcg_bcsr = false;
  const int nc = g->d.nc, nnzb = g->d.s_nnzb, n6 = g->d.n6;
  if (nc <= 0 || nnzb <= 0) return;
  bool cluster16_ok = false;
  if (!gb_func_setup(ctx, (const void*)ba_pcg_bcsr_kernel<false>, GB_SMEM_OPTIN_MAX) ||
      !gb_func_setup(ctx, (const void*)ba_pcg_bcsr_kernel<true>, GB_SMEM_OPTIN_MAX, &cluster16_ok))
    return;
  const size_t budget = (size_t)ctx->max_smem_optin - 2048;  // (static shared memory of the kernel: < 1 KB)
  int G = 0, max_cams = 1, max_blocks = 1, cluster = 0, blk_stride = kBlkStride;
  bool in_smem = true;
  size_t smem = 0;
  // 1) ONE thread-block cluster when S fits the shared memory of <= 16 (8 without the non-portable size) CTAs
  if (!getenv("GB_BA_NO_PCG_CLUSTER")) {
    const int sizes[2] = {16, 8};
    for (int t = 0; t < 2 && !cluster; ++t) {
      const int C = std::min(sizes[t], nc);
      if (C > 8 && !cluster16_ok) continue;
      int mc, mb;
      bcsr_partition(nc, nnzb, s_rowptr, C, cta_cam, &mc, &mb);
      const int strides[2] = {kBlkStride, 36};  // (36: 2-way bank conflicts on the block loads, but 6 % less shared memory)
      for (int q = 0; q < 2 && !cluster; ++q) {
        const size_t need = bcsr_smem_bytes(n6, mc, mb, true, strides[q]);
        if (need > budget) continue;
        GbClusterConfig lc(C, dim3(kBcsrThreads), need, ctx->stream);
        int nclusters = 0;
        if (cudaOccupancyMaxActiveClusters(&nclusters, ba_pcg_bcsr_kernel<true>, &lc.cfg) != cudaSuccess || nclusters < 1) { cudaGetLastError(); continue; }
        cluster = C; G = C; max_cams = mc; max_blocks = mb; blk_stride = strides[q]; smem = need;
      }
    }
  }
  // 2) otherwise a cooperative grid, one CTA per SM at most, global-memory barrier
  if (!cluster) {
    int coop = 0;
    cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, ctx->device);
    if (!coop) return;
    G = std::max(1, std::min(ctx->sm_count, nc));
    bcsr_partition(nc, nnzb, s_rowptr, G, cta_cam, &max_cams, &max_blocks);
    smem = bcsr_smem_bytes(n6, max_cams, max_blocks, true);
    if (smem > budget) {
      in_smem = false;
      smem = bcsr_smem_bytes(n6, max_cams, max_blocks, false);
      if (smem > budget) return;  // not even the vectors fit: generic path
    }
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ba_pcg_bcsr_kernel<false>, kBcsrThreads, smem) != cudaSuccess || per_sm < 1) {
      cudaGetLastError();
      return;
    }
    if ((long long)per_sm * ctx->sm_count < G) return;
  }
  int K = 32;  // lanes per camera in the mat-vec (>= 8: lanes 0..5 publish the six rows)
  while (K > 8 && max_cams * K > kBcsrThreads) K >>= 1;
  g->bcsr_ctas = G; g->bcsr_K = K; g->bcsr_in_smem = in_smem ? 1 : 0; g->bcsr_smem = smem;
  g->bcsr_max_cams = max_cams; g->bcsr_max_blocks = max_blocks; g->bcsr_cluster = cluster; g->bcsr_blk_stride = blk_stride;
  // who reads whose rows of u (cluster mode: the publication of u only goes where it is needed)
  for (int c = 0; c < 16; ++c) g->bcsr_need[c] = 0;
  if (cluster) {
    std::vector<int> owner(nc, 0);
    for (int c = 0; c < G; ++c)
      for (int i = cta_cam[c]; i < cta_cam[c + 1]; ++i) owner[i] = c;
    for (int p = 0; p < G; ++p) {
      g->bcsr_need[p] |= (unsigned short)(1u << p);
      for (int t = s_rowptr[cta_cam[p]]; t < s_rowptr[cta_cam[p + 1]]; ++t) g->bcsr_need[owner[s_col_host[t]]] |= (unsigned short)(1u << p);
    }
  }
  g->pcg_bcsr = true;
}

int ba_pcg_bcsr_launch(gb_ctx* ctx, gb_ba_graph* g, const double* rbuf) {
  if (!ctx || !g || !g->pcg_bcsr || !rbuf) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  BaDev d = g->d;
  d.r_gt = (size_t)d.s_nnzb * 36;
  BcsrArgs a;
  a.cta_cam = g->bcsr_cta_cam; a.part = g->bcsr_part; a.u_glob = g->bcsr_u; a.bar = g->bcsr_bar;
  a.K = g->bcsr_K; a.in_smem = g->bcsr_in_smem; a.maxit = g->opt.pcg_max_iters; a.max_cams = g->bcsr_max_cams; a.max_blocks = g->bcsr_max_blocks;
  a.blk_stride = g->bcsr_blk_stride;
  for (int c = 0; c < 16; ++c) a.need[c] = g->bcsr_need[c];
  double* rb = const_cast<double*>(rbuf);  // (the damped diagonal is written back when S stays in global memory)
  if (g->bcsr_cluster > 0) {
    GbClusterConfig lc(g->bcsr_cluster, dim3(kBcsrThreads), g->bcsr_smem, ctx->stream);
    GB_CUDA(ctx, cudaLaunchKernelEx(&lc.cfg, ba_pcg_bcsr_kernel<true>, d, rb, a));
  } else {
    GB_CUDA(ctx, cudaMemsetAsync(g->bcsr_bar, 0, 4, ctx->stream));
    void* args[3] = {(void*)&d, (void*)&rb, (void*)&a};
    GB_CUDA(ctx, cudaLaunchCooperativeKernel((const void*)ba_pcg_bcsr_kernel<false>, dim3(g->bcsr_ctas), dim3(kBcsrThreads), args, g->bcsr_smem, ctx->stream));
  }
  GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}
