// gslam_b200/csrc/ba_chol.cu — DIRECT solve of the reduced camera system of a local bundle adjustment: block (6x6) skyline
// Cholesky + forward / backward substitution + retraction, ONE CTA, everything in shared memory.
// Behind GSLAM::Optimizer::optimize(BundleGraph&) (GSLAM/core/Optimizer.h:229), selected with gb_ba_options::linear_solver = 1;
// the CPU checker solves the same system with a dense Cholesky (oracle/ba_ref.c::ba_chol_solve).
//
// Why: the block-Jacobi PCG of the local path is a ~2 k-clock dependent chain per iteration on one SM and is capped at 50
// iterations (an INEXACT solve: 70 us per LM iteration at the benchmark window).  The reduced system of a sliding window is a
// narrow band of 6x6 blocks (keyframe i is covisible with i +- 4): its skyline holds a few hundred blocks, the factorisation is
// ~50 block steps of [6x6 Cholesky (one thread, registers) | panel solve | trailing update] and the two substitutions are ~100
// short steps -- about half the time of the 50 PCG iterations, and the solve is EXACT, so LM needs fewer iterations to converge.
// Natural (time) camera order; no fill outside the (monotone) skyline; applies while the skyline fits one SM's shared memory
// (ba_chol_plan), otherwise the solver option is refused loudly.
#include "ba_internal.cuh"

#include <algorithm>
#include <mutex>

using namespace ba;

namespace {

constexpr int kCholThreads = 512;

struct CholArgs {
  const int* first;   // [nc] first block column of block row i (monotone non-decreasing, <= i)
  const int* rowoff;  // [nc] offset (in blocks) of block row i in the skyline
  const int* last;    // [nc] last block row whose skyline reaches column k
  int nblocks;
};

// in-register Cholesky of a 6x6 SPD block (lower), one thread; writes L (lower part; the strict upper part is left as is) and the
// reciprocals of its diagonal.  Returns false on a non-positive pivot.
__device__ __forceinline__ bool chol6(double* A /* smem, 36 */, double* invd /* smem, 6 */) {
  double a[21];  // packed lower triangle, row-major: (i,j) -> i(i+1)/2 + j
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) a[i * (i + 1) / 2 + j] = A[i * 6 + j];
  double r[6];
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const double d = a[j * (j + 1) / 2 + j];
    ok = ok && (d > 0.0) && (d < 1e300);
    const double rs = rsqrt(d);
    r[j] = rs;
    a[j * (j + 1) / 2 + j] = d * rs;
#pragma unroll
    for (int i = j + 1; i < 6; ++i) a[i * (i + 1) / 2 + j] *= rs;
#pragma unroll
    for (int i = j + 1; i < 6; ++i)
#pragma unroll
      for (int m = j + 1; m <= i; ++m) a[i * (i + 1) / 2 + m] -= a[i * (i + 1) / 2 + j] * a[m * (m + 1) / 2 + j];
  }
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) A[i * 6 + j] = a[i * (i + 1) / 2 + j];
#pragma unroll
  for (int j = 0; j < 6; ++j) invd[j] = r[j];
  return ok;
}

__global__ void __launch_bounds__(kCholThreads, 1) ba_chol_kernel(BaDev g, double* __restrict__ buf, CholArgs a) {
  gb_pdl_launch_dependents();
  extern __shared__ __align__(16) double sm[];
  __shared__ int s_fail;
  const int nc = g.nc, n6 = g.n6, tid = threadIdx.x;
  double* L = sm;                                   // [nblocks][36]
  double* y = L + (size_t)a.nblocks * 36;           // [n6] right-hand side -> solution
  double* invd = y + n6;                            // [n6] 1 / L_dd
  int* first = reinterpret_cast<int*>(invd + n6);   // [nc]
  int* rowoff = first + nc;                         // [nc]
  int* last = rowoff + nc;                          // [nc]
  // static structure first (overlaps the Schur kernel under a programmatic dependent launch)
  for (int k = tid; k < nc; k += kCholThreads) { first[k] = a.first[k]; rowoff[k] = a.rowoff[k]; last[k] = a.last[k]; }
  for (int k = tid; k < a.nblocks * 36; k += kCholThreads) L[k] = 0.0;
  if (tid == 0) s_fail = 0;
  gb_pdl_wait();
  if (g.sc->stop) return;
  __syncthreads();
  const double lambda = g.sc->lambda;
  const size_t nS = g.r_gt;
  // ---- A. the lower block triangle of S into the skyline, Marquardt damping (fixed dofs: unit diagonal), right-hand side
  for (int w = tid; w < g.s_nnzb * 36; w += kCholThreads) {
    const int blk = w / 36, k = w - 36 * blk;
    const int i = g.s_brow[blk], c = g.s_col[blk];
    if (c > i) continue;
    double v = g.Sb[w];
    if (c == i && (k % 7) == 0) {
      const int comp = k / 7, d = 6 * i + comp;
      v = lm_damp(v, buf[nS + n6 + d], lambda, (g.dof[i] >> comp) & 1);
    }
    L[(size_t)(rowoff[i] + c - first[i]) * 36 + k] = v;
  }
  for (int d = tid; d < n6; d += kCholThreads) y[d] = buf[nS + d];
  __syncthreads();
  // ---- B. right-looking block Cholesky inside the skyline
  for (int k = 0; k < nc; ++k) {
    double* Lkk = L + (size_t)(rowoff[k] + k - first[k]) * 36;
    if (tid == 0 && !chol6(Lkk, invd + 6 * k)) s_fail = 1;
    __syncthreads();
    const int nrows = last[k] - k;  // block rows k+1 .. last[k] have a block in column k
    // panel: L_ik = A_ik L_kk^-T, one thread per (block row, row of the block)
    for (int t = tid; t < nrows * 6; t += kCholThreads) {
      const int i = k + 1 + t / 6, r = t % 6;
      double* row = L + (size_t)(rowoff[i] + k - first[i]) * 36 + r * 6;
      double x[6];
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        double s = row[c];
#pragma unroll
        for (int m = 0; m < c; ++m) s -= x[m] * Lkk[c * 6 + m];
        x[c] = s * invd[6 * k + c];
      }
#pragma unroll
      for (int c = 0; c < 6; ++c) row[c] = x[c];
    }
    __syncthreads();
    // trailing update: A_ij -= L_ik L_jk' for k < j <= i <= last[k]
    for (int t = tid; t < nrows * nrows * 36; t += kCholThreads) {
      const int q = t / 36, e = t - 36 * q, ii = q / nrows, jj = q - ii * nrows;
      if (jj > ii) continue;
      const int i = k + 1 + ii, j = k + 1 + jj, r = e / 6, c = e - 6 * r;
      const double* Li = L + (size_t)(rowoff[i] + k - first[i]) * 36 + r * 6;
      const double* Lj = L + (size_t)(rowoff[j] + k - first[j]) * 36 + c * 6;
      double s = 0.0;
#pragma unroll
      for (int m = 0; m < 6; ++m) s += Li[m] * Lj[m];
      L[(size_t)(rowoff[i] + j - first[i]) * 36 + e] -= s;
    }
    __syncthreads();
  }
  // ---- C + D. the two substitutions are dependent chains with at most a few dozen independent operations per step: warp 0
  //      alone runs them with warp-level synchronisation (no CTA barrier), the other warps wait once
  if (tid < 32) {
    const int lane = tid;
    // C. forward substitution L z = g~
    for (int k = 0; k < nc; ++k) {
      const double* Lkk = L + (size_t)(rowoff[k] + k - first[k]) * 36;
      if (lane == 0) {
        double z[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) {
          double s = y[6 * k + c];
#pragma unroll
          for (int m = 0; m < c; ++m) s -= Lkk[c * 6 + m] * z[m];
          z[c] = s * invd[6 * k + c];
        }
#pragma unroll
        for (int c = 0; c < 6; ++c) y[6 * k + c] = z[c];
      }
      __syncwarp();
      const int nrows = last[k] - k;
      for (int t = lane; t < nrows * 6; t += 32) {
        const int i = k + 1 + t / 6, r = t % 6;
        const double* row = L + (size_t)(rowoff[i] + k - first[i]) * 36 + r * 6;
        double s = 0.0;
#pragma unroll
        for (int c = 0; c < 6; ++c) s += row[c] * y[6 * k + c];
        y[6 * i + r] -= s;
      }
      __syncwarp();
    }
    // D. backward substitution L' x = z: six lanes gather sum_i L_ik' x_i, lane 0 finishes the 6x6 triangle
    for (int k = nc - 1; k >= 0; --k) {
      const double* Lkk = L + (size_t)(rowoff[k] + k - first[k]) * 36;
      double s = 0.0;
      if (lane < 6) {
        s = y[6 * k + lane];
        for (int i = k + 1; i <= last[k]; ++i) {
          const double* blk = L + (size_t)(rowoff[i] + k - first[i]) * 36;
#pragma unroll
          for (int r = 0; r < 6; ++r) s -= blk[r * 6 + lane] * y[6 * i + r];
        }
      }
      double b[6];
#pragma unroll
      for (int c = 0; c < 6; ++c) b[c] = __shfl_sync(0xffffffffu, s, c);
      if (lane == 0) {
        double x[6];
#pragma unroll
        for (int c = 5; c >= 0; --c) {
          double v = b[c];
#pragma unroll
          for (int m = c + 1; m < 6; ++m) v -= Lkk[m * 6 + c] * x[m];
          x[c] = v * invd[6 * k + c];
        }
#pragma unroll
        for (int c = 0; c < 6; ++c) y[6 * k + c] = x[c];
      }
      __syncwarp();
    }
  }
  __syncthreads();
  // ---- E. solution (the whole step is zero when the factorisation broke down or a substitution left a non-finite component: LM
  //      rejects it and raises lambda) + retraction of the cameras
  int bad = 0;
  for (int d = tid; d < n6; d += kCholThreads) bad |= !isfinite(y[d]);
  const bool fail = __syncthreads_or(s_fail != 0 || bad) != 0;
  for (int d = tid; d < n6; d += kCholThreads) {
    const double v = fail ? 0.0 : y[d];
    y[d] = v;
    g.x[d] = v;
  }
  __syncthreads();
  for (int i = tid; i < nc; i += kCholThreads) retract_camera(g, i, y + 6 * i);
}

}  // namespace

// Skyline of the lower block triangle (natural camera order, made monotone so that the rows touching a column are contiguous).
// Host only: fills plan3 = [first | rowoff | last] (3 x nc ints, uploaded by the caller with the graph blob); false when the skyline
// does not fit one SM's shared memory (no direct solver for this graph).
bool ba_chol_plan_host(gb_ctx* ctx, int nc, const int* s_rowptr, const int* s_col, std::vector<int>& plan3, int* nblocks, size_t* smem_out) {
  plan3.assign(3 * (size_t)std::max(nc, 0), 0);
  *nblocks = 0; *smem_out = 0;
  if (nc <= 0) return false;
  int* first = plan3.data(); int* rowoff = first + nc; int* last = rowoff + nc;
  for (int i = 0; i < nc; ++i) {
    int f = i;
    for (int t = s_rowptr[i]; t < s_rowptr[i + 1]; ++t) f = std::min(f, s_col[t]);
    first[i] = f;
  }
  for (int i = nc - 2; i >= 0; --i) first[i] = std::min(first[i], first[i + 1]);  // monotone non-decreasing
  long long nb = 0;
  for (int i = 0; i < nc; ++i) { rowoff[i] = (int)nb; nb += i - first[i] + 1; }
  for (int k = 0; k < nc; ++k) {
    int l = k;
    while (l + 1 < nc && first[l + 1] <= k) ++l;
    last[k] = l;
  }
  const size_t smem = ((size_t)nb * 36 + 12 * (size_t)nc) * sizeof(double) + 3 * (size_t)nc * sizeof(int) + 64;
  if (smem + 1024 > (size_t)ctx->max_smem_optin) return false;
  if (!gb_func_setup(ctx, (const void*)ba_chol_kernel, GB_SMEM_OPTIN_MAX)) return false;
  *nblocks = (int)nb; *smem_out = smem;
  return true;
}

int ba_chol_launch(gb_ctx* ctx, gb_ba_graph* g, double* buf, bool pdl) {
  if (!ctx || !g || !g->chol_ok) return GB_ERR_INVALID;
  CholArgs a;
  a.first = g->chol_plan; a.rowoff = g->chol_plan + g->d.nc; a.last = g->chol_plan + 2 * (size_t)g->d.nc; a.nblocks = g->chol_blocks;
  if (pdl) GB_CUDA(ctx, gb_launch_pdl(ba_chol_kernel, dim3(1), dim3(kCholThreads), g->chol_smem, ctx->stream, g->d, buf, a));
  else ba_chol_kernel<<<1, kCholThreads, g->chol_smem, ctx->stream>>>(g->d, buf, a);
  GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}
