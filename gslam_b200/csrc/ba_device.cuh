// gslam_b200/csrc/ba_device.cuh — device-side math of the bundle-adjustment path (fp64).
//
// Behind GSLAM::Optimizer::optimize / optimizePnP (GSLAM/core/Optimizer.h:202-207,229).  Conventions consumed from the
// reference types: pose = {qx,qy,qz,qw,tx,ty,tz} (SE3.h:337-339), T_wc camera->world (Optimizer.h:117), quaternion
// rotation / product as SO3.h:486-509, tangent order [translation, rotation] (SE3.h:205-262).  The math is
// SURVEY.md Appendix B; oracle/ba_ref.c is the CPU restatement these functions are tested against.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

struct BaScalars {
  // options (uploaded by gb_ba_graph_begin)
  double delta, ftol, pcg_tol, lambda_init;
  // LM state
  double lambda, nu, cost, cost_new, initial_cost;
  // PCG state (generic multi-kernel path): gamma = r'u, gamma0 its initial value, CG step sizes
  double rz, rz0, pcg_alpha, pcg_beta;
  int pcg_first, pcg_k;
  int need_linearize, stop, status, iterations, accepted;
  unsigned int ticket;  // last-CTA-done counter of the fused back-substitution + commit kernel (ba_backsub_commit_kernel)
  int pending;          // an accepted candidate (pose_new / Rt_new / pts_new) has not been installed yet: the next sweep reads the
                        // candidate arrays and installs them on the fly (ba_install_pending_kernel at the end of a solve)
  int pcg_iters, pcg_done;
};

struct BaDev {
  int nc, np, no, n6, has_info;
  // estimates: T_cw as q(4)+t(3); Rt = R row-major (9) + t (3)
  double *pose, *pose_new, *Rt, *Rt_new, *pts, *pts_new;
  const uint8_t *dof, *pfree;
  // observations sorted by (point, camera)
  const int *o_cam, *o_pt;
  const double *o_uv, *o_info;
  const int *pt_off, *cam_off, *cam_perm;
  // camera-sorted copies (same order as cam_perm) so that the per-camera pass streams instead of chasing indices
  const int* c_pt;
  const double* c_uv;
  // block structure of the reduced camera matrix S (covisibility): CSR over 6x6 blocks, built on the host
  const int *s_rowptr, *s_col, *s_brow;  // s_brow[blk] = block row of blk
  const int *s_upper, *s_tidx;           // list of blocks with col >= row; s_tidx[blk] = index of the transposed block
  int s_nupper;
  double* Sb;                            // [s_nnzb][36] block-CSR values of S (local-BA path)
  int s_nnzb;
  // where [g~ | diag U | cost] start inside the reduced-system buffer handed to a kernel, in doubles: n6*n6 for the dense
  // layout [S (6N x 6N) | ...], s_nnzb*36 for the compact layout [Sb | ...] of the multi-GPU path (set per launch)
  size_t r_gt;
  // landmark-chunk Schur plan (large graphs; ba.cu: ba_schur_chunks_kernel + ba_schur_reduce_kernel), or sp_nchunks == 0
  int sp_nchunks;
  const int* sp_pt0;             // [nchunks+1] range of each chunk in the trajectory-sorted landmark list sp_order
  const int* sp_order;           // [live landmarks] landmark ids sorted by (first camera, last camera, id)
  const unsigned short* sp_mask; // [live landmarks] (same positions) which of the chunk's (<= 16, ascending) cameras observe it
  const int* sp_nused;           // [nchunks] slots of the 16x16 upper triangle the chunk really touches ...
  const unsigned char* sp_slots; // [nchunks][136] ... and which ones (thread t of the chunk's CTA works slot sp_slots[t])
  double *sp_stageS, *sp_stageG; // [nchunks][136][36], [nchunks][16][6] per-chunk partial sums
  const int *sp_boff, *sp_bidx;  // CSR over the UPPER blocks (order of s_upper): staging slots (chunk*136+slot) contributing, ascending
  const int *sp_coff, *sp_cidx;  // CSR over cameras: staging rows (chunk*16+local cam) contributing to g~
  // large-graph sweep (ba_sweep.cu): host-made item records (int4 each) dealt to sw_nteams teams, team k owns
  // [sw_team_off[k], sw_team_off[k+1])
  int vinv_in_sweep;  // 1: the sweep wrote the damped V^-1 (ba.cu's kernel); 0: ba_prepare_schur_kernel forms it (ba_sweep.cu's does not)
  int sw_nteams, sw_nitems;
  const int* sw_items;
  const int* sw_team_off;
  // pose-graph terms (ba_pose.cu): npe = SE3 edges then GPS edges (pe_j = -1); staging records pe_H [npe][121]; gather plans
  int npe, pe_npairs;
  const int *pe_i, *pe_j;
  const double *pe_Zinv, *pe_info;
  double* pe_H;
  const int *pc_off, *pc_ent;           // camera -> incident (edge << 1 | side) in edge order
  const int *pp_off, *pp_ij, *pp_ent;   // unordered camera pair -> (edge << 1 | flipped) in edge order
  // linearisation (cost_pt / cost_pt_new hold np landmark terms followed by npe pose-graph terms)
  double *V, *gp, *Vinv, *W, *U, *gc, *cost_pt, *cost_pt_new;
  // camera pass split: cam_split CTAs per camera, partial [27] sums + a per-camera ticket (the last CTA folds them in order)
  int cam_split;
  double* cam_part;
  unsigned int* cam_ticket;
  // PCG
  double *Minv, *x, *r, *z, *p, *q, *sv;  // generic PCG: z = u = Minv r, q = w = S u, sv = S p
  // grid-wide deterministic sums (cost reductions): per-block partials + a ticket, reused launch after launch
  double* red_part;        // [kRedPartials]
  unsigned int* red_ticket;
  BaScalars* sc;
  long long* prof;  // optional clock64 stamps of the cluster PCG (test hook), or nullptr
};

namespace ba {

__device__ __forceinline__ void quat_to_R(const double* q, double* R) {  // SO3.h:362-374
  const double x = q[0], y = q[1], z = q[2], w = q[3];
  const double x2 = x * x, y2 = y * y, z2 = z * z, xy = x * y, xz = x * z, yz = y * z, wx = w * x, wy = w * y, wz = w * z;
  R[0] = 1.0 - 2.0 * (y2 + z2); R[1] = 2.0 * (xy - wz);       R[2] = 2.0 * (xz + wy);
  R[3] = 2.0 * (xy + wz);       R[4] = 1.0 - 2.0 * (x2 + z2); R[5] = 2.0 * (yz - wx);
  R[6] = 2.0 * (xz - wy);       R[7] = 2.0 * (yz + wx);       R[8] = 1.0 - 2.0 * (x2 + y2);
}
__device__ __forceinline__ void quat_rot(const double* q, const double* p, double* o) {  // SO3.h:499-509
  double ux = q[1] * p[2] - q[2] * p[1], uy = q[2] * p[0] - q[0] * p[2], uz = q[0] * p[1] - q[1] * p[0];
  ux += ux; uy += uy; uz += uz;
  o[0] = p[0] + q[3] * ux + (q[1] * uz - q[2] * uy);
  o[1] = p[1] + q[3] * uy + (q[2] * ux - q[0] * uz);
  o[2] = p[2] + q[3] * uz + (q[0] * uy - q[1] * ux);
}
__device__ __forceinline__ void quat_mul(const double* a, const double* b, double* o) {  // SO3.h:486-493
  o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  o[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  o[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
}
__device__ __forceinline__ void se3_inverse(const double* in, double* out) {  // SE3.h:100-103
  const double n = sqrt(in[0] * in[0] + in[1] * in[1] + in[2] * in[2] + in[3] * in[3]);
  const double qi[4] = {-in[0] / n, -in[1] / n, -in[2] / n, in[3] / n};
  double t[3];
  quat_rot(qi, in + 4, t);
  out[0] = qi[0]; out[1] = qi[1]; out[2] = qi[2]; out[3] = qi[3];
  out[4] = -t[0]; out[5] = -t[1]; out[6] = -t[2];
}
// pose <- Exp([v,w]) * pose, small-angle safe (the reference's SE3::exp is NaN at w=0, SE3.h:284-285)
__device__ __forceinline__ void se3_retract(const double* pose, const double* d, double* out) {
  const double vx = d[0], vy = d[1], vz = d[2], wx = d[3], wy = d[4], wz = d[5];
  const double th2 = wx * wx + wy * wy + wz * wz, th = sqrt(th2);
  double imag, real, B, C;
  if (th < 1e-6) {
    imag = 0.5 - th2 / 48.0; real = 1.0 - th2 / 8.0; B = 0.5 - th2 / 24.0; C = 1.0 / 6.0 - th2 / 120.0;
  } else {
    imag = sin(0.5 * th) / th; real = cos(0.5 * th); B = (1.0 - cos(th)) / th2; C = (th - sin(th)) / (th2 * th);
  }
  const double dq[4] = {imag * wx, imag * wy, imag * wz, real};
  const double c1x = wy * vz - wz * vy, c1y = wz * vx - wx * vz, c1z = wx * vy - wy * vx;
  const double c2x = wy * c1z - wz * c1y, c2y = wz * c1x - wx * c1z, c2z = wx * c1y - wy * c1x;
  const double td[3] = {vx + B * c1x + C * c2x, vy + B * c1y + C * c2y, vz + B * c1z + C * c2z};
  double q[4], t[3];
  quat_mul(dq, pose, q);
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  quat_rot(dq, pose + 4, t);
  out[0] = q[0] / n; out[1] = q[1] / n; out[2] = q[2] / n; out[3] = q[3] / n;
  out[4] = t[0] + td[0]; out[5] = t[1] + td[1]; out[6] = t[2] + td[2];
}

__device__ __forceinline__ double clampd(double d) { return d < 1e-6 ? 1e-6 : (d > 1e32 ? 1e32 : d); }

// Cholesky inverse of a small SPD matrix, row-major, in place; returns false if not positive definite.
template <int N>
__device__ __forceinline__ bool spd_inverse(double* A) {
  double L[N * N], Li[N * N], id[N];  // id[i] = 1 / L_ii (one division per pivot; everything else multiplies)
#pragma unroll
  for (int i = 0; i < N * N; ++i) { L[i] = 0.0; Li[i] = 0.0; }
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      double s = A[i * N + j];
#pragma unroll
      for (int k = 0; k < j; ++k) s -= L[i * N + k] * L[j * N + k];
      if (i == j) {
        if (!(s > 0.0)) return false;
        L[i * N + i] = sqrt(s);
        id[i] = 1.0 / L[i * N + i];
      } else {
        L[i * N + j] = s * id[j];
      }
    }
#pragma unroll
  for (int c = 0; c < N; ++c)
#pragma unroll
    for (int i = c; i < N; ++i) {
      double s = (i == c) ? 1.0 : 0.0;
#pragma unroll
      for (int k = c; k < i; ++k) s -= L[i * N + k] * Li[k * N + c];
      Li[i * N + c] = s * id[i];
    }
#pragma unroll
  for (int i = 0; i < N; ++i)
#pragma unroll
    for (int j = 0; j < N; ++j) {
      double s = 0.0;
#pragma unroll
      for (int k = (i > j ? i : j); k < N; ++k) s += Li[k * N + i] * Li[k * N + j];
      A[i * N + j] = s;
    }
  return true;
}

// ---- the rules of the Levenberg-Marquardt step, each written once for every solver path -----------------------------------------

// LM accept / reject of a step from the cost at the current estimate and at the candidate (one thread).  Accept: lambda / 3 floored
// at 1e-15, nu = 2, stop with status 1 when the relative decrease is under ftol.  Reject: lambda * nu, nu * 2, stop with status 2
// once lambda exceeds 1e16.  Returns whether the step was accepted: lm_accepts, which any thread may evaluate from the two costs.
__device__ __forceinline__ bool lm_accepts(double cost, double cnew) { return (cnew < cost) && isfinite(cnew); }
__device__ __forceinline__ bool lm_decide(BaScalars* sc, double cost, double cnew) {
  if (sc->iterations == 0) sc->initial_cost = cost;
  sc->cost = cost;
  sc->cost_new = cnew;
  sc->iterations++;
  const bool ok = lm_accepts(cost, cnew);
  sc->need_linearize = ok ? 1 : 0;
  if (ok) {
    const double rel = (cost - cnew) / cost;
    sc->cost = cnew;
    const double l = sc->lambda / 3.0;
    sc->lambda = l < 1e-15 ? 1e-15 : l;
    sc->nu = 2.0;
    sc->accepted++;
    if (rel < sc->ftol) { sc->stop = 1; sc->status = 1; }
  } else {
    sc->lambda *= sc->nu;
    sc->nu *= 2.0;
    if (sc->lambda > 1e16) { sc->stop = 1; sc->status = 2; }
  }
  return ok;
}

// Marquardt damping of the diagonal entry s of a normal-equation block whose undamped value is diag; a fixed dof gets a unit diagonal
__device__ __forceinline__ double lm_damp(double s, double diag, double lambda, bool free = true) {
  return free ? s + lambda * clampd(diag) : 1.0;
}

// Block-Jacobi preconditioner block: M (a damped 6x6 diagonal block, read from D with row stride ld) <- its inverse, or the inverse
// of its diagonal when the block is not positive definite
__device__ __forceinline__ void block_jacobi_inverse(double* M, const double* D, size_t ld) {
  if (!spd_inverse<6>(M)) {
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int b = 0; b < 6; ++b) M[a * 6 + b] = (a == b) ? 1.0 / D[a * ld + a] : 0.0;
  }
}

// Damped landmark inverse: Vinv[9] = (V + lambda * clamp(diag V))^-1 for an active landmark (free and observed); zero when the
// landmark is not active or the damped block is not positive definite
__device__ __forceinline__ void damped_vinv(const double* V, bool active, double lambda, double* Vinv) {
  double Vi[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) Vi[k] = active ? V[k] : 0.0;
  if (active) {
#pragma unroll
    for (int a = 0; a < 3; ++a) Vi[a * 4] = lm_damp(Vi[a * 4], Vi[a * 4], lambda);
    if (!spd_inverse<3>(Vi)) {
#pragma unroll
      for (int k = 0; k < 9; ++k) Vi[k] = 0.0;
    }
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) Vinv[k] = Vi[k];
}

// Candidate of camera i: pose_new = Exp(dx) * pose and its Rt_new, with dx[6] restricted to the camera's free dofs
__device__ __forceinline__ void retract_camera(const BaDev& g, int i, const double* dx) {
  double pose[7], d[6], out[7], R[9];
  const int dm = g.dof[i];
#pragma unroll
  for (int k = 0; k < 7; ++k) pose[k] = g.pose[7 * i + k];
#pragma unroll
  for (int a = 0; a < 6; ++a) d[a] = ((dm >> a) & 1) ? dx[a] : 0.0;
  se3_retract(pose, d, out);
#pragma unroll
  for (int k = 0; k < 7; ++k) g.pose_new[7 * i + k] = out[k];
  quat_to_R(out, R);
#pragma unroll
  for (int k = 0; k < 9; ++k) g.Rt_new[12 * i + k] = R[k];
#pragma unroll
  for (int k = 0; k < 3; ++k) g.Rt_new[12 * i + 9 + k] = out[4 + k];
}

struct ObsLin {
  bool valid;
  double r0, r1, rho;
  double A0, A1, A2;  // w * Lambda (xx, xy, yy)
  double a, b, iz;    // normalised coords and 1/z
};

// residual + robust weight of one observation (Appendix B).  Rt = R(9) row-major + t(3) of T_cw.
__device__ __forceinline__ ObsLin eval_obs(const double* __restrict__ Rt, const double* p, double u, double v,
                                           const double* info3, double delta) {
  ObsLin o;
  const double x = Rt[0] * p[0] + Rt[1] * p[1] + Rt[2] * p[2] + Rt[9];
  const double y = Rt[3] * p[0] + Rt[4] * p[1] + Rt[5] * p[2] + Rt[10];
  const double z = Rt[6] * p[0] + Rt[7] * p[1] + Rt[8] * p[2] + Rt[11];
  o.valid = z > 0.0;
  o.rho = 0.0; o.r0 = 0.0; o.r1 = 0.0; o.A0 = 0.0; o.A1 = 0.0; o.A2 = 0.0; o.a = 0.0; o.b = 0.0; o.iz = 0.0;
  if (!o.valid) return o;
  const double iz = 1.0 / z;
  o.iz = iz; o.a = x * iz; o.b = y * iz;
  o.r0 = o.a - u; o.r1 = o.b - v;
  double Lxx = 1.0, Lxy = 0.0, Lyy = 1.0;
  if (info3) { Lxx = info3[0]; Lxy = info3[1]; Lyy = info3[2]; }
  const double e2 = o.r0 * (Lxx * o.r0 + Lxy * o.r1) + o.r1 * (Lxy * o.r0 + Lyy * o.r1);
  const double e = sqrt(e2);
  double w = 1.0;
  if (delta > 0.0 && e > delta) { w = delta / e; o.rho = 2.0 * delta * e - delta * delta; } else { o.rho = e2; }
  o.A0 = w * Lxx; o.A1 = w * Lxy; o.A2 = w * Lyy;
  return o;
}

// 2x6 camera Jacobian rows (left tangent [v,w] of T_cw), masked by the dof bits
__device__ __forceinline__ void jac_cam(const ObsLin& o, int dofmask, double* Jc /*12*/) {
  const double a = o.a, b = o.b, iz = o.iz;
  Jc[0] = iz;  Jc[1] = 0.0; Jc[2] = -a * iz; Jc[3] = -a * b;       Jc[4] = 1.0 + a * a; Jc[5] = -b;
  Jc[6] = 0.0; Jc[7] = iz;  Jc[8] = -b * iz; Jc[9] = -1.0 - b * b; Jc[10] = a * b;      Jc[11] = a;
#pragma unroll
  for (int d = 0; d < 6; ++d)
    if (!((dofmask >> d) & 1)) { Jc[d] = 0.0; Jc[6 + d] = 0.0; }
}
__device__ __forceinline__ void jac_pt(const ObsLin& o, const double* __restrict__ Rt, bool pfree, double* Jp /*6*/) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    Jp[c] = pfree ? (o.iz * Rt[c] - o.a * o.iz * Rt[6 + c]) : 0.0;
    Jp[3 + c] = pfree ? (o.iz * Rt[3 + c] - o.b * o.iz * Rt[6 + c]) : 0.0;
  }
}

// Deterministic block-wide sum (fixed shuffle tree, then warp 0 over the per-warp partials in order). All threads get it.
template <int NT>
__device__ __forceinline__ double block_sum(double v, double* s_part /* >= NT/32 + 1 doubles */) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();  // protect s_part from a previous use
  if (lane == 0) s_part[warp] = v;
  __syncthreads();
  if (warp == 0) {
    double t = (lane < NT / 32) ? s_part[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
    if (lane == 0) s_part[NT / 32] = t;
  }
  __syncthreads();
  return s_part[NT / 32];
}

}  // namespace ba
