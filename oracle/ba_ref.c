/*
 * oracle/ba_ref.c — CPU (fp64, scalar C) restatement of the GSLAM::Optimizer bundle-adjustment path.
 * TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs; never by the product.
 *
 * PARITY UNPINNED by reference tests: the reference ships only the interface (GSLAM/core/Optimizer.h:184-253, every
 * virtual returns false); its Ceres backend (CMakeLists.txt:44, commented out; directory absent; no pinned version)
 * and any test/golden vector for it are not in the tree.  What IS pinned: the conventions this file consumes —
 *   T_wc pose layout & inverse/transform   GSLAM/core/SE3.h:100-103,129-131,337-339  (checked against the reference's
 *                                          own SE3 class through oracle/_ref, tests/test_oracle_ba.py)
 *   quaternion rotate / product            GSLAM/core/SO3.h:486-509
 *   graph PODs, dof bits, Huber default    GSLAM/core/Optimizer.h:58-182
 *   tangent order [translation, rotation]  GSLAM/core/SE3.h:205-262
 * and the optimum itself is cross-checked against scipy.optimize.least_squares on the same residual.
 *
 * Math (SURVEY.md Appendix B — our definition; the reference fixes only types and conventions):
 *   q = R_cw p + t_cw (T_cw = T_wc^-1);  r = (q.x/q.z - u, q.y/q.z - v);  e^2 = r' L r;  Huber IRLS weight
 *   w = e<=d ? 1 : d/e;  rho = e<=d ? e^2 : 2 d e - d^2;  cost = 0.5 sum rho;  observations with q.z <= 0 are skipped.
 *   Left update T_cw <- Exp([v,w]) T_cw:  J_cam = Jpi [I | -[q]x],  J_pt = Jpi R_cw.
 *   Pose-graph terms (SE3Edge / GPSEdge, Optimizer.h:127-148) add e = Log(Z^-1 T_1^-1 T_2) / Log(Z^-1 T) with e' Omega e to the cost
 *   and J' Omega J / J' Omega e to the camera blocks (pose_edge_eval below); a graph may hold them alone (a pose graph).
 *   Levenberg-Marquardt with Marquardt scaling lambda*clamp(diag,1e-6,1e32) on U and V; Schur complement onto the cameras;
 *   block-Jacobi PCG; back-substitution; accept iff cost decreases (lambda/=3, nu=2) else (lambda*=nu, nu*=2).
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "../include/gslam_b200.h"

/* ---- small helpers ------------------------------------------------------------------------------------------------ */
static void quat_to_R(const double* q, double* R) { /* q = x,y,z,w ; R row-major (SO3.h:362-374) */
  double x = q[0], y = q[1], z = q[2], w = q[3];
  double x2 = x * x, y2 = y * y, z2 = z * z, xy = x * y, xz = x * z, yz = y * z, wx = w * x, wy = w * y, wz = w * z;
  R[0] = 1.0 - 2.0 * (y2 + z2); R[1] = 2.0 * (xy - wz);       R[2] = 2.0 * (xz + wy);
  R[3] = 2.0 * (xy + wz);       R[4] = 1.0 - 2.0 * (x2 + z2); R[5] = 2.0 * (yz - wx);
  R[6] = 2.0 * (xz - wy);       R[7] = 2.0 * (yz + wx);       R[8] = 1.0 - 2.0 * (x2 + y2);
}
static void quat_rot(const double* q, const double* p, double* o) { /* SO3.h:499-509 */
  double ux = q[1] * p[2] - q[2] * p[1], uy = q[2] * p[0] - q[0] * p[2], uz = q[0] * p[1] - q[1] * p[0];
  ux += ux; uy += uy; uz += uz;
  o[0] = p[0] + q[3] * ux + (q[1] * uz - q[2] * uy);
  o[1] = p[1] + q[3] * uy + (q[2] * ux - q[0] * uz);
  o[2] = p[2] + q[3] * uz + (q[0] * uy - q[1] * ux);
}
static void quat_mul(const double* a, const double* b, double* o) { /* SO3.h:486-493 */
  o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  o[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  o[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
}
/* pose7 = qx qy qz qw tx ty tz.  out = in^-1 (SE3.h:100-103). */
void orc_se3_inverse(const double* in, double* out) {
  double n = sqrt(in[0] * in[0] + in[1] * in[1] + in[2] * in[2] + in[3] * in[3]);
  double qi[4] = {-in[0] / n, -in[1] / n, -in[2] / n, in[3] / n};
  double t[3];
  quat_rot(qi, in + 4, t);
  out[0] = qi[0]; out[1] = qi[1]; out[2] = qi[2]; out[3] = qi[3];
  out[4] = -t[0]; out[5] = -t[1]; out[6] = -t[2];
}
/* pose <- Exp([v,w]) * pose   (small-angle safe; the reference's SE3::exp is NaN at w=0, SE3.h:284-285) */
void orc_se3_retract(const double* pose, const double* d, double* out) {
  double vx = d[0], vy = d[1], vz = d[2], wx = d[3], wy = d[4], wz = d[5];
  double th2 = wx * wx + wy * wy + wz * wz, th = sqrt(th2);
  double imag, real, B, C;
  if (th < 1e-6) {
    imag = 0.5 - th2 / 48.0;
    real = 1.0 - th2 / 8.0;
    B = 0.5 - th2 / 24.0;
    C = 1.0 / 6.0 - th2 / 120.0;
  } else {
    imag = sin(0.5 * th) / th;
    real = cos(0.5 * th);
    B = (1.0 - cos(th)) / th2;
    C = (th - sin(th)) / (th2 * th);
  }
  double dq[4] = {imag * wx, imag * wy, imag * wz, real};
  /* t_d = v + B w x v + C w x (w x v) */
  double c1x = wy * vz - wz * vy, c1y = wz * vx - wx * vz, c1z = wx * vy - wy * vx;
  double c2x = wy * c1z - wz * c1y, c2y = wz * c1x - wx * c1z, c2z = wx * c1y - wy * c1x;
  double td[3] = {vx + B * c1x + C * c2x, vy + B * c1y + C * c2y, vz + B * c1z + C * c2z};
  double q[4], t[3];
  quat_mul(dq, pose, q);
  double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  quat_rot(dq, pose + 4, t);
  out[0] = q[0] / n; out[1] = q[1] / n; out[2] = q[2] / n; out[3] = q[3] / n;
  out[4] = t[0] + td[0]; out[5] = t[1] + td[1]; out[6] = t[2] + td[2];
}

static double clampd(double d) { return d < 1e-6 ? 1e-6 : (d > 1e32 ? 1e32 : d); }

/* Threads of the solver's heavy loops (the reference arm of bench.py: "OpenMP, all cores" next to the 1-thread figure).  Default 1:
 * the tests compare against the strictly sequential summation order.  With n > 1 the Schur complement accumulates per-thread partial
 * systems (static schedule, folded in thread order: deterministic for a fixed n), the dense mat-vec of the PCG is split by rows
 * (bitwise the same), the cost is a per-thread partial sum. */
static int g_ba_threads = 1;
void orc_ba_set_threads(int n) {
#ifdef _OPENMP
  g_ba_threads = n < 1 ? 1 : (n > 64 ? 64 : n);
#else
  (void)n;
#endif
}

/* ---- pose-graph terms (row f3: GSLAM::SE3Edge / GPSEdge, Optimizer.h:127-148; our definition, see the header) ------------------- */
/* Log of an SE3 given as pose7, tangent order [v, w]: restates the reference's SE3::log (GSLAM/core/SE3.h:205-246, NEAR_ZERO = 1e-10
 * SO3.h:43) -- pinned against the reference class through oracle/_ref in tests/test_oracle_ba.py. */
void orc_se3_log(const double* T, double* out6) {
  const double x = T[0], y = T[1], z = T[2], w = T[3];
  const double* t = T + 4;
  const double n = sqrt(x * x + y * y + z * z);
  double A_inv, r[3], c1[3], c2[3];
  if (n < 1e-10) {
    A_inv = 2.0 / w - 2.0 * (1.0 - w * w) / (w * w * w);
    r[0] = x * A_inv; r[1] = y * A_inv; r[2] = z * A_inv;
    c1[0] = r[1] * t[2] - r[2] * t[1]; c1[1] = r[2] * t[0] - r[0] * t[2]; c1[2] = r[0] * t[1] - r[1] * t[0];
    c2[0] = r[1] * c1[2] - r[2] * c1[1]; c2[1] = r[2] * c1[0] - r[0] * c1[2]; c2[2] = r[0] * c1[1] - r[1] * c1[0];
    for (int k = 0; k < 3; ++k) out6[k] = t[k] - 0.5 * c1[k] + (1.0 / 12.0) * c2[k];
  } else {
    if (fabs(w) < 1e-10) A_inv = (w > 0 ? 3.14159265358979323846 : -3.14159265358979323846) / n;
    else A_inv = 2.0 * atan(n / w) / n;
    const double theta = A_inv * n;
    r[0] = x * A_inv; r[1] = y * A_inv; r[2] = z * A_inv;
    const double a[3] = {r[0] / theta, r[1] / theta, r[2] / theta};
    c1[0] = r[1] * t[2] - r[2] * t[1]; c1[1] = r[2] * t[0] - r[0] * t[2]; c1[2] = r[0] * t[1] - r[1] * t[0];
    double a1[3] = {a[1] * t[2] - a[2] * t[1], a[2] * t[0] - a[0] * t[2], a[0] * t[1] - a[1] * t[0]};
    c2[0] = a[1] * a1[2] - a[2] * a1[1]; c2[1] = a[2] * a1[0] - a[0] * a1[2]; c2[2] = a[0] * a1[1] - a[1] * a1[0];
    const double k2 = 1.0 - theta / (2.0 * tan(0.5 * theta));
    for (int k = 0; k < 3; ++k) out6[k] = t[k] - 0.5 * c1[k] + k2 * c2[k];
  }
  out6[3] = r[0]; out6[4] = r[1]; out6[5] = r[2];
}
/* out = a * b (SE3.h:129-131: rotation product, translation a.R * b.t + a.t) */
void orc_se3_mul(const double* a, const double* b, double* out) {
  double q[4], t[3];
  quat_mul(a, b, q);
  quat_rot(a, b + 4, t);
  out[0] = q[0]; out[1] = q[1]; out[2] = q[2]; out[3] = q[3];
  out[4] = t[0] + a[4]; out[5] = t[1] + a[5]; out[6] = t[2] + a[6];
}
/* 6x6 adjoint of T for the tangent order [v, w]: Ad = [[R, [t]x R], [0, R]]  (Exp(d) T = T Exp(Ad(T^-1) d)) */
static void se3_adjoint(const double* T, double* Ad) {
  double R[9];
  quat_to_R(T, R);
  const double* t = T + 4;
  const double tx[9] = {0.0, -t[2], t[1], t[2], 0.0, -t[0], -t[1], t[0], 0.0};
  memset(Ad, 0, sizeof(double) * 36);
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      Ad[a * 6 + b] = R[a * 3 + b];
      Ad[(3 + a) * 6 + 3 + b] = R[a * 3 + b];
      Ad[a * 6 + 3 + b] = tx[a * 3] * R[b] + tx[a * 3 + 1] * R[3 + b] + tx[a * 3 + 2] * R[6 + b];
    }
}
static void mat6_mul(const double* A, const double* B, double* C) {
  for (int a = 0; a < 6; ++a)
    for (int b = 0; b < 6; ++b) {
      double x = 0.0;
      for (int k = 0; k < 6; ++k) x += A[a * 6 + k] * B[k * 6 + b];
      C[a * 6 + b] = x;
    }
}
/* Inverse left Jacobian of SE3 at xi = [v, w]:  Log(Exp(d) Exp(xi)) = xi + Jl^-1(xi) d + O(d^2).  Bernoulli series in the adjoint
 * ad(xi) = [[w^, v^], [0, w^]]:  I - ad/2 + ad^2/12 - ad^4/720 + ad^6/30240 - ad^8/1209600  (next term 2e-8 |ad|^10: residuals of a
 * pose graph near its optimum are far inside the radius where this is double precision). */
static void se3_jl_inv(const double* xi, double* J) {
  const double* v = xi; const double* w = xi + 3;
  double A[36], A2[36], A4[36], A6[36], A8[36];
  memset(A, 0, sizeof A);
  const double wx[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
  const double vx[9] = {0.0, -v[2], v[1], v[2], 0.0, -v[0], -v[1], v[0], 0.0};
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) { A[a * 6 + b] = wx[a * 3 + b]; A[(3 + a) * 6 + 3 + b] = wx[a * 3 + b]; A[a * 6 + 3 + b] = vx[a * 3 + b]; }
  mat6_mul(A, A, A2); mat6_mul(A2, A2, A4); mat6_mul(A4, A2, A6); mat6_mul(A4, A4, A8);
  for (int k = 0; k < 36; ++k)
    J[k] = ((k % 7) == 0 ? 1.0 : 0.0) - 0.5 * A[k] + A2[k] * (1.0 / 12.0) - A4[k] * (1.0 / 720.0) + A6[k] * (1.0 / 30240.0) - A8[k] * (1.0 / 1209600.0);
}
/* One pose-graph term at the internal estimate (T_cw per camera).
 *   SE3Edge (first = i, second = j, Z = T_wc,i^-1 T_wc,j, Optimizer.h:127-133):  E = Z^-1 T_cw,i T_cw,j^-1,  e = Log(E)
 *        left updates T_cw <- Exp(d) T_cw give  E' = Exp(Ad(Z^-1) d_i) Exp(-Ad(E) d_j) E,  so  J_i = Jl^-1(e) Ad(Z^-1),  J_j = -Jl^-1(e) Ad(E)
 *   GPSEdge (frame i, Z = T_wc,i prior, Optimizer.h:143-148):                    E = Z^-1 T_cw,i^-1,  e = Log(E),  J_i = -Jl^-1(e) Ad(E)
 * Cost term e' Omega e, no robust kernel.  Ji / Jj are 6x6 row-major; Jj unused for a GPS edge. */
static void pose_edge_eval(const double* Zinv, const double* Ti_cw, const double* Tj_cw, int is_gps, double* e, double* Ji, double* Jj) {
  double E[7], tmp[7], inv[7];
  if (is_gps) {
    orc_se3_inverse(Ti_cw, inv);
    orc_se3_mul(Zinv, inv, E);
  } else {
    orc_se3_inverse(Tj_cw, inv);
    orc_se3_mul(Ti_cw, inv, tmp);
    orc_se3_mul(Zinv, tmp, E);
  }
  orc_se3_log(E, e);
  if (!Ji) return;
  double AdE[36], AdZ[36], Jl[36], T[36];
  se3_adjoint(E, AdE);
  se3_jl_inv(e, Jl);
  mat6_mul(Jl, AdE, T);
  if (is_gps) {
    for (int k = 0; k < 36; ++k) Ji[k] = -T[k];
  } else {
    se3_adjoint(Zinv, AdZ);
    mat6_mul(Jl, AdZ, Ji);
    for (int k = 0; k < 36; ++k) Jj[k] = -T[k];
  }
}
static double quad6(const double* info, const double* e) { /* e' Omega e, Omega = identity when info == NULL */
  double s = 0.0;
  for (int a = 0; a < 6; ++a) {
    double r = 0.0;
    if (info) for (int b = 0; b < 6; ++b) r += 0.5 * (info[a * 6 + b] + info[b * 6 + a]) * e[b]; else r = e[a];
    s += e[a] * r;
  }
  return s;
}

/* Cholesky-based inverse of a small SPD matrix (n<=6), row-major, in place.  Returns 0 on success. */
static int spd_inverse(double* A, int n) {
  double L[36], Li[36];
  memset(L, 0, sizeof L);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j <= i; ++j) {
      double s = A[i * n + j];
      for (int k = 0; k < j; ++k) s -= L[i * n + k] * L[j * n + k];
      if (i == j) {
        if (!(s > 0.0)) return 1;
        L[i * n + i] = sqrt(s);
      } else
        L[i * n + j] = s / L[j * n + j];
    }
  memset(Li, 0, sizeof Li);
  for (int c = 0; c < n; ++c) /* Li = L^-1 by forward substitution */
    for (int i = c; i < n; ++i) {
      double s = (i == c) ? 1.0 : 0.0;
      for (int k = c; k < i; ++k) s -= L[i * n + k] * Li[k * n + c];
      Li[i * n + c] = s / L[i * n + i];
    }
  for (int i = 0; i < n; ++i) /* A^-1 = Li' Li */
    for (int j = 0; j < n; ++j) {
      double s = 0.0;
      for (int k = (i > j ? i : j); k < n; ++k) s += Li[k * n + i] * Li[k * n + j];
      A[i * n + j] = s;
    }
  return 0;
}

/* ---- per-observation residual / Jacobian -------------------------------------------------------------------------- */
typedef struct {
  int valid;
  double r[2], w, rho;  /* residual, IRLS weight, robustified squared error */
  double Jc[12], Jp[6]; /* 2x6, 2x3 row-major                               */
  double A[3];          /* w * Lambda (xx, xy, yy)                          */
} obs_lin;

static void eval_obs(const double* R, const double* t, const double* p, const double* m, const double* info,
                     double delta, int want_jac, obs_lin* o) {
  double x = R[0] * p[0] + R[1] * p[1] + R[2] * p[2] + t[0];
  double y = R[3] * p[0] + R[4] * p[1] + R[5] * p[2] + t[1];
  double z = R[6] * p[0] + R[7] * p[1] + R[8] * p[2] + t[2];
  o->valid = 0; o->rho = 0.0; o->w = 0.0;
  if (!(z > 0.0)) return;
  o->valid = 1;
  double iz = 1.0 / z, u = m[0] / m[2], v = m[1] / m[2];
  o->r[0] = x * iz - u;
  o->r[1] = y * iz - v;
  double Lxx = 1.0, Lxy = 0.0, Lyy = 1.0;
  if (info) { Lxx = info[0]; Lxy = 0.5 * (info[1] + info[2]); Lyy = info[3]; }
  double e2 = o->r[0] * (Lxx * o->r[0] + Lxy * o->r[1]) + o->r[1] * (Lxy * o->r[0] + Lyy * o->r[1]);
  double e = sqrt(e2);
  if (delta > 0.0 && e > delta) { o->w = delta / e; o->rho = 2.0 * delta * e - delta * delta; }
  else { o->w = 1.0; o->rho = e2; }
  o->A[0] = o->w * Lxx; o->A[1] = o->w * Lxy; o->A[2] = o->w * Lyy;
  if (!want_jac) return;
  double a = x * iz, b = y * iz; /* normalised coords */
  /* Jpi = [[iz,0,-a iz],[0,iz,-b iz]];  Jc = Jpi [I | -[q]x] */
  o->Jc[0] = iz;  o->Jc[1] = 0.0; o->Jc[2] = -a * iz; o->Jc[3] = -a * b;        o->Jc[4] = 1.0 + a * a; o->Jc[5] = -b;
  o->Jc[6] = 0.0; o->Jc[7] = iz;  o->Jc[8] = -b * iz; o->Jc[9] = -1.0 - b * b;  o->Jc[10] = a * b;      o->Jc[11] = a;
  for (int c = 0; c < 3; ++c) {
    o->Jp[c] = iz * R[c] - a * iz * R[6 + c];
    o->Jp[3 + c] = iz * R[3 + c] - b * iz * R[6 + c];
  }
}

/* ---- solver state ---------------------------------------------------------------------------------------------------- */
typedef struct {
  int nc, np, no;
  double* pose; /* nc x 7, T_cw */
  double* pts;  /* np x 3       */
  const uint8_t* dof; const uint8_t* pfree;
  const int32_t *oc, *op; const double *om, *oi;
  double delta;
  /* linearisation */
  double *U, *gc, *V, *gp, *W; /* nc x 36, nc x 6, np x 9, np x 3, no x 18 */
  /* point -> obs lists, camera -> obs lists (observation indices ascending inside each list) */
  int *poff, *plist, *coff, *clist;
  /* pose-graph terms: SE3 edges then GPS edges; Zinv = measurement^-1; P = off-diagonal block J_i' Omega J_j of each SE3 edge */
  int nse, ngps;
  const int32_t *se_i, *se_j, *gps_i;
  const double *se_info, *gps_info;
  double *se_Zinv, *gps_Zinv, *P;
} ba_state;

static int dofmask(const ba_state* s, int i) { return s->dof ? (s->dof[i] & 63) : 63; }
static int ptfree(const ba_state* s, int j) { return s->pfree ? (s->pfree[j] != 0) : 1; }

static double ba_cost(const ba_state* s, const double* pose, const double* pts) {
  double c = 0.0;
  double* Rs = (double*)malloc(sizeof(double) * 9 * (size_t)s->nc);
  for (int i = 0; i < s->nc; ++i) quat_to_R(pose + 7 * i, Rs + 9 * i);
  if (g_ba_threads > 1 && s->no > 4096) {
    double part[64] = {0};
#ifdef _OPENMP
#pragma omp parallel num_threads(g_ba_threads)
    {
      double acc = 0.0;
#pragma omp for schedule(static)
      for (int k = 0; k < s->no; ++k) {
        obs_lin o;
        int i = s->oc[k], j = s->op[k];
        eval_obs(Rs + 9 * i, pose + 7 * i + 4, pts + 3 * j, s->om + 3 * k, s->oi ? s->oi + 4 * k : NULL, s->delta, 0, &o);
        acc += o.rho;
      }
      part[omp_get_thread_num()] = acc;
    }
#endif
    for (int t = 0; t < 64; ++t) c += part[t];
  } else
  for (int k = 0; k < s->no; ++k) {
    obs_lin o;
    int i = s->oc[k], j = s->op[k];
    eval_obs(Rs + 9 * i, pose + 7 * i + 4, pts + 3 * j, s->om + 3 * k, s->oi ? s->oi + 4 * k : NULL, s->delta, 0, &o);
    c += o.rho;
  }
  free(Rs);
  for (int k = 0; k < s->nse; ++k) {
    double e[6];
    pose_edge_eval(s->se_Zinv + 7 * k, pose + 7 * s->se_i[k], pose + 7 * s->se_j[k], 0, e, NULL, NULL);
    c += quad6(s->se_info ? s->se_info + 36 * k : NULL, e);
  }
  for (int k = 0; k < s->ngps; ++k) {
    double e[6];
    pose_edge_eval(s->gps_Zinv + 7 * k, pose + 7 * s->gps_i[k], NULL, 1, e, NULL, NULL);
    c += quad6(s->gps_info ? s->gps_info + 36 * k : NULL, e);
  }
  return 0.5 * c;
}

/* H_ab += Ja' Omega Jb (6x6), g_a -= Ja' Omega e, with the fixed dofs' columns of the Jacobians zeroed */
static void pose_term_accumulate(const double* info, const double* e, double* Ja, int dma, double* Jb, int dmb, double* Uaa, double* ga, double* Ubb,
                                 double* gb, double* Pab) {
  for (int d = 0; d < 6; ++d) {
    if (!((dma >> d) & 1)) for (int r = 0; r < 6; ++r) Ja[r * 6 + d] = 0.0;
    if (Jb && !((dmb >> d) & 1)) for (int r = 0; r < 6; ++r) Jb[r * 6 + d] = 0.0;
  }
  double Om[36], OJa[36], OJb[36], Oe[6];
  for (int a = 0; a < 6; ++a) for (int b = 0; b < 6; ++b) Om[a * 6 + b] = info ? 0.5 * (info[a * 6 + b] + info[b * 6 + a]) : (a == b ? 1.0 : 0.0);
  for (int a = 0; a < 6; ++a) {
    Oe[a] = 0.0;
    for (int b = 0; b < 6; ++b) Oe[a] += Om[a * 6 + b] * e[b];
    for (int c = 0; c < 6; ++c) {
      double x = 0.0, y = 0.0;
      for (int b = 0; b < 6; ++b) { x += Om[a * 6 + b] * Ja[b * 6 + c]; if (Jb) y += Om[a * 6 + b] * Jb[b * 6 + c]; }
      OJa[a * 6 + c] = x; OJb[a * 6 + c] = y;
    }
  }
  for (int a = 0; a < 6; ++a) {
    double x = 0.0, y = 0.0;
    for (int r = 0; r < 6; ++r) { x += Ja[r * 6 + a] * Oe[r]; if (Jb) y += Jb[r * 6 + a] * Oe[r]; }
    ga[a] -= x; if (Jb) gb[a] -= y;
    for (int c = 0; c < 6; ++c) {
      double haa = 0.0, hbb = 0.0, hab = 0.0;
      for (int r = 0; r < 6; ++r) {
        haa += Ja[r * 6 + a] * OJa[r * 6 + c];
        if (Jb) { hbb += Jb[r * 6 + a] * OJb[r * 6 + c]; hab += Ja[r * 6 + a] * OJb[r * 6 + c]; }
      }
      Uaa[a * 6 + c] += haa;
      if (Jb) { Ubb[a * 6 + c] += hbb; Pab[a * 6 + c] = hab; }
    }
  }
}

static double ba_linearize(ba_state* s) {
  int nc = s->nc, np = s->np, no = s->no;
  memset(s->U, 0, sizeof(double) * 36 * nc); memset(s->gc, 0, sizeof(double) * 6 * nc);
  memset(s->V, 0, sizeof(double) * 9 * np);  memset(s->gp, 0, sizeof(double) * 3 * np);
  memset(s->W, 0, sizeof(double) * 18 * (size_t)no);
  double* Rs = (double*)malloc(sizeof(double) * 9 * (size_t)nc);
  for (int i = 0; i < nc; ++i) quat_to_R(s->pose + 7 * i, Rs + 9 * i);
  double c = 0.0;
#ifdef _OPENMP
  if (g_ba_threads > 1 && no > 4096) {
    /* the same sums as the loop below, regrouped so that threads own disjoint outputs: landmarks (V, g_p, W, cost) then cameras (U, g_c);
     * inside a landmark / camera the observations are visited in ascending index order, i.e. in the sequential loop's order */
    double part[64] = {0};
#pragma omp parallel num_threads(g_ba_threads)
    {
      double acc = 0.0;
#pragma omp for schedule(static)
      for (int j = 0; j < np; ++j) {
        const int pf = ptfree(s, j);
        double* V = s->V + 9 * j;
        for (int e = s->poff[j]; e < s->poff[j + 1]; ++e) {
          const int k = s->plist[e], i = s->oc[k];
          obs_lin o;
          eval_obs(Rs + 9 * i, s->pose + 7 * i + 4, s->pts + 3 * j, s->om + 3 * k, s->oi ? s->oi + 4 * k : NULL, s->delta, 1, &o);
          if (!o.valid) continue;
          acc += o.rho;
          const int dm = dofmask(s, i);
          for (int d = 0; d < 6; ++d) if (!((dm >> d) & 1)) { o.Jc[d] = 0.0; o.Jc[6 + d] = 0.0; }
          if (!pf) for (int d = 0; d < 6; ++d) o.Jp[d] = 0.0;
          double AJp[6], Ar[2];
          for (int d = 0; d < 3; ++d) { AJp[d] = o.A[0] * o.Jp[d] + o.A[1] * o.Jp[3 + d]; AJp[3 + d] = o.A[1] * o.Jp[d] + o.A[2] * o.Jp[3 + d]; }
          Ar[0] = o.A[0] * o.r[0] + o.A[1] * o.r[1]; Ar[1] = o.A[1] * o.r[0] + o.A[2] * o.r[1];
          double* W = s->W + 18 * (size_t)k;
          for (int a = 0; a < 6; ++a) for (int b = 0; b < 3; ++b) W[a * 3 + b] = o.Jc[a] * AJp[b] + o.Jc[6 + a] * AJp[3 + b];
          for (int a = 0; a < 3; ++a) {
            for (int b = 0; b < 3; ++b) V[a * 3 + b] += o.Jp[a] * AJp[b] + o.Jp[3 + a] * AJp[3 + b];
            s->gp[3 * j + a] -= o.Jp[a] * Ar[0] + o.Jp[3 + a] * Ar[1];
          }
        }
      }
      part[omp_get_thread_num()] = acc;
#pragma omp for schedule(static)
      for (int i = 0; i < nc; ++i) {
        const int dm = dofmask(s, i);
        double* U = s->U + 36 * i;
        for (int e = s->coff[i]; e < s->coff[i + 1]; ++e) {
          const int k = s->clist[e], j = s->op[k];
          obs_lin o;
          eval_obs(Rs + 9 * i, s->pose + 7 * i + 4, s->pts + 3 * j, s->om + 3 * k, s->oi ? s->oi + 4 * k : NULL, s->delta, 1, &o);
          if (!o.valid) continue;
          for (int d = 0; d < 6; ++d) if (!((dm >> d) & 1)) { o.Jc[d] = 0.0; o.Jc[6 + d] = 0.0; }
          double AJc[12], Ar[2];
          for (int d = 0; d < 6; ++d) { AJc[d] = o.A[0] * o.Jc[d] + o.A[1] * o.Jc[6 + d]; AJc[6 + d] = o.A[1] * o.Jc[d] + o.A[2] * o.Jc[6 + d]; }
          Ar[0] = o.A[0] * o.r[0] + o.A[1] * o.r[1]; Ar[1] = o.A[1] * o.r[0] + o.A[2] * o.r[1];
          for (int a = 0; a < 6; ++a) {
            for (int b = 0; b < 6; ++b) U[a * 6 + b] += o.Jc[a] * AJc[b] + o.Jc[6 + a] * AJc[6 + b];
            s->gc[6 * i + a] -= o.Jc[a] * Ar[0] + o.Jc[6 + a] * Ar[1];
          }
        }
      }
    }
    for (int t = 0; t < 64; ++t) c += part[t];
    no = 0;  /* (the sequential loop below has nothing left to do) */
  }
#endif
  for (int k = 0; k < no; ++k) {
    obs_lin o;
    int i = s->oc[k], j = s->op[k];
    eval_obs(Rs + 9 * i, s->pose + 7 * i + 4, s->pts + 3 * j, s->om + 3 * k, s->oi ? s->oi + 4 * k : NULL, s->delta, 1, &o);
    if (!o.valid) continue;
    c += o.rho;
    int dm = dofmask(s, i), pf = ptfree(s, j);
    for (int d = 0; d < 6; ++d) if (!((dm >> d) & 1)) { o.Jc[d] = 0.0; o.Jc[6 + d] = 0.0; }
    if (!pf) for (int d = 0; d < 6; ++d) o.Jp[d] = 0.0;
    /* AJc (2x6), AJp (2x3), Ar (2) */
    double AJc[12], AJp[6], Ar[2];
    for (int d = 0; d < 6; ++d) { AJc[d] = o.A[0] * o.Jc[d] + o.A[1] * o.Jc[6 + d]; AJc[6 + d] = o.A[1] * o.Jc[d] + o.A[2] * o.Jc[6 + d]; }
    for (int d = 0; d < 3; ++d) { AJp[d] = o.A[0] * o.Jp[d] + o.A[1] * o.Jp[3 + d]; AJp[3 + d] = o.A[1] * o.Jp[d] + o.A[2] * o.Jp[3 + d]; }
    Ar[0] = o.A[0] * o.r[0] + o.A[1] * o.r[1]; Ar[1] = o.A[1] * o.r[0] + o.A[2] * o.r[1];
    double* U = s->U + 36 * i; double* V = s->V + 9 * j; double* W = s->W + 18 * (size_t)k;
    for (int a = 0; a < 6; ++a) {
      for (int b = 0; b < 6; ++b) U[a * 6 + b] += o.Jc[a] * AJc[b] + o.Jc[6 + a] * AJc[6 + b];
      s->gc[6 * i + a] -= o.Jc[a] * Ar[0] + o.Jc[6 + a] * Ar[1];
      for (int b = 0; b < 3; ++b) W[a * 3 + b] = o.Jc[a] * AJp[b] + o.Jc[6 + a] * AJp[3 + b];
    }
    for (int a = 0; a < 3; ++a) {
      for (int b = 0; b < 3; ++b) V[a * 3 + b] += o.Jp[a] * AJp[b] + o.Jp[3 + a] * AJp[3 + b];
      s->gp[3 * j + a] -= o.Jp[a] * Ar[0] + o.Jp[3 + a] * Ar[1];
    }
  }
  free(Rs);
  for (int k = 0; k < s->nse; ++k) {
    double e[6], Ji[36], Jj[36];
    const int i = s->se_i[k], j = s->se_j[k];
    const double* info = s->se_info ? s->se_info + 36 * k : NULL;
    pose_edge_eval(s->se_Zinv + 7 * k, s->pose + 7 * i, s->pose + 7 * j, 0, e, Ji, Jj);
    c += quad6(info, e);
    pose_term_accumulate(info, e, Ji, dofmask(s, i), Jj, dofmask(s, j), s->U + 36 * i, s->gc + 6 * i, s->U + 36 * j, s->gc + 6 * j, s->P + 36 * (size_t)k);
  }
  for (int k = 0; k < s->ngps; ++k) {
    double e[6], Ji[36];
    const int i = s->gps_i[k];
    const double* info = s->gps_info ? s->gps_info + 36 * k : NULL;
    pose_edge_eval(s->gps_Zinv + 7 * k, s->pose + 7 * i, NULL, 1, e, Ji, NULL);
    c += quad6(info, e);
    pose_term_accumulate(info, e, Ji, dofmask(s, i), NULL, 0, s->U + 36 * i, s->gc + 6 * i, NULL, NULL, NULL);
  }
  return 0.5 * c;
}

/* Exposed for kernel-level parity tests: linearise `problem` at its estimate. Outputs may be NULL.
 * U: nc*36, gc: nc*6, V: np*9, gp: np*3, W: no*18 (in the caller's observation order). */
static void state_init_ex(ba_state* s, const gb_ba_problem* pb, const gb_pose_edges* pe, double delta) {
  memset(s, 0, sizeof *s);
  s->nc = pb->n_cams; s->np = pb->n_points; s->no = pb->n_obs;
  s->dof = pb->cam_dof; s->pfree = pb->point_free; s->oc = pb->obs_cam; s->op = pb->obs_point; s->om = pb->obs_xyz; s->oi = pb->obs_info;
  s->delta = delta;
  s->pose = (double*)malloc(sizeof(double) * 7 * (size_t)(s->nc > 0 ? s->nc : 1));
  s->pts = (double*)malloc(sizeof(double) * 3 * (size_t)(s->np > 0 ? s->np : 1));
  for (int i = 0; i < s->nc; ++i) orc_se3_inverse(pb->cam_pose_wc + 7 * i, s->pose + 7 * i);
  memcpy(s->pts, pb->points, sizeof(double) * 3 * (size_t)s->np);
  s->U = (double*)calloc(36 * (size_t)(s->nc + 1), sizeof(double)); s->gc = (double*)calloc(6 * (size_t)(s->nc + 1), sizeof(double));
  s->V = (double*)calloc(9 * (size_t)(s->np + 1), sizeof(double));  s->gp = (double*)calloc(3 * (size_t)(s->np + 1), sizeof(double));
  s->W = (double*)calloc(18 * (size_t)(s->no + 1), sizeof(double));
  s->poff = (int*)calloc((size_t)s->np + 2, sizeof(int)); s->plist = (int*)calloc((size_t)s->no + 1, sizeof(int));
  for (int k = 0; k < s->no; ++k) s->poff[s->op[k] + 1]++;
  for (int j = 0; j < s->np; ++j) s->poff[j + 1] += s->poff[j];
  int* fill = (int*)calloc((size_t)s->np + 1, sizeof(int));
  for (int k = 0; k < s->no; ++k) { int j = s->op[k]; s->plist[s->poff[j] + fill[j]++] = k; }
  free(fill);
  s->coff = (int*)calloc((size_t)s->nc + 2, sizeof(int)); s->clist = (int*)calloc((size_t)s->no + 1, sizeof(int));
  for (int k = 0; k < s->no; ++k) s->coff[s->oc[k] + 1]++;
  for (int i = 0; i < s->nc; ++i) s->coff[i + 1] += s->coff[i];
  fill = (int*)calloc((size_t)s->nc + 1, sizeof(int));
  for (int k = 0; k < s->no; ++k) { int i = s->oc[k]; s->clist[s->coff[i] + fill[i]++] = k; }
  free(fill);
  if (pe) {
    s->nse = pe->n_se3; s->ngps = pe->n_gps;
    s->se_i = pe->se3_first; s->se_j = pe->se3_second; s->gps_i = pe->gps_frame; s->se_info = pe->se3_info; s->gps_info = pe->gps_info;
  }
  s->se_Zinv = (double*)malloc(sizeof(double) * 7 * (size_t)(s->nse + 1));
  s->gps_Zinv = (double*)malloc(sizeof(double) * 7 * (size_t)(s->ngps + 1));
  s->P = (double*)calloc(36 * (size_t)(s->nse + 1), sizeof(double));
  for (int k = 0; k < s->nse; ++k) orc_se3_inverse(pe->se3_meas + 7 * k, s->se_Zinv + 7 * k);
  for (int k = 0; k < s->ngps; ++k) orc_se3_inverse(pe->gps_meas + 7 * k, s->gps_Zinv + 7 * k);
}
static void state_init(ba_state* s, const gb_ba_problem* pb, double delta) { state_init_ex(s, pb, NULL, delta); }
static void state_free(ba_state* s) {
  free(s->pose); free(s->pts); free(s->U); free(s->gc); free(s->V); free(s->gp); free(s->W); free(s->poff); free(s->plist); free(s->coff); free(s->clist);
  free(s->se_Zinv); free(s->gps_Zinv); free(s->P);
}
static int validate_edges(const gb_ba_problem* pb, const gb_pose_edges* pe) {
  if (!pe) return 0;
  if (pe->n_se3 < 0 || pe->n_gps < 0) return 1;
  for (int k = 0; k < pe->n_se3; ++k)
    if (pe->se3_first[k] < 0 || pe->se3_first[k] >= pb->n_cams || pe->se3_second[k] < 0 || pe->se3_second[k] >= pb->n_cams || pe->se3_first[k] == pe->se3_second[k]) return 1;
  for (int k = 0; k < pe->n_gps; ++k)
    if (pe->gps_frame[k] < 0 || pe->gps_frame[k] >= pb->n_cams) return 1;
  return 0;
}

static int validate(const gb_ba_problem* pb) {
  if (!pb || pb->n_cams < 0 || pb->n_points < 0 || pb->n_obs < 0) return 1;
  for (int k = 0; k < pb->n_obs; ++k)
    if (pb->obs_cam[k] < 0 || pb->obs_cam[k] >= pb->n_cams || pb->obs_point[k] < 0 || pb->obs_point[k] >= pb->n_points) return 1;
  return 0;
}

int orc_ba_linearize_ex(const gb_ba_problem* pb, const gb_pose_edges* pe, double delta, double* U, double* gc, double* V, double* gp, double* W, double* cost) {
  if (validate(pb) || validate_edges(pb, pe)) return GB_ERR_INVALID;
  ba_state s;
  state_init_ex(&s, pb, pe, delta);
  double c = ba_linearize(&s);
  if (U) memcpy(U, s.U, sizeof(double) * 36 * (size_t)s.nc);
  if (gc) memcpy(gc, s.gc, sizeof(double) * 6 * (size_t)s.nc);
  if (V) memcpy(V, s.V, sizeof(double) * 9 * (size_t)s.np);
  if (gp) memcpy(gp, s.gp, sizeof(double) * 3 * (size_t)s.np);
  if (W) memcpy(W, s.W, sizeof(double) * 18 * (size_t)s.no);
  if (cost) *cost = c;
  state_free(&s);
  return GB_OK;
}

int orc_ba_linearize(const gb_ba_problem* pb, double delta, double* U, double* gc, double* V, double* gp, double* W, double* cost) {
  return orc_ba_linearize_ex(pb, NULL, delta, U, gc, V, gp, W, cost);
}

int orc_ba_cost_ex(const gb_ba_problem* pb, const gb_pose_edges* pe, double delta, double* cost) {
  if (validate(pb) || validate_edges(pb, pe)) return GB_ERR_INVALID;
  ba_state s;
  state_init_ex(&s, pb, pe, delta);
  *cost = ba_cost(&s, s.pose, s.pts);
  state_free(&s);
  return GB_OK;
}

int orc_ba_cost(const gb_ba_problem* pb, double delta, double* cost) { return orc_ba_cost_ex(pb, NULL, delta, cost); }

/* Build the damped reduced camera system: S (n6 x n6 dense, row-major), gt (n6), Vinv (np x 9). */
static void ba_schur(const ba_state* s, double lambda, double* S, double* gt, double* Vinv) {
  int nc = s->nc, np = s->np, n6 = 6 * nc;
  memset(S, 0, sizeof(double) * (size_t)n6 * n6);
  for (int i = 0; i < nc; ++i) {
    int dm = dofmask(s, i);
    for (int a = 0; a < 6; ++a) {
      for (int b = 0; b < 6; ++b) S[(size_t)(6 * i + a) * n6 + 6 * i + b] = s->U[36 * i + a * 6 + b];
      if ((dm >> a) & 1) S[(size_t)(6 * i + a) * n6 + 6 * i + a] += lambda * clampd(s->U[36 * i + a * 7]);
      else S[(size_t)(6 * i + a) * n6 + 6 * i + a] = 1.0;
      gt[6 * i + a] = s->gc[6 * i + a];
    }
  }
  for (int k = 0; k < s->nse; ++k) { /* pose-graph coupling: S_ij += J_i' Omega J_j, S_ji += its transpose */
    const int i = s->se_i[k], j = s->se_j[k];
    const double* P = s->P + 36 * (size_t)k;
    for (int a = 0; a < 6; ++a)
      for (int b = 0; b < 6; ++b) {
        S[(size_t)(6 * i + a) * n6 + 6 * j + b] += P[a * 6 + b];
        S[(size_t)(6 * j + b) * n6 + 6 * i + a] += P[a * 6 + b];
      }
  }
  int T = 1;
#ifdef _OPENMP
  if (g_ba_threads > 1 && np > 256) T = g_ba_threads;
#endif
  double* Sall = T > 1 ? (double*)calloc((size_t)T * ((size_t)n6 * n6 + n6), sizeof(double)) : NULL;
#ifdef _OPENMP
#pragma omp parallel num_threads(T) if (T > 1)
#endif
  {
  double* S_acc = S; double* gt_acc = gt;  /* thread-local partial system when T > 1 (folded in thread order below) */
#ifdef _OPENMP
  if (T > 1) { S_acc = Sall + (size_t)omp_get_thread_num() * ((size_t)n6 * n6 + n6); gt_acc = S_acc + (size_t)n6 * n6; }
#pragma omp for schedule(static)
#endif
  for (int j = 0; j < np; ++j) {
    double* Vi = Vinv + 9 * j;
    memset(Vi, 0, sizeof(double) * 9);
    int n = s->poff[j + 1] - s->poff[j];
    if (!ptfree(s, j) || n == 0) continue;
    memcpy(Vi, s->V + 9 * j, sizeof(double) * 9);
    for (int a = 0; a < 3; ++a) Vi[a * 4] += lambda * clampd(s->V[9 * j + a * 4]);
    if (spd_inverse(Vi, 3)) { memset(Vi, 0, sizeof(double) * 9); continue; }
    for (int e = 0; e < n; ++e) {
      int k = s->plist[s->poff[j] + e], i = s->oc[k];
      const double* Wk = s->W + 18 * (size_t)k;
      double Y[18];
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 3; ++b) Y[a * 3 + b] = Wk[a * 3] * Vi[b] + Wk[a * 3 + 1] * Vi[3 + b] + Wk[a * 3 + 2] * Vi[6 + b];
      for (int a = 0; a < 6; ++a)
        gt_acc[6 * i + a] -= Y[a * 3] * s->gp[3 * j] + Y[a * 3 + 1] * s->gp[3 * j + 1] + Y[a * 3 + 2] * s->gp[3 * j + 2];
      for (int f = 0; f < n; ++f) {
        int k2 = s->plist[s->poff[j] + f], i2 = s->oc[k2];
        const double* W2 = s->W + 18 * (size_t)k2;
        for (int a = 0; a < 6; ++a)
          for (int b = 0; b < 6; ++b)
            S_acc[(size_t)(6 * i + a) * n6 + 6 * i2 + b] -= Y[a * 3] * W2[b * 3] + Y[a * 3 + 1] * W2[b * 3 + 1] + Y[a * 3 + 2] * W2[b * 3 + 2];
      }
    }
  }
  }
  if (T > 1) { /* fold the partial systems in thread order */
#ifdef _OPENMP
#pragma omp parallel for schedule(static) num_threads(T)
#endif
    for (int r = 0; r < n6; ++r)
      for (int t = 0; t < T; ++t) {
        const double* P = Sall + (size_t)t * ((size_t)n6 * n6 + n6);
        for (int c = 0; c < n6; ++c) S[(size_t)r * n6 + c] += P[(size_t)r * n6 + c];
        gt[r] += P[(size_t)n6 * n6 + r];
      }
    free(Sall);
  }
}

/* Block-Jacobi preconditioned CG on S x = g in the Chronopoulos-Gear arrangement (one fused pair of inner products per
 * iteration: gamma = r'u and delta = w'u with u = M^-1 r, w = S u; p and s = S p follow by recurrence).  In exact arithmetic it
 * is the classical PCG iteration; it is stated this way because it is what the GPU kernels run (two barriers and one
 * reduction per iteration instead of four and two).  Returns the number of x updates. */
static int ba_pcg(int nc, const double* S, const double* g, double* x, int maxit, double tol) {
  int n6 = 6 * nc;
  double* Minv = (double*)malloc(sizeof(double) * 36 * (size_t)(nc + 1));
  size_t nb = sizeof(double) * (size_t)(n6 + 1);
  double *r = (double*)malloc(nb), *u = (double*)malloc(nb), *w = (double*)malloc(nb), *p = (double*)calloc((size_t)n6 + 1, sizeof(double)),
         *sv = (double*)calloc((size_t)n6 + 1, sizeof(double));
  for (int i = 0; i < nc; ++i) {
    for (int a = 0; a < 6; ++a) for (int b = 0; b < 6; ++b) Minv[36 * i + a * 6 + b] = S[(size_t)(6 * i + a) * n6 + 6 * i + b];
    if (spd_inverse(Minv + 36 * i, 6)) { /* fall back to the diagonal */
      for (int a = 0; a < 6; ++a) for (int b = 0; b < 6; ++b) Minv[36 * i + a * 6 + b] = (a == b) ? 1.0 / S[(size_t)(6 * i + a) * n6 + 6 * i + a] : 0.0;
    }
  }
#define APPLY_MINV(src, dst) \
  for (int i = 0; i < nc; ++i) for (int a = 0; a < 6; ++a) { double sacc = 0.0; for (int b = 0; b < 6; ++b) sacc += Minv[36 * i + a * 6 + b] * (src)[6 * i + b]; (dst)[6 * i + a] = sacc; }
#define MATVEC(src, dst) \
  _Pragma("omp parallel for schedule(static) num_threads(g_ba_threads) if (g_ba_threads > 1 && n6 >= 192)") \
  for (int a = 0; a < n6; ++a) { double sacc = 0.0; const double* row = S + (size_t)a * n6; for (int b = 0; b < n6; ++b) sacc += row[b] * (src)[b]; (dst)[a] = sacc; }
  int it = 0;
  for (int a = 0; a < n6; ++a) { x[a] = 0.0; r[a] = g[a]; }
  APPLY_MINV(r, u);
  MATVEC(u, w);
  double gamma = 0.0, delta = 0.0;
  for (int a = 0; a < n6; ++a) { gamma += r[a] * u[a]; delta += w[a] * u[a]; }
  const double gamma0 = gamma;
  if (gamma0 > 0.0 && delta > 0.0) {
    double alpha = gamma / delta, beta = 0.0;
    while (it < maxit) {
      for (int a = 0; a < n6; ++a) {
        p[a] = u[a] + beta * p[a];
        sv[a] = w[a] + beta * sv[a];
        x[a] += alpha * p[a];
        r[a] -= alpha * sv[a];
      }
      APPLY_MINV(r, u);
      ++it;
      double gn = 0.0;
      for (int a = 0; a < n6; ++a) gn += r[a] * u[a];
      if (!(gn > 0.0) || gn < tol * tol * gamma0) break; /* == sqrt(gn/gamma0) < tol without the sqrt/div */
      MATVEC(u, w);
      delta = 0.0;
      for (int a = 0; a < n6; ++a) delta += w[a] * u[a];
      beta = gn / gamma;
      const double den = delta - beta * gn / alpha;
      if (!(den > 0.0)) break;
      alpha = gn / den;
      gamma = gn;
    }
  }
#undef APPLY_MINV
#undef MATVEC
  free(Minv); free(r); free(u); free(w); free(p); free(sv);
  return it;
}

/* Direct solve of S x = g (S dense SPD, n6 x n6, destroyed): plain Cholesky + two substitutions.  A non-positive pivot gives the zero
 * step (LM then rejects it and raises lambda) -- the convention of gslam_b200/csrc/ba_chol.cu.  Returns 0. */
static int ba_chol_solve(int nc, double* S, const double* g, double* x) {
  int n = 6 * nc, fail = 0;
  for (int j = 0; j < n && !fail; ++j) {
    double d = S[(size_t)j * n + j];
    for (int m = 0; m < j; ++m) d -= S[(size_t)j * n + m] * S[(size_t)j * n + m];
    if (!(d > 0.0) || !(d < 1e300)) { fail = 1; break; }
    double l = sqrt(d);
    S[(size_t)j * n + j] = l;
    for (int i = j + 1; i < n; ++i) {
      double v = S[(size_t)i * n + j];
      for (int m = 0; m < j; ++m) v -= S[(size_t)i * n + m] * S[(size_t)j * n + m];
      S[(size_t)i * n + j] = v / l;
    }
  }
  if (!fail) {
    for (int i = 0; i < n; ++i) {
      double v = g[i];
      for (int m = 0; m < i; ++m) v -= S[(size_t)i * n + m] * x[m];
      x[i] = v / S[(size_t)i * n + i];
    }
    for (int i = n - 1; i >= 0; --i) {
      double v = x[i];
      for (int m = i + 1; m < n; ++m) v -= S[(size_t)m * n + i] * x[m];
      x[i] = v / S[(size_t)i * n + i];
    }
    for (int i = 0; i < n; ++i) if (!isfinite(x[i])) fail = 1;
  }
  if (fail) for (int i = 0; i < n; ++i) x[i] = 0.0;
  return 0;
}

/* Exposed for kernel-level parity tests: S (6nc x 6nc), gt (6nc) and the PCG solution dc (6nc) at the input estimate. */
int orc_ba_reduced_system_ex(const gb_ba_problem* pb, const gb_pose_edges* pe, double delta, double lambda, int pcg_maxit, double pcg_tol, double* S, double* gt, double* dc, int* pcg_iters) {
  if (validate(pb) || validate_edges(pb, pe)) return GB_ERR_INVALID;
  ba_state s;
  state_init_ex(&s, pb, pe, delta);
  ba_linearize(&s);
  double* Vinv = (double*)malloc(sizeof(double) * 9 * (size_t)(s.np + 1));
  ba_schur(&s, lambda, S, gt, Vinv);
  if (dc) { int it = ba_pcg(s.nc, S, gt, dc, pcg_maxit, pcg_tol); if (pcg_iters) *pcg_iters = it; }
  free(Vinv);
  state_free(&s);
  return GB_OK;
}

int orc_ba_reduced_system(const gb_ba_problem* pb, double delta, double lambda, int pcg_maxit, double pcg_tol, double* S, double* gt, double* dc, int* pcg_iters) {
  return orc_ba_reduced_system_ex(pb, NULL, delta, lambda, pcg_maxit, pcg_tol, S, gt, dc, pcg_iters);
}

int orc_ba_solve_ex(gb_ba_problem* pb, const gb_pose_edges* pe, const gb_ba_options* opt_in, gb_ba_result* res);
int orc_ba_solve(gb_ba_problem* pb, const gb_ba_options* opt_in, gb_ba_result* res) { return orc_ba_solve_ex(pb, NULL, opt_in, res); }

int orc_ba_solve_ex(gb_ba_problem* pb, const gb_pose_edges* pe, const gb_ba_options* opt_in, gb_ba_result* res) {
  gb_ba_options opt;
  if (opt_in) opt = *opt_in; else { opt.projection = 0; opt.huber_delta = 0.01; opt.max_iterations = 500; opt.verbose = 0; opt.function_tolerance = 1e-6; opt.lambda_init = 1e-4; opt.pcg_max_iters = 50; opt.pcg_tol = 1e-10; opt.linear_solver = 0; }
  if (validate(pb) || validate_edges(pb, pe) || opt.projection != 0) return GB_ERR_INVALID;
  /* the option checks of gb_ba_graph_begin */
  if (opt.max_iterations < 0 || opt.pcg_max_iters < 0 || !(isfinite(opt.lambda_init) && opt.lambda_init > 0.0) || isnan(opt.huber_delta) ||
      isnan(opt.function_tolerance) || isnan(opt.pcg_tol))
    return GB_ERR_INVALID;
  ba_state s;
  state_init_ex(&s, pb, pe, opt.huber_delta);
  int nc = s.nc, np = s.np, n6 = 6 * nc;
  double* S = (double*)malloc(sizeof(double) * ((size_t)n6 * n6 + 1));
  double *gt = (double*)malloc(sizeof(double) * (size_t)(n6 + 1)), *dc = (double*)malloc(sizeof(double) * (size_t)(n6 + 1));
  double* Vinv = (double*)malloc(sizeof(double) * 9 * (size_t)(np + 1));
  double* pose_new = (double*)malloc(sizeof(double) * 7 * (size_t)(nc + 1));
  double* pts_new = (double*)malloc(sizeof(double) * 3 * (size_t)(np + 1));
  double lambda = opt.lambda_init, nu = 2.0;
  double cost = ba_linearize(&s);
  gb_ba_result R; memset(&R, 0, sizeof R);
  R.initial_cost = cost;
  int it = 0;
  for (; it < opt.max_iterations; ++it) {
    ba_schur(&s, lambda, S, gt, Vinv);
    if (opt.linear_solver == 1) ba_chol_solve(nc, S, gt, dc);
    else R.pcg_iterations += ba_pcg(nc, S, gt, dc, opt.pcg_max_iters, opt.pcg_tol);
    for (int i = 0; i < nc; ++i) {
      double d[6]; int dm = dofmask(&s, i);
      for (int a = 0; a < 6; ++a) d[a] = ((dm >> a) & 1) ? dc[6 * i + a] : 0.0;
      orc_se3_retract(s.pose + 7 * i, d, pose_new + 7 * i);
    }
    for (int j = 0; j < np; ++j) {
      double b[3] = {s.gp[3 * j], s.gp[3 * j + 1], s.gp[3 * j + 2]};
      for (int e = s.poff[j]; e < s.poff[j + 1]; ++e) {
        int k = s.plist[e], i = s.oc[k];
        const double* Wk = s.W + 18 * (size_t)k;
        for (int c = 0; c < 3; ++c) for (int a = 0; a < 6; ++a) b[c] -= Wk[a * 3 + c] * dc[6 * i + a];
      }
      const double* Vi = Vinv + 9 * j;
      for (int a = 0; a < 3; ++a) pts_new[3 * j + a] = s.pts[3 * j + a] + Vi[a * 3] * b[0] + Vi[a * 3 + 1] * b[1] + Vi[a * 3 + 2] * b[2];
    }
    double cnew = ba_cost(&s, pose_new, pts_new);
    int ok = (cnew < cost) && isfinite(cnew);
    if (opt.verbose) fprintf(stderr, "[ba_ref] it %d cost %.12e -> %.12e lambda %.3e %s\n", it, cost, cnew, lambda, ok ? "accept" : "reject");
    if (ok) {
      double rel = (cost - cnew) / cost;
      memcpy(s.pose, pose_new, sizeof(double) * 7 * (size_t)nc);
      memcpy(s.pts, pts_new, sizeof(double) * 3 * (size_t)np);
      cost = ba_linearize(&s);
      lambda = lambda / 3.0; if (lambda < 1e-15) lambda = 1e-15;
      nu = 2.0;
      R.accepted++;
      if (rel < opt.function_tolerance) { R.status = 1; ++it; break; }
    } else {
      lambda *= nu; nu *= 2.0;
      if (lambda > 1e16) { R.status = 2; ++it; break; }
    }
  }
  R.iterations = it; R.final_cost = cost; R.lambda_final = lambda;
  for (int i = 0; i < nc; ++i) orc_se3_inverse(s.pose + 7 * i, pb->cam_pose_wc + 7 * i);
  memcpy(pb->points, s.pts, sizeof(double) * 3 * (size_t)np);
  if (res) *res = R;
  free(S); free(gt); free(dc); free(Vinv); free(pose_new); free(pts_new);
  state_free(&s);
  return GB_OK;
}

/* optimizePnP (Optimizer.h:202-207): one camera, all points fixed. info6x6 (may be NULL) receives U at the result. */
int orc_ba_pnp(int n, const double* xyz, const double* xy1, double* pose_wc, int dof, double* info6x6, const gb_ba_options* opt, gb_ba_result* res) {
  if (n < 0) return GB_ERR_INVALID;
  gb_ba_problem pb; memset(&pb, 0, sizeof pb);
  uint8_t d = (uint8_t)(dof & 63);
  uint8_t* pf = (uint8_t*)calloc((size_t)n + 1, 1);
  int32_t* oc = (int32_t*)calloc((size_t)n + 1, sizeof(int32_t)); int32_t* op = (int32_t*)calloc((size_t)n + 1, sizeof(int32_t));
  double* pts = (double*)malloc(sizeof(double) * 3 * (size_t)(n + 1));
  memcpy(pts, xyz, sizeof(double) * 3 * (size_t)n);
  for (int k = 0; k < n; ++k) op[k] = k;
  pb.n_cams = 1; pb.n_points = n; pb.n_obs = n; pb.cam_pose_wc = pose_wc; pb.cam_dof = &d; pb.points = pts; pb.point_free = pf;
  pb.obs_cam = oc; pb.obs_point = op; pb.obs_xyz = xy1; pb.obs_info = NULL;
  int rc = orc_ba_solve(&pb, opt, res);
  if (rc == GB_OK && info6x6) {
    double delta = opt ? opt->huber_delta : 0.01;
    rc = orc_ba_linearize(&pb, delta, info6x6, NULL, NULL, NULL, NULL, NULL);
  }
  free(pf); free(oc); free(op); free(pts);
  return rc;
}
