// gslam_b200/csrc/pnp.cu — P3P + RANSAC pose estimation from 3D-2D matches: the kernel side of SURVEY.md §8f-1,
// GSLAM::Estimator::findPnP (GSLAM/core/Estimator.h:158-164; factory :175-191).
//
// It mirrors the CPU checker operation for operation; tests/test_pnp_gpu.py compares the two.
//
// Design: RANSAC hypotheses are independent work items.  Hypothesis h draws its three correspondences from a counter-based
// generator (splitmix64 of seed and h: no sequential state), solves P3P (Grunert's distance formulation: quartic in v = s3/s1 built
// by polynomial arithmetic, roots bracketed between the critical points, 64 bisection + 2 Newton steps, then 3 Newton steps on
// the original pair of equations), and scores every solution by its inlier count (z > 0 and squared normalised reprojection error
// < threshold^2).  ONE warp per hypothesis: lane 0 solves the minimal problem (a ~3 kflop latency chain), all 32 lanes score.
// max_hypotheses warps are launched at once (2048 hypotheses x 2000 points is ~0.1 GFLOP of fp64); the host then replays the
// sequential stopping rule of the definition (batches of 64, stop once h >= log(1-confidence)/log(1-w^3)) over the per-hypothesis
// counts, so the result does not depend on how much was computed speculatively.  Refinement = the optimizePnP solver (gb_ba_pnp)
// on the inliers.  Compiled with --fmad=false: inlier counts are integers compared across hypotheses, so the arithmetic is kept
// free of contraction differences.
#include "common.cuh"

#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/gslam_b200.h"

namespace {

constexpr int kHypPerCta = 8;
constexpr double kPi = 3.14159265358979323846;

__host__ __device__ inline uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__host__ __device__ inline void pnp_sample(uint64_t seed, int h, int n, int idx[3]) {
  const uint64_t r0 = splitmix64(seed ^ (0x100000001B3ull * (uint64_t)(3 * h + 1)));
  const uint64_t r1 = splitmix64(seed ^ (0x100000001B3ull * (uint64_t)(3 * h + 2)));
  const uint64_t r2 = splitmix64(seed ^ (0x100000001B3ull * (uint64_t)(3 * h + 3)));
  int i0 = (int)(r0 % (uint64_t)n), i1 = (int)(r1 % (uint64_t)(n - 1)), i2 = (int)(r2 % (uint64_t)(n - 2));
  if (i1 >= i0) ++i1;
  const int lo = i0 < i1 ? i0 : i1, hi = i0 < i1 ? i1 : i0;
  if (i2 >= lo) ++i2;
  if (i2 >= hi) ++i2;
  idx[0] = i0; idx[1] = i1; idx[2] = i2;
}

__host__ __device__ inline void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
__host__ __device__ inline double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// all real roots of x^3 + a x^2 + b x + c
__host__ __device__ int cubic_real_roots(double a, double b, double c, double* x) {
  const double q = (a * a - 3.0 * b) / 9.0, r = (2.0 * a * a * a - 9.0 * a * b + 27.0 * c) / 54.0;
  const double q3 = q * q * q;
  if (r * r < q3) {
    const double t = acos(fmax(-1.0, fmin(1.0, r / sqrt(q3)))), m = -2.0 * sqrt(q);
    x[0] = m * cos(t / 3.0) - a / 3.0;
    x[1] = m * cos((t + 2.0 * kPi) / 3.0) - a / 3.0;
    x[2] = m * cos((t - 2.0 * kPi) / 3.0) - a / 3.0;
    return 3;
  }
  double A = -cbrt(fabs(r) + sqrt(r * r - q3));
  if (r < 0) A = -A;
  const double B = (A == 0.0) ? 0.0 : q / A;
  x[0] = (A + B) - a / 3.0;
  return 1;
}

// real roots of c[0] + ... + c[4] x^4, ascending: brackets between the critical points, bisection + guarded Newton
__host__ __device__ int quartic_roots(const double* c, double* roots) {
  if (c[4] == 0.0) return 0;
  const double a3 = c[3] / c[4], a2 = c[2] / c[4], a1 = c[1] / c[4], a0 = c[0] / c[4];
#define QF(x) (((((x) + a3) * (x) + a2) * (x) + a1) * (x) + a0)
#define QD(x) (((4.0 * (x) + 3.0 * a3) * (x) + 2.0 * a2) * (x) + a1)
  double crit[3];
  const int nc = cubic_real_roots(0.75 * a3, 0.5 * a2, 0.25 * a1, crit);
  for (int i = 0; i < nc; ++i)
    for (int j = i; j > 0 && crit[j] < crit[j - 1]; --j) { const double t = crit[j]; crit[j] = crit[j - 1]; crit[j - 1] = t; }
  const double B = 1.0 + fmax(fmax(fabs(a3), fabs(a2)), fmax(fabs(a1), fabs(a0)));
  double brk[5];
  int nb = 0;
  brk[nb++] = -B;
  for (int i = 0; i < nc; ++i)
    if (crit[i] > -B && crit[i] < B) brk[nb++] = crit[i];
  brk[nb++] = B;
  int n = 0;
  for (int i = 0; i + 1 < nb; ++i) {
    double lo = brk[i], hi = brk[i + 1];
    double flo = QF(lo), fhi = QF(hi);
    if ((flo < 0.0) == (fhi < 0.0) && flo != 0.0 && fhi != 0.0) {
      if (i > 0) {
        const double x = lo, scale = (((fabs(x) + fabs(a3)) * fabs(x) + fabs(a2)) * fabs(x) + fabs(a1)) * fabs(x) + fabs(a0);
        const double fprev = QF(brk[i - 1]);
        if (fabs(flo) <= 1e-12 * scale && (fprev < 0.0) == (flo < 0.0) && n < 4 && (n == 0 || roots[n - 1] != x)) roots[n++] = x;
      }
      continue;
    }
    if (flo == 0.0) { if (n < 4 && (n == 0 || roots[n - 1] != lo)) roots[n++] = lo; if (fhi != 0.0) continue; }
    if (fhi == 0.0) { if (i + 2 == nb && n < 4) roots[n++] = hi; continue; }
    for (int it = 0; it < 64; ++it) {
      const double mid = 0.5 * (lo + hi), fm = QF(mid);
      if (mid == lo || mid == hi) break;
      if ((fm < 0.0) == (flo < 0.0)) { lo = mid; flo = fm; } else { hi = mid; fhi = fm; }
    }
    double x = 0.5 * (lo + hi);
    for (int it = 0; it < 2; ++it) {
      const double d = QD(x);
      if (d != 0.0) {
        const double xn = x - QF(x) / d;
        if (xn >= lo && xn <= hi) x = xn;
      }
    }
    if (n < 4) roots[n++] = x;
  }
#undef QF
#undef QD
  return n;
}

__host__ __device__ inline void poly_mul(const double* a, int da, const double* b, int db, double* o) {
  for (int i = 0; i <= da + db; ++i) o[i] = 0.0;
  for (int i = 0; i <= da; ++i)
    for (int j = 0; j <= db; ++j) o[i + j] += a[i] * b[j];
}

// X: three world points, f: three unit bearings; up to 4 solutions Rt[12] = R (row-major, world->camera) | t
__host__ __device__ int p3p(const double* X, const double* f, double* Rt_out) {
  const double *P1 = X, *P2 = X + 3, *P3 = X + 6, *f1 = f, *f2 = f + 3, *f3 = f + 6;
  double v12[3], v13[3], v23[3];
  for (int k = 0; k < 3; ++k) { v12[k] = P2[k] - P1[k]; v13[k] = P3[k] - P1[k]; v23[k] = P3[k] - P2[k]; }
  const double a2 = dot3(v23, v23), b2 = dot3(v13, v13), c2 = dot3(v12, v12);
  double nrm[3];
  cross3(v12, v13, nrm);
  if (a2 == 0.0 || b2 == 0.0 || c2 == 0.0 || dot3(nrm, nrm) < 1e-24 * b2 * c2) return 0;
  const double ca = dot3(f2, f3), cb = dot3(f1, f3), cg = dot3(f1, f2);
  const double qv[3] = {1.0, -2.0 * cb, 1.0};
  double N[3], D[2];
  for (int k = 0; k < 3; ++k) N[k] = (a2 - c2) * qv[k];
  N[0] += b2; N[2] -= b2;
  D[0] = 2.0 * b2 * cg; D[1] = -2.0 * b2 * ca;
  double NN[5], ND[4], DD[3], K[3], KDD[5], poly[5];
  poly_mul(N, 2, N, 2, NN);
  poly_mul(N, 2, D, 1, ND);
  poly_mul(D, 1, D, 1, DD);
  for (int k = 0; k < 3; ++k) K[k] = -c2 * qv[k];
  K[0] += b2;
  poly_mul(K, 2, DD, 2, KDD);
  for (int k = 0; k < 5; ++k) poly[k] = b2 * NN[k] + KDD[k];
  for (int k = 0; k < 4; ++k) poly[k] -= 2.0 * b2 * cg * ND[k];
  if (fabs(poly[4]) < 1e-14 * (fabs(poly[0]) + fabs(poly[1]) + fabs(poly[2]) + fabs(poly[3]) + 1e-300)) return 0;
  double roots[4];
  const int nr = quartic_roots(poly, roots);
  double ex1[3], ex2[3], ex3[3];
  {
    const double l = sqrt(dot3(v12, v12));
    for (int k = 0; k < 3; ++k) ex1[k] = v12[k] / l;
    const double ln = sqrt(dot3(nrm, nrm));
    for (int k = 0; k < 3; ++k) ex3[k] = nrm[k] / ln;
    cross3(ex3, ex1, ex2);
  }
  int ns = 0;
  for (int r = 0; r < nr; ++r) {
    const double v = roots[r];
    if (!(v > 0.0)) continue;
    const double q = 1.0 + v * v - 2.0 * v * cb;
    if (!(q > 0.0)) continue;
    const double den = 2.0 * b2 * (cg - ca * v);
    double u;
    if (fabs(den) > 1e-12 * b2) u = (b2 * (1.0 - v * v) + (a2 - c2) * q) / den;
    else {
      const double A = b2, Bq = -2.0 * b2 * cg, Cc = b2 - c2 * q, disc = Bq * Bq - 4.0 * A * Cc;
      if (disc < 0.0) continue;
      const double u0 = (-Bq + sqrt(disc)) / (2.0 * A), u1 = (-Bq - sqrt(disc)) / (2.0 * A);
      const double e0 = fabs(b2 * (u0 * u0 + v * v - 2.0 * u0 * v * ca) - a2 * q), e1 = fabs(b2 * (u1 * u1 + v * v - 2.0 * u1 * v * ca) - a2 * q);
      u = e0 <= e1 ? u0 : u1;
    }
    if (!(u > 0.0)) continue;
    double uu = u, vv = v;
    for (int it = 0; it < 3; ++it) {  // Newton on the original pair (the quartic is the squared system)
      const double qq = 1.0 + vv * vv - 2.0 * vv * cb;
      const double E1 = b2 * (1.0 + uu * uu - 2.0 * uu * cg) - c2 * qq, E2 = b2 * (uu * uu + vv * vv - 2.0 * uu * vv * ca) - a2 * qq;
      const double J11 = b2 * (2.0 * uu - 2.0 * cg), J12 = -c2 * (2.0 * vv - 2.0 * cb);
      const double J21 = b2 * (2.0 * uu - 2.0 * vv * ca), J22 = b2 * (2.0 * vv - 2.0 * uu * ca) - a2 * (2.0 * vv - 2.0 * cb);
      const double det = J11 * J22 - J12 * J21;
      if (det == 0.0) break;
      const double du = (E1 * J22 - E2 * J12) / det, dv = (J11 * E2 - J21 * E1) / det;
      if (!(fabs(du) < 0.1 * (1.0 + fabs(uu))) || !(fabs(dv) < 0.1 * (1.0 + fabs(vv)))) break;
      uu -= du; vv -= dv;
    }
    if (!(uu > 0.0) || !(vv > 0.0)) continue;
    const double qr = 1.0 + vv * vv - 2.0 * vv * cb;
    if (!(qr > 0.0)) continue;
    const double s1 = sqrt(b2 / qr), s2 = uu * s1, s3 = vv * s1;
    const double chk = s1 * s1 + s2 * s2 - 2.0 * s1 * s2 * cg;
    if (fabs(chk - c2) > 1e-7 * c2) continue;
    double Y1[3], Y2[3], Y3[3], w12[3], w13[3], wn[3], ey1[3], ey2[3], ey3[3];
    for (int k = 0; k < 3; ++k) { Y1[k] = s1 * f1[k]; Y2[k] = s2 * f2[k]; Y3[k] = s3 * f3[k]; w12[k] = Y2[k] - Y1[k]; w13[k] = Y3[k] - Y1[k]; }
    cross3(w12, w13, wn);
    const double l1 = sqrt(dot3(w12, w12)), l3 = sqrt(dot3(wn, wn));
    if (l1 == 0.0 || l3 == 0.0) continue;
    for (int k = 0; k < 3; ++k) { ey1[k] = w12[k] / l1; ey3[k] = wn[k] / l3; }
    cross3(ey3, ey1, ey2);
    double* Rt = Rt_out + 12 * ns;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Rt[3 * i + j] = ey1[i] * ex1[j] + ey2[i] * ex2[j] + ey3[i] * ex3[j];
    for (int i = 0; i < 3; ++i) Rt[9 + i] = Y1[i] - (Rt[3 * i] * P1[0] + Rt[3 * i + 1] * P1[1] + Rt[3 * i + 2] * P1[2]);
    ++ns;
  }
  return ns;
}

__host__ __device__ inline int is_inlier(const double* P, const double* uv, const double* Rt, double thr2) {
  const double x = Rt[0] * P[0] + Rt[1] * P[1] + Rt[2] * P[2] + Rt[9];
  const double y = Rt[3] * P[0] + Rt[4] * P[1] + Rt[5] * P[2] + Rt[10];
  const double z = Rt[6] * P[0] + Rt[7] * P[1] + Rt[8] * P[2] + Rt[11];
  if (!(z > 0.0)) return 0;
  const double du = x / z - uv[0], dv = y / z - uv[1];
  return du * du + dv * dv < thr2 ? 1 : 0;
}

// one warp per hypothesis: best inlier count over its (<= 4) minimal solutions, the root index and the pose of that solution
__global__ void __launch_bounds__(kHypPerCta * 32) pnp_hypothesis_kernel(int n, const double* __restrict__ xyz, const double* __restrict__ xy,
                                                                         double thr2, uint64_t seed, int n_hyp, int* __restrict__ out_count,
                                                                         int* __restrict__ out_root, double* __restrict__ out_Rt) {
  __shared__ double s_sol[kHypPerCta][48];
  __shared__ int s_ns[kHypPerCta];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.x * kHypPerCta + warp;
  if (h >= n_hyp) return;  // (whole warps leave together; no CTA barrier below)
  if (lane == 0) {
    int idx[3];
    pnp_sample(seed, h, n, idx);
    double X[9], f[9];
    for (int k = 0; k < 3; ++k) {
      X[3 * k] = xyz[3 * (size_t)idx[k]]; X[3 * k + 1] = xyz[3 * (size_t)idx[k] + 1]; X[3 * k + 2] = xyz[3 * (size_t)idx[k] + 2];
      const double bx = xy[2 * (size_t)idx[k]], by = xy[2 * (size_t)idx[k] + 1], l = sqrt(bx * bx + by * by + 1.0);
      f[3 * k] = bx / l; f[3 * k + 1] = by / l; f[3 * k + 2] = 1.0 / l;
    }
    s_ns[warp] = p3p(X, f, s_sol[warp]);
  }
  __syncwarp();
  const int ns = s_ns[warp];
  int best = 0, best_r = -1;
  for (int r = 0; r < ns; ++r) {
    const double* Rt = s_sol[warp] + 12 * r;
    int c = 0;
    for (int k = lane; k < n; k += 32) c += is_inlier(xyz + 3 * (size_t)k, xy + 2 * (size_t)k, Rt, thr2);
    c = __reduce_add_sync(0xffffffffu, c);
    if (c > best) { best = c; best_r = r; }
  }
  if (lane == 0) { out_count[h] = best; out_root[h] = best_r; }
  if (best_r >= 0 && lane < 12) out_Rt[12 * (size_t)h + lane] = s_sol[warp][12 * best_r + lane];
}

void R_to_quat(const double* R, double* q) {  // {x,y,z,w}, w >= 0
  const double tr = R[0] + R[4] + R[8];
  double x, y, z, w;
  if (tr > 0.0) { const double s = sqrt(tr + 1.0) * 2.0; w = 0.25 * s; x = (R[7] - R[5]) / s; y = (R[2] - R[6]) / s; z = (R[3] - R[1]) / s; }
  else if (R[0] > R[4] && R[0] > R[8]) { const double s = sqrt(1.0 + R[0] - R[4] - R[8]) * 2.0; w = (R[7] - R[5]) / s; x = 0.25 * s; y = (R[1] + R[3]) / s; z = (R[2] + R[6]) / s; }
  else if (R[4] > R[8]) { const double s = sqrt(1.0 + R[4] - R[0] - R[8]) * 2.0; w = (R[2] - R[6]) / s; x = (R[1] + R[3]) / s; y = 0.25 * s; z = (R[5] + R[7]) / s; }
  else { const double s = sqrt(1.0 + R[8] - R[0] - R[4]) * 2.0; w = (R[3] - R[1]) / s; x = (R[2] + R[6]) / s; y = (R[5] + R[7]) / s; z = 0.25 * s; }
  if (w < 0.0) { x = -x; y = -y; z = -z; w = -w; }
  q[0] = x; q[1] = y; q[2] = z; q[3] = w;
}
void quat_to_Rt(const double* p, double* Rt) {
  const double x = p[0], y = p[1], z = p[2], w = p[3];
  const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y), 2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                       2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};
  memcpy(Rt, R, sizeof R);
  Rt[9] = p[4]; Rt[10] = p[5]; Rt[11] = p[6];
}
void se3_inverse_h(const double* in, double* out) {  // {q, t} -> {q^-1, -R^T t}
  double Rt[12];
  quat_to_Rt(in, Rt);
  out[0] = -in[0]; out[1] = -in[1]; out[2] = -in[2]; out[3] = in[3];
  for (int j = 0; j < 3; ++j) out[4 + j] = -(Rt[j] * in[4] + Rt[3 + j] * in[5] + Rt[6 + j] * in[6]);
}
int count_inliers_h(int n, const double* xyz, const double* xy, const double* Rt, double thr2, uint8_t* mask) {
  int c = 0;
  for (int k = 0; k < n; ++k) {
    const int in = is_inlier(xyz + 3 * (size_t)k, xy + 2 * (size_t)k, Rt, thr2);
    if (mask) mask[k] = (uint8_t)in;
    c += in;
  }
  return c;
}

// The sequential definition replayed over per-hypothesis results: batches of 64, stop at the first batch boundary where
// h >= log(1-confidence)/log(1-w^3) (w = best inlier ratio so far); best = (most inliers, lowest h).  Returns the hypotheses counted.
int replay_stopping_rule(int n, int H, double confidence, const int* cnt, const int* root, gb_pnp_stats* st, int* best_out) {
  int best = 0, h = 0;
  double needed = (double)H;
  while (h < H && (double)h < needed) {
    const int h_end = h + 64 < H ? h + 64 : H;
    for (; h < h_end; ++h)
      if (cnt[h] > best) { best = cnt[h]; st->best_hypothesis = h; st->best_root = root[h]; }
    const double w = (double)best / (double)n, w3 = w * w * w;
    if (w3 >= 1.0) needed = 0.0;
    else if (w3 > 0.0) needed = log(1.0 - confidence) / log(1.0 - w3);
  }
  *best_out = best;
  return h;
}

}  // namespace

extern "C" {

int gb_pnp_ransac(gb_ctx* ctx, int n, const double* xyz, const double* xy, double threshold, double confidence, int max_hypotheses,
                  uint64_t seed, double* pose_cw, uint8_t* mask, gb_pnp_stats* stats) {
  gb_pnp_stats st;
  memset(&st, 0, sizeof st);
  st.best_hypothesis = -1;
  if (stats) *stats = st;
  if (!ctx || n < 4 || !xyz || !xy || !pose_cw || max_hypotheses < 1 || max_hypotheses > (1 << 20)) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  if (!(threshold > 0.0) || !std::isfinite(threshold) || !(confidence > 0.0) || !(confidence < 1.0)) {  // (NaN fails every comparison)
    gb_set_error(ctx, "gb_pnp_ransac: threshold must be > 0 and confidence in (0,1) (got %g, %g)", threshold, confidence);
    return GB_ERR_INVALID;
  }
  const double thr2 = threshold * threshold;
  const int H = max_hypotheses;
  // device buffers: points, measurements, per-hypothesis results (grow-only scratch owned by the ctx)
  const size_t b_xyz = (size_t)n * 24, b_xy = (size_t)n * 16, b_cnt = (size_t)H * 4, b_Rt = (size_t)H * 96;
  auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t need = al(b_xyz) + al(b_xy) + 2 * al(b_cnt) + al(b_Rt);
  GB_CHECK(gb_dev_realloc(ctx, &ctx->pnp_scratch, &ctx->pnp_scratch_cap, need));
  uint8_t* base = (uint8_t*)ctx->pnp_scratch;
  double* d_xyz = (double*)base; base += al(b_xyz);
  double* d_xy = (double*)base; base += al(b_xy);
  int* d_cnt = (int*)base; base += al(b_cnt);
  int* d_root = (int*)base; base += al(b_cnt);
  double* d_Rt = (double*)base;
  GB_CHECK(gb_stage_reserve(ctx, ctx->h_stage_off + b_xyz + b_xy + 2 * b_cnt + 4096));
  double* h_xyz = (double*)gb_stage_alloc(ctx, b_xyz);
  double* h_xy = (double*)gb_stage_alloc(ctx, b_xy);
  int* h_cnt = (int*)gb_stage_alloc(ctx, b_cnt);
  int* h_root = (int*)gb_stage_alloc(ctx, b_cnt);
  if (!h_xyz || !h_xy || !h_cnt || !h_root) { gb_set_error(ctx, "gb_pnp_ransac: staging exhausted"); return GB_ERR_CUDA; }
  memcpy(h_xyz, xyz, b_xyz);
  memcpy(h_xy, xy, b_xy);
  GB_CUDA(ctx, cudaMemcpyAsync(d_xyz, h_xyz, b_xyz, cudaMemcpyHostToDevice, ctx->stream));
  GB_CUDA(ctx, cudaMemcpyAsync(d_xy, h_xy, b_xy, cudaMemcpyHostToDevice, ctx->stream));
  pnp_hypothesis_kernel<<<gb_div_up(H, kHypPerCta), kHypPerCta * 32, 0, ctx->stream>>>(n, d_xyz, d_xy, thr2, seed, H, d_cnt, d_root, d_Rt);
  GB_LAUNCH_CHECK(ctx);
  GB_CUDA(ctx, cudaMemcpyAsync(h_cnt, d_cnt, b_cnt, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaMemcpyAsync(h_root, d_root, b_cnt, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  // replay of the sequential stopping rule over the speculatively computed hypotheses
  int best = 0;
  const int h = replay_stopping_rule(n, H, confidence, h_cnt, h_root, &st, &best);
  st.hypotheses = h;
  st.inliers_minimal = best;
  if (stats) *stats = st;
  if (best < 4) { gb_set_error(ctx, "gb_pnp_ransac: no pose with at least 4 inliers in %d hypotheses", h); return GB_ERR_NUMERIC; }
  double best_Rt[12];
  GB_CUDA(ctx, cudaMemcpy(best_Rt, d_Rt + 12 * (size_t)st.best_hypothesis, sizeof best_Rt, cudaMemcpyDeviceToHost));
  std::vector<uint8_t> m((size_t)n);
  count_inliers_h(n, xyz, xy, best_Rt, thr2, m.data());
  std::vector<double> ixyz((size_t)best * 3), ixy1((size_t)best * 3);
  int c = 0;
  for (int k = 0; k < n && c < best; ++k)
    if (m[k]) {
      memcpy(&ixyz[3 * (size_t)c], xyz + 3 * (size_t)k, 24);
      ixy1[3 * (size_t)c] = xy[2 * (size_t)k]; ixy1[3 * (size_t)c + 1] = xy[2 * (size_t)k + 1]; ixy1[3 * (size_t)c + 2] = 1.0;
      ++c;
    }
  double cw[7], wc[7];
  R_to_quat(best_Rt, cw);
  cw[4] = best_Rt[9]; cw[5] = best_Rt[10]; cw[6] = best_Rt[11];
  se3_inverse_h(cw, wc);
  gb_ba_options o;
  gb_ba_options_default(&o);
  o.huber_delta = 0.0; o.max_iterations = 20; o.function_tolerance = 1e-12; o.lambda_init = 1e-4; o.pcg_max_iters = 50; o.pcg_tol = 1e-12;
  gb_ba_result res;
  const int rc = gb_ba_pnp(ctx, c, ixyz.data(), ixy1.data(), wc, 63, nullptr, &o, &res);
  st.inliers_refined = best;
  if (rc == GB_OK) {
    double rcw[7], Rt[12];
    se3_inverse_h(wc, rcw);
    quat_to_Rt(rcw, Rt);
    std::vector<uint8_t> m2((size_t)n);
    const int c2 = count_inliers_h(n, xyz, xy, Rt, thr2, m2.data());
    if (c2 >= best) { memcpy(cw, rcw, sizeof cw); st.inliers_refined = c2; m.swap(m2); }  // keep the refinement only if it loses nothing
  }
  memcpy(pose_cw, cw, sizeof cw);
  if (mask) memcpy(mask, m.data(), (size_t)n);
  if (stats) *stats = st;
  return GB_OK;
}

// ---- host-only checks (no device needed): the SAME source as the kernel, instantiated for the host, so that the CPU test suite can
// compare the port with the CPU checker before the kernel has ever run (tests/test_oracle_pnp.py::test_product_host_instantiation_*)
GB_API int gb_dbg_pnp_p3p_host(const double* X, const double* f, double* Rt_out) { return p3p(X, f, Rt_out); }

// the minimal stage of gb_pnp_ransac (sampling, P3P, scoring, stopping-rule replay) with the hypotheses evaluated on the host
GB_API int gb_dbg_pnp_minimal_host(int n, const double* xyz, const double* xy, double threshold, double confidence, int max_hypotheses,
                                   uint64_t seed, double* best_Rt, gb_pnp_stats* stats) {
  if (n < 4 || !xyz || !xy || !best_Rt || !stats || max_hypotheses < 1) return GB_ERR_INVALID;
  const double thr2 = threshold * threshold;
  std::vector<int> cnt((size_t)max_hypotheses), root((size_t)max_hypotheses);
  std::vector<double> Rts((size_t)max_hypotheses * 12);
  for (int h = 0; h < max_hypotheses; ++h) {
    int idx[3];
    pnp_sample(seed, h, n, idx);
    double X[9], f[9], sol[48];
    for (int k = 0; k < 3; ++k) {
      memcpy(X + 3 * k, xyz + 3 * (size_t)idx[k], 24);
      const double bx = xy[2 * (size_t)idx[k]], by = xy[2 * (size_t)idx[k] + 1], l = sqrt(bx * bx + by * by + 1.0);
      f[3 * k] = bx / l; f[3 * k + 1] = by / l; f[3 * k + 2] = 1.0 / l;
    }
    const int ns = p3p(X, f, sol);
    int best = 0, best_r = -1;
    for (int r = 0; r < ns; ++r) {
      const int c = count_inliers_h(n, xyz, xy, sol + 12 * r, thr2, nullptr);
      if (c > best) { best = c; best_r = r; }
    }
    cnt[(size_t)h] = best; root[(size_t)h] = best_r;
    if (best_r >= 0) memcpy(&Rts[12 * (size_t)h], sol + 12 * best_r, 96);
  }
  gb_pnp_stats st;
  memset(&st, 0, sizeof st);
  st.best_hypothesis = -1;
  int best = 0;
  st.hypotheses = replay_stopping_rule(n, max_hypotheses, confidence, cnt.data(), root.data(), &st, &best);
  st.inliers_minimal = best;
  *stats = st;
  if (st.best_hypothesis >= 0) memcpy(best_Rt, &Rts[12 * (size_t)st.best_hypothesis], 96);
  return best >= 4 ? GB_OK : GB_ERR_NUMERIC;
}

}  // extern "C"
