// gslam_b200/csrc/ba_pose.cu — pose-graph terms of a BundleGraph: GSLAM::SE3Edge (relative pose between two keyframes,
// GSLAM/core/Optimizer.h:127-133, BundleGraph::se3Graph :163-164) and GSLAM::GPSEdge (absolute pose prior, :143-148, gpsGraph :167-168)
// next to, or instead of, the reprojection edges.  SURVEY.md section 8f-3.  The arithmetic is our definition (the reference fixes the
// types and the meaning SE3_12 := SE3_1^-1 SE3_2 only); oracle/ba_ref.c::pose_edge_eval is its CPU restatement:
//   e = Log(Z^-1 T_cw,i T_cw,j^-1)  (SE3 edge)   or   Log(Z^-1 T_cw,i^-1)  (GPS edge),   cost term e' Omega e,
//   J_i = Jl^-1(e) Ad(Z^-1),  J_j = -Jl^-1(e) Ad(E)   (GPS: J_i = -Jl^-1(e) Ad(E)),   left updates T_cw <- Exp(d) T_cw,
//   SE3 logarithm as the reference's SE3::log (GSLAM/core/SE3.h:205-246), tangent order [v, w].
// There are few such edges (one per keyframe pair / GPS fix), so the mapping is the plain one: one thread evaluates an edge into a
// staging record, the camera blocks gather their incident records in edge order, the off-diagonal blocks J_i' Omega J_j are added
// to the dense reduced system per unordered camera pair in edge order -- no atomics, bit-reproducible.  Graphs with pose-graph
// terms run the stepwise solver path on the dense reduced system (cluster / generic PCG).
#include <algorithm>
#include <numeric>

#include "ba_device.cuh"
#include "ba_internal.cuh"
#include "common.cuh"

using namespace ba;

namespace {

constexpr int kRec = 121;  // staging record per edge: Hii (36) | Hjj (36) | Hij (36) | g_i (6) | g_j (6) | cost (1)

__device__ __forceinline__ void se3_mul(const double* a, const double* b, double* o) {  // SE3.h:129-131
  double t[3];
  quat_mul(a, b, o);
  quat_rot(a, b + 4, t);
  o[4] = t[0] + a[4]; o[5] = t[1] + a[5]; o[6] = t[2] + a[6];
}
__device__ __forceinline__ void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1]; o[1] = a[2] * b[0] - a[0] * b[2]; o[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ void se3_log(const double* T, double* out) {  // SE3.h:205-246 (NEAR_ZERO = 1e-10, SO3.h:43)
  const double x = T[0], y = T[1], z = T[2], w = T[3];
  const double* t = T + 4;
  const double n = sqrt(x * x + y * y + z * z);
  double r[3], c1[3], c2[3];
  if (n < 1e-10) {
    const double A_inv = 2.0 / w - 2.0 * (1.0 - w * w) / (w * w * w);
    r[0] = x * A_inv; r[1] = y * A_inv; r[2] = z * A_inv;
    cross3(r, t, c1); cross3(r, c1, c2);
    for (int k = 0; k < 3; ++k) out[k] = t[k] - 0.5 * c1[k] + (1.0 / 12.0) * c2[k];
  } else {
    double A_inv;
    if (fabs(w) < 1e-10) A_inv = (w > 0 ? 3.14159265358979323846 : -3.14159265358979323846) / n;
    else A_inv = 2.0 * atan(n / w) / n;
    const double theta = A_inv * n;
    r[0] = x * A_inv; r[1] = y * A_inv; r[2] = z * A_inv;
    const double a[3] = {r[0] / theta, r[1] / theta, r[2] / theta};
    double a1[3];
    cross3(r, t, c1); cross3(a, t, a1); cross3(a, a1, c2);
    const double k2 = 1.0 - theta / (2.0 * tan(0.5 * theta));
    for (int k = 0; k < 3; ++k) out[k] = t[k] - 0.5 * c1[k] + k2 * c2[k];
  }
  out[3] = r[0]; out[4] = r[1]; out[5] = r[2];
}
__device__ void mat6_mul(const double* A, const double* B, double* C) {
  for (int a = 0; a < 6; ++a)
    for (int b = 0; b < 6; ++b) {
      double x = 0.0;
      for (int k = 0; k < 6; ++k) x += A[a * 6 + k] * B[k * 6 + b];
      C[a * 6 + b] = x;
    }
}
__device__ void se3_adjoint(const double* T, double* Ad) {  // [[R, [t]x R], [0, R]] for the tangent order [v, w]
  double R[9];
  quat_to_R(T, R);
  const double* t = T + 4;
  const double tx[9] = {0.0, -t[2], t[1], t[2], 0.0, -t[0], -t[1], t[0], 0.0};
  for (int k = 0; k < 36; ++k) Ad[k] = 0.0;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      Ad[a * 6 + b] = R[a * 3 + b];
      Ad[(3 + a) * 6 + 3 + b] = R[a * 3 + b];
      Ad[a * 6 + 3 + b] = tx[a * 3] * R[b] + tx[a * 3 + 1] * R[3 + b] + tx[a * 3 + 2] * R[6 + b];
    }
}
// Bernoulli series of the inverse left Jacobian in ad(xi) = [[w^, v^], [0, w^]] (see oracle/ba_ref.c::se3_jl_inv)
__device__ void se3_jl_inv(const double* xi, double* J) {
  const double* v = xi; const double* w = xi + 3;
  double A[36], A2[36], A4[36], A6[36], A8[36];
  for (int k = 0; k < 36; ++k) A[k] = 0.0;
  const double wx[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
  const double vx[9] = {0.0, -v[2], v[1], v[2], 0.0, -v[0], -v[1], v[0], 0.0};
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) { A[a * 6 + b] = wx[a * 3 + b]; A[(3 + a) * 6 + 3 + b] = wx[a * 3 + b]; A[a * 6 + 3 + b] = vx[a * 3 + b]; }
  mat6_mul(A, A, A2); mat6_mul(A2, A2, A4); mat6_mul(A4, A2, A6); mat6_mul(A4, A4, A8);
  for (int k = 0; k < 36; ++k)
    J[k] = ((k % 7) == 0 ? 1.0 : 0.0) - 0.5 * A[k] + A2[k] * (1.0 / 12.0) - A4[k] * (1.0 / 720.0) + A6[k] * (1.0 / 30240.0) - A8[k] * (1.0 / 1209600.0);
}
__device__ void edge_residual(const BaDev& g, const double* pose, int k, double* E, double* e) {
  const int i = g.pe_i[k], j = g.pe_j[k];
  double inv[7], tmp[7];
  if (j < 0) {
    se3_inverse(pose + 7 * i, inv);
    se3_mul(g.pe_Zinv + 7 * k, inv, E);
  } else {
    se3_inverse(pose + 7 * j, inv);
    se3_mul(pose + 7 * i, inv, tmp);
    se3_mul(g.pe_Zinv + 7 * k, tmp, E);
  }
  se3_log(E, e);
}
__device__ double quad6(const double* Om, const double* e) {
  double s = 0.0;
  for (int a = 0; a < 6; ++a) {
    double r = 0.0;
    for (int b = 0; b < 6; ++b) r += Om[a * 6 + b] * e[b];
    s += e[a] * r;
  }
  return s;
}

// one thread per edge: residual, Jacobians, J' Omega J / J' Omega e into the staging record; cost into cost_pt[np + k]
__global__ void __launch_bounds__(64) ba_pose_lin_kernel(BaDev g) {
  if (g.sc->stop || !g.sc->need_linearize) return;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= g.npe) return;
  const int i = g.pe_i[k], j = g.pe_j[k];
  double E[7], e[6], AdE[36], Jl[36], T[36], Ji[36], Jj[36];
  edge_residual(g, g.pose, k, E, e);
  se3_adjoint(E, AdE);
  se3_jl_inv(e, Jl);
  mat6_mul(Jl, AdE, T);
  if (j < 0) {
    for (int q = 0; q < 36; ++q) { Ji[q] = -T[q]; Jj[q] = 0.0; }
  } else {
    double AdZ[36];
    se3_adjoint(g.pe_Zinv + 7 * k, AdZ);
    mat6_mul(Jl, AdZ, Ji);
    for (int q = 0; q < 36; ++q) Jj[q] = -T[q];
  }
  const int dmi = g.dof[i], dmj = j < 0 ? 0 : g.dof[j];
  for (int d = 0; d < 6; ++d) {
    if (!((dmi >> d) & 1)) for (int r = 0; r < 6; ++r) Ji[r * 6 + d] = 0.0;
    if (!((dmj >> d) & 1)) for (int r = 0; r < 6; ++r) Jj[r * 6 + d] = 0.0;
  }
  const double* Om = g.pe_info + 36 * (size_t)k;
  double OJi[36], OJj[36], Oe[6];
  mat6_mul(Om, Ji, OJi);
  mat6_mul(Om, Jj, OJj);
  for (int a = 0; a < 6; ++a) {
    double r = 0.0;
    for (int b = 0; b < 6; ++b) r += Om[a * 6 + b] * e[b];
    Oe[a] = r;
  }
  double* rec = g.pe_H + (size_t)kRec * k;
  for (int a = 0; a < 6; ++a) {
    double gi = 0.0, gj = 0.0;
    for (int r = 0; r < 6; ++r) { gi += Ji[r * 6 + a] * Oe[r]; gj += Jj[r * 6 + a] * Oe[r]; }
    rec[108 + a] = -gi; rec[114 + a] = -gj;
    for (int c = 0; c < 6; ++c) {
      double hii = 0.0, hjj = 0.0, hij = 0.0;
      for (int r = 0; r < 6; ++r) {
        hii += Ji[r * 6 + a] * OJi[r * 6 + c];
        hjj += Jj[r * 6 + a] * OJj[r * 6 + c];
        hij += Ji[r * 6 + a] * OJj[r * 6 + c];
      }
      rec[a * 6 + c] = hii; rec[36 + a * 6 + c] = hjj; rec[72 + a * 6 + c] = hij;
    }
  }
  const double c = quad6(Om, e);
  rec[120] = c;
  g.cost_pt[g.np + k] = c;
}

// thread = (camera i, entry q of [U (36) | g (6)]): add the incident edges' records in edge order (after the sweep wrote U, g_c)
__global__ void __launch_bounds__(128) ba_pose_gather_kernel(BaDev g) {
  if (g.sc->stop || !g.sc->need_linearize) return;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = t / 42, q = t - 42 * i;
  if (i >= g.nc) return;
  double s = 0.0;
  for (int n = g.pc_off[i]; n < g.pc_off[i + 1]; ++n) {
    const int ent = g.pc_ent[n], k = ent >> 1, side = ent & 1;
    const double* rec = g.pe_H + (size_t)kRec * k;
    s += q < 36 ? rec[36 * side + q] : rec[108 + 6 * side + (q - 36)];
  }
  if (q < 36) g.U[36 * i + q] += s; else g.gc[6 * i + q - 36] += s;
}

// thread = (unordered camera pair, entry of the 6x6 block): S_ij += sum J_i' Omega J_j, S_ji += its transpose, in edge order.  `buf`
// is the dense reduced system; runs after the Schur complement of EVERY iteration (rejected steps rebuild S from U, so the staged
// blocks of the last linearisation are added again).  The diagonal blocks need nothing here: they went into U before S was formed.
__global__ void __launch_bounds__(128) ba_pose_offdiag_kernel(BaDev g, double* __restrict__ buf) {
  if (g.sc->stop) return;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int p = t / 36, q = t - 36 * p;
  if (p >= g.pe_npairs) return;
  const int i = g.pp_ij[2 * p], j = g.pp_ij[2 * p + 1], a = q / 6, b = q - 6 * a;
  double s = 0.0;
  for (int n = g.pp_off[p]; n < g.pp_off[p + 1]; ++n) {
    const int ent = g.pp_ent[n], k = ent >> 1, flipped = ent & 1;  // flipped: the edge runs j -> i, its block is (j, i)
    const double* H = g.pe_H + (size_t)kRec * k + 72;
    s += flipped ? H[b * 6 + a] : H[a * 6 + b];
  }
  const size_t n6 = g.n6;
  buf[(size_t)(6 * i + a) * n6 + 6 * j + b] += s;
  buf[(size_t)(6 * j + b) * n6 + 6 * i + a] += s;
}

// candidate cost of every edge at pose_new -> cost_pt_new[np + k]
__global__ void __launch_bounds__(64) ba_pose_cost_kernel(BaDev g) {
  if (g.sc->stop) return;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= g.npe) return;
  double E[7], e[6];
  edge_residual(g, g.pose_new, k, E, e);
  g.cost_pt_new[g.np + k] = quad6(g.pe_info + 36 * (size_t)k, e);
}

}  // namespace

int ba_pose_validate(gb_ctx* ctx, const gb_ba_problem* pb, const gb_pose_edges* pe) {
  if (!pe) return GB_OK;
  if (pe->n_se3 < 0 || pe->n_gps < 0 || (pe->n_se3 > 0 && (!pe->se3_first || !pe->se3_second || !pe->se3_meas)) ||
      (pe->n_gps > 0 && (!pe->gps_frame || !pe->gps_meas))) {
    gb_set_error(ctx, "gb_ba: malformed gb_pose_edges");
    return GB_ERR_INVALID;
  }
  for (int k = 0; k < pe->n_se3; ++k) {
    const int a = pe->se3_first[k], b = pe->se3_second[k];
    if (a < 0 || a >= pb->n_cams || b < 0 || b >= pb->n_cams || a == b) {
      gb_set_error(ctx, "gb_ba: SE3 edge %d connects keyframes %d and %d (%d keyframes)", k, a, b, pb->n_cams);
      return GB_ERR_INVALID;
    }
  }
  for (int k = 0; k < pe->n_gps; ++k)
    if (pe->gps_frame[k] < 0 || pe->gps_frame[k] >= pb->n_cams) {
      gb_set_error(ctx, "gb_ba: GPS edge %d refers to keyframe %d (%d keyframes)", k, pe->gps_frame[k], pb->n_cams);
      return GB_ERR_INVALID;
    }
  const int total = pe->n_se3 + pe->n_gps;
  const double* arrays[2] = {pe->se3_meas, pe->gps_meas};
  const int counts[2] = {pe->n_se3, pe->n_gps};
  for (int s = 0; s < 2; ++s)
    for (int k = 0; k < counts[s]; ++k) {
      const double* q = arrays[s] + 7 * (size_t)k;
      const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
      bool fin = true;
      for (int c = 0; c < 7; ++c) fin = fin && std::isfinite(q[c]);
      if (!fin || !(n2 > 1e-12)) { gb_set_error(ctx, "gb_ba: pose-graph measurement %d is not a finite SE3", k); return GB_ERR_INVALID; }
    }
  (void)total;
  return GB_OK;
}

// the edges and the two gather plans (camera -> incident records, unordered pair -> records); graph creation uploads them
void ba_pose_plan(gb_ba_graph* g, const gb_pose_edges* pe, BaPosePlan& p) {
  BaDev& d = g->d;
  const int nse = pe->n_se3, ngps = pe->n_gps, npe = nse + ngps, nc = d.nc;
  std::vector<int> &ei = p.ei, &ej = p.ej;
  std::vector<double> &Zinv = p.Zinv, &info = p.info;
  ei.resize(npe); ej.resize(npe); Zinv.resize((size_t)npe * 7); info.resize((size_t)npe * 36);
  auto inv7 = [](const double* in, double* out) {  // SE3.h:100-103 (as ba_device.cuh::se3_inverse, on the host)
    const double n = std::sqrt(in[0] * in[0] + in[1] * in[1] + in[2] * in[2] + in[3] * in[3]);
    const double q[4] = {-in[0] / n, -in[1] / n, -in[2] / n, in[3] / n};
    const double* p = in + 4;
    double ux = q[1] * p[2] - q[2] * p[1], uy = q[2] * p[0] - q[0] * p[2], uz = q[0] * p[1] - q[1] * p[0];
    ux += ux; uy += uy; uz += uz;
    const double t[3] = {p[0] + q[3] * ux + (q[1] * uz - q[2] * uy), p[1] + q[3] * uy + (q[2] * ux - q[0] * uz), p[2] + q[3] * uz + (q[0] * uy - q[1] * ux)};
    out[0] = q[0]; out[1] = q[1]; out[2] = q[2]; out[3] = q[3]; out[4] = -t[0]; out[5] = -t[1]; out[6] = -t[2];
  };
  for (int k = 0; k < npe; ++k) {
    const bool gps = k >= nse;
    const int s = gps ? k - nse : k;
    ei[k] = gps ? pe->gps_frame[s] : pe->se3_first[s];
    ej[k] = gps ? -1 : pe->se3_second[s];
    inv7((gps ? pe->gps_meas : pe->se3_meas) + 7 * (size_t)s, &Zinv[7 * (size_t)k]);
    const double* src = gps ? (pe->gps_info ? pe->gps_info + 36 * (size_t)s : nullptr) : (pe->se3_info ? pe->se3_info + 36 * (size_t)s : nullptr);
    for (int a = 0; a < 6; ++a)
      for (int b = 0; b < 6; ++b) info[36 * (size_t)k + a * 6 + b] = src ? 0.5 * (src[a * 6 + b] + src[b * 6 + a]) : (a == b ? 1.0 : 0.0);
  }
  // camera -> incident (edge, side) in edge order
  std::vector<int> &pc_off = p.pc_off, &pc_ent = p.pc_ent;
  pc_off.assign(nc + 1, 0);
  for (int k = 0; k < npe; ++k) { pc_off[ei[k] + 1]++; if (ej[k] >= 0) pc_off[ej[k] + 1]++; }
  for (int i = 0; i < nc; ++i) pc_off[i + 1] += pc_off[i];
  pc_ent.resize(pc_off[nc]);
  { std::vector<int> pos(pc_off.begin(), pc_off.end() - 1);
    for (int k = 0; k < npe; ++k) { pc_ent[pos[ei[k]]++] = 2 * k; if (ej[k] >= 0) pc_ent[pos[ej[k]]++] = 2 * k + 1; } }
  // unordered pair -> SE3 edges in edge order
  std::vector<int> order(nse);
  std::iota(order.begin(), order.end(), 0);
  auto key = [&](int k) { return std::make_pair(std::min(ei[k], ej[k]), std::max(ei[k], ej[k])); };
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return key(a) < key(b); });
  std::vector<int> &pp_off = p.pp_off, &pp_ij = p.pp_ij, &pp_ent = p.pp_ent;
  pp_off.assign(1, 0);
  for (int n = 0; n < nse; ++n) {
    const int k = order[n];
    if (n == 0 || key(k) != key(order[n - 1])) {
      if (n) pp_off.push_back((int)pp_ent.size());
      pp_ij.push_back(key(k).first); pp_ij.push_back(key(k).second);
    }
    pp_ent.push_back(2 * k + (ei[k] > ej[k] ? 1 : 0));
  }
  pp_off.push_back((int)pp_ent.size());
  p.rec_doubles = (size_t)npe * kRec;
  d.npe = npe; d.pe_npairs = (int)pp_ij.size() / 2;
}

// after the sweep: edge records, then their sums into U / g_c
int ba_pose_linearize(gb_ctx* ctx, gb_ba_graph* g, cudaStream_t s) {
  const BaDev& d = g->d;
  if (d.npe <= 0) return GB_OK;
  ba_pose_lin_kernel<<<gb_div_up(d.npe, 64), 64, 0, s>>>(d); GB_LAUNCH_CHECK(ctx);
  ba_pose_gather_kernel<<<gb_div_up(d.nc * 42, 128), 128, 0, s>>>(d); GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}
// after the Schur complement (dense layout)
int ba_pose_offdiag(gb_ctx* ctx, gb_ba_graph* g, double* buf, cudaStream_t s) {
  const BaDev& d = g->d;
  if (d.npe <= 0 || d.pe_npairs <= 0) return GB_OK;
  ba_pose_offdiag_kernel<<<gb_div_up(d.pe_npairs * 36, 128), 128, 0, s>>>(d, buf); GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}
// after the retraction of the candidate cameras
int ba_pose_cost(gb_ctx* ctx, gb_ba_graph* g, cudaStream_t s) {
  const BaDev& d = g->d;
  if (d.npe <= 0) return GB_OK;
  ba_pose_cost_kernel<<<gb_div_up(d.npe, 64), 64, 0, s>>>(d); GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}
