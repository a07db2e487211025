"""An INDEPENDENT restatement of the bundle-adjustment definition (SURVEY.md Appendix B / DESIGN.md section 5), used to pin the
CPU oracle oracle/ba_ref.c harder than the reference allows (the reference ships no BA arithmetic, test or vector: parity is
unpinned by it).  Nothing is shared with the oracle's implementation strategy:

  oracle/ba_ref.c                               here (numpy + scipy.sparse)
  ----------------------------------------------------------------------------------------------------------------
  per-landmark / per-camera block accumulation  one global sparse Jacobian, H = J' A J assembled by scipy
  Schur complement onto the cameras             NO Schur complement: the full (cameras + landmarks) damped normal equations
  block-Jacobi PCG / dense Cholesky of S        scipy.sparse.linalg.spsolve (SuperLU) of the full system
  hand-written 6x6 / 3x3 inverses               none

With exact linear solves on both sides (oracle: linear_solver = 1) the two Levenberg-Marquardt runs must produce the same cost
after every iteration, the same accept / reject pattern and the same estimate -- with the Huber kernel active, with per-edge
information matrices, with partially fixed cameras and fixed landmarks, at the benchmark's local-BA size.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import oracle
from gslam_b200 import synth
import ba_graphs  # (tests/ is on sys.path under pytest's rootdir conftest)


def quat_to_R(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0.0]])


def exp_se3(d):
    """Exp([v, w]) as (R, t): Rodrigues + the left Jacobian (closed form; the series below 1e-6 like the product)."""
    v, w = d[:3], d[3:]
    th = np.linalg.norm(w)
    W = skew(w)
    if th < 1e-6:
        A, B, C = 1 - th * th / 6, 0.5 - th * th / 24, 1 / 6 - th * th / 120
    else:
        A, B, C = np.sin(th) / th, (1 - np.cos(th)) / th ** 2, (th - np.sin(th)) / th ** 3
    R = np.eye(3) + A * W + B * W @ W
    V = np.eye(3) + B * W + C * W @ W
    return R, V @ v


class Problem:
    def __init__(self, pb, delta):
        self.delta = delta
        self.nc, self.np_ = pb.n_cams, pb.n_points
        self.Rcw, self.tcw = [], []
        for i in range(pb.n_cams):  # T_cw = T_wc^-1
            R = quat_to_R(pb.cam_pose_wc[i, :4] / np.linalg.norm(pb.cam_pose_wc[i, :4]))
            self.Rcw.append(R.T); self.tcw.append(-R.T @ pb.cam_pose_wc[i, 4:])
        self.pts = pb.points.copy()
        self.dof = pb.cam_dof.astype(int)
        self.pfree = pb.point_free.astype(bool)
        self.oc, self.op = pb.obs_cam.astype(int), pb.obs_point.astype(int)
        self.uv = pb.obs_xyz[:, :2] / pb.obs_xyz[:, 2:3]
        if pb.obs_info is None:
            self.info = np.tile(np.eye(2), (pb.n_obs, 1, 1))
        else:
            L = pb.obs_info.reshape(-1, 2, 2)
            self.info = 0.5 * (L + np.transpose(L, (0, 2, 1)))

    def residuals(self, Rcw=None, tcw=None, pts=None):
        Rcw = self.Rcw if Rcw is None else Rcw; tcw = self.tcw if tcw is None else tcw; pts = self.pts if pts is None else pts
        R = np.stack([Rcw[i] for i in self.oc]); t = np.stack([tcw[i] for i in self.oc])
        q = np.einsum("kij,kj->ki", R, pts[self.op]) + t
        ok = q[:, 2] > 0
        r = np.zeros((len(self.oc), 2))
        r[ok] = q[ok, :2] / q[ok, 2:3] - self.uv[ok]
        return r, q, ok, R

    def cost(self, *a):
        r, q, ok, _ = self.residuals(*a)
        e2 = np.einsum("ki,kij,kj->k", r, self.info, r)
        e = np.sqrt(e2)
        rho = np.where((self.delta > 0) & (e > self.delta), 2 * self.delta * e - self.delta ** 2, e2)
        return 0.5 * rho[ok].sum()

    def normal_equations(self):
        r, q, ok, R = self.residuals()
        e2 = np.einsum("ki,kij,kj->k", r, self.info, r)
        e = np.sqrt(e2)
        w = np.where((self.delta > 0) & (e > self.delta), self.delta / np.maximum(e, 1e-300), 1.0)
        n = 6 * self.nc + 3 * self.np_
        rows, cols, vals = [], [], []
        Ablocks = []
        for k in np.nonzero(ok)[0]:
            x, y, z = q[k]
            Jpi = np.array([[1 / z, 0, -x / z ** 2], [0, 1 / z, -y / z ** 2]])
            Jc = Jpi @ np.hstack([np.eye(3), -skew(q[k])])          # d q / d [v, w] = [I | -[q]x]  (left perturbation of T_cw)
            Jp = Jpi @ R[k]                                          # d q / d p = R_cw
            i, j = self.oc[k], self.op[k]
            for a in range(6):
                if not (self.dof[i] >> a) & 1:
                    Jc[:, a] = 0
            if not self.pfree[j]:
                Jp[:] = 0
            for rr in range(2):
                for a in range(6):
                    rows.append(2 * k + rr); cols.append(6 * i + a); vals.append(Jc[rr, a])
                for a in range(3):
                    rows.append(2 * k + rr); cols.append(6 * self.nc + 3 * j + a); vals.append(Jp[rr, a])
            Ablocks.append((k, w[k] * self.info[k]))
        J = sp.csr_matrix((vals, (rows, cols)), shape=(2 * len(self.oc), n))
        # weight matrix as a block-diagonal over ALL observations (zero blocks for the ones behind the camera)
        blocks = [np.zeros((2, 2))] * len(self.oc)
        for k, blk in Ablocks:
            blocks[k] = blk
        A = sp.block_diag([sp.coo_matrix(b) for b in blocks], format="csr")
        H = (J.T @ A @ J).tocsr()
        g = -(J.T @ (A @ r.reshape(-1)))
        return H, g


def lm_numpy(pb, iters, delta=0.01, lam0=1e-4):
    P = Problem(pb, delta)
    lam, nu = lam0, 2.0
    cost = P.cost()
    trace, accepted = [], 0
    H, g = P.normal_equations()
    for _ in range(iters):
        d = H.diagonal()
        free = np.zeros(H.shape[0], bool)
        for i in range(P.nc):
            for a in range(6):
                free[6 * i + a] = (P.dof[i] >> a) & 1
        deg = np.bincount(P.op, minlength=P.np_)
        for j in range(P.np_):
            free[6 * P.nc + 3 * j: 6 * P.nc + 3 * j + 3] = P.pfree[j] and deg[j] > 0
        idx = np.nonzero(free)[0]
        Hd = H[idx][:, idx] + sp.diags(lam * np.clip(d[idx], 1e-6, 1e32))
        step = np.zeros(H.shape[0])
        step[idx] = spla.spsolve(Hd.tocsc(), g[idx])
        Rn, tn = [], []
        for i in range(P.nc):
            dR, dt = exp_se3(step[6 * i: 6 * i + 6])
            Rn.append(dR @ P.Rcw[i]); tn.append(dR @ P.tcw[i] + dt)
        pn = P.pts + step[6 * P.nc:].reshape(-1, 3)
        cnew = P.cost(Rn, tn, pn)
        ok = cnew < cost and np.isfinite(cnew)
        if ok:
            P.Rcw, P.tcw, P.pts = Rn, tn, pn
            cost = cnew
            lam = max(lam / 3.0, 1e-15); nu = 2.0; accepted += 1
            H, g = P.normal_equations()
        else:
            lam *= nu; nu *= 2.0
        trace.append(cost)
    Twc_t = np.stack([-P.Rcw[i].T @ P.tcw[i] for i in range(P.nc)])
    return trace, accepted, Twc_t, P.pts


def _variant(kind):
    if kind == "config1_huber":
        return synth.synth_ba(10, 200, all_visible=True, n_fixed=2, seed=42), 0.01
    if kind == "local_window_huber":           # the benchmark's local-BA size, Huber active (about a third of the edges start outside)
        return synth.synth_ba(50, 2000, obs_per_point=5, n_fixed=2, seed=42), 0.002
    if kind == "info_and_partial_dof":
        pb = synth.synth_ba(12, 300, obs_per_point=6, n_fixed=1, seed=5)
        rng = np.random.default_rng(1)
        L = rng.normal(size=(pb.n_obs, 2, 2)) * 0.3 + np.eye(2)
        pb.obs_info = np.ascontiguousarray((L @ np.transpose(L, (0, 2, 1))).reshape(-1, 4))
        pb.cam_dof[1] = 0b111000          # rotation only
        pb.cam_dof[2] = 0b000111          # translation only
        pb.point_free[::7] = 0            # some fixed landmarks
        return pb, 0.01
    if kind in ba_graphs.CASES:           # the irregular topologies of tests/ba_graphs.py, local-window size
        c = ba_graphs.build(kind)
        return c.pb, c.delta
    raise KeyError(kind)


@pytest.mark.parametrize("kind,iters", [("config1_huber", 8), ("local_window_huber", 6), ("info_and_partial_dof", 8)] +
                         [(name, 6) for name in ba_graphs.CASES])
def test_oracle_lm_trajectory_equals_independent_sparse_lm(kind, iters):
    pb, delta = _variant(kind)
    trace, accepted, t_wc, pts = lm_numpy(pb, iters, delta)
    # the oracle, stopped after 1, 2, ... iterations: cost after every iteration + the accept count
    for k in range(1, iters + 1):
        q = pb.copy()
        r = oracle.ba_solve(q, max_iterations=k, function_tolerance=0.0, huber_delta=delta, linear_solver=1)
        assert abs(r.final_cost - trace[k - 1]) <= 1e-8 * max(trace[k - 1], 1e-12), (kind, k, r.final_cost, trace[k - 1])
    assert r.accepted == accepted
    assert np.abs(q.cam_pose_wc[:, 4:] - t_wc).max() < 1e-7 * max(1.0, np.abs(t_wc).max())
    assert np.abs(q.points - pts).max() < 1e-7 * np.abs(pts).max()
    if delta > 0:  # the Huber branch really is exercised
        P = Problem(pb, delta)
        r0, _, ok, _ = P.residuals()
        e = np.sqrt(np.einsum("ki,kij,kj->k", r0, P.info, r0))
        assert (e[ok] > delta).mean() > 0.05


def test_oracle_pcg_converged_equals_the_exact_solve():
    """The PCG path of the oracle, run to a tight tolerance, lands on the exact-solve trajectory (ties the solver the product's
    benchmark configuration uses to the independently checked one)."""
    pb, delta = _variant("config1_huber")
    a, b = pb.copy(), pb.copy()
    ra = oracle.ba_solve(a, max_iterations=6, function_tolerance=0.0, huber_delta=delta, linear_solver=1)
    rb = oracle.ba_solve(b, max_iterations=6, function_tolerance=0.0, huber_delta=delta, pcg_max_iters=5000, pcg_tol=1e-15)
    assert ra.accepted == rb.accepted and abs(ra.final_cost - rb.final_cost) / ra.final_cost < 1e-8
    assert np.abs(a.cam_pose_wc - b.cam_pose_wc).max() < 1e-7
