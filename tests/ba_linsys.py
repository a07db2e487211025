"""Extended-precision restatement of the BA reduced camera system's linear solve (a test helper, not product code).

What a solver of the damped system A x = g~ promises is stated against the exact solution of THAT system, so everything here
takes the (S, g~, diag U, lambda, dof) a solver was given and works on it in more precision than fp64:

  damped(...)        A as every device path builds it (csrc/ba_device.cuh lm_damp): a free dof gets S_dd + lambda * clamp(diag U_d,
                     1e-6, 1e32), a fixed one a unit diagonal
  Reference(A, g)    x* (fp64 Cholesky, then iterative refinement with the residuals accumulated in extended precision), kappa_2(A),
                     the block-Jacobi preconditioner, A-norm errors and preconditioned residual ratios of any x
  Reference.pcg      the PCG the device runs, in exact-arithmetic form (classical recurrence, extended precision): the same
                     block-Jacobi preconditioner with the same non-SPD fallback (the inverse of the diagonal), x0 = 0, the stopping
                     test r'z < tol^2 r0'z0 after each update; every iterate's relative A-norm error and sqrt(r'z / r0'z0)

Extended precision is numpy's long double where it carries at least 64 mantissa bits (x86-64); elsewhere the matrix-vector products
and inner products fall back to compensated (double-double) sums of error-free products.
"""
from __future__ import annotations

import math

import numpy as np
import scipy.linalg

from gslam_b200 import synth
import ba_graphs  # (tests/ is on sys.path under pytest's rootdir conftest)

EPS = np.finfo(np.float64).eps
EXTENDED = bool(np.finfo(np.longdouble).eps < 1e-18)
XP = np.longdouble if EXTENDED else np.float64


def dof_mask(cam_dof) -> np.ndarray:
    """Free (True) / fixed (False) per unknown of the 6N camera vector."""
    d = np.asarray(cam_dof, np.int64) & 63
    return ((d[:, None] >> np.arange(6)[None, :]) & 1).astype(bool).reshape(-1)


def damped(S, diagU, lam, cam_dof) -> np.ndarray:
    """The damped reduced camera matrix the device solves (lm_damp on the diagonal of the undamped S)."""
    A = np.array(S, np.float64, copy=True)
    free = dof_mask(cam_dof)
    d = np.arange(A.shape[0])
    A[d, d] = np.where(free, A[d, d] + lam * np.clip(diagU, 1e-6, 1e32), 1.0)
    return A


# ---- double-double fallback: error-free transformations (Dekker, Knuth) ------------------------------------------------------------
def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    c = 134217729.0 * a
    h = c - (c - a)
    return h, a - h


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _dd_matvec(A, x):
    s = np.zeros(A.shape[0]); c = np.zeros(A.shape[0])
    for j in range(A.shape[1]):
        p, e = _two_prod(A[:, j], x[j])
        s, q = _two_sum(s, p)
        c += q + e
    return s + c


def _dd_dot(a, b):
    p, e = _two_prod(np.asarray(a, np.float64), np.asarray(b, np.float64))
    return math.fsum(np.concatenate([p, e]))


class Reference:
    """x*, kappa_2 and the extended-precision PCG of one damped system A x = g (A, g: fp64, taken as exact)."""

    def __init__(self, A: np.ndarray, g: np.ndarray):
        self.A = np.ascontiguousarray(A, np.float64)
        self.g = np.ascontiguousarray(g, np.float64)
        self.n = self.A.shape[0]
        self.Ax = self.A.astype(XP) if EXTENDED else None
        self.kappa = float(np.linalg.cond(self.A, 2))
        self.Minv = self._block_jacobi()
        self.xstar = self._refined_solve()
        self.xA = math.sqrt(max(float(self.dot(self.xstar, self.mv(self.xstar))), 0.0))
        self.gz0 = float(self.dot(self.g, self.precond(self.g.astype(XP))))

    # extended-precision kernels
    def mv(self, x):
        return self.Ax @ np.asarray(x, XP) if EXTENDED else _dd_matvec(self.A, np.asarray(x, np.float64))

    def dot(self, a, b):
        return np.dot(np.asarray(a, XP), np.asarray(b, XP)) if EXTENDED else _dd_dot(a, b)

    def precond(self, r):
        nb = self.n // 6
        return np.einsum("iab,ib->ia", self.Minv, np.asarray(r, XP).reshape(nb, 6)).reshape(-1)

    def _block_jacobi(self):
        """Per camera: the inverse of the damped 6x6 diagonal block, or of its diagonal where the block is not positive definite."""
        nb = self.n // 6
        M = np.zeros((nb, 6, 6), XP)
        for i in range(nb):
            D = self.A[6 * i:6 * i + 6, 6 * i:6 * i + 6]
            try:
                L = np.linalg.cholesky(D)
                Li = scipy.linalg.solve_triangular(L, np.eye(6), lower=True)
                M[i] = (Li.T @ Li).astype(XP)
            except np.linalg.LinAlgError:
                M[i] = np.diag(1.0 / np.diag(D)).astype(XP)
        return M

    def _refined_solve(self):
        c = scipy.linalg.cho_factor(self.A, lower=True)
        x = scipy.linalg.cho_solve(c, self.g).astype(XP)
        for _ in range(10):
            r = np.asarray(self.g, XP) - self.mv(x)
            dx = scipy.linalg.cho_solve(c, np.asarray(r, np.float64))
            x = x + np.asarray(dx, XP)
            if np.abs(dx).max() <= 1e-3 * EPS * max(float(np.abs(x).max()), 1e-300):
                break
        return x

    # what a solution is measured by
    def a_err(self, x) -> float:
        """||x - x*||_A / ||x*||_A."""
        e = np.asarray(x, XP) - self.xstar
        return math.sqrt(max(float(self.dot(e, self.mv(e))), 0.0)) / max(self.xA, 1e-300)

    def res_ratio(self, x) -> float:
        """sqrt(r'M^-1 r / g'M^-1 g) of the TRUE residual r = g - A x: the quantity the PCG's stopping test bounds."""
        r = np.asarray(self.g, XP) - self.mv(x)
        return math.sqrt(max(float(self.dot(r, self.precond(r))), 0.0) / max(self.gz0, 1e-300))

    def backward_err(self, x) -> float:
        r = np.asarray(self.g, XP) - self.mv(x)
        den = np.abs(self.A).sum(axis=1).max() * np.abs(x).max() + np.abs(self.g).max()
        return float(np.abs(r).max()) / max(float(den), 1e-300)

    def forward_err(self, x) -> float:
        return float(np.abs(np.asarray(x, XP) - self.xstar).max()) / max(float(np.abs(self.xstar).max()), 1e-300)

    def pcg(self, maxit: int, tol: float = 0.0, errs_at=()):
        """PCG in extended precision.  Returns (iterations, x, ratios, errs): ratios[k] = sqrt(r_k'z_k / r_0'z_0) for k = 0..iterations,
        errs[k] = relative A-norm error of x_k for each k in errs_at that was reached."""
        x = np.zeros(self.n, XP)
        r = np.asarray(self.g, XP).copy()
        z = self.precond(r)
        p = z.copy()
        rz = self.dot(r, z)
        rz0 = rz
        ratios, errs = [1.0 if rz0 > 0 else 0.0], {}
        k = 0
        if 0 in errs_at:
            errs[0] = self.a_err(x)
        if not rz0 > 0:
            return 0, x, ratios, errs
        while k < maxit:
            q = self.mv(p)
            pq = self.dot(p, q)
            if not pq > 0:
                break
            alpha = rz / pq
            x = x + alpha * p
            r = r - alpha * q
            z = self.precond(r)
            rz_new = self.dot(r, z)
            k += 1
            ratios.append(math.sqrt(max(float(rz_new / rz0), 0.0)))
            if k in errs_at:
                errs[k] = self.a_err(x)
            if not rz_new > 0 or rz_new < tol * tol * rz0:
                break
            p = z + (rz_new / rz) * p
            rz = rz_new
        return k, x, ratios, errs


# ---- bounds, calibrated against the fp64 oracle (tests/test_ba_linsys_reference.py) -----------------------------------------------
def a_err_floor(ref: Reference) -> float:
    """Relative A-norm error at which an fp64 PCG on this system stagnates (see the calibration in test_ba_linsys_reference.py)."""
    return 16.0 * ref.n * EPS * math.sqrt(ref.kappa)


def res_floor(ref: Reference) -> float:
    """kappa * eps term of the true preconditioned residual ratio an fp64 solve can reach."""
    return ref.kappa * EPS


# ---- graphs built for the solver contracts -------------------------------------------------------------------------------------------
def _join(a: synth.BAProblem, b: synth.BAProblem) -> synth.BAProblem:
    """Two graphs side by side in one window (no shared landmark)."""
    nca, npa = a.n_cams, a.n_points
    return synth.BAProblem(cam_pose_wc=np.ascontiguousarray(np.vstack([a.cam_pose_wc, b.cam_pose_wc])), cam_dof=np.concatenate([a.cam_dof, b.cam_dof]),
                           points=np.ascontiguousarray(np.vstack([a.points, b.points])), point_free=np.concatenate([a.point_free, b.point_free]),
                           obs_cam=np.ascontiguousarray(np.concatenate([a.obs_cam, b.obs_cam + nca]).astype(np.int32)),
                           obs_point=np.ascontiguousarray(np.concatenate([a.obs_point, b.obs_point + npa]).astype(np.int32)),
                           obs_xyz=np.ascontiguousarray(np.vstack([a.obs_xyz, b.obs_xyz])),
                           gt_pose_wc=np.vstack([a.gt_pose_wc, b.gt_pose_wc]), gt_points=np.vstack([a.gt_points, b.gt_points]))


def one_active() -> synth.BAProblem:
    """One free camera among 29 fixed ones (a single active camera for the single-CTA PCG)."""
    pb = synth.synth_ba(30, 500, obs_per_point=4, n_fixed=0, seed=121)
    pb.cam_dof[:] = 0
    pb.cam_dof[17] = 63
    return pb


def mixed_scales() -> synth.BAProblem:
    """One window, two scene scales: a trajectory shrunk to millimetres next to one a kilometre away (camera translations ~1e-3 and
    ~1e3; the projections, hence the measurements, do not change with the scale)."""
    a = synth.synth_ba(15, 250, obs_per_point=4, n_fixed=1, seed=131)
    b = synth.synth_ba(15, 250, obs_per_point=4, n_fixed=1, seed=132)
    for p in (a.cam_pose_wc, a.gt_pose_wc):
        p[:, 4:] *= 1e-3
    a.points *= 1e-3; a.gt_points *= 1e-3
    off = np.array([1000.0, 0.0, 0.0])
    for p in (b.cam_pose_wc, b.gt_pose_wc):
        p[:, 4:] += off
    b.points += off; b.gt_points += off
    return _join(a, b)


def zero_rhs() -> synth.BAProblem:
    """A noise-free graph at its optimum whose residuals are exactly zero in fp64: identity rotations, dyadic translations and
    landmarks, depths that are powers of two.  Every gradient, hence g~, is exactly 0 while S is not."""
    rng = np.random.default_rng(151)
    nc, np_ = 8, 60
    pose = np.zeros((nc, 7)); pose[:, 3] = 1.0; pose[:, 4] = 0.5 * np.arange(nc); pose[:, 5] = 0.25 * (np.arange(nc) % 3)
    pts = np.stack([rng.integers(-16, 17, np_) / 8.0, rng.integers(-8, 9, np_) / 8.0, 2.0 ** rng.integers(2, 5, np_)], axis=1)
    oc, op = [], []
    for j in range(np_):
        first = int(rng.integers(0, nc - 3))
        for i in range(first, first + 4):
            oc.append(i); op.append(j)
    oc = np.asarray(oc, np.int32); op = np.asarray(op, np.int32)
    pc = pts[op] - pose[oc, 4:]                       # R = I: camera coordinates, exact
    xyz = np.ascontiguousarray(pc)                    # (x, y, z) with z a power of two: x/z and y/z are exact
    dof = np.full(nc, 63, np.uint8); dof[0] = 0
    return synth.BAProblem(cam_pose_wc=pose, cam_dof=dof, points=np.ascontiguousarray(pts), point_free=np.ones(np_, np.uint8),
                           obs_cam=oc, obs_point=op, obs_xyz=xyz, gt_pose_wc=pose.copy(), gt_points=pts.copy())


def loop_closure() -> synth.BAProblem:
    """A band (3 observers per landmark) plus one landmark seen by the first and the last camera: the block (last, 0) makes the
    monotone skyline's first[] 0 for every row, the whole lower block triangle."""
    pb = synth.synth_ba(30, 500, obs_per_point=3, n_fixed=2, seed=141)
    ba_graphs._add_landmark(pb, [0, pb.n_cams - 1], np.random.default_rng(3), 30.0)
    return pb


def narrow_band_100() -> synth.BAProblem:
    """100 cameras, landmarks seen by 2 consecutive keyframes: 6N = 600 unknowns, more than the 512-thread strides."""
    return synth.synth_ba(100, 1500, obs_per_point=2, n_fixed=2, seed=142)


def skyline(pb: synth.BAProblem) -> np.ndarray:
    """first[] of the monotone block skyline of S (csrc/ba_chol.cu ba_chol_plan_host), from the covisibility of free landmarks."""
    first = np.arange(pb.n_cams)
    free = pb.point_free[pb.obs_point] != 0
    order = np.lexsort((pb.obs_cam[free], pb.obs_point[free]))
    oc, op = pb.obs_cam[free][order], pb.obs_point[free][order]
    starts = np.r_[0, np.nonzero(np.diff(op))[0] + 1, op.shape[0]]
    for s, e in zip(starts[:-1], starts[1:]):
        if e - s >= 2:                                # (cameras sorted: the lowest observer is oc[s])
            first[oc[s:e]] = np.minimum(first[oc[s:e]], oc[s])
    return np.minimum.accumulate(first[::-1])[::-1]


def skyline_blocks(pb) -> int:
    f = skyline(pb)
    return int((np.arange(pb.n_cams) - f + 1).sum())


def chol_fits(nblocks: int, nc: int, max_smem_optin: int) -> bool:
    """ba_chol_plan_host's shared-memory test of a skyline of `nblocks` 6x6 blocks."""
    smem = (nblocks * 36 + 12 * nc) * 8 + 3 * nc * 4 + 64
    return smem + 1024 <= max_smem_optin


def skyline_at(max_smem_optin: int, over: bool) -> synth.BAProblem:
    """A band graph whose skyline is the largest that fits the direct solver's shared memory (over: one block more).  Landmarks seen
    by w+1 consecutive keyframes make a band of width w; each extra landmark seen by cameras (i-w-1, i), from the last row upwards,
    adds exactly one block."""
    for nc in range(48, 160):
        limit = max(n for n in range(nc, nc * (nc + 1) // 2 + 1) if chol_fits(n, nc, max_smem_optin)) if chol_fits(nc, nc, max_smem_optin) else -1
        for w in range(2, 24):
            band = (w + 1) * (w + 2) // 2 + (nc - w - 1) * (w + 1)
            extra = limit + (1 if over else 0) - band
            if 0 <= extra <= nc - w - 2:
                pb = synth.synth_ba(nc, 30 * nc, obs_per_point=w + 1, n_fixed=2, seed=160 + nc)
                assert skyline_blocks(pb) == band
                rng = np.random.default_rng(4)
                for i in range(nc - 1, nc - 1 - extra, -1):
                    ba_graphs._add_landmark(pb, [i - w - 1, i], rng, 30.0)
                assert skyline_blocks(pb) == limit + (1 if over else 0)
                return pb
    raise AssertionError("no band graph reaches the shared-memory limit")
