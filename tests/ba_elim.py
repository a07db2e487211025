"""Extended-precision restatement of the BA landmark elimination and back-substitution (a test helper, not product code).

It takes one linearisation as given -- U, g_c, V, g_p and W in the caller's edge order, as BAGraph.dbg_linearize returns it (or the
oracle's ba_linearize) -- and restates what the device forms from it:

  V~_j        V_j with lm_damp on its diagonal: V_aa + lambda * clamp(V_aa, 1e-6, 1e32) (csrc/ba_device.cuh), for an ACTIVE landmark
              (free and observed); an inactive one has V~^-1 = 0
  V~_j^-1     adjugate / determinant in extended precision, then one refinement step X <- X + X (I - V~ X)
  S           blockdiag(U) - sum_j W_ij V~_j^-1 W_kj' over the landmarks cameras i and k both observe (blocks with i <= k; the lower
              triangle is the transpose)
  g~          g_c,i - sum_j W_ij V~_j^-1 g_p,j
  p_new       p_j + V~_j^-1 (g_p,j - sum_i W_ij' x_i) for a given camera step x

Extended precision is ba_linsys's: numpy's long double where it carries at least 64 mantissa bits, else double-double arithmetic on
(hi, lo) pairs of fp64 arrays built from its error-free transformations.  Either can be asked for (`mode`), so that the CPU tests can
hold the two against each other.

Bounds (u = 2^-53, |.| elementwise, kappa_j = kappa_2(V~_j), sums over the landmarks both cameras observe):

  S block (i, k)   C_S u (delta_ik m_i |U_i| + sum_j (1 + kappa_j) |W_ij| |V~_j^-1| |W_kj|')
  g~_i             C_G u (m_i |g_c,i| + sum_j (1 + kappa_j) |W_ij| |V~_j^-1| |g_p,j|)
  p_new_j          C_P u (|p_j| + (1 + kappa_j) |V~_j^-1| (|g_p,j| + sum_i |W_ij|' |x_i|))
  V~_j^-1          C_V u kappa_j ||V~_j^-1||_2 (normwise)

m_i is 1 where the landmark terms are summed before they are subtracted from U_i and g_c,i (ba_schur_blocks_kernel,
ba_schur_reduce_kernel), and the number of terms of camera i where they are subtracted one by one (`into_u`: ba_schur_accum_kernel,
the oracle).  A landmark whose V~ the device's fp64 Cholesky (mirrored by spd_inverse3_fp64) cannot factor has V~^-1 = 0, as
damped_vinv writes it, and contributes nothing.

The constants are 8x the largest error / bound ratio that fp64 restatements of the same operations reach (landmarks summed forward,
reversed and shuffled, or subtracted one by one from U_i and g_c,i; V~^-1 by the device's Cholesky and by np.linalg.inv) on the
calibration graphs of tests/test_ba_elim_reference.py, which records those ratios.
"""
from __future__ import annotations

import numpy as np

from ba_linsys import EXTENDED, XP, _two_prod, _two_sum, dof_mask  # (tests/ is on sys.path under pytest's rootdir conftest)

U_RND = 2.0 ** -53
# calibrated in tests/test_ba_elim_reference.py (8 x the largest fp64 ratio recorded there)
C_S, C_G, C_P, C_V = 8 * 0.98, 8 * 0.96, 8 * 1.0, 8 * 3.3


# ---- double-double arrays ----------------------------------------------------------------------------------------------------------
def _fast_two_sum(a, b):
    s = a + b
    return s, b - (s - a)


class DD:
    """An array of double-double numbers hi + lo (|lo| <= ulp(hi) / 2), with numpy broadcasting and indexing."""
    __slots__ = ("hi", "lo")

    def __init__(self, hi, lo=None):
        self.hi = np.asarray(hi, np.float64)
        self.lo = np.zeros_like(self.hi) if lo is None else np.asarray(lo, np.float64)

    @staticmethod
    def of(a):
        return a if isinstance(a, DD) else DD(np.asarray(a, np.float64))

    shape = property(lambda self: self.hi.shape)

    def __getitem__(self, k):
        return DD(self.hi[k], self.lo[k])

    def __setitem__(self, k, v):
        v = DD.of(v)
        self.hi[k] = v.hi
        self.lo[k] = v.lo

    def __neg__(self):
        return DD(-self.hi, -self.lo)

    def __add__(self, o):
        o = DD.of(o)
        s, e = _two_sum(self.hi, o.hi)
        return DD(*_fast_two_sum(s, e + (self.lo + o.lo)))

    __radd__ = __add__

    def __sub__(self, o):
        return self + (-DD.of(o))

    def __rsub__(self, o):
        return DD.of(o) + (-self)

    def __mul__(self, o):
        o = DD.of(o)
        p, e = _two_prod(self.hi, o.hi)
        return DD(*_fast_two_sum(p, e + (self.hi * o.lo + self.lo * o.hi)))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = DD.of(o)
        q1 = self.hi / o.hi
        r = self - o * q1
        q2 = r.hi / o.hi
        r = r - o * q2
        return DD(*_fast_two_sum(q1, q2)) + r.hi / o.hi

    def to_float(self):
        return self.hi + self.lo

    def copy(self):
        return DD(self.hi.copy(), self.lo.copy())


class Arith:
    """The extended arithmetic of one mode: 'ld' (numpy long double) or 'dd' (double-double)."""

    def __init__(self, mode: str | None = None):
        self.mode = mode or ("ld" if EXTENDED else "dd")
        assert self.mode in ("ld", "dd")
        if self.mode == "ld":
            assert EXTENDED, "numpy's long double is fp64 here"

    def x(self, a):
        return np.array(a, XP) if self.mode == "ld" else DD(np.array(a, np.float64))

    def zeros(self, shape):
        return np.zeros(shape, XP) if self.mode == "ld" else DD(np.zeros(shape))

    def stack(self, items, axis):
        if self.mode == "ld":
            return np.stack(items, axis=axis)
        return DD(np.stack([i.hi for i in items], axis=axis), np.stack([i.lo for i in items], axis=axis))

    def f64(self, a):
        return np.asarray(a, np.float64) if self.mode == "ld" else a.to_float()

    def diff(self, dev, ref):
        """|dev - ref| in fp64 (dev: fp64, ref: extended)."""
        if self.mode == "ld":
            return np.abs(np.asarray(np.asarray(dev, XP) - ref, np.float64))
        return np.abs((np.asarray(dev, np.float64) - ref.hi) - ref.lo)

    def group_sum(self, vals, grp, n):
        """out[g] = sum of vals[k] over grp[k] == g, each group added in order of k (rows of vals: one per k)."""
        out = self.zeros((n,) + tuple(vals.shape[1:]))
        if len(grp) == 0:
            return out
        order = np.argsort(grp, kind="stable")
        g = grp[order]
        start = np.r_[0, np.nonzero(np.diff(g))[0] + 1]
        rank = np.arange(g.shape[0]) - np.repeat(start, np.diff(np.r_[start, g.shape[0]]))
        for r in range(int(rank.max()) + 1):
            sel = order[rank == r]
            out[grp[sel]] = out[grp[sel]] + vals[sel]
        return out


def mm(A, B):
    """(..., m, k) x (..., k, n) as explicit sums of broadcast products (works for fp64, long double and DD alike)."""
    acc = A[..., :, 0:1] * B[..., 0:1, :]
    for k in range(1, A.shape[-1]):
        acc = acc + A[..., :, k:k + 1] * B[..., k:k + 1, :]
    return acc


def damped_V(V, lam):
    """V~ in fp64 as lm_damp writes it (clamp of the undamped diagonal), for every landmark."""
    Vd = np.array(V, np.float64, copy=True)
    d = np.arange(3)
    Vd[:, d, d] = V[:, d, d] + lam * np.clip(V[:, d, d], 1e-6, 1e32)
    return Vd


def spd_inverse3_fp64(A):
    """fp64 mirror of spd_inverse<3> (csrc/ba_device.cuh) in its operation order, vectorised: (inverse, ok).  A failed landmark gets 0,
    as damped_vinv writes it."""
    A = np.asarray(A, np.float64)
    n = A.shape[0]
    L = np.zeros((n, 3, 3)); Li = np.zeros((n, 3, 3)); idg = np.zeros((n, 3))
    ok = np.ones(n, bool)
    with np.errstate(all="ignore"):
        for i in range(3):
            for j in range(i + 1):
                s = A[:, i, j].copy()
                for k in range(j):
                    s = s - L[:, i, k] * L[:, j, k]
                if i == j:
                    ok &= s > 0.0
                    L[:, i, i] = np.sqrt(np.where(s > 0.0, s, 1.0))
                    idg[:, i] = 1.0 / L[:, i, i]
                else:
                    L[:, i, j] = s * idg[:, j]
        for c in range(3):
            for i in range(c, 3):
                s = np.full(n, 1.0 if i == c else 0.0)
                for k in range(c, i):
                    s = s - L[:, i, k] * Li[:, k, c]
                Li[:, i, c] = s * idg[:, i]
        X = np.zeros((n, 3, 3))
        for i in range(3):
            for j in range(3):
                s = np.zeros(n)
                for k in range(max(i, j), 3):
                    s = s + Li[:, k, i] * Li[:, k, j]
                X[:, i, j] = s
    X[~ok] = 0.0
    return X, ok


def active_landmarks(pb) -> np.ndarray:
    return (np.asarray(pb.point_free) != 0) & (np.bincount(pb.obs_point, minlength=pb.n_points) > 0)


def edge_pairs(pb, keep=None):
    """Every pair (e, f) of edges of one landmark with cam(e) <= cam(f), over the landmarks `keep` (default: active), in landmark order:
    (e, f, j)."""
    keep = active_landmarks(pb) if keep is None else keep
    ne = pb.n_obs
    sel = np.nonzero(keep[pb.obs_point])[0]
    order = sel[np.lexsort((pb.obs_cam[sel], pb.obs_point[sel]))]      # edges by (landmark, camera)
    lm = pb.obs_point[order]
    starts = np.r_[0, np.nonzero(np.diff(lm))[0] + 1] if order.size else np.zeros(0, np.int64)
    deg = np.diff(np.r_[starts, order.size]) if order.size else np.zeros(0, np.int64)
    E, F = [], []
    for d in np.unique(deg):
        a, b = np.triu_indices(int(d))
        s = starts[deg == d]
        E.append(order[s[:, None] + a[None, :]].reshape(-1)); F.append(order[s[:, None] + b[None, :]].reshape(-1))
    if not E:
        z = np.zeros(0, np.int64)
        return z, z, z
    e, f = np.concatenate(E), np.concatenate(F)
    o = np.argsort(pb.obs_point[e], kind="stable")                     # landmark order (then as generated: camera order)
    e, f = e[o], f[o]
    assert ne == 0 or e.max() < ne
    return e, f, pb.obs_point[e]


class Elim:
    """The extended-precision elimination of one linearisation at one lambda, with its componentwise bounds."""

    def __init__(self, pb, lin, lam: float, mode: str | None = None, into_u: bool = False):
        """into_u: bound the accumulation order that subtracts the landmark terms one by one from U_i and g_c,i (ba_schur_accum_kernel,
        the oracle): every one of the n terms of a block rounds at the magnitude of U_i, so |U_i| and |g_c,i| count n times."""
        A = self.A = Arith(mode)
        self.pb, self.lam = pb, float(lam)
        nc, np_ = pb.n_cams, pb.n_points
        self.active = act = active_landmarks(pb)
        U, gc, V, gp, W = (np.asarray(lin[k], np.float64) for k in ("U", "gc", "V", "gp", "W"))
        self.U, self.gc, self.V, self.gp, self.W = U, gc, V, gp, W
        # V~ (damped diagonal exact in extended precision), V~^-1: adjugate, then one refinement step
        Vt = A.x(V[act])
        for a in range(3):
            Vt[:, a, a] = Vt[:, a, a] + A.x(np.full(int(act.sum()), self.lam)) * A.x(np.clip(V[act, a, a], 1e-6, 1e32))
        cof = [[None] * 3 for _ in range(3)]
        for r in range(3):
            for s in range(3):
                r1, r2 = [k for k in range(3) if k != r]
                s1, s2 = [k for k in range(3) if k != s]
                m = Vt[:, r1, s1] * Vt[:, r2, s2] - Vt[:, r1, s2] * Vt[:, r2, s1]
                cof[r][s] = m if (r + s) % 2 == 0 else -m
        det = Vt[:, 0, 0] * cof[0][0] + Vt[:, 0, 1] * cof[0][1] + Vt[:, 0, 2] * cof[0][2]
        X = A.stack([A.stack([cof[s][r] / det for s in range(3)], -1) for r in range(3)], -2)  # X_rs = cof_sr / det
        R = A.x(np.broadcast_to(np.eye(3), X.shape)) - mm(Vt, X)
        X = X + mm(X, R)
        self.Vt64 = damped_V(V, self.lam)
        # where the device's fp64 Cholesky of V~ fails, damped_vinv writes V~^-1 = 0: the landmark then contributes nothing
        self.zeroed = act & ~spd_inverse3_fp64(self.Vt64)[1]
        self.kappa = np.zeros(np_)
        live = act & ~self.zeroed
        if live.any():
            self.kappa[live] = np.linalg.cond(self.Vt64[live], 2)
        Xf = A.zeros((np_, 3, 3))
        Xf[act] = X
        Xf[self.zeroed] = A.zeros((int(self.zeroed.sum()), 3, 3))
        self.X = Xf
        self.X64 = A.f64(Xf)
        self.X_bound = C_V * U_RND * self.kappa * (np.linalg.norm(self.X64, 2, axis=(1, 2)) if np_ else np.zeros(0))
        # S blocks (i <= k) and g~
        e, f, j = edge_pairs(pb)
        oc = pb.obs_cam
        ci, ck = oc[e], oc[f]
        key = np.r_[np.arange(nc, dtype=np.int64) * (nc + 1), ci.astype(np.int64) * nc + ck]
        ukeys, inv = np.unique(key, return_inverse=True)
        self.blocks = np.stack([ukeys // nc, ukeys % nc], axis=1)
        nb = ukeys.shape[0]
        pair_blk = inv[nc:]
        Wx = A.x(W)
        Y = mm(Wx[e], self.X[j])                                            # W_ij V~^-1
        T = mm(Y, A.x(np.swapaxes(W[f], 1, 2)))                             # W_ij V~^-1 W_kj'
        Sb = A.zeros((nb, 6, 6))
        diag_blk = inv[:nc]
        Sb[diag_blk] = A.x(U)
        self.S = Sb - A.group_sum(T, pair_blk, nb)
        w1k = (1.0 + self.kappa[j])[:, None, None]
        aW, aX = np.abs(W), np.abs(self.X64)
        Tb = w1k * np.einsum("pab,pbc,pdc->pad", aW[e], aX[j], aW[f], optimize=True)
        Bb = np.zeros((nb, 6, 6))
        np.add.at(Bb, pair_blk, Tb)
        n_terms = np.bincount(pair_blk, minlength=nb)[diag_blk] if into_u else np.ones(nc)
        Bb[diag_blk] += np.maximum(n_terms, 1)[:, None, None] * np.abs(U)
        self.S_bound = C_S * U_RND * Bb
        # g~: one term per active edge
        ea = np.nonzero(act[pb.obs_point])[0]
        ja = pb.obs_point[ea]
        Ye = mm(Wx[ea], self.X[ja])
        tg = mm(Ye, A.x(gp[ja][:, :, None]))[:, :, 0]
        self.gt = A.x(gc) - A.group_sum(tg, oc[ea], nc)
        gb = np.zeros((nc, 6))
        np.add.at(gb, oc[ea], (1.0 + self.kappa[ja])[:, None] * np.einsum("pab,pbc,pc->pa", aW[ea], aX[ja], np.abs(gp[ja]), optimize=True))
        n_g = np.maximum(np.bincount(oc[ea], minlength=nc), 1) if into_u else np.ones(nc)
        self.gt_bound = C_G * U_RND * (n_g[:, None] * np.abs(gc) + gb)
        self.diagU = np.ascontiguousarray(np.diagonal(U, axis1=1, axis2=2)).reshape(-1)
        self.structural = np.zeros((nc, nc), bool)
        self.structural[self.blocks[:, 0], self.blocks[:, 1]] = True
        self.structural |= self.structural.T

    # ---- the back-substitution at a given camera step -------------------------------------------------------------------------------
    def candidate(self, x, points):
        """(p_new in extended precision, its bound) for camera step x (6N, fp64) and current landmarks `points`."""
        A, pb = self.A, self.pb
        x = np.asarray(x, np.float64).reshape(pb.n_cams, 6)
        e = np.arange(pb.n_obs)
        Wt = A.x(np.swapaxes(self.W, 1, 2))                                  # W' (3 x 6) per edge
        t = mm(Wt, A.x(x[pb.obs_cam][:, :, None]))[:, :, 0]
        b = A.x(self.gp) - A.group_sum(t, pb.obs_point[e], pb.n_points)
        p = A.x(points) + mm(self.X, b[:, :, None])[:, :, 0]
        wx = np.zeros((pb.n_points, 3))
        np.add.at(wx, pb.obs_point, np.einsum("eab,ea->eb", np.abs(self.W), np.abs(x[pb.obs_cam])))
        bound = C_P * U_RND * (np.abs(points) + (1.0 + self.kappa)[:, None] * np.einsum("jab,jb->ja", np.abs(self.X64), np.abs(self.gp) + wx))
        return p, bound

    # ---- comparisons: largest |device - reference| / bound (inf where the bound is 0 and the device is not exact) ---------------------
    @staticmethod
    def ratio(err, bound):
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(err == 0.0, 0.0, err / bound)
        return float(r.max(initial=0.0))

    def s_blocks(self, S):
        """The (i <= k) blocks of a dense 6N x 6N S, in the order of self.blocks."""
        i, k = self.blocks[:, 0], self.blocks[:, 1]
        r = 6 * i[:, None] + np.arange(6)[None, :]
        c = 6 * k[:, None] + np.arange(6)[None, :]
        return S[r[:, :, None], c[:, None, :]]

    def s_ratio(self, S_blocks):
        return self.ratio(self.A.diff(S_blocks, self.S), self.S_bound)

    def gt_ratio(self, gt):
        return self.ratio(self.A.diff(np.asarray(gt).reshape(-1, 6), self.gt), self.gt_bound)

    def vinv_ratio(self, X):
        X = np.asarray(X, np.float64).reshape(-1, 3, 3)
        err = np.linalg.norm(self.A.f64(self.A.x(X) - self.X), 2, axis=(1, 2)) if X.shape[0] else np.zeros(0)
        return self.ratio(err, self.X_bound)

    def cand_ratio(self, p_dev, x, points):
        p, b = self.candidate(x, points)
        return self.ratio(self.A.diff(p_dev, p), b)


# ---- fp64 restatements (calibration) and their deliberate faults (sensitivity) ---------------------------------------------------------
def eliminate_fp64(pb, lin, lam, order="forward", inv="chol", fault=None, seed=0):
    """fp64 S (dense), g~ and V~^-1 of one linearisation: landmarks accumulated in `order` (forward / reversed / shuffled, each summed
    then subtracted from U_i and g_c,i; `into_u`: forward, subtracted one by one from U_i and g_c,i, as ba_schur_accum_kernel and the
    oracle do), V~^-1 by the device's Cholesky (`chol`) or np.linalg.inv (`inv`).  `fault` = (name, arg) plants one defect:
      drop_landmark j, undamped, lambda_nu, transpose_block (i, k), lost_pass j (the pairs of landmark j in chunk slots >= 80),
      y_float32, neighbour_w e (W_kj of edge e replaced by the next edge's)."""
    name, arg = fault if fault else (None, None)
    nc = pb.n_cams
    U, gc, V, gp, W = (np.asarray(lin[k], np.float64) for k in ("U", "gc", "V", "gp", "W"))
    act = active_landmarks(pb)
    lam_v = 0.0 if name == "undamped" else (2.0 * lam if name == "lambda_nu" else lam)
    Vt = damped_V(V, lam_v) if name != "undamped" else np.array(V, copy=True)
    if inv == "chol":
        X, _ = spd_inverse3_fp64(Vt)
    else:
        with np.errstate(all="ignore"):
            X = np.linalg.inv(Vt + np.where(act, 0.0, 1.0)[:, None, None] * np.eye(3))
        X[~spd_inverse3_fp64(Vt)[1]] = 0.0              # (the device's rule: zero where its Cholesky fails)
    X[~act] = 0.0
    e, f, j = edge_pairs(pb)
    if name == "drop_landmark":
        m = j != arg
        e, f, j = e[m], f[m], j[m]
    if name == "lost_pass":
        cams = np.sort(pb.obs_cam[pb.obs_point == arg])
        la, lb = np.searchsorted(cams, pb.obs_cam[e]), np.searchsorted(cams, pb.obs_cam[f])
        m = (j != arg) | (lb * (lb + 1) // 2 + la < 80)
        e, f, j = e[m], f[m], j[m]
    Wf = W[f].copy()
    if name == "neighbour_w":
        Wf[f == arg] = W[arg + 1]
    rng = np.random.default_rng(seed)
    pos = {"forward": np.arange(pb.n_points), "into_u": np.arange(pb.n_points), "reversed": np.arange(pb.n_points)[::-1], "shuffled": rng.permutation(pb.n_points)}[order]
    rank = np.empty(pb.n_points, np.int64); rank[pos] = np.arange(pb.n_points)
    o = np.argsort(rank[j], kind="stable")
    e, f, j, Wf = e[o], f[o], j[o], Wf[o]
    Y = np.einsum("pab,pbc->pac", W[e].astype(np.float32), X[j].astype(np.float32)).astype(np.float64) if name == "y_float32" else mm(W[e], X[j])
    T = mm(Y, np.swapaxes(Wf, 1, 2))
    S = np.zeros((6 * nc, 6 * nc))
    r6 = np.arange(6)
    for i in range(nc):
        S[6 * i:6 * i + 6, 6 * i:6 * i + 6] = U[i]
    blk = pb.obs_cam[e].astype(np.int64) * nc + pb.obs_cam[f]
    if order == "into_u":                               # (-U_i first: -(-U_i + t1 + t2 ...) is U_i - t1 - t2 ... bit for bit)
        T = np.concatenate([-U, T]); blk = np.r_[np.arange(nc, dtype=np.int64) * (nc + 1), blk]
        for i in range(nc):
            S[6 * i:6 * i + 6, 6 * i:6 * i + 6] = 0.0
    for b, v in _group_sum64(T, blk).items():           # (each block accumulated in landmark order)
        i, k = divmod(b, nc)
        S[6 * i + r6[:, None], 6 * k + r6[None, :]] -= v
        if i != k:
            S[6 * k + r6[:, None], 6 * i + r6[None, :]] -= v.T
    if name == "transpose_block":
        i, k = arg
        blkv = S[6 * i:6 * i + 6, 6 * k:6 * k + 6].copy()
        S[6 * i:6 * i + 6, 6 * k:6 * k + 6] = blkv.T
    ea = np.nonzero(act[pb.obs_point])[0]
    ea = ea[np.argsort(rank[pb.obs_point[ea]], kind="stable")]
    ja = pb.obs_point[ea]
    tg = mm(mm(W[ea], X[ja]), gp[ja][:, :, None])[:, :, 0]
    gt = gc.copy()
    gi = pb.obs_cam[ea].astype(np.int64)
    if order == "into_u":
        tg = np.concatenate([-gc, tg]); gi = np.r_[np.arange(nc, dtype=np.int64), gi]
        gt[:] = 0.0
    for i, v in _group_sum64(tg, gi).items():
        gt[i] -= v
    return dict(S=S, gt=gt.reshape(-1), X=X)


def _group_sum64(vals, grp):
    """{g: fp64 sum of vals[k] over grp[k] == g, added in order of k}."""
    out = {}
    if len(grp) == 0:
        return out
    order = np.argsort(grp, kind="stable")
    g = grp[order]
    start = np.r_[0, np.nonzero(np.diff(g))[0] + 1]
    rank = np.arange(g.shape[0]) - np.repeat(start, np.diff(np.r_[start, g.shape[0]]))
    tot = np.zeros((start.shape[0],) + vals.shape[1:])
    slot = np.repeat(np.arange(start.shape[0]), np.diff(np.r_[start, g.shape[0]]))
    for r in range(int(rank.max()) + 1):
        m = rank == r
        tot[slot[m]] = tot[slot[m]] + vals[order[m]]
    return {int(b): tot[s] for s, b in enumerate(g[start])}


def candidate_fp64(pb, lin, X, x, points, fault=None):
    """fp64 back-substitution p + V~^-1 (g_p - sum W' x) with the device's landmark inverses X.  `fault` = (name, arg): drop_camera i
    (x_i taken as 0), negate_edge e (W_e' x negated)."""
    name, arg = fault if fault else (None, None)
    x = np.array(x, np.float64).reshape(pb.n_cams, 6)
    if name == "drop_camera":
        x[arg] = 0.0
    W = np.asarray(lin["W"])
    t = np.einsum("eab,ea->eb", W, x[pb.obs_cam])
    if name == "negate_edge":
        t[arg] = -t[arg]
    b = np.array(lin["gp"], np.float64, copy=True)
    for j, v in _group_sum64(t, pb.obs_point.astype(np.int64)).items():
        b[j] -= v
    return points + np.einsum("jab,jb->ja", X, b)
