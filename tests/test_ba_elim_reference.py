"""Pins the extended-precision landmark elimination of tests/ba_elim.py on the CPU, before any GPU test relies on it.

Self-consistency: the long-double and the double-double arithmetic agree to 1 % of every bound, and the fp64 oracle's reduced system
(oracle/ba_ref.c) is within the bounds on every tests/ba_graphs.py case.

Calibration: fp64 restatements of the elimination (landmarks summed forward, reversed and shuffled, or subtracted one by one from U_i
and g_c,i; V~^-1 by the device's Cholesky and by np.linalg.inv; the back-substitution at a random camera step) on every ba_graphs
case and every numeric-edge graph of ba_graphs.EDGES, at lambda 1e-8, 1e-4 and 1e4.  Largest error / bound ratio with the constants at 1 (RATIOS):

  S      0.98      g~     0.96      p_new  1.0      V~^-1  3.3

(the subtract-one-by-one order against its own bound, with n |U_i| and n |g_c,i|: 0.35 and 0.34)

Each constant of ba_elim is 8x its ratio.

Sensitivity: each deliberate fault below, planted in the fp64 restatement, breaks the bound it should break by the factor given
(largest error / bound on long_tracks at lambda 1e-4, constants as calibrated; ELIM_FAULTS / BACKSUB_FAULTS):

  one landmark's term dropped (a 13-observer one)            2.4e9     S
  V~ undamped                                                 2.4e7     S, g~
  lambda * nu in place of lambda                              2.4e7     S, g~
  one off-diagonal block transposed                           1.8e8     S
  the pairs in chunk slots >= 80 of a 13-observer landmark    1.3e9     S (a lost second pass of ba_schur_chunks_kernel)
  Y = W V~^-1 formed in float32                               4.0e3     S, g~
  one edge's W_kj replaced by its neighbour's                 1.9e5     S
  back-substitution: one camera's x dropped                   1.9e9     p_new
  back-substitution: one edge's W'x negated                   3.3e8     p_new
  V~^-1 at a stale lambda (lambda * nu)                       9.6e9     V~^-1, p_new
"""
import functools

import numpy as np
import pytest

import oracle
import ba_elim as E  # (tests/ is on sys.path under pytest's rootdir conftest)
import ba_graphs

LAMS = (1e-8, 1e-4, 1e4)
RATIOS = dict(S=0.98, G=0.96, P=1.0, V=3.3)


@functools.lru_cache(maxsize=None)
def graph(name):
    if name in ba_graphs.EDGES:
        pb, delta = ba_graphs.EDGES[name]()
    else:
        c = ba_graphs.build(name)
        pb, delta = c.pb, c.delta
    return pb, delta, oracle.ba_linearize(pb, delta)


CALIBRATION = list(ba_graphs.CASES) + list(ba_graphs.EDGES)


@functools.lru_cache(maxsize=None)
def reference(name, lam, mode=None, into_u=False):
    pb, _, lin = graph(name)
    return E.Elim(pb, lin, lam, mode, into_u)


def step(pb, seed=1):
    """A camera step of the size an LM step takes (zero at fixed dofs)."""
    x = 1e-2 * np.random.default_rng(seed).standard_normal(6 * pb.n_cams)
    return np.where(E.dof_mask(pb.cam_dof), x, 0.0)


def unit():
    """Factors that turn a ratio to the calibrated bound into the ratio with the constant at 1."""
    return dict(S=E.C_S, G=E.C_G, P=E.C_P, V=E.C_V)


@pytest.mark.skipif(not E.EXTENDED, reason="numpy's long double is fp64 here: only the double-double arithmetic exists")
@pytest.mark.parametrize("name", ["long_tracks", "sparse_landmarks", "far_landmarks", "narrow_baseline"])
@pytest.mark.parametrize("lam", [1e-8, 1e4])
def test_long_double_and_double_double_agree(name, lam):
    pb, _, lin = graph(name)
    ld, dd = reference(name, lam, "ld"), reference(name, lam, "dd")

    def gap(a, b):  # |long double - double-double|, taken in long double
        return np.abs(np.asarray(a - (b.hi.astype(E.XP) + b.lo.astype(E.XP)), np.float64))

    x = step(pb)
    assert E.Elim.ratio(gap(ld.S, dd.S), ld.S_bound) <= 0.01
    assert E.Elim.ratio(gap(ld.gt, dd.gt), ld.gt_bound) <= 0.01
    assert E.Elim.ratio(np.linalg.norm(gap(ld.X, dd.X), 2, axis=(1, 2)), ld.X_bound) <= 0.01
    pl, bl = ld.candidate(x, pb.points)
    pd, _ = dd.candidate(x, pb.points)
    assert E.Elim.ratio(gap(pl, pd), bl) <= 0.01


@pytest.mark.parametrize("name", list(ba_graphs.CASES))
@pytest.mark.parametrize("lam", LAMS)
def test_oracle_is_within_the_bounds(name, lam):
    """The oracle's damped S0 and g~0, from its own linearisation: off the diagonal against the bounds; on it against the reference
    plus lm_damp, with the damped diagonal in place of |U_i| in the bound (the oracle damps before it subtracts); fixed dofs carry the
    unit diagonal."""
    pb, delta, lin = graph(name)
    ref = reference(name, lam, into_u=True)
    S0, gt0, _, _ = oracle.ba_reduced_system(pb, delta, lam, 1, 1e-10)
    free = E.dof_mask(pb.cam_dof)
    n6 = 6 * pb.n_cams
    d = np.arange(n6)
    damp = lam * np.clip(ref.diagU, 1e-6, 1e32)
    assert np.all(S0[d[~free], d[~free]] == 1.0)
    dS = S0[d, d].copy()
    S0[d, d] = 0.0
    Sb = ref.s_blocks(S0)
    ii = (ref.blocks[:, 0] == ref.blocks[:, 1])
    bound = ref.S_bound.copy()
    diag_ref = np.zeros(n6)
    Sref = ref.A.f64(ref.S)
    for b in np.nonzero(ii)[0]:
        c = ref.blocks[b, 0]
        diag_ref[6 * c:6 * c + 6] = np.diagonal(Sref[b])
        bound[b][np.arange(6), np.arange(6)] = np.inf          # (the diagonal is checked below)
    assert E.Elim.ratio(ref.A.diff(Sb, ref.S), bound) <= 1.0
    err = np.abs(dS - (diag_ref + damp))[free]
    # (the bound's n |U_i| term, with the damped diagonal in place of U_ii)
    n_terms = np.repeat(np.maximum(np.bincount(pb.obs_cam[ref.active[pb.obs_point]], minlength=pb.n_cams), 1), 6)
    allowed = np.concatenate([np.diagonal(b) for b in ref.S_bound[ii]])[free] + (E.C_S * E.U_RND * n_terms * np.abs(dS))[free]
    assert np.all(err <= allowed), (err / allowed).max()
    assert ref.gt_ratio(gt0) <= 1.0


def _calibration_ratios():
    got = dict(S=0.0, G=0.0, P=0.0, V=0.0)
    c = unit()
    for name in CALIBRATION:
        pb, _, lin = graph(name)
        for lam in LAMS:
            for order in ("forward", "reversed", "shuffled", "into_u"):
                ref = reference(name, lam, into_u=order == "into_u")
                for inv in ("chol", "inv"):
                    r = E.eliminate_fp64(pb, lin, lam, order, inv)
                    got["S"] = max(got["S"], c["S"] * ref.s_ratio(ref.s_blocks(r["S"])))
                    got["G"] = max(got["G"], c["G"] * ref.gt_ratio(r["gt"]))
                    got["V"] = max(got["V"], c["V"] * ref.vinv_ratio(r["X"]))
                    if order == "forward":
                        x = step(pb)
                        got["P"] = max(got["P"], c["P"] * ref.cand_ratio(E.candidate_fp64(pb, lin, r["X"], x, pb.points), x, pb.points))
    return got


def test_calibration():
    got = _calibration_ratios()
    for k, v in got.items():
        assert v <= RATIOS[k], (k, v, RATIOS[k])
    assert tuple(unit()[k] for k in "SGPV") == tuple(8 * RATIOS[k] for k in "SGPV")


# ---- sensitivity: the bounds reject each fault ----------------------------------------------------------------------------------------
def _long_track(pb, n):
    cnt = np.bincount(pb.obs_point, minlength=pb.n_points)
    return int(np.nonzero((cnt == n) & (pb.point_free != 0))[0][0])


def _fault_arg(name, pb):
    if name in ("drop_landmark", "lost_pass"):
        return _long_track(pb, 13)
    if name == "transpose_block":
        j = _long_track(pb, 13)
        cams = np.sort(pb.obs_cam[pb.obs_point == j])
        return int(cams[3]), int(cams[8])        # (two free cameras: the block is not zero)
    if name == "neighbour_w":
        j = _long_track(pb, 13)
        return int(np.nonzero(pb.obs_point == j)[0][3])
    return None


# fault -> largest error / bound it produces on long_tracks at lambda 1e-4, as recorded above (each must stay above half of it)
ELIM_FAULTS = dict(drop_landmark=2.4e9, undamped=2.4e7, lambda_nu=2.4e7, transpose_block=1.8e8, lost_pass=1.3e9, y_float32=4.0e3,
                   neighbour_w=1.9e5)
BACKSUB_FAULTS = dict(drop_camera=1.9e9, negate_edge=3.3e8, stale_lambda=9.6e9)


def elim_fault_factor(fault):
    pb, _, lin = graph("long_tracks")
    lam = 1e-4
    ref = reference("long_tracks", lam)
    r = E.eliminate_fp64(pb, lin, lam, fault=(fault, _fault_arg(fault, pb)))
    return max(ref.s_ratio(ref.s_blocks(r["S"])), ref.gt_ratio(r["gt"]))


def backsub_fault_factor(fault):
    pb, _, lin = graph("long_tracks")
    lam = 1e-4
    ref = reference("long_tracks", lam)
    x = step(pb)
    if fault == "stale_lambda":
        X = E.spd_inverse3_fp64(E.damped_V(lin["V"], lam * 2.0))[0]
        X[~ref.active] = 0.0
        return max(ref.vinv_ratio(X), ref.cand_ratio(E.candidate_fp64(pb, lin, X, x, pb.points), x, pb.points))
    arg = int(pb.obs_cam[pb.obs_point == _long_track(pb, 13)][4]) if fault == "drop_camera" else int(np.nonzero(pb.obs_point == _long_track(pb, 13))[0][2])
    return ref.cand_ratio(E.candidate_fp64(pb, lin, ref.X64, x, pb.points, fault=(fault, arg)), x, pb.points)


@pytest.mark.parametrize("fault", list(ELIM_FAULTS))
def test_elimination_bounds_reject(fault):
    f = elim_fault_factor(fault)
    assert f > 1.0, (fault, f)
    assert f >= 0.5 * ELIM_FAULTS[fault], (fault, f, ELIM_FAULTS[fault])


@pytest.mark.parametrize("fault", list(BACKSUB_FAULTS))
def test_back_substitution_bounds_reject(fault):
    f = backsub_fault_factor(fault)
    assert f > 1.0, (fault, f)
    assert f >= 0.5 * BACKSUB_FAULTS[fault], (fault, f, BACKSUB_FAULTS[fault])
