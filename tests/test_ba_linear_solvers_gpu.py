"""Every solver of the BA reduced camera system against an extended-precision solve of the system it was given (tests/ba_linsys.py).

gb_dbg_ba_system hands back what one LM step would solve -- the undamped S, g~, diag U and lambda -- and the answer of the solver
that step runs.  The damped matrix A is rebuilt from them on the host, and the answer is judged by what the solver promises, not by
the recurrence it uses:

  fixed dofs     x is exactly 0 at every fixed dof (unit diagonal, zero row and right-hand side: exact in any correct solver)
  capped PCG     (tolerance 0, caps 1, 2, 5, 20, 50) the reported iterations equal the cap, and the relative A-norm error is within a
                 factor 2 of the extended-precision PCG's at the same iteration -- below max(2 x that, the fp64 floor) once the exact
                 process has reached the floor (bounds from the calibration in test_ba_linsys_reference.py)
  converged PCG  (tolerances 1e-4, 1e-6, 1e-8) the true preconditioned residual ratio at x is <= 1.1 tol + kappa eps, and the exact
                 process had not met 0.9 tol two iterations before the reported count
  direct solver  backward error <= 64 n eps, forward error against x* <= 64 n eps kappa_2(A)

Every case first asserts the path bits it means to cover (BAGraph.paths()), the single-CTA PCG's instantiation bits included."""
import functools

import numpy as np
import pytest

from gslam_b200 import synth
from gslam_b200.api import BAGraph, OptimzeConfig
import ba_graphs  # (tests/ is on sys.path under pytest's rootdir conftest)
import ba_linsys as L
from test_ba_gpu import PROBLEMS

pytestmark = pytest.mark.gpu
B = BAGraph
CAPS = (1, 2, 5, 20, 50)
TOLS = (1e-4, 1e-6, 1e-8)


def cfg(**kw):
    c = OptimzeConfig()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _optin():
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


@functools.lru_cache(maxsize=None)
def graph(name):
    """(problem, Huber delta) of a named graph."""
    if name in PROBLEMS:
        return synth.synth_ba(**PROBLEMS[name]), 0.01
    if name in ba_graphs.CASES:
        c = ba_graphs.build(name)
        return c.pb, c.delta
    if name == "wide_landmarks_large":
        c = ba_graphs.build("wide_landmarks", True)
        return c.pb, c.delta
    if name == "sparse_over_80_cams":
        return ba_graphs.sparse_over_80_cams(), 0.01
    if name == "bcsr_100cams":
        return synth.synth_ba(100, 3000, obs_per_point=3, n_fixed=2, seed=171), 0.01
    if name.startswith("skyline_"):
        return L.skyline_at(_optin(), name == "skyline_over"), 0.01
    return getattr(L, name)(), 0.01


# path -> (force_generic_pcg mode, linear solver, bits that must be set, bits that must be clear)
SP, SM, LR = B.PCG_SPARSE, B.SPARSE_SMALL, B.SPARSE_LONG_ROWS
PATHS = {
    "sparse_small": (0, 0, SP | SM, LR | B.PCG_BCSR),
    "sparse_small_long": (0, 0, SP | SM | LR, B.PCG_BCSR),
    "sparse_large": (0, 0, SP, SM | LR | B.PCG_BCSR),
    "sparse_large_long": (0, 0, SP | LR, SM | B.PCG_BCSR),
    "cluster16": (2, 0, B.PCG_CLUSTER, SP | SM | LR | B.PCG_BCSR),
    "cluster8": (4, 0, B.PCG_CLUSTER, SP | SM | LR | B.PCG_BCSR),
    "generic": (1, 0, 0, SP | SM | LR | B.PCG_CLUSTER | B.PCG_BCSR),
    "bcsr_cluster": (0, 0, B.PCG_BCSR | B.BCSR_CLUSTER, SP | B.LOCAL4),
    "bcsr_grid": (0, 0, B.PCG_BCSR, B.BCSR_CLUSTER | SP | B.LOCAL4),
    "direct": (0, 1, B.CHOL_OK, 0),
}
CLUSTER_SIZE = {"cluster16": 16, "cluster8": 8}

# (path, graph, lambda)
PCG_CASES = [
    ("sparse_small", "scattered_fixed", 1e-4), ("sparse_small_long", "config1_10cam_200pt", 1e-4), ("sparse_small", "tiny", 1e-4),
    ("sparse_small", "one_active", 1e-4), ("sparse_small", "mixed_scales", 1e-4), ("sparse_small", "local_50kf", 1e-4),
    ("sparse_small", "scattered_fixed", 1e4), ("sparse_small", "scattered_fixed", 1e-8),
    ("sparse_small_long", "wide_landmarks", 1e-4), ("sparse_small_long", "wide_band_30kf", 1e-4),
    ("sparse_large", "sparse_over_80_cams", 1e-4),
    ("sparse_large_long", "local_70kf", 1e-4), ("sparse_large_long", "local_70kf", 1e-8),
    ("cluster16", "measurement_forms", 1e-4), ("cluster16", "isolated_cameras", 1e-4), ("cluster16", "mixed_scales", 1e4),
    ("cluster8", "two_components", 1e-4), ("cluster8", "sparse_landmarks", 1e-8),
    ("generic", "isolated_cameras", 1e-4), ("generic", "config1_10cam_200pt", 1e-8), ("generic", "one_active", 1e4),
    ("bcsr_cluster", "bcsr_100cams", 1e-4),
    ("bcsr_grid", "wide_landmarks_large", 1e-4),
]
DIRECT_CASES = [
    ("direct", "scattered_fixed", 1e-4), ("direct", "measurement_forms", 1e-4), ("direct", "mixed_scales", 1e-4),
    ("direct", "one_active", 1e-4), ("direct", "local_50kf", 1e-4), ("direct", "scattered_fixed", 1e4), ("direct", "scattered_fixed", 1e-8),
    ("direct", "loop_closure", 1e-4), ("direct", "narrow_band_100", 1e-4), ("direct", "skyline_fit", 1e-4),
]


def _id(c):
    return f"{c[0]}-{c[1]}-lam{c[2]:g}"


def open_graph(ctx, path, name):
    pb, delta = graph(name)
    g = BAGraph(ctx, pb)
    mode, direct, need, clear = PATHS[path]
    if mode:
        g.force_generic_pcg(mode)
    p = g.paths()
    assert p & need == need and not p & clear, (path, p)
    if path in CLUSTER_SIZE:
        assert g.pcg_cluster_size() == CLUSTER_SIZE[path]
    return g, pb, delta, direct


_REFS = {}


def reference(sysd, pb):
    """Reference of the damped system rebuilt from what the device was given (cached by its bytes: every path of a graph forms the
    same S)."""
    A = L.damped(sysd["S"], sysd["diagU"], sysd["lam"], pb.cam_dof)
    key = (A.tobytes(), sysd["gt"].tobytes())
    if key not in _REFS:
        _REFS.clear()
        _REFS[key] = L.Reference(A, sysd["gt"])
    return _REFS[key]


def check_fixed(x, pb):
    fixed = ~L.dof_mask(pb.cam_dof)
    assert np.all(x[fixed] == 0.0), np.abs(x[fixed]).max()
    assert np.isfinite(x).all()


@pytest.mark.parametrize("case", PCG_CASES, ids=_id)
def test_pcg_contracts(ctx, case):
    path, name, lam = case
    g, pb, delta, _ = open_graph(ctx, path, name)
    opts = dict(projectErrorHuberThreshold=delta, lambdaInit=lam)
    # capped: every iteration runs (tolerance 0)
    ref, errs, floor = None, None, None
    for k in CAPS:
        s = g.dbg_system(cfg(pcgMaxIterations=k, pcgTolerance=0.0, **opts))
        assert s["lam"] == lam
        if ref is None:
            ref = reference(s, pb)
            errs = ref.pcg(max(CAPS), 0.0, errs_at=(0,) + tuple(range(1, max(CAPS) + 1)))[3]
            floor = L.a_err_floor(ref)
        check_fixed(s["x"], pb)
        e = ref.a_err(s["x"])
        if errs.get(k - 1, 0.0) > floor and k in errs:  # (the exact process still makes progress: nothing may stop the loop early)
            assert s["iters"] == k, (k, s["iters"])
        else:
            assert s["iters"] <= k
        exact = errs.get(k, errs[max(errs)])
        if exact > floor:
            assert 0.5 <= e / exact <= 2.0, (k, e, exact)
        else:
            assert e <= max(2 * exact, floor), (k, e, exact, floor)
    # converged: stopped when the rule says so
    for tol in TOLS:
        s = g.dbg_system(cfg(pcgMaxIterations=3000, pcgTolerance=tol, **opts))
        check_fixed(s["x"], pb)
        it = s["iters"]
        assert it < 3000
        rr = ref.res_ratio(s["x"])
        assert rr <= 1.1 * tol + L.res_floor(ref), (tol, rr, it)
        ratios = ref.pcg(it + 2, 0.0)[2]
        assert min(ratios[:max(it - 1, 1)]) >= 0.9 * tol, (tol, it, min(ratios[:max(it - 1, 1)]))
    g.close()


@pytest.mark.parametrize("case", DIRECT_CASES, ids=_id)
def test_direct_solver_contracts(ctx, case):
    path, name, lam = case
    g, pb, delta, _ = open_graph(ctx, path, name)
    s = g.dbg_system(cfg(projectErrorHuberThreshold=delta, lambdaInit=lam, linearSolver=1))
    g.close()
    assert s["iters"] == 0 and s["lam"] == lam
    check_fixed(s["x"], pb)
    ref = reference(s, pb)
    n = ref.n
    assert ref.backward_err(s["x"]) <= 64 * n * L.EPS, ref.backward_err(s["x"])
    assert ref.forward_err(s["x"]) <= 64 * n * L.EPS * ref.kappa, (ref.forward_err(s["x"]), ref.kappa)


@pytest.mark.parametrize("path", ["sparse_small", "cluster16", "cluster8", "generic", "direct"])
def test_zero_right_hand_side(ctx, path):
    """A noise-free graph at its optimum: g~ is exactly 0, so is the step, with no NaN from 0/0 in the first PCG scalars."""
    g, pb, delta, direct = open_graph(ctx, path, "zero_rhs")
    s = g.dbg_system(cfg(pcgMaxIterations=50, pcgTolerance=0.0, linearSolver=direct))
    g.close()
    assert np.all(s["gt"] == 0.0) and np.abs(s["S"]).max() > 1.0
    assert np.all(s["x"] == 0.0) and s["iters"] == 0


def test_damping_restatement_matches_the_device(ctx):
    """damped() is the device's lm_damp: the damped S the single-CTA / one-cluster / generic PCG write back equals it bit for bit."""
    pb, delta = graph("scattered_fixed")
    for mode in (0, 2, 1):
        g = BAGraph(ctx, pb)
        g.force_generic_pcg(mode)
        c = cfg(projectErrorHuberThreshold=delta, lambdaInit=3e-3, pcgMaxIterations=5)
        s = g.dbg_system(c)
        S = g.dbg_reduced(c)[0]
        g.close()
        assert np.array_equal(L.damped(s["S"], s["diagU"], s["lam"], pb.cam_dof), S), mode


def test_direct_solver_skyline_limit(ctx):
    """The largest block skyline that fits one SM's shared memory takes the direct solver; one block more does not (bit 256 of
    paths() flips exactly at ba_chol_plan_host's bound)."""
    optin = _optin()
    for name, fits in (("skyline_fit", True), ("skyline_over", False)):
        pb, _ = graph(name)
        nb = L.skyline_blocks(pb)
        assert L.chol_fits(nb, pb.n_cams, optin) == fits and L.chol_fits(nb + (1 if fits else -1), pb.n_cams, optin) != fits
        g = BAGraph(ctx, pb)
        assert bool(g.paths() & B.CHOL_OK) == fits, (name, nb, g.paths())
        g.close()


def test_every_path_is_covered():
    covered = {c[0] for c in PCG_CASES + DIRECT_CASES}
    assert covered == set(PATHS)
