"""The extended-precision restatement of the reduced camera system's solve (tests/ba_linsys.py), pinned on the CPU against scipy and
against the fp64 oracle's PCG (oracle/ba_ref.c ba_pcg), on the systems oracle.ba_reduced_system forms for tests/ba_graphs.py and
the test_ba_gpu problems.  The device contracts of tests/test_ba_linear_solvers_gpu.py take their bounds from what is recorded here.

Calibration (x86-64 long double), relative A-norm error of the fp64 oracle PCG over that of the extended-precision PCG at the same
iteration k, tolerance 0 (every iteration runs):
  k = 1, 2, 5, 20, 50 while the exact process is above the fp64 floor (a_err_floor = 16 n eps sqrt(kappa)): 1.0000 on every system
  (isolated_cameras, kappa 6.5e11: 1.0196 at k = 50, the largest);
  below the floor the oracle stagnates at rounding level: 1.7e-15 (config1_10cam_200pt, k = 50, exact 5.5e-19; floor 8.7e-11),
  1.6e-15 (tiny, k = 20, exact 8.3e-16; floor 6.4e-11).
  Hence the device bounds: within a factor 2 of the exact process above the floor, below max(2 x exact, floor) once it is there.
Iterations to a relative tolerance (stopping test r'z < tol^2 r0'z0): equal at 1e-4 on every system; at 1e-6 equal except
measurement_forms (oracle 120, exact 119); at 1e-8 one apart on local_50kf (168 / 169), local_70kf (282 / 283) and
sparse_landmarks (108 / 107).  The true preconditioned residual ratio at the oracle's returned x is at most 0.96 tol.
"""
import fractions

import numpy as np
import pytest
import scipy.linalg

import oracle
from gslam_b200 import synth
import ba_graphs  # (tests/ is on sys.path under pytest's rootdir conftest)
import ba_linsys as L
from test_ba_gpu import PROBLEMS

CAPS = (1, 2, 5, 20, 50)
SYSTEMS = [f"graphs:{n}" for n in ba_graphs.CASES] + [f"problems:{n}" for n in PROBLEMS]


def _problem(key):
    kind, name = key.split(":")
    if kind == "graphs":
        c = ba_graphs.build(name)
        return c.pb, c.delta
    return synth.synth_ba(**PROBLEMS[name]), 0.01


def test_extended_residual_is_exact_to_the_last_bit():
    """The residual b - A x that refines x* and judges every solution, against exact rational arithmetic."""
    rng = np.random.default_rng(1)
    n = 12
    A = rng.standard_normal((n, n)) * np.exp(rng.uniform(-20, 20, (n, n)))
    x = rng.standard_normal(n)
    ref = L.Reference(np.eye(6), np.ones(6))
    ref.A, ref.Ax, ref.n = A, A.astype(L.XP) if L.EXTENDED else None, n
    got = ref.mv(x)
    for i in range(n):
        exact = sum(fractions.Fraction(float(A[i, j])) * fractions.Fraction(float(x[j])) for j in range(n))
        scale = sum(abs(fractions.Fraction(float(A[i, j])) * fractions.Fraction(float(x[j]))) for j in range(n))
        assert abs(fractions.Fraction(float(got[i])) - exact) <= scale * fractions.Fraction(1, 2 ** 60) + abs(exact) * fractions.Fraction(1, 2 ** 52)


def test_damping_rule():
    S = np.arange(144, dtype=float).reshape(12, 12)
    dU = np.array([0.0, 1e-9, 2.0, 3.0, 1e40, 5.0, 6.0, 7.0, 8.0, 9.0, 10.0, 11.0])
    dof = np.array([0b111111, 0b000101], np.uint8)
    A = L.damped(S, dU, 0.5, dof)
    d = np.diag(A)
    assert d[0] == S[0, 0] + 0.5e-6 and d[1] == S[1, 1] + 0.5e-6 and d[4] == S[4, 4] + 0.5e32 and d[2] == S[2, 2] + 1.0
    assert d[6] == S[6, 6] + 3.0 and d[7] == 1.0 and d[8] == S[8, 8] + 4.0 and d[9] == 1.0 and d[10] == 1.0 and d[11] == 1.0
    off = ~np.eye(12, dtype=bool)
    assert np.array_equal(A[off], S[off])


@pytest.mark.parametrize("key", SYSTEMS)
def test_reference_pins_against_scipy_and_the_oracle(key):
    pb, delta = _problem(key)
    S0, gt0, _, _ = oracle.ba_reduced_system(pb, delta, 1e-4, 1, 0.0)   # (the oracle's S is damped: lambda 1e-4)
    ref = L.Reference(S0, gt0)
    # x* against scipy's solve, at kappa * eps
    xs = scipy.linalg.solve(S0, gt0, assume_a="pos")
    assert ref.forward_err(xs) <= ref.kappa * L.EPS, (ref.forward_err(xs), ref.kappa)
    assert ref.backward_err(ref.xstar.astype(np.float64)) <= 2 * L.EPS
    # the oracle's fp64 PCG against the extended-precision one, iterate by cap (see the calibration above)
    _, _, _, errs = ref.pcg(max(CAPS), 0.0, errs_at=CAPS)
    floor = L.a_err_floor(ref)
    for k in CAPS:
        dc, it = oracle.ba_reduced_system(pb, delta, 1e-4, k, 0.0)[2:]
        e = ref.a_err(dc)
        if errs[k] > floor:
            assert it == k and 0.5 <= e / errs[k] <= 2.0, (k, e, errs[k])
        else:
            assert e <= max(2 * errs[k], floor), (k, e, errs[k], floor)
    # iteration counts and where the oracle stops
    for tol, slack in ((1e-4, 0), (1e-6, 1)):   # (1e-6: measurement_forms stops one apart, 120 / 119)
        dc, it = oracle.ba_reduced_system(pb, delta, 1e-4, 2000, tol)[2:]
        kx, _, ratios, _ = ref.pcg(2000, tol)
        assert abs(it - kx) <= slack, (tol, it, kx)
        assert ref.res_ratio(dc) <= 1.1 * tol + L.res_floor(ref), (tol, ref.res_ratio(dc))
        assert min(ratios[:max(it - 1, 1)]) >= 0.9 * tol, (tol, it)


def test_new_graphs_have_the_shape_they_are_built_for():
    pb = L.zero_rhs()
    S, gt, dc, it = oracle.ba_reduced_system(pb, 0.01, 1e-4, 50, 1e-10)
    assert np.all(gt == 0.0) and np.abs(S).max() > 1.0 and it == 0 and np.all(dc == 0.0) and oracle.ba_cost(pb) == 0.0
    pb = L.loop_closure()
    assert np.all(L.skyline(pb) == 0)
    pb = L.narrow_band_100()
    assert pb.n_cams > 85 and L.skyline_blocks(pb) == 2 * pb.n_cams - 1
    optin = 232448  # (H100 opt-in shared memory per block, 227 KB; the GPU test reads the device's own)
    a, b = L.skyline_at(optin, False), L.skyline_at(optin, True)
    assert L.chol_fits(L.skyline_blocks(a), a.n_cams, optin) and not L.chol_fits(L.skyline_blocks(b), b.n_cams, optin)
    assert L.skyline_blocks(b) == L.skyline_blocks(a) + 1 and a.n_cams == b.n_cams
    pb = L.mixed_scales()
    t = np.abs(pb.cam_pose_wc[:, 4:]).max(axis=1)
    assert t[:15].max() < 0.1 and t[15:].min() > 999.0
