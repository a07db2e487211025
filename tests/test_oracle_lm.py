"""The Levenberg-Marquardt control of the oracle (oracle/ba_ref.c) on the cases of tests/_lm_cases.py: the closed forms of the exact
zero-cost graphs, the margin of every decision of the reject / accept traces, their accept / reject pattern and lambda against the
independent numpy LM of tests/test_oracle_ba_independent.py, the function-tolerance stops, zero iterations, a non-finite input
cost and the option checks.  These pin the expectations tests/test_lm_paths_gpu.py holds every device path to."""
import ctypes as C
import re

import numpy as np
import pytest

import oracle
from oracle import oracle as O
import _lm_cases as L
from test_oracle_ba_independent import lm_numpy

GB_ERR_INVALID = 1   # (gslam_b200.capi.GB_ERR_INVALID: the two share include/gslam_b200.h)


def exact_solve(kind, **opts):
    """-> (result, input estimate (poses, points), output estimate) of the oracle on an exact zero-cost case"""
    o = dict(max_iterations=50, function_tolerance=0.0)
    o.update(opts)
    if kind == "pnp":
        xyz, xy1, pose = L.exact_pnp()
        out, r, _ = oracle.ba_pnp(xyz, xy1, pose, **o)
        return r, (pose[None], xyz), (out[None], xyz)
    edges = None
    if kind == "posegraph":
        pb, edges = L.exact_posegraph()
    else:
        pb = L.exact_local() if kind == "local" else L.exact_large()
    q = pb.copy()
    r = oracle.ba_solve(q, edges, **o)
    return r, (pb.cam_pose_wc, pb.points), (q.cam_pose_wc, q.points)


@pytest.mark.parametrize("kind", ["local", "large", "posegraph", "pnp"])
def test_exact_graph_rejects_until_lambda_overflows(kind):
    r, (p0, x0), (p1, x1) = exact_solve(kind)
    assert (r.status, r.iterations, r.accepted) == (2, L.REJECTS_TO_OVERFLOW, 0)
    assert r.lambda_final == 1e-4 * 2.0 ** 78
    assert r.initial_cost == 0.0 and r.final_cost == 0.0
    assert np.array_equal(p1, p0) and np.array_equal(x1, x0)   # (the T_wc <-> T_cw round trip is exact for these rotations)


def test_exact_large_graph_has_the_shape_of_the_compact_path():
    pb = L.exact_large()
    cnt = np.bincount(pb.obs_point, minlength=pb.n_points)
    assert int((pb.cam_dof != 0).sum()) > 80 and pb.n_obs >= 65536 and cnt.max() <= 16


def oracle_trace(capfd, pb, opts, iters, **extra):
    """[(cost, candidate cost, accepted)] of every LM decision of the oracle (its verbose lines) and the result"""
    capfd.readouterr()
    o = dict(opts)
    o.update(extra)
    r = oracle.ba_solve(pb.copy(), max_iterations=iters, function_tolerance=o.pop("function_tolerance", 0.0), verbose=1, **o)
    err = capfd.readouterr().err
    rows = [(float(m[0]), float(m[1]), m[2] == "accept") for m in re.findall(r"it \d+ cost (\S+) -> (\S+) lambda \S+ (accept|reject)", err)]
    assert len(rows) == r.iterations
    return rows, r


def pattern(rows):
    return "".join("A" if a else "R" for _, _, a in rows)


@pytest.mark.parametrize("name", list(L.TRACES))
def test_trace_decisions_hold_their_margin(capfd, name):
    pb, opts, iters = L.trace_case(name)
    pats = []
    for solver in (0, 1):   # the same decisions with the PCG and with the direct solver
        rows, r = oracle_trace(capfd, pb, opts, iters, linear_solver=solver)
        assert r.iterations == iters and r.status == 0
        margin = min(abs(c1 - c0) / c0 for c0, c1, _ in rows)
        assert margin >= L.MARGIN, (solver, margin)
        pats.append(pattern(rows))
        assert r.lambda_final == L.lm_replay([a for _, _, a in rows], opts["lambda_init"])[-1]
    assert pats[0] == pats[1], pats
    if name == "floor":
        assert pats[0] == "A" * iters and r.lambda_final == L.LAMBDA_FLOOR
        assert L.lm_replay([True] * 5, opts["lambda_init"])[-1] == L.LAMBDA_FLOOR
    else:   # a streak of >= 2 rejects followed by an accept, and a reject right after an accept
        assert "RRA" in pats[0] and "AR" in pats[0], pats[0]


@pytest.mark.parametrize("name", list(L.TRACES))
def test_trace_equals_independent_lm(name):
    """Accept / reject pattern and lambda after every iteration k = 1 .. N: the oracle stopped after k iterations against the numpy LM
    (a sparse solve of the full damped normal equations: both sides solve exactly)."""
    pb, opts, iters = L.trace_case(name)
    trace, accepted, _, _ = lm_numpy(pb, iters, opts["huber_delta"], opts["lambda_init"])
    from test_oracle_ba_independent import Problem
    costs = [Problem(pb, opts["huber_delta"]).cost()] + list(trace)
    decisions = [costs[k + 1] < costs[k] for k in range(iters)]
    lams = L.lm_replay(decisions, opts["lambda_init"])
    for k in range(1, iters + 1):
        r = oracle.ba_solve(pb.copy(), max_iterations=k, function_tolerance=0.0, linear_solver=1, **opts)
        assert r.iterations == k and r.accepted == sum(decisions[:k]), (k, r.accepted, decisions)
        assert r.lambda_final == lams[k - 1], (k, r.lambda_final, lams[k - 1])
        # (far from the optimum with lambda down to 1e-12 the two exact solves of an ill-conditioned system part in the 4th digit: what
        # is compared exactly is the decisions and lambda, which the margins of test_trace_decisions_hold_their_margin protect)
        assert abs(r.final_cost - costs[k]) <= 1e-3 * costs[k], (k, r.final_cost, costs[k])
    assert accepted == sum(decisions)


def ftol_stops(capfd, name):
    """[(function_tolerance, accepted, iterations)] of every stop the trace allows with margin: always the first accepted step"""
    pb, opts, iters = L.trace_case(name)
    rows, _ = oracle_trace(capfd, pb, opts, iters)
    acc = [k for k, (_, _, a) in enumerate(rows) if a]
    rels = [(rows[k][0] - rows[k][1]) / rows[k][0] for k in acc]
    out = []
    for n in range(1, len(acc) + 1):
        f = L.ftol_between(rels, n)
        if f is not None:
            out.append((f, n, acc[n - 1] + 1))
    return out


@pytest.mark.parametrize("name", list(L.TRACES))
def test_function_tolerance_stops(capfd, name):
    pb, opts, iters = L.trace_case(name)
    stops = ftol_stops(capfd, name)
    assert stops[0][1] == 1 and (name != "floor" or len(stops) >= 2), stops
    for ftol, n, it in stops:
        r = oracle.ba_solve(pb.copy(), max_iterations=iters + 4, function_tolerance=ftol, **opts)
        assert (r.status, r.accepted, r.iterations) == (1, n, it), (ftol, n, it, r.status, r.accepted, r.iterations)


def test_nonfinite_input_cost_rejects_until_lambda_overflows():
    """The oracle states the arithmetic: it returns GB_OK with the non-finite cost in the result (the device API turns that result
    into GB_ERR_NUMERIC)."""
    q = L.nonfinite_graph()
    r = oracle.ba_solve(q, max_iterations=50, function_tolerance=0.0)
    assert (r.status, r.iterations, r.accepted) == (2, L.REJECTS_TO_OVERFLOW, 0)
    assert not np.isfinite(r.initial_cost) and not np.isfinite(r.final_cost)
    assert np.array_equal(q.points, L.exact_local().points)


@pytest.mark.parametrize("name", ["aa_rrrrrrr_aaa", "floor"])
def test_zero_iterations_report_the_input_cost(name):
    pb, opts, _ = L.trace_case(name)
    q = pb.copy()
    r = oracle.ba_solve(q, max_iterations=0, **opts)
    cost = oracle.ba_cost(pb, opts["huber_delta"])
    assert cost > 0 and abs(r.initial_cost - cost) <= 1e-14 * cost and r.final_cost == r.initial_cost
    assert (r.iterations, r.accepted, r.status, r.lambda_final) == (0, 0, 0, opts["lambda_init"])
    assert np.array_equal(q.points, pb.points) and np.abs(q.cam_pose_wc - pb.cam_pose_wc).max() < 1e-13


INVALID = [("lambda_init", float("nan")), ("lambda_init", 0.0), ("lambda_init", -1e-4), ("lambda_init", float("inf")),
           ("huber_delta", float("nan")), ("function_tolerance", float("nan")), ("pcg_tol", float("nan")),
           ("max_iterations", -1), ("pcg_max_iters", -1)]


@pytest.mark.parametrize("field,value", INVALID, ids=[f"{f}={v}" for f, v in INVALID])
def test_invalid_options_are_refused(field, value):
    pb = L.exact_local().copy()
    c, keep = O.ba_problem_c(pb)
    o = O.default_ba_options(**{field: value})
    rc = oracle.lib().orc_ba_solve_ex(C.byref(c), None, C.byref(o), C.byref(O.BaResultC()))
    assert rc == GB_ERR_INVALID
    assert np.array_equal(pb.points, L.exact_local().points)
