"""The Levenberg-Marquardt control of every BA solver path against oracle/ba_ref.c, on the cases of tests/_lm_cases.py whose decisions
do not depend on summation order: the overflow stop of the exact zero-cost graphs, reject / accept traces compared iteration by
iteration, the lambda floor, function-tolerance stops, zero iterations, repeated solves and the option checks.

Every test asserts the path bits it covers (BAGraph.paths() / gb_dbg_ba_last_paths).  Every case runs with function_tolerance = 0
(the host never polls: iterations after a stop must change nothing) and with function_tolerance > 0 (the host polls and stops); the
second must launch exactly what a solve capped at the stopping iteration launches."""
import ctypes as C

import numpy as np
import pytest

import oracle
from gslam_b200 import capi
from gslam_b200.api import BAGraph, GbError, OptimzeConfig, Optimizer, ShardedBAGraph, local_group
import _lm_cases as L
from test_ba_sharded_gpu import on_ranks

pytestmark = pytest.mark.gpu
B = BAGraph
SMALL_PATHS = ["local_pcg", "local_direct", "dense_generic", "dense_cluster", "sweep_large", "cam_split3", "host_cold", "host_cached",
               "shard2", "shard3"]
LARGE_PATHS = ["bcsr_cluster", "bcsr_grid", "shard2"]
NO_POLL_CAP = 20  # max_iterations of the function_tolerance = 0 runs of a case that stops earlier


def dcfg(o):
    return OptimzeConfig(projectErrorHuberThreshold=o.get("huber_delta", 0.01), maxIterations=o["max_iterations"],
                         functionTolerance=o.get("function_tolerance", 0.0), lambdaInit=o.get("lambda_init", 1e-4),
                         pcgMaxIterations=o.get("pcg_max_iters", 50), pcgTolerance=o.get("pcg_tol", 1e-10),
                         linearSolver=o.get("linear_solver", 0))


def expect_paths(path, p):
    if path in ("local_pcg", "host_cold", "host_cached"):
        assert p & B.LOCAL4 and p & B.PCG_SPARSE and not p & (B.PCG_BCSR | B.SWEEP_LARGE | B.CAM_SPLIT), p
    elif path == "local_direct":
        assert p & B.LOCAL4 and p & B.CHOL_OK, p
    elif path == "dense_generic":
        assert not p & (B.LOCAL4 | B.PCG_SPARSE | B.PCG_CLUSTER | B.PCG_BCSR), p
    elif path == "dense_cluster":
        assert p & B.PCG_CLUSTER and not p & (B.LOCAL4 | B.PCG_SPARSE | B.PCG_BCSR), p
    elif path == "sweep_large":
        assert p & B.LOCAL4 and p & B.SWEEP_LARGE, p
    elif path == "cam_split3":
        assert p & B.LOCAL4 and p & B.CAM_SPLIT, p
    elif path == "bcsr_cluster":
        assert p & B.PCG_BCSR and p & B.BCSR_CLUSTER and p & B.SCHUR_CHUNKS and p & B.SWEEP_LARGE and not p & B.LOCAL4, p
    elif path == "bcsr_grid":
        assert p & B.PCG_BCSR and not p & B.BCSR_CLUSTER and not p & B.LOCAL4, p
    elif path.startswith("shard"):
        assert p & B.PCG_BCSR, p
    else:
        raise KeyError(path)


class Runner:
    """One graph on one path: solve(opts) -> (result, T_wc poses, points, launches of the solve); reset(); paths checked on entry."""

    def __init__(self, ctx, path, pb, monkeypatch):
        self.ctx, self.path, self.pb = ctx, path, pb
        self.g = None
        if path == "bcsr_grid":
            monkeypatch.setenv("GB_BA_NO_PCG_CLUSTER", "1")
        if path == "host_cold":
            monkeypatch.setenv("GB_BA_NO_CACHE", "1")
        if path.startswith("shard"):
            world = int(path[5:])
            self.ctxs, self.comms = local_group(ctx, world)
            self.gs = on_ranks(world, lambda r: ShardedBAGraph(self.comms[r], pb))
            for g in self.gs:
                expect_paths(path, g.paths())
        elif path.startswith("host"):
            self.est = pb.copy()
        else:
            self.g = BAGraph(ctx, pb)
            if path == "dense_generic":
                self.g.force_generic_pcg(1)
            elif path == "dense_cluster":
                self.g.force_generic_pcg(2)
            elif path == "sweep_large":
                self.g.set_sweep(2)
            elif path == "cam_split3":
                self.g.set_cam_split(3)
            expect_paths(path, self.g.paths())

    def close(self):
        if self.path.startswith("shard"):
            for g in self.gs:
                g.close()
            for m in self.comms:
                m.close()
            for c in self.ctxs[1:]:
                c.close()
        elif self.g is not None:
            self.g.close()

    def reset(self):
        if self.path.startswith("shard"):
            for g in self.gs:
                g.reset()
        elif self.path.startswith("host"):
            self.est = self.pb.copy()
        else:
            self.g.reset()

    def launches(self):
        # (the loopback all-reduce is launched by whichever rank arrives last: count every rank's context)
        return sum(c.launch_count() for c in self.ctxs) if self.path.startswith("shard") else self.ctx.launch_count()

    def solve(self, o):
        c = dcfg(o)
        n0 = self.launches()
        if self.path.startswith("shard"):
            def rank(r):
                res = self.gs[r].solve(c)
                return res, self.gs[r].download()
            out = on_ranks(len(self.gs), rank)
            res = out[0][0]
            for r, (rr, _) in enumerate(out):   # every rank reports the all-reduced scalars
                assert (rr.iterations, rr.accepted, rr.status, rr.lambda_final, rr.initial_cost, rr.final_cost) == \
                       (res.iterations, res.accepted, res.status, res.lambda_final, res.initial_cost, res.final_cost), r
            poses = out[0][1][0]
            pts = np.concatenate([out[r][1][1] for r in range(len(self.gs))], axis=0)
            return res, poses, pts, self.launches() - n0
        if self.path.startswith("host"):
            if self.path == "host_cached":  # a first call of the same topology fills the cache
                self.ctx.ba_solve(self.pb.copy(), dcfg(dict(o, max_iterations=1)))
                n0 = self.ctx.launch_count()
            q = self.est
            res = self.ctx.ba_solve(q, c)
            expect_paths(self.path, self.ctx._lib.gb_dbg_ba_last_paths(self.ctx.handle))
            return res, q.cam_pose_wc.copy(), q.points.copy(), self.ctx.launch_count() - n0
        res = self.g.solve(c)
        n = self.ctx.launch_count() - n0
        poses, pts = self.g.download()
        return res, poses, pts, n


@pytest.fixture
def runner(ctx, monkeypatch):
    made = []

    def make(path, pb):
        r = Runner(ctx, path, pb, monkeypatch)
        made.append(r)
        return r
    yield make
    for r in made:
        r.close()


def scalars(r):
    return (r.iterations, r.accepted, r.status, r.lambda_final)


# ---- the exact zero-cost graphs: 12 rejects, status 2, lambda_init * 2^78, nothing moves ------------------------------------------
def check_overflow(res, poses, pts, pb):
    assert scalars(res) == (L.REJECTS_TO_OVERFLOW, 0, 2, 1e-4 * 2.0 ** 78), scalars(res)
    assert res.initial_cost == 0.0 and res.final_cost == 0.0
    assert np.array_equal(poses, pb.cam_pose_wc) and np.array_equal(pts, pb.points)


@pytest.mark.parametrize("large,path", [(False, p) for p in SMALL_PATHS] + [(True, p) for p in LARGE_PATHS])
def test_exact_graph_overflows_lambda(runner, large, path):
    pb = L.exact_large() if large else L.exact_local()
    ls = 1 if path == "local_direct" else 0
    run = runner(path, pb)
    for ftol, cap in ((0.0, NO_POLL_CAP), (1e-6, NO_POLL_CAP), (1e-6, L.REJECTS_TO_OVERFLOW)):
        run.reset()
        res, poses, pts, n = run.solve(dict(max_iterations=cap, function_tolerance=ftol, linear_solver=ls))
        check_overflow(res, poses, pts, pb)
        if ftol > 0 and cap == NO_POLL_CAP:
            n_stop = n
    assert n_stop == n   # the polling host stopped at the overflow


def test_exact_posegraph_overflows_lambda(ctx):
    pb, edges = L.exact_posegraph()
    g = BAGraph(ctx, pb, edges)
    p = g.paths()
    g.close()
    assert not p & (B.LOCAL4 | B.PCG_SPARSE | B.PCG_BCSR), p
    for ftol in (0.0, 1e-6):
        q = pb.copy()
        res = ctx.ba_solve_posegraph(q, edges, dcfg(dict(max_iterations=NO_POLL_CAP, function_tolerance=ftol)))
        check_overflow(res, q.cam_pose_wc, q.points, pb)


def test_exact_pnp_overflows_lambda(ctx):
    xyz, xy1, pose = L.exact_pnp()
    _, _, info0 = oracle.ba_pnp(xyz, xy1, pose, want_info=True, max_iterations=0)
    for ftol in (0.0, 1e-6):
        out, res, info = ctx.ba_pnp(xyz, xy1, pose, want_info=True, cfg=dcfg(dict(max_iterations=NO_POLL_CAP, function_tolerance=ftol)))
        assert ctx._lib.gb_dbg_ba_last_paths(ctx.handle) & B.LOCAL4
        check_overflow(res, out[None], xyz, type("P", (), dict(cam_pose_wc=pose[None], points=xyz)))
        assert np.abs(info - info0).max() <= 1e-12 * np.abs(info0).max()


# ---- reject / accept traces, iteration by iteration -----------------------------------------------------------------------------
def oracle_run(pb, o):
    q = pb.copy()
    r = oracle.ba_solve(q, **o)
    return r, q


@pytest.mark.parametrize("path", SMALL_PATHS)
@pytest.mark.parametrize("name", list(L.TRACES))
def test_trace_matches_oracle_iteration_by_iteration(runner, name, path):
    pb, opts, iters = L.trace_case(name)
    ls = 1 if path == "local_direct" else 0
    run = runner(path, pb)
    for k in range(1, iters + 1):
        o = dict(opts, max_iterations=k, function_tolerance=0.0, linear_solver=ls)
        r0, want = oracle_run(pb, o)
        run.reset()
        r1, poses, pts, _ = run.solve(o)
        assert scalars(r1) == scalars(r0), (k, scalars(r1), scalars(r0))
        assert abs(r1.initial_cost - r0.initial_cost) <= 1e-12 * r0.initial_cost
        assert abs(r1.final_cost - r0.final_cost) <= 1e-6 * r0.final_cost, (k, r1.final_cost, r0.final_cost)
    if name == "floor":
        assert r1.lambda_final == L.LAMBDA_FLOOR
        assert abs(r1.final_cost - r0.final_cost) <= 1e-9 * r0.final_cost
        assert np.abs(pts - want.points).max() <= 1e-5 * np.abs(want.points).max()
        assert np.abs(poses[:, 4:] - want.cam_pose_wc[:, 4:]).max() <= 1e-5 * np.abs(want.cam_pose_wc[:, 4:]).max()


@pytest.mark.parametrize("path", SMALL_PATHS)
@pytest.mark.parametrize("name", list(L.TRACES))
def test_function_tolerance_stops_match_oracle(runner, name, path):
    pb, opts, iters = L.trace_case(name)
    ls = 1 if path == "local_direct" else 0
    run = runner(path, pb)
    # the stops of the oracle's run (tests/test_oracle_lm.py::test_function_tolerance_stops pins them)
    stops = []
    for n in range(1, iters + 1):
        r0, _ = oracle_run(pb, dict(opts, max_iterations=n, function_tolerance=0.0, linear_solver=ls))
        stops.append(r0)
    acc = [k for k in range(iters) if stops[k].accepted > (stops[k - 1].accepted if k else 0)]
    before = [stops[k - 1].final_cost if k else stops[0].initial_cost for k in acc]
    rels = [(c - stops[k].final_cost) / c for c, k in zip(before, acc)]
    checked = 0
    for m in range(1, len(acc) + 1):
        ftol = L.ftol_between(rels, m)
        if ftol is None:
            continue
        it = acc[m - 1] + 1
        r0, _ = oracle_run(pb, dict(opts, max_iterations=iters + 4, function_tolerance=ftol, linear_solver=ls))
        assert (r0.status, r0.accepted, r0.iterations) == (1, m, it)
        run.reset()
        r1, p1, x1, n_stop = run.solve(dict(opts, max_iterations=iters + 4, function_tolerance=ftol, linear_solver=ls))
        assert scalars(r1) == scalars(r0), (ftol, scalars(r1), scalars(r0))
        assert abs(r1.final_cost - r0.final_cost) <= 1e-6 * r0.final_cost
        run.reset()
        r2, p2, x2, n_cap = run.solve(dict(opts, max_iterations=it, function_tolerance=ftol, linear_solver=ls))
        assert n_stop == n_cap and scalars(r2) == scalars(r1)            # the polling host stopped at the stop
        assert r2.final_cost == r1.final_cost and np.array_equal(x1, x2) and np.array_equal(p1, p2)
        checked += 1
    assert checked >= 1


# ---- zero iterations ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", SMALL_PATHS + ["stepwise"])
def test_zero_iterations_report_the_input_cost(runner, path):
    name = "aa_rrrrrrr_aaa"
    pb, opts, _ = L.trace_case(name)
    o = dict(opts, max_iterations=0, function_tolerance=0.0, linear_solver=1 if path == "local_direct" else 0)
    r0, _ = oracle_run(pb, o)
    assert r0.initial_cost > 0
    run = runner("local_pcg" if path == "stepwise" else path, pb)
    if path == "stepwise":   # the stepwise interface: begin + finish, no LM step in between
        run.g.begin(dcfg(o))
        r1 = run.g.finish()
        poses, pts = run.g.download()
    else:
        r1, poses, pts, _ = run.solve(o)
    assert scalars(r1) == (0, 0, 0, opts["lambda_init"]), scalars(r1)
    assert abs(r1.initial_cost - r0.initial_cost) <= 1e-12 * r0.initial_cost and r1.final_cost == r1.initial_cost
    assert np.array_equal(pts, pb.points)
    assert np.abs(poses - pb.cam_pose_wc).max() <= 1e-13 * max(1.0, np.abs(pb.cam_pose_wc).max())


def test_zero_iterations_large_and_posegraph_and_pnp(ctx, runner):
    pb = L.exact_large()
    run = runner("bcsr_cluster", pb)
    r1, poses, pts, _ = run.solve(dict(max_iterations=0))
    assert scalars(r1) == (0, 0, 0, 1e-4) and r1.initial_cost == 0.0 and r1.final_cost == 0.0
    run = runner("shard2", pb)
    r1, poses, pts, _ = run.solve(dict(max_iterations=0))
    assert scalars(r1) == (0, 0, 0, 1e-4) and r1.initial_cost == 0.0 and np.array_equal(pts, pb.points)
    # (a shard's partial cost would show: the sharded solve of a graph off its optimum)
    tpb, opts, _ = L.trace_case("floor")
    r0, _ = oracle_run(tpb, dict(opts, max_iterations=0))
    run = runner("shard3", tpb)
    r1, _, _, _ = run.solve(dict(opts, max_iterations=0))
    assert abs(r1.initial_cost - r0.initial_cost) <= 1e-12 * r0.initial_cost and r1.final_cost == r1.initial_cost
    # pose graph: the cost of the pose-graph terms counts too
    ppb, edges = L.exact_posegraph()
    q = ppb.copy()
    q.cam_pose_wc[3, 4] += 0.5
    r0 = oracle.ba_solve(q.copy(), edges, max_iterations=0)
    r1 = ctx.ba_solve_posegraph(q, edges, dcfg(dict(max_iterations=0)))
    assert r0.initial_cost > 0 and abs(r1.initial_cost - r0.initial_cost) <= 1e-12 * r0.initial_cost and r1.final_cost == r1.initial_cost
    # optimizePnP: the information matrix is still returned
    tpb, opts, _ = L.trace_case("floor")
    xyz, xy1 = tpb.points[:40], np.concatenate([tpb.gt_points[:40, :2] / 30.0, np.ones((40, 1))], axis=1)
    pose = tpb.cam_pose_wc[3]
    p0, r0, info0 = oracle.ba_pnp(xyz, xy1, pose, want_info=True, max_iterations=0)
    p1, r1, info1 = ctx.ba_pnp(xyz, xy1, pose, want_info=True, cfg=dcfg(dict(max_iterations=0)))
    assert scalars(r1) == (0, 0, 0, 1e-4) and abs(r1.initial_cost - r0.initial_cost) <= 1e-12 * r0.initial_cost
    assert np.abs(p1 - pose).max() <= 1e-14 * 10 and np.abs(info1 - info0).max() <= 1e-10 * np.abs(info0).max()


# ---- a non-finite input cost ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ftol", [0.0, 1e-6])
def test_nonfinite_input_cost(ctx, ftol):
    pb = L.nonfinite_graph()
    g = BAGraph(ctx, pb)
    expect_paths("local_pcg", g.paths())
    g.close()
    from gslam_b200.api import _problem_c
    c, keep = _problem_c(pb)
    o = dcfg(dict(max_iterations=NO_POLL_CAP, function_tolerance=ftol)).to_c()
    res = capi.BaResult()
    rc = ctx._lib.gb_ba_solve(ctx.handle, C.byref(c), C.byref(o), C.byref(res))
    assert rc == capi.GB_ERR_NUMERIC and b"non-finite" in ctx._lib.gb_last_error(ctx.handle)
    assert (res.iterations, res.accepted, res.status) == (L.REJECTS_TO_OVERFLOW, 0, 2)
    assert not np.isfinite(res.initial_cost) and not np.isfinite(res.final_cost)
    assert np.array_equal(pb.points, L.exact_local().points) and np.array_equal(pb.cam_pose_wc, L.exact_local().cam_pose_wc)


# ---- repeated solves --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", [p for p in SMALL_PATHS if not p.startswith("host")])
def test_second_solve_continues_from_the_first(runner, path):
    ls = 1 if path == "local_direct" else 0
    # after an overflow stop: the second solve runs its own full LM from lambda_init
    pb = L.exact_local()
    run = runner(path, pb)
    for _ in range(2):
        res, poses, pts, _ = run.solve(dict(max_iterations=NO_POLL_CAP, function_tolerance=0.0, linear_solver=ls))
        check_overflow(res, poses, pts, pb)
    # after a function-tolerance stop at the first accepted step: the second starts at the first one's estimate and cost
    tpb, opts, iters = L.trace_case("floor")
    run = runner(path, tpb)
    first, p1, x1, _ = run.solve(dict(opts, max_iterations=iters, function_tolerance=10.0, linear_solver=ls))
    assert (first.status, first.accepted, first.iterations) == (1, 1, 1)
    second, p2, x2, _ = run.solve(dict(opts, max_iterations=3, function_tolerance=0.0, linear_solver=ls))
    assert abs(second.initial_cost - first.final_cost) <= 1e-12 * first.final_cost
    q = tpb.copy()
    q.cam_pose_wc[...], q.points[...] = p1, x1
    r0, _ = oracle_run(q, dict(opts, max_iterations=3, function_tolerance=0.0, linear_solver=ls))
    assert scalars(second) == scalars(r0), (scalars(second), scalars(r0))
    assert abs(second.final_cost - r0.final_cost) <= 1e-6 * r0.final_cost
    # reset: the first solve's bits again
    run.reset()
    again, p3, x3, _ = run.solve(dict(opts, max_iterations=iters, function_tolerance=10.0, linear_solver=ls))
    assert scalars(again) == scalars(first) and again.final_cost == first.final_cost
    assert np.array_equal(p3, p1) and np.array_equal(x3, x1)


# ---- option checks ----------------------------------------------------------------------------------------------------------------
INVALID = [("lambdaInit", float("nan")), ("lambdaInit", 0.0), ("lambdaInit", -1e-4), ("lambdaInit", float("inf")),
           ("projectErrorHuberThreshold", float("nan")), ("functionTolerance", float("nan")), ("pcgTolerance", float("nan")),
           ("maxIterations", -1), ("pcgMaxIterations", -1)]


@pytest.mark.parametrize("field,value", INVALID, ids=[f"{f}={v}" for f, v in INVALID])
def test_invalid_options_are_refused(ctx, field, value):
    pb = L.exact_local()
    c = OptimzeConfig()
    setattr(c, field, value)
    g = BAGraph(ctx, pb)
    with pytest.raises(GbError) as e:
        g.solve(c)
    g.close()
    assert e.value.code == capi.GB_ERR_INVALID and "gb_ba:" in str(e.value)
    opt = Optimizer(c)
    q = pb.copy()
    assert opt.optimize(q) is False
    assert np.array_equal(q.points, pb.points)
    opt._ctx.close()
