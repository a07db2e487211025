"""gb_ba_graph_solve and gb_ba_shard_solve are one LM driver: a landmark-sharded solve at world 1 is the single-GPU solve.

A shard of world 1 holds the whole problem, so a ShardedBAGraph on a world-1 communicator and a BAGraph of the same problem must
take the same iterations on the same layout.  For graphs that iterate on the compact block-CSR reduced system, each pair of solves
must give the same bits for every pose and landmark, every BaResult field but gpu_ms, and the same number of kernel launches: with a
fixed iteration count, with none (the cost at the input, which the sharded solve all-reduces), under a function tolerance (the
polling loop, whose verbose line differs only in its tag), and on a graph whose steps are rejected.

The direct solver is the one option that sends such a graph off the compact system: a world-1 shard that asks for it is solved as
gb_ba_graph_solve solves it, by the Cholesky solver on the dense reduced system."""
import contextlib
import functools

import pytest

from gslam_b200 import synth
from gslam_b200.api import BAGraph, Comm, OptimzeConfig, ShardedBAGraph
import ba_graphs  # (tests/ is on sys.path under pytest's rootdir conftest)
import ba_linsys

pytestmark = pytest.mark.gpu
B = BAGraph
RESULT = ("initial_cost", "final_cost", "iterations", "accepted", "pcg_iterations", "status", "lambda_final")


def rejected_steps():
    """ba_graphs.rejected_step's start (20 degree rotation noise, no Huber kernel, lambda 1e-8) on 100 cameras instead of 30: a
    local-BA window has no block-CSR plan, so a shard of it cannot be solved; this one iterates on the compact system."""
    return synth.synth_ba(100, 3000, obs_per_point=4, n_fixed=2, seed=191, pose_sigma_deg=20.0, pose_sigma_t=0.5), 0.0


@functools.lru_cache(maxsize=None)
def problem(name):
    """(problem, Huber delta)"""
    if name == "flagship":   # the sharded solve's test graph (tests/test_ba_sharded_gpu.py)
        return synth.synth_ba(60, 6000, obs_per_point=8, seed=11, n_fixed=2), 0.01
    if name == "rejected_steps":
        return rejected_steps()
    if name == "narrow_band_100":
        return ba_linsys.narrow_band_100(), 0.01
    c = ba_graphs.build(name, True)
    return c.pb, c.delta


MODES = {
    "fixed": dict(maxIterations=4, functionTolerance=0.0),
    "zero": dict(maxIterations=0),
    "poll": dict(maxIterations=50, functionTolerance=1e-6, verbose=True),
}


def opts(delta, **kw):
    c = OptimzeConfig(projectErrorHuberThreshold=delta)
    for k, v in kw.items():
        setattr(c, k, v)
    return c


@contextlib.contextmanager
def world1(ctx):
    comm = Comm(ctx, world=1, rank=0)
    try:
        yield comm
    finally:
        comm.close()


def solve(ctx, g, o):
    n0 = ctx.launch_count()
    r = g.solve(o)
    n = ctx.launch_count() - n0
    pose, pts = g.download()
    return r, pose, pts, n


def both(ctx, pb, o):
    """(paths, BAGraph solve, world-1 ShardedBAGraph solve), each as (result, poses, points, launches)."""
    g = BAGraph(ctx, pb)
    try:
        paths = g.paths()
        single = solve(ctx, g, o)
    finally:
        g.close()
    with world1(ctx) as comm:
        s = ShardedBAGraph(comm, pb)
        try:
            sharded = solve(ctx, s, o)
        finally:
            s.close()
    return paths, single, sharded


def check_same(single, sharded):
    r1, p1, x1, n1 = single
    r2, p2, x2, n2 = sharded
    for f in RESULT:
        assert getattr(r2, f) == getattr(r1, f), (f, getattr(r2, f), getattr(r1, f))
    assert p2.tobytes() == p1.tobytes(), "poses differ"
    assert x2.tobytes() == x1.tobytes(), "landmarks differ"
    assert n2 == n1, ("launches", n2, n1)


COMPACT = ["flagship"] + list(ba_graphs.CASES)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", COMPACT)
def test_world1_shard_is_the_single_gpu_solve(ctx, capfd, name, mode):
    pb, delta = problem(name)
    capfd.readouterr()
    paths, single, sharded = both(ctx, pb, opts(delta, **MODES[mode]))
    assert paths & B.PCG_BCSR and not paths & B.LOCAL4, paths
    check_same(single, sharded)
    r = single[0]
    if mode == "zero":
        assert r.iterations == 0 and r.initial_cost == r.final_cost > 0.0, (r.iterations, r.initial_cost, r.final_cost)
    if mode == "poll":   # one verbose line per iteration from each front end, equal but for the tag
        err = capfd.readouterr().err.splitlines()
        one = [ln[len("[gb_ba] "):] for ln in err if ln.startswith("[gb_ba] it ")]
        shard = [ln[len("[gb_ba x1] "):] for ln in err if ln.startswith("[gb_ba x1] it ")]
        assert len(one) == r.iterations and shard == one, err


def test_world1_shard_rejected_steps(ctx):
    pb, delta = problem("rejected_steps")
    paths, single, sharded = both(ctx, pb, opts(delta, maxIterations=4, functionTolerance=0.0, lambdaInit=1e-8))
    assert paths & B.PCG_BCSR and not paths & B.LOCAL4, paths
    check_same(single, sharded)
    r = single[0]
    assert r.iterations == 4 and r.accepted < r.iterations, (r.iterations, r.accepted)


def test_world1_shard_takes_the_direct_solver(ctx):
    """narrow_band_100: 98 active cameras (more than the single-CTA PCG's 80), so a block-CSR plan, and a skyline that fits the
    direct solver.  With linearSolver = 1 both front ends run the Cholesky solver on the dense system: no PCG iteration, same bits."""
    pb, delta = problem("narrow_band_100")
    paths, single, sharded = both(ctx, pb, opts(delta, maxIterations=4, functionTolerance=0.0, linearSolver=1))
    assert paths & B.PCG_BCSR and paths & B.CHOL_OK and not paths & B.LOCAL4, paths
    check_same(single, sharded)
    assert single[0].iterations == 4 and single[0].pcg_iterations == 0, (single[0].iterations, single[0].pcg_iterations)
    # (with linearSolver = 0 both run the block-CSR PCG on the compact system, which reports its iterations)
    _, single, sharded = both(ctx, pb, opts(delta, maxIterations=4, functionTolerance=0.0))
    check_same(single, sharded)
    assert single[0].pcg_iterations > 0
