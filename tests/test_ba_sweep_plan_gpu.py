"""The item plan of the large-graph sweep (csrc/ba_sweep.cu), checked by what the solves return.

A graph that takes that sweep by size gets its plan when it is created, in its own slab.  gb_dbg_ba_set_cam_split and
gb_dbg_ba_set_sweep re-cut it in place whenever their change leaves the graph on that sweep, and a graph that gb_ba_solve creates and
destroys within the call (GB_BA_NO_CACHE) plans in the ctx's scratch.  Each solve must give the same bytes as a fresh graph set up
the same way: the poses, the points and every BaResult field but gpu_ms."""
import pytest

from gslam_b200 import synth
from gslam_b200.api import BAGraph, Context, OptimzeConfig

pytestmark = pytest.mark.gpu
BA_FIELDS = ("initial_cost", "final_cost", "iterations", "accepted", "pcg_iterations", "status", "lambda_final")
CFG = OptimzeConfig(maxIterations=5, functionTolerance=0.0)


def large():
    """70 000 observations: over the 65 536 from which a graph takes the large-graph sweep by size."""
    return synth.synth_ba(100, 14_000, obs_per_point=5, seed=21)


def small():
    """50 000 observations, and too many landmarks for the local-BA chain: its solves run the sweep the graph is set to."""
    return synth.synth_ba(80, 25_000, obs_per_point=2, seed=22)


@pytest.fixture
def fresh():
    """Context(0) factory; every ctx it made is closed after the test."""
    made = []

    def make():
        made.append(Context(0))
        return made[-1]
    yield make
    for c in made:
        c.close()


def outcome(g):
    """(BaResult fields, pose bytes, point bytes) of a solve of g."""
    r = g.solve(CFG)
    pose, pts = g.download()
    assert r.accepted > 0
    return [getattr(r, k) for k in BA_FIELDS], pose.tobytes(), pts.tobytes()


def fresh_outcome(ctx, pb, split=None, sweep=None):
    g = BAGraph(ctx, pb)
    try:
        if sweep is not None:
            g.set_sweep(sweep)
        if split is not None:
            g.set_cam_split(split)
        return outcome(g)
    finally:
        g.close()


def test_set_cam_split_replans_a_solved_graph(fresh):
    """A large graph solved with the plan it was created with, then re-split 1..4 and solved again from its input each time."""
    pb = large()
    g = BAGraph(fresh(), pb)
    assert g.paths() & BAGraph.SWEEP_LARGE and not g.paths() & BAGraph.CAM_SPLIT
    first = outcome(g)
    ref = fresh()
    for split in (1, 2, 3, 4):
        g.set_cam_split(split)
        assert bool(g.paths() & BAGraph.CAM_SPLIT) == (split > 1)
        g.reset()
        want = fresh_outcome(ref, pb, split=split)
        assert outcome(g) == want
        if split == 1:
            assert first == want
    g.close()


@pytest.mark.parametrize("split", [1, 3])
def test_set_sweep_switches_a_solved_graph(fresh, split):
    """A small graph solved on ba.cu's sweep, then on ba_sweep.cu's (planned for the split it has then), then on the one its size
    picks."""
    pb = small()
    g = BAGraph(fresh(), pb)
    g.set_cam_split(split)
    ref = fresh()
    for sweep in (1, 2, 0):
        g.set_sweep(sweep)
        assert not g.paths() & BAGraph.LOCAL4
        assert bool(g.paths() & BAGraph.SWEEP_LARGE) == (sweep == 2)
        g.reset()
        assert outcome(g) == fresh_outcome(ref, pb, split=split, sweep=sweep)
    g.close()


def test_uncached_solve_plans_in_the_scratch(fresh, monkeypatch):
    """gb_ba_solve of a large graph three times on one ctx with the topology cache off: its graph, plan included, is made in the
    ctx's scratch each time."""
    monkeypatch.setenv("GB_BA_NO_CACHE", "1")
    pb = large()
    want = fresh_outcome(fresh(), pb)
    ctx = fresh()
    for _ in range(3):
        got = pb.copy()
        r = ctx.ba_solve(got, CFG)
        assert ctx._lib.gb_dbg_ba_last_paths(ctx.handle) & BAGraph.SWEEP_LARGE
        assert ([getattr(r, k) for k in BA_FIELDS], got.cam_pose_wc.tobytes(), got.points.tobytes()) == want
