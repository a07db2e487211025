"""Where a BA graph's device memory lives (BaPlace, csrc/ba_internal.cuh), checked by what the solves return.

gb_ba_solve keeps the graph of its last call in the topology cache's own buffer, so the one-shot calls between two solves on a ctx
(gb_pnp_ransac and the gb_ba_pnp nested in it) leave that graph alone.  The graphs that gb_ba_pnp, gb_ba_solve_posegraph and an
uncached gb_ba_solve create and destroy within the call live in the ctx's device scratch, over whatever the previous call left
there.  Each such solve must give the same bytes as the same problem solved as a BAGraph (its own allocation) on a fresh ctx:
the poses, the points and every BaResult field but gpu_ms.  The cases cover the local-BA chain of programmatic dependent launches
(BAGraph.LOCAL4), which reads the graph's structure before it waits for its predecessor, and graphs that grow the scratch."""
import numpy as np
import pytest

from gslam_b200 import synth
from gslam_b200.api import BAGraph, Context, OptimzeConfig
from gslam_b200.synth import BAProblem
import pnp_scenes  # (tests/ is on sys.path under pytest's rootdir conftest)

pytestmark = pytest.mark.gpu
BA_FIELDS = ("initial_cost", "final_cost", "iterations", "accepted", "pcg_iterations", "status", "lambda_final")
CFG = OptimzeConfig(maxIterations=5, functionTolerance=0.0)


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


def last_paths(ctx):
    return ctx._lib.gb_dbg_ba_last_paths(ctx.handle)


def fields(r):
    return [getattr(r, k) for k in BA_FIELDS]


def own_solve(ctx, pb, edges=None, cfg=CFG):
    """The problem as a caller-held graph: (result, poses, points)."""
    g = BAGraph(ctx, pb, edges)
    try:
        r = g.solve(cfg)
        return (r,) + g.download()
    finally:
        g.close()


def assert_same(r, pose, pts, want):
    w, wpose, wpts = want
    assert fields(r) == fields(w)
    assert r.accepted > 0
    assert pose.tobytes() == wpose.tobytes() and pts.tobytes() == wpts.tobytes()


def moved(pb, seed):
    """pb with new estimates and measurements on the same topology (a sliding window re-solved)."""
    rng = np.random.default_rng(seed)
    out = pb.copy()
    out.cam_pose_wc[2:, 4:] += rng.normal(0, 0.01, out.cam_pose_wc[2:, 4:].shape)
    out.points += rng.normal(0, 0.02, out.points.shape)
    out.obs_xyz[:, :2] += rng.normal(0, 1e-4, (out.n_obs, 2))
    return out


def stale_scratch(ctx):
    """A match of 20 000 x 20 000 descriptors: its feature sets and partials (some MB) are left in the ctx's scratch."""
    q, t = synth.random_descriptors(20000, 41), synth.random_descriptors(20000, 42)
    ctx.match_hamming(q, t)


def test_pnp_ransac_keeps_the_solve_cache(fresh, capfd, monkeypatch):
    """gb_ba_solve, gb_pnp_ransac, gb_ba_solve of the same topology on one ctx: the second solve refreshes the kept graph and returns
    what it returns with no gb_pnp_ransac in between."""
    monkeypatch.setenv("GB_BA_TRACE", "1")
    pb1 = synth.synth_ba(10, 300, seed=3)
    pb2 = moved(pb1, 4)
    xyz, xy = pnp_scenes.scene(np.random.default_rng(5), 2000, outliers=0.2)[:2]
    ctx = fresh()
    ctx.ba_solve(pb1.copy(), CFG)
    assert last_paths(ctx) & BAGraph.LOCAL4
    assert ctx.pnp_ransac(xyz, xy)[2].inliers_minimal >= 4  # (so it refines the pose with gb_ba_pnp)
    capfd.readouterr()
    got = pb2.copy()
    r = ctx.ba_solve(got, CFG)
    assert "cached topology: refresh" in capfd.readouterr().err
    ref = fresh()
    ref.ba_solve(pb1.copy(), CFG)
    want = pb2.copy()
    w = ref.ba_solve(want, CFG)
    assert_same(r, got.cam_pose_wc, got.points, (w, want.cam_pose_wc, want.points))


def pnp_problem(xyz, xy1, pose_wc, dof=63):
    """gb_ba_pnp's graph: one camera, every landmark fixed and observed once."""
    n = xyz.shape[0]
    return BAProblem(cam_pose_wc=pose_wc.reshape(1, 7).copy(), cam_dof=np.array([dof], np.uint8), points=xyz.copy(),
                     point_free=np.zeros(n, np.uint8), obs_cam=np.zeros(n, np.int32), obs_point=np.arange(n, dtype=np.int32),
                     obs_xyz=xy1.copy())


# 2 000 correspondences fit in what the match left and take the local-BA chain; 200 000 grow the scratch
@pytest.mark.parametrize("n", [2000, 200_000])
def test_ba_pnp_over_stale_scratch(fresh, n):
    rng = np.random.default_rng(n)
    xyz, xy, Rg, tg = pnp_scenes.scene(rng, n, outliers=0.05, sigma=1e-3)
    xy1 = np.ascontiguousarray(np.column_stack([xy, np.ones(n)]))
    init = pnp_scenes.Rt_to_pose_wc(Rg, tg)
    init[4:] += 0.05
    ctx = fresh()
    stale_scratch(ctx)
    pose, r, _ = ctx.ba_pnp(xyz, xy1, init, cfg=CFG)
    assert bool(last_paths(ctx) & BAGraph.LOCAL4) == (n == 2000)
    w, wpose, wpts = own_solve(fresh(), pnp_problem(xyz, xy1, init))
    assert fields(r) == fields(w) and r.accepted > 0
    assert pose.tobytes() == wpose[0].tobytes()


def test_ba_solve_posegraph(fresh):
    """A pose graph, then bundle adjustment with pose-graph terms, on one ctx after a match left its scratch."""
    pg = synth.synth_ba(40, 0, n_fixed=1, seed=7)
    pg_edges = synth.synth_pose_edges(pg, seed=2, n_loops=6, gps_every=5, with_info=True)
    ba = synth.synth_ba(30, 3000, seed=8)
    ba_edges = synth.synth_pose_edges(ba, seed=3, n_loops=3, gps_every=4)
    ctx = fresh()
    stale_scratch(ctx)
    for pb, edges in ((pg, pg_edges), (ba, ba_edges)):
        got = pb.copy()
        r = ctx.ba_solve_posegraph(got, edges, CFG)
        assert_same(r, got.cam_pose_wc, got.points, own_solve(fresh(), pb, edges))


def test_ba_solve_uncached(fresh, monkeypatch):
    """gb_ba_solve with the topology cache off: a local-BA window, then a 300 000-edge graph that grows the scratch."""
    monkeypatch.setenv("GB_BA_NO_CACHE", "1")
    ctx = fresh()
    stale_scratch(ctx)
    for pb, local4 in ((synth.synth_ba(10, 300, seed=11), True), (synth.synth_ba(200, 60_000, obs_per_point=5, seed=12), False)):
        got = pb.copy()
        r = ctx.ba_solve(got, CFG)
        assert bool(last_paths(ctx) & BAGraph.LOCAL4) == local4
        assert_same(r, got.cam_pose_wc, got.points, own_solve(fresh(), pb))
