"""Pose-graph terms (csrc/ba_pose.cu: SE3Edge / GPSEdge) at large and degenerate residuals and on every solver path they take,
against oracle/ba_ref.c, on the named cases of tests/pose_graphs.py.

Every test first asserts the path bits it means to cover (BAGraph.paths()), so that a threshold change cannot quietly turn it
into a duplicate of another test.  Graphs with pose-graph terms always run the stepwise iteration on the dense reduced system:
never the local-BA chain, the single-CTA sparse PCG, the block-CSR PCG or the landmark-chunk Schur plan.

Bars: the edge sweep compares each camera's 6x6 / 6-vector blocks scaled by the block's own largest entry (1e-12 for U, g_c and
the cost, 1e-11 for S and g~); every other case compares whole arrays (1e-10 linearisation, 1e-9 reduced system, 1e-5 after a
fixed-iteration solve).  Measured on an H100 the edge sweep stays below 2e-14 and the other linearisations below 2e-12 (the UTM
frame, whose residuals are differences of 1e5 m translations: |t| 2^-52 ~ 2e-11 m each), so every case meets the common bars."""
import functools

import numpy as np
import pytest

import oracle
from gslam_b200.api import BAGraph, OptimzeConfig
import pose_graphs  # (tests/ is on sys.path under pytest's rootdir conftest)

pytestmark = pytest.mark.gpu
RTOL = 1e-5
B = BAGraph
NEVER = B.LOCAL4 | B.PCG_SPARSE | B.PCG_BCSR | B.SCHUR_CHUNKS   # never taken by a graph with pose-graph terms


def rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300)


def block_rel(got, want):
    """Per-block relative error (rows of the (n, ...) arrays), each scaled by the block's largest entry; a block that is exactly
    zero in `want` must be exactly zero in `got`."""
    g = np.asarray(got).reshape(np.shape(got)[0], -1); w = np.asarray(want).reshape(np.shape(want)[0], -1)
    num = np.abs(g - w).max(axis=1); den = np.abs(w).max(axis=1)
    return np.where(den > 0, num / np.where(den > 0, den, 1.0), np.where(num > 0, np.inf, 0.0))


def blocks6(S, nc):
    return S.reshape(nc, 6, nc, 6).transpose(0, 2, 1, 3).reshape(nc * nc, 36)


def cfg(**kw):
    c = OptimzeConfig()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def pose_close(a, b, tol):
    s = np.sign(np.sum(a[:, :4] * b[:, :4], axis=1))[:, None]
    assert np.abs(a[:, :4] * s - b[:, :4]).max() < tol, np.abs(a[:, :4] * s - b[:, :4]).max()
    assert np.abs(a[:, 4:] - b[:, 4:]).max() < tol * max(1.0, np.abs(b[:, 4:]).max()), np.abs(a[:, 4:] - b[:, 4:]).max()


def expect_paths(p, nc, large_sweep=False):
    assert not p & NEVER, p
    assert bool(p & B.PCG_CLUSTER) == (nc <= 85), p          # one-cluster PCG while 6N <= 512, else the generic PCG
    assert bool(p & B.DENSE_ATOMIC) == (nc > 2048), p
    assert bool(p & B.SWEEP_LARGE) == large_sweep, p


# ---- 1. one edge per block, every angle class -----------------------------------------------------------------------------------
@pytest.mark.parametrize("angle", list(pose_graphs.ANGLES))
@pytest.mark.parametrize("kind", ["se3", "gps"])
def test_edge_sweep_matches_oracle_block_by_block(ctx, kind, angle):
    pb, pe = pose_graphs.edge_sweep(kind, angle)
    nc = pb.n_cams
    want = oracle.ba_linearize(pb, 0.01, pe)
    g = BAGraph(ctx, pb, pe)
    expect_paths(g.paths(), nc)
    got = g.dbg_linearize(0.01)
    for k in ("U", "gc"):
        err = block_rel(got[k], want[k])
        assert err.max() < 1e-12, (k, err)
    assert abs(got["cost"] - want["cost"]) <= 1e-12 * want["cost"], (got["cost"], want["cost"])
    # (each pair's gauge is free: only lambda holds it, so the PCG solution is not compared)
    S0, gt0, _, _ = oracle.ba_reduced_system(pb, 0.01, 1e-4, 50, 1e-10, pe)
    S, gt, _, _ = g.dbg_reduced(cfg(pcgMaxIterations=50, pcgTolerance=1e-10))
    g.close()
    err = block_rel(blocks6(S, nc), blocks6(S0, nc))
    assert err.max() < 1e-11, err.reshape(nc, nc)
    err = block_rel(gt.reshape(nc, 6), gt0.reshape(nc, 6))
    assert err.max() < 1e-11, err


# ---- 2. whole graphs: linearisation, reduced system, fixed-iteration solve -----------------------------------------------------------
CASES = {"large_residuals": pose_graphs.large_residuals, "masks_and_fixed": pose_graphs.masks_and_fixed,
         **{f"info_{f}": functools.partial(pose_graphs.info_forms, f) for f in pose_graphs.INFO_FORMS},
         "hub_and_parallel": pose_graphs.hub_and_parallel, "size_300": functools.partial(pose_graphs.size_case, 300)}
ITERS = {"large_residuals": 8}   # (the others converge to rounding level within a few iterations, where accept / reject is decided
#                                   by the last bit of the cost on either side: they are compared while the cost still moves)


@functools.lru_cache(maxsize=None)
def case(name):
    pb, pe = CASES[name]() if name in CASES else pose_graphs.mixed_large(name)
    pose_graphs.check(pb, pe)
    return pb, pe


def solve_opts(name, nc):
    """The same options on both sides.  From 160 cameras on, a PCG cap with tolerance 0: no exit depends on summation order."""
    it = ITERS.get(name, 6 if name in pose_graphs.MIXED_LARGE else 4)
    cap, tol = (300, 0.0) if nc >= 160 else (600, 1e-13)
    return (dict(max_iterations=it, function_tolerance=0.0, pcg_max_iters=cap, pcg_tol=tol),
            cfg(maxIterations=it, functionTolerance=0.0, pcgMaxIterations=cap, pcgTolerance=tol))


@functools.lru_cache(maxsize=None)
def oracle_solve(name):
    pb, pe = case(name)
    want = pb.copy()
    r0 = oracle.ba_solve(want, pe, **solve_opts(name, pb.n_cams)[0])
    return r0, want


def check_solve(pb, r0, want, r1, got):
    assert r1.iterations == r0.iterations and r1.accepted == r0.accepted and r0.accepted > 0, (r1.iterations, r1.accepted, r0.iterations, r0.accepted)
    assert abs(r1.initial_cost - r0.initial_cost) <= 1e-10 * r0.initial_cost
    assert abs(r1.final_cost - r0.final_cost) <= RTOL * r0.final_cost, (r1.final_cost, r0.final_cost)
    pose_close(got.cam_pose_wc, want.cam_pose_wc, RTOL)
    if pb.n_points:
        assert rel(got.points, want.points) < RTOL
    fixed = pb.cam_dof == 0   # (the T_wc <-> T_cw round trip of the download may move last bits: see test_fixed_cameras_...)
    assert np.abs(got.cam_pose_wc[fixed] - pb.cam_pose_wc[fixed]).max(initial=0) <= 1e-15 * max(1.0, np.abs(pb.cam_pose_wc[:, 4:]).max())


@pytest.mark.parametrize("name", list(CASES))
def test_case_linearisation_and_reduced_system_match_oracle(ctx, name):
    pb, pe = case(name)
    want = oracle.ba_linearize(pb, 0.01, pe)
    g = BAGraph(ctx, pb, pe)
    expect_paths(g.paths(), pb.n_cams)
    got = g.dbg_linearize(0.01); again = g.dbg_linearize(0.01)
    assert rel(got["U"], want["U"]) < 1e-10, rel(got["U"], want["U"])
    assert rel(got["gc"], want["gc"]) < 1e-10, rel(got["gc"], want["gc"])   # (info_utm: ~2e-12, the |t| 2^-52 of its 1e5 m frame)
    assert abs(got["cost"] - want["cost"]) <= 1e-10 * want["cost"]
    for k in ("U", "gc"):
        assert np.array_equal(got[k], again[k]), k
    S0, gt0, _, _ = oracle.ba_reduced_system(pb, 0.01, 1e-4, 50, 1e-10, pe)
    S, gt, _, _ = g.dbg_reduced(cfg(pcgMaxIterations=50, pcgTolerance=1e-10))
    g.close()
    assert rel(S, S0) < 1e-9, rel(S, S0)
    assert np.abs(S - S.T).max() < 1e-9 * np.abs(S).max()
    assert rel(gt, gt0) < 1e-9, rel(gt, gt0)


@pytest.mark.parametrize("name", list(CASES))
def test_case_solve_matches_oracle_and_repeats_bitwise(ctx, name):
    pb, pe = case(name)
    r0, want = oracle_solve(name)
    opts = solve_opts(name, pb.n_cams)[1]
    g = BAGraph(ctx, pb, pe)
    runs = []
    for _ in range(2):   # (<= 2048 cameras: every reduction has a fixed order, so a repeat after reset() gives the same bits)
        g.reset()
        r1 = g.solve(opts)
        got = pb.copy()
        got.cam_pose_wc[...], got.points[...] = g.download()
        runs.append((r1, got))
    g.close()
    (r1, got), (r2, got2) = runs
    check_solve(pb, r0, want, r1, got)
    assert (r1.final_cost, r1.accepted, r1.pcg_iterations) == (r2.final_cost, r2.accepted, r2.pcg_iterations)
    assert np.array_equal(got.cam_pose_wc, got2.cam_pose_wc) and np.array_equal(got.points, got2.points)
    # the host-buffer entry point (gb_ba_solve_posegraph) computes the same bits
    host = pb.copy()
    r3 = ctx.ba_solve_posegraph(host, pe, opts)
    assert (r3.final_cost, r3.iterations, r3.accepted, r3.pcg_iterations) == (r1.final_cost, r1.iterations, r1.accepted, r1.pcg_iterations)
    assert np.array_equal(host.cam_pose_wc, got.cam_pose_wc) and np.array_equal(host.points, got.points)


def test_fixed_cameras_keep_their_pose_and_masked_components_stay(ctx):
    """masks_and_fixed: the fully fixed cameras' internal pose is not touched by a solve (the download of a reset graph and of the
    solved one agree bit for bit there); the masked tangent components are checked through the oracle agreement above, and here
    directly: U and g_c rows and columns of a masked component are exactly zero."""
    pb, pe = case("masks_and_fixed")
    g = BAGraph(ctx, pb, pe)
    lin = g.dbg_linearize(0.01)
    for i, m in list(pose_graphs.MASKS.items()) + [(0, 0), (1, 0)]:
        off = [d for d in range(6) if not (m >> d) & 1]
        assert not lin["U"][i][off, :].any() and not lin["U"][i][:, off].any() and not lin["gc"][i][off].any(), i
    g.reset()
    before = g.download()[0]
    g.solve(solve_opts("masks_and_fixed", pb.n_cams)[1])
    after = g.download()[0]
    g.close()
    fixed = pb.cam_dof == 0
    assert np.array_equal(after[fixed], before[fixed])
    assert not np.array_equal(after[~fixed], before[~fixed])


# ---- 3. the large mixed graphs under every sweep kernel and camera split -------------------------------------------------------------
@pytest.mark.parametrize("sweep,split", [(1, 1), (2, 1), (1, 3), (2, 3)])
@pytest.mark.parametrize("name", list(pose_graphs.MIXED_LARGE))
def test_mixed_large_graph_every_sweep_matches_oracle(ctx, name, sweep, split):
    pb, pe = case(name)
    assert pb.n_cams == 160 and pb.n_obs > 65536
    g = BAGraph(ctx, pb, pe)
    expect_paths(g.paths(), pb.n_cams, large_sweep=True)
    g.set_sweep(sweep)
    g.set_cam_split(split)
    p = g.paths()
    assert not p & NEVER and bool(p & B.SWEEP_LARGE) == (sweep == 2) and bool(p & B.CAM_SPLIT) == (split > 1), p
    want = oracle.ba_linearize(pb, 0.01, pe)
    got = g.dbg_linearize(0.01); again = g.dbg_linearize(0.01)
    for k in ("U", "gc", "V", "gp", "W"):
        assert rel(got[k], want[k]) < 1e-10, (k, rel(got[k], want[k]))
        assert np.array_equal(got[k], again[k]), k
    assert abs(got["cost"] - want["cost"]) <= 1e-10 * want["cost"]
    S0, gt0, _, _ = oracle.ba_reduced_system(pb, 0.01, 1e-4, 20, 0.0, pe)
    S, gt, _, _ = g.dbg_reduced(cfg(pcgMaxIterations=20, pcgTolerance=0.0))
    assert rel(S, S0) < 1e-9 and rel(gt, gt0) < 1e-9, (rel(S, S0), rel(gt, gt0))
    assert np.abs(S - S.T).max() < 1e-9 * np.abs(S).max()
    r0, want_pb = oracle_solve(name)
    g.reset()
    r1 = g.solve(solve_opts(name, pb.n_cams)[1])
    got_pb = pb.copy()
    got_pb.cam_pose_wc[...], got_pb.points[...] = g.download()
    g.close()
    check_solve(pb, r0, want_pb, r1, got_pb)


# ---- 4. the stepwise interface on caller-owned buffers ------------------------------------------------------------------------------
def _stepwise(g, opts):
    import torch
    buf = torch.zeros(g.reduce_size(), dtype=torch.float64, device="cuda")
    cost = torch.zeros(1, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()  # (the library works on its own stream)
    g.begin(opts)
    for _ in range(opts.maxIterations):
        g.reduce_local(buf.data_ptr())
        g.step(buf.data_ptr(), cost.data_ptr())
        g.commit(buf.data_ptr(), cost.data_ptr())
    return g.finish()


@pytest.mark.parametrize("name", ["large_residuals", "isolated_cameras"])
def test_stepwise_interface_with_caller_buffers_equals_solve(ctx, name):
    pb, pe = case(name)
    opts = solve_opts(name, pb.n_cams)[1]
    g = BAGraph(ctx, pb, pe)
    assert not g.paths() & NEVER
    g.reset()
    r1 = g.solve(opts)
    p1, x1 = g.download()
    g.reset()
    r2 = _stepwise(g, opts)
    p2, x2 = g.download()
    g.close()
    assert (r2.final_cost, r2.iterations, r2.accepted, r2.pcg_iterations) == (r1.final_cost, r1.iterations, r1.accepted, r1.pcg_iterations)
    assert np.array_equal(p1, p2) and np.array_equal(x1, x2)
    r0, want = oracle_solve(name)
    got = pb.copy(); got.cam_pose_wc[...], got.points[...] = p2, x2
    check_solve(pb, r0, want, r2, got)


# ---- 5. above 2048 cameras: no block structure, S by fp64 atomics --------------------------------------------------------------------
def _rel_rows(a, b, rows=1024):
    num = max(np.abs(a[r:r + rows] - b[r:r + rows]).max() for r in range(0, a.shape[0], rows))
    return num / max(np.abs(b).max(), 1e-300)


def test_pose_graph_above_2048_cameras(ctx):
    pb, pe = pose_graphs.size_case(2100)
    g = BAGraph(ctx, pb, pe)
    expect_paths(g.paths(), pb.n_cams)
    want = oracle.ba_linearize(pb, 0.01, pe)
    got = g.dbg_linearize(0.01)
    assert rel(got["U"], want["U"]) < 1e-10 and rel(got["gc"], want["gc"]) < 1e-10
    assert abs(got["cost"] - want["cost"]) <= 1e-10 * want["cost"]
    del want, got
    S0, gt0, _, _ = oracle.ba_reduced_system(pb, 0.01, 1e-4, 20, 0.0, pe)
    S, gt, _, _ = g.dbg_reduced(cfg(pcgMaxIterations=20, pcgTolerance=0.0))
    assert _rel_rows(S, S0) < 1e-9 and rel(gt, gt0) < 1e-9
    del S0
    assert _rel_rows(S, S.T) < 1e-9
    del S
    # a 2-iteration solve, twice: no fixed reduction order here, so the repeat agrees to 1e-9, not bitwise
    a = pb.copy()
    r0 = oracle.ba_solve(a, pe, max_iterations=2, function_tolerance=0.0, pcg_max_iters=50, pcg_tol=0.0)
    runs = []
    for _ in range(2):
        g.reset()
        r1 = g.solve(cfg(maxIterations=2, functionTolerance=0.0, pcgMaxIterations=50, pcgTolerance=0.0))
        runs.append((r1,) + g.download())
    g.close()
    (r1, p1, _), (r2, p2, _) = runs
    assert r1.iterations == r0.iterations == 2 and r1.accepted == r0.accepted
    assert abs(r1.final_cost - r0.final_cost) <= RTOL * r0.final_cost
    pose_close(p1, a.cam_pose_wc, RTOL)
    assert r1.accepted == r2.accepted and abs(r1.final_cost - r2.final_cost) <= 1e-9 * r1.final_cost
    pose_close(p2, p1, 1e-9)
