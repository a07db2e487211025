"""A device-resident BAGraph.solve waits for the device without holding its context: while the mapping thread is blocked in a
solve, a tracking thread can still order work on that context (Context.wait_for), and the solve returns what it returns alone.
A second solve of the same graph started during that wait does not disturb the first."""
import threading
import time

import numpy as np
import pytest

from gslam_b200 import synth
from gslam_b200.api import BAGraph, Context, Features, OptimzeConfig

pytestmark = pytest.mark.gpu

W, H, NKP = 1920, 1080, 2000
CFG = dict(maxIterations=10, functionTolerance=0.0, pcgMaxIterations=50, pcgTolerance=1e-10)
RESULT = ("initial_cost", "final_cost", "iterations", "accepted", "pcg_iterations", "status", "lambda_final")


def _hold_behind_extractions(ctx, ctx_m, n=100):
    """Order ctx_m's stream after n 1080p extractions on ctx (~20 ms of device work), so that a solve enqueued on ctx_m next
    stays blocked on the device long after its enqueue; returns the Features to close."""
    import torch
    frames = torch.from_numpy(synth.synth_stream(W, H, 2, seed=7)).cuda()
    ocfg = ctx.orb_cfg(nfeatures=NKP)
    f = Features(ctx, 2 * NKP + 256)
    torch.cuda.synchronize()
    for k in range(n):
        f.extract(frames[k & 1].data_ptr(), W, H, ocfg, device_ptr=True, pitch=W)
    ctx_m.wait_for(ctx)
    return f


def _same(a, b):
    for k in RESULT:
        assert getattr(a, k) == getattr(b, k), k


def test_wait_for_is_not_held_up_by_a_solve_in_flight():
    ctx, ctx_m, other = Context(0), Context(0), Context(0)
    try:
        pb = synth.synth_ba(50, 2000, 5, seed=42, n_fixed=2)
        cfg = OptimzeConfig(**CFG)
        g = BAGraph(ctx_m, pb)
        alone = g.solve(cfg)
        poses0, pts0 = g.download()

        f = _hold_behind_extractions(ctx, ctx_m)
        g.reset()
        out = {}

        def mapper():
            out["res"] = g.solve(cfg)
            out["t_solve"] = time.perf_counter()
        th = threading.Thread(target=mapper)
        t0 = time.perf_counter()
        th.start()
        time.sleep(0.004)
        t1 = time.perf_counter()
        ctx_m.wait_for(other)  # needs ctx_m while the mapping thread waits in its solve
        t2 = time.perf_counter()
        th.join()
        # the solve stayed blocked well past the wait_for call (else this test shows nothing) ...
        assert out["t_solve"] - t0 > 0.010, f"the solve returned after {(out['t_solve'] - t0) * 1e3:.1f} ms: not held on the device"
        # ... and wait_for did not wait for it to return
        assert t2 - t1 < 0.002, f"wait_for took {(t2 - t1) * 1e3:.2f} ms while a solve waited on the device"

        res = out["res"]
        poses, pts = g.download()
        assert np.array_equal(poses, poses0) and np.array_equal(pts, pts0)
        _same(res, alone)
        assert res.gpu_ms > 0.0
        g.close(); f.close()
    finally:
        other.close(); ctx_m.close(); ctx.close()


def test_second_solve_of_a_graph_during_its_unlocked_wait():
    """While thread A waits unlocked in g.solve(), thread B solves g again (without a reset: from A's result): B's solve takes the
    locked wait and gives the sequential second solve's result, and A's result is the single-threaded one."""
    ctx, ctx_m = Context(0), Context(0)
    try:
        pb = synth.synth_ba(50, 2000, 5, seed=42, n_fixed=2)
        cfg = OptimzeConfig(**CFG)
        g = BAGraph(ctx_m, pb)
        first = g.solve(cfg)
        second = g.solve(cfg)  # continues from the first solve's estimate
        want_p, want_x = g.download()

        g.reset()
        f = _hold_behind_extractions(ctx, ctx_m)
        out, started = {}, threading.Event()

        def solver_a():
            started.set()
            out["a"] = g.solve(cfg)
        th = threading.Thread(target=solver_a)
        th.start()
        started.wait()
        time.sleep(0.003)
        b = g.solve(cfg)
        a_done_before_b = "a" in out
        th.join()
        assert not a_done_before_b, "the first solve returned before the second was enqueued: the overlap was not exercised"
        _same(out["a"], first)
        _same(b, second)
        assert out["a"].gpu_ms > 0.0 and b.gpu_ms > 0.0
        p, x = g.download()
        assert np.array_equal(p, want_p) and np.array_equal(x, want_x)
        g.close(); f.close()
    finally:
        ctx_m.close(); ctx.close()


def test_repeated_device_resident_solves_from_two_threads_match_one_thread():
    """reset()/solve() on a mapping ctx from its own thread while a tracking thread keeps ordering it after its ctx: every solve
    gives the single-threaded result bit for bit."""
    ctx = Context(0)
    ctx_m = Context(0, high_priority=True)
    try:
        pb = synth.synth_ba(20, 600, 4, seed=3, n_fixed=1)
        cfg = OptimzeConfig(maxIterations=6, functionTolerance=0.0)
        g = BAGraph(ctx_m, pb)
        want = g.solve(cfg)
        wp, wx = g.download()
        got, err = [], []

        def mapper():
            try:
                for _ in range(20):
                    g.reset()
                    r = g.solve(cfg)
                    got.append((r, *g.download()))
            except Exception as e:  # surfaced after the join
                err.append(e)
        th = threading.Thread(target=mapper)
        th.start()
        while th.is_alive():
            ctx_m.wait_for(ctx)
        th.join()
        assert not err, err
        assert len(got) == 20
        for r, p, x in got:
            _same(r, want)
            assert np.array_equal(p, wp) and np.array_equal(x, wx)
        g.close()
    finally:
        ctx_m.close(); ctx.close()
