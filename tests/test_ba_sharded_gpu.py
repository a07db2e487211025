"""The landmark-sharded global BA at 2 to 8 ranks on ONE GPU, against oracle/ba_ref.c.

The ranks talk through the loopback communicator (gb_dbg_comm_create_local, api.local_group): rank r runs on its own context, all
contexts share one stream, and each all-reduce is one kernel that sums the ranks' buffers in rank order.  One Python thread drives
each rank (ctypes releases the GIL), exactly as gb_ba_solve_multi drives one device per thread.  NCCL itself is covered only by the
two-GPU test in tests/test_dist.py; everything else of the sharded engine -- the shard's slice of the graph, its chunk / sweep plans,
its Schur contribution, the replicated PCG and LM decisions -- runs here.

Comparison rules are those of tests/test_ba_topology_gpu.py: PCG to convergence (500 iterations, 1e-12), equal LM iteration counts on
both sides, fixed cameras and landmarks untouched, unobserved landmarks unchanged, isolated cameras."""
import contextlib
import ctypes as C
import functools
import threading

import numpy as np
import pytest

import oracle
from gslam_b200 import capi, synth
from gslam_b200.api import BAGraph, OptimzeConfig, ShardedBAGraph, ba_solve_multi, local_group
from gslam_b200.capi import GbError
from gslam_b200.dist import shard_bounds, shard_landmarks
import ba_graphs
from test_ba_topology_gpu import NAMES, case, cfg, check_solve, oracle_solve, rel, solve_opts

gpu = pytest.mark.gpu
B = BAGraph
LAM = 1e-4          # lambda_init on both sides of the reduced-system comparisons
ITERS = 6


# ---- driving the ranks -------------------------------------------------------------------------------------------------------------------
def on_ranks(world, fn, timeout=900):
    """fn(rank) on one thread per rank; returns the results in rank order, re-raises the first rank's error."""
    out, err = [None] * world, [None] * world

    def run(r):
        try:
            out[r] = fn(r)
        except BaseException as e:  # noqa: BLE001 (reported below, per rank)
            err[r] = e
    th = [threading.Thread(target=run, args=(r,), daemon=True) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout)
    assert not any(t.is_alive() for t in th), "a rank did not return"
    for r, e in enumerate(err):
        if e is not None:
            raise AssertionError(f"rank {r} of {world}: {e!r}") from e
    return out


@contextlib.contextmanager
def group(ctx, world):
    ctxs, comms = local_group(ctx, world)
    try:
        yield ctxs, comms
    finally:
        for m in comms:
            m.close()
        for c in ctxs[1:]:
            c.close()


def opts_of(iters, delta=0.01, **kw):
    o = dict(max_iterations=iters, function_tolerance=0.0, huber_delta=delta, pcg_max_iters=500, pcg_tol=1e-12)
    o.update(kw)
    d = cfg(maxIterations=o["max_iterations"], functionTolerance=o["function_tolerance"], projectErrorHuberThreshold=delta,
            pcgMaxIterations=500, pcgTolerance=1e-12, lambdaInit=o.get("lambda_init", 1e-4))
    return o, d


def chunks_expected(pb, lo, hi):
    """Whether the landmark-chunk Schur planner takes this shard: it has a free observed landmark and none has > 16 observers."""
    cnt = np.bincount(pb.obs_point, minlength=pb.n_points)[lo:hi]
    live = (cnt > 0) & (pb.point_free[lo:hi] != 0)
    return bool(live.any()) and int(cnt[live].max()) <= 16


def solve_sharded(ctx, pb, world, opts, sweep=0, cam_split=0, repeat=True):
    """Every rank: create its shard, apply the hooks, solve (twice, with a reset between, when `repeat`), download.
    -> per rank (lo, hi, paths, [(result, poses, points) per run])."""
    with group(ctx, world) as (ctxs, comms):
        def rank(r):
            g = ShardedBAGraph(comms[r], pb)
            try:
                if sweep:
                    g.set_sweep(sweep)
                if cam_split:
                    g.set_cam_split(cam_split)
                runs = []
                for _ in range(2 if repeat else 1):
                    g.reset()
                    res = g.solve(opts)
                    runs.append((res,) + g.download())
                return g.lo, g.hi, g.paths(), runs
            finally:
                g.close()
        return on_ranks(world, rank)


def check_sharded(c, r0, want, out, world, chunks_env=True):
    """Ranges, paths, replication across ranks, the repeat's bits, and the oracle comparison of check_solve."""
    pb = c.pb
    b = shard_bounds(pb, world)
    for r, (lo, hi, p, runs) in enumerate(out):
        assert (lo, hi) == (b[r], b[r + 1]), (r, lo, hi, b)
        assert p & B.PCG_BCSR, (r, p)
        if chunks_env:
            assert bool(p & B.SCHUR_CHUNKS) == chunks_expected(pb, lo, hi), (r, p)
    n_runs = len(out[0][3])
    for k in range(n_runs):
        res = [o[3][k][0] for o in out]
        for r in range(1, world):   # every rank took the same LM decisions on the same (all-reduced) costs
            assert (res[r].iterations, res[r].accepted, res[r].initial_cost, res[r].final_cost, res[r].lambda_final) == \
                   (res[0].iterations, res[0].accepted, res[0].initial_cost, res[0].final_cost, res[0].lambda_final), r
            assert np.array_equal(out[r][3][k][1], out[0][3][k][1]), f"rank {r}'s cameras differ from rank 0's"
        got = pb.copy()
        got.cam_pose_wc[...] = out[0][3][k][1]
        got.points = np.ascontiguousarray(np.concatenate([o[3][k][2] for o in out]).reshape(-1, 3))
        assert got.points.shape == pb.points.shape
        check_solve(c, r0, want, res[0], got)
        if k == 0:
            first = got
        else:   # the repeat after reset(): same bits
            assert res[0].final_cost == out[0][3][0][0].final_cost and res[0].pcg_iterations == out[0][3][0][0].pcg_iterations
            assert np.array_equal(got.cam_pose_wc, first.cam_pose_wc) and np.array_equal(got.points, first.points)
    return first


# ---- graphs ----------------------------------------------------------------------------------------------------------------------------------
def relabel_landmarks(pb, order):
    """The same graph with landmark k := old landmark order[k]."""
    order = np.asarray(order)
    inv = np.empty_like(order)
    inv[order] = np.arange(order.shape[0])
    q = pb.copy()
    q.points = np.ascontiguousarray(pb.points[order])
    q.point_free = np.ascontiguousarray(pb.point_free[order])
    if pb.gt_points is not None:
        q.gt_points = pb.gt_points[order]
    q.obs_point = np.ascontiguousarray(inv[pb.obs_point].astype(np.int32))
    return q


def by_trajectory(pb):
    """Landmarks numbered along the trajectory (by first observing camera): a contiguous landmark shard sees a window of cameras."""
    first = np.full(pb.n_points, pb.n_cams, np.int64)
    np.minimum.at(first, pb.obs_point, pb.obs_cam)
    return relabel_landmarks(pb, np.argsort(first, kind="stable"))


@functools.lru_cache(maxsize=None)
def flagship():
    """The sharded solve's test graph of tests/test_dist.py (60 cameras, 6000 landmarks, 8 observers each)."""
    return ba_graphs.Case("flagship", synth.synth_ba(60, 6000, obs_per_point=8, seed=11, n_fixed=2))


@functools.lru_cache(maxsize=None)
def windowed():
    """A 60-camera trajectory, landmarks numbered along it: at 3 ranks each shard sees ~24 of the 60 cameras, so most structurally
    non-zero blocks of S get nothing from a given shard."""
    return ba_graphs.Case("windowed", by_trajectory(synth.synth_ba(60, 3000, obs_per_point=5, seed=12, n_fixed=2)))


def more_ranks_than_landmarks():
    """6 landmarks seen by all 4 cameras, 8 ranks: some ranks hold no landmark at all (np = no = 0)."""
    pb = synth.synth_ba(4, 6, all_visible=True, n_fixed=2, seed=120)
    return ba_graphs.Case("more_ranks_than_landmarks", pb), 8


def _heavy(nc, n_small, seed, at):
    """n_small landmarks of 3 consecutive observers (half of the cameras fixed) plus one seen by every camera, numbered `at`."""
    pb = synth.synth_ba(nc, n_small, obs_per_point=3, n_fixed=nc // 2, seed=seed)
    j = ba_graphs._add_landmark(pb, range(nc), np.random.default_rng(seed), 20.0)
    order = list(range(j))
    order.insert(at, j)
    return relabel_landmarks(pb, order), at


def heavy_middle_landmark():
    """One landmark seen by all 16 cameras carries 16 of the 64 observations (> 1/8): two shard targets fall inside it, so a middle
    rank is empty."""
    pb, at = _heavy(16, 16, 121, 8)
    return ba_graphs.Case("heavy_middle_landmark", pb), 8


def fixed_rank():
    """Rank 1 of 3 holds only fixed landmarks: it adds to U, g_c and the cost but no off-diagonal block of S."""
    pb = by_trajectory(synth.synth_ba(40, 2000, obs_per_point=4, seed=122, n_fixed=2))
    b = shard_bounds(pb, 3)
    pb.point_free[b[1]:b[2]] = 0
    return ba_graphs.Case("fixed_rank", pb), 3


def unobserved_rank():
    """The heavy landmark last among the observed ones, then 6 free landmarks nobody observes: the last of 8 ranks holds only
    those (np > 0, no = 0)."""
    pb, at = _heavy(16, 16, 123, 16)
    rng = np.random.default_rng(5)
    extra = pb.gt_points[:6] + rng.standard_normal((6, 3))
    pb.points = np.ascontiguousarray(np.vstack([pb.points, extra]))
    pb.gt_points = np.vstack([pb.gt_points, extra])
    pb.point_free = np.append(pb.point_free, np.ones(6, np.uint8))
    n = pb.n_points
    return ba_graphs.Case("unobserved_rank", pb, unobserved=list(range(n - 6, n))), 8


def trajectory_windows():
    """A 120-camera trajectory at 4 ranks: each rank observes only a window of about a quarter of the cameras."""
    pb = by_trajectory(synth.synth_ba(120, 3000, obs_per_point=4, seed=124, n_fixed=2))
    return ba_graphs.Case("trajectory_windows", pb), 4


DEGENERATE = {f.__name__: f for f in (more_ranks_than_landmarks, heavy_middle_landmark, fixed_rank, unobserved_rank, trajectory_windows)}


def assert_shape(name, pb, world):
    """The shard shape `name` stands for really occurs at `world` ranks (dist.shard_bounds)."""
    b = shard_bounds(pb, world)
    cnt = np.bincount(pb.obs_point, minlength=pb.n_points)
    empty = [r for r in range(world) if b[r] == b[r + 1]]
    if name == "more_ranks_than_landmarks":
        assert int((cnt > 0).sum()) < world and empty, b
    elif name == "heavy_middle_landmark":
        assert cnt.max() * world > pb.n_obs and any(0 < r < world - 1 for r in empty), b
    elif name == "fixed_rank":
        assert b[2] > b[1] and not pb.point_free[b[1]:b[2]].any() and pb.point_free[:b[1]].all() and not empty, b
    elif name == "unobserved_rank":
        lo, hi = b[world - 1], b[world]
        assert hi > lo and cnt[lo:hi].sum() == 0 and cnt[:lo].sum() == pb.n_obs, b
    elif name == "trajectory_windows":
        for r in range(world):
            sel = (pb.obs_point >= b[r]) & (pb.obs_point < b[r + 1])
            cams = np.unique(pb.obs_cam[sel])
            assert 0 < cams.shape[0] <= pb.n_cams // 3 and cams[-1] - cams[0] + 1 == cams.shape[0], (r, cams)
    return b


# ---- CPU: shard bounds of the degenerate shapes -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(DEGENERATE))
def test_cabi_shard_bounds_of_degenerate_shapes(name):
    """gb_dbg_ba_shard_bounds (the ranges ba_graph_create_impl uses, host only) == dist.shard_bounds where ranks are empty, hold one
    landmark, only fixed or only unobserved landmarks."""
    c, world = DEGENERATE[name]()
    L = capi.lib()
    assert_shape(name, c.pb, world)
    for w in sorted({1, 2, 3, 4, 8, world}):
        out = np.zeros(w + 1, np.int32)
        op = np.ascontiguousarray(c.pb.obs_point, np.int32)
        assert L.gb_dbg_ba_shard_bounds(c.pb.n_points, c.pb.n_obs, capi.ptr(op), w, capi.ptr(out)) == 0
        assert out.tolist() == shard_bounds(c.pb, w), (name, w)


# ---- the loopback all-reduce itself ------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("n", [0, 1, 255, 1_000_003])
def test_loopback_allreduce_sums_in_rank_order(ctx, n):
    """W = 3: every rank ends with ((b0 + b1) + b2), bit for bit, as numpy computes it."""
    import torch
    rng = np.random.default_rng(n)
    host = [rng.standard_normal(max(n, 1)) * 10.0 ** rng.integers(-8, 9, max(n, 1)) for _ in range(3)]
    want = (host[0] + host[1]) + host[2]
    if n > 1000:   # (the order is observable: another association gives other bits somewhere)
        assert not np.array_equal(want, host[0] + (host[1] + host[2]))
    bufs = [torch.from_numpy(h.copy()).cuda() for h in host]
    torch.cuda.synchronize()
    with group(ctx, 3) as (ctxs, comms):
        on_ranks(3, lambda r: comms[r].allreduce_sum_f64(bufs[r].data_ptr(), n))
        ctx.sync()
    for r in range(3):
        got = bufs[r].cpu().numpy()
        if n == 0:
            assert np.array_equal(got, host[r]), r   # nothing to sum: untouched
        else:
            assert np.array_equal(got[:n], want[:n]), r


@gpu
def test_loopback_allreduce_refuses_unequal_lengths(ctx):
    """Ranks that pass different lengths to one collective all fail (none hangs, none sums)."""
    import torch
    bufs = [torch.ones(8, dtype=torch.float64, device="cuda") for _ in range(2)]
    torch.cuda.synchronize()
    with group(ctx, 2) as (ctxs, comms):
        def rank(r):
            with pytest.raises(GbError, match="different lengths"):
                comms[r].allreduce_sum_f64(bufs[r].data_ptr(), 8 if r == 0 else 7)
        on_ranks(2, rank)
        ctx.sync()
    assert all(float(b.sum()) == 8.0 for b in bufs)


# ---- the reduced system of one shard, before and after the all-reduce ---------------------------------------------------------------------------
def damp(S, dU, lam, dof):
    """lm_damp / clampd (csrc/ba_device.cuh) restated: s + lam * clamp(diag U, 1e-6, 1e32) on a free dof, 1.0 on a fixed one."""
    S = S.copy()
    free = ((dof.astype(np.int64)[:, None] >> np.arange(6)) & 1).reshape(-1).astype(bool)
    k = np.arange(S.shape[0])
    S[k, k] = np.where(free, S[k, k] + lam * np.clip(dU, 1e-6, 1e32), 1.0)
    return S


def coupled_blocks(pb):
    """(i, i') camera pairs that share a free landmark, plus (i, i) for every observed camera."""
    cam = pb.obs_cam.astype(np.int64)
    order = np.argsort(pb.obs_point, kind="stable")
    pairs = set((int(i), int(i)) for i in np.unique(cam))
    pts = pb.obs_point[order]
    cams = cam[order]
    starts = np.flatnonzero(np.r_[True, pts[1:] != pts[:-1]])
    ends = np.r_[starts[1:], pts.shape[0]]
    for a, e in zip(starts, ends):
        if not pb.point_free[pts[a]]:
            continue
        cs = cams[a:e]
        pairs.update((int(x), int(y)) for x in cs for y in cs)
    return pairs


@gpu
def test_shard_reduced_systems_match_oracle_and_sum_exactly(ctx):
    """W = 3 on a trajectory whose shards each see a window of the cameras.  Per rank, BEFORE the all-reduce: S, g~, diag U and cost
    are the oracle's system of dist.shard_landmarks(pb, r, 3), and every block of the whole graph's structure that this shard does not
    touch is exactly 0.0 -- read after a full solve, so stale rbuf contents would show.  AFTER it: every rank holds the same bits,
    ((c0 + c1) + c2) of the contributions, and the oracle's system of the whole problem."""
    c = windowed()
    pb, W = c.pb, 3
    o = cfg(maxIterations=4, functionTolerance=0.0, pcgMaxIterations=500, pcgTolerance=1e-12, lambdaInit=LAM)
    present = coupled_blocks(pb)
    touched = [coupled_blocks(shard_landmarks(pb, r, W)[0]) for r in range(W)]
    with group(ctx, W) as (ctxs, comms):
        def rank(r):
            g = ShardedBAGraph(comms[r], pb)
            try:
                g.solve(o)          # leaves the all-reduced (and, in part, damped) system of its last iteration in rbuf
                g.reset()
                mine = g.dbg_shard_reduced(o, allreduce=False)
                g.reset()
                summed = g.dbg_shard_reduced(o, allreduce=True)
                return g.lo, g.hi, mine, summed
            finally:
                g.close()
        out = on_ranks(W, rank)
    b = shard_bounds(pb, W)
    n_zero_blocks = 0
    for r, (lo, hi, (S, gt, dU, cost), _) in enumerate(out):
        assert (lo, hi) == (b[r], b[r + 1])
        loc, ids = shard_landmarks(pb, r, W)
        S0, gt0, _, _ = oracle.ba_reduced_system(loc, 0.01, LAM, 1, 1e-10)
        lin = oracle.ba_linearize(loc, 0.01)
        dU0 = np.einsum("nii->ni", lin["U"]).reshape(-1)
        assert rel(damp(S, dU, LAM, pb.cam_dof), S0) < 1e-10, (r, rel(damp(S, dU, LAM, pb.cam_dof), S0))
        assert rel(gt, gt0) < 1e-10 and rel(dU, dU0) < 1e-10, (r, rel(gt, gt0), rel(dU, dU0))
        assert abs(cost - lin["cost"]) / lin["cost"] < 1e-12, r
        untouched = [(i, k) for (i, k) in present if (i, k) not in touched[r]]
        for i, k in untouched:
            blk = S[6 * i:6 * i + 6, 6 * k:6 * k + 6]
            assert np.array_equal(blk, np.zeros((6, 6))), (r, i, k, blk)
            if i == k:
                assert not gt[6 * i:6 * i + 6].any() and not dU[6 * i:6 * i + 6].any(), (r, i)
        n_zero_blocks += len(untouched)
    assert n_zero_blocks > len(present), n_zero_blocks   # the shape: most blocks are untouched by a given shard
    # after the all-reduce
    Ss, gts, dUs, costs = out[0][3]
    for r in range(1, W):
        S, gt, dU, cost = out[r][3]
        assert np.array_equal(S, Ss) and np.array_equal(gt, gts) and np.array_equal(dU, dUs) and cost == costs, r
    parts = [o_[2] for o_ in out]
    for k in range(3):
        assert np.array_equal(Ss if k == 0 else (gts if k == 1 else dUs), (parts[0][k] + parts[1][k]) + parts[2][k]), k
    assert costs == (parts[0][3] + parts[1][3]) + parts[2][3]
    stale = sum(1 for r in range(W) for (i, k) in present if (i, k) not in touched[r] and np.abs(Ss[6 * i:6 * i + 6, 6 * k:6 * k + 6]).max() > 0)
    assert stale > 0   # (those blocks are non-zero in the sum, so a shard that left them alone would have added stale values)
    S0, gt0, _, _ = oracle.ba_reduced_system(pb, 0.01, LAM, 1, 1e-10)
    lin = oracle.ba_linearize(pb, 0.01)
    assert rel(damp(Ss, dUs, LAM, pb.cam_dof), S0) < 1e-10 and rel(gts, gt0) < 1e-10
    assert rel(dUs, np.einsum("nii->ni", lin["U"]).reshape(-1)) < 1e-10
    assert abs(costs - lin["cost"]) / lin["cost"] < 1e-12


# ---- solves ----------------------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def flagship_oracle():
    want = flagship().pb.copy()
    return oracle.ba_solve(want, **opts_of(ITERS)[0]), want


@gpu
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_flagship_graph_at_2_to_8_ranks(ctx, world):
    """synth_ba(60, 6000, 8 observers): every landmark shard sees all cameras; chunk Schur, sweep by size, block-CSR PCG."""
    c = flagship()
    r0, want = flagship_oracle()
    out = solve_sharded(ctx, c.pb, world, opts_of(ITERS)[1])
    check_sharded(c, r0, want, out, world)


@gpu
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("large", [False, True], ids=["small", "large"])
@pytest.mark.parametrize("name", NAMES)
def test_irregular_graphs_sharded(ctx, name, large, world):
    """The six tests/ba_graphs.py shapes, sharded.  On large wide_landmarks the landmarks with > 16 observers all fall in the last
    shard: its chunk planner refuses (block gather) while the other shards take the chunk Schur complement."""
    c = case(name, large)
    r0, want = oracle_solve(name, large)
    out = solve_sharded(ctx, c.pb, world, solve_opts(c)[1])
    if name == "wide_landmarks" and large:
        chunks = [bool(o[2] & B.SCHUR_CHUNKS) for o in out]
        assert chunks[:-1] == [True] * (world - 1) and not chunks[-1], chunks
    check_sharded(c, r0, want, out, world)


VARIANTS = ["sweep2_split3", "no_chunks", "bcsr_grid"]


@gpu
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", NAMES)
def test_irregular_graphs_sharded_variants(ctx, monkeypatch, name, variant):
    """Large cases at W = 2 under: the persistent sweep with the camera pass in 3 slices on every rank (on each shard's observation
    slice), the block-gather Schur complement (GB_BA_NO_SCHUR_CHUNKS), the cooperative-grid PCG (GB_BA_NO_PCG_CLUSTER).

    two_components has one free scale per trajectory, damped by lambda alone; after 6 iterations the order in which the sliced
    camera pass sums U and g_c moves its far landmarks by up to 1e-5 relative -- on ONE GPU with the same hooks too (9.6e-6; sharded
    1.03e-5 at W = 2, 6.8e-6 at W = 3; every other hook setting 2e-6..8e-6).  That variant stops after 4 iterations, where lambda is
    still larger, and keeps the 1e-5 bar."""
    c = case(name, True)
    r0, want = oracle_solve(name, True)
    opts = solve_opts(c)[1]
    if variant == "sweep2_split3" and name == "two_components":
        o4, opts = opts_of(4, c.delta)
        want = c.pb.copy()
        r0 = oracle.ba_solve(want, **o4)
    if variant == "no_chunks":
        monkeypatch.setenv("GB_BA_NO_SCHUR_CHUNKS", "1")
    if variant == "bcsr_grid":
        monkeypatch.setenv("GB_BA_NO_PCG_CLUSTER", "1")
    hooks = dict(sweep=2, cam_split=3) if variant == "sweep2_split3" else {}
    out = solve_sharded(ctx, c.pb, 2, opts, **hooks)
    for r, (_, _, p, _) in enumerate(out):
        assert p & B.PCG_BCSR, (r, p)
        if variant == "sweep2_split3":
            assert p & B.SWEEP_LARGE and p & B.CAM_SPLIT, (r, p)
        elif variant == "no_chunks":
            assert not p & B.SCHUR_CHUNKS, (r, p)
        else:
            assert not p & B.BCSR_CLUSTER, (r, p)
    check_sharded(c, r0, want, out, 2, chunks_env=variant != "no_chunks")


@gpu
@pytest.mark.parametrize("sweep", [1, 2])
@pytest.mark.parametrize("name", list(DEGENERATE))
def test_degenerate_shards(ctx, name, sweep):
    """Empty ranks, an empty middle rank behind one heavy landmark, a rank of fixed landmarks only, a rank of unobserved landmarks
    only, and ranks that each see a window of the trajectory -- with the latency-tuned (1) and the persistent (2) sweep."""
    c, world = DEGENERATE[name]()
    assert_shape(name, c.pb, world)
    want = c.pb.copy()
    r0 = oracle.ba_solve(want, **opts_of(5)[0])
    out = solve_sharded(ctx, c.pb, world, opts_of(5)[1], sweep=sweep)
    for r, (_, _, p, _) in enumerate(out):
        assert bool(p & B.SWEEP_LARGE) == (sweep == 2), (r, p)
    check_sharded(c, r0, want, out, world)


# ---- replicated LM control -----------------------------------------------------------------------------------------------------------------------
@gpu
def test_rejected_steps_are_replicated(ctx):
    """A start far from the optimum with lambda_init = 1e-8: the oracle rejects steps; every rank rejects the same ones."""
    pb = synth.synth_ba(40, 3000, obs_per_point=5, seed=11, n_fixed=2, pose_sigma_t=0.3, point_sigma=0.5, pose_sigma_deg=2.0)
    c = ba_graphs.Case("rejects", pb)
    o, d = opts_of(8, lambda_init=1e-8)
    want = pb.copy()
    r0 = oracle.ba_solve(want, **o)
    assert r0.accepted < r0.iterations, (r0.accepted, r0.iterations)
    out = solve_sharded(ctx, pb, 3, d)
    check_sharded(c, r0, want, out, 3)


@gpu
def test_function_tolerance_stops_every_rank_at_the_oracle_iteration(ctx):
    """functionTolerance > 0 takes the polling branch of gb_ba_shard_solve: each rank reads the reduced scalars and stops."""
    c = flagship()
    o, d = opts_of(50, function_tolerance=1e-6)
    want = c.pb.copy()
    r0 = oracle.ba_solve(want, **o)
    assert r0.iterations < 50
    out = solve_sharded(ctx, c.pb, 4, d)
    check_sharded(c, r0, want, out, 4)


# ---- gb_ba_solve_multi on a local group ---------------------------------------------------------------------------------------------------
@gpu
def test_solve_multi_on_a_local_group_equals_the_thread_driven_run(ctx):
    """gb_ba_solve_multi (one host thread per rank inside the library) writes rank 0's cameras and each shard's points at its offsets:
    bit for bit what the ranks driven from Python computed."""
    c = flagship()
    d = opts_of(ITERS)[1]
    out = solve_sharded(ctx, c.pb, 3, d, repeat=False)
    got = c.pb.copy()
    with group(ctx, 3) as (ctxs, comms):
        r1 = ba_solve_multi(ctxs, got, d, comms=comms)
    assert r1.final_cost == out[0][3][0][0].final_cost and r1.accepted == out[0][3][0][0].accepted
    assert np.array_equal(got.cam_pose_wc, out[0][3][0][1])
    for lo, hi, _, runs in out:
        assert np.array_equal(got.points[lo:hi], runs[0][2]), (lo, hi)


# ---- argument errors fail every rank without hanging ---------------------------------------------------------------------------------------------
@gpu
def test_more_than_2048_cameras_refused_on_every_rank(ctx):
    pb = ba_graphs.over_2048_cams()
    with group(ctx, 2) as (ctxs, comms):
        def rank(r):
            with pytest.raises(GbError, match="needs the block-CSR reduced system") as e:
                ShardedBAGraph(comms[r], pb)
            assert e.value.code == capi.GB_ERR_INVALID
        on_ranks(2, rank)


@gpu
def test_graph_communicator_mismatch(ctx):
    """A shard solved with another rank's communicator is refused before any collective."""
    c = flagship()
    L = capi.lib()
    with group(ctx, 2) as (ctxs, comms):
        gs = [ShardedBAGraph(comms[r], c.pb) for r in range(2)]
        try:
            for r in range(2):
                o, res = opts_of(ITERS)[1].to_c(), capi.BaResult()
                other = comms[1 - r]
                assert L.gb_ba_shard_solve(other._h, gs[r]._h, C.byref(o), C.byref(res)) == capi.GB_ERR_INVALID
                assert "graph / communicator mismatch" in L.gb_last_error(other.ctx._h).decode()
        finally:
            for g in gs:
                g.close()
