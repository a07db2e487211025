"""The BA landmark elimination and back-substitution, block by block, against an extended-precision elimination of the device's own
linearisation (tests/ba_elim.py, pinned on the CPU by tests/test_ba_elim_reference.py).

Elimination: g.reset(), lin = g.dbg_linearize(delta), then the system one LM step would solve (g.dbg_system) at lambda in
{1e-8, 1e-4, 1e4}.  Every S entry, g~ entry and diag U entry is held to its componentwise bound; on top of that, bit for bit: every
block outside the covisibility structure is 0.0, every lower block is the transpose of its mirror, diag U is the diagonal of U and a
camera that sees only fixed landmarks has S_ii == U_i.  On every kernel that forms S: ba_schur_blocks_kernel (local windows, and large
graphs under GB_BA_NO_SCHUR_CHUNKS), ba_schur_chunks_kernel + ba_schur_reduce_kernel in one and in two slot passes, the dense
ba_schur_accum_kernel + mirror above 2048 cameras, and the per-shard contribution of the landmark-sharded solve and its all-reduce.

Back-substitution: one LM iteration (maxIterations = 1), then what it left on the device (g.dbg_last_step): the candidate landmarks
against the reference at the device's own camera step, V~^-1 against the reference inverse at the lambda the path holds after the
iteration (the local-BA chain refreshes it after a rejection), exact zeros where V~^-1 must be zero and nowhere else.

Numeric-edge graphs (here only: their conditioning would loosen the trajectory bars of the parity tests) each assert the property they
are named for."""
import contextlib

import numpy as np
import pytest

from gslam_b200 import synth
from gslam_b200.api import BAGraph, OptimzeConfig, ShardedBAGraph, local_group
from gslam_b200.dist import shard_landmarks
import ba_elim as E  # (tests/ is on sys.path under pytest's rootdir conftest)
import ba_graphs
import ba_linsys

pytestmark = pytest.mark.gpu
B = BAGraph
LAMS = (1e-8, 1e-4, 1e4)


def cfg(**kw):
    c = OptimzeConfig()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def edge_property(name, pb, delta, lin, ref):
    """The property each numeric-edge graph is named for, asserted on the host."""
    dV = np.einsum("jaa->ja", lin["V"])
    act = ref.active
    if name == "far_landmarks":
        assert (dV[act] < 1e-6).any(), dV[act].min()                               # the 1e-6 clamp binds
    elif name == "near_landmarks":
        pose = pb.cam_pose_wc
        for c in range(3, 29, 3):
            j = pb.n_points - len(range(3, 29, 3)) + (c - 3) // 3
            R = synth._quat_to_R((pose[c, :4] / np.linalg.norm(pose[c, :4]))[None])[0]
            assert abs((R.T @ (pb.points[j] - pose[c, 4:]))[2] - 0.05) < 1e-12
    elif name == "narrow_baseline":
        for j in range(pb.n_points - 13, pb.n_points):
            c = pb.obs_cam[pb.obs_point == j]
            base = np.linalg.norm(pb.cam_pose_wc[c[1], 4:] - pb.cam_pose_wc[c[0], 4:])
            depth = np.linalg.norm(pb.points[j] - pb.cam_pose_wc[c[0], 4:])
            assert 0.9e-4 < base / depth < 1.1e-4
    elif name == "huber_linear":
        Rwc = synth._quat_to_R(pb.cam_pose_wc[:, :4])
        q = np.einsum("nji,nj->ni", Rwc[pb.obs_cam], pb.points[pb.obs_point] - pb.cam_pose_wc[pb.obs_cam, 4:])
        e = np.linalg.norm(q[:, :2] / q[:, 2:3] - pb.obs_xyz[:, :2], axis=1)
        assert (e > delta).mean() > 0.75
    elif name == "fixed_only_cameras":
        for c in (9, 21):
            assert not ref.active[pb.obs_point[pb.obs_cam == c]].any()
    elif name == "single_low_lambda":
        assert ref.kappa.max() >= 1e7, ref.kappa.max()
    elif name == "indefinite_info":      # damped V of those landmarks far from positive definite (robustly zeroed), all others factor
        if ref.lam <= 1e-4:
            ev = np.linalg.eigvalsh(ref.Vt64[list(ba_graphs.INDEFINITE)])
            assert (ev[:, 0] < -1e-2 * np.abs(ev).max(axis=1)).all(), ev
            assert sorted(np.nonzero(ref.zeroed)[0]) == sorted(ba_graphs.INDEFINITE)
        assert (ref.kappa[ref.active & ~ref.zeroed] < 1e12).all()


def problem(name, large=False):
    if name in ba_graphs.EDGES:
        return ba_graphs.EDGES[name]()
    if name == "rejected_step":
        return ba_graphs.rejected_step()
    if name == "zero_rhs":
        return ba_linsys.zero_rhs(), 0.01
    if name == "single_low_lambda":
        c = ba_graphs.build("sparse_landmarks")
        return c.pb, c.delta
    if name == "over_2048_cams":
        return ba_graphs.over_2048_cams(), 0.01
    c = ba_graphs.build(name, large)
    return c.pb, c.delta


# ---- the elimination -----------------------------------------------------------------------------------------------------------------
def check_system(ref, s, pb):
    nc = pb.n_cams
    S = s["S"]
    Sb = ref.s_blocks(S)
    r = ref.s_ratio(Sb)
    assert r <= 1.0, ("S", r)
    i, k = ref.blocks[:, 0], ref.blocks[:, 1]
    off = i != k
    r6 = np.arange(6)
    lower = S[(6 * k[off])[:, None, None] + r6[None, :, None], (6 * i[off])[:, None, None] + r6[None, None, :]]
    assert np.array_equal(lower, np.swapaxes(Sb[off], 1, 2)), "a lower block is not the transpose of its mirror"
    assert ref.gt_ratio(s["gt"]) <= 1.0, ("g~", ref.gt_ratio(s["gt"]))
    assert np.array_equal(s["diagU"], ref.diagU), "diag U"
    alone = np.setdiff1d(np.arange(nc), pb.obs_cam[ref.active[pb.obs_point]])
    for c in alone:                     # no active landmark: S_ii is U_i
        assert np.array_equal(S[6 * c:6 * c + 6, 6 * c:6 * c + 6], ref.U[c]), c
    S4 = S.reshape(nc, 6, nc, 6)       # (in place: what is left outside the structure must be exactly zero)
    I, K = np.nonzero(ref.structural)
    S4[I, :, K, :] = 0.0
    assert not S.any(), "an entry outside the covisibility structure is not 0.0"
    return r, alone


def run_elimination(g, pb, delta, lams, edge=None, into_u=False):
    ratios = []
    for lam in lams:
        g.reset()
        lin = g.dbg_linearize(delta)
        s = g.dbg_system(cfg(lambdaInit=lam, projectErrorHuberThreshold=delta, pcgMaxIterations=5))
        assert s["lam"] == lam
        ref = E.Elim(pb, lin, lam, into_u=into_u)
        if edge:
            edge_property(edge, pb, delta, lin, ref)
        ratios.append(check_system(ref, s, pb)[0])
    return ratios


SMALL = list(ba_graphs.CASES)


@pytest.mark.parametrize("name", SMALL + list(ba_graphs.EDGES) + ["single_low_lambda"])
def test_elimination_blocks_kernel_local(ctx, name):
    pb, delta = problem(name)
    g = BAGraph(ctx, pb)
    p = g.paths()
    assert p & B.LOCAL4 and p & B.PCG_SPARSE and not p & (B.SCHUR_CHUNKS | B.DENSE_ATOMIC), p
    run_elimination(g, pb, delta, (1e-8,) if name == "single_low_lambda" else LAMS, name if name in ba_graphs.EDGES or name == "single_low_lambda" else None)
    g.close()


@pytest.mark.parametrize("name", SMALL)
def test_elimination_large_graphs(ctx, monkeypatch, name):
    """The large form on the chunk kernel (one pass; two on long_tracks) and, created under GB_BA_NO_SCHUR_CHUNKS, on the block-gather
    kernel (wide_landmarks: the planner refuses its > 16-observer landmarks, block gather only)."""
    pb, delta = problem(name, True)
    g = BAGraph(ctx, pb)
    p = g.paths()
    assert p & B.PCG_BCSR and not p & (B.LOCAL4 | B.DENSE_ATOMIC), p
    assert bool(p & B.SCHUR_CHUNKS) == (name != "wide_landmarks"), p
    assert bool(p & B.SCHUR_PASSES) == (name == "long_tracks"), p
    run_elimination(g, pb, delta, LAMS if name == "long_tracks" else (1e-4,))
    g.close()
    if name == "wide_landmarks":
        return
    monkeypatch.setenv("GB_BA_NO_SCHUR_CHUNKS", "1")
    g = BAGraph(ctx, pb)
    p = g.paths()
    assert p & B.PCG_BCSR and not p & (B.SCHUR_CHUNKS | B.SCHUR_PASSES | B.LOCAL4), p
    run_elimination(g, pb, delta, (1e-4,))
    g.close()


def test_elimination_dense_atomic(ctx):
    pb, delta = problem("over_2048_cams")
    g = BAGraph(ctx, pb)
    assert g.paths() & B.DENSE_ATOMIC, g.paths()
    run_elimination(g, pb, delta, (1e-4,), into_u=True)      # (S and g~ start at U_i and g_c,i; every term is subtracted by an atomic)
    g.close()


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


@pytest.mark.parametrize("world", [2, 3])
def test_elimination_sharded(ctx, world):
    """Per rank, the shard's contribution (before the all-reduce) against the reference of a single-GPU graph of that shard; after the
    all-reduce, the system of the whole problem."""
    from test_ba_sharded_gpu import on_ranks
    c = ba_graphs.build("long_tracks", True)
    pb, delta, lam = c.pb, c.delta, 1e-4
    o = cfg(lambdaInit=lam, projectErrorHuberThreshold=delta)
    with group(ctx, world) as (ctxs, comms):
        def rank(r):
            g = ShardedBAGraph(comms[r], pb)
            try:
                g.reset()
                mine = g.dbg_shard_reduced(o, allreduce=False)
                g.reset()
                return mine, g.dbg_shard_reduced(o, allreduce=True)
            finally:
                g.close()
        out = on_ranks(world, rank)
    for r in range(world):
        loc, _ = shard_landmarks(pb, r, world)
        gl = BAGraph(ctx, loc)
        ref = E.Elim(loc, gl.dbg_linearize(delta), lam)
        gl.close()
        S, gt, dU, _ = out[r][0]
        check_system(ref, dict(S=S, gt=gt, diagU=dU), loc)
    g = BAGraph(ctx, pb)
    ref = E.Elim(pb, g.dbg_linearize(delta), lam)
    g.close()
    S, gt, dU, _ = out[0][1]
    for r in range(1, world):
        assert all(np.array_equal(a, b) for a, b in zip(out[r][1][:3], (S, gt, dU))), r
    # (the all-reduce adds the shards' U_i: diag U and S within the bounds of the whole problem, not bit for bit)
    assert ref.s_ratio(ref.s_blocks(S)) <= 1.0 and ref.gt_ratio(gt) <= 1.0
    assert np.abs(dU - ref.diagU).max() <= 4 * E.U_RND * np.abs(ref.diagU).max()


# ---- the back-substitution and V~^-1 ---------------------------------------------------------------------------------------------------
# path -> (graph, large, force_generic_pcg mode, linear solver, bits set, bits clear, lambdas at which the first step is rejected)
BOTH = (1e-4, 1e-8)
BACKSUB = {
    "local_sparse": ("long_tracks", False, 0, 0, B.LOCAL4 | B.PCG_SPARSE, B.PCG_BCSR, ()),
    "local_direct": ("long_tracks", False, 0, 1, B.LOCAL4 | B.CHOL_OK, B.PCG_BCSR, ()),
    "stepwise_dense": ("measurement_forms", False, 1, 0, 0, B.LOCAL4 | B.PCG_SPARSE | B.PCG_CLUSTER | B.PCG_BCSR, ()),
    "compact_chunks": ("long_tracks", True, 0, 0, B.PCG_BCSR | B.SCHUR_CHUNKS | B.SCHUR_PASSES, B.LOCAL4, ()),
    "compact_gather": ("wide_landmarks", True, 0, 0, B.PCG_BCSR, B.LOCAL4 | B.SCHUR_CHUNKS, ()),
    "local_edges_far": ("far_landmarks", False, 0, 0, B.LOCAL4, 0, ()),
    "local_edges_baseline": ("narrow_baseline", False, 0, 0, B.LOCAL4, 0, ()),
    "local_zeroed": ("indefinite_info", False, 0, 0, B.LOCAL4, 0, None),     # (zeroed inverses: whichever LM decision follows)
    # a step of exactly zero (g~ = 0: x = 0, p_new = p) and a Gauss-Newton step that overshoots
    "local_zero_step": ("zero_rhs", False, 0, 0, B.LOCAL4 | B.PCG_SPARSE, 0, BOTH),
    "stepwise_zero_step": ("zero_rhs", False, 1, 0, 0, B.LOCAL4 | B.PCG_SPARSE, BOTH),
    "local_overshoot": ("rejected_step", False, 0, 0, B.LOCAL4 | B.PCG_SPARSE, 0, (1e-8,)),
    "stepwise_overshoot": ("rejected_step", False, 1, 0, 0, B.LOCAL4 | B.PCG_SPARSE, (1e-8,)),
}


def check_last_step(st, pb, lin, lam_step, lam_vinv):
    """st: dbg_last_step after one iteration whose candidate was formed at lam_step and whose V~^-1 is held at lam_vinv."""
    ref = E.Elim(pb, lin, lam_step)
    r_p = ref.cand_ratio(st["pts_new"], st["x"], pb.points)
    assert r_p <= 1.0, ("p_new", r_p)
    idle = ~ref.active
    assert np.array_equal(st["pts_new"][idle], pb.points[idle]), "a fixed or unobserved landmark moved"
    rv = ref if lam_vinv == lam_step else E.Elim(pb, lin, lam_vinv)
    X = st["vinv"]
    _, ok = E.spd_inverse3_fp64(rv.Vt64)
    zero = ~(X != 0.0).any(axis=(1, 2))
    assert np.array_equal(zero, idle | ~ok), "V~^-1 is zero somewhere else than where it must be"
    ev = np.linalg.eigvalsh(rv.Vt64[rv.zeroed])        # (never where the exact V~ is positive definite with kappa < 1e12)
    assert not ((ev[:, 0] > 0) & (ev[:, 2] < 1e12 * ev[:, 0])).any()
    assert rv.vinv_ratio(X) <= 1.0, ("V~^-1", rv.vinv_ratio(X))
    return r_p


@pytest.mark.parametrize("path", list(BACKSUB))
@pytest.mark.parametrize("lam", [1e-4, 1e-8])
def test_back_substitution(ctx, path, lam):
    name, large, mode, direct, need, clear, rejects = BACKSUB[path]
    pb, delta = problem(name, large)
    g = BAGraph(ctx, pb)
    if mode:
        g.force_generic_pcg(mode)
    p = g.paths()
    assert p & need == need and not p & clear, (path, p)
    g.reset()
    lin = g.dbg_linearize(delta)
    g.reset()
    r = g.solve(cfg(maxIterations=1, functionTolerance=0.0, lambdaInit=lam, projectErrorHuberThreshold=delta, pcgMaxIterations=500,
                    pcgTolerance=1e-12, linearSolver=direct))
    st = g.dbg_last_step()
    g.close()
    assert r.iterations == 1
    rejected = r.accepted == 0
    if rejects is not None:
        assert rejected == (lam in rejects), (r.accepted, r.initial_cost, r.final_cost)
    if name == "rejected_step":
        assert np.abs(st["x"]).max() > 1e-2, np.abs(st["x"]).max()
    if name == "indefinite_info" and lam <= 1e-4:
        assert st["vinv"][list(ba_graphs.INDEFINITE)].any(axis=(1, 2)).sum() == 0
    assert r.lambda_final == (2.0 * lam if rejected else max(lam / 3.0, 1e-15))
    # the local-BA chain refreshes V~^-1 at the new lambda after a rejection; every other path keeps the lambda of the iteration
    lam_vinv = r.lambda_final if (rejected and p & B.LOCAL4) else lam
    check_last_step(st, pb, lin, lam, lam_vinv)


def test_back_substitution_sharded(ctx):
    """One rank of the landmark-sharded solve: its landmarks' candidates and inverses against a single-GPU graph of its shard."""
    from test_ba_sharded_gpu import on_ranks
    c = ba_graphs.build("long_tracks", True)
    pb, delta, lam, world = c.pb, c.delta, 1e-4, 2
    o = cfg(maxIterations=1, functionTolerance=0.0, lambdaInit=lam, projectErrorHuberThreshold=delta, pcgMaxIterations=500, pcgTolerance=1e-12)
    with group(ctx, world) as (ctxs, comms):
        def rank(r):
            g = ShardedBAGraph(comms[r], pb)
            try:
                return g.solve(o), g.dbg_last_step()
            finally:
                g.close()
        out = on_ranks(world, rank)
    for r in range(world):
        res, st = out[r]
        assert res.iterations == 1 and res.accepted == 1
        assert np.array_equal(st["x"], out[0][1]["x"])
        loc, _ = shard_landmarks(pb, r, world)
        gl = BAGraph(ctx, loc)
        lin = gl.dbg_linearize(delta)
        gl.close()
        check_last_step(st, loc, lin, lam, lam)
