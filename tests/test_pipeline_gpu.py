"""The tracking / mapping pipeline that bench.py times, checked for what it computes.

bench.py drives two contexts on one device from two host threads: a tracking ctx extracts ORB features from device-resident
1920x1080 frames into two reused `Features` and matches each frame against the previous one without a host round trip, and a
high-priority mapping ctx solves local BA windows, ordered after the tracking stream with `gb_ctx_wait_for`.  The header promises
that one ctx per calling thread is safe (include/gslam_b200.h: tracking does extract / match / PnP, mapping does local BA).  These
tests run that arrangement and compare every output with the oracle or with the same call on a lone ctx:

* device frames with a row pitch (torch tensors, column slices of wider tensors) and host frames with a pitch, pageable and pinned;
* the bench's tracking loop on one ctx and pipelined against a mapping thread, with and without downloads between steps;
* the mapping side under that load, on resident graphs and through the host-buffer entry points (topology cache, PnP in between);
* the host-buffer end-to-end pipeline from two threads;
* gb_ctx_wait_for carrying a real data dependency between two contexts (the stepwise BA on caller-owned buffers);
* first use of the process-wide kernel state from several threads at once, in a fresh process.

Extraction and match results must equal the oracle in every keypoint field and descriptor bit; BA results must equal a lone
solve bit for bit (DESIGN.md section 5: every reduction has a fixed order) and the oracle within 1e-5.

Frames handed over by device pointer are read on the library's own stream.  Whoever wrote them on another stream (here torch's)
must synchronise that stream before the call: the library cannot know about the writer.
"""
import os
import queue
import subprocess
import sys
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oracle
from gslam_b200 import capi, synth
from gslam_b200.api import BAGraph, Context, Features, OptimzeConfig

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("octave", "x", "y", "size", "angle", "response", "class_id")
RESULT_FIELDS = ("initial_cost", "final_cost", "iterations", "accepted", "pcg_iterations", "status", "lambda_final")

# bench.py's timed step: 1920x1080, 2000 keypoints, two feature sets of 2 * 2000 + 256 rows, a ring of np.roll-shifted copies of
# eight synth_stream frames (seed 7), the 50-keyframe window with 10 LM iterations and a 50-iteration PCG cap
W, H, NKP = 1920, 1080, 2000
CAP = 2 * NKP + 256
RING = 10   # the oracle needs about a second per 1080p frame on one core: ten distinct frames keep the file well under a minute
STEPS = 10
BA_CFG = OptimzeConfig(maxIterations=10, functionTolerance=0.0, pcgMaxIterations=50, pcgTolerance=1e-10)
WINDOWS = [dict(n_cams=50, n_points=2000, obs_per_point=5, seed=42, n_fixed=2),   # the bench's window
           dict(n_cams=40, n_points=1500, obs_per_point=6, seed=7, n_fixed=2)]


def assert_features(kps, desc, wk, wd, what=""):
    assert len(kps) == len(wk), (what, len(kps), len(wk))
    for f in FIELDS:
        assert np.array_equal(kps[f], wk[f]), (what, f)
    assert np.array_equal(desc, wd), what


def assert_matches(got, want, what=""):
    for g, w, name in zip(got, want, ("idx", "d1", "d2")):
        assert np.array_equal(g, w), (what, name)


def result(r):
    return tuple(getattr(r, f) for f in RESULT_FIELDS)


def oracle_extract_all(frames, n):
    oracle.orb_extract(np.zeros((64, 64), np.uint8), 10)  # binds the oracle's ctypes signatures before the threads use them
    with ThreadPoolExecutor(max(1, min(len(frames), os.cpu_count() or 1))) as ex:  # the oracle releases the GIL
        return list(ex.map(lambda f: oracle.orb_extract(f, n), frames))


# ---- fixtures ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ring_host():
    base = synth.synth_stream(W, H, 8, seed=7)
    return [np.ascontiguousarray(np.roll(base[k % 8], shift=(k // 8) * 7, axis=1)) for k in range(RING)]


@pytest.fixture(scope="module")
def ring_dev(ring_host):
    import torch
    t = torch.empty((RING, H, W), dtype=torch.uint8, device="cuda")
    for k in range(RING):
        t[k] = torch.from_numpy(ring_host[k]).cuda()
    torch.cuda.synchronize()  # the library reads the ring on its own streams
    return t


@pytest.fixture(scope="module")
def ring_oracle(ring_host):
    return oracle_extract_all(ring_host, NKP)


@pytest.fixture(scope="module")
def lone_windows():
    """Each window solved on a ctx of its own with nothing else running: (result, poses, points)."""
    c = Context(0)
    out = []
    for kw in WINDOWS:
        g = BAGraph(c, synth.synth_ba(**kw))
        r = g.solve(BA_CFG)
        out.append((result(r),) + g.download())
        g.close()
    c.close()
    return out


def pnp_case(seed):
    """An optimizePnP problem: 1500 points in front of a camera, 1e-3 noise, every 50th correspondence an outlier."""
    rng = np.random.default_rng(seed)
    q = rng.standard_normal(4); q /= np.linalg.norm(q)
    pose = np.concatenate([q, 0.1 * rng.standard_normal(3)])
    cw = np.zeros(7); oracle.lib().orc_se3_inverse(pose.ctypes.data, cw.ctypes.data)
    pc = np.stack([rng.uniform(-2, 2, 1500), rng.uniform(-2, 2, 1500), rng.uniform(4, 10, 1500)], axis=1)
    xyz = (pc - cw[4:]) @ synth._quat_to_R(cw[:4])
    xy1 = np.concatenate([pc[:, :2] / pc[:, 2:3] + 1e-3 * rng.standard_normal((1500, 2)), np.ones((1500, 1))], axis=1)
    xy1[::50, :2] += 0.2
    init = pose.copy(); init[4:] += 0.05; init[:4] += 0.01; init[:4] /= np.linalg.norm(init[:4])
    return xyz, xy1, init


def host_mapping_sequence():
    """A sliding window through gb_ba_solve: the same topology with new estimates (cache hits), a changed mask and another window
    (misses), optimizePnP calls in between (each drops the ctx's cached graph)."""
    rng = np.random.default_rng(3)
    pb1 = synth.synth_ba(**WINDOWS[0])
    pb2 = pb1.copy()
    pb2.cam_pose_wc[2:, 4:] += rng.normal(0, 0.01, pb2.cam_pose_wc[2:, 4:].shape)
    pb2.points += rng.normal(0, 0.02, pb2.points.shape)
    pb2.obs_xyz[:, :2] += rng.normal(0, 1e-4, (pb2.n_obs, 2))
    pb3 = pb2.copy(); pb3.point_free[5] = 0
    pb4 = synth.synth_ba(**WINDOWS[1])
    return [("ba", pb1), ("ba", pb2), ("pnp", pnp_case(1)), ("ba", pb2), ("ba", pb3), ("pnp", pnp_case(2)), ("ba", pb4), ("ba", pb1)]


HOST_BA_CFG = OptimzeConfig(maxIterations=6, functionTolerance=0.0)
PNP_CFG = OptimzeConfig(maxIterations=10, functionTolerance=0.0)


def run_host_item(c, item):
    kind, x = item
    if kind == "ba":
        pb = x.copy()
        r = c.ba_solve(pb, HOST_BA_CFG)
        return result(r), pb.cam_pose_wc, pb.points
    xyz, xy1, init = x
    pose, r, info = c.ba_pnp(xyz, xy1, init, want_info=True, cfg=PNP_CFG)
    return result(r), pose, info


def assert_same_outputs(got, want, what=""):
    assert len(got) == len(want), what
    for k, (a, b) in enumerate(zip(got, want)):
        assert a[0] == b[0], (what, k, a[0], b[0])
        for x, y in zip(a[1:], b[1:]):
            assert np.array_equal(x, y), (what, k)


@pytest.fixture(scope="module")
def host_sequence():
    seq = host_mapping_sequence()
    c = Context(0)
    want = [run_host_item(c, it) for it in seq]
    c.close()
    return seq, want


class Mapper:
    """The mapping thread of bench.py's run_pipelined: one job per tracking step from a queue of two, results in order.  After a
    failure it keeps draining the queue so that the tracking thread never blocks on it; the failure is raised by join()."""

    def __init__(self, job):
        self.q = queue.Queue(maxsize=2)
        self.out, self.err = [], []
        self.th = threading.Thread(target=self._run, args=(job,), daemon=True)
        self.th.start()

    def _run(self, job):
        while True:
            k = self.q.get()
            if k is None:
                return
            if self.err:
                continue
            try:
                self.out.append(job(k))
            except Exception as e:
                self.err.append(e)

    def put(self, k):
        self.q.put(k)

    def join(self):
        self.q.put(None)
        self.th.join()
        if self.err:
            raise self.err[0]
        return self.out


def stale_rows(ring_oracle):
    """CAP descriptor rows taken in turn from every frame of the ring: loaded into both feature sets before the loop, they stay
    behind every extraction's count, where a match that read past the device-side count would find exact copies of its queries."""
    d = [w[1] for w in ring_oracle]
    return np.stack([d[i % RING][(i // RING) % len(d[i % RING])] for i in range(CAP)])


def track(ctx, feats, ring_dev, steps, download, stale, after_match=None):
    """bench.py's track(k) for k = 0 .. steps - 1, frame k - 1 extracted first: extract(k) into feats[k & 1], match against
    feats[(k + 1) & 1], no host synchronisation in between.  With `download`, the tracking thread reads each frame's features and
    matches right after its match (which synchronises the tracking stream only)."""
    cfg = ctx.orb_cfg(nfeatures=NKP)
    for f in feats:
        f.upload(stale)
    feats[1].extract(ring_dev[(-1) % RING].data_ptr(), W, H, cfg, device_ptr=True, pitch=W)
    out = {}
    for k in range(steps):
        f, fp = feats[k & 1], feats[(k + 1) & 1]
        f.extract(ring_dev[k % RING].data_ptr(), W, H, cfg, device_ptr=True, pitch=W)
        f.match(fp)
        if after_match:
            after_match(k)
        if download:
            out[k] = f.download() + (f.matches(),)
    return out


def check_step(k, got, ring_oracle):
    kps, desc, m = got
    wk, wd = ring_oracle[k % RING]
    assert_features(kps, desc, wk, wd, f"frame {k}")
    assert_matches(m, oracle.match_hamming(wd, ring_oracle[(k - 1) % RING][1]), f"match {k}")


# ---- 1. device frames with a pitch, host frames with a pitch ---------------------------------------------------------------------
def _extract_device(ctx, t, width, height, pitch, n):
    import torch
    torch.cuda.synchronize()  # the caller's side of the contract: the frame is written on torch's stream, read on the ctx's
    f = Features(ctx, 2 * n + 256)
    f.extract(t.data_ptr(), width, height, ctx.orb_cfg(nfeatures=n), device_ptr=True, pitch=pitch)
    kps, desc = f.download()
    f.close()
    return kps, desc


def test_device_frame_dense(ctx):
    import torch
    img = synth.synth_frame(517, 389, seed=31)
    t = torch.from_numpy(img).cuda()
    assert_features(*_extract_device(ctx, t, 517, 389, 517, 350), *oracle.orb_extract(img, 350))


@pytest.mark.parametrize("pitch", [640, 523])
def test_device_frame_column_slice_with_pitch(ctx, pitch):
    """A 517-column slice of a wider tensor: the rows start `pitch` bytes apart and the columns past the slice hold other data."""
    import torch
    img = synth.synth_frame(517, 389, seed=32)
    wide = torch.from_numpy(np.random.default_rng(pitch).integers(0, 256, (389, pitch), dtype=np.uint8)).cuda()
    wide[:, :517] = torch.from_numpy(img).cuda()
    view = wide[:, :517]
    assert view.stride(0) == pitch and not view.is_contiguous()
    assert_features(*_extract_device(ctx, view, 517, 389, pitch, 350), *oracle.orb_extract(img, 350))


def test_device_frame_bench_size(ctx, ring_dev, ring_oracle):
    assert_features(*_extract_device(ctx, ring_dev[3], W, H, W, NKP), *ring_oracle[3])


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("pitch", [640, 523])
def test_host_frame_with_pitch(ctx, pinned, pitch):
    """The host-pointer path with pitch > width: pageable rows are staged one by one, pinned ones go over in one 2-D copy."""
    import torch
    img = synth.synth_frame(517, 389, seed=33)
    wide = np.random.default_rng(pitch + 1).integers(0, 256, (389, pitch), dtype=np.uint8)
    wide[:, :517] = img
    if pinned:
        t = torch.from_numpy(wide).pin_memory()
        assert t.is_pinned()
        wide = t.numpy()
    f = Features(ctx, 956)
    f.extract(wide, 517, 389, ctx.orb_cfg(nfeatures=350), pitch=pitch)
    kps, desc = f.download()
    f.close()
    assert_features(kps, desc, *oracle.orb_extract(img, 350))


# ---- 2 + 3. the bench's tracking loop, alone and against a mapping thread ------------------------------------------------------
@pytest.mark.parametrize("mode", ["one_ctx", "graphs", "graphs_no_download", "host_buffers"])
def test_tracking_loop(mode, ring_dev, ring_oracle, lone_windows, host_sequence):
    """STEPS steps of bench.py's tracking loop, each frame's features and matches bit-exact against the oracle.
    one_ctx: the tracking ctx alone.  graphs: run_pipelined -- a high-priority mapping ctx on a second thread re-solves two resident
    windows in turn (BAGraph.reset + solve), ordered after each match by ctx_m.wait_for(ctx); every solve must equal the lone solve
    of its window bit for bit.  graphs_no_download: the same with nothing read back until the end, so that every match reads both
    keypoint counts on the device; only the last frame is checked, as bench.py --dump-outputs sees it.  host_buffers: the mapping
    thread runs the host-buffer sliding window (gb_ba_solve with its topology cache, gb_ba_pnp in between) instead.  Both feature
    sets start with stale rows past every count (stale_rows)."""
    ctx = Context(0)
    feats = [Features(ctx, CAP), Features(ctx, CAP)]
    ctx_m = mapper = graphs = None
    if mode != "one_ctx":
        ctx_m = Context(0, high_priority=True)
        if mode == "host_buffers":
            seq, want_seq = host_sequence
            mapper = Mapper(lambda k: run_host_item(ctx_m, seq[k % len(seq)]))
        else:
            graphs = [BAGraph(ctx_m, synth.synth_ba(**kw)) for kw in WINDOWS]

            def solve(k):
                g = graphs[k & 1]
                g.reset()
                r = g.solve(BA_CFG)
                return (k & 1, result(r)) + g.download()
            mapper = Mapper(solve)

    def after_match(k):
        ctx_m.wait_for(ctx)  # BA(k) after match(k); extract(k + 1) does not wait for BA(k)
        mapper.put(k)
    try:
        got = track(ctx, feats, ring_dev, STEPS, download=mode != "graphs_no_download", stale=stale_rows(ring_oracle),
                    after_match=after_match if mapper else None)
    finally:
        mapped = mapper.join() if mapper else []
    if mode == "graphs_no_download":
        last = STEPS - 1
        f = feats[last & 1]
        got = {last: f.download() + (f.matches(),)}
    for k, v in got.items():
        check_step(k, v, ring_oracle)
    if mode == "host_buffers":
        assert_same_outputs(mapped, [want_seq[k % len(seq)] for k in range(STEPS)], "host-buffer mapping")
    elif graphs:
        assert len(mapped) == STEPS
        for w, res, poses, points in mapped:
            want = lone_windows[w]
            assert res == want[0], (w, res, want[0])
            assert np.array_equal(poses, want[1]) and np.array_equal(points, want[2]), w
        for g in graphs:
            g.close()
    for f in feats:
        f.close()
    ctx.close()
    if ctx_m:
        ctx_m.close()


def test_lone_window_matches_oracle(lone_windows):
    """The bench's window, solved alone (and so, by test_tracking_loop, under load), against oracle/ba_ref.c after the same LM and
    PCG iteration counts."""
    pb = synth.synth_ba(**WINDOWS[0])
    r0 = oracle.ba_solve(pb, max_iterations=BA_CFG.maxIterations, function_tolerance=0.0, pcg_max_iters=BA_CFG.pcgMaxIterations,
                         pcg_tol=BA_CFG.pcgTolerance)
    res, poses, points = lone_windows[0]
    got = dict(zip(RESULT_FIELDS, res))
    assert got["iterations"] == r0.iterations and got["accepted"] == r0.accepted
    assert abs(got["final_cost"] - r0.final_cost) / r0.final_cost < 1e-5
    s = np.sign(np.sum(poses[:, :4] * pb.cam_pose_wc[:, :4], axis=1))[:, None]
    assert np.abs(poses[:, :4] * s - pb.cam_pose_wc[:, :4]).max() < 1e-5
    assert np.abs(poses[:, 4:] - pb.cam_pose_wc[:, 4:]).max() < 1e-5 * max(1.0, np.abs(pb.cam_pose_wc[:, 4:]).max())
    assert np.abs(points - pb.points).max() / np.abs(pb.points).max() < 1e-5


# ---- 4. host-buffer end to end from two threads -----------------------------------------------------------------------------
def _pnp_scene(k):
    rng = np.random.default_rng(100 + k)
    from scipy.spatial.transform import Rotation as R
    Rg = R.from_rotvec(rng.normal(0, 0.3, 3)).as_matrix(); tg = rng.uniform(-1, 1, 3)
    Xc = np.column_stack([rng.uniform(-4, 4, 800), rng.uniform(-3, 3, 800), rng.uniform(3, 20, 800)])
    xy = Xc[:, :2] / Xc[:, 2:3] + rng.normal(0, 1 / 718, (800, 2))
    bad = rng.permutation(800)[:240]
    xy[bad] = np.column_stack([rng.uniform(-1.3, 1.3, 240), rng.uniform(-1, 1, 240)])
    return np.ascontiguousarray((Xc - tg) @ Rg), np.ascontiguousarray(xy)


PNP_KW = dict(threshold=4 / 718, confidence=0.99, max_hypotheses=512)


def _e2e(frames, seq, scenes, threaded):
    """bench.py's e2e_pipelined (threaded) or the same calls on one thread: tracking does orb_extract + match_hamming + pnp_ransac
    on host frames, mapping does ba_solve / ba_pnp, each on its own ctx."""
    ctx, ctx_m = Context(0), Context(0, high_priority=True)
    mapper = Mapper(lambda k: run_host_item(ctx_m, seq[k])) if threaded else None
    tracked, mapped = [], []
    try:
        prev = ctx.orb_extract(frames[-1], NKP)[1]
        for k, img in enumerate(frames):
            kps, desc = ctx.orb_extract(img, NKP)
            m = ctx.match_hamming(desc, prev)
            prev = desc
            Xw, xy = scenes[k]
            pose, mask, st = ctx.pnp_ransac(Xw, xy, seed=k + 1, **PNP_KW)
            tracked.append((kps, desc, m, pose, mask, tuple(getattr(st, f) for f, _ in st._fields_)))
            if threaded:
                mapper.put(k)
            else:
                mapped.append(run_host_item(ctx_m, seq[k]))
    finally:
        if threaded:
            mapped = mapper.join()
    ctx.close(); ctx_m.close()
    return tracked, mapped


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
def test_host_buffer_pipeline_two_threads(pinned, ring_host, ring_oracle, host_sequence):
    import torch
    frames = [np.array(ring_host[k], copy=True) for k in range(8)]
    if pinned:
        keep = [torch.from_numpy(f).pin_memory() for f in frames]
        frames = [t.numpy() for t in keep]
    seq, want_seq = host_sequence
    scenes = [_pnp_scene(k) for k in range(len(frames))]
    tracked, mapped = _e2e(frames, seq, scenes, threaded=True)
    tracked1, mapped1 = _e2e(frames, seq, scenes, threaded=False)
    assert_same_outputs(mapped, want_seq[:len(frames)], "mapping thread")
    assert_same_outputs(mapped1, want_seq[:len(frames)], "one thread")
    for k, (a, b) in enumerate(zip(tracked, tracked1)):
        assert_features(a[0], a[1], b[0], b[1], f"frame {k} vs one thread")
        assert_matches(a[2], b[2], f"match {k} vs one thread")
        assert np.array_equal(a[3], b[3]) and np.array_equal(a[4], b[4]) and a[5] == b[5], k
    for k, (kps, desc, m, pose, mask, st) in enumerate(tracked):
        assert_features(kps, desc, *ring_oracle[k], f"frame {k}")
        assert_matches(m, oracle.match_hamming(desc, ring_oracle[(k - 1) % 8][1]), f"match {k}")
        # tests/test_pnp_gpu.py's bar: same hypotheses, winner and root, same inlier mask, pose within 1e-7
        wp, wm, ws = oracle.pnp_ransac(*scenes[k], seed=k + 1, **PNP_KW)
        assert st == tuple(getattr(ws, f) for f, _ in ws._fields_), k
        assert np.array_equal(mask, wm) and np.abs(pose - wp).max() < 1e-7, k


# ---- 5. gb_ctx_wait_for with a real data dependency ------------------------------------------------------------------------
def test_wait_for_orders_a_handoff_between_contexts():
    """Two graphs of the same problem on two contexts run the stepwise LM on caller-owned buffers and swap them: each graph reduces
    into its own buffer (gb_ba_graph_reduce_local writes S, g~, diag U and the current cost there, and prepares the graph's own
    per-landmark state), then steps and commits from the OTHER graph's buffer (gb_ba_graph_step damps the diagonal of S in place and
    writes the candidate cost into its own cost word; commit reads the buffer's cost and that word).  Only gb_ctx_wait_for orders
    the contexts: each waits for the other after the reductions (read after write) and after the commits (the next reduction
    overwrites a buffer the other side has just read).  The producer's stream is held back by a sleep before it writes, so a wait
    that does not hold shows up as a step on stale data.  Both graphs must end bit-identical to a solve on one ctx."""
    import torch
    pb = synth.synth_ba(**WINDOWS[0])
    c = OptimzeConfig(maxIterations=6, functionTolerance=0.0)
    lone = Context(0)
    gl = BAGraph(lone, pb)
    gl.force_generic_pcg(1)  # the dense reduced layout: what the stepwise interface exchanges
    want = result(gl.solve(c)); wp, wx = gl.download()
    gl.close(); lone.close()

    ca, cb = Context(0), Context(0)
    ga, gb = BAGraph(ca, pb), BAGraph(cb, pb)
    ga.force_generic_pcg(1); gb.force_generic_pcg(1)
    n = ga.reduce_size()
    buf_a = torch.zeros(n, dtype=torch.float64, device="cuda"); buf_b = torch.zeros(n, dtype=torch.float64, device="cuda")
    cost_a = torch.zeros(1, dtype=torch.float64, device="cuda"); cost_b = torch.zeros(1, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()  # (allocated and zeroed on torch's stream)
    sa, sb = torch.cuda.ExternalStream(ca.stream()), torch.cuda.ExternalStream(cb.stream())

    def hold(s):  # about a millisecond of nothing on stream s
        with torch.cuda.stream(s):
            torch.cuda._sleep(2_000_000)
    ga.begin(c); gb.begin(c)
    for it in range(c.maxIterations):
        hold(sa if it % 2 == 0 else sb)
        ga.reduce_local(buf_a.data_ptr())
        gb.reduce_local(buf_b.data_ptr())
        cb.wait_for(ca); ca.wait_for(cb)
        gb.step(buf_a.data_ptr(), cost_b.data_ptr()); gb.commit(buf_a.data_ptr(), cost_b.data_ptr())
        ga.step(buf_b.data_ptr(), cost_a.data_ptr()); ga.commit(buf_b.data_ptr(), cost_a.data_ptr())
        ca.wait_for(cb); cb.wait_for(ca)
    got_a, got_b = result(ga.finish()), result(gb.finish())
    pa, xa = ga.download(); pb_, xb = gb.download()
    ga.close(); gb.close(); ca.close(); cb.close()
    assert got_b == want and got_a == want, (got_a, got_b, want)
    assert np.array_equal(pb_, wp) and np.array_equal(xb, wx)
    assert np.array_equal(pa, wp) and np.array_equal(xa, wx)


def test_wait_for_argument_rules(ctx):
    L = capi.lib()
    other = Context(0)
    ctx.wait_for(ctx)          # waiting for oneself is a no-op
    ctx.wait_for(other); other.wait_for(ctx)
    assert L.gb_ctx_wait_for(ctx.handle, None) == capi.GB_ERR_INVALID
    assert L.gb_ctx_wait_for(None, ctx.handle) == capi.GB_ERR_INVALID
    assert L.gb_ctx_wait_for(None, None) == capi.GB_ERR_INVALID
    other.sync(); other.close()


# ---- 6. first use of the process-wide state from several threads ---------------------------------------------------------------
FIRST_USE = r"""
import sys, threading
import numpy as np
sys.path.insert(0, sys.argv[1])
from gslam_b200 import synth
from gslam_b200.api import BAGraph, Context, OptimzeConfig
out = sys.argv[2]
small, mid = synth.synth_frame(640, 480, seed=41), synth.synth_frame(1280, 720, seed=42)
local, large = synth.synth_ba(50, 2000, 5, seed=42, n_fixed=2), synth.synth_ba(120, 12000, 8, seed=6, n_fixed=2)
ctxs = [Context(0), Context(0), Context(0, high_priority=True), Context(0)]
go = threading.Barrier(4)
err = []

def extract(i, img, n, name):
    go.wait()
    kps, desc = ctxs[i].orb_extract(img, n)
    np.savez(f"{out}/{name}.npz", kps=kps, desc=desc)

def ba(i, pb, cfg, name):
    go.wait()
    g = BAGraph(ctxs[i], pb)
    r = g.solve(cfg)
    p, x = g.download()
    np.savez(f"{out}/{name}.npz", poses=p, points=x, paths=g.paths(),
             res=np.array([r.initial_cost, r.final_cost, r.iterations, r.accepted, r.pcg_iterations, r.status, r.lambda_final]))

def run(fn, *a):
    try:
        fn(*a)
    except BaseException as e:
        err.append(repr(e))
        go.abort()

th = [threading.Thread(target=run, args=a) for a in (
    (extract, 0, small, 500, "small"), (extract, 1, mid, 1000, "mid"),
    (ba, 2, local, OptimzeConfig(maxIterations=10, functionTolerance=0.0, pcgMaxIterations=50, pcgTolerance=1e-10), "local"),
    (ba, 3, large, OptimzeConfig(maxIterations=3, functionTolerance=0.0, pcgMaxIterations=30), "large"))]
for t in th:
    t.start()
for t in th:
    t.join()
if err:
    sys.exit("; ".join(err))
print("ok")
"""


def test_first_use_from_four_threads_in_a_fresh_process(ctx, tmp_path):
    """The kernel attribute table (gb_func_setup) and the tensor-map encoder of the ORB path are set on first use and shared by
    every ctx of the process; in this process they are set long ago.  A fresh process creates four contexts and starts one thread
    per ctx at once: extractions at two frame sizes, a local BA and a large-graph BA (block-CSR PCG in a thread-block cluster).
    Each result must equal the same call made here."""
    r = subprocess.run([sys.executable, "-c", FIRST_USE, ROOT, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout + r.stderr
    for name, seed, w, h, n in (("small", 41, 640, 480, 500), ("mid", 42, 1280, 720, 1000)):
        got = np.load(tmp_path / f"{name}.npz")
        kps, desc = ctx.orb_extract(synth.synth_frame(w, h, seed=seed), n)
        assert_features(got["kps"], got["desc"], kps, desc, name)
    for name, pb, c in (("local", synth.synth_ba(50, 2000, 5, seed=42, n_fixed=2), BA_CFG),
                        ("large", synth.synth_ba(120, 12000, 8, seed=6, n_fixed=2),
                         OptimzeConfig(maxIterations=3, functionTolerance=0.0, pcgMaxIterations=30))):
        got = np.load(tmp_path / f"{name}.npz")
        g = BAGraph(ctx, pb)
        res = g.solve(c)
        p, x = g.download()
        paths = g.paths()
        g.close()
        assert int(got["paths"]) == paths, name
        if name == "large":
            assert paths & BAGraph.PCG_BCSR and paths & BAGraph.BCSR_CLUSTER, paths
        assert np.array_equal(got["res"], np.array(result(res), np.float64)), name
        assert np.array_equal(got["poses"], p) and np.array_equal(got["points"], x), name
