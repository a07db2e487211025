"""The GSLAM-facing plugins, driven ONLY through the reference's public API by gslam_b200_host_test (a stand-in for a SLAM
plugin): Optimizer::create() -> optimize / optimizePnP, Registry::load("b200") -> orb_extract / match_hamming.
CPU part: discovery + symbol export + the no-device failure convention.  GPU part: plugin-level parity with the oracle."""
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from gslam_b200 import capi, synth

LIB = oracle.PLUGIN_DIR
EXE = os.path.join(LIB, "gslam_b200_host_test")
needs_plugins = pytest.mark.skipif(not all(os.path.exists(os.path.join(LIB, f)) for f in
                                           ("gslam_b200_host_test", "libgslam_optimizer.so", "libgslam_b200.so")),
                                   reason="oracle/_ref/plugins not built (they need the headers of a GSLAM checkout at build time)")


def write_ba(path, pb, iters, ftol, edges=None):
    with open(path, "wb") as f:
        nse = 0 if edges is None else edges.n_se3; ngps = 0 if edges is None else edges.n_gps
        pinfo = 0 if edges is None or edges.se3_info is None else 1
        f.write(struct.pack("<8i", pb.n_cams, pb.n_points, pb.n_obs, iters, 0 if pb.obs_info is None else 1, nse, ngps, pinfo))
        f.write(struct.pack("<d", ftol))
        for a, dt in ((pb.cam_pose_wc, np.float64), (pb.cam_dof, np.uint8), (pb.points, np.float64), (pb.point_free, np.uint8),
                      (pb.obs_cam, np.int32), (pb.obs_point, np.int32), (pb.obs_xyz, np.float64)):
            f.write(np.ascontiguousarray(a, dt).tobytes())
        if pb.obs_info is not None:
            f.write(np.ascontiguousarray(pb.obs_info, np.float64).tobytes())
        if edges is not None:
            for a, dt in ((edges.se3_first, np.int32), (edges.se3_second, np.int32), (edges.se3_meas, np.float64)):
                f.write(np.ascontiguousarray(a, dt).tobytes())
            if pinfo:
                f.write(np.ascontiguousarray(edges.se3_info, np.float64).tobytes())
            for a, dt in ((edges.gps_frame, np.int32), (edges.gps_meas, np.float64)):
                f.write(np.ascontiguousarray(a, dt).tobytes())
            if pinfo:
                f.write(np.ascontiguousarray(edges.gps_info, np.float64).tobytes())


def run(mode, inp, out, *svar_settings):
    return subprocess.run([EXE, mode, LIB, inp, out, *svar_settings], capture_output=True, text=True, timeout=300)


@needs_plugins
def test_exports():
    import ctypes
    o = ctypes.CDLL(os.path.join(LIB, "libgslam_optimizer.so"))
    assert hasattr(o, "createOptimizerInstance")       # Optimizer.h:43-45,241-247
    m = ctypes.CDLL(os.path.join(LIB, "libgslam_b200.so"))
    assert hasattr(m, "svarInstance")                  # Svar.h:71


@needs_plugins
def test_discovery_and_failure_convention_without_gpu():
    """Optimizer::create() must find the plugin; without a device optimize() returns false (no throw, no CPU fallback)."""
    import ctypes
    n = ctypes.c_int(0)
    if capi.lib().gb_device_count(ctypes.byref(n)) == 0 and n.value > 0:
        pytest.skip("GPU present: covered by the gpu tests")
    pb = synth.synth_ba(4, 12, obs_per_point=3, n_fixed=1, seed=1)
    with tempfile.TemporaryDirectory() as d:
        write_ba(os.path.join(d, "in.bin"), pb, 3, 0.0)
        r = run("ba", os.path.join(d, "in.bin"), os.path.join(d, "out.bin"))
        assert r.returncode == 1, (r.returncode, r.stderr)   # 2 would mean create() returned null
        assert "no usable CUDA device" in (r.stderr + r.stdout)
        ok = struct.unpack("<i", open(os.path.join(d, "out.bin"), "rb").read(4))[0]
        assert ok == 0


@needs_plugins
def test_estimator_discovery_and_failure_convention_without_gpu():
    """Estimator::create() must find libgslam_estimator.so (Estimator.h:175-191); without a device findPnP returns false."""
    import ctypes
    if not os.path.exists(os.path.join(LIB, "libgslam_estimator.so")):
        pytest.skip("estimator plugin not built")
    n = ctypes.c_int(0)
    if capi.lib().gb_device_count(ctypes.byref(n)) == 0 and n.value > 0:
        pytest.skip("GPU present: the no-device convention cannot be observed (findPnP on hardware: tests/test_pnp_gpu.py)")
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "in.bin"), "wb") as f:
            f.write(struct.pack("<4i", 20, 0, 0, 0)); f.write(struct.pack("<2d", 0.01, 0.99))
            f.write(rng.normal(size=(20, 3)).tobytes()); f.write(rng.normal(size=(20, 2)).tobytes())
        r = run("findpnp", os.path.join(d, "in.bin"), os.path.join(d, "out.bin"))
        assert r.returncode == 3, (r.returncode, r.stderr)   # 2 would mean create() returned null
        assert "no usable CUDA device" in (r.stderr + r.stdout)
        assert struct.unpack("<i", open(os.path.join(d, "out.bin"), "rb").read(4))[0] == 0


@needs_plugins
@pytest.mark.gpu
def test_optimize_through_reference_api_matches_oracle():
    """BASELINE config 1 (10 cams / 200 pts) + a local-BA window through GSLAM::Optimizer::create()->optimize(BundleGraph&)."""
    for kw, iters in ((dict(n_cams=10, n_points=200, all_visible=True, n_fixed=2, seed=42), 8), (dict(n_cams=50, n_points=2000, obs_per_point=5, n_fixed=2, seed=42), 6)):
        pb = synth.synth_ba(**kw)
        want = pb.copy()
        oracle.ba_solve(want, max_iterations=iters, function_tolerance=0.0)
        with tempfile.TemporaryDirectory() as d:
            write_ba(os.path.join(d, "in.bin"), pb, iters, 0.0)
            r = run("ba", os.path.join(d, "in.bin"), os.path.join(d, "out.bin"))
            assert r.returncode == 0, r.stderr
            raw = open(os.path.join(d, "out.bin"), "rb").read()
        ok = struct.unpack("<i", raw[:4])[0]
        assert ok == 1
        poses = np.frombuffer(raw[4:4 + 64 * pb.n_cams], np.float64).reshape(-1, 8)
        pts = np.frombuffer(raw[4 + 64 * pb.n_cams:], np.float64).reshape(-1, 3)
        s = np.sign(np.sum(poses[:, :4] * want.cam_pose_wc[:, :4], axis=1))[:, None]
        assert np.abs(poses[:, :4] * s - want.cam_pose_wc[:, :4]).max() < 1e-5
        assert np.abs(poses[:, 4:7] - want.cam_pose_wc[:, 4:]).max() < 1e-5 * max(1.0, np.abs(want.cam_pose_wc[:, 4:]).max())
        assert np.abs(pts - want.points).max() < 1e-5 * np.abs(want.points).max()
        assert np.allclose(poses[:, 7], 1.0 + 0.01 * np.arange(pb.n_cams))   # SIM3 scale untouched (UPDATE_KF_SE3)


@needs_plugins
@pytest.mark.gpu
def test_global_ba_sharded_over_all_gpus_through_reference_api():
    """Optimizer::create()->optimize(BundleGraph&) (Optimizer.h:229) with the svar option b200.devices naming every visible GPU:
    the plugin shards the landmarks itself (gb_ba_solve_multi: one NCCL all-reduce of the reduced camera system per LM iteration).
    On a 1-GPU box the option names one device and the call must stay on the single-GPU path with the same result."""
    import ctypes
    n = ctypes.c_int(0)
    assert capi.lib().gb_device_count(ctypes.byref(n)) == 0 and n.value > 0
    ndev = min(n.value, 8)
    pb = synth.synth_ba(n_cams=50, n_points=2000, obs_per_point=5, n_fixed=2, seed=42)  # (the local-BA window of the other tests)
    want = pb.copy()
    oracle.ba_solve(want, max_iterations=6, function_tolerance=0.0)
    with tempfile.TemporaryDirectory() as d:
        write_ba(os.path.join(d, "in.bin"), pb, 6, 0.0)
        r = run("ba", os.path.join(d, "in.bin"), os.path.join(d, "out.bin"), "b200.devices=" + ",".join(str(k) for k in range(ndev)),
                "b200.multi_min_obs=1000")
        assert r.returncode == 0, r.stderr
        raw = open(os.path.join(d, "out.bin"), "rb").read()
    assert struct.unpack("<i", raw[:4])[0] == 1
    poses = np.frombuffer(raw[4:4 + 64 * pb.n_cams], np.float64).reshape(-1, 8)
    pts = np.frombuffer(raw[4 + 64 * pb.n_cams:], np.float64).reshape(-1, 3)
    s_ = np.sign(np.sum(poses[:, :4] * want.cam_pose_wc[:, :4], axis=1))[:, None]
    # same iteration counts on both sides (a long straight trajectory has a very weak scale-drift mode: Krylov solves run "to
    # convergence" on the two sides would differ along it by condition number x tolerance); 1e-4 on the unit quaternions,
    # translations / points relative to the scene scale as in tests/test_dist.py
    assert np.abs(poses[:, :4] * s_ - want.cam_pose_wc[:, :4]).max() < 1e-4
    assert np.abs(poses[:, 4:7] - want.cam_pose_wc[:, 4:]).max() < 1e-5 * max(1.0, np.abs(want.cam_pose_wc[:, 4:]).max())
    assert np.abs(pts - want.points).max() < 1e-5 * np.abs(want.points).max()


@needs_plugins
@pytest.mark.gpu
def test_optimize_pnp_through_reference_api():
    rng = np.random.default_rng(5)
    q = rng.standard_normal(4); q /= np.linalg.norm(q)
    pose = np.concatenate([q, 0.1 * rng.standard_normal(3)])
    cw = np.zeros(7); oracle.lib().orc_se3_inverse(pose.ctypes.data, cw.ctypes.data)
    Rm = synth._quat_to_R(cw[:4])
    pc = np.stack([rng.uniform(-2, 2, 500), rng.uniform(-2, 2, 500), rng.uniform(4, 10, 500)], axis=1)
    xyz = (pc - cw[4:]) @ Rm
    xy1 = np.concatenate([pc[:, :2] / pc[:, 2:3] + 1e-3 * rng.standard_normal((500, 2)), np.ones((500, 1))], axis=1)
    init = pose.copy(); init[4:] += 0.05; init[:4] += 0.01; init[:4] /= np.linalg.norm(init[:4])
    p0, r0, i0 = oracle.ba_pnp(xyz, xy1, init, want_info=True, max_iterations=10, function_tolerance=0.0)
    pb = synth.BAProblem(cam_pose_wc=init[None].copy(), cam_dof=np.array([63], np.uint8), points=xyz.copy(), point_free=np.zeros(500, np.uint8),
                         obs_cam=np.zeros(500, np.int32), obs_point=np.arange(500, dtype=np.int32), obs_xyz=xy1)
    with tempfile.TemporaryDirectory() as d:
        write_ba(os.path.join(d, "in.bin"), pb, 10, 0.0)
        r = run("pnp", os.path.join(d, "in.bin"), os.path.join(d, "out.bin"))
        assert r.returncode == 0, r.stderr
        raw = open(os.path.join(d, "out.bin"), "rb").read()
    got = np.frombuffer(raw[4:4 + 56], np.float64); info = np.frombuffer(raw[60:60 + 288], np.float64).reshape(6, 6)
    if got[3] * p0[3] < 0:
        got = np.concatenate([-got[:4], got[4:]])
    assert np.abs(got - p0).max() < 1e-5
    assert np.abs(info - i0).max() < 1e-6 * np.abs(i0).max()


@needs_plugins
@pytest.mark.gpu
def test_orb_and_match_through_svar_module():
    frames = synth.synth_stream(640, 480, 2, seed=12)
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "in.bin"), "wb") as f:
            f.write(struct.pack("<4i", 640, 480, 500, 0)); f.write(frames[0].tobytes()); f.write(frames[1].tobytes())
        r = run("orb", os.path.join(d, "in.bin"), os.path.join(d, "out.bin"))
        assert r.returncode == 0, r.stderr
        raw = open(os.path.join(d, "out.bin"), "rb").read()
    na, nb = struct.unpack("<2i", raw[:8]); off = 8
    ka = np.frombuffer(raw[off:off + 28 * na], capi.KP_DTYPE); off += 28 * na
    da = np.frombuffer(raw[off:off + 32 * na], np.uint8).reshape(-1, 32); off += 32 * na
    kb = np.frombuffer(raw[off:off + 28 * nb], capi.KP_DTYPE); off += 28 * nb
    db = np.frombuffer(raw[off:off + 32 * nb], np.uint8).reshape(-1, 32); off += 32 * nb
    idx = np.frombuffer(raw[off:off + 4 * nb], np.int32); off += 4 * nb
    d1 = np.frombuffer(raw[off:off + 4 * nb], np.int32); off += 4 * nb
    d2 = np.frombuffer(raw[off:off + 4 * nb], np.int32)
    wa, wda = oracle.orb_extract(frames[0], 500); wb, wdb = oracle.orb_extract(frames[1], 500)
    for got, want in ((ka, wa), (kb, wb)):
        assert len(got) == len(want)
        for fld in ("x", "y", "size", "angle", "response", "octave", "class_id"):
            assert np.array_equal(got[fld], want[fld]), fld
    assert np.array_equal(da, wda) and np.array_equal(db, wdb)
    w = oracle.match_hamming(wdb, wda)
    assert np.array_equal(idx, w[0]) and np.array_equal(d1, w[1]) and np.array_equal(d2, w[2])


@needs_plugins
def test_synth_dataset_frames_equal_python_generator(tmp_path):
    """GSLAM::Dataset::open("x.synth") finds libgslamDB_synth.so through the reference's loader (Dataset.h:124-162,
    GSLAM_REGISTER_DATASET GSLAM.h:35-41) and its frames are bit-identical to gslam_b200.synth.synth_stream.  No GPU involved."""
    if not os.path.exists(os.path.join(LIB, "libgslamDB_synth.so")):
        pytest.skip("dataset plugin not built")
    cfg = tmp_path / "x.synth"
    cfg.write_text("width 320\nheight 240\nframes 3\nseed 5\n")
    out = tmp_path / "out.bin"
    r = run("dataset", str(cfg), str(out))
    assert r.returncode == 0, r.stderr
    raw = open(out, "rb").read()
    n, cams, w, h = struct.unpack("<4i", raw[:16])
    assert (n, cams, w, h) == (3, 1, 320, 240)
    got = np.frombuffer(raw[16:], np.uint8).reshape(n, h, w)
    want = synth.synth_stream(320, 240, 3, seed=5)
    assert np.array_equal(got, want)
    # stereo: two cameras per frame, the right eye displaced by the configured disparity
    cfg.write_text("width 256\nheight 192\nframes 2\nseed 2\nstereo 1\ndisparity 9\n")
    r = run("dataset", str(cfg), str(out))
    assert r.returncode == 0, r.stderr
    raw = open(out, "rb").read()
    n, cams, w, h = struct.unpack("<4i", raw[:16])
    assert (n, cams, w, h) == (2, 2, 256, 192)


@needs_plugins
@pytest.mark.gpu
def test_features_app_over_messenger_matches_direct_calls(tmp_path):
    """The Messenger-level pipeline of SURVEY.md 8f-2, wired like `gslam play b200_features -dataset x.synth`: dataset/frame ->
    gslam.apps.b200_features (ORB extract on the GPU, MapFrame::setKeyPoints, Hamming match against the previous frame) ->
    b200/curframe.  Every frame's keypoints / descriptors / matches equal direct C-ABI calls on the same frames."""
    from gslam_b200.api import Context
    cfg = tmp_path / "x.synth"
    cfg.write_text("width 640\nheight 480\nframes 4\nseed 3\n")
    out = tmp_path / "out.bin"
    r = run("features", str(cfg), str(out), "nfeatures=500")
    assert r.returncode == 0, r.stderr[-2000:]
    raw = open(out, "rb").read()
    n = struct.unpack("<i", raw[:4])[0]
    assert n == 4
    frames = synth.synth_stream(640, 480, 4, seed=3)
    ctx = Context(0)
    off = 4
    prev = None
    for k in range(n):
        fid, nk = struct.unpack("<2i", raw[off:off + 8]); off += 8
        kps = np.frombuffer(raw[off:off + 28 * nk], capi.KP_DTYPE); off += 28 * nk
        desc = np.frombuffer(raw[off:off + 32 * nk], np.uint8).reshape(nk, 32); off += 32 * nk
        nm = struct.unpack("<i", raw[off:off + 4])[0]; off += 4
        idx = np.frombuffer(raw[off:off + 4 * nm], np.int32); off += 4 * nm
        ns = struct.unpack("<i", raw[off:off + 4])[0]; off += 4 + 4 * ns
        k0, d0 = ctx.orb_extract(frames[k], 500)
        assert fid == k + 1 and nk == len(k0) and np.array_equal(kps, k0) and np.array_equal(desc, d0)
        if prev is None:
            assert nm == 0
        else:
            assert np.array_equal(idx, ctx.match_hamming(d0, prev)[0])
        prev = d0
    ctx.close()


@needs_plugins
@pytest.mark.gpu
@pytest.mark.parametrize("ch", [1, 3])
def test_undistort_function_equals_the_reference_undistorter_in_process(tmp_path, ch):
    """gslam.b200.undistort(GImage, Camera, Camera) next to the UNMODIFIED GSLAM::Undistorter (a header: host_test runs both on the
    same frame): every pixel the reference defines is bit-identical, at the benchmark's frame size, for the OpenCV camera model."""
    w, h = 1920, 1080
    cam_in = [w, h, 1400.0, 1402.0, 961.5, 539.25, -0.28, 0.07, 0.0002, 0.00002, 0.0]
    cam_out = [w, h, 1250.0, 1250.0, 960.0, 540.0]
    img = synth.synth_frame(w, h, seed=4)
    if ch == 3:
        img = np.stack([img, np.roll(img, 11, axis=1), 255 - img], axis=2)
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(struct.pack("<8i", w, h, ch, len(cam_in), len(cam_out), 0, 0, 0))
        f.write(np.array(cam_in, np.float64).tobytes()); f.write(np.array(cam_out, np.float64).tobytes())
        f.write(np.ascontiguousarray(img).tobytes())
    r = run("undistort", str(inp), str(out))
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    raw = open(out, "rb").read()
    wo, ho, c, bad = struct.unpack("<4i", raw[:16])
    n = wo * ho * c
    mine = np.frombuffer(raw[16:16 + n], np.uint8).reshape(ho, wo, c)
    want = np.frombuffer(raw[16 + n:16 + 2 * n], np.uint8).reshape(ho, wo, c)
    inside = np.frombuffer(raw[16 + 2 * n:], np.uint8).reshape(ho, wo).astype(bool)
    assert (wo, ho, c, bad) == (w, h, ch, 0)
    assert inside.mean() > 0.9 and np.array_equal(mine[inside], want[inside]) and mine[inside].std() > 10


@needs_plugins
@pytest.mark.gpu
@pytest.mark.parametrize("tree,weighting,scoring,levelsup", [("trained", 0, 0, 0), ("trained", 0, 0, 2), ("synthetic", 1, 1, 1), ("synthetic", 2, 5, 0),
                                                            ("synthetic", 0, 3, 4)])
def test_vocabulary_from_the_module_equals_the_reference_vocabulary_in_process(tmp_path, tree, weighting, scoring, levelsup):
    """gslam.b200.vocabulary(VocabularyPtr) returns a GSLAM::Vocabulary whose virtual batch transforms run on the device.  host_test
    loads a tree into the REFERENCE class with its own binary loader -- the one tests/golden/bow_golden.npz holds (trained by the
    reference's Vocabulary::create) or a synthetic 10^4-word one --, hands it to the module, lets both objects transform the same 2000
    descriptors in one process and compares the BowVector / FeatureVector std::maps with ==: key for key, float for float."""
    from gslam_b200 import synth as S
    if tree == "trained":
        z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bow_golden.npz"))
        k, L, child, weight, desc = int(z["k"]), int(z["L"]), z["child_num"], z["weight"], z["desc"]
    else:
        v = S.synth_vocabulary(10, 4, seed=21, stop=0.05)   # (complete tree: the node id "levelsup levels up" is defined for every word)
        k, L, child, weight, desc = v.k, v.L, v.child_num, v.weight, v.desc
    rng = np.random.default_rng(11)
    nq = 2000
    q = desc[rng.integers(1, desc.shape[0], nq)] ^ np.packbits(rng.random((nq, 256)) < 0.06, axis=1)
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(struct.pack("<8i", k, L, weighting, scoring, child.shape[0], nq, levelsup, 0))
        f.write(np.ascontiguousarray(child, np.uint32).tobytes()); f.write(np.ascontiguousarray(weight, np.float32).tobytes())
        f.write(np.ascontiguousarray(desc, np.uint8).tobytes()); f.write(np.ascontiguousarray(q, np.uint8).tobytes())
    r = run("bow", str(inp), str(out))
    assert r.returncode == 0, (r.returncode, r.stderr[-2000:])
    raw = open(out, "rb").read()
    eq_bow, eq_fv, eq_bow_only, nw, nfv, us_ref, us_dev, _ = struct.unpack("<8i", raw[:32])
    assert (eq_bow, eq_fv, eq_bow_only) == (1, 1, 1)
    assert 50 < nw <= nq and 0 < nfv <= nw
    words = np.frombuffer(raw[32:32 + 8 * nw], np.uint64); values = np.frombuffer(raw[32 + 8 * nw:32 + 12 * nw], np.float32)
    assert np.all(np.diff(words.astype(np.int64)) > 0) and np.all(values > 0)
    # ... and equal to the oracle on the same tree (itself pinned to the reference in tests/test_oracle_bow.py)
    from oracle import oracle as O
    want = O.bow_transform(O.VocabularyArrays(k, L, weighting, scoring, child, weight, desc), q, levelsup)
    assert np.array_equal(words.astype(np.int64), want["words"]) and np.array_equal(values, want["values"])
    print(f"bow transform of {nq} descriptors: reference {us_ref} us, plugin {us_dev} us")


@needs_plugins
@pytest.mark.gpu
@pytest.mark.parametrize("kw,ekw", [(dict(n_cams=20, n_points=300, obs_per_point=4, n_fixed=2, seed=3), dict(seed=1, n_loops=5, gps_every=4, with_info=True)),
                                    (dict(n_cams=40, n_points=0, n_fixed=1, seed=7, pose_sigma_t=0.05, pose_sigma_deg=0.5), dict(seed=2, n_loops=12, gps_every=0, with_info=False))])
def test_pose_graph_edges_through_reference_api(kw, ekw):
    """BundleGraph::se3Graph / gpsGraph (Optimizer.h:163-168) through GSLAM::Optimizer::create()->optimize(BundleGraph&): a bundle
    adjustment with odometry / loop-closure / GPS terms and a pure POSEGRAPH, against the oracle after the same iteration counts."""
    pb = synth.synth_ba(**kw)
    pe = synth.synth_pose_edges(pb, **ekw)
    want = pb.copy()
    r0 = oracle.ba_solve(want, pe, max_iterations=8, function_tolerance=0.0)
    with tempfile.TemporaryDirectory() as d:
        write_ba(os.path.join(d, "in.bin"), pb, 8, 0.0, pe)
        r = run("ba", os.path.join(d, "in.bin"), os.path.join(d, "out.bin"))
        assert r.returncode == 0, r.stderr
        raw = open(os.path.join(d, "out.bin"), "rb").read()
    assert struct.unpack("<i", raw[:4])[0] == 1
    poses = np.frombuffer(raw[4:4 + 64 * pb.n_cams], np.float64).reshape(-1, 8)
    sgn = np.sign(np.sum(poses[:, :4] * want.cam_pose_wc[:, :4], axis=1))[:, None]
    assert np.abs(poses[:, :4] * sgn - want.cam_pose_wc[:, :4]).max() < 1e-5
    assert np.abs(poses[:, 4:7] - want.cam_pose_wc[:, 4:]).max() < 1e-5 * max(1.0, np.abs(want.cam_pose_wc[:, 4:]).max())
    assert r0.final_cost < r0.initial_cost
    moved = np.abs(poses[:, 4:7] - pb.cam_pose_wc[:, 4:]).max()
    assert moved > 1e-4        # the graph was really optimised
