"""The host-buffer entry points when the ctx's pinned staging has to grow, compared byte for byte with the device-resident route.

A ctx is created with 8 MiB of pinned staging (about 10.5 MB with the growth slack).  Every call here stages more than that, so it
grows the staging.  In the extraction, PnP and smaller match cases the staging grows in a later take of a call that has already
taken staging: gb_stage_take then synchronises the stream before it frees the buffer that the earlier take's copies read.  Each
call starts on a fresh ctx, whose staging no earlier test has grown."""
import numpy as np
import pytest

from gslam_b200 import synth
from gslam_b200.api import BAGraph, Context, Features, OptimzeConfig
import pnp_scenes  # (tests/ is on sys.path under pytest's rootdir conftest)

pytestmark = pytest.mark.gpu
BA_FIELDS = ("initial_cost", "final_cost", "iterations", "accepted", "pcg_iterations", "status", "lambda_final")


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


def test_orb_extract_pageable_frame_larger_than_staging(fresh):
    """A pageable 4096x3072 gray frame (12.6 MB) is staged row by row and grows the staging; the download of 65 536 rows (3.9 MB)
    behind it in the same call grows it again."""
    import torch
    img = synth.synth_frame(4096, 3072, seed=11)
    cap = 65536
    kps, desc = fresh().orb_extract(img, 2000, capacity=cap)
    assert len(kps) > 1000
    dev = fresh()
    t = torch.from_numpy(img).cuda()
    torch.cuda.synchronize()  # (the frame is written on torch's stream, read on the ctx's)
    f = Features(dev, cap)
    f.extract(t.data_ptr(), 4096, 3072, dev.orb_cfg(nfeatures=2000), device_ptr=True)
    wk, wd = f.download()
    f.close()
    assert kps.tobytes() == wk.tobytes() and desc.tobytes() == wd.tobytes()


@pytest.mark.parametrize("n", [200_000, 150_000], ids=["grow_on_upload", "grow_on_results"])
def test_match_hamming_larger_than_staging(fresh, n):
    """200 000 query and train rows (12.8 MB) grow the staging with the upload; 150 000 (9.6 MB) fit, and the three result arrays
    taken after them in the same call (1.8 MB) grow it once the upload and the match are enqueued."""
    q = synth.random_descriptors(n, 21)
    t = synth.random_descriptors(n, 22)
    got = fresh().match_hamming(q, t)
    dev = fresh()
    fq, ft = Features(dev, n), Features(dev, n)
    fq.upload(q)
    ft.upload(t)
    fq.match(ft)
    want = fq.matches()
    fq.close(); ft.close()
    for g, w in zip(got, want):
        assert g.tobytes() == w.tobytes()


def test_ba_solve_blob_larger_than_staging(fresh):
    """gb_ba_solve of a 300 000-edge graph, whose upload blob is larger than the staging: cold, then with new estimates and
    measurements through the topology cache, each equal to a resident graph of the same problem on a fresh ctx."""
    c = OptimzeConfig(maxIterations=4, functionTolerance=0.0)
    rng = np.random.default_rng(5)
    pb1 = synth.synth_ba(200, 60_000, obs_per_point=5, n_fixed=2, seed=9)
    pb2 = pb1.copy()
    pb2.cam_pose_wc[2:, 4:] += rng.normal(0, 0.01, pb2.cam_pose_wc[2:, 4:].shape)
    pb2.points += rng.normal(0, 0.02, pb2.points.shape)
    pb2.obs_xyz[:, :2] += rng.normal(0, 1e-4, (pb2.n_obs, 2))
    host = fresh()
    for pb in (pb1, pb2):  # cold, then a cache hit
        got = pb.copy()
        r = host.ba_solve(got, c)
        g = BAGraph(fresh(), pb)
        w = g.solve(c)
        pose, pts = g.download()
        g.close()
        assert [getattr(r, k) for k in BA_FIELDS] == [getattr(w, k) for k in BA_FIELDS]
        assert r.accepted > 0
        assert got.cam_pose_wc.tobytes() == pose.tobytes() and got.points.tobytes() == pts.tobytes()


def test_pnp_ransac_nested_solve_larger_than_staging(fresh):
    """gb_pnp_ransac of 300 000 correspondences: the upload (12 MB) grows the staging, and the optimizePnP solve of its inliers
    (gb_ba_pnp, nested in the same call) grows it again with its upload blob.  The same call on that ctx, whose staging has just
    grown, and on the fresh ctx give the same bytes."""
    from scipy.spatial.transform import Rotation
    n = 300_000
    xyz, xy, Rg, tg = pnp_scenes.scene(np.random.default_rng(7), n, outliers=0.2)
    ctx = fresh()
    first = ctx.pnp_ransac(xyz, xy)
    again = ctx.pnp_ransac(xyz, xy)
    (p0, m0, s0), (p1, m1, s1) = first, again
    assert p0.tobytes() == p1.tobytes() and m0.tobytes() == m1.tobytes() and bytes(s0) == bytes(s1)
    assert s0.inliers_refined >= int(0.8 * n) - 1 and int(m0.sum()) == s0.inliers_refined
    assert np.abs(Rotation.from_quat(p0[:4]).as_matrix() - Rg).max() < 1e-6 and np.abs(p0[4:] - tg).max() < 1e-6
