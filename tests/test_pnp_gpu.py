"""GPU parity of gb_pnp_ransac and of Estimator::findPnP through the reference API against oracle/pnp_ref.c.

Bar: same number of counted hypotheses, same winning hypothesis and root, identical inlier mask, pose within 1e-7 (the refinement is an LM solve on both sides: agreement at its convergence level; the minimal
solver runs in fp64 on both sides with contraction disabled; only libm-vs-CUDA-math ulp differences in acos/cos/cbrt can move a
bracket, and the bisection + Newton steps converge to the same root)."""
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from gslam_b200 import capi

pytestmark = pytest.mark.gpu
LIB = oracle.PLUGIN_DIR
EXE = os.path.join(LIB, "gslam_b200_host_test")


def scene(rng, n, outlier_fraction, sigma):
    from scipy.spatial.transform import Rotation as R
    Rg = R.from_rotvec(rng.normal(0, 0.3, 3)).as_matrix(); tg = rng.uniform(-1, 1, 3)
    Xc = np.column_stack([rng.uniform(-4, 4, n), rng.uniform(-3, 3, n), rng.uniform(3, 20, n)])
    Xw = (Xc - tg) @ Rg
    xy = Xc[:, :2] / Xc[:, 2:3] + rng.normal(0, sigma, (n, 2))
    bad = rng.permutation(n)[:int(outlier_fraction * n)]
    xy[bad] = np.column_stack([rng.uniform(-1.3, 1.3, bad.size), rng.uniform(-1, 1, bad.size)])
    return np.ascontiguousarray(Xw), np.ascontiguousarray(xy)


@pytest.mark.parametrize("n,outliers,sigma", [(50, 0.0, 0.0), (200, 0.3, 1 / 718), (2000, 0.5, 1 / 718), (1000, 0.7, 1 / 718), (4, 0.0, 0.0)])
def test_ransac_matches_oracle(ctx, n, outliers, sigma):
    rng = np.random.default_rng(n)
    for rep in range(4):
        Xw, xy = scene(rng, n, outliers, sigma)
        want = oracle.pnp_ransac(Xw, xy, threshold=4 / 718, confidence=0.99, max_hypotheses=1024, seed=rep + 1)
        got = ctx.pnp_ransac(Xw, xy, threshold=4 / 718, confidence=0.99, max_hypotheses=1024, seed=rep + 1)
        for f in ("hypotheses", "best_hypothesis", "best_root", "inliers_minimal", "inliers_refined"):
            assert getattr(got[2], f) == getattr(want[2], f), f
        assert np.array_equal(got[1], want[1])
        assert np.abs(got[0] - want[0]).max() < 1e-7


def test_no_consistent_pose_is_an_error(ctx):
    rng = np.random.default_rng(5)
    Xw = rng.uniform(-5, 5, (100, 3)) + np.array([0, 0, 10.0]); xy = rng.uniform(-1, 1, (100, 2))
    with pytest.raises(capi.GbError):
        ctx.pnp_ransac(Xw, xy, threshold=1e-4, max_hypotheses=256)


def test_find_pnp_through_reference_api():
    """GSLAM::Estimator::create() -> findPnP (Estimator.h:158-164,175-191) via gslam_b200_host_test."""
    if not all(os.path.exists(os.path.join(LIB, f)) for f in ("gslam_b200_host_test", "libgslam_estimator.so")):
        pytest.skip("plugins not built")
    rng = np.random.default_rng(7)
    Xw, xy = scene(rng, 500, 0.4, 1 / 718)
    want = oracle.pnp_ransac(Xw, xy, threshold=4 / 718, confidence=0.99, max_hypotheses=1024, seed=1)  # plugin defaults
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "in.bin"), "wb") as f:
            f.write(struct.pack("<4i", 500, 0, 0, 0)); f.write(struct.pack("<2d", 4 / 718, 0.99)); f.write(Xw.tobytes()); f.write(xy.tobytes())
        r = subprocess.run([EXE, "findpnp", LIB, os.path.join(d, "in.bin"), os.path.join(d, "out.bin")], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        raw = open(os.path.join(d, "out.bin"), "rb").read()
    assert struct.unpack("<i", raw[:4])[0] == 1
    pose = np.frombuffer(raw[4:60], np.float64); mask = np.frombuffer(raw[60:560], np.uint8)
    assert np.abs(pose - want[0]).max() < 1e-7 and np.array_equal(mask, want[1])
