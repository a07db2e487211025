"""Frame undistortion (SURVEY.md section 8f-4): the oracle's restatement of the bilinear LUT remap against the UNMODIFIED reference
(GSLAM::Undistorter through oracle/_ref, GSLAM/core/Undistorter.h:120-348) -- tables from the reference's prepareReMap, image from
the reference's undistort(), byte for byte."""
import numpy as np
import pytest

import oracle
from gslam_b200 import synth

W, H = 320, 240
PINHOLE = [W, H, 250.0, 251.0, 160.5, 119.25]
OPENCV = [W, H, 250.0, 251.0, 160.5, 119.25, -0.28, 0.07, 0.0002, 0.00002, 0.0]   # k1 k2 p1 p2 k3 (Camera.h:435-444)
ATAN = [W, H, 256.0, 252.0, 160.0, 120.0, 0.9]                                   # PTAM model: fx fy cx cy, w


def _need_ref():
    if not oracle.have_ref():
        pytest.skip("oracle/_ref not built (needs a GSLAM checkout)")


def _frame(ch):
    g = synth.synth_frame(W, H, seed=3)
    if ch == 1:
        return g
    rng = np.random.default_rng(0)
    return np.stack([g, np.roll(g, 5, axis=1), rng.integers(0, 256, g.shape, dtype=np.uint8)], axis=2)


@pytest.mark.parametrize("cam_in,cam_out", [(OPENCV, PINHOLE), (ATAN, PINHOLE), (PINHOLE, [200, 150, 180.0, 180.0, 100.0, 75.0])])
@pytest.mark.parametrize("ch", [1, 3])
def test_remap_restatement_equals_reference_undistort(cam_in, cam_out, ch):
    _need_ref()
    img = _frame(ch)
    idx4, coef4, rx, ref_out = oracle.ref_undistort(cam_in, cam_out, img)
    ho, wo = int(cam_out[1]), int(cam_out[0])
    mine = oracle.remap_apply(img, idx4, coef4, rx, (ho, wo))
    inside = (rx >= 0) if ch == 1 else (rx > 0)
    assert inside.mean() > 0.5          # the comparison is not vacuous
    if ch == 1:
        assert np.array_equal(mine, ref_out)                       # every pixel (outside ones are 0 in the reference too)
    else:
        m = inside.reshape(ho, wo)                                 # the reference leaves multi-channel outside pixels uninitialised
        assert np.array_equal(mine[m], ref_out[m])
        assert not mine[~m].any()
    assert mine[inside.reshape(ho, wo)].std() > 10                 # and it is an image, not a constant


def test_remap_identity_cameras_reproduce_the_frame():
    _need_ref()
    img = _frame(1)
    idx4, coef4, rx, out = oracle.ref_undistort(PINHOLE, PINHOLE, img)
    assert np.array_equal(out, img) and np.array_equal(oracle.remap_apply(img, idx4, coef4, rx, (H, W)), img)


def test_remap_last_row_taps_count_as_zero():
    """Taps beyond the input image (the reference reads past its buffer there) contribute 0: a table that points every tap one row
    below the last row gives 0, and a table whose first tap is valid keeps only that tap."""
    img = np.full((4, 4), 200, np.uint8)
    idx4 = np.tile(np.array([[15, 16, 19, 20]], np.int32), (16, 1))
    coef4 = np.tile(np.array([[0.5, 0.25, 0.125, 0.125]], np.float32), (16, 1))
    out = oracle.remap_apply(img, idx4, coef4, np.ones(16, np.float32), (4, 4))
    assert (out == 100).all()


def test_remap_restatement_equals_the_committed_reference_vectors():
    """tests/golden/remap_opencv_96x72.npz was written by the reference itself (make_golden_remap.py); this runs on boxes
    without the reference too."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "remap_opencv_96x72.npz"))
    h, w = g["out1"].shape
    assert np.array_equal(oracle.remap_apply(g["img"], g["idx4"], g["coef4"], g["remap_x"], (h, w)), g["out1"])
    m = (g["remap_x"] > 0).reshape(h, w)
    assert np.array_equal(oracle.remap_apply(g["rgb"], g["idx4"], g["coef4"], g["remap_x"], (h, w))[m], g["out3"][m])
