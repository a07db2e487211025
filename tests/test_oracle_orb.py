"""Pins oracle/orb_ref.c against cv2 4.13 golden vectors, stage by stage and end to end (SURVEY.md App. A, §8c KAT-O).
OpenCV is the third-party dependency that holds the ORB arithmetic of the reference's CPU path (absent from the tree)."""
import hashlib
import os

import numpy as np
import pytest

import oracle
from gslam_b200 import synth

GD = os.path.join(os.path.dirname(__file__), "golden")
ST = np.load(os.path.join(GD, "orb_stages.npz"))
CASES = ["orb_320x240_n300", "orb_480x360_n400", "orb_752x480_n2000", "orb_1280x720_n1000", "orb_1920x1080_n2000"]


def load_case(name):
    g = np.load(os.path.join(GD, name + ".npz"))
    img = g["image"] if "image" in g else synth.synth_frame(int(g["width"]), int(g["height"]), int(g["seed"]))
    if hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest() != str(g["image_sha256"]):
        pytest.skip("synthetic image generator drifted from the fixture")
    return g, img


def test_gauss_kernel_bits():
    import struct
    bits = [0x3d8fafb1, 0x3e06387e, 0x3e434a39, 0x3e5d4ae0, 0x3e434a39, 0x3e06387e, 0x3d8fafb1]
    assert [struct.unpack("<I", struct.pack("<f", float(v)))[0] for v in ST["gauss_kernel"]] == bits


def test_resize_linear_exact_golden():
    assert np.array_equal(oracle.resize_linear_exact(ST["image"], 167, 125), ST["resized_167x125"])


def test_fast_golden():
    for nms, key in ((True, "fast_nms"), (False, "fast_all")):
        xs, ys, sc = oracle.fast_detect(ST["image"], 20, nms)
        got = np.stack([xs, ys, sc], axis=1)
        if not nms:  # cv2 reports response 0 when it does not run NMS: compare positions only
            got[:, 2] = 0
        assert np.array_equal(got, ST[key]), key  # same positions, same row-major order, same scores


def test_fast_atan2_golden():
    got = np.array([oracle.fast_atan2(y, x) for y, x in zip(ST["atan_y"], ST["atan_x"])], np.float32)
    assert np.array_equal(got, ST["atan"])


def test_blur_golden():
    assert np.array_equal(oracle.blur7(ST["image"]), ST["blur"])
    img = ST["image"]
    for (x, y) in [(0, 0), (199, 149), (50, 60), (3, 146)]:
        assert oracle.lib().orc_blur_pixel(img.ctypes.data, 200, 150, x, y) == ST["blur"][y, x]


def test_quotas_and_level_sizes():
    assert oracle.orb_quotas(2000).tolist() == [434, 362, 302, 251, 209, 175, 145, 122]  # SURVEY.md App. A.3
    assert [oracle.orb_level_size(1920, 1080, l) for l in range(8)] == [(1920, 1080), (1600, 900), (1333, 750), (1111, 625), (926, 521), (772, 434), (643, 362), (536, 301)]
    assert [oracle.orb_level_size(1280, 720, l) for l in range(8)] == [(1280, 720), (1067, 600), (889, 500), (741, 417), (617, 347), (514, 289), (429, 241), (357, 201)]


# cv2 4.13 level sizes, recovered from cv2 itself (the Harris responses of its keypoints only reproduce on a level image of
# exactly the right size): cv2 evaluates cols/scale as cols*(1/scale) in float, so 477/1.2f -> 397.5f -> 398 where a true float
# division rounds to 397.  Rows where the two rules differ (found by fuzzing the oracle against live cv2):
CV2_LEVEL_SIZES = {
    (456, 477, 1.2): [(456, 477), (380, 398), (317, 331), (264, 276), (220, 230), (183, 192), (153, 160), (127, 133)],
    (303, 249, 1.2): [(303, 249), (252, 208), (210, 173), (175, 144), (146, 120), (122, 100), (101, 83), (85, 69)],
    (645, 333, 1.2): [(645, 333), (538, 278), (448, 231), (373, 193), (311, 161), (259, 134), (216, 112), (180, 93)],
    (342, 630, 1.2): [(342, 630), (285, 525), (237, 437), (198, 365), (165, 304), (137, 253), (115, 211), (95, 176)],
    (702, 342, 1.2): [(702, 342), (585, 285), (487, 237), (406, 198), (339, 165), (282, 137), (235, 115), (196, 95)],
    (432, 522, 1.25): [(432, 522), (346, 418), (276, 334), (221, 267), (177, 214), (142, 171), (113, 137), (91, 109)],
}


def test_level_sizes_match_cv2():
    for (w, h, sf), want in CV2_LEVEL_SIZES.items():
        assert [oracle.orb_level_size(w, h, l, sf) for l in range(len(want))] == want, (w, h, sf)


def test_level_size_rule_live_cv2():
    """Re-derive one discriminating size from the installed cv2: only a level-1 image of 380x398 reproduces its responses."""
    cv2 = pytest.importorskip("cv2")
    import sys
    sys.path.insert(0, GD)
    from make_golden_orb import cv2_orb_canonical
    img = synth.synth_frame(456, 477, 5634)
    want, _, lvl = cv2_orb_canonical(img, 1500)
    sel = np.nonzero(want["octave"] == 1)[0][:60]
    assert len(sel) > 20
    hits = {}
    for size in ((380, 397), (380, 398)):
        im = cv2.resize(img, size, interpolation=cv2.INTER_LINEAR_EXACT)
        hits[size] = sum(float(oracle.harris_response(im, int(lvl[i, 2]), int(lvl[i, 1]))) == float(want["response"][i]) for i in sel)
    assert hits[(380, 398)] == len(sel) and hits[(380, 397)] == 0
    assert oracle.orb_level_size(456, 477, 1) == (380, 398)


def test_full_pipeline_live_cv2_at_sizes_with_half_way_levels():
    cv2 = pytest.importorskip("cv2")
    import sys
    sys.path.insert(0, GD)
    from make_golden_orb import cv2_orb_canonical
    for (w, h, seed, n, kw, okw) in [(456, 477, 5634, 4000, dict(fastThreshold=30), dict(fast_threshold=30)),
                                     (303, 249, 11, 600, {}, {}), (702, 342, 12, 900, {}, {})]:
        img = synth.synth_frame(w, h, seed)
        want, wdesc, _ = cv2_orb_canonical(img, n, **kw)
        kps, desc = oracle.orb_extract(img, n, **okw)
        assert len(kps) == len(want), (w, h)
        for f in ("octave", "x", "y", "size", "angle", "response"):
            assert np.array_equal(kps[f], want[f]), (f, w, h)
        assert np.array_equal(desc, wdesc)


from _images import KIND_CASES, image_of_kind  # noqa: E402


@pytest.mark.parametrize("kind,w,h,seed,n,nl,sf,ft", KIND_CASES)
def test_live_cv2_image_kinds(kind, w, h, seed, n, nl, sf, ft):
    """Other image statistics than the synthetic scene generator (ties, saturation, flat regions), odd parameter corners."""
    pytest.importorskip("cv2")
    import sys
    sys.path.insert(0, GD)
    from make_golden_orb import cv2_orb_canonical
    img = np.ascontiguousarray(image_of_kind(kind, w, h, seed))
    want, wdesc, _ = cv2_orb_canonical(img, n, nlevels=nl, scaleFactor=sf, fastThreshold=ft)
    kps, desc = oracle.orb_extract(img, n, nlevels=nl, scale_factor=sf, fast_threshold=ft)
    assert len(kps) == len(want)
    for f in ("octave", "x", "y", "size", "angle", "response"):
        assert np.array_equal(kps[f], want[f]), f
    assert np.array_equal(desc, wdesc)


def test_product_level_size_rule_equals_oracle():
    """The extractor's host code (gslam_b200/csrc/orb.cu) and the oracle must size the pyramid identically; the helper is pure
    host code, so this runs without a GPU."""
    import ctypes as C
    from gslam_b200 import capi
    L = C.CDLL(capi.LIB_PATH)
    L.gb_dbg_orb_level_size.argtypes = [C.c_int, C.c_int, C.c_float, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.gb_dbg_orb_level_size.restype = C.c_int
    lw, lh = C.c_int(), C.c_int()
    rng = np.random.default_rng(9)
    cases = [(w, h, sf) for (w, h, sf) in CV2_LEVEL_SIZES] + [(int(rng.integers(40, 4000)), int(rng.integers(40, 3000)), float(sf))
                                                             for sf in (1.1, 1.2, 1.25, 1.35, 1.5, 2.0) for _ in range(60)]
    for w, h, sf in cases:
        for l in range(8):
            assert L.gb_dbg_orb_level_size(w, h, sf, l, C.byref(lw), C.byref(lh)) == 0
            assert (lw.value, lh.value) == oracle.orb_level_size(w, h, l, sf), (w, h, sf, l)


def test_det_sincos_matches_libm_after_float_rounding():
    ang = np.float32(np.linspace(0, 360, 20001, dtype=np.float32))
    th = ang * np.float32(np.pi / 180.0)
    bad = 0
    for t in th:
        s, c = oracle.det_sincos(float(t))
        bad += (np.float32(s) != np.float32(np.sin(np.float64(t)))) + (np.float32(c) != np.float32(np.cos(np.float64(t))))
        assert abs(s - np.sin(np.float64(t))) < 4e-16 and abs(c - np.cos(np.float64(t))) < 4e-16
    assert bad == 0


@pytest.mark.parametrize("name", CASES)
def test_full_pipeline_matches_cv2_golden(name):
    g, img = load_case(name)
    kps, desc = oracle.orb_extract(img, int(g["nfeatures"]))
    want = g["kps"]
    assert len(kps) == len(want)
    for f in ("octave", "x", "y", "size", "angle", "response", "class_id"):
        assert np.array_equal(kps[f], want[f]), f  # bit-exact, canonical order
    assert np.array_equal(desc, g["desc"])


def test_live_cv2_other_resolution_and_params():
    cv2 = pytest.importorskip("cv2")
    import sys
    sys.path.insert(0, GD)
    from make_golden_orb import cv2_orb_canonical
    img = synth.synth_frame(517, 389, 77)  # odd sizes: level sizes land on non-trivial roundings
    for n, kw, okw in [(350, {}, {}), (200, dict(nlevels=5, fastThreshold=12), dict(nlevels=5, fast_threshold=12)),
                       (300, dict(scaleFactor=1.35, nlevels=6), dict(scale_factor=1.35, nlevels=6))]:
        want, wdesc, _ = cv2_orb_canonical(img, n, **kw)
        kps, desc = oracle.orb_extract(img, n, **okw)
        assert len(kps) == len(want)
        for f in ("octave", "x", "y", "size", "angle", "response"):
            assert np.array_equal(kps[f], want[f]), (f, kw)
        assert np.array_equal(desc, wdesc)


def test_degenerate_images():
    flat = np.full((100, 120), 77, np.uint8)
    kps, desc = oracle.orb_extract(flat, 100)
    assert len(kps) == 0 and desc.shape == (0, 32)
    tiny = synth.synth_frame(40, 40, 1)  # smaller than 2*edgeThreshold: nothing can be kept
    kps, _ = oracle.orb_extract(tiny, 100)
    assert len(kps) == 0


def test_gray_conversion_equals_cv2():
    """oracle.to_gray (the rule the device-side conversion of colour frames follows) == cv2.cvtColor on 8-bit images."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    grid = np.stack(np.meshgrid(np.arange(0, 256, 5), np.arange(0, 256, 3), np.arange(0, 256, 7), indexing="ij"), -1).reshape(-1, 1, 3).astype(np.uint8)
    assert np.array_equal(oracle.to_gray(grid), cv2.cvtColor(grid, cv2.COLOR_BGR2GRAY))
    img3 = rng.integers(0, 256, (97, 131, 3), dtype=np.uint8); img4 = rng.integers(0, 256, (64, 80, 4), dtype=np.uint8)
    assert np.array_equal(oracle.to_gray(img3), cv2.cvtColor(img3, cv2.COLOR_BGR2GRAY))
    assert np.array_equal(oracle.to_gray(img3, rgb=True), cv2.cvtColor(img3, cv2.COLOR_RGB2GRAY))
    assert np.array_equal(oracle.to_gray(img4), cv2.cvtColor(img4, cv2.COLOR_BGRA2GRAY))
    assert np.array_equal(oracle.to_gray(img4, rgb=True), cv2.cvtColor(img4, cv2.COLOR_RGBA2GRAY))


from _orb_limits import CASES as LIMIT_CASES, OVER_CAP, check_reach, level0_fast_corners  # noqa: E402


@pytest.mark.parametrize("case", LIMIT_CASES + [OVER_CAP], ids=lambda c: c.id)
def test_limit_case_oracle_equals_cv2(case):
    """The ORB limit cases (edge thresholds 22..239, 12 levels, scale factors 1.01..3.7, FAST thresholds 1 and 254, the 4096-keypoint
    level cap and one past it, 16384-pixel sides): the oracle reaches each case's boundary and equals live cv2 in every keypoint field
    and descriptor bit, so the device parity tests of tests/test_orb_limits_gpu.py compare against cv2's answer."""
    img = case.image()
    kps, desc = oracle.orb_extract(img, case.nfeatures, **case.kw)
    check_reach(case, kps, fast0=level0_fast_corners(case, img))
    pytest.importorskip("cv2")
    import sys
    sys.path.insert(0, GD)
    from make_golden_orb import cv2_orb_canonical
    want, wdesc, _ = cv2_orb_canonical(img, case.nfeatures, **case.cv2_kw)
    assert len(kps) == len(want)
    for f in ("octave", "x", "y", "size", "angle", "response"):
        assert np.array_equal(kps[f], want[f]), f
    assert np.array_equal(desc, wdesc)
