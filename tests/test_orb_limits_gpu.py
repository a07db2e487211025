"""ORB extraction at the edges of its configuration range and at its fixed limits, bit-exact against the oracle.

The cases (tests/_orb_limits.py) are pinned to live cv2 by tests/test_oracle_orb.py::test_limit_case_oracle_equals_cv2.  Besides
every keypoint field and descriptor bit, each case asserts on the device's per-level counts that it reached the boundary it was
written for: the 4096-keypoint level cap, the full 4096-entry sort, the usable levels at large edge thresholds and extreme aspect
ratios, positions near 16383.  The other tests cover what happens over the limits -- more than 4096 keypoints on one level, frames
wider than 16384 -- and that one context stays correct when the frame size or the configuration changes from call to call."""
import ctypes as C

import numpy as np
import pytest

import oracle
from gslam_b200 import capi, synth
from gslam_b200.api import Features

from _orb_limits import CASES, LEVEL_CAP, N_AT_CAP, N_OVER_CAP, OVER_CAP, BY_ID, check_reach, usable_levels

pytestmark = pytest.mark.gpu
FIELDS = ("octave", "x", "y", "size", "angle", "response", "class_id")


def assert_same(kps, desc, wk, wd):
    assert len(kps) == len(wk), (len(kps), len(wk))
    for f in FIELDS:
        assert np.array_equal(kps[f], wk[f]), f
    assert np.array_equal(desc, wd)


def level_counts(ctx, nlevels):
    """Per level of the last extraction on ctx: (FAST corners after NMS and the border filter, keypoints kept)."""
    L = capi.lib()
    cand, kept = [], []
    for l in range(nlevels):
        n, nk = C.c_int(), C.c_int()
        assert L.gb_dbg_orb_candidates(ctx.handle, l, None, None, None, None, 0, C.byref(n), None, 0, C.byref(nk)) == capi.GB_OK
        cand.append(n.value); kept.append(nk.value)
    return cand, kept


def extract_and_compare(ctx, img, n, **kw):
    gray = oracle.to_gray(img, rgb=kw.get("rgb", False)) if img.ndim == 3 else img
    wk, wd = oracle.orb_extract(gray, n, **{k: v for k, v in kw.items() if k != "rgb"})
    kps, desc = ctx.orb_extract(img, n, **kw)
    assert_same(kps, desc, wk, wd)
    return kps


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_limit_case_matches_oracle(ctx, case):
    kps = extract_and_compare(ctx, case.image(), case.nfeatures, **case.kw)
    cand, kept = level_counts(ctx, case.kw.get("nlevels", 8))
    per = check_reach(case, kps, fast0=cand[0])
    assert kept == per, (kept, per)                   # what the device's selection kept, level by level
    assert not any(cand[usable_levels(case):]), cand   # levels within 2 * edge_threshold of their size get no FAST tile


def test_level_cap_at_4096(ctx):
    """Level 0 keeps exactly 4096 at nfeatures 18862 (its whole sort runs); at 18863 it would keep 4097 (the oracle and cv2 do),
    and every way of reading that extraction fails with GB_ERR_CAPACITY naming the limit, without writing the caller's buffers and
    without breaking the context."""
    img = OVER_CAP.image()
    h, w = img.shape
    assert check_reach(OVER_CAP, oracle.orb_extract(img, N_OVER_CAP)[0])[0] == LEVEL_CAP + 1
    # host buffers
    cfg = ctx.orb_cfg(nfeatures=N_OVER_CAP)
    cap = 2 * N_OVER_CAP + 256
    kps = np.zeros(cap, capi.KP_DTYPE); desc = np.zeros((cap, 32), np.uint8); n = C.c_int(cap)
    rc = ctx._lib.gb_orb_extract(ctx.handle, capi.ptr(img), w, h, C.byref(cfg), capi.ptr(kps), capi.ptr(desc), C.byref(n))
    assert rc == capi.GB_ERR_CAPACITY and n.value == 0
    assert "4096" in ctx._lib.gb_last_error(ctx.handle).decode()
    assert not kps.view(np.uint8).any() and not desc.any()
    with pytest.raises(capi.GbError) as e:
        ctx.orb_extract(img, N_OVER_CAP)
    assert e.value.code == capi.GB_ERR_CAPACITY and "4096" in str(e.value)
    # device-resident feature sets: count, download, and the matches of a match enqueued behind the extraction
    f, train = Features(ctx, cap), Features(ctx, cap)
    try:
        train.extract(img, w, h, ctx.orb_cfg(nfeatures=2000))
        f.extract(img, w, h, cfg)
        for read in (f.count, f.download, f.count):
            with pytest.raises(capi.GbError) as e:
                read()
            assert e.value.code == capi.GB_ERR_CAPACITY and "4096" in str(e.value)
        f.extract(img, w, h, cfg)
        f.match(train)
        for _ in range(2):  # asking again must not turn the failure into an empty result
            with pytest.raises(capi.GbError) as e:
                f.matches()
            assert e.value.code == capi.GB_ERR_CAPACITY and "4096" in str(e.value)
        # the same context and feature set at the cap, then at the defaults: bit-exact again
        wk, wd = oracle.orb_extract(img, N_AT_CAP)
        f.extract(img, w, h, ctx.orb_cfg(nfeatures=N_AT_CAP))
        assert f.count() == len(wk)
        got = f.download()
        assert_same(got[0], got[1], wk, wd)
        assert level_counts(ctx, 1)[1] == [LEVEL_CAP]
        kps, desc = ctx.orb_extract(img, N_AT_CAP)
        assert_same(kps, desc, wk, wd)
        assert check_reach(BY_ID["cap_noise"], kps)[0] == LEVEL_CAP
        extract_and_compare(ctx, img, 500)
    finally:
        f.close(); train.close()


@pytest.mark.parametrize("w,h", [(16385, 64), (64, 16385)])
def test_oversize_frame_rejected_then_next_extraction_exact(ctx, w, h):
    """A frame over 16384 on a side is refused (positions are packed in 16 bits); the refusal frees the context's buffers, so the
    next call -- at the size the context was built for before -- must rebuild them."""
    ok = synth.synth_frame(640, 480, 31)
    extract_and_compare(ctx, ok, 500)
    img = np.zeros((h, w), np.uint8)
    with pytest.raises(capi.GbError) as e:
        ctx.orb_extract(img, 500)
    assert e.value.code == capi.GB_ERR_INVALID and "16384" in str(e.value)
    extract_and_compare(ctx, ok, 500)


def _colour(w, h, channels, seed):
    rng = np.random.default_rng(seed)
    base = synth.synth_frame(w, h, seed).astype(np.int64)
    return np.stack([np.clip(base + rng.integers(-40, 41, base.shape), 0, 255) for _ in range(channels)], -1).astype(np.uint8)


def test_rebuild_sequence_one_context(ctx):
    """One context through frame sizes, configurations and channel counts that each rebuild (or grow) its state: pyramid, resize
    tables, TMA tensor maps, candidate slices, the colour staging buffer.  Every call is checked against the oracle."""
    hd = synth.synth_frame(1280, 720, 41)
    c3 = _colour(480, 360, 3, 42)
    steps = [
        (hd, 1000, {}),
        (BY_ID["wide_16384x80"].image(), 2000, {}),
        (synth.synth_frame(517, 389, 77), 500, dict(nlevels=12, edge_threshold=22)),
        (c3, 400, {}),
        (_colour(480, 360, 4, 43), 400, {}),                 # same size and config: the colour buffer grows in place
        (_colour(752, 480, 4, 44), 600, dict(rgb=True)),     # another size
        (_colour(752, 480, 3, 45), 600, {}),                 # fewer channels into the grown buffer
        (c3, 400, {}),
        (hd, 1000, {}),
    ]
    for img, n, kw in steps:
        assert len(extract_and_compare(ctx, img, n, **kw)) > 0
