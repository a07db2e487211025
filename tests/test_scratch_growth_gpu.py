"""A ctx's device scratch grows inside the call whose take no longer fits it (gb_scratch_take, csrc/ctx.cu): the stream is synchronised,
the buffer replaced, and the call's buffers are laid out in the new one.  Each case runs a call on a ctx whose scratch earlier calls
sized too small, and compares its outputs byte for byte with the same call on a fresh ctx."""
import numpy as np
import pytest

from gslam_b200 import synth
from gslam_b200.api import Context, Remap, Vocabulary
from oracle import oracle as O

import _bow_cases as BC

pytestmark = pytest.mark.gpu


def fresh(call):
    c = Context(0)
    try:
        return call(c)
    finally:
        c.close()


def scale_map(ctx, w_in, h_in, w_out, h_out):
    """A bilinear downscale in the reference's table format: every output pixel inside the input, four taps each."""
    y, x = np.mgrid[0:h_out, 0:w_out].astype(np.float64)
    sx = ((x + 0.5) * (w_in - 1) / w_out).astype(np.float32); sy = ((y + 0.5) * (h_in - 1) / h_out).astype(np.float32)
    xi, yi = sx.astype(np.int32), sy.astype(np.int32)
    fx, fy = sx - xi, sy - yi
    idx = np.stack([yi * w_in + xi, yi * w_in + xi + 1, (yi + 1) * w_in + xi, (yi + 1) * w_in + xi + 1], -1).astype(np.int32)
    coef = np.stack([(1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy], -1).astype(np.float32)
    return Remap(ctx, w_in, h_in, w_out, h_out, idx.reshape(-1, 4), coef.reshape(-1, 4), sx.reshape(-1))


def colour(w, h, seed):
    g = synth.synth_frame(w, h, seed=seed)
    return np.stack([g, np.roll(g, 7, axis=1), 255 - g], axis=2)


def assert_same(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if isinstance(g, np.ndarray):
            assert g.dtype == w.dtype and np.array_equal(g, w)
        else:
            assert g == w


def test_bow_transform_larger_than_any_earlier_take():
    """Host-buffer gb_bow_transform: the uploaded descriptors, the walk's outputs, the global-memory sort keys and the results are one
    take, larger than everything the ctx took before."""
    v = O.synth_vocabulary(10, 4, seed=5, stop=0.05)
    small, big = BC.queries(v, 300, seed=1), BC.queries(v, 20000, seed=2)

    def transform(ctx, descs):
        dv = Vocabulary(ctx, v.k, v.L, v.weighting, v.scoring, v.child_num, v.weight, v.desc)
        try:
            return [dv.transform(d, 1) for d in descs]
        finally:
            dv.close()
    got = fresh(lambda c: transform(c, (small, big)))
    want = [fresh(lambda c: transform(c, (d,)))[0] for d in (small, big)]
    for g, w in zip(got, want):
        for k in ("words", "values", "fv_node", "fv_feat"):
            assert g[k].dtype == w[k].dtype and np.array_equal(g[k], w[k]), k


def test_orb_colour_frame_then_larger_undistorted_frame():
    """A pageable colour gb_orb_extract_image stages its frame in the scratch; a gb_orb_extract_undistorted of a larger colour frame
    then grows it."""
    small, big = colour(320, 240, seed=3), colour(1920, 1080, seed=4)
    c = Context(0)
    m = scale_map(c, 1920, 1080, 1280, 720)
    try:
        got_small = c.orb_extract(small, 300)
        got = c.orb_extract_undistorted(m, big, 1500)
        assert len(got[0]) > 500
        assert_same(got_small, fresh(lambda f: f.orb_extract(small, 300)))
        assert_same(got, fresh(lambda f: f.orb_extract_undistorted(m, big, 1500)))
    finally:
        m.close()
        c.close()


def scene(rng, n, outliers):
    R, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    t = rng.uniform(-1, 1, 3)
    Xc = np.column_stack([rng.uniform(-4, 4, n), rng.uniform(-3, 3, n), rng.uniform(3, 20, n)])
    xy = Xc[:, :2] / Xc[:, 2:3] + rng.normal(0, 1 / 718, (n, 2))
    bad = rng.permutation(n)[:int(outliers * n)]
    xy[bad] = np.column_stack([rng.uniform(-1.3, 1.3, bad.size), rng.uniform(-1, 1, bad.size)])
    return np.ascontiguousarray((Xc - t) @ R), np.ascontiguousarray(xy)


def test_pnp_ransac_scratch_grows():
    """gb_pnp_ransac's points, measurements and per-hypothesis results: a small call, then one with more of each."""
    rng = np.random.default_rng(7)
    small, big = scene(rng, 60, 0.2), scene(rng, 3000, 0.6)
    kw_small = dict(threshold=4 / 718, max_hypotheses=128, seed=3)
    kw_big = dict(threshold=4 / 718, max_hypotheses=8192, confidence=0.9999, seed=4)
    c = Context(0)
    try:
        got_small = c.pnp_ransac(*small, **kw_small)
        got = c.pnp_ransac(*big, **kw_big)
    finally:
        c.close()
    for g, w in ((got_small, fresh(lambda f: f.pnp_ransac(*small, **kw_small))), (got, fresh(lambda f: f.pnp_ransac(*big, **kw_big)))):
        assert np.array_equal(g[0], w[0]) and np.array_equal(g[1], w[1])
        for f in ("hypotheses", "best_hypothesis", "best_root", "inliers_minimal", "inliers_refined"):
            assert getattr(g[2], f) == getattr(w[2], f), f
