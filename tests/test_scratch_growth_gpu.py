"""A ctx's device scratch grows inside the call whose take no longer fits it (gb_scratch_take, csrc/ctx.cu): the stream is synchronised,
the buffer replaced, and the call's buffers are laid out in the new one.  Each case runs a call on a ctx whose scratch earlier calls
sized too small, and compares its outputs byte for byte with the same call on a fresh ctx -- for the matcher with the work split it
planned (gb_dbg_match_last_plan)."""
import numpy as np
import pytest

from gslam_b200 import capi, synth
from gslam_b200.api import Context, Features, Remap, Vocabulary
from oracle import oracle as O

import _bow_cases as BC
from _match_cases import grid_keypoints

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


def last_plan(ctx):
    out = np.zeros(4, np.int32)
    assert capi.lib().gb_dbg_match_last_plan(ctx.handle, capi.ptr(out)) == capi.GB_OK
    return tuple(int(x) for x in out)


def test_device_match_partials_grow_then_tickets_rearm():
    """Features.match takes its split partials from the scratch.  A small pair, then a pending pair (an extraction in flight) whose
    partials grow the scratch and whose query capacity, 4001, leaves the last query tile -- and its ticket -- 33 rows, then the small
    pair again, on the tickets its first match re-armed."""
    small = synth.random_descriptors(200, 1), synth.random_descriptors(300, 2)
    big = synth.random_descriptors(4001, 3), synth.random_descriptors(6000, 4)

    def run(ctx, which):
        sets = {}

        def pair(name):
            if name not in sets:
                q, t = small if name == "small" else big
                fq, ft = Features(ctx, len(q)), Features(ctx, len(t))
                fq.upload(q)
                ft.upload(t)
                sets[name] = fq, ft
            return sets[name]
        out = []
        try:
            for name in which:
                fq, ft = pair(name)
                if name == "big":  # device-side counts: the launch covers the capacities, the last tile holds 28 real rows
                    for f, n in ((fq, 3996), (ft, 5990)):
                        assert capi.lib().gb_dbg_features_set_pending(ctx.handle, f._h, n, 0, n - 100) == capi.GB_OK
                fq.match(ft)
                out.append((last_plan(ctx), fq.matches()))
        finally:
            for fq, ft in sets.values():
                fq.close()
                ft.close()
        return out
    got = fresh(lambda c: run(c, ("small", "big", "small")))
    want = [fresh(lambda c: run(c, (name,)))[0] for name in ("small", "big", "small")]
    assert got[1][0][0] == 32 and got[1][0][1] > 1 and got[0][0][1] > 1, (got[0][0], got[1][0])
    for (gp, gm), (wp, wm) in zip(got, want):
        assert gp == wp
        assert_same(gm, wm)
    assert np.array_equal(got[0][1][0], got[2][1][0])


def test_host_match_hamming_then_larger():
    """gb_match_hamming: its two feature sets and the partials are one take, larger than the earlier call's."""
    calls = [(synth.random_descriptors(150, 5), synth.random_descriptors(700, 6)),
             (synth.random_descriptors(3000, 7), synth.random_descriptors(9000, 8))]

    def run(ctx, cs):
        return [(ctx.match_hamming(q, t), last_plan(ctx)) for q, t in cs]
    got = fresh(lambda c: run(c, calls))
    for g, call in zip(got, calls):
        w = fresh(lambda c: run(c, [call]))[0]
        assert g[1] == w[1]
        assert_same(g[0], w[0])


def test_host_match_stereo_then_larger():
    """gb_match_stereo: the same for the rectified-stereo matcher, whose feature sets carry the keypoints."""
    rng = np.random.default_rng(11)
    calls = [(grid_keypoints(rng, n), synth.random_descriptors(n, 20 + n), grid_keypoints(rng, m), synth.random_descriptors(m, 30 + m))
             for n, m in ((120, 400), (2500, 7000))]

    def run(ctx, cs):
        return [(ctx.match_stereo(*c, band=1.0, min_disp=0.0, max_disp=20.0), last_plan(ctx)) for c in cs]
    got = fresh(lambda c: run(c, calls))
    for g, call in zip(got, calls):
        w = fresh(lambda c: run(c, [call]))[0]
        assert g[1] == w[1] and g[1][3] == 1
        assert_same(g[0], w[0])


def test_orb_extract_large_capacity_then_small():
    """gb_orb_extract's feature set is sized to the call, max(capacity, 2 nfeatures + 256), not to the largest earlier call."""
    img = synth.synth_frame(640, 480, seed=9)
    c = Context(0)
    try:
        got_big = c.orb_extract(img, 500, capacity=40000)
        got = c.orb_extract(img, 500, capacity=600)
    finally:
        c.close()
    assert len(got[0]) > 400
    assert_same(got_big, fresh(lambda f: f.orb_extract(img, 500, capacity=40000)))
    assert_same(got, fresh(lambda f: f.orb_extract(img, 500, capacity=600)))
