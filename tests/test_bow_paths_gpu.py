"""The bag-of-words transform on every walk width and sort path, at device-side counts and from two contexts, bit-exact against
the oracle.

The cases (tests/_bow_cases.py) reach the launch plan's boundaries -- 16- and 32-lane walks (k = 1, 2, 15, 16, 17, 31, 32), a
root-only tree, trees deeper than L and one level deep, a 10^6-node tree, every kind of levelsup, row counts around 1024, 2048
and 8192 keys (shared- and global-memory sorts), word runs that start and end on chunk boundaries or span chunks, the node sort
skipped and run because of one feature, stopped words of every odd weight (-0.0, negative, NaN, subnormal) and the norm's
exactness bound on both sides.  Every case asserts that the device planned exactly what the mirror plans (gb_dbg_bow_last_plan)
and so reached its boundary.  The other tests run the device-side counts of an extraction in flight, every weighting with every
scoring, one vocabulary through growing and shrinking inputs, the call contracts, and one vocabulary shared by two contexts
driven from two threads."""
import ctypes as C
import threading

import numpy as np
import pytest

from gslam_b200 import capi, synth
from gslam_b200.api import Context, Features, Vocabulary
from oracle import oracle as O

import _bow_cases as BC
from _bow_cases import CASES

pytestmark = pytest.mark.gpu
KEYS = ("words", "values", "fv_node", "fv_feat")


def dev_voc(ctx, v):
    return Vocabulary(ctx, v.k, v.L, v.weighting, v.scoring, v.child_num, v.weight, v.desc)


def last_plan(voc):
    out = np.zeros(5, np.int32)
    assert capi.lib().gb_dbg_bow_last_plan(voc._h, capi.ptr(out)) == capi.GB_OK
    return tuple(int(x) for x in out)


def set_pending(ctx, f, count, status=0, expect=0):
    assert capi.lib().gb_dbg_features_set_pending(ctx.handle, f._h, count, status, expect) == capi.GB_OK


def check(got, want, where=""):
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), (k, where)


def transform_on(ctx, voc, features, levelsup, n_out):
    """gb_bow_transform / gb_bow_transform_features on `ctx`, which need not be the ctx the vocabulary was created on."""
    L = capi.lib()
    words = np.zeros(max(n_out, 1), np.uint64); values = np.zeros(max(n_out, 1), np.float32)
    fvn = np.zeros(max(n_out, 1), np.uint64); fvf = np.zeros(max(n_out, 1), np.uint32)
    nw, m = C.c_int(0), C.c_int(0)
    if isinstance(features, Features):
        rc = L.gb_bow_transform_features(ctx.handle, voc._h, features._h, levelsup, capi.ptr(words), capi.ptr(values), C.byref(nw),
                                         capi.ptr(fvn), capi.ptr(fvf), C.byref(m))
    else:
        rc = L.gb_bow_transform(ctx.handle, voc._h, capi.ptr(features), len(features), levelsup, capi.ptr(words), capi.ptr(values),
                                C.byref(nw), capi.ptr(fvn), capi.ptr(fvf), C.byref(m))
    ctx._check(rc)
    return dict(words=words[:nw.value].astype(np.int64), values=values[:nw.value], fv_node=fvn[:m.value].astype(np.int64),
                fv_feat=fvf[:m.value].astype(np.int32))


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_case_matches_oracle(ctx, case):
    v, f, lu = case.data
    dv = dev_voc(ctx, v)
    try:
        got = dv.transform(f, lu)
        plan = last_plan(dv)
    finally:
        dv.close()
    ref = O.bow_transform(v, f, lu)
    for k in KEYS:
        bad = np.nonzero(got[k] != ref[k])[0] if got[k].shape == ref[k].shape else [0]
        assert len(bad) == 0, (k, [(i, got[k][i], ref[k][i]) for i in bad[:3]] if got[k].shape == ref[k].shape else got[k].shape)
    assert plan == BC.device_plan(v, ref, len(f)), plan
    BC.check_reach(case, plan)


# ---- device-side counts ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cap,count", [(3000, 0), (3000, 1), (3000, 3000), (3000, 1234), (12000, 5000), (12000, 8192), (12000, 8193),
                                       (12000, 12000)])
def test_device_count(ctx, cap, count):
    """All `cap` rows uploaded, the count on the device: rows past it are real descriptors that would add words.  The transform of
    the feature set equals the host transform of the first `count` rows; the sort is clipped to the count's power of two."""
    v = O.synth_vocabulary(10, 4, seed=cap + count, prune=0.1, stop=0.05)
    rows = BC.queries(v, cap, seed=count)
    dv = dev_voc(ctx, v)
    fs = Features(ctx, cap)
    try:
        fs.upload(rows)
        set_pending(ctx, fs, count, 0, cap)
        got = dv.transform(fs, 1)
        plan = last_plan(dv)
        ref_all = O.bow_transform(v, rows, 1)
        assert plan == BC.device_plan(v, ref_all, cap, count), plan
        assert plan[2] == BC.next_pow2(cap) and plan[3] == min(plan[2], BC.next_pow2(max(count, 2)))
        want = O.bow_transform(v, rows[:count], 1)
        check(got, want)
        if count > 0:
            check(dv.transform(rows[:count], 1), want)
        if count < cap:
            assert not all(np.array_equal(ref_all[k], want[k]) for k in ("words", "fv_feat"))
        # a failed extraction's status: GB_ERR_CAPACITY on every call, then exact again
        fs.upload(rows)
        set_pending(ctx, fs, count, cap + 5, cap)
        for _ in range(2):
            with pytest.raises(capi.GbError) as e:
                dv.transform(fs, 1)
            assert e.value.code == capi.GB_ERR_CAPACITY
        fs.upload(rows[:count]) if count else fs.upload(np.zeros((0, 32), np.uint8))
        check(dv.transform(fs, 1), want)
    finally:
        fs.close(); dv.close()


def test_cross_ctx_device_count(ctx):
    """Extract on ctx A, order ctx B after it (gb_ctx_wait_for), transform on B while the count is still on the device."""
    b = Context(0)
    v = O.synth_vocabulary(10, 4, seed=11)
    dv = dev_voc(ctx, v)
    fs = Features(ctx, 2000)
    try:
        img = synth.synth_frame(640, 480, seed=5)
        fs.extract(img, 640, 480, ctx.orb_cfg(nfeatures=700))
        b.wait_for(ctx)
        got = transform_on(b, dv, fs, 2, fs.capacity)
        _, desc = fs.download()
        assert len(desc) > 100
        check(got, O.bow_transform(v, desc, 2))
    finally:
        fs.close(); dv.close(); b.close()


# ---- every weighting with every scoring -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("weighting", [O.W_TF_IDF, O.W_TF, O.W_IDF, O.W_BINARY])
@pytest.mark.parametrize("scoring", [O.S_L1, O.S_L2, O.S_CHI_SQUARE, O.S_KL, O.S_BHATTACHARYYA, O.S_DOT_PRODUCT])
def test_weighting_and_scoring(ctx, weighting, scoring):
    v = O.synth_vocabulary(10, 4, seed=3 + weighting, weighting=weighting, scoring=scoring, prune=0.1, stop=0.1)
    f = BC.queries(v, 9000, seed=scoring)
    dv = dev_voc(ctx, v)
    try:
        for lu in (0, 2):
            ref = O.bow_transform(v, f, lu)
            check(dv.transform(f, lu), ref, lu)
            assert last_plan(dv) == BC.device_plan(v, ref, len(f))
    finally:
        dv.close()


# ---- one vocabulary through growing and shrinking inputs ------------------------------------------------------------------------
def test_size_sequence_on_one_vocabulary(ctx):
    v = O.synth_vocabulary(20, 3, seed=8, stop=0.05)
    dv = dev_voc(ctx, v)
    try:
        for i, n in enumerate((1, 9000, 1, 8192, 9000, 2)):
            f = BC.queries(v, n, seed=i)
            ref = O.bow_transform(v, f, 1)
            check(dv.transform(f, 1), ref, n)
            assert last_plan(dv) == BC.device_plan(v, ref, n)
        dv.transform(np.zeros((0, 32), np.uint8), 1)
        assert last_plan(dv) == (0, 0, 0, 0, 0)
    finally:
        dv.close()


# ---- contracts ------------------------------------------------------------------------------------------------------------------
def test_voc_create_contracts(ctx):
    L = capi.lib()
    v = O.synth_vocabulary(4, 2, seed=1)
    ch, w, d = v.child_num.copy(), v.weight, v.desc
    P = capi.ptr

    def create(c=ctx.handle, k=4, Lv=2, we=0, sc=0, n=None, child=ch, weight=w, desc=d, out=True):
        h = C.c_void_p()
        rc = L.gb_voc_create(c, k, Lv, we, sc, len(ch) if n is None else n, P(child), P(weight), P(desc), C.byref(h) if out else None)
        if rc == capi.GB_OK:
            assert L.gb_voc_destroy(ctx.handle, h) == capi.GB_OK
        else:
            assert not h.value
        return rc

    assert create() == capi.GB_OK
    bad = [dict(c=None), dict(out=False), dict(k=0), dict(k=33), dict(Lv=-1), dict(we=-1), dict(we=4), dict(sc=-1), dict(sc=6), dict(n=0),
           dict(child=None), dict(weight=None), dict(desc=None)]
    for kw in bad:
        assert create(**kw) == capi.GB_ERR_INVALID, kw
    c2 = ch.copy(); c2[1] = 5                        # more children than k
    assert create(child=c2) == capi.GB_ERR_INVALID
    # the last node with children: its last child id at n_nodes - 1 is accepted, at n_nodes rejected
    small = np.zeros(7, np.uint32); small[0] = 2; small[1] = 4     # children of 1: 5, 6, 7, 8 -> ids up to 8
    ws, ds = np.ones(9, np.float32), np.zeros((9, 32), np.uint8)
    assert create(n=9, child=np.append(small, [0, 0]).astype(np.uint32), weight=ws, desc=ds) == capi.GB_OK
    assert create(n=8, child=np.append(small, [0]).astype(np.uint32), weight=ws, desc=ds) == capi.GB_ERR_INVALID
    # a k = 1 chain, and a root-only tree
    assert create(k=1, n=3, child=np.uint32([1, 1, 0]), weight=ws, desc=ds) == capi.GB_OK
    assert create(n=1, child=np.zeros(1, np.uint32), weight=ws, desc=ds) == capi.GB_OK


def test_transform_contracts(ctx):
    L = capi.lib()
    v = O.synth_vocabulary(10, 2, seed=1)
    dv = dev_voc(ctx, v)
    f = BC.queries(v, 50, 2)
    o = [np.zeros(50, t) for t in (np.uint64, np.float32, np.uint64, np.uint32)]
    nw, m = C.c_int(-1), C.c_int(-1)
    P = capi.ptr
    try:
        args = [ctx.handle, dv._h, P(f), 50, 0, P(o[0]), P(o[1]), C.byref(nw), P(o[2]), P(o[3]), C.byref(m)]
        for i in (0, 1, 2, 5, 6, 7, 8, 9, 10):
            a = list(args); a[i] = None
            assert L.gb_bow_transform(*a) == capi.GB_ERR_INVALID, i
        a = list(args); a[3] = -1
        assert L.gb_bow_transform(*a) == capi.GB_ERR_INVALID
        a = list(args); a[2] = None; a[3] = 0                      # n = 0: no rows needed, empty maps
        assert L.gb_bow_transform(*a) == capi.GB_OK and nw.value == 0 and m.value == 0
        fs = Features(ctx, 64)
        try:
            fa = [ctx.handle, dv._h, fs._h, 0, P(o[0]), P(o[1]), C.byref(nw), P(o[2]), P(o[3]), C.byref(m)]
            for i in (0, 1, 2, 4, 5, 6, 7, 8, 9):
                a = list(fa); a[i] = None
                assert L.gb_bow_transform_features(*a) == capi.GB_ERR_INVALID, i
        finally:
            fs.close()
        check(dv.transform(f, 0), O.bow_transform(v, f, 0))
    finally:
        dv.close()


# ---- one vocabulary, two contexts, two threads -----------------------------------------------------------------------------------
def test_one_vocabulary_two_contexts_two_threads(ctx):
    """Two threads, each with its own ctx, transform their own descriptor sets through one vocabulary many times, each set both from
    host memory and as a device-resident feature set, so that host-buffer and device-feature transforms overlap; every result equals
    the oracle.  Both use the same row count, and one call at that count ran first."""
    n, iters = 3000, 30
    v = O.synth_vocabulary(10, 4, seed=21, stop=0.05)
    dv = dev_voc(ctx, v)
    dv.transform(BC.queries(v, n, 0), 1)
    sets = [[BC.queries(v, n, 100 * t + j) for j in range(2)] for t in range(2)]
    wants = [[O.bow_transform(v, s, 1) for s in ss] for ss in sets]
    ctxs = [ctx, Context(0)]
    feats = [[Features(ctxs[t], n) for _ in range(2)] for t in range(2)]
    for t in range(2):
        for j in range(2):
            feats[t][j].upload(sets[t][j])
    errors = []

    def run(t):
        try:
            for i in range(iters):
                # thread 0 starts on host buffers, thread 1 on device features: the two forms run side by side
                for src in ((sets, feats) if (i + t) % 2 == 0 else (feats, sets)):
                    got = transform_on(ctxs[t], dv, src[t][i % 2], 1, n)
                    for k in KEYS:
                        if not np.array_equal(got[k], wants[t][i % 2][k]):
                            errors.append((t, i, k, type(src[t][i % 2]).__name__))
                            return
        except Exception as e:  # noqa: BLE001
            errors.append((t, repr(e)))

    th = [threading.Thread(target=run, args=(t,)) for t in range(2)]
    try:
        for x in th:
            x.start()
        for x in th:
            x.join()
    finally:
        for fs in feats[0] + feats[1]:
            fs.close()
        dv.close()
        ctxs[1].close()
    assert not errors, errors
