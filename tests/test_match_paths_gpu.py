"""The Hamming and stereo matchers on every work split, at device-side counts and at the edges of the candidate window, bit-exact
against the oracle.

The cases (tests/_match_cases.py) reach the planner's boundaries -- one split with few and with many train rows, 1024-row
chunks, more than 256 splits, a last split of one row, query counts around the tile size and around two tiles per SM, empty and
one-row sets -- and the device-side counts of an extraction in flight: 0, 1, the capacity, counts that need fewer splits than
were launched, and expect hints below, at and above the real count.  Every case asserts that the device planned exactly what the
mirror plans (gb_dbg_match_last_plan) and so reached its boundary.  The other tests plant ties on the split boundaries the device
reports, run the stereo predicate at its edges through both entry points, pin the call contracts, and check that a failed
extraction on the train (right) side fails the download -- and the bag-of-words transform -- instead of reading as an empty set."""
import ctypes as C

import numpy as np
import pytest

import oracle
from gslam_b200 import capi, synth
from gslam_b200.api import Context, Features, Vocabulary

import _match_cases as MC
from _match_cases import CASES, STEREO_EDGES, D, S, check_reach

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def last_plan(ctx):
    out = np.zeros(4, np.int32)
    assert capi.lib().gb_dbg_match_last_plan(ctx.handle, capi.ptr(out)) == capi.GB_OK
    return tuple(int(x) for x in out[:3]), bool(out[3])


def set_pending(ctx, f, count, status=0, expect=0):
    """Put `f` back into the state of an extraction in flight: {count, status} on the device, host count unknown."""
    assert capi.lib().gb_dbg_features_set_pending(ctx.handle, f._h, count, status, expect) == capi.GB_OK


def assert_same(got, want):
    for g, w, name in zip(got, want, ("idx", "d1", "d2")):
        assert np.array_equal(g, w), name


def expect_error(code, fn, *args, text=None):
    with pytest.raises(capi.GbError) as e:
        fn(*args)
    assert e.value.code == code, str(e.value)
    if text:
        assert text in str(e.value), str(e.value)


def run_case(ctx, case, sm):
    """One launch of `case` on ctx: the plan the device used == the mirror's (and reaches the case's boundary), the results ==
    the oracle's on the real rows."""
    s, d = case.shape(sm), case.data(sm)
    q, t, kl, kr = d["q"], d["t"], d["kl"], d["kr"]
    if not s.device:
        got = ctx.match_stereo(kl, q, kr, t, *case.stereo) if case.stereo else ctx.match_hamming(q, t)
    else:
        fq, ft = Features(ctx, s.qcap), Features(ctx, s.tcap)
        try:
            fq.upload(q, kl)
            fq.match(fq)   # outputs of an earlier match in place (distance 0 everywhere): a launch that writes nothing keeps them
            assert (fq.matches()[1] == 0).all()
            ft.upload(t, kr)
            if s.q_dev:
                set_pending(ctx, fq, s.nq, 0, s.eq)
            if s.t_dev:
                set_pending(ctx, ft, s.nt, 0, s.et)
            if case.stereo:
                fq.match_stereo(ft, *case.stereo)
            else:
                fq.match(ft)
            plan_used = last_plan(ctx)
            got = fq.matches()
        finally:
            fq.close(); ft.close()
    if not s.device:
        plan_used = last_plan(ctx)
    assert plan_used == (case.plan(sm), case.stereo is not None), (plan_used, case.plan(sm))
    check_reach(case, plan_used[0], sm)
    if case.stereo:
        want = oracle.match_stereo(kl[:s.nq], q[:s.nq], kr[:s.nt], t[:s.nt], *case.stereo)
    else:
        want = oracle.match_hamming(q[:s.nq], t[:s.nt])
    assert len(got[0]) == s.nq
    assert_same(got, want)
    return got


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_case_matches_oracle(ctx, sm, case):
    run_case(ctx, case, sm)


# ---- ties planted on the split boundaries --------------------------------------------------------------------------------------
def _flip(row, bits):
    r = row.copy()
    for b in bits:
        r[b // 8] ^= np.uint8(1 << (b % 8))
    return r


@pytest.mark.parametrize("nq,nt,dev", [(256, 2000, False), (2000, 2000, False), (40, 50000, False), (3, 8193, True)])
def test_ties_on_split_boundaries(ctx, sm, nq, nt, dev):
    """The merge of the per-split partials keeps the sequential scan's answer where the splits meet: the best distance in the last
    row of split s and again in the first row of s+1 (the index from s, d2 = d1); the best only in s+1 with the runner-up in s; the
    runner-up in the best's own split.  The chunk is the one the device reports for these shapes."""
    rng = np.random.default_rng(nq + nt)
    q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    eq, et = (0, 256) if dev else (0, 0)

    def launch(qq, tt):
        if not dev:
            return ctx.match_hamming(qq, tt), last_plan(ctx)[0]
        fq, ft = Features(ctx, nq), Features(ctx, nt)
        try:
            fq.upload(qq); ft.upload(tt)
            set_pending(ctx, ft, nt, 0, et)
            fq.match(ft)
            return fq.matches(), last_plan(ctx)[0]
        finally:
            fq.close(); ft.close()

    _, (qtiles, nsplit, chunk) = launch(q, t)
    assert (qtiles, nsplit, chunk) == MC.plan(nq, nt, eq, et, sm) and nsplit >= 3
    # one query per boundary (its planted rows are its own), the last boundary always among them
    bounds = np.unique(np.linspace(0, nsplit - 2, min(nq, nsplit - 1)).astype(int))
    want = {}
    for i, s in enumerate(bounds):
        a, b = (s + 1) * chunk - 1, (s + 1) * chunk           # last row of split s, first row of s+1
        kind = i % 3
        if kind == 0:      # the same best distance on both sides of the boundary: the index from s
            t[a] = _flip(q[i], [3]); t[b] = _flip(q[i], [200])
            want[i] = (a, 1, 1)
        elif kind == 1:    # the best only in s+1, the runner-up in s
            t[b] = _flip(q[i], [5]); t[a] = _flip(q[i], [6, 7])
            want[i] = (b, 1, 2)
        else:              # the runner-up in the best's own split
            t[a - 1] = _flip(q[i], [9, 10, 11]); t[a] = q[i]
            want[i] = (a, 0, 3)
    assert bounds[-1] == nsplit - 2 and len(want) >= 3
    got, p = launch(q, t)
    assert p == (qtiles, nsplit, chunk)
    assert_same(got, oracle.match_hamming(q, t))
    for i, w in want.items():
        assert (got[0][i], got[1][i], got[2][i]) == w, (i, bounds[i])


def test_identical_rows_and_extreme_distances(ctx):
    """Every train row identical (the first one wins, d2 = d1 in every split), distances 0 and 256."""
    r = np.full(32, 0x5A, np.uint8)
    q = np.stack([r, ~r, np.zeros(32, np.uint8), np.full(32, 255, np.uint8)] + list(synth.random_descriptors(300, 4)))
    for nt in (1, 33, 5000):
        t = np.repeat(r[None], nt, 0)
        got = ctx.match_hamming(q, t)
        assert_same(got, oracle.match_hamming(q, t))
        assert (got[0] == 0).all() and got[1][0] == 0 and got[1][1] == 256 and got[1][2] == got[1][3] == 128
        assert (got[2] == (got[1] if nt > 1 else 257)).all()
    z, o = np.zeros((130, 32), np.uint8), np.full((3000, 32), 255, np.uint8)
    got = ctx.match_hamming(z, o)
    assert (got[0] == 0).all() and (got[1] == 256).all() and (got[2] == 256).all()


# ---- the stereo predicate at its edges, through both entry points ------------------------------------------------------------
@pytest.mark.parametrize("path", ["host", "dev_left", "dev_right", "dev_both"])
@pytest.mark.parametrize("edge", STEREO_EDGES, ids=lambda e: e.id)
def test_stereo_edge_matches_oracle(ctx, edge, path):
    kl, dl, kr, dr, band, mind, maxd = edge.make(np.random.default_rng(5))
    want = oracle.match_stereo(kl, dl, kr, dr, band, mind, maxd)
    if path == "host":
        got = ctx.match_stereo(kl, dl, kr, dr, band, mind, maxd)
    else:
        fl, fr = Features(ctx, len(kl) + 40), Features(ctx, len(kr) + 40)
        try:
            fl.upload(dl, kl); fr.upload(dr, kr)
            if path in ("dev_left", "dev_both"):
                set_pending(ctx, fl, len(kl), 0, len(kl))
            if path in ("dev_right", "dev_both"):
                set_pending(ctx, fr, len(kr), 0, 0)
            fl.match_stereo(fr, band, mind, maxd)
            assert last_plan(ctx)[1]
            got = fl.matches()
        finally:
            fl.close(); fr.close()
    assert_same(got, want)


# ---- contracts ------------------------------------------------------------------------------------------------------------------
def test_null_outputs_and_download_capacity(ctx):
    L = capi.lib()
    q = synth.random_descriptors(300, 1); t = synth.random_descriptors(500, 2)
    want = oracle.match_hamming(q, t)
    for keep in range(4):  # every output alone, then none
        outs = [np.full(300, -7, np.int32) if k == keep else None for k in range(3)]
        assert L.gb_match_hamming(ctx.handle, capi.ptr(q), 300, capi.ptr(t), 500, *[capi.ptr(o) for o in outs]) == capi.GB_OK
        if keep < 3:
            assert np.array_equal(outs[keep], want[keep])
    kl = MC.grid_keypoints(np.random.default_rng(1), 300); kr = MC.grid_keypoints(np.random.default_rng(2), 500)
    swant = oracle.match_stereo(kl, q, kr, t, 1.0, 2.0, 10.0)
    d1 = np.full(300, -7, np.int32)
    assert L.gb_match_stereo(ctx.handle, capi.ptr(kl), capi.ptr(q), 300, capi.ptr(kr), capi.ptr(t), 500, 1.0, 2.0, 10.0, None, capi.ptr(d1),
                             None) == capi.GB_OK
    assert np.array_equal(d1, swant[1])
    fq, ft = Features(ctx, 400), Features(ctx, 600)
    try:
        fq.upload(q); ft.upload(t)
        set_pending(ctx, ft, 500, 0, 0)
        fq.match(ft)
        n = C.c_int(300)
        assert L.gb_match_download(ctx.handle, fq._h, None, None, None, C.byref(n)) == capi.GB_OK and n.value == 300
        bufs = [np.full(300, 12345, np.int32) for _ in range(3)]
        n = C.c_int(299)
        rc = L.gb_match_download(ctx.handle, fq._h, *[capi.ptr(b) for b in bufs], C.byref(n))
        assert rc == capi.GB_ERR_CAPACITY and n.value == 300
        assert all((b == 12345).all() for b in bufs)
        n = C.c_int(300)
        idx = np.full(300, -7, np.int32)
        assert L.gb_match_download(ctx.handle, fq._h, capi.ptr(idx), None, None, C.byref(n)) == capi.GB_OK
        assert np.array_equal(idx, want[0])
        assert_same(fq.matches(), want)
    finally:
        fq.close(); ft.close()


@pytest.mark.parametrize("band,mind,maxd", [(-1.0, 0.0, 10.0), (float("nan"), 0.0, 10.0), (1.0, 10.0, 9.0), (1.0, 0.0, -1e-3)])
def test_invalid_stereo_arguments(ctx, band, mind, maxd):
    kl = MC.grid_keypoints(np.random.default_rng(1), 10)
    d = synth.random_descriptors(10, 3)
    expect_error(capi.GB_ERR_INVALID, ctx.match_stereo, kl, d, kl, d, band, mind, maxd)
    f = Features(ctx, 16)
    try:
        f.upload(d, kl)
        expect_error(capi.GB_ERR_INVALID, f.match_stereo, f, band, mind, maxd)
    finally:
        f.close()
    assert_same(ctx.match_stereo(kl, d, kl, d, 1.0, 0.0, 10.0), oracle.match_stereo(kl, d, kl, d, 1.0, 0.0, 10.0))


# ---- a failed extraction on the train / right side ------------------------------------------------------------------------------
def _exact_again(ctx, fq, ft, stereo=None):
    img = synth.synth_frame(640, 480, 8)
    cfg = ctx.orb_cfg(nfeatures=500)
    fq.extract(img, 640, 480, cfg); ft.extract(np.roll(img, -6, axis=1), 640, 480, cfg)
    if stereo:
        fq.match_stereo(ft, *stereo)
    else:
        fq.match(ft)
    got = fq.matches()
    kq, dq = fq.download(); kt, dt = ft.download()
    assert_same(got, oracle.match_stereo(kq, dq, kt, dt, *stereo) if stereo else oracle.match_hamming(dq, dt))
    assert (got[0] >= 0).sum() > 100


@pytest.mark.parametrize("stereo", [None, (2.0, 0.0, 96.0)], ids=["match", "stereo"])
def test_failed_train_extraction_fails_download(ctx, stereo):
    """A match enqueued behind a train (right) extraction that kept more keypoints than its feature set holds: the download fails
    with GB_ERR_CAPACITY naming the train side, on every call, whether the query count is on the device or on the host -- not -1 /
    257 / 257 for every query.  The same context and feature sets are bit-exact again afterwards."""
    img = synth.synth_frame(640, 480, 3)
    cfg = ctx.orb_cfg(nfeatures=500)
    fq, small, good = Features(ctx, 2000), Features(ctx, 16), Features(ctx, 2000)

    def enqueue(q, t):
        q.match_stereo(t, *stereo) if stereo else q.match(t)

    try:
        for query_on_device in (True, False):
            if query_on_device:
                fq.extract(img, 640, 480, cfg)
            else:
                fq.upload(synth.random_descriptors(700, 1), MC.grid_keypoints(np.random.default_rng(0), 700))
            small.extract(img, 640, 480, cfg)
            enqueue(fq, small)
            for _ in range(2):
                expect_error(capi.GB_ERR_CAPACITY, fq.matches, text="train set")
            _exact_again(ctx, fq, good, stereo)
        # a train set whose status word says it failed although its count is plausible (the hook), and an empty query set
        t = synth.random_descriptors(900, 2)
        good.upload(t, MC.grid_keypoints(np.random.default_rng(1), 900))
        set_pending(ctx, good, 900, 950, 900)
        fq.upload(synth.random_descriptors(50, 3), MC.grid_keypoints(np.random.default_rng(2), 50))
        enqueue(fq, good)
        for _ in range(2):
            expect_error(capi.GB_ERR_CAPACITY, fq.matches, text="950")
        good.upload(t, MC.grid_keypoints(np.random.default_rng(1), 900))
        set_pending(ctx, good, 0, -2, 900)
        fq.upload(np.zeros((0, 32), np.uint8))
        enqueue(fq, good)
        expect_error(capi.GB_ERR_CAPACITY, fq.matches, text="4096")
        _exact_again(ctx, fq, good, stereo)
    finally:
        fq.close(); small.close(); good.close()


def test_failed_extraction_fails_bow_transform(ctx):
    """gb_bow_transform_features after an extraction that kept more keypoints than the feature set holds: GB_ERR_CAPACITY on every
    call, not an empty BowVector; the same vocabulary and context are exact again on the next frame."""
    from oracle import oracle as O
    vt = synth.synth_vocabulary(10, 3, seed=1)
    voc = Vocabulary(ctx, vt.k, vt.L, vt.weighting, vt.scoring, vt.child_num, vt.weight, vt.desc)
    img = synth.synth_frame(640, 480, 3)
    cfg = ctx.orb_cfg(nfeatures=500)
    small, good = Features(ctx, 16), Features(ctx, 2000)
    try:
        small.extract(img, 640, 480, cfg)
        for _ in range(2):
            expect_error(capi.GB_ERR_CAPACITY, voc.transform, small, 1, text="holds 16")
        good.extract(img, 640, 480, cfg)
        got = voc.transform(good, 1)
        _, desc = good.download()
        want = O.bow_transform(O.VocabularyArrays(vt.k, vt.L, vt.weighting, vt.scoring, vt.child_num, vt.weight, vt.desc), desc, 1)
        assert len(desc) > 100 and all(np.array_equal(got[k], want[k]) for k in ("words", "values", "fv_node", "fv_feat"))
    finally:
        voc.close(); small.close(); good.close()


# ---- one context through a fixed sequence of plans ------------------------------------------------------------------------------
SEQUENCE = [
    MC._c("seq_plain_q5", S(5), S(700), "near", seed=31, qtiles=1),
    MC._c("seq_stereo_dev_right", S(300), D(2000, 2400, 2000), seed=32, stereo=(1.0, 2.0, 10.0), qtiles=3),
    MC._c("seq_plain_q300tiles", S(300 * 128 - 5), S(900), "pool", seed=33, qtiles=300),
    MC._c("seq_dev_both_q300tiles", D(1000, 300 * 128, 1000), D(3000, 3000), "near", seed=34, qtiles=300),
    MC._c("seq_stereo_host", S(129), S(1000), seed=35, stereo=(0.0, -3.0, 3.0), qtiles=2),
    MC._c("seq_dev_splits257", D(1, 1, 1), D(8193, 8193, 256), "near", seed=36, qtiles=1, nsplit=257),
    MC._c("seq_plain_q1", S(1), S(1), seed=37, qtiles=1, nsplit=1),
    MC._c("seq_dev_t0", S(700), D(0, 900, 900), seed=38, t_count=0),
]


def test_plan_sequence_on_one_context(sm):
    """The partials and the tickets grow and shrink (query tiles 1 -> 300 -> 1) while plain, stereo, host-count and device-count
    launches alternate on one context; every launch == the oracle."""
    c = Context(0)
    try:
        for case in SEQUENCE + SEQUENCE[::-1]:
            run_case(c, case, sm)
    finally:
        c.close()
