"""ORB extraction from a distorted frame in one device-resident pass (gb_orb_extract_undistorted*, gb_remap_apply_to): the remap
writes the undistorted gray image straight into pyramid level 0 (remap_level0_kernel, csrc/remap.cu).

The result is by construction the composition of three operations that are each pinned bit for bit elsewhere -- oracle.remap_apply
(tests/test_oracle_remap.py: the reference's Undistorter), oracle.to_gray (cv2.cvtColor) and oracle.orb_extract (cv2.ORB) -- so every
comparison here is equality: all seven keypoint fields, every descriptor bit, every byte of level 0."""
import ctypes as C
import functools
import threading

import numpy as np
import pytest

import oracle
from oracle import oracle as O
from gslam_b200 import api, capi, synth
from gslam_b200.api import Context, Features, GbError, Remap, Vocabulary

pytestmark = pytest.mark.gpu
FIELDS = ("octave", "x", "y", "size", "angle", "response", "class_id")
BIG, MID, ODD = (1920, 1080, 1920, 1080), (752, 480, 640, 400), (203, 167, 161, 131)   # (w_in, h_in, w_out, h_out)
NKP = {BIG: 2000, MID: 1000, ODD: 150}
KINDS = ("gray", "bgr", "rgb")


def _bilinear_table(w_in, h_in, w_out, h_out, seed):
    """A smooth synthetic distortion in the reference's table format (indices / weights as prepareReMap lays them out)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h_out, 0:w_out].astype(np.float64)
    u = (x - w_out / 2) / w_out; v = (y - h_out / 2) / h_out
    r2 = u * u + v * v
    k = 1 + rng.uniform(-0.4, -0.1) * r2 + 0.1 * r2 * r2
    sx = (u * k * 1.15 + 0.5) * w_in; sy = (v * k * 1.15 + 0.5) * h_in
    out = (sx < 0) | (sy < 0) | (sx >= w_in) | (sy >= h_in)
    rx = np.where(out, -1, sx).astype(np.float32)
    ry = np.where(out, -1, sy).astype(np.float32)
    xi = rx.astype(np.int32); yi = ry.astype(np.int32)
    fx = rx - xi; fy = ry - yi; fxy = fx * fy
    idx = np.stack([yi * w_in + xi, yi * w_in + xi + 1, (yi + 1) * w_in + xi, (yi + 1) * w_in + xi + 1], -1).astype(np.int32)
    coef = np.stack([1 - fx - fy + fxy, fx - fxy, fy - fxy, fxy], -1).astype(np.float32)
    idx[out] = 0; coef[out] = 0
    return idx.reshape(-1, 4), coef.reshape(-1, 4), rx.reshape(-1)


@functools.lru_cache(maxsize=None)
def table(size, seed=None):
    w_in, h_in, w_out, h_out = size
    idx, coef, rx = _bilinear_table(w_in, h_in, w_out, h_out, seed=w_in if seed is None else seed)
    inside = rx >= 0
    # the table has what the kernel must get right: pixels outside the input, and last-row / last-column taps beyond it
    assert 0.5 < inside.mean() < 1.0 and (idx[inside].max(axis=1) >= w_in * h_in).any()
    assert (idx[inside, 1] % w_in == 0).any()
    return idx, coef, rx


def frame(size, kind, seed=2):
    img = synth.synth_frame(size[0], size[1], seed=seed)
    return img if kind == "gray" else np.stack([img, np.roll(img, 9, axis=1), 255 - img], axis=2)


def undistorted_gray(size, kind, img, seed=None):
    und = oracle.remap_apply(img, *table(size, seed), (size[3], size[2]))
    return und if kind == "gray" else oracle.to_gray(und, rgb=kind == "rgb")


@functools.lru_cache(maxsize=None)
def expected(size, kind, seed=2):
    """(keypoints, descriptors) of the composition, and the undistorted gray frame it saw."""
    g = undistorted_gray(size, kind, frame(size, kind, seed))
    return oracle.orb_extract(g, NKP[size]) + (g,)


def new_map(ctx, size, seed=None):
    return Remap(ctx, *size, *table(size, seed))


def assert_features(kps, desc, wk, wd, what=""):
    assert len(kps) == len(wk), (what, len(kps), len(wk))
    for f in FIELDS:
        assert np.array_equal(kps[f], wk[f]), (what, f)
    assert np.array_equal(desc, wd), what


def level0(ctx, w, h):
    L = capi.lib()
    L.gb_dbg_orb_level.restype = C.c_int
    L.gb_dbg_orb_level.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    out = np.zeros((h, w), np.uint8); lw, lh = C.c_int(), C.c_int()
    ctx._check(L.gb_dbg_orb_level(ctx._h, 0, api.ptr(out), out.size, C.byref(lw), C.byref(lh)))
    assert (lw.value, lh.value) == (w, h)
    return out


def to_device(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()   # written on torch's stream, read on the ctx's
    return t


# ---- 1. equality with the composition, and with the two-call route ------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", [BIG, MID, ODD], ids=["1080p", "752x480_to_640x400", "203x167_to_161x131"])
def test_equals_composition_and_two_call_route(ctx, size, kind):
    wk, wd, gray = expected(size, kind)
    assert len(wk) > NKP[size] // 2
    img = frame(size, kind)
    m = new_map(ctx, size)
    kps, desc = ctx.orb_extract_undistorted(m, img, NKP[size], rgb=kind == "rgb")
    assert_features(kps, desc, wk, wd, "fused vs oracle")
    assert size[2] % 4 == 0 or (size[2] + 127) // 128 * 128 > size[2]
    assert np.array_equal(level0(ctx, size[2], size[3]), gray)
    k2, d2 = ctx.orb_extract(m.apply(img), NKP[size], rgb=kind == "rgb")
    assert_features(kps, desc, k2, d2, "fused vs apply + orb_extract")
    m.close()


# ---- 2. gb_remap_apply_to -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("source", ["host", "host_pitched", "device", "device_pitched"])
@pytest.mark.parametrize("ch", [1, 3])
@pytest.mark.parametrize("size", [MID, ODD], ids=["752x480_to_640x400", "203x167_to_161x131"])
def test_apply_to_equals_apply(ctx, size, ch, source):
    import torch
    w_in, h_in, w_out, h_out = size
    img = frame(size, "gray" if ch == 1 else "bgr", seed=5)
    m = new_map(ctx, size)
    want = m.apply(img).reshape(h_out, w_out * ch)
    assert np.array_equal(want, oracle.remap_apply(img, *table(size), (h_out, w_out)).reshape(h_out, w_out * ch))
    dst_pitch = w_out * ch + 13
    dst = torch.full((h_out, dst_pitch), 0xA5, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    row, pitch = w_in * ch, w_in * ch + 29
    wide = np.random.default_rng(ch).integers(0, 256, (h_in, pitch), dtype=np.uint8)
    wide[:, :row] = img.reshape(h_in, row)
    if source == "host":
        m.apply_to(img, dst.data_ptr(), dst_pitch)
    elif source == "host_pitched":
        m.apply_to(wide, dst.data_ptr(), dst_pitch, channels=ch, pitch=pitch)
    elif source == "device":
        t = to_device(img)
        m.apply_to(t.data_ptr(), dst.data_ptr(), dst_pitch, channels=ch, device_ptr=True)
    else:
        t = to_device(wide)
        m.apply_to(t.data_ptr(), dst.data_ptr(), dst_pitch, channels=ch, device_ptr=True, pitch=pitch)
    ctx.sync()
    got = dst.cpu().numpy()
    assert np.array_equal(got[:, :w_out * ch], want)
    assert (got[:, w_out * ch:] == 0xA5).all()
    m.close()


# ---- 3. device-resident chaining ----------------------------------------------------------------------------------------------------
def test_match_and_bow_chain_behind_device_frames(ctx):
    size, n = MID, NKP[MID]
    a, b = frame(size, "bgr", seed=2), frame(size, "bgr", seed=2).copy()
    b = np.ascontiguousarray(np.roll(b, 5, axis=1))
    ka, da, _ = expected(size, "bgr")
    kb, db = oracle.orb_extract(undistorted_gray(size, "bgr", b), n)
    ta, tb = to_device(a), to_device(b)
    m = new_map(ctx, size)
    v = O.synth_vocabulary(10, 4, seed=11)
    dv = Vocabulary(ctx, v.k, v.L, v.weighting, v.scoring, v.child_num, v.weight, v.desc)
    cfg = ctx.orb_cfg(nfeatures=n)
    fa, fb = Features(ctx, 2 * n + 256), Features(ctx, 2 * n + 256)
    fa.extract_undistorted(m, ta.data_ptr(), cfg, channels=3, device_ptr=True)
    fb.extract_undistorted(m, tb.data_ptr(), cfg, channels=3, device_ptr=True)
    fa.match(fb)
    bow = dv.transform(fa, 1)
    got_m = fa.matches()
    assert_features(*fa.download(), ka, da, "frame a")
    assert_features(*fb.download(), kb, db, "frame b")
    ua, ub = Features(ctx, 2 * n + 256), Features(ctx, 2 * n + 256)
    ua.upload(da, ka); ub.upload(db, kb)
    ua.match(ub)
    want_bow = dv.transform(ua, 1)
    for g, w, o in zip(got_m, ua.matches(), oracle.match_hamming(da, db)):
        assert np.array_equal(g, w) and np.array_equal(g, o)
    ob = O.bow_transform(v, da, 1)
    for k in ("words", "values", "fv_node", "fv_feat"):
        assert np.array_equal(bow[k], want_bow[k]) and np.array_equal(bow[k], ob[k]), k
    for x in (fa, fb, ua, ub, dv, m):
        x.close()


def test_stereo_match_chains_behind_two_maps(ctx):
    size, n = MID, NKP[MID]
    left = frame(size, "gray", seed=8)
    right = np.ascontiguousarray(np.roll(left, -12, axis=1))
    ml, mr = new_map(ctx, size), new_map(ctx, size, seed=753)
    kl, dl = oracle.orb_extract(undistorted_gray(size, "gray", left), n)
    kr, dr = oracle.orb_extract(undistorted_gray(size, "gray", right, seed=753), n)
    tl, tr = to_device(left), to_device(right)
    cfg = ctx.orb_cfg(nfeatures=n)
    fl, fr = Features(ctx, 2 * n + 256), Features(ctx, 2 * n + 256)
    fl.extract_undistorted(ml, tl.data_ptr(), cfg, device_ptr=True)
    fr.extract_undistorted(mr, tr.data_ptr(), cfg, device_ptr=True)
    fl.match_stereo(fr, band=2.0, min_disp=0.0, max_disp=64.0)
    got = fl.matches()
    want = oracle.match_stereo(kl, dl, kr, dr, 2.0, 0.0, 64.0)
    assert (want[0] >= 0).sum() > 100
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert_features(*fl.download(), kl, dl, "left")
    assert_features(*fr.download(), kr, dr, "right")
    for x in (fl, fr, ml, mr):
        x.close()


# ---- 4. one map, two contexts, two threads ------------------------------------------------------------------------------------------
def test_one_map_serves_two_contexts_on_two_threads(ctx):
    size, n = MID, NKP[MID]
    m = new_map(ctx, size)
    kinds = ("gray", "bgr")
    want = [expected(size, k) for k in kinds]
    frames = [frame(size, k) for k in kinds]
    want_und = [m.apply(f) for f in frames]  # gb_remap_apply from one thread: the map holds no per-call state
    ctxs = [Context(0), Context(0)]
    go = threading.Barrier(2)
    got, und, err = [[], []], [[], []], []

    def run(i):
        try:
            go.wait()
            for _ in range(4):
                got[i].append(ctxs[i].orb_extract_undistorted(m, frames[i], n))
                und[i].append(m.apply(frames[i], ctx=ctxs[i]))
        except BaseException as e:
            err.append(e)
            go.abort()
    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not err, err
    for i in range(2):
        for kps, desc in got[i]:
            assert_features(kps, desc, want[i][0], want[i][1], kinds[i])
        for u in und[i]:
            assert np.array_equal(u, want_und[i]), kinds[i]
    for c in ctxs:
        c.close()
    m.close()


# ---- 5. repeated use and size changes -----------------------------------------------------------------------------------------------
def test_size_changes_on_one_ctx():
    c = Context(0)
    ms, mm = new_map(c, ODD), new_map(c, MID)
    plain = synth.synth_frame(517, 389, seed=31)
    want_plain = oracle.orb_extract(plain, 350)
    for _ in range(2):
        assert_features(*c.orb_extract_undistorted(ms, frame(ODD, "rgb"), NKP[ODD], rgb=True), *expected(ODD, "rgb")[:2], "odd rgb")
        assert_features(*c.orb_extract(plain, 350), *want_plain, "plain")
        assert_features(*c.orb_extract_undistorted(mm, frame(MID, "bgr"), NKP[MID]), *expected(MID, "bgr")[:2], "mid bgr")
        assert_features(*c.orb_extract_undistorted(mm, frame(MID, "gray"), NKP[MID]), *expected(MID, "gray")[:2], "mid gray")
    ms.close(); mm.close(); c.close()


# ---- 6. capacity and argument errors: all rejected on the host, before any launch ------------------------------------------------
def test_capacity_protocol(ctx):
    wk, wd, _ = expected(ODD, "gray")
    m = new_map(ctx, ODD)
    img = frame(ODD, "gray")
    cfg = ctx.orb_cfg(nfeatures=NKP[ODD])
    cap = len(wk) - 1
    kps = np.zeros(cap, capi.KP_DTYPE); desc = np.full((cap, 32), 0x5A, np.uint8); kps["class_id"] = 77
    n = C.c_int(cap)
    rc = ctx._lib.gb_orb_extract_undistorted(ctx._h, m._h, api.ptr(img), 1, 0, C.byref(cfg), api.ptr(kps), api.ptr(desc), C.byref(n))
    assert rc == capi.GB_ERR_CAPACITY and n.value == len(wk)
    assert (desc == 0x5A).all() and (kps["class_id"] == 77).all() and not kps["x"].any()
    n = C.c_int(0)   # capacity 0: the count alone
    rc = ctx._lib.gb_orb_extract_undistorted(ctx._h, m._h, api.ptr(img), 1, 0, C.byref(cfg), None, None, C.byref(n))
    assert rc == capi.GB_ERR_CAPACITY and n.value == len(wk)
    f = Features(ctx, cap)   # the device-resident form reports it where gb_orb_extract_to does: at the count
    f.extract_undistorted(m, img, cfg)
    with pytest.raises(GbError) as e:
        f.count()
    assert e.value.code == capi.GB_ERR_CAPACITY
    f.close(); m.close()


def test_argument_errors(ctx):
    import torch
    L = ctx._lib
    w_in, h_in, w_out, h_out = ODD
    m = new_map(ctx, ODD)
    cfg = ctx.orb_cfg(nfeatures=100)
    img = np.zeros((h_in, w_in, 4), np.uint8)
    f = Features(ctx, 456)
    kps = np.zeros(456, capi.KP_DTYPE); desc = np.zeros((456, 32), np.uint8)
    dst = torch.zeros((h_out, w_out * 4), dtype=torch.uint8, device="cuda")
    before = ctx.launch_count()

    def invalid(rc, needs_text=True):
        assert rc == capi.GB_ERR_INVALID
        assert not needs_text or len(L.gb_last_error(ctx._h)) > 0

    for ch in (2, 4):
        invalid(L.gb_orb_extract_undistorted(ctx._h, m._h, api.ptr(img), ch, 0, C.byref(cfg), api.ptr(kps), api.ptr(desc), C.byref(C.c_int(456))))
        invalid(L.gb_orb_extract_undistorted_to(ctx._h, m._h, api.ptr(img), 0, w_in * ch, ch, 0, C.byref(cfg), f._h))
        invalid(L.gb_remap_apply_to(ctx._h, m._h, api.ptr(img), 0, w_in * ch, ch, C.c_void_p(dst.data_ptr()), w_out * ch))
    invalid(L.gb_orb_extract_undistorted_to(ctx._h, m._h, api.ptr(img), 0, w_in * 3 - 1, 3, 0, C.byref(cfg), f._h))
    invalid(L.gb_remap_apply_to(ctx._h, m._h, api.ptr(img), 0, w_in - 1, 1, C.c_void_p(dst.data_ptr()), w_out))
    invalid(L.gb_remap_apply_to(ctx._h, m._h, api.ptr(img), 0, w_in * 3, 3, C.c_void_p(dst.data_ptr()), w_out * 3 - 1))
    invalid(L.gb_orb_extract_undistorted(ctx._h, None, api.ptr(img), 1, 0, C.byref(cfg), api.ptr(kps), api.ptr(desc), C.byref(C.c_int(456))), False)
    invalid(L.gb_orb_extract_undistorted_to(ctx._h, None, api.ptr(img), 0, w_in, 1, 0, C.byref(cfg), f._h), False)
    invalid(L.gb_orb_extract_undistorted_to(ctx._h, m._h, None, 0, w_in, 1, 0, C.byref(cfg), f._h), False)
    invalid(L.gb_orb_extract_undistorted_to(ctx._h, m._h, api.ptr(img), 0, w_in, 1, 0, C.byref(cfg), None), False)
    invalid(L.gb_remap_apply_to(ctx._h, None, api.ptr(img), 0, w_in, 1, C.c_void_p(dst.data_ptr()), w_out), False)
    invalid(L.gb_remap_apply_to(ctx._h, m._h, api.ptr(img), 0, w_in, 1, None, w_out), False)
    bad_cfg = ctx.orb_cfg(nfeatures=100, edge_threshold=10)
    invalid(L.gb_orb_extract_undistorted_to(ctx._h, m._h, api.ptr(img), 0, w_in, 1, 0, C.byref(bad_cfg), f._h))
    for wrong in (np.zeros((h_in, w_in + 1), np.uint8), np.zeros((h_out, w_out), np.uint8), np.zeros((h_in * w_in,), np.uint8)):
        with pytest.raises(GbError) as e:
            ctx.orb_extract_undistorted(m, wrong, 100)
        assert e.value.code == capi.GB_ERR_INVALID and "shape" in str(e.value)
        with pytest.raises(GbError):
            f.extract_undistorted(m, wrong, cfg)
        with pytest.raises(GbError):
            m.apply_to(wrong, dst.data_ptr(), w_out * 4)
    assert ctx.launch_count() == before
    f.close(); m.close()


def test_output_too_small_for_the_border_behaves_as_a_frame_of_that_size(ctx):
    def outcome(fn):
        try:
            return ("ok", len(fn()[0]))
        except GbError as e:
            return ("error", e.code)
    size = (96, 72, 48, 40)
    idx, coef, rx = _bilinear_table(*size, seed=1)
    m = Remap(ctx, *size, idx, coef, rx)
    img = synth.synth_frame(96, 72, seed=4)
    und = oracle.remap_apply(img, idx, coef, rx, (40, 48))
    assert outcome(lambda: ctx.orb_extract_undistorted(m, img, 100)) == outcome(lambda: ctx.orb_extract(und, 100))
    m.close()


# ---- 7. one launch more than a plain extraction ---------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["gray", "bgr"])
def test_one_more_launch_than_a_plain_device_extraction(ctx, kind):
    size, n = MID, NKP[MID]
    w_in, h_in, w_out, h_out = size
    m = new_map(ctx, size)
    cfg = ctx.orb_cfg(nfeatures=n)
    f = Features(ctx, 2 * n + 256)
    t_plain = to_device(expected(size, kind)[2])
    t_src = to_device(frame(size, kind))
    f.extract(t_plain.data_ptr(), w_out, h_out, cfg, device_ptr=True, pitch=w_out)
    c0 = ctx.launch_count()
    f.extract(t_plain.data_ptr(), w_out, h_out, cfg, device_ptr=True, pitch=w_out)
    c1 = ctx.launch_count()
    f.extract_undistorted(m, t_src.data_ptr(), cfg, channels=1 if kind == "gray" else 3, device_ptr=True)
    c2 = ctx.launch_count()
    assert c2 - c1 == c1 - c0 + 1
    assert_features(*f.download(), *expected(size, kind)[:2])
    f.close(); m.close()
