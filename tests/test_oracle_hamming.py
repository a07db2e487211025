"""Pins oracle/hamming_ref.c against (a) the reference's own hamming32 (oracle/_ref, compiled from Vocabulary.h:485-491),
(b) cv2.BFMatcher golden vectors (tests/golden/hamming_golden.npz) and (c) known answers (SURVEY.md §8c KAT-H / KAT-M)."""
import os

import numpy as np
import pytest

import oracle
from gslam_b200 import synth

import _match_cases as MC

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "hamming_golden.npz"))


def test_kat_distance():
    z = np.zeros(32, np.uint8); o = np.full(32, 255, np.uint8)
    L = oracle.lib()
    assert L.orc_hamming256(z.ctypes.data, o.ctypes.data) == 256
    assert L.orc_hamming256(o.ctypes.data, o.ctypes.data) == 0
    for bit in range(256):  # single-bit walk
        a = np.zeros(32, np.uint8); a[bit // 8] = 1 << (bit % 8)
        assert L.orc_hamming256(a.ctypes.data, z.ctypes.data) == 1
        assert L.orc_hamming256(a.ctypes.data, o.ctypes.data) == 255


def test_against_numpy_popcount():
    q = synth.random_descriptors(64, 1); t = synth.random_descriptors(80, 2)
    d = np.unpackbits(q[:, None, :] ^ t[None, :, :], axis=2).sum(axis=2)
    idx, d1, d2 = oracle.match_hamming(q, t)
    assert np.array_equal(idx, d.argmin(axis=1))  # argmin takes the first minimum == lowest index
    assert np.array_equal(d1, d.min(axis=1))
    assert np.array_equal(d2, np.sort(d, axis=1)[:, 1])


@pytest.mark.skipif(not oracle.have_ref(), reason="oracle/_ref not built (needs a GSLAM checkout)")
def test_against_reference_hamming32_live():
    q = synth.random_descriptors(1000, 42); t = synth.random_descriptors(1000, 43)
    R = oracle.ref(); L = oracle.lib()
    for a, b in zip(q, t):
        assert int(R.ref_hamming32(a.ctypes.data, b.ctypes.data)) == L.orc_hamming256(a.ctypes.data, b.ctypes.data)


def test_against_reference_hamming32_golden():
    if "ref_hamming32" not in G:
        pytest.skip("fixture generated without oracle/_ref")
    L = oracle.lib()
    q, t = np.ascontiguousarray(G["q"]), np.ascontiguousarray(G["t"])
    for (a, b), want in zip(G["ref_pairs"], G["ref_hamming32"]):
        assert L.orc_hamming256(q[a].ctypes.data, t[b].ctypes.data) == int(want)


def test_against_cv2_bfmatcher_golden():
    idx, d1, d2 = oracle.match_hamming(G["q"], G["t"])
    assert np.array_equal(idx, G["idx"]) and np.array_equal(idx, G["idx_knn"])
    assert np.array_equal(d1, G["d1"])
    assert np.array_equal(d2, G["d2"])
    # the engineered ties resolved to the lowest train index
    assert idx[0] == 7 and idx[1] == 49 and d1[0] == 0 and d2[0] == 0


def test_against_cv2_live():
    cv2 = pytest.importorskip("cv2")
    q = synth.random_descriptors(200, 5); t = synth.random_descriptors(150, 6)
    t[20] = t[3]; q[9] = t[3]
    m = cv2.BFMatcher(cv2.NORM_HAMMING).match(q, t)
    idx, d1, _ = oracle.match_hamming(q, t)
    assert [x.trainIdx for x in m] == idx.tolist()
    assert [int(x.distance) for x in m] == d1.tolist()


def test_edge_cases():
    q = synth.random_descriptors(5, 1)
    idx, d1, d2 = oracle.match_hamming(q, np.zeros((0, 32), np.uint8))
    assert (idx == -1).all() and (d1 == 257).all() and (d2 == 257).all()
    idx, d1, d2 = oracle.match_hamming(q, q[:1])
    assert (idx == 0).all() and d1[0] == 0 and (d2 == 257).all()
    idx, d1, d2 = oracle.match_hamming(np.zeros((0, 32), np.uint8), q)
    assert idx.size == 0


_stereo_numpy = MC.stereo_numpy


def _stereo_case(rng, nl, nr, dup=False):
    kl = np.zeros(nl, oracle.KP_DTYPE); kr = np.zeros(nr, oracle.KP_DTYPE)
    kl["x"] = rng.uniform(0, 752, nl).astype(np.float32); kl["y"] = np.round(rng.uniform(0, 480, nl) * 2) / 2
    kr["x"] = rng.uniform(0, 752, nr).astype(np.float32); kr["y"] = np.round(rng.uniform(0, 480, nr) * 2) / 2
    dl = rng.integers(0, 256, (nl, 32), dtype=np.uint8); dr = rng.integers(0, 256, (nr, 32), dtype=np.uint8)
    if dup and nr > 8:   # engineered ties: identical right descriptors on the same row
        dr[5] = dr[2]; kr["y"][5] = kr["y"][2]; dr[7] = dr[2]; kr["y"][7] = kr["y"][2]
    return kl, dl, kr, dr


def test_stereo_rowband_match_equals_numpy_restatement():
    rng = np.random.default_rng(3)
    for (nl, nr, band, mind, maxd, dup) in [(300, 280, 2.0, 0.0, 96.0, False), (64, 500, 0.0, -5.0, 1e9, True), (200, 0, 2.0, 0.0, 50.0, False),
                                            (1, 1, 1000.0, -1e9, 1e9, False), (500, 500, 2.5, 3.0, 200.0, True)]:
        kl, dl, kr, dr = _stereo_case(rng, nl, nr, dup)
        got = oracle.match_stereo(kl, dl, kr, dr, band, mind, maxd)
        want = _stereo_numpy(kl, dl, kr, dr, band, mind, maxd)
        for g, w in zip(got, want):
            assert np.array_equal(g, w)
    # unrestricted band == the plain matcher
    kl, dl, kr, dr = _stereo_case(rng, 100, 120)
    a = oracle.match_stereo(kl, dl, kr, dr, 1e9, -1e9, 1e9); b = oracle.match_hamming(dl, dr)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


# ---- the matcher's work split and the stereo predicate at their edges (tests/_match_cases.py; the device side is
# tests/test_match_paths_gpu.py) ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sm", MC.SM_COUNTS)
@pytest.mark.parametrize("case", MC.CASES, ids=lambda c: c.id)
def test_match_case_reaches_its_boundary(case, sm):
    MC.check_reach(case, case.plan(sm), sm)


def test_match_plan_mirror_known_splits():
    """The planner's splits for the shapes of the parity tests and beyond them, at 132 SMs."""
    want = {(2000, 2000): (16, 17, 120), (513, 4097): (5, 52, 80), (3000, 50): (24, 2, 32), (40000, 5000): (313, 5, 1024),
            (1, 100000): (1, 261, 384), (33665, 100): (264, 1, 104), (33536, 100): (262, 2, 56), (10, 0): (1, 1, 8), (0, 10): (0, 0, 0)}
    for (nq, nt), p in want.items():
        assert MC.plan(nq, nt, sm_count=132) == p, (nq, nt)
    # the expect hints of a count still on the device: below the launch size they shape the split, above it they are ignored
    assert MC.plan(4256, 4256, 2039, 2039) == (34, 36, 120)
    assert MC.plan(4256, 4256, 9999, 9999) == MC.plan(4256, 4256) == MC.plan(4256, 4256, 0, 0)
    for sm in MC.SM_COUNTS:  # every split but the last is full, and the splits cover the train rows
        for nq, nt, eq, et in [(1, 1, 0, 0), (7, 33, 0, 0), (300, 2000, 0, 500), (5000, 70000, 100, 0), (1, 8193, 0, 256)]:
            qt, ns, ch = MC.plan(nq, nt, eq, et, sm)
            assert qt * MC.KQ >= nq and (ns - 1) * ch < nt <= ns * ch and ch % 8 == 0 and ch <= MC.MAX_CHUNK


@pytest.mark.parametrize("case", [c for c in MC.CASES if c.stereo is not None], ids=lambda c: c.id)
def test_stereo_case_oracle_equals_numpy(case):
    s = case.shape(132); d = case.data(132)
    kl, kr = d["kl"][:s.nq], d["kr"][:s.nt]
    got = oracle.match_stereo(kl, d["q"][:s.nq], kr, d["t"][:s.nt], *case.stereo)
    want = _stereo_numpy(kl, d["q"][:s.nq], kr, d["t"][:s.nt], *case.stereo)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert (got[0] >= 0).sum() > s.nq // 2 if s.nt else (got[0] == -1).all()


@pytest.mark.parametrize("edge", MC.STEREO_EDGES, ids=lambda e: e.id)
def test_stereo_edge_oracle_equals_numpy(edge):
    """The oracle's stereo predicate against the numpy restatement exactly where it is decided: |dy| == band (band 0 too),
    disparities on min_disp and max_disp (min == max, negative windows), infinite windows and bands, -0.0, float disparities that
    round near 16384, NaN coordinates."""
    kl, dl, kr, dr, band, mind, maxd = edge.make(np.random.default_rng(5))
    MC.stereo_hits(edge, kl, kr, band, mind, maxd)
    got = oracle.match_stereo(kl, dl, kr, dr, band, mind, maxd)
    want = _stereo_numpy(kl, dl, kr, dr, band, mind, maxd)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    if "nan" in edge.hits:  # a NaN coordinate is never a candidate, whatever the band and window
        assert (got[0][np.isnan(kl["x"]) | np.isnan(kl["y"])] == -1).all()
        bad = np.isnan(kr["x"]) | np.isnan(kr["y"])
        assert not np.isin(got[0], np.nonzero(bad)[0]).any()
        assert (got[0][~(np.isnan(kl["x"]) | np.isnan(kl["y"]))] >= 0).all()
    if edge.id == "one_candidate":
        assert (got[0][:-1] == np.arange(len(kl) - 1)).all() and (got[2] == 257).all() and got[0][-1] == -1 and got[1][-1] == 257
