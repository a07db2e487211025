"""Hamming / stereo matcher cases at the boundaries of its work split, shared by the CPU checks of the split planner
(tests/test_oracle_hamming.py) and the device-vs-oracle parity tests (tests/test_match_paths_gpu.py).

gb_match_launch (gslam_b200/csrc/match.cu) splits the work into `qtiles` tiles of 128 queries (blockIdx.x) times `nsplit` splits of
`chunk` train rows (blockIdx.y), planned on the host from the SM count, the launch sizes and -- while a count is still on the
device -- the `expect` hints of the feature sets.  When the train count is on the device the kernel recomputes the number of
splits that hold rows (at least one) and the other y-CTAs leave; the last CTA of a query tile to arrive merges the partials of
the splits in ascending order.  `plan` mirrors the host planner; each case states the boundary it exists to reach as facts
about that plan and its own shape, which `check_reach` asserts, so that an edit to a case or to the planner cannot quietly turn a
boundary case into an easy one.  Shapes whose boundary depends on the SM count are functions of it: every case reaches its
boundary on a 132-SM and on a 114-SM H100.

Facts (values may be functions of the SM count):
  qtiles, nsplit, chunk       the plan's value
  nsplit_gt                   nsplit is larger than this
  nt_max / nt_min             the real train count is at most / at least this
  last_rows                   rows of the real train count in its last split
  tail_q                      queries in the last query tile of the real query count (128: a full tile)
  dev_splits                  splits that hold train rows when the kernel reads the train count on the device
  dev_splits_lt_launch        ... fewer than the launch has
  q_count / t_count           the real count read on the device
  q_at_cap / t_at_cap         the count read on the device equals the launch size (the feature set's capacity)
  q_expect / t_expect         the expect hint is "below", "equal" to or "above" the real count (or "unknown": 0)
"""
import dataclasses

import numpy as np

KQ = 128            # queries per CTA (kQPerCta)
MAX_CHUNK = 1024    # train rows per split at most (32 KB of shared memory)
SM_COUNTS = (132, 114)  # H100 SXM and H100 PCIe


def _du(a, b):
    return (a + b - 1) // b


def plan(nq, nt, eq=0, et=0, sm_count=132):
    """Mirror of gb_match_launch's work split -> (qtiles, nsplit, chunk).  nq / nt: the launch sizes (the capacities when a count
    is on the device), eq / et: the expect hints (<= 0 or above the launch size: use the launch size).  (0, 0, 0): no launch."""
    if nq <= 0:
        return 0, 0, 0
    qtiles = _du(nq, KQ)
    if eq <= 0 or eq > nq:
        eq = nq
    if et <= 0 or et > nt:
        et = nt
    if nt <= 0:
        return qtiles, 1, 8
    nsplit = max(1, min(_du(2 * sm_count, _du(eq, KQ)), _du(et, 32)))
    chunk = min(_du(_du(et, nsplit), 8) * 8, MAX_CHUNK)
    return qtiles, _du(nt, chunk), chunk


def device_splits(nt, chunk):
    """Splits that hold train rows when the kernel reads the train count nt on the device (at least one: it writes the outputs of
    an empty train set)."""
    return max(1, _du(nt, chunk))


def _v(x, sm):
    return x(sm) if callable(x) else x


@dataclasses.dataclass(frozen=True)
class Side:
    n: object               # rows the match sees
    cap: object = None      # None: the count is on the host; else the count is on the device and the launch covers `cap` rows
    expect: object = 0      # the launch hint while the count is on the device (0: unknown)


@dataclasses.dataclass(frozen=True)
class Shape:
    nq: int
    nt: int
    qcap: int
    tcap: int
    eq: int
    et: int
    q_dev: bool
    t_dev: bool

    @property
    def device(self):
        return self.q_dev or self.t_dev


@dataclasses.dataclass(frozen=True)
class MatchCase:
    id: str
    q: Side
    t: Side
    desc: str = "random"    # "random", "pool" (train rows drawn from 5 rows: ties in every split) or "near" (queries are train
                            # rows with 0..3 bits flipped: small distances)
    seed: int = 0
    stereo: tuple = None    # (band, min_disp, max_disp) on integer keypoint coordinates, or None for the plain matcher
    reach: tuple = ()

    def shape(self, sm):
        nq, nt = _v(self.q.n, sm), _v(self.t.n, sm)
        qd, td = self.q.cap is not None, self.t.cap is not None
        qcap = _v(self.q.cap, sm) if qd else nq
        tcap = _v(self.t.cap, sm) if td else nt
        # gb_match_features passes both sets' hints once either count is on the device; a set whose count is on the host has 0
        eq = _v(self.q.expect, sm) if qd else 0
        et = _v(self.t.expect, sm) if td else 0
        return Shape(nq, nt, qcap, tcap, eq, et, qd, td)

    def plan(self, sm):
        s = self.shape(sm)
        if s.device:
            return plan(s.qcap, s.tcap, s.eq, s.et, sm)
        return plan(s.nq, s.nt, 0, 0, sm)

    def data(self, sm):
        """Descriptors (and keypoints) at the launch sizes.  Rows beyond a count read on the device are poison: train rows equal
        to query rows (distance 0, and for stereo at a disparity inside the window), so that reading past a count changes the
        answer."""
        s = self.shape(sm)
        rng = np.random.default_rng(self.seed)
        t = rng.integers(0, 256, (s.tcap, 32), dtype=np.uint8)
        if self.desc == "pool":
            pool = rng.integers(0, 256, (5, 32), dtype=np.uint8)
            t = pool[rng.integers(0, 5, s.tcap)]
        q = rng.integers(0, 256, (s.qcap, 32), dtype=np.uint8)
        if self.desc == "near" and s.nt > 0:
            q = t[rng.integers(0, s.nt, s.qcap)].copy()
            for i in range(s.qcap):
                for b in rng.integers(0, 256, rng.integers(0, 4)):
                    q[i, b // 8] ^= np.uint8(1 << (b % 8))
        out = dict(q=q, t=t, kl=None, kr=None)
        if s.tcap > s.nt and s.qcap > 0:
            t[s.nt:] = q[np.arange(s.nt, s.tcap) % s.qcap]
        if self.stereo is not None:
            kl, kr = grid_keypoints(rng, s.qcap), grid_keypoints(rng, s.tcap)
            if s.tcap > s.nt and s.qcap > 0:
                src = np.arange(s.nt, s.tcap) % s.qcap
                kr["x"][s.nt:] = kl["x"][src] - np.float32(self.stereo[1])
                kr["y"][s.nt:] = kl["y"][src]
            out.update(kl=kl, kr=kr)
        return out


def grid_keypoints(rng, n, w=48, h=6):
    """Keypoints on a small integer grid: disparities and row offsets land exactly on the window's and the band's edges."""
    from gslam_b200.capi import KP_DTYPE
    k = np.zeros(n, KP_DTYPE)
    k["x"] = rng.integers(16, 16 + w, n).astype(np.float32)
    k["y"] = rng.integers(0, h, n).astype(np.float32)
    return k


def S(n):
    return Side(n)


def D(n, cap, expect=0):
    return Side(n, cap, expect)


def _c(id, q, t, desc="random", seed=0, stereo=None, **reach):
    return MatchCase(id, q, t, desc, seed, stereo, tuple(sorted(reach.items())))


TWO_SM = lambda sm: 2 * sm  # noqa: E731

CASES = [
    # counts on the host (gb_match_hamming / gb_match_stereo)
    _c("q1_t1", S(1), S(1), seed=1, nsplit=1, nt_max=32, tail_q=1),
    _c("q127_t32", S(127), S(32), "near", seed=2, nsplit=1, nt_max=32, tail_q=127),
    _c("q128_t33", S(128), S(33), "pool", seed=3, qtiles=1, nsplit=2, chunk=24, last_rows=9, tail_q=128),
    _c("q129_t1000", S(129), S(1000), "pool", seed=4, qtiles=2, nsplit=32, chunk=32, last_rows=8, tail_q=1),
    _c("one_split_wide", S(lambda sm: 2 * sm * KQ - 127), S(1000), "near", seed=5, qtiles=TWO_SM, nsplit=1, nt_min=33, tail_q=1),
    _c("tiles_2sm_minus1", S(lambda sm: 2 * sm * KQ - 1), S(33), "pool", seed=6, qtiles=TWO_SM, nsplit=1, nt_min=33, tail_q=127),
    _c("chunk1024_last1", S(lambda sm: 2 * sm * KQ + 1), S(4 * MAX_CHUNK + 1), "pool", seed=7, qtiles=lambda sm: 2 * sm + 1, nsplit=5,
       chunk=MAX_CHUNK, last_rows=1, tail_q=1),
    _c("two_splits_last", S(lambda sm: (2 * sm - 1) * KQ), S(2000), "near", seed=8, qtiles=lambda sm: 2 * sm - 1, nsplit=2, chunk=1000,
       tail_q=128),
    _c("q1_splits_2sm", S(1), S(lambda sm: 2 * sm * 384), "near", seed=9, nsplit=TWO_SM, chunk=384, last_rows=384),
    _c("t0", S(300), S(0), seed=10, qtiles=3, nsplit=1, chunk=8, nt_max=0),
    # a count on the device (gb_match_features behind an extraction in flight)
    _c("dev_splits257_last1", S(3), D(8193, 8193, 256), "near", seed=11, nsplit=257, nsplit_gt=256, chunk=32, last_rows=1,
       t_at_cap=True, t_expect="below"),
    _c("dev_q0", D(0, 1000, 1000), S(500), seed=12, q_count=0, q_expect="above"),
    _c("dev_t0", S(300), D(0, 2000, 2000), "pool", seed=13, nsplit=63, chunk=32, t_count=0, dev_splits=1, dev_splits_lt_launch=True,
       t_expect="above"),
    _c("dev_t1", S(200), D(1, 1500), seed=14, nsplit=47, chunk=32, t_count=1, dev_splits=1, dev_splits_lt_launch=True,
       t_expect="unknown"),
    _c("dev_both_at_cap", D(700, 700, 700), D(900, 900, 900), "pool", seed=15, q_at_cap=True, t_at_cap=True, q_expect="equal",
       t_expect="equal"),
    _c("dev_t_few_splits", S(2000), D(2100, 40000, 40000), "near", seed=16, qtiles=16, nsplit=40, chunk=MAX_CHUNK, last_rows=52,
       dev_splits=3, dev_splits_lt_launch=True, t_expect="above"),
    _c("dev_expect_above", D(1000, 1200, 1200), D(1000, 3000, 2500), "pool", seed=17, dev_splits_lt_launch=True, q_expect="above",
       t_expect="above"),
    _c("dev_q_expect_below", D(3000, 4000, 500), D(2500, 2600, 2600), "near", seed=18, qtiles=32, q_expect="below",
       t_expect="above", tail_q=56),
    _c("dev_expect_equal", D(1500, 2000, 1500), D(1800, 2048, 1800), "pool", seed=19, q_expect="equal", t_expect="equal"),
    _c("dev_q1_t_at_cap", D(1, 64, 1), D(5000, 5000, 5000), "near", seed=20, qtiles=1, nsplit=157, chunk=32, last_rows=8,
       q_count=1, t_at_cap=True, t_expect="equal"),
    # the stereo matcher on the same split (integer keypoints: disparities and row offsets exactly on the window's edges)
    _c("stereo_host", S(300), S(3000), seed=21, stereo=(1.0, 2.0, 10.0), qtiles=3),
    _c("stereo_dev_right", S(800), D(900, 1200, 1000), "pool", seed=22, stereo=(1.0, 2.0, 10.0), t_expect="above"),
    _c("stereo_dev_left", D(700, 1000, 700), S(1000), seed=23, stereo=(0.0, -4.0, 4.0), q_expect="equal"),
    _c("stereo_dev_both_t0", D(500, 640, 0), D(0, 700, 700), seed=24, stereo=(2.0, 0.0, 8.0), t_count=0, dev_splits=1,
       q_expect="unknown"),
]

BY_ID = {c.id: c for c in CASES}


def _expect_rel(expect, n):
    if expect <= 0:
        return "unknown"
    return "below" if expect < n else ("equal" if expect == n else "above")


def check_reach(case, got_plan, sm):
    """Assert that `got_plan` (the plan of a launch of `case` on an `sm`-SM device: the mirror's or the device's own) reaches the
    boundary the case was written for."""
    s = case.shape(sm)
    qtiles, nsplit, chunk = got_plan
    r = {k: _v(v, sm) for k, v in case.reach}
    where = (case.id, sm, got_plan, s)
    for name, val in (("qtiles", qtiles), ("nsplit", nsplit), ("chunk", chunk)):
        if name in r:
            assert val == r[name], (name,) + where
    if "nsplit_gt" in r:
        assert nsplit > r["nsplit_gt"], where
    if "nt_max" in r:
        assert s.nt <= r["nt_max"], where
    if "nt_min" in r:
        assert s.nt >= r["nt_min"], where
    if "last_rows" in r:
        assert s.nt > 0 and s.nt - (_du(s.nt, chunk) - 1) * chunk == r["last_rows"], where
    if "tail_q" in r:
        assert s.nq > 0 and s.nq - (_du(s.nq, KQ) - 1) * KQ == r["tail_q"], where
    if "dev_splits" in r or "dev_splits_lt_launch" in r:
        assert s.t_dev, where
        ds = device_splits(s.nt, chunk)
        if "dev_splits" in r:
            assert ds == r["dev_splits"], where
        if "dev_splits_lt_launch" in r:
            assert ds < nsplit, where
    for side, dev, n, cap, e in (("q", s.q_dev, s.nq, s.qcap, s.eq), ("t", s.t_dev, s.nt, s.tcap, s.et)):
        if side + "_count" in r:
            assert dev and n == r[side + "_count"], where
        if side + "_at_cap" in r:
            assert dev and n == cap, where
        if side + "_expect" in r:
            assert dev and _expect_rel(e, n) == r[side + "_expect"], where
    return got_plan


# ---- the stereo predicate at its edges ---------------------------------------------------------------------------------------
# A right keypoint is a candidate of a left one iff |y_R - y_L| <= band and min_disp <= x_L - x_R <= max_disp, float compares on
# float differences.  Each case is (kl, kr, band, min_disp, max_disp) plus the facts it must reach, checked by `stereo_hits`:
#   dy_eq_band      some pair has |y_R - y_L| == band exactly (and its disparity inside the window)
#   disp_eq_min / disp_eq_max   some pair has x_L - x_R == min_disp (max_disp) exactly (and |dy| <= band)
#   just_outside    some pair misses the band or the window by less than 1e-3 (and meets the other condition)
#   rounds          some pair's float disparity differs from the real one (and sits on a window edge)
#   nan             some keypoint coordinate is NaN
#   neg_zero        some coordinate or window bound is -0.0


@dataclasses.dataclass(frozen=True)
class StereoEdge:
    id: str
    make: object        # rng -> (kl, dl, kr, dr, band, min_disp, max_disp)
    hits: tuple


def _kps(xy):
    from gslam_b200.capi import KP_DTYPE
    k = np.zeros(len(xy), KP_DTYPE)
    if len(xy):
        a = np.asarray(xy, np.float32).reshape(-1, 2)
        k["x"], k["y"] = a[:, 0], a[:, 1]
    return k


def _desc(rng, n):
    return rng.integers(0, 256, (n, 32), dtype=np.uint8)


def _f32(x):
    return float(np.float32(x))


def _up(x):
    return float(np.nextafter(np.float32(x), np.float32(np.inf)))


def _dn(x):
    return float(np.nextafter(np.float32(x), np.float32(-np.inf)))


def _band_edge(band):
    def make(rng):
        y0 = 100.0
        kl = _kps([(50.0, y0), (60.0, y0), (70.0, y0)])
        kr = _kps([(45.0, y0 + band), (46.0, y0 - band), (47.0, _up(y0 + band)), (48.0, _dn(y0 - band)), (55.0, y0), (65.0, y0 + band),
                   (66.0, _up(y0 + band))])
        return kl, _desc(rng, 3), kr, _desc(rng, 7), band, 0.0, 96.0
    return make


def _disp_edges(mind, maxd):
    def make(rng):
        xl = [200.0, 300.0, 400.0, 500.0]
        kl = _kps([(x, 10.0) for x in xl])
        xr = []
        for x in xl:
            xr += [x - mind, x - maxd, _up(x - mind), _dn(x - maxd), x - (mind + maxd) / 2]
        kr = _kps([(x, 10.0) for x in xr])
        return kl, _desc(rng, len(xl)), kr, _desc(rng, len(xr)), 0.0, mind, maxd
    return make


def _near_16384(rng):
    # float32 steps are 2^-10 below 16384 and 2^-9 above it: x_L - x_R rounds, and the window bounds are set to rounded values
    xl = (16384.0 + rng.integers(-300, 300, 64) / 512.0 + 1 / 1024.0).astype(np.float32)
    xr = (rng.uniform(0.05, 3.0, 96)).astype(np.float32)
    kl = _kps(np.stack([xl, np.zeros(64, np.float32)], 1))
    kr = _kps(np.stack([xr, np.zeros(96, np.float32)], 1))
    disp = (xl[:, None] - xr[None, :]).astype(np.float32)
    exact = xl[:, None].astype(np.float64) - xr[None, :].astype(np.float64)
    rounded = np.argwhere(disp.astype(np.float64) != exact)
    lo = disp[tuple(rounded[0])]
    hi = disp[tuple(rounded[len(rounded) // 2])]
    mind, maxd = (float(lo), float(hi)) if lo <= hi else (float(hi), float(lo))
    return kl, _desc(rng, 64), kr, _desc(rng, 96), 0.0, mind, maxd


def _nan(rng):
    nan = float("nan")
    kl = _kps([(50.0, 5.0), (nan, 5.0), (60.0, nan), (70.0, 5.0)])
    kr = _kps([(45.0, 5.0), (nan, 5.0), (55.0, nan), (46.0, 5.0), (65.0, 5.0)])
    return kl, _desc(rng, 4), kr, _desc(rng, 5), float("inf"), float("-inf"), float("inf")


def _neg_zero(rng):
    kl = _kps([(0.0, 0.0), (-0.0, -0.0), (3.0, 0.0)])
    kr = _kps([(-0.0, 0.0), (0.0, -0.0), (3.0, -0.0), (_up(0.0), 0.0), (0.0, _up(0.0))])
    return kl, _desc(rng, 3), kr, _desc(rng, 5), 0.0, -0.0, 0.0


def _inf_window(mind, maxd, band):
    def make(rng):
        kl = _kps([(100.0 + i, float(i % 7)) for i in range(20)])
        kr = _kps([(float(rng.integers(0, 250)), float(rng.integers(0, 7))) for _ in range(30)])
        return kl, _desc(rng, 20), kr, _desc(rng, 30), band, mind, maxd
    return make


def _one_candidate(rng):
    # every left keypoint has exactly one candidate (d2 = 257), the last one none (-1 / 257 / 257)
    kl = _kps([(100.0 + 10 * i, float(i)) for i in range(8)])
    kr = _kps([(100.0 + 10 * i - 3.0, float(i)) for i in range(7)] + [(0.0, 50.0)])
    return kl, _desc(rng, 8), kr, _desc(rng, 8), 0.0, 3.0, 3.0


INF = float("inf")
STEREO_EDGES = [
    StereoEdge("band_eq", _band_edge(2.0), ("dy_eq_band", "just_outside")),
    StereoEdge("band0", _band_edge(0.0), ("dy_eq_band", "just_outside")),
    StereoEdge("band_frac", _band_edge(_f32(2.5)), ("dy_eq_band", "just_outside")),
    StereoEdge("disp_edges", _disp_edges(0.0, 96.0), ("disp_eq_min", "disp_eq_max", "just_outside")),
    StereoEdge("disp_edges_frac", _disp_edges(_f32(3.25), _f32(17.75)), ("disp_eq_min", "disp_eq_max", "just_outside")),
    StereoEdge("min_eq_max", _disp_edges(14.0, 14.0), ("disp_eq_min", "disp_eq_max", "just_outside")),
    StereoEdge("negative_window", _disp_edges(-10.0, -2.0), ("disp_eq_min", "disp_eq_max", "just_outside")),
    StereoEdge("inf_window", _inf_window(-INF, INF, 1.0), ()),
    StereoEdge("inf_band", _inf_window(0.0, INF, INF), ()),
    StereoEdge("neg_inf_min", _inf_window(-INF, 5.0, 0.0), ()),
    StereoEdge("neg_zero", _neg_zero, ("neg_zero", "disp_eq_min", "disp_eq_max", "dy_eq_band", "just_outside")),
    StereoEdge("near_16384", _near_16384, ("rounds", "disp_eq_min", "disp_eq_max")),
    StereoEdge("nan_coords", _nan, ("nan",)),
    StereoEdge("one_candidate", _one_candidate, ("disp_eq_min", "disp_eq_max", "dy_eq_band")),
]


def stereo_hits(edge, kl, kr, band, mind, maxd):
    """Assert that the arrays of `edge` reach its facts (see above)."""
    f = np.float32
    dy = np.abs(kr["y"][None, :] - kl["y"][:, None]).astype(f)
    disp = (kl["x"][:, None] - kr["x"][None, :]).astype(f)
    with np.errstate(invalid="ignore"):
        in_band = dy <= f(band)
        in_win = (disp >= f(mind)) & (disp <= f(maxd))
    for h in edge.hits:
        if h == "dy_eq_band":
            assert ((dy == f(band)) & in_win).any(), (edge.id, h)
        elif h == "disp_eq_min":
            assert ((disp == f(mind)) & in_band).any(), (edge.id, h)
        elif h == "disp_eq_max":
            assert ((disp == f(maxd)) & in_band).any(), (edge.id, h)
        elif h == "just_outside":
            eps = f(1e-3)
            miss_band = (dy > f(band)) & (dy <= f(band) + eps) & in_win
            miss_win = (((disp < f(mind)) & (disp >= f(mind) - eps)) | ((disp > f(maxd)) & (disp <= f(maxd) + eps))) & in_band
            assert (miss_band | miss_win).any(), (edge.id, h)
        elif h == "rounds":
            exact = kl["x"][:, None].astype(np.float64) - kr["x"][None, :].astype(np.float64)
            edge_hit = (disp == f(mind)) | (disp == f(maxd))
            assert (edge_hit & (disp.astype(np.float64) != exact)).any(), (edge.id, h)
        elif h == "nan":
            assert np.isnan(kl["x"]).any() and np.isnan(kl["y"]).any() and np.isnan(kr["x"]).any() and np.isnan(kr["y"]).any(), edge.id
        elif h == "neg_zero":
            z = lambda a: (a == 0) & np.signbit(a)  # noqa: E731
            assert z(kl["x"]).any() and z(kr["x"]).any() and np.signbit(f(mind)), edge.id
        else:
            raise AssertionError(f"unknown fact {h}")


def stereo_numpy(kl, dl, kr, dr, band, mind, maxd):
    """Independent restatement of the stereo row-band rule (vectorised numpy, stable argsort on (distance, index))."""
    nl = len(kl)
    idx = np.full(nl, -1, np.int32); d1 = np.full(nl, 257, np.int32); d2 = np.full(nl, 257, np.int32)
    if len(kr) == 0:
        return idx, d1, d2
    bits_r = np.unpackbits(dr, axis=1)
    for i in range(nl):
        dy = np.abs(kr["y"] - kl["y"][i]).astype(np.float32)
        disp = (kl["x"][i] - kr["x"]).astype(np.float32)
        with np.errstate(invalid="ignore"):
            cand = np.nonzero((dy <= np.float32(band)) & (disp >= np.float32(mind)) & (disp <= np.float32(maxd)))[0]
        if cand.size == 0:
            continue
        d = (np.unpackbits(dl[i])[None, :] != bits_r[cand]).sum(axis=1)
        order = np.lexsort((cand, d))
        idx[i] = cand[order[0]]; d1[i] = d[order[0]]
        if cand.size > 1:
            d2[i] = d[order[1]]
    return idx, d1, d2
