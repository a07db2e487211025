"""ORB extraction cases at the edges of its configuration range and of its fixed limits, shared by the oracle-vs-cv2 pins
(tests/test_oracle_orb.py) and the device-vs-oracle parity tests (tests/test_orb_limits_gpu.py).

Each case names an image, nfeatures, the extractor configuration and the boundary it exists to reach.  `reach` states that
boundary as facts about the result, which `check_reach` asserts on the keypoints (and the GPU tests also on the device's per-level
counts), so that a change to an image generator cannot quietly turn a limit case into an easy one:
  kept        exact number of keypoints kept on each of the first len(kept) levels
  total       exact number of keypoints
  usable      number of levels larger than 2 * edge_threshold on both sides (the others get no FAST tile); the last of them keeps
              keypoints
  full_sort   number of levels keeping more than 2048 and at most 4096 keypoints (the whole 4096-entry sort of a level)
  edge_x      level-0 keypoints sit on the first and on the last column the border allows (x == edge and x == w - 1 - edge); on
              a width that is a multiple of 128 the device row pitch equals the width, so the last word of that keypoint's 45x45
              patch ends on column w - 1 with no padding column behind it
  edge_y      the same for rows
  min_x / min_y   some level-0 keypoint has x (resp. y) at least this large (positions are packed as 16-bit fields)
  min_fast0   level 0 has at least this many FAST corners after the non-maximum suppression and the border filter
"""
import dataclasses

import numpy as np

# A pyramid level keeps at most this many keypoints on the device (include/gslam_b200.h, above gb_orb_cfg_default).
LEVEL_CAP = 4096
# The largest nfeatures whose level-0 quota at the defaults (scale 1.2, 8 levels) is LEVEL_CAP (18859..18862 all give it), and the
# first one above it.
N_AT_CAP, N_OVER_CAP = 18862, 18863


@dataclasses.dataclass(frozen=True)
class LimitCase:
    id: str
    kind: str                  # "synth" (gslam_b200.synth.synth_frame) or an image_of_kind kind
    w: int
    h: int
    seed: int
    nfeatures: int
    cfg: tuple = ()            # ((name, value), ...) in gb_orb_cfg / oracle.orb_extract names
    reach: tuple = ()          # ((fact, value), ...), see the module docstring

    def image(self):
        if self.kind == "synth":
            from gslam_b200 import synth
            return synth.synth_frame(self.w, self.h, self.seed)
        from _images import image_of_kind
        return np.ascontiguousarray(image_of_kind(self.kind, self.w, self.h, self.seed))

    @property
    def kw(self):
        return dict(self.cfg)

    @property
    def cv2_kw(self):
        names = dict(edge_threshold="edgeThreshold", nlevels="nlevels", scale_factor="scaleFactor", fast_threshold="fastThreshold")
        return {names[k]: v for k, v in self.cfg}


def _c(id, kind, w, h, seed, n, cfg=None, **reach):
    return LimitCase(id, kind, w, h, seed, n, tuple(sorted((cfg or {}).items())), tuple(sorted(reach.items())))


CASES = [
    # edge_threshold: the minimum 22 (45x45 describe patch touching column / row 0 and w-1), odd and pitch == width widths
    _c("edge22_odd", "synth", 517, 389, 77, 400, dict(edge_threshold=22), usable=8),
    _c("edge23", "synth", 517, 389, 77, 400, dict(edge_threshold=23), usable=8),
    _c("edge40", "synth", 517, 389, 77, 400, dict(edge_threshold=40), usable=8),
    _c("edge64", "synth", 517, 389, 77, 400, dict(edge_threshold=64), usable=7),
    _c("edge22_noise_w640", "noise", 640, 480, 21, 6000, dict(edge_threshold=22), usable=8, edge_x=True, edge_y=True),
    _c("edge22_noise_odd", "noise", 517, 389, 22, 4000, dict(edge_threshold=22), usable=8, edge_x=True),
    _c("edge22_synth_w1280", "synth", 1280, 720, 23, 3000, dict(edge_threshold=22), usable=8),
    _c("edge22_binary_w256", "binary", 256, 200, 24, 2000, dict(edge_threshold=22, fast_threshold=40), usable=8, edge_x=True),
    # edge_threshold so large that only level 0 is usable
    _c("edge200", "synth", 640, 480, 8, 400, dict(edge_threshold=200), usable=1, kept=[87, 0]),
    _c("edge239", "synth", 640, 480, 8, 400, dict(edge_threshold=239), usable=1, kept=[1, 0]),
    # nlevels 12 (every slot of the level arrays), scale factors near 1 and large, zero quotas between positive ones
    _c("lv12_sf105", "synth", 517, 389, 77, 500, dict(nlevels=12, scale_factor=1.05), usable=12),
    _c("lv12_sf12", "synth", 517, 389, 77, 500, dict(nlevels=12, scale_factor=1.2), usable=11),
    _c("lv12_sf101", "synth", 640, 480, 8, 600, dict(nlevels=12, scale_factor=1.01), usable=12),
    _c("lv3_sf37", "synth", 640, 480, 8, 300, dict(nlevels=3, scale_factor=3.7), usable=2),
    _c("lv12_zero_quotas", "synth", 640, 480, 8, 5, dict(nlevels=12), kept=[1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1]),
    # FAST threshold extremes: 1 (fullest candidate lists and score histograms) and 254 (only 0 / 255 contrasts are corners)
    _c("fast1", "synth", 517, 389, 77, 500, dict(fast_threshold=1), min_fast0=10000),  # 11048 corners; 1808 at threshold 20
    _c("fast254_synth", "synth", 517, 389, 77, 500, dict(fast_threshold=254), total=0),
    _c("fast254_binary", "binary", 300, 240, 3, 500, dict(fast_threshold=254), total=109),
    _c("fast1_noise_lv12", "noise", 1024, 768, 4, 3000, dict(fast_threshold=1, nlevels=12, scale_factor=1.1), usable=12),
    # the 4096-keypoint level cap, reached exactly
    _c("cap_noise", "noise", 1920, 1080, 11, N_AT_CAP, kept=[LEVEL_CAP]),
    _c("cap_synth", "synth", 1920, 1080, 5, N_AT_CAP, kept=[LEVEL_CAP]),
    _c("full_sort_12lv", "noise", 4096, 3072, 2, 30000, dict(nlevels=12, scale_factor=1.1), full_sort=8),
    # frame shape: 16384 on one side (x or y near 16383 in the packed positions), extreme aspect ratios
    _c("wide_16384x80", "synth", 16384, 80, 3, 2000, usable=2, kept=[434, 362], min_x=16300),
    _c("tall_80x16384", "synth", 80, 16384, 3, 2000, usable=2, kept=[434, 362], min_y=16250),
    _c("wide_16384x1024", "synth", 16384, 1024, 6, 2000, usable=8, min_x=16300),
    _c("tall_1024x16384", "synth", 1024, 16384, 7, 2000, usable=8, min_y=16300),
]

# Over the level cap: the oracle (like cv2) keeps 4097 on level 0, the device refuses the configuration.
OVER_CAP = _c("over_cap_noise", "noise", 1920, 1080, 11, N_OVER_CAP, kept=[LEVEL_CAP + 1])

BY_ID = {c.id: c for c in CASES + [OVER_CAP]}


def level_sizes(case):
    import oracle
    kw = case.kw
    nl, sf = kw.get("nlevels", 8), kw.get("scale_factor", 1.2)
    return [oracle.orb_level_size(case.w, case.h, l, sf) for l in range(nl)]


def usable_levels(case):
    e = case.kw.get("edge_threshold", 31)
    return sum(1 for lw, lh in level_sizes(case) if lw > 2 * e and lh > 2 * e)


def kept_per_level(kps, nlevels):
    return np.bincount(np.asarray(kps["octave"], np.int64), minlength=nlevels)[:nlevels].tolist()


def level0_fast_corners(case, img):
    """The oracle's level-0 FAST corners of `case` after the non-maximum suppression and the border filter."""
    import oracle
    kw = case.kw
    e = kw.get("edge_threshold", 31)
    xs, ys, _ = oracle.fast_detect(img, kw.get("fast_threshold", 20), True)
    return int(((xs >= e) & (xs < case.w - e) & (ys >= e) & (ys < case.h - e)).sum())


def check_reach(case, kps, fast0=None):
    """Assert that the keypoints `kps` (an extraction of `case`, any source) reach the case's boundary; `fast0` is the number of
    level-0 FAST corners of the same extraction."""
    kw = case.kw
    nl, e = kw.get("nlevels", 8), kw.get("edge_threshold", 31)
    per = kept_per_level(kps, nl)
    r = dict(case.reach)
    if "kept" in r:
        want = list(r["kept"])
        assert per[:len(want)] == want, (case.id, per)
    if "total" in r:
        assert len(kps) == r["total"], (case.id, len(kps))
    if "usable" in r:
        assert usable_levels(case) == r["usable"], (case.id, level_sizes(case))
        assert per[r["usable"] - 1] > 0 and not any(per[r["usable"]:]), (case.id, per)
    if "full_sort" in r:
        assert sum(2048 < k <= LEVEL_CAP for k in per) == r["full_sort"], (case.id, per)
    if "min_fast0" in r:
        assert fast0 is not None and fast0 >= r["min_fast0"], (case.id, fast0)
    l0 = kps[kps["octave"] == 0]
    # level 0 has scale 1: the keypoint coordinates are the level-0 pixel positions
    x0, y0 = l0["x"].astype(np.int64), l0["y"].astype(np.int64)
    if "edge_x" in r:
        assert x0.min() == e and x0.max() == case.w - 1 - e, (case.id, x0.min(), x0.max())
    if "edge_y" in r:
        assert y0.min() == e and y0.max() == case.h - 1 - e, (case.id, y0.min(), y0.max())
    if "min_x" in r:
        assert x0.max() >= r["min_x"], (case.id, x0.max())
    if "min_y" in r:
        assert y0.max() >= r["min_y"], (case.id, y0.max())
    return per
