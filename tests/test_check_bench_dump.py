"""tools/check_bench_dump.py reads what bench.py's dump_outputs writes: a dump made from the oracle's own outputs passes, and one
flipped descriptor bit, one changed match or a BA result off by more than the tolerance fails."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench  # noqa: E402
import check_bench_dump as cbd  # noqa: E402


class _Feats:
    def __init__(self, kps, desc, m):
        self.kps, self.desc, self.m = kps, desc, m

    def download(self):
        return self.kps, self.desc

    def matches(self):
        return self.m


class _Graph:
    def __init__(self, pb):
        self.pb = pb

    def download(self):
        return self.pb.cam_pose_wc, self.pb.points


class _Res:
    def __init__(self, r):
        self.initial_cost, self.final_cost, self.iterations = r.initial_cost, r.final_cost, r.iterations
        self.accepted, self.pcg_iterations = r.accepted, r.pcg_iterations


@pytest.fixture(scope="module")
def want():
    return cbd.expected(1, 0)


def _dump(d, want, mutate=None):
    kps, desc, m, r, pb = want
    kps, desc, m, pb = kps.copy(), desc.copy(), tuple(x.copy() for x in m), pb.copy()
    if mutate:
        mutate(kps, desc, m, pb)
    bench.dump_outputs(str(d), _Feats(kps, desc, m), _Graph(pb), _Res(r))


def _failed(d, want, monkeypatch):
    monkeypatch.setattr(cbd, "expected", lambda steps, warmup: want)
    return [n for n, ok, _ in cbd.check(str(d), 1, 0) if not ok]


def test_oracle_dump_agrees(tmp_path, want, monkeypatch):
    _dump(tmp_path, want)
    assert _failed(tmp_path, want, monkeypatch) == []


@pytest.mark.parametrize("what,mutate", [
    ("descriptors", lambda k, d, m, pb: d.__setitem__((17, 3), d[17, 3] ^ 4)),
    ("keypoints", lambda k, d, m, pb: k["response"].__setitem__(5, np.nextafter(k["response"][5], np.float32(1)))),
    ("match_index", lambda k, d, m, pb: m[0].__setitem__(9, m[0][9] + 1)),
    ("ba_points", lambda k, d, m, pb: pb.points.__setitem__((7, 2), pb.points[7, 2] + 1e-4 * np.abs(pb.points).max())),
])
def test_a_wrong_output_is_reported(tmp_path, want, monkeypatch, what, mutate):
    _dump(tmp_path, want, mutate)
    assert _failed(tmp_path, want, monkeypatch) == [what]
