#!/usr/bin/env python
"""Check what `bench.py --dump-outputs DIR` wrote against the CPU oracle.

  python tools/check_bench_dump.py DIR --steps S --warmup W

bench.py's inputs depend only on its arguments, so the last timed step can be rebuilt here from bench.py's own constants: the
frame is ring slot (W + S - 1) % RING, the frame before it slot (W + S - 2) % RING (slot k is synth_stream(1920, 1080, 8, seed=7)
frame k % 8 rolled by (k // 8) * 7 columns), and the BA window is synth_ba(50, 2000, 5, seed=42, n_fixed=2).  Keypoints,
descriptors and matches must equal oracle ORB + oracle Hamming match bit for bit; the solved window must agree with
oracle.ba_solve after the same LM and PCG iteration counts within 1e-5 (final cost, every camera pose, every landmark).
Prints one line per check and exits non-zero on any disagreement.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (constants only; its main() is not run)
import oracle  # noqa: E402
from gslam_b200 import synth  # noqa: E402

RTOL = 1e-5


def ring_frame(base, slot):
    return np.ascontiguousarray(np.roll(base[slot % 8], shift=(slot // 8) * 7, axis=1))


def expected(steps, warmup):
    """The oracle's outputs of the last timed step: (keypoint rows, descriptors, (idx, d1, d2), ba result, problem after solve)."""
    base = synth.synth_stream(bench.W, bench.H, 8, seed=7)
    k = warmup + steps - 1
    kps, desc = oracle.orb_extract(ring_frame(base, k % bench.RING), bench.NKP)
    _, desc_prev = oracle.orb_extract(ring_frame(base, (k - 1) % bench.RING), bench.NKP)
    m = oracle.match_hamming(desc, desc_prev)
    pb = synth.synth_ba(bench.BA_CAMS, bench.BA_PTS, bench.BA_OBS_PER_PT, seed=42, n_fixed=2)
    r = oracle.ba_solve(pb, max_iterations=bench.BA_ITERS, function_tolerance=0.0, pcg_max_iters=bench.PCG_ITERS, pcg_tol=1e-10)
    return kps, desc, m, r, pb


def check(out_dir, steps, warmup) -> list[tuple[str, bool, str]]:
    kps, desc, (idx, d1, d2), r, pb = expected(steps, warmup)
    ld = lambda name: np.load(os.path.join(out_dir, name + ".npy"))
    res = []
    # bench.py's dump: the keypoint record's fields in dtype order, each as float32 (exact for every field: small integers, floats)
    want_k = np.stack([kps[f].astype(np.float32) for f in kps.dtype.names], axis=1).reshape(-1, len(kps.dtype.names))
    got_k = ld("keypoints")
    res.append(("keypoints", got_k.shape == want_k.shape and np.array_equal(got_k, want_k), f"{got_k.shape[0]} vs {want_k.shape[0]} rows"))
    got_d = ld("descriptors")
    res.append(("descriptors", np.array_equal(got_d, desc.astype(np.float32)), f"{got_d.shape[0]} rows"))
    for name, want in (("match_index", idx), ("match_distance", d1), ("match_distance2", d2)):
        got = ld(name)
        res.append((name, np.array_equal(got, want.astype(np.float32)), f"{got.shape[0]} queries"))
    ba = ld("ba_result")  # [initial_cost, final_cost, iterations, accepted, pcg_iterations]
    rc = abs(ba[1] - r.final_cost) / r.final_cost
    res.append(("ba_lm", int(ba[2]) == r.iterations and int(ba[3]) == r.accepted,
                f"iterations {int(ba[2])} / {r.iterations}, accepted {int(ba[3])} / {r.accepted}"))
    res.append(("ba_final_cost", rc < RTOL, f"relative difference {rc:.2e}"))
    poses, points = ld("ba_poses_wc"), ld("ba_points")
    want_p = pb.cam_pose_wc
    s = np.sign(np.sum(poses[:, :4] * want_p[:, :4], axis=1))[:, None]
    eq = np.abs(poses[:, :4] * s - want_p[:, :4]).max()
    et = np.abs(poses[:, 4:] - want_p[:, 4:]).max() / max(1.0, np.abs(want_p[:, 4:]).max())
    res.append(("ba_poses", eq < RTOL and et < RTOL, f"quaternion {eq:.2e}, translation {et:.2e}"))
    ep = np.abs(points - pb.points).max() / np.abs(pb.points).max()
    res.append(("ba_points", ep < RTOL, f"relative difference {ep:.2e}"))
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[1])
    ap.add_argument("dir")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args(argv)
    if a.steps < 1 or a.warmup < 0:
        ap.error("--steps must be at least 1 and --warmup at least 0")
    res = check(a.dir, a.steps, a.warmup)
    for name, ok, note in res:
        print(f"{'ok  ' if ok else 'FAIL'} {name}: {note}")
    bad = [n for n, ok, _ in res if not ok]
    print("agreement with the oracle" if not bad else f"{len(bad)} disagreement(s): {', '.join(bad)}")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
