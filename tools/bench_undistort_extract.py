"""What the device-resident undistort + extract costs against the two-call route through host buffers.

  python tools/bench_undistort_extract.py [--reps N] [--warmup W] [--kernel-launches K] [--out FILE]

Needs a CUDA device (there is no fallback: context creation raises without one) and reads nothing outside the tree.  For 1920x1080
gray and BGR frames and a 752x480 stereo pair (two maps, two extractions per step), 2000 keypoints each, every shape warmed up first,
the routes are run alternately, N rounds of a / b / c, and the median and the 10th / 90th percentile of each are reported in ms:

  a  two_calls_host     gb_remap_apply, then gb_orb_extract_image on its result: host buffers in and out (host clock; both calls end
                        in a synchronisation)
  b  fused_host         gb_orb_extract_undistorted: host frame in, keypoints and descriptors out (host clock, one synchronisation)
  c  fused_device       gb_orb_extract_undistorted_to on a frame resident in HBM: device events around the enqueue

  d  the remap kernel alone (remap_level0_kernel), in a run of its own under torch.profiler with a synchronisation between the
     extractions (so that the kernel, a programmatic dependent launch, never waits inside its own duration for a predecessor): mean
     duration over K launches, and its algorithmic bytes over that time as a share of the H100 SXM data sheet's 3.35 TB/s.  The kernel
     is bandwidth-bound (a gather: per output pixel 36 B of table read and 1 B written, plus the source frame read once).

The card's name and power limit are read in the same run and are part of every number.  Prints one JSON line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

NKP = 2000
HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
SHAPES = [("1080p_gray", 1920, 1080, 1, 1), ("1080p_bgr", 1920, 1080, 3, 1), ("752x480_stereo", 752, 480, 1, 2)]  # name, w, h, channels, eyes


def card() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    return r.stdout.strip()


def distortion_table(w, h, k1):
    """A radial distortion in the reference's table format (four taps + weights per output pixel, remap_x < 0 outside the input)."""
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    u = (x - w / 2) / w; v = (y - h / 2) / h
    r2 = u * u + v * v
    k = 1 + k1 * r2 + 0.1 * r2 * r2
    sx = (u * k * 1.15 + 0.5) * w; sy = (v * k * 1.15 + 0.5) * h
    out = (sx < 0) | (sy < 0) | (sx >= w) | (sy >= h)
    rx = np.where(out, -1, sx).astype(np.float32); ry = np.where(out, -1, sy).astype(np.float32)
    xi = rx.astype(np.int32); yi = ry.astype(np.int32)
    fx = rx - xi; fy = ry - yi; fxy = fx * fy
    idx = np.stack([yi * w + xi, yi * w + xi + 1, (yi + 1) * w + xi, (yi + 1) * w + xi + 1], -1).astype(np.int32)
    coef = np.stack([1 - fx - fy + fxy, fx - fxy, fy - fxy, fxy], -1).astype(np.float32)
    idx[out] = 0; coef[out] = 0
    return idx.reshape(-1, 4), coef.reshape(-1, 4), rx.reshape(-1)


def remap_bytes(w_in, h_in, w_out, h_out, channels):
    """Bytes the level-0 remap has to move: 16 B indices + 16 B weights + 4 B remap_x read and 1 B written per output pixel, and the
    source frame read once (the four taps of neighbouring pixels overlap: every further read of a source byte is a cache hit)."""
    return 37 * w_out * h_out + w_in * h_in * channels


def stats(v):
    a = np.asarray(v, np.float64)
    return dict(median=round(float(np.median(a)), 4), p10=round(float(np.percentile(a, 10)), 4), p90=round(float(np.percentile(a, 90)), 4), n=len(v))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kernel-launches", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the JSON there")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from gslam_b200 import synth
    from gslam_b200.api import Context, Features, Remap

    ctx = Context(0)  # raises without a device
    result = dict(card=card(), nfeatures=NKP, reps=args.reps, shapes={})
    for name, w, h, ch, eyes in SHAPES:
        cfg = ctx.orb_cfg(nfeatures=NKP)
        maps, frames, dev, feats = [], [], [], []
        for e in range(eyes):
            maps.append(Remap(ctx, w, h, w, h, *distortion_table(w, h, -0.25 - 0.05 * e)))
            g = synth.synth_frame(w, h, seed=3 + e)
            img = g if ch == 1 else np.ascontiguousarray(np.stack([g, np.roll(g, 9, axis=1), 255 - g], axis=2))
            frames.append(img)
            dev.append(torch.from_numpy(img).cuda())
            feats.append(Features(ctx, 2 * NKP + 256))
        torch.cuda.synchronize()  # the frames were written on torch's stream, the ctx reads them on its own

        def two_calls():
            return [ctx.orb_extract(m.apply(f), NKP) for m, f in zip(maps, frames)]

        def fused_host():
            return [ctx.orb_extract_undistorted(m, f, NKP) for m, f in zip(maps, frames)]

        def fused_device_enqueue():
            for m, t, ft in zip(maps, dev, feats):
                ft.extract_undistorted(m, t.data_ptr(), cfg, channels=ch, device_ptr=True)

        ra, rb = two_calls(), fused_host()   # first use of the shape, and the check that the routes agree
        fused_device_enqueue()
        for (ka, da), (kb, db), ft in zip(ra, rb, feats):
            kc, dc = ft.download()
            if not (np.array_equal(ka, kb) and np.array_equal(da, db) and np.array_equal(ka, kc) and np.array_equal(da, dc)):
                sys.exit(f"{name}: the routes disagree")
        for _ in range(args.warmup):
            two_calls(); fused_host(); fused_device_enqueue()
        ctx.sync()
        t = dict(two_calls_host=[], fused_host=[], fused_device=[])
        for _ in range(args.reps):
            t0 = time.perf_counter(); two_calls(); t["two_calls_host"].append((time.perf_counter() - t0) * 1e3)
            t0 = time.perf_counter(); fused_host(); t["fused_host"].append((time.perf_counter() - t0) * 1e3)
            ctx.timer_begin(); fused_device_enqueue(); t["fused_device"].append(ctx.timer_end())
        entry = {k: stats(v) for k, v in t.items()}
        entry["keypoints"] = [int(len(k)) for k, _ in ra]

        # d: the kernel alone
        with tempfile.TemporaryDirectory() as tmp:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(max(1, args.kernel_launches // eyes)):
                    fused_device_enqueue()
                    ctx.sync()
            trace = os.path.join(tmp, "trace.json")
            prof.export_chrome_trace(trace)
            ev = json.load(open(trace))["traceEvents"]
        durs = [e["dur"] for e in ev if e.get("cat") == "kernel" and "remap_level0_kernel" in e.get("name", "")]
        if not durs:
            sys.exit(f"{name}: no remap_level0_kernel in the trace")
        us = float(np.mean(durs))
        nbytes = remap_bytes(w, h, w, h, ch)
        entry["remap_level0_kernel"] = dict(launches=len(durs), mean_us=round(us, 3), median_us=round(float(np.median(durs)), 3), algorithmic_bytes=nbytes,
                                            gb_per_s=round(nbytes / us * 1e-3, 1), share_of_hbm_peak=round(nbytes / (us * 1e-6) / HBM_PEAK, 4),
                                            bound="HBM bandwidth (3.35 TB/s, H100 SXM data sheet)")
        result["shapes"][name] = entry
        for x in feats + maps:
            x.close()
    ctx.close()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
