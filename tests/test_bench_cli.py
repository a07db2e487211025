"""bench.py's reference arm (`--impl reference`): the CPU path of the same workload.  Under torchrun rank 0 alone runs and prints ONE JSON
line, the other ranks leave without work -- checked here with two CPU processes (no GPU is involved in this arm)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_under_torchrun_prints_one_line():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29547",
           os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1", "--warmup", "1"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, r.stdout[-2000:]
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 2 and d["higher_is_better"] is True
    assert d["metric"].startswith("frames/sec") and d["unit"] == "frames/s" and d["value"] > 0
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]
    assert d["cpu_baseline"]["kind"] == "port" and "OpenMP" in d["cpu_baseline"]["sample"]
    assert set(d["config"]) >= {"workload", "l2", "parallelism"}


def test_gpu_arm_refuses_to_run_without_a_device():
    """No CPU fallback: on a box without a GPU the product arm of bench.py exits non-zero and prints no result line."""
    import ctypes
    from gslam_b200 import capi
    n = ctypes.c_int(0)
    if capi.lib().gb_device_count(ctypes.byref(n)) == 0 and n.value > 0:
        import pytest
        pytest.skip("a GPU is present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode != 0
    assert not any(l.startswith("{") for l in r.stdout.splitlines())


def test_dump_outputs_writes_the_last_step_as_float_arrays(tmp_path):
    """bench.py --dump-outputs: what a caller of the timed step receives, one float32 / float64 .npy per array, from stand-ins for
    the device objects (the device path itself is exercised by the GPU runs of bench.py)."""
    import importlib.util
    import types
    import numpy as np
    from gslam_b200.capi import KP_DTYPE
    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec); spec.loader.exec_module(bench)
    n, nc, npts = 5, 3, 4
    kps = np.zeros(n, KP_DTYPE); kps["x"] = np.arange(n); kps["octave"] = 2
    feats = types.SimpleNamespace(download=lambda: (kps, np.full((n, 32), 7, np.uint8)),
                                  matches=lambda: (np.arange(n, dtype=np.int32), np.full(n, 3, np.int32), np.full(n, 9, np.int32)))
    graph = types.SimpleNamespace(download=lambda: (np.ones((nc, 7)), np.ones((npts, 3))))
    res = types.SimpleNamespace(initial_cost=2.0, final_cost=1.0, iterations=10, accepted=9, pcg_iterations=50)
    bench.dump_outputs(str(tmp_path), feats, graph, res)
    want = {"keypoints": ((n, 7), np.float32), "descriptors": ((n, 32), np.float32), "match_index": ((n,), np.float32),
            "match_distance": ((n,), np.float32), "match_distance2": ((n,), np.float32), "ba_poses_wc": ((nc, 7), np.float64),
            "ba_points": ((npts, 3), np.float64), "ba_result": ((5,), np.float64)}
    assert sorted(os.listdir(tmp_path)) == sorted(k + ".npy" for k in want)
    for name, (shape, dtype) in want.items():
        a = np.load(tmp_path / (name + ".npy"))
        assert a.shape == shape and a.dtype == dtype, name
    assert np.array_equal(np.load(tmp_path / "keypoints.npy")[:, 0], np.arange(n)) and (np.load(tmp_path / "keypoints.npy")[:, 5] == 2).all()
    assert np.load(tmp_path / "ba_result.npy").tolist() == [2.0, 1.0, 10.0, 9.0, 50.0]


def test_zero_steps_are_refused():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "0"], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode != 0 and "--steps" in r.stderr
