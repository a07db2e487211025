"""The N>1 path: landmark sharding host logic (CPU, world_size-2 gloo) and the NCCL-reduced global BA (gpu, needs 2 GPUs)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import oracle
from gslam_b200 import synth
from gslam_b200.dist import shard_bounds, shard_landmarks

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_shards_partition_the_graph():
    pb = synth.synth_ba(20, 500, obs_per_point=6, seed=3)
    for world in (1, 2, 3, 8):
        seen_pts, n_obs = [], 0
        loads = []
        for r in range(world):
            loc, ids = shard_landmarks(pb, r, world)
            seen_pts.append(ids); n_obs += loc.n_obs; loads.append(loc.n_obs)
            assert np.array_equal(loc.points, pb.points[ids])
            assert loc.n_cams == pb.n_cams and np.array_equal(loc.cam_pose_wc, pb.cam_pose_wc)
            assert loc.obs_point.min(initial=0) >= 0 and loc.obs_point.max(initial=-1) < loc.n_points
        assert np.array_equal(np.concatenate(seen_pts), np.arange(pb.n_points))   # every landmark exactly once
        assert n_obs == pb.n_obs                                                   # every edge exactly once
        assert max(loads) - min(loads) <= 2 * 6 + pb.n_obs // (10 * world)         # balanced by edge count


def test_cabi_shard_bounds_equal_the_python_restatement():
    """The landmark ranges ba_graph_create_impl uses (host-only hook, no device) == gslam_b200.dist.shard_bounds."""
    import ctypes as C
    from gslam_b200 import capi
    L = capi.lib()
    rng = np.random.default_rng(0)
    for (nc, npts, opp, seed) in [(20, 500, 6, 3), (5, 37, 3, 1), (50, 2000, 5, 42), (8, 1, 8, 2)]:
        pb = synth.synth_ba(nc, npts, obs_per_point=min(opp, nc), seed=seed)
        op = np.ascontiguousarray(pb.obs_point[rng.permutation(pb.n_obs)], np.int32)   # edge order must not matter
        for world in (1, 2, 3, 4, 8, 16):
            out = np.zeros(world + 1, np.int32)
            assert L.gb_dbg_ba_shard_bounds(pb.n_points, pb.n_obs, capi.ptr(op), world, capi.ptr(out)) == 0
            assert out.tolist() == shard_bounds(pb, world), (nc, npts, world)
            assert out[0] == 0 and out[-1] == pb.n_points and np.all(np.diff(out) >= 0)


WORKER = r'''
import os, sys
sys.path.insert(0, sys.argv[1])
import numpy as np, torch, torch.distributed as dist
import oracle
from gslam_b200 import synth
from gslam_b200.dist import shard_landmarks
dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
pb = synth.synth_ba(12, 300, obs_per_point=5, seed=9)
loc, ids = shard_landmarks(pb, rank, world)
lin = oracle.ba_linearize(loc, 0.01)
# the path's exchange step: sum over ranks of the camera-side blocks and the cost
buf = torch.from_numpy(np.concatenate([lin["U"].ravel(), lin["gc"].ravel(), [lin["cost"]]]))
dist.all_reduce(buf)
full = oracle.ba_linearize(pb, 0.01)
want = np.concatenate([full["U"].ravel(), full["gc"].ravel(), [full["cost"]]])
err = np.abs(buf.numpy() - want).max() / np.abs(want).max()
# landmark-side blocks are a partition, not a sum
okV = np.allclose(lin["V"], full["V"][ids], rtol=1e-12, atol=0)
print("RESULT", rank, err, okV)
assert err < 1e-12 and okV
dist.destroy_process_group()
'''


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def test_world2_gloo_exchange_step_matches_unsharded(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script), ROOT]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env={**os.environ, "OMP_NUM_THREADS": "1"})
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("RESULT") == 2


GPU_WORKER = r'''
import os, sys
sys.path.insert(0, sys.argv[1])
import numpy as np, torch, torch.distributed as dist
from gslam_b200 import synth
from gslam_b200.api import Context, OptimzeConfig
from gslam_b200.dist import DistributedBA
local = int(os.environ["LOCAL_RANK"]); torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
rank, world = dist.get_rank(), dist.get_world_size()
ctx = Context(local)
pb = synth.synth_ba(60, 6000, obs_per_point=8, seed=11, n_fixed=2)
cfg = OptimzeConfig(maxIterations=6, functionTolerance=0.0, pcgMaxIterations=40)
d = DistributedBA(ctx, pb, rank, world)
res = d.solve(cfg)
pose, pts, ids = d.download()
# every rank must hold bit-identical cameras (replicated deterministic PCG, no broadcast)
t = torch.from_numpy(pose.copy()).cuda(); lo = t.clone(); hi = t.clone()
dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX)
assert torch.equal(lo, hi), "ranks diverged"
full = torch.zeros((pb.n_points, 3), dtype=torch.float64, device="cuda"); full[torch.from_numpy(ids).cuda()] = torch.from_numpy(pts).cuda()
dist.all_reduce(full)
if rank == 0:
    import oracle
    ref = pb.copy()
    r0 = oracle.ba_solve(ref, max_iterations=6, function_tolerance=0.0, pcg_max_iters=40)
    ep = np.abs(pose[:, 4:] - ref.cam_pose_wc[:, 4:]).max(); ex = np.abs(full.cpu().numpy() - ref.points).max() / np.abs(ref.points).max()
    ec = abs(res.final_cost - r0.final_cost) / r0.final_cost
    print("RESULT", world, res.final_cost, r0.final_cost, ec, ep, ex, res.accepted, r0.accepted)
    assert ec < 1e-5 and ep < 1e-5 * max(1.0, np.abs(ref.cam_pose_wc[:, 4:]).max()) and ex < 1e-5 and res.accepted == r0.accepted
d.close(); dist.destroy_process_group()
'''


@pytest.mark.gpu
def test_world2_nccl_global_ba_matches_oracle(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(GPU_WORKER)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script), ROOT]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "RESULT 2" in r.stdout


@pytest.mark.gpu
def test_single_process_multi_gpu_solve_matches_oracle():
    """gb_comm_create_all + gb_ba_solve_multi: ONE process drives every visible GPU (1 GPU: world 1, no NCCL) -- the entry point
    the optimizer plugin uses for `b200.devices`."""
    import ctypes as C
    from gslam_b200 import capi
    from gslam_b200.api import Context, OptimzeConfig, ba_solve_multi
    n = C.c_int(0)
    assert capi.lib().gb_device_count(C.byref(n)) == 0
    ndev = min(n.value, 8)
    ctxs = [Context(k) for k in range(ndev)]
    pb = synth.synth_ba(60, 6000, obs_per_point=8, seed=11, n_fixed=2)
    ref = pb.copy()
    r0 = oracle.ba_solve(ref, max_iterations=6, function_tolerance=0.0, pcg_max_iters=40)
    r1 = ba_solve_multi(ctxs, pb, OptimzeConfig(maxIterations=6, functionTolerance=0.0, pcgMaxIterations=40))
    assert r1.accepted == r0.accepted and abs(r1.final_cost - r0.final_cost) / r0.final_cost < 1e-5
    assert np.abs(pb.cam_pose_wc - ref.cam_pose_wc).max() < 1e-5 * max(1.0, np.abs(ref.cam_pose_wc).max())
    assert np.abs(pb.points - ref.points).max() / np.abs(ref.points).max() < 1e-5
    for c in ctxs:
        c.close()


@pytest.mark.gpu
def test_world1_stepwise_path_matches_oracle(tmp_path):
    """The sharded engine with world=1 (communicator without NCCL): runs on a single-GPU box."""
    script = tmp_path / "worker.py"
    script.write_text(GPU_WORKER)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=1", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(script), ROOT]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "RESULT 1" in r.stdout
