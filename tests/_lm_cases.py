"""Bundle-adjustment graphs whose Levenberg-Marquardt decisions do not depend on summation order.

Near an optimum, accept / reject turns on the last bits of two costs that the device and the oracle sum in different orders.  The
cases here are built so that rounding cannot decide any of them:

* exact zero-cost graphs: rotations from {identity, the three 180-degree rotations} (R has entries in {0, +-1}), integer translations
  and landmarks, camera-frame depths that are powers of two, so every measurement x/z, y/z is exact in binary.  Every residual is
  exactly 0 on both sides, so the gradient, the step and the retraction of the step are exact zeros, the candidate cost equals the
  cost, and every step is rejected: status 2 after 12 rejects, lambda = lambda_init * 2^78 bit for bit, the estimate unchanged;
* reject / accept traces: graphs started far from the optimum with a small lambda_init, so that early Gauss-Newton steps overshoot;
  every decision of the oracle's run holds a relative margin of at least MARGIN (checked in tests/test_oracle_lm.py);
* the lambda floor: a graph whose first steps are all accepted from lambda_init = 1e-13;
* function-tolerance stops placed geometrically between the relative decrease of an accepted step of the oracle's run and the least
  one before it (ftol_between);
* a non-finite input cost: one observation with an infinite information entry.
"""
import functools

import numpy as np

from gslam_b200 import synth

MARGIN = 1e-6            # least |cnew - cost| / cost of every LM decision of a trace case
REJECTS_TO_OVERFLOW = 12  # lambda_init * 2^(1 + 2 + ... + 12) = lambda_init * 2^78 > 1e16 from lambda_init = 1e-4
LAMBDA_FLOOR = 1e-15

# x, y, z, w: the identity, then 180 degrees about x, y and z
QUATS = np.array([[0.0, 0.0, 0.0, 1.0], [1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0]])
# landmarks on the plane z = 32; a camera looking along +z (identity, 180 about z) at one of these heights, or along -z (180 about x
# or y) at one of the others, sees each of them at a depth of 32, 16, 8 or 4
PLANE_Z = 32.0
FORWARD_Z = (0.0, 16.0, 24.0, 28.0)
BACKWARD_Z = (64.0, 48.0, 40.0, 36.0)


def _R(q):
    return synth._quat_to_R(q)


def exact_graph(n_cams, n_points, obs_per_point, n_fixed=2, seed=0, with_info=False):
    """A zero-cost graph: landmark j is seen by `obs_per_point` consecutive cameras (a band of the reduced camera system)."""
    rng = np.random.default_rng(seed)
    k = np.arange(n_cams)
    q = QUATS[k % 4]
    t = np.zeros((n_cams, 3))
    t[:, :2] = rng.integers(-8, 9, (n_cams, 2))
    forward = (k % 4 == 0) | (k % 4 == 3)
    t[:, 2] = np.where(forward, np.take(FORWARD_Z, (k // 4) % 4), np.take(BACKWARD_Z, (k // 4) % 4))
    pts = np.zeros((n_points, 3))
    pts[:, :2] = rng.integers(-64, 65, (n_points, 2))
    pts[:, 2] = PLANE_Z
    first = rng.integers(0, n_cams - obs_per_point + 1, n_points)
    oc = (first[:, None] + np.arange(obs_per_point)[None, :]).reshape(-1).astype(np.int32)
    op = np.repeat(np.arange(n_points, dtype=np.int32), obs_per_point)
    pc = np.einsum("nji,nj->ni", _R(q)[oc], pts[op] - t[oc])  # R^T (p - t): integers
    assert np.all(pc == np.round(pc)) and set(np.unique(pc[:, 2])) <= {4.0, 8.0, 16.0, 32.0}
    xyz = np.concatenate([pc[:, :2] / pc[:, 2:3], np.ones((oc.shape[0], 1))], axis=1)
    perm = rng.permutation(oc.shape[0])
    dof = np.full(n_cams, 63, np.uint8)
    dof[:n_fixed] = 0
    info = None
    if with_info:  # integer SPD information: the residuals stay exact zeros
        info = np.tile(np.array([2.0, 1.0, 1.0, 3.0]), (oc.shape[0], 1))
    pose = np.ascontiguousarray(np.concatenate([q, t], axis=1))
    return synth.BAProblem(cam_pose_wc=pose, cam_dof=dof, points=np.ascontiguousarray(pts), point_free=np.ones(n_points, np.uint8),
                           obs_cam=np.ascontiguousarray(oc[perm]), obs_point=np.ascontiguousarray(op[perm]),
                           obs_xyz=np.ascontiguousarray(xyz[perm]), obs_info=info, gt_pose_wc=pose.copy(), gt_points=pts.copy())


@functools.lru_cache(maxsize=None)
def exact_local():
    """Local-window size: the 4-launch chain, the single-CTA sparse PCG and the direct solver all apply."""
    return exact_graph(24, 600, 5, seed=1, with_info=True)


@functools.lru_cache(maxsize=None)
def exact_large():
    """> 80 active cameras, 65 536 observations, 8 observers per landmark: the compact block-CSR path with the chunked Schur
    complement and the persistent sweep."""
    return exact_graph(96, 8192, 8, seed=2)


@functools.lru_cache(maxsize=None)
def exact_posegraph():
    """A zero-cost graph with exactly consistent SE3 and GPS edges (the pose-graph terms of the stepwise path)."""
    pb = exact_graph(16, 300, 4, seed=3)
    T = pb.cam_pose_wc
    first = np.arange(15, dtype=np.int32)
    second = first + 1
    loops_a = np.array([0, 3, 5], np.int32)
    loops_b = np.array([9, 14, 12], np.int32)
    first = np.concatenate([first, loops_a]); second = np.concatenate([second, loops_b])
    meas = synth.se3_mul(synth.se3_inv(T[first]), T[second])
    gps = np.array([0, 7, 15], np.int32)
    edges = synth.PoseEdges(first, second, np.ascontiguousarray(meas), None, gps, np.ascontiguousarray(T[gps]), None)
    return pb, edges


@functools.lru_cache(maxsize=None)
def exact_pnp():
    """One camera (180 degrees about y, looking along -z), 64 fixed landmarks at exact depths: (xyz, xy1, pose_wc)."""
    rng = np.random.default_rng(4)
    pose = np.array([0.0, 1.0, 0.0, 0.0, 3.0, -2.0, 48.0])
    xyz = np.zeros((64, 3))
    xyz[:, :2] = rng.integers(-20, 21, (64, 2))
    xyz[:, 2] = PLANE_Z
    pc = (xyz - pose[4:]) @ _R(pose[:4])
    assert np.all(pc[:, 2] == 16.0)
    xy1 = np.concatenate([pc[:, :2] / pc[:, 2:3], np.ones((64, 1))], axis=1)
    return xyz, xy1, pose


# ---- reject / accept traces ------------------------------------------------------------------------------------------------------
# (chosen by scanning seeds of synth.synth_ba with a large initial perturbation: the oracle's run of each has a streak of >= 2 rejects
# followed by accepts, a reject right after an accept, and a margin of >= MARGIN at every decision)
#   name: (n_cams, n_points, observers per landmark, seed, pose sigma t / deg, point sigma, huber delta, lambda_init, iterations)
TRACES = {
    "aa_rrrrrrr_aaa": (8, 120, 4, 1, 1.0, 10.0, 2.0, 0.01, 1e-10, 12),
    "rrrrrr_aaaa_rr": (10, 200, 5, 0, 1.0, 10.0, 2.0, 0.01, 1e-12, 12),
    # the lambda floor: six accepted steps from 1e-13 (1e-13 / 3^5 < 1e-15)
    "floor": (10, 200, 5, 3, 0.3, 3.0, 0.5, 0.01, 1e-13, 6),
}


@functools.lru_cache(maxsize=None)
def trace_case(name):
    """-> (problem, oracle options, iterations)"""
    nc, npt, obs, seed, st, sd, sp, delta, lam, iters = TRACES[name]
    pb = synth.synth_ba(nc, npt, obs_per_point=obs, seed=seed, n_fixed=2, pose_sigma_t=st, pose_sigma_deg=sd, point_sigma=sp)
    return pb, dict(huber_delta=delta, lambda_init=lam, pcg_max_iters=500, pcg_tol=1e-12), iters


def lm_replay(decisions, lam0):
    """lambda after each decision (True = accept) under the rule of lm_decide, from lam0"""
    lam, nu, out = lam0, 2.0, []
    for a in decisions:
        if a:
            lam = max(lam / 3.0, LAMBDA_FLOOR); nu = 2.0
        else:
            lam *= nu; nu *= 2.0
        out.append(lam)
    return out


def ftol_between(rels, k):
    """A function tolerance that stops a run at its k-th accepted step (k >= 1), geometrically between the relative decrease of that
    step and the least one before it, or None when they are less than a factor of 4 apart: the tolerance then stands a factor >= 2
    from both, where summation order moves a relative decrease by ~1e-12.  `rels`: relative decreases of the accepted steps in order."""
    lo = rels[k - 1]
    hi = min(rels[:k - 1]) if k > 1 else 4.0 * lo
    if hi < 4.0 * lo:
        return None
    return float(np.sqrt(hi * lo))


def nonfinite_graph():
    """The local zero-cost graph with one observation's information entry set to +inf (a residual of 0 times inf: a NaN cost)."""
    pb = exact_local().copy()
    pb.obs_info[7, 0] = np.inf
    return pb
