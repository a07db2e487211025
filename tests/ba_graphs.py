"""Irregular bundle-adjustment graphs for the parity tests (a test helper, not product code).

`synth.synth_ba` builds one shape only: every landmark seen by >= 3 consecutive keyframes, a fixed prefix of cameras, every
camera observed, free landmarks.  A real map is messier, and the solver's host-side planners branch on exactly the differences.
Each builder here starts from `synth_ba` and edits it into one named shape, deterministically, keeping the graph valid for
`gb_ba_graph_create` (no duplicate (camera, point) edge, no zero measurement z):

  scattered_fixed     fully fixed cameras at non-prefix indices, single-axis and mixed dof masks
  isolated_cameras    free cameras without observations (one in the middle, the last one), a free camera whose landmarks are all fixed
  sparse_landmarks    free landmarks with one observation and with none, fixed landmarks with many observers
  wide_landmarks      landmarks seen by 17..40 cameras (large: also one seen by more than 128)
  two_components      two disconnected trajectories, each with its own fixed camera
  measurement_forms   obs_xyz with z != 1 (negative too), non-unit quaternions, non-symmetric information, a Huber delta that
                      residuals straddle, landmarks behind some of their observing cameras

`build(name, large)`: the small size is a local-BA window (<= 80 active cameras); the large one has more than 80 active cameras and
more than 65 536 observations, so the compact path and the persistent sweep run by their own thresholds.
"""
from __future__ import annotations

import dataclasses

import numpy as np

from gslam_b200 import synth

PIXEL = 1.0 / 718.0  # synth_ba's measurement noise (one pixel at its focal length)


@dataclasses.dataclass
class Case:
    name: str
    pb: synth.BAProblem
    delta: float = 0.01                                   # Huber threshold the case is meant to be solved with
    isolated: list = dataclasses.field(default_factory=list)     # free cameras without observations
    unobserved: list = dataclasses.field(default_factory=list)   # free landmarks without observations
    single: list = dataclasses.field(default_factory=list)       # free landmarks with exactly one observation


def _keep_edges(pb: synth.BAProblem, keep: np.ndarray) -> None:
    pb.obs_cam = np.ascontiguousarray(pb.obs_cam[keep])
    pb.obs_point = np.ascontiguousarray(pb.obs_point[keep])
    pb.obs_xyz = np.ascontiguousarray(pb.obs_xyz[keep])
    if pb.obs_info is not None:
        pb.obs_info = np.ascontiguousarray(pb.obs_info[keep])


def _add_landmark(pb: synth.BAProblem, cams, rng, ahead: float, free: bool = True) -> int:
    """A new landmark `ahead` metres beyond the farthest of `cams` along the trajectory (in front of all of them), observed by each of
    them with synth_ba's pixel noise; its estimate is the truth perturbed like synth_ba's (exact when fixed).  Returns its index."""
    cams = np.asarray(sorted(set(int(c) for c in cams)), np.int32)
    T = pb.gt_pose_wc
    p = np.array([rng.uniform(-2, 2), rng.uniform(-1, 1), T[cams, 6].max() + ahead])
    R = synth._quat_to_R(T[cams, :4])
    pc = np.einsum("nji,nj->ni", R, p[None] - T[cams, 4:])
    assert (pc[:, 2] > 1.0).all()
    uv = pc[:, :2] / pc[:, 2:3] + PIXEL * rng.standard_normal((cams.shape[0], 2))
    j = pb.n_points
    pb.points = np.ascontiguousarray(np.vstack([pb.points, p + (0.1 * rng.standard_normal(3) if free else 0.0)]))
    pb.gt_points = np.vstack([pb.gt_points, p])
    pb.point_free = np.append(pb.point_free, np.uint8(1 if free else 0))
    pb.obs_cam = np.ascontiguousarray(np.append(pb.obs_cam, cams))
    pb.obs_point = np.ascontiguousarray(np.append(pb.obs_point, np.full(cams.shape[0], j, np.int32)))
    pb.obs_xyz = np.ascontiguousarray(np.vstack([pb.obs_xyz, np.concatenate([uv, np.ones((cams.shape[0], 1))], axis=1)]))
    assert pb.obs_info is None
    return j


def _base(large: bool, seed: int, **kw) -> synth.BAProblem:
    # small: 30 cameras, 500 landmarks, 2000 edges; large: 160 cameras, 18 000 landmarks, 72 000 edges
    if large:
        return synth.synth_ba(160, 18000, obs_per_point=4, seed=seed, **kw)
    return synth.synth_ba(30, 500, obs_per_point=4, seed=seed, **kw)


def scattered_fixed(large: bool) -> Case:
    pb = _base(large, 101, n_fixed=0)
    pb.cam_dof[3::7] = 0                                    # fully fixed keyframes in the middle of the window
    masks = [1, 2, 4, 8, 16, 32, 0b000111, 0b111000, 0b010101]
    free = [i for i in range(pb.n_cams) if pb.cam_dof[i] != 0]
    for m, i in zip(masks, free[1::2]):
        pb.cam_dof[i] = m
    return Case("scattered_fixed", pb)


def isolated_cameras(large: bool) -> Case:
    pb = _base(large, 102)
    nc = pb.n_cams
    mid, last, fixed_lm = nc // 2, nc - 1, nc // 3
    _keep_edges(pb, (pb.obs_cam != mid) & (pb.obs_cam != last))
    pb.point_free[np.unique(pb.obs_point[pb.obs_cam == fixed_lm])] = 0   # every landmark of this free camera is fixed
    return Case("isolated_cameras", pb, isolated=[mid, last])


def sparse_landmarks(large: bool) -> Case:
    pb = _base(large, 103)
    rng = np.random.default_rng(7)
    np_ = pb.n_points
    pick = rng.permutation(np_)
    single, none = np.sort(pick[:np_ // 20]), np.sort(pick[np_ // 20:np_ // 20 + np_ // 50])
    keep = ~np.isin(pb.obs_point, none)
    for j in single:                                        # keep the first edge of each of these landmarks only
        e = np.nonzero(pb.obs_point == j)[0]
        keep[e[1:]] = False
    _keep_edges(pb, keep)
    for k in range(4):                                      # fixed landmarks with many observers (more than a Schur chunk's 16)
        _add_landmark(pb, range(2 + 5 * k, min(pb.n_cams, 22 + 5 * k)), rng, 25.0, free=False)
    return Case("sparse_landmarks", pb, unobserved=none.tolist(), single=single.tolist())


def wide_landmarks(large: bool) -> Case:
    pb = _base(large, 104)
    rng = np.random.default_rng(8)
    nc = pb.n_cams
    # (small: S keeps 698 of its 900 blocks, so the single-CTA sparse PCG still fits one SM's shared memory; observed by all 30
    #  cameras, a landmark would fill S and send the window to the compact path)
    spans = [(0, 17, 1), (13, 30, 1), (1, 30, 4), (3, 23, 1)] if not large else [(0, 17, 1), (20, 60, 1), (5, 85, 2), (100, 157, 2)]
    for a, b, s in spans:
        _add_landmark(pb, range(a, min(b, nc), s), rng, 30.0)
    if large:                                               # more observers than one 128-lane chunk of the persistent sweep
        _add_landmark(pb, range(2, 150), rng, 60.0)
    return Case("wide_landmarks", pb)


def two_components(large: bool) -> Case:
    kw = dict(n_cams=80, n_points=8500) if large else dict(n_cams=15, n_points=250)
    a = synth.synth_ba(obs_per_point=4, n_fixed=1, seed=105, **kw)
    b = synth.synth_ba(obs_per_point=4, n_fixed=1, seed=106, **kw)
    off = np.array([1000.0, 0.0, 0.0])                      # the second trajectory far away: no landmark is shared
    nca, npa = a.n_cams, a.n_points
    pose_b, gt_b = b.cam_pose_wc.copy(), b.gt_pose_wc.copy()
    pose_b[:, 4:] += off; gt_b[:, 4:] += off
    pb = synth.BAProblem(cam_pose_wc=np.ascontiguousarray(np.vstack([a.cam_pose_wc, pose_b])), cam_dof=np.concatenate([a.cam_dof, b.cam_dof]),
                         points=np.ascontiguousarray(np.vstack([a.points, b.points + off])), point_free=np.concatenate([a.point_free, b.point_free]),
                         obs_cam=np.ascontiguousarray(np.concatenate([a.obs_cam, b.obs_cam + nca]).astype(np.int32)),
                         obs_point=np.ascontiguousarray(np.concatenate([a.obs_point, b.obs_point + npa]).astype(np.int32)),
                         obs_xyz=np.ascontiguousarray(np.vstack([a.obs_xyz, b.obs_xyz])),
                         gt_pose_wc=np.vstack([a.gt_pose_wc, gt_b]), gt_points=np.vstack([a.gt_points, b.gt_points + off]))
    return Case("two_components", pb)


def measurement_forms(large: bool) -> Case:
    pb = _base(large, 107)
    rng = np.random.default_rng(9)
    n = pb.n_obs
    s = rng.uniform(0.5, 3.0, n) * np.where(rng.random(n) < 0.3, -1.0, 1.0)   # the same ray: (x, y, z) * s, z negative for some
    pb.obs_xyz = np.ascontiguousarray(pb.obs_xyz * s[:, None])
    free = pb.cam_dof != 0
    pb.cam_pose_wc[free, :4] *= rng.uniform(0.8, 1.25, (int(free.sum()), 1))  # non-unit quaternions (normalised on input)
    L = rng.uniform(0.3, 1.0, (n, 2, 2))
    info = L @ np.transpose(L, (0, 2, 1)) + 0.5 * np.eye(2)
    info[:, 0, 1] += rng.uniform(-0.4, 0.4, n)              # non-symmetric: both sides average the off-diagonals
    info[:, 1, 0] -= rng.uniform(-0.4, 0.4, n)
    pb.obs_info = np.ascontiguousarray(info.reshape(n, 4))
    # a few landmarks moved between their observing cameras: behind the later ones, in front of the earlier ones
    for j in (3, 11, 29):
        cams = np.sort(pb.obs_cam[pb.obs_point == j])
        pb.points[j] = pb.cam_pose_wc[cams[1], 4:] + np.array([0.2, -0.1, 1.5])
    # the Huber threshold at the 60th percentile of the initial whitened residuals: both branches are taken
    Rwc = synth._quat_to_R(pb.cam_pose_wc[:, :4] / np.linalg.norm(pb.cam_pose_wc[:, :4], axis=1, keepdims=True))
    q = np.einsum("nji,nj->ni", Rwc[pb.obs_cam], pb.points[pb.obs_point] - pb.cam_pose_wc[pb.obs_cam, 4:])
    ok = q[:, 2] > 0
    r = q[ok, :2] / q[ok, 2:3] - pb.obs_xyz[ok, :2] / pb.obs_xyz[ok, 2:3]
    Ls = 0.5 * (info + np.transpose(info, (0, 2, 1)))[ok]
    e = np.sqrt(np.einsum("ki,kij,kj->k", r, Ls, r))
    assert (~ok).sum() >= 3
    return Case("measurement_forms", pb, delta=float(np.quantile(e, 0.6)))


CASES = {f.__name__: f for f in (scattered_fixed, isolated_cameras, sparse_landmarks, wide_landmarks, two_components, measurement_forms)}


def build(name: str, large: bool = False) -> Case:
    c = CASES[name](large)
    check(c.pb)
    return c


# ---- boundary graphs: one just under / over each host-side threshold ------------------------------------------------------------------
def local4_under() -> synth.BAProblem:
    """np*3 + nc*19 == 65536 exactly: the last graph the 4-launch local-BA chain takes."""
    return synth.synth_ba(40, 21592, obs_per_point=3, n_fixed=2, seed=110)


def local4_over() -> synth.BAProblem:
    """np*3 + nc*19 == 65539: the same window with one landmark more leaves the chain for the stepwise iteration."""
    return synth.synth_ba(40, 21593, obs_per_point=3, n_fixed=2, seed=110)


def sparse_over_80_cams() -> synth.BAProblem:
    """96 cameras, every 6th fixed: 80 active cameras, so the single-CTA sparse PCG takes a graph with more than 80 cameras."""
    pb = synth.synth_ba(96, 1500, obs_per_point=3, n_fixed=0, seed=111)
    pb.cam_dof[::6] = 0
    return pb


def natural_cam_split() -> synth.BAProblem:
    """4 cameras seeing all of 20 000 landmarks: 20 000 observations per camera slice the camera pass without any hook."""
    return synth.synth_ba(4, 20000, all_visible=True, n_fixed=1, seed=112)


def over_2048_cams() -> synth.BAProblem:
    """More cameras than the host derives the covisibility block structure for: the dense 6N x 6N reduced system."""
    return synth.synth_ba(2100, 6000, obs_per_point=3, n_fixed=2, seed=113)


def check(pb: synth.BAProblem) -> None:
    """The invariants gb_ba_graph_create checks, asserted on the host."""
    assert pb.obs_cam.dtype == np.int32 and pb.obs_point.dtype == np.int32
    assert pb.cam_pose_wc.flags.c_contiguous and pb.points.flags.c_contiguous and pb.obs_xyz.flags.c_contiguous
    assert ((pb.obs_cam >= 0) & (pb.obs_cam < pb.n_cams)).all() and ((pb.obs_point >= 0) & (pb.obs_point < pb.n_points)).all()
    assert (pb.obs_xyz[:, 2] != 0).all() and np.isfinite(pb.obs_xyz).all()
    key = pb.obs_cam.astype(np.int64) * pb.n_points + pb.obs_point
    assert np.unique(key).shape[0] == key.shape[0], "duplicate (camera, point) edge"
    assert pb.point_free.shape[0] == pb.n_points and pb.cam_dof.shape[0] == pb.n_cams
