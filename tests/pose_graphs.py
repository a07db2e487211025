"""Named pose-graph cases for the parity tests of the SE3 / GPS edges (csrc/ba_pose.cu) -- a test helper, not product code.

`synth.synth_pose_edges` measures every edge on the ground truth with small noise, so its residuals stay far from the branches of
the SE3 logarithm and from the radius where the Bernoulli series of J_l^-1 loses digits.  The builders here aim at those places,
deterministically; each returns `(pb, edges)` that `gb_ba_graph_create_ex` accepts:

  edge_sweep(kind, angle)  one edge per independent block (disjoint camera pairs for "se3", single cameras for "gps"), so that a
                           camera's rows of U, g_c and S are exactly its edge's record; residual rotation angle `angle` (ANGLES)
  large_residuals          a drifted 60-keyframe pose graph: consistent odometry, loop closures 30..150 degrees off
  masks_and_fixed          single-axis / translation-only / rotation-only dof masks on either side of an edge, fixed-fixed edge
  info_forms(form)         non-symmetric, rank-deficient, zero-row and scaled information; a GPS frame around 1e5 m
  hub_and_parallel         300 keyframes, 20 000 edges, one keyframe with 600 incident edges, 20 parallel edges both ways
  mixed_large(name)        tests/ba_graphs.py's large graphs (160 cameras, > 65 536 observations) plus odometry, loops and GPS
  size_case(n)             a plain pose graph of n keyframes (300: generic PCG by size; 2100: no covisibility structure)

The rounding-sensitive angles (exactly pi, w within 1e-10 of 0) are built from exactly representable quaternions on cameras with
identity rotation, so the residual quaternion E is formed without rounding on either side: its w, and so the sign the logarithm
gives at pi, cannot depend on the order or contraction of floating-point operations.
"""
from __future__ import annotations

import math

import numpy as np

from gslam_b200 import synth
import ba_graphs  # (tests/ is on sys.path under pytest's rootdir conftest)

# residual rotation of an edge: an angle in rad, or an exact quaternion w with a unit axis (w = 0: exactly pi)
ANGLES = {
    "0": 0.0, "1e-14": 1e-14, "1e-11": 1e-11, "1e-9": 1e-9, "1e-6": 1e-6, "1e-3": 1e-3, "0.1": 0.1, "0.5": 0.5, "1": 1.0, "2": 2.0,
    "2.5": 2.5, "3": 3.0, "pi-1e-6": math.pi - 1e-6, "pi": ("w", 0.0), "w+5e-11": ("w", 5e-11), "w-5e-11": ("w", -5e-11),
    "w+2e-10": ("w", 2e-10), "w-2e-10": ("w", -2e-10),
}
EXACT_ONLY = {"pi", "w+5e-11", "w-5e-11", "w+2e-10", "w-2e-10"}  # (no rounded variant: the sign of w would be decided by rounding)


def _unit(v):
    return v / np.linalg.norm(v)


def _rand_quat(rng):
    return _unit(rng.standard_normal(4))


def _spd(rng, scale=1.0):
    A = rng.standard_normal((6, 6))
    M = A @ A.T + 6.0 * np.eye(6)
    M[:3, :3] *= 4.0
    return scale * M


def _residual_quat(angle, axis):
    if isinstance(angle, tuple):
        return np.concatenate([axis, [angle[1]]])
    return np.concatenate([math.sin(0.5 * angle) * axis, [math.cos(0.5 * angle)]])


def _pose_graph(pose_wc, dof=None):
    n = pose_wc.shape[0]
    return synth.BAProblem(cam_pose_wc=np.ascontiguousarray(pose_wc, np.float64), cam_dof=np.full(n, 63, np.uint8) if dof is None else dof,
                           points=np.zeros((0, 3)), point_free=np.zeros(0, np.uint8), obs_cam=np.zeros(0, np.int32),
                           obs_point=np.zeros(0, np.int32), obs_xyz=np.zeros((0, 3)), gt_pose_wc=np.array(pose_wc, copy=True))


def _edges(first=(), second=(), meas=None, info=None, gps=(), gmeas=None, ginfo=None):
    f = np.ascontiguousarray(first, np.int32); s = np.ascontiguousarray(second, np.int32); g = np.ascontiguousarray(gps, np.int32)
    return synth.PoseEdges(f, s, np.ascontiguousarray(np.reshape(meas, (-1, 7)) if meas is not None else np.zeros((0, 7))),
                           None if info is None else np.ascontiguousarray(np.reshape(info, (-1, 36))), g,
                           np.ascontiguousarray(np.reshape(gmeas, (-1, 7)) if gmeas is not None else np.zeros((0, 7))),
                           None if ginfo is None else np.ascontiguousarray(np.reshape(ginfo, (-1, 36))))


# ---- one edge per block ----------------------------------------------------------------------------------------------------------
def edge_sweep(kind: str, angle: str):
    """Independent blocks whose single edge has residual rotation ANGLES[angle].  Variants per block:
      exact  identity-rotation cameras (the first given with -q in two of them: E's w flips sign for every angle), the measurement
             quaternion scaled by 0.5..2, residual translation 0, ~3 m and ~100 m; E = +-Z^-1 without rounding
      rounded (not for EXACT_ONLY) random camera rotations and translations up to 100 m, the residual translation 1..100 m (so the
             rounding of E stays ~1e-16 of each block's largest entry)
    SE3 blocks alternate the edge's direction (first > second for odd blocks)."""
    assert kind in ("se3", "gps")
    a = ANGLES[angle]
    rng = np.random.default_rng(1000 + list(ANGLES).index(angle) + (0 if kind == "se3" else 500))
    variants = [("exact", +1, 0.0, 1.0), ("exact", -1, 3.0, rng.uniform(0.5, 2.0)), ("exact", -1, 100.0, rng.uniform(0.5, 2.0)),
                ("exact", +1, 100.0, 0.5)]
    if angle not in EXACT_ONLY:
        variants += [("rounded", +1, rng.uniform(1.0, 100.0), 1.0), ("rounded", -1, rng.uniform(1.0, 100.0), rng.uniform(0.5, 2.0))]
    first, second, meas, info, gps, gmeas, ginfo, pose = [], [], [], [], [], [], [], []
    for b, (how, sgn, tnorm, qscale) in enumerate(variants):
        E = np.concatenate([_residual_quat(a, _unit(rng.standard_normal(3))), tnorm * _unit(rng.standard_normal(3)) if tnorm else np.zeros(3)])
        Om = np.eye(6) if b == 0 else _spd(rng)
        if how == "exact":
            Pi = np.array([0.0, 0.0, 0.0, float(sgn), 0.0, 0.0, 0.0])
            Pj = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
            if kind == "se3":   # equal translations: T_cw,i T_cw,j^-1 = (+-1 | 0) exactly
                Pi[4:] = Pj[4:] = np.round(rng.uniform(-50, 50, 3))
        else:
            q = _rand_quat(rng)
            Pi = np.concatenate([sgn * np.copysign(1.0, q[3]) * q, rng.uniform(-100, 100, 3)])
            Pj = np.concatenate([_rand_quat(rng), rng.uniform(-100, 100, 3)])
        # E = Z^-1 M with M = T_wc,i^-1 T_wc,j (SE3) or T_wc,i (GPS)  ->  Z = M E^-1;  exact: Z = E^-1 (and E = +-Z^-1 back)
        if how == "exact":
            Z = synth.se3_inv(E)
        else:
            M = synth.se3_mul(synth.se3_inv(Pi), Pj) if kind == "se3" else Pi
            Z = synth.se3_mul(M, synth.se3_inv(E))
        Z[:4] *= qscale
        if kind == "se3":   # odd blocks: the edge runs from camera 2b+1 (holding Pi) to camera 2b
            i, j = (2 * b, 2 * b + 1) if b % 2 == 0 else (2 * b + 1, 2 * b)
            pose += [Pi, Pj] if b % 2 == 0 else [Pj, Pi]
            first.append(i); second.append(j); meas.append(Z); info.append(Om)
        else:
            pose.append(Pi)
            gps.append(b); gmeas.append(Z); ginfo.append(Om)
    pb = _pose_graph(np.array(pose))
    if kind == "se3":
        return pb, _edges(first, second, np.array(meas), np.array(info))
    return pb, _edges(gps=gps, gmeas=np.array(gmeas), ginfo=np.array(ginfo))


# ---- whole graphs ------------------------------------------------------------------------------------------------------------------
def _spd_many(rng, m, scale=1.0):
    A = rng.standard_normal((m, 6, 6))
    M = np.einsum("nij,nkj->nik", A, A) + 6.0 * np.eye(6)
    M[:, :3, :3] *= 4.0
    return scale * M


def _measure(T, first, second, rng, sigma_t=0.02, sigma_r=0.002):
    """SE3 measurements SE3_12 = T_1^-1 T_2 of the poses T (n, 7), with synth_pose_edges' noise."""
    first, second = np.asarray(first), np.asarray(second)
    return synth.se3_mul(synth.se3_mul(synth.se3_inv(T[first]), T[second]), synth._small_se3(rng, first.shape[0], sigma_t, sigma_r))


def large_residuals():
    """60 keyframes whose estimate has drifted: keyframe k is turned by 150 deg * k / 59 about the world's vertical axis through the
    first one.  Odometry is measured on the estimate (consistent), the 8 loop closures and the GPS priors at both ends on the ground
    truth, so the loops disagree with the estimate by 38..142 deg."""
    pb = synth.synth_ba(60, 0, n_fixed=1, seed=21)
    gt = pb.gt_pose_wc
    n = gt.shape[0]
    d = np.deg2rad(150.0) * np.arange(n) / (n - 1)
    D = np.zeros((n, 7)); D[:, 1] = np.sin(0.5 * d); D[:, 3] = np.cos(0.5 * d)
    est = synth.se3_mul(D, gt)
    pb.cam_pose_wc = np.ascontiguousarray(est)
    rng = np.random.default_rng(22)
    odo_f, odo_s = np.arange(n - 1), np.arange(1, n)
    loops = np.array([(0, 15), (5, 30), (10, 45), (3, 59), (20, 50), (30, 55), (12, 40), (25, 59)])
    first = np.concatenate([odo_f, loops[:, 0]]); second = np.concatenate([odo_s, loops[:, 1]])
    meas = np.concatenate([synth.se3_mul(synth.se3_inv(est[odo_f]), est[odo_s]), _measure(gt, loops[:, 0], loops[:, 1], rng)])
    gps = np.array([0, n - 1])
    gmeas = synth.se3_mul(gt[gps], synth._small_se3(rng, 2, 0.05, 0.005))
    return pb, _edges(first, second, meas, _spd_many(rng, first.shape[0]), gps, gmeas, _spd_many(rng, 2))


# dof masks (bit d frees tangent component d, order [v, w])
MASKS = {2: 0b000001, 3: 0b000111, 4: 0b111000, 5: 0b100000, 6: 0b010101}


def masks_and_fixed():
    """14 keyframes: 0 and 1 fully fixed, 2..6 with the partial masks of MASKS.  Odometry, masked cameras as the first and as the
    second camera of loop edges, an edge between the two fixed cameras (cost only) and GPS priors on a fixed and on masked cameras."""
    pb = synth.synth_ba(14, 0, n_fixed=0, seed=23, pose_sigma_t=0.1, pose_sigma_deg=2.0)
    pb.cam_dof[:2] = 0
    for i, m in MASKS.items():
        pb.cam_dof[i] = m
    rng = np.random.default_rng(24)
    loops = [(2, 9), (9, 3), (4, 10), (11, 4), (5, 12), (13, 6), (2, 6), (6, 3), (1, 0)]
    first = list(range(13)) + [a for a, _ in loops]; second = list(range(1, 14)) + [b for _, b in loops]
    gps = [0, 3, 4, 6, 12]
    T = pb.gt_pose_wc
    return pb, _edges(first, second, _measure(T, first, second, rng), _spd_many(rng, len(first)), gps,
                      synth.se3_mul(T[gps], synth._small_se3(rng, len(gps), 0.1, 0.01)), _spd_many(rng, len(gps)))


INFO_FORMS = ("nonsymmetric", "translation_only_gps", "zero_row", "scaled_1e-6", "scaled_1e6", "utm")
UTM = np.array([123456.0, 78.0, 98765.0])   # the frame offset of info_forms("utm")


def info_forms(form: str):
    """12 keyframes with odometry, 4 loops and a GPS prior on every 3rd keyframe; the information matrices (or the frame) in `form`:
      nonsymmetric          a random strictly upper-triangular part added to every matrix (the solver uses (O + O') / 2)
      translation_only_gps  GPS information with zero rotation rows and columns (rank 3)
      zero_row              SE3 information with row k % 6 zeroed (even edges: its column too, rank 5; odd edges: the row only)
      scaled_1e-6 / 1e6     every matrix scaled
      utm                   the whole trajectory and the GPS priors moved by UTM (~1e5 m)"""
    assert form in INFO_FORMS
    pb = synth.synth_ba(12, 0, n_fixed=1, seed=31, pose_sigma_t=0.1, pose_sigma_deg=2.0)
    if form == "utm":
        pb.cam_pose_wc[:, 4:] += UTM; pb.gt_pose_wc[:, 4:] += UTM
    pe = synth.synth_pose_edges(pb, seed=5, n_loops=4, gps_every=3, with_info=True)
    rng = np.random.default_rng(32)
    si, gi = pe.se3_info.reshape(-1, 6, 6), pe.gps_info.reshape(-1, 6, 6)
    if form == "nonsymmetric":
        for M in (si, gi):
            M += np.triu(rng.uniform(-3, 3, M.shape), 1)
    elif form == "translation_only_gps":
        gi[:, 3:, :] = 0.0; gi[:, :, 3:] = 0.0
    elif form == "zero_row":
        for k in range(si.shape[0]):
            si[k, k % 6, :] = 0.0
            if k % 2 == 0:
                si[k, :, k % 6] = 0.0
    elif form.startswith("scaled"):
        s = float(form.split("_")[1])
        si *= s; gi *= s
    pe.se3_info = np.ascontiguousarray(si.reshape(-1, 36)); pe.gps_info = np.ascontiguousarray(gi.reshape(-1, 36))
    return pb, pe


def hub_and_parallel():
    """300 keyframes and 20 000 SE3 edges: odometry; keyframe 150 joined to every other keyframe twice, once in each direction
    (600 incident edges with its odometry); 20 parallel edges between keyframes 7 and 8 alternating in direction; random pairs
    for the rest.  GPS priors on every 25th keyframe."""
    pb = synth.synth_ba(300, 0, n_fixed=1, seed=41)
    n, hub = 300, 150
    rng = np.random.default_rng(42)
    others = np.array([c for c in range(n) if c != hub])
    first = [np.arange(n - 1), np.full(others.shape[0], hub), others, np.where(np.arange(20) % 2 == 0, 7, 8)]
    second = [np.arange(1, n), others, np.full(others.shape[0], hub), np.where(np.arange(20) % 2 == 0, 8, 7)]
    m = 20000 - sum(f.shape[0] for f in first)
    a = rng.integers(0, n, m); b = (a + rng.integers(1, n, m)) % n   # (b != a)
    first.append(a); second.append(b)
    first = np.concatenate(first); second = np.concatenate(second)
    T = pb.gt_pose_wc
    gps = np.arange(0, n, 25)
    return pb, _edges(first, second, _measure(T, first, second, rng), _spd_many(rng, first.shape[0]), gps,
                      synth.se3_mul(T[gps], synth._small_se3(rng, gps.shape[0], 0.1, 0.01)), _spd_many(rng, gps.shape[0]))


MIXED_LARGE = ("scattered_fixed", "isolated_cameras")


def mixed_large(name: str):
    """tests/ba_graphs.py's large `name` (160 cameras, > 65 536 observations) with odometry, 20 loops and a GPS prior on every 10th
    keyframe.  In isolated_cameras the two cameras without observations are held by their odometry and GPS edges alone."""
    assert name in MIXED_LARGE
    c = ba_graphs.build(name, True)
    return c.pb, synth.synth_pose_edges(c.pb, seed=61, n_loops=20, gps_every=10, with_info=True)


def size_case(n: int):
    """A plain pose graph of n keyframes: odometry, n / 10 loops, a GPS prior on every 50th keyframe."""
    pb = synth.synth_ba(n, 0, n_fixed=1, seed=50 + n)
    return pb, synth.synth_pose_edges(pb, seed=7, n_loops=n // 10, gps_every=50, with_info=True)


def check(pb: synth.BAProblem, pe: synth.PoseEdges) -> None:
    """The invariants gb_ba_graph_create_ex checks on the edges, asserted on the host."""
    ba_graphs.check(pb)
    assert pe.se3_first.dtype == np.int32 and pe.se3_second.dtype == np.int32 and pe.gps_frame.dtype == np.int32
    assert ((pe.se3_first >= 0) & (pe.se3_first < pb.n_cams) & (pe.se3_second >= 0) & (pe.se3_second < pb.n_cams)).all()
    assert (pe.se3_first != pe.se3_second).all() and ((pe.gps_frame >= 0) & (pe.gps_frame < pb.n_cams)).all()
    for m in (pe.se3_meas, pe.gps_meas):
        assert np.isfinite(m).all() and (np.sum(m[:, :4] ** 2, axis=1) > 1e-12).all()


# ---- inputs of the SE3 logarithm's branches (tests/test_oracle_posegraph.py, tests/golden/make_golden_reference.py) ----------------
def se3_log_edge_inputs() -> np.ndarray:
    """(n, 7) poses at the logarithm's branch points, each with translation 0 and a random one: exactly the identity (+-q), angles
    1e-14 and 1e-11 (n < 1e-10), exactly pi (w = +0 and -0), w = +-5e-11 (inside the |w| < 1e-10 branch) and +-2e-10 (just
    outside), pi - 1e-6, and -q of 0.5, 1 and 3 rad (w < 0 for a small rotation).  Quaternions with a unit axis and an exact w."""
    rng = np.random.default_rng(77)
    quats = [np.array([0.0, 0.0, 0.0, 1.0]), np.array([0.0, 0.0, 0.0, -1.0])]
    for w in (0.0, -0.0, 5e-11, -5e-11, 2e-10, -2e-10):
        quats.append(np.concatenate([_unit(rng.standard_normal(3)), [w]]))
    for th in (1e-14, 1e-11, math.pi - 1e-6):
        quats.append(_residual_quat(th, _unit(rng.standard_normal(3))))
    for th in (0.5, 1.0, 3.0):
        quats.append(-_residual_quat(th, _unit(rng.standard_normal(3))))
    out = []
    for q in quats:
        out.append(np.concatenate([q, np.zeros(3)]))
        out.append(np.concatenate([q, rng.uniform(-10, 10, 3)]))
    return np.ascontiguousarray(out)
