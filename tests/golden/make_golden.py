"""Regenerates the committed golden fixtures in tests/golden/ (oracle/_ref parts need GSLAM_REFERENCE at build time).

  python tests/golden/make_golden.py [hamming] [ba] [orb]

* hamming_golden.npz : seeded descriptor sets (with engineered duplicates / ties) + cv2.BFMatcher(NORM_HAMMING)
                       match / knnMatch(k=2) results + the reference's own hamming32 (oracle/_ref) on sampled pairs.
* ba_golden.npz      : BASELINE config 1 (10 cams / 200 points, all visible) + the optimum found by
                       scipy.optimize.least_squares on the same residual (independent algorithm).
* orb_*.npz          : cv2.ORB_create(...).detectAndCompute on synthetic frames (keypoints + descriptors), plus the
                       per-stage cv2 outputs the oracle is pinned against.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from gslam_b200 import synth  # noqa: E402


def make_hamming():
    import cv2
    import oracle
    q = synth.random_descriptors(300, seed=11)
    t = synth.random_descriptors(257, seed=12)
    # engineered ties: duplicate train rows, a query equal to a train row, near-duplicates differing in one bit
    t[100] = t[7]; t[200] = t[7]; t[50] = t[49]
    q[0] = t[7]; q[1] = t[49]; q[2] = t[256]
    q[3] = t[7]; q[3, 0] ^= 1
    t[10] = 0; t[11] = 255; q[4] = 0; q[5] = 255
    bf = cv2.BFMatcher(cv2.NORM_HAMMING)
    m = bf.match(q, t)
    assert [x.queryIdx for x in m] == list(range(q.shape[0]))
    idx = np.array([x.trainIdx for x in m], np.int32)
    d1 = np.array([int(x.distance) for x in m], np.int32)
    knn = bf.knnMatch(q, t, k=2)
    idx_knn = np.array([k[0].trainIdx for k in knn], np.int32)
    d2 = np.array([int(k[1].distance) for k in knn], np.int32)
    idx2 = np.array([k[1].trainIdx for k in knn], np.int32)
    out = dict(q=q, t=t, idx=idx, d1=d1, d2=d2, idx_knn=idx_knn, idx2=idx2)
    if oracle.have_ref():
        pairs = np.stack([np.arange(300) % 300, (np.arange(300) * 7) % 257], axis=1).astype(np.int32)
        ref = np.array([oracle.ref().ref_hamming32(q[a].ctypes.data, t[b].ctypes.data) for a, b in pairs], np.float32)
        out.update(ref_pairs=pairs, ref_hamming32=ref)
    np.savez_compressed(os.path.join(HERE, "hamming_golden.npz"), **out)
    print("hamming_golden.npz", {k: v.shape for k, v in out.items()})


def ba_residuals(x, pb, delta=None):
    """Plain numpy residual of the BA path (SURVEY.md App. B) in the parameterisation x = [rotvec,t]_cw per free cam + points."""
    from scipy.spatial.transform import Rotation as R
    nc, npnt = pb.n_cams, pb.n_points
    free = np.flatnonzero(pb.cam_dof != 0)
    Rcw = np.empty((nc, 3, 3)); tcw = np.empty((nc, 3))
    q = pb.cam_pose_wc[:, :4]; t = pb.cam_pose_wc[:, 4:]
    Rwc = R.from_quat(q).as_matrix()
    Rcw[:] = np.transpose(Rwc, (0, 2, 1)); tcw[:] = -np.einsum("nij,nj->ni", Rcw, t)
    xc = x[:6 * free.size].reshape(-1, 6)
    Rcw[free] = R.from_rotvec(xc[:, :3]).as_matrix(); tcw[free] = xc[:, 3:]
    P = x[6 * free.size:].reshape(npnt, 3)
    pc = np.einsum("nij,nj->ni", Rcw[pb.obs_cam], P[pb.obs_point]) + tcw[pb.obs_cam]
    r = pc[:, :2] / pc[:, 2:3] - pb.obs_xyz[:, :2] / pb.obs_xyz[:, 2:3]
    return r.reshape(-1)


def make_ba():
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation as R
    pb = synth.synth_ba(10, 200, all_visible=True, n_fixed=2, seed=42)
    free = np.flatnonzero(pb.cam_dof != 0)
    Rwc = R.from_quat(pb.cam_pose_wc[:, :4]).as_matrix()
    Rcw = np.transpose(Rwc, (0, 2, 1)); tcw = -np.einsum("nij,nj->ni", Rcw, pb.cam_pose_wc[:, 4:])
    x0 = np.concatenate([np.concatenate([R.from_matrix(Rcw[free]).as_rotvec(), tcw[free]], axis=1).reshape(-1), pb.points.reshape(-1)])
    # Huber in scipy: rho(z) with z = (r/f_scale)^2 per scalar residual — not the 2-D norm Huber of the path, so compare
    # on the NON-robust problem (huber disabled on both sides): delta = 0.
    sol = least_squares(ba_residuals, x0, args=(pb,), method="trf", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=200)
    cost = 0.5 * float(np.sum(sol.fun ** 2))
    out = dict(cam_pose_wc=pb.cam_pose_wc, cam_dof=pb.cam_dof, points=pb.points, point_free=pb.point_free,
               obs_cam=pb.obs_cam, obs_point=pb.obs_point, obs_xyz=pb.obs_xyz, scipy_cost_nohuber=np.array(cost),
               scipy_x=sol.x)
    np.savez_compressed(os.path.join(HERE, "ba_golden.npz"), **out)
    print("ba_golden.npz scipy optimum cost (no huber):", cost, "nfev", sol.nfev)


if __name__ == "__main__":
    what = sys.argv[1:] or ["hamming", "ba", "orb"]
    if "hamming" in what:
        make_hamming()
    if "ba" in what:
        make_ba()
    if "orb" in what:
        from make_golden_orb import make_orb  # noqa
        make_orb()
