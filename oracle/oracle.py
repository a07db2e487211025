"""ctypes bindings of oracle/liboracle.so (our C restatements) and oracle/_ref/libgslam_ref.so (the unmodified
reference headers behind an extern "C" shim).  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# a checkout of the GSLAM sources (GSLAM_REFERENCE, else the default location below): the reference checkers and the GSLAM plugins
# compile against its headers into _ref/, which is built where the checkout is and used as built everywhere else
REFERENCE = os.environ.get("GSLAM_REFERENCE") or "/root/reference"
# the GSLAM-facing plugins (gslam_b200/plugin) and the host program that drives them through the reference API
PLUGIN_DIR = os.path.join(_HERE, "_ref", "plugins")
KERNEL_LIB = os.path.join(os.path.dirname(_HERE), "gslam_b200", "lib", "libgslam_b200_kernels.so")
_LIB = None
_REF = None

u8p = C.POINTER(C.c_uint8)
i32p = C.POINTER(C.c_int32)
f64p = C.POINTER(C.c_double)


class BaProblemC(C.Structure):
    _fields_ = [("n_cams", C.c_int32), ("n_points", C.c_int32), ("n_obs", C.c_int32),
                ("cam_pose_wc", f64p), ("cam_dof", u8p), ("points", f64p), ("point_free", u8p),
                ("obs_cam", i32p), ("obs_point", i32p), ("obs_xyz", f64p), ("obs_info", f64p)]


class PoseEdgesC(C.Structure):
    _fields_ = [("n_se3", C.c_int32), ("se3_first", i32p), ("se3_second", i32p), ("se3_meas", f64p), ("se3_info", f64p),
                ("n_gps", C.c_int32), ("gps_frame", i32p), ("gps_meas", f64p), ("gps_info", f64p)]


class BaOptionsC(C.Structure):
    _fields_ = [("projection", C.c_int32), ("huber_delta", C.c_double), ("max_iterations", C.c_int32),
                ("verbose", C.c_int32), ("function_tolerance", C.c_double), ("lambda_init", C.c_double),
                ("pcg_max_iters", C.c_int32), ("pcg_tol", C.c_double), ("linear_solver", C.c_int32)]


class BaResultC(C.Structure):
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double), ("iterations", C.c_int32),
                ("accepted", C.c_int32), ("pcg_iterations", C.c_int32), ("status", C.c_int32),
                ("lambda_final", C.c_double), ("gpu_ms", C.c_float)]


class KeyPointC(C.Structure):
    _fields_ = [("x", C.c_float), ("y", C.c_float), ("size", C.c_float), ("angle", C.c_float),
                ("response", C.c_float), ("octave", C.c_int32), ("class_id", C.c_int32)]


KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"), ("response", "<f4"),
                     ("octave", "<i4"), ("class_id", "<i4")])


class OrbCfgC(C.Structure):
    _fields_ = [("nfeatures", C.c_int32), ("scale_factor", C.c_float), ("nlevels", C.c_int32),
                ("edge_threshold", C.c_int32), ("first_level", C.c_int32), ("wta_k", C.c_int32),
                ("score_type", C.c_int32), ("patch_size", C.c_int32), ("fast_threshold", C.c_int32)]


def default_ba_options(**kw) -> BaOptionsC:
    o = BaOptionsC(0, 0.01, 500, 0, 1e-6, 1e-4, 50, 1e-10, 0)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def default_orb_cfg(**kw) -> OrbCfgC:
    o = OrbCfgC(500, 1.2, 8, 31, 0, 2, 0, 31, 20)
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def build(force: bool = False) -> None:
    """Compile liboracle.so (always possible) and, where a GSLAM checkout is found (REFERENCE), _ref/libgslam_ref.so and the plugins
    in _ref/plugins (these link against the CUDA library, so they are built once it is)."""
    srcs = [os.path.join(_HERE, f) for f in ("hamming_ref.c", "ba_ref.c", "orb_ref.c", "pnp_ref.c", "bow_ref.c", "Makefile")]
    lib = os.path.join(_HERE, "liboracle.so")
    if force or not os.path.exists(lib) or any(os.path.getmtime(s) > os.path.getmtime(lib) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s", "liboracle.so", "CC=gcc"])
    ref = os.path.join(_HERE, "_ref", "libgslam_ref.so")
    if not os.path.isdir(os.path.join(REFERENCE, "GSLAM", "core")):
        return
    if force or not os.path.exists(ref) or os.path.getmtime(os.path.join(_HERE, "ref_shim.cpp")) > os.path.getmtime(ref):
        subprocess.check_call(["make", "-C", _HERE, "-s", "ref", "CXX=g++", f"REF={REFERENCE}"])
    if os.path.exists(KERNEL_LIB):
        subprocess.check_call(["make", "-C", _HERE, "-s", "plugins", "CXX=g++", f"REF={REFERENCE}"])


def digest(a) -> str:
    """SHA-256 of an array's dtype, shape and bytes: stored golden outputs compared exactly without storing them whole."""
    import hashlib
    a = np.ascontiguousarray(a)
    return hashlib.sha256(f"{a.dtype.str}{a.shape}".encode() + a.tobytes()).hexdigest()[:32]


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        build()
        L = C.CDLL(os.path.join(_HERE, "liboracle.so"))
        L.orc_hamming256.restype = C.c_int
        L.orc_hamming256.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_match_hamming.restype = None
        L.orc_match_hamming.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_remap_apply.restype = None
        L.orc_remap_apply.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_match_stereo.restype = None
        L.orc_match_stereo.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float,
                                       C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_ba_solve.restype = C.c_int
        L.orc_ba_solve.argtypes = [C.POINTER(BaProblemC), C.POINTER(BaOptionsC), C.POINTER(BaResultC)]
        L.orc_ba_linearize.restype = C.c_int
        L.orc_ba_linearize.argtypes = [C.POINTER(BaProblemC), C.c_double] + [C.c_void_p] * 6
        L.orc_ba_cost.restype = C.c_int
        L.orc_ba_cost.argtypes = [C.POINTER(BaProblemC), C.c_double, f64p]
        L.orc_ba_reduced_system.restype = C.c_int
        L.orc_ba_reduced_system.argtypes = [C.POINTER(BaProblemC), C.c_double, C.c_double, C.c_int, C.c_double,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
        L.orc_ba_solve_ex.restype = C.c_int
        L.orc_ba_solve_ex.argtypes = [C.POINTER(BaProblemC), C.POINTER(PoseEdgesC), C.POINTER(BaOptionsC), C.POINTER(BaResultC)]
        L.orc_ba_linearize_ex.restype = C.c_int
        L.orc_ba_linearize_ex.argtypes = [C.POINTER(BaProblemC), C.POINTER(PoseEdgesC), C.c_double] + [C.c_void_p] * 6
        L.orc_ba_cost_ex.restype = C.c_int
        L.orc_ba_cost_ex.argtypes = [C.POINTER(BaProblemC), C.POINTER(PoseEdgesC), C.c_double, f64p]
        L.orc_ba_reduced_system_ex.restype = C.c_int
        L.orc_ba_reduced_system_ex.argtypes = [C.POINTER(BaProblemC), C.POINTER(PoseEdgesC), C.c_double, C.c_double, C.c_int, C.c_double,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
        L.orc_ba_set_threads.restype = None
        L.orc_ba_set_threads.argtypes = [C.c_int]
        L.orc_se3_log.restype = None
        L.orc_se3_log.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_se3_mul.restype = None
        L.orc_se3_mul.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_ba_pnp.restype = C.c_int
        L.orc_ba_pnp.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                 C.POINTER(BaOptionsC), C.POINTER(BaResultC)]
        L.orc_bow_transform.restype = C.c_int
        L.orc_bow_transform.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.c_void_p]
        L.orc_se3_inverse.restype = None
        L.orc_se3_inverse.argtypes = [C.c_void_p, C.c_void_p]
        L.orc_se3_retract.restype = None
        L.orc_se3_retract.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


def have_ref() -> bool:
    return os.path.exists(os.path.join(_HERE, "_ref", "libgslam_ref.so"))


def ref() -> C.CDLL:
    global _REF
    if _REF is None:
        build()
        R = C.CDLL(os.path.join(_HERE, "_ref", "libgslam_ref.so"))
        R.ref_hamming32.restype = C.c_float
        R.ref_hamming32.argtypes = [C.c_void_p, C.c_void_p]
        for name in ("ref_se3_inverse", "ref_se3_exp", "ref_se3_log"):
            getattr(R, name).restype = None
            getattr(R, name).argtypes = [C.c_void_p, C.c_void_p]
        for name in ("ref_se3_transform", "ref_se3_mul"):
            getattr(R, name).restype = None
            getattr(R, name).argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        R.ref_sim3_raw.restype = None
        R.ref_sim3_raw.argtypes = [C.c_void_p, C.c_double, C.c_void_p]
        R.ref_undistort.restype = C.c_int
        R.ref_undistort.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        R.ref_voc_train.restype = C.c_void_p
        R.ref_voc_train.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        R.ref_voc_from_arrays.restype = C.c_void_p
        R.ref_voc_from_arrays.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint, C.c_void_p, C.c_void_p, C.c_void_p]
        R.ref_voc_destroy.restype = None
        R.ref_voc_destroy.argtypes = [C.c_void_p]
        R.ref_voc_info.restype = C.c_int
        R.ref_voc_info.argtypes = [C.c_void_p] + [C.POINTER(C.c_int)] * 4
        R.ref_voc_export.restype = None
        R.ref_voc_export.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        R.ref_voc_transform.restype = C.c_int
        R.ref_voc_transform.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.c_void_p,
                                        C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_double)]
        R.ref_voc_transform_one.restype = None
        R.ref_voc_transform_one.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        R.ref_sizeof.restype = C.c_int
        R.ref_sizeof.argtypes = [C.c_char_p]
        R.ref_keypoint_offsets.restype = C.c_int
        R.ref_keypoint_offsets.argtypes = [C.c_void_p]
        _REF = R
    return _REF


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def match_stereo(kps_left, desc_left, kps_right, desc_right, band=2.0, min_disp=0.0, max_disp=1e9):
    kl = np.ascontiguousarray(kps_left, KP_DTYPE); kr = np.ascontiguousarray(kps_right, KP_DTYPE)
    dl = np.ascontiguousarray(desc_left, np.uint8).reshape(-1, 32); dr = np.ascontiguousarray(desc_right, np.uint8).reshape(-1, 32)
    nl, nr = dl.shape[0], dr.shape[0]
    idx = np.empty(nl, np.int32); d1 = np.empty(nl, np.int32); d2 = np.empty(nl, np.int32)
    lib().orc_match_stereo(_p(kl), _p(dl), nl, _p(kr), _p(dr), nr, band, min_disp, max_disp, _p(idx), _p(d1), _p(d2))
    return idx, d1, d2


def remap_apply(img: np.ndarray, idx4, coef4, remap_x, out_shape) -> np.ndarray:
    """The bilinear LUT remap (orc_remap_apply): img (H,W) or (H,W,3) uint8 -> out_shape (+channels)."""
    img = np.ascontiguousarray(img, np.uint8)
    ch = 1 if img.ndim == 2 else img.shape[2]
    n_in = img.shape[0] * img.shape[1]; n_out = out_shape[0] * out_shape[1]
    idx4 = np.ascontiguousarray(idx4, np.int32); coef4 = np.ascontiguousarray(coef4, np.float32); rx = np.ascontiguousarray(remap_x, np.float32)
    out = np.zeros(tuple(out_shape) + ((ch,) if img.ndim == 3 else ()), np.uint8)
    lib().orc_remap_apply(n_in, n_out, ch, _p(idx4), _p(coef4), _p(rx), _p(img), _p(out))
    return out


def ref_undistort(cam_in, cam_out, img=None):
    """The UNMODIFIED reference (oracle/_ref): remap tables of UndistorterImpl::prepareReMap and, with an image, Undistorter::undistort.
    cam_*: GSLAM camera parameter vectors [w, h, fx, fy, cx, cy(, ...)].  -> (idx4, coef4, remap_x, out or None)"""
    ci = np.ascontiguousarray(cam_in, np.float64); co = np.ascontiguousarray(cam_out, np.float64)
    wo, ho = int(co[0]), int(co[1])
    idx4 = np.zeros((ho * wo, 4), np.int32); coef4 = np.zeros((ho * wo, 4), np.float32); rx = np.zeros(ho * wo, np.float32)
    out = None
    ch = 1
    if img is not None:
        img = np.ascontiguousarray(img, np.uint8)
        ch = 1 if img.ndim == 2 else img.shape[2]
        out = np.zeros((ho, wo) + ((ch,) if img.ndim == 3 else ()), np.uint8)
    rc = ref().ref_undistort(_p(ci), ci.size, _p(co), co.size, _p(img), ch, _p(idx4), _p(coef4), _p(rx), _p(out))
    if rc != 0:
        raise RuntimeError(f"ref_undistort failed rc={rc}")
    return idx4, coef4, rx, out


def to_gray(img: np.ndarray, rgb: bool = False) -> np.ndarray:
    """Colour (H, W, 3|4) uint8 -> gray uint8 as cv2.cvtColor(..., COLOR_BGR[A]2GRAY / COLOR_RGB[A]2GRAY) computes it for 8-bit
    images (cv2 4.13: 15-bit fixed point, B 3735 / G 19235 / R 9798, round to nearest) -- pinned against cv2 in
    tests/test_oracle_orb.py::test_gray_conversion_equals_cv2.  The frames GSLAM's dataset plugins deliver are 8UC3 / 8UC4
    (GSLAM/plugins/datasets/IO.h:86-110)."""
    a = np.asarray(img, np.uint8)
    c0, c1, c2 = (a[..., i].astype(np.int64) for i in range(3))
    b, r = (c2, c0) if rgb else (c0, c2)
    return ((b * 3735 + c1 * 19235 + r * 9798 + (1 << 14)) >> 15).astype(np.uint8)


# ---- Hamming -----------------------------------------------------------------------------------------------------
def match_hamming(query: np.ndarray, train: np.ndarray):
    q = np.ascontiguousarray(query, dtype=np.uint8).reshape(-1, 32)
    t = np.ascontiguousarray(train, dtype=np.uint8).reshape(-1, 32)
    nq, nt = q.shape[0], t.shape[0]
    idx = np.empty(nq, np.int32); d1 = np.empty(nq, np.int32); d2 = np.empty(nq, np.int32)
    lib().orc_match_hamming(_p(q), nq, _p(t), nt, _p(idx), _p(d1), _p(d2))
    return idx, d1, d2


# ---- BA ------------------------------------------------------------------------------------------------------------
def ba_problem_c(pb) -> tuple[BaProblemC, list]:
    """pb: gslam_b200.synth.BAProblem (arrays are used in place; poses/points are IN/OUT)."""
    keep = []

    def arr(a, dt):
        if a is None:
            return None
        b = np.ascontiguousarray(a, dtype=dt)
        keep.append(b)
        return b
    pose = pb.cam_pose_wc; pts = pb.points
    assert pose.dtype == np.float64 and pose.flags.c_contiguous and pts.dtype == np.float64 and pts.flags.c_contiguous
    dof = arr(pb.cam_dof, np.uint8); pf = arr(pb.point_free, np.uint8)
    oc = arr(pb.obs_cam, np.int32); op = arr(pb.obs_point, np.int32); ox = arr(pb.obs_xyz, np.float64); oi = arr(pb.obs_info, np.float64)
    c = BaProblemC(pb.n_cams, pb.n_points, pb.n_obs, pose.ctypes.data_as(f64p),
                   None if dof is None else dof.ctypes.data_as(u8p), pts.ctypes.data_as(f64p),
                   None if pf is None else pf.ctypes.data_as(u8p), oc.ctypes.data_as(i32p), op.ctypes.data_as(i32p),
                   ox.ctypes.data_as(f64p), None if oi is None else oi.ctypes.data_as(f64p))
    return c, keep


def pose_edges_c(edges):
    """edges: an object with se3_first / se3_second / se3_meas / se3_info / gps_frame / gps_meas / gps_info (gslam_b200.synth.PoseEdges)
    or None -> (ctypes struct or None, keep-alive list)"""
    if edges is None:
        return None, []
    f = np.ascontiguousarray(edges.se3_first, np.int32); s_ = np.ascontiguousarray(edges.se3_second, np.int32)
    m = np.ascontiguousarray(edges.se3_meas, np.float64).reshape(-1, 7)
    si = None if edges.se3_info is None else np.ascontiguousarray(edges.se3_info, np.float64).reshape(-1, 36)
    gf = np.ascontiguousarray(edges.gps_frame, np.int32); gm = np.ascontiguousarray(edges.gps_meas, np.float64).reshape(-1, 7)
    gi = None if edges.gps_info is None else np.ascontiguousarray(edges.gps_info, np.float64).reshape(-1, 36)
    cast = lambda a, t: None if a is None else a.ctypes.data_as(t)
    c = PoseEdgesC(f.shape[0], cast(f, i32p), cast(s_, i32p), cast(m, f64p), cast(si, f64p), gf.shape[0], cast(gf, i32p), cast(gm, f64p), cast(gi, f64p))
    return c, [f, s_, m, si, gf, gm, gi]


def _pe(edges):
    c, keep = pose_edges_c(edges)
    return (C.byref(c) if c is not None else None), (c, keep)


def ba_set_threads(n: int) -> None:
    """OpenMP threads of the BA oracle's heavy loops (default 1 = the strictly sequential order the parity tests compare against)."""
    lib().orc_ba_set_threads(int(n))


def ba_solve(pb, edges=None, **opts):
    c, keep = ba_problem_c(pb)
    o = default_ba_options(**opts)
    r = BaResultC()
    e, keep2 = _pe(edges)
    rc = lib().orc_ba_solve_ex(C.byref(c), e, C.byref(o), C.byref(r))
    if rc != 0:
        raise RuntimeError(f"orc_ba_solve failed rc={rc}")
    return r


def ba_linearize(pb, delta=0.01, edges=None):
    c, keep = ba_problem_c(pb)
    U = np.zeros((pb.n_cams, 6, 6)); gc = np.zeros((pb.n_cams, 6)); V = np.zeros((pb.n_points, 3, 3)); gp = np.zeros((pb.n_points, 3))
    W = np.zeros((pb.n_obs, 6, 3)); cost = np.zeros(1)
    e, keep2 = _pe(edges)
    rc = lib().orc_ba_linearize_ex(C.byref(c), e, delta, _p(U), _p(gc), _p(V), _p(gp), _p(W), _p(cost))
    assert rc == 0
    return dict(U=U, gc=gc, V=V, gp=gp, W=W, cost=float(cost[0]))


def ba_cost(pb, delta=0.01, edges=None) -> float:
    c, keep = ba_problem_c(pb)
    out = C.c_double()
    e, keep2 = _pe(edges)
    rc = lib().orc_ba_cost_ex(C.byref(c), e, delta, C.byref(out))
    assert rc == 0
    return out.value


def ba_reduced_system(pb, delta=0.01, lam=1e-4, pcg_max_iters=50, pcg_tol=1e-10, edges=None):
    c, keep = ba_problem_c(pb)
    n6 = 6 * pb.n_cams
    S = np.zeros((n6, n6)); gt = np.zeros(n6); dc = np.zeros(n6); it = C.c_int()
    e, keep2 = _pe(edges)
    rc = lib().orc_ba_reduced_system_ex(C.byref(c), e, delta, lam, pcg_max_iters, pcg_tol, _p(S), _p(gt), _p(dc), C.byref(it))
    assert rc == 0
    return S, gt, dc, it.value


def se3_log(pose7):
    p = np.ascontiguousarray(pose7, np.float64); out = np.zeros(6)
    lib().orc_se3_log(_p(p), _p(out))
    return out


def se3_mul(a7, b7):
    a = np.ascontiguousarray(a7, np.float64); b = np.ascontiguousarray(b7, np.float64); out = np.zeros(7)
    lib().orc_se3_mul(_p(a), _p(b), _p(out))
    return out


def ba_pnp(xyz, xy1, pose_wc, dof=63, want_info=False, **opts):
    xyz = np.ascontiguousarray(xyz, np.float64); xy1 = np.ascontiguousarray(xy1, np.float64)
    pose = np.ascontiguousarray(pose_wc, np.float64).copy()
    info = np.zeros((6, 6)) if want_info else None
    o = default_ba_options(**opts); r = BaResultC()
    rc = lib().orc_ba_pnp(xyz.shape[0], _p(xyz), _p(xy1), _p(pose), dof, _p(info), C.byref(o), C.byref(r))
    if rc != 0:
        raise RuntimeError(f"orc_ba_pnp failed rc={rc}")
    return pose, r, info


# ---- ORB -----------------------------------------------------------------------------------------------------------
_ORB_BOUND = False


def _orb():
    global _ORB_BOUND
    L = lib()
    if not _ORB_BOUND:
        L.orc_orb_scale.restype = C.c_float; L.orc_orb_scale.argtypes = [C.c_float, C.c_int]
        L.orc_orb_level_size.restype = None
        L.orc_orb_level_size.argtypes = [C.c_int, C.c_int, C.c_float, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.orc_resize_linear_exact.restype = None
        L.orc_resize_linear_exact.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
        L.orc_fast_score_map.restype = None
        L.orc_fast_score_map.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
        L.orc_fast_detect.restype = C.c_int
        L.orc_fast_detect.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.orc_harris_response.restype = C.c_float; L.orc_harris_response.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.orc_fast_atan2.restype = C.c_float; L.orc_fast_atan2.argtypes = [C.c_float, C.c_float]
        L.orc_ic_angle.restype = C.c_float; L.orc_ic_angle.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.orc_blur7.restype = None; L.orc_blur7.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.orc_blur_pixel.restype = C.c_uint8; L.orc_blur_pixel.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        L.orc_det_sincos.restype = None; L.orc_det_sincos.argtypes = [C.c_double, f64p, f64p]
        L.orc_brief_descriptor.restype = None
        L.orc_brief_descriptor.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]
        L.orc_orb_quotas.restype = None; L.orc_orb_quotas.argtypes = [C.c_int, C.c_float, C.c_int, C.c_void_p]
        L.orc_orb_pyramid_level.restype = C.c_void_p
        L.orc_orb_pyramid_level.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.orc_orb_extract.restype = C.c_int
        L.orc_orb_extract.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(OrbCfgC), C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
        _ORB_BOUND = True
    return L


def orb_level_size(w, h, level, scale_factor=1.2):
    lw, lh = C.c_int(), C.c_int()
    _orb().orc_orb_level_size(w, h, scale_factor, level, C.byref(lw), C.byref(lh))
    return lw.value, lh.value


def orb_quotas(nfeatures, nlevels=8, scale_factor=1.2):
    q = np.zeros(nlevels, np.int32)
    _orb().orc_orb_quotas(nfeatures, scale_factor, nlevels, _p(q))
    return q


def resize_linear_exact(img, dw, dh):
    img = np.ascontiguousarray(img, np.uint8)
    out = np.empty((dh, dw), np.uint8)
    _orb().orc_resize_linear_exact(_p(img), img.shape[1], img.shape[0], _p(out), dw, dh)
    return out


def orb_pyramid_level(img, level, scale_factor=1.2):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    cur = img
    for l in range(1, level + 1):
        lw, lh = orb_level_size(w, h, l, scale_factor)
        cur = resize_linear_exact(cur, lw, lh)
    return cur


def fast_detect(img, threshold=20, nms=True):
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    cap = 1 << 16
    while True:
        xs = np.empty(cap, np.int32); ys = np.empty(cap, np.int32); sc = np.empty(cap, np.int32)
        n = _orb().orc_fast_detect(_p(img), w, h, threshold, int(nms), _p(xs), _p(ys), _p(sc), cap)
        if n <= cap:
            return xs[:n].copy(), ys[:n].copy(), sc[:n].copy()
        cap = n


def fast_score_map(img, threshold=20):
    img = np.ascontiguousarray(img, np.uint8)
    out = np.empty_like(img)
    _orb().orc_fast_score_map(_p(img), img.shape[1], img.shape[0], threshold, _p(out))
    return out


def harris_response(img, x, y):
    img = np.ascontiguousarray(img, np.uint8)
    return float(_orb().orc_harris_response(_p(img), img.shape[1], int(x), int(y)))


def ic_angle(img, x, y):
    img = np.ascontiguousarray(img, np.uint8)
    return float(_orb().orc_ic_angle(_p(img), img.shape[1], int(x), int(y)))


def fast_atan2(y, x):
    return float(_orb().orc_fast_atan2(float(y), float(x)))


def blur7(img):
    img = np.ascontiguousarray(img, np.uint8)
    out = np.empty_like(img)
    _orb().orc_blur7(_p(img), img.shape[1], img.shape[0], _p(out))
    return out


def det_sincos(x):
    s, c = C.c_double(), C.c_double()
    _orb().orc_det_sincos(float(x), C.byref(s), C.byref(c))
    return s.value, c.value


def brief_descriptor(blurred, x, y, angle_deg):
    b = np.ascontiguousarray(blurred, np.uint8)
    d = np.zeros(32, np.uint8)
    _orb().orc_brief_descriptor(_p(b), b.shape[1], int(x), int(y), float(angle_deg), _p(d))
    return d


def orb_extract(img, nfeatures=500, **cfg_kw):
    """Full pipeline. Returns (keypoints[KP_DTYPE], descriptors (n,32) u8) in canonical (octave, y, x) order."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    cfg = default_orb_cfg(nfeatures=nfeatures, **cfg_kw)
    cap = 2 * nfeatures + 1024
    while True:
        kps = np.zeros(cap, KP_DTYPE); desc = np.zeros((cap, 32), np.uint8); n = C.c_int(cap)
        rc = _orb().orc_orb_extract(_p(img), w, h, C.byref(cfg), _p(kps), _p(desc), C.byref(n))
        if rc == 3 and n.value > cap:
            cap = n.value
            continue
        if rc != 0:
            raise RuntimeError(f"orc_orb_extract failed rc={rc}")
        return kps[:n.value].copy(), desc[:n.value].copy()


# ---- PnP (SURVEY.md §8f-1: Estimator::findPnP) -------------------------------------------------------------------------
class PnpStatsC(C.Structure):
    _fields_ = [("hypotheses", C.c_int), ("best_hypothesis", C.c_int), ("best_root", C.c_int), ("inliers_minimal", C.c_int),
                ("inliers_refined", C.c_int)]


def quartic_roots(coeffs):
    """Real roots of c[0] + c[1] x + ... + c[4] x^4 (orc_quartic_roots)."""
    c = np.ascontiguousarray(coeffs, np.float64); out = np.zeros(4)
    L = lib(); L.orc_quartic_roots.restype = C.c_int
    n = L.orc_quartic_roots(_p(c), _p(out))
    return out[:n]


def p3p(X, f):
    """X: 3x3 world points, f: 3x3 unit bearings -> list of (R, t) with x_cam = R X + t."""
    X = np.ascontiguousarray(X, np.float64); f = np.ascontiguousarray(f, np.float64); out = np.zeros(48)
    L = lib(); L.orc_p3p.restype = C.c_int
    n = L.orc_p3p(_p(X), _p(f), _p(out))
    return [(out[12 * k:12 * k + 9].reshape(3, 3).copy(), out[12 * k + 9:12 * k + 12].copy()) for k in range(n)]


def pnp_sample(seed, h, n):
    idx = (C.c_int * 3)()
    L = lib(); L.orc_pnp_sample.argtypes = [C.c_uint64, C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.orc_pnp_sample(seed, h, n, idx)
    return list(idx)


def pnp_ransac(xyz, xy, threshold=0.01, confidence=0.99, max_hypotheses=1024, seed=1):
    """-> (pose_cw[7] {qx,qy,qz,qw,tx,ty,tz}, mask[n] uint8, stats) or raises."""
    xyz = np.ascontiguousarray(xyz, np.float64); xy = np.ascontiguousarray(xy, np.float64)
    pose = np.zeros(7); mask = np.zeros(xyz.shape[0], np.uint8); st = PnpStatsC()
    L = lib()
    L.orc_pnp_ransac.restype = C.c_int
    L.orc_pnp_ransac.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p,
                                 C.POINTER(PnpStatsC)]
    rc = L.orc_pnp_ransac(xyz.shape[0], _p(xyz), _p(xy), threshold, confidence, max_hypotheses, seed, _p(pose), _p(mask), C.byref(st))
    if rc != 0:
        raise RuntimeError(f"orc_pnp_ransac failed rc={rc}")
    return pose, mask, st


# ---- bag-of-words transform (bow_ref.c restates GSLAM/core/Vocabulary.h:1558-1736; RefVocabulary IS the reference, oracle/_ref) -------
W_TF_IDF, W_TF, W_IDF, W_BINARY = 0, 1, 2, 3                                  # Vocabulary.h:88-94
S_L1, S_L2, S_CHI_SQUARE, S_KL, S_BHATTACHARYYA, S_DOT_PRODUCT = 0, 1, 2, 3, 4, 5  # Vocabulary.h:97-105


class VocabularyArrays:
    """The vocabulary tree as the flat arrays the reference keeps (Vocabulary.h:583-601): children of node p are rows
    p*k+1 .. p*k+child_num[p] of `desc`; the word id of a leaf is its node id."""

    def __init__(self, k, L, weighting, scoring, child_num, weight, desc):
        self.k, self.L, self.weighting, self.scoring = int(k), int(L), int(weighting), int(scoring)
        self.child_num = np.ascontiguousarray(child_num, np.uint32)
        self.weight = np.ascontiguousarray(weight, np.float32)
        self.desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        assert self.child_num.shape[0] == self.weight.shape[0] == self.desc.shape[0]

    @property
    def n_nodes(self):
        return int(self.child_num.shape[0])


def synth_vocabulary(k=10, L=4, seed=1, weighting=W_TF_IDF, scoring=S_L1, prune=0.0, stop=0.0) -> VocabularyArrays:
    """gslam_b200.synth.synth_vocabulary (the bench and the tests share one generator) as VocabularyArrays."""
    from gslam_b200 import synth
    v = synth.synth_vocabulary(k, L, seed, weighting, scoring, prune, stop)
    return VocabularyArrays(v.k, v.L, v.weighting, v.scoring, v.child_num, v.weight, v.desc)


def bow_transform(voc: VocabularyArrays, feats, levelsup=0):
    """-> dict(words int64[nw], values float32[nw], fv_node int64[m], fv_feat int32[m], f_word int64[n], f_node int64[n])"""
    f = np.ascontiguousarray(feats, np.uint8).reshape(-1, 32)
    n = f.shape[0]
    words = np.zeros(max(n, 1), np.int64); values = np.zeros(max(n, 1), np.float32)
    fvn = np.zeros(max(n, 1), np.int64); fvf = np.zeros(max(n, 1), np.int32)
    fw = np.zeros(max(n, 1), np.int64); fn = np.zeros(max(n, 1), np.int64)
    m = C.c_int(0)
    nw = lib().orc_bow_transform(voc.k, voc.L, voc.weighting, voc.scoring, _p(voc.child_num), _p(voc.weight), _p(voc.desc), _p(f), n, int(levelsup),
                                 _p(words), _p(values), _p(fvn), _p(fvf), C.byref(m), _p(fw), _p(fn))
    return dict(words=words[:nw], values=values[:nw], fv_node=fvn[:m.value], fv_feat=fvf[:m.value], f_word=fw[:n], f_node=fn[:n])


class RefVocabulary:
    """GSLAM::Vocabulary itself (oracle/_ref): trained by Vocabulary::create or loaded from arrays by Vocabulary::load."""

    def __init__(self, handle):
        if not handle:
            raise RuntimeError("reference vocabulary could not be created")
        self._h = C.c_void_p(handle)

    @classmethod
    def train(cls, descriptors, n_images, k, L, weighting=W_TF_IDF, scoring=S_L1):
        d = np.ascontiguousarray(descriptors, np.uint8).reshape(n_images, -1, 32)
        return cls(ref().ref_voc_train(_p(d), n_images, d.shape[1], k, L, weighting, scoring))

    @classmethod
    def from_arrays(cls, v: VocabularyArrays):
        return cls(ref().ref_voc_from_arrays(v.k, v.L, v.weighting, v.scoring, v.n_nodes, _p(v.child_num), _p(v.weight), _p(v.desc)))

    def arrays(self) -> VocabularyArrays:
        k, L, w, s = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        n = ref().ref_voc_info(self._h, C.byref(k), C.byref(L), C.byref(w), C.byref(s))
        child = np.zeros(n, np.uint32); weight = np.zeros(n, np.float32); desc = np.zeros((n, 32), np.uint8)
        ref().ref_voc_export(self._h, _p(child), _p(weight), _p(desc))
        return VocabularyArrays(k.value, L.value, w.value, s.value, child, weight, desc)

    def transform(self, feats, levelsup=0, repeat=1):
        f = np.ascontiguousarray(feats, np.uint8).reshape(-1, 32)
        n = f.shape[0]
        words = np.zeros(max(n, 1), np.uint64); values = np.zeros(max(n, 1), np.float32)
        fvn = np.zeros(max(n, 1), np.uint64); fvf = np.zeros(max(n, 1), np.uint32)
        nw, m, sec = C.c_int(0), C.c_int(0), C.c_double(0)
        ref().ref_voc_transform(self._h, _p(f), n, int(levelsup), _p(words), _p(values), C.byref(nw), _p(fvn), _p(fvf), C.byref(m), int(repeat),
                                C.byref(sec))
        return dict(words=words[:nw.value].astype(np.int64), values=values[:nw.value], fv_node=fvn[:m.value].astype(np.int64),
                    fv_feat=fvf[:m.value].astype(np.int32), seconds=sec.value)

    def transform_one(self, feat, levelsup=0):
        f = np.ascontiguousarray(feat, np.uint8).reshape(32)
        w, n, val = C.c_ulonglong(0), C.c_ulonglong(0), C.c_float(0)
        ref().ref_voc_transform_one(self._h, _p(f), int(levelsup), C.byref(w), C.byref(val), C.byref(n))
        return int(w.value), float(val.value), int(n.value)

    def close(self):
        if self._h:
            ref().ref_voc_destroy(self._h)
            self._h = None
