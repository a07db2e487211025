"""Host-side Python mirror of the reference-facing interface, one thin layer above the C-ABI.

Names and argument meaning follow the reference (the production host side is the C++ plugins under plugin/):
  Context.orb_extract(img, nfeatures)   ~ the Svar module function gslam.b200.orb_extract(GImage, cfg)
  Context.match_hamming(q, t)           ~ gslam.b200.match_hamming(GImage q, GImage t)
  Optimizer.optimize(graph)             ~ GSLAM::Optimizer::optimize(BundleGraph&)        Optimizer.h:229
  Optimizer.optimizePnP(matches, pose)  ~ GSLAM::Optimizer::optimizePnP(...)              Optimizer.h:202-207
Errors: like the reference plugins, `Optimizer` methods return bool and never raise across the boundary
(Optimizer.h:193-232); the lower-level Context methods raise GbError.
"""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np

from . import capi
from .capi import GbError, KP_DTYPE, ptr
from .synth import BAProblem


@dataclasses.dataclass
class OptimzeConfig:  # spelling follows GSLAM::OptimzeConfig (Optimizer.h:174-182)
    cameraProjectionType: int = 0            # PROJECTION_PINHOLE
    projectErrorHuberThreshold: float = 0.01
    maxIterations: int = 500
    verbose: bool = False
    # solver knobs the reference leaves to its backend
    functionTolerance: float = 1e-6
    lambdaInit: float = 1e-4
    pcgMaxIterations: int = 50
    pcgTolerance: float = 1e-10
    linearSolver: int = 0                    # 0 = block-Jacobi PCG, 1 = direct (block-skyline Cholesky; local-BA sizes)

    def to_c(self) -> capi.BaOptions:
        return capi.BaOptions(self.cameraProjectionType, self.projectErrorHuberThreshold, self.maxIterations,
                              int(self.verbose), self.functionTolerance, self.lambdaInit, self.pcgMaxIterations,
                              self.pcgTolerance, self.linearSolver)


def _edges_c(edges):
    """gslam_b200.synth.PoseEdges -> (capi.PoseEdges or None, keep-alive list)"""
    if edges is None:
        return None, []
    f = np.ascontiguousarray(edges.se3_first, np.int32); s_ = np.ascontiguousarray(edges.se3_second, np.int32)
    m = np.ascontiguousarray(edges.se3_meas, np.float64).reshape(-1, 7)
    si = None if edges.se3_info is None else np.ascontiguousarray(edges.se3_info, np.float64).reshape(-1, 36)
    gf = np.ascontiguousarray(edges.gps_frame, np.int32); gm = np.ascontiguousarray(edges.gps_meas, np.float64).reshape(-1, 7)
    gi = None if edges.gps_info is None else np.ascontiguousarray(edges.gps_info, np.float64).reshape(-1, 36)
    cast = lambda a, t: None if a is None else a.ctypes.data_as(t)
    c = capi.PoseEdges(f.shape[0], cast(f, capi.i32p), cast(s_, capi.i32p), cast(m, capi.f64p), cast(si, capi.f64p), gf.shape[0], cast(gf, capi.i32p),
                       cast(gm, capi.f64p), cast(gi, capi.f64p))
    return c, [f, s_, m, si, gf, gm, gi]


def _problem_c(pb: BAProblem):
    keep = []

    def arr(a, dt):
        if a is None:
            return None
        b = np.ascontiguousarray(a, dtype=dt)
        keep.append(b)
        return b
    assert pb.cam_pose_wc.dtype == np.float64 and pb.cam_pose_wc.flags.c_contiguous
    assert pb.points.dtype == np.float64 and pb.points.flags.c_contiguous
    dof = arr(pb.cam_dof, np.uint8); pf = arr(pb.point_free, np.uint8)
    oc = arr(pb.obs_cam, np.int32); op = arr(pb.obs_point, np.int32)
    ox = arr(pb.obs_xyz, np.float64); oi = arr(pb.obs_info, np.float64)

    def p(a, t):
        return None if a is None else a.ctypes.data_as(t)
    c = capi.BaProblem(pb.n_cams, pb.n_points, pb.n_obs, p(pb.cam_pose_wc, capi.f64p), p(dof, capi.u8p),
                       p(pb.points, capi.f64p), p(pf, capi.u8p), p(oc, capi.i32p), p(op, capi.i32p), p(ox, capi.f64p),
                       p(oi, capi.f64p))
    return c, keep


class Context:
    """One device + one stream (gb_ctx)."""

    def __init__(self, device: int = 0, high_priority: bool = False):
        self._lib = capi.lib()
        h = C.c_void_p()
        rc = self._lib.gb_ctx_create_priority(device, 1 if high_priority else 0, C.byref(h))
        if rc != capi.GB_OK:
            raise GbError(rc, self._lib.gb_last_error(None).decode())
        self._h = h
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            self._lib.gb_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != capi.GB_OK:
            raise GbError(rc, self._lib.gb_last_error(self._h).decode())

    @property
    def handle(self):
        return self._h

    def sync(self):
        self._check(self._lib.gb_ctx_sync(self._h))

    def wait_for(self, producer: "Context"):
        """Order this ctx's stream after everything enqueued so far on `producer`'s stream (no host sync)."""
        self._check(self._lib.gb_ctx_wait_for(self._h, producer._h))

    def popc_peak(self) -> float:
        """Measured POPC throughput of the device (popc32 per second): the matcher's roofline denominator."""
        v = C.c_double()
        self._check(self._lib.gb_dbg_popc_peak(self._h, C.byref(v)))
        return float(v.value)

    def stream(self) -> int:
        return int(self._lib.gb_ctx_stream(self._h) or 0)

    def timer_begin(self):
        self._check(self._lib.gb_timer_begin(self._h))

    def timer_end(self) -> float:
        ms = C.c_float()
        self._check(self._lib.gb_timer_end(self._h, C.byref(ms)))
        return float(ms.value)

    def launch_count(self) -> int:
        return int(self._lib.gb_launch_count(self._h))

    # ---- ORB ---------------------------------------------------------------------------------------------------------
    def orb_cfg(self, **kw) -> capi.OrbCfg:
        cfg = capi.OrbCfg()
        self._lib.gb_orb_cfg_default(C.byref(cfg))
        for k, v in kw.items():
            setattr(cfg, k, v)
        return cfg

    def orb_extract(self, img: np.ndarray, nfeatures: int = 500, capacity: int | None = None, **cfg_kw):
        """img: (H, W) uint8 gray, or (H, W, 3|4) colour (B,G,R[,A] unless rgb=True).  Returns (keypoints[KP_DTYPE], descriptors
        (n,32) uint8) in canonical (octave,y,x) order."""
        rgb = bool(cfg_kw.pop("rgb", False))
        img = np.ascontiguousarray(img, dtype=np.uint8)
        h, w = img.shape[:2]
        ch = 1 if img.ndim == 2 else img.shape[2]
        cfg = self.orb_cfg(nfeatures=nfeatures, **cfg_kw)
        cap = capacity or (2 * nfeatures + 256)
        while True:
            kps = np.zeros(cap, dtype=KP_DTYPE)
            desc = np.zeros((cap, 32), dtype=np.uint8)
            n = C.c_int(cap)
            rc = self._lib.gb_orb_extract_image(self._h, ptr(img), w, h, ch, 1 if rgb else 0, C.byref(cfg), ptr(kps), ptr(desc), C.byref(n))
            if rc == capi.GB_ERR_CAPACITY and capacity is None and n.value > cap:
                cap = n.value
                continue
            self._check(rc)
            return kps[:n.value].copy(), desc[:n.value].copy()

    # ---- match -------------------------------------------------------------------------------------------------------
    def match_hamming(self, query: np.ndarray, train: np.ndarray):
        """Returns (best_idx, best_dist, second_dist) int32 arrays, cv::BFMatcher(NORM_HAMMING) tie rules."""
        q = np.ascontiguousarray(query, dtype=np.uint8).reshape(-1, 32)
        t = np.ascontiguousarray(train, dtype=np.uint8).reshape(-1, 32)
        nq, nt = q.shape[0], t.shape[0]
        idx = np.empty(nq, np.int32); d1 = np.empty(nq, np.int32); d2 = np.empty(nq, np.int32)
        self._check(self._lib.gb_match_hamming(self._h, ptr(q), nq, ptr(t), nt, ptr(idx), ptr(d1), ptr(d2)))
        return idx, d1, d2

    def match_stereo(self, kps_left, desc_left, kps_right, desc_right, band=2.0, min_disp=0.0, max_disp=1e9):
        """Rectified-stereo row-band match (left = query): (best_idx, best_dist, second_dist); idx -1 when no candidate."""
        kl = np.ascontiguousarray(kps_left, KP_DTYPE); kr = np.ascontiguousarray(kps_right, KP_DTYPE)
        dl = np.ascontiguousarray(desc_left, np.uint8).reshape(-1, 32); dr = np.ascontiguousarray(desc_right, np.uint8).reshape(-1, 32)
        nl, nr = dl.shape[0], dr.shape[0]
        idx = np.empty(nl, np.int32); d1 = np.empty(nl, np.int32); d2 = np.empty(nl, np.int32)
        self._check(self._lib.gb_match_stereo(self._h, ptr(kl), ptr(dl), nl, ptr(kr), ptr(dr), nr, band, min_disp, max_disp,
                                              ptr(idx), ptr(d1), ptr(d2)))
        return idx, d1, d2

    # ---- BA ----------------------------------------------------------------------------------------------------------
    def pnp_ransac(self, xyz, xy, threshold=0.01, confidence=0.99, max_hypotheses=1024, seed=1):
        """Estimator::findPnP (P3P + RANSAC + refinement): -> (pose_cw[7] {qx,qy,qz,qw,tx,ty,tz}, mask[n] uint8, PnpStats)."""
        xyz = np.ascontiguousarray(xyz, np.float64); xy = np.ascontiguousarray(xy, np.float64)
        pose = np.zeros(7); mask = np.zeros(xyz.shape[0], np.uint8); st = capi.PnpStats()
        self._check(self._lib.gb_pnp_ransac(self._h, xyz.shape[0], ptr(xyz), ptr(xy), float(threshold), float(confidence),
                                            int(max_hypotheses), int(seed), ptr(pose), ptr(mask), C.byref(st)))
        return pose, mask, st

    def ba_solve(self, pb: BAProblem, cfg: OptimzeConfig | None = None) -> capi.BaResult:
        c, keep = _problem_c(pb)
        o = (cfg or OptimzeConfig()).to_c()
        r = capi.BaResult()
        self._check(self._lib.gb_ba_solve(self._h, C.byref(c), C.byref(o), C.byref(r)))
        return r

    def ba_solve_posegraph(self, pb: BAProblem, edges, cfg: OptimzeConfig | None = None) -> capi.BaResult:
        """Optimizer::optimize on a BundleGraph with SE3 / GPS edges (`edges`: gslam_b200.synth.PoseEdges)."""
        c, keep = _problem_c(pb)
        e, keep2 = _edges_c(edges)
        o = (cfg or OptimzeConfig()).to_c()
        r = capi.BaResult()
        self._check(self._lib.gb_ba_solve_posegraph(self._h, C.byref(c), C.byref(e) if e is not None else None, C.byref(o), C.byref(r)))
        return r

    def ba_pnp(self, xyz, xy1, pose_wc, dof: int = 63, want_info: bool = False, cfg: OptimzeConfig | None = None):
        xyz = np.ascontiguousarray(xyz, np.float64); xy1 = np.ascontiguousarray(xy1, np.float64)
        pose = np.ascontiguousarray(pose_wc, np.float64).copy()
        info = np.zeros((6, 6)) if want_info else None
        o = (cfg or OptimzeConfig()).to_c(); r = capi.BaResult()
        self._check(self._lib.gb_ba_pnp(self._h, xyz.shape[0], ptr(xyz), ptr(xy1), ptr(pose), dof, ptr(info),
                                        C.byref(o), C.byref(r)))
        return pose, r, info


class Remap:
    """A bilinear remap table resident in HBM (gb_remap): GSLAM::Undistorter::undistort on the device."""

    def __init__(self, ctx: Context, w_in, h_in, w_out, h_out, idx4, coef4, remap_x):
        self.ctx = ctx
        self.shape_in, self.shape_out = (h_in, w_in), (h_out, w_out)
        idx4 = np.ascontiguousarray(idx4, np.int32); coef4 = np.ascontiguousarray(coef4, np.float32); rx = np.ascontiguousarray(remap_x, np.float32)
        h = C.c_void_p()
        ctx._check(ctx._lib.gb_remap_create(ctx._h, w_in, h_in, w_out, h_out, ptr(idx4), ptr(coef4), ptr(rx), C.byref(h)))
        self._h = h

    def apply(self, img: np.ndarray) -> np.ndarray:
        img = np.ascontiguousarray(img, np.uint8)
        ch = 1 if img.ndim == 2 else img.shape[2]
        out = np.zeros(self.shape_out + ((ch,) if img.ndim == 3 else ()), np.uint8)
        self.ctx._check(self.ctx._lib.gb_remap_apply(self.ctx._h, self._h, ptr(img), ch, ptr(out)))
        return out

    def close(self):
        if getattr(self, "_h", None) and getattr(self.ctx, "_h", None):
            self.ctx._lib.gb_remap_destroy(self.ctx._h, self._h)
        self._h = None


class Vocabulary:
    """A GSLAM::Vocabulary tree resident in HBM (gb_vocabulary); method names follow the reference (Vocabulary.h:168-193)."""

    def __init__(self, ctx: Context, k, L, weighting, scoring, child_num, weight, desc):
        self.ctx = ctx
        child = np.ascontiguousarray(child_num, np.uint32); w = np.ascontiguousarray(weight, np.float32)
        d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        h = C.c_void_p()
        ctx._check(ctx._lib.gb_voc_create(ctx._h, int(k), int(L), int(weighting), int(scoring), child.shape[0], ptr(child), ptr(w), ptr(d), C.byref(h)))
        self._h = h

    def transform(self, features, levelsup: int = 0):
        """features: (N,32) uint8 host array, or a `Features` object resident in HBM.
        -> dict(words int64[nw], values float32[nw], fv_node int64[m], fv_feat int32[m]) in std::map order."""
        c = self.ctx
        if isinstance(features, Features):
            n = features.capacity
        else:
            features = np.ascontiguousarray(features, np.uint8).reshape(-1, 32)
            n = features.shape[0]
        words = np.zeros(max(n, 1), np.uint64); values = np.zeros(max(n, 1), np.float32)
        fvn = np.zeros(max(n, 1), np.uint64); fvf = np.zeros(max(n, 1), np.uint32)
        nw, m = C.c_int(0), C.c_int(0)
        if isinstance(features, Features):
            c._check(c._lib.gb_bow_transform_features(c._h, self._h, features._h, int(levelsup), ptr(words), ptr(values), C.byref(nw), ptr(fvn), ptr(fvf),
                                                      C.byref(m)))
        else:
            c._check(c._lib.gb_bow_transform(c._h, self._h, ptr(features), n, int(levelsup), ptr(words), ptr(values), C.byref(nw), ptr(fvn), ptr(fvf),
                                             C.byref(m)))
        return dict(words=words[:nw.value].astype(np.int64), values=values[:nw.value], fv_node=fvn[:m.value].astype(np.int64),
                    fv_feat=fvf[:m.value].astype(np.int32))

    def close(self):
        if getattr(self, "_h", None) and getattr(self.ctx, "_h", None):
            self.ctx._lib.gb_voc_destroy(self.ctx._h, self._h)
        self._h = None


class Features:
    """A frame's keypoints + descriptors resident in HBM (gb_features)."""

    def __init__(self, ctx: Context, capacity: int):
        self.ctx = ctx
        h = C.c_void_p()
        ctx._check(ctx._lib.gb_features_create(ctx._h, capacity, C.byref(h)))
        self._h = h
        self.capacity = capacity

    def close(self):
        if getattr(self, "_h", None) and getattr(self.ctx, "_h", None):
            self.ctx._lib.gb_features_destroy(self.ctx._h, self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def extract(self, img, width: int, height: int, cfg: capi.OrbCfg, device_ptr: bool = False, pitch: int | None = None):
        """img: numpy (H,W) uint8 host array, or an integer device pointer when device_ptr."""
        c = self.ctx
        if device_ptr:
            p = C.c_void_p(int(img))
        else:
            p = ptr(img)
        c._check(c._lib.gb_orb_extract_to(c._h, p, 1 if device_ptr else 0, width, height, pitch or width, C.byref(cfg), self._h))

    def count(self) -> int:
        n = C.c_int()
        self.ctx._check(self.ctx._lib.gb_features_count(self.ctx._h, self._h, C.byref(n)))
        return n.value

    def upload(self, desc: np.ndarray, kps: np.ndarray | None = None):
        d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        k = None if kps is None else np.ascontiguousarray(kps, KP_DTYPE)
        self.ctx._check(self.ctx._lib.gb_features_upload(self.ctx._h, self._h, ptr(k), ptr(d), d.shape[0]))

    def download(self):
        n = C.c_int(self.capacity)
        kps = np.zeros(self.capacity, KP_DTYPE); desc = np.zeros((self.capacity, 32), np.uint8)
        self.ctx._check(self.ctx._lib.gb_features_download(self.ctx._h, self._h, ptr(kps), ptr(desc), C.byref(n)))
        return kps[:n.value].copy(), desc[:n.value].copy()

    def match(self, train: "Features"):
        self.ctx._check(self.ctx._lib.gb_match_features(self.ctx._h, self._h, train._h))

    def match_stereo(self, right: "Features", band=2.0, min_disp=0.0, max_disp=1e9):
        self.ctx._check(self.ctx._lib.gb_match_stereo_features(self.ctx._h, self._h, right._h, band, min_disp, max_disp))

    def matches(self):
        n = C.c_int(self.capacity)
        idx = np.empty(self.capacity, np.int32); d1 = np.empty(self.capacity, np.int32); d2 = np.empty(self.capacity, np.int32)
        self.ctx._check(self.ctx._lib.gb_match_download(self.ctx._h, self._h, ptr(idx), ptr(d1), ptr(d2), C.byref(n)))
        return idx[:n.value].copy(), d1[:n.value].copy(), d2[:n.value].copy()


class BAGraph:
    """A bundle-adjustment graph resident in HBM (gb_ba_graph)."""

    def __init__(self, ctx: Context, pb: BAProblem, edges=None):
        self.ctx = ctx
        self.n_cams, self.n_points, self.n_obs = pb.n_cams, pb.n_points, pb.n_obs
        c, keep = _problem_c(pb)
        h = C.c_void_p()
        if edges is None:
            ctx._check(ctx._lib.gb_ba_graph_create(ctx._h, C.byref(c), C.byref(h)))
        else:
            e, keep2 = _edges_c(edges)
            ctx._check(ctx._lib.gb_ba_graph_create_ex(ctx._h, C.byref(c), C.byref(e), C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None) and getattr(self.ctx, "_h", None):
            self.ctx._lib.gb_ba_graph_destroy(self.ctx._h, self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        self.ctx._check(self.ctx._lib.gb_ba_graph_reset(self.ctx._h, self._h))

    def solve(self, cfg: OptimzeConfig | None = None) -> capi.BaResult:
        o = (cfg or OptimzeConfig()).to_c(); r = capi.BaResult()
        self.ctx._check(self.ctx._lib.gb_ba_graph_solve(self.ctx._h, self._h, C.byref(o), C.byref(r)))
        return r

    def sweep(self, delta: float = 0.01):
        """One fused residual+Jacobian sweep (K6) at the current estimate, enqueued on the ctx stream."""
        self.ctx._check(self.ctx._lib.gb_ba_graph_sweep(self.ctx._h, self._h, delta))

    def download(self):
        pose = np.zeros((self.n_cams, 7)); pts = np.zeros((self.n_points, 3))
        self.ctx._check(self.ctx._lib.gb_ba_graph_download(self.ctx._h, self._h, ptr(pose), ptr(pts)))
        return pose, pts

    # stepwise interface (landmark-sharded multi-GPU BA; see gslam_b200/dist.py)
    def reduce_size(self) -> int:
        n = C.c_size_t()
        self.ctx._check(self.ctx._lib.gb_ba_graph_reduce_size(self.ctx._h, self._h, C.byref(n)))
        return int(n.value)

    def begin(self, cfg: OptimzeConfig | None = None):
        o = (cfg or OptimzeConfig()).to_c()
        self.ctx._check(self.ctx._lib.gb_ba_graph_begin(self.ctx._h, self._h, C.byref(o)))

    def reduce_local(self, d_buf: int):
        self.ctx._check(self.ctx._lib.gb_ba_graph_reduce_local(self.ctx._h, self._h, C.c_void_p(d_buf)))

    def step(self, d_buf: int, d_cost: int):
        self.ctx._check(self.ctx._lib.gb_ba_graph_step(self.ctx._h, self._h, C.c_void_p(d_buf), C.c_void_p(d_cost)))

    def commit(self, d_buf: int, d_cost: int):
        self.ctx._check(self.ctx._lib.gb_ba_graph_commit(self.ctx._h, self._h, C.c_void_p(d_buf), C.c_void_p(d_cost)))

    def finish(self) -> capi.BaResult:
        r = capi.BaResult()
        self.ctx._check(self.ctx._lib.gb_ba_graph_finish(self.ctx._h, self._h, C.byref(r)))
        return r

    # test hooks
    def dbg_linearize(self, delta: float = 0.01):
        U = np.zeros((self.n_cams, 6, 6)); gc = np.zeros((self.n_cams, 6)); V = np.zeros((self.n_points, 3, 3))
        gp = np.zeros((self.n_points, 3)); W = np.zeros((self.n_obs, 6, 3)); cost = np.zeros(1)
        self.ctx._check(self.ctx._lib.gb_dbg_ba_linearize(self.ctx._h, self._h, delta, ptr(U), ptr(gc), ptr(V), ptr(gp),
                                                          ptr(W), ptr(cost)))
        return dict(U=U, gc=gc, V=V, gp=gp, W=W, cost=float(cost[0]))

    def force_generic_pcg(self, mode=1):
        """PCG dispatch override (test hook): 0 auto, 1 generic multi-kernel, 2 one-cluster DSMEM, 3 single-CTA block-sparse."""
        self.ctx._check(self.ctx._lib.gb_dbg_ba_force_generic_pcg(self.ctx._h, self._h, int(mode)))

    def set_cam_split(self, split: int):
        """CTAs per camera of the sweep's camera pass (test hook, 1..4; production graphs pick it from the longest camera)."""
        self.ctx._check(self.ctx._lib.gb_dbg_ba_set_cam_split(self.ctx._h, self._h, int(split)))

    def set_sweep(self, mode: int):
        """Sweep kernel (test hook): 0 by size, 1 the latency-tuned local-BA kernel, 2 the bandwidth-tuned large-graph kernel."""
        self.ctx._check(self.ctx._lib.gb_dbg_ba_set_sweep(self.ctx._h, self._h, int(mode)))

    def pcg_sparse_blocks(self) -> int:
        return int(self.ctx._lib.gb_dbg_ba_pcg_sparse(self.ctx._h, self._h))

    def pcg_cluster_size(self) -> int:
        return int(self.ctx._lib.gb_dbg_ba_pcg_cluster_size(self.ctx._h, self._h))

    # bits of paths(): what a solve of this graph would run, as planned now (gb_dbg_ba_paths in csrc/ba.cu)
    LOCAL4, PCG_SPARSE, PCG_CLUSTER, PCG_BCSR, BCSR_CLUSTER, SCHUR_CHUNKS, SWEEP_LARGE, DENSE_ATOMIC, CHOL_OK, CAM_SPLIT = (1 << k for k in range(10))

    def paths(self) -> int:
        """Bitmask of the solver paths (test hook): see the BAGraph.LOCAL4 ... CAM_SPLIT constants."""
        v = int(self.ctx._lib.gb_dbg_ba_paths(self.ctx._h, self._h))
        if v < 0:
            raise GbError(v, "gb_dbg_ba_paths")
        return v

    def dbg_reduced(self, cfg: OptimzeConfig | None = None):
        n6 = 6 * self.n_cams
        S = np.zeros((n6, n6)); gt = np.zeros(n6); dc = np.zeros(n6); it = C.c_int()
        o = (cfg or OptimzeConfig()).to_c()
        self.ctx._check(self.ctx._lib.gb_dbg_ba_reduced(self.ctx._h, self._h, C.byref(o), ptr(S), ptr(gt), ptr(dc), C.byref(it)))
        return S, gt, dc, it.value



class Comm:
    """A rank of the multi-GPU communicator (gb_comm): NCCL under the C-ABI.  `unique_id` is the 128 bytes rank 0 obtained from
    Comm.unique_id() and the host distributed (torch.distributed broadcast in bench.py / tests)."""

    def __init__(self, ctx: Context, world: int = 1, rank: int = 0, unique_id: bytes | None = None, _handle=None):
        self.ctx = ctx
        h = C.c_void_p(_handle) if _handle is not None else C.c_void_p()
        if _handle is None:
            buf = (C.c_uint8 * 128).from_buffer_copy(unique_id) if unique_id is not None else None
            ctx._check(ctx._lib.gb_comm_create(ctx._h, world, rank, C.cast(buf, C.c_void_p) if buf is not None else None, C.byref(h)))
        self._h = h
        self.rank, self.world = rank, world

    @staticmethod
    def unique_id() -> bytes:
        L = capi.lib()
        buf = (C.c_uint8 * 128)()
        rc = L.gb_comm_unique_id(C.cast(buf, C.c_void_p))
        if rc != capi.GB_OK:
            raise GbError(rc, L.gb_last_error(None).decode())
        return bytes(buf)

    def allreduce_sum_f64(self, d_ptr: int, n: int):
        self.ctx._check(self.ctx._lib.gb_comm_allreduce_sum_f64(self._h, C.c_void_p(d_ptr), n))

    def close(self):
        if getattr(self, "_h", None):
            self.ctx._lib.gb_comm_destroy(self._h)
            self._h = None


class ShardedBAGraph(BAGraph):
    """This rank's landmark shard of a global BA problem (gb_ba_shard_*): every rank passes the SAME full problem."""

    def __init__(self, comm: Comm, pb: BAProblem):
        self.ctx, self.comm = comm.ctx, comm
        c, keep = _problem_c(pb)
        h = C.c_void_p()
        self.ctx._check(self.ctx._lib.gb_ba_shard_create(comm._h, C.byref(c), C.byref(h)))
        self._h = h
        lo, hi = C.c_int(), C.c_int()
        self.ctx._check(self.ctx._lib.gb_ba_shard_range(self._h, C.byref(lo), C.byref(hi)))
        self.lo, self.hi = lo.value, hi.value
        self.n_cams, self.n_points = pb.n_cams, self.hi - self.lo
        nb = C.c_size_t()
        self.ctx._check(self.ctx._lib.gb_ba_shard_reduce_bytes(self._h, C.byref(nb)))
        self.reduce_bytes = int(nb.value)

    def solve(self, cfg: OptimzeConfig | None = None) -> capi.BaResult:
        o = (cfg or OptimzeConfig()).to_c(); r = capi.BaResult()
        self.ctx._check(self.ctx._lib.gb_ba_shard_solve(self.comm._h, self._h, C.byref(o), C.byref(r)))
        return r

    def dbg_shard_reduced(self, cfg: OptimzeConfig | None = None, allreduce: bool = False):
        """(S dense 6N x 6N undamped, g~, diag U, cost) of one iteration at the current estimate (test hook); with `allreduce` a
        collective that every rank calls."""
        n6 = 6 * self.n_cams
        S = np.zeros((n6, n6)); gt = np.zeros(n6); dU = np.zeros(n6); cost = np.zeros(1)
        o = (cfg or OptimzeConfig()).to_c()
        self.ctx._check(self.ctx._lib.gb_dbg_ba_shard_reduced(self.comm._h, self._h, C.byref(o), int(allreduce), ptr(S), ptr(gt), ptr(dU),
                                                              ptr(cost)))
        return S, gt, dU, float(cost[0])


def local_group(ctx: Context, world: int):
    """A loopback communicator of `world` ranks on ctx's device (test hook gb_dbg_comm_create_local): -> (ctxs, comms).  ctxs[0] is
    `ctx`; the others share its stream.  Close the comms, then ctxs[1:], before `ctx`."""
    L = ctx._lib
    hc = (C.c_void_p * world)()
    hm = (C.c_void_p * world)()
    rc = L.gb_dbg_comm_create_local(ctx._h, world, hc, hm)
    if rc != capi.GB_OK:
        raise GbError(rc, L.gb_last_error(None).decode())
    ctxs = [ctx]
    for r in range(1, world):
        c = Context.__new__(Context)
        c._lib, c._h, c.device = L, C.c_void_p(hc[r]), ctx.device
        ctxs.append(c)
    return ctxs, [Comm(ctxs[r], world, r, _handle=hm[r]) for r in range(world)]


def ba_solve_multi(ctxs, pb: BAProblem, cfg: OptimzeConfig | None = None, comms=None) -> capi.BaResult:
    """One process, len(ctxs) GPUs: gb_comm_create_all + gb_ba_solve_multi (what the optimizer plugin does for b200.devices).  With
    `comms` (Comm objects, e.g. from local_group) those communicators are used instead, and the caller keeps them."""
    L = capi.lib()
    n = len(ctxs)
    own = comms is None
    if own:
        hs = (C.c_void_p * n)(*[c._h for c in ctxs])
        hm = (C.c_void_p * n)()
        ctxs[0]._check(L.gb_comm_create_all(n, hs, hm))
    else:
        hm = (C.c_void_p * n)(*[m._h.value for m in comms])
    try:
        c, keep = _problem_c(pb)
        o = (cfg or OptimzeConfig()).to_c(); r = capi.BaResult()
        ctxs[0]._check(L.gb_ba_solve_multi(n, hm, C.byref(c), C.byref(o), C.byref(r)))
        return r
    finally:
        if own:
            for k in range(n):
                L.gb_comm_destroy(hm[k])

class Optimizer:
    """Mirror of GSLAM::Optimizer (Optimizer.h:184-253): bool returns, graph / pose updated in place, `_config` public."""

    def __init__(self, config: OptimzeConfig | None = None, device: int = 0):
        self._config = config or OptimzeConfig()
        self._ctx = Context(device)
        self.last_result: capi.BaResult | None = None

    def optimize(self, graph: BAProblem) -> bool:
        try:
            self.last_result = self._ctx.ba_solve(graph, self._config)
            return True
        except GbError:
            return False

    def optimizePnP(self, matches_xyz, matches_anchor, pose: np.ndarray, dof: int = 63, information: np.ndarray | None = None) -> bool:
        try:
            out, res, info = self._ctx.ba_pnp(matches_xyz, matches_anchor, pose, dof, want_info=information is not None,
                                              cfg=self._config)
            pose[...] = out
            if information is not None:
                information[...] = info
            self.last_result = res
            return True
        except GbError:
            return False

    @staticmethod
    def create(pluginName: str = "", device: int = 0):
        """GSLAM::Optimizer::create (Optimizer.h:234-248): returns None (the reference returns a null shared_ptr) on failure."""
        try:
            return Optimizer(device=device)
        except (GbError, ImportError, OSError):
            return None
