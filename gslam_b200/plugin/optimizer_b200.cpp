// gslam_b200/plugin/optimizer_b200.cpp -> libgslam_optimizer.so
//
// The drop-in: a GSLAM::Optimizer (GSLAM/core/Optimizer.h:184-253) whose optimize()/optimizePnP() run on the GPU through
// the C-ABI of include/gslam_b200.h.  Found by GSLAM::Optimizer::create() exactly like the (absent) Ceres plugin:
// Registry::get("libgslam_optimizer") -> dlsym("createOptimizerInstance") (Optimizer.h:234-248, 42-51).
// This TU is built with default symbol visibility: GSLAM_REGISTER_OPTIMIZER adds no visibility attribute (SURVEY.md §8b).
//
// Contract kept from the reference: bool returns, never throws across the boundary, BundleGraph& / SE3& updated in place,
// `_config` is honoured on every call (callers may edit it between calls, Optimizer.h:252).
#include <GSLAM/core/GSLAM.h>
#include <GSLAM/core/Optimizer.h>

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/gslam_b200.h"

namespace {

class OptimizerB200 : public GSLAM::Optimizer {
 public:
  OptimizerB200() : ctx_(nullptr), multi_failed_(false) {}
  ~OptimizerB200() override {
    for (size_t k = 0; k < comms_.size(); ++k) gb_comm_destroy(comms_[k]);
    for (size_t k = 0; k < ctxs_.size(); ++k)
      if (ctxs_[k] != ctx_) gb_ctx_destroy(ctxs_[k]);
    if (ctx_) gb_ctx_destroy(ctx_);
  }

  // MAPPING: bundle adjustment over BundleGraph::keyframes / mappoints / mappointObserves, pose-graph terms se3Graph / gpsGraph --
  // BUNDLEADJUST and POSEGRAPH of Optimizer.h:227-229 (graph PODs :106-172)
  bool optimize(GSLAM::BundleGraph& graph) override {
    try {
      if (!graph.invDepths.empty() || !graph.invDepthObserves.empty() || !graph.sim3Graph.empty()) {
        LOG(ERROR) << "gslam_b200 optimizer: inverse-depth landmarks and SIM3 edges are not implemented (SURVEY.md §8f-3)";
        return false;
      }
      if (graph.camera.isValid() && graph.cameraDOF != GSLAM::UPDATE_CAMERA_NONE) {
        LOG(ERROR) << "gslam_b200 optimizer: camera self-calibration (cameraDOF) is not implemented";
        return false;
      }
      if (_config.cameraProjectionType != GSLAM::PROJECTION_PINHOLE) {
        LOG(ERROR) << "gslam_b200 optimizer: only PROJECTION_PINHOLE is implemented";
        return false;
      }
      if (!ensureContext()) return false;
      const size_t nc = graph.keyframes.size(), np = graph.mappoints.size(), no = graph.mappointObserves.size();
      // AoS -> SoA repack into member buffers (capacity is kept across calls: a sliding window re-uses them without touching the
      // allocator; the edge loop runs on all cores for global-BA-sized graphs: 48 MB of BundleEdge at config 5)
      std::lock_guard<std::mutex> call_lock(call_mu_);
      std::vector<double>&pose = pose_, &pts = pts_, &xyz = xyz_, &info = info_;
      std::vector<uint8_t>&dof = dof_, &pfree = pfree_;
      std::vector<int32_t>&oc = oc_, &op = op_;
      pose.resize(7 * nc); pts.resize(3 * np); xyz.resize(3 * no); info.clear(); dof.resize(nc); pfree.resize(np); oc.resize(no); op.resize(no);
      for (size_t i = 0; i < nc; ++i) {
        // SIM3 memory = {SO3{x,y,z,w}, Point3d, scale}: the first 7 doubles are the SE3 T_wc (SE3.h:337-339, SIM3.h:290-291)
        const GSLAM::SE3& T = graph.keyframes[i].estimation.get_se3();
        const GSLAM::SO3& r = T.get_rotation();
        const GSLAM::Point3d& t = T.get_translation();
        double* p = &pose[7 * i];
        p[0] = r.x; p[1] = r.y; p[2] = r.z; p[3] = r.w; p[4] = t.x; p[5] = t.y; p[6] = t.z;
        dof[i] = (uint8_t)(graph.keyframes[i].dof & 63);
      }
      for (size_t j = 0; j < np; ++j) {
        const GSLAM::Point3d& p = graph.mappoints[j].first;
        pts[3 * j] = p.x; pts[3 * j + 1] = p.y; pts[3 * j + 2] = p.z;
        pfree[j] = graph.mappoints[j].second ? 1 : 0;
      }
      bool any_info = false;
      for (size_t k = 0; k < no; ++k) any_info |= graph.mappointObserves[k].information != NULL;
      if (any_info) info.resize(4 * no);
      std::atomic<long> bad_edge_a(-1);
      auto repack = [&](size_t k0, size_t k1) {
        for (size_t k = k0; k < k1; ++k) {
          const GSLAM::BundleEdge& e = graph.mappointObserves[k];
          if (e.frameId >= nc || e.pointId >= np) { bad_edge_a = (long)k; continue; }
          oc[k] = (int32_t)e.frameId; op[k] = (int32_t)e.pointId;
          xyz[3 * k] = e.measurement.x; xyz[3 * k + 1] = e.measurement.y; xyz[3 * k + 2] = e.measurement.z;
          if (any_info) {
            double* L = &info[4 * k];
            if (e.information) std::memcpy(L, e.information, 4 * sizeof(double));
            else { L[0] = 1; L[1] = 0; L[2] = 0; L[3] = 1; }
          }
        }
      };
      if (no > 65536) {  // global-BA-sized: split the edge list over a few host threads
        const size_t nt = std::min<size_t>(std::max(2u, std::thread::hardware_concurrency()), 16);
        std::vector<std::thread> th;
        for (size_t t = 1; t < nt; ++t) th.emplace_back(repack, no * t / nt, no * (t + 1) / nt);
        repack(0, no / nt);
        for (size_t t = 0; t < th.size(); ++t) th[t].join();
      } else {
        repack(0, no);
      }
      const long bad_edge = bad_edge_a;
      if (bad_edge >= 0) {
        const GSLAM::BundleEdge& e = graph.mappointObserves[bad_edge];
        LOG(ERROR) << "gslam_b200 optimizer: edge " << bad_edge << " references frame " << e.frameId << " / point " << e.pointId;
        return false;
      }
      gb_ba_problem pb;
      std::memset(&pb, 0, sizeof pb);
      pb.n_cams = (int32_t)nc; pb.n_points = (int32_t)np; pb.n_obs = (int32_t)no;
      pb.cam_pose_wc = pose.data(); pb.cam_dof = dof.data(); pb.points = pts.data(); pb.point_free = pfree.data();
      pb.obs_cam = oc.data(); pb.obs_point = op.data(); pb.obs_xyz = xyz.data(); pb.obs_info = any_info ? info.data() : NULL;
      // pose-graph terms: SE3Edge {firstId, secondId, SE3_12, information 6x6} and GPSEdge {frameId, SE3_gps, information 6x6}
      // (Optimizer.h:127-148) -> gb_pose_edges; a NULL information is the identity, a mix of NULL and non-NULL is filled in
      const size_t nse = graph.se3Graph.size(), ngps = graph.gpsGraph.size();
      std::vector<int32_t> se_a(nse), se_b(nse), gps_f(ngps);
      std::vector<double> se_m(7 * nse), gps_m(7 * ngps), se_i, gps_i;
      auto put7 = [](const GSLAM::SE3& T, double* p) {
        const GSLAM::SO3& r = T.get_rotation();
        const GSLAM::Point3d& t = T.get_translation();
        p[0] = r.x; p[1] = r.y; p[2] = r.z; p[3] = r.w; p[4] = t.x; p[5] = t.y; p[6] = t.z;
      };
      auto put36 = [](const double* info, double* dst) {
        for (int k = 0; k < 36; ++k) dst[k] = info ? info[k] : ((k % 7) == 0 ? 1.0 : 0.0);
      };
      bool se_info = false, gps_info = false;
      for (size_t k = 0; k < nse; ++k) se_info |= graph.se3Graph[k].information != NULL;
      for (size_t k = 0; k < ngps; ++k) gps_info |= graph.gpsGraph[k].information != NULL;
      if (se_info) se_i.resize(36 * nse);
      if (gps_info) gps_i.resize(36 * ngps);
      for (size_t k = 0; k < nse; ++k) {
        const GSLAM::SE3Edge& e = graph.se3Graph[k];
        if (e.firstId >= nc || e.secondId >= nc) { LOG(ERROR) << "gslam_b200 optimizer: SE3 edge " << k << " references a missing keyframe"; return false; }
        se_a[k] = (int32_t)e.firstId; se_b[k] = (int32_t)e.secondId;
        put7(e.measurement, &se_m[7 * k]);
        if (se_info) put36(e.information, &se_i[36 * k]);
      }
      for (size_t k = 0; k < ngps; ++k) {
        const GSLAM::GPSEdge& e = graph.gpsGraph[k];
        if (e.frameId >= nc) { LOG(ERROR) << "gslam_b200 optimizer: GPS edge " << k << " references a missing keyframe"; return false; }
        gps_f[k] = (int32_t)e.frameId;
        put7(e.measurement, &gps_m[7 * k]);
        if (gps_info) put36(e.information, &gps_i[36 * k]);
      }
      gb_pose_edges pe;
      std::memset(&pe, 0, sizeof pe);
      pe.n_se3 = (int32_t)nse; pe.se3_first = se_a.data(); pe.se3_second = se_b.data(); pe.se3_meas = se_m.data(); pe.se3_info = se_info ? se_i.data() : NULL;
      pe.n_gps = (int32_t)ngps; pe.gps_frame = gps_f.data(); pe.gps_meas = gps_m.data(); pe.gps_info = gps_info ? gps_i.data() : NULL;
      gb_ba_options opt = options();
      gb_ba_result res;
      // global-BA-sized graphs on several GPUs when the svar option `b200.devices` (e.g. "0,1,2,3") names more than one device:
      // landmark-sharded solve, one NCCL all-reduce of the reduced camera system per LM iteration (gb_ba_solve_multi)
      int rc;
      if (nse + ngps > 0)
        rc = gb_ba_solve_posegraph(ctx_, &pb, &pe, &opt, &res);
      else if (no >= (size_t)svar.GetInt("b200.multi_min_obs", 200000) && ensureMulti())
        rc = gb_ba_solve_multi((int)comms_.size(), comms_.data(), &pb, &opt, &res);
      else
        rc = gb_ba_solve(ctx_, &pb, &opt, &res);
      if (rc != GB_OK) {
        LOG(ERROR) << "gslam_b200 optimizer: " << gb_last_error(ctx_);
        return false;
      }
      for (size_t i = 0; i < nc; ++i) {
        const double* p = &pose[7 * i];
        GSLAM::SIM3& S = graph.keyframes[i].estimation;
        S = GSLAM::SIM3(GSLAM::SE3(GSLAM::SO3(p[0], p[1], p[2], p[3]), GSLAM::Point3d(p[4], p[5], p[6])), S.get_scale());
      }
      for (size_t j = 0; j < np; ++j) graph.mappoints[j].first = GSLAM::Point3d(pts[3 * j], pts[3 * j + 1], pts[3 * j + 2]);
      if (_config.verbose)
        LOG(INFO) << "gslam_b200 optimizer: cost " << res.initial_cost << " -> " << res.final_cost << " in " << res.iterations
                  << " iterations (" << res.gpu_ms << " ms on device)";
      return true;
    } catch (...) {
      return false;  // nothing may escape a plugin (Optimizer.h:193-232 convention)
    }
  }

  // TRACKING: pose from 3D-2D correspondences (Optimizer.h:202-207)
  bool optimizePnP(const std::vector<std::pair<GSLAM::Point3d, GSLAM::CameraAnchor> >& matches, GSLAM::SE3& pose,
                   GSLAM::KeyFrameEstimzationDOF dof = GSLAM::UPDATE_KF_SE3, double* information = NULL) override {
    try {
      if (!ensureContext()) return false;
      const size_t n = matches.size();
      std::vector<double> xyz(3 * n), xy1(3 * n);
      for (size_t k = 0; k < n; ++k) {
        xyz[3 * k] = matches[k].first.x; xyz[3 * k + 1] = matches[k].first.y; xyz[3 * k + 2] = matches[k].first.z;
        xy1[3 * k] = matches[k].second.x; xy1[3 * k + 1] = matches[k].second.y; xy1[3 * k + 2] = matches[k].second.z;
      }
      const GSLAM::SO3& r = pose.get_rotation();
      const GSLAM::Point3d& t = pose.get_translation();
      double p[7] = {r.x, r.y, r.z, r.w, t.x, t.y, t.z};
      gb_ba_options opt = options();
      gb_ba_result res;
      const int rc = gb_ba_pnp(ctx_, (int)n, xyz.data(), xy1.data(), p, (int)dof & 63, information, &opt, &res);
      if (rc != GB_OK) {
        LOG(ERROR) << "gslam_b200 optimizer: " << gb_last_error(ctx_);
        return false;
      }
      pose = GSLAM::SE3(GSLAM::SO3(p[0], p[1], p[2], p[3]), GSLAM::Point3d(p[4], p[5], p[6]));
      return true;
    } catch (...) {
      return false;
    }
  }

 private:
  bool ensureContext() {
    std::lock_guard<std::mutex> lk(mu_);
    if (ctx_) return true;
    const int device = svar.GetInt("b200.device", 0);
    if (gb_ctx_create(device, &ctx_) != GB_OK) {
      LOG(ERROR) << "gslam_b200 optimizer: no usable CUDA device (" << gb_last_error(NULL) << "); there is no CPU fallback";
      ctx_ = nullptr;
      return false;
    }
    return true;
  }

  // contexts + communicators for `b200.devices`; false (single-GPU path) when fewer than two devices are named or usable
  bool ensureMulti() {
    std::lock_guard<std::mutex> lk(mu_);
    if (!comms_.empty()) return true;
    if (multi_failed_) return false;
    const std::string list = svar.GetString("b200.devices", "");
    std::vector<int> devs;
    for (size_t i = 0; i < list.size();) {
      size_t j = list.find(',', i);
      if (j == std::string::npos) j = list.size();
      if (j > i) devs.push_back(atoi(list.substr(i, j - i).c_str()));
      i = j + 1;
    }
    if (devs.size() < 2) { multi_failed_ = true; return false; }
    for (size_t k = 0; k < devs.size(); ++k) {
      gb_ctx* c = nullptr;
      if (ctx_ && devs[k] == svar.GetInt("b200.device", 0)) c = ctx_;
      else if (gb_ctx_create(devs[k], &c) != GB_OK) {
        LOG(ERROR) << "gslam_b200 optimizer: b200.devices names device " << devs[k] << " which is not usable (" << gb_last_error(NULL)
                   << "); staying on one GPU";
        for (size_t t = 0; t < ctxs_.size(); ++t)
          if (ctxs_[t] != ctx_) gb_ctx_destroy(ctxs_[t]);
        ctxs_.clear();
        multi_failed_ = true;
        return false;
      }
      ctxs_.push_back(c);
    }
    comms_.resize(ctxs_.size(), nullptr);
    if (gb_comm_create_all((int)ctxs_.size(), ctxs_.data(), comms_.data()) != GB_OK) {
      LOG(ERROR) << "gslam_b200 optimizer: communicator over b200.devices failed (" << gb_last_error(ctxs_[0]) << "); staying on one GPU";
      for (size_t t = 0; t < ctxs_.size(); ++t)
        if (ctxs_[t] != ctx_) gb_ctx_destroy(ctxs_[t]);
      ctxs_.clear(); comms_.clear();
      multi_failed_ = true;
      return false;
    }
    return true;
  }

  gb_ba_options options() const {
    gb_ba_options o;
    gb_ba_options_default(&o);
    o.huber_delta = _config.projectErrorHuberThreshold;  // OptimzeConfig, Optimizer.h:174-182
    o.max_iterations = _config.maxIterations;
    o.verbose = _config.verbose ? 1 : 0;
    o.function_tolerance = svar.GetDouble("b200.ftol", o.function_tolerance);
    o.lambda_init = svar.GetDouble("b200.lambda", o.lambda_init);
    o.pcg_max_iters = svar.GetInt("b200.pcg_iters", o.pcg_max_iters);
    o.pcg_tol = svar.GetDouble("b200.pcg_tol", o.pcg_tol);
    o.linear_solver = svar.GetInt("b200.linear_solver", o.linear_solver);  // 1 = direct block-skyline Cholesky (local-BA sizes)
    return o;
  }

  gb_ctx* ctx_;
  std::mutex mu_, call_mu_;
  std::vector<gb_ctx*> ctxs_;     // b200.devices
  std::vector<gb_comm*> comms_;
  bool multi_failed_;
  std::vector<double> pose_, pts_, xyz_, info_;  // repack buffers (kept across calls)
  std::vector<uint8_t> dof_, pfree_;
  std::vector<int32_t> oc_, op_;
};

}  // namespace

GSLAM_REGISTER_OPTIMIZER(OptimizerB200)
