// gslam_b200/plugin/estimator_b200.cpp -> libgslam_estimator.so
//
// A GSLAM::Estimator (GSLAM/core/Estimator.h:93-193) whose findPnP() runs P3P + RANSAC + refinement on the GPU through
// gb_pnp_ransac (include/gslam_b200.h).  Found by GSLAM::Estimator::create() like the (absent) default estimator plugin:
// Registry::get(svar "EstimatorPlugin" = "libgslam_estimator") -> dlsym("createEstimatorInstance") (Estimator.h:175-191, 43-45).
// SURVEY.md §8f-1.
//
// Contract kept from the reference: bool returns, never throws across the boundary, `const` methods, the optional mask receives one
// byte per correspondence.  Only findPnP is implemented; every other model returns false (the reference's own convention for an
// estimator without that solver) with one log line.
#include <GSLAM/core/GSLAM.h>
#include <GSLAM/core/Estimator.h>

#include <mutex>
#include <vector>

#include "../../include/gslam_b200.h"

namespace {

class EstimatorB200 : public GSLAM::Estimator {
 public:
  EstimatorB200() : ctx_(nullptr) {}
  ~EstimatorB200() override {
    if (ctx_) gb_ctx_destroy(ctx_);
  }
  std::string type() const override { return "EstimatorB200"; }

  // 2D&3D correspondences (Estimator.h:158-164): imagePoints are normalised (unit focal plane), threshold in the same unit.
  // `method`: the reference's default P3_ITERATIVE&RANSAC evaluates to 0; every value selects P3P + RANSAC + LM refinement here.
  bool findPnP(GSLAM::SE3* world2camera, const std::vector<GSLAM::Point3d>& objectPoints, const std::vector<GSLAM::Point2d>& imagePoints,
               int method, double threshold, double confidence, std::vector<GSLAM::uchar>* mask) const override {
    (void)method;
    try {
      if (!world2camera || objectPoints.size() != imagePoints.size() || objectPoints.size() < 4) return false;
      if (!ensureContext()) return false;
      const size_t n = objectPoints.size();
      std::vector<double> xyz(3 * n), xy(2 * n);
      for (size_t k = 0; k < n; ++k) {
        xyz[3 * k] = objectPoints[k].x; xyz[3 * k + 1] = objectPoints[k].y; xyz[3 * k + 2] = objectPoints[k].z;
        xy[2 * k] = imagePoints[k].x; xy[2 * k + 1] = imagePoints[k].y;
      }
      std::vector<uint8_t> m(n);
      double p[7];
      gb_pnp_stats st;
      const int rc = gb_pnp_ransac(ctx_, (int)n, xyz.data(), xy.data(), threshold, confidence, svar.GetInt("b200.pnp_hypotheses", 1024),
                                   (uint64_t)svar.GetInt("b200.pnp_seed", 1), p, m.data(), &st);
      if (rc != GB_OK) {
        LOG(WARNING) << "gslam_b200 estimator: " << gb_last_error(ctx_);
        return false;
      }
      *world2camera = GSLAM::SE3(GSLAM::SO3(p[0], p[1], p[2], p[3]), GSLAM::Point3d(p[4], p[5], p[6]));
      if (mask) mask->assign(m.begin(), m.end());
      return true;
    } catch (...) {
      return false;
    }
  }

#define GB_UNIMPLEMENTED(what)                                                                     \
  LOG(ERROR) << "gslam_b200 estimator: " what " is not implemented (only findPnP, SURVEY.md §8f)"; \
  return false
  bool findHomography(GSLAM::Homography2D*, const std::vector<GSLAM::Point2d>&, const std::vector<GSLAM::Point2d>&, int, double, double,
                      std::vector<GSLAM::uchar>*) const override { GB_UNIMPLEMENTED("findHomography"); }
  bool findAffine2D(GSLAM::Affine2D*, const std::vector<GSLAM::Point2d>&, const std::vector<GSLAM::Point2d>&, int, double, double,
                    std::vector<GSLAM::uchar>*) const override { GB_UNIMPLEMENTED("findAffine2D"); }
  bool findFundamental(GSLAM::Fundamental*, const std::vector<GSLAM::Point2d>&, const std::vector<GSLAM::Point2d>&, int, double, double,
                       std::vector<GSLAM::uchar>*) const override { GB_UNIMPLEMENTED("findFundamental"); }
  bool findEssentialMatrix(GSLAM::Essential*, const std::vector<GSLAM::Point2d>&, const std::vector<GSLAM::Point2d>&, int, double, double,
                           std::vector<GSLAM::uchar>*) const override { GB_UNIMPLEMENTED("findEssentialMatrix"); }
  bool findSIM3(GSLAM::SIM3*, const std::vector<GSLAM::Point3d>&, const std::vector<GSLAM::Point3d>&, int, double, double,
                std::vector<GSLAM::uchar>*) const override { GB_UNIMPLEMENTED("findSIM3"); }
  bool findAffine3D(GSLAM::Affine3D*, const std::vector<GSLAM::Point3d>&, const std::vector<GSLAM::Point3d>&, int, double, double,
                    std::vector<GSLAM::uchar>*) const override { GB_UNIMPLEMENTED("findAffine3D"); }
  bool findPlane(GSLAM::SE3*, const std::vector<GSLAM::Point3d>&, int, double, double, std::vector<GSLAM::uchar>*) const override {
    GB_UNIMPLEMENTED("findPlane");
  }
  bool trianglate(GSLAM::Point3d*, const GSLAM::SE3&, const GSLAM::Point3d&, const GSLAM::Point3d&) const override {
    GB_UNIMPLEMENTED("trianglate");
  }
#undef GB_UNIMPLEMENTED

 private:
  bool ensureContext() const {
    std::lock_guard<std::mutex> lk(mu_);
    if (ctx_) return true;
    if (gb_ctx_create(svar.GetInt("b200.device", 0), &ctx_) != GB_OK) {
      LOG(ERROR) << "gslam_b200 estimator: no usable CUDA device (" << gb_last_error(NULL) << "); there is no CPU fallback";
      ctx_ = nullptr;
      return false;
    }
    return true;
  }
  mutable gb_ctx* ctx_;
  mutable std::mutex mu_;
};

}  // namespace

using GSLAM::funcCreateEstimatorInstance;  // (the reference macro names it unqualified, Estimator.h:50)
USE_ESTIMATOR_PLUGIN(EstimatorB200)
