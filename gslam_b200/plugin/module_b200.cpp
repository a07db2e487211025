// gslam_b200/plugin/module_b200.cpp -> libgslam_b200.so
//
// Svar module (GSLAM/core/Svar.h:71-76, loaded with GSLAM::Registry::load("b200"), Registry.h:48-77) that exposes the feature
// path the reference has no interface for (the ORB calls live in external SLAM plugins, README.md:130-133):
//   svar["gslam"]["b200"]["orb_extract"]   (GImage gray8, Svar cfg) -> {"keypoints": vector<KeyPoint>, "descriptors": GImage Nx32 8UC1}
//   svar["gslam"]["b200"]["match_hamming"] (GImage query Nx32, GImage train Mx32) -> {"trainIdx": vector<int>, "distance": vector<int>,
//                                                                                    "distance2": vector<int>}
//   svar["gslam"]["b200"]["extract_to_frame"] (FramePtr, Svar cfg) -> bool : getImage() -> orb_extract -> setKeyPoints()
//                                                                     (Map.h:287,311-312)
//   svar["gslam"]["b200"]["match_stereo"]  (kps_left, desc_left, kps_right, desc_right, Svar cfg) -> {"rightIdx", "distance", "distance2"}
//   svar["gslam"]["b200"]["undistort"]     (GImage, Camera in, Camera out) -> GImage : GSLAM::Undistorter::undistort (Undistorter.h:271-348)
//   svar["gslam"]["b200"]["vocabulary"]    (std::shared_ptr<Vocabulary>) -> std::shared_ptr<Vocabulary> : the same vocabulary with the
//                                          batch transforms (Vocabulary.h:174,192: virtual) answered by the device; any code holding
//                                          a GSLAM::Vocabulary* / VocabularyPtr keeps working unchanged
//   svar["gslam"]["apps"]["b200_features"] the Messenger application: "dataset/frame" -> extract -> "b200_features/curframe"
// Outputs are the reference's own carrier types: GSLAM::KeyPoint (Map.h:122-195) and an owning GImage (GImage.h:160-443).
// Functions do not throw; on failure they return an undefined Svar / false and log through GSLAM's LOG.
#include <GSLAM/core/GSLAM.h>
#include <GSLAM/core/Undistorter.h>
#include <GSLAM/core/Vocabulary.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/gslam_b200.h"

namespace {

static_assert(sizeof(GSLAM::KeyPoint) == sizeof(gb_keypoint), "gb_keypoint must be field-compatible with GSLAM::KeyPoint");

struct SharedCtx {
  gb_ctx* ctx = nullptr;
  std::mutex mu;
  gb_ctx* get() {
    std::lock_guard<std::mutex> lk(mu);
    if (!ctx) {
      if (gb_ctx_create(svar.GetInt("b200.device", 0), &ctx) != GB_OK) {
        LOG(ERROR) << "gslam_b200: no usable CUDA device (" << gb_last_error(NULL) << "); there is no CPU fallback";
        ctx = nullptr;
      }
    }
    return ctx;
  }
};
SharedCtx& shared() {
  static SharedCtx s;
  return s;
}

gb_orb_cfg cfgFrom(GSLAM::Svar cfg) {
  gb_orb_cfg c;
  gb_orb_cfg_default(&c);
  if (cfg.isObject()) {
    c.nfeatures = cfg.get<int>("nfeatures", c.nfeatures);
    c.scale_factor = (float)cfg.get<double>("scaleFactor", c.scale_factor);
    c.nlevels = cfg.get<int>("nlevels", c.nlevels);
    c.edge_threshold = cfg.get<int>("edgeThreshold", c.edge_threshold);
    c.fast_threshold = cfg.get<int>("fastThreshold", c.fast_threshold);
  }
  return c;
}

bool extract(const GSLAM::GImage& img, GSLAM::Svar cfg, std::vector<GSLAM::KeyPoint>& kps, GSLAM::GImage& desc) {
  // 8UC1 gray, or the 8UC3 / 8UC4 colour frames GSLAM's dataset plugins deliver (B,G,R[,A] unless cfg.rgb): converted on the device
  const int channels = img.channels();
  if (img.empty() || img.elemSize1() != 1 || (channels != 1 && channels != 3 && channels != 4)) {
    LOG(ERROR) << "gslam_b200 orb_extract: need a non-empty 8-bit image with 1, 3 or 4 channels";
    return false;
  }
  const int rgb = cfg.isObject() ? (cfg.get<bool>("rgb", false) ? 1 : 0) : 0;
  gb_ctx* ctx = shared().get();
  if (!ctx) return false;
  gb_orb_cfg c = cfgFrom(cfg);
  if (c.nfeatures <= 0 || c.nfeatures > (1 << 20)) {  // (validated before any buffer is sized from it: nothing may throw out of a Svar function)
    LOG(ERROR) << "gslam_b200 orb_extract: nfeatures must be in 1 .. 1048576";
    return false;
  }
  int n = 2 * c.nfeatures + 256;
  for (int attempt = 0; attempt < 2; ++attempt) {
    kps.resize(n);
    std::vector<uint8_t> d((size_t)n * 32);
    int got = n;
    // GImage has no row stride: row i at data + i*cols (GImage.h:378)
    const int rc = gb_orb_extract_image(ctx, img.data, img.cols, img.rows, channels, rgb, &c, reinterpret_cast<gb_keypoint*>(kps.data()), d.data(), &got);
    if (rc == GB_ERR_CAPACITY && got > n) { n = got; continue; }
    if (rc != GB_OK) {
      LOG(ERROR) << "gslam_b200 orb_extract: " << gb_last_error(ctx);
      return false;
    }
    kps.resize(got);
    desc = GSLAM::GImage(got, 32, GSLAM::GImageType<uchar, 1>::Type, got ? d.data() : NULL, true);  // owning copy
    return true;
  }
  return false;
}

// ---- the vocabulary (SURVEY.md section 8f-4) -----------------------------------------------------------------------------------------
// A GSLAM::Vocabulary whose batch transforms (virtual, Vocabulary.h:174-175,192-193) run on the device.  Everything else -- load /
// save, single-descriptor transform, score, getWord ... -- is the base class, working on the same tree.  The tree is uploaded once,
// on the first transform (gb_voc_create); the BowVector / FeatureVector are std::maps as the reference defines them (:47-48), filled in
// ascending key order with an end() hint (amortised O(1) per entry).
class B200Vocabulary : public GSLAM::Vocabulary {
 public:
  explicit B200Vocabulary(const GSLAM::Vocabulary& src) : GSLAM::Vocabulary(src) {}
  ~B200Vocabulary() {
    if (dev_ && ctx_) gb_voc_destroy(ctx_, dev_);
  }
  virtual void transform(const GSLAM::TinyMat& features, GSLAM::BowVector& v) const {
    GSLAM::FeatureVector fv;
    if (!run(features, v, fv, 0, false)) GSLAM::Vocabulary::transform(features, v);
  }
  virtual void transform(const GSLAM::TinyMat& features, GSLAM::BowVector& v, GSLAM::FeatureVector& fv, int levelsup = 0) const {
    if (!run(features, v, fv, levelsup, true)) GSLAM::Vocabulary::transform(features, v, fv, levelsup);
  }

 private:
  // false: this input is not the device path's (not 32-byte 8-bit rows, k > 32): the caller forwards to the base class -- the same
  // answer from the reference's own code, NOT a fallback for a missing device (a missing device is an error: empty vectors + LOG)
  bool run(const GSLAM::TinyMat& features, GSLAM::BowVector& v, GSLAM::FeatureVector& fv, int levelsup, bool want_fv) const {
    if (m_nodeDescriptors.cols != 32 || m_nodeDescriptors.elemSize() != 1 || m_k > 32) return false;
    v.clear(); fv.clear();
    if (empty() || features.rows <= 0) { if (getenv("GB_DEBUG")) fprintf(stderr, "gslam_b200 vocabulary: empty input (%zu nodes, %d rows)\n", m_nodes.size(), features.rows); return true; }
    if (features.cols != 32 || features.elemSize() != 1) {
      LOG(ERROR) << "gslam_b200 vocabulary: features must be N x 32 8UC1";
      fprintf(stderr, "gslam_b200 vocabulary: features must be N x 32 8UC1 (got %d cols, elemSize %d)\n", features.cols, (int)features.elemSize());
      return true;
    }
    std::lock_guard<std::mutex> lk(mu_);
    if (!dev_) {
      ctx_ = shared().get();
      if (!ctx_) { fprintf(stderr, "gslam_b200 vocabulary: no device context\n"); return true; }  // (also logged by shared(): no CPU fallback)
      std::vector<uint32_t> child(m_nodes.size());
      std::vector<float> weight(m_nodes.size());
      for (size_t i = 0; i < m_nodes.size(); ++i) { child[i] = m_nodes[i].childNum; weight[i] = m_nodes[i].weight; }
      if (gb_voc_create(ctx_, m_k, m_L, (int)m_weighting, (int)m_scoring, (uint32_t)m_nodes.size(), child.data(), weight.data(), m_nodeDescriptors.data,
                        &dev_) != GB_OK) {
        LOG(ERROR) << "gslam_b200 vocabulary: " << gb_last_error(ctx_);
        fprintf(stderr, "gslam_b200 vocabulary: %s\n", gb_last_error(ctx_));
        dev_ = nullptr;
        return true;
      }
    }
    const int n = features.rows;
    words_.resize(n); values_.resize(n); fv_node_.resize(n); fv_feat_.resize(n);
    int nw = 0, m = 0;
    if (gb_bow_transform(ctx_, dev_, features.data, n, levelsup, words_.data(), values_.data(), &nw, fv_node_.data(), fv_feat_.data(), &m) != GB_OK) {
      LOG(ERROR) << "gslam_b200 vocabulary: " << gb_last_error(ctx_);
      fprintf(stderr, "gslam_b200 vocabulary: %s\n", gb_last_error(ctx_));
      return true;
    }
    if (getenv("GB_DEBUG")) fprintf(stderr, "gslam_b200 vocabulary: %d rows -> %d words, %d feature entries\n", n, nw, m);
    for (int i = 0; i < nw; ++i) v.insert(v.end(), GSLAM::BowVector::value_type((GSLAM::WordId)words_[i], values_[i]));
    if (want_fv)
      for (int i = 0; i < m;) {
        int j = i;
        while (j < m && fv_node_[j] == fv_node_[i]) ++j;
        GSLAM::FeatureVector::iterator it = fv.insert(fv.end(), GSLAM::FeatureVector::value_type((GSLAM::NodeId)fv_node_[i], std::vector<unsigned int>()));
        it->second.assign(fv_feat_.begin() + i, fv_feat_.begin() + j);
        i = j;
      }
    return true;
  }
  mutable std::mutex mu_;
  mutable gb_ctx* ctx_ = nullptr;
  mutable gb_vocabulary* dev_ = nullptr;
  mutable std::vector<uint64_t> words_, fv_node_;
  mutable std::vector<float> values_;
  mutable std::vector<uint32_t> fv_feat_;
};

// ---- the Messenger-level application (SURVEY.md section 8f-2) ---------------------------------------------------------------------
// `gslam play b200_features [metric_time -slam b200] -dataset x.synth`: subscribes "dataset/frame" (published by the reference's
// player, GSLAM/plugins/play/main.cpp:15,126-132), runs the GPU feature path on every frame -- ORB extract on each camera of the
// frame, MapFrame::setKeyPoints (Map.h:311), Hamming match against the previous frame, row-band stereo match for two-camera frames
// -- and publishes the frame on "<name>/curframe", the topic GSLAM's own latency tool listens to
// (GSLAM/evaluation/metric_time/main.cpp:11-21), plus the associations on "<name>/matches".
int runFeatures(GSLAM::Svar config) {
  const std::string name = config.arg<std::string>("name", "b200", "topic prefix: frames leave on <name>/curframe, matches on <name>/matches");
  const int nfeatures = config.arg<int>("nfeatures", 2000, "ORB keypoints per image");
  const bool do_match = config.arg<bool>("match", true, "Hamming-match every frame against the previous one");
  const double band = config.arg<double>("stereo_band", 2.0, "row band (pixels) of the stereo association");
  const double max_disp = config.arg<double>("stereo_max_disparity", 128.0, "largest accepted disparity (pixels)");
  if (config.get("help", false)) return config.help();
  GSLAM::Svar cfg = GSLAM::Svar::object();
  cfg["nfeatures"] = nfeatures;
  GSLAM::Publisher pub_cur = messenger.advertise<GSLAM::FramePtr>(name + "/curframe", 0);
  GSLAM::Publisher pub_match = messenger.advertise<GSLAM::Svar>(name + "/matches", 0);
  GSLAM::GImage prev_desc;
  std::mutex mu;
  GSLAM::Subscriber sub = messenger.subscribe("dataset/frame", 0, [&](GSLAM::FramePtr fr) {
    if (!fr || !fr->cameraNum()) return;
    std::lock_guard<std::mutex> lk(mu);
    std::vector<GSLAM::KeyPoint> kps, kps_r;
    GSLAM::GImage desc, desc_r;
    if (!extract(fr->getImage(0, GSLAM::IMAGE_GRAY), cfg, kps, desc)) return;
    fr->setKeyPoints(kps, desc);  // Map.h:311-312
    GSLAM::Svar out = GSLAM::Svar::object();
    out["id"] = (int)fr->id();
    out["keypoints"] = (int)kps.size();
    gb_ctx* ctx = shared().get();
    if (fr->cameraNum() > 1 && ctx && extract(fr->getImage(1, GSLAM::IMAGE_GRAY), cfg, kps_r, desc_r)) {
      std::vector<int> idx(kps.size()), d1(kps.size()), d2(kps.size());
      if (gb_match_stereo(ctx, reinterpret_cast<const gb_keypoint*>(kps.data()), desc.data, (int)kps.size(), reinterpret_cast<const gb_keypoint*>(kps_r.data()),
                          desc_r.data, (int)kps_r.size(), (float)band, 0.f, (float)max_disp, idx.data(), d1.data(), d2.data()) == GB_OK) {
        out["stereoIdx"] = idx;
        out["stereoDistance"] = d1;
      } else {
        LOG(ERROR) << "gslam_b200 b200_features: " << gb_last_error(ctx);
      }
    }
    if (do_match && ctx && !prev_desc.empty() && !desc.empty()) {
      std::vector<int> idx(desc.rows), d1(desc.rows), d2(desc.rows);
      if (gb_match_hamming(ctx, desc.data, desc.rows, prev_desc.data, prev_desc.rows, idx.data(), d1.data(), d2.data()) == GB_OK) {
        out["trainIdx"] = idx;
        out["distance"] = d1;
        out["distance2"] = d2;
      } else {
        LOG(ERROR) << "gslam_b200 b200_features: " << gb_last_error(ctx);
      }
    }
    prev_desc = desc;
    pub_match.publish(out);
    pub_cur.publish(fr);
  });
  LOG(INFO) << "gslam_b200 b200_features ready: dataset/frame -> " << name << "/curframe";
  return GSLAM::Messenger::exec();  // until "messenger/stop" (Messenger.h:610-620)
}

}  // namespace

EXPORT_SVAR_INSTANCE
REGISTER_SVAR_MODULE(b200) {
  GSLAM_REGISTER_GLOG_SINKS
  GSLAM_REGISTER_MESSENGER
  svar["gslam"]["b200"]["orb_extract"] = GSLAM::Svar::lambda([](GSLAM::GImage img, GSLAM::Svar cfg) -> GSLAM::Svar {
    std::vector<GSLAM::KeyPoint> kps;
    GSLAM::GImage desc;
    if (!extract(img, cfg, kps, desc)) return GSLAM::Svar();
    GSLAM::Svar out = GSLAM::Svar::object();
    out["keypoints"] = kps;
    out["descriptors"] = desc;
    return out;
  });
  svar["gslam"]["b200"]["match_hamming"] = GSLAM::Svar::lambda([](GSLAM::GImage q, GSLAM::GImage t) -> GSLAM::Svar {
    if (q.cols != 32 || (t.rows > 0 && t.cols != 32) || q.elemSize() != 1 || (t.rows > 0 && t.elemSize() != 1)) {
      LOG(ERROR) << "gslam_b200 match_hamming: descriptors must be N x 32 8UC1";
      return GSLAM::Svar();
    }
    gb_ctx* ctx = shared().get();
    if (!ctx) return GSLAM::Svar();
    std::vector<int> idx(q.rows), d1(q.rows), d2(q.rows);
    if (gb_match_hamming(ctx, q.data, q.rows, t.data, t.rows, idx.data(), d1.data(), d2.data()) != GB_OK) {
      LOG(ERROR) << "gslam_b200 match_hamming: " << gb_last_error(ctx);
      return GSLAM::Svar();
    }
    GSLAM::Svar out = GSLAM::Svar::object();
    out["trainIdx"] = idx;
    out["distance"] = d1;
    out["distance2"] = d2;
    return out;
  });
  svar["gslam"]["apps"]["b200_features"] = GSLAM::SvarFunction(runFeatures);  // (what GSLAM_REGISTER_APPLICATION would register, GSLAM.h:26-33)
  svar["gslam"]["b200"]["match_stereo"] = GSLAM::Svar::lambda([](std::vector<GSLAM::KeyPoint> kl, GSLAM::GImage dl, std::vector<GSLAM::KeyPoint> kr,
                                                                   GSLAM::GImage dr, GSLAM::Svar cfg) -> GSLAM::Svar {
    if ((int)kl.size() != dl.rows || (int)kr.size() != dr.rows || (dl.rows > 0 && (dl.cols != 32 || dl.elemSize() != 1)) ||
        (dr.rows > 0 && (dr.cols != 32 || dr.elemSize() != 1))) {
      LOG(ERROR) << "gslam_b200 match_stereo: keypoints / N x 32 8UC1 descriptors of the two images do not fit together";
      return GSLAM::Svar();
    }
    gb_ctx* ctx = shared().get();
    if (!ctx) return GSLAM::Svar();
    const double band = cfg.isObject() ? cfg.get<double>("band", 2.0) : 2.0, mind = cfg.isObject() ? cfg.get<double>("minDisparity", 0.0) : 0.0,
                 maxd = cfg.isObject() ? cfg.get<double>("maxDisparity", 1e9) : 1e9;
    std::vector<int> idx(kl.size()), d1(kl.size()), d2(kl.size());
    if (gb_match_stereo(ctx, reinterpret_cast<const gb_keypoint*>(kl.data()), dl.data, (int)kl.size(), reinterpret_cast<const gb_keypoint*>(kr.data()), dr.data,
                        (int)kr.size(), (float)band, (float)mind, (float)maxd, idx.data(), d1.data(), d2.data()) != GB_OK) {
      LOG(ERROR) << "gslam_b200 match_stereo: " << gb_last_error(ctx);
      return GSLAM::Svar();
    }
    GSLAM::Svar out = GSLAM::Svar::object();
    out["rightIdx"] = idx;
    out["distance"] = d1;
    out["distance2"] = d2;
    return out;
  });
  // undistort(image, camera_in, camera_out) -> image: GSLAM::Undistorter::undistort (GSLAM/core/Undistorter.h:271-348) with the table
  // of the reference's own prepareReMap (:120-203; every camera model stays the reference's) applied on the device.  The table of the
  // last camera pair is kept resident in HBM.
  svar["gslam"]["b200"]["undistort"] = GSLAM::Svar::lambda([](GSLAM::GImage img, GSLAM::Camera in, GSLAM::Camera out) -> GSLAM::GImage {
    static std::mutex mtx;
    static std::string cached_key;
    static gb_remap* cached_map = nullptr;  // lives as long as the process-wide context it was created on
    if (img.empty() || (img.channels() != 1 && img.channels() != 3) || img.elemSize1() != 1 || !in.isValid() || !out.isValid() ||
        img.cols != in.width() || img.rows != in.height()) {
      LOG(ERROR) << "gslam_b200 undistort: needs an 8-bit 1- or 3-channel image of camera_in's size and two valid cameras";
      return GSLAM::GImage();
    }
    gb_ctx* ctx = shared().get();
    if (!ctx) return GSLAM::GImage();
    std::lock_guard<std::mutex> lk(mtx);
    const std::string key = in.info() + "|" + out.info();
    if (cached_key != key || !cached_map) {
      if (cached_map) gb_remap_destroy(ctx, cached_map);
      cached_map = nullptr;
      GSLAM::UndistorterImpl table(in, out);
      if (!table.valid || gb_remap_create(ctx, in.width(), in.height(), out.width(), out.height(), table.remapIdx, table.remapCoef, table.remapX,
                                          &cached_map) != GB_OK) {
        LOG(ERROR) << "gslam_b200 undistort: " << gb_last_error(ctx);
        return GSLAM::GImage();
      }
      cached_key = key;
    }
    GSLAM::GImage result(out.height(), out.width(), img.type());
    if (gb_remap_apply(ctx, cached_map, img.data, img.channels(), result.data) != GB_OK) {
      LOG(ERROR) << "gslam_b200 undistort: " << gb_last_error(ctx);
      return GSLAM::GImage();
    }
    return result;
  });
  svar["gslam"]["b200"]["vocabulary"] = GSLAM::Svar::lambda([](std::shared_ptr<GSLAM::Vocabulary> src) -> std::shared_ptr<GSLAM::Vocabulary> {
    if (!src) return std::shared_ptr<GSLAM::Vocabulary>();
    return std::shared_ptr<GSLAM::Vocabulary>(new B200Vocabulary(*src));
  });
  svar["gslam"]["b200"]["extract_to_frame"] = GSLAM::Svar::lambda([](GSLAM::FramePtr fr, GSLAM::Svar cfg) -> bool {
    if (!fr) return false;
    std::vector<GSLAM::KeyPoint> kps;
    GSLAM::GImage desc;
    if (!extract(fr->getImage(), cfg, kps, desc)) return false;
    return fr->setKeyPoints(kps, desc);  // Map.h:311-312
  });
}
