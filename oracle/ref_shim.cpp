// oracle/ref_shim.cpp — NOT a restatement: a thin extern "C" window onto the UNMODIFIED reference headers, compiled from
// where they lie in the GSLAM checkout named by REF into oracle/_ref/libgslam_ref.so (recipe: oracle/Makefile, target `ref`).
// TEST INFRASTRUCTURE ONLY.  It pins the parts of the hot path that DO exist in the reference tree:
//   * Vocabulary::DistanceFactory::hamming32          GSLAM/core/Vocabulary.h:485-491
//   * SE3 inverse / point transform / product / exp / log   GSLAM/core/SE3.h:100-131,205-287  (pose conventions of BA)
//   * sizeof / layout of the carrier PODs             Map.h:122-195, Optimizer.h:106-172, SE3.h:337-339, SIM3.h:290-291
//   * Undistorter::undistort + the remap table of prepareReMap   GSLAM/core/Undistorter.h:120-348 (the frame-undistortion row)
//   * Vocabulary::create / load / transform (BoW + feature vector)  GSLAM/core/Vocabulary.h:1051-1130,1890-1930,1558-1736 (the BoW row)
// No reference source is copied into this repository; the .so is git-ignored.
#include <cstring>
#include <GSLAM/core/GSLAM.h>
#include <GSLAM/core/Optimizer.h>
#include <GSLAM/core/Vocabulary.h>
#include <GSLAM/core/Undistorter.h>
#include <sstream>

using namespace GSLAM;

static SE3 mk(const double* p) { return SE3(SO3(p[0], p[1], p[2], p[3]), Point3d(p[4], p[5], p[6])); }
static void put(const SE3& T, double* o) {
  const SO3& r = T.get_rotation();
  const Point3d& t = T.get_translation();
  o[0] = r.x; o[1] = r.y; o[2] = r.z; o[3] = r.w; o[4] = t.x; o[5] = t.y; o[6] = t.z;
}

extern "C" {
__attribute__((visibility("default"))) float ref_hamming32(const unsigned char* a, const unsigned char* b) {
  return Vocabulary::DistanceFactory::hamming32(a, b);
}
__attribute__((visibility("default"))) void ref_se3_inverse(const double* pose7, double* out7) { put(mk(pose7).inverse(), out7); }
__attribute__((visibility("default"))) void ref_se3_transform(const double* pose7, const double* p3, double* out3) {
  Point3d q = mk(pose7) * Point3d(p3[0], p3[1], p3[2]);
  out3[0] = q.x; out3[1] = q.y; out3[2] = q.z;
}
__attribute__((visibility("default"))) void ref_se3_mul(const double* a7, const double* b7, double* out7) { put(mk(a7) * mk(b7), out7); }
__attribute__((visibility("default"))) void ref_se3_exp(const double* d6, double* out7) {
  Vector<double, 6> v;
  for (int i = 0; i < 6; ++i) v[i] = d6[i];
  put(SE3::exp(v), out7);
}
__attribute__((visibility("default"))) void ref_se3_log(const double* pose7, double* out6) {
  Vector<double, 6> v = mk(pose7).log();
  for (int i = 0; i < 6; ++i) out6[i] = v[i];
}
// The in-memory layout the BA boundary relies on: SIM3 = {SO3{x,y,z,w}, Point3d, scale} as 8 contiguous doubles.
__attribute__((visibility("default"))) void ref_sim3_raw(const double* pose7, double scale, double* out8) {
  SIM3 s(mk(pose7), scale);
  static_assert(sizeof(SIM3) == 64, "SIM3 layout");
  std::memcpy(out8, &s, 64);
}
__attribute__((visibility("default"))) int ref_sizeof(const char* name) {
  if (!std::strcmp(name, "KeyPoint")) return sizeof(KeyPoint);
  if (!std::strcmp(name, "SE3")) return sizeof(SE3);
  if (!std::strcmp(name, "SIM3")) return sizeof(SIM3);
  if (!std::strcmp(name, "Point3d")) return sizeof(Point3d);
  if (!std::strcmp(name, "BundleEdge")) return sizeof(BundleEdge);
  if (!std::strcmp(name, "KeyFrameEstimzation")) return sizeof(KeyFrameEstimzation);
  if (!std::strcmp(name, "MapPointEstimation")) return sizeof(MapPointEstimation);
  if (!std::strcmp(name, "GImage")) return sizeof(GImage);
  return -1;
}
// field offsets of KeyPoint, to prove gb_keypoint is field-compatible
__attribute__((visibility("default"))) int ref_keypoint_offsets(int* o7) {
  KeyPoint k;
  char* b = (char*)&k;
  o7[0] = (char*)&k.pt.x - b; o7[1] = (char*)&k.pt.y - b; o7[2] = (char*)&k.size - b; o7[3] = (char*)&k.angle - b;
  o7[4] = (char*)&k.response - b; o7[5] = (char*)&k.octave - b; o7[6] = (char*)&k.class_id - b;
  return 7;
}

// The reference's undistorter, run as is: cameras from parameter vectors (Camera.h:435-444), tables from prepareReMap, output from
// undistort().  tables: idx4 / coef4 / remap_x may be NULL; out may be NULL.  Returns 0 when both cameras are valid.
__attribute__((visibility("default"))) int ref_undistort(const double* cam_in, int n_in, const double* cam_out, int n_out, const unsigned char* img,
                                                         int channels, int* idx4, float* coef4, float* remap_x, unsigned char* out) {
  Camera in(std::vector<double>(cam_in, cam_in + n_in)), outc(std::vector<double>(cam_out, cam_out + n_out));
  if (!in.isValid() || !outc.isValid()) return 1;
  UndistorterImpl u(in, outc);  // (prepareReMap prints the two camera models on stdout)
  if (!u.valid) return 2;
  const size_t n = (size_t)outc.width() * outc.height();
  if (idx4) std::memcpy(idx4, u.remapIdx, n * 16);
  if (coef4) std::memcpy(coef4, u.remapCoef, n * 16);
  if (remap_x) std::memcpy(remap_x, u.remapX, n * 4);
  if (img && out) {
    // the reference reads up to one row + one pixel past the end of the image for taps of the last row: let it read zeros from a
    // padded buffer it does not own (GImage.h:169, copy = false) -- which is the value the product defines for those taps
    const size_t bytes = (size_t)in.width() * in.height() * channels;
    std::vector<unsigned char> padded(bytes + (size_t)(in.width() + 2) * channels, 0);
    std::memcpy(padded.data(), img, bytes);
    GImage src(in.height(), in.width(), channels == 1 ? GImageType<uchar, 1>::Type : GImageType<uchar, 3>::Type, padded.data(), false);
    GImage dst;
    if (!u.undistort(src, dst)) return 3;
    std::memcpy(out, dst.data, n * channels);
  }
  return 0;
}

// ---- the reference's vocabulary, run as is (BoW row) ---------------------------------------------------------------------------
// ref_voc_train: Vocabulary::create (hierarchical k-medians + idf weights) on n_images x per_image 32-byte descriptors.
// ref_voc_from_arrays: any tree, through the reference's own binary loader (Vocabulary::load(std::istream&), :1890-1930).
__attribute__((visibility("default"))) void* ref_voc_train(const unsigned char* desc, int n_images, int per_image, int k, int L, int weighting, int scoring) {
  std::vector<TinyMat> imgs;
  for (int i = 0; i < n_images; ++i) {
    TinyMat m(per_image, 32, GImageType<uchar, 1>::Type, nullptr, false, 32);
    std::memcpy(m.data, desc + (size_t)i * per_image * 32, (size_t)per_image * 32);
    imgs.push_back(m);
  }
  std::shared_ptr<Vocabulary> v = Vocabulary::create(imgs, k, L, (Vocabulary::WeightingType)weighting, (Vocabulary::ScoringType)scoring);
  return v ? new std::shared_ptr<Vocabulary>(v) : nullptr;
}
__attribute__((visibility("default"))) void* ref_voc_from_arrays(int k, int L, int weighting, int scoring, unsigned nnodes, const unsigned* child_num,
                                                                const float* weight, const unsigned char* desc32) {
  std::stringstream ss;
  const uint64_t sig = 88877711233ull;
  const bool compressed = false;
  ss.write((const char*)&sig, sizeof sig); ss.write((const char*)&compressed, sizeof compressed); ss.write((const char*)&nnodes, sizeof nnodes);
  Vocabulary::ScoringType sc = (Vocabulary::ScoringType)scoring; Vocabulary::WeightingType we = (Vocabulary::WeightingType)weighting;
  ss.write((const char*)&k, sizeof k); ss.write((const char*)&L, sizeof L); ss.write((const char*)&sc, sizeof sc); ss.write((const char*)&we, sizeof we);
  const int cols = 32, rows = 1, type = GImageType<uchar, 1>::Type;
  ss.write((const char*)&cols, sizeof cols); ss.write((const char*)&rows, sizeof rows); ss.write((const char*)&type, sizeof type);
  std::vector<Vocabulary::Node> nodes(nnodes);
  for (unsigned i = 0; i < nnodes; ++i) { nodes[i].childNum = child_num[i]; nodes[i].weight = weight[i]; }
  ss.write((const char*)nodes.data(), sizeof(Vocabulary::Node) * nnodes);
  ss.write((const char*)desc32, (size_t)nnodes * 32);
  std::shared_ptr<Vocabulary> v(new Vocabulary());
  if (!v->load(ss)) return nullptr;
  return new std::shared_ptr<Vocabulary>(v);
}
__attribute__((visibility("default"))) void ref_voc_destroy(void* h) { delete (std::shared_ptr<Vocabulary>*)h; }
__attribute__((visibility("default"))) int ref_voc_info(void* h, int* k, int* L, int* weighting, int* scoring) {
  Vocabulary& v = **(std::shared_ptr<Vocabulary>*)h;
  *k = v.m_k; *L = v.m_L; *weighting = (int)v.m_weighting; *scoring = (int)v.m_scoring;
  return (int)v.m_nodes.size();
}
__attribute__((visibility("default"))) void ref_voc_export(void* h, unsigned* child_num, float* weight, unsigned char* desc32) {
  Vocabulary& v = **(std::shared_ptr<Vocabulary>*)h;
  for (size_t i = 0; i < v.m_nodes.size(); ++i) { child_num[i] = v.m_nodes[i].childNum; weight[i] = v.m_nodes[i].weight; }
  std::memcpy(desc32, v.m_nodeDescriptors.data, v.m_nodes.size() * 32);
}
// Vocabulary::transform(features, BowVector&, FeatureVector&, levelsup) (:1558-1622).  words/values: the BowVector in map order;
// fv_node/fv_feat: the FeatureVector flattened in map order (node ascending, feature indices in insertion order).
__attribute__((visibility("default"))) int ref_voc_transform(void* h, const unsigned char* feats, int n, int levelsup, unsigned long long* words, float* values,
                                                             int* n_words, unsigned long long* fv_node, unsigned* fv_feat, int* n_fv, int repeat,
                                                             double* seconds) {
  Vocabulary& v = **(std::shared_ptr<Vocabulary>*)h;
  TinyMat f(n, 32, GImageType<uchar, 1>::Type, nullptr, false, 32);
  std::memcpy(f.data, feats, (size_t)n * 32);
  BowVector bv; FeatureVector fv;
  auto t0 = std::chrono::steady_clock::now();
  for (int r = 0; r < (repeat > 0 ? repeat : 1); ++r) v.transform(f, bv, fv, levelsup);
  if (seconds) *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() / (repeat > 0 ? repeat : 1);
  int a = 0, b = 0;
  for (auto& it : bv) { if (words) { words[a] = it.first; values[a] = it.second; } ++a; }
  for (auto& it : fv) for (unsigned idx : it.second) { if (fv_node) { fv_node[b] = it.first; fv_feat[b] = idx; } ++b; }
  *n_words = a; *n_fv = b;
  return 0;
}
// one descriptor down the tree (:1692-1736): word id, weight, node id `levelsup` levels above the leaf
__attribute__((visibility("default"))) void ref_voc_transform_one(void* h, const unsigned char* feat, int levelsup, unsigned long long* word, float* weight,
                                                                 unsigned long long* node) {
  Vocabulary& v = **(std::shared_ptr<Vocabulary>*)h;
  TinyMat f(1, 32, GImageType<uchar, 1>::Type, nullptr, false, 32);
  std::memcpy(f.data, feat, 32);
  WordId w; WordValue val; NodeId nid = (NodeId)-1;
  v.transform(f, w, val, &nid, levelsup);
  *word = w; *weight = val; *node = nid;
}
}
