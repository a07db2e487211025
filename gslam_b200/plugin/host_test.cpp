// gslam_b200/plugin/host_test.cpp -> gslam_b200_host_test
//
// A stand-in for a GSLAM SLAM plugin: it uses ONLY the reference's public API (Optimizer::create, Registry::load, Svar calls,
// BundleGraph, GImage, KeyPoint) to drive the GPU backends, reading a case from a binary file and writing the results back,
// so the Python tests can compare the plugin-level outputs with the oracle.  Usage:
//   gslam_b200_host_test ba   <plugin-dir> in.bin out.bin      optimize(BundleGraph&) through GSLAM::Optimizer::create()
//   gslam_b200_host_test pnp  <plugin-dir> in.bin out.bin      optimizePnP(...)
//   gslam_b200_host_test orb  <plugin-dir> in.bin out.bin      Registry::load("b200") -> gslam.b200.orb_extract + match_hamming
//   gslam_b200_host_test findpnp <plugin-dir> in.bin out.bin   Estimator::create() -> findPnP (P3P + RANSAC), Estimator.h:158-164
//   gslam_b200_host_test dataset <plugin-dir> x.synth out.bin  GSLAM::Dataset::open -> libgslamDB_synth.so -> grabFrame (Dataset.h:124-162)
//   gslam_b200_host_test features <plugin-dir> x.synth out.bin dataset/frame -> gslam.apps.b200_features -> b200/curframe (Messenger)
//   gslam_b200_host_test undistort <plugin-dir> in.bin out.bin  gslam.b200.undistort next to the reference's own GSLAM::Undistorter
//   gslam_b200_host_test bow <plugin-dir> in.bin out.bin        gslam.b200.vocabulary(Vocabulary::create(...))->transform next to the
//                                                               reference's own Vocabulary::transform (Vocabulary.h:1558-1622)
// Trailing "key=value" arguments become svar settings the plugins read (b200.devices=0,1 shards a global BA over two GPUs).
#include <GSLAM/core/GSLAM.h>
#include <GSLAM/core/Dataset.h>
#include <GSLAM/core/Estimator.h>
#include <GSLAM/core/Optimizer.h>
#include <GSLAM/core/Undistorter.h>
#include <GSLAM/core/Vocabulary.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <fstream>
#include <sstream>
#include <vector>

using namespace GSLAM;

template <typename T>
static void rd(std::ifstream& f, T* p, size_t n) { f.read(reinterpret_cast<char*>(p), sizeof(T) * n); }
template <typename T>
static void wr(std::ofstream& f, const T* p, size_t n) { f.write(reinterpret_cast<const char*>(p), sizeof(T) * n); }

static int runBA(const std::string& dir, const char* in, const char* out, bool pnp) {
  svar.Set<std::string>("GSLAM_LIBRARY_PATH", dir);  // Registry search path is a svar variable, not process env (Registry.h:95-131)
  OptimizerPtr opt = Optimizer::create();             // default name "libgslam_optimizer" (Optimizer.h:237)
  if (!opt) { fprintf(stderr, "Optimizer::create() returned null\n"); return 2; }
  std::ifstream f(in, std::ios::binary);
  int32_t hdr[8];
  rd(f, hdr, 8);
  const int nc = hdr[0], np = hdr[1], no = hdr[2], iters = hdr[3], has_info = hdr[4];
  double ftol; rd(f, &ftol, 1);
  svar.Set<double>("b200.ftol", ftol);
  opt->_config.maxIterations = iters;
  std::vector<double> pose(7 * (size_t)nc), pts(3 * (size_t)np), xyz(3 * (size_t)no), info(has_info ? 4 * (size_t)no : 0);
  std::vector<uint8_t> dof(nc), pf(np);
  std::vector<int32_t> oc(no), op(no);
  rd(f, pose.data(), pose.size()); rd(f, dof.data(), dof.size()); rd(f, pts.data(), pts.size()); rd(f, pf.data(), pf.size());
  rd(f, oc.data(), oc.size()); rd(f, op.data(), op.size()); rd(f, xyz.data(), xyz.size());
  if (has_info) rd(f, info.data(), info.size());
  // optional pose-graph terms (Optimizer.h:127-148): hdr[5] SE3 edges, hdr[6] GPS edges, hdr[7] != 0: 6x6 information matrices follow
  const int nse = hdr[5], ngps = hdr[6], pinfo = hdr[7];
  std::vector<int32_t> sa(nse), sb(nse), gf(ngps);
  std::vector<double> sm(7 * (size_t)nse), si(pinfo ? 36 * (size_t)nse : 0), gm(7 * (size_t)ngps), gi(pinfo ? 36 * (size_t)ngps : 0);
  rd(f, sa.data(), sa.size()); rd(f, sb.data(), sb.size()); rd(f, sm.data(), sm.size()); rd(f, si.data(), si.size());
  rd(f, gf.data(), gf.size()); rd(f, gm.data(), gm.size()); rd(f, gi.data(), gi.size());
  bool ok;
  std::ofstream o(out, std::ios::binary);
  if (pnp) {
    std::vector<std::pair<Point3d, CameraAnchor> > matches(no);
    for (int k = 0; k < no; ++k)
      matches[k] = std::make_pair(Point3d(pts[3 * op[k]], pts[3 * op[k] + 1], pts[3 * op[k] + 2]), CameraAnchor(xyz[3 * k], xyz[3 * k + 1], xyz[3 * k + 2]));
    SE3 T(SO3(pose[0], pose[1], pose[2], pose[3]), Point3d(pose[4], pose[5], pose[6]));
    double information[36];
    ok = opt->optimizePnP(matches, T, (KeyFrameEstimzationDOF)dof[0], information);
    double p[7] = {T.get_rotation().x, T.get_rotation().y, T.get_rotation().z, T.get_rotation().w, T.get_translation().x, T.get_translation().y, T.get_translation().z};
    int32_t okv = ok; wr(o, &okv, 1); wr(o, p, 7); wr(o, information, 36);
    return ok ? 0 : 1;
  }
  BundleGraph g;
  g.keyframes.resize(nc); g.mappoints.resize(np); g.mappointObserves.resize(no);
  for (int i = 0; i < nc; ++i) {
    const double* p = &pose[7 * i];
    g.keyframes[i].estimation = SIM3(SE3(SO3(p[0], p[1], p[2], p[3]), Point3d(p[4], p[5], p[6])), 1.0 + 0.01 * i);  // scales must survive
    g.keyframes[i].dof = (KeyFrameEstimzationDOF)dof[i];
  }
  for (int j = 0; j < np; ++j) g.mappoints[j] = MapPointEstimation(Point3d(pts[3 * j], pts[3 * j + 1], pts[3 * j + 2]), pf[j] != 0);
  for (int k = 0; k < no; ++k) {
    BundleEdge& e = g.mappointObserves[k];
    e.pointId = op[k]; e.frameId = oc[k]; e.measurement = CameraAnchor(xyz[3 * k], xyz[3 * k + 1], xyz[3 * k + 2]);
    e.information = has_info ? &info[4 * (size_t)k] : NULL;
  }
  g.se3Graph.resize(nse); g.gpsGraph.resize(ngps);
  for (int k = 0; k < nse; ++k) {
    const double* p = &sm[7 * (size_t)k];
    g.se3Graph[k].firstId = sa[k]; g.se3Graph[k].secondId = sb[k];
    g.se3Graph[k].measurement = SE3(SO3(p[0], p[1], p[2], p[3]), Point3d(p[4], p[5], p[6]));
    g.se3Graph[k].information = pinfo ? &si[36 * (size_t)k] : NULL;
  }
  for (int k = 0; k < ngps; ++k) {
    const double* p = &gm[7 * (size_t)k];
    g.gpsGraph[k].frameId = gf[k];
    g.gpsGraph[k].measurement = SE3(SO3(p[0], p[1], p[2], p[3]), Point3d(p[4], p[5], p[6]));
    g.gpsGraph[k].information = pinfo ? &gi[36 * (size_t)k] : NULL;
  }
  g.cameraDOF = UPDATE_CAMERA_NONE;
  ok = opt->optimize(g);
  int32_t okv = ok; wr(o, &okv, 1);
  for (int i = 0; i < nc; ++i) {
    const SE3& T = g.keyframes[i].estimation.get_se3();
    double p[8] = {T.get_rotation().x, T.get_rotation().y, T.get_rotation().z, T.get_rotation().w, T.get_translation().x, T.get_translation().y, T.get_translation().z,
                   g.keyframes[i].estimation.get_scale()};
    wr(o, p, 8);
  }
  for (int j = 0; j < np; ++j) { double p[3] = {g.mappoints[j].first.x, g.mappoints[j].first.y, g.mappoints[j].first.z}; wr(o, p, 3); }
  return ok ? 0 : 1;
}

static int runORB(const std::string& dir, const char* in, const char* out) {
  svar.Set<std::string>("GSLAM_LIBRARY_PATH", dir);
  Svar mod = Registry::load("b200");  // dlopen + svarInstance() (Registry.h:48-77)
  if (mod.isUndefined()) { fprintf(stderr, "Registry::load(\"b200\") failed\n"); return 2; }
  Svar orb = mod["gslam"]["b200"]["orb_extract"], match = mod["gslam"]["b200"]["match_hamming"];
  std::ifstream f(in, std::ios::binary);
  int32_t hdr[4];
  rd(f, hdr, 4);
  const int w = hdr[0], h = hdr[1], nfeat = hdr[2];
  GImage a(h, w, GImageType<uchar, 1>::Type), b(h, w, GImageType<uchar, 1>::Type);
  rd(f, a.data, (size_t)w * h); rd(f, b.data, (size_t)w * h);
  Svar cfg = Svar::object();
  cfg["nfeatures"] = nfeat;
  Svar ra = orb(a, cfg), rb = orb(b, cfg);
  if (ra.isUndefined() || rb.isUndefined()) return 1;
  std::vector<KeyPoint> ka = ra["keypoints"].castAs<std::vector<KeyPoint> >(), kb = rb["keypoints"].castAs<std::vector<KeyPoint> >();
  GImage da = ra["descriptors"].castAs<GImage>(), db = rb["descriptors"].castAs<GImage>();
  Svar m = match(db, da);
  if (m.isUndefined()) return 1;
  std::vector<int> idx = m["trainIdx"].castAs<std::vector<int> >(), d1 = m["distance"].castAs<std::vector<int> >(), d2 = m["distance2"].castAs<std::vector<int> >();
  std::ofstream o(out, std::ios::binary);
  int32_t n[2] = {(int32_t)ka.size(), (int32_t)kb.size()};
  wr(o, n, 2);
  wr(o, ka.data(), ka.size()); wr(o, da.data, (size_t)da.rows * 32);
  wr(o, kb.data(), kb.size()); wr(o, db.data, (size_t)db.rows * 32);
  wr(o, idx.data(), idx.size()); wr(o, d1.data(), d1.size()); wr(o, d2.data(), d2.size());
  return 0;
}

// in : int32 w, h, channels, n_in_params, n_out_params, 3 x pad; doubles camera_in params, doubles camera_out params; image bytes
// out: int32 w_out, h_out, channels, mismatching_inside_pixels; plugin image bytes; reference image bytes; inside mask bytes
// The plugin's output and the reference's own Undistorter::undistort run side by side in this process (the reference is a header).
static int runUndistort(const std::string& dir, const char* in, const char* out) {
  svar.Set<std::string>("GSLAM_LIBRARY_PATH", dir);
  Svar mod = Registry::load("b200");
  if (mod.isUndefined()) { fprintf(stderr, "Registry::load(\"b200\") failed\n"); return 2; }
  Svar und = mod["gslam"]["b200"]["undistort"];
  std::ifstream f(in, std::ios::binary);
  int32_t hdr[8];
  rd(f, hdr, 8);
  const int w = hdr[0], h = hdr[1], ch = hdr[2];
  std::vector<double> pi(hdr[3]), po(hdr[4]);
  rd(f, pi.data(), pi.size()); rd(f, po.data(), po.size());
  Camera cin(pi), cout_(po);
  // (one spare row behind the image: the reference's last-row taps read there)
  std::vector<uchar> buf((size_t)w * (h + 2) * ch, 0);
  rd(f, buf.data(), (size_t)w * h * ch);
  GImage img(h, w, ch == 1 ? GImageType<uchar, 1>::Type : GImageType<uchar, 3>::Type, buf.data(), false);
  Svar r = und(img, cin, cout_);
  if (!r.is<GImage>()) return 1;
  GImage mine = r.castAs<GImage>();
  if (mine.empty()) return 1;
  Svar again = und(img, cin, cout_);  // the cached table
  if (std::memcmp(again.castAs<GImage>().data, mine.data, (size_t)mine.total() * mine.elemSize()) != 0) return 3;
  UndistorterImpl ref(cin, cout_);
  GImage want;
  if (!ref.undistort(img, want)) return 4;
  const int wo = cout_.width(), ho = cout_.height();
  std::vector<uchar> inside((size_t)wo * ho);
  int32_t bad = 0;
  for (int i = 0; i < wo * ho; ++i) {
    inside[i] = ch == 1 ? !(ref.remapX[i] < 0) : (ref.remapX[i] > 0);
    if (inside[i] && std::memcmp(mine.data + (size_t)i * ch, want.data + (size_t)i * ch, ch) != 0) ++bad;
  }
  std::ofstream o(out, std::ios::binary);
  int32_t oh[4] = {wo, ho, ch, bad};
  wr(o, oh, 4);
  wr(o, mine.data, (size_t)wo * ho * ch); wr(o, want.data, (size_t)wo * ho * ch); wr(o, inside.data(), inside.size());
  return 0;
}

// in : int32 k, L, weighting, scoring, n_nodes, n_query, levelsup, pad; child counts (uint32 x n_nodes), weights (float x n_nodes), node
//      descriptors (n_nodes x 32 bytes), queries (n_query x 32 bytes)
// out: int32 equal_bow, equal_fv, equal_bow_only_overload, n_words, n_fv_nodes, microseconds reference, microseconds plugin, pad;
//      words (uint64 x n_words), values (float x n_words)
// The tree enters the REFERENCE class through its own binary loader (Vocabulary::load(std::istream&), Vocabulary.h:1890-1930), is
// handed to the plugin as the VocabularyPtr any GSLAM code holds, and both objects transform the same descriptors in this process;
// the std::maps must compare equal, key for key and float for float.  (Training stays out of this program: Vocabulary::create leaves
// the descriptor rows of unused cluster slots uninitialised, so a tree trained in a fresh process differs from one trained elsewhere.)
static int runBow(const std::string& dir, const char* in, const char* out) {
  svar.Set<std::string>("GSLAM_LIBRARY_PATH", dir);
  Svar mod = Registry::load("b200");
  if (mod.isUndefined()) { fprintf(stderr, "Registry::load(\"b200\") failed\n"); return 2; }
  std::ifstream f(in, std::ios::binary);
  int32_t hdr[8];
  rd(f, hdr, 8);
  const int k = hdr[0], L = hdr[1], nq = hdr[5], levelsup = hdr[6];
  const uint32_t nnodes = (uint32_t)hdr[4];
  std::vector<uint32_t> child(nnodes);
  std::vector<float> weight(nnodes);
  std::vector<uchar> desc((size_t)nnodes * 32);
  rd(f, child.data(), child.size()); rd(f, weight.data(), weight.size()); rd(f, desc.data(), desc.size());
  TinyMat q(nq, 32, GImageType<uchar, 1>::Type, nullptr, false, 32);
  rd(f, q.data, (size_t)nq * 32);
  std::shared_ptr<Vocabulary> ref(new Vocabulary());
  {
    std::stringstream ss;
    const uint64_t sig = 88877711233ull;
    const bool compressed = false;
    Vocabulary::ScoringType sc = (Vocabulary::ScoringType)hdr[3];
    Vocabulary::WeightingType we = (Vocabulary::WeightingType)hdr[2];
    const int cols = 32, rows = 1, type = GImageType<uchar, 1>::Type;
    ss.write((const char*)&sig, sizeof sig); ss.write((const char*)&compressed, sizeof compressed); ss.write((const char*)&nnodes, sizeof nnodes);
    ss.write((const char*)&k, sizeof k); ss.write((const char*)&L, sizeof L); ss.write((const char*)&sc, sizeof sc); ss.write((const char*)&we, sizeof we);
    ss.write((const char*)&cols, sizeof cols); ss.write((const char*)&rows, sizeof rows); ss.write((const char*)&type, sizeof type);
    std::vector<Vocabulary::Node> nodes(nnodes);
    for (uint32_t i = 0; i < nnodes; ++i) { nodes[i].childNum = child[i]; nodes[i].weight = weight[i]; }
    ss.write((const char*)nodes.data(), sizeof(Vocabulary::Node) * nnodes);
    ss.write((const char*)desc.data(), desc.size());
    if (!ref->load(ss)) return 3;
  }
  Svar made = mod["gslam"]["b200"]["vocabulary"](ref);
  std::shared_ptr<Vocabulary> dev;
  try { dev = made.castAs<std::shared_ptr<Vocabulary> >(); } catch (...) { return 4; }  // (Svar holds shared_ptr<T> as a pointer holder of T, Svar.h:2834-2850)
  if (!dev || dev->size() != ref->size()) return 5;
  BowVector v0, v1, v2, v3;
  FeatureVector f0, f1;
  dev->transform(q, v1, f1, levelsup);  // (first call uploads the tree)
  auto t0 = std::chrono::steady_clock::now();
  for (int r = 0; r < 20; ++r) ref->transform(q, v0, f0, levelsup);
  auto t1 = std::chrono::steady_clock::now();
  for (int r = 0; r < 20; ++r) dev->transform(q, v1, f1, levelsup);
  auto t2 = std::chrono::steady_clock::now();
  ref->transform(q, v2);
  dev->transform(q, v3);
  // the untouched parts of the interface still answer from the same tree
  WordId w0, w1; WordValue a0, a1;
  ref->transform(q.row(0), w0, a0);
  dev->transform(q.row(0), w1, a1);
  if (w0 != w1 || a0 != a1 || dev->getWordWeight(w1) != ref->getWordWeight(w0) || dev->getEffectiveLevels() != ref->getEffectiveLevels()) return 6;
  if (v1.empty()) { fprintf(stderr, "bow: reference %zu words, plugin %zu words, vocabulary %u words, %d query rows x %d cols\n", v0.size(), v1.size(), dev->size(), q.rows, q.cols); return 7; }
  std::ofstream o(out, std::ios::binary);
  int32_t oh[8] = {v0 == v1, f0 == f1, v2 == v3, (int32_t)v1.size(), (int32_t)f1.size(),
                   (int32_t)(std::chrono::duration<double>(t1 - t0).count() / 20 * 1e6), (int32_t)(std::chrono::duration<double>(t2 - t1).count() / 20 * 1e6), 0};
  wr(o, oh, 8);
  for (auto& it : v1) { uint64_t w = it.first; wr(o, &w, 1); }
  for (auto& it : v1) { float x = it.second; wr(o, &x, 1); }
  return 0;
}

// in : int32 n, 3 x int32 pad, double threshold, double confidence, n x 3 doubles (world points), n x 2 doubles (normalised image points)
// out: int32 ok, 7 doubles world2camera {qx,qy,qz,qw,tx,ty,tz}, n bytes mask
static int runFindPnP(const std::string& dir, const char* in, const char* out) {
  svar.Set<std::string>("GSLAM_LIBRARY_PATH", dir);
  EstimatorPtr est = Estimator::create();  // default name "libgslam_estimator" (Estimator.h:181)
  if (!est) { fprintf(stderr, "Estimator::create() returned null\n"); return 2; }
  std::ifstream f(in, std::ios::binary);
  int32_t hdr[4];
  rd(f, hdr, 4);
  const int n = hdr[0];
  double thr, conf;
  rd(f, &thr, 1); rd(f, &conf, 1);
  std::vector<double> xyz(3 * (size_t)n), xy(2 * (size_t)n);
  rd(f, xyz.data(), xyz.size()); rd(f, xy.data(), xy.size());
  std::vector<Point3d> obj(n);
  std::vector<Point2d> img(n);
  for (int k = 0; k < n; ++k) { obj[k] = Point3d(xyz[3 * k], xyz[3 * k + 1], xyz[3 * k + 2]); img[k] = Point2d(xy[2 * k], xy[2 * k + 1]); }
  SE3 w2c;
  std::vector<uchar> mask;
  const bool ok = est->findPnP(&w2c, obj, img, P3_ITERATIVE & RANSAC, thr, conf, &mask);
  std::ofstream o(out, std::ios::binary);
  const int32_t okv = ok ? 1 : 0;
  wr(o, &okv, 1);
  const SO3& r = w2c.get_rotation();
  const Point3d& t = w2c.get_translation();
  const double p[7] = {r.x, r.y, r.z, r.w, t.x, t.y, t.z};
  wr(o, p, 7);
  mask.resize((size_t)n, 0);
  wr(o, mask.data(), mask.size());
  return ok ? 0 : 3;
}

// Dataset through the reference's loader: GSLAM::Dataset::open("x.synth") -> Registry::load("gslamDB_synth") (Dataset.h:124-162).
// out: int32 n_frames, cams, w, h, then for every frame and camera w*h bytes.
static int runDataset(const std::string& dir, const char* in, const char* out) {
  svar.Set<std::string>("GSLAM_LIBRARY_PATH", dir);
  Dataset ds;
  if (!ds.open(in)) { fprintf(stderr, "Dataset::open(%s) failed\n", in); return 2; }
  std::ofstream o(out, std::ios::binary);
  std::vector<FramePtr> frames;
  while (FramePtr fr = ds.grabFrame()) frames.push_back(fr);
  if (frames.empty()) return 1;
  GImage im0 = frames[0]->getImage(0);
  int32_t hdr[4] = {(int32_t)frames.size(), frames[0]->cameraNum(), im0.cols, im0.rows};
  wr(o, hdr, 4);
  for (size_t k = 0; k < frames.size(); ++k)
    for (int c = 0; c < hdr[1]; ++c) {
      GImage im = frames[k]->getImage(c);
      wr(o, im.data, (size_t)im.cols * im.rows);
    }
  return 0;
}

// The Messenger-level pipeline, wired the way `gslam play b200_features -dataset x.synth` wires it (gslam/main.cpp:12-46,
// plugins/play/main.cpp:126-132): the app gslam.apps.b200_features of libgslam_b200.so runs on its own thread with OUR messenger
// injected; this thread plays the dataset onto "dataset/frame", listens on "b200/curframe" / "b200/matches" and finally publishes
// "messenger/stop".  out: int32 n_frames, then per frame: int32 id, int32 n_kp, n_kp x 28 B keypoints, n_kp x 32 B descriptors,
// int32 n_match, n_match x int32 trainIdx, int32 n_stereo, n_stereo x int32 stereoIdx.
static int runFeaturesApp(const std::string& dir, const char* in, const char* out) {
  svar.Set<std::string>("GSLAM_LIBRARY_PATH", dir);
  Svar mod = Registry::load("b200");
  if (mod.isUndefined()) { fprintf(stderr, "Registry::load(\"b200\") failed\n"); return 2; }
  Svar run = mod["gslam"]["apps"]["b200_features"];
  if (!run.isFunction()) { fprintf(stderr, "gslam.apps.b200_features missing\n"); return 2; }
  Svar setMsg = mod["gslam"]["setGlobalMessenger"], setLog = mod["gslam"]["setGlobalLogSinks"];
  if (setLog.isFunction()) setLog(getLogSinksGlobal());
  if (setMsg.isFunction()) setMsg(messenger);
  Dataset ds;
  if (!ds.open(in)) { fprintf(stderr, "Dataset::open(%s) failed\n", in); return 2; }
  std::mutex mu;
  std::vector<FramePtr> got;
  std::vector<Svar> matches;
  Subscriber s1 = messenger.subscribe("b200/curframe", 0, [&](FramePtr fr) { std::lock_guard<std::mutex> lk(mu); got.push_back(fr); });
  Subscriber s2 = messenger.subscribe("b200/matches", 0, [&](Svar m) { std::lock_guard<std::mutex> lk(mu); matches.push_back(m); });
  std::thread app([run]() { run(svar); });
  // wait until the app subscribed (it has no ready signal: poll the subscriber count of the topic)
  Publisher pub = messenger.advertise<FramePtr>("dataset/frame", 0);
  for (int spin = 0; spin < 2000 && pub.getNumSubscribers() == 0; ++spin) std::this_thread::sleep_for(std::chrono::milliseconds(5));
  int sent = 0;
  while (FramePtr fr = ds.grabFrame()) { pub.publish(fr); ++sent; }
  messenger.publish("messenger/stop", true);
  app.join();
  std::ofstream o(out, std::ios::binary);
  int32_t n = (int32_t)got.size();
  wr(o, &n, 1);
  for (size_t k = 0; k < got.size(); ++k) {
    std::vector<KeyPoint> kps;
    got[k]->getKeyPoints(kps);
    GImage d = got[k]->getDescriptor();
    int32_t h2[2] = {(int32_t)got[k]->id(), (int32_t)kps.size()};
    wr(o, h2, 2);
    wr(o, kps.data(), kps.size());
    if (d.rows) wr(o, d.data, (size_t)d.rows * 32);
    std::vector<int> idx, st;
    if (k < matches.size() && matches[k].exist("trainIdx")) idx = matches[k]["trainIdx"].castAs<std::vector<int> >();
    if (k < matches.size() && matches[k].exist("stereoIdx")) st = matches[k]["stereoIdx"].castAs<std::vector<int> >();
    int32_t nm = (int32_t)idx.size(), ns = (int32_t)st.size();
    wr(o, &nm, 1); wr(o, idx.data(), idx.size());
    wr(o, &ns, 1); wr(o, st.data(), st.size());
  }
  return (int)got.size() == sent ? 0 : 1;
}

int main(int argc, char** argv) {
  if (argc < 5) { fprintf(stderr, "usage: %s ba|pnp|orb|findpnp|dataset|undistort|features|bow <plugin-dir> in.bin out.bin\n", argv[0]); return 64; }
  // optional svar settings for the plugins, "key=value" (e.g. b200.devices=0,1  b200.multi_min_obs=1000)
  for (int i = 5; i < argc; ++i) {
    const std::string kv = argv[i];
    const size_t eq = kv.find('=');
    if (eq == std::string::npos) continue;
    const std::string key = kv.substr(0, eq), val = kv.substr(eq + 1);
    char* end = NULL;
    const long iv = strtol(val.c_str(), &end, 10);
    if (end && *end == 0 && !val.empty()) { svar.Set<int>(key, (int)iv); continue; }  // typed like `gslam -key value` would be read back
    const double dv = strtod(val.c_str(), &end);
    if (end && *end == 0 && !val.empty()) { svar.Set<double>(key, dv); continue; }
    svar.Set<std::string>(key, val);
  }
  const std::string mode = argv[1];
  if (mode == "ba") return runBA(argv[2], argv[3], argv[4], false);
  if (mode == "pnp") return runBA(argv[2], argv[3], argv[4], true);
  if (mode == "orb") return runORB(argv[2], argv[3], argv[4]);
  if (mode == "findpnp") return runFindPnP(argv[2], argv[3], argv[4]);
  if (mode == "dataset") return runDataset(argv[2], argv[3], argv[4]);
  if (mode == "undistort") return runUndistort(argv[2], argv[3], argv[4]);
  if (mode == "features") return runFeaturesApp(argv[2], argv[3], argv[4]);
  if (mode == "bow") return runBow(argv[2], argv[3], argv[4]);
  return 64;
}
