/*
 * gslam_b200.h — the C-ABI drop-in boundary of the H100 (sm_90a) backends for GSLAM's per-frame numeric hot path
 * (ORB extract -> 256-bit Hamming brute-force match -> GSLAM::Optimizer bundle adjustment).
 *
 * Plain C: opaque handles, plain pointers and sizes, `int` status returns, caller-owned output buffers.  No STL, no
 * Svar, no torch types.  Everything the reference-facing C++ plugins (under gslam_b200/plugin: `libgslam_optimizer.so`
 * exporting `createOptimizerInstance`, and the Svar module `libgslam_b200.so`) need is here; so is everything a
 * ctypes / cgo / JNI binding would need (INTEGRATION.md shows the stubs).
 *
 * Reference interfaces each entry point sits behind (paths relative to the GSLAM tree):
 *   gb_orb_extract      <- consumes GSLAM::GImage            GSLAM/core/GImage.h:160-443   (dense 8UC1, no row stride :378)
 *                          emits    GSLAM::KeyPoint           GSLAM/core/Map.h:122-195      (28-byte record, == gb_keypoint)
 *                          emits    N x 32 8UC1 descriptors   GSLAM/core/Map.h:311-312,321  (MapFrame::setKeyPoints/getDescriptor)
 *   gb_match_hamming    <- distance == Vocabulary::DistanceFactory::hamming32  GSLAM/core/Vocabulary.h:485-491
 *   gb_ba_solve         <- GSLAM::Optimizer::optimize(BundleGraph&)            GSLAM/core/Optimizer.h:229 (graph PODs :106-172)
 *   gb_ba_pnp           <- GSLAM::Optimizer::optimizePnP(matches, SE3&, dof, information)  GSLAM/core/Optimizer.h:202-207
 *   gb_ba_options       <- GSLAM::OptimzeConfig                                GSLAM/core/Optimizer.h:174-182
 *
 * Error behaviour mirrors the reference's plugin convention (Optimizer.h:193-232: every virtual returns bool, nothing
 * throws across the boundary): every function returns GB_OK (0) or a GB_ERR_* code and never throws; a human-readable
 * message is available from gb_last_error().  There is NO CPU fallback: without a usable CUDA device gb_ctx_create
 * fails with GB_ERR_NODEVICE and every compute entry point fails loudly.
 *
 * Threading: a gb_ctx owns one CUDA stream, its device buffers and pinned staging; calls on one ctx are serialised by an
 * internal mutex (the reference documents no re-entrancy guarantee, SURVEY.md §8b).  Use one ctx per calling thread for
 * concurrency (e.g. tracking thread: extract/match/pnp; mapping thread: local BA).
 */
#ifndef GSLAM_B200_H_
#define GSLAM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define GB_API __attribute__((visibility("default")))
#else
#define GB_API
#endif

#define GB_VERSION 100 /* major*100 + minor */

/* ---- status codes --------------------------------------------------------------------------------------------- */
enum {
  GB_OK = 0,
  GB_ERR_INVALID = 1,  /* bad argument / unsupported configuration                         */
  GB_ERR_CUDA = 2,     /* a CUDA runtime call or kernel failed (message in gb_last_error)  */
  GB_ERR_CAPACITY = 3, /* caller buffer too small; required size reported via the in/out n */
  GB_ERR_NODEVICE = 4, /* no usable CUDA device (there is no CPU fallback)                 */
  GB_ERR_NUMERIC = 5   /* solver produced a non-finite value                               */
};

typedef struct gb_ctx gb_ctx;           /* one device + one stream + cached buffers            */
typedef struct gb_features gb_features; /* a frame's keypoints + descriptors resident in HBM   */
typedef struct gb_ba_graph gb_ba_graph; /* a bundle-adjustment graph resident in HBM           */

/* ---- context ---------------------------------------------------------------------------------------------------- */
GB_API int gb_version(void);
GB_API int gb_device_count(int* n);
GB_API int gb_ctx_create(int device, gb_ctx** out);
/* high_priority != 0: the ctx's stream gets the device's greatest priority, so that its (few-CTA) kernels are scheduled ahead of
 * the big grids of another ctx on the same GPU -- the mapping ctx (local BA) of a tracking / mapping pair. */
GB_API int gb_ctx_create_priority(int device, int high_priority, gb_ctx** out);
GB_API int gb_ctx_destroy(gb_ctx* ctx);
/* Last error message of `ctx` (or of the calling thread when ctx==NULL).  Never NULL; valid until the next call. */
GB_API const char* gb_last_error(const gb_ctx* ctx);
/* The ctx's cudaStream_t (as void*) so a host can order its own work / record its own events on it. */
GB_API void* gb_ctx_stream(gb_ctx* ctx);
GB_API int gb_ctx_sync(gb_ctx* ctx);
/* Order `waiter`'s stream after everything enqueued so far on `producer`'s stream (same device; no host synchronisation): the
 * pipelining primitive between a tracking ctx (extract / match) and a mapping ctx (local BA). */
GB_API int gb_ctx_wait_for(gb_ctx* waiter, gb_ctx* producer);
/* CUDA-event stopwatch on the ctx stream (begin records an event; end records another, synchronises, returns ms). */
GB_API int gb_timer_begin(gb_ctx* ctx);
GB_API int gb_timer_end(gb_ctx* ctx, float* ms);
/* Number of kernels this ctx has launched so far (for bench.py's gpu_launches). */
GB_API int64_t gb_launch_count(const gb_ctx* ctx);

/* ---- ORB extract ------------------------------------------------------------------------------------------------ */
/* Field-for-field GSLAM::KeyPoint (Map.h:180-194) == cv::KeyPoint: 28 bytes. */
typedef struct gb_keypoint {
  float x, y;       /* pt: level coords * float(scale^octave)          */
  float size;       /* 31 * scale^octave                               */
  float angle;      /* degrees [0,360), intensity-centroid orientation */
  float response;   /* Harris response                                 */
  int32_t octave;   /* pyramid level                                   */
  int32_t class_id; /* -1                                              */
} gb_keypoint;

/* Same knobs (and defaults) as cv::ORB::create — the CPU path GSLAM's SLAM plugins call (SURVEY.md §8 a4, App. A). */
typedef struct gb_orb_cfg {
  int32_t nfeatures;      /* 500 in OpenCV; benchmarks use 1000 / 2000 */
  float scale_factor;     /* 1.2f                                       */
  int32_t nlevels;        /* 8   (1..GB_ORB_MAX_LEVELS)                 */
  int32_t edge_threshold; /* 31  (must be >= 22; see DESIGN.md)         */
  int32_t first_level;    /* 0   (only 0 supported)                     */
  int32_t wta_k;          /* 2   (only 2 supported)                     */
  int32_t score_type;     /* 0 = HARRIS_SCORE (only 0 supported)        */
  int32_t patch_size;     /* 31  (only 31 supported)                    */
  int32_t fast_threshold; /* 20                                         */
} gb_orb_cfg;
#define GB_ORB_MAX_LEVELS 12
/* A pyramid level keeps at most 4096 keypoints (its selection sorts in shared memory): the level's quota plus the keypoints tied with
 * the last one kept (equal Harris response) must be <= 4096, or the extraction fails with GB_ERR_CAPACITY instead of truncating
 * (cv::ORB has no such limit; the SLAM configurations of BASELINE.json use 1000 / 2000).  Level 0 has the largest quota: at the
 * default scale 1.2 and 8 levels it is 4096 at nfeatures = 18 862 and 4097 at 18 863, so frames without such ties extract up to
 * nfeatures = 18 862. */
GB_API void gb_orb_cfg_default(gb_orb_cfg* cfg);

/*
 * Host-buffer entry point (what the Svar plugin's orb_extract binds).  `img` is a dense 8UC1 GImage payload
 * (rows*cols bytes, row i at img + i*width, GImage.h:378), host memory, read-only.  On input *n is the capacity of `kps`
 * (records) and `desc` (rows of 32 bytes); on output the number of keypoints.  Output order is canonical:
 * ascending (octave, y, x) — OpenCV's own intra-level order is an artefact of std::nth_element (SURVEY.md App. A.3).
 * If more keypoints are kept than capacity (ties at the selection thresholds are kept, like OpenCV's retainBest) the
 * call returns GB_ERR_CAPACITY with *n = required capacity and writes nothing.
 */
GB_API int gb_orb_extract(gb_ctx* ctx, const uint8_t* img, int width, int height, const gb_orb_cfg* cfg,
                          gb_keypoint* kps, uint8_t* desc, int* n);

/* Colour frames (GSLAM's dataset plugins deliver 8UC3 / 8UC4, GSLAM/plugins/datasets/IO.h:86-110): channels = 1, 3 or 4 interleaved
 * bytes per pixel, rgb_order 0 = B,G,R[,A] (OpenCV / IMAGE_BGRA), 1 = R,G,B[,A]; the gray conversion is cv2.cvtColor's 8-bit fixed
 * point, fused into the level-0 upload on the device.  channels = 1 is gb_orb_extract. */
GB_API int gb_orb_extract_image(gb_ctx* ctx, const uint8_t* img, int width, int height, int channels, int rgb_order,
                                const gb_orb_cfg* cfg, gb_keypoint* kps, uint8_t* desc, int* n);

/* Device-resident variants: the frame and/or the results stay in HBM (bench `value`, chained pipelines). */
GB_API int gb_features_create(gb_ctx* ctx, int capacity, gb_features** out);
GB_API int gb_features_destroy(gb_ctx* ctx, gb_features* f);
/* img_is_device: 0 = host pointer (copied H2D through pinned staging), 1 = device pointer, `pitch` bytes per row. */
GB_API int gb_orb_extract_to(gb_ctx* ctx, const uint8_t* img, int img_is_device, int width, int height, int pitch,
                             const gb_orb_cfg* cfg, gb_features* out);
/* Blocks until the extraction on `f` finished; returns its keypoint count. */
GB_API int gb_features_count(gb_ctx* ctx, gb_features* f, int* n);
/* Replace the contents of `f` with caller-provided descriptors (and optional keypoints) — e.g. map-point descriptors. */
GB_API int gb_features_upload(gb_ctx* ctx, gb_features* f, const gb_keypoint* kps, const uint8_t* desc, int n);
GB_API int gb_features_download(gb_ctx* ctx, gb_features* f, gb_keypoint* kps, uint8_t* desc, int* n);

/* ---- 256-bit Hamming brute-force match ---------------------------------------------------------------------------- */
/*
 * For every query row q (32 bytes) find the train row with the smallest popcount(q XOR t) (== hamming32,
 * Vocabulary.h:485-491); ties -> lowest train index (cv::BFMatcher(NORM_HAMMING) semantics, SURVEY.md App. A.7).
 * best_idx[i] = argmin (-1 if nt==0), best_dist[i] = its distance, second_dist[i] = distance of the 2nd-nearest
 * neighbour in (distance, index) order (== knnMatch(k=2)[1].distance; 257 if nt<2).  Any output pointer may be NULL.
 */
GB_API int gb_match_hamming(gb_ctx* ctx, const uint8_t* query, int nq, const uint8_t* train, int nt, int32_t* best_idx,
                            int32_t* best_dist, int32_t* second_dist);
/* Device-resident: match fq against ft; results stay on device until gb_match_download.  Either set may be the output of an
 * extraction still in flight (gb_orb_extract_to): the match is then enqueued behind it and reads the row counts on the device.
 * gb_match_download: on input *n is the capacity of the (nullable) output arrays, on output the number of queries matched; when
 * that is more than the capacity it returns GB_ERR_CAPACITY and writes none of the arrays.  If the extraction of fq OR of ft
 * failed (more keypoints kept than the feature set holds, or an internal overflow) it returns GB_ERR_CAPACITY naming the failed
 * side, on every call, rather than matches against an empty set. */
GB_API int gb_match_features(gb_ctx* ctx, gb_features* fq, gb_features* ft);
GB_API int gb_match_download(gb_ctx* ctx, gb_features* fq, int32_t* best_idx, int32_t* best_dist, int32_t* second_dist,
                             int* n);

/*
 * Rectified-stereo row-band match (SURVEY.md section 8f-1; BASELINE config 4: EuRoC-shaped stereo 752x480): left = query,
 * right = train.  A right keypoint is a candidate of a left one iff |y_R - y_L| <= band_rows and
 * min_disparity <= x_L - x_R <= max_disparity (float compares on GSLAM::KeyPoint::pt, level-0 pixels, Map.h:180-194); among the
 * candidates the same distance (hamming32, Vocabulary.h:485-491), (distance, index) order and tie rule as gb_match_hamming.
 * best_idx = -1 / distances 257 when a left keypoint has no candidate.  The reference has no stereo matcher: this definition is
 * ours (DESIGN.md).  band_rows < 0 or NaN, or max_disparity < min_disparity: GB_ERR_INVALID.  Device-resident variant: results stay
 * with `left` until gb_match_download(left), which fails as above when the extraction of `left` or of `right` failed.
 */
GB_API int gb_match_stereo(gb_ctx* ctx, const gb_keypoint* kps_left, const uint8_t* desc_left, int n_left,
                           const gb_keypoint* kps_right, const uint8_t* desc_right, int n_right, float band_rows,
                           float min_disparity, float max_disparity, int32_t* best_idx, int32_t* best_dist, int32_t* second_dist);
GB_API int gb_match_stereo_features(gb_ctx* ctx, gb_features* left, gb_features* right, float band_rows, float min_disparity,
                                    float max_disparity);

/* ---- frame undistortion (SURVEY.md section 8f-4) -----------------------------------------------------------------------------------
 * The bilinear LUT remap of GSLAM::Undistorter::undistort (GSLAM/core/Undistorter.h:271-348).  The table is the reference's own
 * (UndistorterImpl::prepareReMap :120-203 -- remapIdx, remapCoef, remapX; the plugin builds it with the reference's camera models):
 * per output pixel four source pixel indices (row-major, in pixels, >= 0) and four float weights; remap_x < 0 marks output pixels
 * that fall outside the input image.  gb_remap_apply: src = w_in*h_in*channels bytes, dst = w_out*h_out*channels bytes, host
 * buffers, channels 1 or 3; out = p[i0]*c0 + p[i1]*c1 + p[i2]*c2 + p[i3]*c3 in float, left to right, truncated to uchar --
 * bit-identical to the reference wherever the reference is defined (taps beyond the input image count as 0; outside pixels are 0). */
typedef struct gb_remap gb_remap;
GB_API int gb_remap_create(gb_ctx* ctx, int w_in, int h_in, int w_out, int h_out, const int32_t* idx4, const float* coef4,
                           const float* remap_x, gb_remap** out);
GB_API int gb_remap_destroy(gb_ctx* ctx, gb_remap* map);
GB_API int gb_remap_apply(gb_ctx* ctx, gb_remap* map, const uint8_t* src, int channels, uint8_t* dst);

/* ---- bag-of-words transform (SURVEY.md section 8f-4) --------------------------------------------------------------------------------
 * GSLAM::Vocabulary::transform(features, BowVector&, FeatureVector&, levelsup)  (GSLAM/core/Vocabulary.h:1558-1622; tree walk
 * :1692-1736; distance hamming32 :485-491).  gb_voc_create uploads the reference's own flat tree (the public members
 * Vocabulary::m_k, m_L, m_weighting, m_scoring, m_nodes[].childNum / .weight, m_nodeDescriptors, :583-601): children of node p are rows
 * p*k+1 .. p*k+child_num[p] of desc32 (32-byte rows: ORB / 256-bit vocabularies), k <= 32; weighting / scoring are the reference's
 * enum values (:88-105).  gb_bow_transform: desc = n x 32 bytes (the N x 32 8UC1 descriptor GImage of MapFrame::getDescriptor,
 * Map.h:321), host memory.  Outputs, caller-owned, capacity n each: the BowVector (std::map<WordId,float>, :47) as parallel arrays
 * in map order (words ascending) and the FeatureVector (std::map<NodeId,std::vector<unsigned>>, :48) flattened in map order (node
 * ascending, feature indices ascending).  Word / node / feature indices are bit-exact with the reference; values are the reference's
 * floats, bit-exact for every vocabulary (accumulated with the same operations; the double L1 / L2 norm equals the reference's
 * sum in ascending word order).  One vocabulary may be used from any ctx on the device it was created on, from any thread: calls
 * on it are serialised by the vocabulary itself.  A leaf above level L - levelsup files under itself (the reference
 * reads an uninitialised node id there).  gb_bow_transform_features: the same for descriptors already resident in HBM (the output
 * of gb_orb_extract_to), no host round trip before the walk; the output arrays must hold the CAPACITY of `f` entries (the row
 * count of an extraction still in flight is only known on the device; the launch is clipped by it).  If that extraction failed
 * (more keypoints kept than `f` holds, or an internal overflow) it returns GB_ERR_CAPACITY with *n_words = *n_fv = 0, on every
 * call, rather than an empty BowVector. */
typedef struct gb_vocabulary gb_vocabulary;
GB_API int gb_voc_create(gb_ctx* ctx, int k, int L, int weighting, int scoring, uint32_t n_nodes, const uint32_t* child_num, const float* weight,
                         const uint8_t* desc32, gb_vocabulary** out);
GB_API int gb_voc_destroy(gb_ctx* ctx, gb_vocabulary* voc);
GB_API int gb_bow_transform(gb_ctx* ctx, gb_vocabulary* voc, const uint8_t* desc, int n, int levelsup, uint64_t* words, float* values, int* n_words,
                            uint64_t* fv_node, uint32_t* fv_feat, int* n_fv);
GB_API int gb_bow_transform_features(gb_ctx* ctx, gb_vocabulary* voc, gb_features* f, int levelsup, uint64_t* words, float* values, int* n_words,
                                     uint64_t* fv_node, uint32_t* fv_feat, int* n_fv);

/* ---- bundle adjustment ---------------------------------------------------------------------------------------------- */
/*
 * SoA mirror of GSLAM::BundleGraph's mappoint part (Optimizer.h:150-172).  The C++ plugin repacks the graph's AoS
 * vectors into these arrays (and back) — INTEGRATION.md.
 *   cam_pose_wc : n_cams x 7 doubles {qx,qy,qz,qw, tx,ty,tz} = the first 7 doubles of KeyFrameEstimzation::estimation
 *                 (SIM3 = SE3{SO3{x,y,z,w},Point3d} + scale, SE3.h:337-339, SIM3.h:290-291): T_wc, camera -> world
 *                 (Optimizer.h:117).  IN/OUT.
 *   cam_dof     : n_cams bytes, low 6 bits of KeyFrameEstimzationDOF (Optimizer.h:70-84): bit k frees component k of the
 *                 left tangent [v(3), w(3)] of T_cw.  0 = UPDATE_KF_NONE (fixed), 63 = UPDATE_KF_SE3.  NULL = all 63.
 *   points      : n_points x 3 world coordinates (MapPointEstimation.first, Optimizer.h:113-114).  IN/OUT.
 *   point_free  : n_points bytes, MapPointEstimation.second (true = NOT fixed).  NULL = all free.
 *   obs_cam/obs_point : BundleEdge::frameId / pointId (indices into the two arrays above, Optimizer.h:121-125).
 *   obs_xyz     : n_obs x 3, BundleEdge::measurement, a CameraAnchor (Optimizer.h:102-103); PROJECTION_PINHOLE uses
 *                 (x/z, y/z).
 *   obs_info    : n_obs x 4 row-major 2x2 information matrices, or NULL (= identity for every edge, the usual
 *                 BundleEdge::information == NULL case).
 */
typedef struct gb_ba_problem {
  int32_t n_cams, n_points, n_obs;
  double* cam_pose_wc;
  const uint8_t* cam_dof;
  double* points;
  const uint8_t* point_free;
  const int32_t* obs_cam;
  const int32_t* obs_point;
  const double* obs_xyz;
  const double* obs_info;
} gb_ba_problem;

/* Pose-graph terms of a BundleGraph (SURVEY.md section 8f-3): GSLAM::SE3Edge (Optimizer.h:127-133, BundleGraph::se3Graph :163-164) and
 * GSLAM::GPSEdge (:143-148, gpsGraph :167-168).  All indices are keyframe indices of the gb_ba_problem they accompany.
 *   se3_meas : n_se3 x 7 doubles, SE3_12 := SE3_1^-1 * SE3_2 (T_wc conventions, SE3 layout {qx,qy,qz,qw,tx,ty,tz});
 *   gps_meas : n_gps x 7 doubles, SE3_gps := SE3_frame (a prior on T_wc of the frame);
 *   *_info   : row-major 6x6 information matrices in the tangent order [v(3), w(3)] (SE3.h:205-262), one per edge, or NULL = identity.
 * Residual e = Log(Z^-1 * T_wc,1^-1 * T_wc,2) resp. Log(Z^-1 * T_wc), cost term e' Omega e (no robust kernel), Jacobians with the
 * first-order approximation of the logarithm's Jacobian (DESIGN.md section 5: our definition -- the reference fixes only the types). */
typedef struct gb_pose_edges {
  int32_t n_se3;
  const int32_t* se3_first;
  const int32_t* se3_second;
  const double* se3_meas;
  const double* se3_info;
  int32_t n_gps;
  const int32_t* gps_frame;
  const double* gps_meas;
  const double* gps_info;
} gb_pose_edges;

/* GSLAM::OptimzeConfig (Optimizer.h:174-182) + the solver knobs the reference leaves to its (absent) Ceres plugin.
 * A solve rejects (GB_ERR_INVALID) negative integer knobs, a lambda_init that is not finite and > 0, and a NaN huber_delta,
 * function_tolerance or pcg_tol.  max_iterations = 0 runs no LM iteration and reports the cost at the input estimate. */
typedef struct gb_ba_options {
  int32_t projection;       /* 0 = PROJECTION_PINHOLE (only 0 supported)                               */
  double huber_delta;       /* projectErrorHuberThreshold, 0.01 (normalised units); <=0 disables Huber */
  int32_t max_iterations;   /* LM iterations (linear solves), reference default 500                    */
  int32_t verbose;          /* print one line per iteration to stderr                                  */
  double function_tolerance;/* stop when |dcost|/cost < tol after an accepted step (1e-6); 0 = never   */
  double lambda_init;       /* initial LM damping, 1e-4                                                 */
  int32_t pcg_max_iters;    /* block-Jacobi PCG iteration cap on the reduced camera system, 50         */
  double pcg_tol;           /* stop when sqrt(r'z / r0'z0) < tol, 1e-10                                 */
  int32_t linear_solver;    /* 0 = block-Jacobi PCG on the reduced camera system (default); 1 = DIRECT: block-skyline Cholesky
                               (exact solve; local-BA sizes: the skyline must fit one SM's shared memory, single GPU)       */
} gb_ba_options;
GB_API void gb_ba_options_default(gb_ba_options* opt);

typedef struct gb_ba_result {
  double initial_cost; /* 0.5 * sum rho(e^2) at the input estimate (Ceres convention) */
  double final_cost;   /* ... at the returned estimate                                */
  int32_t iterations;  /* LM iterations performed (linear solves)                     */
  int32_t accepted;    /* of which accepted                                           */
  int32_t pcg_iterations; /* total PCG iterations                                     */
  int32_t status;      /* 0 = iteration cap, 1 = function tolerance, 2 = no progress (lambda overflow) */
  double lambda_final;
  float gpu_ms;        /* device time of the solve (CUDA events on the ctx stream)    */
} gb_ba_result;

/* Host-buffer entry point (what libgslam_optimizer.so's optimize() binds): uploads, solves, writes poses/points back. */
GB_API int gb_ba_solve(gb_ctx* ctx, gb_ba_problem* problem, const gb_ba_options* opt, gb_ba_result* result);
/* The same for a BundleGraph that carries SE3 / GPS edges (BundleGraph::se3Graph / gpsGraph, Optimizer.h:163-168): a pose graph
 * (n_points == n_obs == 0) or a bundle adjustment with pose-graph terms.  edges == NULL or empty == gb_ba_solve. */
GB_API int gb_ba_solve_posegraph(gb_ctx* ctx, gb_ba_problem* problem, const gb_pose_edges* edges, const gb_ba_options* opt, gb_ba_result* result);

/*
 * Pose-only refinement from 3D-2D matches (Optimizer::optimizePnP, Optimizer.h:202-207).
 *   xyz: n x 3 world points; xy1: n x 3 CameraAnchor measurements; pose_wc: 7 doubles IN/OUT (SE3 layout, T_wc);
 *   dof: KeyFrameEstimzationDOF low 6 bits; info6x6: NULL, or 36 doubles that RECEIVE the row-major 6x6 information
 *   (Gauss-Newton Hessian sum w J'J, undamped, tangent order [v,w] of T_cw) of the returned pose.  The reference leaves
 *   the meaning of this non-const `double* information` unspecified; an output is the reading we fix (DESIGN.md).
 */
GB_API int gb_ba_pnp(gb_ctx* ctx, int n, const double* xyz, const double* xy1, double* pose_wc, int dof,
                     double* info6x6, const gb_ba_options* opt, gb_ba_result* result);

/* Device-resident graph: upload once (host-side ordering + H2D), solve many times from the same initial estimate. */
GB_API int gb_ba_graph_create(gb_ctx* ctx, const gb_ba_problem* problem, gb_ba_graph** out);
/* ... with pose-graph terms (`edges` may be NULL); such a graph runs the stepwise solver on the dense reduced camera system */
GB_API int gb_ba_graph_create_ex(gb_ctx* ctx, const gb_ba_problem* problem, const gb_pose_edges* edges, gb_ba_graph** out);
GB_API int gb_ba_graph_destroy(gb_ctx* ctx, gb_ba_graph* g);
GB_API int gb_ba_graph_reset(gb_ctx* ctx, gb_ba_graph* g); /* restore the uploaded estimate (device-to-device) */
GB_API int gb_ba_graph_solve(gb_ctx* ctx, gb_ba_graph* g, const gb_ba_options* opt, gb_ba_result* result);
GB_API int gb_ba_graph_download(gb_ctx* ctx, gb_ba_graph* g, double* cam_pose_wc, double* points);
/* One fused residual + Jacobian sweep at the current estimate (K6: V, g_p, W, U, g_c, cost stay on the device) — the
 * "BA Jacobian-eval" of the BASELINE metric in isolation; enqueued on the ctx stream, no host synchronisation. */
GB_API int gb_ba_graph_sweep(gb_ctx* ctx, gb_ba_graph* g, double huber_delta);

/*
 * Stepwise interface for landmark-sharded multi-GPU global BA (SURVEY.md §8e): every rank holds all cameras and a
 * shard of the landmarks with all their edges.  One LM iteration is
 *   gb_ba_graph_reduce_local   : linearise the shard at the current estimate (if needed), form the shard's Schur
 *                                contribution into `d_buf` (device, gb_ba_graph_reduce_size doubles):
 *                                [ S (6n x 6n, undamped) | g~ (6n) | diag U (6n) | cost (1) | pad ]
 *   <all-reduce d_buf across ranks, sum, f64 — the path's single exchange step; the host does it with NCCL>
 *   gb_ba_graph_step           : damp, block-Jacobi PCG on the reduced camera system (replicated, deterministic),
 *                                back-substitute the shard's landmarks, build the candidate estimate and write the
 *                                shard's candidate cost to d_cost[0] (device)
 *   <all-reduce d_cost (1 double)>
 *   gb_ba_graph_commit         : accept/reject on the device from the reduced costs, update lambda.
 * No host synchronisation is needed between the calls.
 */
GB_API int gb_ba_graph_reduce_size(gb_ctx* ctx, gb_ba_graph* g, size_t* n_doubles);
GB_API int gb_ba_graph_begin(gb_ctx* ctx, gb_ba_graph* g, const gb_ba_options* opt);
GB_API int gb_ba_graph_reduce_local(gb_ctx* ctx, gb_ba_graph* g, double* d_buf);
GB_API int gb_ba_graph_step(gb_ctx* ctx, gb_ba_graph* g, const double* d_buf, double* d_cost);
GB_API int gb_ba_graph_commit(gb_ctx* ctx, gb_ba_graph* g, const double* d_buf, const double* d_cost);
GB_API int gb_ba_graph_finish(gb_ctx* ctx, gb_ba_graph* g, gb_ba_result* result);

/* =====================================================================================================================
 * Pose from 3D-2D matches with outliers: minimal P3P solver + RANSAC + non-linear refinement.
 * Sits behind GSLAM::Estimator::findPnP(SE3* world2camera, objectPoints, imagePoints, method = P3_ITERATIVE&RANSAC,
 * threshold = 0.01, confidence = 0.99, mask)  GSLAM/core/Estimator.h:158-164 (factory createEstimatorInstance :43-45,175-191);
 * SURVEY.md section 8f-1.  Mirrors the CPU checker operation for operation (tests/test_pnp_gpu.py).
 *   xyz: n x 3 world points; xy: n x 2 normalised image points (x/z, y/z);
 *   threshold: inlier bound on the normalised reprojection error; confidence in (0,1); max_hypotheses >= 1; seed: any;
 *   pose_cw: 7 doubles OUT, world->camera as the reference signature asks, layout {qx,qy,qz,qw,tx,ty,tz};
 *   mask: NULL or n bytes OUT (1 = inlier of the returned pose).
 * Definition (deterministic, independent of how many hypotheses run in parallel): hypothesis h draws its three matches from
 * splitmix64(seed, h); best = (most inliers, lowest h, lowest root); hypotheses count in batches of 64 and stop at the first batch
 * boundary with h >= log(1-confidence)/log(1-w^3), w the best inlier ratio so far; the winner is refined by the optimizePnP solver
 * on its inliers and kept if it loses none.  GB_ERR_NUMERIC when no pose reaches 4 inliers. */
typedef struct gb_pnp_stats {
  int32_t hypotheses;       /* hypotheses that counted (a multiple of 64, or max_hypotheses) */
  int32_t best_hypothesis;  /* index of the winning hypothesis, -1 if none */
  int32_t best_root;        /* which P3P solution of that hypothesis */
  int32_t inliers_minimal;  /* inliers of the winning minimal solution */
  int32_t inliers_refined;  /* inliers of the returned pose */
} gb_pnp_stats;
GB_API int gb_pnp_ransac(gb_ctx* ctx, int n, const double* xyz, const double* xy, double threshold, double confidence,
                         int max_hypotheses, uint64_t seed, double* pose_cw, uint8_t* mask, gb_pnp_stats* stats);

/* =====================================================================================================================
 * Multi-GPU global bundle adjustment (SURVEY.md section 8e; BASELINE config 5: 500 cameras / 100k landmarks / 1M observations).
 * Still behind GSLAM::Optimizer::optimize(BundleGraph&) (GSLAM/core/Optimizer.h:229): the landmarks (and all their edges) are
 * sharded over the ranks, every rank holds all cameras; per LM iteration ONE all-reduce (f64 sum over NVLink, NCCL bound at run
 * time with dlopen) of the shard contributions to the compact reduced camera system [S in covisibility block-CSR | g~ | diag U |
 * cost], then a replicated, bit-identical block-CSR PCG (so every rank takes the same LM decisions), the shard's
 * back-substitution and a 1-double all-reduce of the candidate cost.  No host synchronisation inside the loop.
 *
 * Two front ends over the same engine:
 *   one process per GPU : gb_comm_unique_id on rank 0, the host distributes the 128 bytes (torch.distributed broadcast, MPI,
 *                         a file ...), every rank calls gb_comm_create; then gb_ba_shard_create / _solve / gb_ba_graph_download.
 *   one process, N GPUs : gb_comm_create_all over N contexts, gb_ba_solve_multi(problem) -- one host thread per device inside;
 *                         this is what libgslam_optimizer.so's optimize() calls when the svar option `b200.devices` names
 *                         several devices.
 * A communicator of world size 1 needs no NCCL and makes every call below a single-GPU call. */
typedef struct gb_comm gb_comm;
#define GB_COMM_ID_BYTES 128
GB_API int gb_comm_unique_id(uint8_t* id128);
GB_API int gb_comm_create(gb_ctx* ctx, int world, int rank, const uint8_t* id128, gb_comm** out);
GB_API int gb_comm_create_all(int n_dev, gb_ctx* const* ctxs, gb_comm** out /* [n_dev] */);
GB_API int gb_comm_destroy(gb_comm* comm);
GB_API int gb_comm_rank(const gb_comm* comm);
GB_API int gb_comm_world(const gb_comm* comm);
/* In-place f64 sum over the ranks, enqueued on the communicator's ctx stream. */
GB_API int gb_comm_allreduce_sum_f64(gb_comm* comm, double* d_buf, size_t n);
/* The rank's shard of `full` (every rank passes the SAME full problem): a contiguous landmark range balanced by observation
 * count, all cameras, the covisibility block structure of the whole graph.  Needs <= 2048 cameras. */
GB_API int gb_ba_shard_create(gb_comm* comm, const gb_ba_problem* full, gb_ba_graph** out);
/* Landmarks [lo, hi) of the full problem live on this rank; gb_ba_graph_download returns exactly those (hi-lo) x 3 points. */
GB_API int gb_ba_shard_range(const gb_ba_graph* g, int* lo, int* hi);
GB_API int gb_ba_shard_reduce_bytes(const gb_ba_graph* g, size_t* bytes); /* size of the per-iteration all-reduce */
GB_API int gb_ba_shard_solve(gb_comm* comm, gb_ba_graph* g, const gb_ba_options* opt, gb_ba_result* result);
/* Shard, solve and write poses / points back into `problem` (gpu_ms = max over the devices). */
GB_API int gb_ba_solve_multi(int n_dev, gb_comm* const* comms, gb_ba_problem* problem, const gb_ba_options* opt,
                             gb_ba_result* result);

#ifdef __cplusplus
}
#endif
#endif /* GSLAM_B200_H_ */
