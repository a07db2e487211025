// gslam_b200/csrc/ba_sweep.cu — the residual + Jacobian sweep of LARGE bundle-adjustment graphs (global BA, BASELINE config 5:
// 500 cameras / 100k landmarks / 1M observations) behind GSLAM::Optimizer::optimize (GSLAM/core/Optimizer.h:229).
//
// Same arithmetic per observation as ba.cu's ba_linearize_kernel (ba_device.cuh: eval_obs / jac_cam / jac_pt; oracle:
// oracle/ba_ref.c), different machine mapping — the local-BA kernel is latency-tuned for 10k observations, this one is
// throughput-tuned: the sweep reads 24 B and writes one 144-byte W block per observation (168 B/observation, SURVEY.md §8d).
//
//   * ONE persistent launch, one 512-thread CTA per SM = FOUR independent 128-thread teams (named barriers) that share one copy
//     of the pose table T_cw (R row-major + t, 96 B per camera, <= 512 cameras) and the dof masks in SHARED memory: an
//     observation's pose is six LDS.128 instead of six L1 tag look-ups per lane (every lane of a warp reads a different camera).
//   * work items are cut and dealt to the teams ON THE HOST at graph creation (static, balanced by a cost model: a team's list =
//     some cameras, then a contiguous run of landmark groups), so a team knows its next items in advance: the record of item n+2
//     and the DATA of item n+1 (camera index / landmark index / measurement of its 128 observations, the landmarks' coordinates,
//     offsets and free flags: cp.async into a double-buffered shared-memory stage) are in flight while item n is computed.  The
//     dependent load chain item -> offsets -> observation -> point that left the first version of this kernel waiting on the long
//     scoreboard for 46 % of its cycles is gone from the critical path.
//   * landmark item = a run of consecutive landmarks with <= 128 observations: ONE LANE PER OBSERVATION (the 8-lanes-per-landmark
//     mapping of ba.cu idles 38 % of the lane rounds at 10 observations per landmark).  The 6x3 W block goes to a shared-memory
//     tile that is contiguous in the global W array and leaves the SM as ONE bulk asynchronous copy
//     (cp.async.bulk.global.shared::cta — the TMA engine: no LDS/STG instructions, no L1 wavefronts; `UBLKCP` in SASS).  The ten
//     per-observation terms of V_j / g_p,j / cost_j are summed per landmark from shared memory in ascending observation order
//     -> bit-reproducible, and the same order as the oracle.
//   * camera item = one camera (or one slice of a camera with > 8192 observations): the team strides its camera-sorted
//     observation list with the next iteration's indices / point prefetched, 27 accumulators per thread, folded through shared
//     memory in a fixed order (no atomics).  Sliced cameras: last-slice-folds, as in ba.cu.
#include <algorithm>

#include "ba_device.cuh"
#include "ba_internal.cuh"
#include "common.cuh"

using namespace ba;

namespace {

constexpr int kTeam = 128;       // threads per team = observations per landmark chunk
constexpr int kTeams = 4;        // teams per CTA
constexpr int kSwThreads = kTeam * kTeams;
constexpr int kSwMaxPts = 32;    // landmarks per group (host plan)
constexpr int kSwPoseCams = 512; // pose table in shared memory up to this many cameras
constexpr int kPoseStride = 14;  // doubles per camera row of the shared-memory table (12 used): an ODD number of 16-byte chunks, so that
                                 // the rows of a warp's 32 different cameras spread over all eight chunk slots of the banks (12 -> only four)

// one stage of prefetched item data, in doubles
constexpr int kStUv = 0;                         // [128] double2
constexpr int kStPts = kStUv + 2 * kTeam;        // [32][3] landmark coordinates
constexpr int kStCam = kStPts + 3 * kSwMaxPts;   // [128] int camera of the observation
constexpr int kStPt = kStCam + kTeam / 2;        // [128] int landmark of the observation
constexpr int kStOff = kStPt + kTeam / 2;        // [33] int pt_off[j0 ..j1]
constexpr int kStPf = kStOff + 18;               // [<= 36] bytes point_free[j0 & ~3 ...]
constexpr int kStage = kStPf + 6;
// one team's region, in doubles
constexpr int kOffW = 0;                               // [128][18]  W tile (bulk-copy source, 16-byte aligned)
constexpr int kOffC = kOffW + kTeam * 18;              // [10][128]  per-observation V / g_p / cost terms, term-major
constexpr int kOffAcc = kOffC + kTeam * 10;            // [32][10]   per-landmark sums of the group; camera fold result [27]
constexpr int kOffStage = kOffAcc + kSwMaxPts * 10;    // [2] stages
constexpr int kOffMisc = kOffStage + 2 * kStage;       // flag
constexpr int kRecs = 32;                              // item records of the team kept in shared memory
constexpr int kOffRec = kOffMisc + 4;                  // [32] int4
constexpr int kTeamDoubles = kOffRec + 2 * kRecs;
static_assert(kTeam * 28 >= 27 * kTeam, "camera fold scratch spans the W and contribution tiles");
static_assert((kTeamDoubles % 2) == 0 && (kStage % 2) == 0, "16-byte alignment of the team regions and stages");
constexpr int kOffPose = kTeams * kTeamDoubles;        // [nc][12] pose table, then [nc] dof bytes (POSE_SMEM)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bulk_store(void* gdst, const void* ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
template <int BYTES>
__device__ __forceinline__ void cp_async(void* sdst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(smem_u32(sdst)), "l"(gsrc), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void team_sync(int team) { asm volatile("bar.sync %0, %1;" ::"r"(team + 1), "n"(kTeam) : "memory"); }

template <bool POSE_SMEM>
__device__ __forceinline__ void load_rt(const double* __restrict__ table, int i, double* Rt) {
  const double2* src = reinterpret_cast<const double2*>(table + (POSE_SMEM ? kPoseStride : 12) * (size_t)i);
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    const double2 v = POSE_SMEM ? src[k] : __ldg(src + k);
    Rt[2 * k] = v.x; Rt[2 * k + 1] = v.y;
  }
}

struct SweepCtx {
  const double* pose_tab;  // shared (POSE_SMEM) or global
  const uint8_t* dof_tab;
  const double* PTS;
  bool pend;
  double delta;
};

// issue the asynchronous copies of a landmark item's chunk [c0, c0 + 128) into `st` (thread t: observation c0 + t; the first
// threads also copy the group's landmark rows / offsets / free flags when `head`)
__device__ __forceinline__ void stage_fill(const BaDev& g, const SweepCtx& cx, double* st, int t, int j0, int j1, int c0, int e1, bool head) {
  const int e = c0 + t;
  if (e < e1) {
    cp_async<16>(st + kStUv + 2 * t, g.o_uv + 2 * (size_t)e);
    cp_async<4>(reinterpret_cast<int*>(st + kStCam) + t, g.o_cam + e);
    cp_async<4>(reinterpret_cast<int*>(st + kStPt) + t, g.o_pt + e);
  }
  if (head) {
    const int L = j1 - j0;
    if (t < 3 * L) cp_async<8>(st + kStPts + t, cx.PTS + 3 * (size_t)j0 + t);
    if (t <= L) cp_async<4>(reinterpret_cast<int*>(st + kStOff) + t, g.pt_off + j0 + t);
    const int w0 = j0 >> 2, nw = ((j1 + 3) >> 2) - w0;  // the words of point_free covering [j0, j1)
    if (t < nw) cp_async<4>(reinterpret_cast<int*>(st + kStPf) + t, reinterpret_cast<const int*>(g.pfree) + w0 + t);
  }
  cp_async_commit();
}

// ---- landmark item: landmarks [j0, j1), observations [e0, e1) in chunks of 128; chunk 0 is already staged in `st` ---------------
template <bool POSE_SMEM>
__device__ __forceinline__ void sweep_landmarks(const BaDev& g, const SweepCtx& cx, double* tm, double* st, int team, int t, int j0, int j1, int e0, int e1) {
  double* s_w = tm + kOffW;
  double* s_c = tm + kOffC;
  double* s_acc = tm + kOffAcc;
  const int* s_cam = reinterpret_cast<const int*>(st + kStCam);
  const int* s_pt = reinterpret_cast<const int*>(st + kStPt);
  const int* s_off = reinterpret_cast<const int*>(st + kStOff);
  const uint8_t* s_pf = reinterpret_cast<const uint8_t*>(st + kStPf) + (j0 & 3);
  const double* s_pts = st + kStPts;
  const int L = j1 - j0;
  for (int c0 = e0; c0 < e1 || c0 == e0; c0 += kTeam) {
    if (c0 != e0) {  // (a landmark with more observations than one chunk) later chunks are fetched in place
      if (t == 0) bulk_wait_read();
      team_sync(team);  // the W tile, the contribution tile and the stage's observation slots are free again
      stage_fill(g, cx, st, t, j0, j1, c0, e1, false);
      cp_async_wait_all();
    }
    const int e = c0 + t;
    double2* mine = reinterpret_cast<double2*>(s_w + 18 * t);
    bool done = false;
    if (e < e1) {
      const int i = s_cam[t], l = s_pt[t] - j0;
      const double2 uv = *reinterpret_cast<const double2*>(st + kStUv + 2 * t);
      const bool pf = s_pf[l] != 0;
      const double p[3] = {s_pts[3 * l], s_pts[3 * l + 1], s_pts[3 * l + 2]};
      double Rt[12];
      load_rt<POSE_SMEM>(cx.pose_tab, i, Rt);
      const ObsLin o = eval_obs(Rt, p, uv.x, uv.y, g.has_info ? g.o_info + 3 * (size_t)e : nullptr, cx.delta);
      if (o.valid) {
        done = true;
        double Jc[12], Jp[6], AJp[6];
        jac_cam(o, cx.dof_tab[i], Jc);
        jac_pt(o, Rt, pf, Jp);
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          AJp[d] = o.A0 * Jp[d] + o.A1 * Jp[3 + d];
          AJp[3 + d] = o.A1 * Jp[d] + o.A2 * Jp[3 + d];
        }
        const double Ar0 = o.A0 * o.r0 + o.A1 * o.r1, Ar1 = o.A1 * o.r0 + o.A2 * o.r1;
        // W = Jc' A Jp, row-major 6x3, leaving as nine 16-byte pieces as soon as each is complete
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          const int a0 = (2 * k) / 3, c0_ = (2 * k) % 3, a1 = (2 * k + 1) / 3, c1_ = (2 * k + 1) % 3;
          mine[k] = make_double2(Jc[a0] * AJp[c0_] + Jc[6 + a0] * AJp[3 + c0_], Jc[a1] * AJp[c1_] + Jc[6 + a1] * AJp[3 + c1_]);
        }
        int q = 0;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
#pragma unroll
          for (int c = a; c < 3; ++c) s_c[(q++) * kTeam + t] = Jp[a] * AJp[c] + Jp[3 + a] * AJp[3 + c];
          s_c[(6 + a) * kTeam + t] = -(Jp[a] * Ar0 + Jp[3 + a] * Ar1);
        }
        s_c[9 * kTeam + t] = o.rho;
      }
    }
    if (!done) {  // behind the camera / no observation in this lane: a zero block, zero terms
#pragma unroll
      for (int k = 0; k < 9; ++k) mine[k] = make_double2(0.0, 0.0);
#pragma unroll
      for (int k = 0; k < 10; ++k) s_c[k * kTeam + t] = 0.0;
    }
    fence_async_smem();  // the tile is read by the async proxy next
    team_sync(team);
    const int nobs = min(kTeam, e1 - c0);
    if (t == 0 && nobs > 0) bulk_store(g.W + 18 * (size_t)c0, s_w, (uint32_t)nobs * 144u);
    // per-landmark sums: thread = (landmark l, term k); the observations of a landmark are added in ascending order, even and odd
    // positions in two chains (fixed order, half the dependent latency).  The sums leave straight from the threads that made them:
    // k = 0..5 the upper triangle of V_j (mirrored), 6..8 g_p,j, 9 cost_j.  (V^-1 is NOT formed here: ba_prepare_schur_kernel does it
    // for every landmark in parallel -- BaDev::vinv_in_sweep = 0 -- instead of one lane per landmark behind a team barrier.)
    const bool last = c0 + kTeam >= e1, first = c0 == e0;
    for (int it = t; it < L * 10; it += kTeam) {
      const int l = it / 10, k = it - l * 10;
      const int a = max(s_off[l], c0) - c0, b = min(s_off[l + 1], c0 + kTeam) - c0;
      const double* col = s_c + k * kTeam;
      // eight observations at a time: the loads leave together (zero for positions past the landmark's end), the adds form a fixed
      // three-level tree -- one shared-memory latency and three add latencies per batch instead of eight dependent ones
      double s = 0.0;
      for (int o = a; o < b; o += 8) {
        double v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = o + q < b ? col[o + q] : 0.0;
        s += ((v[0] + v[1]) + (v[2] + v[3])) + ((v[4] + v[5]) + (v[6] + v[7]));
      }
      if (!first) s += s_acc[it];
      if (!last) { s_acc[it] = s; continue; }
      const int j = j0 + l;
      if (k < 6) {
        const int r = k < 3 ? 0 : (k < 5 ? 1 : 2), c = k < 3 ? k : (k < 5 ? k - 2 : 2);  // (0,0) (0,1) (0,2) (1,1) (1,2) (2,2)
        double* Vg = g.V + 9 * (size_t)j;
        Vg[r * 3 + c] = s;
        if (r != c) Vg[c * 3 + r] = s;
      } else if (k < 9) {
        g.gp[3 * (size_t)j + (k - 6)] = s;
        if (cx.pend) g.pts[3 * (size_t)j + (k - 6)] = s_pts[3 * l + (k - 6)];  // install the accepted candidate point
      } else {
        g.cost_pt[j] = s;
      }
    }
  }
}

// ---- camera item: slice `slice` of camera i, observations [s0, s1) of the camera-sorted list -----------------------------------
template <bool POSE_SMEM>
__device__ __forceinline__ void sweep_camera(const BaDev& g, const SweepCtx& cx, double* tm, int team, int t, int i, int slice, int s0, int s1) {
  const int K = g.cam_split;
  const int dm = cx.dof_tab[i];
  // (the camera's pose stays in the shared-memory table: broadcast LDS per use instead of 24 registers next to the 54 of the sums)
  double Rt_reg[12];
  if (!POSE_SMEM) load_rt<false>(cx.pose_tab, i, Rt_reg);
  const double* Rt = POSE_SMEM ? cx.pose_tab + kPoseStride * (size_t)i : Rt_reg;
  if (cx.pend && slice == 0) {  // install this camera's accepted pose
    if (t < 12) g.Rt[12 * i + t] = g.Rt_new[12 * i + t];
    else if (t >= 32 && t < 39) g.pose[7 * i + t - 32] = g.pose_new[7 * i + t - 32];
  }
  double acc[27];
#pragma unroll
  for (int k = 0; k < 27; ++k) acc[k] = 0.0;
  // software pipeline over the camera's (camera-sorted) observations: the landmark INDEX is fetched two iterations ahead, the
  // measurement and the landmark coordinates one iteration ahead, so that neither the index -> address dependency nor the gather
  // latency sits in the iteration that consumes them
  int idx = s0 + t;
  double2 uv = make_double2(0.0, 0.0);
  double p[3] = {0.0, 0.0, 0.0};
  int j_nx = 0;
  if (idx < s1) {
    const int j = g.c_pt[idx];
    uv = *reinterpret_cast<const double2*>(g.c_uv + 2 * (size_t)idx);
    if (idx + kTeam < s1) j_nx = g.c_pt[idx + kTeam];
    p[0] = cx.PTS[3 * (size_t)j]; p[1] = cx.PTS[3 * (size_t)j + 1]; p[2] = cx.PTS[3 * (size_t)j + 2];
  }
  while (idx < s1) {
    const int nx = idx + kTeam;
    double2 uv_n = make_double2(0.0, 0.0);
    double pn[3] = {0.0, 0.0, 0.0};
    int j_nx2 = 0;
    if (nx < s1) {
      uv_n = *reinterpret_cast<const double2*>(g.c_uv + 2 * (size_t)nx);
      pn[0] = cx.PTS[3 * (size_t)j_nx]; pn[1] = cx.PTS[3 * (size_t)j_nx + 1]; pn[2] = cx.PTS[3 * (size_t)j_nx + 2];
      if (nx + kTeam < s1) j_nx2 = g.c_pt[nx + kTeam];
    }
    const double* Rt_it = Rt;
    if (POSE_SMEM) asm volatile("" : "+l"(Rt_it));  // (opaque per iteration: keeps the pose loads in the loop instead of 24 live registers)
    const ObsLin o = eval_obs(Rt_it, p, uv.x, uv.y, g.has_info ? g.o_info + 3 * (size_t)g.cam_perm[idx] : nullptr, cx.delta);
    if (o.valid) {
      double Jc[12], AJc[12];
      jac_cam(o, dm, Jc);
#pragma unroll
      for (int d = 0; d < 6; ++d) {
        AJc[d] = o.A0 * Jc[d] + o.A1 * Jc[6 + d];
        AJc[6 + d] = o.A1 * Jc[d] + o.A2 * Jc[6 + d];
      }
      const double Ar0 = o.A0 * o.r0 + o.A1 * o.r1, Ar1 = o.A1 * o.r0 + o.A2 * o.r1;
      int q = 0;
#pragma unroll
      for (int a = 0; a < 6; ++a) {
#pragma unroll
        for (int b = a; b < 6; ++b) acc[q++] += Jc[a] * AJc[b] + Jc[6 + a] * AJc[6 + b];
      }
#pragma unroll
      for (int a = 0; a < 6; ++a) acc[21 + a] -= Jc[a] * Ar0 + Jc[6 + a] * Ar1;
    }
    idx = nx; uv = uv_n; p[0] = pn[0]; p[1] = pn[1]; p[2] = pn[2]; j_nx = j_nx2;
  }
  // fixed-order fold: term-major scratch [27][128]; warp w folds terms w, w+4, ...: four strided entries per lane in order, then a
  // fixed shuffle tree
  double* s_red = tm + kOffW;
  double* s_out = tm + kOffAcc;  // [27]
  int* s_flag = reinterpret_cast<int*>(tm + kOffMisc);
#pragma unroll
  for (int k = 0; k < 27; ++k) s_red[k * kTeam + t] = acc[k];
  team_sync(team);
  const int lane = t & 31, warp = t >> 5;
  for (int k = warp; k < 27; k += kTeam / 32) {
    double r = 0.0;
#pragma unroll
    for (int m = 0; m < kTeam / 32; ++m) r += s_red[k * kTeam + lane + 32 * m];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_down_sync(0xffffffffu, r, o);
    if (lane == 0) {
      s_out[k] = r;
      if (K > 1) g.cam_part[((size_t)i * K + slice) * 27 + k] = r;
    }
  }
  if (K > 1) {
    __threadfence();
    team_sync(team);
    if (t == 0) *s_flag = (atomicAdd(&g.cam_ticket[i], 1u) == (unsigned)(K - 1)) ? 1 : 0;
    team_sync(team);
    if (!*s_flag) return;
    __threadfence();
    if (t < 27) {
      double r = 0.0;
      for (int k = 0; k < K; ++k) r += __ldcg(&g.cam_part[((size_t)i * K + k) * 27 + t]);
      s_out[t] = r;
    }
    if (t == 0) g.cam_ticket[i] = 0;
  }
  team_sync(team);
  if (t < 36) {
    const int a = t / 6, c = t % 6, lo = a < c ? a : c, hi = a < c ? c : a;
    const int q = lo * 6 - lo * (lo - 1) / 2 + (hi - lo);
    g.U[36 * i + t] = s_out[q];
  }
  if (t < 6) g.gc[6 * i + t] = s_out[21 + t];
}

// item records (host plan): landmark group {j0, j1, e0, e1}; camera slice {-1 - camera, slice, s0, s1}
// which: 3 = whole sweep, 1 = camera items only, 2 = landmark items only (timing experiments)
template <bool POSE_SMEM>
__global__ void __launch_bounds__(kSwThreads, 1) ba_sweep_kernel(BaDev g, int which) {
  extern __shared__ __align__(128) double sm[];
  if (g.sc->stop || !g.sc->need_linearize) return;
  const int team = threadIdx.x / kTeam, t = threadIdx.x % kTeam;
  SweepCtx cx;
  cx.delta = g.sc->delta;
  cx.pend = g.sc->pending != 0;  // an accepted candidate not installed yet: read the candidate arrays, install on the fly
  cx.PTS = cx.pend ? g.pts_new : g.pts;
  const double* RT = cx.pend ? g.Rt_new : g.Rt;
  cx.pose_tab = RT;
  cx.dof_tab = g.dof;
  if (POSE_SMEM) {
    double2* dst = reinterpret_cast<double2*>(sm + kOffPose);
    const double2* src = reinterpret_cast<const double2*>(RT);
    for (int k = threadIdx.x; k < g.nc * 6; k += kSwThreads) dst[(k / 6) * (kPoseStride / 2) + (k % 6)] = src[k];
    uint8_t* sd = reinterpret_cast<uint8_t*>(sm + kOffPose + kPoseStride * (size_t)g.nc);
    for (int k = threadIdx.x; k < g.nc; k += kSwThreads) sd[k] = g.dof[k];
    cx.pose_tab = sm + kOffPose;
    cx.dof_tab = sd;
    __syncthreads();
  }
  double* tm = sm + team * kTeamDoubles;
  const int gteam = blockIdx.x * kTeams + team;
  const int n0 = g.sw_team_off[gteam], n1 = g.sw_team_off[gteam + 1];
  const int4* items = reinterpret_cast<const int4*>(g.sw_items);
  // the team's item records: the first kRecs of them into shared memory once (a team gets ~15), the rest (if any) from global memory
  int4* s_rec = reinterpret_cast<int4*>(tm + kOffRec);
  if (t < min(n1 - n0, kRecs)) s_rec[t] = items[n0 + t];
  team_sync(team);
  auto record = [&](int n) -> int4 { return n - n0 < kRecs ? s_rec[n - n0] : items[n]; };
  auto wanted = [&](const int4& r) { return r.x < 0 ? (which & 1) != 0 : (which & 2) != 0; };
  if (n0 < n1) {
    const int4 r = record(n0);
    if (r.x >= 0 && wanted(r)) stage_fill(g, cx, tm + kOffStage, t, r.x, r.y, r.z, r.w, true);
  }
  for (int n = n0; n < n1; ++n) {
    cp_async_wait_all();           // this thread's share of item n's stage
    if (t == 0) bulk_wait_read();  // the W tile of the previous landmark item has left
    team_sync(team);
    double* st = tm + kOffStage + ((n - n0) & 1) * kStage;
    if (n + 1 < n1) {
      const int4 r = record(n + 1);
      if (r.x >= 0 && wanted(r)) stage_fill(g, cx, tm + kOffStage + ((n + 1 - n0) & 1) * kStage, t, r.x, r.y, r.z, r.w, true);
    }
    const int4 rec = record(n);
    if (wanted(rec)) {
      if (rec.x < 0) sweep_camera<POSE_SMEM>(g, cx, tm, team, t, -1 - rec.x, rec.y, rec.z, rec.w);
      else sweep_landmarks<POSE_SMEM>(g, cx, tm, st, team, t, rec.x, rec.y, rec.z, rec.w);
    }
  }
  cp_async_wait_all();
  if (t == 0) bulk_wait_all();
}

}  // namespace

// Host plan.  Landmark groups: consecutive landmarks with <= 128 observations and <= 32 landmarks together (a landmark with more
// observations than a chunk is a group of its own, swept in several chunks).  Camera slices as ba.cu cuts them.  The items are dealt
// to n_teams teams so that every team carries about the same cost (cost model: a camera-pass observation is
// 0.4 of a landmark-pass observation, plus a fixed fold per camera slice): team k gets camera slices k, k + n_teams, ... and then a
// CONTIGUOUS run of landmark groups (neighbouring groups share pose-table and landmark cache lines).
void ba_sweep_plan_host(int nc, int np, int cam_split, const std::vector<int>& cam_off, const std::vector<int>& pt_off, int n_teams,
                        std::vector<int>& items4, std::vector<int>& team_off) {
  struct Grp { int j0, j1; };
  std::vector<Grp> groups;
  for (int j = 0; j < np;) {
    int k = j + 1;
    while (k < np && k - j < kSwMaxPts && pt_off[k + 1] - pt_off[j] <= kTeam) ++k;
    groups.push_back({j, k});
    j = k;
  }
  const int n_cam_items = nc * cam_split;
  auto cam_range = [&](int item, int* s0, int* s1) {
    const int i = item / cam_split, slice = item - i * cam_split;
    const int c0 = cam_off[i], c1 = cam_off[i + 1], per = (c1 - c0 + cam_split - 1) / cam_split;
    *s0 = std::min(c0 + slice * per, c1); *s1 = std::min(*s0 + per, c1);
  };
  auto cam_cost = [&](int item) { int s0, s1; cam_range(item, &s0, &s1); return 0.4 * (s1 - s0) + 150.0; };
  auto grp_cost = [&](const Grp& gr) { return (double)(pt_off[gr.j1] - pt_off[gr.j0]) + 40.0; };
  double total = 0.0;
  for (int c = 0; c < n_cam_items; ++c) total += cam_cost(c);
  for (const Grp& gr : groups) total += grp_cost(gr);
  items4.clear();
  team_off.assign(n_teams + 1, 0);
  size_t next_grp = 0;
  double given = 0.0;
  for (int k = 0; k < n_teams; ++k) {
    team_off[k] = (int)(items4.size() / 4);
    double mine = 0.0;
    for (int c = k; c < n_cam_items; c += n_teams) {
      int s0, s1; cam_range(c, &s0, &s1);
      const int i = c / cam_split;
      items4.insert(items4.end(), {-1 - i, c - i * cam_split, s0, s1});
      mine += cam_cost(c);
    }
    // a contiguous run of groups up to this team's share of what is left
    const double target = k == n_teams - 1 ? 1e300 : std::max(0.0, (total - given) / (n_teams - k) - mine);
    double got = 0.0;
    while (next_grp < groups.size() && (got + 0.5 * grp_cost(groups[next_grp]) <= target)) {
      const Grp& gr = groups[next_grp++];
      items4.insert(items4.end(), {gr.j0, gr.j1, pt_off[gr.j0], pt_off[gr.j1]});
      got += grp_cost(gr);
    }
    given += mine + got;
  }
  team_off[n_teams] = (int)(items4.size() / 4);
}

int ba_sweep_teams(const gb_ctx* ctx) { return ctx->sm_count * kTeams; }

static size_t ba_sweep_smem(int nc) {
  const bool pose = nc <= kSwPoseCams;
  return (size_t)kOffPose * sizeof(double) + (pose ? (size_t)nc * kPoseStride * 8 + (((size_t)nc + 15) & ~(size_t)15) : 0);
}

static int ba_sweep_setup(gb_ctx* ctx) {  // once per device: opt in to the large dynamic shared memory (never lowered)
  static std::once_flag once[64];
  cudaError_t e = cudaSuccess;
  std::call_once(once[ctx->device & 63], [&] {
    e = cudaFuncSetAttribute(ba_sweep_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ba_sweep_smem(kSwPoseCams));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(ba_sweep_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ba_sweep_smem(kSwPoseCams + 1));
  });
  if (e != cudaSuccess) { gb_set_error(ctx, "ba_sweep_setup: %s", cudaGetErrorString(e)); return GB_ERR_CUDA; }
  return GB_OK;
}

void ba_sweep_plan_drop(gb_ba_graph* g) {
  if (g->sw_alloc) cudaFree(g->sw_alloc);
  g->sw_alloc = nullptr;
  g->d.sw_items = nullptr; g->d.sw_team_off = nullptr; g->d.sw_nteams = 0; g->d.sw_nitems = 0;
}

// made on first use (the local-BA sizes never come here): cut the items, deal them to the teams, upload
static int ba_sweep_plan(gb_ctx* ctx, gb_ba_graph* g) {
  std::vector<int> items4, team_off;
  const int n_teams = ba_sweep_teams(ctx);
  ba_sweep_plan_host(g->d.nc, g->d.np, g->d.cam_split, g->cam_off_h, g->pt_off_h, n_teams, items4, team_off);
  const size_t b_items = (items4.size() * 4 + 255) & ~(size_t)255, b_off = team_off.size() * 4;
  GB_CUDA(ctx, cudaMalloc(&g->sw_alloc, b_items + b_off + 256));
  uint8_t* base = (uint8_t*)g->sw_alloc;
  if (!items4.empty()) GB_CUDA(ctx, cudaMemcpyAsync(base, items4.data(), items4.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  GB_CUDA(ctx, cudaMemcpyAsync(base + b_items, team_off.data(), b_off, cudaMemcpyHostToDevice, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // (the host vectors die with this frame)
  g->d.sw_items = (const int*)base; g->d.sw_team_off = (const int*)(base + b_items);
  g->d.sw_nteams = n_teams; g->d.sw_nitems = (int)(items4.size() / 4);
  return GB_OK;
}

int ba_sweep_launch(gb_ctx* ctx, gb_ba_graph* g, const BaDev& d_in, cudaStream_t s, int which) {
  GB_CHECK(ba_sweep_setup(ctx));
  if (!g->sw_alloc) GB_CHECK(ba_sweep_plan(ctx, g));
  if (g->d.sw_nitems <= 0) return GB_OK;
  BaDev d = d_in;  // (the caller's copy may predate the plan)
  d.sw_items = g->d.sw_items; d.sw_team_off = g->d.sw_team_off; d.sw_nteams = g->d.sw_nteams; d.sw_nitems = g->d.sw_nitems;
  const int grid = d.sw_nteams / kTeams;
  if (d.nc <= kSwPoseCams) ba_sweep_kernel<true><<<grid, kSwThreads, ba_sweep_smem(d.nc), s>>>(d, which);
  else ba_sweep_kernel<false><<<grid, kSwThreads, ba_sweep_smem(d.nc), s>>>(d, which);
  GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}

// host-only test hook: the item records and per-team ranges the sweep would use -- no device needed.  items4: capacity cap_items
// records of 4 ints; team_off: n_teams + 1 ints.  Returns the number of items through *n_items.
extern "C" GB_API int gb_dbg_ba_sweep_plan(int nc, int np, int cam_split, const int32_t* cam_off, const int32_t* pt_off, int n_teams, int32_t* items4,
                                           int cap_items, int32_t* team_off, int* n_items) {
  if (nc < 0 || np < 0 || cam_split < 1 || n_teams < 1 || !cam_off || !pt_off || !team_off || !n_items) return GB_ERR_INVALID;
  std::vector<int> co(cam_off, cam_off + nc + 1), po(pt_off, pt_off + np + 1), it, to;
  ba_sweep_plan_host(nc, np, cam_split, co, po, n_teams, it, to);
  *n_items = (int)(it.size() / 4);
  if (*n_items > cap_items) return GB_ERR_CAPACITY;
  if (items4 && !it.empty()) memcpy(items4, it.data(), it.size() * 4);
  memcpy(team_off, to.data(), to.size() * 4);
  return GB_OK;
}
