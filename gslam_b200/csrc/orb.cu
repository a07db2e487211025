// gslam_b200/csrc/orb.cu — ORB extract (K1-K4): pyramid -> FAST-9/16 + NMS -> Harris / per-level top-N -> IC angle + rBRIEF.
//
// Consumes a GSLAM::GImage payload (dense 8UC1, GSLAM/core/GImage.h:160-443, no row stride :378); produces
// GSLAM::KeyPoint records (GSLAM/core/Map.h:122-195 == gb_keypoint) and N x 32 8UC1 descriptor rows for
// MapFrame::setKeyPoints (Map.h:311-312).  The arithmetic is OpenCV's ORB as specified in SURVEY.md Appendix A and
// restated by oracle/orb_ref.c; every stage here is bit-exact against it (integer stages trivially; float stages by
// using explicitly rounded intrinsics / explicit fma in the same order).
//
// Launch structure per frame (all on the ctx stream, no host sync inside):
//   orb_resize_kernel   x (nlevels-1) : INTER_LINEAR_EXACT from the previous level (Q8 fixed point), padded pitch
//   orb_fast_kernel     x 1           : all levels, 64x16 tiles staged in shared memory; quick-reject -> shared worklist ->
//                                       dense score pass -> strict 3x3 NMS -> border filter -> candidate append + histogram
//   orb_harris_kernel   x 1           : FAST-score threshold from the histogram (top 2n, ties kept), Harris response
//   orb_select_kernel   x 1           : one CTA per level: 4-pass radix select of the n-th largest response (ties kept),
//                                       compaction, bitonic sort by (y,x) -> canonical order
//   orb_describe_kernel x 1           : one warp per keypoint: 45x45 patch in shared memory, IC angle, 7x7 float blur of the
//                                       patch, 256 rotated tests, coalesced 32-byte descriptor row + KeyPoint record
#include "common.cuh"
#include "orb_pattern.h"

#include <cuda.h>  // CUtensorMap (types only: the encoder is fetched with cudaGetDriverEntryPoint, libcuda is not linked)

#include <cmath>

namespace {

constexpr int kMaxLevels = GB_ORB_MAX_LEVELS;
constexpr int kTileW = 128, kTileH = 32;               // interior of a FAST tile
constexpr int kInX0 = 16, kInY0 = 4;                   // input-box coordinates of tile pixel (0,0)
constexpr int kInW = kTileW + 32, kInH = kTileH + 8;   // 160 x 40 input box: 3 ring + 1 nms halo each side; the box must START on a
                                                       // 16-byte boundary of the image row (TMA: tools/mb/tma_probe.cu -- any other x
                                                       // faults with "illegal instruction"), so 16 columns are fetched on the left and
                                                       // the width is a multiple of 16 bytes
constexpr int kScW = kTileW + 2, kScH = kTileH + 2;    // 130 x 34 score tile (1-pixel halo for the non-maximum suppression)
constexpr int kFastThreads = 256;
constexpr int kInWords = kInW / 4;                     // 40 32-bit words per input row
constexpr int kWorkCap = 2048;                         // quick-test survivors per tile handled in shared memory (rest: rounds)
constexpr int kSelThreads = 1024;
constexpr int kSelMax = 4096;                          // max kept keypoints per level (bitonic sort in shared memory)
constexpr int kDescWarps = 4;

struct LevelInfo {
  int w, h, pitch;        // pitch in bytes, multiple of 128
  int quota;              // n_l
  size_t off;             // byte offset of the level in the pyramid buffer
  int tiles_x, tile_start;  // FAST tiling
  int cand_off, cand_cap;   // slice of the candidate arrays
  int coef_off;           // offset (in entries) of this level's resize tables: x table then y table
  float scale;            // s_l = (float)pow((double)scaleFactor, l)
};

struct OrbParams {
  int nlevels, total_tiles, fast_threshold, border;
  LevelInfo lv[kMaxLevels];
};

// ---- K1: pyramid ---------------------------------------------------------------------------------------------------------
// dst(x,y) = (b0*(a0*S[iy][ix] + a1*S[iy][ix+1]) + b1*(a0*S[iy+1][ix] + a1*S[iy+1][ix+1]) + 2^15) >> 16, weights Q8.
// Table entry: idx | (a1 << 16).  One thread writes 4 consecutive pixels as one 32-bit store.
__global__ void __launch_bounds__(256) orb_resize_kernel(const uint8_t* __restrict__ src, int sw, int sh, int spitch,
                                                         uint8_t* __restrict__ dst, int dw, int dh, int dpitch,
                                                         const uint32_t* __restrict__ xtab, const uint32_t* __restrict__ ytab) {
  gb_pdl_launch_dependents();
  gb_pdl_wait();
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x4 >= dw || y >= dh) return;
  const uint32_t ye = ytab[y];
  const int iy = ye & 0xffff, b1 = ye >> 16, b0 = 256 - b1;
  const uint8_t* r0 = src + (size_t)iy * spitch;
  const uint8_t* r1 = src + (size_t)min(iy + 1, sh - 1) * spitch;
  uint32_t out = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int x = x4 + k;
    uint32_t v = 0;
    if (x < dw) {
      const uint32_t xe = xtab[x];
      const int ix = xe & 0xffff, a1 = xe >> 16, a0 = 256 - a1, ix1 = min(ix + 1, sw - 1);
      const uint32_t h0 = a0 * r0[ix] + a1 * r0[ix1];
      const uint32_t h1 = a0 * r1[ix] + a1 * r1[ix1];
      v = (b0 * h0 + b1 * h1 + (1u << 15)) >> 16;
    }
    out |= v << (8 * k);
  }
  *reinterpret_cast<uint32_t*>(dst + (size_t)y * dpitch + x4) = out;
}

// ---- K0: colour -> gray into pyramid level 0 (frames arrive BGR / BGRA / RGB / RGBA from the dataset plugins, IO.h:86-110) ----
// OpenCV's 8-bit fixed point (cv2 4.13: 15-bit coefficients B 3735, G 19235, R 9798, round to nearest; pinned against
// cv2.cvtColor in tests/test_oracle_orb.py::test_gray_conversion_equals_cv2).
__global__ void __launch_bounds__(256) orb_gray_kernel(const uint8_t* __restrict__ src, int w, int h, int channels, int rgb_order,
                                                       uint8_t* __restrict__ dst, int dpitch) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w || y >= h) return;
  const uint8_t* p = src + ((size_t)y * w + x) * channels;
  const int c0 = p[0], c1 = p[1], c2 = p[2];
  const int b = rgb_order ? c2 : c0, r = rgb_order ? c0 : c2;
  dst[(size_t)y * dpitch + x] = (uint8_t)((b * 3735 + c1 * 19235 + r * 9798 + (1 << 14)) >> 15);
}

// ---- K2: FAST-9/16 -----------------------------------------------------------------------------------------------------
// Corner score of one pixel: m = max over the 16 cyclic 9-arcs of max(min_i d_i, min_i -d_i), score = m-1 if m > t.
// Sliding 9-window minimum over the ring by doubling (windows 2, 4, 8, then +1), once on d = ring - centre (bright arcs) and
// once on the explicitly negated array (dark arcs).  NB: the obvious formulation max(best, max(mn, -mx)) inside one unrolled
// loop is MISCOMPILED by ptxas 12.9 for sm_100a (the negation is dropped when it fuses the chain into VIMNMX3) — keep the
// two arrays separate; tests/test_orb_gpu.py::test_fast_candidates_match_oracle guards this.
__device__ __forceinline__ int ring_arc9_maxmin(const int* v) {
  int m2[16], m4[16], m8[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) m2[i] = min(v[i], v[(i + 1) & 15]);
#pragma unroll
  for (int i = 0; i < 16; ++i) m4[i] = min(m2[i], m2[(i + 2) & 15]);
#pragma unroll
  for (int i = 0; i < 16; ++i) m8[i] = min(m4[i], m4[(i + 4) & 15]);
  int best = min(m8[0], v[8]);
#pragma unroll
  for (int i = 1; i < 16; ++i) best = max(best, min(m8[i], v[(i + 8) & 15]));
  return best;
}

// Is there a 9-arc of the 16-ring entirely brighter than c+t or entirely darker than c-t?  (bit masks + doubling)
__device__ __forceinline__ bool fast_is_corner(const uint8_t* p, int threshold) {
  const int c = p[0], hi = c + threshold, lo = c - threshold;
  int r[16];
  r[0] = p[3 * kInW + 0]; r[1] = p[3 * kInW + 1]; r[2] = p[2 * kInW + 2]; r[3] = p[1 * kInW + 3];
  r[4] = p[3]; r[5] = p[-1 * kInW + 3]; r[6] = p[-2 * kInW + 2]; r[7] = p[-3 * kInW + 1];
  r[8] = p[-3 * kInW]; r[9] = p[-3 * kInW - 1]; r[10] = p[-2 * kInW - 2]; r[11] = p[-1 * kInW - 3];
  r[12] = p[-3]; r[13] = p[1 * kInW - 3]; r[14] = p[2 * kInW - 2]; r[15] = p[3 * kInW - 1];
  unsigned mb = 0, md = 0;
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    mb |= (r[k] > hi ? 1u : 0u) << k;
    md |= (r[k] < lo ? 1u : 0u) << k;
  }
  mb |= mb << 16;
  md |= md << 16;
  unsigned b = mb & (mb >> 1); b &= b >> 2; b &= b >> 4; b &= mb >> 8;  // bit i set <=> bits i..i+8 all set
  unsigned d = md & (md >> 1); d &= d >> 2; d &= d >> 4; d &= md >> 8;
  return ((b | d) & 0xffffu) != 0;
}

__device__ __forceinline__ int fast_full_score(const uint8_t* p /* centre inside the shared tile */, int threshold) {
  // ring offsets (dx,dy), radius 3 (SURVEY.md App. A.2)
  const int c = p[0];
  int r[16];
  r[0] = p[3 * kInW + 0]; r[1] = p[3 * kInW + 1]; r[2] = p[2 * kInW + 2]; r[3] = p[1 * kInW + 3];
  r[4] = p[3]; r[5] = p[-1 * kInW + 3]; r[6] = p[-2 * kInW + 2]; r[7] = p[-3 * kInW + 1];
  r[8] = p[-3 * kInW]; r[9] = p[-3 * kInW - 1]; r[10] = p[-2 * kInW - 2]; r[11] = p[-1 * kInW - 3];
  r[12] = p[-3]; r[13] = p[1 * kInW - 3]; r[14] = p[2 * kInW - 2]; r[15] = p[3 * kInW - 1];
  int d[16], nd[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    d[k] = r[k] - c;
    nd[k] = c - r[k];
    asm volatile("" : "+r"(nd[k]));  // opaque to the optimiser: it must not re-derive nd from d (see NB above)
  }
  const int bright = ring_arc9_maxmin(d);
  const int dark = ring_arc9_maxmin(nd);
  const int best = bright > dark ? bright : dark;
  return best > threshold ? best - 1 : 0;
}

// ---- TMA + mbarrier plumbing (sm_90+ PTX; SASS: UTMALDG / SYNCS) ----------------------------------------------------------------
struct FastMaps {
  CUtensorMap m[kMaxLevels];  // one 2-D u8 tensor map per pyramid level: dims {w, h}, row stride = pitch, box {kInW, kInH}
};
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int x, int y, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst)),
               "l"(map), "r"(x), "r"(y), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  for (int spin = 0; spin < (1 << 24) && !ok; ++spin)
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  if (!ok) __trap();  // a copy that never lands must not hang the device
}

// K2.  Persistent CTAs walk the FAST tiles of all levels; the 160 x 40 input box of tile i+1 is fetched by the TMA unit
// (cp.async.bulk.tensor.2d, zero fill outside the image) into the other half of a double buffer while tile i is processed:
//   A  packed quick test, four pixels per thread-step on 32-bit words (byte-SIMD compares): a 9-arc of the 16-ring always
//      contains two CONSECUTIVE compass points (S,E / E,N / N,W / W,S), so a corner needs (S|N) & (E|W) all brighter than c+t or
//      all darker than c-t -- survivors (a few percent) go to a shared-memory worklist;
//   B  per survivor: exact 9-contiguity test on bit masks, then the exact score (max threshold) for true corners only;
//   C  strict 3x3 non-maximum suppression over the corner list (not over the pixels), border filter, append + score histogram.
__global__ void __launch_bounds__(kFastThreads) orb_fast_kernel(const __grid_constant__ OrbParams P, const __grid_constant__ FastMaps M,
                                                                uint32_t* __restrict__ cand_pos, uint8_t* __restrict__ cand_score,
                                                                int* __restrict__ counts, int* __restrict__ hist) {
  gb_pdl_launch_dependents();
  __shared__ __align__(128) uint8_t s_in[2][kInH * kInW];
  __shared__ __align__(16) uint8_t s_sc[kScH * kScW + 12];
  __shared__ uint16_t s_work[kScH * kScW];   // quick-test survivors: input-tile offsets ry * kInW + col
  __shared__ uint16_t s_work2[kScH * kScW];  // true corners: score-tile offsets
  __shared__ __align__(8) uint64_t s_bar[2];
  __shared__ int s_nwork, s_nwork2;
  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(&s_bar[0], 1);
    mbar_init(&s_bar[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  gb_pdl_wait();  // the pyramid levels are written by the predecessor kernels
  auto locate = [&](int tile, int* lvl, int* x0, int* y0) {
    int l = 0;
#pragma unroll 1
    for (int k = 1; k < P.nlevels; ++k)
      if (tile >= P.lv[k].tile_start && P.lv[k].tiles_x > 0) l = k;
    const int t = tile - P.lv[l].tile_start;
    *lvl = l; *x0 = (t % P.lv[l].tiles_x) * kTileW; *y0 = (t / P.lv[l].tiles_x) * kTileH;
  };
  auto fetch = [&](int tile, int buf) {  // thread 0 only
    int l, x0, y0;
    locate(tile, &l, &x0, &y0);
    mbar_expect_tx(&s_bar[buf], kInH * kInW);
    tma_load_2d(&s_in[buf][0], &M.m[l], x0 - kInX0, y0 - kInY0, &s_bar[buf]);
  };
  const int thr = P.fast_threshold;
  const uint32_t t4 = (uint32_t)thr * 0x01010101u;
  int tile = blockIdx.x;
  if (tile < P.total_tiles && tid == 0) fetch(tile, 0);
  for (int it = 0; tile < P.total_tiles; ++it, tile += gridDim.x) {
    const int buf = it & 1;
    if (tid == 0 && tile + (int)gridDim.x < P.total_tiles) fetch(tile + gridDim.x, buf ^ 1);  // (that buffer was released by the barrier ending step it-1)
    int l, x0, y0;
    locate(tile, &l, &x0, &y0);
    const LevelInfo& L = P.lv[l];
    if (tid == 0) { s_nwork = 0; s_nwork2 = 0; }
    for (int i = tid; i < (kScH * kScW + 12) / 16; i += kFastThreads) reinterpret_cast<uint4*>(s_sc)[i] = make_uint4(0, 0, 0, 0);
    mbar_wait(&s_bar[buf], (it >> 1) & 1);
    __syncthreads();
    const uint8_t* in = s_in[buf];
    const uint32_t* inw = reinterpret_cast<const uint32_t*>(in);
    // ---- A: packed quick test over the score region (input rows 3..36; input columns 15..144 = words 3..36)
    for (int i = tid; i < kScH * 34; i += kFastThreads) {  // 34 rows x 34 words
      const int ry = 3 + i / 34, wx = 3 + i - (i / 34) * 34;
      const uint32_t C = inw[ry * kInWords + wx];
      const uint32_t S = inw[(ry + 3) * kInWords + wx], N = inw[(ry - 3) * kInWords + wx];
      const uint32_t Wm = inw[ry * kInWords + wx - 1], Wp = inw[ry * kInWords + wx + 1];
      const uint32_t E = __byte_perm(C, Wp, 0x6543), Wst = __byte_perm(Wm, C, 0x4321);
      const uint32_t hi = __vaddus4(C, t4), lo = __vsubus4(C, t4);
      const uint32_t bright = (__vcmpgtu4(S, hi) | __vcmpgtu4(N, hi)) & (__vcmpgtu4(E, hi) | __vcmpgtu4(Wst, hi));
      const uint32_t dark = (__vcmpgtu4(lo, S) | __vcmpgtu4(lo, N)) & (__vcmpgtu4(lo, E) | __vcmpgtu4(lo, Wst));
      uint32_t pass = bright | dark;
      if (pass == 0) continue;
      const int gy = y0 - kInY0 + ry;
      if (gy < 3 || gy >= L.h - 3) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (!((pass >> (8 * j)) & 1u)) continue;
        const int col = 4 * wx + j, gx = x0 - kInX0 + col;
        if (col < kInX0 - 1 || col >= kInX0 - 1 + kScW || gx < 3 || gx >= L.w - 3) continue;
        s_work[atomicAdd(&s_nwork, 1)] = (uint16_t)(ry * kInW + col);
      }
    }
    __syncthreads();
    // ---- B: exact 9-contiguity test, exact score for the true corners
    const int nwork = s_nwork;
    for (int k = tid; k < nwork; k += kFastThreads) {
      const int o = s_work[k];
      const uint8_t* p = in + o;
      if (!fast_is_corner(p, thr)) continue;
      const int ry = o / kInW, col = o - ry * kInW;
      const int so = (ry - (kInY0 - 1)) * kScW + (col - (kInX0 - 1));
      s_sc[so] = (uint8_t)fast_full_score(p, thr);
      s_work2[atomicAdd(&s_nwork2, 1)] = (uint16_t)so;
    }
    __syncthreads();
    // ---- C: strict 3x3 NMS over the corner list, border filter, emit
    const int ncorner = s_nwork2;
    for (int k = tid; k < ncorner; k += kFastThreads) {
      const int so = s_work2[k];
      const int sr = so / kScW, scol = so - sr * kScW;
      if (sr < 1 || sr > kTileH || scol < 1 || scol > kTileW) continue;  // halo ring: belongs to the neighbouring tile
      const int gx = x0 + scol - 1, gy = y0 + sr - 1;
      if (gx < P.border || gx >= L.w - P.border || gy < P.border || gy >= L.h - P.border) continue;
      const uint8_t* q = &s_sc[so];
      const int sv = q[0];
      if (sv > q[-1] && sv > q[1] && sv > q[-kScW - 1] && sv > q[-kScW] && sv > q[-kScW + 1] && sv > q[kScW - 1] && sv > q[kScW] && sv > q[kScW + 1]) {
        const int idx = atomicAdd(&counts[l], 1);
        if (idx < L.cand_cap) {
          cand_pos[L.cand_off + idx] = ((uint32_t)gy << 16) | (uint32_t)gx;
          cand_score[L.cand_off + idx] = (uint8_t)sv;
        }
        atomicAdd(&hist[l * 256 + sv], 1);
      }
    }
    __syncthreads();  // every read of s_in[buf] / s_sc / the worklists is done: the buffer may be refilled, the lists reset
  }
}

// ---- K3: Harris ----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t float_key(float f) {  // order-preserving map float -> uint32 (larger float, larger key)
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float harris_response(const uint8_t* __restrict__ img, int pitch, int x, int y) {
  // 9x9 byte window held in a rolling 3-row register file: 81 loads instead of 49 x 6
  int a = 0, b = 0, c = 0;
  int r0[9], r1[9], r2[9];
  const uint8_t* p = img + (size_t)(y - 4) * pitch + (x - 4);
#pragma unroll
  for (int k = 0; k < 9; ++k) { r0[k] = p[k]; r1[k] = p[pitch + k]; }
#pragma unroll
  for (int dy = 0; dy < 7; ++dy) {
    const uint8_t* q = p + (size_t)(dy + 2) * pitch;
#pragma unroll
    for (int k = 0; k < 9; ++k) r2[k] = q[k];
#pragma unroll
    for (int dx = 0; dx < 7; ++dx) {
      const int Ix = (r1[dx + 2] - r1[dx]) * 2 + (r0[dx + 2] - r0[dx]) + (r2[dx + 2] - r2[dx]);
      const int Iy = (r2[dx + 1] - r0[dx + 1]) * 2 + (r2[dx] - r0[dx]) + (r2[dx + 2] - r0[dx + 2]);
      a += Ix * Ix; b += Iy * Iy; c += Ix * Iy;
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) { r0[k] = r1[k]; r1[k] = r2[k]; }
  }
  const float scale = __fdiv_rn(1.f, __fmul_rn((float)(4 * 7), 255.f));
  const float s4 = __fmul_rn(__fmul_rn(__fmul_rn(scale, scale), scale), scale);
  const float fa = (float)a, fb = (float)b, fc = (float)c, sab = __fadd_rn(fa, fb);
  const float v = __fsub_rn(__fsub_rn(__fmul_rn(fa, fb), __fmul_rn(fc, fc)), __fmul_rn(__fmul_rn(0.04f, sab), sab));
  return __fmul_rn(v, s4);
}

__global__ void __launch_bounds__(256) orb_harris_kernel(const __grid_constant__ OrbParams P, const uint8_t* __restrict__ pyr,
                                                         const uint32_t* __restrict__ cand_pos, const uint8_t* __restrict__ cand_score,
                                                         const int* __restrict__ counts, const int* __restrict__ hist,
                                                         uint32_t* __restrict__ surv_key, float* __restrict__ surv_resp,
                                                         uint32_t* __restrict__ surv_pos, int* __restrict__ surv_count) {
  gb_pdl_launch_dependents();
  gb_pdl_wait();
  // FAST-score threshold of this level = the (2 n_l)-th largest score (ties kept): suffix sums of the 256-bin histogram,
  // one bin per thread (blockDim.x == 256), thr = number of scores s whose suffix count  #{score >= s}  reaches 2 n_l
  __shared__ int s_suffix[256];
  __shared__ int s_thr;
  const int l = blockIdx.y;
  const LevelInfo& L = P.lv[l];
  {
    const int t = threadIdx.x;
    int v = t >= 1 ? hist[l * 256 + t] : 0;
    s_suffix[t] = v;
    if (t == 0) s_thr = 0;
    __syncthreads();
    // inclusive suffix scan (Hillis-Steele, 8 steps)
    for (int off = 1; off < 256; off <<= 1) {
      const int add = (t + off < 256) ? s_suffix[t + off] : 0;
      __syncthreads();
      s_suffix[t] += add;
      __syncthreads();
    }
    const int want = 2 * L.quota;
    // suffix counts are non-increasing in s: the threshold is the LARGEST s >= 1 with suffix[s] >= want (0 if none)
    if (want > 0 && t >= 1 && s_suffix[t] >= want && (t == 255 || s_suffix[t + 1] < want)) s_thr = t;
    if (want <= 0 && t == 0) s_thr = 256;
    __syncthreads();
  }
  const int thr = s_thr;
  const int n = min(counts[l], L.cand_cap);
  const uint8_t* img = pyr + L.off;
  // survivors of the FAST-score cut are appended to a compact per-level list (order is irrelevant: the selection below is
  // order-independent and ends with a sort), so the selection kernel scans ~2n entries instead of every FAST corner
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int g = L.cand_off + i;
    if ((int)cand_score[g] >= thr) {
      const uint32_t pos = cand_pos[g];
      const float r = harris_response(img, L.pitch, pos & 0xffff, pos >> 16);
      const int slot = L.cand_off + atomicAdd(&surv_count[l], 1);
      surv_key[slot] = float_key(r);
      surv_resp[slot] = r;
      surv_pos[slot] = pos;
    }
  }
}

// ---- K3b: per-level selection + canonical ordering ------------------------------------------------------------------------
__global__ void __launch_bounds__(kSelThreads) orb_select_kernel(const __grid_constant__ OrbParams P, const uint32_t* __restrict__ cand_pos,
                                                                 const uint32_t* __restrict__ cand_key, const float* __restrict__ cand_resp,
                                                                 const int* __restrict__ counts, const int* __restrict__ raw_counts,
                                                                 uint32_t* __restrict__ kept_pos,
                                                                 float* __restrict__ kept_resp, int* __restrict__ kept_count,
                                                                 int* __restrict__ status) {
  gb_pdl_launch_dependents();
  gb_pdl_wait();
  __shared__ int s_hist[256];
  __shared__ unsigned long long s_keys[kSelMax];
  __shared__ int s_n, s_k;
  __shared__ uint32_t s_prefix;
  const int l = blockIdx.x, tid = threadIdx.x;
  const LevelInfo& L = P.lv[l];
  const int n = min(counts[l], L.cand_cap);  // counts here = number of survivors of the FAST-score cut (compact list)
  const uint32_t* keys = cand_key + L.cand_off;
  if (raw_counts[l] > L.cand_cap && tid == 0) atomicMin(status, -1);  // cannot happen (cap = w*h/4): flag loudly if it does
  const int m = n;
  uint32_t T = 1;  // keep every key >= T; key 0 = dropped
  if (L.quota <= 0) T = 0xffffffffu;
  else if (m > L.quota) {
    // 4-pass MSB-first radix select of the quota-th largest key
    if (tid == 0) { s_prefix = 0; s_k = L.quota; }
    uint32_t mask = 0;
    for (int pass = 3; pass >= 0; --pass) {
      const int shift = 8 * pass;
      for (int b = tid; b < 256; b += kSelThreads) s_hist[b] = 0;
      __syncthreads();
      const uint32_t prefix = s_prefix;
      for (int i = tid; i < n; i += kSelThreads) {
        const uint32_t k = keys[i];
        if (k != 0 && (k & mask) == prefix) atomicAdd(&s_hist[(k >> shift) & 255], 1);
      }
      __syncthreads();
      if (tid == 0) {
        int cum = 0, b = 255, want = s_k;
        for (; b > 0; --b) {
          if (cum + s_hist[b] >= want) break;
          cum += s_hist[b];
        }
        s_k = want - cum;
        s_prefix = prefix | ((uint32_t)b << shift);
      }
      __syncthreads();
      mask |= 0xffu << shift;
    }
    T = s_prefix;
  }
  // compaction of the kept candidates: (pos << 32) | candidate index
  if (tid == 0) s_n = 0;
  __syncthreads();
  for (int i = tid; i < n; i += kSelThreads) {
    const uint32_t k = keys[i];
    if (k != 0 && k >= T) {
      const int slot = atomicAdd(&s_n, 1);
      if (slot < kSelMax) s_keys[slot] = ((unsigned long long)cand_pos[L.cand_off + i] << 32) | (unsigned)i;
    }
  }
  __syncthreads();
  const int cnt = s_n;
  if (cnt > kSelMax) {
    if (tid == 0) { atomicMin(status, -2); kept_count[l] = 0; }
    return;
  }
  int np2 = 1;
  while (np2 < cnt) np2 <<= 1;
  for (int i = cnt + tid; i < np2; i += kSelThreads) s_keys[i] = ~0ull;
  __syncthreads();
  for (int k = 2; k <= np2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < np2; i += kSelThreads) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = s_keys[i], b = s_keys[ixj];
          const bool up = (i & k) == 0;
          if ((a > b) == up) { s_keys[i] = b; s_keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  for (int i = tid; i < cnt; i += kSelThreads) {
    const unsigned long long e = s_keys[i];
    kept_pos[l * kSelMax + i] = (uint32_t)(e >> 32);
    kept_resp[l * kSelMax + i] = cand_resp[L.cand_off + (uint32_t)e];
  }
  if (tid == 0) kept_count[l] = cnt;
}

// ---- K4: orientation + rBRIEF ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float fast_atan2_deg(float y, float x) {  // cv::fastAtan2, bit-exact (App. A.4): no FMA
  const float k = (float)(180.0 / 3.14159265358979323846);
  const float p1 = __fmul_rn(0.9997878412794807f, k), p3 = __fmul_rn(-0.3258083974640975f, k),
              p5 = __fmul_rn(0.1555786518463281f, k), p7 = __fmul_rn(-0.04432655554792128f, k);
  const float ax = fabsf(x), ay = fabsf(y);
  const float eps = (float)2.220446049250313e-16;
  float a;
  if (ax >= ay) {
    const float c = __fdiv_rn(ay, __fadd_rn(ax, eps)), c2 = __fmul_rn(c, c);
    a = __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c);
  } else {
    const float c = __fdiv_rn(ax, __fadd_rn(ay, eps)), c2 = __fmul_rn(c, c);
    a = __fsub_rn(90.f, __fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(p7, c2), p5), c2), p3), c2), p1), c));
  }
  if (x < 0.f) a = __fsub_rn(180.f, a);
  if (y < 0.f) a = __fsub_rn(360.f, a);
  return a;
}

// deterministic double sincos: Cody-Waite by pi/2 + fdlibm kernel polynomials, explicit fma only (same op sequence as the oracle)
__device__ __forceinline__ void det_sincos(double x, double* sn, double* cs) {
  const double kf = rint(__dmul_rn(x, 0.63661977236758134308));
  const int q = (int)kf & 3;
  double r = fma(-kf, 1.57079632673412561417e+00, x);
  r = fma(-kf, 6.07710050650619224932e-11, r);
  const double z = __dmul_rn(r, r);
  double ps = fma(z, 1.58969099521155010221e-10, -2.50507602534068634195e-08);
  ps = fma(z, ps, 2.75573137070700676789e-06);
  ps = fma(z, ps, -1.98412698298579493134e-04);
  ps = fma(z, ps, 8.33333333332248946124e-03);
  ps = fma(z, ps, -1.66666666666666324348e-01);
  const double s = fma(__dmul_rn(z, r), ps, r);
  double pc = fma(z, -1.13596475577881948265e-11, 2.08757232129817482790e-09);
  pc = fma(z, pc, -2.75573143513906633035e-07);
  pc = fma(z, pc, 2.48015872894767294178e-05);
  pc = fma(z, pc, -1.38888888888741095749e-03);
  pc = fma(z, pc, 4.16666666666666019037e-02);
  const double c = fma(__dmul_rn(z, z), pc, fma(z, -0.5, 1.0));
  switch (q) {
    case 0: *sn = s; *cs = c; break;
    case 1: *sn = c; *cs = -s; break;
    case 2: *sn = -s; *cs = -c; break;
    default: *sn = -c; *cs = s; break;
  }
}

constexpr int kPatch = 45, kPatchWords = 13, kPatchPitch = 52, kPR = 22;  // raw patch: rows/cols -22..22 (13 aligned words per row)
constexpr int kBl = 39, kBlPitch = 40, kBR = 19;        // blurred patch: -19..19
__constant__ int c_umax[16] = {15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3};

struct DescSmem {
  uint8_t patch[kPatch * kPatchPitch];
  float rows[kPatch * kBlPitch];
  uint8_t blur[kBl * kBlPitch];
};

__global__ void __launch_bounds__(kDescWarps * 32) orb_describe_kernel(const __grid_constant__ OrbParams P, const uint8_t* __restrict__ pyr,
                                                                      const uint32_t* __restrict__ kept_pos, const float* __restrict__ kept_resp,
                                                                      const int* __restrict__ kept_count, const signed char* __restrict__ pattern,
                                                                      gb_keypoint* __restrict__ out_kps, uint8_t* __restrict__ out_desc,
                                                                      int capacity, int* __restrict__ out_count, int* __restrict__ out_status,
                                                                      const int* __restrict__ status_in) {
  gb_pdl_launch_dependents();
  gb_pdl_wait();
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ signed char s_pat[1024];
  DescSmem* sm = reinterpret_cast<DescSmem*>(smem_raw) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) reinterpret_cast<int*>(s_pat)[i] = __ldg(reinterpret_cast<const int*>(pattern) + i);
  // level prefix
  int total = 0, l = -1, base = 0;
  const int g = blockIdx.x * kDescWarps + warp;
  for (int k = 0; k < P.nlevels; ++k) {
    const int c = kept_count[k];
    if (l < 0 && g < total + c) { l = k; base = total; }
    total += c;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const int st = *status_in;
    out_count[0] = (total <= capacity && st == 0) ? total : 0;
    out_status[0] = st != 0 ? st : (total > capacity ? total : 0);
  }
  __syncthreads();
  if (l < 0 || total > capacity || *status_in != 0) return;
  const LevelInfo& L = P.lv[l];
  const uint32_t pos = kept_pos[l * kSelMax + (g - base)];
  const int x = pos & 0xffff, y = pos >> 16;
  const uint8_t* img = pyr + L.off;
  // raw 45x45 patch (always inside the level: border >= 22), staged with aligned 32-bit loads: 12 (or 13) words cover the 45
  // columns starting at the 4-byte boundary below x-22; `sh` is the byte offset of column x-22 inside the staged row
  const int xa = (x - kPR) & ~3, sh = (x - kPR) - xa;
  for (int i = lane; i < kPatch * kPatchWords; i += 32) {
    const int r = i / kPatchWords, wq = i - r * kPatchWords;
    const int gx = xa + 4 * wq;
    uint32_t v = 0;
    if (gx + 3 < L.pitch) v = __ldg(reinterpret_cast<const uint32_t*>(img + (size_t)(y - kPR + r) * L.pitch + gx));
    *reinterpret_cast<uint32_t*>(&sm->patch[r * kPatchPitch + 4 * wq]) = v;
  }
  __syncwarp();
  const uint8_t* patch = sm->patch + sh;  // patch[r * kPatchPitch + c] == level(y-22+r, x-22+c)
  // intensity-centroid orientation over the radius-15 disc: lane = row v+15
  int m01 = 0, m10 = 0;
  if (lane < 31) {
    const int v = lane - 15, d = c_umax[v < 0 ? -v : v];
    const uint8_t* row = &patch[(kPR + v) * kPatchPitch + kPR];
    int rs = 0, ru = 0;
    for (int u = -d; u <= d; ++u) { const int val = row[u]; rs += val; ru += u * val; }
    m01 = v * rs; m10 = ru;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { m01 += __shfl_xor_sync(0xffffffffu, m01, o); m10 += __shfl_xor_sync(0xffffffffu, m10, o); }
  const float angle = fast_atan2_deg((float)m01, (float)m10);
  // separable 7-tap float blur of the patch, cv2.sepFilter2D order: rows sequential-fma, columns symmetric-fma
  const float k0 = __uint_as_float(0x3d8fafb1u), k1 = __uint_as_float(0x3e06387eu), k2 = __uint_as_float(0x3e434a39u), k3 = __uint_as_float(0x3e5d4ae0u);
  for (int i = lane; i < kPatch * kBl; i += 32) {
    const int r = i / kBl, c = i % kBl;  // output col c <-> patch cols c..c+6
    const uint8_t* p = &patch[r * kPatchPitch + c];
    float s = __fmul_rn(k0, (float)p[0]);
    s = __fmaf_rn((float)p[1], k1, s);
    s = __fmaf_rn((float)p[2], k2, s);
    s = __fmaf_rn((float)p[3], k3, s);
    s = __fmaf_rn((float)p[4], k2, s);
    s = __fmaf_rn((float)p[5], k1, s);
    s = __fmaf_rn((float)p[6], k0, s);
    sm->rows[r * kBlPitch + c] = s;
  }
  __syncwarp();
  for (int i = lane; i < kBl * kBl; i += 32) {
    const int r = i / kBl, c = i % kBl;
    const float* q = &sm->rows[r * kBlPitch + c];
    float s = __fmul_rn(k3, q[3 * kBlPitch]);
    s = __fmaf_rn(__fadd_rn(q[2 * kBlPitch], q[4 * kBlPitch]), k2, s);
    s = __fmaf_rn(__fadd_rn(q[1 * kBlPitch], q[5 * kBlPitch]), k1, s);
    s = __fmaf_rn(__fadd_rn(q[0], q[6 * kBlPitch]), k0, s);
    int v = __float2int_rn(s);
    v = v < 0 ? 0 : (v > 255 ? 255 : v);
    sm->blur[r * kBlPitch + c] = (uint8_t)v;
  }
  __syncwarp();
  // 256 rotated binary tests: lane j produces descriptor byte j
  const float theta = __fmul_rn(angle, (float)(3.14159265358979323846 / 180.0));
  double sd, cd;
  det_sincos((double)theta, &sd, &cd);
  const float a = (float)cd, b = (float)sd;
  const uint8_t* center = &sm->blur[kBR * kBlPitch + kBR];
  int byte = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const signed char* pt = &s_pat[4 * (8 * lane + k)];
    const float px0 = (float)pt[0], py0 = (float)pt[1], px1 = (float)pt[2], py1 = (float)pt[3];
    const int ix0 = __float2int_rn(__fsub_rn(__fmul_rn(px0, a), __fmul_rn(py0, b)));
    const int iy0 = __float2int_rn(__fadd_rn(__fmul_rn(px0, b), __fmul_rn(py0, a)));
    const int ix1 = __float2int_rn(__fsub_rn(__fmul_rn(px1, a), __fmul_rn(py1, b)));
    const int iy1 = __float2int_rn(__fadd_rn(__fmul_rn(px1, b), __fmul_rn(py1, a)));
    const int t0 = center[iy0 * kBlPitch + ix0], t1 = center[iy1 * kBlPitch + ix1];
    byte |= (t0 < t1) << k;
  }
  out_desc[(size_t)g * 32 + lane] = (uint8_t)byte;
  if (lane == 0) {
    gb_keypoint kp;
    kp.x = __fmul_rn((float)x, L.scale);
    kp.y = __fmul_rn((float)y, L.scale);
    kp.size = __fmul_rn(31.f, L.scale);
    kp.angle = angle;
    kp.response = kept_resp[l * kSelMax + (g - base)];
    kp.octave = l;
    kp.class_id = -1;
    out_kps[g] = kp;
  }
}

}  // namespace

// ==========================================================================================================================
// host side
// ==========================================================================================================================
struct OrbState {
  // configuration the buffers were built for
  int w = 0, h = 0;
  gb_orb_cfg cfg{};
  OrbParams P{};
  FastMaps maps{};                      // TMA tensor maps of the pyramid levels (built with the buffers)
  // device buffers
  uint8_t* d_pyr = nullptr; size_t pyr_bytes = 0;
  void* d_color = nullptr; size_t color_cap = 0;  // packed colour frame before the gray conversion (grow-only)
  uint32_t* d_tabs = nullptr;           // resize tables
  uint32_t* d_cand_pos = nullptr; uint8_t* d_cand_score = nullptr; uint32_t* d_cand_key = nullptr; float* d_cand_resp = nullptr;
  uint32_t* d_surv_pos = nullptr;       // compact survivor lists share d_cand_key / d_cand_resp
  int* d_counts = nullptr;              // [kMaxLevels] candidates | [kMaxLevels] kept | [1] status | hist [kMaxLevels*256]
  uint32_t* d_kept_pos = nullptr; float* d_kept_resp = nullptr;
  signed char* d_pattern = nullptr;
  int total_cand = 0;
  bool valid = false;
};

static void orb_free_buffers(OrbState* s) {
  cudaFree(s->d_surv_pos); s->d_surv_pos = nullptr;
  cudaFree(s->d_color); s->d_color = nullptr; s->color_cap = 0;
  cudaFree(s->d_pyr); cudaFree(s->d_tabs); cudaFree(s->d_cand_pos); cudaFree(s->d_cand_score); cudaFree(s->d_cand_key);
  cudaFree(s->d_cand_resp); cudaFree(s->d_counts); cudaFree(s->d_kept_pos); cudaFree(s->d_kept_resp);
  s->d_pyr = nullptr; s->d_tabs = nullptr; s->d_cand_pos = nullptr; s->d_cand_score = nullptr; s->d_cand_key = nullptr;
  s->d_cand_resp = nullptr; s->d_counts = nullptr; s->d_kept_pos = nullptr; s->d_kept_resp = nullptr;
  s->valid = false;
}

void gb_orb_state_free(gb_ctx* ctx) {
  if (!ctx->orb) return;
  orb_free_buffers(ctx->orb);
  cudaFree(ctx->orb->d_pattern);
  delete ctx->orb;
  ctx->orb = nullptr;
}

static inline int cv_round_f(float v) { return (int)lrintf(v); }
// level size as cv2 computes it: cols * (1/scale) in float, round-half-even (NOT cols / scale: 477 / 1.2f -> 397, cv2 -> 398;
// pinned by tests/test_oracle_orb.py::test_level_sizes_match_cv2 and ::test_product_level_size_rule_equals_oracle)
static inline void orb_level_size(int w, int h, float scale, int* lw, int* lh) {
  const volatile float inv = 1.0f / scale;  // (volatile: the reciprocal must be rounded to float before the multiply)
  *lw = cv_round_f((float)w * inv);
  *lh = cv_round_f((float)h * inv);
}

static int orb_cfg_check(gb_ctx* ctx, const gb_orb_cfg* c) {
  if (!c || c->nfeatures <= 0 || c->nlevels < 1 || c->nlevels > kMaxLevels || !(c->scale_factor > 1.0f) || c->edge_threshold < 22 ||
      c->first_level != 0 || c->wta_k != 2 || c->score_type != 0 || c->patch_size != 31 || c->fast_threshold < 1 || c->fast_threshold > 254) {
    gb_set_error(ctx, "gb_orb: unsupported configuration (need nlevels 1..%d, scale>1, edge_threshold>=22, first_level 0, wta_k 2, "
                 "HARRIS score, patch 31, fast_threshold 1..254)", kMaxLevels);
    return GB_ERR_INVALID;
  }
  return GB_OK;
}

// (Re)build the per-resolution state: level geometry, quotas, resize tables, buffers.
static int orb_prepare(gb_ctx* ctx, int w, int h, const gb_orb_cfg* cfg) {
  if (!ctx->orb) {
    ctx->orb = new OrbState();
    GB_CUDA(ctx, cudaMalloc((void**)&ctx->orb->d_pattern, 1024));
    GB_CUDA(ctx, cudaMemcpyAsync(ctx->orb->d_pattern, kOrbPattern, 1024, cudaMemcpyHostToDevice, ctx->stream));
    GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  OrbState* s = ctx->orb;
  if (s->valid && s->w == w && s->h == h && memcmp(&s->cfg, cfg, sizeof *cfg) == 0) return GB_OK;
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  orb_free_buffers(s);
  if (w > 16384 || h > 16384) {
    gb_set_error(ctx, "gb_orb: image %dx%d too large (max 16384)", w, h);
    return GB_ERR_INVALID;
  }
  OrbParams& P = s->P;
  memset(&P, 0, sizeof P);
  P.fast_threshold = cfg->fast_threshold;
  P.border = cfg->edge_threshold;
  // quotas (App. A.3, float arithmetic as OpenCV)
  int quota[kMaxLevels];
  {
    const float factor = (float)(1.0 / (double)cfg->scale_factor);
    float nd = (float)cfg->nfeatures * (1.f - factor) / (1.f - (float)pow((double)factor, (double)cfg->nlevels));
    int sum = 0;
    for (int l = 0; l < cfg->nlevels - 1; ++l) {
      quota[l] = cv_round_f(nd);
      sum += quota[l];
      nd *= factor;
    }
    quota[cfg->nlevels - 1] = std::max(cfg->nfeatures - sum, 0);
  }
  size_t off = 0;
  int tiles = 0, cand = 0, coef = 0, nl = 0;
  for (int l = 0; l < cfg->nlevels; ++l) {
    const float sc = (float)pow((double)cfg->scale_factor, (double)l);
    int lw, lh;
    orb_level_size(w, h, sc, &lw, &lh);
    if (lw < 1 || lh < 1) break;
    LevelInfo& L = P.lv[l];
    L.w = lw; L.h = lh; L.pitch = (lw + 127) & ~127; L.quota = quota[l]; L.scale = sc;
    L.off = off;
    off += (size_t)L.pitch * lh;
    L.tiles_x = gb_div_up(lw, kTileW);
    L.tile_start = tiles;
    // levels too small to hold a keypoint produce none (and the oracle skips them): give them zero tiles
    const bool usable = lw > 2 * P.border && lh > 2 * P.border;
    if (!usable) L.tiles_x = 0;
    tiles += usable ? L.tiles_x * gb_div_up(lh, kTileH) : 0;
    L.cand_off = cand;
    L.cand_cap = usable ? (lw * lh) / 4 + 1024 : 0;
    cand += L.cand_cap;
    L.coef_off = coef;
    coef += lw + lh;
    nl = l + 1;
  }
  P.nlevels = nl;
  P.total_tiles = tiles;
  s->total_cand = cand;
  s->pyr_bytes = off + 256;
  // resize tables
  std::vector<uint32_t> tabs((size_t)coef + 1, 0);
  for (int l = 1; l < nl; ++l) {
    const LevelInfo &S = P.lv[l - 1], &D = P.lv[l];
    auto fill = [&](int src, int dst, uint32_t* out) {
      const double scale = (double)src / (double)dst;
      for (int d = 0; d < dst; ++d) {
        const double f = ((double)d + 0.5) * scale - 0.5;
        int i = (int)floor(f);
        int a = (int)lrint((f - (double)i) * 256.0);
        if (i < 0) { i = 0; a = 0; }
        if (i >= src - 1) { i = src - 1; a = 0; }
        out[d] = (uint32_t)i | ((uint32_t)a << 16);
      }
    };
    fill(S.w, D.w, tabs.data() + D.coef_off);
    fill(S.h, D.h, tabs.data() + D.coef_off + D.w);
  }
  GB_CUDA(ctx, cudaMalloc((void**)&s->d_pyr, s->pyr_bytes));
  GB_CUDA(ctx, cudaMemsetAsync(s->d_pyr, 0, s->pyr_bytes, ctx->stream));
  GB_CUDA(ctx, cudaMalloc((void**)&s->d_tabs, tabs.size() * 4));
  GB_CUDA(ctx, cudaMemcpyAsync(s->d_tabs, tabs.data(), tabs.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  const size_t nc = (size_t)std::max(cand, 1);
  GB_CUDA(ctx, cudaMalloc((void**)&s->d_cand_pos, nc * 4));
  GB_CUDA(ctx, cudaMalloc((void**)&s->d_cand_score, nc));
  GB_CUDA(ctx, cudaMalloc((void**)&s->d_cand_key, nc * 4));
  GB_CUDA(ctx, cudaMalloc((void**)&s->d_cand_resp, nc * 4));
  GB_CUDA(ctx, cudaMalloc((void**)&s->d_counts, (3 * kMaxLevels + 8 + kMaxLevels * 256) * sizeof(int)));
  GB_CUDA(ctx, cudaMalloc((void**)&s->d_surv_pos, nc * 4));
  GB_CUDA(ctx, cudaMalloc((void**)&s->d_kept_pos, (size_t)kMaxLevels * kSelMax * 4));
  GB_CUDA(ctx, cudaMalloc((void**)&s->d_kept_resp, (size_t)kMaxLevels * kSelMax * 4));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // tabs is a local vector
  {  // TMA tensor maps: one per level over the padded-pitch buffer, u8, box = the FAST input tile; out-of-image reads give 0
    typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                 const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    // looked up once per process; contexts on other threads may reach here at the same time (a function-local static is
    // initialised exactly once, the others wait for it)
    static const EncodeFn encode = []() -> EncodeFn {
      void* fn = nullptr;
      cudaDriverEntryPointQueryResult qr;
      if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || qr != cudaDriverEntryPointSuccess) {
        cudaGetLastError();
        fn = nullptr;
      }
      return (EncodeFn)fn;
    }();
    if (!encode) {
      gb_set_error(ctx, "gb_orb: cuTensorMapEncodeTiled is not available from this driver (the FAST kernel stages its tiles with TMA)");
      return GB_ERR_CUDA;
    }
    memset(&s->maps, 0, sizeof s->maps);
    for (int l = 0; l < nl; ++l) {
      const LevelInfo& L = P.lv[l];
      const cuuint64_t gdim[2] = {(cuuint64_t)L.w, (cuuint64_t)L.h};
      const cuuint64_t gstride[1] = {(cuuint64_t)L.pitch};
      const cuuint32_t box[2] = {(cuuint32_t)kInW, (cuuint32_t)kInH}, estr[2] = {1, 1};
      const CUresult r = encode(&s->maps.m[l], CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, s->d_pyr + L.off, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) {
        gb_set_error(ctx, "gb_orb: cuTensorMapEncodeTiled failed for level %d (%dx%d pitch %d): CUresult %d", l, L.w, L.h, L.pitch, (int)r);
        return GB_ERR_CUDA;
      }
    }
  }
  if (!gb_func_setup(ctx, (const void*)orb_describe_kernel, (int)(sizeof(DescSmem) * kDescWarps))) {
    gb_set_error(ctx, "gb_orb: cannot set the shared-memory limit of the describe kernel");
    return GB_ERR_CUDA;
  }
  s->w = w; s->h = h; s->cfg = *cfg; s->valid = true;
  return GB_OK;
}

// Enqueue the whole extraction of the frame already sitting in level 0 of the pyramid buffer.
static int orb_launch(gb_ctx* ctx, gb_features* out) {
  OrbState* s = ctx->orb;
  const OrbParams& P = s->P;
  cudaStream_t st = ctx->stream;
  int* d_counts = s->d_counts;
  int* d_kept = d_counts + kMaxLevels;
  int* d_status = d_counts + 2 * kMaxLevels;
  int* d_hist = d_counts + 2 * kMaxLevels + 8;
  int* d_surv = d_hist + kMaxLevels * 256;
  GB_CUDA(ctx, cudaMemsetAsync(d_counts, 0, (3 * kMaxLevels + 8 + kMaxLevels * 256) * sizeof(int), st));
  for (int l = 1; l < P.nlevels; ++l) {
    const LevelInfo &S = P.lv[l - 1], &D = P.lv[l];
    dim3 blk(64, 4), grd(gb_div_up(gb_div_up(D.w, 4), 64), gb_div_up(D.h, 4));
    GB_CUDA(ctx, gb_launch_pdl(orb_resize_kernel, grd, blk, 0, st, s->d_pyr + S.off, S.w, S.h, S.pitch, s->d_pyr + D.off, D.w, D.h, D.pitch,
                               s->d_tabs + D.coef_off, s->d_tabs + D.coef_off + D.w));
    GB_LAUNCH_CHECK(ctx);
  }
  if (P.total_tiles > 0) {
    const int fast_ctas = std::min(P.total_tiles, ctx->sm_count * 3);  // persistent: each CTA walks tiles blockIdx.x, +grid, ...
    GB_CUDA(ctx, gb_launch_pdl(orb_fast_kernel, dim3(fast_ctas), dim3(kFastThreads), 0, st, P, s->maps, s->d_cand_pos, s->d_cand_score, d_counts, d_hist));
    GB_LAUNCH_CHECK(ctx);
    GB_CUDA(ctx, gb_launch_pdl(orb_harris_kernel, dim3(32, P.nlevels), dim3(256), 0, st, P, s->d_pyr, s->d_cand_pos, s->d_cand_score, d_counts,
                               d_hist, s->d_cand_key, s->d_cand_resp, s->d_surv_pos, d_surv));
    GB_LAUNCH_CHECK(ctx);
    GB_CUDA(ctx, gb_launch_pdl(orb_select_kernel, dim3(P.nlevels), dim3(kSelThreads), 0, st, P, s->d_surv_pos, s->d_cand_key, s->d_cand_resp, d_surv,
                               d_counts, s->d_kept_pos, s->d_kept_resp, d_kept, d_status));
    GB_LAUNCH_CHECK(ctx);
  }
  const int blocks = std::max(1, gb_div_up(out->capacity, kDescWarps));
  GB_CUDA(ctx, gb_launch_pdl(orb_describe_kernel, dim3(blocks), dim3(kDescWarps * 32), sizeof(DescSmem) * kDescWarps, st, P, s->d_pyr, s->d_kept_pos,
                             s->d_kept_resp, d_kept, s->d_pattern, out->d_kps, out->d_desc, out->capacity, out->d_count, out->d_status, d_status));
  GB_LAUNCH_CHECK(ctx);
  out->h_count = -1;
  out->expect = std::min(out->capacity, s->cfg.nfeatures + s->cfg.nfeatures / 64 + 8);  // (a few ties above nfeatures are usual)
  return GB_OK;
}

extern "C" {

void gb_orb_cfg_default(gb_orb_cfg* c) {
  if (!c) return;
  c->nfeatures = 500;
  c->scale_factor = 1.2f;
  c->nlevels = 8;
  c->edge_threshold = 31;
  c->first_level = 0;
  c->wta_k = 2;
  c->score_type = 0;
  c->patch_size = 31;
  c->fast_threshold = 20;
}

// sync_after: a host image (or its staging copy) must have been consumed before the caller may touch it again; the one-shot
// gb_orb_extract synchronises in its own download instead (one synchronisation per host-buffer extraction)
// channels: 1 = gray (GImage 8UC1), 3 / 4 = packed colour (8UC3 / 8UC4), converted on the device; rgb_order: 0 = B,G,R[,A] (OpenCV,
// GSLAM IMAGE_BGRA), 1 = R,G,B[,A].  `pitch` is in bytes (>= width * channels).
static int orb_extract_to_impl(gb_ctx* ctx, const uint8_t* img, int img_is_device, int width, int height, int pitch, const gb_orb_cfg* cfg_in,
                               gb_features* out, bool sync_after, int channels = 1, int rgb_order = 0) {
  if (!ctx || !img || !out || width < 1 || height < 1 || (channels != 1 && channels != 3 && channels != 4) || pitch < width * channels) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  gb_orb_cfg cfg;
  if (cfg_in) cfg = *cfg_in; else gb_orb_cfg_default(&cfg);
  GB_CHECK(orb_cfg_check(ctx, &cfg));
  GB_CHECK(orb_prepare(ctx, width, height, &cfg));
  OrbState* s = ctx->orb;
  const LevelInfo& L0 = s->P.lv[0];
  if (channels != 1) {
    const size_t row = (size_t)width * channels, bytes = row * height;
    GB_CHECK(gb_dev_realloc(ctx, &s->d_color, &s->color_cap, bytes));
    if (img_is_device) {
      GB_CUDA(ctx, cudaMemcpy2DAsync(s->d_color, row, img, pitch, row, height, cudaMemcpyDeviceToDevice, ctx->stream));
    } else {
      cudaPointerAttributes at;
      const bool pinned = cudaPointerGetAttributes(&at, img) == cudaSuccess && at.type == cudaMemoryTypeHost;
      cudaGetLastError();
      const uint8_t* src = img;
      int spitch = pitch;
      if (!pinned) {
        GB_CHECK(gb_stage_reserve(ctx, ctx->h_stage_off + bytes + 1024));
        uint8_t* hs = (uint8_t*)gb_stage_alloc(ctx, bytes);
        for (int y = 0; y < height; ++y) memcpy(hs + (size_t)y * row, img + (size_t)y * pitch, row);
        src = hs;
        spitch = (int)row;
      }
      GB_CUDA(ctx, cudaMemcpy2DAsync(s->d_color, row, src, spitch, row, height, cudaMemcpyHostToDevice, ctx->stream));
    }
    orb_gray_kernel<<<dim3(gb_div_up(width, 256), height), 256, 0, ctx->stream>>>((const uint8_t*)s->d_color, width, height, channels, rgb_order,
                                                                                 s->d_pyr + L0.off, L0.pitch);
    GB_LAUNCH_CHECK(ctx);
  } else if (img_is_device) {
    GB_CUDA(ctx, cudaMemcpy2DAsync(s->d_pyr + L0.off, L0.pitch, img, pitch, width, height, cudaMemcpyDeviceToDevice, ctx->stream));
  } else {
    // pinned caller memory goes straight over PCIe; pageable memory is staged through the ctx's pinned buffer
    cudaPointerAttributes at;
    const bool pinned = cudaPointerGetAttributes(&at, img) == cudaSuccess && at.type == cudaMemoryTypeHost;
    cudaGetLastError();
    const uint8_t* src = img;
    int spitch = pitch;
    if (!pinned) {
      GB_CHECK(gb_stage_reserve(ctx, ctx->h_stage_off + (size_t)width * height + 1024));
      uint8_t* hs = (uint8_t*)gb_stage_alloc(ctx, (size_t)width * height);
      for (int y = 0; y < height; ++y) memcpy(hs + (size_t)y * width, img + (size_t)y * pitch, width);
      src = hs;
      spitch = width;
    }
    GB_CUDA(ctx, cudaMemcpy2DAsync(s->d_pyr + L0.off, L0.pitch, src, spitch, width, height, cudaMemcpyHostToDevice, ctx->stream));
  }
  GB_CHECK(orb_launch(ctx, out));
  if (!img_is_device && sync_after) GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // staging / caller buffer may be reused
  return GB_OK;
}

int gb_orb_extract_to(gb_ctx* ctx, const uint8_t* img, int img_is_device, int width, int height, int pitch, const gb_orb_cfg* cfg_in,
                      gb_features* out) {
  return orb_extract_to_impl(ctx, img, img_is_device, width, height, pitch, cfg_in, out, true);
}

static int orb_extract_host(gb_ctx* ctx, const uint8_t* img, int width, int height, int channels, int rgb_order, const gb_orb_cfg* cfg_in, gb_keypoint* kps,
                            uint8_t* desc, int* n);

int gb_orb_extract(gb_ctx* ctx, const uint8_t* img, int width, int height, const gb_orb_cfg* cfg_in, gb_keypoint* kps, uint8_t* desc,
                   int* n) {
  return orb_extract_host(ctx, img, width, height, 1, 0, cfg_in, kps, desc, n);
}

int gb_orb_extract_image(gb_ctx* ctx, const uint8_t* img, int width, int height, int channels, int rgb_order, const gb_orb_cfg* cfg_in, gb_keypoint* kps,
                         uint8_t* desc, int* n) {
  return orb_extract_host(ctx, img, width, height, channels, rgb_order, cfg_in, kps, desc, n);
}

static int orb_extract_host(gb_ctx* ctx, const uint8_t* img, int width, int height, int channels, int rgb_order, const gb_orb_cfg* cfg_in, gb_keypoint* kps,
                            uint8_t* desc, int* n) {
  if (!ctx || !img || !n || *n < 0) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  gb_orb_cfg cfg;
  if (cfg_in) cfg = *cfg_in; else gb_orb_cfg_default(&cfg);
  GB_CHECK(orb_cfg_check(ctx, &cfg));
  const int want_cap = std::max(*n, 2 * cfg.nfeatures + 256);
  if (!ctx->tmp_f || ctx->tmp_f->capacity < want_cap) {
    if (ctx->tmp_f) gb_features_destroy(ctx, ctx->tmp_f);
    ctx->tmp_f = nullptr;
    GB_CHECK(gb_features_create(ctx, want_cap, &ctx->tmp_f));
  }
  gb_features* f = ctx->tmp_f;
  GB_CHECK(orb_extract_to_impl(ctx, img, 0, width, height, width * channels, &cfg, f, *n <= 0, channels, rgb_order));
  const int cap = *n;
  if (cap > 0) {  // one synchronisation: the count travels with the rows
    int m = cap;
    const int rc = gb_features_download(ctx, f, kps, desc, &m);
    *n = m;
    if (rc == GB_ERR_CAPACITY && m > cap) gb_set_error(ctx, "gb_orb_extract: %d keypoints > caller capacity %d", m, cap);
    return rc;
  }
  int cnt = 0;
  const int rc = gb_features_count(ctx, f, &cnt);
  *n = cnt;
  if (rc != GB_OK) return rc;
  if (cnt > 0) {
    gb_set_error(ctx, "gb_orb_extract: %d keypoints > caller capacity %d", cnt, cap);
    return GB_ERR_CAPACITY;
  }
  return GB_OK;
}

// host-only (no device needed): the pyramid level size the extractor uses, for the CPU parity test against the oracle / cv2
GB_API int gb_dbg_orb_level_size(int w, int h, float scale_factor, int level, int* lw, int* lh) {
  if (!lw || !lh || level < 0) return GB_ERR_INVALID;
  orb_level_size(w, h, (float)pow((double)scale_factor, (double)level), lw, lh);
  return GB_OK;
}

// ---- test hook: candidates of the LAST extraction on this ctx (after FAST+NMS+border), and the kept lists --------------
GB_API int gb_dbg_orb_candidates(gb_ctx* ctx, int level, uint32_t* pos, uint8_t* score, float* resp, uint32_t* key, int cap, int* n,
                                 uint32_t* kept_pos, int kept_cap, int* n_kept) {
  if (!ctx || !ctx->orb || !ctx->orb->valid || level < 0 || level >= ctx->orb->P.nlevels) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  OrbState* s = ctx->orb;
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int counts[2 * kMaxLevels];
  GB_CUDA(ctx, cudaMemcpy(counts, s->d_counts, sizeof counts, cudaMemcpyDeviceToHost));
  const LevelInfo& L = s->P.lv[level];
  const int c = std::min(counts[level], L.cand_cap);
  *n = c;
  const int m = std::min(c, cap);
  if (pos) GB_CUDA(ctx, cudaMemcpy(pos, s->d_cand_pos + L.cand_off, (size_t)m * 4, cudaMemcpyDeviceToHost));
  if (score) GB_CUDA(ctx, cudaMemcpy(score, s->d_cand_score + L.cand_off, (size_t)m, cudaMemcpyDeviceToHost));
  if (resp) GB_CUDA(ctx, cudaMemcpy(resp, s->d_cand_resp + L.cand_off, (size_t)m * 4, cudaMemcpyDeviceToHost));
  if (key) GB_CUDA(ctx, cudaMemcpy(key, s->d_cand_key + L.cand_off, (size_t)m * 4, cudaMemcpyDeviceToHost));
  const int k = counts[kMaxLevels + level];
  if (n_kept) *n_kept = k;
  if (kept_pos) GB_CUDA(ctx, cudaMemcpy(kept_pos, s->d_kept_pos + (size_t)level * kSelMax, (size_t)std::min(k, kept_cap) * 4, cudaMemcpyDeviceToHost));
  return GB_OK;
}

// test hook: download pyramid level `level` of the LAST extraction (dense w*h bytes); returns its size through w/h
GB_API int gb_dbg_orb_level(gb_ctx* ctx, int level, uint8_t* out, int cap, int* w, int* h) {
  if (!ctx || !ctx->orb || !ctx->orb->valid || level < 0 || level >= ctx->orb->P.nlevels) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  OrbState* s = ctx->orb;
  const LevelInfo& L = s->P.lv[level];
  *w = L.w; *h = L.h;
  if (!out || cap < L.w * L.h) return GB_ERR_CAPACITY;
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  GB_CUDA(ctx, cudaMemcpy2D(out, L.w, s->d_pyr + L.off, L.pitch, L.w, L.h, cudaMemcpyDeviceToHost));
  return GB_OK;
}

}  // extern "C"
