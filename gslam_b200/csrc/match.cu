// gslam_b200/csrc/match.cu — 256-bit Hamming brute-force matcher (K5).
//
// Behind: Vocabulary::DistanceFactory::hamming32 (GSLAM/core/Vocabulary.h:485-491) as the distance; argmin/2nd-best with
// cv::BFMatcher(NORM_HAMMING) tie rules (lowest train index; SURVEY.md App. A.7).
//
// Shape of the work: Q x T pairs, each 8 XOR + 8 POPC + adds on 32-byte rows.  Algorithmic HBM traffic is only
// 32(Q+T)+12Q bytes, so this kernel is bound by the integer POPC pipe, not by HBM (DESIGN.md §match).  One thread owns
// one query row in registers; a CTA stages a chunk of train rows in shared memory and every lane reads the same row
// (broadcast, conflict-free).  The train dimension is split across blockIdx.y so that Q=2000 still fills 132 SMs; the
// last CTA of each query tile (atomic ticket) merges the per-chunk (best, 2nd) partials in ascending chunk order, which
// reproduces the sequential "first minimum wins" tie rule exactly.  One launch, no atomics on the data path.
#include "common.cuh"

namespace {

constexpr int kQPerCta = 128;  // threads per CTA == queries per CTA

struct MatchPartial {
  int32_t d0, b0, d1;
};

__device__ __forceinline__ int ham256(const uint4& a0, const uint4& a1, const uint4& b0, const uint4& b1) {
  return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) + __popc(a1.x ^ b1.x) +
         __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// d_nq / d_nt (nullable): device-side row counts of an extraction still in flight -- the launch is then sized for the capacities
// passed as nq / nt and the kernel clips to the real counts, so that extract -> match chains without a host round trip.
// STEREO (rectified pair, left = query, right = train): a right keypoint is a candidate of a left one iff
// |y_R - y_L| <= band and min_disp <= x_L - x_R <= max_disp (level-0 pixel coordinates, float compares); everything else -- the
// distance, the (distance, index) order, the tie rule -- is the matcher's.  The right keypoints' (x, y) ride along with the staged
// descriptors; the popcounts are only evaluated for candidates (a few percent of the pairs).
struct StereoArgs {
  const gb_keypoint* qk;
  const gb_keypoint* tk;
  float band, min_disp, max_disp;
};

template <bool STEREO>
__global__ void __launch_bounds__(kQPerCta) match_kernel(const uint4* __restrict__ q, int nq, const uint4* __restrict__ t,
                                                         int nt, int chunk, MatchPartial* __restrict__ partial,
                                                         unsigned int* __restrict__ tickets, int32_t* __restrict__ best_idx,
                                                         int32_t* __restrict__ best_dist, int32_t* __restrict__ second_dist,
                                                         const int* __restrict__ d_nq, const int* __restrict__ d_nt, StereoArgs st) {
  gb_pdl_launch_dependents();
  gb_pdl_wait();
  const int pstride = nq;  // layout of the partials: [split][query capacity]
  if (d_nq) nq = min(max(*d_nq, 0), nq);
  if (d_nt) nt = min(max(*d_nt, 0), nt);
  if ((int)(blockIdx.x * kQPerCta) >= nq) return;  // a query tile beyond the real count: none of its CTAs has anything to merge
  const int nsplit = d_nt ? max(1, (nt + chunk - 1) / chunk) : (int)gridDim.y;  // splits that hold train rows (>= 1: the empty-train case)
  if ((int)blockIdx.y >= nsplit) return;
  extern __shared__ uint4 s_train[];  // chunk rows x 2 uint4
  __shared__ bool s_last;
  const int tid = threadIdx.x;
  const int qi = blockIdx.x * kQPerCta + tid;
  const int t0 = blockIdx.y * chunk;
  const int tn = min(chunk, nt - t0);

  // stage the train chunk: 2 uint4 per row, fully coalesced
  for (int i = tid; i < tn * 2; i += kQPerCta) s_train[i] = __ldg(t + (size_t)t0 * 2 + i);
  float2* s_xy = reinterpret_cast<float2*>(s_train + 2 * chunk);  // STEREO: (x, y) of the staged right keypoints
  if (STEREO)
    for (int i = tid; i < tn; i += kQPerCta) s_xy[i] = make_float2(st.tk[t0 + i].x, st.tk[t0 + i].y);
  uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0;
  float qx = 0.f, qy = 0.f;
  if (qi < nq) {
    q0 = __ldg(q + (size_t)qi * 2);
    q1 = __ldg(q + (size_t)qi * 2 + 1);
    if (STEREO) { qx = st.qk[qi].x; qy = st.qk[qi].y; }
  }
  __syncthreads();

  int d0 = 257, d1 = 257, b0 = -1;
  if (STEREO) {
    for (int j = 0; j < tn; ++j) {
      const float2 p = s_xy[j];
      const float disp = qx - p.x;
      if (!(fabsf(p.y - qy) <= st.band && disp >= st.min_disp && disp <= st.max_disp)) continue;
      const uint4 a = s_train[2 * j], b = s_train[2 * j + 1];
      const int d = ham256(q0, q1, a, b);
      const bool lt = d < d0;
      d1 = lt ? d0 : min(d1, d);
      b0 = lt ? (t0 + j) : b0;
      d0 = lt ? d : d0;
    }
  } else {
#pragma unroll 4
    for (int j = 0; j < tn; ++j) {
      const uint4 a = s_train[2 * j], b = s_train[2 * j + 1];
      const int d = ham256(q0, q1, a, b);
      const bool lt = d < d0;
      d1 = lt ? d0 : min(d1, d);
      b0 = lt ? (t0 + j) : b0;
      d0 = lt ? d : d0;
    }
  }

  if (nsplit == 1) {
    if (qi < nq) {
      if (best_idx) best_idx[qi] = b0;
      if (best_dist) best_dist[qi] = d0;
      if (second_dist) second_dist[qi] = d1;
    }
    return;
  }
  if (qi < nq) {
    MatchPartial p;
    p.d0 = d0;
    p.b0 = b0;
    p.d1 = d1;
    partial[(size_t)blockIdx.y * pstride + qi] = p;  // [split][query]: coalesced across the CTA
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned int prev = atomicAdd(&tickets[blockIdx.x], 1u);
    s_last = (prev == (unsigned int)nsplit - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  if (qi < nq) {
    int D0 = 257, D1 = 257, B0 = -1;
    for (int s = 0; s < nsplit; ++s) {  // ascending train index == sequential scan order
      const MatchPartial* pp = partial + (size_t)s * pstride + qi;
      const int pd0 = __ldcg(&pp->d0), pb0 = __ldcg(&pp->b0), pd1 = __ldcg(&pp->d1);
      if (pd0 < D0) {
        D1 = min(D0, pd1);
        D0 = pd0;
        B0 = pb0;
      } else {
        D1 = min(D1, pd0);
      }
    }
    if (best_idx) best_idx[qi] = B0;
    if (best_dist) best_dist[qi] = D0;
    if (second_dist) second_dist[qi] = D1;
  }
  if (tid == 0) tickets[blockIdx.x] = 0;  // re-arm for the next launch on this stream
}

// POPC-pipe ceiling of this device, measured (bench.py: the matcher's roofline denominator): every thread keeps 16 independent
// x = popc(x ^ m) chains in flight -- the same LOP3 + POPC pair as the matcher's inner loop, nothing else.
__global__ void __launch_bounds__(256) popc_peak_kernel(unsigned int* __restrict__ out, int iters, unsigned int seed) {
  unsigned int x[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) x[k] = seed * (threadIdx.x + 1u) + 0x9e3779b9u * (k + 1u) + blockIdx.x;
  unsigned int m = seed | 0x80000001u;
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int k = 0; k < 16; ++k) x[k] = __popc(x[k] ^ m) | (x[k] << 7);  // (the shift/or keeps the chain from collapsing to a constant)
    m = m * 1664525u + 1013904223u;
  }
  unsigned int acc = 0;
#pragma unroll
  for (int k = 0; k < 16; ++k) acc ^= x[k];
  if (acc == 0x12345u) out[0] = acc;  // (never true in practice; keeps the loop alive)
}

}  // namespace

struct MatchState {
  void* d_partial = nullptr;
  size_t partial_cap = 0;
  void* d_tickets = nullptr;
  size_t tickets_cap = 0;
};

void gb_match_state_free(gb_ctx* ctx) {
  if (!ctx->match) return;
  cudaFree(ctx->match->d_partial);
  cudaFree(ctx->match->d_tickets);
  delete ctx->match;
  ctx->match = nullptr;
}

// Enqueue the match of (d_q, nq) against (d_t, nt) on the ctx stream.  Outputs are device pointers (may be null).
// nq / nt: row counts, or -- with d_nq / d_nt -- CAPACITIES the launch must cover while the real counts are read on the device; the
// work split is then tuned for the expected counts eq / et (<= 0: unknown, use the capacities).
int gb_match_launch(gb_ctx* ctx, const uint8_t* d_q, int nq, const uint8_t* d_t, int nt, int32_t* d_best, int32_t* d_dist,
                    int32_t* d_dist2, const int* d_nq = nullptr, const int* d_nt = nullptr, const StereoArgs* stereo = nullptr, int eq = 0,
                    int et = 0) {
  if (nq <= 0) return GB_OK;
  if (!ctx->match) ctx->match = new MatchState();
  MatchState* ms = ctx->match;
  const int qtiles = gb_div_up(nq, kQPerCta);
  if (eq <= 0 || eq > nq) eq = nq;
  if (et <= 0 || et > nt) et = nt;
  // split the train rows so that ~2 CTAs land on every SM; chunk is a multiple of 8 rows, at most 1024 rows (32 KB)
  int nsplit = 1, chunk = nt > 0 ? nt : 1;
  if (nt > 0) {
    nsplit = gb_div_up(2 * ctx->sm_count, gb_div_up(eq, kQPerCta));
    const int max_split = gb_div_up(et, 32);
    if (nsplit > max_split) nsplit = max_split;
    if (nsplit < 1) nsplit = 1;
    chunk = gb_div_up(gb_div_up(et, nsplit), 8) * 8;
    if (chunk > 1024) chunk = 1024;
    nsplit = gb_div_up(nt, chunk);
  }
  if (nt <= 0) {  // nothing to match against: -1 / 257 / 257 through the same kernel with an empty chunk
    nsplit = 1;
    chunk = 8;
  }
  GB_CHECK(gb_dev_realloc(ctx, &ms->d_partial, &ms->partial_cap, (size_t)nsplit * nq * sizeof(MatchPartial)));
  if ((size_t)qtiles * sizeof(unsigned int) > ms->tickets_cap) {
    GB_CHECK(gb_dev_realloc(ctx, &ms->d_tickets, &ms->tickets_cap, (size_t)qtiles * sizeof(unsigned int)));
    GB_CUDA(ctx, cudaMemsetAsync(ms->d_tickets, 0, ms->tickets_cap, ctx->stream));
  }
  dim3 grid(qtiles, nsplit);
  const size_t smem = (size_t)chunk * (stereo ? 40 : 32);
  StereoArgs sa = {};
  if (stereo) sa = *stereo;
  if (stereo)
    GB_CUDA(ctx, gb_launch_pdl(match_kernel<true>, grid, dim3(kQPerCta), smem, ctx->stream, (const uint4*)d_q, nq, (const uint4*)d_t, nt > 0 ? nt : 0, chunk,
                               (MatchPartial*)ms->d_partial, (unsigned int*)ms->d_tickets, d_best, d_dist, d_dist2, d_nq, d_nt, sa));
  else
    GB_CUDA(ctx, gb_launch_pdl(match_kernel<false>, grid, dim3(kQPerCta), smem, ctx->stream, (const uint4*)d_q, nq, (const uint4*)d_t, nt > 0 ? nt : 0, chunk,
                               (MatchPartial*)ms->d_partial, (unsigned int*)ms->d_tickets, d_best, d_dist, d_dist2, d_nq, d_nt, sa));
  GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}

extern "C" {

// test / bench hook: measured POPC throughput of the device in popc32 per second (all SMs, 16 independent chains per thread)
GB_API int gb_dbg_popc_peak(gb_ctx* ctx, double* popc_per_s) {
  if (!ctx || !popc_per_s) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  unsigned int* d_out = nullptr;
  GB_CUDA(ctx, cudaMalloc((void**)&d_out, 64));
  const int ctas = ctx->sm_count * 8, iters = 4096;
  cudaEvent_t e0, e1;
  GB_CUDA(ctx, cudaEventCreate(&e0));
  GB_CUDA(ctx, cudaEventCreate(&e1));
  float best = 1e30f;
  for (int rep = 0; rep < 4; ++rep) {  // rep 0 warms up
    GB_CUDA(ctx, cudaEventRecord(e0, ctx->stream));
    popc_peak_kernel<<<ctas, 256, 0, ctx->stream>>>(d_out, iters, 12345u + rep);
    GB_LAUNCH_CHECK(ctx);
    GB_CUDA(ctx, cudaEventRecord(e1, ctx->stream));
    GB_CUDA(ctx, cudaEventSynchronize(e1));
    float ms = 0.f;
    GB_CUDA(ctx, cudaEventElapsedTime(&ms, e0, e1));
    if (rep > 0 && ms < best) best = ms;
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaFree(d_out);
  *popc_per_s = (double)ctas * 256.0 * iters * 16.0 / (best * 1e-3);
  return GB_OK;
}

int gb_match_features(gb_ctx* ctx, gb_features* fq, gb_features* ft) {
  if (!ctx || !fq || !ft) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  if (fq->h_count < 0 || ft->h_count < 0) {
    // an extraction is still in flight: no host round trip -- launch for the capacities, the kernel reads the device-side counts
    fq->n_matched = -1;  // resolved by gb_match_download
    return gb_match_launch(ctx, fq->d_desc, fq->h_count >= 0 ? fq->h_count : fq->capacity, ft->d_desc, ft->h_count >= 0 ? ft->h_count : ft->capacity,
                           fq->d_best, fq->d_dist, fq->d_dist2, fq->h_count >= 0 ? nullptr : fq->d_count, ft->h_count >= 0 ? nullptr : ft->d_count,
                           nullptr, fq->expect, ft->expect);
  }
  const int nq = fq->h_count, nt = ft->h_count;
  fq->n_matched = nq;
  return gb_match_launch(ctx, fq->d_desc, nq, ft->d_desc, nt, fq->d_best, fq->d_dist, fq->d_dist2);
}

// Rectified-stereo row-band match, device-resident: left = query, right = train; results with gb_match_download(left).
int gb_match_stereo_features(gb_ctx* ctx, gb_features* left, gb_features* right, float band_rows, float min_disparity, float max_disparity) {
  if (!ctx || !left || !right || !(band_rows >= 0.f) || !(max_disparity >= min_disparity)) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  StereoArgs sa;
  sa.qk = left->d_kps; sa.tk = right->d_kps; sa.band = band_rows; sa.min_disp = min_disparity; sa.max_disp = max_disparity;
  const bool async = left->h_count < 0 || right->h_count < 0;
  left->n_matched = async ? -1 : left->h_count;
  return gb_match_launch(ctx, left->d_desc, left->h_count >= 0 ? left->h_count : left->capacity, right->d_desc,
                         right->h_count >= 0 ? right->h_count : right->capacity, left->d_best, left->d_dist, left->d_dist2,
                         left->h_count >= 0 ? nullptr : left->d_count, right->h_count >= 0 ? nullptr : right->d_count, &sa, left->expect, right->expect);
}

// Host-buffer variant (what the Svar module's match_stereo binds).
int gb_match_stereo(gb_ctx* ctx, const gb_keypoint* kps_left, const uint8_t* desc_left, int nl, const gb_keypoint* kps_right, const uint8_t* desc_right,
                    int nr, float band_rows, float min_disparity, float max_disparity, int32_t* best_idx, int32_t* best_dist, int32_t* second_dist) {
  if (!ctx || nl < 0 || nr < 0 || (nl > 0 && (!kps_left || !desc_left)) || (nr > 0 && (!kps_right || !desc_right))) return GB_ERR_INVALID;
  if (nl == 0) return GB_OK;
  CtxLock lk(ctx);
  auto ensure = [&](gb_features** f, int n) -> int {
    if (*f && (*f)->capacity >= n) return GB_OK;
    if (*f) gb_features_destroy(ctx, *f);
    *f = nullptr;
    return gb_features_create(ctx, n + n / 4 + 64, f);
  };
  GB_CHECK(ensure(&ctx->tmp_q, nl));
  GB_CHECK(ensure(&ctx->tmp_t, nr > 0 ? nr : 1));
  GB_CHECK(gb_features_upload(ctx, ctx->tmp_q, kps_left, desc_left, nl));
  GB_CHECK(gb_features_upload(ctx, ctx->tmp_t, nr > 0 ? kps_right : nullptr, nr > 0 ? desc_right : desc_left, nr));
  GB_CHECK(gb_match_stereo_features(ctx, ctx->tmp_q, ctx->tmp_t, band_rows, min_disparity, max_disparity));
  int n = nl;
  return gb_match_download(ctx, ctx->tmp_q, best_idx, best_dist, second_dist, &n);
}

int gb_match_download(gb_ctx* ctx, gb_features* fq, int32_t* best_idx, int32_t* best_dist, int32_t* second_dist, int* n) {
  if (!ctx || !fq || !n) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  if (fq->n_matched < 0) GB_CHECK(gb_features_count(ctx, fq, &fq->n_matched));  // (the match was enqueued behind an extraction in flight)
  const int cap = *n, cnt = fq->n_matched;
  *n = cnt;
  if (cnt > cap) {
    gb_set_error(ctx, "gb_match_download: %d matches > caller capacity %d", cnt, cap);
    return GB_ERR_CAPACITY;
  }
  if (cnt == 0) return GB_OK;
  const size_t bytes = (size_t)cnt * sizeof(int32_t);
  GB_CHECK(gb_stage_reserve(ctx, ctx->h_stage_off + 3 * bytes + 1024));
  int32_t* h0 = (int32_t*)gb_stage_alloc(ctx, bytes);
  int32_t* h1 = (int32_t*)gb_stage_alloc(ctx, bytes);
  int32_t* h2 = (int32_t*)gb_stage_alloc(ctx, bytes);
  if (best_idx) GB_CUDA(ctx, cudaMemcpyAsync(h0, fq->d_best, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  if (best_dist) GB_CUDA(ctx, cudaMemcpyAsync(h1, fq->d_dist, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  if (second_dist) GB_CUDA(ctx, cudaMemcpyAsync(h2, fq->d_dist2, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (best_idx) memcpy(best_idx, h0, bytes);
  if (best_dist) memcpy(best_dist, h1, bytes);
  if (second_dist) memcpy(second_dist, h2, bytes);
  return GB_OK;
}

int gb_match_hamming(gb_ctx* ctx, const uint8_t* query, int nq, const uint8_t* train, int nt, int32_t* best_idx,
                     int32_t* best_dist, int32_t* second_dist) {
  if (!ctx || nq < 0 || nt < 0 || (nq > 0 && !query) || (nt > 0 && !train)) return GB_ERR_INVALID;
  if (nq == 0) return GB_OK;
  CtxLock lk(ctx);
  auto ensure = [&](gb_features** f, int n) -> int {
    if (*f && (*f)->capacity >= n) return GB_OK;
    if (*f) gb_features_destroy(ctx, *f);
    *f = nullptr;
    return gb_features_create(ctx, n + n / 4 + 64, f);
  };
  GB_CHECK(ensure(&ctx->tmp_q, nq));
  GB_CHECK(ensure(&ctx->tmp_t, nt > 0 ? nt : 1));
  gb_features *fq = ctx->tmp_q, *ft = ctx->tmp_t;
  const size_t bq = (size_t)nq * 32, bt = (size_t)nt * 32, bo = (size_t)nq * sizeof(int32_t);
  GB_CHECK(gb_stage_reserve(ctx, bq + bt + 3 * bo + 4096));
  uint8_t* hq = (uint8_t*)gb_stage_alloc(ctx, bq);
  memcpy(hq, query, bq);
  GB_CUDA(ctx, cudaMemcpyAsync(fq->d_desc, hq, bq, cudaMemcpyHostToDevice, ctx->stream));
  if (nt > 0) {
    uint8_t* ht = (uint8_t*)gb_stage_alloc(ctx, bt);
    memcpy(ht, train, bt);
    GB_CUDA(ctx, cudaMemcpyAsync(ft->d_desc, ht, bt, cudaMemcpyHostToDevice, ctx->stream));
  }
  fq->h_count = nq;
  ft->h_count = nt;
  fq->n_matched = nq;
  GB_CHECK(gb_match_launch(ctx, fq->d_desc, nq, ft->d_desc, nt, fq->d_best, fq->d_dist, fq->d_dist2));
  int32_t* h0 = (int32_t*)gb_stage_alloc(ctx, bo);
  int32_t* h1 = (int32_t*)gb_stage_alloc(ctx, bo);
  int32_t* h2 = (int32_t*)gb_stage_alloc(ctx, bo);
  if (best_idx) GB_CUDA(ctx, cudaMemcpyAsync(h0, fq->d_best, bo, cudaMemcpyDeviceToHost, ctx->stream));
  if (best_dist) GB_CUDA(ctx, cudaMemcpyAsync(h1, fq->d_dist, bo, cudaMemcpyDeviceToHost, ctx->stream));
  if (second_dist) GB_CUDA(ctx, cudaMemcpyAsync(h2, fq->d_dist2, bo, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (best_idx) memcpy(best_idx, h0, bo);
  if (best_dist) memcpy(best_dist, h1, bo);
  if (second_dist) memcpy(second_dist, h2, bo);
  return GB_OK;
}

}  // extern "C"
