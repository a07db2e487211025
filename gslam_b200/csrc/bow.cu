// gslam_b200/csrc/bow.cu — bag-of-words transform of a frame's descriptors: GSLAM::Vocabulary::transform(features, BowVector&,
// FeatureVector&, levelsup)  (GSLAM/core/Vocabulary.h:1558-1622; the tree walk :1692-1736; distance hamming32 :485-491; accumulation
// helpers addWeight / addIfNotExist / normalize / addFeature :357-425; which scoring normalises how :667-684).  SURVEY.md section 8f-4.
// The published CPU figure for this call is 615.5 us (doc/doxygen/4_2_tools.dox:43, "Trans ORB-4").
//
// The vocabulary is the reference's own flat layout (Vocabulary.h:583-601): node p's children are rows p*k+1 .. p*k+childNum[p] of
// the node-descriptor matrix (32-byte rows here: ORB / 256-bit binary vocabularies); a leaf's node id IS its word id.
//   K-bow1 bow_walk_kernel : a group of 16 (k <= 16) or 32 lanes per descriptor; lane c reads child c (two 16-byte loads + its child
//            count, so the next level needs no extra dependent load), Hamming distance with POPC, packed (distance, child) minimum
//            over the group = the reference's first-strict-minimum rule; one dependent memory round per tree level.
//   K-bow2 bow_reduce_kernel : one CTA; bitonic sort of (word << 32 | feature) and (node << 32 | feature) keys in shared memory,
//            run heads -> the BowVector in std::map order, values accumulated exactly as the reference does (float, += the word's
//            weight once per occurrence in feature order; first occurrence only for IDF / BINARY), L1 / L2 norm in double over the
//            words in ascending order, FeatureVector flattened in map order.
// Integer outputs (words, nodes, feature indices) are bit-exact; values are bit-exact unless the double norm needs more than 53 bits
// (the norm is folded in a fixed tree, the reference adds sequentially: both are exact for float weights spanning < 2^29).
// A leaf met above level L - levelsup leaves the reference's node id uninitialised (:1579,1728); it files under the leaf itself here.
#include "common.cuh"

struct gb_vocabulary {
  int k = 0, L = 0, weighting = 0, scoring = 0;
  uint32_t n_nodes = 0;
  uint32_t* d_child = nullptr;  // [n_nodes]
  float* d_weight = nullptr;    // [n_nodes]
  uint4* d_desc = nullptr;      // [n_nodes][2]
  // per-call scratch (grow-only): per-feature word / node / weight, sorted keys (large inputs), outputs
  uint8_t* d_feat = nullptr; size_t feat_cap = 0;
  uint32_t* d_fword = nullptr; size_t fword_cap = 0;  // [n] word, [n] node, [n] weight bits
  unsigned long long* d_keys = nullptr; size_t keys_cap = 0;  // [2][npad] when the keys do not fit shared memory
  uint8_t* d_out = nullptr; size_t out_cap = 0;       // [counts(4 ints) | words u64[n] | fv_node u64[n] | values f32[n] | fv_feat u32[n]]
};

namespace {

enum { W_TF_IDF = 0, W_TF = 1, W_IDF = 2, W_BINARY = 3 };  // Vocabulary.h:88-94
enum { S_L1 = 0, S_L2 = 1, S_CHI = 2, S_KL = 3, S_BHATT = 4, S_DOT = 5 };  // Vocabulary.h:97-105

constexpr int kWalkThreads = 256;
constexpr int kRedThreads = 1024;
constexpr int kSmemKeys = 8192;  // keys per sort held in shared memory (2 arrays x 8192 x 8 B = 128 KB)

template <int G>  // lanes per descriptor
__global__ void __launch_bounds__(kWalkThreads) bow_walk_kernel(int k, int L, const uint32_t* __restrict__ child, const float* __restrict__ weight,
                                                                const uint4* __restrict__ desc, const uint4* __restrict__ feats, int n,
                                                                const int* __restrict__ d_count, int levelsup, uint32_t* __restrict__ f_word,
                                                                uint32_t* __restrict__ f_node, float* __restrict__ f_weight) {
  const int gt = blockIdx.x * kWalkThreads + threadIdx.x;
  const int f = gt / G, c = gt % G;
  if (d_count) n = min(n, *d_count);
  if (f >= n) return;  // (whole groups leave together: kWalkThreads % G == 0)
  const uint4 a0 = __ldg(feats + 2 * (size_t)f), a1 = __ldg(feats + 2 * (size_t)f + 1);
  const int nid_level = L - levelsup;
  uint32_t cur = 0, nid = nid_level <= 0 ? 0u : 0xffffffffu;
  uint32_t nch = __ldg(child);
  int level = 0;
  const unsigned gmask = G == 32 ? 0xffffffffu : (0xffffu << ((threadIdx.x & 16)));
  while (nch != 0) {
    ++level;
    const uint32_t id = cur * (uint32_t)k + 1u + (uint32_t)c;
    uint32_t key = 0xffffffffu, my_nch = 0;
    if ((uint32_t)c < nch) {
      const uint4 b0 = __ldg(desc + 2 * (size_t)id), b1 = __ldg(desc + 2 * (size_t)id + 1);
      my_nch = __ldg(child + id);
      const uint32_t d = __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) + __popc(a1.x ^ b1.x) +
                         __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
      key = (d << 8) | (uint32_t)c;  // smallest distance, then smallest child index = the first strict minimum of the reference's scan
    }
    uint32_t best = key;
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(gmask, best, o, G));
    const int win = (int)(best & 0xffu);
    cur = cur * (uint32_t)k + 1u + (uint32_t)win;
    nch = __shfl_sync(gmask, my_nch, win, G);
    if (level == nid_level) nid = cur;
  }
  if (c == 0) {
    f_word[f] = cur;
    f_node[f] = nid == 0xffffffffu ? cur : nid;
    f_weight[f] = __ldg(weight + cur);
  }
}

__device__ __forceinline__ void bitonic_sort(unsigned long long* keys, int npad) {
  for (int size = 2; size <= npad; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < npad / 2; t += kRedThreads) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const bool up = (lo & size) == 0;
        const unsigned long long a = keys[lo], b = keys[hi];
        if ((a > b) == up) { keys[lo] = b; keys[hi] = a; }
      }
    }
  __syncthreads();
}

// block-wide exclusive scan of one int per thread (kRedThreads threads); returns the exclusive prefix, *total = the sum
__device__ __forceinline__ int block_exscan(int v, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  __syncthreads();
  if (lane == 31) s_warp[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
    s_warp[lane] = w;
  }
  __syncthreads();
  const int base = warp > 0 ? s_warp[warp - 1] : 0;
  *total = s_warp[kRedThreads / 32 - 1];
  return base + x - v;
}

__device__ __forceinline__ double block_sum_d(double v, double* s_part) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    double t = s_part[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) s_part[32] = t;
  }
  __syncthreads();
  return s_part[32];
}

// out_counts: [0] words, [1] feature-vector entries
__global__ void __launch_bounds__(kRedThreads, 1) bow_reduce_kernel(int n, const int* __restrict__ d_count, int npad, int weighting, int scoring,
                                                                    const uint32_t* __restrict__ f_word, const uint32_t* __restrict__ f_node,
                                                                    const float* __restrict__ f_weight, unsigned long long* __restrict__ gkeys,
                                                                    int* __restrict__ out_counts, unsigned long long* __restrict__ words,
                                                                    float* __restrict__ values, unsigned long long* __restrict__ fv_node,
                                                                    uint32_t* __restrict__ fv_feat) {
  extern __shared__ __align__(16) unsigned long long s_keys[];
  __shared__ int s_warp[32];
  __shared__ double s_part[33];
  __shared__ int s_same;
  unsigned long long* kw = gkeys ? gkeys : s_keys;  // word keys
  unsigned long long* kn = kw + npad;               // node keys (npad = the allocated power of two, sized for the capacity)
  if (d_count) {  // descriptors of an extraction in flight: the launch was sized for the capacity, sort only what the count needs
    n = max(0, min(n, *d_count));
    int p2 = 2;
    while (p2 < n) p2 <<= 1;
    npad = min(npad, p2);
  }
  if (threadIdx.x == 0) s_same = 1;
  __syncthreads();
  int differ = 0;
  for (int i = threadIdx.x; i < npad; i += kRedThreads) {
    unsigned long long a = ~0ull, b = ~0ull;
    if (i < n && f_weight[i] > 0.f) {  // stopped words (weight 0) take no part (Vocabulary.h:1585)
      a = ((unsigned long long)f_word[i] << 32) | (unsigned)i;
      b = ((unsigned long long)f_node[i] << 32) | (unsigned)i;
      differ |= f_word[i] != f_node[i];
    }
    kw[i] = a; kn[i] = b;
  }
  if (differ) s_same = 0;
  bitonic_sort(kw, npad);
  const bool same = s_same != 0;
  if (!same) bitonic_sort(kn, npad);
  // ---- BowVector: run heads of the sorted word keys --------------------------------------------------------------------------
  const int per = (npad + kRedThreads - 1) / kRedThreads, i0 = threadIdx.x * per, i1 = min(i0 + per, npad);
  int heads = 0, live = 0;
  for (int i = i0; i < i1; ++i) {
    const unsigned long long key = kw[i];
    if (key == ~0ull) break;
    ++live;
    if (i == 0 || (kw[i - 1] >> 32) != (key >> 32)) ++heads;
  }
  int nw = 0, m = 0;
  int pos = block_exscan(heads, s_warp, &nw);
  (void)block_exscan(live, s_warp, &m);
  const bool tf = weighting == W_TF || weighting == W_TF_IDF;
  double local = 0.0;  // this thread's share of the norm, its words in ascending order
  for (int i = i0; i < i1; ++i) {
    const unsigned long long key = kw[i];
    if (key == ~0ull) break;
    if (i == 0 || (kw[i - 1] >> 32) != (key >> 32)) {
      const float w = f_weight[(unsigned)key];
      float v = w;
      if (tf)
        for (int t = i + 1; t < npad && (kw[t] >> 32) == (key >> 32); ++t) v = __fadd_rn(v, w);  // += per occurrence (:357-369)
      words[pos] = key >> 32;
      values[pos] = v;
      local += scoring == S_L2 ? (double)__fmul_rn(v, v) : (double)fabsf(v);
      ++pos;
    }
  }
  const bool must = scoring != S_DOT;
  if (must || (tf && nw > 0)) {
    double norm = block_sum_d(local, s_part);  // (values of other threads are visible after its barriers)
    if (must && scoring == S_L2) norm = sqrt(norm);
    if (!must) norm = (double)nw;                // TF / TF_IDF without normalisation: divided by the number of words (:1592-1598)
    if (norm > 0.0)
      for (int a = threadIdx.x; a < nw; a += kRedThreads) values[a] = (float)((double)values[a] / norm);
  }
  // ---- FeatureVector: the sorted node keys, flattened --------------------------------------------------------------------------
  const unsigned long long* src = same ? kw : kn;
  for (int i = threadIdx.x; i < m; i += kRedThreads) {
    fv_node[i] = src[i] >> 32;
    fv_feat[i] = (uint32_t)src[i];
  }
  if (threadIdx.x == 0) { out_counts[0] = nw; out_counts[1] = m; }
}

int next_pow2(int n) { int p = 2; while (p < n) p <<= 1; return p; }

}  // namespace

extern "C" {

int gb_voc_create(gb_ctx* ctx, int k, int L, int weighting, int scoring, uint32_t n_nodes, const uint32_t* child_num, const float* weight,
                  const uint8_t* desc32, gb_vocabulary** out) {
  if (!ctx || !out) return GB_ERR_INVALID;
  *out = nullptr;
  if (k < 1 || k > 32 || L < 0 || weighting < 0 || weighting > 3 || scoring < 0 || scoring > 5 || n_nodes < 1 || !child_num || !weight || !desc32) {
    gb_set_error(ctx, "gb_voc_create: needs 1 <= k <= 32, a weighting in 0..3 (Vocabulary.h:88-94), a scoring in 0..5 (:97-105) and the node arrays");
    return GB_ERR_INVALID;
  }
  for (uint32_t p = 0; p < n_nodes; ++p) {
    if (child_num[p] > (uint32_t)k || (child_num[p] && (uint64_t)p * k + child_num[p] >= n_nodes)) {
      gb_set_error(ctx, "gb_voc_create: node %u has %u children (k = %d, %u nodes): not the implicit k-ary layout of Vocabulary.h:1714-1716", p, child_num[p], k, n_nodes);
      return GB_ERR_INVALID;
    }
  }
  CtxLock lk(ctx);
  gb_vocabulary* v = new gb_vocabulary();
  v->k = k; v->L = L; v->weighting = weighting; v->scoring = scoring; v->n_nodes = n_nodes;
  cudaError_t e = cudaMalloc((void**)&v->d_child, (size_t)n_nodes * 4);
  if (e == cudaSuccess) e = cudaMalloc((void**)&v->d_weight, (size_t)n_nodes * 4);
  if (e == cudaSuccess) e = cudaMalloc((void**)&v->d_desc, (size_t)n_nodes * 32);
  if (e == cudaSuccess) e = cudaMemcpy(v->d_child, child_num, (size_t)n_nodes * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(v->d_weight, weight, (size_t)n_nodes * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(v->d_desc, desc32, (size_t)n_nodes * 32, cudaMemcpyHostToDevice);
  const bool smem_ok = e == cudaSuccess && gb_func_setup(ctx, (const void*)bow_reduce_kernel, 2 * kSmemKeys * (int)sizeof(unsigned long long));
  if (!smem_ok) {
    gb_set_error(ctx, "gb_voc_create -> %s", e != cudaSuccess ? cudaGetErrorString(e) : "cannot set the shared-memory limit of the reduce kernel");
    cudaFree(v->d_child); cudaFree(v->d_weight); cudaFree(v->d_desc);
    delete v;
    return GB_ERR_CUDA;
  }
  *out = v;
  return GB_OK;
}

int gb_voc_destroy(gb_ctx* ctx, gb_vocabulary* v) {
  if (!v) return GB_OK;
  if (ctx) { CtxLock lk(ctx); cudaStreamSynchronize(ctx->stream); }
  cudaFree(v->d_child); cudaFree(v->d_weight); cudaFree(v->d_desc); cudaFree(v->d_feat); cudaFree(v->d_fword); cudaFree(v->d_keys); cudaFree(v->d_out);
  delete v;
  return GB_OK;
}

static int bow_run(gb_ctx* ctx, gb_vocabulary* v, const uint4* d_feats, int n, const int* d_count, int levelsup, uint64_t* words, float* values,
                   int* n_words, uint64_t* fv_node, uint32_t* fv_feat, int* n_fv) {
  if (n == 0) { *n_words = 0; *n_fv = 0; return GB_OK; }
  const int npad = next_pow2(n);
  const bool in_smem = npad <= kSmemKeys;
  GB_CHECK(gb_dev_realloc(ctx, (void**)&v->d_fword, &v->fword_cap, (size_t)n * 12));
  if (!in_smem) GB_CHECK(gb_dev_realloc(ctx, (void**)&v->d_keys, &v->keys_cap, (size_t)npad * 16));
  const size_t o_words = 16, o_node = o_words + (size_t)n * 8, o_val = o_node + (size_t)n * 8, o_feat = o_val + (size_t)n * 4, bytes = o_feat + (size_t)n * 4;
  GB_CHECK(gb_dev_realloc(ctx, (void**)&v->d_out, &v->out_cap, bytes));
  uint32_t* f_word = v->d_fword; uint32_t* f_node = f_word + n; float* f_weight = (float*)(f_node + n);
  const int G = v->k <= 16 ? 16 : 32;
  const int blocks = gb_div_up(n * G, kWalkThreads);
  if (G == 16) bow_walk_kernel<16><<<blocks, kWalkThreads, 0, ctx->stream>>>(v->k, v->L, v->d_child, v->d_weight, v->d_desc, d_feats, n, d_count, levelsup, f_word, f_node, f_weight);
  else bow_walk_kernel<32><<<blocks, kWalkThreads, 0, ctx->stream>>>(v->k, v->L, v->d_child, v->d_weight, v->d_desc, d_feats, n, d_count, levelsup, f_word, f_node, f_weight);
  GB_LAUNCH_CHECK(ctx);
  bow_reduce_kernel<<<1, kRedThreads, in_smem ? (size_t)npad * 16 : 0, ctx->stream>>>(
      n, d_count, npad, v->weighting, v->scoring, f_word, f_node, f_weight, in_smem ? nullptr : v->d_keys, (int*)v->d_out,
      (unsigned long long*)(v->d_out + o_words), (float*)(v->d_out + o_val), (unsigned long long*)(v->d_out + o_node), (uint32_t*)(v->d_out + o_feat));
  GB_LAUNCH_CHECK(ctx);
  GB_CHECK(gb_stage_reserve(ctx, ctx->h_stage_off + bytes + 1024));
  uint8_t* h = (uint8_t*)gb_stage_alloc(ctx, bytes);
  GB_CUDA(ctx, cudaMemcpyAsync(h, v->d_out, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const int nw = ((int*)h)[0], m = ((int*)h)[1];
  *n_words = nw; *n_fv = m;
  memcpy(words, h + o_words, (size_t)nw * 8);
  memcpy(values, h + o_val, (size_t)nw * 4);
  memcpy(fv_node, h + o_node, (size_t)m * 8);
  memcpy(fv_feat, h + o_feat, (size_t)m * 4);
  return GB_OK;
}

int gb_bow_transform(gb_ctx* ctx, gb_vocabulary* v, const uint8_t* desc, int n, int levelsup, uint64_t* words, float* values, int* n_words,
                     uint64_t* fv_node, uint32_t* fv_feat, int* n_fv) {
  if (!ctx || !v || n < 0 || (n > 0 && !desc) || !words || !values || !n_words || !fv_node || !fv_feat || !n_fv) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  if (n == 0) { *n_words = 0; *n_fv = 0; return GB_OK; }
  GB_CHECK(gb_dev_realloc(ctx, (void**)&v->d_feat, &v->feat_cap, (size_t)n * 32));
  GB_CHECK(gb_stage_reserve(ctx, ctx->h_stage_off + (size_t)n * 32 + 1024));
  uint8_t* h = (uint8_t*)gb_stage_alloc(ctx, (size_t)n * 32);
  memcpy(h, desc, (size_t)n * 32);
  GB_CUDA(ctx, cudaMemcpyAsync(v->d_feat, h, (size_t)n * 32, cudaMemcpyHostToDevice, ctx->stream));
  return bow_run(ctx, v, (const uint4*)v->d_feat, n, nullptr, levelsup, words, values, n_words, fv_node, fv_feat, n_fv);
}

int gb_bow_transform_features(gb_ctx* ctx, gb_vocabulary* v, gb_features* f, int levelsup, uint64_t* words, float* values, int* n_words,
                              uint64_t* fv_node, uint32_t* fv_feat, int* n_fv) {
  if (!ctx || !v || !f || !words || !values || !n_words || !fv_node || !fv_feat || !n_fv) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  // the descriptors of an extraction still in flight: the launch is sized for the capacity and clipped by the device-side count
  const int n = f->h_count >= 0 ? f->h_count : f->capacity;
  return bow_run(ctx, v, (const uint4*)f->d_desc, n, f->h_count >= 0 ? nullptr : f->d_count, levelsup, words, values, n_words, fv_node, fv_feat, n_fv);
}

}  // extern "C"
