// gslam_b200/csrc/ctx.cu — gb_ctx lifetime, error strings, pinned staging and device scratch, timers, gb_features containers.
#include <map>

#include "common.cuh"

static thread_local std::string g_tls_err = "";

void gb_set_error(gb_ctx* ctx, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (ctx) ctx->err = buf;
  g_tls_err = buf;
}

static size_t take_align(size_t off) { return (off + 255) & ~(size_t)255; }

// Replaces b's buffer by one of at least `bytes` (device memory or pinned host memory), with room to spare, and empties it.
static int bump_grow(gb_ctx* ctx, GbBump& b, bool device, size_t bytes) {
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // (nothing may be in flight from the old buffer)
  if (device) cudaFree(b.base);
  else cudaFreeHost(b.base);
  b = GbBump{};
  const size_t want = device ? bytes + (bytes >> 3) + 256 : bytes + (bytes >> 2) + 4096;
  GB_CUDA(ctx, device ? cudaMalloc((void**)&b.base, want) : cudaHostAlloc((void**)&b.base, want, cudaHostAllocDefault));
  b.bytes = want;
  return GB_OK;
}

static int bump_take(gb_ctx* ctx, GbBump& b, bool device, std::initializer_list<GbBuf> bufs) {
  size_t end = b.off;
  for (const GbBuf& x : bufs)
    if (x.bytes) end = take_align(end) + x.bytes;
  if (end > b.bytes) GB_CHECK(bump_grow(ctx, b, device, end));  // (a grown buffer starts empty: the layout below then fits)
  for (const GbBuf& x : bufs) {
    *x.p = nullptr;
    if (!x.bytes) continue;
    b.off = take_align(b.off);
    *x.p = b.base + b.off;
    b.off += x.bytes;
  }
  return GB_OK;
}

int gb_stage_take(gb_ctx* ctx, std::initializer_list<GbBuf> bufs) { return bump_take(ctx, ctx->stage, false, bufs); }

int gb_scratch_take(gb_ctx* ctx, std::initializer_list<GbBuf> bufs) { return bump_take(ctx, ctx->scratch, true, bufs); }

int gb_upload_2d(gb_ctx* ctx, void* d_dst, size_t dpitch, const void* src, int src_is_device, size_t spitch, size_t row_bytes, int rows) {
  if (!src_is_device) {
    cudaPointerAttributes at;
    const bool pinned = cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeHost;
    cudaGetLastError();
    if (!pinned) {
      uint8_t* hs;
      GB_CHECK(gb_stage_take(ctx, {{&hs, row_bytes * rows}}));
      for (int y = 0; y < rows; ++y) memcpy(hs + (size_t)y * row_bytes, (const uint8_t*)src + (size_t)y * spitch, row_bytes);
      src = hs;
      spitch = row_bytes;
    }
  }
  GB_CUDA(ctx, cudaMemcpy2DAsync(d_dst, dpitch, src, spitch, row_bytes, rows, src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice,
                                 ctx->stream));
  return GB_OK;
}

int gb_stage_frame(gb_ctx* ctx, const uint8_t* img, int img_is_device, size_t row_bytes, int height, int pitch, const uint8_t** d_frame) {
  if (img_is_device && (size_t)pitch == row_bytes) {
    *d_frame = img;
    return GB_OK;
  }
  uint8_t* d;
  GB_CHECK(gb_scratch_take(ctx, {{&d, row_bytes * height}}));
  GB_CHECK(gb_upload_2d(ctx, d, row_bytes, img, img_is_device, pitch, row_bytes, height));
  *d_frame = d;
  return GB_OK;
}

namespace {
struct FuncSetup {
  bool smem_ok = false;
  int nonportable = 0;  // 0 not asked for yet, 1 permitted, -1 refused
};
std::mutex g_func_mu;
std::map<std::pair<int, const void*>, FuncSetup> g_func_done;  // (device, kernel) -> what was set
}  // namespace

bool gb_func_setup(gb_ctx* ctx, const void* fn, int smem, bool* nonportable_cluster) {
  std::lock_guard<std::mutex> lk(g_func_mu);
  const auto key = std::make_pair(ctx->device, fn);
  auto it = g_func_done.find(key);
  if (it == g_func_done.end()) {
    FuncSetup s;
    s.smem_ok = true;
    if (smem == GB_SMEM_OPTIN_MAX) {
      cudaFuncAttributes fa{};
      s.smem_ok = cudaFuncGetAttributes(&fa, fn) == cudaSuccess;
      if (s.smem_ok) smem = ctx->max_smem_optin - (int)fa.sharedSizeBytes;
    }
    s.smem_ok = s.smem_ok && cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess;
    cudaGetLastError();  // (a refused attribute must not surface as the error of a later launch)
    it = g_func_done.emplace(key, s).first;
  }
  if (nonportable_cluster && it->second.nonportable == 0) {
    it->second.nonportable = cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess ? 1 : -1;
    cudaGetLastError();
  }
  if (nonportable_cluster) *nonportable_cluster = it->second.nonportable > 0;
  return it->second.smem_ok;
}

extern void gb_orb_state_free(gb_ctx* ctx);
extern void ba_cache_free(gb_ctx* ctx);

extern "C" {

int gb_version(void) { return GB_VERSION; }

int gb_device_count(int* n) {
  int c = 0;
  cudaError_t e = cudaGetDeviceCount(&c);
  if (e != cudaSuccess) {
    gb_set_error(nullptr, "cudaGetDeviceCount -> %s", cudaGetErrorString(e));
    if (n) *n = 0;
    return GB_ERR_NODEVICE;
  }
  if (n) *n = c;
  return GB_OK;
}

static int ctx_create_impl(int device, int high_priority, cudaStream_t borrowed, gb_ctx** out);

int gb_ctx_create(int device, gb_ctx** out) { return ctx_create_impl(device, 0, nullptr, out); }

// A ctx whose stream has the device's greatest priority: the block scheduler hands free SM slots to its CTAs first.  For the
// mapping ctx of a tracking/mapping pair: the few-CTA local-BA kernels then do not queue behind the thousands of CTAs of the
// tracking ctx's FAST / describe grids (without it the two streams barely overlap).
int gb_ctx_create_priority(int device, int high_priority, gb_ctx** out) { return ctx_create_impl(device, high_priority, nullptr, out); }

}  // extern "C"

int gb_ctx_create_on_stream(int device, cudaStream_t stream, gb_ctx** out) {
  if (!stream) return GB_ERR_INVALID;
  return ctx_create_impl(device, 0, stream, out);
}

extern "C" {

static int ctx_create_impl(int device, int high_priority, cudaStream_t borrowed, gb_ctx** out) {
  if (!out) return GB_ERR_INVALID;
  *out = nullptr;
  int n = 0;
  if (gb_device_count(&n) != GB_OK || n <= 0) {
    if (n <= 0 && g_tls_err.empty()) gb_set_error(nullptr, "no CUDA device");
    return GB_ERR_NODEVICE;  // no CPU fallback, by design
  }
  if (device < 0 || device >= n) {
    gb_set_error(nullptr, "device %d out of range (have %d)", device, n);
    return GB_ERR_INVALID;
  }
  gb_ctx* ctx = new gb_ctx();
  ctx->device = device;
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess && borrowed) {
    ctx->stream = borrowed;
    ctx->owns_stream = false;
  } else if (e == cudaSuccess) {
    int lo = 0, hi = 0;  // (numerically lower = higher priority)
    if (high_priority && cudaDeviceGetStreamPriorityRange(&lo, &hi) == cudaSuccess) e = cudaStreamCreateWithPriority(&ctx->stream, cudaStreamNonBlocking, hi);
    else e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
  }
  if (e == cudaSuccess) e = cudaEventCreate(&ctx->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&ctx->ev1);
  if (e == cudaSuccess) e = cudaEventCreate(&ctx->evs);
  if (e == cudaSuccess) e = cudaEventCreate(&ctx->eve);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx->max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
  auto drop = [&]() {  // whatever was created before the failure
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->evs) cudaEventDestroy(ctx->evs);
    if (ctx->eve) cudaEventDestroy(ctx->eve);
    if (ctx->stream && ctx->owns_stream) cudaStreamDestroy(ctx->stream);
    if (ctx->stage.base) cudaFreeHost(ctx->stage.base);
    delete ctx;
  };
  if (e != cudaSuccess) {
    gb_set_error(nullptr, "gb_ctx_create(device %d) -> %s", device, cudaGetErrorString(e));
    drop();
    return GB_ERR_CUDA;
  }
  if (bump_grow(ctx, ctx->stage, false, 8u << 20) != GB_OK) {
    drop();
    return GB_ERR_CUDA;
  }
  *out = ctx;
  return GB_OK;
}

int gb_ctx_destroy(gb_ctx* ctx) {
  if (!ctx) return GB_OK;
  {
    CtxLock lk(ctx);
    cudaStreamSynchronize(ctx->stream);
    ba_cache_free(ctx);
    gb_orb_state_free(ctx);
    if (ctx->stage.base) cudaFreeHost(ctx->stage.base);
    cudaFree(ctx->scratch.base);
    cudaEventDestroy(ctx->ev0);
    cudaEventDestroy(ctx->ev1);
    cudaEventDestroy(ctx->evs);
    cudaEventDestroy(ctx->eve);
    if (ctx->ev_x) cudaEventDestroy(ctx->ev_x);
    if (ctx->owns_stream) cudaStreamDestroy(ctx->stream);
  }
  delete ctx;
  return GB_OK;
}

const char* gb_last_error(const gb_ctx* ctx) { return ctx ? ctx->err.c_str() : g_tls_err.c_str(); }

void* gb_ctx_stream(gb_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

int gb_ctx_sync(gb_ctx* ctx) {
  if (!ctx) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return GB_OK;
}

// Order `waiter`'s stream after everything enqueued so far on `producer`'s stream (event record + stream wait; no host sync).
// This is how a tracking ctx (extract / match) and a mapping ctx (local BA) pipeline on one GPU: BA(k) waits for match(k) while
// extract(k+1) already runs.
int gb_ctx_wait_for(gb_ctx* waiter, gb_ctx* producer) {
  if (!waiter || !producer) return GB_ERR_INVALID;
  if (waiter == producer) return GB_OK;
  std::lock(waiter->mu, producer->mu);
  std::lock_guard<std::recursive_mutex> l0(waiter->mu, std::adopt_lock), l1(producer->mu, std::adopt_lock);
  if (waiter->device != producer->device) { gb_set_error(waiter, "gb_ctx_wait_for: contexts on different devices"); return GB_ERR_INVALID; }
  cudaSetDevice(producer->device);
  if (!producer->ev_x) GB_CUDA(producer, cudaEventCreateWithFlags(&producer->ev_x, cudaEventDisableTiming));
  GB_CUDA(producer, cudaEventRecord(producer->ev_x, producer->stream));
  GB_CUDA(waiter, cudaStreamWaitEvent(waiter->stream, producer->ev_x, 0));
  return GB_OK;
}

int gb_timer_begin(gb_ctx* ctx) {
  if (!ctx) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  GB_CUDA(ctx, cudaEventRecord(ctx->ev0, ctx->stream));
  return GB_OK;
}

int gb_timer_end(gb_ctx* ctx, float* ms) {
  if (!ctx || !ms) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  GB_CUDA(ctx, cudaEventRecord(ctx->ev1, ctx->stream));
  GB_CUDA(ctx, cudaEventSynchronize(ctx->ev1));
  GB_CUDA(ctx, cudaEventElapsedTime(ms, ctx->ev0, ctx->ev1));
  return GB_OK;
}

int64_t gb_launch_count(const gb_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ---- gb_features ---------------------------------------------------------------------------------------------------
int gb_features_create(gb_ctx* ctx, int capacity, gb_features** out) {
  if (!ctx || !out || capacity <= 0) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  gb_features* f = new gb_features();
  f->capacity = capacity;
  int rc = gb_slab_alloc(ctx, &f->d_slab, [&](Slab& sl) { gb_features_layout(sl, f); });
  if (rc == GB_OK && cudaMemsetAsync(f->d_count, 0, gb_features_words(capacity) * sizeof(int), ctx->stream) != cudaSuccess) {
    gb_set_error(ctx, "gb_features_create(%d) -> %s", capacity, cudaGetErrorString(cudaGetLastError()));
    rc = GB_ERR_CUDA;
  }
  if (rc != GB_OK) {
    gb_features_destroy(ctx, f);
    return rc;
  }
  f->h_count = 0;
  *out = f;
  return GB_OK;
}

int gb_features_destroy(gb_ctx* ctx, gb_features* f) {
  if (!f) return GB_OK;
  if (ctx) {
    CtxLock lk(ctx);
    cudaStreamSynchronize(ctx->stream);
  }
  cudaFree(f->d_slab);
  delete f;
  return GB_OK;
}

}  // extern "C"

void gb_features_layout(Slab& sl, gb_features* f) {
  const size_t cap = (size_t)f->capacity;
  sl.take(&f->d_kps, cap);
  sl.take(&f->d_desc, cap * 32);
  sl.take(&f->d_count, gb_features_words(f->capacity));  // count, status, train status, (pad), tickets: after d_desc (gb_match_hamming)
  sl.take(&f->d_best, cap);
  sl.take(&f->d_dist, cap);
  sl.take(&f->d_dist2, cap);
  if (!sl.base) return;  // (measuring)
  f->d_status = f->d_count + 1;
  f->d_train_status = f->d_count + 2;
  f->d_tickets = (unsigned int*)(f->d_count + 4);
}

int gb_features_resolve(gb_ctx* ctx, gb_features* f, const int* hc, int* n) {
  if (hc[1] < 0) {
    *n = 0;
    gb_set_error(ctx, "extract: internal overflow (%s)", hc[1] == -2 ? "more than 4096 keypoints kept on one level" : "candidate buffer");
    return GB_ERR_CAPACITY;
  }
  if (hc[1] != 0) {
    *n = hc[1];
    gb_set_error(ctx, "extract kept %d keypoints but the feature set holds %d", hc[1], f->capacity);
    return GB_ERR_CAPACITY;
  }
  f->h_count = *n = hc[0];
  return GB_OK;
}

extern "C" {

int gb_features_count(gb_ctx* ctx, gb_features* f, int* n) {
  if (!ctx || !f || !n) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  if (f->h_count < 0) {
    int hc[2] = {0, 0};
    GB_CUDA(ctx, cudaMemcpyAsync(hc, f->d_count, sizeof hc, cudaMemcpyDeviceToHost, ctx->stream));
    GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return gb_features_resolve(ctx, f, hc, n);
  }
  *n = f->h_count;
  return GB_OK;
}

// test hook: put a feature set back into the state of an extraction in flight -- device-side {count, status} as given, host count
// unknown, `expect` as the launch hint -- so that the device-count paths run on chosen rows (uploaded before)
GB_API int gb_dbg_features_set_pending(gb_ctx* ctx, gb_features* f, int count, int status, int expect) {
  if (!ctx || !f || count < 0 || count > f->capacity) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  int* hc;
  GB_CHECK(gb_stage_take(ctx, {{&hc, 2 * sizeof(int)}}));
  hc[0] = count;
  hc[1] = status;
  GB_CUDA(ctx, cudaMemcpyAsync(f->d_count, hc, 2 * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  f->h_count = -1;
  f->expect = expect;
  return GB_OK;
}

int gb_features_upload(gb_ctx* ctx, gb_features* f, const gb_keypoint* kps, const uint8_t* desc, int n) {
  if (!ctx || !f || n < 0 || (n > 0 && !desc)) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  if (n > f->capacity) {
    gb_set_error(ctx, "gb_features_upload: %d rows > capacity %d", n, f->capacity);
    return GB_ERR_CAPACITY;
  }
  uint8_t* hd;
  gb_keypoint* hk;
  int* hc;
  GB_CHECK(gb_stage_take(ctx, {{&hd, (size_t)n * 32}, {&hk, kps ? (size_t)n * sizeof(gb_keypoint) : 0}, {&hc, 2 * sizeof(int)}}));
  if (n > 0) {
    memcpy(hd, desc, (size_t)n * 32);
    GB_CUDA(ctx, cudaMemcpyAsync(f->d_desc, hd, (size_t)n * 32, cudaMemcpyHostToDevice, ctx->stream));
    if (kps) {
      memcpy(hk, kps, (size_t)n * sizeof(gb_keypoint));
      GB_CUDA(ctx, cudaMemcpyAsync(f->d_kps, hk, (size_t)n * sizeof(gb_keypoint), cudaMemcpyHostToDevice, ctx->stream));
    }
  }
  hc[0] = n;
  hc[1] = 0;
  GB_CUDA(ctx, cudaMemcpyAsync(f->d_count, hc, 2 * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
  f->h_count = n;
  // the staging is reused by the next API call: make sure the copies left it
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return GB_OK;
}

int gb_features_download(gb_ctx* ctx, gb_features* f, gb_keypoint* kps, uint8_t* desc, int* n) {
  if (!ctx || !f || !n) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  const int cap = *n;
  int cnt = 0;
  if (f->h_count >= 0) {
    cnt = f->h_count;
  } else if (cap <= 0) {
    GB_CHECK(gb_features_count(ctx, f, &cnt));
  }
  // When the count is not on the host yet (the extraction is still in flight) the count word travels WITH the rows: up to
  // min(cap, capacity) rows are copied speculatively, so that a host-buffer extraction costs ONE synchronisation, not two.
  const bool speculative = f->h_count < 0 && cap > 0;
  const int rows = speculative ? std::min(cap, f->capacity) : cnt;
  if (!speculative) {
    *n = cnt;
    if (cnt > cap) {
      gb_set_error(ctx, "gb_features_download: %d keypoints > caller capacity %d", cnt, cap);
      return GB_ERR_CAPACITY;
    }
    if (cnt == 0) return GB_OK;
  }
  int* hc;
  gb_keypoint* hk;
  uint8_t* hd;
  GB_CHECK(gb_stage_take(ctx, {{&hc, 16}, {&hk, kps ? (size_t)rows * sizeof(gb_keypoint) : 0}, {&hd, desc ? (size_t)rows * 32 : 0}}));
  if (speculative) GB_CUDA(ctx, cudaMemcpyAsync(hc, f->d_count, 2 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  if (hk && rows > 0) GB_CUDA(ctx, cudaMemcpyAsync(hk, f->d_kps, (size_t)rows * sizeof(gb_keypoint), cudaMemcpyDeviceToHost, ctx->stream));
  if (hd && rows > 0) GB_CUDA(ctx, cudaMemcpyAsync(hd, f->d_desc, (size_t)rows * 32, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (speculative) {
    GB_CHECK(gb_features_resolve(ctx, f, hc, n));
    cnt = *n;
    if (cnt > cap) {
      gb_set_error(ctx, "gb_features_download: %d keypoints > caller capacity %d", cnt, cap);
      return GB_ERR_CAPACITY;
    }
  }
  if (hk && cnt > 0) memcpy(kps, hk, (size_t)cnt * sizeof(gb_keypoint));
  if (hd && cnt > 0) memcpy(desc, hd, (size_t)cnt * 32);
  return GB_OK;
}

}  // extern "C"
