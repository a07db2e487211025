// gslam_b200/csrc/remap.cu — frame undistortion: the bilinear LUT remap of GSLAM::Undistorter::undistort
// (GSLAM/core/Undistorter.h:271-348; tables built by UndistorterImpl::prepareReMap :120-203).  SURVEY.md section 8f-4.
//
// The table (four source pixel indices + four float weights per output pixel, remapX < 0 = outside the input image) is built by the
// REFERENCE's own prepareReMap in the plugin (camera models stay the reference's); this file applies it: one thread per output
// pixel, p_out = p[i0]*c0 + p[i1]*c1 + p[i2]*c2 + p[i3]*c3 in float with the reference's left-to-right order, no FMA contraction,
// truncation to uchar -- bit-identical to the reference wherever the reference is defined.  Two places where the reference reads or
// leaves undefined memory are given a defined value here (documented in DESIGN.md, excluded from the parity comparison):
//   * taps whose index lies beyond the input image (last row / last column: the reference reads past its buffer) contribute 0;
//   * multi-channel images: output pixels outside the input image are 0 (the reference leaves them uninitialised) and the pixel
//     test is remapX > 0 as in the reference's multi-channel branch (:318), remapX >= 0 in the 1-channel branch (:297).
//
// Two kernels share that arithmetic (remap_inside / remap_tap): remap_kernel writes the undistorted image itself, 1 or 3 channels, at
// any row pitch (gb_remap_apply, gb_remap_apply_to); remap_level0_kernel is the first stage of gb_orb_extract_undistorted*: it
// writes the undistorted GRAY image straight into level 0 of the ORB pyramid, the colour conversion done in registers.
#include "common.cuh"

struct gb_remap {  // immutable after creation
  int device = 0;             // the table lives there: usable from every ctx on that device
  int w_in = 0, h_in = 0, w_out = 0, h_out = 0;
  void* d_slab = nullptr;     // one allocation holding the three arrays below
  int32_t* d_idx = nullptr;   // [w_out*h_out][4]
  float* d_coef = nullptr;    // [w_out*h_out][4]
  float* d_x = nullptr;       // [w_out*h_out] remapX
};

namespace {

// Is the output pixel with this remapX inside the input image?  (1-channel: remapX >= 0; multi-channel: remapX > 0)
__device__ __forceinline__ bool remap_inside(float xx, int channels) { return channels == 1 ? !(xx < 0.f) : (xx > 0.f); }

// Channel j of one inside output pixel: the four taps in the reference's order, taps beyond the input image count as 0.
__device__ __forceinline__ uint8_t remap_tap(const uint8_t* __restrict__ src, const int4 t, const float4 c, int n_in, int channels, int j) {
  const float p0 = t.x < n_in ? (float)__ldg(src + (size_t)t.x * channels + j) : 0.f, p1 = t.y < n_in ? (float)__ldg(src + (size_t)t.y * channels + j) : 0.f;
  const float p2 = t.z < n_in ? (float)__ldg(src + (size_t)t.z * channels + j) : 0.f, p3 = t.w < n_in ? (float)__ldg(src + (size_t)t.w * channels + j) : 0.f;
  const float v = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(p0, c.x), __fmul_rn(p1, c.y)), __fmul_rn(p2, c.z)), __fmul_rn(p3, c.w));
  return (uint8_t)__float2int_rz(v);
}

// One thread per output pixel; row y of the output starts at dst + y * dpitch.
__global__ void __launch_bounds__(256) remap_kernel(const int4* __restrict__ idx, const float4* __restrict__ coef, const float* __restrict__ rx, int n_out,
                                                    int n_in, int channels, const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int w_out, int dpitch) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  const int y = i / w_out;
  uint8_t* o = dst + (size_t)y * dpitch + (size_t)(i - y * w_out) * channels;
  if (!remap_inside(rx[i], channels)) {
    for (int j = 0; j < channels; ++j) o[j] = 0;
    return;
  }
  const int4 t = idx[i];
  const float4 c = coef[i];
  for (int j = 0; j < channels; ++j) o[j] = remap_tap(src, t, c, n_in, channels, j);
}

// The remap as the producer of ORB pyramid level 0: one thread per 4 consecutive output pixels of a row, their table entries
// (36 B per pixel: the bound of this kernel, a gather) fetched with 128-bit loads BEFORE the wait on the predecessor -- the table
// never changes, so under programmatic dependent launch those loads overlap the tail of whatever ran before -- then the source taps
// through the read-only path and one aligned 32-bit store (level rows start 128-byte aligned; the bytes of the last word past
// w_out are row padding and are written 0, as the pyramid kernel writes them).  CH == 3: the three channels are remapped to bytes as
// remap_kernel does and the gray value of cv2.cvtColor (orb_gray_kernel's fixed point) is formed from them in registers.
template <int CH>
__global__ void __launch_bounds__(256) remap_level0_kernel(const int4* __restrict__ idx, const float4* __restrict__ coef, const float* __restrict__ rx, int w_out,
                                                           int h_out, int n_in, int rgb_order, const uint8_t* __restrict__ src, uint8_t* __restrict__ dst,
                                                           int dpitch) {
  gb_pdl_launch_dependents();
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int y = blockIdx.y * blockDim.y + threadIdx.y;
  const bool active = x4 < w_out && y < h_out;
  int4 t[4];
  float4 c[4];
  bool in[4];
  if (active) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const bool valid = x4 + k < w_out;
      const size_t i = (size_t)y * w_out + (valid ? x4 + k : w_out - 1);
      in[k] = valid && remap_inside(__ldg(rx + i), CH);
      t[k] = __ldg(idx + i);
      c[k] = __ldg(coef + i);
    }
  }
  gb_pdl_wait();  // the source frame may have been written, and level 0 read, by the predecessors on the stream
  if (!active) return;
  uint32_t out = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    uint32_t v;
    if (CH == 1) {
      v = remap_tap(src, t[k], c[k], n_in, 1, 0);
    } else {
      const int c0 = remap_tap(src, t[k], c[k], n_in, 3, 0), c1 = remap_tap(src, t[k], c[k], n_in, 3, 1), c2 = remap_tap(src, t[k], c[k], n_in, 3, 2);
      const int b = rgb_order ? c2 : c0, r = rgb_order ? c0 : c2;
      v = (uint32_t)((b * 3735 + c1 * 19235 + r * 9798 + (1 << 14)) >> 15);
    }
    out |= (in[k] ? v : 0u) << (8 * k);
  }
  *reinterpret_cast<uint32_t*>(dst + (size_t)y * dpitch + x4) = out;
}

}  // namespace

void gb_remap_geometry(const gb_remap* m, int* device, int* w_in, int* h_in, int* w_out, int* h_out) {
  *device = m->device; *w_in = m->w_in; *h_in = m->h_in; *w_out = m->w_out; *h_out = m->h_out;
}

int gb_remap_enqueue_level0(gb_ctx* ctx, const gb_remap* m, const uint8_t* d_src, int channels, int rgb_order, uint8_t* d_dst, int dst_pitch) {
  const dim3 blk(64, 4), grd(gb_div_up(gb_div_up(m->w_out, 4), 64), gb_div_up(m->h_out, 4));
  const int n_in = m->w_in * m->h_in;
  if (channels == 1)
    GB_CUDA(ctx, gb_launch_pdl(remap_level0_kernel<1>, grd, blk, 0, ctx->stream, (const int4*)m->d_idx, (const float4*)m->d_coef, m->d_x, m->w_out, m->h_out, n_in,
                               rgb_order, d_src, d_dst, dst_pitch));
  else
    GB_CUDA(ctx, gb_launch_pdl(remap_level0_kernel<3>, grd, blk, 0, ctx->stream, (const int4*)m->d_idx, (const float4*)m->d_coef, m->d_x, m->w_out, m->h_out, n_in,
                               rgb_order, d_src, d_dst, dst_pitch));
  GB_LAUNCH_CHECK(ctx);
  return GB_OK;
}

extern "C" {

int gb_remap_create(gb_ctx* ctx, int w_in, int h_in, int w_out, int h_out, const int32_t* idx4, const float* coef4, const float* remap_x, gb_remap** out) {
  if (!ctx || !out || w_in < 1 || h_in < 1 || w_out < 1 || h_out < 1 || !idx4 || !coef4 || !remap_x) return GB_ERR_INVALID;
  *out = nullptr;
  CtxLock lk(ctx);
  const size_t n = (size_t)w_out * h_out;
  for (size_t k = 0; k < 4 * n; ++k)
    if (idx4[k] < 0) { gb_set_error(ctx, "gb_remap_create: negative source index at entry %zu", k); return GB_ERR_INVALID; }
  gb_remap* m = new gb_remap();
  m->device = ctx->device;
  m->w_in = w_in; m->h_in = h_in; m->w_out = w_out; m->h_out = h_out;
  int rc = gb_slab_alloc(ctx, &m->d_slab, [&](Slab& sl) { sl.take(&m->d_idx, 4 * n); sl.take(&m->d_coef, 4 * n); sl.take(&m->d_x, n); });
  cudaError_t e = cudaSuccess;
  if (rc == GB_OK) e = cudaMemcpy(m->d_idx, idx4, n * 16, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(m->d_coef, coef4, n * 16, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(m->d_x, remap_x, n * 4, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    gb_set_error(ctx, "gb_remap_create -> %s", cudaGetErrorString(e));
    rc = GB_ERR_CUDA;
  }
  if (rc != GB_OK) {
    cudaFree(m->d_slab);
    delete m;
    return rc;
  }
  *out = m;
  return GB_OK;
}

int gb_remap_destroy(gb_ctx* ctx, gb_remap* m) {
  if (!m) return GB_OK;
  if (ctx) { CtxLock lk(ctx); cudaStreamSynchronize(ctx->stream); }
  cudaFree(m->d_slab);
  delete m;
  return GB_OK;
}

int gb_remap_apply(gb_ctx* ctx, gb_remap* m, const uint8_t* src, int channels, uint8_t* dst) {
  if (!ctx || !m || !src || !dst || (channels != 1 && channels != 3)) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  const size_t n_in = (size_t)m->w_in * m->h_in, n_out = (size_t)m->w_out * m->h_out, b_in = n_in * channels, b_out = n_out * channels;
  uint8_t *d_src, *d_dst, *hd;
  GB_CHECK(gb_scratch_take(ctx, {{&d_src, b_in}, {&d_dst, b_out}}));
  GB_CHECK(gb_upload_2d(ctx, d_src, b_in, src, 0, b_in, b_in, 1));
  remap_kernel<<<gb_div_up((int)n_out, 256), 256, 0, ctx->stream>>>((const int4*)m->d_idx, (const float4*)m->d_coef, m->d_x, (int)n_out, (int)n_in, channels,
                                                                   d_src, d_dst, m->w_out, m->w_out * channels);
  GB_LAUNCH_CHECK(ctx);
  GB_CHECK(gb_stage_take(ctx, {{&hd, b_out}}));  // (after the upload's own take: a growth here synchronises first)
  GB_CUDA(ctx, cudaMemcpyAsync(hd, d_dst, b_out, cudaMemcpyDeviceToHost, ctx->stream));
  GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  memcpy(dst, hd, b_out);
  return GB_OK;
}

int gb_remap_apply_to(gb_ctx* ctx, gb_remap* m, const uint8_t* src, int src_is_device, int src_pitch, int channels, uint8_t* d_dst, int dst_pitch) {
  if (!ctx || !m || !src || !d_dst) return GB_ERR_INVALID;
  CtxLock lk(ctx);
  if (channels != 1 && channels != 3) {
    gb_set_error(ctx, "gb_remap_apply_to: %d channels (1 or 3 are supported; the reference's 4-channel branch writes 3-channel pixels)", channels);
    return GB_ERR_INVALID;
  }
  if (m->device != ctx->device) {
    gb_set_error(ctx, "gb_remap_apply_to: the map was created on device %d, the ctx is on device %d", m->device, ctx->device);
    return GB_ERR_INVALID;
  }
  if (src_pitch < m->w_in * channels || dst_pitch < m->w_out * channels) {
    gb_set_error(ctx, "gb_remap_apply_to: pitches %d / %d are shorter than rows of %d / %d bytes", src_pitch, dst_pitch, m->w_in * channels, m->w_out * channels);
    return GB_ERR_INVALID;
  }
  const uint8_t* d_src = nullptr;
  GB_CHECK(gb_stage_frame(ctx, src, src_is_device, (size_t)m->w_in * channels, m->h_in, src_pitch, &d_src));
  const int n_out = m->w_out * m->h_out;
  remap_kernel<<<gb_div_up(n_out, 256), 256, 0, ctx->stream>>>((const int4*)m->d_idx, (const float4*)m->d_coef, m->d_x, n_out, m->w_in * m->h_in, channels, d_src,
                                                                d_dst, m->w_out, dst_pitch);
  GB_LAUNCH_CHECK(ctx);
  if (!src_is_device) GB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the caller's buffer / the pinned staging may be reused
  return GB_OK;
}

}  // extern "C"
