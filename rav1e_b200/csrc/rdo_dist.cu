// rdo_dist.cu — the RDO distortion kernels of rav1e for batches of blocks (sm_90a).
//
//   get_weighted_sse   src/dist.rs:234-283   (asm: rav1e_weighted_sse_{W}x{H}, asm/x86/dist/sse.rs:18-35)
//   cdef_dist_kernel   src/dist.rs:302-372   (asm: rav1e_cdef_dist_kernel_{W}x{H}, asm/x86/dist/cdef_dist.rs:18-52)
//   apply_ssim_boost   src/activity.rs:159-186 (+ ssim_boost_rsqrt :107-143)
// Callers: sse_wxh / cdef_dist_wxh / compute_distortion (rdo.rs:142-250, :254-330): one call per
// block per RDO candidate.  Here one launch covers every block of a frame (or of a candidate set).
//
// weighted SSE: one warp per block, a lane per 4x4 chunk (one DistortionScale each), u64 partial
// sums reduced by shuffles, the final (sse + den/2) / den in lane 0.
// cdef_dist: one thread per <= 8x8 block, five u32 sums (wrapping like the reference), integer
// variance scaling through the reciprocal table, fixed-point rsqrt and boost.
#include <cuda_runtime.h>

#include <algorithm>
#include <mutex>

#include "host_stage.cuh"
#include "rdo_dist_dev.cuh"

namespace {

// dist.rs:234-283.  scale: one Q14 DistortionScale per 4x4 chunk of the plane (chunk (cx, cy)
// at scale[cy * scale_stride + cx]); blocks sit on 4-pixel positions.
template <typename T>
__global__ void __launch_bounds__(256) weighted_sse_kernel(PlaneView a, PlaneView b, const b200_block *blocks,
                                                           size_t n, int w, int h, const uint32_t *scale,
                                                           long long scale_stride, unsigned long long *out) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  const int cw = w >> 2, ch = h >> 2;  // whole chunks only (vert/horz_windows(4).step_by(4))
  for (size_t i = warp0; i < n; i += nwarps) {
    const b200_block blk = blocks[i];
    unsigned long long acc = 0;
    for (int c = lane; c < cw * ch; c += 32) {
      const int cy = c / cw, cx = c - cy * cw;
      uint32_t sum = 0;
#pragma unroll
      for (int y = 0; y < 4; y++) {
        const T *pa = px<T>(a, blk.x + 4 * cx, blk.y + 4 * cy + y);
        const T *pb = px<T>(b, blk.x + 4 * cx, blk.y + 4 * cy + y);
#pragma unroll
        for (int x = 0; x < 4; x++) {
          const int d = (int)pa[x] - (int)pb[x];
          sum += (uint32_t)(d * d);
        }
      }
      acc += wsse_chunk(sum, scale[(long long)((blk.y >> 2) + cy) * scale_stride + (blk.x >> 2) + cx]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) out[i] = wsse_finish(acc);
  }
}

// dist.rs:302-372
template <typename T>
__global__ void __launch_bounds__(128) cdef_dist_kernel(PlaneView src, PlaneView dst, const b200_block *blocks,
                                                        size_t n, int w, int h, int bit_depth, uint32_t *out,
                                                        uint32_t *raw) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const b200_block blk = blocks[i];
    uint32_t sum_s = 0, sum_d = 0, sum_s2 = 0, sum_d2 = 0, sum_sd = 0;
    for (int y = 0; y < h; y++) {
      const T *ps = px<T>(src, blk.x, blk.y + y);
      const T *pd = px<T>(dst, blk.x, blk.y + y);
      for (int x = 0; x < w; x++) {
        const uint32_t s = ps[x], d = pd[x];
        sum_s += s;
        sum_d += d;
        sum_s2 += s * s;
        sum_d2 += d * d;
        sum_sd += s * d;
      }
    }
    uint32_t svar, dvar;
    const uint32_t sse = cdef_dist_vars(sum_s, sum_d, sum_s2, sum_d2, sum_sd, w * h, &svar, &dvar);
    if (raw) {  // what the asm kernels return (asm/x86/dist/cdef_dist.rs:18-24)
      raw[3 * i + 0] = svar;
      raw[3 * i + 1] = dvar;
      raw[3 * i + 2] = sse;
    }
    if (out) out[i] = apply_ssim_boost(sse, svar, dvar, bit_depth);
  }
}

int check_pair(b200_ctx *ctx, const b200_plane *a, const b200_plane *b) {
  B200_REQUIRE(ctx, a && b && a->data && b->data, "bad planes");
  B200_REQUIRE(ctx, a->bpp == b->bpp && (a->bpp == 1 || a->bpp == 2), "planes must share bpp (1 or 2)");
  return B200_OK;
}


// A host block (w x h, byte stride) staged as a device plane with a 16-byte row pitch.
size_t staged_block_bytes(int w, int h, int bpp) { return b200_align_up((size_t)w * bpp, 16) * h; }

b200_plane stage_block(HostStage &s, const void *src, ptrdiff_t stride, int w, int h, int bpp) {
  const size_t pitch = b200_align_up((size_t)w * bpp, 16);
  b200_plane p{};
  p.data = s.take(pitch * h);
  p.stride = (int32_t)(pitch / bpp);
  p.width = w;
  p.height = h;
  p.bpp = bpp;
  s.up2d(p.data, pitch, src, (size_t)stride, (size_t)w * bpp, h);
  return p;
}

}  // namespace

extern "C" int b200_weighted_sse_dev(b200_ctx *ctx, const b200_plane *src1, const b200_plane *src2,
                                     const b200_block *d_blocks, size_t nblocks, int w, int h,
                                     const uint32_t *d_scale, size_t scale_stride, uint64_t *d_out) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (int st = check_pair(ctx, src1, src2)) return st;
  B200_REQUIRE(ctx, w >= 4 && h >= 4 && w <= 128 && h <= 128, "block size %dx%d out of range (4..128)", w, h);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && d_scale && d_out, "NULL blocks / scale / output");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const int wpc = 8;
  const int grid = (int)std::min<size_t>((nblocks + wpc - 1) / wpc, (size_t)ctx->num_sms * 32);
  PlaneView a{src1->data, src1->stride}, b{src2->data, src2->stride};
  if (src1->bpp == 1)
    weighted_sse_kernel<uint8_t><<<grid, wpc * 32, 0, ctx->stream>>>(a, b, d_blocks, nblocks, w, h, d_scale,
                                                                     (long long)scale_stride,
                                                                     (unsigned long long *)d_out);
  else
    weighted_sse_kernel<uint16_t><<<grid, wpc * 32, 0, ctx->stream>>>(a, b, d_blocks, nblocks, w, h, d_scale,
                                                                      (long long)scale_stride,
                                                                      (unsigned long long *)d_out);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_cdef_dist_dev(b200_ctx *ctx, const b200_plane *src, const b200_plane *dst,
                                  const b200_block *d_blocks, size_t nblocks, int w, int h, int bit_depth,
                                  uint32_t *d_out, uint32_t *d_raw) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (int st = check_pair(ctx, src, dst)) return st;
  // dist.rs:317-318: the kernel is limited to 8x8
  B200_REQUIRE(ctx, w >= 1 && h >= 1 && w <= 8 && h <= 8, "cdef_dist_kernel: w, h must be <= 8, got %dx%d", w, h);
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bit depth %d not in {8,10,12}", bit_depth);
  B200_REQUIRE(ctx, (src->bpp == 1) == (bit_depth == 8), "bpp %d does not match bit depth %d", src->bpp, bit_depth);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && (d_out || d_raw), "NULL blocks / outputs");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const int grid = (int)std::min<size_t>((nblocks + 127) / 128, (size_t)ctx->num_sms * 32);
  PlaneView a{src->data, src->stride}, b{dst->data, dst->stride};
  if (src->bpp == 1)
    cdef_dist_kernel<uint8_t><<<grid, 128, 0, ctx->stream>>>(a, b, d_blocks, nblocks, w, h, bit_depth, d_out, d_raw);
  else
    cdef_dist_kernel<uint16_t><<<grid, 128, 0, ctx->stream>>>(a, b, d_blocks, nblocks, w, h, bit_depth, d_out, d_raw);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// ---- per-call forms (host pointers, BYTE strides): what the reference's tables bind
// (asm/x86/dist/sse.rs:18-35, asm/x86/dist/cdef_dist.rs:18-52).  Latency-bound by design.
extern "C" uint64_t b200_weighted_sse(const void *src, ptrdiff_t src_stride, const void *dst,
                                      ptrdiff_t dst_stride, const uint32_t *scale,
                                      ptrdiff_t scale_stride_bytes, int w, int h, int bpp) {
  b200_ctx *ctx = b200_default_ctx();
  const int cw = w / 4, ch = h / 4;
  const size_t plane_bytes = b200_align_up(staged_block_bytes(w, h, bpp), 256);
  const size_t scale_bytes = b200_align_up((size_t)cw * ch * 4, 256);
  HostStage s(ctx, 2 * plane_bytes + scale_bytes + 256 + 64 + 256);
  const b200_plane a = stage_block(s, src, src_stride, w, h, bpp);
  const b200_plane b = stage_block(s, dst, dst_stride, w, h, bpp);
  uint32_t *d_scale = (uint32_t *)s.take((size_t)cw * ch * 4);
  b200_block *d_blk = (b200_block *)s.take(sizeof(b200_block));
  uint64_t *d_out = (uint64_t *)s.take(8);
  const b200_block blk{0, 0};
  uint64_t out = 0;
  s.up2d(d_scale, (size_t)cw * 4, scale, (size_t)scale_stride_bytes, (size_t)cw * 4, ch);
  s.up(d_blk, &blk, sizeof blk);
  if (s.ok()) s.run(b200_weighted_sse_dev(ctx, &a, &b, d_blk, 1, w, h, d_scale, (size_t)cw, d_out));
  s.down(&out, d_out, 8);
  b200_percall_check(ctx, s.finish(true), "weighted_sse");
  return out;
}

extern "C" uint32_t b200_cdef_dist_kernel(const void *src, ptrdiff_t src_stride, const void *dst,
                                          ptrdiff_t dst_stride, int w, int h, int bit_depth, uint32_t ret[3]) {
  b200_ctx *ctx = b200_default_ctx();
  const int bpp = bit_depth == 8 ? 1 : 2;
  HostStage s(ctx, 2 * b200_align_up(staged_block_bytes(w, h, bpp), 256) + 512 + 256);
  const b200_plane a = stage_block(s, src, src_stride, w, h, bpp);
  const b200_plane b = stage_block(s, dst, dst_stride, w, h, bpp);
  b200_block *d_blk = (b200_block *)s.take(sizeof(b200_block));
  uint32_t *d_out = (uint32_t *)s.take(16);
  const b200_block blk{0, 0};
  uint32_t host[4] = {0, 0, 0, 0};
  s.up(d_blk, &blk, sizeof blk);
  if (s.ok()) s.run(b200_cdef_dist_dev(ctx, &a, &b, d_blk, 1, w, h, bit_depth, d_out, d_out + 1));
  s.down(host, d_out, 16);
  b200_percall_check(ctx, s.finish(true), "cdef_dist_kernel");
  if (ret) ret[0] = host[1], ret[1] = host[2], ret[2] = host[3];
  return host[0];
}

// ---------------------------------------------------------------- activity mask
// ActivityMask::from_plane (src/activity.rs:21-55): variance_8x8 (:71-100) of every 8x8 luma
// block of the plane rounded up to whole blocks, and fill_scales (:58-68): ssim_boost(var, var,
// bit_depth) = apply_ssim_boost(1 << 14, ..) (:147-154).  One thread per 8x8 block.
namespace {

// host+device so that tests/cpp/activity_emul.cu can replay it on the CPU against the oracle
template <typename T>
__host__ __device__ __forceinline__ uint32_t variance_8x8_px(const T *src, long long stride) {
  unsigned short sum_s_cols[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // u16 column sums, activity.rs:76
  uint32_t sum_s2_cols[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = 0; j < 8; j++)
    for (int i = 0; i < 8; i++) {
      const unsigned short s = (unsigned short)src[j * stride + i];
      sum_s_cols[i] = (unsigned short)(sum_s_cols[i] + s);
      sum_s2_cols[i] += (uint32_t)s * (uint32_t)s;
    }
  unsigned long long sum_s = 0, sum_s2 = 0;
  for (int i = 0; i < 8; i++) {
    sum_s += sum_s_cols[i];
    sum_s2 += sum_s2_cols[i];
  }
  const unsigned long long v = sum_s2 - ((sum_s * sum_s + 32) >> 6);
  return v > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)v;  // u32::try_from(..).unwrap_or(u32::MAX)
}

template <typename T>
__global__ void __launch_bounds__(128) activity_mask_kernel(PlaneView luma, int wb, int hb, int bit_depth,
                                                            uint32_t *variances, uint32_t *scales) {
  const long long n = (long long)wb * hb;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / wb), x = (int)(i - (long long)y * wb);
    const uint32_t v = variance_8x8_px<T>(px<T>(luma, 8 * x, 8 * y), luma.stride);
    variances[i] = v;
    if (scales) scales[i] = apply_ssim_boost(1u << 14, v, v, bit_depth);
  }
}

}  // namespace

extern "C" int b200_activity_mask_dev(b200_ctx *ctx, const b200_plane *luma, int bit_depth,
                                      uint32_t *d_variances, uint32_t *d_scales) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, luma && luma->data && (luma->bpp == 1 || luma->bpp == 2), "bad plane");
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bit depth %d not in {8,10,12}", bit_depth);
  B200_REQUIRE(ctx, (luma->bpp == 1) == (bit_depth == 8), "bpp %d does not match bit depth %d", luma->bpp, bit_depth);
  const int wb = (luma->width + 7) >> 3, hb = (luma->height + 7) >> 3;
  // the region is rounded up to whole 8x8 blocks (activity.rs:26-35): it reads into the padding
  B200_REQUIRE(ctx, luma->pad >= wb * 8 - luma->width && luma->pad >= hb * 8 - luma->height,
               "plane padding %d too small for the %dx%d region rounded up to 8", luma->pad, luma->width, luma->height);
  B200_REQUIRE(ctx, d_variances != nullptr, "NULL output");
  const long long n = (long long)wb * hb;
  if (n == 0) return B200_OK;  // an empty plane: a zero-block grid is not a valid launch
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const int grid = (int)std::min<long long>((n + 127) / 128, (long long)ctx->num_sms * 32);
  PlaneView p{luma->data, luma->stride};
  if (luma->bpp == 1)
    activity_mask_kernel<uint8_t><<<grid, 128, 0, ctx->stream>>>(p, wb, hb, bit_depth, d_variances, d_scales);
  else
    activity_mask_kernel<uint16_t><<<grid, 128, 0, ctx->stream>>>(p, wb, hb, bit_depth, d_variances, d_scales);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
