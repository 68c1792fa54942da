// lookahead.cu — the frame-wide, dependence-free consumers of the SATD / intra kernels (sm_90a).
//
//   Plane::downsampled + Plane::pad        v_frame 0.3.9 (off disk); src/encoder.rs:476-477 builds the half
//                                          and quarter resolution planes of the ME pyramid with it
//   estimate_intra_costs                   src/api/lookahead.rs:30-128
//   estimate_importance_block_difference   src/api/lookahead.rs:131-180
//   estimate_inter_costs (cost part)       src/api/lookahead.rs:238-270
//
// Every 8x8 importance block of a frame is independent here (the source frame is its own neighbour),
// so one launch covers a frame: 32 400 blocks at 1080p.  The intra cost fuses what the reference does
// in three calls per block - get_intra_edges(DC_PRED) -> DC prediction -> get_satd - without the edge
// buffer or the prediction ever existing in memory: a thread reads its block, the row above and the
// column to the left, forms the DC of its PredictionVariant and runs the 8x8 Hadamard on org - dc.
#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"
#include "hadamard.cuh"

namespace {

template <typename T>
__device__ __forceinline__ int at(const PlaneView &v, int x, int y) {
  return *px<T>(v, x, y);
}

// ---- Plane::downsampled + Plane::pad
template <typename T>
__global__ void downsample_kernel(PlaneView src, T *dst, int dst_stride, int w, int h, int pad, int pad_w, int pad_h) {
  const int tw = w + 2 * pad, th = h + 2 * pad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)tw * th;
       i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / tw) - pad, x = (int)(i % tw) - pad;
    // everything outside [0, pad_w) x [0, pad_h) is a replica of the nearest pixel inside (Plane::pad)
    const int cx = min(max(x, 0), pad_w - 1), cy = min(max(y, 0), pad_h - 1);
    const int sum = at<T>(src, 2 * cx, 2 * cy) + at<T>(src, 2 * cx + 1, 2 * cy) + at<T>(src, 2 * cx, 2 * cy + 1) +
                    at<T>(src, 2 * cx + 1, 2 * cy + 1);
    dst[(long long)y * dst_stride + x] = (T)((sum + 2) >> 2);
  }
}

// ---- estimate_intra_costs
template <typename T>
__global__ void __launch_bounds__(128) intra_cost_kernel(PlaneView luma, int wb, int hb, int bit_depth, uint32_t *costs) {
  const int n = wb * hb;
  for (int blk = blockIdx.x * blockDim.x + threadIdx.x; blk < n; blk += gridDim.x * blockDim.x) {
    const int by = blk / wb, bx = blk - by * wb, x = 8 * bx, y = 8 * by;
    int d[64];
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
      for (int c = 0; c < 8; c++) d[r * 8 + c] = at<T>(luma, x + c, y + r);
    // PredictionVariant::new (predict.rs:126-135) and pred_dc* (predict.rs:795-858) on the edges
    // get_intra_edges(DC_PRED) would gather (partition.rs:711-762): real pixels wherever they are used
    int dc;
    if (x != 0 && y != 0) {
      int s = 0;
#pragma unroll
      for (int k = 0; k < 8; k++) s += at<T>(luma, x - 1, y + k) + at<T>(luma, x + k, y - 1);
      dc = (s + 8) >> 4;
    } else if (x != 0) {  // LEFT
      int s = 0;
#pragma unroll
      for (int k = 0; k < 8; k++) s += at<T>(luma, x - 1, y + k);
      dc = (s + 4) >> 3;
    } else if (y != 0) {  // TOP
      int s = 0;
#pragma unroll
      for (int k = 0; k < 8; k++) s += at<T>(luma, x + k, y - 1);
      dc = (s + 4) >> 3;
    } else {
      dc = 128 << (bit_depth - 8);
    }
#pragma unroll
    for (int i = 0; i < 64; i++) d[i] -= dc;
    costs[blk] = satd8x8(d);
  }
}

// ---- estimate_inter_costs: SATD(org block, reference block displaced by the block's mv)
template <typename T>
__global__ void __launch_bounds__(128) inter_cost_kernel(PlaneView org, PlaneView ref, int wb, int hb, const short *mvs,
                                                         uint32_t *costs, unsigned long long *total) {
  const int n = wb * hb;
  unsigned long long mine = 0;
  for (int blk = blockIdx.x * blockDim.x + threadIdx.x; blk < n; blk += gridDim.x * blockDim.x) {
    const int by = blk / wb, bx = blk - by * wb;
    // lookahead.rs:246-260: (x * 64 + mv.col) as isize / 8 - the SUM truncates toward zero
    const int rx = (bx * 64 + (int)mvs[2 * blk + 1]) / 8, ry = (by * 64 + (int)mvs[2 * blk]) / 8;
    int d[64];
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
      for (int c = 0; c < 8; c++) d[r * 8 + c] = at<T>(org, 8 * bx + c, 8 * by + r) - at<T>(ref, rx + c, ry + r);
    const uint32_t s = satd8x8(d);
    if (costs) costs[blk] = s;
    mine += s;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(total, mine);
}

// ---- estimate_importance_block_difference
template <typename T>
__global__ void __launch_bounds__(128) imp_diff_kernel(PlaneView org, PlaneView ref, int wb, int hb, unsigned long long *total) {
  const int n = wb * hb;
  unsigned long long mine = 0;
  for (int blk = blockIdx.x * blockDim.x + threadIdx.x; blk < n; blk += gridDim.x * blockDim.x) {
    const int by = blk / wb, bx = blk - by * wb;
    long long so = 0, sr = 0;
    for (int r = 0; r < 8; r++) {
      unsigned ro = 0, rr = 0;  // u16 row sums upstream: 8 x 4095 < 65536, no wrap
#pragma unroll
      for (int c = 0; c < 8; c++) {
        ro += (unsigned)at<T>(org, 8 * bx + c, 8 * by + r);
        rr += (unsigned)at<T>(ref, 8 * bx + c, 8 * by + r);
      }
      so += ro;
      sr += rr;
    }
    const long long m = (so + 32) / 64 - (sr + 32) / 64;
    mine += (unsigned long long)(m < 0 ? -m : m);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(total, mine);
}

// `imp_block_costs as f64 / (w_in_imp_b * h_in_imp_b) as f64`: one correctly rounded division
__global__ void mean_kernel(const unsigned long long *total, unsigned long long count, double *out) {
  *out = __ddiv_rn(__ull2double_rn(*total), __ull2double_rn(count));
}

int check_pair(b200_ctx *ctx, const b200_plane *a, const b200_plane *b) {
  B200_REQUIRE(ctx, a && b && a->data && b->data, "NULL plane");
  B200_REQUIRE(ctx, a->bpp == b->bpp && (a->bpp == 1 || a->bpp == 2), "planes must share bpp (1 or 2)");
  B200_REQUIRE(ctx, a->width == b->width && a->height == b->height, "planes must share their size");
  return B200_OK;
}

}  // namespace

extern "C" int b200_plane_downsample_dev(b200_ctx *ctx, const b200_plane *src, const b200_plane *dst, int pad_w,
                                         int pad_h) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, src && dst && src->data && dst->data && src->bpp == dst->bpp && (src->bpp == 1 || src->bpp == 2),
               "bad planes");
  const int w = (src->width + 1) / 2, h = (src->height + 1) / 2;
  B200_REQUIRE(ctx, dst->width == w && dst->height == h, "destination must be %d x %d (is %d x %d)", w, h, dst->width,
               dst->height);
  B200_REQUIRE(ctx, pad_w >= 1 && pad_w <= w && pad_h >= 1 && pad_h <= h, "pad size %d x %d outside 1..%d x 1..%d",
               pad_w, pad_h, w, h);
  // the last column / row of an odd-sized source reads one pixel of its padding
  B200_REQUIRE(ctx, src->pad >= 1 || ((src->width & 1) == 0 && (src->height & 1) == 0),
               "an odd-sized source needs at least one padding pixel");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const long long total = (long long)(w + 2 * dst->pad) * (h + 2 * dst->pad);
  const int grid = (int)std::min<long long>((total + 255) / 256, (long long)ctx->num_sms * 16);
  const PlaneView s{src->data, src->stride};
  if (src->bpp == 1)
    downsample_kernel<uint8_t><<<grid, 256, 0, ctx->stream>>>(s, (uint8_t *)dst->data, dst->stride, w, h, dst->pad, pad_w, pad_h);
  else
    downsample_kernel<uint16_t><<<grid, 256, 0, ctx->stream>>>(s, (uint16_t *)dst->data, dst->stride, w, h, dst->pad, pad_w, pad_h);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_estimate_intra_costs_dev(b200_ctx *ctx, const b200_plane *luma, int bit_depth, uint32_t *d_costs) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, luma && luma->data && d_costs, "NULL plane / output");
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bit depth %d not in {8,10,12}", bit_depth);
  B200_REQUIRE(ctx, (luma->bpp == 1 || luma->bpp == 2) && (luma->bpp == 1) == (bit_depth == 8),
               "bpp %d vs bit depth %d", luma->bpp, bit_depth);
  const int wb = luma->width / 8, hb = luma->height / 8;
  if (wb == 0 || hb == 0) return B200_OK;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const int grid = std::min((wb * hb + 127) / 128, ctx->num_sms * 8);
  const PlaneView v{luma->data, luma->stride};
  if (luma->bpp == 1)
    intra_cost_kernel<uint8_t><<<grid, 128, 0, ctx->stream>>>(v, wb, hb, bit_depth, d_costs);
  else
    intra_cost_kernel<uint16_t><<<grid, 128, 0, ctx->stream>>>(v, wb, hb, bit_depth, d_costs);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_estimate_inter_costs_dev(b200_ctx *ctx, const b200_plane *org, const b200_plane *ref,
                                             const int16_t *d_mvs, uint32_t *d_costs, uint64_t *d_scratch,
                                             double *d_mean) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (int st = check_pair(ctx, org, ref)) return st;
  B200_REQUIRE(ctx, d_mvs && d_scratch && d_mean, "NULL motion vectors / scratch / output");
  const int wb = org->width / 8, hb = org->height / 8;
  B200_REQUIRE(ctx, wb > 0 && hb > 0, "plane smaller than an importance block");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  B200_CUDA(ctx, cudaMemsetAsync(d_scratch, 0, 8, ctx->stream));
  const int grid = std::min((wb * hb + 127) / 128, ctx->num_sms * 8);
  const PlaneView o{org->data, org->stride}, r{ref->data, ref->stride};
  if (org->bpp == 1)
    inter_cost_kernel<uint8_t><<<grid, 128, 0, ctx->stream>>>(o, r, wb, hb, d_mvs, d_costs, (unsigned long long *)d_scratch);
  else
    inter_cost_kernel<uint16_t><<<grid, 128, 0, ctx->stream>>>(o, r, wb, hb, d_mvs, d_costs, (unsigned long long *)d_scratch);
  B200_LAUNCH_CHECK(ctx);
  mean_kernel<<<1, 1, 0, ctx->stream>>>((const unsigned long long *)d_scratch, (unsigned long long)wb * hb, d_mean);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_importance_block_difference_dev(b200_ctx *ctx, const b200_plane *org, const b200_plane *ref,
                                                    uint64_t *d_scratch, double *d_mean) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (int st = check_pair(ctx, org, ref)) return st;
  B200_REQUIRE(ctx, d_scratch && d_mean, "NULL scratch / output");
  const int wb = org->width / 8, hb = org->height / 8;
  B200_REQUIRE(ctx, wb > 0 && hb > 0, "plane smaller than an importance block");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  B200_CUDA(ctx, cudaMemsetAsync(d_scratch, 0, 8, ctx->stream));
  const int grid = std::min((wb * hb + 127) / 128, ctx->num_sms * 8);
  const PlaneView o{org->data, org->stride}, r{ref->data, ref->stride};
  if (org->bpp == 1)
    imp_diff_kernel<uint8_t><<<grid, 128, 0, ctx->stream>>>(o, r, wb, hb, (unsigned long long *)d_scratch);
  else
    imp_diff_kernel<uint16_t><<<grid, 128, 0, ctx->stream>>>(o, r, wb, hb, (unsigned long long *)d_scratch);
  B200_LAUNCH_CHECK(ctx);
  mean_kernel<<<1, 1, 0, ctx->stream>>>((const unsigned long long *)d_scratch, (unsigned long long)wb * hb, d_mean);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
