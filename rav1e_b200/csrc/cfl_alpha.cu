// cfl_alpha.cu — the CfL alpha search of rdo_mode_decision for sm_90a: rdo_cfl_alpha (rav1e
// src/rdo.rs:1593-1689) with luma_ac (src/predict.rs:644-698) and clip_visible_bsize (src/rdo.rs:228-253)
// for a batch of blocks in one launch.
//
// One CTA (4 warps) per block, grid-stride over the items:
//   1. the block's geometry (uniform over the CTA): validity, uv_tx_size, the visible chroma area, the
//      sub-8x8 luma offset and the per-block w_pad / h_pad; invalid and invisible blocks get the sentinels;
//   2. the CTA stages the luma AC samples (pred_cfl_ac, once for both planes), per chroma plane the
//      IntraEdge buffer (get_intra_edges with UV_CFL_PRED, rdo.rs:1625-1638) and the visible whole 4x4
//      chunks of the source;
//   3. one thread per plane forms the DC value, one thread the AC average;
//   4. the (plane, alpha, 4x4 chunk) triples are spread over the threads: a thread forms its chunk's 16
//      predicted pixels in registers (DC, then pred_cfl_inner for alpha != 0), subtracts the source and adds
//      the chunk's get_weighted_sse term at the default scale into the (plane, alpha) shared accumulator;
//   5. one thread per plane replays the early exit of rdo.rs:1664-1680 on the 33 costs, and the CTA writes
//      the chosen alpha and the SSE of every alpha the reference evaluates (UINT64_MAX for the others).
// All 33 alphas are evaluated: a prediction costs a multiply, a round and a clamp per pixel, less than the
// barriers a round-by-round search would add.  Predictions never exist in memory and `rec` is not written.
// Integer sums are order independent, so the shared-memory atomics give the reference's result exactly.
#include <algorithm>

#include "common.cuh"
#include "intra_edges_dev.cuh"
#include "ipred_dev.cuh"
#include "rdo_dist_dev.cuh"

namespace {

using namespace ipred;
using intra_edges::EdgeGeom;
using intra_edges::EdgeLens;

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kAlphas = 33;        // -16 ..= 16
constexpr int kMaxCfl = 32;        // largest chroma block of a cfl_allowed size (BLOCK_32X32 at 4:4:4)
constexpr int kMaxBsize = 9;       // BLOCK_32X32: cfl_allowed() is `self <= BLOCK_32X32` (partition.rs:228-231)
constexpr uint32_t kUnitScale = 1u << 14;  // DistortionScale::default() (rdo.rs:639-643)

struct CflArgs {
  EdgeGeom rec[2];           // the tile region of each chroma plane of rec
  const void *src[2];        // the chroma planes of src at the region's (0, 0)
  int src_stride[2];
  const void *luma;          // rec's luma plane at the region's (0, 0)
  int luma_stride;
  int rect_x, rect_y, rect_w, rect_h;  // the region, luma pixels
  int cw, ch;                // the chroma frame: ((fi.width + xdec) >> xdec, (fi.height + ydec) >> ydec)
  int w_in_b, h_in_b;        // fi.w_in_b / fi.h_in_b (encoder.rs:852-853)
  int xdec, ydec, bit_depth;
  const b200_cfl_item *items;
  size_t n;
  int8_t *alpha;             // n x 2 or NULL
  unsigned long long *sse;   // n x 2 x 33 or NULL
};

// The TxSize of a w x h block (transform/mod.rs:101-123): max_txsize_rect_lookup of a chroma block of a
// cfl_allowed size is the TxSize of its own dimensions, and av1_get_coded_tx_size leaves it (all <= 32).
__device__ __forceinline__ int tx_of_dims(int w, int h) {
  int t = 0;
  while (t < 19 && !(intra_edges::kTxW[t] == w && intra_edges::kTxH[t] == h)) t++;
  return t;
}

// clip_visible_bsize (rdo.rs:228-253), one direction
__device__ __forceinline__ int clip_visible(int frame, int blk, int pos) {
  return pos + blk <= frame ? blk : pos >= frame ? 0 : frame - pos;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) cfl_alpha_kernel(const __grid_constant__ CflArgs a) {
  __shared__ short s_ac[kMaxCfl * kMaxCfl];   // AC samples, average not yet removed
  __shared__ int s_edge[2][kEdgeLen];
  __shared__ T s_src[2][kMaxCfl * kMaxCfl];   // the visible whole chunks of each plane's source block
  __shared__ unsigned long long s_sse[2][kAlphas];
  __shared__ unsigned long long s_mask[2];    // the alphas the reference evaluates, bit alpha + 16
  __shared__ int s_red[kWarps];
  __shared__ int s_dc[2];
  __shared__ int s_avg;
  const int tid = threadIdx.x;
  const int xdec = a.xdec, ydec = a.ydec, bd = a.bit_depth;
  for (size_t it = blockIdx.x; it < a.n; it += gridDim.x) {
    const b200_cfl_item item = a.items[it];
    const int x = item.x, y = item.y, bs = item.bsize, luma_tx = item.tx_size;
    __syncthreads();  // the previous item's readers are done with shared memory

    // 1. geometry.  BlockSize::subsampled_size (partition.rs:337-379): 4:2:2 has no 4x8, 8x16 or 16x32.
    bool ok = bs <= kMaxBsize && !(xdec && !ydec && (bs == 1 || bs == 4 || bs == 7)) && luma_tx < 19 && x >= 0 &&
              y >= 0 && x < a.rect_w && y < a.rect_h && !(x & 3) && !(y & 3);
    const int bw = intra_edges::kBsW[min(bs, kMaxBsize)], bh = intra_edges::kBsH[min(bs, kMaxBsize)];
    const int txw = intra_edges::kTxW[min(luma_tx, 18)], txh = intra_edges::kTxH[min(luma_tx, 18)];
    ok = ok && txw <= bw && txh <= bh;
    const int bx = x >> 2, by = y >> 2;  // tile_bo
    // has_chroma (context/transform_unit.rs:108-121)
    ok = ok && ((bx & 1) || !((bw >> 2) & 1) || !xdec) && ((by & 1) || !((bh >> 2) & 1) || !ydec);
    // plane_bsize = uv_tx_size.block_size() (rdo.rs:1598-1601)
    const int tw = max(bw >> xdec, 4), th = max(bh >> ydec, 4);
    // visible area (rdo.rs:1603-1614): x / y from the frame block offset, not the 4-aligned chroma origin
    const int vis_w = clip_visible(a.cw, tw, (a.rect_x + x) >> xdec);
    const int vis_h = clip_visible(a.ch, th, (a.rect_y + y) >> ydec);
    if (!ok || vis_w == 0 || vis_h == 0) {
      if (a.sse && tid < 2 * kAlphas) a.sse[it * 2 * kAlphas + tid] = ~0ull;
      if (a.alpha && tid < 2) a.alpha[it * 2 + tid] = 0;
      continue;
    }

    // 2. luma AC (luma_ac, predict.rs:644-698): sub-8x8 blocks read the luma of tile_bo + sub8x8_offset
    const int sub_x = xdec && bw == 4, sub_y = ydec && bh == 4;
    const int lx = x - 4 * sub_x, ly = y - 4 * sub_y;
    int max_luma_w = bw, max_luma_h = bh;
    if (bw > 8) {  // frame_clipped_bw rounded up to the luma tx width
      const int clipped = min((a.w_in_b - ((a.rect_x + lx) >> 2)) << 2, bw);
      max_luma_w = (clipped + txw - 1) / txw * txw;
    }
    if (bh > 8) {
      const int clipped = min((a.h_in_b - ((a.rect_y + ly) >> 2)) << 2, bh);
      max_luma_h = (clipped + txh - 1) / txh * txh;
    }
    const CflAcShape shape =
        cfl_ac_shape(tw, th, (bw - max_luma_w) >> (2 + xdec), (bh - max_luma_h) >> (2 + ydec), xdec, ydec);
    const T *luma = (const T *)a.luma + (long long)ly * a.luma_stride + lx;
    int local = 0;
    for (int i = tid; i < tw * th; i += kThreads) {
      const short s = cfl_ac_sample(shape, luma, a.luma_stride, i);
      s_ac[i] = s;
      local += s;
    }
    local = (int)warp_sum_u32((uint32_t)local);
    if ((tid & 31) == 0) s_red[tid >> 5] = local;

    // edges, once per chroma plane: get_intra_edges(rec, tile_bo, 0, 0, bsize, po, uv_tx_size, UV_CFL_PRED)
    const int po_x = (bx >> xdec) << 2, po_y = (by >> ydec) << 2;  // tile_bo.plane_offset
    b200_edge_item e{};
    e.po_x = (int16_t)po_x;
    e.po_y = (int16_t)po_y;
    e.part_x = (int16_t)bx;
    e.part_y = (int16_t)by;
    e.bsize = (uint8_t)bs;
    e.tx_size = (uint8_t)tx_of_dims(tw, th);
    e.mode = UV_CFL_PRED;
    const EdgeLens lens0 = intra_edges::gather_intra_edge<T>(a.rec[0], e, tid, kThreads, s_edge[0]);
    const EdgeLens lens1 = intra_edges::gather_intra_edge<T>(a.rec[1], e, tid, kThreads, s_edge[1]);

    // the source chunks sse_wxh reads: whole 4x4 chunks of the visible area (dist.rs:248-251)
    const int ncx = vis_w >> 2, nch = ncx * (vis_h >> 2);
    const int sw = ncx * 4;
    for (int p = 0; p < 2; p++) {
      const T *src = (const T *)a.src[p] + (long long)po_y * a.src_stride[p] + po_x;
      for (int i = tid; i < nch * 16; i += kThreads) {
        const int r = i / sw, c = i - r * sw;
        s_src[p][r * tw + c] = src[(long long)r * a.src_stride[p] + c];
      }
    }
    if (tid < 2 * kAlphas) s_sse[tid / kAlphas][tid % kAlphas] = 0;
    __syncthreads();

    // 3. the DC value of each plane (predict_intra with UV_CFL_PRED, predict.rs:212-248: the variant from the
    //    4-aligned chroma origin in the tile) and the AC average
    if (tid < 2) {
      const int variant = (po_x == 0 && po_y == 0) ? VAR_NONE : po_y == 0 ? VAR_LEFT : po_x == 0 ? VAR_TOP : VAR_BOTH;
      s_dc[tid] = ipred_dc(s_edge[tid], variant, tw, th, tid ? lens1.left : lens0.left, bd);
    } else if (tid == 32) {
      int sum = 0;
      for (int k = 0; k < kWarps; k++) sum += s_red[k];
      s_avg = cfl_ac_average(shape, sum);
    }
    __syncthreads();

    // 4. the chunk SSE of every (plane, alpha)
    const short avg = (short)s_avg;
    const int maxv = (1 << bd) - 1;
    for (int u = tid; u < 2 * kAlphas * nch; u += kThreads) {
      const int p = u / (kAlphas * nch), rem = u - p * kAlphas * nch;
      const int ai = rem / nch, ch = rem - ai * nch;
      const int r0 = (ch / ncx) * 4, c0 = (ch - (ch / ncx) * ncx) * 4;
      const int dc = s_dc[p], alpha = ai - 16;
      uint32_t sum = 0;
#pragma unroll
      for (int k = 0; k < 16; k++) {
        const int idx = (r0 + (k >> 2)) * tw + c0 + (k & 3);
        // alpha 0 is DC_PRED (predict.rs:236); cfl_pixel adds nothing for it
        const int pred = cfl_pixel(dc, alpha, (short)(s_ac[idx] - avg), maxv);
        const int d = (int)s_src[p][idx] - pred;
        sum += (uint32_t)(d * d);
      }
      atomicAdd(&s_sse[p][ai], wsse_chunk(sum, kUnitScale));
    }
    __syncthreads();

    // 5. the selection (rdo.rs:1664-1680): +alpha, then -alpha against the updated best; a strict
    //    improvement adds 2 to count; stop once count < alpha
    if (tid < 2) {
      unsigned long long *cost = s_sse[tid];
      for (int k = 0; k < kAlphas; k++) cost[k] = wsse_finish(cost[k]);
      unsigned long long best_cost = cost[16], mask = 1ull << 16;
      int best = 0, count = 2;
      for (int al = 1; al <= 16; al++) {
        mask |= 1ull << (16 + al) | 1ull << (16 - al);
        if (cost[16 + al] < best_cost) {
          best_cost = cost[16 + al];
          best = al;
          count += 2;
        }
        if (cost[16 - al] < best_cost) {
          best_cost = cost[16 - al];
          best = -al;
          count += 2;
        }
        if (count < al) break;
      }
      s_mask[tid] = mask;
      if (a.alpha) a.alpha[it * 2 + tid] = (int8_t)best;
    }
    __syncthreads();
    if (a.sse && tid < 2 * kAlphas) {
      const int p = tid / kAlphas, ai = tid - p * kAlphas;
      a.sse[it * 2 * kAlphas + tid] = (s_mask[p] >> ai) & 1ull ? s_sse[p][ai] : ~0ull;
    }
  }
}

}  // namespace

extern "C" int b200_cfl_alpha_dev(b200_ctx *ctx, const b200_plane rec[3], const b200_plane src[3], int xdec, int ydec,
                                  int rect_x, int rect_y, int rect_w, int rect_h, int frame_width, int frame_height,
                                  int bit_depth, const b200_cfl_item *d_items, size_t nitems, int8_t *d_alpha,
                                  uint64_t *d_sse) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, rec && src, "NULL rec / src");
  B200_REQUIRE(ctx, d_alpha || d_sse, "both outputs are NULL");
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  B200_REQUIRE(ctx, (xdec == 1 && ydec == 1) || (xdec == 1 && ydec == 0) || (xdec == 0 && ydec == 0),
               "chroma layout (xdec %d, ydec %d) is not 4:2:0, 4:2:2 or 4:4:4", xdec, ydec);
  B200_REQUIRE(ctx, frame_width > 0 && frame_height > 0 && frame_width <= 32760 && frame_height <= 32760,
               "bad frame size %dx%d", frame_width, frame_height);
  const int bpp = bit_depth == 8 ? 1 : 2;
  const int cw = (frame_width + xdec) >> xdec, ch = (frame_height + ydec) >> ydec;
  for (int k = 0; k < 5; k++) {
    const b200_plane &pl = k < 3 ? rec[k] : src[k - 2];
    const int p = k < 3 ? k : k - 2;
    const int fw = p ? cw : frame_width, fh = p ? ch : frame_height;
    B200_REQUIRE(ctx, pl.data != nullptr, "NULL %s plane %d", k < 3 ? "rec" : "src", p);
    B200_REQUIRE(ctx, pl.bpp == bpp, "%s plane %d: bpp %d does not match bit depth %d", k < 3 ? "rec" : "src", p,
                 pl.bpp, bit_depth);
    B200_REQUIRE(ctx, pl.width >= fw && pl.height >= fh && pl.stride >= pl.width,
                 "%s plane %d (%dx%d) smaller than the frame's (%dx%d)", k < 3 ? "rec" : "src", p, pl.width,
                 pl.height, fw, fh);
  }
  for (int p = 1; p < 3; p++)
    B200_REQUIRE(ctx, src[p].width == rec[p].width && src[p].height == rec[p].height,
                 "src plane %d (%dx%d) and rec plane %d (%dx%d) differ", p, src[p].width, src[p].height, p,
                 rec[p].width, rec[p].height);
  // luma_ac reads up to 31 pixels past the last visible column / row (frame_clipped_bw counts the frame's
  // 8x8 blocks, and max_luma_w rounds that up to the luma tx width)
  B200_REQUIRE(ctx, rec[0].width + rec[0].pad >= frame_width + 31 && rec[0].height + rec[0].pad >= frame_height + 31,
               "rec luma plane %dx%d with pad %d does not reach %d pixels past the %dx%d frame", rec[0].width,
               rec[0].height, rec[0].pad, 31, frame_width, frame_height);
  const int w_in_b = 2 * ((frame_width + 7) >> 3), h_in_b = 2 * ((frame_height + 7) >> 3);
  B200_REQUIRE(ctx, rect_x >= 0 && rect_y >= 0 && rect_w > 0 && rect_h > 0 && !(rect_x & 7) && !(rect_y & 7) &&
                        rect_x + rect_w <= 4 * w_in_b && rect_y + rect_h <= 4 * h_in_b,
               "region (%d, %d, %d, %d) outside the %dx%d frame's 8x8 blocks or not 8-aligned", rect_x, rect_y,
               rect_w, rect_h, 4 * w_in_b, 4 * h_in_b);
  if (nitems == 0) return B200_OK;
  B200_REQUIRE(ctx, d_items != nullptr, "NULL items");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  CflArgs a{};
  for (int p = 0; p < 2; p++) {
    const b200_plane &r = rec[p + 1], &s = src[p + 1];
    const int crx = rect_x >> xdec, cry = rect_y >> ydec;
    a.rec[p].data = (const uint8_t *)r.data + ((long long)cry * r.stride + crx) * bpp;
    a.rec[p].stride = r.stride;
    a.rec[p].plane_w = r.width;
    a.rec[p].plane_h = r.height;
    a.rec[p].rect_x = crx, a.rec[p].rect_y = cry;
    a.rec[p].rect_w = rect_w >> xdec, a.rec[p].rect_h = rect_h >> ydec;  // TileRect::decimated (tile.rs:29-36)
    a.rec[p].xdec = xdec, a.rec[p].ydec = ydec;
    a.rec[p].bit_depth = bit_depth;
    a.src[p] = (const uint8_t *)s.data + ((long long)cry * s.stride + crx) * bpp;
    a.src_stride[p] = s.stride;
  }
  a.luma = (const uint8_t *)rec[0].data + ((long long)rect_y * rec[0].stride + rect_x) * bpp;
  a.luma_stride = rec[0].stride;
  a.rect_x = rect_x, a.rect_y = rect_y, a.rect_w = rect_w, a.rect_h = rect_h;
  a.cw = cw, a.ch = ch;
  a.w_in_b = w_in_b, a.h_in_b = h_in_b;
  a.xdec = xdec, a.ydec = ydec, a.bit_depth = bit_depth;
  a.items = d_items;
  a.n = nitems;
  a.alpha = d_alpha;
  a.sse = (unsigned long long *)d_sse;
  const int grid = (int)std::min<size_t>(nitems, (size_t)ctx->num_sms * 16);
  if (bpp == 1)
    cfl_alpha_kernel<uint8_t><<<grid, kThreads, 0, ctx->stream>>>(a);
  else
    cfl_alpha_kernel<uint16_t><<<grid, kThreads, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
