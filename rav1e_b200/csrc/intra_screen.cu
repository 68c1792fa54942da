// intra_screen.cu — intra mode screening for sm_90a: the pruning metric of
// intra_frame_rdo_mode_decision (rav1e src/rdo.rs:1433-1511) with PredictionMode::predict_intra
// (src/predict.rs:205-249) for a batch of luma blocks in one launch.
//
// One CTA (4 warps) per block, grid-stride over the items:
//   1. the CTA gathers the block's IntraEdge buffer (get_intra_edges, mode None) from `rec` straight
//      into shared memory and stages the tx-sized source block next to it;
//   2. thread 0 forms the DC value (shared by DC_PRED and PAETH_PRED remapped to DC), and each warp
//      filters / upsamples the edges of the screened directional modes it owns (D45..D67, one edge
//      pair each, ipred_filter_edges on a warp);
//   3. the (screened mode, Hadamard chunk) pairs are spread over the threads: a thread evaluates its
//      chunk's predicted pixels straight into registers (ipred_pixel_k after one dispatch on the
//      predictor kind when its warp agrees on the kind, ipred_pixel otherwise), subtracts the source and
//      adds the 8x8 (4x4 when a side is 4) Hadamard abs-sum into the mode's shared accumulator;
//   4. thread 0 applies get_satd's one final rounding and stable-sorts the tail of the mode list.
// Predictions never exist in memory.  Integer sums are order independent, so the shared-memory
// atomics give the reference's result exactly.
#include <algorithm>

#include "common.cuh"
#include "hadamard.cuh"
#include "intra_edges_dev.cuh"
#include "ipred_dev.cuh"

namespace {

using namespace ipred;
using intra_edges::EdgeGeom;
using intra_edges::EdgeLens;

constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kModes = 13;  // RAV1E_INTRA_MODES
constexpr int kDir = 6;     // D45_PRED..D67_PRED: the modes whose edges are filtered

// BlockSize::tx_size (partition.rs:306-328), BlockSize order
__constant__ uint8_t kBsTx[22] = {0, 5, 6, 1, 7, 8, 2, 9, 10, 3, 11, 12, 4, 4, 4, 4, 13, 14, 15, 16, 17, 18};

struct ScreenArgs {
  EdgeGeom rec;            // the tile region of rec
  const void *src;         // src pixel at the region's (0, 0)
  int src_stride;
  int num_modes_rdo;
  const b200_intra_screen_item *items;
  size_t n;
  uint32_t *satd;          // n x 13 or NULL
  uint8_t *modes;          // n x 13 or NULL
};

template <typename T>
__global__ void __launch_bounds__(kThreads) intra_screen_kernel(const __grid_constant__ ScreenArgs a) {
  __shared__ int s_edge[kEdgeLen];
  __shared__ int s_fa[kDir][kEdgeLen], s_fl[kDir][kEdgeLen];  // per directional mode: filtered edges
  __shared__ int s_sa[kWarps][kEdgeLen], s_sl[kWarps][kEdgeLen];  // per warp: filter staging
  __shared__ T s_src[kMaxTx * kMaxTx];
  __shared__ uint32_t s_sum[kModes];
  __shared__ uint8_t s_list[kModes];
  __shared__ int s_dc;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int skip = a.num_modes_rdo >> 1;
  for (size_t it = blockIdx.x; it < a.n; it += gridDim.x) {
    const b200_intra_screen_item item = a.items[it];
    const int x = item.x, y = item.y;
    bool ok = item.bsize < 22 && x >= 0 && y >= 0 && x < a.rec.rect_w && y < a.rec.rect_h && !(x & 3) && !(y & 3);
    unsigned seen = 0, screened = 0;
#pragma unroll
    for (int k = 0; k < kModes; k++) {
      const int m = item.modes[k];
      ok = ok && m < kModes && !((seen >> m) & 1u);
      seen |= 1u << (m & 31);
      if (k >= skip) screened |= 1u << (m & 31);
    }
    __syncthreads();  // the previous item's readers are done with shared memory
    if (!ok) {
      if (tid < kModes) {
        if (a.satd) a.satd[it * kModes + tid] = UINT32_MAX;
        if (a.modes) a.modes[it * kModes + tid] = a.items[it].modes[tid];
      }
      continue;
    }
    const int tx = kBsTx[item.bsize];
    const int w = intra_edges::kTxW[tx], h = intra_edges::kTxH[tx];
    const int bd = a.rec.bit_depth;

    // 1. edges (get_intra_edges with mode None, rdo.rs:1443-1461) and the source block
    b200_edge_item e{};
    e.po_x = (int16_t)x;
    e.po_y = (int16_t)y;
    e.part_x = (int16_t)(x >> 2);
    e.part_y = (int16_t)(y >> 2);
    e.bsize = item.bsize;
    e.tx_size = (uint8_t)tx;
    e.mode = 255;
    e.enable_ief = item.ief >= 0;
    const EdgeLens lens = intra_edges::gather_intra_edge<T>(a.rec, e, tid, kThreads, s_edge);
    const int lw = 31 - __clz(w);
    const T *src = (const T *)a.src + (long long)y * a.src_stride + x;
    for (int i = tid; i < w * h; i += kThreads) s_src[i] = src[(long long)(i >> lw) * a.src_stride + (i & (w - 1))];
    if (tid < kModes) {
      s_sum[tid] = 0;
      s_list[tid] = a.items[it].modes[tid];
    }
    __syncthreads();

    // 2. preparation: DC value, filtered edges of the screened directional modes
    const int variant = (x == 0 && y == 0) ? VAR_NONE : y == 0 ? VAR_LEFT : x == 0 ? VAR_TOP : VAR_BOTH;
    if (tid == 0) s_dc = ipred_dc(s_edge, variant, w, h, lens.left, bd);
    if (item.ief >= 0) {
      for (int j = warp; j < kDir; j += kWarps) {
        if (!((screened >> (D45_PRED + j)) & 1u)) continue;
        const IpredPix p = ipred_setup(s_edge, D45_PRED + j, intra_edges::kModeAngle[D45_PRED + j], item.ief,
                                       lens.left, w, h, bd, s_fa[j], s_fl[j], 0);
        ipred_filter_edges(WarpGroup(), p, lens.above, a.rec.plane_w, a.rec.plane_h, a.rec.rect_x + x,
                           a.rec.rect_y + y, s_sa[warp], s_sl[warp], s_fa[j], s_fl[j]);
      }
    }
    __syncthreads();

    // 3. SATD chunks of every screened mode
    const int cs = min(w, h) == 4 ? 4 : 8;
    const int cw = w / cs, nch = cw * (h / cs);
    for (int u = tid; u < (kModes - skip) * nch; u += kThreads) {
      const int mi = u / nch, ch = u - mi * nch;
      const int luma_mode = s_list[skip + mi];
      // predict_intra (predict.rs:214-248): PAETH at the tile's edges, the angle, ief for directional modes
      int mode = luma_mode;
      if (mode == PAETH_PRED)
        mode = variant == VAR_NONE ? DC_PRED : variant == VAR_TOP ? V_PRED : variant == VAR_LEFT ? H_PRED : PAETH_PRED;
      const int angle = mode >= V_PRED && mode <= D67_PRED ? intra_edges::kModeAngle[mode] : 0;
      const int ief = luma_mode >= V_PRED && luma_mode <= D67_PRED ? item.ief : -1;
      const int dj = min(max(mode - D45_PRED, 0), kDir - 1);
      const IpredPix p = ipred_setup(s_edge, mode, angle, ief, lens.left, w, h, bd, s_fa[dj], s_fl[dj], s_dc);
      const int r0 = (ch / cw) * cs, c0 = (ch - (ch / cw) * cw) * cs;
      // d = source - prediction.  When every active lane of the warp runs the same predictor kind
      // (the modes of the larger blocks span whole warps), one dispatch per chunk puts a single
      // predictor's code in the unrolled loop; lanes of mixed kinds (a warp of 4x4 / 8x8 blocks' modes)
      // run the generic per-pixel form instead of serialising one whole unrolled loop per kind.
      const unsigned active = __activemask();
      const bool uniform = __match_any_sync(active, p.kind) == active;
      uint32_t s;
      if (cs == 4) {
        int d[16];
        auto fill = [&](auto kind) {
#pragma unroll
          for (int k = 0; k < 16; k++)
            d[k] = (int)s_src[(r0 + (k >> 2)) * w + c0 + (k & 3)] -
                   ipred_pixel_k<decltype(kind)::value>(p, r0 + (k >> 2), c0 + (k & 3));
        };
        if (uniform) {
          ipred_dispatch(p, fill);
        } else {
#pragma unroll
          for (int k = 0; k < 16; k++)
            d[k] = (int)s_src[(r0 + (k >> 2)) * w + c0 + (k & 3)] - ipred_pixel(p, r0 + (k >> 2), c0 + (k & 3));
        }
        s = hadamard4x4_abs_sum(d);
      } else {
        int d[64];
        auto fill = [&](auto kind) {
#pragma unroll
          for (int k = 0; k < 64; k++)
            d[k] = (int)s_src[(r0 + (k >> 3)) * w + c0 + (k & 7)] -
                   ipred_pixel_k<decltype(kind)::value>(p, r0 + (k >> 3), c0 + (k & 7));
        };
        if (uniform) {
          ipred_dispatch(p, fill);
        } else {
#pragma unroll
          for (int k = 0; k < 64; k++)
            d[k] = (int)s_src[(r0 + (k >> 3)) * w + c0 + (k & 7)] - ipred_pixel(p, r0 + (k >> 3), c0 + (k & 7));
        }
        s = hadamard8x8_abs_sum(d);
      }
      atomicAdd(&s_sum[luma_mode], s);
    }
    __syncthreads();

    // 4. get_satd's rounding (dist.rs:156-221), the stable tail sort (rdo.rs:1511), the outputs
    if (tid == 0) {
      const int ln = cs == 4 ? 2 : 3;
      for (int m = 0; m < kModes; m++)
        s_sum[m] = ((screened >> m) & 1u) ? (s_sum[m] + ((1u << ln) >> 1)) >> ln : 0u;
      for (int k = skip + 1; k < kModes; k++) {
        const uint8_t m = s_list[k];
        int j = k;
        for (; j > skip && s_sum[s_list[j - 1]] > s_sum[m]; j--) s_list[j] = s_list[j - 1];
        s_list[j] = m;
      }
    }
    __syncthreads();
    if (tid < kModes) {
      if (a.satd) a.satd[it * kModes + tid] = s_sum[tid];
      if (a.modes) a.modes[it * kModes + tid] = s_list[tid];
    }
  }
}

}  // namespace

extern "C" int b200_intra_mode_screen_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src, int rect_x,
                                          int rect_y, int rect_w, int rect_h, int bit_depth, int num_modes_rdo,
                                          const b200_intra_screen_item *d_items, size_t nitems, uint32_t *d_satd,
                                          uint8_t *d_modes) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, num_modes_rdo == 3 || num_modes_rdo == 7, "num_modes_rdo %d is not 3 or 7", num_modes_rdo);
  B200_REQUIRE(ctx, rec && rec->data && src && src->data, "NULL plane");
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  B200_REQUIRE(ctx, rec->bpp == (bit_depth == 8 ? 1 : 2) && src->bpp == rec->bpp, "bpp %d / %d vs bit depth %d",
               rec->bpp, src->bpp, bit_depth);
  B200_REQUIRE(ctx, rec->width == src->width && rec->height == src->height, "rec %dx%d vs src %dx%d", rec->width,
               rec->height, src->width, src->height);
  B200_REQUIRE(ctx, rect_x >= 0 && rect_y >= 0 && rect_w > 0 && rect_h > 0 && rect_x + rect_w <= rec->width &&
                        rect_y + rect_h <= rec->height,
               "region (%d, %d, %d, %d) outside the %dx%d plane", rect_x, rect_y, rect_w, rect_h, rec->width,
               rec->height);
  B200_REQUIRE(ctx, rec->pad >= kMaxTx && src->pad >= kMaxTx, "plane padding %d / %d below %d", rec->pad, src->pad,
               kMaxTx);
  B200_REQUIRE(ctx, d_satd || d_modes, "both outputs are NULL");
  if (nitems == 0) return B200_OK;
  B200_REQUIRE(ctx, d_items != nullptr, "NULL items");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  ScreenArgs a{};
  a.rec.data = (const uint8_t *)rec->data + ((long long)rect_y * rec->stride + rect_x) * rec->bpp;
  a.rec.stride = rec->stride;
  a.rec.plane_w = rec->width;
  a.rec.plane_h = rec->height;
  a.rec.rect_x = rect_x, a.rec.rect_y = rect_y, a.rec.rect_w = rect_w, a.rec.rect_h = rect_h;
  a.rec.bit_depth = bit_depth;
  a.src = (const uint8_t *)src->data + ((long long)rect_y * src->stride + rect_x) * src->bpp;
  a.src_stride = src->stride;
  a.num_modes_rdo = num_modes_rdo;
  a.items = d_items;
  a.n = nitems;
  a.satd = d_satd;
  a.modes = d_modes;
  const int grid = (int)std::min<size_t>(nitems, (size_t)ctx->num_sms * 8);
  if (bit_depth == 8)
    intra_screen_kernel<uint8_t><<<grid, kThreads, 0, ctx->stream>>>(a);
  else
    intra_screen_kernel<uint16_t><<<grid, kThreads, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
