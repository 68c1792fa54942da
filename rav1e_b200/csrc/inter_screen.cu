// inter_screen.cu — inter mode screening for sm_90a: the SATD pruning of inter_frame_rdo_mode_decision
// (rav1e src/rdo.rs:1281-1363) with PredictionMode::predict_inter (src/predict.rs:284-421) for a batch of
// luma blocks in one call.
//
// Per item (a block and its resolved mode list of up to 20 (reference pair, vectors) entries), ONE warp:
//   1. stages the source block in shared memory;
//   2. per entry: get_mv_params with PlaneSlice::clamp picks the (w+7) x (h+7) footprint, which is
//      staged; a single reference goes through mc_put_warp, a compound pair through mc_prep_warp twice
//      and mc_avg_warp (mc_dev.cuh); get_satd of the prediction against the staged source (warp_satd.cuh);
//      the lane whose index is the entry's keeps the value;
//   3. one shuffle pass ranks the entries: entry i's rank is the number of entries with a smaller SATD,
//      or an equal SATD and a smaller index (sort_by_key is stable).
// Predictions never leave shared memory.
//
// Items of every block size share a call and the host cannot see them, so a first kernel validates
// each item (invalid ones get their output rows there) and buckets the valid ones by size class (longest
// side <= 16, 32, 64) into context scratch.  Then one launch per class, with shared memory sized for the
// class's largest block, walks its bucket; the warps read the bucket's count on the device.  No host
// synchronisation anywhere.
#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"
#include "mc_dev.cuh"
#include "warp_satd.cuh"

namespace {

constexpr int kEntries = 20;   // ArrayVec<_, 20>, rdo.rs:1158
constexpr int kClasses = 3;    // longest side <= 16, 32, 64
constexpr int kBucketThreads = 256;
constexpr int kMaxWarps = 8;

// BlockSize (partition.rs:130-153) -> width, height; 0 for the 128-sided sizes
__constant__ uint8_t kBsW[22] = {4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 0, 0, 0, 4, 16, 8, 32, 16, 64};
__constant__ uint8_t kBsH[22] = {4, 8, 4, 8, 16, 8, 16, 32, 16, 32, 64, 32, 64, 0, 0, 0, 16, 4, 32, 8, 64, 16};

struct ScreenArgs {
  const void *src;                       // src pixel at the region's (0, 0)
  int src_stride;
  const void *ref[8];                    // pixel (0, 0) of each reference frame
  int ref_stride[8];
  int nrefs;
  int rect_x, rect_y, rect_w, rect_h;
  int x_lo, x_hi, y_lo, y_hi;            // PlaneSlice::clamp: [-xorigin, width] x [-yorigin, height]
  int mode, bit_depth;
  const b200_inter_screen_item *items;
  size_t n;
  uint32_t *satd;                        // n x 20 or NULL
  uint8_t *order;                        // n x 20 or NULL
  uint32_t *count;                       // [kClasses] valid items per class (scratch)
  uint32_t *bucket;                      // [kClasses][n] item indices (scratch)
  int smem_per_warp;
};

__device__ __forceinline__ bool item_valid(const b200_inter_screen_item &it, const ScreenArgs &a) {
  if (it.bsize >= 22 || kBsW[it.bsize] == 0 || it.n > kEntries) return false;
  if (it.x < 0 || it.y < 0 || it.x >= a.rect_w || it.y >= a.rect_h || (it.x & 3) || (it.y & 3)) return false;
  for (int k = 0; k < it.n; k++) {
    if (it.cands[k].ref[0] >= a.nrefs) return false;
    if (it.cands[k].ref[1] != 0xFF && it.cands[k].ref[1] >= a.nrefs) return false;
  }
  return true;
}

// Validate every item: invalid ones get UINT32_MAX and the identity order; valid ones go to their bucket
__global__ void __launch_bounds__(kBucketThreads) inter_screen_bucket_kernel(const __grid_constant__ ScreenArgs a) {
  const int lane = threadIdx.x & 31;
  for (size_t base = (size_t)blockIdx.x * blockDim.x; base < a.n; base += (size_t)gridDim.x * blockDim.x) {
    const size_t i = base + threadIdx.x;
    int cls = -1;
    if (i < a.n) {
      const b200_inter_screen_item &it = a.items[i];
      if (item_valid(it, a)) {
        const int side = max(kBsW[it.bsize], kBsH[it.bsize]);
        cls = side <= 16 ? 0 : side <= 32 ? 1 : 2;
      } else {
        for (int k = 0; k < kEntries; k++) {
          if (a.satd) a.satd[i * kEntries + k] = UINT32_MAX;
          if (a.order) a.order[i * kEntries + k] = (uint8_t)k;
        }
      }
    }
    // warp-aggregated append to the class buckets
#pragma unroll
    for (int c = 0; c < kClasses; c++) {
      const unsigned m = __ballot_sync(0xffffffffu, cls == c);
      if (!m) continue;
      const int leader = __ffs(m) - 1;
      uint32_t at = 0;
      if (lane == leader) at = atomicAdd(&a.count[c], (uint32_t)__popc(m));
      at = __shfl_sync(0xffffffffu, at, leader);
      if (cls == c) a.bucket[c * a.n + at + __popc(m & ((1u << lane) - 1))] = (uint32_t)i;
    }
  }
}

// Per-warp shared-memory layout for blocks up to S x S: footprint tile (the prediction aliases it once the
// last H pass has read it), transposed intermediate, two i16 preps, the source block.
constexpr size_t align16(size_t v) { return (v + 15) / 16 * 16; }

template <typename T, int S>
struct ScreenLayout {
  using ML = McLayout<T, S, S>;
  static constexpr size_t INTER_OFF = align16(ML::TILE_BYTES);
  static constexpr size_t TMP0_OFF = INTER_OFF + align16(ML::INTER_BYTES);
  static constexpr size_t TMP1_OFF = TMP0_OFF + (size_t)S * S * 2;
  static constexpr size_t SRC_OFF = TMP1_OFF + (size_t)S * S * 2;
  static constexpr size_t BYTES = align16(SRC_OFF + (size_t)S * S * sizeof(T));
};

// get_mv_params (predict.rs:284-297): rec_plane.slice(po + (mv >> 3) - 3).clamp().subslice(3, 3).  Returns
// the clamped slice's origin, where the staged footprint starts (the block's source pixel (-3, -3)).
// mv = row << 16 | col.
template <typename T>
__device__ __forceinline__ const T *footprint(const ScreenArgs &a, int r, int mv, int po_x, int po_y, int &row_frac,
                                              int &col_frac) {
  const int mv_row = (short)(mv >> 16), mv_col = (short)(mv & 0xffff);
  row_frac = (int)(((unsigned)mv_row << 1) & 0xf);
  col_frac = (int)(((unsigned)mv_col << 1) & 0xf);
  const int qx = min(max(po_x + (mv_col >> 3) - 3, a.x_lo), a.x_hi);
  const int qy = min(max(po_y + (mv_row >> 3) - 3, a.y_lo), a.y_hi);
  return (const T *)a.ref[r] + (long long)qy * a.ref_stride[r] + qx;
}

// One item at W x H: the whole list, then the rank pass and the outputs
template <typename T, int W, int H, int S>
__device__ __forceinline__ void screen_item(const ScreenArgs &a, unsigned char *base, uint32_t idx, int x, int y,
                                            int n, int lane) {
  using ML = McLayout<T, W, H>;
  using SL = ScreenLayout<T, S>;
  T *tile = (T *)base;
  T *pred = tile;  // written only after the last H pass of an entry has read the tile
  short *inter = (short *)(base + SL::INTER_OFF);
  short *tmp0 = (short *)(base + SL::TMP0_OFF), *tmp1 = (short *)(base + SL::TMP1_OFF);
  T *org = (T *)(base + SL::SRC_OFF);
  static_assert(ML::TILE_BYTES <= SL::INTER_OFF && ML::INTER_BYTES <= SL::TMP0_OFF - SL::INTER_OFF, "layout");
  const int xb = filter_bank(a.mode, W), yb = filter_bank(a.mode, H);

  // the entries: lane k holds entry k's descriptor
  const b200_inter_screen_cand *cands = a.items[idx].cands;
  int mv0 = 0, mv1 = 0, refs = 0xFFFF;  // mv = row << 16 | col (u16); refs = ref0 | ref1 << 8
  if (lane < n) {
    const b200_inter_screen_cand c = cands[lane];
    mv0 = (int)((uint32_t)(uint16_t)c.mv[0][0] << 16 | (uint16_t)c.mv[0][1]);
    mv1 = (int)((uint32_t)(uint16_t)c.mv[1][0] << 16 | (uint16_t)c.mv[1][1]);
    refs = c.ref[0] | c.ref[1] << 8;
  }

  __syncwarp();  // the previous item's readers are done with the source block
  const T *src = (const T *)a.src + (long long)y * a.src_stride + x;
  for (int i = lane; i < W * H; i += 32) org[i] = src[(long long)(i / W) * a.src_stride + (i % W)];

  const int po_x = a.rect_x + x, po_y = a.rect_y + y;  // tile_rect.to_frame_plane_offset

  uint32_t mine = UINT32_MAX;
  for (int e = 0; e < n; e++) {
    const int m0 = __shfl_sync(0xffffffffu, mv0, e), m1 = __shfl_sync(0xffffffffu, mv1, e);
    const int rr = __shfl_sync(0xffffffffu, refs, e);
    const int r0 = rr & 0xff, r1 = rr >> 8;
    int rf, cf;
    const T *fp = footprint<T>(a, r0, m0, po_x, po_y, rf, cf);
    __syncwarp();  // the previous entry's SATD is done with the prediction
    mc_stage_tile<T, W, H>(tile, fp, a.ref_stride[r0], lane);
    __syncwarp();
    if (r1 == 0xFF) {
      // predict_inter_single (predict.rs:304-336): put_8tap
      mc_put_warp<T, W, H>(tile, inter, pred, xb, cf, yb, rf, a.bit_depth, lane);
    } else {
      // predict_inter_compound (predict.rs:339-382): prep_8tap of each reference, then mc_avg
      mc_prep_warp<T, W, H>(tile, inter, tmp0, xb, cf, yb, rf, a.bit_depth, lane);
      fp = footprint<T>(a, r1, m1, po_x, po_y, rf, cf);
      mc_stage_tile<T, W, H>(tile, fp, a.ref_stride[r1], lane);  // the H pass above is done with the tile
      __syncwarp();
      mc_prep_warp<T, W, H>(tile, inter, tmp1, xb, cf, yb, rf, a.bit_depth, lane);
      __syncwarp();
      mc_avg_warp<T, W, H>(tmp0, tmp1, pred, a.bit_depth, lane);
    }
    __syncwarp();
    const uint32_t s = block_satd<T, W, H>(org, W, pred, lane);
    if (lane == e) mine = s;
  }

  // the stable sort (rdo.rs:1363 sort_by_key): entries past n hold UINT32_MAX and follow in index order
  int rank = 0;
#pragma unroll
  for (int j = 0; j < kEntries; j++) {
    const uint32_t v = __shfl_sync(0xffffffffu, mine, j);
    rank += (v < mine) || (v == mine && j < lane);
  }
  if (lane < kEntries) {
    if (a.satd) a.satd[(size_t)idx * kEntries + lane] = mine;
    if (a.order) a.order[(size_t)idx * kEntries + rank] = (uint8_t)lane;
  }
}

template <typename T, int CLS>
__global__ void __launch_bounds__(kMaxWarps * 32, 2) inter_screen_kernel(const __grid_constant__ ScreenArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int S = 16 << CLS;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  unsigned char *base = smem_raw + (size_t)wid * a.smem_per_warp;
  const uint32_t cnt = a.count[CLS];
  for (uint32_t k = blockIdx.x * nw + wid; k < cnt; k += gridDim.x * nw) {
    const uint32_t idx = a.bucket[CLS * a.n + k];
    const int x = a.items[idx].x, y = a.items[idx].y, n = a.items[idx].n;
    switch (a.items[idx].bsize) {
      // the sizes of this class, by BlockSize
#define B200_IS_IF(BS, W_, H_) \
  case BS:                     \
    if constexpr (((W_ > H_ ? W_ : H_) <= S) && ((W_ > H_ ? W_ : H_) > S / 2 || S == 16)) \
      screen_item<T, W_, H_, S>(a, base, idx, x, y, n, lane); \
    break;
      B200_IS_IF(0, 4, 4)
      B200_IS_IF(1, 4, 8)
      B200_IS_IF(2, 8, 4)
      B200_IS_IF(3, 8, 8)
      B200_IS_IF(4, 8, 16)
      B200_IS_IF(5, 16, 8)
      B200_IS_IF(6, 16, 16)
      B200_IS_IF(7, 16, 32)
      B200_IS_IF(8, 32, 16)
      B200_IS_IF(9, 32, 32)
      B200_IS_IF(10, 32, 64)
      B200_IS_IF(11, 64, 32)
      B200_IS_IF(12, 64, 64)
      B200_IS_IF(16, 4, 16)
      B200_IS_IF(17, 16, 4)
      B200_IS_IF(18, 8, 32)
      B200_IS_IF(19, 32, 8)
      B200_IS_IF(20, 16, 64)
      B200_IS_IF(21, 64, 16)
#undef B200_IS_IF
      default:
        break;
    }
  }
}

template <typename T, int CLS>
int launch_class(b200_ctx *ctx, ScreenArgs a) {
  constexpr int S = 16 << CLS;
  const size_t per_warp = ScreenLayout<T, S>::BYTES;
  const int wpc = (int)std::min<size_t>(kMaxWarps, std::max<size_t>(1, (200 * 1024) / per_warp));
  if (int st = b200_smem_opt_in(ctx, (const void *)inter_screen_kernel<T, CLS>, 200 * 1024)) return st;
  a.smem_per_warp = (int)per_warp;
  // the class's item count lives on the device: enough warps for every item up to a few waves
  const int grid = (int)std::min<size_t>((a.n + wpc - 1) / wpc, (size_t)ctx->num_sms * 8);
  inter_screen_kernel<T, CLS><<<grid, wpc * 32, per_warp * wpc, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

template <typename T>
int launch_all(b200_ctx *ctx, const ScreenArgs &a) {
  const int grid = (int)std::min<size_t>((a.n + kBucketThreads - 1) / kBucketThreads, (size_t)ctx->num_sms * 8);
  inter_screen_bucket_kernel<<<grid, kBucketThreads, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  if (int st = launch_class<T, 0>(ctx, a)) return st;
  if (int st = launch_class<T, 1>(ctx, a)) return st;
  return launch_class<T, 2>(ctx, a);
}

}  // namespace

extern "C" int b200_inter_mode_screen_dev(b200_ctx *ctx, const b200_plane *src, int rect_x, int rect_y, int rect_w,
                                          int rect_h, const b200_plane *refs, int nrefs, int xorigin, int yorigin,
                                          int filter_mode, int bit_depth, const b200_inter_screen_item *d_items,
                                          size_t nitems, uint32_t *d_satd, uint8_t *d_order) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, src && src->data && refs, "NULL plane");
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  B200_REQUIRE(ctx, src->bpp == (bit_depth == 8 ? 1 : 2), "bpp %d vs bit depth %d", src->bpp, bit_depth);
  B200_REQUIRE(ctx, nrefs >= 1 && nrefs <= 8, "nrefs %d outside 1..8", nrefs);
  B200_REQUIRE(ctx, xorigin >= 0 && yorigin >= 0, "negative origin (%d, %d)", xorigin, yorigin);
  const int ref_pad = std::max(std::max(xorigin, yorigin), 64 + 7);
  for (int r = 0; r < nrefs; r++) {
    B200_REQUIRE(ctx, refs[r].data, "NULL reference %d", r);
    B200_REQUIRE(ctx, refs[r].width == src->width && refs[r].height == src->height && refs[r].bpp == src->bpp,
                 "reference %d is %dx%d bpp %d, src %dx%d bpp %d", r, refs[r].width, refs[r].height, refs[r].bpp,
                 src->width, src->height, src->bpp);
    // the clamped footprint spans [-origin, size + 64 + 6]
    B200_REQUIRE(ctx, refs[r].pad >= ref_pad, "reference %d padding %d below %d", r, refs[r].pad, ref_pad);
  }
  B200_REQUIRE(ctx, rect_x >= 0 && rect_y >= 0 && rect_w > 0 && rect_h > 0 && rect_x + rect_w <= src->width &&
                        rect_y + rect_h <= src->height,
               "region (%d, %d, %d, %d) outside the %dx%d plane", rect_x, rect_y, rect_w, rect_h, src->width,
               src->height);
  B200_REQUIRE(ctx, filter_mode >= 0 && filter_mode <= 3, "bad FilterMode %d", filter_mode);
  B200_REQUIRE(ctx, src->pad >= 64, "src padding %d below 64", src->pad);
  B200_REQUIRE(ctx, d_satd || d_order, "both outputs are NULL");
  if (nitems == 0) return B200_OK;
  B200_REQUIRE(ctx, d_items != nullptr, "NULL items");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  if (int st = b200_reserve_dwork(ctx, 16 + (size_t)kClasses * nitems * 4)) return st;
  ScreenArgs a{};
  a.src = (const uint8_t *)src->data + ((long long)rect_y * src->stride + rect_x) * src->bpp;
  a.src_stride = src->stride;
  for (int r = 0; r < nrefs; r++) {
    a.ref[r] = refs[r].data;
    a.ref_stride[r] = refs[r].stride;
  }
  a.nrefs = nrefs;
  a.rect_x = rect_x, a.rect_y = rect_y, a.rect_w = rect_w, a.rect_h = rect_h;
  a.x_lo = -xorigin, a.x_hi = src->width, a.y_lo = -yorigin, a.y_hi = src->height;
  a.mode = filter_mode;
  a.bit_depth = bit_depth;
  a.items = d_items;
  a.n = nitems;
  a.satd = d_satd;
  a.order = d_order;
  a.count = (uint32_t *)ctx->dwork;
  a.bucket = (uint32_t *)((uint8_t *)ctx->dwork + 16);
  B200_CUDA(ctx, cudaMemsetAsync(a.count, 0, kClasses * sizeof(uint32_t), ctx->stream));
  return src->bpp == 1 ? launch_all<uint8_t>(ctx, a) : launch_all<uint16_t>(ctx, a);
}
