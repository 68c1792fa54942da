// subpel_rdo.cu — sub-pel refinement fused with the winner's residual and forward transform (sm_90a):
// BASELINE configs[3] "speed-2 inter RDO (mc subpel + SATD + fwd-txfm fused)".
//
//   get_subpel_mv_rd           src/me.rs:1411-1442   (per candidate: predict_inter_single -> compute_mv_rd)
//   predict_inter_single       src/predict.rs:304-336 -> put_8tap, src/mc.rs:250-353
//   get_sad / get_satd         src/dist.rs:31-52, :156-221
//   compute_mv_rd, get_mv_rate src/me.rs:1445-1461, :1512-1523
//   diff + forward_transform   src/encoder.rs:1533-1544, src/transform/forward.rs:71-161
//
// The two-launch form (b200_me_subpel_candidates_dev: mc kernel -> packed predictions in HBM ->
// distortion kernel) writes and re-reads w*h pixels per candidate.  Here ONE warp owns a block and walks
// its candidates: the (w+7) x (h+7) source footprint is staged in shared memory, the 8-tap prediction is
// formed in shared memory (the reference's four cases incl. the double-rounded H-only path and the i16
// intermediate), measured against the source block where it sits - SAD by lanes striding the pixels,
// SATD with 8 lanes per 8x8 chunk (lane = row: horizontal butterflies in registers, vertical ones by
// shfl.xor), or a lane per 4x4 chunk when a side is 4 - and the best prediction so far is kept by swapping
// two shared buffers.  When the list is exhausted the winner's prediction is still on chip: its residual
// goes straight through the column / row passes of the forward transform (thread per column, padded
// transposition tile, thread per row; the reference's 32x32-chunked store when a side is 64).
// Nothing but the source footprints is read from HBM and nothing but results is written.
// Every AV1 block size 4x4 .. 64x64 is an instantiation of the same warp-per-block kernel.
#include <cuda_runtime.h>

#include <algorithm>

#include "fwd_txfm_dev.cuh"
#include "subpel_dev.cuh"

namespace {

struct SrdoArgs {
  const void *cur, *ref;
  int cur_stride, ref_stride;
  const b200_block *blocks;
  const b200_cand *cands;
  const uint32_t *cand_offsets;
  const short *pmv;
  const b200_me_result *start;  // non-NULL: subpel_diamond_search from this result instead of a list
  size_t nblocks;
  int w_in_b, h_in_b;
  uint32_t lambda;
  int allow_hp, use_satd, mode, bit_depth;
  uint32_t *out_sad;
  unsigned long long *out_cost;
  b200_me_result *out_best;
  int tx_on;
  TxSetup tx;
  void *out_coef;
  int smem_per_warp, pred_off;  // bytes: a warp's slice, and where its two prediction buffers start
};

template <typename T, int W, int H>
__global__ void __launch_bounds__(256) subpel_rdo_kernel(const __grid_constant__ SrdoArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using CoefT = typename std::conditional<sizeof(T) == 1, int16_t, int32_t>::type;
  using ML = McLayout<T, W, H>;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  unsigned char *base = smem_raw + (size_t)wid * a.smem_per_warp;
  T *tile = (T *)base;                                  // [H+7][W+8] source footprint
  short *inter = (short *)(base + ML::TILE_BYTES);      // [W][H+8] transposed i16 intermediate
  T *pred0 = (T *)(base + a.pred_off);                  // two W x H predictions: current / best so far
  T *pred1 = pred0 + W * H;
  int *txtile = (int *)base;                            // aliases tile + inter once the list is done
  const int xb = filter_bank(a.mode, W), yb = filter_bank(a.mode, H);

  for (size_t blk = (size_t)blockIdx.x * nw + wid; blk < a.nblocks; blk += (size_t)gridDim.x * nw) {
    const b200_block b = a.blocks[blk];
    const uint32_t lo = a.start ? 0u : a.cand_offsets[blk], hi = a.start ? 0u : a.cand_offsets[blk + 1];
    const T *org = (const T *)a.cur + (long long)b.y * a.cur_stride + b.x;
    const SubpelBlock<T, W, H> sp{org, a.cur_stride, (const T *)a.ref, a.ref_stride, b.x, b.y,
                                  b200_mv_range(a.w_in_b, a.h_in_b, b.x / MI_SIZE, b.y / MI_SIZE, W, H),
                                  load_pmv(a.pmv, blk), a.lambda, a.allow_hp, a.use_satd, a.bit_depth, xb, yb, tile,
                                  inter};
    T *pcur = pred0, *pbest = pred1;
    unsigned long long best_cost = kEmptyCost;
    uint32_t best_sad = kEmptySad;
    int best_row = 0, best_col = 0;
    auto eval = [&](int mv_row, int mv_col, uint32_t &sad) { return sp.rd(mv_row, mv_col, pcur, sad, lane); };
    if (a.start) {
      // ---- subpel_diamond_search, me.rs:1311-1383 (subpel_dev.cuh)
      const b200_me_result st = a.start[blk];
      best_cost = st.cost, best_sad = st.sad, best_row = st.mv_row, best_col = st.mv_col;
      sp.diamond(best_cost, best_sad, best_row, best_col, pcur, lane);
      if (a.tx_on && best_cost != kEmptyCost) {  // the winner's prediction for the transform below
        uint32_t sad;
        (void)eval(best_row, best_col, sad);
        T *t = pcur;
        pcur = pbest;
        pbest = t;
      }
    } else {
      for (uint32_t i = lo; i < hi; i++) {
        const b200_cand c = a.cands[i];
        uint32_t sad;
        const unsigned long long cost = eval(c.mv_row, c.mv_col, sad);
        if (cost < best_cost) {  // strict: the first minimum in list order wins (me.rs:1360-1365)
          best_cost = cost;
          best_sad = sad;
          best_row = c.mv_row;
          best_col = c.mv_col;
          T *t = pcur;
          pcur = pbest;
          pbest = t;
        }
        if (lane == 0) {
          if (a.out_sad) a.out_sad[i] = sad;
          if (a.out_cost) a.out_cost[i] = cost;
        }
      }
    }
    if (lane == 0 && a.out_best) {
      b200_me_result res;
      res.cost = best_cost;
      res.sad = best_sad;
      res.mv_row = (int16_t)best_row;
      res.mv_col = (int16_t)best_col;
      a.out_best[blk] = res;
    }
    if (a.tx_on) {
      // ---- residual of the winner's prediction -> forward transform (forward.rs:94-160)
      constexpr int PITCH = W + 1;
      CoefT *dst = (CoefT *)a.out_coef + blk * (size_t)(W * H);
      __syncwarp();
      if (best_cost == kEmptyCost) {
        for (int k = lane; k < W * H; k += 32) dst[k] = 0;
      } else {
        for (int t = lane; t < W; t += 32) {
          TXV c[H];
#pragma unroll
          for (int r = 0; r < H; r++) {
            const int rr = a.tx.ud_flip ? H - 1 - r : r;
            c[r] = round_shift_bit((int)org[(long long)rr * a.cur_stride + t] - (int)pbest[rr * W + t], a.tx.bit0);
          }
          run_1d<H>(a.tx.col_type, c);
          const int cc = a.tx.lr_flip ? W - 1 - t : t;
#pragma unroll
          for (int r = 0; r < H; r++) txtile[r * PITCH + cc] = round_shift_bit(c[r], a.tx.bit1);
        }
        __syncwarp();
        for (int t = lane; t < H; t += 32) {
          TXV c[W];
#pragma unroll
          for (int k = 0; k < W; k++) c[k] = txtile[t * PITCH + k];
          run_1d<W>(a.tx.row_type, c);
          if constexpr (W == 64 || H == 64) {
            CoefT *d = dst + CoefOrder<W, H>::row(t);  // the reference's 32x32-chunked order
#pragma unroll
            for (int k = 0; k < W; k++) d[CoefOrder<W, H>::col(k)] = (CoefT)round_shift_bit(c[k], a.tx.bit2);
          } else {
            // the same order: t < H <= 32 here, written as the plain transpose it reduces to
#pragma unroll
            for (int k = 0; k < W; k++) dst[k * H + t] = (CoefT)round_shift_bit(c[k], a.tx.bit2);
          }
        }
      }
      __syncwarp();
    }
  }
}

template <typename T, int W, int H>
int launch_srdo(b200_ctx *ctx, SrdoArgs a) {
  using ML = McLayout<T, W, H>;
  const size_t mc_bytes = b200_align_up(ML::TILE_BYTES, 4) + ML::INTER_BYTES;
  const size_t tx_bytes = (size_t)H * (W + 1) * 4;  // aliases the MC buffers
  // the predictions sit behind whichever of the two is larger
  const size_t pred_off = b200_align_up(std::max(mc_bytes, tx_bytes), 16);
  const size_t per_warp = b200_align_up(pred_off + 2 * (size_t)W * H * sizeof(T), 16);
  const int wpc = (int)std::min<size_t>(8, std::max<size_t>(1, (160 * 1024) / per_warp));
  const size_t smem = per_warp * wpc;
  if (int st = b200_smem_opt_in(ctx, (const void *)subpel_rdo_kernel<T, W, H>, 200 * 1024)) return st;
  a.smem_per_warp = (int)per_warp;
  a.pred_off = (int)pred_off;
  const int grid = (int)std::min<size_t>((a.nblocks + wpc - 1) / wpc, (size_t)ctx->num_sms * 16);
  subpel_rdo_kernel<T, W, H><<<grid, wpc * 32, smem, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

}  // namespace

static int subpel_rdo_impl(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref, const b200_block *d_blocks,
                           size_t nblocks, const b200_cand *d_cands, size_t ncands, const uint32_t *d_cand_offsets,
                           const b200_me_result *d_start, const int16_t *d_pmv, const b200_me_params *p,
                           int filter_mode, int tx_size, int tx_type, uint32_t *d_sad, uint64_t *d_cost,
                           b200_me_result *d_best, void *d_coeffs) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && ref && p && cur->data && ref->data, "NULL plane / params");
  B200_REQUIRE(ctx, cur->bpp == ref->bpp && (cur->bpp == 1 || cur->bpp == 2), "planes must share bpp (1 or 2)");
  B200_REQUIRE(ctx, (cur->bpp == 1) == (p->bit_depth == 8) && (p->bit_depth == 8 || p->bit_depth == 10 || p->bit_depth == 12),
               "bpp %d vs bit depth %d", cur->bpp, p->bit_depth);
  int bsize = -1;  // the block sizes are the 19 transform sizes: 4x4 .. 64x64
  for (int s = 0; s < 19; s++)
    if (kTxW[s] == p->w && kTxH[s] == p->h) bsize = s;
  B200_REQUIRE(ctx, bsize >= 0, "fused sub-pel RDO serves the AV1 block sizes 4x4 .. 64x64 (got %dx%d)", p->w, p->h);
  B200_REQUIRE(ctx, filter_mode >= 0 && filter_mode <= 3, "bad FilterMode %d", filter_mode);
  B200_REQUIRE(ctx, d_start != nullptr || d_cand_offsets != nullptr, "candidates must be grouped by block (CSR d_cand_offsets)");
  B200_REQUIRE(ctx, tx_size < 0 || (valid_transform(tx_size, tx_type) && kTxW[tx_size] == p->w && kTxH[tx_size] == p->h),
               "transform %d/%d does not match the %dx%d blocks", tx_size, tx_type, p->w, p->h);
  B200_REQUIRE(ctx, tx_size < 0 || d_coeffs, "transform requested without an output buffer");
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && (d_start || d_cands || ncands == 0), "NULL blocks / candidates");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  SrdoArgs a{};
  a.cur = cur->data, a.ref = ref->data;
  a.cur_stride = cur->stride, a.ref_stride = ref->stride;
  a.blocks = d_blocks;
  a.cands = d_cands;
  a.cand_offsets = d_cand_offsets;
  a.start = d_start;
  a.pmv = d_pmv;
  a.nblocks = nblocks;
  a.w_in_b = p->frame_w_in_b, a.h_in_b = p->frame_h_in_b;
  a.lambda = p->lambda;
  a.allow_hp = p->allow_high_precision_mv;
  a.use_satd = p->use_satd;
  a.mode = filter_mode;
  a.bit_depth = p->bit_depth;
  a.out_sad = d_sad;
  a.out_cost = (unsigned long long *)d_cost;
  a.out_best = d_best;
  a.tx_on = tx_size >= 0;
  if (a.tx_on) a.tx = tx_setup(tx_size, tx_type, p->bit_depth);
  a.out_coef = d_coeffs;
  switch (bsize) {
#define B200_SRDO(ID, W_, H_) \
  case ID:                    \
    return cur->bpp == 1 ? launch_srdo<uint8_t, W_, H_>(ctx, a) : launch_srdo<uint16_t, W_, H_>(ctx, a);
    B200_SRDO(0, 4, 4)
    B200_SRDO(1, 8, 8)
    B200_SRDO(2, 16, 16)
    B200_SRDO(3, 32, 32)
    B200_SRDO(4, 64, 64)
    B200_SRDO(5, 4, 8)
    B200_SRDO(6, 8, 4)
    B200_SRDO(7, 8, 16)
    B200_SRDO(8, 16, 8)
    B200_SRDO(9, 16, 32)
    B200_SRDO(10, 32, 16)
    B200_SRDO(11, 32, 64)
    B200_SRDO(12, 64, 32)
    B200_SRDO(13, 4, 16)
    B200_SRDO(14, 16, 4)
    B200_SRDO(15, 8, 32)
    B200_SRDO(16, 32, 8)
    B200_SRDO(17, 16, 64)
    B200_SRDO(18, 64, 16)
#undef B200_SRDO
  }
  return b200_fail(ctx, B200_ERR_ARG, "unreachable block size");
}

extern "C" int b200_subpel_rdo_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                   const b200_block *d_blocks, size_t nblocks, const b200_cand *d_cands,
                                   size_t ncands, const uint32_t *d_cand_offsets, const int16_t *d_pmv,
                                   const b200_me_params *p, int filter_mode, int tx_size, int tx_type,
                                   uint32_t *d_sad, uint64_t *d_cost, b200_me_result *d_best, void *d_coeffs) {
  B200_REQUIRE(ctx, ctx != nullptr && d_cand_offsets != nullptr, "NULL ctx / candidates must be grouped by block (CSR)");
  return subpel_rdo_impl(ctx, cur, ref, d_blocks, nblocks, d_cands, ncands, d_cand_offsets, nullptr, d_pmv, p,
                         filter_mode, tx_size, tx_type, d_sad, d_cost, d_best, d_coeffs);
}

extern "C" int b200_subpel_search_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                      const b200_block *d_blocks, size_t nblocks, const b200_me_result *d_start,
                                      const int16_t *d_pmv, const b200_me_params *p, int filter_mode, int tx_size,
                                      int tx_type, b200_me_result *d_best, void *d_coeffs) {
  B200_REQUIRE(ctx, ctx != nullptr && d_start != nullptr && d_best != nullptr, "NULL ctx / start results / output");
  return subpel_rdo_impl(ctx, cur, ref, d_blocks, nblocks, nullptr, 0, nullptr, d_start, d_pmv, p, filter_mode, tx_size,
                         tx_type, nullptr, nullptr, d_best, d_coeffs);
}
