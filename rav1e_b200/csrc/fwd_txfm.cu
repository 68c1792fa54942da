// fwd_txfm.cu — batched 2-D forward transforms (rav1e src/transform/forward.rs:71-161) for sm_90a.
//
// One thread owns one whole column (pass 1) and then one whole row (pass 2) of a block in
// registers and runs the straight-line lifting network on it (txfm_networks.cuh); the
// transposition between the passes goes through a padded shared-memory tile, so both the
// int16 residual loads and the coefficient stores (the reference's transposed, 32x32-chunked
// order, forward.rs:135-159) are coalesced.  A CTA of 128 threads carries 128/max(W,H) blocks
// at a time.  Warp shuffles are deliberately NOT used for the butterflies: the Daala networks
// are irregular lifting ladders with per-node constants, so a lane-per-coefficient layout
// would diverge on every step, while a thread-per-vector layout needs no communication at all
// inside a 1-D pass.
#include "fwd_txfm_dev.cuh"
#include "host_stage.cuh"

namespace {

// Several (cur, ref) plane pairs per launch (see b200_me_candidates_multi_dev): pair k owns
// blocks [block_end[k-1], block_end[k]) of the launch.
constexpr int kTxMaxPairs = 32;
struct TxPairs {
  int n;  // <= 1: TxArgs::cur / ref
  uint32_t block_end[kTxMaxPairs];
  const void *cur[kTxMaxPairs], *ref[kTxMaxPairs];
  int cur_stride[kTxMaxPairs], ref_stride[kTxMaxPairs];
};

struct TxArgs {
  // fused residual source (PLANES variants): cur - ref displaced by the full-pel winner mv
  const void *cur, *ref;
  int cur_stride, ref_stride;
  TxPairs pr;
  const b200_block *blocks;
  const b200_me_result *mv_src;
  const void *pred_packed;  // PLANES variants: prediction given as packed W x H blocks instead of a plane
  const int16_t *in;
  void *out;
  size_t n;
  size_t in_block_stride;  // elements between consecutive blocks
  int in_row_stride;       // elements between rows of a block
  int col_type, row_type;
  int ud_flip, lr_flip;
  int bit0, bit1, bit2;    // av1_round_shift_array `bit` = -shift[k]: >0 round-shift right, <0 left
};

constexpr int kTxThreads = 128;

template <int W, int H, typename CoefT, bool PLANES>
__global__ void __launch_bounds__(kTxThreads) fwd_txfm_kernel(const __grid_constant__ TxArgs a) {
  constexpr int T = W > H ? W : H;       // threads per block-transform
  constexpr int PER = kTxThreads / T;    // transforms in flight per CTA
  constexpr int PITCH = W + 1;           // padded row pitch: conflict-free transposition
  constexpr int REGION = H * PITCH + ((H * PITCH) % 2 == 0 ? 1 : 0);
  __shared__ int buf[PER * REGION];
  const int slot = threadIdx.x / T, t = threadIdx.x - slot * T;
  int *tile = buf + slot * REGION;
  const size_t stride_blk = (size_t)gridDim.x * PER;
  for (size_t base = (size_t)blockIdx.x * PER; base < a.n; base += stride_blk) {
    const size_t blk = base + slot;
    const bool valid = blk < a.n;
    // ---- columns (forward.rs:95-126)
    if (valid && t < W) {
      TXV c[H];
      if constexpr (PLANES) {
        // residual computed on the fly (encoder.rs:1533 `diff`): u8 planes pair with i16
        // coefficients, u16 planes with i32 (T::Coeff)
        using Px = typename std::conditional<sizeof(CoefT) == 2, uint8_t, uint16_t>::type;
        const b200_block b = a.blocks[blk];
        int dx = 0, dy = 0;
        if (a.mv_src && a.mv_src[blk].cost != ~0ull) {
          dx = a.mv_src[blk].mv_col / 8;
          dy = a.mv_src[blk].mv_row / 8;
        }
        const void *cur_p = a.cur, *ref_p = a.ref;
        int cur_stride = a.cur_stride, ref_stride = a.ref_stride;
        if (a.pr.n > 1) {  // first pair whose block range holds blk
          int lo = 0, hi = a.pr.n - 1;
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if ((uint32_t)blk < a.pr.block_end[mid])
              hi = mid;
            else
              lo = mid + 1;
          }
          cur_p = a.pr.cur[lo], ref_p = a.pr.ref[lo];
          cur_stride = a.pr.cur_stride[lo], ref_stride = a.pr.ref_stride[lo];
        }
        const Px *pc = (const Px *)cur_p + (long long)b.y * cur_stride + b.x + t;
        const Px *pr;
        long long rstride;
        if (a.pred_packed) {
          pr = (const Px *)a.pred_packed + blk * (size_t)(W * H) + t;
          rstride = W;
        } else {
          pr = (const Px *)ref_p + (long long)(b.y + dy) * ref_stride + b.x + dx + t;
          rstride = ref_stride;
        }
#pragma unroll
        for (int r = 0; r < H; r++) {
          const int rr = a.ud_flip ? H - 1 - r : r;
          c[r] = round_shift_bit((int)pc[(long long)rr * cur_stride] - (int)pr[rr * rstride], a.bit0);
        }
      } else {
        const int16_t *src = a.in + blk * a.in_block_stride + t;
#pragma unroll
        for (int r = 0; r < H; r++) {
          const int rr = a.ud_flip ? H - 1 - r : r;
          c[r] = round_shift_bit((int)src[(size_t)rr * a.in_row_stride], a.bit0);
        }
      }
      run_1d<H>(a.col_type, c);
      const int cc = a.lr_flip ? W - 1 - t : t;
#pragma unroll
      for (int r = 0; r < H; r++) tile[r * PITCH + cc] = round_shift_bit(c[r], a.bit1);
    }
    __syncthreads();
    // ---- rows (forward.rs:131-160)
    if (valid && t < H) {
      TXV c[W];
#pragma unroll
      for (int k = 0; k < W; k++) c[k] = tile[t * PITCH + k];
      run_1d<W>(a.row_type, c);
      constexpr int HS = H < 32 ? H : 32, WC = W < 32 ? W : 32;
      CoefT *dst = (CoefT *)a.out + blk * (size_t)(W * H) + (t >= 32 ? HS * WC : 0) + (t & 31);
#pragma unroll
      for (int k = 0; k < W; k++)
        dst[(size_t)H * 32 * (k >= 32) + (k & 31) * HS] = (CoefT)round_shift_bit(c[k], a.bit2);
    }
    __syncthreads();
  }
}

template <int W, int H>
int launch_txfm(b200_ctx *ctx, const TxArgs &a, int coeff_is_i32) {
  constexpr int T = W > H ? W : H;
  constexpr int PER = kTxThreads / T;
  const size_t ctas = (a.n + PER - 1) / PER;
  const int grid = (int)std::min<size_t>(ctas, (size_t)ctx->num_sms * 32);
  if (a.cur) {
    if (coeff_is_i32)
      fwd_txfm_kernel<W, H, int32_t, true><<<grid, kTxThreads, 0, ctx->stream>>>(a);
    else
      fwd_txfm_kernel<W, H, int16_t, true><<<grid, kTxThreads, 0, ctx->stream>>>(a);
  } else if (coeff_is_i32) {
    fwd_txfm_kernel<W, H, int32_t, false><<<grid, kTxThreads, 0, ctx->stream>>>(a);
  } else {
    fwd_txfm_kernel<W, H, int16_t, false><<<grid, kTxThreads, 0, ctx->stream>>>(a);
  }
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

}  // namespace

extern "C" int b200_valid_av1_transform(int tx_size, int tx_type) {
  return valid_transform(tx_size, tx_type) ? 1 : 0;
}
extern "C" int b200_tx_width(int tx_size) { return tx_size >= 0 && tx_size < 19 ? kTxW[tx_size] : 0; }
extern "C" int b200_tx_height(int tx_size) { return tx_size >= 0 && tx_size < 19 ? kTxH[tx_size] : 0; }

static int fwd_txfm_impl(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                         const TxPairs *pairs, const void *d_pred_packed, const b200_block *d_blocks,
                         const b200_me_result *d_mv_src,
                         const int16_t *d_input, size_t in_block_stride, size_t in_row_stride,
                         void *d_output, size_t nblocks, int tx_size, int tx_type, int bd,
                         int coeff_is_i32) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  // forward.rs:75: assert!(valid_av1_transform(tx_size, tx_type))
  B200_REQUIRE(ctx, valid_transform(tx_size, tx_type), "invalid transform: tx_size %d tx_type %d",
               tx_size, tx_type);
  B200_REQUIRE(ctx, bd == 8 || bd == 10 || bd == 12, "bit depth %d not in {8,10,12}", bd);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, (d_input || cur) && d_output, "NULL input/output");
  const int w = kTxW[tx_size], h = kTxH[tx_size];
  B200_REQUIRE(ctx, cur || in_row_stride >= (size_t)w, "row stride %zu < width %d", in_row_stride, w);
  (void)h;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const TxSetup ts = tx_setup(tx_size, tx_type, bd);
  TxArgs a;
  a.cur = cur ? cur->data : nullptr;
  a.ref = ref ? ref->data : nullptr;
  a.cur_stride = cur ? cur->stride : 0;
  a.ref_stride = ref ? ref->stride : 0;
  if (pairs)
    a.pr = *pairs;
  else
    a.pr.n = 0;
  a.blocks = d_blocks;
  a.mv_src = d_mv_src;
  a.pred_packed = d_pred_packed;
  a.in = d_input;
  a.out = d_output;
  a.n = nblocks;
  a.in_block_stride = in_block_stride;
  a.in_row_stride = (int)in_row_stride;
  a.col_type = ts.col_type;
  a.row_type = ts.row_type;
  a.ud_flip = ts.ud_flip;
  a.lr_flip = ts.lr_flip;
  a.bit0 = ts.bit0;
  a.bit1 = ts.bit1;
  a.bit2 = ts.bit2;
  switch (tx_size) {
#define B200_TX(ID, W_, H_) \
  case ID:                  \
    return launch_txfm<W_, H_>(ctx, a, coeff_is_i32);
    B200_TX(0, 4, 4)
    B200_TX(1, 8, 8)
    B200_TX(2, 16, 16)
    B200_TX(3, 32, 32)
    B200_TX(4, 64, 64)
    B200_TX(5, 4, 8)
    B200_TX(6, 8, 4)
    B200_TX(7, 8, 16)
    B200_TX(8, 16, 8)
    B200_TX(9, 16, 32)
    B200_TX(10, 32, 16)
    B200_TX(11, 32, 64)
    B200_TX(12, 64, 32)
    B200_TX(13, 4, 16)
    B200_TX(14, 16, 4)
    B200_TX(15, 8, 32)
    B200_TX(16, 32, 8)
    B200_TX(17, 16, 64)
    B200_TX(18, 64, 16)
#undef B200_TX
  }
  return b200_fail(ctx, B200_ERR_ARG, "unreachable tx_size %d", tx_size);
}

extern "C" int b200_fwd_txfm_dev(b200_ctx *ctx, const int16_t *d_input, size_t in_block_stride,
                                 size_t in_row_stride, void *d_output, size_t nblocks, int tx_size,
                                 int tx_type, int bd, int coeff_is_i32) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, d_input || nblocks == 0, "NULL input");
  return fwd_txfm_impl(ctx, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, d_input, in_block_stride,
                       in_row_stride, d_output, nblocks, tx_size, tx_type, bd, coeff_is_i32);
}

// Fused `diff` + forward transform (encoder.rs:1533-1544): residual of each block against the
// reference displaced by the full-pel part of d_mv_src (NULL = zero motion), transformed without
// a round trip of the residual through HBM.  u8 planes give i16 coefficients, u16 planes i32.
extern "C" int b200_fwd_txfm_residual_dev(b200_ctx *ctx, const b200_plane *cur,
                                          const b200_plane *ref, const b200_block *d_blocks,
                                          size_t nblocks, const b200_me_result *d_mv_src,
                                          void *d_output, int tx_size, int tx_type, int bd) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && ref && cur->data && ref->data && cur->bpp == ref->bpp, "bad planes");
  B200_REQUIRE(ctx, (cur->bpp == 1) == (bd == 8), "bpp %d does not match bit depth %d", cur->bpp, bd);
  B200_REQUIRE(ctx, d_blocks || nblocks == 0, "NULL blocks");
  return fwd_txfm_impl(ctx, cur, ref, nullptr, nullptr, d_blocks, d_mv_src, nullptr, 0, 0, d_output,
                       nblocks, tx_size, tx_type, bd, cur->bpp == 2);
}

// The fused residual + transform over several plane pairs in one launch (block ranges as in
// b200_me_candidates_multi_dev; d_mv_src / d_output follow the concatenated block order).
extern "C" int b200_fwd_txfm_residual_multi_dev(b200_ctx *ctx, size_t npairs, const b200_plane *curs,
                                                const b200_plane *refs, const uint32_t *pair_block_end,
                                                const b200_block *d_blocks, size_t nblocks,
                                                const b200_me_result *d_mv_src, void *d_output,
                                                int tx_size, int tx_type, int bd) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, npairs >= 1 && curs && refs && pair_block_end, "NULL plane pair table");
  B200_REQUIRE(ctx, valid_transform(tx_size, tx_type), "invalid transform: tx_size %d tx_type %d",
               tx_size, tx_type);
  B200_REQUIRE(ctx, d_blocks || nblocks == 0, "NULL blocks");
  B200_REQUIRE(ctx, pair_block_end[npairs - 1] == nblocks && nblocks < (1ull << 32),
               "last pair must end at nblocks");
  for (size_t k = 0; k < npairs; k++) {
    B200_REQUIRE(ctx, curs[k].data && refs[k].data && curs[k].bpp == refs[k].bpp &&
                          curs[k].bpp == curs[0].bpp, "pair %zu: bad planes", k);
    B200_REQUIRE(ctx, pair_block_end[k] >= (k ? pair_block_end[k - 1] : 0),
                 "pair %zu: block ends must be non-decreasing", k);
  }
  B200_REQUIRE(ctx, (curs[0].bpp == 1) == (bd == 8), "bpp %d does not match bit depth %d", curs[0].bpp, bd);
  const size_t coef_bytes = (size_t)kTxW[tx_size] * kTxH[tx_size] * (curs[0].bpp == 2 ? 4 : 2);
  for (size_t k0 = 0; k0 < npairs; k0 += kTxMaxPairs) {
    const int n = (int)std::min<size_t>(kTxMaxPairs, npairs - k0);
    const uint32_t b0 = k0 ? pair_block_end[k0 - 1] : 0;
    TxPairs t;
    t.n = n;
    for (int k = 0; k < n; k++) {
      t.block_end[k] = pair_block_end[k0 + k] - b0;
      t.cur[k] = curs[k0 + k].data;
      t.ref[k] = refs[k0 + k].data;
      t.cur_stride[k] = curs[k0 + k].stride;
      t.ref_stride[k] = refs[k0 + k].stride;
    }
    const size_t nb = t.block_end[n - 1];
    if (nb == 0) continue;
    if (int st = fwd_txfm_impl(ctx, &curs[k0], &refs[k0], &t, nullptr, d_blocks + b0,
                               d_mv_src ? d_mv_src + b0 : nullptr, nullptr, 0, 0,
                               (uint8_t *)d_output + (size_t)b0 * coef_bytes, nb, tx_size, tx_type, bd,
                               curs[0].bpp == 2))
      return st;
  }
  return B200_OK;
}

// Residual against PACKED predictions (the output layout of b200_mc_blocks_dev /
// b200_predict_intra_dev): block i = cur(d_blocks[i]) - d_pred[i], then the forward transform.
// This is encode_tx_block's predict -> diff -> forward_transform chain (encoder.rs:1492-1544)
// for sub-pel inter or intra predictions.
extern "C" int b200_fwd_txfm_pred_dev(b200_ctx *ctx, const b200_plane *cur, const void *d_pred,
                                      const b200_block *d_blocks, size_t nblocks, void *d_output,
                                      int tx_size, int tx_type, int bd) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && cur->data && d_pred, "bad plane / prediction");
  B200_REQUIRE(ctx, (cur->bpp == 1) == (bd == 8), "bpp %d does not match bit depth %d", cur->bpp, bd);
  B200_REQUIRE(ctx, d_blocks || nblocks == 0, "NULL blocks");
  return fwd_txfm_impl(ctx, cur, cur, nullptr, d_pred, d_blocks, nullptr, nullptr, 0, 0, d_output, nblocks,
                       tx_size, tx_type, bd, cur->bpp == 2);
}

// Host-buffer form: packed residual blocks in, coefficients out.
extern "C" int b200_fwd_txfm_batch(b200_ctx *ctx, const int16_t *input, size_t in_block_stride,
                                   size_t in_row_stride, void *output, size_t nblocks, int tx_size,
                                   int tx_type, int bd, int coeff_is_i32) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, valid_transform(tx_size, tx_type), "invalid transform: tx_size %d tx_type %d",
               tx_size, tx_type);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, input && output, "NULL input/output");
  const int w = kTxW[tx_size], h = kTxH[tx_size];
  const size_t in_elems = (nblocks - 1) * in_block_stride + (size_t)(h - 1) * in_row_stride + w;
  const size_t out_bytes = nblocks * (size_t)w * h * (coeff_is_i32 ? 4 : 2);
  HostStage s(ctx, b200_align_up(in_elems * 2, 256) + out_bytes);
  int16_t *d_in = (int16_t *)s.take(in_elems * 2);
  uint8_t *d_out = s.take(out_bytes);
  s.up(d_in, input, in_elems * 2);
  if (s.ok())
    s.run(b200_fwd_txfm_dev(ctx, d_in, in_block_stride, in_row_stride, d_out, nblocks, tx_size, tx_type, bd,
                            coeff_is_i32));
  s.down(output, d_out, out_bytes);
  return s.finish(!ctx->async_batch);
}

extern "C" int b200_fwd_txfm_residual_resident(b200_ctx *ctx, const b200_plane *cur,
                                               const b200_plane *ref, const b200_block *blocks,
                                               size_t nblocks, const b200_me_result *mv_src,
                                               void *output, int tx_size, int tx_type, int bd) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, valid_transform(tx_size, tx_type), "invalid transform: tx_size %d tx_type %d",
               tx_size, tx_type);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, cur && ref && blocks && output, "NULL argument");
  const size_t area = (size_t)kTxW[tx_size] * kTxH[tx_size];
  const size_t out_bytes = nblocks * area * (cur->bpp == 2 ? 4 : 2);
  const size_t blk_bytes = b200_align_up(nblocks * sizeof(b200_block), 256);
  const size_t mv_bytes = mv_src ? b200_align_up(nblocks * sizeof(b200_me_result), 256) : 0;
  HostStage s(ctx, blk_bytes + mv_bytes + out_bytes);
  b200_block *d_blk = (b200_block *)s.take(nblocks * sizeof(b200_block));
  b200_me_result *d_mv = mv_src ? (b200_me_result *)s.take(nblocks * sizeof(b200_me_result)) : nullptr;
  uint8_t *d_out = s.take(out_bytes);
  s.up(d_blk, blocks, nblocks * sizeof(b200_block));
  if (mv_src) s.up(d_mv, mv_src, nblocks * sizeof(b200_me_result));
  if (s.ok()) s.run(b200_fwd_txfm_residual_dev(ctx, cur, ref, d_blk, nblocks, d_mv, d_out, tx_size, tx_type, bd));
  s.down(output, d_out, out_bytes);
  return s.finish(!ctx->async_batch);
}

// Per-call form with the reference's signature (asm/x86/transform/forward.rs:444-447):
// forward_transform(input: &[i16], output: &mut [T::Coeff], stride, tx_size, tx_type, bd, cpu).
extern "C" void b200_forward_transform(const int16_t *input, void *output, size_t stride,
                                       int tx_size, int tx_type, int bd, int coeff_is_i32) {
  b200_ctx *ctx = b200_default_ctx();
  // the reference panics on an invalid (size, type) pair (forward.rs:75)
  b200_percall_check(ctx, b200_fwd_txfm_batch(ctx, input, 0, stride, output, 1, tx_size, tx_type, bd, coeff_is_i32),
                     "forward_transform");
}
