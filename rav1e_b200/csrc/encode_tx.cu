// encode_tx.cu — encode_tx_block's numeric core (src/encoder.rs:1492-1655) for a batch of transform
// blocks in ONE kernel: the coefficients of a block never leave the SM between the steps
//   diff (:1533) + forward_transform (:1544)                     forward.rs:71-161
//   ts.qc.quantize (:1556) + dequantize (:1590) + raw tx-domain distortion (:1611-1640)   quantize/mod.rs
//   inverse_transform_add (:1600-1609)                            inverse.rs:1637-1704
//
// A CTA of 128 threads carries PER = 128 / max(W, H) blocks at a time, each with its own slice of shared
// memory: the padded transposition tile (shared by the forward and the inverse pass), the block's
// coefficients and its dequantized coefficients.
//   phase 1  thread per column, then per row: residual -> forward transform -> coefficients in shared
//            memory in the reference's order (and to d_coeffs when the caller wants them);
//   phase 2  one warp per block: the quantize chain of quantize_dev.cuh on the shared coefficients
//            (end of block by REDUX.MAX, the scan-order loop's one bit of state by a warp scan),
//            qcoeffs / eob / distortion to global memory, dequantized coefficients to shared memory;
//   phase 3  thread per row, then per column: inverse transform of the dequantized coefficients, added
//            into the reconstruction plane with the pixel clamp.
// The prediction is the reference plane displaced by the full-pel part of d_mv_src (NULL: zero motion);
// `rec` must already hold that prediction in the blocks' areas (predict-then-add, like the reference
// writes the prediction into `rec` before reconstructing).  Entropy coding of the quantized
// coefficients (write_coeffs_lv_map) and the rate / bias terms stay with the caller.
#include "fwd_txfm_dev.cuh"
#include "inv_txfm_dev.cuh"
#include "quantize_dev.cuh"

namespace {

struct EncArgs {
  const void *cur, *ref;
  int cur_stride, ref_stride;
  const b200_block *blocks;
  const b200_me_result *mv_src;
  size_t n;
  TxSetup tx;
  QuantArgs q;   // buffers unused: per-block pointers are formed in the kernel
  InvArgs inv;   // dst / dst_stride / kinds / shifts
  int need_recon;
  void *out_coef;   // may be NULL
  void *out_q, *out_r;  // out_r may be NULL
  uint16_t *out_eob;
  unsigned long long *out_dist;
};

constexpr int kEncThreads = 128;

template <int W, int H, typename CoefT>
struct EncLayout {
  static constexpr int T = W > H ? W : H;
  static constexpr int PER = kEncThreads / T;
  static constexpr int PITCH = W + 1;
  static constexpr int TILE = H * PITCH + ((H * PITCH) & 1);                       // ints
  static constexpr int CODED = (W < 32 ? W : 32) * (H < 32 ? H : 32);
  static constexpr size_t SLOT = (size_t)TILE * 4 + (size_t)(W * H + CODED) * sizeof(CoefT);
  static constexpr size_t SLOT_A = (SLOT + 15) / 16 * 16;
  static constexpr size_t SMEM = SLOT_A * PER;
};

template <int W, int H, typename CoefT>
__global__ void __launch_bounds__(kEncThreads) encode_tx_kernel(const __grid_constant__ EncArgs a) {
  using Px = typename std::conditional<sizeof(CoefT) == 2, uint8_t, uint16_t>::type;
  using L = EncLayout<W, H, CoefT>;
  constexpr int T = L::T, PER = L::PER, PITCH = L::PITCH;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int slot = threadIdx.x / T, t = threadIdx.x - slot * T;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  auto slot_tile = [&](int s) { return (int *)(smem_raw + (size_t)s * L::SLOT_A); };
  auto slot_coef = [&](int s) { return (CoefT *)(smem_raw + (size_t)s * L::SLOT_A + (size_t)L::TILE * 4); };
  auto slot_rcoef = [&](int s) { return slot_coef(s) + W * H; };
  int *tile = slot_tile(slot);
  CoefT *coef = slot_coef(slot);
  const size_t stride_blk = (size_t)gridDim.x * PER;
  for (size_t base = (size_t)blockIdx.x * PER; base < a.n; base += stride_blk) {
    const size_t blk = base + slot;
    const bool valid = blk < a.n;
    // ---- phase 1: residual + forward transform (forward.rs:94-160)
    if (valid && t < W) {
      const b200_block b = a.blocks[blk];
      int dx = 0, dy = 0;
      if (a.mv_src && a.mv_src[blk].cost != ~0ull) {
        dx = a.mv_src[blk].mv_col / 8;
        dy = a.mv_src[blk].mv_row / 8;
      }
      const Px *pc = (const Px *)a.cur + (long long)b.y * a.cur_stride + b.x + t;
      const Px *pr = (const Px *)a.ref + (long long)(b.y + dy) * a.ref_stride + b.x + dx + t;
      TXV c[H];
#pragma unroll
      for (int r = 0; r < H; r++) {
        const int rr = a.tx.ud_flip ? H - 1 - r : r;
        c[r] = round_shift_bit((int)pc[(long long)rr * a.cur_stride] - (int)pr[(long long)rr * a.ref_stride], a.tx.bit0);
      }
      run_1d<H>(a.tx.col_type, c);
      const int cc = a.tx.lr_flip ? W - 1 - t : t;
#pragma unroll
      for (int r = 0; r < H; r++) tile[r * PITCH + cc] = round_shift_bit(c[r], a.tx.bit1);
    }
    __syncthreads();
    if (valid && t < H) {
      TXV c[W];
#pragma unroll
      for (int k = 0; k < W; k++) c[k] = tile[t * PITCH + k];
      run_1d<W>(a.tx.row_type, c);
      const int off0 = CoefOrder<W, H>::row(t);
      CoefT *g = a.out_coef ? (CoefT *)a.out_coef + blk * (size_t)(W * H) : nullptr;
#pragma unroll
      for (int k = 0; k < W; k++) {
        const int idx = off0 + CoefOrder<W, H>::col(k);  // forward.rs:145-158
        const CoefT v = (CoefT)round_shift_bit(c[k], a.tx.bit2);
        coef[idx] = v;
        if (g) g[idx] = v;
      }
    }
    __syncthreads();
    // ---- phase 2: quantize -> dequantize -> tx-domain distortion, one warp per block
    for (int s = warp; s < PER; s += kEncThreads / 32) {
      const size_t b2 = base + s;
      if (b2 < a.n) {
        quantize_block_warp<CoefT>(a.q, slot_coef(s), (CoefT *)a.out_q + b2 * (size_t)a.q.coded, slot_rcoef(s),
                                   a.out_eob ? a.out_eob + b2 : nullptr, a.out_dist ? a.out_dist + b2 : nullptr, lane);
        if (a.out_r) {
          __syncwarp();
          CoefT *gr = (CoefT *)a.out_r + b2 * (size_t)a.q.coded;
          const CoefT *sr = slot_rcoef(s);
          for (int i = lane; i < a.q.coded; i += 32) gr[i] = sr[i];
        }
      }
    }
    __syncthreads();
    // ---- phase 3: inverse transform of the dequantized coefficients, added into the reconstruction
    if (a.need_recon) {
      if (valid && t < H) inv_row_pass_ptr<W, H, CoefT>(a.inv, slot_rcoef(slot), t, tile);
      __syncthreads();
      if (valid && t < W) {
        const b200_block b = a.blocks[blk];
        inv_col_pass_ptr<W, H, Px>(a.inv, (Px *)a.inv.dst + (long long)b.y * a.inv.dst_stride + b.x, t, tile);
      }
      __syncthreads();
    }
  }
}

template <int W, int H>
int launch_enc(b200_ctx *ctx, const EncArgs &a, int hbd) {
  const auto go = [&](auto tag) -> int {
    using CoefT = decltype(tag);
    using L = EncLayout<W, H, CoefT>;
    if (int st = b200_smem_opt_in(ctx, (const void *)encode_tx_kernel<W, H, CoefT>, (int)L::SMEM)) return st;
    const size_t ctas = (a.n + L::PER - 1) / L::PER;
    const int grid = (int)std::min<size_t>(ctas, (size_t)ctx->num_sms * 16);
    encode_tx_kernel<W, H, CoefT><<<grid, kEncThreads, L::SMEM, ctx->stream>>>(a);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
  };
  return hbd ? go(int32_t{}) : go(int16_t{});
}

}  // namespace

extern "C" int b200_encode_tx_blocks_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                         const b200_plane *rec, const b200_block *d_blocks, size_t nblocks,
                                         const b200_me_result *d_mv_src, int tx_size, int tx_type, int bd,
                                         uint32_t dc_quant, uint32_t ac_quant, int is_intra,
                                         int need_recon_pixel, void *d_coeffs, void *d_qcoeffs,
                                         void *d_rcoeffs, uint16_t *d_eob, uint64_t *d_tx_dist) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && ref && cur->data && ref->data && cur->bpp == ref->bpp, "bad planes");
  B200_REQUIRE(ctx, d_qcoeffs != nullptr, "NULL quantized-coefficient buffer");
  B200_REQUIRE(ctx, !need_recon_pixel || (rec && rec->data && rec->bpp == cur->bpp),
               "need_recon_pixel without a reconstruction plane");
  B200_REQUIRE(ctx, bd == 8 || bd == 10 || bd == 12, "bit depth %d not in {8,10,12}", bd);
  B200_REQUIRE(ctx, (cur->bpp == 1) == (bd == 8), "bpp %d does not match bit depth %d", cur->bpp, bd);
  B200_REQUIRE(ctx, valid_transform(tx_size, tx_type), "invalid transform: tx_size %d tx_type %d", tx_size, tx_type);
  // av1_scan_orders has TX_TYPES = 16 columns: WHT_WHT (lossless only) never reaches quantize
  B200_REQUIRE(ctx, tx_type >= 0 && tx_type < 16, "tx_type %d out of range (0..15)", tx_type);
  B200_REQUIRE(ctx, dc_quant >= 1 && dc_quant <= 65535 && ac_quant >= 1 && ac_quant <= 65535,
               "quantizer step sizes must be NonZeroU16 (dc %u, ac %u)", dc_quant, ac_quant);
  const int w = kItxW[tx_size], h = kItxH[tx_size];
  B200_REQUIRE(ctx, !need_recon_pixel || (inv_1d_exists(kTx1D[tx_type][1], w) && inv_1d_exists(kTx1D[tx_type][0], h)),
               "tx_type %d has no inverse at %dx%d (INV_TXFM_FNS, inverse.rs:1593-1623)", tx_type, w, h);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_blocks != nullptr, "NULL blocks");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  EncArgs a{};
  a.cur = cur->data, a.ref = ref->data;
  a.cur_stride = cur->stride, a.ref_stride = ref->stride;
  a.blocks = d_blocks;
  a.mv_src = d_mv_src;
  a.n = nblocks;
  a.tx = tx_setup(tx_size, tx_type, bd);
  if (int st = quant_setup(ctx, tx_size, tx_type, dc_quant, ac_quant, is_intra, cur->bpp == 2, &a.q)) return st;
  inv_setup(tx_size, tx_type, bd, &a.inv);
  a.inv.dst = need_recon_pixel ? rec->data : nullptr;
  a.inv.dst_stride = need_recon_pixel ? rec->stride : 0;
  a.need_recon = need_recon_pixel ? 1 : 0;
  a.out_coef = d_coeffs;
  a.out_q = d_qcoeffs;
  a.out_r = d_rcoeffs;
  a.out_eob = d_eob;
  a.out_dist = (unsigned long long *)d_tx_dist;
  const int hbd = bd > 8;
  switch (tx_size) {
#define B200_ETX(ID, W_, H_) \
  case ID:                   \
    return launch_enc<W_, H_>(ctx, a, hbd);
    B200_ETX(0, 4, 4)
    B200_ETX(1, 8, 8)
    B200_ETX(2, 16, 16)
    B200_ETX(3, 32, 32)
    B200_ETX(4, 64, 64)
    B200_ETX(5, 4, 8)
    B200_ETX(6, 8, 4)
    B200_ETX(7, 8, 16)
    B200_ETX(8, 16, 8)
    B200_ETX(9, 16, 32)
    B200_ETX(10, 32, 16)
    B200_ETX(11, 32, 64)
    B200_ETX(12, 64, 32)
    B200_ETX(13, 4, 16)
    B200_ETX(14, 16, 4)
    B200_ETX(15, 8, 32)
    B200_ETX(16, 32, 8)
    B200_ETX(17, 16, 64)
    B200_ETX(18, 64, 16)
#undef B200_ETX
  }
  return b200_fail(ctx, B200_ERR_ARG, "unreachable tx_size %d", tx_size);
}
