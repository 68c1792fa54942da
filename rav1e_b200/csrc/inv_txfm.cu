// inv_txfm.cu — inverse transform + reconstruction for batches of transform blocks (sm_90a).
//
//   rust::inverse_transform_add   src/transform/inverse.rs:1637-1704
//   INV_TXFM_FNS                  :1593-1623   INV_INTERMEDIATE_SHIFTS :1710-1711
//   av1_iwht4 :35-53, identity :150-157 / :299-304 / :579-584 / :886-891, flipped ADSTs
//   half_btf / clamp_value        src/transform/mod.rs:296-315
// The 1-D DCT / ADST butterfly networks are the generated single-assignment programs of
// inv_txfm_networks.cuh (tools/gen_inv_txfm.py), shared word for word with the oracle's copy.
//
// Same shape as the forward kernel: T = max(W, H) threads per block-transform, several transforms
// per CTA.  Row pass: thread r reads its row of the (transposed, 32x32-coded) coefficients — threads
// walk consecutive addresses — applies the rectangular / lossless scaling and clamp, runs the
// 1-D row transform in registers and parks the row in a padded shared tile.  Column pass: thread c
// reads its column, intermediate round shift + clamp, 1-D column transform, final round shift, and
// adds into the destination plane with the pixel clamp (rows of the plane are written by
// consecutive threads).  Blocks of one call must not overlap.
//
// The per-thread row / column passes (inv_txfm_dev.cuh) are host+device functions:
// tests/test_inv_txfm_emul.py replays them on the CPU against the oracle (all 160 valid pairs, 8, 10 and
// 12 bit, also with coefficients at the limits of their type); tests/test_zz_inv_txfm_gpu.py and
// tests/test_tx_paths_gpu.py check the launch on hardware, the latter at the clamps and past one grid stride.
#include "inv_txfm_dev.cuh"

namespace {

template <int W, int H, typename CoefT, typename Px>
__global__ void __launch_bounds__(kInvThreads) inv_txfm_add_kernel(const __grid_constant__ InvArgs a) {
  constexpr int T = W > H ? W : H;
  constexpr int PER = kInvThreads / T;
  constexpr int PITCH = W + 1;
  constexpr int REGION = H * PITCH + ((H * PITCH) % 2 == 0 ? 1 : 0);
  __shared__ int buf[PER * REGION];
  const int slot = threadIdx.x / T, t = threadIdx.x - slot * T;
  int *tile = buf + slot * REGION;
  const size_t stride_blk = (size_t)gridDim.x * PER;
  for (size_t base = (size_t)blockIdx.x * PER; base < a.n; base += stride_blk) {
    const size_t blk = base + slot;
    const bool valid = blk < a.n;
    if (valid && t < H) inv_row_pass<W, H, CoefT>(a, blk, t, tile);
    __syncthreads();
    if (valid && t < W) inv_col_pass<W, H, Px>(a, blk, t, tile);
    __syncthreads();
  }
}

template <int W, int H>
int launch_inv(b200_ctx *ctx, const InvArgs &a, int hbd) {
  constexpr int T = W > H ? W : H;
  constexpr int PER = kInvThreads / T;
  const size_t ctas = (a.n + PER - 1) / PER;
  const int grid = (int)std::min<size_t>(ctas, (size_t)ctx->num_sms * 32);
  if (hbd)
    inv_txfm_add_kernel<W, H, int32_t, uint16_t><<<grid, kInvThreads, 0, ctx->stream>>>(a);
  else
    inv_txfm_add_kernel<W, H, int16_t, uint8_t><<<grid, kInvThreads, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

}  // namespace

// inverse_transform_add for nblocks blocks of one (tx_size, tx_type): the destination area of
// block i is the w x h rectangle at d_blocks[i] of `dst` (u8 planes take i16 coefficients, u16
// planes i32, T::Coeff); d_coeffs holds b200_coded_tx_area(tx_size) coefficients per block in the
// forward transform's layout (what b200_quantize_dev writes to d_rcoeffs).
extern "C" int b200_inverse_transform_add_dev(b200_ctx *ctx, const void *d_coeffs, const b200_plane *dst,
                                              const b200_block *d_blocks, size_t nblocks, int tx_size,
                                              int tx_type, int bd) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, tx_size >= 0 && tx_size < 19 && tx_type >= 0 && tx_type <= 16,
               "tx_size %d / tx_type %d out of range", tx_size, tx_type);
  B200_REQUIRE(ctx, bd == 8 || bd == 10 || bd == 12, "bit depth %d not in {8,10,12}", bd);
  B200_REQUIRE(ctx, dst && dst->data && (dst->bpp == 1) == (bd == 8), "bad destination plane for bit depth %d", bd);
  const int w = kItxW[tx_size], h = kItxH[tx_size];
  B200_REQUIRE(ctx, inv_1d_exists(kTx1D[tx_type][1], w) && inv_1d_exists(kTx1D[tx_type][0], h),
               "tx_type %d has no inverse at %dx%d (INV_TXFM_FNS, inverse.rs:1593-1623)", tx_type, w, h);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_coeffs && d_blocks, "NULL coefficients / blocks");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  InvArgs a{};
  a.coeffs = d_coeffs;
  a.dst = dst->data;
  a.dst_stride = dst->stride;
  a.blocks = d_blocks;
  a.n = nblocks;
  inv_setup(tx_size, tx_type, bd, &a);
  const int hbd = bd > 8;
  switch (tx_size) {
#define B200_ITX(ID, W_, H_) \
  case ID:                   \
    return launch_inv<W_, H_>(ctx, a, hbd);
    B200_ITX(0, 4, 4)
    B200_ITX(1, 8, 8)
    B200_ITX(2, 16, 16)
    B200_ITX(3, 32, 32)
    B200_ITX(4, 64, 64)
    B200_ITX(5, 4, 8)
    B200_ITX(6, 8, 4)
    B200_ITX(7, 8, 16)
    B200_ITX(8, 16, 8)
    B200_ITX(9, 16, 32)
    B200_ITX(10, 32, 16)
    B200_ITX(11, 32, 64)
    B200_ITX(12, 64, 32)
    B200_ITX(13, 4, 16)
    B200_ITX(14, 16, 4)
    B200_ITX(15, 8, 32)
    B200_ITX(16, 32, 8)
    B200_ITX(17, 16, 64)
    B200_ITX(18, 64, 16)
#undef B200_ITX
  }
  return b200_fail(ctx, B200_ERR_ARG, "unreachable tx_size %d", tx_size);
}
