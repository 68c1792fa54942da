// quantize.cu — quantize -> dequantize -> transform-domain distortion for batches of transform
// blocks (sm_90a): the steps of encode_tx_block that follow the forward transform
// (src/encoder.rs:1556-1655).
//
//   QuantizationContext::update / quantize   src/quantize/mod.rs:219-361
//   rust::dequantize                          src/quantize/mod.rs:368-392
//   raw tx-domain distortion                  src/encoder.rs:1611-1640
//   scan orders                               src/scan_order.rs (regenerated from their rule)
//
// One warp per block.  The reference's loop over the scan order carries one bit of state
// (`level_mode`: which rounding offset the next coefficient gets), so it looks serial; but each
// coefficient is a function {0,1} -> {0,1} of that bit, and function composition is associative:
// lanes take 32 consecutive scan positions, compute both outcomes, and an inclusive warp scan of
// the 2-bit function tables hands every lane its incoming state (5 shuffles per 32 coefficients).
// The end-of-block search is a REDUX.MAX over iscan, the distortion a shuffle reduction.
#include "quantize_dev.cuh"

extern "C" int b200_coded_tx_area(int tx_size) {
  return tx_size >= 0 && tx_size < 19 ? std::min(kQtxW[tx_size], 32) * std::min(kQtxH[tx_size], 32) : 0;
}

int b200_scan_table_internal(b200_ctx *ctx, int tx_size, int tx_type, const uint16_t **d_scan) {
  const uint16_t *iscan = nullptr;
  const int kind = tx_type < 10 ? 0 : ((tx_type & 1) ? 2 : 1);  // as quant_setup
  return scan_tables(ctx, tx_size, kind, d_scan, &iscan);
}

extern "C" int b200_quantize_dev(b200_ctx *ctx, const void *d_coeffs, size_t nblocks, int tx_size,
                                 int tx_type, uint32_t dc_quant, uint32_t ac_quant, int is_intra,
                                 int coeff_is_i32, void *d_qcoeffs, void *d_rcoeffs, uint16_t *d_eob,
                                 uint64_t *d_tx_dist) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, tx_size >= 0 && tx_size < 19, "tx_size %d out of range", tx_size);
  // av1_scan_orders has TX_TYPES = 16 columns: WHT_WHT (lossless only) never reaches quantize
  B200_REQUIRE(ctx, tx_type >= 0 && tx_type < 16, "tx_type %d out of range (0..15)", tx_type);
  B200_REQUIRE(ctx, dc_quant >= 1 && dc_quant <= 65535 && ac_quant >= 1 && ac_quant <= 65535,
               "quantizer step sizes must be NonZeroU16 (dc %u, ac %u)", dc_quant, ac_quant);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_coeffs && d_qcoeffs, "NULL coefficients / output");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  QuantArgs a{};
  if (int st = quant_setup(ctx, tx_size, tx_type, dc_quant, ac_quant, is_intra, coeff_is_i32, &a)) return st;
  a.coeffs = d_coeffs;
  a.qcoeffs = d_qcoeffs;
  a.rcoeffs = d_rcoeffs;
  a.eob = d_eob;
  a.tx_dist = (unsigned long long *)d_tx_dist;
  a.n = nblocks;
  const int wpc = 8;
  const int grid = (int)std::min<size_t>((nblocks + wpc - 1) / wpc, (size_t)ctx->num_sms * 16);
  if (coeff_is_i32)
    quantize_chain_kernel<int32_t><<<grid, wpc * 32, 0, ctx->stream>>>(a);
  else
    quantize_chain_kernel<int16_t><<<grid, wpc * 32, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
