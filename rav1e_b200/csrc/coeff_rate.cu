// Coefficient rate: write_coeffs_lv_map's symbols (context/block_unit.rs:1783-2016) counted by a
// WriterCounter (ec.rs:193-222) for batches of chains of transform blocks.  Contract and rules:
// include/b200rdo.h (b200_coeff_rate_dev).
//
// One warp per chain; the per-block counter is coeff_rate_dev.cuh's count_item.
#include "coeff_rate_dev.cuh"

namespace {

constexpr int kWarps = 4;  // warps (chains in flight) per CTA

template <typename T>
__device__ bool item_valid(const b200_coeff_item &it, const T *q, unsigned long long ncoeffs, const ScanTables &st,
                           int lane) {
  if (it.tx_size >= 19 || it.tx_type >= 16 || it.plane > 2 || it.plane_bsize >= 22 || it.mode > 33) return false;
  if (it.plane == 0 && it.mode == 13) return false;
  const int t = it.tx_size, cw = min(1 << cWl[t], 32), ch = min(1 << cHl[t], 32), area = cw * ch;
  if ((unsigned long long)it.block * area + area > ncoeffs || it.eob > area) return false;
  if (!it.clip_w4 || !it.clip_h4) return false;
  if (it.x4 + max(1 << (cWl[t] - 2), (int)it.clip_w4) > 16 || it.y4 + max(1 << (cHl[t] - 2), (int)it.clip_h4) > 16)
    return false;
  const T *blk = q + (size_t)it.block * area;
  const T tmin = sizeof(T) == 4 ? (T)INT32_MIN : (T)INT16_MIN;
  bool bad = false;
  for (int i = lane; i < area; i += 32) bad |= blk[i] == tmin;
  if (__any_sync(0xffffffffu, bad)) return false;
  if (it.eob > 0) {
    const uint16_t *scan = st.p[t][it.tx_type < 10 ? 0 : ((it.tx_type & 1) ? 2 : 1)];
    if (blk[scan[it.eob - 1]] == 0) return false;
    if (it.plane == 0) {
      int num;
      if (tx_ind(tx_set_of(t, it.mode >= 14, it.reduced_tx_set), it.tx_type, &num) < 0 && num > 1) return false;
    }
  }
  return true;
}

template <typename T>
__global__ void __launch_bounds__(32 * kWarps) coeff_rate_kernel(const b200_coeff_cdfs *cdfs, unsigned long long ncdfs,
                                                                 const b200_coeff_chain *chains, long long nchains,
                                                                 const b200_coeff_item *items,
                                                                 unsigned long long nitems, const T *q,
                                                                 unsigned long long ncoeffs, ScanTables st,
                                                                 uint32_t *rate_out, uint8_t *cul_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  WarpSmem &s = reinterpret_cast<WarpSmem *>(smem_raw)[wid];
  const long long nwarps = (long long)gridDim.x * kWarps;
  for (long long ci = (long long)blockIdx.x * kWarps + wid; ci < nchains; ci += nwarps) {
    const b200_coeff_chain &ch = chains[ci];
    const uint32_t snap = ch.snapshot, init_rng = ch.init_rng, ib = ch.item_begin, nit = ch.item_count;
    // ---- validity of the whole chain before any symbol
    bool ok = snap < ncdfs && init_rng >= 32768u && init_rng <= 65535u && (unsigned long long)ib + nit <= nitems;
    for (uint32_t k = 0; ok && k < nit; k++) ok = item_valid<T>(items[ib + k], q, ncoeffs, st, lane);
    if (!ok) {
      if (lane == 0) rate_out[ci] = 0xFFFFFFFFu;
      continue;
    }
    const uint16_t *g = reinterpret_cast<const uint16_t *>(cdfs + snap);
    if (lane < 24) reinterpret_cast<uint32_t *>(&s.above[0][0])[lane] = reinterpret_cast<const uint32_t *>(&ch.above[0][0])[lane];
    __syncwarp();
    uint64_t m0 = 0, m1 = 0, m2 = 0;  // regions copied so far
    count_begin(m0, s.cdf, g, lane);
    Coder w{init_rng, 0};
    for (uint32_t k = 0; k < nit; k++) {
      const b200_coeff_item it = items[ib + k];
      const int area = min(1 << cWl[it.tx_size], 32) * min(1 << cHl[it.tx_size], 32);
      count_item<T>(s, m0, m1, m2, g, st, it, q + (size_t)it.block * area, w, cul_out ? cul_out + ib + k : nullptr,
                    lane);
    }
    // tell_frac(end) - tell_frac(start); a counter's tell is bits + 1 (ec.rs:782-798)
    if (lane == 0) rate_out[ci] = frac(w.bits + 1, w.rng) - frac(1, init_rng);
    __syncwarp();
  }
}

#undef OFF

}  // namespace

extern "C" int b200_coeff_rate_dev(b200_ctx *ctx, const b200_coeff_cdfs *d_cdfs, size_t ncdfs,
                                   const b200_coeff_chain *d_chains, size_t nchains, const b200_coeff_item *d_items,
                                   size_t nitems, const void *d_qcoeffs, size_t ncoeffs, int coeff_is_i32,
                                   uint32_t *d_rate, uint8_t *d_cul_level) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, coeff_is_i32 == 0 || coeff_is_i32 == 1, "coeff_is_i32 %d not 0 / 1", coeff_is_i32);
  B200_REQUIRE(ctx, nchains < (1ull << 31) && nitems < (1ull << 31), "nchains %zu / nitems %zu >= 2^31", nchains,
               nitems);
  B200_REQUIRE(ctx, nchains == 0 || (d_chains != nullptr && d_cdfs != nullptr && d_rate != nullptr),
               "NULL chains / CDF snapshots / rate output");
  B200_REQUIRE(ctx, nchains == 0 || ncdfs > 0, "no CDF snapshot for %zu chains", nchains);
  B200_REQUIRE(ctx, nitems == 0 || (d_items != nullptr && d_qcoeffs != nullptr), "NULL items / coefficients");
  if (nchains == 0) return B200_OK;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  ScanTables st;
  for (int t = 0; t < 19; t++) {
    static const int kKindType[3] = {0, 10, 11};  // a tx_type of each scan kind
    for (int k = 0; k < 3; k++)
      if (int e = b200_scan_table_internal(ctx, t, kKindType[k], &st.p[t][k])) return e;
  }
  const int smem = kWarps * (int)sizeof(WarpSmem);
  const int grid = (int)std::min<size_t>((nchains + kWarps - 1) / kWarps, (size_t)ctx->num_sms * 16);
  if (coeff_is_i32) {
    if (int e = b200_smem_opt_in(ctx, (const void *)coeff_rate_kernel<int32_t>, smem)) return e;
    coeff_rate_kernel<int32_t><<<grid, 32 * kWarps, smem, ctx->stream>>>(
        d_cdfs, ncdfs, d_chains, (long long)nchains, d_items, nitems, (const int32_t *)d_qcoeffs, ncoeffs, st, d_rate,
        d_cul_level);
  } else {
    if (int e = b200_smem_opt_in(ctx, (const void *)coeff_rate_kernel<int16_t>, smem)) return e;
    coeff_rate_kernel<int16_t><<<grid, 32 * kWarps, smem, ctx->stream>>>(
        d_cdfs, ncdfs, d_chains, (long long)nchains, d_items, nitems, (const int16_t *)d_qcoeffs, ncoeffs, st, d_rate,
        d_cul_level);
  }
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
