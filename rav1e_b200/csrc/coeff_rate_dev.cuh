// coeff_rate_dev.cuh — write_coeffs_lv_map's symbols (context/block_unit.rs:1783-2016) counted by a
// WriterCounter (ec.rs:193-222), one transform block at a time by one warp: shared by the batched
// coefficient rate (coeff_rate.cu) and the transform size / type decision (tx_size_type.cu).
//
// Per transform block the warp works in parallel: it builds the padded levels tile (txb_init_levels,
// rav1e's transposed layout) and, for every scan position below eob, the base-symbol context, the br
// context, the clipped level and the sign, packed in 16 bits; cul_level is a warp reduction.  Contexts
// depend only on the final levels, so what stays serial is the range coder's (bits, rng) recurrence and
// the CDF adaptation, which lane 0 runs from the packed words.  Each warp owns a copy of its chain's CDF
// snapshot in shared memory, filled region by region on first use (a transform-size slice, a tx-type
// row), so a chain reads only the rows it codes.
#pragma once
#include <cstddef>

#include "common.cuh"

namespace {
constexpr int kCdfLen = (int)(sizeof(b200_coeff_cdfs) / 2);
static_assert(kCdfLen == 3930, "b200_coeff_cdfs layout");
static_assert(sizeof(b200_coeff_chain) == 112 && sizeof(b200_coeff_item) == 16, "record layout");

#define OFF(F) ((int)(offsetof(b200_coeff_cdfs, F) / 2))

struct WarpSmem {
  uint16_t cdf[kCdfLen + 2];
  uint16_t pk[1024];             // per scan index c < eob: ctx | br_ctx << 6 | min(level, 15) << 11 | sign << 15
  uint8_t lv[36 * 36];           // levels, column-major with stride H + 4, zero in the padding
  uint8_t above[3][16], left[3][16];
};

struct ScanTables {
  const uint16_t *p[19][3];  // av1_scan_orders by (tx_size, kind): default / V_* rows / H_* identity
};

// TxSize (transform/mod.rs:130-240) and BlockSize (partition.rs:130-153) log2 dimensions
__constant__ uint8_t cWl[19] = {2, 3, 4, 5, 6, 2, 3, 3, 4, 4, 5, 5, 6, 2, 4, 3, 5, 4, 6};
__constant__ uint8_t cHl[19] = {2, 3, 4, 5, 6, 3, 2, 4, 3, 5, 4, 6, 5, 4, 2, 5, 3, 6, 4};
__constant__ uint8_t cBwl[22] = {2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5, 6, 6, 6, 7, 7, 2, 4, 3, 5, 4, 6};
__constant__ uint8_t cBhl[22] = {2, 3, 2, 3, 4, 3, 4, 5, 4, 5, 6, 5, 6, 7, 6, 7, 4, 2, 5, 3, 6, 4};
// the AV1 specification's inverse tx-type lists per TxSet (DCTONLY, INTER_3, INTRA_2, INTRA_1, INTER_2,
// INTER_1); av1_tx_ind is a type's position in its list, -1 ends a list
__constant__ int8_t cInvSet[6][16] = {{0, -1},
                                      {9, 0, -1},
                                      {9, 0, 3, 1, 2, -1},
                                      {9, 0, 10, 11, 3, 1, 2, -1},
                                      {9, 10, 11, 0, 1, 2, 4, 5, 3, 6, 7, 8, -1},
                                      {9, 10, 11, 12, 13, 14, 15, 0, 1, 2, 4, 5, 3, 6, 7, 8}};

__device__ __forceinline__ int tx_set_of(int t, int is_inter, int reduced) {  // get_tx_set, transform_unit.rs:123-148
  const int up = max(cWl[t], cHl[t]) - 2, sq = min(cWl[t], cHl[t]) - 2;
  if (up > 3) return 0;
  if (is_inter) return (reduced || up == 3) ? 1 : sq == 2 ? 4 : 5;
  if (up == 3) return 0;
  return (reduced || sq == 2) ? 2 : 3;
}
__device__ __forceinline__ int tx_ind(int set, int type, int *num) {  // av1_tx_ind / num_tx_set, -1: unused
  int ind = -1, n = 0;
  for (; n < 16 && cInvSet[set][n] >= 0; n++)
    if (cInvSet[set][n] == type) ind = n;
  *num = n;
  return ind;
}

struct Coder {
  uint32_t rng, bits;
};

// symbol (ec.rs:520-537): lr_compute (:334-346) + the counter's store (:195-201)
__device__ __forceinline__ void code(Coder &w, uint32_t fl, uint32_t fh, uint32_t nms) {
  const uint32_t r = w.rng;
  const uint32_t u = fl >= 32768u ? r : ((((r >> 8) * (fl >> 6)) >> 1) + 4u * nms);
  const uint32_t v = (((r >> 8) * (fh >> 6)) >> 1) + 4u * (nms - 1);
  const uint32_t rr = (u - v) & 0xFFFFu;
  const int d = __clz(rr) - 16;
  w.bits += (uint32_t)d;
  w.rng = (rr << d) & 0xFFFFu;
}
// symbol_with_update: the symbol, then update_cdf (ec.rs:935-955)
__device__ __forceinline__ void put(Coder &w, uint16_t *cdf, int n, uint32_t s) {
  code(w, s ? cdf[s - 1] : 32768u, cdf[s], (uint32_t)(n - (int)s));
  const uint32_t cnt = cdf[n - 1];
  const int rate = 3 + min(n >> 1, 2) + (int)(cnt >> 4);
  cdf[n - 1] = (uint16_t)(cnt + 1 - (cnt >> 5));
  for (int i = 0; i < n - 1; i++) {
    const uint32_t v = cdf[i];
    cdf[i] = (uint16_t)((uint32_t)i >= s ? v - (v >> rate) : v + ((32768u - v) >> rate));
  }
}
// bit (ec.rs:494-496): bool(bit == 1, 16384) over the CDF [16384, 0]
__device__ __forceinline__ void bit(Coder &w, uint32_t b) { code(w, b ? 16384u : 32768u, b ? 0u : 16384u, 2u - b); }

// frac_compute (ec.rs:357-379)
__device__ __forceinline__ uint32_t frac(uint32_t nbits_total, uint32_t rng) {
  uint32_t l = 0;
  for (int i = 0; i < 3; i++) {
    rng = (rng * rng) >> 15;
    const uint32_t b = rng >> 16;
    l = (l << 1) | b;
    rng >>= b;
  }
  return (nbits_total << 3) - l;
}

// get_nz_map_ctx_from_stats' offsets (transform_unit.rs:846-883) by their generating rule: the
// Coeff_Base_Ctx_Offset table for 2-D classes, Coeff_Base_Pos_Ctx_Offset for 1-D ones
__device__ __forceinline__ int nz_offset_2d(int t, int row, int col) {
  const int w = 1 << cWl[t], h = 1 << cHl[t];
  if (row == 0 && col == 0) return 0;
  if (w < h && row < 2) return 11;
  if (w > h && col < 2) return 16;
  if (row + col < 2) return 1;
  if (row + col < 4) return 6;
  return 21;
}

// eob_flag_cdf16 .. eob_flag_cdf1024 by tx_size.area_log2() - 4 (encode_eob's match, block_unit.rs:1869-1898);
// each is [2][2][n] with n = 5 + multi, laid out back to back
__device__ __forceinline__ int eob_flag_off(int multi) {
  int off = OFF(eob_flag16);
  for (int i = 0; i < multi; i++) off += 4 * (5 + i);
  return off;
}
static_assert(OFF(eob_flag1024) == OFF(eob_flag16) + 4 * (5 + 6 + 7 + 8 + 9 + 10), "eob_flag fields back to back");

// window read of get_txb_ctx (block_unit.rs:442-526)
__device__ __forceinline__ void txb_ctx(const WarpSmem &s, const b200_coeff_item &it, int *skip_ctx, int *dc_ctx) {
  const uint8_t *above = &s.above[it.plane][it.x4], *left = &s.left[it.plane][it.y4];
  int dc = 0;
  uint32_t top = 0, lft = 0;
  for (int i = 0; i < it.clip_w4; i++) {
    const int sg = above[i] >> 6;
    dc += sg == 1 ? -1 : sg == 2 ? 1 : 0;
    top |= above[i];
  }
  for (int i = 0; i < it.clip_h4; i++) {
    const int sg = left[i] >> 6;
    dc += sg == 1 ? -1 : sg == 2 ? 1 : 0;
    lft |= left[i];
  }
  *dc_ctx = dc < 0 ? 1 : dc > 0 ? 2 : 0;
  const int t = it.tx_size;
  if (it.plane == 0) {
    if (cBwl[it.plane_bsize] == cWl[t] && cBhl[it.plane_bsize] == cHl[t]) {
      *skip_ctx = 0;
    } else {
      top &= 63;
      lft &= 63;
      const int mx = min((int)(top | lft), 4), mn = min(min((int)top, (int)lft), 4);
      *skip_ctx = !mx ? 1 : !mn ? 2 + (mx > 3) : mx <= 3 ? 4 : mn <= 3 ? 5 : 6;
    }
  } else {
    *skip_ctx = (top != 0) + (lft != 0) + (cBwl[it.plane_bsize] + cBhl[it.plane_bsize] > cWl[t] + cHl[t] ? 10 : 7);
  }
}

// first use of a CDF region by this chain: copy it from the snapshot (warp-uniform control flow)
__device__ __forceinline__ void ensure(uint64_t &mask, int bit_idx, uint16_t *dst, const uint16_t *src, int off,
                                       int len, int lane) {
  if ((mask >> bit_idx) & 1) return;
  for (int i = lane; i < len; i += 32) dst[off + i] = src[off + i];
  mask |= 1ull << bit_idx;
  __syncwarp();
}

// The regions every chain codes with, copied when the chain starts.
__device__ __forceinline__ void count_begin(uint64_t &m0, uint16_t *cdf, const uint16_t *g, int lane) {
  ensure(m0, 63, cdf, g, OFF(dc_sign), OFF(eob_extra) - OFF(dc_sign), lane);
  ensure(m0, 62, cdf, g, OFF(eob_flag16), OFF(coeff_base_eob) - OFF(eob_flag16), lane);
}

// One transform block of a chain (write_coeffs_lv_map, block_unit.rs:1783-2016) by one warp: its symbols
// through the counter w (lane 0), the CDF regions it codes with copied from the snapshot g on first use,
// its cul_level written into s's window (and to *cul_out unless NULL).  blk: the coded block, any address
// space.  Ends with __syncwarp().
template <typename T>
__device__ __forceinline__ void count_item(WarpSmem &s, uint64_t &m0, uint64_t &m1, uint64_t &m2, const uint16_t *g,
                                           const ScanTables &st, const b200_coeff_item &it, const T *blk, Coder &w,
                                           uint8_t *cul_out, int lane) {
  const int t = it.tx_size, eob = it.eob, ptype = it.plane != 0;
  const int cw = min(1 << cWl[t], 32), chh = min(1 << cHl[t], 32), area = cw * chh, bhl = min((int)cHl[t], 5);
  const int txs_ctx = (min(cWl[t], cHl[t]) + max(cWl[t], cHl[t]) - 4 + 1) >> 1;
  const int cls = it.tx_type < 10 ? 0 : ((it.tx_type & 1) ? 1 : 2);
  const uint16_t *scan = st.p[t][cls == 0 ? 0 : (cls == 1 ? 2 : 1)];
  ensure(m0, txs_ctx, s.cdf, g, OFF(txb_skip) + txs_ctx * 26, 26, lane);
  int skip_ctx = 0, dc_ctx = 0;
  if (lane == 0) txb_ctx(s, it, &skip_ctx, &dc_ctx);
  if (eob == 0) {
    if (lane == 0) {
      put(w, &s.cdf[OFF(txb_skip) + (txs_ctx * 13 + skip_ctx) * 2], 2, 1);
      for (int i = 0; i < (1 << (cWl[t] - 2)); i++) s.above[it.plane][it.x4 + i] = 0;
      for (int i = 0; i < (1 << (cHl[t] - 2)); i++) s.left[it.plane][it.y4 + i] = 0;
      if (cul_out) *cul_out = 0;
    }
    __syncwarp();
    return;
  }
  // ---- CDF regions this block codes with
  const int tp = txs_ctx * 2 + ptype, brt = min(txs_ctx, 3) * 2 + ptype;
  ensure(m0, 5 + tp, s.cdf, g, OFF(eob_extra) + tp * 18, 18, lane);
  ensure(m0, 35 + tp, s.cdf, g, OFF(coeff_base_eob) + tp * 12, 12, lane);
  ensure(m0, 45 + tp, s.cdf, g, OFF(coeff_base) + tp * 168, 168, lane);
  ensure(m0, 15 + brt, s.cdf, g, OFF(coeff_br) + brt * 84, 84, lane);
  const int is_inter = it.mode >= 14;
  int tx_s = -1, tx_n = 0, tx_off = 0;
  if (it.plane == 0) {
    const int set = tx_set_of(t, is_inter, it.reduced_tx_set), sq = min(cWl[t], cHl[t]) - 2;
    int num;
    tx_s = tx_ind(set, it.tx_type, &num);
    if (num > 1) {
      if (is_inter) {
        const int idx = set == 5 ? 1 : set == 4 ? 2 : 3;
        tx_n = idx == 1 ? 16 : idx == 2 ? 12 : 2;
        tx_off = (idx == 1 ? OFF(inter_tx_1) : idx == 2 ? OFF(inter_tx_2) : OFF(inter_tx_3)) + sq * tx_n;
        ensure(m0, 23 + (idx - 1) * 4 + sq, s.cdf, g, tx_off, tx_n, lane);
      } else {
        const int idx = set == 3 ? 1 : 2;
        tx_n = idx == 1 ? 7 : 5;
        tx_off = (idx == 1 ? OFF(intra_tx_1) : OFF(intra_tx_2)) + (sq * 13 + it.mode) * tx_n;
        ensure(idx == 1 ? m1 : m2, sq * 13 + it.mode, s.cdf, g, tx_off, tx_n, lane);
      }
    }
  }
  // ---- levels (txb_init_levels, transform_unit.rs:780-792) over the padded (cw + 4) x (chh + 4) tile
  const int stride = chh + 4;
  for (int i = lane; i < (cw + 4) * stride; i += 32) {
    const int col = i / stride, row = i - col * stride;
    uint32_t a = 0;
    if (col < cw && row < chh) {
      const int v = (int)blk[col * chh + row];
      a = min((uint32_t)(v < 0 ? -v : v), 127u);
    }
    s.lv[i] = (uint8_t)a;
  }
  __syncwarp();
  // ---- per scan position: contexts (get_nz_map_contexts :911-936, get_br_ctx :938-985), level, sign
  uint32_t cul = 0;
  for (int c = lane; c < eob; c += 32) {
    const int pos = scan[c];
    const int v = (int)blk[pos];
    const uint32_t level = (uint32_t)(v < 0 ? -v : v);
    cul += level;
    const int col = pos >> bhl, row = pos - (col << bhl);
    const uint8_t *lp = &s.lv[col * stride + row];
    int ctx;
    if (c == eob - 1) {
      ctx = c == 0 ? 0 : c <= area / 8 ? 1 : c <= area / 4 ? 2 : 3;
    } else {
      int mag = min(3, (int)lp[1]) + min(3, (int)lp[stride]);
      if (cls == 0) mag += min(3, (int)lp[stride + 1]) + min(3, (int)lp[2]) + min(3, (int)lp[2 * stride]);
      else if (cls == 2) mag += min(3, (int)lp[2]) + min(3, (int)lp[3]) + min(3, (int)lp[4]);
      else mag += min(3, (int)lp[2 * stride]) + min(3, (int)lp[3 * stride]) + min(3, (int)lp[4 * stride]);
      if ((cls | pos) == 0) {
        ctx = 0;
      } else {
        ctx = min((mag + 1) >> 1, 4);
        if (cls == 0) ctx += nz_offset_2d(t, min(row, 4), min(col, 4));
        else ctx += 26 + 5 * min(cls == 1 ? col : row, 2);
      }
    }
    int br = 0;
    if (level > 2) {
      int mag = (uint8_t)(lp[1] + lp[stride]);
      mag += cls == 0 ? lp[stride + 1] : cls == 1 ? lp[2 * stride] : lp[2];
      mag = min((mag + 1) >> 1, 6);
      const bool near = cls == 0 ? (row < 2 && col < 2) : cls == 1 ? col == 0 : row == 0;
      br = pos == 0 ? mag : near ? mag + 7 : mag + 14;
    }
    s.pk[c] = (uint16_t)(ctx | br << 6 | min(level, 15u) << 11 | (uint32_t)(v < 0) << 15);
  }
  cul = __reduce_add_sync(0xffffffffu, cul);
  __syncwarp();
  if (lane == 0) {
    put(w, &s.cdf[OFF(txb_skip) + (txs_ctx * 13 + skip_ctx) * 2], 2, 0);
    if (tx_n) put(w, &s.cdf[tx_off], tx_n, (uint32_t)tx_s);
    // encode_eob (block_unit.rs:1861-1914): eob_pt is the spec's group of eob
    const int eob_pt = eob < 3 ? eob : 33 - __clz(eob - 1);
    const int eob_extra = eob - (eob_pt < 3 ? eob_pt : (1 << (eob_pt - 2)) + 1);
    const int multi = min(cWl[t] + cHl[t] - 4, 6), n = 5 + multi;
    put(w, &s.cdf[eob_flag_off(multi) + (ptype * 2 + (cls != 0)) * n], n, (uint32_t)(eob_pt - 1));
    const int obits = eob_pt < 3 ? 0 : eob_pt - 2;
    if (obits > 0) {
      put(w, &s.cdf[OFF(eob_extra) + (tp * 9 + eob_pt - 3) * 2], 2, (uint32_t)(eob_extra >> (obits - 1)) & 1u);
      for (int i = 1; i < obits; i++) bit(w, (uint32_t)(eob_extra >> (obits - 1 - i)) & 1u);
    }
    // encode_coeffs (:1916-1981): reverse scan, the base symbol then its br loop
    uint16_t *base_eob = &s.cdf[OFF(coeff_base_eob) + tp * 12], *base = &s.cdf[OFF(coeff_base) + tp * 168];
    uint16_t *brc = &s.cdf[OFF(coeff_br) + brt * 84];
    for (int c = eob - 1; c >= 0; c--) {
      const uint32_t p = s.pk[c], level = (p >> 11) & 15u;
      if (c == eob - 1) put(w, base_eob + (p & 63u) * 3, 3, min(level, 3u) - 1);
      else put(w, base + (p & 63u) * 4, 4, min(level, 3u));
      if (level > 2) {
        uint16_t *row = brc + ((p >> 6) & 31u) * 4;
        const uint32_t range = level - 3;
        for (uint32_t idx = 0; idx < 12; idx += 3) {
          const uint32_t kk = min(range - idx, 3u);
          put(w, row, 4, kk);
          if (kk < 3) break;
        }
      }
    }
    // encode_coeff_signs (:1983-2016): dc_sign, bypass sign bits, write_golomb (ec.rs:609-620)
    for (int c = 0; c < eob; c++) {
      const uint32_t p = s.pk[c], level = (p >> 11) & 15u, sign = p >> 15;
      if (level == 0) continue;
      if (c == 0) put(w, &s.cdf[OFF(dc_sign) + (ptype * 3 + dc_ctx) * 2], 2, sign);
      else bit(w, sign);
      if (level > 14) {
        const int v = (int)blk[scan[c]];
        const uint32_t x = (uint32_t)(v < 0 ? -v : v) - 14u;  // (level - 15) + 1
        const int len = 32 - __clz(x);
        for (int i = 0; i < len - 1; i++) bit(w, 0);
        for (int i = len - 1; i >= 0; i--) bit(w, (x >> i) & 1u);
      }
    }
    uint32_t cl = min(cul, 63u);
    const uint32_t p0 = s.pk[0];
    if ((p0 >> 11) & 15u) cl = (p0 >> 15) ? (cl | 64u) : cl + 128u;
    for (int i = 0; i < (1 << (cWl[t] - 2)); i++) s.above[it.plane][it.x4 + i] = (uint8_t)cl;
    for (int i = 0; i < (1 << (cHl[t] - 2)); i++) s.left[it.plane][it.y4 + i] = (uint8_t)cl;
    if (cul_out) *cul_out = (uint8_t)cl;
  }
  __syncwarp();
}

}  // namespace
