/*
 * coeff_rate.c — write_coeffs_lv_map through rav1e's range-coder backends (see coeff_rate.h).
 * Serial and literal: one writer, one private copy of the chain's CDF snapshot, symbols in the
 * reference's order.  The tables are restated from the AV1 specification's rules and compared with the
 * reference's by digest (tests/test_oracle_coeff_rate.py).
 */
#include "coeff_rate.h"

#include <stdlib.h>
#include <string.h>

#include "oracle.h"

/* ---------------------------------------------------------------- sizes (transform/mod.rs:130-240) */
static const uint8_t kWl[19] = {2, 3, 4, 5, 6, 2, 3, 3, 4, 4, 5, 5, 6, 2, 4, 3, 5, 4, 6};
static const uint8_t kHl[19] = {2, 3, 4, 5, 6, 3, 2, 4, 3, 5, 4, 6, 5, 4, 2, 5, 3, 6, 4};
/* BlockSize 0..21 (partition.rs:130-153): log2 width / height */
static const uint8_t kBwl[22] = {2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5, 6, 6, 6, 7, 7, 2, 4, 3, 5, 4, 6};
static const uint8_t kBhl[22] = {2, 3, 2, 3, 4, 3, 4, 5, 4, 5, 6, 5, 6, 7, 6, 7, 4, 2, 5, 3, 6, 4};
static int imin(int a, int b) { return a < b ? a : b; }
static int imax(int a, int b) { return a > b ? a : b; }
static int sqr_log2(int t) { return imin(kWl[t], kHl[t]); }
static int sqr_up_log2(int t) { return imax(kWl[t], kHl[t]); }
/* TxSize::sqr() / sqr_up() as TxSize discriminants: the square sizes are 0..4 for log2 2..6 */
static int tx_sqr(int t) { return sqr_log2(t) - 2; }
static int tx_sqr_up(int t) { return sqr_up_log2(t) - 2; }

/* ---------------------------------------------------------------- tables, restated from the spec */
enum { SET_DCTONLY, SET_INTER_3, SET_INTRA_2, SET_INTRA_1, SET_INTER_2, SET_INTER_1 };
/* the spec's inverse lists Tx_Type_{Intra,Inter}_Inv_Set* (TxType discriminants, transform/mod.rs:101-123):
 * av1_tx_ind is the position of a type in its set's list, av1_tx_used its membership */
static const int8_t kInvSet[6][16] = {
    {0, -1},
    {9, 0, -1},
    {9, 0, 3, 1, 2, -1},
    {9, 0, 10, 11, 3, 1, 2, -1},
    {9, 10, 11, 0, 1, 2, 4, 5, 3, 6, 7, 8, -1},
    {9, 10, 11, 12, 13, 14, 15, 0, 1, 2, 4, 5, 3, 6, 7, 8}};
static int num_tx_set[6], av1_tx_used[6][16], av1_tx_ind[6][16], tx_type_to_class[16];
static int eob_to_pos_small[33], eob_to_pos_large[17], k_eob_group_start[12], k_eob_offset_bits[12];
static int av1_nz_map_ctx_offset[19][5][5], nz_map_ctx_offset_1d[32], skip_contexts[5][5], dc_sign_contexts[65];
static const int tx_set_index_intra[6] = {0, -1, 2, 1, -1, -1};
static const int tx_set_index_inter[6] = {0, 3, -1, -1, 2, 1};
static int tables_ready;

static int eob_group(int eob) { /* the spec's eob_pt: group t holds k_eob_group_start[t] ..< start[t + 1] */
  if (eob < 3) return eob;
  int t = 3;
  while ((1 << (t - 1)) < eob) t++;
  return t;
}

static void init_tables(void) {
  if (tables_ready) return;
  for (int s = 0; s < 6; s++) {
    int n = 0;
    for (; n < 16 && kInvSet[s][n] >= 0; n++) {
      av1_tx_used[s][kInvSet[s][n]] = 1;
      av1_tx_ind[s][kInvSet[s][n]] = n;
    }
    num_tx_set[s] = n;
  }
  for (int t = 0; t < 16; t++) tx_type_to_class[t] = t < 10 ? 0 : ((t & 1) ? 1 : 2); /* V_* vertical, H_* horizontal */
  for (int t = 0; t < 12; t++) {
    k_eob_group_start[t] = t < 3 ? t : (1 << (t - 2)) + 1;
    k_eob_offset_bits[t] = t < 3 ? 0 : t - 2;
  }
  for (int e = 0; e <= 32; e++) eob_to_pos_small[e] = eob_group(e);
  for (int i = 0; i <= 16; i++) eob_to_pos_large[i] = i == 0 ? 6 : eob_group(32 * i + 1); /* [0] is unused */
  /* Coeff_Base_Ctx_Offset: row < 2 of a tall block, col < 2 of a wide one, then the row + col bands; 0 at
   * DC and outside the coded block */
  for (int t = 0; t < 19; t++) {
    const int w = 1 << kWl[t], h = 1 << kHl[t], cw = imin(w, 32), ch = imin(h, 32);
    for (int r = 0; r < 5; r++)
      for (int c = 0; c < 5; c++) {
        int v;
        if ((r == 0 && c == 0) || r >= ch || c >= cw) v = 0;
        else if (w < h && r < 2) v = 11;
        else if (w > h && c < 2) v = 16;
        else if (r + c < 2) v = 1;
        else if (r + c < 4) v = 6;
        else v = 21;
        av1_nz_map_ctx_offset[t][r][c] = v;
      }
  }
  for (int i = 0; i < 32; i++) nz_map_ctx_offset_1d[i] = 26 + 5 * imin(i, 2); /* Coeff_Base_Pos_Ctx_Offset */
  for (int mn = 0; mn < 5; mn++)
    for (int mx = 0; mx < 5; mx++)
      skip_contexts[mn][mx] = !mx ? 1 : !mn ? 2 + (mx > 3) : mx <= 3 ? 4 : mn <= 3 ? 5 : 6;
  for (int i = 0; i < 65; i++) dc_sign_contexts[i] = i < 32 ? 1 : i == 32 ? 0 : 2;
  tables_ready = 1;
}

int orc_coeff_table(const char *name, int32_t *out) {
  init_tables();
#define ORC_T(NAME, ARR)                                                      \
  if (!strcmp(name, NAME)) {                                                  \
    const int *p = (const int *)(ARR);                                        \
    const int n = (int)(sizeof(ARR) / sizeof(int));                           \
    for (int i = 0; i < n; i++) out[i] = p[i];                                \
    return n;                                                                 \
  }
  ORC_T("num_tx_set", num_tx_set)
  ORC_T("av1_tx_used", av1_tx_used)
  ORC_T("av1_tx_ind", av1_tx_ind)
  ORC_T("tx_type_to_class", tx_type_to_class)
  ORC_T("eob_to_pos_small", eob_to_pos_small)
  ORC_T("eob_to_pos_large", eob_to_pos_large)
  ORC_T("k_eob_group_start", k_eob_group_start)
  ORC_T("k_eob_offset_bits", k_eob_offset_bits)
  ORC_T("av1_nz_map_ctx_offset", av1_nz_map_ctx_offset)
  ORC_T("nz_map_ctx_offset_1d", nz_map_ctx_offset_1d)
  ORC_T("skip_contexts", skip_contexts)
  ORC_T("dc_sign_contexts", dc_sign_contexts)
#undef ORC_T
  return 0;
}

/* get_tx_set, transform_unit.rs:123-148 */
static int get_tx_set(int tx_size, int is_inter, int reduced) {
  const int up = tx_sqr_up(tx_size), sq = tx_sqr(tx_size);
  if (up > 3) return SET_DCTONLY;
  if (is_inter) return (reduced || up == 3) ? SET_INTER_3 : sq == 2 ? SET_INTER_2 : SET_INTER_1;
  if (up == 3) return SET_DCTONLY;
  return (reduced || sq == 2) ? SET_INTRA_2 : SET_INTRA_1;
}

/* ---------------------------------------------------------------- the writer (ec.rs) */
typedef struct {
  int enc;          /* 0: WriterCounter, 1: WriterEncoder */
  uint32_t rng;     /* u16 */
  int cnt;          /* i16, -9 at new() */
  uint32_t low;     /* ec_window */
  uint64_t bits;    /* the counter's s.bits */
  uint16_t *pre;    /* the encoder's precarry */
  size_t npre, cap;
  long nsym;
  int oom;
} writer;

static void w_init(writer *w, int enc, uint32_t rng) {
  memset(w, 0, sizeof(*w));
  w->enc = enc;
  w->rng = rng;
  w->cnt = -9;
}

static void w_push(writer *w, uint16_t v) {
  if (w->npre == w->cap) {
    w->cap = w->cap ? 2 * w->cap : 4096;
    uint16_t *p = (uint16_t *)realloc(w->pre, w->cap * sizeof(uint16_t));
    if (!p) {
      w->oom = 1;
      return;
    }
    w->pre = p;
  }
  w->pre[w->npre++] = v;
}

static int clz16(uint32_t r) {
  int d = 0;
  while (d < 16 && !(r & (0x8000u >> d))) d++;
  return d;
}

/* lr_compute, ec.rs:334-346, then store of the counter (:195-201) or the encoder (:265-288) */
static void w_store(writer *w, uint32_t fl, uint32_t fh, uint32_t nms) {
  const uint32_t r = w->rng;
  uint32_t u = (((r >> 8) * (fl >> 6)) >> 1) + 4 * nms;
  if (fl >= 32768) u = r;
  const uint32_t v = (((r >> 8) * (fh >> 6)) >> 1) + 4 * (nms - 1);
  const uint32_t l = r - u, rr = (u - v) & 0xFFFF;
  const int d = clz16(rr);
  w->nsym++;
  if (!w->enc) {
    w->bits += (uint64_t)d;
    w->rng = (rr << d) & 0xFFFF;
    return;
  }
  uint32_t low = l + w->low;
  int c = w->cnt, s = c + d;
  if (s >= 0) {
    c += 16;
    uint32_t m = (1u << c) - 1;
    if (s >= 8) {
      w_push(w, (uint16_t)(low >> c));
      low &= m;
      c -= 8;
      m >>= 8;
    }
    w_push(w, (uint16_t)(low >> c));
    s = c + d - 24;
    low &= m;
  }
  w->low = low << d;
  w->rng = (rr << d) & 0xFFFF;
  w->cnt = s;
}

/* symbol (ec.rs:520-537) with update_cdf (:935-955) when adapt */
static void w_symbol(writer *w, uint32_t s, uint16_t *cdf, int n, int adapt) {
  const uint32_t fl = s > 0 ? cdf[s - 1] : 32768, fh = cdf[s];
  w_store(w, fl, fh, (uint32_t)(n - (int)s));
  if (!adapt) return;
  int rate = 3 + imin(n >> 1, 2);
  uint16_t *count = &cdf[n - 1];
  rate += *count >> 4;
  *count = (uint16_t)(*count + 1 - (*count >> 5));
  for (int i = 0; i < n - 1 && i < 15; i++) {
    if ((uint32_t)i >= s) cdf[i] = (uint16_t)(cdf[i] - (cdf[i] >> rate));
    else cdf[i] = (uint16_t)(cdf[i] + ((32768 - cdf[i]) >> rate));
  }
}

/* bool / bit, ec.rs:485-496 */
static void w_bool(writer *w, int val, uint32_t f) {
  uint16_t cdf[2] = {(uint16_t)f, 0};
  w_symbol(w, (uint32_t)(val != 0), cdf, 2, 0);
}
static void w_bit(writer *w, int bit) { w_bool(w, bit == 1, 16384); }

/* write_golomb, ec.rs:609-620 */
static void w_golomb(writer *w, uint32_t level) {
  const uint32_t x = level + 1;
  int length = 0;
  while (length < 32 && (x >> length)) length++;
  for (int i = 0; i < length - 1; i++) w_bit(w, 0);
  for (int i = length - 1; i >= 0; i--) w_bit(w, (int)((x >> i) & 1));
}

/* frac_compute, ec.rs:357-379 */
static uint32_t frac_compute(uint32_t nbits_total, uint32_t rng) {
  const uint32_t nbits = nbits_total << 3;
  uint32_t l = 0;
  for (int i = 0; i < 3; i++) {
    rng = (rng * rng) >> 15;
    const uint32_t b = rng >> 16;
    l = (l << 1) | b;
    rng >>= b;
  }
  return nbits - l;
}

/* tell / tell_frac, ec.rs:782-798: stream_bits is s.bits (counter) or precarry.len() * 8 (encoder) */
static uint32_t w_tell_frac(const writer *w) {
  const uint64_t sb = w->enc ? 8 * (uint64_t)w->npre : w->bits;
  return frac_compute((uint32_t)((int64_t)sb + w->cnt + 10), w->rng);
}

/* done, ec.rs:434-473 */
static long w_done(writer *w, uint8_t *out, size_t cap) {
  const uint32_t l = w->low, m = 0x3FFF;
  int c = w->cnt, s = 10 + c;
  uint32_t e = ((l + m) & ~m) | (m + 1);
  if (s > 0) {
    uint32_t n = (1u << (c + 16)) - 1;
    for (;;) {
      w_push(w, (uint16_t)(e >> (c + 16)));
      e &= n;
      s -= 8;
      c -= 8;
      n >>= 8;
      if (s <= 0) break;
    }
  }
  if (w->npre > cap) return -2;
  uint32_t carry = 0;
  for (size_t offs = w->npre; offs > 0; offs--) {
    carry += w->pre[offs - 1];
    out[offs - 1] = (uint8_t)carry;
    carry >>= 8;
  }
  return (long)w->npre;
}

/* ---------------------------------------------------------------- write_coeffs_lv_map */
enum { TX_PAD_HOR = 4, TX_PAD_TOP = 2, TX_PAD_2D = (32 + 4) * (32 + 6) + 16 };

static int64_t coeff_at(const void *q, int is32, size_t i) {
  return is32 ? (int64_t)((const int32_t *)q)[i] : (int64_t)((const int16_t *)q)[i];
}

/* b200_coeff_rate_dev's validity rules (include/b200rdo.h) for one item */
static int item_valid(const orc_coeff_item *it, const void *q, size_t ncoeffs, int is32, const uint16_t *scan) {
  if (it->tx_size >= 19 || it->tx_type >= 16 || it->plane > 2 || it->plane_bsize >= 22 || it->mode > 33) return 0;
  if (it->plane == 0 && it->mode == 13) return 0;
  const int t = it->tx_size, area = orc_coded_tx_area(t);
  if ((uint64_t)it->block * (uint64_t)area + (uint64_t)area > ncoeffs) return 0;
  if (it->eob > area) return 0;
  if (!it->clip_w4 || !it->clip_h4) return 0;
  if (it->x4 + imax(1 << (kWl[t] - 2), it->clip_w4) > 16 || it->y4 + imax(1 << (kHl[t] - 2), it->clip_h4) > 16)
    return 0;
  const size_t base = (size_t)it->block * (size_t)area;
  for (int i = 0; i < area; i++) {
    const int64_t v = coeff_at(q, is32, base + (size_t)i);
    if (v == (is32 ? (int64_t)INT32_MIN : (int64_t)INT16_MIN)) return 0;
  }
  if (it->eob > 0) {
    if (coeff_at(q, is32, base + scan[it->eob - 1]) == 0) return 0;
    if (it->plane == 0) {
      const int set = get_tx_set(t, it->mode >= 14, it->reduced_tx_set);
      if (num_tx_set[set] > 1 && !av1_tx_used[set][it->tx_type]) return 0;
    }
  }
  return 1;
}

typedef struct {
  orc_coeff_cdfs f;
  uint8_t above[3][16], left[3][16];
} chain_state;

/* get_txb_ctx, block_unit.rs:442-526 */
static void get_txb_ctx(const chain_state *cs, const orc_coeff_item *it, int *skip_ctx, int *dc_ctx) {
  const uint8_t *above = &cs->above[it->plane][it->x4], *left = &cs->left[it->plane][it->y4];
  static const int signs[3] = {0, -1, 1};
  int dc_sign = 0;
  for (int i = 0; i < it->clip_w4; i++) dc_sign += signs[above[i] >> 6];
  for (int i = 0; i < it->clip_h4; i++) dc_sign += signs[left[i] >> 6];
  *dc_ctx = dc_sign_contexts[dc_sign + 32];
  const int t = it->tx_size;
  uint32_t top = 0, lft = 0;
  for (int i = 0; i < it->clip_w4; i++) top |= above[i];
  for (int i = 0; i < it->clip_h4; i++) lft |= left[i];
  if (it->plane == 0) {
    if (kBwl[it->plane_bsize] == kWl[t] && kBhl[it->plane_bsize] == kHl[t]) {
      *skip_ctx = 0;
    } else {
      top &= 63;
      lft &= 63;
      const int mx = imin((int)(top | lft), 4), mn = imin(imin((int)top, (int)lft), 4);
      *skip_ctx = skip_contexts[mn][mx];
    }
  } else {
    const int base = (top != 0) + (lft != 0);
    *skip_ctx = base + ((kBwl[it->plane_bsize] + kBhl[it->plane_bsize] > kWl[t] + kHl[t]) ? 10 : 7);
  }
}

/* get_nz_mag, transform_unit.rs:821-844 (levels at the padded position) */
static int get_nz_mag(const uint8_t *lv, int bhl, int cls) {
  int mag = imin(3, lv[1]) + imin(3, lv[(1 << bhl) + TX_PAD_HOR]);
  if (cls == 0) {
    mag += imin(3, lv[(1 << bhl) + TX_PAD_HOR + 1]) + imin(3, lv[2]) + imin(3, lv[(2 << bhl) + (2 << 2)]);
  } else if (cls == 2) {
    mag += imin(3, lv[2]) + imin(3, lv[3]) + imin(3, lv[4]);
  } else {
    mag += imin(3, lv[(2 << bhl) + (2 << 2)]) + imin(3, lv[(3 << bhl) + (3 << 2)]) +
           imin(3, lv[(4 << bhl) + (4 << 2)]);
  }
  return mag;
}

/* get_nz_map_ctx + get_nz_map_ctx_from_stats, transform_unit.rs:846-907 */
static int get_nz_map_ctx(const uint8_t *levels, int pos, int bhl, int area, int c, int is_eob, int t, int cls) {
  if (is_eob) {
    if (c == 0) return 0;
    if (c <= area / 8) return 1;
    if (c <= area / 4) return 2;
    return 3;
  }
  const int padded = pos + ((pos >> bhl) << 2);
  const int stats = get_nz_mag(levels + padded, bhl, cls);
  if ((cls | pos) == 0) return 0;
  const int col = pos >> bhl, row = pos - (col << bhl);
  const int ctx = imin((stats + 1) >> 1, 4);
  if (cls == 0) return ctx + av1_nz_map_ctx_offset[t][imin(row, 4)][imin(col, 4)];
  return ctx + (cls == 1 ? nz_map_ctx_offset_1d[col] : nz_map_ctx_offset_1d[row]);
}

/* get_br_ctx, transform_unit.rs:938-985 */
static int get_br_ctx(const uint8_t *levels, int pos, int bhl, int cls) {
  const int col = pos >> bhl, row = pos - (col << bhl), stride = (1 << bhl) + TX_PAD_HOR, p = col * stride + row;
  int mag = (uint8_t)(levels[p + 1] + levels[p + stride]);
  if (cls == 0) {
    mag += levels[p + stride + 1];
    mag = imin((mag + 1) >> 1, 6);
    if (pos == 0) return mag;
    if (row < 2 && col < 2) return mag + 7;
  } else if (cls == 1) {
    mag += levels[p + (stride << 1)];
    mag = imin((mag + 1) >> 1, 6);
    if (pos == 0) return mag;
    if (col == 0) return mag + 7;
  } else {
    mag += levels[p + 2];
    mag = imin((mag + 1) >> 1, 6);
    if (pos == 0) return mag;
    if (row == 0) return mag + 7;
  }
  return mag + 14;
}

static void set_coeff_context(chain_state *cs, const orc_coeff_item *it, uint8_t value) {
  for (int i = 0; i < (1 << (kWl[it->tx_size] - 2)); i++) cs->above[it->plane][it->x4 + i] = value;
  for (int i = 0; i < (1 << (kHl[it->tx_size] - 2)); i++) cs->left[it->plane][it->y4 + i] = value;
}

static uint16_t *eob_flag_row(orc_coeff_cdfs *f, int multi, int ptype, int ctx, int *n) {
  *n = 5 + imin(multi, 6);
  switch (imin(multi, 6)) {
    case 0: return f->eob_flag16[ptype][ctx];
    case 1: return f->eob_flag32[ptype][ctx];
    case 2: return f->eob_flag64[ptype][ctx];
    case 3: return f->eob_flag128[ptype][ctx];
    case 4: return f->eob_flag256[ptype][ctx];
    case 5: return f->eob_flag512[ptype][ctx];
    default: return f->eob_flag1024[ptype][ctx];
  }
}

/* write_coeffs_lv_map, block_unit.rs:1783-1859, with write_tx_type (transform_unit.rs:530-574), encode_eob
 * (:1861-1914), encode_coeffs (:1916-1981) and encode_coeff_signs (:1983-2016); returns cul_level */
static uint8_t write_item(writer *w, chain_state *cs, const orc_coeff_item *it, const void *q, int is32,
                          const uint16_t *scan) {
  const int t = it->tx_size, eob = it->eob, area = orc_coded_tx_area(t);
  const int height = imin(1 << kHl[t], 32), bhl = imin(kHl[t], 5);
  const size_t base = (size_t)it->block * (size_t)area;
  const int is_inter = it->mode >= 14;
  uint32_t cul_level = 0;
  for (int c = 0; c < eob; c++) {
    const int64_t v = coeff_at(q, is32, base + scan[c]);
    cul_level += (uint32_t)(v < 0 ? -v : v);
  }
  const int txs_ctx = (tx_sqr(t) + tx_sqr_up(t) + 1) >> 1;
  int skip_ctx, dc_ctx;
  get_txb_ctx(cs, it, &skip_ctx, &dc_ctx);
  w_symbol(w, eob == 0, cs->f.txb_skip[txs_ctx][skip_ctx], 2, 1);
  if (eob == 0) {
    set_coeff_context(cs, it, 0);
    return 0;
  }
  uint8_t levels_buf[TX_PAD_2D];
  memset(levels_buf, 0, sizeof(levels_buf));
  uint8_t *levels = levels_buf + TX_PAD_TOP * (height + TX_PAD_HOR);
  for (int i = 0; i < area; i++) { /* txb_init_levels, transform_unit.rs:780-792 */
    const int64_t v = coeff_at(q, is32, base + (size_t)i);
    const int64_t a = v < 0 ? -v : v;
    levels[(i / height) * (height + TX_PAD_HOR) + i % height] = (uint8_t)(a < 127 ? a : 127);
  }
  const int cls = tx_type_to_class[it->tx_type], ptype = it->plane != 0;
  if (it->plane == 0) {
    const int set = get_tx_set(t, is_inter, it->reduced_tx_set);
    if (num_tx_set[set] > 1) {
      const int idx = is_inter ? tx_set_index_inter[set] : tx_set_index_intra[set], sq = tx_sqr(t);
      const uint32_t s = (uint32_t)av1_tx_ind[set][it->tx_type];
      if (is_inter) {
        if (idx == 1) w_symbol(w, s, cs->f.inter_tx_1[sq], 16, 1);
        else if (idx == 2) w_symbol(w, s, cs->f.inter_tx_2[sq], 12, 1);
        else w_symbol(w, s, cs->f.inter_tx_3[sq], 2, 1);
      } else {
        if (idx == 1) w_symbol(w, s, cs->f.intra_tx_1[sq][it->mode], 7, 1);
        else w_symbol(w, s, cs->f.intra_tx_2[sq][it->mode], 5, 1);
      }
    }
  }
  /* encode_eob */
  const int eob_pt = eob < 33 ? eob_to_pos_small[eob] : eob_to_pos_large[imin((eob - 1) >> 5, 16)];
  const int eob_extra = eob - k_eob_group_start[eob_pt];
  int n;
  uint16_t *cdf = eob_flag_row(&cs->f, kWl[t] + kHl[t] - 4, ptype, cls != 0, &n);
  w_symbol(w, (uint32_t)(eob_pt - 1), cdf, n, 1);
  const int eob_offset_bits = k_eob_offset_bits[eob_pt];
  if (eob_offset_bits > 0) {
    int eob_shift = eob_offset_bits - 1;
    w_symbol(w, (eob_extra >> eob_shift) & 1, cs->f.eob_extra[txs_ctx][ptype][eob_pt - 3], 2, 1);
    for (int i = 1; i < eob_offset_bits; i++) {
      eob_shift = eob_offset_bits - 1 - i;
      w_bit(w, (eob_extra >> eob_shift) & 1);
    }
  }
  /* encode_coeffs: get_nz_map_contexts (transform_unit.rs:911-936), then the reverse scan */
  for (int c = eob - 1; c >= 0; c--) {
    const int pos = scan[c];
    const int ctx = get_nz_map_ctx(levels, pos, bhl, area, c, c == eob - 1, t, cls);
    const int64_t v = coeff_at(q, is32, base + (size_t)pos);
    const uint32_t level = (uint32_t)(v < 0 ? -v : v);
    if (c == eob - 1) w_symbol(w, (level < 3 ? level : 3) - 1, cs->f.coeff_base_eob[txs_ctx][ptype][ctx], 3, 1);
    else w_symbol(w, level < 3 ? level : 3, cs->f.coeff_base[txs_ctx][ptype][ctx], 4, 1);
    if (level > 2) {
      const uint32_t base_range = level - 3;
      const int br_ctx = get_br_ctx(levels, pos, bhl, cls);
      for (uint32_t idx = 0; idx < 12; idx += 3) {
        const uint32_t k = base_range - idx < 3 ? base_range - idx : 3;
        w_symbol(w, k, cs->f.coeff_br[imin(txs_ctx, 3)][ptype][br_ctx], 4, 1);
        if (k < 3) break;
      }
    }
  }
  /* encode_coeff_signs */
  for (int c = 0; c < eob; c++) {
    const int64_t v = coeff_at(q, is32, base + scan[c]);
    if (v == 0) continue;
    const uint32_t level = (uint32_t)(v < 0 ? -v : v);
    const int sign = v < 0;
    if (c == 0) w_symbol(w, (uint32_t)sign, cs->f.dc_sign[ptype][dc_ctx], 2, 1);
    else w_bit(w, sign);
    if (level > 14) w_golomb(w, level - 15);
  }
  uint32_t ncl = cul_level < 63 ? cul_level : 63;
  const int64_t dc = coeff_at(q, is32, base + scan[0]);
  if (dc < 0) ncl |= 1u << 6;
  else if (dc > 0) ncl += 2u << 6;
  set_coeff_context(cs, it, (uint8_t)ncl);
  return (uint8_t)ncl;
}

/* validity of a whole chain; fills scans[i] for its items */
static int chain_valid(size_t ncdfs, const orc_coeff_chain *ch, const orc_coeff_item *items, size_t nitems,
                       const void *q, size_t ncoeffs, int is32, uint16_t (*scans)[1024]) {
  if (ch->snapshot >= ncdfs || ch->init_rng < 32768 || ch->init_rng > 65535) return 0;
  if ((uint64_t)ch->item_begin + ch->item_count > nitems) return 0;
  for (uint32_t i = 0; i < ch->item_count; i++) {
    const orc_coeff_item *it = &items[ch->item_begin + i];
    if (it->tx_size >= 19 || it->tx_type >= 16) return 0;
    orc_scan_order(it->tx_size, it->tx_type, scans[i], NULL);
    if (!item_valid(it, q, ncoeffs, is32, scans[i])) return 0;
  }
  return 1;
}

static int run_chain(writer *w, const orc_coeff_cdfs *cdfs, size_t ncdfs, const orc_coeff_chain *ch,
                     const orc_coeff_item *items, size_t nitems, const void *q, size_t ncoeffs, int is32,
                     uint8_t *cul_level) {
  uint16_t(*scans)[1024] = (uint16_t(*)[1024])malloc((ch->item_count ? ch->item_count : 1) * sizeof(*scans));
  chain_state *cs = (chain_state *)malloc(sizeof(chain_state));
  int ok = scans && cs && chain_valid(ncdfs, ch, items, nitems, q, ncoeffs, is32, scans);
  if (ok) {
    cs->f = cdfs[ch->snapshot];
    memcpy(cs->above, ch->above, sizeof(cs->above));
    memcpy(cs->left, ch->left, sizeof(cs->left));
    for (uint32_t i = 0; i < ch->item_count; i++) {
      const uint8_t cl = write_item(w, cs, &items[ch->item_begin + i], q, is32, scans[i]);
      if (cul_level) cul_level[ch->item_begin + i] = cl;
    }
  }
  free(scans);
  free(cs);
  return ok;
}

void orc_coeff_rate(const orc_coeff_cdfs *cdfs, size_t ncdfs, const orc_coeff_chain *chains, size_t nchains,
                    const orc_coeff_item *items, size_t nitems, const void *qcoeffs, size_t ncoeffs, int coeff_is_i32,
                    uint32_t *rate, uint8_t *cul_level) {
  init_tables();
#pragma omp parallel for schedule(dynamic, 16)
  for (long c = 0; c < (long)nchains; c++) {
    writer w;
    w_init(&w, 0, chains[c].init_rng);
    const uint32_t start = w_tell_frac(&w);
    if (run_chain(&w, cdfs, ncdfs, &chains[c], items, nitems, qcoeffs, ncoeffs, coeff_is_i32, cul_level))
      rate[c] = w_tell_frac(&w) - start;
    else
      rate[c] = UINT32_MAX;
  }
}

long orc_coeff_encode_chain(const orc_coeff_cdfs *cdfs, size_t ncdfs, const orc_coeff_chain *chain,
                            const orc_coeff_item *items, size_t nitems, const void *qcoeffs, size_t ncoeffs,
                            int coeff_is_i32, uint8_t *out, size_t cap, uint32_t *tell_frac, long *nsymbols) {
  init_tables();
  if (chain->init_rng != 32768) return -1;
  writer we, wc;
  w_init(&we, 1, 32768);
  w_init(&wc, 0, 32768);
  if (!run_chain(&we, cdfs, ncdfs, chain, items, nitems, qcoeffs, ncoeffs, coeff_is_i32, NULL)) return -1;
  run_chain(&wc, cdfs, ncdfs, chain, items, nitems, qcoeffs, ncoeffs, coeff_is_i32, NULL);
  tell_frac[0] = w_tell_frac(&we);
  tell_frac[1] = w_tell_frac(&wc);
  *nsymbols = we.nsym;
  const long n = we.oom ? -2 : w_done(&we, out, cap);
  free(we.pre);
  return n;
}

long orc_ec_encode_script(const int32_t *ops, size_t nops, const uint16_t *cdf, int ncdf, uint8_t *out, size_t cap,
                          uint32_t *tell_frac) {
  writer we, wc;
  w_init(&we, 1, 32768);
  w_init(&wc, 0, 32768);
  uint16_t *c = (uint16_t *)malloc((size_t)(ncdf > 0 ? ncdf : 1) * sizeof(uint16_t));
  for (size_t k = 0; k < nops; k++) {
    const int32_t kind = ops[3 * k], s = ops[3 * k + 1], f = ops[3 * k + 2];
    for (writer *w = &we; w; w = w == &we ? &wc : NULL) {
      if (kind == 0) {
        w_bool(w, s, (uint32_t)f);
      } else {
        memcpy(c, cdf, (size_t)ncdf * sizeof(uint16_t));
        w_symbol(w, (uint32_t)s, c, ncdf, 0);
      }
    }
  }
  free(c);
  tell_frac[0] = w_tell_frac(&we);
  tell_frac[1] = w_tell_frac(&wc);
  const long n = we.oom ? -2 : w_done(&we, out, cap);
  free(we.pre);
  return n;
}
