/* tx_size_type.c — CPU restatement of rav1e's intra transform size and type decision (TEST INFRASTRUCTURE
 * ONLY, see oracle.h and tx_size_type.h).
 *
 *   rdo_tx_size_type            src/rdo.rs:725-802
 *   rdo_tx_type_decision        src/rdo.rs:1701-1823
 *   write_tx_blocks (luma)      src/encoder.rs:2243-2311
 *   encode_tx_block             src/encoder.rs:1404-1658
 *   compute_distortion          src/rdo.rs:254-307 (luma only), compute_tx_distortion :310-394
 *   cdef_dist_wxh / sse_wxh     src/rdo.rs:142-224, clip_visible_bsize :228-250
 *   max_txsize_rect_lookup, sub_tx_size_map, get_tx_set   context/transform_unit.rs:60-148
 *   RAV1E_TX_TYPES              transform/mod.rs:28-44
 *
 * Serial and literal: one candidate after the other in the reference's order, each from the same
 * coefficient-context checkpoint.  The partition's reconstruction lives in a private window: the
 * reference writes each candidate's prediction and reconstruction into `rec` and the next candidate
 * overwrites them before reading them, so what a candidate reads inside the partition is only its own.
 * The orchestration has no stored vectors upstream ("parity unpinned"); tests/test_oracle_tx_size_type.py
 * checks it against an independent Python restatement driving the same pieces.
 */
#include "tx_size_type.h"

#include <float.h>
#include <stdlib.h>
#include <string.h>

#include "oracle.h"

static const uint8_t BS_W[22] = {4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 64, 128, 128, 4, 16, 8, 32, 16, 64};
static const uint8_t BS_H[22] = {4, 8, 4, 8, 16, 8, 16, 32, 16, 32, 64, 32, 64, 128, 64, 128, 16, 4, 32, 8, 64, 16};
static const uint8_t MAX_TX[22] = {0, 5, 6, 1, 7, 8, 2, 9, 10, 3, 11, 12, 4, 4, 4, 4, 13, 14, 15, 16, 17, 18};
static const uint8_t SUB_TX[19] = {0, 0, 1, 2, 3, 0, 0, 1, 1, 2, 2, 3, 3, 5, 6, 7, 8, 9, 10};
static const uint8_t TX_TYPES[7] = {0, 1, 2, 3, 9, 10, 11}; /* DCT_DCT ADST_DCT DCT_ADST ADST_ADST IDTX V_DCT H_DCT */
enum { SET_DCTONLY = 0, SET_INTRA_2 = 2, SET_INTRA_1 = 3 };

static int ilog2i(int v) { return 31 - __builtin_clz((unsigned)v); }

/* get_tx_set (transform_unit.rs:123-148) for intra */
static int intra_tx_set(int t, int reduced) {
  const int wl = ilog2i(orc_tx_width(t)), hl = ilog2i(orc_tx_height(t));
  const int up = (wl > hl ? wl : hl) - 2, sq = (wl < hl ? wl : hl) - 2;
  if (up >= 3) return SET_DCTONLY;
  return (reduced || sq == 2) ? SET_INTRA_2 : SET_INTRA_1;
}
/* av1_tx_used (transform_unit.rs:19-58) of the intra sets */
static int tx_used(int set, int type) {
  if (set == SET_DCTONLY) return type == 0;
  if (set == SET_INTRA_2) return type <= 3 || type == 9;
  return 1;
}

static int item_valid(const orc_tx_item *it, int rect_w, int rect_h, size_t ncdfs) {
  if (it->bsize >= 22 || (it->bsize >= 13 && it->bsize <= 15) || it->mode >= 13) return 0;
  if (it->x < 0 || it->y < 0 || it->x >= rect_w || it->y >= rect_h || (it->x & 3) || (it->y & 3)) return 0;
  if (it->dc_quant < 1 || it->dc_quant > 65535 || it->ac_quant < 1 || it->ac_quant > 65535) return 0;
  return it->snapshot < ncdfs;
}

typedef struct {
  const uint8_t *rec0, *src0;
  ptrdiff_t rec_stride, src_stride;
  int bpp, plane_w, plane_h, rect_x, rect_y, rect_w, rect_h, frame_w, frame_h, bit_depth, dist_mode, reduced;
  double lambda_;
  uint32_t dist_scale;
  const uint32_t *scale4x4;
  size_t scale_stride;
  const orc_coeff_cdfs *cdfs;
  size_t ncdfs;
  int ws; /* the window's stride: rect_w + 64 */
} call_t;

static uint32_t bias(const call_t *c, int fx4, int fy4) { /* distortion_scale, rdo.rs:443-459 */
  return c->scale4x4 ? c->scale4x4[(size_t)fy4 * c->scale_stride + (size_t)fx4] : 1u << 14;
}
static int getpx(const uint8_t *p, ptrdiff_t i, int bpp) { return bpp == 1 ? p[i] : ((const uint16_t *)p)[i]; }
static void setpx(uint8_t *p, ptrdiff_t i, int bpp, int v) {
  if (bpp == 1) p[i] = (uint8_t)v;
  else ((uint16_t *)p)[i] = (uint16_t)v;
}

/* The window: region coordinates [0, rect_w + 64) x [0, rect_h + 64) (a partition may reach 63 px past the
 * region), pixel (xx, yy) at WOFF(xx, yy).  Only the pixels an item reads are loaded. */
#define WOFF(xx, yy) ((ptrdiff_t)(yy) * c->ws + (xx))

static void load_window(const call_t *c, const orc_tx_item *it, uint8_t *win) {
  const int x0 = it->x, y0 = it->y, bw = BS_W[it->bsize], bh = BS_H[it->bsize];
  const int rw = c->rect_w < c->plane_w - c->rect_x ? c->rect_w : c->plane_w - c->rect_x;
  const int rh = c->rect_h < c->plane_h - c->rect_y ? c->rect_h : c->plane_h - c->rect_y;
  const uint8_t *reg = c->rec0 + ((ptrdiff_t)c->rect_y * c->rec_stride + c->rect_x) * c->bpp;
  /* get_intra_edges reads inside the region only: the line above and the rows of the partition up to 64
     px past its right side, and the column left of it up to 64 px below */
  for (int yy = y0 - 1 > 0 ? y0 - 1 : 0; yy < y0 + bh + 64 && yy < rh; yy++) {
    const int xe = yy < y0 + bh ? x0 + bw + 64 : x0;
    for (int xx = x0 - 1 > 0 ? x0 - 1 : 0; xx < xe && xx < rw; xx++)
      setpx(win, WOFF(xx, yy), c->bpp, getpx(reg, (ptrdiff_t)yy * c->rec_stride + xx, c->bpp));
  }
}

/* One candidate of rdo_tx_type_decision: write_tx_blocks' luma loop with the counter, then the
 * distortion.  win holds rec around the partition and receives this candidate's reconstruction. */
static void eval_candidate(const call_t *c, const orc_tx_item *it, int tx, int type, uint8_t *win, uint32_t *rate_out,
                           uint64_t *dist_out) {
  const int bpp = c->bpp, is32 = bpp == 2, bs = it->bsize;
  const int x0 = it->x, y0 = it->y, bw = BS_W[bs], bh = BS_H[bs];
  const int tw = orc_tx_width(tx), th = orc_tx_height(tx), coded = orc_coded_tx_area(tx);
  const int nbx = bw / tw, nby = bh / th;
  const int mi_w = (c->rect_w + 3) >> 2, mi_h = (c->rect_h + 3) >> 2;
  const int w_in_b = 2 * ((c->frame_w + 7) >> 3), h_in_b = 2 * ((c->frame_h + 7) >> 3);
  const int need_recon_pixel = tw != bw || th != bh;
  const uint8_t *src = c->src0 + ((ptrdiff_t)c->rect_y * c->src_stride + c->rect_x) * bpp;
  int32_t qbuf[16 * 1024];
  orc_coeff_item items[16];
  uint64_t tx_dist = 0;
  int nk = 0;
  for (int by = 0; by < nby; by++)
    for (int bx = 0; bx < nbx; bx++) {
      const int px = x0 + bx * tw, py = y0 + by * th; /* the tx block in the region */
      if ((px >> 2) >= mi_w || (py >> 2) >= mi_h) continue; /* encoder.rs:2282 */
      /* get_intra_edges + predict_intra (encoder.rs:1468-1499, predict.rs:205-249) */
      uint16_t edge[4 * 64 + 1];
      int init_left = 0, init_above = 0;
      orc_get_intra_edges(edge, win, c->ws, bpp, c->plane_w, c->plane_h, c->rect_x, c->rect_y, c->rect_w, c->rect_h,
                          0, 0, x0 >> 2, y0 >> 2, bx, by, bs, px, py, tw, th, c->bit_depth, it->mode, it->ief >= 0, 0,
                          &init_left, &init_above);
      const int variant = px == 0 && py == 0 ? 0 : py == 0 ? 1 : px == 0 ? 2 : 3;
      int mode = it->mode;
      if (mode == 12) mode = variant == 0 ? 0 : variant == 2 ? 1 : variant == 1 ? 2 : 12;
      static const int ANGLE[9] = {0, 90, 180, 45, 135, 113, 157, 203, 67};
      const int angle = mode >= 1 && mode <= 8 ? ANGLE[mode] : 0;
      const int ief = it->mode >= 1 && it->mode <= 8 ? it->ief : -1;
      uint8_t *dst = win + WOFF(px, py) * bpp;
      orc_predict_intra(mode, variant, dst, c->ws, bpp, tw, th, c->bit_depth, NULL, angle, ief, edge, init_left,
                        init_above, c->plane_w, c->plane_h, c->rect_x + px, c->rect_y + py);
      /* residual (zero when invisible), forward_transform, quantize, dequantize, raw tx distortion */
      const int fx = c->rect_x + px, fy = c->rect_y + py;
      const int visible = fx < c->frame_w && fy < c->frame_h;
      int16_t residual[64 * 64];
      for (int r = 0; r < th; r++)
        for (int k = 0; k < tw; k++)
          residual[r * tw + k] = visible ? (int16_t)(getpx(src, (ptrdiff_t)(py + r) * c->src_stride + px + k, bpp) -
                                                     getpx(dst, (ptrdiff_t)r * c->ws + k, bpp))
                                         : 0;
      int32_t coeffs[64 * 64], rcoeffs[32 * 32];
      orc_forward_transform(residual, coeffs, tw, tx, type, c->bit_depth, is32);
      uint16_t eob;
      uint64_t raw;
      void *q = is32 ? (void *)(qbuf + nk * coded) : (void *)((int16_t *)qbuf + nk * coded);
      orc_quantize_chain_batch(coeffs, 1, tx, type, it->dc_quant, it->ac_quant, 1, is32, q, rcoeffs, &eob, &raw, 1);
      /* write_coeffs_lv_map's item: frame_clipped_txw / txh (encoder.rs:1561-1566) */
      const int cw = ((w_in_b - (fx >> 2)) << 2) < tw ? ((w_in_b - (fx >> 2)) << 2) : tw;
      const int ch = ((h_in_b - (fy >> 2)) << 2) < th ? ((h_in_b - (fy >> 2)) << 2) : th;
      orc_coeff_item ci = {(uint32_t)nk, eob, (uint8_t)tx, (uint8_t)type, 0, (uint8_t)bs, it->mode,
                           (uint8_t)c->reduced, (uint8_t)(bx * tw / 4), (uint8_t)(by * th / 4), (uint8_t)(cw >> 2),
                           (uint8_t)(ch >> 2)};
      items[nk++] = ci;
      if (eob > 0 && (need_recon_pixel || c->dist_mode != 0))
        orc_inverse_transform_add(rcoeffs, is32, dst, c->ws, bpp, tx, type, c->bit_depth);
      if (c->dist_mode == 0 && visible) /* RawDistortion * bias * dist_scale[0] (encoder.rs:1642-1652) */
        tx_dist += orc_distortion_scale_mul(c->dist_scale, orc_distortion_scale_mul(bias(c, fx >> 2, fy >> 2), raw));
    }
  orc_coeff_chain chain;
  memset(&chain, 0, sizeof chain);
  chain.snapshot = it->snapshot;
  chain.init_rng = 32768; /* WriterCounter::new() */
  chain.item_count = (uint32_t)nk;
  memcpy(chain.above[0], it->above, 16);
  memcpy(chain.left[0], it->left, 16);
  uint32_t rate = 0;
  orc_coeff_rate(c->cdfs, c->ncdfs, &chain, 1, items, (size_t)nk, qbuf, (size_t)nk * coded, is32, &rate, NULL);
  *rate_out = rate;
  if (c->dist_mode == 0) {
    *dist_out = tx_dist;
    return;
  }
  /* compute_distortion's luma term over the visible block (rdo.rs:254-293) */
  const int fx0 = c->rect_x + x0, fy0 = c->rect_y + y0;
  const int vw = fx0 + bw <= c->frame_w ? bw : fx0 >= c->frame_w ? 0 : c->frame_w - fx0;
  const int vh = fy0 + bh <= c->frame_h ? bh : fy0 >= c->frame_h ? 0 : c->frame_h - fy0;
  if (vw == 0 || vh == 0) {
    *dist_out = 0;
    return;
  }
  const uint8_t *s = src + ((ptrdiff_t)y0 * c->src_stride + x0) * bpp, *d = win + WOFF(x0, y0) * bpp;
  uint64_t dist = 0;
  if (c->dist_mode == 1) { /* sse_wxh: the bias of every 4x4 chunk */
    uint32_t sc[16 * 16];
    const int nw = (vw + 3) >> 2, nh = (vh + 3) >> 2;
    for (int cy = 0; cy < nh; cy++)
      for (int cx = 0; cx < nw; cx++) sc[cy * nw + cx] = bias(c, (fx0 >> 2) + cx, (fy0 >> 2) + cy);
    dist = bpp == 1 ? orc_weighted_sse_u8(s, c->src_stride, d, c->ws, sc, (size_t)nw, vw, vh)
                    : orc_weighted_sse_u16((const uint16_t *)s, c->src_stride, (const uint16_t *)d, c->ws, sc,
                                           (size_t)nw, vw, vh);
  } else { /* cdef_dist_wxh: 8x8 steps, each with its own bias */
    for (int yy = 0; yy < vh; yy += 8)
      for (int xx = 0; xx < vw; xx += 8) {
        const int kw = vw - xx < 8 ? vw - xx : 8, kh = vh - yy < 8 ? vh - yy : 8;
        const uint32_t v =
            bpp == 1 ? orc_cdef_dist_kernel_u8(s + (ptrdiff_t)yy * c->src_stride + xx, c->src_stride,
                                               d + (ptrdiff_t)yy * c->ws + xx, c->ws, kw, kh, c->bit_depth, NULL)
                     : orc_cdef_dist_kernel_u16((const uint16_t *)s + (ptrdiff_t)yy * c->src_stride + xx,
                                                c->src_stride, (const uint16_t *)d + (ptrdiff_t)yy * c->ws + xx, c->ws,
                                                kw, kh, c->bit_depth, NULL);
        dist += orc_distortion_scale_mul(bias(c, (fx0 + xx) >> 2, (fy0 + yy) >> 2), v);
      }
  }
  *dist_out = orc_distortion_scale_mul(c->dist_scale, dist);
}

static void decide(const call_t *c, const orc_tx_item *it, uint8_t *win, orc_tx_best *best, orc_tx_cand *cands) {
  load_window(c, it, win);
  int tx = MAX_TX[it->bsize];
  int best_size = tx, best_type = 0;
  double best_rd = DBL_MAX;
  for (int l = 0; l < 3; l++) {
    orc_tx_cand *row = cands + l * 7;
    if (tx < 0) { /* the ladder stopped */
      for (int k = 0; k < 7; k++) row[k] = (orc_tx_cand){0, 0, 0, ORC_TX_NOT_IN_LADDER};
      continue;
    }
    const int set = intra_tx_set(tx, c->reduced);
    const int all = set != SET_DCTONLY && !it->skip; /* do_rdo_tx_type, rdo.rs:751-761 */
    int first = 1, cut = 0, size_type = 0;
    double size_rd = DBL_MAX;
    for (int k = 0; k < 7; k++) {
      const int type = TX_TYPES[k];
      if (!(all || k == 0) || !tx_used(set, type)) {
        row[k] = (orc_tx_cand){0, 0, 0, ORC_TX_NOT_IN_SET};
        continue;
      }
      if (cut) {
        row[k] = (orc_tx_cand){0, 0, 0, ORC_TX_CUT};
        continue;
      }
      uint32_t rate;
      uint64_t dist;
      eval_candidate(c, it, tx, type, win, &rate, &dist);
      const double rd = orc_compute_rd_cost(c->lambda_, rate, dist);
      row[k] = (orc_tx_cand){rd, dist, rate, ORC_TX_EVALUATED};
      if (first) { /* rdo.rs:1806-1815 */
        first = 0;
        if (rd > best_rd) {
          cut = 1;
          continue;
        }
      }
      if (rd < size_rd) {
        size_rd = rd;
        size_type = type;
      }
    }
    if (size_rd < best_rd) { /* rdo.rs:780-784 */
      best_size = tx;
      best_type = size_type;
      best_rd = size_rd;
    }
    const int next = SUB_TX[tx];
    tx = next == tx ? -1 : next;
  }
  best->rd = best_rd;
  best->tx_size = (uint8_t)best_size;
  best->tx_type = (uint8_t)best_type;
  memset(best->pad_, 0, sizeof best->pad_);
}

void orc_intra_tx_size_type(const void *rec0, ptrdiff_t rec_stride, const void *src0, ptrdiff_t src_stride, int bpp,
                            int plane_w, int plane_h, int rect_x, int rect_y, int rect_w, int rect_h, int frame_w,
                            int frame_h, int bit_depth, int dist_mode, int reduced_tx_set, double lambda,
                            uint32_t dist_scale, const uint32_t *scale4x4, size_t scale_stride,
                            const orc_coeff_cdfs *cdfs, size_t ncdfs, const orc_tx_item *items, size_t n,
                            orc_tx_best *best, orc_tx_cand *cands, int threads) {
  const call_t c = {(const uint8_t *)rec0, (const uint8_t *)src0, rec_stride, src_stride, bpp, plane_w, plane_h,
                    rect_x, rect_y, rect_w, rect_h, frame_w, frame_h, bit_depth, dist_mode, reduced_tx_set, lambda,
                    dist_scale, scale4x4, scale_stride, cdfs, ncdfs, rect_w + 64};
#pragma omp parallel num_threads(threads > 0 ? threads : orc_num_threads())
  {
    uint8_t *win = (uint8_t *)malloc((size_t)(rect_h + 64) * (size_t)c.ws * 2);
#pragma omp for schedule(dynamic, 4)
  for (long i = 0; i < (long)n; i++) {
    orc_tx_cand tmp[21];
    orc_tx_cand *cd = cands ? cands + (size_t)i * 21 : tmp;
    if (!item_valid(&items[i], rect_w, rect_h, ncdfs)) {
      best[i] = (orc_tx_best){-1.0, 0xFF, 0xFF, {0}};
      for (int k = 0; k < 21; k++) cd[k] = (orc_tx_cand){0, 0, 0, ORC_TX_INVALID};
      continue;
    }
    decide(&c, &items[i], win, &best[i], cd);
  }
    free(win);
  }
}
