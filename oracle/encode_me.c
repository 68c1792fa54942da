/*
 * oracle/encode_me.c — the encode-time motion search, serially per item: get_subset_predictors (me.rs:386-534)
 * in CORNER mode with tile-local subset B, and estimate_motion (me.rs:536-632) with a pmv and no extensive search.
 * TEST INFRASTRUCTURE ONLY (see oracle.h); declared in encode_me.h.
 *
 * The stages after the gathering are me.c's: orc_full_pixel_me_blocks with one subset (all_mvs, me.rs:757-759),
 * orc_fullpel_candidates with SATD for the re-measure (me.rs:596-616) and orc_subpel_diamond_search_blocks for
 * sub_pixel_me (me.rs:857-882), each called on the items of one (block size, slot) group.
 */
#include "encode_me.h"

#include <stdlib.h>

#define MI_SIZE 4 /* context/superblock_unit.rs:12 */

static const int TXW[19] = {4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64};
static const int TXH[19] = {4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16};

static inline int imin(int a, int b) { return a < b ? a : b; }
static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

typedef struct {
  int mvx_min, mvx_max, mvy_min, mvy_max;
  uint32_t min_sad;
} gather;

/* process_cand, me.rs:405-412: min_sad, quantize_to_fullpel (i16 `/ 8 * 8`), clamp to the range */
static orc_mv proc_cand(gather *g, orc_me_stats st) {
  if (st.normalized_sad < g->min_sad) g->min_sad = st.normalized_sad;
  orc_mv mv;
  mv.col = (int16_t)clampi((st.mv_col / 8) * 8, g->mvx_min, g->mvx_max);
  mv.row = (int16_t)clampi((st.mv_row / 8) * 8, g->mvy_min, g->mvy_max);
  return mv;
}

/* me.rs:386-534 with corner = CORNER { right: true, bottom: true } and ssdec = 0 (dec_mv is the identity) */
int orc_enc_subset_predictors(const orc_me_stats *stats, const orc_me_stats *prev, int w_in_b, int h_in_b,
                              int tile_w_sb, int tile_h_sb, int x4, int y4, int w, int h, orc_mv *out,
                              uint32_t *min_sad) {
  gather g;
  orc_get_mv_range(w_in_b, h_in_b, x4, y4, w, h, &g.mvx_min, &g.mvx_max, &g.mvy_min, &g.mvy_max);
  g.min_sad = UINT32_MAX;
  /* the block's tile: TileMEStats over the 8-aligned frame, the last tiles cropped (tile_state.rs:130-176) */
  const int tw = tile_w_sb * 16, th = tile_h_sb * 16;
  const int tx0 = x4 / tw * tw, ty0 = y4 / th * th;
  const int cols = imin(tw, w_in_b - tx0), rows = imin(th, h_in_b - ty0);
  const int bx = x4 - tx0, by = y4 - ty0; /* tile_bo */
#define TS(x, y) stats[(size_t)(ty0 + (y)) * w_in_b + tx0 + (x)]
  const int wb = (w + MI_SIZE - 1) >> 2, hb = (h + MI_SIZE - 1) >> 2; /* me.rs:397-398 */
  const int chw = imin(wb >> 1, cols - 1 - bx), chh = imin(hb >> 1, rows - 1 - by); /* :402-403 */
  orc_mv b[5], c[5];
  int nb = 0, nc = 0;
  if (bx > 0) b[nb++] = proc_cand(&g, TS(bx - 1, by + chh));        /* left, :420-424 */
  if (by > 0) b[nb++] = proc_cand(&g, TS(bx + chw, by - 1));        /* top, :426-430 */
  if (bx + wb < cols) b[nb++] = proc_cand(&g, TS(bx + wb, by + chh)); /* right, :437-443 */
  if (by + hb < rows) b[nb++] = proc_cand(&g, TS(bx + chw, by + hb)); /* bottom, :445-451 */
  const orc_mv median = proc_cand(&g, TS(bx + chw, by + chh));       /* centre, :453-458 */
#undef TS
  b[nb].row = b[nb].col = 0; /* zero vector, :470 */
  nb++;
  if (prev) { /* subset C, :477-515: frame coordinates */
    const int fx = x4, fy = y4;
    const int hw = imin(wb >> 1, w_in_b - 1 - fx), hh = imin(hb >> 1, h_in_b - 1 - fy);
#define PS(x, y) prev[(size_t)(y) * w_in_b + (x)]
    if (fx > 0) c[nc++] = proc_cand(&g, PS(fx - 1, fy + hh));
    if (fy > 0) c[nc++] = proc_cand(&g, PS(fx + hw, fy - 1));
    if (fx + wb < w_in_b) c[nc++] = proc_cand(&g, PS(fx + wb, fy + hh));
    if (fy + hb < h_in_b) c[nc++] = proc_cand(&g, PS(fx + hw, fy + hb));
    c[nc++] = proc_cand(&g, PS(fx + hw, fy + hh));
#undef PS
  }
  if (min_sad) *min_sad = (uint32_t)(((uint64_t)g.min_sad * (uint64_t)(w * h)) >> 14); /* :518-519 */
  int n = 0; /* all_mvs, :372-382 */
  out[n++] = median;
  for (int i = 0; i < nb; i++) out[n++] = b[i];
  for (int i = 0; i < nc; i++) out[n++] = c[i];
  return n;
}

/* estimate_motion, me.rs:536-632, for the items of one (size, slot) group at once */
void orc_estimate_motion_items(const void *src0, ptrdiff_t src_stride, const void *const *refs,
                               const ptrdiff_t *ref_stride, int nslots, int bpp, int width, int height,
                               const orc_me_stats *stats, const orc_me_stats *prev, const uint8_t *has_prev,
                               int bit_depth, int allow_hp, double me_lambda, int use_satd, int filter_mode,
                               int tile_w_sb, int tile_h_sb, const uint32_t size_end[19],
                               const orc_enc_me_item *items, size_t nitems, orc_me_result *out, int threads) {
  const int w_in_b = 2 * ((width + 7) >> 3), h_in_b = 2 * ((height + 7) >> 3);
  const size_t ncells = (size_t)w_in_b * h_in_b;
  /* me.rs:549-552: (fi.me_lambda * 256.0 * 0.5) as u32, saturating */
  const double l = me_lambda * 256.0 * 0.5;
  const uint32_t lambda = !(l > 0.0) ? 0u : l >= 4294967295.0 ? UINT32_MAX : (uint32_t)l;
  for (size_t i = 0; i < nitems; i++) {
    out[i].cost = UINT64_MAX;
    out[i].sad = UINT32_MAX;
    out[i].mv.row = out[i].mv.col = 0;
  }
  orc_block *blocks = malloc(sizeof(orc_block) * (nitems + 1));
  orc_mv *pmv = malloc(sizeof(orc_mv) * 2 * (nitems + 1));
  orc_cand *preds = malloc(sizeof(orc_cand) * 11 * (nitems + 1));
  orc_cand *best_mv = malloc(sizeof(orc_cand) * (nitems + 1));
  uint32_t *offs = malloc(sizeof(uint32_t) * (nitems + 2));
  size_t *idx = malloc(sizeof(size_t) * (nitems + 1));
  orc_me_result *res = malloc(sizeof(orc_me_result) * (nitems + 1));
  uint32_t *sad = malloc(sizeof(uint32_t) * (nitems + 1));
  uint64_t *cost = malloc(sizeof(uint64_t) * (nitems + 1));
  for (int s = 0; s < 19; s++) {
    const size_t lo = s ? size_end[s - 1] : 0, hi = size_end[s];
    const int w = TXW[s], h = TXH[s];
    for (int slot = 0; slot < nslots; slot++) {
      const orc_me_stats *S = stats + (size_t)slot * ncells;
      const orc_me_stats *P = prev && has_prev[slot] ? prev + (size_t)slot * ncells : NULL;
      size_t n = 0;
      offs[0] = 0;
      for (size_t i = lo; i < hi; i++) {
        const orc_enc_me_item it = items[i];
        if (it.slot != slot || it.x4 >= w_in_b || it.y4 >= h_in_b) continue;
        blocks[n].x = (int16_t)(it.x4 * MI_SIZE);
        blocks[n].y = (int16_t)(it.y4 * MI_SIZE);
        pmv[2 * n].row = it.pmv[0][0], pmv[2 * n].col = it.pmv[0][1];
        pmv[2 * n + 1].row = it.pmv[1][0], pmv[2 * n + 1].col = it.pmv[1][1];
        orc_mv mv[11];
        const int k = orc_enc_subset_predictors(S, P, w_in_b, h_in_b, tile_w_sb, tile_h_sb, it.x4, it.y4, w, h, mv,
                                                NULL);
        for (int j = 0; j < k; j++) {
          orc_cand *q = &preds[offs[n] + j];
          q->block = (uint32_t)n;
          q->mv_row = mv[j].row;
          q->mv_col = mv[j].col;
        }
        offs[n + 1] = offs[n] + (uint32_t)k;
        idx[n++] = i;
      }
      if (n == 0) continue;
      /* full_pixel_me's non-extensive branch: try_cands(all_mvs), me.rs:757-759 */
      orc_full_pixel_me_blocks(src0, src_stride, refs[slot], ref_stride[slot], bpp, w_in_b, h_in_b, blocks, n, preds,
                               offs, 1, pmv, NULL, w, h, lambda, allow_hp, 0, res, threads);
      /* the items whose full-pel result is empty (no candidate in range) keep the empty result */
      size_t m = 0;
      for (size_t j = 0; j < n; j++) {
        if (res[j].cost == UINT64_MAX) continue;
        blocks[m] = blocks[j];
        pmv[2 * m] = pmv[2 * j];
        pmv[2 * m + 1] = pmv[2 * j + 1];
        res[m] = res[j];
        idx[m] = idx[j];
        m++;
      }
      if (m == 0) continue;
      if (use_satd) { /* best.rd = get_fullpel_mv_rd(.., use_satd, .., best.mv), me.rs:596-616 */
        for (size_t j = 0; j < m; j++) {
          best_mv[j].block = (uint32_t)j;
          best_mv[j].mv_row = res[j].mv.row;
          best_mv[j].mv_col = res[j].mv.col;
        }
        orc_fullpel_candidates(src0, src_stride, refs[slot], ref_stride[slot], bpp, w_in_b, h_in_b, blocks, best_mv,
                               m, w, h, 1, lambda, pmv, allow_hp, sad, cost, threads);
        for (size_t j = 0; j < m; j++) res[j].sad = sad[j], res[j].cost = cost[j];
      }
      /* sub_pixel_me, me.rs:857-882 */
      orc_subpel_diamond_search_blocks(src0, src_stride, refs[slot], ref_stride[slot], bpp, w_in_b, h_in_b, blocks, m,
                                       w, h, use_satd, lambda, pmv, allow_hp, filter_mode, bit_depth, res, threads);
      for (size_t j = 0; j < m; j++) out[idx[j]] = res[j];
    }
  }
  free(blocks);
  free(pmv);
  free(preds);
  free(best_mv);
  free(offs);
  free(idx);
  free(res);
  free(sad);
  free(cost);
}
