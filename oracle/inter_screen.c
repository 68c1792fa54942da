/* inter_screen.c — CPU restatement of rav1e's inter mode screening (TEST INFRASTRUCTURE ONLY, see
 * oracle.h and inter_screen.h).
 *
 *   inter_frame_rdo_mode_decision's SATD pruning   src/rdo.rs:1281-1363
 *   PredictionMode::predict_inter (+ _single,     src/predict.rs:284-421
 *     _compound, get_mv_params)
 *   PlaneSlice::clamp                              v_frame 0.3.9 (off disk; published semantics)
 *
 * Composed of orc_get_mv_params, orc_put_8tap, orc_prep_8tap, orc_mc_avg and orc_get_satd_*, plus the
 * clamp and a stable sort.
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "inter_screen.h"
#include "oracle.h"

enum { ENTRIES = 20 };

/* BlockSize (partition.rs:130-153) -> width, height; 0 for the 128-sided sizes */
static const uint8_t BS_W[22] = {4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 0, 0, 0, 4, 16, 8, 32, 16, 64};
static const uint8_t BS_H[22] = {4, 8, 4, 8, 16, 8, 16, 32, 16, 32, 64, 32, 64, 0, 0, 0, 16, 4, 32, 8, 64, 16};

static int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

static int item_valid(const orc_inter_screen_item *it, int rect_w, int rect_h, int nrefs) {
  if (it->bsize >= 22 || BS_W[it->bsize] == 0 || it->n > ENTRIES) return 0;
  if (it->x < 0 || it->y < 0 || it->x >= rect_w || it->y >= rect_h || (it->x & 3) || (it->y & 3)) return 0;
  for (int k = 0; k < it->n; k++) {
    if (it->cands[k].ref[0] >= nrefs) return 0;
    if (it->cands[k].ref[1] != 0xFF && it->cands[k].ref[1] >= nrefs) return 0;
  }
  return 1;
}

/* predict.rs:284-297 get_mv_params: rec_plane.slice(po + (mv >> 3) - 3).clamp().subslice(3, 3) */
static const uint8_t *mv_source(const uint8_t *ref0, ptrdiff_t stride, int bpp, int plane_w, int plane_h,
                                int xorigin, int yorigin, int po_x, int po_y, const int16_t mv[2], int *row_frac,
                                int *col_frac) {
  int ro, co;
  orc_get_mv_params(mv[0], mv[1], 0, 0, &ro, &co, row_frac, col_frac);
  const int qx = clampi(po_x + co - 3, -xorigin, plane_w), qy = clampi(po_y + ro - 3, -yorigin, plane_h);
  return ref0 + ((ptrdiff_t)(qy + 3) * stride + qx + 3) * bpp;
}

static void screen_one(const uint8_t *src0, ptrdiff_t src_stride, int rect_x, int rect_y, const void *const *refs0,
                       const ptrdiff_t *ref_strides, int bpp, int plane_w, int plane_h, int xorigin, int yorigin,
                       int mode, int bit_depth, const orc_inter_screen_item *it, uint32_t *satd_out,
                       uint8_t *order_out) {
  const int w = BS_W[it->bsize], h = BS_H[it->bsize];
  const int po_x = rect_x + it->x, po_y = rect_y + it->y; /* tile_rect.to_frame_plane_offset */
  const uint8_t *org = src0 + ((ptrdiff_t)po_y * src_stride + po_x) * bpp;
  uint16_t pred[64 * 64];
  int16_t tmp[2][64 * 64];
  uint32_t satd[ENTRIES];
  for (int k = 0; k < ENTRIES; k++) satd[k] = UINT32_MAX;
  for (int k = 0; k < it->n; k++) { /* rdo.rs:1334-1357 */
    const orc_inter_screen_cand *c = &it->cands[k];
    int rf, cf;
    if (c->ref[1] == 0xFF) { /* predict_inter_single, predict.rs:304-336 */
      const int r = c->ref[0];
      const uint8_t *s = mv_source((const uint8_t *)refs0[r], ref_strides[r], bpp, plane_w, plane_h, xorigin, yorigin,
                                   po_x, po_y, c->mv[0], &rf, &cf);
      orc_put_8tap(pred, w, s, ref_strides[r], bpp, w, h, cf, rf, mode, mode, bit_depth);
    } else { /* predict_inter_compound, predict.rs:339-382 */
      for (int i = 0; i < 2; i++) {
        const int r = c->ref[i];
        const uint8_t *s = mv_source((const uint8_t *)refs0[r], ref_strides[r], bpp, plane_w, plane_h, xorigin,
                                     yorigin, po_x, po_y, c->mv[i], &rf, &cf);
        orc_prep_8tap(tmp[i], s, ref_strides[r], bpp, w, h, cf, rf, mode, mode, bit_depth);
      }
      orc_mc_avg(pred, w, bpp, tmp[0], tmp[1], w, h, bit_depth);
    }
    satd[k] = bpp == 1 ? orc_get_satd_u8(org, src_stride, (const uint8_t *)pred, w, w, h)
                       : orc_get_satd_u16((const uint16_t *)org, src_stride, pred, w, w, h);
  }
  /* rdo.rs:1363 sorted.sort_by_key(satd): stable; the unused tail keeps its order */
  uint8_t order[ENTRIES];
  for (int k = 0; k < ENTRIES; k++) order[k] = (uint8_t)k;
  for (int k = 1; k < it->n; k++) {
    const uint8_t e = order[k];
    int j = k;
    for (; j > 0 && satd[order[j - 1]] > satd[e]; j--) order[j] = order[j - 1];
    order[j] = e;
  }
  if (satd_out) memcpy(satd_out, satd, sizeof satd);
  if (order_out) memcpy(order_out, order, sizeof order);
}

void orc_inter_mode_screen(const void *src0, ptrdiff_t src_stride, int rect_x, int rect_y, int rect_w, int rect_h,
                           const void *const *refs0, const ptrdiff_t *ref_strides, int nrefs, int bpp, int plane_w,
                           int plane_h, int xorigin, int yorigin, int filter_mode, int bit_depth,
                           const orc_inter_screen_item *items, size_t n, uint32_t *satd, uint8_t *order,
                           int threads) {
#pragma omp parallel for schedule(dynamic, 16) num_threads(threads > 0 ? threads : orc_num_threads())
  for (size_t i = 0; i < n; i++) {
    uint32_t *s = satd ? satd + i * ENTRIES : NULL;
    uint8_t *o = order ? order + i * ENTRIES : NULL;
    if (!item_valid(&items[i], rect_w, rect_h, nrefs)) {
      for (int k = 0; k < ENTRIES; k++) {
        if (s) s[k] = UINT32_MAX;
        if (o) o[k] = (uint8_t)k;
      }
      continue;
    }
    screen_one((const uint8_t *)src0, src_stride, rect_x, rect_y, refs0, ref_strides, bpp, plane_w, plane_h, xorigin,
               yorigin, filter_mode, bit_depth, &items[i], s, o);
  }
}
