/* intra_screen.c — CPU restatement of rav1e's intra mode screening (TEST INFRASTRUCTURE ONLY, see
 * oracle.h and intra_screen.h).
 *
 *   intra_frame_rdo_mode_decision's pruning metric   src/rdo.rs:1433-1511
 *   PredictionMode::predict_intra                    src/predict.rs:205-249
 *   PredictionVariant::new, intra_mode_to_angle      src/predict.rs:126-150
 *   BlockSize::tx_size                               src/partition.rs:306-328
 *
 * Composed of the pinned pieces orc_get_intra_edges, orc_predict_intra and orc_get_satd_*; the
 * orchestration itself has no stored vectors upstream ("parity unpinned") and is cross-checked
 * against an independent Python restatement (tests/test_oracle_intra_screen.py).
 */
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "intra_screen.h"
#include "oracle.h"

static const uint8_t BS_TX[22] = {0, 5, 6, 1, 7, 8, 2, 9, 10, 3, 11, 12, 4, 4, 4, 4, 13, 14, 15, 16, 17, 18};
enum { DC = 0, V = 1, H = 2, D67 = 8, PAETH = 12, NMODES = 13 };

static int mode_angle(int mode) { /* predict.rs:138-150 */
  static const int a[9] = {0, 90, 180, 45, 135, 113, 157, 203, 67};
  return mode >= 1 && mode <= 8 ? a[mode] : 0;
}

static int item_valid(const orc_intra_screen_item *it, int rect_w, int rect_h) {
  if (it->bsize >= 22 || it->x < 0 || it->y < 0 || it->x >= rect_w || it->y >= rect_h || (it->x & 3) || (it->y & 3))
    return 0;
  unsigned seen = 0;
  for (int k = 0; k < NMODES; k++) {
    if (it->modes[k] >= NMODES || (seen >> it->modes[k]) & 1u) return 0;
    seen |= 1u << it->modes[k];
  }
  return 1;
}

static void screen_one(const uint8_t *rec0, ptrdiff_t rec_stride, const uint8_t *src0, ptrdiff_t src_stride, int bpp,
                       int plane_w, int plane_h, int rect_x, int rect_y, int rect_w, int rect_h, int bit_depth,
                       int num_modes_rdo, const orc_intra_screen_item *it, uint32_t *satd, uint8_t *modes) {
  const int tx = BS_TX[it->bsize], w = orc_tx_width(tx), h = orc_tx_height(tx);
  const int x = it->x, y = it->y;
  /* rdo.rs:1443-1461: get_intra_edges(rec, tile_bo, 0, 0, bsize, po, tx_size, bd, None, ...) */
  uint16_t edge_buf[4 * 64 + 1];
  int init_left = 0, init_above = 0;
  const uint8_t *region = rec0 + ((ptrdiff_t)rect_y * rec_stride + rect_x) * bpp;
  orc_get_intra_edges(edge_buf, region, rec_stride, bpp, plane_w, plane_h, rect_x, rect_y, rect_w, rect_h, 0, 0,
                      x >> 2, y >> 2, 0, 0, it->bsize, x, y, w, h, bit_depth, -1, it->ief >= 0, 0, &init_left,
                      &init_above);
  /* predict.rs:214-219: the variant from the tile-relative position */
  const int variant = x == 0 && y == 0 ? 0 : y == 0 ? 1 : x == 0 ? 2 : 3;
  const uint8_t *org = src0 + ((ptrdiff_t)(rect_y + y) * src_stride + rect_x + x) * bpp;
  uint16_t pred[64 * 64];
  uint32_t satds_all[NMODES] = {0};
  uint8_t list[NMODES];
  memcpy(list, it->modes, NMODES);
  /* rdo.rs:1477-1508: every mode after the first num_modes_rdo / 2 */
  for (int k = num_modes_rdo / 2; k < NMODES; k++) {
    const int luma_mode = list[k];
    int mode = luma_mode; /* predict.rs:231-239: PAETH at the tile's top / left edges */
    if (mode == PAETH) mode = variant == 0 ? DC : variant == 2 ? V : variant == 1 ? H : PAETH;
    const int ief = luma_mode >= V && luma_mode <= D67 ? it->ief : -1; /* is_directional() */
    orc_predict_intra(mode, variant, pred, w, bpp, w, h, bit_depth, NULL, mode_angle(mode), ief, edge_buf, init_left,
                      init_above, plane_w, plane_h, rect_x + x, rect_y + y);
    satds_all[luma_mode] = bpp == 1 ? orc_get_satd_u8(org, src_stride, (const uint8_t *)pred, w, w, h)
                                    : orc_get_satd_u16((const uint16_t *)org, src_stride, pred, w, w, h);
  }
  /* rdo.rs:1511: modes[num_modes_rdo / 2..].sort_by_key(satds) — stable */
  for (int k = num_modes_rdo / 2 + 1; k < NMODES; k++) {
    const uint8_t m = list[k];
    int j = k;
    for (; j > num_modes_rdo / 2 && satds_all[list[j - 1]] > satds_all[m]; j--) list[j] = list[j - 1];
    list[j] = m;
  }
  if (satd) memcpy(satd, satds_all, sizeof satds_all);
  if (modes) memcpy(modes, list, NMODES);
}

void orc_intra_mode_screen(const void *rec0, ptrdiff_t rec_stride, const void *src0, ptrdiff_t src_stride, int bpp,
                           int plane_w, int plane_h, int rect_x, int rect_y, int rect_w, int rect_h, int bit_depth,
                           int num_modes_rdo, const orc_intra_screen_item *items, size_t n, uint32_t *satd,
                           uint8_t *modes, int threads) {
#pragma omp parallel for schedule(dynamic, 16) num_threads(threads > 0 ? threads : orc_num_threads())
  for (size_t i = 0; i < n; i++) {
    uint32_t *s = satd ? satd + i * NMODES : NULL;
    uint8_t *m = modes ? modes + i * NMODES : NULL;
    if (!item_valid(&items[i], rect_w, rect_h)) {
      if (s)
        for (int k = 0; k < NMODES; k++) s[k] = UINT32_MAX;
      if (m) memcpy(m, items[i].modes, NMODES);
      continue;
    }
    screen_one((const uint8_t *)rec0, rec_stride, (const uint8_t *)src0, src_stride, bpp, plane_w, plane_h, rect_x,
               rect_y, rect_w, rect_h, bit_depth, num_modes_rdo, &items[i], s, m);
  }
}
