/*
 * encode_me.h — CPU restatement of the encode-time motion search (TEST INFRASTRUCTURE ONLY, like oracle.h):
 * estimate_motion (me.rs:536-632) with a pmv, CORNER { right: true, bottom: true } sampling, no extensive
 * search and ssdec 0, as inter_frame_rdo_mode_decision calls it (rdo.rs:1164-1196).  Implemented in
 * encode_me.c, which cites the lines each function follows; the search and sub-pel stages are me.c's.
 *
 * Parity pinning status (see DESIGN.md §2): unpinned upstream (no stored vectors); the predictor gathering is
 * checked against an independent Python model (tests/test_oracle_encode_me.py), the driver against me.c's
 * stages composed by hand.
 */
#ifndef RAV1E_B200_ORACLE_ENCODE_ME_H
#define RAV1E_B200_ORACLE_ENCODE_ME_H

#include "lookahead_me.h"
#include "oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { /* b200_enc_me_item */
  uint16_t x4, y4;
  uint8_t slot, pad_;
  int16_t pmv[2][2]; /* (row, col) of the two mv-stack predictors */
} orc_enc_me_item;

/* get_subset_predictors (me.rs:386-534) in CORNER { right, bottom } mode at ssdec 0, returned as all_mvs()
 * (me.rs:372-382): the median (the centre sample), subset B (left, top, right, bottom, zero), subset C (from
 * `prev`, NULL = LAST has no stats).  stats / prev: w_in_b x h_in_b grids (w_in_b = 2 * ceil(width / 8)) of the
 * block's slot; the block is w x h px at frame 4x4 offset (x4, y4) in the tile grid of tile_w_sb x tile_h_sb
 * superblocks.  Writes up to 11 vectors to out and returns their count; *min_sad receives the un-normalized
 * min_sad (may be NULL). */
int orc_enc_subset_predictors(const orc_me_stats *stats, const orc_me_stats *prev, int w_in_b, int h_in_b,
                              int tile_w_sb, int tile_h_sb, int x4, int y4, int w, int h, orc_mv *out,
                              uint32_t *min_sad);

/* estimate_motion for every item (b200_estimate_motion_dev's contract, include/b200rdo.h): items grouped by
 * size in TxSize order through size_end[19]; refs[k] / ref_stride[k]: pixel (0,0) of slot k's reconstructed
 * luma; stats / prev: nslots grids (prev NULL or with has_prev flags per slot).  Invalid items (slot >= nslots,
 * offset outside the 4x4 grid) get the empty result. */
void orc_estimate_motion_items(const void *src0, ptrdiff_t src_stride, const void *const *refs,
                               const ptrdiff_t *ref_stride, int nslots, int bpp, int width, int height,
                               const orc_me_stats *stats, const orc_me_stats *prev, const uint8_t *has_prev,
                               int bit_depth, int allow_hp, double me_lambda, int use_satd, int filter_mode,
                               int tile_w_sb, int tile_h_sb, const uint32_t size_end[19],
                               const orc_enc_me_item *items, size_t nitems, orc_me_result *out, int threads);

#ifdef __cplusplus
}
#endif

#endif
