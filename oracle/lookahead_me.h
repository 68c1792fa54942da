/*
 * lookahead_me.h — CPU restatement of the lookahead's motion estimation (TEST INFRASTRUCTURE ONLY, like
 * oracle.h): estimate_tile_motion and what it calls, me.rs:153-337, 386-534, 633-856.  Implemented in
 * lookahead_me.c, which cites the lines each function follows.
 *
 * Parity pinning status (see DESIGN.md §2): unpinned upstream (no stored vectors; the reference's tests
 * need rustc); checked against an independent Python model of the driver (tests/test_oracle_lookahead_me.py).
 */
#ifndef RAV1E_B200_ORACLE_LOOKAHEAD_ME_H
#define RAV1E_B200_ORACLE_LOOKAHEAD_ME_H

#include "oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* estimate_tile_motion (me.rs:153-337, 386-534, 633-690) for every tile of one (frame, reference
 * slot) pair, serially in the reference's loop order.  cur[k] / ref[k] point at pixel (0,0) of the
 * full (k = 0), half (1) and quarter (2) resolution planes; width x height is the full-resolution
 * frame.  The stats grid is w_in_b x h_in_b (2 * ceil(width / 8) x 2 * ceil(height / 8)) row-major,
 * like FrameMEStats; prev is LAST's final grid for the same slot, or NULL. */
typedef struct {
  int16_t mv_row, mv_col;
  uint32_t normalized_sad;
} orc_me_stats;
void orc_lookahead_motion(const void *const cur[3], const ptrdiff_t cur_stride[3], const void *const ref[3],
                          const ptrdiff_t ref_stride[3], int bpp, int width, int height, int bit_depth,
                          int allow_hp, double me_lambda, int me_allow_full_search, int me_range_scale,
                          int tile_w_sb, int tile_h_sb, const orc_me_stats *prev, orc_me_stats *out);
/* thresh of full_pixel_me's extensive ladder (me.rs:771-772) from the un-normalized min_sad */
uint32_t orc_lookahead_me_thresh(uint32_t min_sad, int w, int h, int bit_depth);

#ifdef __cplusplus
}
#endif

#endif
