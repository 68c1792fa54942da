/* inter_screen.h — CPU restatement of rav1e's inter mode screening (TEST INFRASTRUCTURE ONLY, see oracle.h).
 *
 * rdo.rs:1281-1363 + predict.rs:284-421.  Per item: every entry of its resolved mode list predicted at the
 * full block size by predict_inter (put_8tap for a single reference; prep_8tap of both references and
 * mc_avg for a compound pair; FilterMode filter_mode in both directions), from the source position of
 * get_mv_params including PlaneSlice::clamp to [-xorigin, plane_w] x [-yorigin, plane_h]; get_satd
 * against src; the entries stable-sorted by SATD.  refs0[r] / src0 address plane pixel (0,0) (refs padded
 * by >= max(xorigin, yorigin, 71), src by >= 64); satd: n x 20 in list order (UINT32_MAX past n), order:
 * n x 20 (the sorted entries, then n .. 19); either may be NULL.  Invalid items (bsize >= 22 or 128-sided,
 * n > 20, a ref index >= nrefs, (x, y) outside the region or not a multiple of 4) get UINT32_MAX and the
 * identity order.  Item layout = b200_inter_screen_item.
 *
 * Pinning: put_8tap / prep_8tap / mc_avg / get_mv_params and get_satd are as pinned as oracle.h states
 * (MC parity unpinned upstream, checked against the AV1 specification's two-pass form; SATD pinned).
 * PlaneSlice::clamp lives in v_frame 0.3.9, which is not on disk: it is restated from its published
 * semantics (x clamped to [-xorigin, width], y to [-yorigin, height]) and is parity unpinned, like
 * Plane::downsampled.  The orchestration has no stored vectors upstream; it is cross-checked against an
 * independent Python restatement (tests/test_oracle_inter_screen.py).
 */
#ifndef RAV1E_B200_ORACLE_INTER_SCREEN_H
#define RAV1E_B200_ORACLE_INTER_SCREEN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int16_t mv[2][2]; /* {row, col} per reference, 1/8 pel */
  uint8_t ref[2];   /* index into refs0[]; ref[1] = 0xFF: single reference */
  uint8_t pad_[2];
} orc_inter_screen_cand;

typedef struct {
  int16_t x, y;
  uint8_t bsize;
  uint8_t n;
  uint8_t pad_[2];
  orc_inter_screen_cand cands[20];
} orc_inter_screen_item;

void orc_inter_mode_screen(const void *src0, ptrdiff_t src_stride, int rect_x, int rect_y, int rect_w, int rect_h,
                           const void *const *refs0, const ptrdiff_t *ref_strides, int nrefs, int bpp, int plane_w,
                           int plane_h, int xorigin, int yorigin, int filter_mode, int bit_depth,
                           const orc_inter_screen_item *items, size_t n, uint32_t *satd, uint8_t *order,
                           int threads);

#ifdef __cplusplus
}
#endif
#endif
