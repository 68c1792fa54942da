/* intra_screen.h — CPU restatement of rav1e's intra mode screening (TEST INFRASTRUCTURE ONLY, see oracle.h).
 *
 * rdo.rs:1433-1511 + predict.rs:205-249.  Per item: get_intra_edges (mode None) from the rec region, the
 * modes after the first num_modes_rdo / 2 predicted at bsize.tx_size() with predict_intra's wrapper logic,
 * get_satd against src, the tail stable-sorted by SATD.  rec0 / src0 address plane pixel (0,0) (both padded
 * by >= 64); satd: n x 13 by discriminant (0 = not screened), modes: n x 13; either may be NULL.  Invalid
 * items (bsize >= 22, an entry >= 13 or repeated, (x, y) outside the region or not a multiple of 4) get
 * UINT32_MAX and their list unchanged.  Item layout = b200_intra_screen_item.
 */
#ifndef RAV1E_B200_ORACLE_INTRA_SCREEN_H
#define RAV1E_B200_ORACLE_INTRA_SCREEN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int16_t x, y;
  uint8_t bsize;
  int8_t ief;
  uint8_t modes[13];
  uint8_t pad_;
} orc_intra_screen_item;

void orc_intra_mode_screen(const void *rec0, ptrdiff_t rec_stride, const void *src0, ptrdiff_t src_stride, int bpp,
                           int plane_w, int plane_h, int rect_x, int rect_y, int rect_w, int rect_h, int bit_depth,
                           int num_modes_rdo, const orc_intra_screen_item *items, size_t n, uint32_t *satd,
                           uint8_t *modes, int threads);

#ifdef __cplusplus
}
#endif
#endif
