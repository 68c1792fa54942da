/* cfl_alpha.h — CPU restatement of rav1e's CfL alpha search (TEST INFRASTRUCTURE ONLY, see oracle.h).
 *
 * rdo_cfl_alpha (rdo.rs:1593-1689) with luma_ac (predict.rs:644-698) and clip_visible_bsize (rdo.rs:228-253).
 * rec[p] / src[p] address plane p's pixel (0, 0) with element strides rec_stride[p] / src_stride[p] (src[0] is
 * not read); chroma_w / chroma_h = the chroma planes' plane_cfg width / height; the luma plane must be
 * readable 31 pixels past the frame.  (rect_x, rect_y, rect_w, rect_h) is the tile in luma pixels;
 * frame_width / frame_height = fi.width / fi.height.  alpha: n x 2 (best_alpha of planes 1, 2), sse: n x 2 x 33
 * ([item][plane - 1][alpha + 16], UINT64_MAX for alphas the reference never evaluates); either may be NULL.
 * Invalid items (bsize > BLOCK_32X32, no subsampled_size, no chroma, tx_size >= 19 or larger than the block,
 * (x, y) outside the region or not a multiple of 4) and items with no visible chroma get {0, 0} and UINT64_MAX.
 * Item layout = b200_cfl_item.
 */
#ifndef RAV1E_B200_ORACLE_CFL_ALPHA_H
#define RAV1E_B200_ORACLE_CFL_ALPHA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int16_t x, y;
  uint8_t bsize, tx_size;
  uint8_t pad_[2];
} orc_cfl_item;

void orc_cfl_alpha(const void *const rec[3], const ptrdiff_t rec_stride[3], const void *const src[3],
                   const ptrdiff_t src_stride[3], int bpp, int chroma_w, int chroma_h, int xdec, int ydec, int rect_x,
                   int rect_y, int rect_w, int rect_h, int frame_width, int frame_height, int bit_depth,
                   const orc_cfl_item *items, size_t n, int8_t *alpha, uint64_t *sse, int threads);

#ifdef __cplusplus
}
#endif
#endif
