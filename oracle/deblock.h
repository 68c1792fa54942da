/*
 * oracle/deblock.h — the deblocking filter's level search and edge filter (TEST INFRASTRUCTURE ONLY, see
 * oracle.h).
 *
 * orc_deblock_levels restates sse_optimize (rav1e src/deblock.rs:1553-1617, with sse_plane :1460-1540,
 * sse_v_edge / sse_h_edge :1145-1193, :1241-1290 and sse_size4/6/8/14) per item.  orc_deblock_filter
 * restates deblock_filter_frame -> deblock_plane (:1292-1551) in the reference's lagged edge order, per
 * item, in place, behind the call sites' gate (encoder.rs:3280, :3598, rdo.rs:2311: nothing is filtered
 * when both luma levels are 0).  Deblocking is normative (AV1 specification section 7.14) and the
 * reference stores no vectors for it, so it is parity-unpinned upstream and second-sourced from the
 * specification: tests/test_oracle_deblock_spec.py checks the filter against an independent model of
 * section 7.14, tests/test_oracle_deblock.py the level search against a brute-force search over that model.
 *
 * Planes: pl[p] addresses pixel (0,0) of the frame plane, strides in elements, `bpp` bytes per pixel; the
 * level search reads up to 4 luma rows outside an item's working rect (see include/b200rdo.h), so the
 * caller pads.  mi: 12-byte b200_deblock_mi records, mi_stride per row, frame-absolute.  items: n_items x
 * {mi_x, mi_y, mi_w, mi_h, vis_w, vis_h}.  state: the 16-byte b200_deblock_state.  levels: 4 per item.
 * tally (may be NULL): per item x 3 planes x {vertical, horizontal} x 64 prefix-summed i64 (zeros for
 * planes >= `planes`).
 */
#ifndef ORC_DEBLOCK_H
#define ORC_DEBLOCK_H

#include <stddef.h>
#include <stdint.h>

void orc_deblock_levels(const void *const *rec, const ptrdiff_t *rec_stride, const void *const *src,
                        const ptrdiff_t *src_stride, int bpp, int planes, int xdec, int ydec, int bit_depth,
                        const uint8_t *mi, ptrdiff_t mi_stride, const int32_t *items, size_t n_items,
                        uint8_t *levels, int64_t *tally);

void orc_deblock_filter(void *const *pl, const ptrdiff_t *stride, int bpp, int planes, int xdec, int ydec,
                        int bit_depth, const uint8_t *state, const uint8_t *levels, const uint8_t *mi,
                        ptrdiff_t mi_stride, const int32_t *items, size_t n_items);

#endif
