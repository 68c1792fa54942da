/*
 * oracle/lrf.h — loop restoration's frame filter (TEST INFRASTRUCTURE ONLY, see oracle.h).
 *
 * orc_lrf_filter_frame restates RestorationState::lrf_filter_frame (rav1e src/lrf.rs:1482-1585) with its
 * stripe and unit loops, restoration_unit_by_stripe (:1295-1312), wiener_stripe_filter (:1099-1207),
 * setup_integral_image with VertPaddedIter / HorzPaddedIter (:381-627, wrapping u32 integral images
 * included) and sgrproj_stripe_filter (:629-830) with the Rust box helpers (:175-342) and
 * sgrproj_sum_finish (:344-362).  Loop restoration is normative (AV1 specification, loop restoration
 * process) and the reference stores no vectors for it, so it is parity-unpinned upstream and second-sourced
 * from the specification: tests/test_oracle_lrf_spec.py checks it against an independent model of the
 * specification, pixel for pixel, and shows the three places where rav1e departs from it:
 *   1. Wiener units read the deblocked frame's row 0 for the 3 rows above the frame and its row crop_h - 1
 *      for rows below the last stripe (:1157-1169); the specification reads the CDEF output there.
 *   2. With enable_cdef == 0 Sgrproj units are skipped (:1545-1547).
 *   3. When crop_h < 56 >> ydec, Sgrproj units also write stripe 0's rows at and below crop_h.
 *
 * Planes: out[p] / cdeffed[p] / deblocked[p] address pixel (0,0), strides in elements, `bpp` bytes per
 * pixel.  out holds a copy of cdeffed on entry (lrf_filter_frame's `out`; cdeffed is its clone) and is
 * filtered in place.  Difference 3 reads cdeffed and writes out at rows up to (56 >> ydec) - 1, so for
 * such frames the planes need that many rows.  units[p]: cols x rows 12-byte b200_lrf_unit records,
 * row-major, with cols / rows derived from unit_size[p] and the crop as lrf.rs:1431-1440 does.
 */
#ifndef ORC_LRF_H
#define ORC_LRF_H

#include <stddef.h>
#include <stdint.h>

void orc_lrf_filter_frame(void *const *out, const ptrdiff_t *out_stride, const void *const *cdeffed,
                          const ptrdiff_t *cdeffed_stride, const void *const *deblocked,
                          const ptrdiff_t *deblocked_stride, int bpp, int planes, int xdec, int ydec,
                          int frame_width, int frame_height, int bit_depth, int enable_cdef, const int *unit_size,
                          const uint8_t *const *units);

#endif
