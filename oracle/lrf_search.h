/*
 * oracle/lrf_search.h — the restoration search of one rdo_loop_decision pass (TEST INFRASTRUCTURE ONLY).
 *
 * orc_lrf_search restates rav1e src/rdo.rs:2575-2740 for a list of b200_lrf_search_item records (see
 * include/b200rdo.h for the contract): the None candidate (rdo_loop_plane_error, rdo.rs:2027-2093, with the
 * incoming filter's rate), then for every set of get_sgr_sets (lrf.rs:75-93) sgrproj_solve (lrf.rs:846-1096),
 * sgrproj_stripe_filter over the visible rect, rdo_loop_plane_error and count_lrf_switchable
 * (context/frame_header.rs:14-45 with ec.rs:381-389, 639-773), and the winner under a strict `<`.  The
 * integral image and the filter are oracle/lrf.c's; the distortion pieces are the ones orc_cdef_rdo
 * composes.  The solve is restated operation for operation in f64, line sums in i64 as the reference.
 *
 * Parity: rdo_loop_decision has no stored vectors upstream, so the orchestration is parity-unpinned and
 * checked against an independent Python restatement (tests/test_oracle_lrf_search.py).  lrf_work's pixels
 * outside the visible rect come from v_frame's Plane::new fill, restated as B200_LRF_WORK_FILL.
 *
 * Planes: lrf_in[p] / src[p] address pixel (0,0) of the frame, strides in elements, `bpp` bytes per
 * pixel, covering the frame rounded up to 8 luma pixels.  Outputs per item i: best[i], cost[i],
 * changed[i]; optional (NULL = not wanted) xqd[(i * 16 + set) * 2 + k], err[i * 17 + c] and
 * cand_cost[i * 17 + c] with c = 0 for None and 1 + set for the searched sets.
 */
#ifndef ORC_LRF_SEARCH_H
#define ORC_LRF_SEARCH_H

#include <stddef.h>
#include <stdint.h>

#include "../include/b200rdo.h"

void orc_lrf_search(const void *const *lrf_in, const ptrdiff_t *lrf_in_stride, const void *const *src,
                    const ptrdiff_t *src_stride, int bpp, int xdec, int ydec, int frame_width, int frame_height,
                    int bit_depth, const int *unit_size, int reduced_sets, const uint32_t *imp_scales,
                    const uint32_t *dist_scale, double lambda, const b200_cdef_rdo_area *areas,
                    const b200_lrf_search_item *items, size_t n_items, b200_lrf_unit *best, double *cost,
                    uint8_t *changed, int8_t *xqd, uint64_t *err, double *cand_cost);

#endif
