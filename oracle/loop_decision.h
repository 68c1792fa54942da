/*
 * oracle/loop_decision.h — rdo_loop_decision's CDEF / restoration pass loop (TEST INFRASTRUCTURE ONLY).
 *
 * orc_loop_decision restates rav1e src/rdo.rs:2104-2745 after the optional deblock for a list of
 * loop-restoration areas (see b200_loop_decision_dev in include/b200rdo.h for the contract): per area its
 * scratch copies, the CDEF analysis, then C, L, C, L, .. stages until one changes nothing, walking
 * superblocks and units in the reference's order.  The C stage is orc_cdef_rdo's superblock loop with the
 * restoration branches of rdo.rs:2424-2527 added literally: for a unit holding Sgrproj, the candidate is
 * filtered into the CDEF scratch copy, the integral image is taken from that copy (so it sees this pass's
 * winners to the left and above), the self-guided filter runs over the superblock's visible rect and the
 * distortion is measured on lrf_work.  The L stage is orc_lrf_search's per-unit search with the incumbent
 * and its cost carried.  The pieces are cdef_rdo.c's, lrf_search.c's and lrf.c's own, compiled in.
 *
 * Parity: rdo_loop_decision has no stored vectors upstream, so the orchestration is parity-unpinned and
 * checked against an independent Python restatement (tests/test_oracle_loop_decision.py).
 *
 * Planes: rec[p] / src[p] / work[p] address pixel (0,0) of the frame, strides in elements, `bpp` bytes per
 * pixel.  Outputs as b200_loop_decision_dev's; err / cost (slot * 8 + i) may be NULL.  Returns the stage
 * count of the longest area, or -1 when an area is still changing after B200_LOOP_MAX_STAGES stages.
 */
#ifndef ORC_LOOP_DECISION_H
#define ORC_LOOP_DECISION_H

#include <stddef.h>
#include <stdint.h>

#include "../include/b200rdo.h"

int orc_loop_decision(const void *const *rec, const ptrdiff_t *rec_stride, const void *const *src,
                      const ptrdiff_t *src_stride, void *const *work, const ptrdiff_t *work_stride, int bpp,
                      int planes, int xdec, int ydec, int width, int height, int bit_depth, int enable_cdef,
                      int damping, int cdef_bits, const uint8_t *y_strengths, const uint8_t *uv_strengths,
                      const uint8_t *skip8, int enable_restoration, const int *unit_size, int reduced_sets,
                      const uint32_t *imp_scales, const uint32_t *dist_scale, double lambda,
                      const b200_cdef_rdo_area *areas, size_t n_areas, const b200_loop_unit *units,
                      size_t n_units, const int32_t *sb_unit, int8_t *best_index, b200_lrf_unit *unit_out,
                      double *unit_cost, uint8_t *written, uint64_t *err, double *cost);

#endif
