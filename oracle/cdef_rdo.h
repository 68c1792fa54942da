/*
 * oracle/cdef_rdo.h — the CDEF pass of rdo_loop_decision (TEST INFRASTRUCTURE ONLY, see oracle.h).
 *
 * orc_cdef_rdo restates rav1e src/rdo.rs:2104-2567 for the RestorationFilter::None / no-LRU branches
 * (with rdo_loop_plane_error :2027-2093 and cdef_filter_superblock, cdef.rs:401-570) for a list of
 * loop-restoration areas, composed only of pinned pieces: orc_cdef_find_dir, orc_cdef_filter_block_px
 * with the edge flags of the area's scratch copy, orc_cdef_dist_kernel_*, orc_weighted_sse_*,
 * orc_distortion_scale_mul and orc_compute_rd_cost.  The orchestration itself is parity-unpinned
 * upstream; tests/test_oracle_cdef_rdo.py checks it against an independent Python restatement.
 *
 * Planes: rec[p] / src[p] / out[p] address pixel (0,0), strides in elements, `bpp` bytes per pixel;
 * out may be NULL.  areas: n_areas x {sbx, sby, sb_w, sb_h} in frame-absolute superblocks.  skip8 /
 * imp_scales: ceil(W/8) entries per row (NULL = none skipped / default scale).  rate: one per slot
 * (NULL = 0).  Outputs per slot (area * 16 + sby * 4 + sbx): err[slot * 8 + i], cost[slot * 8 + i]
 * for i < 1 << cdef_bits of decided superblocks, best[slot] (-1 = CDEF-skipped); slots outside an area
 * are not written.  out receives the area's CDEF output over each area's scratch rect.
 */
#ifndef ORC_CDEF_RDO_H
#define ORC_CDEF_RDO_H

#include <stddef.h>
#include <stdint.h>

void orc_cdef_rdo(const void *const *rec, const ptrdiff_t *rec_stride, const void *const *src,
                  const ptrdiff_t *src_stride, void *const *out, const ptrdiff_t *out_stride, int bpp,
                  int planes, int xdec, int ydec, int width, int height, int bit_depth, int damping,
                  int cdef_bits, const uint8_t *y_strengths, const uint8_t *uv_strengths,
                  const uint8_t *skip8, const uint32_t *imp_scales, const uint32_t *dist_scale,
                  double lambda, const int32_t *areas, size_t n_areas, const uint32_t *rate,
                  uint64_t *err, double *cost, int8_t *best);

#endif
