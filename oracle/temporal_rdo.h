/*
 * temporal_rdo.h — CPU restatement of rav1e's temporal RDO (TEST INFRASTRUCTURE ONLY, like oracle.h):
 * api/internal.rs:912-1230, rdo.rs:506-630, encoder.rs:744-777, util/logexp.rs.  Implemented in
 * temporal_rdo.c, which cites the lines each function follows.
 *
 * Importance blocks sit on the CEIL grid (w_imp = ceil(W/8), h_imp = ceil(H/8)); the intra-cost maps
 * are floor(W/8) x floor(H/8) and are read flat in rows of w_imp, as the reference does.
 *
 * Parity pinning status (see DESIGN.md §2):
 *   blog64 / bexp64   : pinned by util/logexp.rs:292-314 (KATs in tests/golden/logexp_kats.json + the
 *                       round-trip test)
 *   blog32_q11        : pinned by its round-trip test (:345-358)
 *   propagation,      : unpinned upstream; checked against an independent float32 numpy model and
 *   scales, scores      Python restatements (tests/test_oracle_temporal_rdo.py)
 */
#ifndef RAV1E_B200_ORACLE_TEMPORAL_RDO_H
#define RAV1E_B200_ORACLE_TEMPORAL_RDO_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

int64_t orc_bexp64(int64_t logq57);
int64_t orc_blog64(int64_t n);
int32_t orc_blog32_q11(uint32_t w);
uint32_t orc_dscale_mul(uint32_t a, uint32_t b);
uint32_t orc_dscale_inv_mean(const uint32_t *s, size_t n);
int64_t orc_dscale_blog64(uint32_t s);
uint32_t orc_distortion_scale_for(double propagate_cost, double intra_cost);
void orc_distortion_scales(const float *importances, size_t n_imp, const uint32_t *intra_costs, size_t n_intra,
                           uint32_t *scales);
int64_t orc_temporal_scores(uint32_t *scales, size_t n, const uint32_t *activity, uint32_t *spatiotemporal,
                            uint32_t *inv_mean_out);
void orc_update_block_importances(const void *org, ptrdiff_t org_stride, const void *ref, ptrdiff_t ref_stride,
                                  int bpp, int w_imp, int h_imp, const uint32_t *intra_costs, size_t n_intra,
                                  const int16_t *mvs, const float *future, uint32_t len, float *ref_importances);
void orc_block_importances(size_t nframes, const void *const *frames, ptrdiff_t stride, int bpp, int width,
                           int height, const uint32_t *intra_costs, const int16_t *mvs, size_t nsteps,
                           const uint32_t *steps, float *importances);

#ifdef __cplusplus
}
#endif
#endif
