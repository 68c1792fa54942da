/*
 * segmentation.h — CPU restatement of rav1e's segmentation (TEST INFRASTRUCTURE ONLY, like oracle.h):
 * segmentation.rs:23-196, util/kmeans.rs:11-102, quantize/mod.rs:44-97 (ac_q, select_qi), encoder.rs:566-580
 * (update_threshold), encoder.rs:1383-1394 (get_qidx), rdo.rs:464-504 (spatiotemporal_scale).  Implemented in
 * segmentation.c, which cites the lines each function follows.
 *
 * orc_segmentation has the layout of b200_segmentation (include/b200rdo.h): SegmentationState field for field
 * plus qidx[] (get_qidx per segment) and status (0, or 1 / 2 where the reference panics).
 *
 * Parity pinning status (see DESIGN.md §2):
 *   kmeans            : pinned by util/kmeans.rs:108-122 (tests/golden/segmentation_kats.json)
 *   blog32_q11 / bexp64 / blog64 : temporal_rdo.h's, pinned there
 *   the rest          : unpinned upstream; checked against an independent Python restatement
 *                       (tests/test_oracle_segmentation.py)
 *   segment_idx_from_distortion on non-monotone thresholds: parity-unpinned, follows Rust 1.83's
 *                       binary_search_by probe order
 */
#ifndef RAV1E_B200_ORACLE_SEGMENTATION_H
#define RAV1E_B200_ORACLE_SEGMENTATION_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  uint8_t enabled, update_data, update_map, preskip;
  uint8_t last_active_segid, min_segment, max_segment, pad_;
  uint8_t features[8][8];
  int16_t data[8][8];
  uint32_t threshold[7];
  uint8_t qidx[8];
  int32_t status;
} orc_segmentation;

typedef struct {
  int16_t x, y;
  uint8_t bsize, skip, pad_[2];
} orc_segment_item;

/* kmeans::<i16, k> over sorted data (n >= 1), 2 <= k <= 8 */
void orc_kmeans_i16(const int16_t *sorted, size_t n, int k, int16_t *means);
/* select_qi over a strictly increasing 256-entry table */
int orc_select_qi(int64_t quantizer, const uint16_t *table);
/* segmentation_optimize on a copy of *prev (NULL = SegmentationState::default()); returns out->status */
int orc_segmentation_optimize(const uint32_t *scores, size_t n, int base_q_idx, int bit_depth, const uint16_t *ac_q,
                              int update_data, const orc_segmentation *prev, orc_segmentation *out);
/* spatiotemporal_scale of one block (x, y luma px; scales_off: DistortionScale::default()) */
uint32_t orc_spatiotemporal_scale(const uint32_t *scales, const uint32_t *activity, size_t w_imp, size_t h_imp,
                                  int x, int y, int bsize, int scales_off);
/* select_segment for a batch, with b200_select_segment_dev's item conventions (sidx: n x 2, scale may be NULL) */
void orc_select_segment(const orc_segment_item *items, size_t n, const uint32_t *scales, const uint32_t *activity,
                        size_t w_imp, size_t h_imp, int scales_off, int level, const orc_segmentation *seg,
                        uint8_t *sidx, uint32_t *scale);

#ifdef __cplusplus
}
#endif
#endif
