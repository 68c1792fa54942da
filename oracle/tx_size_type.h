/* tx_size_type.h — CPU restatement of rav1e's intra transform size and type decision (TEST INFRASTRUCTURE
 * ONLY, see oracle.h).
 *
 *   rdo_tx_size_type       src/rdo.rs:725-802  (intra luma, rdo_tx_decision and tx_mode_select on)
 *   rdo_tx_type_decision   src/rdo.rs:1701-1823
 *   write_tx_blocks (luma) src/encoder.rs:2243-2311 -> encode_tx_block :1404-1658
 *
 * Composed of the oracle's own pieces: orc_get_intra_edges, orc_predict_intra, orc_forward_transform,
 * orc_quantize_chain_batch, orc_inverse_transform_add, orc_coeff_rate (counter backend),
 * orc_weighted_sse_*, orc_cdef_dist_kernel_*, orc_distortion_scale_mul and orc_compute_rd_cost.  The records
 * have the layout of b200_tx_item / b200_tx_best / b200_tx_cand (include/b200rdo.h) and
 * orc_intra_tx_size_type follows b200_intra_tx_size_type_dev's rules, invalid items included.
 */
#ifndef RAV1E_B200_ORACLE_TX_SIZE_TYPE_H
#define RAV1E_B200_ORACLE_TX_SIZE_TYPE_H

#include <stddef.h>
#include <stdint.h>

#include "coeff_rate.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  int16_t x, y;
  uint8_t bsize, mode;
  int8_t ief;
  uint8_t skip;
  uint32_t dc_quant, ac_quant, snapshot;
  uint8_t above[16], left[16];
} orc_tx_item; /* 52 B */

typedef struct {
  double rd;
  uint8_t tx_size, tx_type, pad_[6];
} orc_tx_best; /* 16 B */

typedef struct {
  double rd;
  uint64_t dist;
  uint32_t rate, state;
} orc_tx_cand; /* 24 B */

enum { ORC_TX_EVALUATED = 0, ORC_TX_NOT_IN_SET = 1, ORC_TX_CUT = 2, ORC_TX_NOT_IN_LADDER = 3, ORC_TX_INVALID = 255 };

/* rec0 / src0 address plane pixel (0,0) (padded by >= 64).  cands may be NULL: else n x 21 records,
 * [item][level * 7 + k] with k the position in RAV1E_TX_TYPES. */
void orc_intra_tx_size_type(const void *rec0, ptrdiff_t rec_stride, const void *src0, ptrdiff_t src_stride, int bpp,
                            int plane_w, int plane_h, int rect_x, int rect_y, int rect_w, int rect_h, int frame_w,
                            int frame_h, int bit_depth, int dist_mode, int reduced_tx_set, double lambda,
                            uint32_t dist_scale, const uint32_t *scale4x4, size_t scale_stride,
                            const orc_coeff_cdfs *cdfs, size_t ncdfs, const orc_tx_item *items, size_t n,
                            orc_tx_best *best, orc_tx_cand *cands, int threads);

#ifdef __cplusplus
}
#endif
#endif
