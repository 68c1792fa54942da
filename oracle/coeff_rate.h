/*
 * coeff_rate.h — CPU restatement of rav1e's coefficient rate (TEST INFRASTRUCTURE ONLY, like oracle.h):
 * write_coeffs_lv_map and its helpers (context/block_unit.rs:333-348, :442-526, :1783-2016,
 * context/transform_unit.rs:123-160, :530-574, :776-985) driving the range coder's counter and encoder
 * backends (ec.rs:193-222, :265-308, :334-379, :434-473, :485-620, :782-798, :935-955).  Implemented in
 * coeff_rate.c, which cites the lines each function follows.
 *
 * The records have the layout of b200_coeff_cdfs / b200_coeff_chain / b200_coeff_item (include/b200rdo.h),
 * and orc_coeff_rate follows b200_coeff_rate_dev's rules, invalid chains included.
 *
 * Parity pinning status (see DESIGN.md §2):
 *   default CDFs and the context / tx-set tables : sha256 of the reference's tables
 *                       (tests/golden/coeff_cdf_kats.json); the tables here are restated from the AV1
 *                       specification's rules and compared by digest
 *   symbol order and contexts : an independent decoder written from the AV1 specification (8.2, 5.11.39,
 *                       8.3.2) decodes the encoder backend's bytes (tests/test_oracle_coeff_rate.py)
 *   counter           : an independent Python WriterCounter fed with the decoded symbols
 */
#ifndef RAV1E_B200_ORACLE_COEFF_RATE_H
#define RAV1E_B200_ORACLE_COEFF_RATE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  uint16_t txb_skip[5][13][2];
  uint16_t dc_sign[2][3][2];
  uint16_t eob_extra[5][2][9][2];
  uint16_t eob_flag16[2][2][5];
  uint16_t eob_flag32[2][2][6];
  uint16_t eob_flag64[2][2][7];
  uint16_t eob_flag128[2][2][8];
  uint16_t eob_flag256[2][2][9];
  uint16_t eob_flag512[2][2][10];
  uint16_t eob_flag1024[2][2][11];
  uint16_t coeff_base_eob[5][2][4][3];
  uint16_t coeff_base[5][2][42][4];
  uint16_t coeff_br[5][2][21][4];
  uint16_t intra_tx_1[4][13][7];
  uint16_t intra_tx_2[4][13][5];
  uint16_t inter_tx_1[4][16];
  uint16_t inter_tx_2[4][12];
  uint16_t inter_tx_3[4][2];
} orc_coeff_cdfs;

typedef struct {
  uint32_t snapshot, init_rng, item_begin, item_count;
  uint8_t above[3][16], left[3][16];
} orc_coeff_chain;

typedef struct {
  uint32_t block;
  uint16_t eob;
  uint8_t tx_size, tx_type, plane, plane_bsize, mode, reduced_tx_set;
  uint8_t x4, y4, clip_w4, clip_h4;
} orc_coeff_item;

/* b200_coeff_rate_dev's semantics: rate[c] (UINT32_MAX for an invalid chain), cul_level[i] (may be NULL) */
void orc_coeff_rate(const orc_coeff_cdfs *cdfs, size_t ncdfs, const orc_coeff_chain *chains, size_t nchains,
                    const orc_coeff_item *items, size_t nitems, const void *qcoeffs, size_t ncoeffs, int coeff_is_i32,
                    uint32_t *rate, uint8_t *cul_level);
/* One chain through the encoder backend (WriterEncoder::new(), so init_rng must be 32768): writes done()'s
 * bytes to out (cap bytes) and returns their count, -1 for an invalid chain, -2 if cap is too small.
 * tell_frac[0] is the encoder's tell_frac before done(), tell_frac[1] the counter's on the same symbols;
 * *nsymbols counts every symbol / bool coded. */
long orc_coeff_encode_chain(const orc_coeff_cdfs *cdfs, size_t ncdfs, const orc_coeff_chain *chain,
                            const orc_coeff_item *items, size_t nitems, const void *qcoeffs, size_t ncoeffs,
                            int coeff_is_i32, uint8_t *out, size_t cap, uint32_t *tell_frac, long *nsymbols);
/* A script of raw coder calls through the encoder backend, for the range coder's own round-trip tests:
 * ops[3k..3k+2] = (0, val, f) for bool(val, f), (1, s, 0) for symbol(s, cdf) without adaptation.
 * Returns the byte count (-2: cap too small); tell_frac as orc_coeff_encode_chain. */
long orc_ec_encode_script(const int32_t *ops, size_t nops, const uint16_t *cdf, int ncdf, uint8_t *out, size_t cap,
                          uint32_t *tell_frac);
/* The spec-restated tables under the reference's names (see tests/golden/make_coeff_cdf_kats.py), as int32
 * in row-major order; returns the count, 0 for an unknown name. */
int orc_coeff_table(const char *name, int32_t *out);

#ifdef __cplusplus
}
#endif
#endif
