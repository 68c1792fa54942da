/* temporal_rdo.c — CPU restatement of rav1e's temporal RDO: block-importance propagation over the
 * lookahead window, the distortion scales derived from it and their normalisation (TEST
 * INFRASTRUCTURE ONLY, see oracle.h; declared in temporal_rdo.h).
 *
 *   update_block_importances        src/api/internal.rs:912-1071
 *   compute_block_importances       src/api/internal.rs:1075-1230 (window driver + distortion scales)
 *   distortion_scale_for            src/rdo.rs:506-553
 *   DistortionScale new / From<f64> src/rdo.rs:579-583, :652-658
 *   DistortionScale inv_mean / blog64 / Mul   src/rdo.rs:585-594, :605-608, :618-630
 *   compute_{spatio,}temporal_scores          src/encoder.rs:744-777
 *   q57 / bexp64 / blog64 / blog32_q11        src/util/logexp.rs:11-14, :34-125, :130-174, :271-286
 *
 * The f32 sequence of the propagation is evaluated exactly as written (one rounding per operation,
 * nothing fused: -std=c11 makes GCC use -ffp-contract=off).  pow() is glibc's, which Rust's
 * f64::powf calls on Linux.  The logexp helpers are restated from their published semantics
 * (hyperbolic CORDIC in Q61/Q62 with the iterations 3k+1 = 4, 13, 40 repeated); only the
 * atanh(2^-i)/ln 2 table is data.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "oracle.h"
#include "temporal_rdo.h"

/* ------------------------------------------------------------------ util/logexp.rs */
/* ATANH_LOG2[i] = atanh(2^-(i+1)) / ln(2) in Q62 (logexp.rs:17-29) */
static const int64_t K_ATANH[32] = {
    0x32B803473F7AD0F4, 0x2F2A71BD4E25E916, 0x2E68B244BB93BA06, 0x2E39FB9198CE62E4, 0x2E2E683F68565C8F,
    0x2E2B850BE2077FC1, 0x2E2ACC58FE7B78DB, 0x2E2A9E2DE52FD5F2, 0x2E2A92A338D53EEC, 0x2E2A8FC08F5E19B6,
    0x2E2A8F07E51A485E, 0x2E2A8ED9BA8AF388, 0x2E2A8ECE2FE7384A, 0x2E2A8ECB4D3E4B1A, 0x2E2A8ECA94940FE8,
    0x2E2A8ECA6669811D, 0x2E2A8ECA5ADEDD6A, 0x2E2A8ECA57FC347E, 0x2E2A8ECA57438A43, 0x2E2A8ECA57155FB4,
    0x2E2A8ECA5709D510, 0x2E2A8ECA5706F267, 0x2E2A8ECA570639BD, 0x2E2A8ECA57060B92, 0x2E2A8ECA57060008,
    0x2E2A8ECA5705FD25, 0x2E2A8ECA5705FC6C, 0x2E2A8ECA5705FC3E, 0x2E2A8ECA5705FC33, 0x2E2A8ECA5705FC30,
    0x2E2A8ECA5705FC2F, 0x2E2A8ECA5705FC2F};

static int64_t q57(int v) { return (int64_t)((uint64_t)(int64_t)v << 57); }
static int64_t dbl(int64_t v) { return (int64_t)((uint64_t)v << 1); } /* `* 2`, wrapping */
/* conditional negation by a 0 / -1 mask: (v + m) ^ m */
static int64_t cneg(int64_t v, int64_t m) { return (int64_t)(((uint64_t)v + (uint64_t)m) ^ (uint64_t)m); }
/* the CORDIC's repeated iteration after `r` is 3 r + 3 (3 -> 12 -> 39), i.e. the 1-based 4, 13, 40 */
static int next_repeat(int r) { return 3 * r + 3; }

/* logexp.rs:34-125: 2^(logq57 / 2^57) rounded to an integer, 0 below 1, i64::MAX from 2^63 on */
int64_t orc_bexp64(int64_t logq57) {
  const int ipart = (int)(logq57 >> 57);
  if (ipart < 0) return 0;
  if (ipart >= 63) return INT64_MAX;
  int64_t z = logq57 - q57(ipart), w;
  if (z == 0) {
    w = (int64_t)1 << 62;
  } else {
    z = (int64_t)((uint64_t)z << 5); /* fractional part in Q62 */
    w = 0x26A3D0E401DD846D;          /* 2^61 / prod sqrt(1 - 2^-2i), repeats included */
    int i = 0, rep = 3;
    while (i < 32) {
      const int64_t m = -(int64_t)(z < 0);
      w += cneg(w >> (i + 1), m);
      z -= cneg(K_ATANH[i], m);
      if (i == rep) {
        rep = next_repeat(rep);
        continue;
      }
      z = dbl(z);
      i++;
    }
    int32_t wlo = 0;
    if (ipart > 30) { /* only the low bits move from here on; the table has converged */
      while (i < 61) {
        const int64_t m = -(int64_t)(z < 0);
        wlo += (int32_t)cneg(w >> i, m);
        z -= cneg(K_ATANH[31], m);
        if (i == rep) {
          rep = next_repeat(rep);
          continue;
        }
        z = dbl(z);
        i++;
      }
    }
    w = dbl(w) + wlo;
  }
  if (ipart < 62) w = ((w >> (61 - ipart)) + 1) >> 1;
  return w;
}

/* logexp.rs:130-174: log2(n) in Q57, -1 for n <= 0 */
int64_t orc_blog64(int64_t n) {
  if (n <= 0) return -1;
  const int ipart = 63 - __builtin_clzll((unsigned long long)n);
  const int64_t w = ipart > 61 ? n >> (ipart - 61) : (int64_t)((uint64_t)n << (61 - ipart));
  if ((w & (w - 1)) == 0) return q57(ipart);
  /* z = 2 atanh((w - 1) / (w + 1)) with x, y = cosh, sinh in Q61 */
  int64_t z = 0, x = w + ((int64_t)1 << 61), y = w - ((int64_t)1 << 61);
  int i = 0, rep = 3;
  while (i <= 61) {
    const int64_t m = -(int64_t)(y < 0);
    z += cneg(K_ATANH[i < 31 ? i : 31] >> i, m);
    const int64_t u = x >> (i + 1);
    x -= cneg(y >> (i + 1), m);
    y -= cneg(u, m);
    if (i == rep) {
      rep = next_repeat(rep);
      continue;
    }
    i++;
  }
  return q57(ipart) + ((z + 8) >> 4);
}

/* logexp.rs:271-286: polynomial log2 of a u32, Q11; -1 for 0 */
int32_t orc_blog32_q11(uint32_t w) {
  if (w == 0) return -1;
  const int ipart = 32 - __builtin_clz(w);
  const uint32_t norm = ipart > 16 ? w >> (ipart - 16) : w << (16 - ipart); /* [2^15, 2^16) */
  const int32_t n = (int32_t)norm - 49152;
  static const int32_t coef[4] = {2546, -5216, 15745, -6797}; /* Horner from the leading -1402 */
  int32_t p = -1402;
  for (int k = 0; k < 4; k++) p = ((n * p) >> 15) + coef[k];
  return (ipart << 11) + (p >> 3);
}

/* ------------------------------------------------------------------ DistortionScale (rdo.rs) */
#define DS_SHIFT 14
#define DS_MAX ((1u << 28) - 1)

static uint32_t clamp_scale(uint64_t v) { return v < 1 ? 1u : v > DS_MAX ? DS_MAX : (uint32_t)v; }

/* rdo.rs:618-630 */
uint32_t orc_dscale_mul(uint32_t a, uint32_t b) {
  return clamp_scale(((uint64_t)a * b + (1u << (DS_SHIFT - 1))) >> DS_SHIFT);
}

/* rdo.rs:585-594 */
uint32_t orc_dscale_inv_mean(const uint32_t *s, size_t n) {
  int64_t sum = 0;
  for (size_t i = 0; i < n; i++) sum += orc_blog32_q11(s[i]);
  const int64_t log_inv_mean_q11 = ((int64_t)DS_SHIFT << 11) - sum / (int64_t)n;
  const int64_t e = orc_bexp64((int64_t)((uint64_t)(log_inv_mean_q11 + ((int64_t)DS_SHIFT << 11)) << (57 - 11)));
  return e < 1 ? 1u : e > (int64_t)DS_MAX ? DS_MAX : (uint32_t)e;
}

/* rdo.rs:605-608 DistortionScale::blog64 */
int64_t orc_dscale_blog64(uint32_t s) { return orc_blog64((int64_t)s) - q57(DS_SHIFT); }

/* rdo.rs:506-553 + From<f64> (:652-658) + new (:579-583) */
uint32_t orc_distortion_scale_for(double propagate_cost, double intra_cost) {
  if (intra_cost == 0.) return 1u << DS_SHIFT;
  const double frac = (intra_cost + propagate_cost) / intra_cost;
  const double s = pow(frac, 1.0 / 3.0);
  const uint64_t den = 1u << (DS_SHIFT + 1);
  const double scaled = s * (double)den;
  /* `as u64` saturates (NaN -> 0) */
  const uint64_t num = !(scaled > 0.) ? 0 : scaled >= 18446744073709551616.0 ? UINT64_MAX : (uint64_t)scaled;
  const uint64_t sh = num << DS_SHIFT;
  const uint64_t raw = (sh > UINT64_MAX - den / 2 ? UINT64_MAX : sh + den / 2) / den;
  return raw <= DS_MAX ? (uint32_t)raw : DS_MAX;
}

/* api/internal.rs:1219-1230: the zip stops at the shorter map; later entries keep the default */
void orc_distortion_scales(const float *importances, size_t n_imp, const uint32_t *intra_costs, size_t n_intra,
                           uint32_t *scales) {
  for (size_t i = 0; i < n_imp; i++)
    scales[i] = i < n_intra ? orc_distortion_scale_for((double)importances[i], (double)intra_costs[i]) : 1u << DS_SHIFT;
}

/* encoder.rs:744-777.  activity NULL: compute_temporal_scores (spatiotemporal, when given, receives
 * the scaled distortion scales); else compute_spatiotemporal_scores.  Returns inv_mean.blog64() >> 1. */
int64_t orc_temporal_scores(uint32_t *scales, size_t n, const uint32_t *activity, uint32_t *spatiotemporal,
                            uint32_t *inv_mean_out) {
  uint32_t inv;
  if (activity) {
    for (size_t i = 0; i < n; i++) spatiotemporal[i] = orc_dscale_mul(scales[i], activity[i]);
    inv = orc_dscale_inv_mean(spatiotemporal, n);
    for (size_t i = 0; i < n; i++) spatiotemporal[i] = orc_dscale_mul(spatiotemporal[i], inv);
    for (size_t i = 0; i < n; i++) scales[i] = orc_dscale_mul(scales[i], inv);
  } else {
    inv = orc_dscale_inv_mean(scales, n);
    for (size_t i = 0; i < n; i++) scales[i] = orc_dscale_mul(scales[i], inv);
    if (spatiotemporal) memcpy(spatiotemporal, scales, n * sizeof *scales);
  }
  if (inv_mean_out) *inv_mean_out = inv;
  return orc_dscale_blog64(inv) >> 1;
}

/* ------------------------------------------------------------------ api/internal.rs */
/* floor division by 64 (internal.rs:1010-1017: `(v - (v < 0 ? 63 : 0)) / 64`) */
static int64_t floor64(int64_t v) { return (v - (v < 0 ? 63 : 0)) / 64; }

/* internal.rs:912-1071: one (frame, reference) step.  org / ref: pixel (0,0) of the two source luma
 * planes (readable wherever an 8x8 block at a vector's truncated position, or a ceil-grid block
 * past the frame edge, reads); w_imp x h_imp = ceil(W / 8) x ceil(H / 8); intra_costs: the source
 * frame's floor(W / 8) x floor(H / 8) map read flat in rows of w_imp (`chunks_exact(w_in_imp_b)`);
 * mvs: (row, col) per importance block on the ceil grid; future: the source frame's importances;
 * ref_importances += the propagated amounts. */
void orc_update_block_importances(const void *org, ptrdiff_t org_stride, const void *ref, ptrdiff_t ref_stride,
                                  int bpp, int w_imp, int h_imp, const uint32_t *intra_costs, size_t n_intra,
                                  const int16_t *mvs, const float *future, uint32_t len, float *ref_importances) {
  const size_t rows_by_intra = n_intra / (size_t)w_imp;
  const int rows = rows_by_intra < (size_t)h_imp ? (int)rows_by_intra : h_imp;
  for (int y = 0; y < rows; y++)
    for (int x = 0; x < w_imp; x++) {
      const size_t i = (size_t)y * w_imp + x;
      const int64_t rx = (int64_t)x * 64 + mvs[2 * i + 1], ry = (int64_t)y * 64 + mvs[2 * i];
      const ptrdiff_t px = (ptrdiff_t)(rx / 8), py = (ptrdiff_t)(ry / 8); /* truncating, as `isize / 8` */
      const uint8_t *o = (const uint8_t *)org + ((ptrdiff_t)(8 * y) * org_stride + 8 * x) * bpp;
      const uint8_t *r = (const uint8_t *)ref + (py * ref_stride + px) * bpp;
      const uint32_t satd = bpp == 1 ? orc_get_satd_u8(o, org_stride, r, ref_stride, 8, 8)
                                     : orc_get_satd_u16((const uint16_t *)o, org_stride, (const uint16_t *)r,
                                                        ref_stride, 8, 8);
      const float inter = (float)satd, intra = (float)intra_costs[i];
      const float frac = intra <= inter ? 0.f : 1.f - inter / intra;
      const float amount = (intra + future[i]) * frac / (float)len;
      const int64_t tlx = floor64(rx) * 64, tly = floor64(ry) * 64;
      const int64_t fx = rx - tlx, fy = ry - tly;
      const int64_t wts[4] = {(64 - fx) * (64 - fy), fx * (64 - fy), (64 - fx) * fy, fx * fy};
      for (int k = 0; k < 4; k++) { /* TL, TR, BL, BR */
        const int64_t bx = tlx / 64 + (k & 1), by = tly / 64 + (k >> 1);
        const float weight = (float)wts[k] / 4096.f;
        if (bx >= 0 && by >= 0 && bx < w_imp && by < h_imp) ref_importances[by * w_imp + bx] += amount * weight;
      }
    }
}

/* internal.rs:1095-1206: zero every frame's importances, then run the steps in the given order.
 * frames[f]: pixel (0,0) of frame f's source luma (all share stride / bpp / size);
 * intra_costs: nframes x floor(W/8)*floor(H/8); mvs: per mv_index a ceil-grid map of (row, col);
 * steps: 4 u32 per step {src, dst, len, mv_index}; importances: nframes x w_imp*h_imp. */
void orc_block_importances(size_t nframes, const void *const *frames, ptrdiff_t stride, int bpp, int width,
                           int height, const uint32_t *intra_costs, const int16_t *mvs, size_t nsteps,
                           const uint32_t *steps, float *importances) {
  const int w_imp = (width + 7) / 8, h_imp = (height + 7) / 8;
  const size_t n_imp = (size_t)w_imp * h_imp, n_intra = (size_t)(width / 8) * (height / 8);
  for (size_t k = 0; k < nframes * n_imp; k++) importances[k] = 0.f;
  for (size_t s = 0; s < nsteps; s++) {
    const uint32_t src = steps[4 * s], dst = steps[4 * s + 1], len = steps[4 * s + 2], mvi = steps[4 * s + 3];
    orc_update_block_importances(frames[src], stride, frames[dst], stride, bpp, w_imp, h_imp,
                                 intra_costs + (size_t)src * n_intra, n_intra, mvs + (size_t)mvi * 2 * n_imp,
                                 importances + (size_t)src * n_imp, len, importances + (size_t)dst * n_imp);
  }
}
