/*
 * oracle/lrf.c — loop restoration's frame filter, stripe by stripe and unit by unit, the way rav1e runs it
 * (TEST INFRASTRUCTURE ONLY; see lrf.h for the contract and what pins it).
 */
#include "lrf.h"

#include <stdlib.h>
#include <string.h>

#include "oracle.h"

#define SGRPROJ_RST_BITS 4
#define SGRPROJ_PRJ_BITS 7
#define SGRPROJ_MTABLE_BITS 20
#define SGRPROJ_SGR_BITS 8
#define SGRPROJ_RECIP_BITS 12
#define STRIPE_IMAGE_MAX (256 + 128)                      /* lrf.rs:100-104 */
#define STRIPE_IMAGE_STRIDE (STRIPE_IMAGE_MAX + 6 + 2)
#define STRIPE_IMAGE_HEIGHT (64 + 6 + 2)
#define IMAGE_WIDTH_MAX STRIPE_IMAGE_MAX                  /* max(STRIPE_IMAGE_MAX, SOLVE_IMAGE_MAX) */

/* SGRPROJ_PARAMS_S (lrf.rs:56-73): s for radius 2, s for radius 1 */
static const uint32_t kSgrS[16][2] = {{140, 3236}, {112, 2158}, {93, 1618}, {80, 1438}, {70, 1295}, {58, 1177},
                                      {47, 1079},  {37, 996},   {30, 925},  {25, 863},  {0, 2589},  {0, 1618},
                                      {0, 1177},   {0, 925},    {56, 0},    {22, 0}};

typedef struct {
  const uint8_t *d;
  ptrdiff_t stride; /* elements */
  int bpp;
} Src;

static int rd(const Src *s, long x, long y) {
  const ptrdiff_t i = (ptrdiff_t)y * s->stride + x;
  return s->bpp == 1 ? s->d[i] : ((const uint16_t *)s->d)[i];
}

static void wr(const Src *s, long x, long y, int v) {
  const ptrdiff_t i = (ptrdiff_t)y * s->stride + x;
  if (s->bpp == 1) ((uint8_t *)s->d)[i] = (uint8_t)v;
  else ((uint16_t *)s->d)[i] = (uint16_t)v;
}

static long clampl(long v, long lo, long hi) { return v < lo ? lo : v > hi ? hi : v; }
static long minl(long a, long b) { return a < b ? a : b; }
static long maxl(long a, long b) { return a > b ? a : b; }

/* ---------------------------------------------------------------- Wiener (lrf.rs:1099-1207) */
static void wiener_stripe_filter(const int8_t coeffs[2][3], int bd, long crop_w, long crop_h, long stripe_w,
                                 long stripe_h, long stripe_x, long stripe_y, const Src *cdeffed,
                                 const Src *deblocked, const Src *out) {
  const int round_h = bd == 12 ? 5 : 3, round_v = bd == 12 ? 9 : 11;
  const int offset = 1 << (bd + 7 - round_h - 1);
  const int limit = (1 << (bd + 1 + 7 - round_h)) - 1;
  int vf[7], hf[7], work[64 + 7];
  for (int k = 0; k < 3; k++) {
    vf[k] = vf[6 - k] = coeffs[0][k];
    hf[k] = hf[6 - k] = coeffs[1][k];
  }
  vf[3] = 128 - 2 * (coeffs[0][0] + coeffs[0][1] + coeffs[0][2]);
  hf[3] = 128 - 2 * (coeffs[1][0] + coeffs[1][1] + coeffs[1][2]);

  const long start_wi = stripe_y < 0 ? -stripe_y : 0;
  const long start_yi = stripe_y < 0 ? 0 : stripe_y;
  const long end_i =
      maxl(0, stripe_h + stripe_y > crop_h ? crop_h - stripe_y - start_wi : stripe_h - start_wi);

  for (long xi = stripe_x; xi < stripe_x + stripe_w; xi++) {
    const long n = minl(7, crop_w + 3 - xi);
    for (long yi = stripe_y - 3; yi < stripe_y + stripe_h + 4; yi++) {
      const Src *src;
      long ly;
      if (yi < stripe_y) {
        ly = maxl(clampl(yi, 0, crop_h - 1), stripe_y - 2);
        src = deblocked;
      } else if (yi < stripe_y + stripe_h) {
        ly = clampl(yi, 0, crop_h - 1);
        src = cdeffed;
      } else {
        ly = minl(clampl(yi, 0, crop_h - 1), stripe_y + stripe_h + 1);
        src = deblocked;
      }
      const int start = rd(src, 0, ly), end = rd(src, crop_w - 1, ly);
      int acc = 0;
      for (long i = 0; i < 3 - xi; i++) acc += hf[i] * start;
      const long off = 3 - xi, s = maxl(0, off);
      for (long i = s; i < n; i++) acc += hf[i] * rd(src, i - off, ly);
      for (long i = n; i < 7; i++) acc += hf[i] * end;
      acc = (acc + (1 << round_h >> 1)) >> round_h;
      work[yi - stripe_y + 3] = (int)clampl(acc, -offset, limit - offset);
    }
    for (long k = 0; k < end_i; k++) {
      int acc = 0;
      for (int i = 0; i < 7; i++) acc += vf[i] * work[start_wi + k + i];
      wr(out, xi, start_yi + k, (int)clampl((acc + (1 << round_v >> 1)) >> round_v, 0, (1 << bd) - 1));
    }
  }
}

/* ---------------------------------------------------------------- self-guided */
/* setup_integral_image (lrf.rs:529-627) with VertPaddedIter (:381-479) and HorzPaddedIter (:481-527).  x, y:
 * the stripe's origin in the plane; crop_w / crop_h relative to it, as the call site passes them. */
static void setup_integral_image(uint32_t *ii, uint32_t *sq, long crop_w, long crop_h, long stripe_w,
                                 long stripe_h, long x, long y, const Src *cdeffed, const Src *deblocked) {
  const long left_w = 4, right_w = 3;
  const long left_uniques = x == 0 ? 0 : left_w;
  const long right_uniques = minl(right_w, crop_w - stripe_w);
  const long row_uniques = left_uniques + stripe_w + right_uniques;
  const long start_index_x = x == 0 ? -left_w : 0;
  const long x0 = x - left_uniques; /* the slices go_left(left_uniques) */
  /* VertPaddedIter::new with stripe_h rounded up to even, r = 2 */
  const long sh = stripe_h + (stripe_h & 1);
  const long crop = crop_h + y, stripe_begin = y, stripe_end = sh + y;
  const long y_first = y - 4, y_end = 4 + sh + 2 + y_first;
  const long width = left_w + stripe_w + right_w;
  for (long yy = y_first; yy < y_end; yy++) {
    const long cropped_y = clampl(yy, 0, crop - 1);
    const long ly = clampl(cropped_y, stripe_begin - 2, stripe_end + 1);
    const Src *src = (ly >= stripe_begin && ly < stripe_end) ? cdeffed : deblocked;
    const long r = yy - y_first;
    uint32_t sum = 0, sq_sum = 0;
    for (long j = 0; j < width; j++) {
      const long xi = clampl(start_index_x + j, 0, row_uniques - 1);
      const uint32_t cur = (uint32_t)rd(src, x0 + xi, ly);
      sum += cur;
      sq_sum += cur * cur;
      ii[r * STRIPE_IMAGE_STRIDE + j] = r ? sum + ii[(r - 1) * STRIPE_IMAGE_STRIDE + j] : sum;
      sq[r * STRIPE_IMAGE_STRIDE + j] = r ? sq_sum + sq[(r - 1) * STRIPE_IMAGE_STRIDE + j] : sq_sum;
    }
  }
}

/* get_integral_square (:364-379), wrapping */
static uint32_t integral_square(const uint32_t *im, long x, long y, long size) {
  const long s = STRIPE_IMAGE_STRIDE;
  return im[y * s + x] + im[(y + size) * s + x + size] - im[(y + size) * s + x] - im[y * s + x + size];
}

/* sgrproj_sum_finish (:344-362) */
static void sum_finish(uint32_t ssq, uint32_t sum, uint32_t n, uint32_t one_over_n, uint32_t s, int bd, uint32_t *ra,
                       uint32_t *rb) {
  const int bdm8 = bd - 8;
  const uint32_t scaled_ssq = (ssq + ((1u << (2 * bdm8)) >> 1)) >> (2 * bdm8);
  const uint32_t scaled_sum = (sum + ((1u << bdm8) >> 1)) >> bdm8;
  const uint32_t t0 = scaled_ssq * n, t1 = scaled_sum * scaled_sum;
  const uint32_t p = t0 > t1 ? t0 - t1 : 0;
  const uint32_t z = (p * s + (1u << SGRPROJ_MTABLE_BITS >> 1)) >> SGRPROJ_MTABLE_BITS;
  const uint32_t a = z >= 255 ? 256 : z == 0 ? 1 : ((z << SGRPROJ_SGR_BITS) + z / 2) / (z + 1);
  const uint32_t b = ((1u << SGRPROJ_SGR_BITS) - a) * sum * one_over_n;
  *ra = a;
  *rb = (b + (1u << SGRPROJ_RECIP_BITS >> 1)) >> SGRPROJ_RECIP_BITS;
}

/* sgrproj_box_ab_internal (:175-200): one a / b row for stripe_w + 2 columns.  off = 0 for r = 2 and
 * stride + 1 for r = 1, as the callers offset the images. */
static void box_ab(int r, uint32_t *af, uint32_t *bf, const uint32_t *ii, const uint32_t *sq, long y,
                   long stripe_w, uint32_t s, int bd) {
  const long d = 2 * r + 1, off = r == 1 ? STRIPE_IMAGE_STRIDE + 1 : 0;
  const uint32_t n = (uint32_t)(d * d), one_over_n = r == 1 ? 455 : 164;
  for (long x = 0; x < stripe_w + 2; x++)
    sum_finish(integral_square(sq + off, x, y, d), integral_square(ii + off, x, y, d), n, one_over_n, s, bd, &af[x],
               &bf[x]);
}

/* sgrproj_stripe_filter (:629-830); cdeffed and out are addressed from the stripe's origin (x, y) */
static void sgrproj_stripe_filter(int set, const int8_t xqd[2], int bd, const uint32_t *ii, const uint32_t *sq,
                                  long stripe_w, long stripe_h, long x, long y, const Src *cdeffed, const Src *out) {
  static __thread uint32_t a_r2[2][IMAGE_WIDTH_MAX + 2], b_r2[2][IMAGE_WIDTH_MAX + 2];
  static __thread uint32_t a_r1[3][IMAGE_WIDTH_MAX + 2], b_r1[3][IMAGE_WIDTH_MAX + 2];
  static __thread uint32_t f_r2_0[IMAGE_WIDTH_MAX], f_r2_1[IMAGE_WIDTH_MAX], f_r1[IMAGE_WIDTH_MAX];
  const uint32_t s_r2 = kSgrS[set][0], s_r1 = kSgrS[set][1];
  const int shift = 5 + SGRPROJ_SGR_BITS - SGRPROJ_RST_BITS, shifto = 4 + SGRPROJ_SGR_BITS - SGRPROJ_RST_BITS;
  if (s_r2 > 0) box_ab(2, a_r2[0], b_r2[0], ii, sq, 0, stripe_w, s_r2, bd);
  if (s_r1 > 0) {
    box_ab(1, a_r1[0], b_r1[0], ii, sq, 0, stripe_w, s_r1, bd);
    box_ab(1, a_r1[1], b_r1[1], ii, sq, 1, stripe_w, s_r1, bd);
  }
  for (long yy = 0; yy < stripe_h; yy += 2) {
    const uint32_t *f_r2_ab[2];
    if (s_r2 > 0) {
      const int c = (int)((yy / 2) % 2), o = (int)((yy / 2 + 1) % 2);
      box_ab(2, a_r2[o], b_r2[o], ii, sq, yy + 2, stripe_w, s_r2, bd);
      /* sgrproj_box_f_r2 (:300-342).  Row yy + 1's output is only used when it is inside the stripe, so it
       * is only formed there: the reference also reads cdeffed row yy + 1 past an odd stripe's end. */
      const int two = yy + 1 < stripe_h;
      for (long i = 0; i < stripe_w; i++) {
        const uint32_t a = 5 * (a_r2[c][i] + a_r2[c][i + 2]) + 6 * a_r2[c][i + 1];
        const uint32_t b = 5 * (b_r2[c][i] + b_r2[c][i + 2]) + 6 * b_r2[c][i + 1];
        const uint32_t ao = 5 * (a_r2[o][i] + a_r2[o][i + 2]) + 6 * a_r2[o][i + 1];
        const uint32_t bo = 5 * (b_r2[o][i] + b_r2[o][i + 2]) + 6 * b_r2[o][i + 1];
        const uint32_t v = (a + ao) * (uint32_t)rd(cdeffed, x + i, y + yy) + b + bo;
        f_r2_0[i] = (v + (1u << shift >> 1)) >> shift;
        if (two) {
          const uint32_t vo = ao * (uint32_t)rd(cdeffed, x + i, y + yy + 1) + bo;
          f_r2_1[i] = (vo + (1u << shifto >> 1)) >> shifto;
        }
      }
      f_r2_ab[0] = f_r2_0;
      f_r2_ab[1] = f_r2_1;
    } else {
      /* sgrproj_box_f_r0 for row yy, shared by both rows (:740-749) */
      for (long i = 0; i < stripe_w; i++) f_r2_0[i] = (uint32_t)rd(cdeffed, x + i, y + yy) << SGRPROJ_RST_BITS;
      f_r2_ab[0] = f_r2_ab[1] = f_r2_0;
    }
    for (long dy = 0; dy < minl(2, stripe_h - yy); dy++) {
      const long row = yy + dy;
      if (s_r1 > 0) {
        const int i0 = (int)(row % 3), i1 = (int)((row + 1) % 3), i2 = (int)((row + 2) % 3);
        box_ab(1, a_r1[i2], b_r1[i2], ii, sq, row + 2, stripe_w, s_r1, bd);
        for (long i = 0; i < stripe_w; i++) { /* sgrproj_box_f_r1 (:266-291) */
          const uint32_t a = 3 * (a_r1[i0][i] + a_r1[i2][i] + a_r1[i0][i + 2] + a_r1[i2][i + 2]) +
                             4 * (a_r1[i1][i] + a_r1[i0][i + 1] + a_r1[i1][i + 1] + a_r1[i2][i + 1] + a_r1[i1][i + 2]);
          const uint32_t b = 3 * (b_r1[i0][i] + b_r1[i2][i] + b_r1[i0][i + 2] + b_r1[i2][i + 2]) +
                             4 * (b_r1[i1][i] + b_r1[i0][i + 1] + b_r1[i1][i + 1] + b_r1[i2][i + 1] + b_r1[i1][i + 2]);
          const uint32_t v = a * (uint32_t)rd(cdeffed, x + i, y + row) + b;
          f_r1[i] = (v + (1u << shift >> 1)) >> shift;
        }
      } else {
        for (long i = 0; i < stripe_w; i++) f_r1[i] = (uint32_t)rd(cdeffed, x + i, y + row) << SGRPROJ_RST_BITS;
      }
      const int w0 = xqd[0], w1 = xqd[1], w2 = (1 << SGRPROJ_PRJ_BITS) - w0 - w1;
      for (long i = 0; i < stripe_w; i++) { /* apply_filter (:796-815) */
        const int u = rd(cdeffed, x + i, y + row) << SGRPROJ_RST_BITS;
        const int v = w0 * (int)f_r2_ab[dy][i] + w1 * u + w2 * (int)f_r1[i];
        const int s = (v + (1 << (SGRPROJ_RST_BITS + SGRPROJ_PRJ_BITS) >> 1)) >> (SGRPROJ_RST_BITS + SGRPROJ_PRJ_BITS);
        wr(out, x + i, y + row, (int)clampl(s, 0, (1 << bd) - 1));
      }
    }
  }
}

/* ---------------------------------------------------------------- lrf_filter_frame (:1481-1585) */
void orc_lrf_filter_frame(void *const *out, const ptrdiff_t *out_stride, const void *const *cdeffed,
                          const ptrdiff_t *cdeffed_stride, const void *const *deblocked,
                          const ptrdiff_t *deblocked_stride, int bpp, int planes, int xdec, int ydec,
                          int frame_width, int frame_height, int bit_depth, int enable_cdef, const int *unit_size,
                          const uint8_t *const *units) {
  uint32_t *ii = calloc((size_t)STRIPE_IMAGE_STRIDE * STRIPE_IMAGE_HEIGHT, sizeof(uint32_t));
  uint32_t *sq = calloc((size_t)STRIPE_IMAGE_STRIDE * STRIPE_IMAGE_HEIGHT, sizeof(uint32_t));
  const long stripe_n = (frame_height + 7) / 64 + 1;
  for (int p = 0; p < planes; p++) {
    const int xd = p ? xdec : 0, yd = p ? ydec : 0;
    const long crop_w = (frame_width + (1 << xd >> 1)) >> xd;
    const long crop_h = (frame_height + (1 << yd >> 1)) >> yd;
    const long us = unit_size[p];
    /* RestorationState::new (:1323-1324, :1431-1440) and RestorationPlane::new (:1275) */
    const long cols = maxl(1, (crop_w + (us >> 1)) / us), rows = maxl(1, (crop_h + (us >> 1)) / us);
    const long stripe_height = (p && xdec && ydec) ? 32 : 64;
    const Src C_ = {cdeffed[p], cdeffed_stride[p], bpp}, D = {deblocked[p], deblocked_stride[p], bpp};
    const Src O = {out[p], out_stride[p], bpp};
    for (long si = 0; si < stripe_n; si++) {
      long sy, ssize;
      if (si == 0) {
        sy = 0;
        ssize = (64 - 8) >> yd;
      } else {
        sy = (si * 64 - 8) >> yd;
        ssize = minl(64 >> yd, crop_h - sy);
      }
      for (long rux = 0; rux < cols; rux++) {
        const long x = rux * us, size = rux == cols - 1 ? crop_w - x : us;
        /* restoration_unit_by_stripe (:1295-1312) */
        const long ruy = minl(si * stripe_height / us, rows - 1);
        const uint8_t *u = units[p] + (ruy * cols + minl(rux, cols - 1)) * 12;
        if (u[0] == 1) {
          const int8_t coeffs[2][3] = {{(int8_t)u[4], (int8_t)u[5], (int8_t)u[6]},
                                       {(int8_t)u[7], (int8_t)u[8], (int8_t)u[9]}};
          wiener_stripe_filter(coeffs, bit_depth, crop_w, crop_h, size, ssize, x, sy, &C_, &D, &O);
        } else if (u[0] == 2) {
          if (!enable_cdef) continue;
          const int8_t xqd[2] = {(int8_t)u[2], (int8_t)u[3]};
          setup_integral_image(ii, sq, crop_w - x, crop_h - sy, size, ssize, x, sy, &C_, &D);
          sgrproj_stripe_filter(u[1], xqd, bit_depth, ii, sq, size, ssize, x, sy, &C_, &O);
        }
      }
    }
  }
  free(ii);
  free(sq);
}
