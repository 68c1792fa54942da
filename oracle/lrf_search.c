/*
 * oracle/lrf_search.c — the restoration search of rdo_loop_decision, item by item, the way rav1e runs it
 * (TEST INFRASTRUCTURE ONLY; see lrf_search.h for the contract and what pins it).
 */
#include "lrf_search.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "lrf.h"
#include "oracle.h"

/* The integral image, the box helpers and the stripe filter are oracle/lrf.c's own file-static functions: this
 * file compiles them in rather than restating them.  lrf.c's frame filter comes along under another name so the
 * library keeps one orc_lrf_filter_frame; that copy is hidden and never called.  The headers lrf.c includes come
 * first, so only the definitions below take the hidden visibility, not the library's shared declarations. */
#define orc_lrf_filter_frame orc_lrf_filter_frame_in_lrf_search_
#pragma GCC visibility push(hidden)
#include "lrf.c"
#pragma GCC visibility pop
#undef orc_lrf_filter_frame

#define SOLVE_MAX 256
#define OD_BITRES 3

static const int kXqdMin[2] = {-96, -32}, kXqdMax[2] = {31, 95}; /* lrf.rs:46-48 */



/* ---------------------------------------------------------------- rates (ec.rs) */
/* count_quniform (ec.rs:639-652) */
static uint32_t count_quniform(uint32_t n, uint32_t v) {
  uint32_t bits = 0;
  if (n > 1) {
    const uint32_t l = 32 - (uint32_t)__builtin_clz(n), m = (1u << l) - n;
    bits += (l - 1) << OD_BITRES;
    if (v >= m) bits += 1 << OD_BITRES;
  }
  return bits;
}

/* count_subexp (ec.rs:683-707) */
static uint32_t count_subexp(uint32_t n, uint32_t k, uint32_t v) {
  uint32_t i = 0, mk = 0, bits = 0;
  for (;;) {
    const uint32_t b = i ? k + i - 1 : k, a = 1u << b;
    if (n <= mk + 3 * a) {
      bits += count_quniform(n - mk, v - mk);
      break;
    }
    bits += 1 << OD_BITRES;
    if (v >= mk + a) {
      i++;
      mk += a;
    } else {
      bits += b << OD_BITRES;
      break;
    }
  }
  return bits;
}

/* recenter (ec.rs:381-389) */
static uint32_t recenter(uint32_t r, uint32_t v) { return v > (r << 1) ? v : v >= r ? (v - r) << 1 : ((r - v) << 1) - 1; }

/* count_signed_subexp_with_ref -> count_unsigned_subexp_with_ref (ec.rs:726-773) */
static uint32_t count_signed_subexp_with_ref(int v, int low, int high, uint32_t k, int r) {
  const uint32_t uv = (uint32_t)(v - low), n = (uint32_t)(high - low), ur = (uint32_t)(r - low);
  return (ur << 1) <= n ? count_subexp(n, k, recenter(ur, uv)) : count_subexp(n, k, recenter(n - 1 - ur, n - 1 - uv));
}

/* count_lrf_switchable (context/frame_header.rs:14-45) of a None (type 0) or Sgrproj (type 2) filter */
static uint32_t lrf_rate(const b200_lrf_search_item *it, int type, int set, const int8_t xqd[2]) {
  if (type == 0) return it->none_bits;
  uint32_t bits = it->sgr_bits + (4u << OD_BITRES); /* SGRPROJ_PARAMS_BITS << OD_BITRES */
  for (int i = 0; i < 2; i++)
    if (kSgrS[set][i] > 0)
      bits += count_signed_subexp_with_ref(xqd[i], kXqdMin[i], kXqdMax[i] + 1, 4, it->sgrproj_ref[i]);
  return bits;
}

/* ---------------------------------------------------------------- sgrproj_solve (lrf.rs:846-1096) */
/* Rust's saturating `as i32` (NaN -> 0) */
static int32_t sat_i32(double v) {
  if (v != v) return 0;
  if (v >= 2147483647.0) return INT32_MAX;
  if (v <= -2147483648.0) return INT32_MIN;
  return (int32_t)v;
}

static int32_t clampi(int32_t v, int32_t lo, int32_t hi) { return v < lo ? lo : v > hi ? hi : v; }

/* in / src addressed from the area's origin, the unit at (x, y), w x h = vis */
static void sgrproj_solve(int set, int bd, const uint32_t *ii, const uint32_t *sq, const Src *src, const Src *in,
                          long w, long h, long x, long y, int8_t out[2]) {
  uint32_t a_r2[2][SOLVE_MAX + 2], b_r2[2][SOLVE_MAX + 2], a_r1[3][SOLVE_MAX + 2], b_r1[3][SOLVE_MAX + 2];
  uint32_t f_r2_0[SOLVE_MAX], f_r2_1[SOLVE_MAX], f_r1[SOLVE_MAX];
  const uint32_t s_r2 = kSgrS[set][0], s_r1 = kSgrS[set][1];
  double H[2][2] = {{0., 0.}, {0., 0.}}, c[2] = {0., 0.};
  if (s_r2 > 0) box_ab(2, a_r2[0], b_r2[0], ii, sq, 0, w, s_r2, bd);
  if (s_r1 > 0) {
    box_ab(1, a_r1[0], b_r1[0], ii, sq, 0, w, s_r1, bd);
    box_ab(1, a_r1[1], b_r1[1], ii, sq, 1, w, s_r1, bd);
  }
  for (long yy = 0; yy < h; yy += 2) {
    const uint32_t *f2ab[2];
    if (s_r2 > 0) {
      const int cu = (int)((yy / 2) % 2), o = (int)((yy / 2 + 1) % 2);
      box_ab(2, a_r2[o], b_r2[o], ii, sq, yy + 2, w, s_r2, bd);
      for (long i = 0; i < w; i++) { /* sgrproj_box_f_r2 (lrf.rs:300-342) */
        const uint32_t a = 5 * (a_r2[cu][i] + a_r2[cu][i + 2]) + 6 * a_r2[cu][i + 1];
        const uint32_t b = 5 * (b_r2[cu][i] + b_r2[cu][i + 2]) + 6 * b_r2[cu][i + 1];
        const uint32_t ao = 5 * (a_r2[o][i] + a_r2[o][i + 2]) + 6 * a_r2[o][i + 1];
        const uint32_t bo = 5 * (b_r2[o][i] + b_r2[o][i + 2]) + 6 * b_r2[o][i + 1];
        f_r2_0[i] = ((a + ao) * (uint32_t)rd(in, x + i, y + yy) + b + bo + (1u << 8)) >> 9;
        if (yy + 1 < h) f_r2_1[i] = (ao * (uint32_t)rd(in, x + i, y + yy + 1) + bo + (1u << 7)) >> 8;
      }
      f2ab[0] = f_r2_0;
      f2ab[1] = f_r2_1;
    } else {
      for (long i = 0; i < w; i++) f_r2_0[i] = (uint32_t)rd(in, x + i, y + yy) << 4;
      f2ab[0] = f2ab[1] = f_r2_0;
    }
    for (long dy = 0; dy < minl(2, h - yy); dy++) {
      const long row = yy + dy;
      if (s_r1 > 0) {
        const int i0 = (int)(row % 3), i1 = (int)((row + 1) % 3), i2 = (int)((row + 2) % 3);
        box_ab(1, a_r1[i2], b_r1[i2], ii, sq, row + 2, w, s_r1, bd);
        for (long i = 0; i < w; i++) { /* sgrproj_box_f_r1 (lrf.rs:266-291) */
          const uint32_t a = 3 * (a_r1[i0][i] + a_r1[i2][i] + a_r1[i0][i + 2] + a_r1[i2][i + 2]) +
                             4 * (a_r1[i1][i] + a_r1[i0][i + 1] + a_r1[i1][i + 1] + a_r1[i2][i + 1] + a_r1[i1][i + 2]);
          const uint32_t b = 3 * (b_r1[i0][i] + b_r1[i2][i] + b_r1[i0][i + 2] + b_r1[i2][i + 2]) +
                             4 * (b_r1[i1][i] + b_r1[i0][i + 1] + b_r1[i1][i + 1] + b_r1[i2][i + 1] + b_r1[i1][i + 2]);
          f_r1[i] = (a * (uint32_t)rd(in, x + i, y + row) + b + (1u << 8)) >> 9;
        }
      } else {
        for (long i = 0; i < w; i++) f_r1[i] = (uint32_t)rd(in, x + i, y + row) << 4;
      }
      /* process_line (lrf.rs:997-1037): i64 line sums, added to the f64 totals */
      int64_t h00 = 0, h11 = 0, h01 = 0, c0 = 0, c1 = 0;
      for (long i = 0; i < w; i++) {
        const int32_t u = rd(in, x + i, y + row) << 4;
        const int64_t s = (int64_t)((rd(src, x + i, y + row) << 4) - u);
        const int64_t f2 = (int64_t)((int32_t)f2ab[dy][i] - u), f1 = (int64_t)((int32_t)f_r1[i] - u);
        h00 += f2 * f2;
        h11 += f1 * f1;
        h01 += f1 * f2;
        c0 += f2 * s;
        c1 += f1 * s;
      }
      H[0][0] += (double)h00;
      H[1][1] += (double)h11;
      H[0][1] += (double)h01;
      c[0] += (double)c0;
      c[1] += (double)c1;
    }
  }
  const double n = (double)w * (double)h;
  H[0][0] /= n;
  H[0][1] /= n;
  H[1][1] /= n;
  H[1][0] = H[0][1];
  c[0] *= 128.0 / n;
  c[1] *= 128.0 / n;
  int32_t xq0, xq1;
  if (s_r2 == 0) {
    xq0 = 0;
    xq1 = H[1][1] == 0. ? 0 : sat_i32(round(c[1] / H[1][1]));
  } else if (s_r1 == 0) {
    xq0 = H[0][0] == 0. ? 0 : sat_i32(round(c[0] / H[0][0]));
    xq1 = 0;
  } else {
    const double det = fma(H[0][0], H[1][1], -(H[0][1] * H[1][0]));
    if (det == 0.) {
      xq0 = xq1 = 0;
    } else {
      const double div1 = fma(H[1][1], c[0], -(H[0][1] * c[1]));
      const double div2 = fma(H[0][0], c[1], -(H[1][0] * c[0]));
      xq0 = sat_i32(round(div1 / det));
      xq1 = sat_i32(round(div2 / det));
    }
  }
  const int32_t xqd0 = clampi(xq0, kXqdMin[0], kXqdMax[0]);
  /* (1 << SGRPROJ_PRJ_BITS) - xqd0 - xq1 in i32; wrapping, as a release build computes it */
  const int32_t xqd1 = clampi((int32_t)(128u - (uint32_t)xqd0 - (uint32_t)xq1), kXqdMin[1], kXqdMax[1]);
  out[0] = (int8_t)xqd0;
  out[1] = (int8_t)xqd1;
}

/* ---------------------------------------------------------------- rdo_loop_plane_error (rdo.rs:2027-2093) */
/* src / test addressed from the area's origin; blocks [bx0, bx0 + nb) x [by0, by0 + nb) of the area's 8x8
 * grid, those inside cols8 x rows8 counted; gbx0 / gby0: the area's first 8x8 block in the frame */
static uint64_t plane_error(const Src *src, const Src *test, int p, int xd, int yd, int bd, long bx0, long by0,
                            long nbx, long nby, long cols8, long rows8, const uint32_t *imp, long w8, long gbx0,
                            long gby0, uint32_t dscale) {
  uint64_t e = 0;
  const int bw = 8 >> xd, bh = 8 >> yd;
  for (long by = by0; by < by0 + nby && by < rows8; by++)
    for (long bx = bx0; bx < bx0 + nbx && bx < cols8; bx++) {
      const uint32_t bias = imp ? imp[(size_t)(gby0 + by) * w8 + gbx0 + bx] : (1u << 14);
      const ptrdiff_t so = ((ptrdiff_t)by * bh * src->stride + bx * bw) * src->bpp;
      const ptrdiff_t to = ((ptrdiff_t)by * bh * test->stride + bx * bw) * test->bpp;
      const void *s = src->d + so, *t = test->d + to;
      if (p == 0) {
        const uint32_t d = src->bpp == 1 ? orc_cdef_dist_kernel_u8(s, src->stride, t, test->stride, 8, 8, bd, NULL)
                                         : orc_cdef_dist_kernel_u16(s, src->stride, t, test->stride, 8, 8, bd, NULL);
        e += orc_distortion_scale_mul(bias, d);
      } else {
        const uint32_t scale[4] = {bias, bias, bias, bias};
        e += src->bpp == 1 ? orc_weighted_sse_u8(s, src->stride, t, test->stride, scale, 2, bw, bh)
                           : orc_weighted_sse_u16(s, src->stride, t, test->stride, scale, 2, bw, bh);
      }
    }
  return orc_distortion_scale_mul(dscale, e);
}

/* RestorationFilter::notequal (lrf.rs:139-160) for None / Sgrproj */
static int notequal(const b200_lrf_unit *a, const b200_lrf_unit *b) {
  if (a->type != b->type) return 1;
  return a->type == 2 && !(a->set == b->set && a->xqd[0] == b->xqd[0] && a->xqd[1] == b->xqd[1]);
}

void orc_lrf_search(const void *const *lrf_in, const ptrdiff_t *lrf_in_stride, const void *const *src,
                    const ptrdiff_t *src_stride, int bpp, int xdec, int ydec, int frame_width, int frame_height,
                    int bit_depth, const int *unit_size, int reduced_sets, const uint32_t *imp_scales,
                    const uint32_t *dist_scale, double lambda, const b200_cdef_rdo_area *areas,
                    const b200_lrf_search_item *items, size_t n_items, b200_lrf_unit *best, double *cost,
                    uint8_t *changed, int8_t *xqd, uint64_t *err, double *cand_cost) {
  const size_t ii_n = (size_t)STRIPE_IMAGE_STRIDE * (SOLVE_MAX + 8);
  uint32_t *ii = calloc(ii_n, sizeof(uint32_t)), *sq = calloc(ii_n, sizeof(uint32_t));
  const long w8 = (frame_width + 7) >> 3;
  for (size_t k = 0; k < n_items; k++) {
    const b200_lrf_search_item *it = &items[k];
    const b200_cdef_rdo_area *ar = &areas[it->area];
    const int p = it->plane, xd = p ? xdec : 0, yd = p ? ydec : 0;
    const long ax = ar->sbx * 64L, ay = ar->sby * 64L;
    /* the area's scratch copy (rdo.rs:2152-2157, 2277-2284) */
    const long crop_w = frame_width - ax, crop_h = frame_height - ay;
    const long aw = (minl(crop_w, ar->sb_w * 64L) + 7) & ~7L, ah = (minl(crop_h, ar->sb_h * 64L) + 7) & ~7L;
    const long us = unit_size[p], lru_sb_w = (us << xd) / 64, lru_sb_h = (us << yd) / 64;
    const long po_x = it->lru_x * lru_sb_w * 64 >> xd, po_y = it->lru_y * lru_sb_h * 64 >> yd;
    const long vis_w = minl(us, (crop_w >> xd) - po_x), vis_h = minl(us, (crop_h >> yd) - po_y);
    const Src in = {(const uint8_t *)lrf_in[p] + ((ay >> yd) * lrf_in_stride[p] + (ax >> xd)) * bpp,
                    lrf_in_stride[p], bpp};
    const Src sr = {(const uint8_t *)src[p] + ((ay >> yd) * src_stride[p] + (ax >> xd)) * bpp, src_stride[p], bpp};
    /* lrf_work (rdo.rs:2331-2341): Plane::new of the scratch copy's size */
    const long ww = aw >> xd, wh = ah >> yd;
    uint8_t *work = malloc((size_t)ww * wh * bpp);
    for (long i = 0; i < ww * wh; i++) {
      if (bpp == 1) work[i] = B200_LRF_WORK_FILL;
      else ((uint16_t *)work)[i] = B200_LRF_WORK_FILL;
    }
    const Src wk = {work, ww, bpp};
    const long bx0 = it->lru_x * lru_sb_w * 8, by0 = it->lru_y * lru_sb_h * 8;
    const long nbx = lru_sb_w * 8, nby = lru_sb_h * 8, cols8 = aw >> 3, rows8 = ah >> 3;
    const long gbx0 = ax >> 3, gby0 = ay >> 3;

    b200_lrf_unit bst = it->incoming;
    double best_cost = it->incoming_cost;
    { /* the no-filter option, rated with the incoming filter (rdo.rs:2619-2647) */
      const uint64_t e = plane_error(&sr, &in, p, xd, yd, bit_depth, bx0, by0, nbx, nby, cols8, rows8, imp_scales,
                                     w8, gbx0, gby0, dist_scale[p]);
      const uint32_t rate = lrf_rate(it, it->incoming.type, it->incoming.set, it->incoming.xqd);
      const double c = orc_compute_rd_cost(lambda, rate, e);
      if (err) err[k * 17] = e;
      if (cand_cost) cand_cost[k * 17] = c;
      if (best_cost < 0. || c < best_cost) {
        best_cost = c;
        memset(&bst, 0, sizeof(bst));
      }
    }
    setup_integral_image(ii, sq, vis_w, vis_h, vis_w, vis_h, po_x, po_y, &in, &in);
    for (int si = 0; si < (reduced_sets ? 8 : 16); si++) {
      const int set = reduced_sets ? 2 * si + 1 : si; /* get_sgr_sets (lrf.rs:77-93) */
      int8_t q[2];
      sgrproj_solve(set, bit_depth, ii, sq, &sr, &in, vis_w, vis_h, po_x, po_y, q);
      sgrproj_stripe_filter(set, q, bit_depth, ii, sq, vis_w, vis_h, po_x, po_y, &in, &wk);
      const uint64_t e = plane_error(&sr, &wk, p, xd, yd, bit_depth, bx0, by0, nbx, nby, cols8, rows8, imp_scales,
                                     w8, gbx0, gby0, dist_scale[p]);
      const double c = orc_compute_rd_cost(lambda, lrf_rate(it, 2, set, q), e);
      if (xqd) {
        xqd[(k * 16 + set) * 2] = q[0];
        xqd[(k * 16 + set) * 2 + 1] = q[1];
      }
      if (err) err[k * 17 + 1 + set] = e;
      if (cand_cost) cand_cost[k * 17 + 1 + set] = c;
      if (c < best_cost) {
        best_cost = c;
        memset(&bst, 0, sizeof(bst));
        bst.type = 2;
        bst.set = (uint8_t)set;
        bst.xqd[0] = q[0];
        bst.xqd[1] = q[1];
      }
    }
    best[k] = bst;
    cost[k] = best_cost;
    changed[k] = (uint8_t)notequal(&it->incoming, &bst);
    free(work);
  }
  free(ii);
  free(sq);
}
