/*
 * oracle/cdef_rdo.c — the CDEF pass of rdo_loop_decision, area by area, the way rav1e runs it
 * (TEST INFRASTRUCTURE ONLY; see cdef_rdo.h for the contract and what pins it).
 */
#include "cdef_rdo.h"

#include <stdlib.h>
#include <string.h>

#include "oracle.h"

#define HAVE_LEFT 1
#define HAVE_RIGHT 2
#define HAVE_TOP 4
#define HAVE_BOTTOM 8

/* one plane of an area's scratch copy (plane_region.rs:390-401): w x h pixels, no padding */
typedef struct {
  uint8_t *px;
  int w, h, bpp;
} Scratch;

static void *at(const void *base, ptrdiff_t stride, int bpp, int x, int y) {
  return (uint8_t *)base + ((ptrdiff_t)y * stride + x) * bpp;
}

static void copy_rect(void *dst, ptrdiff_t ds, const void *src, ptrdiff_t ss, int bpp, int w, int h) {
  for (int y = 0; y < h; y++) memcpy(at(dst, ds, bpp, 0, y), at(src, ss, bpp, 0, y), (size_t)w * bpp);
}

/* cdef_filter_superblock (cdef.rs:401-570) of superblock (sbx, sby) of the area: input = the rec
 * scratch copy, output = the cdef_ref copy, the tile rect = the whole copy (x = y = 0). */
static void filter_superblock(Scratch *in, Scratch *outp, int planes, int xdec, int ydec, int sbx, int sby,
                              int cols8, int rows8, const uint8_t *skip, const uint8_t *dirs,
                              const int32_t *vars, int y_str, int uv_str, int damping, int bit_depth) {
  const int coeff_shift = bit_depth - 8;
  const int pri_y = y_str / 4, pri_uv = uv_str / 4;
  int sec_y = y_str % 4, sec_uv = uv_str % 4;
  if (sec_y == 3) sec_y += 1;
  if (sec_uv == 3) sec_uv += 1;
  const int input_xavail = in[0].w - 64 * sbx, input_yavail = in[0].h - 64 * sby;
  const int have_top = sby > 0 ? HAVE_TOP : 0, have_left = sbx > 0 ? HAVE_LEFT : 0;
  int edges = have_top | HAVE_BOTTOM;
  static const uint8_t uv_dir_422[8] = {7, 0, 2, 4, 5, 6, 6, 6};
  for (int by = 0; by < 8; by++) {
    if (by + 1 >= (input_yavail >> 3)) edges &= ~HAVE_BOTTOM;
    edges &= ~HAVE_LEFT;
    edges |= have_left;
    edges |= HAVE_RIGHT;
    for (int bx = 0; bx < 8; bx++) {
      if (bx + 1 >= (input_xavail >> 3)) edges &= ~HAVE_RIGHT;
      const int gx = 8 * sbx + bx, gy = 8 * sby + by; /* 8x8 block inside the area */
      if (gx < cols8 && gy < rows8) {
        const int k = gy * cols8 + gx;
        for (int p = 0; p < planes; p++) {
          const int xd = p ? xdec : 0, yd = p ? ydec : 0;
          const int xs = 8 >> xd, ys = 8 >> yd;
          const void *src = at(in[p].px, in[p].w, in[p].bpp, gx * xs, gy * ys);
          void *dst = at(outp[p].px, outp[p].w, outp[p].bpp, gx * xs, gy * ys);
          if (skip[k]) {
            copy_rect(dst, outp[p].w, src, in[p].w, in[p].bpp, xs, ys);
            continue;
          }
          int lpri, lsec, ldir, ldamp = damping + coeff_shift;
          if (p == 0) {
            lpri = orc_cdef_adjust_strength(pri_y << coeff_shift, vars[k]);
            lsec = sec_y << coeff_shift;
            ldir = pri_y ? dirs[k] : 0;
          } else {
            lpri = pri_uv << coeff_shift;
            lsec = sec_uv << coeff_shift;
            ldamp -= 1;
            ldir = pri_uv ? (xdec != ydec ? uv_dir_422[dirs[k]] : dirs[k]) : 0;
          }
          orc_cdef_filter_block_px(dst, outp[p].w, src, in[p].w, in[p].bpp, lpri, lsec, ldir, ldamp, bit_depth,
                                   xd, yd, edges);
        }
      }
      edges |= HAVE_LEFT;
    }
    edges |= HAVE_TOP;
  }
}

void orc_cdef_rdo(const void *const *rec, const ptrdiff_t *rec_stride, const void *const *src,
                  const ptrdiff_t *src_stride, void *const *out, const ptrdiff_t *out_stride, int bpp,
                  int planes, int xdec, int ydec, int width, int height, int bit_depth, int damping,
                  int cdef_bits, const uint8_t *y_strengths, const uint8_t *uv_strengths,
                  const uint8_t *skip8, const uint32_t *imp_scales, const uint32_t *dist_scale,
                  double lambda, const int32_t *areas, size_t n_areas, const uint32_t *rate,
                  uint64_t *err, double *cost, int8_t *best) {
  const int w8 = (width + 7) >> 3;
  for (size_t a = 0; a < n_areas; a++) {
    const int ax = areas[4 * a] * 64, ay = areas[4 * a + 1] * 64;
    const int sb_w = areas[4 * a + 2], sb_h = areas[4 * a + 3];
    /* rdo.rs:2152-2157, 2281-2282 */
    const int crop_w = width - ax, crop_h = height - ay;
    const int pixel_w = crop_w < sb_w * 64 ? crop_w : sb_w * 64, pixel_h = crop_h < sb_h * 64 ? crop_h : sb_h * 64;
    const int aw = (pixel_w + 7) >> 3 << 3, ah = (pixel_h + 7) >> 3 << 3;
    const int cols8 = aw >> 3, rows8 = ah >> 3; /* blocks.cols() / rows() of the area, in 8x8 units */
    Scratch rc[3], cr[3];
    for (int p = 0; p < planes; p++) {
      const int xd = p ? xdec : 0, yd = p ? ydec : 0;
      rc[p].w = cr[p].w = aw >> xd;
      rc[p].h = cr[p].h = ah >> yd;
      rc[p].bpp = cr[p].bpp = bpp;
      rc[p].px = malloc((size_t)rc[p].w * rc[p].h * bpp);
      cr[p].px = malloc((size_t)rc[p].w * rc[p].h * bpp);
      copy_rect(rc[p].px, rc[p].w, at(rec[p], rec_stride[p], bpp, ax >> xd, ay >> yd), rec_stride[p], bpp, rc[p].w,
                rc[p].h);
      memcpy(cr[p].px, rc[p].px, (size_t)rc[p].w * rc[p].h * bpp); /* cdef_work = rec_subset.clone() */
    }
    /* skip per 8x8 block of the area, and cdef_analyze_superblock_range on the copy */
    uint8_t *skip = malloc((size_t)cols8 * rows8), *dirs = calloc((size_t)cols8 * rows8, 1);
    int32_t *vars = calloc((size_t)cols8 * rows8, sizeof(int32_t));
    for (int y = 0; y < rows8; y++)
      for (int x = 0; x < cols8; x++) {
        const int k = y * cols8 + x;
        skip[k] = skip8 ? skip8[(size_t)((ay >> 3) + y) * w8 + (ax >> 3) + x] : 0;
        if (!skip[k]) {
          uint32_t v = 0;
          dirs[k] = (uint8_t)orc_cdef_find_dir(at(rc[0].px, rc[0].w, bpp, 8 * x, 8 * y), rc[0].w, bpp, &v,
                                               bit_depth - 8);
          vars[k] = (int32_t)v;
        }
      }
    for (int sby = 0; sby < sb_h; sby++)
      for (int sbx = 0; sbx < sb_w; sbx++) {
        const size_t slot = a * 16 + (size_t)sby * 4 + sbx;
        int all_skip = 1;
        for (int y = 8 * sby; y < 8 * sby + 8 && y < rows8; y++)
          for (int x = 8 * sbx; x < 8 * sbx + 8 && x < cols8; x++) all_skip &= skip[y * cols8 + x];
        if (all_skip) { /* rdo.rs:2380 */
          best[slot] = -1;
          continue;
        }
        double best_cost = -1.;
        int best_index = -1;
        for (int i = 0; i < (1 << cdef_bits); i++) {
          filter_superblock(rc, cr, planes, xdec, ydec, sbx, sby, cols8, rows8, skip, dirs, vars, y_strengths[i],
                            uv_strengths[i], damping, bit_depth);
          uint64_t e = 0;
          for (int p = 0; p < planes; p++) { /* rdo_loop_plane_error, rdo.rs:2027-2093 */
            const int xd = p ? xdec : 0, yd = p ? ydec : 0;
            uint64_t pe = 0;
            for (int by = 8 * sby; by < 8 * sby + 8 && by < rows8; by++)
              for (int bx = 8 * sbx; bx < 8 * sbx + 8 && bx < cols8; bx++) {
                const size_t gb = (size_t)((ay >> 3) + by) * w8 + (ax >> 3) + bx;
                const uint32_t bias = imp_scales ? imp_scales[gb] : (1u << 14);
                const void *s = at(src[p], src_stride[p], bpp, (ax >> xd) + bx * (8 >> xd), (ay >> yd) + by * (8 >> yd));
                const void *t = at(cr[p].px, cr[p].w, bpp, bx * (8 >> xd), by * (8 >> yd));
                if (p == 0) {
                  const uint32_t d = bpp == 1 ? orc_cdef_dist_kernel_u8(s, src_stride[p], t, cr[p].w, 8, 8, bit_depth, NULL)
                                              : orc_cdef_dist_kernel_u16(s, src_stride[p], t, cr[p].w, 8, 8, bit_depth, NULL);
                  pe += orc_distortion_scale_mul(bias, d);
                } else {
                  const uint32_t scale[4] = {bias, bias, bias, bias}; /* sse_wxh's per-chunk bias buffer */
                  pe += bpp == 1 ? orc_weighted_sse_u8(s, src_stride[p], t, cr[p].w, scale, 2, 8 >> xd, 8 >> yd)
                                 : orc_weighted_sse_u16(s, src_stride[p], t, cr[p].w, scale, 2, 8 >> xd, 8 >> yd);
                }
              }
            e += orc_distortion_scale_mul(dist_scale[p], pe);
          }
          const double c = orc_compute_rd_cost(lambda, rate ? rate[slot] : 0, e);
          err[slot * 8 + i] = e;
          cost[slot * 8 + i] = c;
          if (best_cost < 0. || c < best_cost) {
            best_cost = c;
            best_index = i;
          }
        }
        best[slot] = (int8_t)best_index;
        /* keep the CDEF output up to date with the winner (rdo.rs:2544-2564) */
        filter_superblock(rc, cr, planes, xdec, ydec, sbx, sby, cols8, rows8, skip, dirs, vars,
                          y_strengths[best_index], uv_strengths[best_index], damping, bit_depth);
      }
    for (int p = 0; p < planes; p++) {
      const int xd = p ? xdec : 0, yd = p ? ydec : 0;
      if (out)
        copy_rect(at(out[p], out_stride[p], bpp, ax >> xd, ay >> yd), out_stride[p], cr[p].px, cr[p].w, bpp, cr[p].w,
                  cr[p].h);
      free(rc[p].px);
      free(cr[p].px);
    }
    free(skip);
    free(dirs);
    free(vars);
  }
}
