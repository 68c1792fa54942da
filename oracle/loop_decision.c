/*
 * oracle/loop_decision.c — rdo_loop_decision's pass loop, area by area, the way rav1e runs it
 * (TEST INFRASTRUCTURE ONLY; see loop_decision.h for the contract and what pins it).
 */
#include "loop_decision.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "cdef_rdo.h"
#include "lrf.h"
#include "lrf_search.h"
#include "oracle.h"

/* cdef_rdo.c's superblock filter and lrf_search.c's (and through it lrf.c's) integral image, stripe filter,
 * solve, distortion and rate are file-static: this file compiles them in, as lrf_search.c compiles lrf.c in.
 * Their exported functions come along under other names and hidden, so the library keeps one copy of each. */
#define orc_cdef_rdo orc_cdef_rdo_in_loop_decision_
#pragma GCC visibility push(hidden)
#include "cdef_rdo.c"
#pragma GCC visibility pop
#undef orc_cdef_rdo
#define orc_lrf_search orc_lrf_search_in_loop_decision_
#define orc_lrf_filter_frame_in_lrf_search_ orc_lrf_filter_frame_in_loop_decision_
#pragma GCC visibility push(hidden)
#include "lrf_search.c"
#pragma GCC visibility pop
#undef orc_lrf_search
#undef orc_lrf_filter_frame_in_lrf_search_

/* count_lrf_switchable of a unit's current filter */
static uint32_t unit_rate(const b200_loop_unit *u, const b200_lrf_unit *f) {
  b200_lrf_search_item it;
  memset(&it, 0, sizeof(it));
  it.none_bits = u->none_bits;
  it.sgr_bits = u->sgr_bits;
  it.sgrproj_ref[0] = u->sgrproj_ref[0];
  it.sgrproj_ref[1] = u->sgrproj_ref[1];
  return lrf_rate(&it, f->type, f->set, f->xqd);
}

int orc_loop_decision(const void *const *rec, const ptrdiff_t *rec_stride, const void *const *src,
                      const ptrdiff_t *src_stride, void *const *work, const ptrdiff_t *work_stride, int bpp,
                      int planes, int xdec, int ydec, int width, int height, int bit_depth, int enable_cdef,
                      int damping, int cdef_bits, const uint8_t *y_strengths, const uint8_t *uv_strengths,
                      const uint8_t *skip8, int enable_restoration, const int *unit_size, int reduced_sets,
                      const uint32_t *imp_scales, const uint32_t *dist_scale, double lambda,
                      const b200_cdef_rdo_area *areas, size_t n_areas, const b200_loop_unit *units,
                      size_t n_units, const int32_t *sb_unit, int8_t *best_index, b200_lrf_unit *unit_out,
                      double *unit_cost, uint8_t *written, uint64_t *err, double *cost) {
  const size_t ii_n = (size_t)STRIPE_IMAGE_STRIDE * (SOLVE_MAX + 8);
  uint32_t *ii = calloc(ii_n, sizeof(uint32_t)), *sq = calloc(ii_n, sizeof(uint32_t));
  const long w8 = (width + 7) >> 3;
  int longest = 0, unbounded = 0;
  for (size_t a = 0; a < n_areas; a++) {
    const int ax = areas[a].sbx * 64, ay = areas[a].sby * 64, sb_w = areas[a].sb_w, sb_h = areas[a].sb_h;
    /* rdo.rs:2152-2157, 2281-2282 */
    const int crop_w = width - ax, crop_h = height - ay;
    const int aw = ((crop_w < sb_w * 64 ? crop_w : sb_w * 64) + 7) >> 3 << 3;
    const int ah = ((crop_h < sb_h * 64 ? crop_h : sb_h * 64) + 7) >> 3 << 3;
    const int cols8 = aw >> 3, rows8 = ah >> 3;
    /* cdef_skip / cdef_skip_all (rdo.rs:2189-2205), lru_skip_all (rdo.rs:2212-2264) */
    uint8_t *skip = malloc((size_t)cols8 * rows8);
    int sb_skip[16], cdef_work = 0, lrf_work = 0;
    for (int k = 0; k < cols8 * rows8; k++)
      skip[k] = skip8 ? skip8[(size_t)((ay >> 3) + k / cols8) * w8 + (ax >> 3) + k % cols8] : 0;
    for (int sby = 0; sby < sb_h; sby++)
      for (int sbx = 0; sbx < sb_w; sbx++) {
        int s = 1;
        for (int y = 8 * sby; y < 8 * sby + 8 && y < rows8; y++)
          for (int x = 8 * sbx; x < 8 * sbx + 8 && x < cols8; x++) s &= skip[y * cols8 + x];
        sb_skip[sby * 4 + sbx] = s || !enable_cdef;
        cdef_work |= !sb_skip[sby * 4 + sbx];
      }
    for (size_t u = 0; u < n_units; u++) lrf_work |= enable_restoration && units[u].area == (int)a && units[u].search;
    if (!cdef_work && !lrf_work) { /* rdo.rs:2267 */
      free(skip);
      continue;
    }
    for (int k = 0; k < 16; k++)
      if (k % 4 < sb_w && k / 4 < sb_h) best_index[a * 16 + k] = -1;
    for (size_t u = 0; u < n_units; u++)
      if (units[u].area == (int)a) {
        memset(&unit_out[u], 0, sizeof(unit_out[u]));
        unit_cost[u] = -1.;
        written[u] = 0;
      }
    /* rec_subset, cdef_work and lrf_work (rdo.rs:2277-2344) */
    Scratch rc[3], cr[3];
    uint8_t *lw[3];
    for (int p = 0; p < planes; p++) {
      const int xd = p ? xdec : 0, yd = p ? ydec : 0;
      rc[p].w = cr[p].w = aw >> xd;
      rc[p].h = cr[p].h = ah >> yd;
      rc[p].bpp = cr[p].bpp = bpp;
      rc[p].px = malloc((size_t)rc[p].w * rc[p].h * bpp);
      cr[p].px = malloc((size_t)rc[p].w * rc[p].h * bpp);
      copy_rect(rc[p].px, rc[p].w, at(rec[p], rec_stride[p], bpp, ax >> xd, ay >> yd), rec_stride[p], bpp, rc[p].w,
                rc[p].h);
      memcpy(cr[p].px, rc[p].px, (size_t)rc[p].w * rc[p].h * bpp);
      lw[p] = malloc((size_t)rc[p].w * rc[p].h * bpp);
      for (long i = 0; i < (long)rc[p].w * rc[p].h; i++) {
        if (bpp == 1) lw[p][i] = B200_LRF_WORK_FILL;
        else ((uint16_t *)lw[p])[i] = B200_LRF_WORK_FILL;
      }
    }
    /* cdef_analyze_superblock_range */
    uint8_t *dirs = calloc((size_t)cols8 * rows8, 1);
    int32_t *vars = calloc((size_t)cols8 * rows8, sizeof(int32_t));
    for (int k = 0; k < cols8 * rows8 && cdef_work; k++)
      if (!skip[k]) {
        uint32_t v = 0;
        dirs[k] = (uint8_t)orc_cdef_find_dir(at(rc[0].px, rc[0].w, bpp, 8 * (k % cols8), 8 * (k / cols8)), rc[0].w,
                                             bpp, &v, bit_depth - 8);
        vars[k] = (int32_t)v;
      }
    /* the restoration input: the CDEF output, or the deblocked copy without CDEF (rdo.rs:2577-2584) */
    Scratch *lin = cdef_work ? cr : rc;

    int stage = 0;
    for (;;) {
      if (stage == B200_LOOP_MAX_STAGES) {
        unbounded = 1;
        break;
      }
      int changed = 0;
      if (!(stage & 1)) { /* ---- C (rdo.rs:2373-2567) */
        changed = stage == 0;
        for (int sby = 0; sby < sb_h && cdef_work; sby++)
          for (int sbx = 0; sbx < sb_w; sbx++) {
            if (sb_skip[sby * 4 + sbx]) continue;
            const size_t slot = a * 16 + (size_t)sby * 4 + sbx;
            double best_cost = -1.;
            int best = -1;
            for (int i = 0; i < (1 << cdef_bits); i++) {
              filter_superblock(rc, cr, planes, xdec, ydec, sbx, sby, cols8, rows8, skip, dirs, vars, y_strengths[i],
                                uv_strengths[i], damping, bit_depth);
              uint64_t e = 0;
              uint32_t rate = 0;
              for (int p = 0; p < planes; p++) {
                const int xd = p ? xdec : 0, yd = p ? ydec : 0;
                const Src sr = {(const uint8_t *)src[p] + ((ptrdiff_t)(ay >> yd) * src_stride[p] + (ax >> xd)) * bpp,
                                src_stride[p], bpp};
                const Src cw = {cr[p].px, cr[p].w, bpp};
                const Src *test = &cw;
                const Src lwk = {lw[p], cr[p].w, bpp};
                const int32_t u = sb_unit[slot * 3 + p];
                if (u >= 0 && lrf_work) { /* rdo.rs:2424-2507 */
                  const b200_lrf_unit *f = &unit_out[u];
                  rate += unit_rate(&units[u], f);
                  if (f->type == 2) {
                    const long po_x = (sbx * 64L) >> xd, po_y = (sby * 64L) >> yd;
                    const long vis_w = minl(64 >> xd, (crop_w >> xd) - po_x), vis_h = minl(64 >> yd, (crop_h >> yd) - po_y);
                    setup_integral_image(ii, sq, vis_w, vis_h, vis_w, vis_h, po_x, po_y, &cw, &cw);
                    sgrproj_stripe_filter(f->set, f->xqd, bit_depth, ii, sq, vis_w, vis_h, po_x, po_y, &cw, &lwk);
                    test = &lwk;
                  }
                }
                e += plane_error(&sr, test, p, xd, yd, bit_depth, 8 * sbx, 8 * sby, 8, 8, cols8, rows8, imp_scales, w8,
                                 ax >> 3, ay >> 3, dist_scale[p]);
              }
              const double c = orc_compute_rd_cost(lambda, rate, e);
              if (err) err[slot * 8 + i] = e;
              if (cost) cost[slot * 8 + i] = c;
              if (best_cost < 0. || c < best_cost) {
                best_cost = c;
                best = i;
              }
            }
            if (best != best_index[slot]) {
              changed = 1;
              best_index[slot] = (int8_t)best;
            }
            filter_superblock(rc, cr, planes, xdec, ydec, sbx, sby, cols8, rows8, skip, dirs, vars,
                              y_strengths[best], uv_strengths[best], damping, bit_depth);
          }
      } else if (lrf_work) { /* ---- L (rdo.rs:2575-2745) */
        for (size_t u = 0; u < n_units; u++) {
          const b200_loop_unit *un = &units[u];
          if (un->area != (int)a || !un->search) continue;
          const int p = un->plane, xd = p ? xdec : 0, yd = p ? ydec : 0;
          const long us = unit_size[p], lsw = (us << xd) / 64, lsh = (us << yd) / 64;
          const long po_x = un->lru_x * lsw * 64 >> xd, po_y = un->lru_y * lsh * 64 >> yd;
          const long vis_w = minl(us, (crop_w >> xd) - po_x), vis_h = minl(us, (crop_h >> yd) - po_y);
          const Src in = {lin[p].px, lin[p].w, bpp}, wk = {lw[p], lin[p].w, bpp};
          const Src sr = {(const uint8_t *)src[p] + ((ptrdiff_t)(ay >> yd) * src_stride[p] + (ax >> xd)) * bpp,
                          src_stride[p], bpp};
          const long bx0 = un->lru_x * lsw * 8, by0 = un->lru_y * lsh * 8;
          b200_lrf_search_item it;
          memset(&it, 0, sizeof(it));
          it.none_bits = un->none_bits;
          it.sgr_bits = un->sgr_bits;
          it.sgrproj_ref[0] = un->sgrproj_ref[0];
          it.sgrproj_ref[1] = un->sgrproj_ref[1];
          b200_lrf_unit bst = unit_out[u];
          double best_cost = unit_cost[u];
          { /* the no-filter option, rated with the incumbent (rdo.rs:2619-2647) */
            const uint64_t e = plane_error(&sr, &in, p, xd, yd, bit_depth, bx0, by0, lsw * 8, lsh * 8, cols8, rows8,
                                           imp_scales, w8, ax >> 3, ay >> 3, dist_scale[p]);
            const double c = orc_compute_rd_cost(lambda, lrf_rate(&it, bst.type, bst.set, bst.xqd), e);
            if (best_cost < 0. || c < best_cost) {
              best_cost = c;
              memset(&bst, 0, sizeof(bst));
            }
          }
          setup_integral_image(ii, sq, vis_w, vis_h, vis_w, vis_h, po_x, po_y, &in, &in);
          for (int si = 0; si < (reduced_sets ? 8 : 16); si++) {
            const int set = reduced_sets ? 2 * si + 1 : si;
            int8_t q[2];
            sgrproj_solve(set, bit_depth, ii, sq, &sr, &in, vis_w, vis_h, po_x, po_y, q);
            sgrproj_stripe_filter(set, q, bit_depth, ii, sq, vis_w, vis_h, po_x, po_y, &in, &wk);
            const uint64_t e = plane_error(&sr, &wk, p, xd, yd, bit_depth, bx0, by0, lsw * 8, lsh * 8, cols8, rows8,
                                           imp_scales, w8, ax >> 3, ay >> 3, dist_scale[p]);
            const double c = orc_compute_rd_cost(lambda, lrf_rate(&it, 2, set, q), e);
            if (c < best_cost) {
              best_cost = c;
              memset(&bst, 0, sizeof(bst));
              bst.type = 2;
              bst.set = (uint8_t)set;
              bst.xqd[0] = q[0];
              bst.xqd[1] = q[1];
            }
          }
          unit_cost[u] = best_cost;
          if (notequal(&unit_out[u], &bst)) { /* rdo.rs:2730-2741 */
            unit_out[u] = bst;
            written[u] = 1;
            changed = 1;
          }
        }
      }
      stage++;
      if (!changed) break;
    }
    if (stage > longest) longest = stage;
    for (int p = 0; p < planes; p++) {
      const int xd = p ? xdec : 0, yd = p ? ydec : 0;
      copy_rect(at(work[p], work_stride[p], bpp, ax >> xd, ay >> yd), work_stride[p], lin[p].px, lin[p].w, bpp,
                lin[p].w, lin[p].h);
      free(rc[p].px);
      free(cr[p].px);
      free(lw[p]);
    }
    free(skip);
    free(dirs);
    free(vars);
  }
  free(ii);
  free(sq);
  return unbounded ? -1 : longest;
}
