/*
 * oracle/lookahead_me.c — the lookahead's motion vectors, serially: estimate_tile_motion (me.rs:153-218)
 * with estimate_sb_motion (:220-282), refine_subsampled_sb_motion (:284-322), save_me_stats (:324-337),
 * get_subset_predictors (:386-534), estimate_motion without a pmv (:536-631),
 * refine_subsampled_motion_estimate (:633-690) and full_pixel_me (:692-856), in the reference's loop
 * order.  TEST INFRASTRUCTURE ONLY (see oracle.h); declared in lookahead_me.h.
 *
 * The search stages below restate full_pixel_me's (get_best_predictor, fullpel_diamond_search,
 * hexagon_search, uneven_multi_hex_search) as me.c does for orc_full_pixel_me_blocks.  They are
 * restated here rather than reused because me.c's take the mv range of a full-resolution block, while
 * the subsampled levels search within get_mv_range(full-size block) >> ssdec.  Distortion, rate,
 * range and the exhaustive grid are me.c's exported orc_get_sad_*, orc_mv_cost, orc_get_mv_range
 * and orc_full_search.
 */
#include "lookahead_me.h"

#define MI_SIZE 4 /* context/superblock_unit.rs:12 */

static inline const void *px_at(const void *p0, ptrdiff_t stride, int bpp, int x, int y) {
  return (const uint8_t *)p0 + ((ptrdiff_t)y * stride + x) * bpp;
}

static inline uint32_t sad_any(const void *org, ptrdiff_t os, const void *ref, ptrdiff_t rs, int bpp, int w,
                               int h) {
  return bpp == 1 ? orc_get_sad_u8((const uint8_t *)org, os, (const uint8_t *)ref, rs, w, h)
                  : orc_get_sad_u16((const uint16_t *)org, os, (const uint16_t *)ref, rs, w, h);
}

/* ------------------------------------------------------------------------------------------
 * Search stages: full_pixel_me's, me.rs:884-1303.  MotionVector arithmetic is i16 (release builds
 * wrap); every "if rd.cost < best.cost" keeps the first minimum.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const void *org; /* block pixel (0,0) in cur */
  ptrdiff_t org_stride;
  const void *ref0;
  ptrdiff_t ref_stride;
  int bpp, w, h, po_x, po_y;
  int mvx_min, mvx_max, mvy_min, mvy_max;
  uint32_t lambda;
  orc_mv pmv0, pmv1;
  int allow_hp;
} srch;

static inline orc_mv mv_add(orc_mv a, orc_mv b) {
  orc_mv r = {(int16_t)(a.row + b.row), (int16_t)(a.col + b.col)};
  return r;
}
static inline orc_mv mv_mul(orc_mv a, int16_t k) {
  orc_mv r = {(int16_t)(a.row * k), (int16_t)(a.col * k)};
  return r;
}
static inline orc_mv mv_shl(orc_mv a, int s) {
  orc_mv r = {(int16_t)((int)a.row * (1 << s)), (int16_t)((int)a.col * (1 << s))};
  return r;
}
static inline orc_me_result res_empty(void) { /* MotionSearchResult::empty(), me.rs:111-116 */
  orc_me_result r;
  r.cost = UINT64_MAX;
  r.sad = UINT32_MAX;
  r.mv.row = 0;
  r.mv.col = 0;
  return r;
}

/* get_fullpel_mv_rd, me.rs:1386-1409 (use_satd = false in every full-pel stage) */
static orc_me_result fullpel_rd(const srch *s, orc_mv mv) {
  orc_me_result r = res_empty();
  r.mv = mv;
  if (mv.col < s->mvx_min || mv.col > s->mvx_max || mv.row < s->mvy_min || mv.row > s->mvy_max)
    return r;
  r.sad = sad_any(s->org, s->org_stride,
                  px_at(s->ref0, s->ref_stride, s->bpp, s->po_x + mv.col / 8, s->po_y + mv.row / 8), s->ref_stride,
                  s->bpp, s->w, s->h);
  r.cost = orc_mv_cost(r.sad, mv, s->pmv0, s->pmv1, s->lambda, s->allow_hp);
  return r;
}

/* me.rs:884-909 */
static orc_me_result best_predictor(const srch *s, const orc_cand *preds, size_t n) {
  orc_me_result best = res_empty();
  for (size_t i = 0; i < n; i++) {
    orc_mv mv = {preds[i].mv_row, preds[i].mv_col};
    orc_me_result rd = fullpel_rd(s, mv);
    if (rd.cost < best.cost) best = rd;
  }
  return best;
}

#define FP(c, r) {(int16_t)((r) * 8), (int16_t)((c) * 8)} /* search_pattern!: {row, col} << 3 */
static const orc_mv DIAMOND_R1[4] = {FP(0, 1), FP(1, 0), FP(0, -1), FP(-1, 0)}; /* me.rs:944-947 */
static const orc_mv HEXAGON[6] = {FP(0, -2), FP(2, -1), FP(2, 1), FP(0, 2), FP(-2, 1), FP(-2, -1)}; /* :1022-1025 */
static const orc_mv SQUARE_REFINE[8] = {FP(-1, 1), FP(0, 1),  FP(1, 1),  FP(-1, 0),
                                        FP(1, 0),  FP(-1, -1), FP(0, -1), FP(1, -1)}; /* :1035-1038 */
static const orc_mv UMH[16] = {FP(-2, 4), FP(-1, 4), FP(0, 4),  FP(1, 4),  FP(2, 4),  FP(3, 2),
                               FP(4, 0),  FP(3, -2), FP(2, -4), FP(1, -4), FP(0, -4), FP(-1, -4),
                               FP(-2, -4), FP(3, -2), FP(-4, 0), FP(-3, 2)}; /* :1153-1156 */

/* me.rs:955-998 */
static void fullpel_diamond(const srch *s, orc_me_result *current) {
  int radius_log2 = 1;
  const int end_log2 = 0;
  for (;;) {
    orc_me_result best_cand = res_empty();
    for (int k = 0; k < 4; k++) {
      orc_me_result rd = fullpel_rd(s, mv_add(current->mv, mv_shl(DIAMOND_R1[k], radius_log2)));
      if (rd.cost < best_cand.cost) best_cand = rd;
    }
    if (current->cost <= best_cand.cost) {
      if (radius_log2 == end_log2) break;
      radius_log2--;
    } else {
      *current = best_cand;
    }
  }
}

/* me.rs:1055-1135 */
static void hexagon(const srch *s, orc_me_result *current) {
  int best_idx = 0;
  orc_me_result best_cand = res_empty();
  for (int i = 0; i < 6; i++) {
    orc_me_result rd = fullpel_rd(s, mv_add(current->mv, HEXAGON[i]));
    if (rd.cost < best_cand.cost) {
      best_idx = i;
      best_cand = rd;
    }
  }
  while (best_cand.cost < current->cost) {
    *current = best_cand;
    best_cand = res_empty();
    const int center_idx = best_idx;
    for (int off = 5; off <= 7; off++) {
      const int i = (center_idx + off) % 6;
      orc_me_result rd = fullpel_rd(s, mv_add(current->mv, HEXAGON[i]));
      if (rd.cost < best_cand.cost) {
        best_idx = i;
        best_cand = rd;
      }
    }
  }
  best_cand = res_empty();
  for (int k = 0; k < 8; k++) {
    orc_me_result rd = fullpel_rd(s, mv_add(current->mv, SQUARE_REFINE[k]));
    if (rd.cost < best_cand.cost) best_cand = rd;
  }
  if (best_cand.cost < current->cost) *current = best_cand;
}

/* me.rs:1170-1303.  Quirks kept as they are: the "horizontal" line steps the ROW component
 * (:1195-1198), and the 5x5 stage adds raw {row, col} in 1/8 pel, not full pixels (:1240-1246). */
static void umh(const srch *s, orc_me_result *current, int me_range) {
  orc_mv center = current->mv;
  for (int i = 1; i <= me_range; i += 2) {
    static const orc_mv line[2] = {FP(0, -1), FP(0, 1)};
    for (int k = 0; k < 2; k++) {
      orc_me_result rd = fullpel_rd(s, mv_add(center, mv_mul(line[k], (int16_t)i)));
      if (rd.cost < current->cost) *current = rd;
    }
  }
  for (int i = 1; i <= (me_range >> 1); i += 2) {
    static const orc_mv line[2] = {FP(-1, 0), FP(1, 0)};
    for (int k = 0; k < 2; k++) {
      orc_me_result rd = fullpel_rd(s, mv_add(center, mv_mul(line[k], (int16_t)i)));
      if (rd.cost < current->cost) *current = rd;
    }
  }
  center = current->mv;
  for (int row = -2; row <= 2; row++)
    for (int col = -2; col <= 2; col++) {
      if (row == 0 && col == 0) continue;
      orc_mv off = {(int16_t)row, (int16_t)col};
      orc_me_result rd = fullpel_rd(s, mv_add(center, off));
      if (rd.cost < current->cost) *current = rd;
    }
  center = current->mv;
  const int iterations = me_range >> 2;
  for (int i = 1; i <= iterations; i++)
    for (int k = 0; k < 16; k++) {
      orc_me_result rd = fullpel_rd(s, mv_add(center, mv_mul(UMH[k], (int16_t)i)));
      if (rd.cost < current->cost) *current = rd;
    }
  hexagon(s, current);
}

/* ------------------------------------------------------------------------------------------
 * The driver.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  const void *const *cur;
  const ptrdiff_t *cur_stride;
  const void *const *ref;
  const ptrdiff_t *ref_stride;
  int bpp, bit_depth, allow_hp, full_search, range_scale;
  int w_in_b, h_in_b;
  int tx0, ty0, mi_w, mi_h, tile_w, tile_h; /* tile origin (4x4 units), size (4x4 units, px) */
  const orc_me_stats *prev;
  orc_me_stats *out;
} la_ctx;

uint32_t orc_lookahead_me_thresh(uint32_t min_sad, int w, int h, int bit_depth) {
  const float t = (float)min_sad * 1.2f; /* `min_sad as f32 * 1.2`, then a saturating `as u32` */
  const uint32_t f = t >= 4294967296.0f ? UINT32_MAX : (uint32_t)t;
  return f + ((uint32_t)(w * h) << (bit_depth - 8));
}

static inline orc_me_stats *la_tile(const la_ctx *c, int bx, int by) { /* TileMEStats[by][bx] */
  return &c->out[(size_t)(c->ty0 + by) * c->w_in_b + c->tx0 + bx];
}

static inline int16_t shr16(int16_t v, int s) { return (int16_t)(v >> s); }

static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

/* block geometry shared by the search and the refinement: range (>> ssdec), po, org */
static void la_srch(const la_ctx *c, srch *s, int bx, int by, int w, int h, int ssdec, uint32_t lambda) {
  const int fx = c->tx0 + bx, fy = c->ty0 + by;
  orc_get_mv_range(c->w_in_b, c->h_in_b, fx, fy, w << ssdec, h << ssdec, &s->mvx_min, &s->mvx_max, &s->mvy_min,
                   &s->mvy_max);
  s->mvx_min >>= ssdec, s->mvx_max >>= ssdec, s->mvy_min >>= ssdec, s->mvy_max >>= ssdec;
  s->po_x = (fx * MI_SIZE) >> ssdec;
  s->po_y = (fy * MI_SIZE) >> ssdec;
  s->bpp = c->bpp;
  s->org = px_at(c->cur[ssdec], c->cur_stride[ssdec], c->bpp, s->po_x, s->po_y);
  s->org_stride = c->cur_stride[ssdec];
  s->ref0 = c->ref[ssdec];
  s->ref_stride = c->ref_stride[ssdec];
  s->w = w;
  s->h = h;
  s->lambda = lambda;
  s->pmv0.row = s->pmv0.col = s->pmv1.row = s->pmv1.col = 0;
  s->allow_hp = c->allow_hp;
}

static void la_save(const la_ctx *c, int log2, int bx, int by, orc_me_result r, int w, int h, int ssdec) {
  orc_me_stats st;
  st.mv_row = (int16_t)(r.mv.row * (1 << ssdec)); /* `best.mv << ssdec` on i16 */
  st.mv_col = (int16_t)(r.mv.col * (1 << ssdec));
  st.normalized_sad = (uint32_t)(((uint64_t)r.sad << 14) / (uint64_t)(w * h));
  const int xe = bx + (1 << log2) < c->mi_w ? bx + (1 << log2) : c->mi_w;
  const int ye = by + (1 << log2) < c->mi_h ? by + (1 << log2) : c->mi_h;
  for (int y = by; y < ye; y++)
    for (int x = bx; x < xe; x++) *la_tile(c, x, y) = st;
}

typedef struct {
  uint32_t min_sad;
  int has_median;
  orc_mv median;
  orc_mv b[5], cc[5];
  int nb, nc;
} la_subsets;

static orc_mv la_proc(const srch *s, uint32_t *min_sad, orc_me_stats st) {
  if (st.normalized_sad < *min_sad) *min_sad = st.normalized_sad;
  orc_mv mv;
  mv.col = (int16_t)clampi((st.mv_col / 8) * 8, s->mvx_min, s->mvx_max);
  mv.row = (int16_t)clampi((st.mv_row / 8) * 8, s->mvy_min, s->mvy_max);
  return mv;
}

/* me.rs:386-534; corner: -1 = INIT, else bit 0 right, bit 1 bottom */
static la_subsets la_predictors(const la_ctx *c, const srch *s, int bx, int by, int corner, int ssdec) {
  la_subsets r;
  r.min_sad = UINT32_MAX;
  r.nb = r.nc = 0;
  r.has_median = 0;
  const int w = ((s->w << ssdec) + MI_SIZE - 1) >> 2, h = ((s->h << ssdec) + MI_SIZE - 1) >> 2;
  const int chw = (w >> 1) < c->mi_w - 1 - bx ? (w >> 1) : c->mi_w - 1 - bx;
  const int chh = (h >> 1) < c->mi_h - 1 - by ? (h >> 1) : c->mi_h - 1 - by;
  if (bx > 0) r.b[r.nb++] = la_proc(s, &r.min_sad, *la_tile(c, bx - 1, by + chh));
  if (by > 0) r.b[r.nb++] = la_proc(s, &r.min_sad, *la_tile(c, bx + chw, by - 1));
  if (corner >= 0 && (corner & 1) && bx + w < c->mi_w) r.b[r.nb++] = la_proc(s, &r.min_sad, *la_tile(c, bx + w, by + chh));
  if (corner >= 0 && (corner & 2) && by + h < c->mi_h) r.b[r.nb++] = la_proc(s, &r.min_sad, *la_tile(c, bx + chw, by + h));
  if (corner >= 0) {
    r.has_median = 1;
    r.median = la_proc(s, &r.min_sad, *la_tile(c, bx + chw, by + chh));
  } else if (r.nb == 3) {
    int16_t rows[3] = {r.b[0].row, r.b[1].row, r.b[2].row}, cols[3] = {r.b[0].col, r.b[1].col, r.b[2].col};
    for (int i = 0; i < 3; i++)
      for (int j = i + 1; j < 3; j++) {
        if (rows[j] < rows[i]) { int16_t t = rows[i]; rows[i] = rows[j]; rows[j] = t; }
        if (cols[j] < cols[i]) { int16_t t = cols[i]; cols[i] = cols[j]; cols[j] = t; }
      }
    r.has_median = 1;
    r.median.row = rows[1];
    r.median.col = cols[1];
  }
  r.b[r.nb].row = r.b[r.nb].col = 0;
  r.nb++;
  if (c->prev) {
    const int fx = c->tx0 + bx, fy = c->ty0 + by, W = c->w_in_b, H = c->h_in_b;
    const orc_me_stats *P = c->prev;
    const int hw = (w >> 1) < W - 1 - fx ? (w >> 1) : W - 1 - fx;
    const int hh = (h >> 1) < H - 1 - fy ? (h >> 1) : H - 1 - fy;
    if (fx > 0) r.cc[r.nc++] = la_proc(s, &r.min_sad, P[(size_t)(fy + hh) * W + fx - 1]);
    if (fy > 0) r.cc[r.nc++] = la_proc(s, &r.min_sad, P[(size_t)(fy - 1) * W + fx + hw]);
    if (fx + w < W) r.cc[r.nc++] = la_proc(s, &r.min_sad, P[(size_t)(fy + hh) * W + fx + w]);
    if (fy + h < H) r.cc[r.nc++] = la_proc(s, &r.min_sad, P[(size_t)(fy + h) * W + fx + hw]);
    r.cc[r.nc++] = la_proc(s, &r.min_sad, P[(size_t)(fy + hh) * W + fx + hw]);
  }
  r.min_sad = (uint32_t)(((uint64_t)r.min_sad * (uint64_t)(s->w * s->h)) >> 14);
  r.median.row = shr16(r.median.row, ssdec), r.median.col = shr16(r.median.col, ssdec);
  for (int i = 0; i < r.nb; i++) r.b[i].row = shr16(r.b[i].row, ssdec), r.b[i].col = shr16(r.b[i].col, ssdec);
  for (int i = 0; i < r.nc; i++) r.cc[i].row = shr16(r.cc[i].row, ssdec), r.cc[i].col = shr16(r.cc[i].col, ssdec);
  return r;
}

static orc_me_result la_try(const srch *s, const orc_mv *preds, int n, orc_me_result best) {
  orc_cand cands[11];
  for (int i = 0; i < n; i++) cands[i].mv_row = preds[i].row, cands[i].mv_col = preds[i].col;
  orc_me_result r = best_predictor(s, cands, (size_t)n);
  fullpel_diamond(s, &r);
  return r.cost < best.cost ? r : best;
}

/* full_pixel_me, me.rs:692-856 */
static orc_me_result la_full_pixel_me(const la_ctx *c, const srch *s, int bx, int by, int corner, int extensive,
                                      int ssdec) {
  const la_subsets ss = la_predictors(c, s, bx, by, corner, ssdec);
  orc_me_result best = res_empty();
  if (!extensive) { /* all_mvs */
    orc_mv all[11];
    int n = 0;
    if (ss.has_median) all[n++] = ss.median;
    for (int i = 0; i < ss.nb; i++) all[n++] = ss.b[i];
    for (int i = 0; i < ss.nc; i++) all[n++] = ss.cc[i];
    return la_try(s, all, n, best);
  }
  const uint32_t thresh = orc_lookahead_me_thresh(ss.min_sad, s->w, s->h, c->bit_depth);
  if (ss.has_median) {
    best = la_try(s, &ss.median, 1, best);
    if (best.sad < thresh) return best;
  }
  best = la_try(s, ss.b, ss.nb, best);
  if (best.sad < thresh) return best;
  best = la_try(s, ss.cc, ss.nc, best);
  if (best.sad < thresh) return best;
  umh(s, &best, 24);
  if (!c->full_search || best.sad < thresh) return best;
  const int range_x = (192 * c->range_scale) >> ssdec, range_y = (64 * c->range_scale) >> ssdec;
  const int x_lo = s->po_x + (-range_x > s->mvx_min / 8 ? -range_x : s->mvx_min / 8);
  const int x_hi = s->po_x + (range_x < s->mvx_max / 8 ? range_x : s->mvx_max / 8);
  const int y_lo = s->po_y + (-range_y > s->mvy_min / 8 ? -range_y : s->mvy_min / 8);
  const int y_hi = s->po_y + (range_y < s->mvy_max / 8 ? range_y : s->mvy_max / 8);
  const orc_mv z = {0, 0};
  orc_me_result r = orc_full_search(s->org, s->org_stride, s->ref0, s->ref_stride, s->bpp, x_lo, x_hi, y_lo, y_hi,
                                    s->w, s->h, s->po_x, s->po_y, 4 >> ssdec, s->lambda, z, z, s->allow_hp);
  return r.cost < best.cost ? r : best;
}

static void la_sb(const la_ctx *c, int sbx, int sby, int log2, int ssdec, uint32_t lambda, int refine) {
  const int px = sbx * 64, py = sby * 64;
  const int sb_w = c->tile_w - px < 64 ? c->tile_w - px : 64;
  const int sb_h = c->tile_h - py < 64 ? c->tile_h - py : 64;
  const int mv_size = MI_SIZE << log2;
  for (int y = 0; y < sb_h; y += mv_size)
    for (int x = 0; x < sb_w; x += mv_size) {
      const int bx = (px + x) >> 2, by = (py + y) >> 2;
      const int w = (mv_size < sb_w - x + (1 << ssdec) - 1 ? mv_size : sb_w - x + (1 << ssdec) - 1) >> ssdec;
      const int h = (mv_size < sb_h - y + (1 << ssdec) - 1 ? mv_size : sb_h - y + (1 << ssdec) - 1) >> ssdec;
      srch s;
      la_srch(c, &s, bx, by, w, h, ssdec, lambda);
      orc_me_result r;
      if (refine) { /* refine_subsampled_motion_estimate: 4x4 full search around the stored mv */
        const orc_me_stats st = *la_tile(c, bx, by);
        const int mc = shr16(st.mv_col, ssdec) / 8, mr = shr16(st.mv_row, ssdec) / 8;
        const int x_lo = s.po_x + (mc - 1 > s.mvx_min / 8 ? mc - 1 : s.mvx_min / 8);
        const int x_hi = s.po_x + (mc + 2 < s.mvx_max / 8 ? mc + 2 : s.mvx_max / 8);
        const int y_lo = s.po_y + (mr - 1 > s.mvy_min / 8 ? mr - 1 : s.mvy_min / 8);
        const int y_hi = s.po_y + (mr + 2 < s.mvy_max / 8 ? mr + 2 : s.mvy_max / 8);
        const orc_mv z = {0, 0};
        r = orc_full_search(s.org, s.org_stride, s.ref0, s.ref_stride, s.bpp, x_lo, x_hi, y_lo, y_hi, w, h, s.po_x,
                            s.po_y, 1, lambda, z, z, c->allow_hp);
      } else {
        const int corner = log2 == 4 ? -1 : ((x & mv_size) ? 1 : 0) | ((y & mv_size) ? 2 : 0);
        r = la_full_pixel_me(c, &s, bx, by, corner, log2 == 4, ssdec);
      }
      la_save(c, log2, bx, by, r, w, h, ssdec);
    }
}

void orc_lookahead_motion(const void *const cur[3], const ptrdiff_t cur_stride[3], const void *const ref[3],
                          const ptrdiff_t ref_stride[3], int bpp, int width, int height, int bit_depth,
                          int allow_hp, double me_lambda, int me_allow_full_search, int me_range_scale,
                          int tile_w_sb, int tile_h_sb, const orc_me_stats *prev, orc_me_stats *out) {
  la_ctx c;
  c.cur = cur, c.cur_stride = cur_stride, c.ref = ref, c.ref_stride = ref_stride;
  c.bpp = bpp, c.bit_depth = bit_depth, c.allow_hp = allow_hp;
  c.full_search = me_allow_full_search, c.range_scale = me_range_scale;
  const int W8 = (width + 7) & ~7, H8 = (height + 7) & ~7;
  c.w_in_b = W8 >> 2, c.h_in_b = H8 >> 2;
  c.prev = prev, c.out = out;
  const int tw = tile_w_sb * 64, th = tile_h_sb * 64;
  for (int ty = 0; ty < H8; ty += th)
    for (int tx = 0; tx < W8; tx += tw) { /* tiles are independent */
      c.tx0 = tx >> 2, c.ty0 = ty >> 2;
      c.tile_w = W8 - tx < tw ? W8 - tx : tw;
      c.tile_h = H8 - ty < th ? H8 - ty : th;
      c.mi_w = c.tile_w >> 2, c.mi_h = c.tile_h >> 2;
      const int sbw = (c.tile_w + 63) >> 6, sbh = (c.tile_h + 63) >> 6;
      for (int log2 = 4; log2 >= 2; log2--) {
        const int ssdec = log2 - 2; /* 64 px on the quarter, 32 on the half, 16 on the full plane */
        const double l = me_lambda * 256.0 / (double)(1 << (2 * ssdec)) * (ssdec == 0 ? 0.5 : 0.125);
        const uint32_t lambda = !(l > 0.0) ? 0u : l >= 4294967295.0 ? UINT32_MAX : (uint32_t)l; /* `as u32` */
        for (int sby = 0; sby < sbh; sby++)
          for (int sbx = 0; sbx < sbw; sbx++) {
            if (log2 < 4) la_sb(&c, sbx, sby, log2 + 1, ssdec, lambda, 1);
            la_sb(&c, sbx, sby, log2, ssdec, lambda, 0);
          }
      }
    }
}
