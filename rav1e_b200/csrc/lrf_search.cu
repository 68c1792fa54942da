// lrf_search.cu — the restoration search of one rdo_loop_decision pass (rav1e src/rdo.rs:2575-2740) for many
// (area, plane, unit) items in one call: the None candidate, then per self-guided set sgrproj_solve
// (lrf.rs:846-1096), sgrproj_stripe_filter over the unit's visible rect, rdo_loop_plane_error
// (rdo.rs:2027-2093), count_lrf_switchable (context/frame_header.rs:14-45) and compute_rd_cost.
//
// Four launches, whatever the item count:
//  1. lrf_search_tiles<T, false>, per (item, 32x32 tile of the unit): the tile plus a 3-pixel halo is staged
//     once through setup_integral_image's clip rule (lrf.rs:529-627), the radius-1 and radius-2 box sums
//     are formed once, and for every set the a / b values, the two filter outputs f1 / f2 and the five
//     solve sums are formed; the sums go to per-(item, set) i64 accumulators.
//  2. lrf_search_solve, per (item, set): the 2x2 solve in f64, operation for operation as the reference.
//  3. lrf_search_tiles<T, true>, per (item, tile): the same staging, then the None candidate's and every
//     set's filtered tile are measured block by block; the per-block scaled distortions go to per-(item,
//     candidate) u64 accumulators.
//  4. lrf_search_decide, per item: dist_scale, the rates, compute_rd_cost and the winner.
// Integer sums are exact in any order, so atomics keep the results bit exact.
#include <algorithm>
#include <vector>

#include "host_stage.cuh"
#include "lrf_search_dev.cuh"

namespace {

bool is_unit_size(int s) { return s >= 32 && s <= 256 && (s & (s - 1)) == 0; }

}  // namespace

extern "C" int b200_lrf_search_dev(b200_ctx *ctx, const b200_plane *lrf_in, const b200_plane *src, int planes,
                                   int xdec, int ydec, int frame_width, int frame_height, int bit_depth,
                                   const int unit_size[3], int reduced_sets, const uint32_t *d_imp_scales,
                                   const uint32_t dist_scale[3], double lambda, const b200_cdef_rdo_area *areas,
                                   size_t n_areas, const b200_lrf_search_item *items, size_t n_items,
                                   b200_lrf_unit *d_best, double *d_cost, uint8_t *d_changed, int8_t *d_xqd,
                                   uint64_t *d_err, double *d_cand_cost) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, lrf_in && src && unit_size && dist_scale && d_best && d_cost && d_changed,
               "NULL lrf_in / src / unit_size / dist_scale / outputs");
  B200_REQUIRE(ctx, planes == 1 || planes == 3, "planes must be 1 or 3, got %d", planes);
  B200_REQUIRE(ctx, (xdec == 1 && ydec == 1) || (xdec == 1 && ydec == 0) || (xdec == 0 && ydec == 0),
               "chroma layout (xdec %d, ydec %d) is not 4:2:0, 4:2:2 or 4:4:4", xdec, ydec);
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  B200_REQUIRE(ctx, frame_width > 0 && frame_height > 0 && frame_width <= 65536 && frame_height <= 65536,
               "bad frame size %dx%d", frame_width, frame_height);
  const int bpp = bit_depth == 8 ? 1 : 2;
  const int w8px = (frame_width + 7) & ~7, h8px = (frame_height + 7) & ~7;
  for (int p = 0; p < planes; p++) {
    const int xd = p ? xdec : 0, yd = p ? ydec : 0;
    for (const b200_plane *pl : {lrf_in, src}) {
      B200_REQUIRE(ctx, pl[p].data != nullptr, "NULL plane %d", p);
      B200_REQUIRE(ctx, pl[p].bpp == bpp, "plane %d: bpp %d does not match bit depth %d", p, pl[p].bpp, bit_depth);
      B200_REQUIRE(ctx, pl[p].width >= (w8px >> xd) && pl[p].height >= (h8px >> yd) && pl[p].stride >= pl[p].width,
                   "plane %d (%dx%d) smaller than the frame's 8x8 blocks (%dx%d)", p, pl[p].width, pl[p].height,
                   w8px >> xd, h8px >> yd);
    }
    const int us = unit_size[p];
    // whole superblocks, at most the 4x4 of an area (rdo.rs:2160-2162)
    B200_REQUIRE(ctx, is_unit_size(us) && ((us << xd) % 64) == 0 && ((us << yd) % 64) == 0 && (us << xd) <= 256 &&
                          (us << yd) <= 256,
                 "plane %d: unit size %d is not 32..256 in whole superblocks", p, us);
  }
  if (n_items == 0) return B200_OK;
  B200_REQUIRE(ctx, areas != nullptr && items != nullptr, "NULL areas / items");
  const int sbw = (frame_width + 63) >> 6, sbh = (frame_height + 63) >> 6;
  for (size_t k = 0; k < n_areas; k++) {
    const b200_cdef_rdo_area &r = areas[k];
    B200_REQUIRE(ctx, r.sb_w >= 1 && r.sb_w <= 4 && r.sb_h >= 1 && r.sb_h <= 4, "area %zu: %dx%d superblocks", k,
                 r.sb_w, r.sb_h);
    B200_REQUIRE(ctx, r.sbx >= 0 && r.sby >= 0 && r.sbx + r.sb_w <= sbw && r.sby + r.sb_h <= sbh,
                 "area %zu (%d, %d, %dx%d) outside the %dx%d superblock frame", k, r.sbx, r.sby, r.sb_w, r.sb_h, sbw,
                 sbh);
  }
  B200_REQUIRE(ctx, n_items <= (1u << 24), "%zu items: at most 2^24 per call", n_items);
  std::vector<Geo> geo(n_items);
  std::vector<Tile> tiles;
  for (size_t i = 0; i < n_items; i++) {
    const b200_lrf_search_item &it = items[i];
    B200_REQUIRE(ctx, it.area >= 0 && (size_t)it.area < n_areas, "item %zu: area %d of %zu", i, it.area, n_areas);
    B200_REQUIRE(ctx, it.plane >= 0 && it.plane < planes, "item %zu: plane %d", i, it.plane);
    const b200_cdef_rdo_area &r = areas[it.area];
    const int p = it.plane, xd = p ? xdec : 0, yd = p ? ydec : 0, us = unit_size[p];
    const int lsw = (us << xd) / 64, lsh = (us << yd) / 64;
    B200_REQUIRE(ctx, it.lru_x >= 0 && it.lru_y >= 0 && it.lru_x * lsw < r.sb_w && it.lru_y * lsh < r.sb_h,
                 "item %zu: unit (%d, %d) outside its %dx%d area", i, it.lru_x, it.lru_y, r.sb_w, r.sb_h);
    Geo &g = geo[i];
    g = lrf_unit_geo(r, p, xd, yd, us, it.lru_x, it.lru_y, frame_width, frame_height);
    B200_REQUIRE(ctx, g.vis_w > 0 && g.vis_h > 0, "item %zu: unit (%d, %d) outside the visible frame", i, it.lru_x,
                 it.lru_y);
    const b200_lrf_unit &u = it.incoming;
    B200_REQUIRE(ctx, u.type == 0 || u.type == 2, "item %zu: incoming filter type %d is not None or Sgrproj", i,
                 u.type);
    if (u.type == 2)
      B200_REQUIRE(ctx, u.set <= 15 && u.xqd[0] >= -96 && u.xqd[0] <= 31 && u.xqd[1] >= -32 && u.xqd[1] <= 95,
                   "item %zu: incoming Sgrproj (set %d, xqd %d %d) out of range", i, u.set, u.xqd[0], u.xqd[1]);
    B200_REQUIRE(ctx, it.sgrproj_ref[0] >= -96 && it.sgrproj_ref[0] <= 31 && it.sgrproj_ref[1] >= -32 &&
                          it.sgrproj_ref[1] <= 95,
                 "item %zu: sgrproj_ref (%d, %d) out of range", i, it.sgrproj_ref[0], it.sgrproj_ref[1]);
    for (int ty = 0; ty < g.eh; ty += kT)
      for (int tx = 0; tx < g.ew; tx += kT) tiles.push_back(Tile{(uint32_t)i, (uint16_t)tx, (uint16_t)ty});
  }

  SearchArgs a{};
  for (int p = 0; p < planes; p++) {
    a.in[p] = PlaneView{lrf_in[p].data, lrf_in[p].stride};
    a.src[p] = PlaneView{src[p].data, src[p].stride};
  }
  a.xdec = xdec, a.ydec = ydec, a.bit_depth = bit_depth, a.w8 = w8px >> 3;
  a.reduced = reduced_sets != 0;
  a.nsets = a.reduced ? 8 : 16;
  a.imp = d_imp_scales;
  for (int p = 0; p < 3; p++) a.dist_scale[p] = p < planes ? dist_scale[p] : 0;
  a.lambda = lambda;
  a.n_items = (uint32_t)n_items;
  a.n_tiles = (uint32_t)tiles.size();
  a.best = d_best, a.cost = d_cost, a.changed = d_changed;
  a.out_xqd = d_xqd, a.out_err = d_err, a.out_cand_cost = d_cand_cost;

  // items, geometry and tiles go up in one copy; the accumulators live in the same stream-ordered arena
  const size_t b_items = n_items * sizeof(b200_lrf_search_item), b_geo = n_items * sizeof(Geo);
  const size_t b_tiles = tiles.size() * sizeof(Tile), b_acc = n_items * 16 * 5 * sizeof(long long);
  const size_t b_err = n_items * kCands * sizeof(unsigned long long), b_xq = n_items * 32;
  const size_t o_geo = b200_align_up(b_items, 256), o_tiles = o_geo + b200_align_up(b_geo, 256);
  const size_t up_bytes = o_tiles + b_tiles;
  std::vector<uint8_t> packed(up_bytes);
  memcpy(packed.data(), items, b_items);
  memcpy(packed.data() + o_geo, geo.data(), b_geo);
  memcpy(packed.data() + o_tiles, tiles.data(), b_tiles);
  HostStage s(ctx, b200_align_up(up_bytes, 256) + b200_align_up(b_acc, 256) + b200_align_up(b_err, 256) + b_xq);
  uint8_t *d_up = s.take(up_bytes);
  a.acc = (long long *)s.take(b_acc);
  a.err = (unsigned long long *)s.take(b_err);
  a.xq = (int8_t *)s.take(b_xq);
  s.up(d_up, packed.data(), up_bytes);
  if (!s.ok()) return s.finish(false);
  a.items = (const b200_lrf_search_item *)d_up;
  a.geo = (const Geo *)(d_up + o_geo);
  a.tiles = (const Tile *)(d_up + o_tiles);
  s.run(cudaMemsetAsync(a.acc, 0, b_acc, ctx->stream) == cudaSuccess ? B200_OK : B200_ERR_CUDA);
  s.run(cudaMemsetAsync(a.err, 0, b_err, ctx->stream) == cudaSuccess ? B200_OK : B200_ERR_CUDA);
  if (!s.ok()) return s.finish(false);

  const unsigned tile_grid = (unsigned)std::min<size_t>(tiles.size(), 8192);
  const unsigned solve_grid = (unsigned)std::min<size_t>((n_items * a.nsets + 255) / 256, 4096);
  const unsigned item_grid = (unsigned)std::min<size_t>((n_items + 255) / 256, 4096);
  if (bpp == 1) lrf_search_tiles<uint8_t, false><<<tile_grid, kThreads, 0, ctx->stream>>>(a);
  else lrf_search_tiles<uint16_t, false><<<tile_grid, kThreads, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  lrf_search_solve<<<solve_grid, 256, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  if (bpp == 1) lrf_search_tiles<uint8_t, true><<<tile_grid, kThreads, 0, ctx->stream>>>(a);
  else lrf_search_tiles<uint16_t, true><<<tile_grid, kThreads, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  lrf_search_decide<<<item_grid, 256, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return s.finish(false);
}
