// lrf_search.cu — the restoration search of one rdo_loop_decision pass (rav1e src/rdo.rs:2575-2740) for many
// (area, plane, unit) items in one call: the None candidate, then per self-guided set sgrproj_solve
// (lrf.rs:846-1096), sgrproj_stripe_filter over the unit's visible rect, rdo_loop_plane_error
// (rdo.rs:2027-2093), count_lrf_switchable (context/frame_header.rs:14-45) and compute_rd_cost.
//
// Four launches, whatever the item count, made by lrf_search_launch for this entry point and for each
// restoration stage of b200_loop_decision_dev (loop_decision.cu):
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

#include "loop_filter_checks.cuh"
#include "lrf_search_dev.cuh"

namespace {

__device__ __forceinline__ int set_of(const SearchArgs &A, int si) { return A.reduced ? 2 * si + 1 : si; }

template <typename T, bool ERR>
__global__ void __launch_bounds__(kThreads) lrf_search_tiles(const __grid_constant__ SearchArgs A) {
  __shared__ uint16_t sp[kSP][kSP];            // lrf_in through the clip rule
  __shared__ uint16_t ss[kT][kT];              // src
  __shared__ uint16_t st[kT][kT];              // ERR: the candidate's test pixels
  __shared__ uint32_t box1[2][kAB][kAB];       // radius-1 sum / sum of squares
  __shared__ uint32_t box2[2][kR2][kAB];       // radius-2 sum / sum of squares
  __shared__ uint32_t a1[kAB][kAB], b1[kAB][kAB], a2[kR2][kAB], b2[kR2][kAB];
  __shared__ unsigned long long red[kThreads / 32][5];

  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int bd = A.bit_depth, bdm8 = bd - 8;
  for (uint32_t k = blockIdx.x; k < A.n_tiles; k += gridDim.x) {
    const Tile tl = A.tiles[k];
    if (A.active && !A.active[A.items[tl.item].area]) continue;
    const Geo g = A.geo[tl.item];
    const int tx = tl.tx, ty = tl.ty;
    const T *in = (const T *)A.in[g.p].data + (long long)g.ay * A.in[g.p].stride + g.ax;
    const T *sr = (const T *)A.src[g.p].data + (long long)g.ay * A.src[g.p].stride + g.ax;
    const int is = A.in[g.p].stride, ssd = A.src[g.p].stride;
    sgr_stage_tile<T>(sp, in, is, g.po_x, g.po_y, g.vis_w, g.vis_h, tx, ty);
    const int tw = min(kT, g.ew - tx), th = min(kT, g.eh - ty);  // the tile's part of the unit's blocks
    for (int i = t; i < kT * kT; i += kThreads) {
      const int r = i / kT, c = i - r * kT;
      ss[r][c] = r < th && c < tw ? (uint16_t)sr[(long long)(g.po_y + ty + r) * ssd + g.po_x + tx + c] : 0;
    }
    __syncthreads();
    sgr_box_sums(sp, box1, box2);

    // ERR: the unit's 8x8 blocks in this tile, one thread each (rdo_loop_plane_error)
    const int bw = 8 >> g.xd, bh = 8 >> g.yd, nbx = kT / bw, nb = nbx * (kT / bh);
    const int bx = t % nbx, by = t / nbx;
    const bool blk = ERR && t < nb && bx * bw < tw && by * bh < th;
    uint32_t bias = 1u << 14;
    if (blk && A.imp) bias = A.imp[(size_t)(g.gby0 + ((ty + by * bh) / bh)) * A.w8 + g.gbx0 + (tx + bx * bw) / bw];
    auto block_err = [&]() -> unsigned long long {  // of st against ss
      if (!blk) return 0ull;
      const int x0 = bx * bw, y0 = by * bh;
      if (g.p == 0) {  // cdef_dist_kernel 8x8 times the bias (mul_u64)
        uint32_t s1 = 0, d1 = 0, s2 = 0, d2 = 0, sd = 0;
        for (int r = 0; r < 8; r++)
          for (int c = 0; c < 8; c++) {
            const uint32_t s = ss[y0 + r][x0 + c], d = st[y0 + r][x0 + c];
            s1 += s, d1 += d, s2 += s * s, d2 += d * d, sd += s * d;
          }
        uint32_t sv, dv;
        const uint32_t sse = cdef_dist_vars(s1, d1, s2, d2, sd, 64, &sv, &dv);
        return ((unsigned long long)bias * apply_ssim_boost(sse, sv, dv, bd) + (1u << 13)) >> 14;
      }
      unsigned long long acc = 0;  // sse_wxh: get_weighted_sse with the bias on every 4x4 chunk
      for (int cy = 0; cy < bh; cy += 4)
        for (int cx = 0; cx < bw; cx += 4) {
          uint32_t e = 0;
          for (int r = 0; r < 4; r++)
            for (int c = 0; c < 4; c++) {
              const int d = (int)ss[y0 + cy + r][x0 + cx + c] - (int)st[y0 + cy + r][x0 + cx + c];
              e += (uint32_t)(d * d);
            }
          acc += wsse_chunk(e, bias);
        }
      return wsse_finish(acc);
    };
    auto reduce_add = [&](unsigned long long v, unsigned long long *dst) {
#pragma unroll
      for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) red[warp][0] = v;
      __syncthreads();
      if (t == 0) {
        unsigned long long s = 0;
        for (int w = 0; w < kThreads / 32; w++) s += red[w][0];
        atomicAdd(dst, s);
      }
    };
    if (ERR) {  // the None candidate: lrf_in itself over the blocks
      for (int i = t; i < kT * kT; i += kThreads) {
        const int r = i / kT, c = i - r * kT;
        st[r][c] = r < th && c < tw ? (uint16_t)in[(long long)(g.po_y + ty + r) * is + g.po_x + tx + c] : 0;
      }
      __syncthreads();
      reduce_add(block_err(), &A.err[(size_t)tl.item * kCands]);
    }

    for (int si = 0; si < A.nsets; si++) {
      const int set = set_of(A, si);
      const uint32_t s2 = kSgrS[set][0], s1 = kSgrS[set][1];
      __syncthreads();
      sgr_ab(box1, box2, a1, b1, a2, b2, s1, s2, bdm8);
      __syncthreads();
      int w0 = 0, w1 = 0, w2 = 0;
      if (ERR) {
        const int8_t *q = &A.xq[((size_t)tl.item * 16 + set) * 2];
        w0 = q[0], w1 = q[1], w2 = 128 - w0 - w1;
      }
      long long h00 = 0, h11 = 0, h01 = 0, c0 = 0, c1 = 0;
      for (int i = t; i < kT * kT; i += kThreads) {
        const int y = i / kT, x = i - y * kT;
        const bool vis = tx + x < g.vis_w && ty + y < g.vis_h;
        if (!vis) {
          if (ERR) st[y][x] = B200_LRF_WORK_FILL;
          continue;
        }
        uint32_t f1, f2;
        const uint32_t px = sgr_f(sp, a1, b1, a2, b2, s1, s2, y, x, f1, f2);
        const int u = (int)(px << 4);
        if (ERR) {
          st[y][x] = sgr_apply(w0, w1, w2, f1, f2, px, bd);
        } else {  // process_line (lrf.rs:997-1037)
          const long long s = (long long)(((int)ss[y][x] << 4) - u), e2 = (int)f2 - u, e1 = (int)f1 - u;
          h00 += e2 * e2;
          h11 += e1 * e1;
          h01 += e1 * e2;
          c0 += e2 * s;
          c1 += e1 * s;
        }
      }
      if (ERR) {
        __syncthreads();
        reduce_add(block_err(), &A.err[(size_t)tl.item * kCands + 1 + set]);
      } else {
        long long v[5] = {h00, h11, h01, c0, c1};
#pragma unroll
        for (int q = 0; q < 5; q++) {
#pragma unroll
          for (int o = 16; o; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
          if (lane == 0) red[warp][q] = (unsigned long long)v[q];
        }
        __syncthreads();
        if (t < 5) {
          unsigned long long s = 0;
          for (int w = 0; w < kThreads / 32; w++) s += red[w][t];
          atomicAdd((unsigned long long *)&A.acc[((size_t)tl.item * 16 + set) * 5 + t], s);
        }
      }
    }
    __syncthreads();
  }
}

// Rust's saturating `f64 as i32` (NaN -> 0)
__device__ __forceinline__ int sat_i32(double v) {
  return v != v ? 0 : v >= 2147483647.0 ? INT_MAX : v <= -2147483648.0 ? INT_MIN : (int)v;
}

// sgrproj_solve's closing arithmetic (lrf.rs:1051-1095).  The sums are exact integers: |s|, |f1 - u|,
// |f2 - u| < 2^17, so a product is below 2^34 and a 256x256 unit's total below 2^50 < 2^53; the
// reference's f64 accumulation of i64 line sums therefore equals the i64 total converted once.  The
// explicit _rn intrinsics keep nvcc from contracting or reordering the reference's f64 operations.
__global__ void lrf_search_solve(const __grid_constant__ SearchArgs A) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < A.n_items * (uint32_t)A.nsets;
       k += gridDim.x * blockDim.x) {
    const uint32_t item = k / A.nsets;
    if (A.active && !A.active[A.items[item].area]) continue;
    const int set = set_of(A, (int)(k % A.nsets));
    const Geo g = A.geo[item];
    const long long *acc = &A.acc[((size_t)item * 16 + set) * 5];
    const double n = __dmul_rn((double)g.vis_w, (double)g.vis_h);
    const double h00 = __ddiv_rn((double)acc[0], n), h11 = __ddiv_rn((double)acc[1], n);
    const double h01 = __ddiv_rn((double)acc[2], n), h10 = h01;
    const double sc = __ddiv_rn(128.0, n);
    const double c0 = __dmul_rn((double)acc[3], sc), c1 = __dmul_rn((double)acc[4], sc);
    int xq0 = 0, xq1 = 0;
    if (kSgrS[set][0] == 0) {
      if (h11 != 0.) xq1 = sat_i32(round(__ddiv_rn(c1, h11)));
    } else if (kSgrS[set][1] == 0) {
      if (h00 != 0.) xq0 = sat_i32(round(__ddiv_rn(c0, h00)));
    } else {
      const double det = __fma_rn(h00, h11, -__dmul_rn(h01, h10));
      if (det != 0.) {
        const double div1 = __fma_rn(h11, c0, -__dmul_rn(h01, c1));
        const double div2 = __fma_rn(h00, c1, -__dmul_rn(h10, c0));
        xq0 = sat_i32(round(__ddiv_rn(div1, det)));
        xq1 = sat_i32(round(__ddiv_rn(div2, det)));
      }
    }
    const int xqd0 = min(max(xq0, -96), 31);
    // (1 << SGRPROJ_PRJ_BITS) - xqd0 - xq1 in i32, wrapping as a release build computes it
    const int xqd1 = min(max((int)(128u - (uint32_t)xqd0 - (uint32_t)xq1), -32), 95);
    int8_t *q = &A.xq[((size_t)item * 16 + set) * 2];
    q[0] = (int8_t)xqd0;
    q[1] = (int8_t)xqd1;
    if (A.out_xqd) {
      A.out_xqd[((size_t)item * 16 + set) * 2] = (int8_t)xqd0;
      A.out_xqd[((size_t)item * 16 + set) * 2 + 1] = (int8_t)xqd1;
    }
  }
}

__global__ void lrf_search_decide(const __grid_constant__ SearchArgs A) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < A.n_items; i += gridDim.x * blockDim.x) {
    b200_lrf_search_item it = A.items[i];
    if (A.active && !A.active[it.area]) continue;
    if (A.inc) {  // the incumbent carried from the previous restoration stage
      it.incoming = A.inc[A.unit_of[i]];
      it.incoming_cost = A.inc_cost[A.unit_of[i]];
    }
    const uint32_t ds = A.dist_scale[A.geo[i].p];
    b200_lrf_unit best = it.incoming;
    double best_cost = it.incoming_cost;
    {  // None, rated with the incoming filter (rdo.rs:2633-2638)
      const unsigned long long e = ((unsigned long long)ds * A.err[(size_t)i * kCands] + (1u << 13)) >> 14;
      const double c = rd_cost(A.lambda, lrf_rate(it, it.incoming.type, it.incoming.set, it.incoming.xqd[0],
                                                  it.incoming.xqd[1]), e);
      if (A.out_err) A.out_err[(size_t)i * kCands] = e;
      if (A.out_cand_cost) A.out_cand_cost[(size_t)i * kCands] = c;
      if (best_cost < 0. || c < best_cost) {
        best_cost = c;
        best = b200_lrf_unit{};
      }
    }
    for (int si = 0; si < A.nsets; si++) {
      const int set = set_of(A, si);
      const int8_t *q = &A.xq[((size_t)i * 16 + set) * 2];
      const size_t slot = (size_t)i * kCands + 1 + set;
      const unsigned long long e = ((unsigned long long)ds * A.err[slot] + (1u << 13)) >> 14;
      const double c = rd_cost(A.lambda, lrf_rate(it, 2, set, q[0], q[1]), e);
      if (A.out_err) A.out_err[slot] = e;
      if (A.out_cand_cost) A.out_cand_cost[slot] = c;
      if (c < best_cost) {
        best_cost = c;
        best = b200_lrf_unit{};
        best.type = 2;
        best.set = (uint8_t)set;
        best.xqd[0] = q[0];
        best.xqd[1] = q[1];
      }
    }
    A.best[i] = best;
    A.cost[i] = best_cost;
    // RestorationFilter::notequal (lrf.rs:139-160)
    const bool ne = it.incoming.type != best.type ||
                    (best.type == 2 && !(it.incoming.set == best.set && it.incoming.xqd[0] == best.xqd[0] &&
                                         it.incoming.xqd[1] == best.xqd[1]));
    A.changed[i] = ne;
    if (A.inc) {  // rdo.rs:2730-2741
      const uint32_t u = A.unit_of[i];
      A.inc_cost[u] = best_cost;
      if (ne) {
        A.inc[u] = best;
        A.written[u] = 1;
        A.area_changed[it.area] = 1;
      }
    }
  }
}

}  // namespace

int lrf_search::lrf_search_launch(b200_ctx *ctx, HostStage &s, const SearchArgs &a) {
  auto zero = [&](void *p, size_t bytes) {
    s.run(cudaMemsetAsync(p, 0, bytes, ctx->stream) == cudaSuccess ? B200_OK : B200_ERR_CUDA);
  };
  zero(a.acc, (size_t)a.n_items * 16 * 5 * sizeof(long long));
  zero(a.err, (size_t)a.n_items * kCands * sizeof(unsigned long long));
  if (!s.ok()) return s.finish(false);
  const unsigned tile_grid = std::min<unsigned>(a.n_tiles, 8192);
  const unsigned solve_grid = (unsigned)std::min<size_t>(((size_t)a.n_items * a.nsets + 255) / 256, 4096);
  const unsigned item_grid = (unsigned)std::min<size_t>(((size_t)a.n_items + 255) / 256, 4096);
  const bool u8 = a.bit_depth == 8;
  if (u8) lrf_search_tiles<uint8_t, false><<<tile_grid, kThreads, 0, ctx->stream>>>(a);
  else lrf_search_tiles<uint16_t, false><<<tile_grid, kThreads, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  lrf_search_solve<<<solve_grid, 256, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  if (u8) lrf_search_tiles<uint8_t, true><<<tile_grid, kThreads, 0, ctx->stream>>>(a);
  else lrf_search_tiles<uint16_t, true><<<tile_grid, kThreads, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  lrf_search_decide<<<item_grid, 256, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_lrf_search_dev(b200_ctx *ctx, const b200_plane *lrf_in, const b200_plane *src, int planes,
                                   int xdec, int ydec, int frame_width, int frame_height, int bit_depth,
                                   const int unit_size[3], int reduced_sets, const uint32_t *d_imp_scales,
                                   const uint32_t dist_scale[3], double lambda, const b200_cdef_rdo_area *areas,
                                   size_t n_areas, const b200_lrf_search_item *items, size_t n_items,
                                   b200_lrf_unit *d_best, double *d_cost, uint8_t *d_changed, int8_t *d_xqd,
                                   uint64_t *d_err, double *d_cand_cost) {
  if (int st = lf_check_frame(ctx, planes, xdec, ydec, bit_depth, frame_width, frame_height)) return st;
  B200_REQUIRE(ctx, lrf_in && src && dist_scale && d_best && d_cost && d_changed,
               "NULL lrf_in / src / dist_scale / outputs");
  for (const b200_plane *pl : {lrf_in, src})
    if (int st = lf_check_planes(ctx, pl, planes, xdec, ydec, bit_depth, frame_width, frame_height)) return st;
  if (int st = lf_check_unit_sizes(ctx, unit_size, planes, xdec, ydec)) return st;
  if (n_items == 0) return B200_OK;
  B200_REQUIRE(ctx, items != nullptr, "NULL items");
  if (int st = lf_check_areas(ctx, areas, n_areas, frame_width, frame_height, false)) return st;
  B200_REQUIRE(ctx, n_items <= (1u << 24), "%zu items: at most 2^24 per call", n_items);
  std::vector<Geo> geo(n_items);
  std::vector<Tile> tiles;
  for (size_t i = 0; i < n_items; i++) {
    const b200_lrf_search_item &it = items[i];
    B200_REQUIRE(ctx, it.area >= 0 && (size_t)it.area < n_areas, "item %zu: area %d of %zu", i, it.area, n_areas);
    B200_REQUIRE(ctx, it.plane >= 0 && it.plane < planes, "item %zu: plane %d", i, it.plane);
    if (int st = lrf_item_geo(ctx, i, areas[it.area], it.plane, xdec, ydec, unit_size[it.plane], it.lru_x, it.lru_y,
                              frame_width, frame_height, geo[i]))
      return st;
    const b200_lrf_unit &u = it.incoming;
    B200_REQUIRE(ctx, u.type == 0 || u.type == 2, "item %zu: incoming filter type %d is not None or Sgrproj", i,
                 u.type);
    if (u.type == 2)
      B200_REQUIRE(ctx, u.set <= 15 && sgrproj_xqd_ok(u.xqd[0], u.xqd[1]),
                   "item %zu: incoming Sgrproj (set %d, xqd %d %d) out of range", i, u.set, u.xqd[0], u.xqd[1]);
    B200_REQUIRE(ctx, sgrproj_xqd_ok(it.sgrproj_ref[0], it.sgrproj_ref[1]), "item %zu: sgrproj_ref (%d, %d) out of range",
                 i, it.sgrproj_ref[0], it.sgrproj_ref[1]);
    lrf_item_tiles(geo[i], (uint32_t)i, tiles);
  }

  SearchArgs a = search_args(lrf_in, src, planes, xdec, ydec, bit_depth, frame_width, reduced_sets, d_imp_scales,
                             dist_scale, lambda);
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
  if (int st = lrf_search::lrf_search_launch(ctx, s, a)) return st;
  return s.finish(false);
}
