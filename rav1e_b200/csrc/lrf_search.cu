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
#include "lrf_dev.cuh"
#include "rdo_dist_dev.cuh"

namespace {

constexpr int kT = 32;              // tile side, plane pixels
constexpr int kThreads = 256;
constexpr int kSP = kT + 6;         // staged pixels per side: the tile plus 3 on each side
constexpr int kAB = kT + 2;         // a / b columns (and radius-1 rows): -1 .. kT
constexpr int kR2 = kT / 2 + 1;     // radius-2 a / b rows: the odd rows -1 .. kT - 1
constexpr int kCands = 17;          // None, then sets 0 .. 15

struct Tile {
  uint32_t item;
  uint16_t tx, ty;  // tile origin inside the unit, plane pixels
};

struct Geo {  // an item's unit, in its plane's pixels
  int ax, ay;                   // the area's origin
  int po_x, po_y;               // the unit's origin inside the area
  int vis_w, vis_h;             // the visible rect (rdo.rs:2651-2658)
  int ew, eh;                   // the unit's 8x8 blocks that lie inside the area's block grid
  int gbx0, gby0;               // the unit's first 8x8 block, frame-absolute
  int p, xd, yd;
};

struct SearchArgs {
  PlaneView in[3], src[3];
  int xdec, ydec, bit_depth, w8, nsets, reduced;
  const uint32_t *imp;
  uint32_t dist_scale[3];
  double lambda;
  const b200_lrf_search_item *items;
  const Geo *geo;
  const Tile *tiles;
  uint32_t n_items, n_tiles;
  long long *acc;               // [item][set][5]: H00, H11, H01, C0, C1
  unsigned long long *err;      // [item][17]
  int8_t *xq;                   // [item][16][2]
  b200_lrf_unit *best;
  double *cost;
  uint8_t *changed;
  int8_t *out_xqd;
  uint64_t *out_err;
  double *out_cand_cost;
};

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
    const Geo g = A.geo[tl.item];
    const int tx = tl.tx, ty = tl.ty;
    const T *in = (const T *)A.in[g.p].data + (long long)g.ay * A.in[g.p].stride + g.ax;
    const T *sr = (const T *)A.src[g.p].data + (long long)g.ay * A.src[g.p].stride + g.ax;
    const int is = A.in[g.p].stride, ssd = A.src[g.p].stride;
    // setup_integral_image's clip rule: columns clamp to [0, po_x + vis_w) of the area (4 real columns on
    // the left, none past the right edge), rows to [max(0, po_y - 2), po_y + vis_h)
    const int c_lo = 0, c_hi = g.po_x + g.vis_w - 1, r_lo = max(0, g.po_y - 2), r_hi = g.po_y + g.vis_h - 1;
    for (int i = t; i < kSP * kSP; i += kThreads) {
      const int r = i / kSP, c = i - r * kSP;
      const int y = min(max(g.po_y + ty - 3 + r, r_lo), r_hi), x = min(max(g.po_x + tx - 3 + c, c_lo), c_hi);
      sp[r][c] = (uint16_t)in[(long long)y * is + x];
    }
    const int tw = min(kT, g.ew - tx), th = min(kT, g.eh - ty);  // the tile's part of the unit's blocks
    for (int i = t; i < kT * kT; i += kThreads) {
      const int r = i / kT, c = i - r * kT;
      ss[r][c] = r < th && c < tw ? (uint16_t)sr[(long long)(g.po_y + ty + r) * ssd + g.po_x + tx + c] : 0;
    }
    __syncthreads();
    for (int i = t; i < kAB * kAB; i += kThreads) {  // radius 1: every row -1 .. kT
      const int j = i / kAB, m = i - j * kAB;
      uint32_t sum = 0, ssq = 0;
#pragma unroll
      for (int dy = 0; dy < 3; dy++)
#pragma unroll
        for (int dx = 0; dx < 3; dx++) {
          const uint32_t v = sp[j + 1 + dy][m + 1 + dx];
          sum += v;
          ssq += v * v;
        }
      box1[0][j][m] = sum;
      box1[1][j][m] = ssq;
    }
    for (int i = t; i < kR2 * kAB; i += kThreads) {  // radius 2: odd rows -1, 1, .. kT - 1
      const int j = i / kAB, m = i - j * kAB;
      uint32_t sum = 0, ssq = 0;
#pragma unroll
      for (int dy = 0; dy < 5; dy++)
#pragma unroll
        for (int dx = 0; dx < 5; dx++) {
          const uint32_t v = sp[2 * j + dy][m + dx];
          sum += v;
          ssq += v * v;
        }
      box2[0][j][m] = sum;
      box2[1][j][m] = ssq;
    }

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
      if (s1)
        for (int i = t; i < kAB * kAB; i += kThreads) {
          const int j = i / kAB, m = i - j * kAB;
          sum_finish(box1[1][j][m], box1[0][j][m], 9, 455, s1, bdm8, a1[j][m], b1[j][m]);
        }
      if (s2)
        for (int i = t; i < kR2 * kAB; i += kThreads) {
          const int j = i / kAB, m = i - j * kAB;
          sum_finish(box2[1][j][m], box2[0][j][m], 25, 164, s2, bdm8, a2[j][m], b2[j][m]);
        }
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
        const uint32_t px = sp[y + 3][x + 3];
        uint32_t f2, f1 = px << 4;
        if (s2) {  // even rows weigh the a / b rows above and below, odd rows their own
          const int j = (y + 1) >> 1;
          uint32_t av = r2_row(a2[j], x), bv = r2_row(b2[j], x);
          if (y & 1) {
            f2 = (av * px + bv + (1u << 7)) >> 8;
          } else {
            av += r2_row(a2[j + 1], x);
            bv += r2_row(b2[j + 1], x);
            f2 = (av * px + bv + (1u << 8)) >> 9;
          }
        } else {  // sgrproj_box_f_r0 of the even row, shared by the odd row below it (lrf.rs:740-749)
          f2 = (uint32_t)sp[(y & ~1) + 3][x + 3] << 4;
        }
        if (s1) f1 = (r1_weigh(a1, y, x) * px + r1_weigh(b1, y, x) + (1u << 8)) >> 9;
        const int u = (int)(px << 4);
        if (ERR) {  // apply_filter (lrf.rs:796-815)
          const int v = w0 * (int)f2 + w1 * u + w2 * (int)f1;
          st[y][x] = (uint16_t)min(max((v + (1 << 10)) >> 11, 0), (1 << bd) - 1);
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

// count_quniform / count_subexp / recenter / count_signed_subexp_with_ref (ec.rs:381-389, 639-773)
__device__ uint32_t count_quniform(uint32_t n, uint32_t v) {
  if (n <= 1) return 0;
  const uint32_t l = 32 - __clz(n), m = (1u << l) - n;
  return ((l - 1) << 3) + (v >= m ? 8u : 0u);
}
__device__ uint32_t count_subexp(uint32_t n, uint32_t k, uint32_t v) {
  uint32_t i = 0, mk = 0, bits = 0;
  for (;;) {
    const uint32_t b = i ? k + i - 1 : k, a = 1u << b;
    if (n <= mk + 3 * a) return bits + count_quniform(n - mk, v - mk);
    bits += 8;
    if (v < mk + a) return bits + (b << 3);
    i++;
    mk += a;
  }
}
__device__ uint32_t recenter(uint32_t r, uint32_t v) {
  return v > (r << 1) ? v : v >= r ? (v - r) << 1 : ((r - v) << 1) - 1;
}
__device__ uint32_t count_signed_subexp_with_ref(int v, int low, int high, uint32_t k, int r) {
  const uint32_t uv = (uint32_t)(v - low), n = (uint32_t)(high - low), ur = (uint32_t)(r - low);
  return (ur << 1) <= n ? count_subexp(n, k, recenter(ur, uv)) : count_subexp(n, k, recenter(n - 1 - ur, n - 1 - uv));
}
// count_lrf_switchable (context/frame_header.rs:14-45) for None (type 0) or Sgrproj
__device__ uint32_t lrf_rate(const b200_lrf_search_item &it, int type, int set, int x0, int x1) {
  if (type == 0) return it.none_bits;
  uint32_t bits = it.sgr_bits + (4u << 3);
  if (kSgrS[set][0]) bits += count_signed_subexp_with_ref(x0, -96, 32, 4, it.sgrproj_ref[0]);
  if (kSgrS[set][1]) bits += count_signed_subexp_with_ref(x1, -32, 96, 4, it.sgrproj_ref[1]);
  return bits;
}

__device__ __forceinline__ double rd_cost(double lambda, uint32_t rate, unsigned long long dist) {
  return __fma_rn(lambda, (double)rate / 8.0, (double)dist);  // compute_rd_cost, rdo.rs:718-723
}

__global__ void lrf_search_decide(const __grid_constant__ SearchArgs A) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < A.n_items; i += gridDim.x * blockDim.x) {
    const b200_lrf_search_item it = A.items[i];
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
  }
}

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
    g.ax = (r.sbx * 64) >> xd, g.ay = (r.sby * 64) >> yd;
    const int crop_w = frame_width - r.sbx * 64, crop_h = frame_height - r.sby * 64;
    g.po_x = (it.lru_x * lsw * 64) >> xd, g.po_y = (it.lru_y * lsh * 64) >> yd;
    g.vis_w = std::min(us, (crop_w >> xd) - g.po_x), g.vis_h = std::min(us, (crop_h >> yd) - g.po_y);
    B200_REQUIRE(ctx, g.vis_w > 0 && g.vis_h > 0, "item %zu: unit (%d, %d) outside the visible frame", i, it.lru_x,
                 it.lru_y);
    const int aw = (std::min(crop_w, r.sb_w * 64) + 7) & ~7, ah = (std::min(crop_h, r.sb_h * 64) + 7) & ~7;
    g.ew = std::min(us, (aw >> xd) - g.po_x), g.eh = std::min(us, (ah >> yd) - g.po_y);
    g.gbx0 = r.sbx * 8 + it.lru_x * lsw * 8, g.gby0 = r.sby * 8 + it.lru_y * lsh * 8;
    g.p = p, g.xd = xd, g.yd = yd;
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
