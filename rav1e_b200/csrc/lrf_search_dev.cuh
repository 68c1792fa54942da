// lrf_search_dev.cuh — the restoration search's kernels (rav1e src/rdo.rs:2575-2740), shared by the search
// entry point (lrf_search.cu) and the pass loop of rdo_loop_decision (loop_decision.cu), which launches them
// once per restoration stage with the incumbents carried on the device.  The self-guided tile pieces
// (staging through setup_integral_image's clip rule, box sums, a / b, the two filter outputs) are also the
// C stage's Sgrproj branch.  See lrf_search.cu for the launch sequence.
#pragma once
#include <algorithm>
#include <vector>

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
  // the restoration stage of rdo_loop_decision's pass loop (loop_decision.cu); all NULL for b200_lrf_search_dev
  const uint32_t *unit_of;  // [item] -> the carried unit
  b200_lrf_unit *inc;       // [unit] the incumbent filter, updated in place
  double *inc_cost;         // [unit] best_lrf_cost, updated in place
  uint8_t *written;         // [unit] set when the unit's filter changes
  const uint8_t *active;    // [area] areas still in the pass loop; the others' items are skipped
  uint8_t *area_changed;    // [area] set when a unit of the area changes
};

// setup_integral_image's clip rule (lrf.rs:529-627) for a unit at (po_x, po_y) of its area with visible rect
// vis_w x vis_h: columns clamp to [0, po_x + vis_w) of the area (4 real columns on the left, none past the
// right edge), rows to [max(0, po_y - 2), po_y + vis_h).  Stages the 32x32 tile at (tx, ty) of the unit plus
// 3 pixels on every side; `in` addresses the area's origin.
template <typename T>
__device__ __forceinline__ void sgr_stage_tile(uint16_t (*sp)[kSP], const T *in, int is, int po_x, int po_y,
                                               int vis_w, int vis_h, int tx, int ty) {
  const int c_lo = 0, c_hi = po_x + vis_w - 1, r_lo = max(0, po_y - 2), r_hi = po_y + vis_h - 1;
  for (int i = threadIdx.x; i < kSP * kSP; i += kThreads) {
    const int r = i / kSP, c = i - r * kSP;
    const int y = min(max(po_y + ty - 3 + r, r_lo), r_hi), x = min(max(po_x + tx - 3 + c, c_lo), c_hi);
    sp[r][c] = (uint16_t)in[(long long)y * is + x];
  }
}

// the radius-1 (every row -1 .. kT) and radius-2 (odd rows -1, 1, .. kT - 1) box sums and sums of squares
__device__ __forceinline__ void sgr_box_sums(const uint16_t (*sp)[kSP], uint32_t (*box1)[kAB][kAB],
                                             uint32_t (*box2)[kR2][kAB]) {
  for (int i = threadIdx.x; i < kAB * kAB; i += kThreads) {
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
  for (int i = threadIdx.x; i < kR2 * kAB; i += kThreads) {
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
}

// one set's a / b values from the box sums (sgrproj_box_ab_internal)
__device__ __forceinline__ void sgr_ab(const uint32_t (*box1)[kAB][kAB], const uint32_t (*box2)[kR2][kAB],
                                       uint32_t (*a1)[kAB], uint32_t (*b1)[kAB], uint32_t (*a2)[kAB],
                                       uint32_t (*b2)[kAB], uint32_t s1, uint32_t s2, int bdm8) {
  if (s1)
    for (int i = threadIdx.x; i < kAB * kAB; i += kThreads) {
      const int j = i / kAB, m = i - j * kAB;
      sum_finish(box1[1][j][m], box1[0][j][m], 9, 455, s1, bdm8, a1[j][m], b1[j][m]);
    }
  if (s2)
    for (int i = threadIdx.x; i < kR2 * kAB; i += kThreads) {
      const int j = i / kAB, m = i - j * kAB;
      sum_finish(box2[1][j][m], box2[0][j][m], 25, 164, s2, bdm8, a2[j][m], b2[j][m]);
    }
}

// the two filter outputs f1 / f2 of tile pixel (y, x) (sgrproj_box_f_r0 / r1 / r2), and the pixel itself
__device__ __forceinline__ uint32_t sgr_f(const uint16_t (*sp)[kSP], const uint32_t (*a1)[kAB],
                                          const uint32_t (*b1)[kAB], const uint32_t (*a2)[kAB],
                                          const uint32_t (*b2)[kAB], uint32_t s1, uint32_t s2, int y, int x,
                                          uint32_t &f1, uint32_t &f2) {
  const uint32_t px = sp[y + 3][x + 3];
  f1 = px << 4;
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
  return px;
}

// apply_filter (lrf.rs:796-815)
__device__ __forceinline__ uint16_t sgr_apply(int w0, int w1, int w2, uint32_t f1, uint32_t f2, uint32_t px, int bd) {
  const int v = w0 * (int)f2 + w1 * (int)(px << 4) + w2 * (int)f1;
  return (uint16_t)min(max((v + (1 << 10)) >> 11, 0), (1 << bd) - 1);
}

// a unit's geometry in its plane's pixels (rdo.rs:2651-2658; the area's scratch rect, rdo.rs:2152-2157);
// the unit is inside its area when lru_x * lru_sb_w < sb_w and likewise vertically
inline Geo lrf_unit_geo(const b200_cdef_rdo_area &r, int p, int xd, int yd, int us, int lru_x, int lru_y,
                        int frame_width, int frame_height) {
  Geo g;
  const int lsw = (us << xd) / 64, lsh = (us << yd) / 64;
  g.ax = (r.sbx * 64) >> xd, g.ay = (r.sby * 64) >> yd;
  const int crop_w = frame_width - r.sbx * 64, crop_h = frame_height - r.sby * 64;
  g.po_x = (lru_x * lsw * 64) >> xd, g.po_y = (lru_y * lsh * 64) >> yd;
  g.vis_w = std::min(us, (crop_w >> xd) - g.po_x), g.vis_h = std::min(us, (crop_h >> yd) - g.po_y);
  const int aw = (std::min(crop_w, r.sb_w * 64) + 7) & ~7, ah = (std::min(crop_h, r.sb_h * 64) + 7) & ~7;
  g.ew = std::min(us, (aw >> xd) - g.po_x), g.eh = std::min(us, (ah >> yd) - g.po_y);
  g.gbx0 = r.sbx * 8 + lru_x * lsw * 8, g.gby0 = r.sby * 8 + lru_y * lsh * 8;
  g.p = p, g.xd = xd, g.yd = yd;
  return g;
}

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
template <typename Rec>  // b200_lrf_search_item or b200_loop_unit
__device__ uint32_t lrf_rate(const Rec &it, int type, int set, int x0, int x1) {
  if (type == 0) return it.none_bits;
  uint32_t bits = it.sgr_bits + (4u << 3);
  if (kSgrS[set][0]) bits += count_signed_subexp_with_ref(x0, -96, 32, 4, it.sgrproj_ref[0]);
  if (kSgrS[set][1]) bits += count_signed_subexp_with_ref(x1, -32, 96, 4, it.sgrproj_ref[1]);
  return bits;
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
