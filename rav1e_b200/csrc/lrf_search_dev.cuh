// lrf_search_dev.cuh — what the restoration search (rav1e src/rdo.rs:2575-2740) shares between its two
// callers, b200_lrf_search_dev and the L stage of b200_loop_decision_dev's pass loop: the argument types and
// lrf_search_launch (its kernels and launch sequence are in lrf_search.cu), the per-item host set-up, and the
// pieces the pass loop's C stage also runs for its Sgrproj branch: the self-guided tile steps (staging through
// setup_integral_image's clip rule, box sums, a / b, the two filter outputs) and lrf_rate.
#pragma once
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

}  // namespace

// named, because lrf_search_launch is called from two translation units
namespace lrf_search {

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

// Zeroes a.acc / a.err (n_items x 16 x 5 and n_items x kCands) and makes the search's four launches on the
// context's stream: the tile statistics, the solve, the tile errors and the decision.  On a failed memset it
// returns s.finish(false).
int lrf_search_launch(b200_ctx *ctx, HostStage &s, const SearchArgs &a);

}  // namespace lrf_search

namespace {

using lrf_search::Geo;
using lrf_search::SearchArgs;
using lrf_search::Tile;

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

// the SearchArgs fields both callers fill alike; `in` is the plane list the units are filtered from
inline SearchArgs search_args(const b200_plane *in, const b200_plane *src, int planes, int xdec, int ydec,
                              int bit_depth, int frame_width, int reduced_sets, const uint32_t *d_imp_scales,
                              const uint32_t dist_scale[3], double lambda) {
  SearchArgs a{};
  for (int p = 0; p < planes; p++) {
    a.in[p] = PlaneView{in[p].data, in[p].stride};
    a.src[p] = PlaneView{src[p].data, src[p].stride};
    a.dist_scale[p] = dist_scale[p];
  }
  a.xdec = xdec, a.ydec = ydec, a.bit_depth = bit_depth, a.w8 = (frame_width + 7) >> 3;
  a.reduced = reduced_sets != 0;
  a.nsets = a.reduced ? 8 : 16;
  a.imp = d_imp_scales;
  a.lambda = lambda;
  return a;
}

// Unit (lru_x, lru_y) of plane p in area r, item or unit `i` of the call: its geometry in the plane's pixels
// (rdo.rs:2651-2658; the area's scratch rect, rdo.rs:2152-2157).  Rejects a unit outside its area or the
// visible frame.
inline int lrf_item_geo(b200_ctx *ctx, size_t i, const b200_cdef_rdo_area &r, int p, int xdec, int ydec, int us,
                        int lru_x, int lru_y, int frame_width, int frame_height, Geo &g) {
  const int xd = p ? xdec : 0, yd = p ? ydec : 0;
  const int lsw = (us << xd) / 64, lsh = (us << yd) / 64;
  B200_REQUIRE(ctx, lru_x >= 0 && lru_y >= 0 && lru_x * lsw < r.sb_w && lru_y * lsh < r.sb_h,
               "unit %zu: (%d, %d) outside its %dx%d area", i, lru_x, lru_y, r.sb_w, r.sb_h);
  g.ax = (r.sbx * 64) >> xd, g.ay = (r.sby * 64) >> yd;
  const int crop_w = frame_width - r.sbx * 64, crop_h = frame_height - r.sby * 64;
  g.po_x = (lru_x * lsw * 64) >> xd, g.po_y = (lru_y * lsh * 64) >> yd;
  g.vis_w = std::min(us, (crop_w >> xd) - g.po_x), g.vis_h = std::min(us, (crop_h >> yd) - g.po_y);
  const int aw = (std::min(crop_w, r.sb_w * 64) + 7) & ~7, ah = (std::min(crop_h, r.sb_h * 64) + 7) & ~7;
  g.ew = std::min(us, (aw >> xd) - g.po_x), g.eh = std::min(us, (ah >> yd) - g.po_y);
  g.gbx0 = r.sbx * 8 + lru_x * lsw * 8, g.gby0 = r.sby * 8 + lru_y * lsh * 8;
  g.p = p, g.xd = xd, g.yd = yd;
  B200_REQUIRE(ctx, g.vis_w > 0 && g.vis_h > 0, "unit %zu: (%d, %d) outside the visible frame", i, lru_x, lru_y);
  return B200_OK;
}

// the 32x32 tiles of item `item`'s unit, over its 8x8 blocks inside the area
inline void lrf_item_tiles(const Geo &g, uint32_t item, std::vector<Tile> &tiles) {
  for (int ty = 0; ty < g.eh; ty += kT)
    for (int tx = 0; tx < g.ew; tx += kT) tiles.push_back(Tile{item, (uint16_t)tx, (uint16_t)ty});
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

}  // namespace
