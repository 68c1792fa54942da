// lrf.cu — loop restoration's frame filter (rav1e RestorationState::lrf_filter_frame, src/lrf.rs:1482-1585):
// Wiener (wiener_stripe_filter, :1099-1207) and self-guided (setup_integral_image + sgrproj_stripe_filter,
// :529-830) units over whole frames, reading the CDEF output and the deblocked frame.
//
// One 128-thread CTA per tile of (plane, stripe, 32-column span).  Units start at multiples of their size
// (>= 32), so a span lies inside one unit and the filter type is uniform over the CTA.  An output pixel
// depends only on its unit's record and on at most 3 rows and columns around it, read through the
// stripe's source rule, so the tile stages its rows plus a 3-pixel halo into shared memory once, with the
// rule applied there (Wiener's and self-guided's rules differ only at the frame's top and bottom), and the
// filters then run on shared memory with no boundary branches.
//  - Wiener: the horizontal pass writes the i16 intermediate (it fits at every bit depth) for the tile's
//    rows plus 3 above and below, then the vertical pass writes the output.
//  - Self-guided: the radius-2 a / b values on the stripe's odd rows, then (reusing the buffer) the
//    radius-1 values on every row, are formed from direct box sums of the staged pixels.  The true 5x5
//    sum of squares at 12 bit (25 * 4095^2) fits in u32, so a direct sum equals the reference's wrapping
//    integral-image difference.  Each thread keeps its pixels' radius-2 filter output in registers while
//    the radius-1 values are formed.
// Warp w owns rows w, w + 4, ... of the tile and lane l column l, so stores are row-contiguous.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "host_stage.cuh"
#include "loop_filter_checks.cuh"
#include "lrf_dev.cuh"

namespace {

constexpr int kTW = 32;                 // tile columns
constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kRowsPerWarp = 64 / kWarps;
constexpr int kMaxRows = 64 + 6;        // staged rows: a stripe plus 3 above and below
constexpr int kSW = kTW + 6;            // staged columns: the span plus 3 left and right
constexpr int kAbRows = 64 + 2;         // radius-1 a / b rows: -1 .. 64
constexpr int kAbCols = kTW + 2;        // a / b columns: -1 .. kTW

struct LrfArgs {
  PlaneView cdef[3], deb[3], out[3];
  int cw[3], ch[3], yd[3];       // crop and vertical decimation per plane
  int unit[3], cols[3], rows[3]; // unit grid per plane
  int stripe_h[3];               // RestorationPlaneConfig::stripe_height: 32 for 4:2:0 chroma, else 64
  int ntx[3];                    // 32-column spans per stripe
  uint32_t tile0[4];             // first tile of each plane
  const b200_lrf_unit *units[3];
  int bit_depth, enable_cdef;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) lrf_filter_kernel(const LrfArgs a) {
  __shared__ uint16_t sp[kMaxRows][kSW];
  __shared__ union {
    struct {
      uint32_t A[kAbRows][kAbCols], B[kAbRows][kAbCols];
    } ab;
    int16_t w[kMaxRows][kTW];
  } u;

  const uint32_t b = blockIdx.x;
  const int p = b >= a.tile0[2] ? 2 : b >= a.tile0[1] ? 1 : 0;
  const uint32_t t = b - a.tile0[p];
  const int si = (int)(t / (uint32_t)a.ntx[p]), x0 = (int)(t % (uint32_t)a.ntx[p]) * kTW;
  const int yd = a.yd[p], cw = a.cw[p], ch = a.ch[p];
  // lrf_filter_frame's stripes (lrf.rs:1509-1519): stripe 0 is not clipped to the crop
  const int sy = si == 0 ? 0 : (si * 64 - 8) >> yd;
  const int sh = si == 0 ? 56 >> yd : min(64 >> yd, ch - sy);
  const int nout = min(sh, ch - sy);  // rows written: the crop only
  const int tw = min(kTW, cw - x0);
  // restoration_unit_by_stripe (lrf.rs:1295-1312)
  const int us = a.unit[p];
  const int ruy = min(si * a.stripe_h[p] / us, a.rows[p] - 1), rux = min(x0 / us, a.cols[p] - 1);
  const b200_lrf_unit un = a.units[p][ruy * a.cols[p] + rux];
  const int type = (un.type == 2 && !a.enable_cdef) ? 0 : un.type;  // lrf.rs:1545-1547

  const T *cdef = (const T *)a.cdef[p].data, *deb = (const T *)a.deb[p].data;
  const int cs = a.cdef[p].stride, ds = a.deb[p].stride, os = a.out[p].stride;
  T *out = (T *)a.out[p].data;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x = x0 + lane;

  if (type == 0) {
    for (int y = warp; y < nout; y += kWarps)
      if (lane < tw) out[(long long)(sy + y) * os + x] = cdef[(long long)(sy + y) * cs + x];
    return;
  }

  // Stage rows sy - 3 .. sy + nout + 2 and columns x0 - 3 .. x0 + kTW + 2 through the source rule.
  const int nr = nout + 6;
  const int sh2 = sh + (sh & 1);  // VertPaddedIter's stripe end: the height rounded up to even
  for (int i = threadIdx.x; i < nr * kSW; i += kThreads) {
    const int r = i / kSW, c = i - r * kSW;
    const int yi = sy - 3 + r, xi = min(max(x0 - 3 + c, 0), cw - 1);
    const int cy = min(max(yi, 0), ch - 1);
    int ly;
    bool from_cdef;
    if (type == 1) {  // wiener_stripe_filter (lrf.rs:1157-1169)
      from_cdef = yi >= sy && yi < sy + sh;
      ly = yi < sy ? max(cy, sy - 2) : from_cdef ? cy : min(cy, sy + sh + 1);
    } else {  // VertPaddedIter (lrf.rs:446-467)
      ly = min(max(cy, sy - 2), sy + sh2 + 1);
      from_cdef = ly >= sy && ly < sy + sh2;
    }
    sp[r][c] = from_cdef ? cdef[(long long)ly * cs + xi] : deb[(long long)ly * ds + xi];
  }
  __syncthreads();

  const int bd = a.bit_depth, pmax = (1 << bd) - 1;
  if (type == 1) {
    int hf[7], vf[7];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      vf[k] = vf[6 - k] = un.coeffs[0][k];
      hf[k] = hf[6 - k] = un.coeffs[1][k];
    }
    vf[3] = 128 - 2 * (vf[0] + vf[1] + vf[2]);
    hf[3] = 128 - 2 * (hf[0] + hf[1] + hf[2]);
    const int round_h = bd == 12 ? 5 : 3, round_v = bd == 12 ? 9 : 11;
    const int offset = 1 << (bd + 7 - round_h - 1), limit = (1 << (bd + 1 + 7 - round_h)) - 1;
    for (int r = warp; r < nr; r += kWarps) {
      int acc = 0;
#pragma unroll
      for (int k = 0; k < 7; k++) acc += hf[k] * sp[r][lane + k];
      acc = (acc + (1 << round_h >> 1)) >> round_h;
      u.w[r][lane] = (int16_t)min(max(acc, -offset), limit - offset);
    }
    __syncthreads();
    for (int y = warp; y < nout; y += kWarps) {
      int acc = 0;
#pragma unroll
      for (int k = 0; k < 7; k++) acc += vf[k] * u.w[y + k][lane];
      if (lane < tw) out[(long long)(sy + y) * os + x] = (T)min(max((acc + (1 << round_v >> 1)) >> round_v, 0), pmax);
    }
    return;
  }

  // self-guided (sgrproj_stripe_filter, lrf.rs:629-830)
  const int bdm8 = bd - 8;
  const uint32_t s2 = kSgrS[un.set][0], s1 = kSgrS[un.set][1];
  uint32_t f2[kRowsPerWarp];
  if (s2) {
    // a / b row j sits on stripe row 2j - 1 (lrf.rs:665-668: only every other row is used)
    const int n2 = (nout + 1) / 2 + 1;
    for (int i = threadIdx.x; i < n2 * kAbCols; i += kThreads) {
      const int j = i / kAbCols, m = i - j * kAbCols;
      uint32_t sum = 0, ssq = 0;
#pragma unroll
      for (int dy = 0; dy < 5; dy++)
#pragma unroll
        for (int dx = 0; dx < 5; dx++) {
          const uint32_t v = sp[2 * j + dy][m + dx];
          sum += v;
          ssq += v * v;
        }
      sum_finish(ssq, sum, 25, 164, s2, bdm8, u.ab.A[j][m], u.ab.B[j][m]);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kRowsPerWarp; k++) {
      const int y = warp + kWarps * k;
      if (y >= nout) break;
      const uint32_t px = sp[y + 3][lane + 3];
      // sgrproj_box_f_r2 (lrf.rs:300-342): even rows weigh rows y - 1 and y + 1, odd rows their own
      const int j = (y + 1) >> 1;
      uint32_t av = r2_row(u.ab.A[j], lane);
      uint32_t bv = r2_row(u.ab.B[j], lane);
      if (y & 1) {
        f2[k] = (av * px + bv + (1u << 7)) >> 8;
      } else {
        av += r2_row(u.ab.A[j + 1], lane);
        bv += r2_row(u.ab.B[j + 1], lane);
        f2[k] = (av * px + bv + (1u << 8)) >> 9;
      }
    }
    if (s1) __syncthreads();  // the radius-1 values reuse the buffer
  } else {
    // sgrproj_box_f_r0 of the even row, shared by the odd row below it (lrf.rs:740-749)
#pragma unroll
    for (int k = 0; k < kRowsPerWarp; k++) {
      const int y = warp + kWarps * k;
      if (y >= nout) break;
      f2[k] = (uint32_t)sp[(y & ~1) + 3][lane + 3] << 4;
    }
  }
  if (s1) {
    // a / b row j sits on stripe row j - 1
    for (int i = threadIdx.x; i < (nout + 2) * kAbCols; i += kThreads) {
      const int j = i / kAbCols, m = i - j * kAbCols;
      uint32_t sum = 0, ssq = 0;
#pragma unroll
      for (int dy = 0; dy < 3; dy++)
#pragma unroll
        for (int dx = 0; dx < 3; dx++) {
          const uint32_t v = sp[j + 1 + dy][m + 1 + dx];
          sum += v;
          ssq += v * v;
        }
      sum_finish(ssq, sum, 9, 455, s1, bdm8, u.ab.A[j][m], u.ab.B[j][m]);
    }
    __syncthreads();
  }
  const int w0 = un.xqd[0], w1 = un.xqd[1], w2 = 128 - w0 - w1;
#pragma unroll
  for (int k = 0; k < kRowsPerWarp; k++) {
    const int y = warp + kWarps * k;
    if (y >= nout) break;
    const uint32_t px = sp[y + 3][lane + 3];
    uint32_t f1 = px << 4;
    if (s1) {  // sgrproj_box_f_r1 (lrf.rs:266-291)
      const uint32_t av = r1_weigh(u.ab.A, y, lane), bv = r1_weigh(u.ab.B, y, lane);
      f1 = (av * px + bv + (1u << 8)) >> 9;
    }
    // apply_filter (lrf.rs:796-815)
    const int v = w0 * (int)f2[k] + w1 * (int)(px << 4) + w2 * (int)f1;
    if (lane < tw) out[(long long)(sy + y) * os + x] = (T)min(max((v + (1 << 10)) >> 11, 0), pmax);
  }
}

// bytes [lo, hi) a plane's crop rect spans
struct Span {
  uintptr_t lo, hi;
};
Span crop_span(const b200_plane &pl, long long cw, long long ch) {
  const uintptr_t lo = (uintptr_t)pl.data;
  return Span{lo, lo + (uintptr_t)(((ch - 1) * pl.stride + cw) * pl.bpp)};
}

// A record's ranges (lrf.rs:39-48), for the fields of its own type
int check_unit(b200_ctx *ctx, const b200_lrf_unit &r, int p, size_t i) {
  static const int kTapMin[3] = {-5, -23, -17}, kTapMax[3] = {10, 8, 46};
  B200_REQUIRE(ctx, r.type <= 2, "plane %d unit %zu: type %d", p, i, r.type);
  if (r.type == 2) {
    B200_REQUIRE(ctx, r.set <= 15, "plane %d unit %zu: sgrproj set %d", p, i, r.set);
    B200_REQUIRE(ctx, sgrproj_xqd_ok(r.xqd[0], r.xqd[1]), "plane %d unit %zu: xqd (%d, %d) out of range", p, i,
                 r.xqd[0], r.xqd[1]);
  } else if (r.type == 1) {
    for (int d = 0; d < 2; d++)
      for (int k = 0; k < 3; k++)
        B200_REQUIRE(ctx, r.coeffs[d][k] >= kTapMin[k] && r.coeffs[d][k] <= kTapMax[k],
                     "plane %d unit %zu: wiener tap [%d][%d] = %d out of range", p, i, d, k, r.coeffs[d][k]);
  }
  return B200_OK;
}

}  // namespace

extern "C" int b200_lrf_filter_dev(b200_ctx *ctx, const b200_plane *cdeffed, const b200_plane *deblocked,
                                   const b200_plane *out, int planes, int xdec, int ydec, int frame_width,
                                   int frame_height, int bit_depth, int enable_cdef, const int unit_size[3],
                                   const b200_lrf_unit *const units[3]) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cdeffed && deblocked && out && unit_size && units, "NULL planes / unit_size / units");
  B200_REQUIRE(ctx, planes == 1 || planes == 3, "planes must be 1 or 3, got %d", planes);
  B200_REQUIRE(ctx, (xdec == 1 && ydec == 1) || (xdec == 1 && ydec == 0) || (xdec == 0 && ydec == 0),
               "chroma layout (xdec %d, ydec %d) is not 4:2:0, 4:2:2 or 4:4:4", xdec, ydec);
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  // enable_restoration_filters (encoder.rs:232)
  B200_REQUIRE(ctx, frame_width >= 32 && frame_height >= 32, "frame %dx%d is under 32x32", frame_width,
               frame_height);
  const int bpp = bit_depth == 8 ? 1 : 2;
  LrfArgs a{};
  size_t total_units = 0;
  long long cwv[3], chv[3];
  uint32_t tiles = 0;
  for (int p = 0; p < planes; p++) {
    const int xd = p ? xdec : 0, yd = p ? ydec : 0;
    const long long cw = ((long long)frame_width + (1 << xd >> 1)) >> xd;
    const long long ch = ((long long)frame_height + (1 << yd >> 1)) >> yd;
    cwv[p] = cw, chv[p] = ch;
    B200_REQUIRE(ctx, lrf_unit_size_ok(unit_size[p]), "plane %d: unit size %d is not a power of two in 32..256", p,
                 unit_size[p]);
    B200_REQUIRE(ctx, units[p] != nullptr, "NULL units for plane %d", p);
    for (const b200_plane *pl : {cdeffed, deblocked, out}) {
      B200_REQUIRE(ctx, pl[p].data != nullptr, "NULL plane %d", p);
      B200_REQUIRE(ctx, pl[p].bpp == bpp, "plane %d: bpp %d does not match bit depth %d", p, pl[p].bpp, bit_depth);
      B200_REQUIRE(ctx, pl[p].width >= cw && pl[p].height >= ch && pl[p].stride >= pl[p].width,
                   "plane %d: %dx%d (stride %d) is smaller than the %lldx%lld crop", p, pl[p].width, pl[p].height,
                   pl[p].stride, cw, ch);
    }
    const int us = unit_size[p];
    const int cols = (int)std::max(1LL, (cw + (us >> 1)) / us), rows = (int)std::max(1LL, (ch + (us >> 1)) / us);
    for (size_t i = 0; i < (size_t)cols * rows; i++)
      if (int st = check_unit(ctx, units[p][i], p, i)) return st;
    a.cdef[p] = PlaneView{cdeffed[p].data, cdeffed[p].stride};
    a.deb[p] = PlaneView{deblocked[p].data, deblocked[p].stride};
    a.out[p] = PlaneView{out[p].data, out[p].stride};
    a.cw[p] = (int)cw, a.ch[p] = (int)ch, a.yd[p] = yd;
    a.unit[p] = us, a.cols[p] = cols, a.rows[p] = rows;
    a.stripe_h[p] = (p && xdec && ydec) ? 32 : 64;
    a.ntx[p] = (int)((cw + kTW - 1) / kTW);
    a.tile0[p] = tiles;
    tiles += (uint32_t)(((long long)frame_height + 7) / 64 + 1) * (uint32_t)a.ntx[p];
    total_units += (size_t)cols * rows;
  }
  for (int p = planes; p < 4; p++) a.tile0[p] = tiles;
  for (int p = 0; p < planes; p++)
    for (int q = 0; q < planes; q++)
      for (const b200_plane *in : {cdeffed, deblocked}) {
        const Span o = crop_span(out[p], cwv[p], chv[p]), s = crop_span(in[q], cwv[q], chv[q]);
        B200_REQUIRE(ctx, o.hi <= s.lo || s.hi <= o.lo, "out plane %d overlaps input plane %d", p, q);
      }
  a.bit_depth = bit_depth;
  a.enable_cdef = enable_cdef != 0;

  // every plane's records in one upload; a copy from pageable memory has left `packed` when it returns
  std::vector<b200_lrf_unit> packed;
  packed.reserve(total_units);
  size_t first[3] = {0, 0, 0};
  for (int p = 0; p < planes; p++) {
    first[p] = packed.size();
    packed.insert(packed.end(), units[p], units[p] + (size_t)a.cols[p] * a.rows[p]);
  }
  const size_t bytes = packed.size() * sizeof(b200_lrf_unit);
  HostStage s(ctx, bytes);
  b200_lrf_unit *d_units = (b200_lrf_unit *)s.take(bytes);
  s.up(d_units, packed.data(), bytes);
  if (!s.ok()) return s.finish(false);
  for (int p = 0; p < planes; p++) a.units[p] = d_units + first[p];
  if (bit_depth > 8) lrf_filter_kernel<uint16_t><<<tiles, kThreads, 0, ctx->stream>>>(a);
  else lrf_filter_kernel<uint8_t><<<tiles, kThreads, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return s.finish(false);
}
