// cdef_rdo.cu — the CDEF pass of rdo_loop_decision (rav1e src/rdo.rs:2104-2567, RestorationFilter::None
// and no-LRU branches) for many loop-restoration areas in one call: for every superblock of every area,
// every cdef index 0 .. 1 << cdef_bits is filtered (cdef_filter_superblock, cdef.rs:401-570), measured
// (rdo_loop_plane_error, rdo.rs:2027-2093) and costed (compute_rd_cost, rdo.rs:718-723); the first
// minimum wins and, on request, the winner's pixels are written.
//
// One CTA of 256 threads per area superblock.  The superblock's tiles of `rec` (+ 2-pixel halo) are
// staged once per plane as int16 with the CDEF_VERY_LARGE sentinel wherever the reference's scratch
// copy of the AREA (rdo.rs:2277-2284, plane_region.rs:390-401) has no pixel: availability is relative
// to the area, not to the frame or tile.  The source blocks are staged once, the 64 directions and
// variances are computed in shared memory, and each index is filtered into registers and reduced to
// integer sums right away: four threads own one 8x8 luma block (a 4x4 quarter each) and the matching
// chroma block.  Only distortions, costs, the winner and the winner's pixels leave the chip.
#include <algorithm>
#include <vector>

#include "cdef_dev.cuh"
#include "rdo_dist_dev.cuh"

namespace {

constexpr int kRdoThreads = 256;
constexpr int kRdoMaxAreas = 256;   // areas per launch (kernel-parameter table)
constexpr int kRdoMaxSlots = 1024;  // superblocks per launch
constexpr int kLumaPitch = 70;      // 68 staged columns; rows 35 words apart -> odd bank shift

struct CdefRdoArgs {
  PlaneView rec[3], src[3];
  void *out[3];
  int out_stride[3];
  int planes, width, height, w8, bit_depth, damping, nidx;
  uint8_t ystr[8], uvstr[8];
  const uint8_t *skip8;
  const uint32_t *imp;
  uint32_t dist_scale[3];
  double lambda;
  const uint32_t *rate;
  unsigned long long *err;
  double *cost;
  int8_t *best;
};

// The areas and superblocks of one launch.  slot[k] = local area index << 4 | sby << 2 | sbx.
struct CdefRdoSlots {
  uint32_t area0;  // index of local area 0 in the caller's array
  uint16_t ax[kRdoMaxAreas], ay[kRdoMaxAreas];
  uint8_t wh[kRdoMaxAreas];  // sb_w | sb_h << 4
  uint16_t slot[kRdoMaxSlots];
};
static_assert(sizeof(CdefRdoArgs) + sizeof(CdefRdoSlots) <= 4096, "kernel parameters over 4 KB");

template <int XDEC, int YDEC>
struct RdoLayout {
  static constexpr int CW = 64 >> XDEC, CH = 64 >> YDEC;  // chroma superblock
  static constexpr int CP = CW + 6;                       // chroma tile pitch
  static constexpr int LT = 68 * kLumaPitch, CT = (CH + 4) * CP;
  // shorts: luma tile, 2 chroma tiles, luma source, 2 chroma sources
  static constexpr int SHORTS = LT + 2 * CT + 64 * 64 + 2 * CW * CH;
  static constexpr size_t BYTES = SHORTS * 2 + 64 * (4 + 4 + 1 + 1) + 8 * 3 * 8 + 16;
};

template <typename T, int XDEC, int YDEC>
__global__ void __launch_bounds__(kRdoThreads, 2)
    cdef_rdo_kernel(const __grid_constant__ CdefRdoArgs A, const __grid_constant__ CdefRdoSlots S) {
  using L = RdoLayout<XDEC, YDEC>;
  constexpr int CW8 = 8 >> XDEC, CH8 = 8 >> YDEC;  // chroma block of one 8x8 luma block
  constexpr int CROWS = CW8 * CH8 / 16;            // rows of 4 pixels per thread: 4 / 2 / 1
  constexpr int LPC = 4 / (CW8 * CH8 / 16);        // lanes per 4x4 chunk: 1 / 2 / 4
  extern __shared__ __align__(16) unsigned char smem[];
  short *lt = (short *)smem;
  short *ct[2] = {lt + L::LT, lt + L::LT + L::CT};
  short *ls = lt + L::LT + 2 * L::CT;
  short *cs[2] = {ls + 64 * 64, ls + 64 * 64 + L::CW * L::CH};
  int *s_var = (int *)(smem + L::SHORTS * 2);
  uint32_t *s_bias = (uint32_t *)(s_var + 64);
  uint8_t *s_dir = (uint8_t *)(s_bias + 64);
  uint8_t *s_skip = s_dir + 64;
  unsigned long long *s_red = (unsigned long long *)(s_skip + 64);  // [8 warps][3 planes]
  int *s_best = (int *)(s_red + 24);

  const int t = threadIdx.x;
  const uint32_t e = S.slot[blockIdx.x];
  const int la = e >> 4, sbx = e & 3, sby = (e >> 2) & 3;
  const int ax = S.ax[la] * 64, ay = S.ay[la] * 64;  // area origin, luma px
  const int sb_w = S.wh[la] & 15, sb_h = S.wh[la] >> 4;
  const size_t slot = (size_t)(S.area0 + la) * 16 + (e & 15);
  // the scratch copy: the area cropped to the visible frame, rounded up to 8 (rdo.rs:2152-2157, 2281-2282)
  const int wa = (min(A.width - ax, sb_w * 64) + 7) & ~7, ha = (min(A.height - ay, sb_h * 64) + 7) & ~7;
  const int x0 = sbx * 64, y0 = sby * 64;                                   // superblock, area-relative
  const int bw8 = min(64, wa - x0) >> 3, bh8 = min(64, ha - y0) >> 3;      // blocks in range (rdo.rs:2042)
  const int coeff_shift = A.bit_depth - 8;

  // ---- skip flags and 8x8 distortion biases (distortion_scale, rdo.rs:443-462, frame-absolute)
  int coded_blk = 0;
  if (t < 64) {
    const int bx = t & 7, by = t >> 3;
    const bool inr = bx < bw8 && by < bh8;
    const size_t gb = (size_t)(((ay + y0) >> 3) + by) * A.w8 + ((ax + x0) >> 3) + bx;
    const bool sk = !inr || (A.skip8 && A.skip8[gb]);
    s_skip[t] = sk;
    s_bias[t] = inr && A.imp ? A.imp[gb] : (1u << 14);
    coded_blk = !sk;
  }
  const int coded = __syncthreads_or(coded_blk);  // rdo.rs:2185-2205: an all-skip superblock gets no decision

  // ---- stage rec (+ halo, sentinel outside the area) and src
#pragma unroll
  for (int p = 0; p < 3; p++) {
    if (p >= A.planes) break;
    const int xd = p ? XDEC : 0, yd = p ? YDEC : 0;
    const int tw = (64 >> xd) + 4, th = (64 >> yd) + 4, pitch = p ? L::CP : kLumaPitch;
    const int aw = wa >> xd, ah = ha >> yd, sx = x0 >> xd, sy = y0 >> yd;
    const T *rp = (const T *)A.rec[p].data + (long long)(ay >> yd) * A.rec[p].stride + (ax >> xd);
    short *tile = p ? ct[p - 1] : lt;
    for (int i = t; i < tw * th; i += kRdoThreads) {
      const int r = i / tw, c = i - r * tw;
      const int x = sx + c - 2, y = sy + r - 2;
      short v = (short)0x8000;
      if (x >= 0 && x < aw && y >= 0 && y < ah) v = (short)rp[(long long)y * A.rec[p].stride + x];
      tile[r * pitch + c] = v;
    }
    if (coded) {
      const T *sp = (const T *)A.src[p].data + (long long)(ay >> yd) * A.src[p].stride + (ax >> xd);
      short *dst = p ? cs[p - 1] : ls;
      const int sw = 64 >> xd, sh = 64 >> yd;
      for (int i = t; i < sw * sh; i += kRdoThreads) {
        const int r = i / sw, c = i - r * sw;
        const int x = sx + c, y = sy + r;
        dst[i] = x < aw && y < ah ? (short)sp[(long long)y * A.src[p].stride + x] : (short)0;
      }
    }
  }
  __syncthreads();
  // ---- directions and variances (cdef_analyze_superblock, cdef.rs:340-374)
  if (t < 64) {
    unsigned v = 0;
    int d = 0;
    if (!s_skip[t]) d = find_dir_8x8<short>(lt + (2 + 8 * (t >> 3)) * kLumaPitch + 2 + 8 * (t & 7), kLumaPitch, coeff_shift, &v);
    s_dir[t] = (uint8_t)d;
    s_var[t] = (int)v;
  }
  __syncthreads();

  // ---- four threads per 8x8 block: a 4x4 quarter of luma, CROWS rows of 4 chroma pixels each
  const int b = t >> 2, q = t & 3, bx = b & 7, by = b >> 3;
  const bool inr = bx < bw8 && by < bh8;
  const bool sk = s_skip[b];
  const int lx = 8 * bx + 4 * (q & 1), ly = 8 * by + 4 * (q >> 1);
  const int cx = CW8 * bx + (XDEC ? 0 : 4 * (q & 1)), cy = CH8 * by + (XDEC ? q * CROWS : 4 * (q >> 1));
  const int warp = t >> 5, lane = t & 31;

  int best = -1;
  double best_cost = -1.;
  for (int i = 0; i < A.nidx && coded; i++) {
    unsigned long long acc[3] = {0, 0, 0};
    {  // luma: cdef_dist_kernel(src, test, 8, 8) * bias
      const CdefBlockTaps tp = cdef_block_taps(A.ystr + i, 0, XDEC, YDEC, s_dir, s_var, b, A.damping, coeff_shift,
                                               kLumaPitch);
      uint32_t ss = 0, sd = 0, ss2 = 0, sd2 = 0, ssd = 0;
#pragma unroll
      for (int r = 0; r < 4; r++)
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const short *ctr = lt + (2 + ly + r) * kLumaPitch + 2 + lx + c;
          const uint32_t d = (uint32_t)(sk ? (int)ctr[0] : cdef_filter_tile_px(ctr, tp));
          const uint32_t s = (uint32_t)ls[(ly + r) * 64 + lx + c];
          ss += s, sd += d, ss2 += s * s, sd2 += d * d, ssd += s * d;
        }
#pragma unroll
      for (int o = 1; o < 4; o <<= 1) {
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
        sd += __shfl_xor_sync(0xffffffffu, sd, o);
        ss2 += __shfl_xor_sync(0xffffffffu, ss2, o);
        sd2 += __shfl_xor_sync(0xffffffffu, sd2, o);
        ssd += __shfl_xor_sync(0xffffffffu, ssd, o);
      }
      uint32_t svar, dvar;
      const uint32_t sse = cdef_dist_vars(ss, sd, ss2, sd2, ssd, 64, &svar, &dvar);
      const uint32_t dist = apply_ssim_boost(sse, svar, dvar, A.bit_depth);
      if (q == 0 && inr) acc[0] = ((unsigned long long)s_bias[b] * dist + (1u << 13)) >> 14;  // mul_u64
    }
#pragma unroll
    for (int p = 1; p < 3; p++) {  // chroma: sse_wxh(8 >> xdec, 8 >> ydec) with the bias per chunk
      if (p >= A.planes) break;
      const short *tile = ct[p - 1], *src = cs[p - 1];
      const CdefBlockTaps tp = cdef_block_taps(A.uvstr + i, p, XDEC, YDEC, s_dir, s_var, b, A.damping, coeff_shift,
                                               L::CP);
      uint32_t sse = 0;
#pragma unroll
      for (int r = 0; r < CROWS; r++)
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const short *ctr = tile + (2 + cy + r) * L::CP + 2 + cx + c;
          const int d = sk ? (int)ctr[0] : cdef_filter_tile_px(ctr, tp);
          const int df = d - (int)src[(cy + r) * L::CW + cx + c];
          sse += (uint32_t)(df * df);
        }
      if (LPC >= 2) sse += __shfl_xor_sync(0xffffffffu, sse, 1);
      if (LPC == 4) sse += __shfl_xor_sync(0xffffffffu, sse, 2);
      unsigned long long term = (q % LPC) == 0 ? wsse_chunk(sse, s_bias[b]) : 0ull;
      term += __shfl_xor_sync(0xffffffffu, term, 1);
      term += __shfl_xor_sync(0xffffffffu, term, 2);
      if (q == 0 && inr) acc[p] = wsse_finish(term);
    }
    // ---- per-plane sums over the superblock
#pragma unroll
    for (int p = 0; p < 3; p++) {
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) acc[p] += __shfl_xor_sync(0xffffffffu, acc[p], o);
      if (lane == 0) s_red[warp * 3 + p] = acc[p];
    }
    __syncthreads();
    if (t == 0) {
      unsigned long long err = 0;
      for (int p = 0; p < A.planes; p++) {
        unsigned long long sum = 0;
        for (int w = 0; w < kRdoThreads / 32; w++) sum += s_red[w * 3 + p];
        err += ((unsigned long long)A.dist_scale[p] * sum + (1u << 13)) >> 14;  // err * fi.dist_scale[p]
      }
      const double rate_in_bits = (double)(A.rate ? A.rate[slot] : 0u) / 8.0;
      const double cost = __fma_rn(A.lambda, rate_in_bits, (double)err);
      A.err[slot * 8 + i] = err;
      A.cost[slot * 8 + i] = cost;
      if (best_cost < 0. || cost < best_cost) {  // first minimum, rdo.rs:2531-2534
        best_cost = cost;
        best = i;
      }
    }
    __syncthreads();
  }
  if (t == 0) {
    A.best[slot] = (int8_t)best;
    *s_best = best;
  }
  if (!A.out[0]) return;
  __syncthreads();
  // ---- the area's CDEF output: the winner, or a copy of rec for skipped blocks and superblocks
  if (!inr) return;
  const int wi = max(*s_best, 0);
  {
    const CdefBlockTaps tp = cdef_block_taps(A.ystr + wi, 0, XDEC, YDEC, s_dir, s_var, b, A.damping, coeff_shift,
                                             kLumaPitch);
    T *o = (T *)A.out[0] + (long long)(ay + y0 + ly) * A.out_stride[0] + ax + x0 + lx;
#pragma unroll
    for (int r = 0; r < 4; r++)
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const short *ctr = lt + (2 + ly + r) * kLumaPitch + 2 + lx + c;
        o[(long long)r * A.out_stride[0] + c] = (T)(sk ? (int)ctr[0] : cdef_filter_tile_px(ctr, tp));
      }
  }
#pragma unroll
  for (int p = 1; p < 3; p++) {
    if (p >= A.planes) break;
    const short *tile = ct[p - 1];
    const CdefBlockTaps tp = cdef_block_taps(A.uvstr + wi, p, XDEC, YDEC, s_dir, s_var, b, A.damping, coeff_shift,
                                             L::CP);
    T *o = (T *)A.out[p] + (long long)(((ay + y0) >> YDEC) + cy) * A.out_stride[p] + ((ax + x0) >> XDEC) + cx;
#pragma unroll
    for (int r = 0; r < CROWS; r++)
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const short *ctr = tile + (2 + cy + r) * L::CP + 2 + cx + c;
        o[(long long)r * A.out_stride[p] + c] = (T)(sk ? (int)ctr[0] : cdef_filter_tile_px(ctr, tp));
      }
  }
}

template <typename T, int XDEC, int YDEC>
int cdef_rdo_launch(b200_ctx *ctx, const CdefRdoArgs &a, const CdefRdoSlots &s, int nslots) {
  constexpr size_t bytes = RdoLayout<XDEC, YDEC>::BYTES;
  if (int st = b200_smem_opt_in(ctx, (const void *)cdef_rdo_kernel<T, XDEC, YDEC>, (int)bytes)) return st;
  cdef_rdo_kernel<T, XDEC, YDEC><<<nslots, kRdoThreads, bytes, ctx->stream>>>(a, s);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

int cdef_rdo_dispatch(b200_ctx *ctx, int bpp, int xdec, int ydec, const CdefRdoArgs &a, const CdefRdoSlots &s,
                      int nslots) {
  if (bpp == 1) {
    if (xdec && ydec) return cdef_rdo_launch<uint8_t, 1, 1>(ctx, a, s, nslots);
    if (xdec) return cdef_rdo_launch<uint8_t, 1, 0>(ctx, a, s, nslots);
    return cdef_rdo_launch<uint8_t, 0, 0>(ctx, a, s, nslots);
  }
  if (xdec && ydec) return cdef_rdo_launch<uint16_t, 1, 1>(ctx, a, s, nslots);
  if (xdec) return cdef_rdo_launch<uint16_t, 1, 0>(ctx, a, s, nslots);
  return cdef_rdo_launch<uint16_t, 0, 0>(ctx, a, s, nslots);
}

}  // namespace

extern "C" int b200_cdef_rdo_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src, const b200_plane *out,
                                 int planes, int xdec, int ydec, int frame_width, int frame_height, int bit_depth,
                                 int damping, int cdef_bits, const uint8_t y_strengths[8],
                                 const uint8_t uv_strengths[8], const uint8_t *d_skip8, const uint32_t *d_imp_scales,
                                 const uint32_t dist_scale[3], double lambda, const b200_cdef_rdo_area *areas,
                                 size_t n_areas, const uint32_t *d_rate, uint64_t *d_err, double *d_cost,
                                 int8_t *d_best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, rec && src && y_strengths && uv_strengths && dist_scale && d_err && d_cost && d_best,
               "NULL rec / src / strengths / dist_scale / outputs");
  B200_REQUIRE(ctx, planes == 1 || planes == 3, "planes must be 1 or 3, got %d", planes);
  B200_REQUIRE(ctx, (xdec == 1 && ydec == 1) || (xdec == 1 && ydec == 0) || (xdec == 0 && ydec == 0),
               "chroma layout (xdec %d, ydec %d) is not 4:2:0, 4:2:2 or 4:4:4", xdec, ydec);
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  B200_REQUIRE(ctx, frame_width > 0 && frame_height > 0 && frame_width <= 65536 && frame_height <= 65536,
               "bad frame size %dx%d", frame_width, frame_height);
  // fi.cdef_damping = 3 + (base_q_idx >> 6) (encoder.rs:1221)
  B200_REQUIRE(ctx, damping >= 3 && damping <= 6, "damping %d outside 3..6", damping);
  B200_REQUIRE(ctx, cdef_bits >= 0 && cdef_bits <= 3, "cdef_bits %d outside 0..3", cdef_bits);
  const int nidx = 1 << cdef_bits;
  for (int i = 0; i < nidx; i++)
    B200_REQUIRE(ctx, y_strengths[i] <= 63 && uv_strengths[i] <= 63, "strength %d above 63 at index %d",
                 std::max(y_strengths[i], uv_strengths[i]), i);
  const int bpp = bit_depth == 8 ? 1 : 2;
  const int w8px = (frame_width + 7) & ~7, h8px = (frame_height + 7) & ~7;  // the frame's 8x8 blocks
  for (int p = 0; p < planes; p++) {
    const int xd = p ? xdec : 0, yd = p ? ydec : 0;
    for (int k = 0; k < 3; k++) {
      const b200_plane *pl = k == 0 ? rec : k == 1 ? src : out;
      if (!pl) continue;
      B200_REQUIRE(ctx, pl[p].data != nullptr, "NULL plane %d", p);
      B200_REQUIRE(ctx, pl[p].bpp == bpp, "plane %d: bpp %d does not match bit depth %d", p, pl[p].bpp, bit_depth);
      B200_REQUIRE(ctx, pl[p].width >= (w8px >> xd) && pl[p].height >= (h8px >> yd) && pl[p].stride >= pl[p].width,
                   "plane %d (%dx%d) smaller than the frame's 8x8 blocks (%dx%d)", p, pl[p].width, pl[p].height,
                   w8px >> xd, h8px >> yd);
    }
    if (out)
      for (int r = 0; r < planes; r++)
        B200_REQUIRE(ctx, out[p].data != rec[r].data, "out plane %d aliases rec plane %d", p, r);
  }
  if (n_areas == 0) return B200_OK;
  B200_REQUIRE(ctx, areas != nullptr, "NULL areas");
  const int sbw = (frame_width + 63) >> 6, sbh = (frame_height + 63) >> 6;
  std::vector<uint8_t> used((size_t)sbw * sbh, 0);
  for (size_t k = 0; k < n_areas; k++) {
    const b200_cdef_rdo_area &r = areas[k];
    B200_REQUIRE(ctx, r.sb_w >= 1 && r.sb_w <= 4 && r.sb_h >= 1 && r.sb_h <= 4, "area %zu: %dx%d superblocks", k,
                 r.sb_w, r.sb_h);
    B200_REQUIRE(ctx, r.sbx >= 0 && r.sby >= 0 && r.sbx + r.sb_w <= sbw && r.sby + r.sb_h <= sbh,
                 "area %zu (%d, %d, %dx%d) outside the %dx%d superblock frame", k, r.sbx, r.sby, r.sb_w, r.sb_h, sbw,
                 sbh);
    for (int y = r.sby; y < r.sby + r.sb_h; y++)
      for (int x = r.sbx; x < r.sbx + r.sb_w; x++) {
        B200_REQUIRE(ctx, !used[(size_t)y * sbw + x], "area %zu overlaps an earlier area at superblock (%d, %d)", k,
                     x, y);
        used[(size_t)y * sbw + x] = 1;
      }
  }
  B200_CUDA(ctx, cudaSetDevice(ctx->device));

  CdefRdoArgs a{};
  for (int p = 0; p < planes; p++) {
    a.rec[p] = PlaneView{rec[p].data, rec[p].stride};
    a.src[p] = PlaneView{src[p].data, src[p].stride};
    a.out[p] = out ? out[p].data : nullptr;
    a.out_stride[p] = out ? out[p].stride : 0;
  }
  a.planes = planes;
  a.width = frame_width;
  a.height = frame_height;
  a.w8 = w8px >> 3;
  a.bit_depth = bit_depth;
  a.damping = damping;
  a.nidx = nidx;
  for (int i = 0; i < 8; i++) {
    a.ystr[i] = i < nidx ? y_strengths[i] : 0;
    a.uvstr[i] = i < nidx ? uv_strengths[i] : 0;
  }
  a.skip8 = d_skip8;
  a.imp = d_imp_scales;
  for (int p = 0; p < 3; p++) a.dist_scale[p] = dist_scale[p];
  a.lambda = lambda;
  a.rate = d_rate;
  a.err = (unsigned long long *)d_err;
  a.cost = d_cost;
  a.best = d_best;

  // areas in launch-sized groups: up to kRdoMaxAreas areas and kRdoMaxSlots superblocks each
  CdefRdoSlots s;
  size_t k = 0;
  while (k < n_areas) {
    s.area0 = (uint32_t)k;
    int na = 0, ns = 0;
    while (k < n_areas && na < kRdoMaxAreas && ns + areas[k].sb_w * areas[k].sb_h <= kRdoMaxSlots) {
      const b200_cdef_rdo_area &r = areas[k];
      s.ax[na] = (uint16_t)r.sbx;
      s.ay[na] = (uint16_t)r.sby;
      s.wh[na] = (uint8_t)(r.sb_w | r.sb_h << 4);
      for (int y = 0; y < r.sb_h; y++)
        for (int x = 0; x < r.sb_w; x++) s.slot[ns++] = (uint16_t)(na << 4 | y << 2 | x);
      na++, k++;
    }
    if (int st = cdef_rdo_dispatch(ctx, bpp, xdec, ydec, a, s, ns)) return st;
  }
  return B200_OK;
}
