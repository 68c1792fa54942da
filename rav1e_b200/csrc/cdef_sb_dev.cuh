// cdef_sb_dev.cuh — one superblock of the CDEF loop-filter RDO (rav1e src/rdo.rs:2373-2567): for every cdef
// index the superblock is filtered (cdef_filter_superblock, cdef.rs:401-570), measured (rdo_loop_plane_error,
// rdo.rs:2027-2093) and costed (compute_rd_cost, rdo.rs:718-723), the first minimum wins and the winner's
// pixels can be written.  The stand-alone RDO call (cdef_rdo.cu) and the C stage of the pass loop
// (loop_decision.cu) are two kernels built from these pieces; each finds its own superblock and keeps its
// own epilogue.
//
// One CTA of 256 threads per superblock.  The superblock's tiles of `rec` (+ 2-pixel halo) are staged once
// per plane as int16 with the CDEF_VERY_LARGE sentinel wherever the reference's scratch copy of the AREA
// (rdo.rs:2277-2284, plane_region.rs:390-401) has no pixel: availability is relative to the area, not to the
// frame or tile.  The source blocks are staged once, the 64 directions and variances are computed in shared
// memory, and each index is filtered into registers and reduced to integer sums right away: four threads own
// one 8x8 luma block (a 4x4 quarter each) and the matching chroma block.
#pragma once
#include "cdef_dev.cuh"
#include "rdo_dist_dev.cuh"

namespace {

constexpr int kSbThreads = 256;
constexpr int kLumaPitch = 70;  // 68 staged columns; rows 35 words apart -> odd bank shift
constexpr int kSbPx = 64 * 64;  // one plane of a superblock's self-guided output

// the frame and CDEF parameters both kernels read
struct CdefSbArgs {
  PlaneView rec[3], src[3];
  int planes, width, height, w8, bit_depth, damping, nidx;
  uint8_t ystr[8], uvstr[8];
  const uint8_t *skip8;
  const uint32_t *imp;
  uint32_t dist_scale[3];
  double lambda;
};

inline CdefSbArgs cdef_sb_args(const b200_plane *rec, const b200_plane *src, int planes, int frame_width,
                               int frame_height, int bit_depth, int damping, int nidx, const uint8_t *y_strengths,
                               const uint8_t *uv_strengths, const uint8_t *d_skip8, const uint32_t *d_imp_scales,
                               const uint32_t dist_scale[3], double lambda) {
  CdefSbArgs a{};
  for (int p = 0; p < planes; p++) {
    a.rec[p] = PlaneView{rec[p].data, rec[p].stride};
    a.src[p] = PlaneView{src[p].data, src[p].stride};
    a.dist_scale[p] = dist_scale[p];
  }
  a.planes = planes, a.width = frame_width, a.height = frame_height, a.w8 = (frame_width + 7) >> 3;
  a.bit_depth = bit_depth, a.damping = damping, a.nidx = nidx;
  for (int i = 0; i < nidx; i++) a.ystr[i] = y_strengths[i], a.uvstr[i] = uv_strengths[i];
  a.skip8 = d_skip8, a.imp = d_imp_scales, a.lambda = lambda;
  return a;
}

// Dynamic shared memory: luma tile, 2 chroma tiles, luma source, 2 chroma sources and, with SGR, the 3
// self-guided outputs, in shorts; then variances, biases, directions, skip flags, the reduction and the winner.
template <int XDEC, int YDEC, bool SGR>
struct SbLayout {
  static constexpr int CW = 64 >> XDEC, CH = 64 >> YDEC;  // chroma superblock
  static constexpr int CP = CW + 6;                       // chroma tile pitch
  static constexpr int LT = 68 * kLumaPitch, CT = (CH + 4) * CP;
  static constexpr int SHORTS = LT + 2 * CT + 64 * 64 + 2 * CW * CH + (SGR ? 3 * kSbPx : 0);
  static constexpr size_t BYTES = SHORTS * 2 + 64 * (4 + 4 + 1 + 1) + 8 * 3 * 8 + 16;
};

// the superblock's rect inside its area, luma px
struct SbGeo {
  int ax, ay;    // the area's origin
  int wa, ha;    // the scratch copy: the area cropped to the visible frame, rounded up to 8 (rdo.rs:2152-2157, 2281-2282)
  int x0, y0;    // the superblock, area-relative
  int bw8, bh8;  // its 8x8 blocks in range (rdo.rs:2042)
};
// the superblock s = sby << 2 | sbx of the area at superblock (asbx, asby), sb_w x sb_h superblocks
__device__ __forceinline__ SbGeo sb_geo(const CdefSbArgs &A, int asbx, int asby, int sb_w, int sb_h, uint32_t s) {
  SbGeo g;
  g.ax = asbx * 64, g.ay = asby * 64;
  g.wa = (min(A.width - g.ax, sb_w * 64) + 7) & ~7, g.ha = (min(A.height - g.ay, sb_h * 64) + 7) & ~7;
  g.x0 = (s & 3) * 64, g.y0 = ((s >> 2) & 3) * 64;
  g.bw8 = min(64, g.wa - g.x0) >> 3, g.bh8 = min(64, g.ha - g.y0) >> 3;
  return g;
}

// One CTA's view of its superblock: the shared-memory layout and this thread's pixels.  SGR adds the
// self-guided outputs, which a plane's distortion reads instead of the CDEF output when s_mode[p] >= 0.
template <typename T, int XDEC, int YDEC, bool SGR>
struct CdefSb {
  using L = SbLayout<XDEC, YDEC, SGR>;
  static constexpr int CW8 = 8 >> XDEC, CH8 = 8 >> YDEC;  // chroma block of one 8x8 luma block
  static constexpr int CROWS = CW8 * CH8 / 16;            // rows of 4 pixels per thread: 4 / 2 / 1
  static constexpr int LPC = 4 / CROWS;                   // lanes per 4x4 chunk: 1 / 2 / 4

  short *lt, *ct[2], *ls, *cs[2];
  uint16_t *sg;  // SGR: [3][kSbPx]
  int *s_var;
  uint32_t *s_bias;
  uint8_t *s_dir, *s_skip;
  unsigned long long *s_red;  // [8 warps][3 planes]
  int *s_best;
  SbGeo g;
  int coeff_shift;
  // four threads per 8x8 block: a 4x4 quarter of luma, CROWS rows of 4 chroma pixels each
  int t, b, lx, ly, cx, cy;
  bool inr, sk;

  __device__ __forceinline__ CdefSb(unsigned char *smem, const SbGeo &geo, int bit_depth)
      : g(geo), coeff_shift(bit_depth - 8), t(threadIdx.x) {
    lt = (short *)smem;
    ct[0] = lt + L::LT, ct[1] = ct[0] + L::CT;
    ls = ct[1] + L::CT;
    cs[0] = ls + 64 * 64, cs[1] = cs[0] + L::CW * L::CH;
    sg = (uint16_t *)(cs[1] + L::CW * L::CH);
    s_var = (int *)(smem + L::SHORTS * 2);
    s_bias = (uint32_t *)(s_var + 64);
    s_dir = (uint8_t *)(s_bias + 64);
    s_skip = s_dir + 64;
    s_red = (unsigned long long *)(s_skip + 64);
    s_best = (int *)(s_red + 24);
    b = t >> 2;
    const int q = t & 3, bx = b & 7, by = b >> 3;
    inr = bx < g.bw8 && by < g.bh8;
    lx = 8 * bx + 4 * (q & 1), ly = 8 * by + 4 * (q >> 1);
    cx = CW8 * bx + (XDEC ? 0 : 4 * (q & 1)), cy = CH8 * by + (XDEC ? q * CROWS : 4 * (q >> 1));
  }

  // skip flags and 8x8 distortion biases (distortion_scale, rdo.rs:443-462, frame-absolute); whether any block
  // is coded (rdo.rs:2185-2205: an all-skip superblock gets no decision)
  __device__ __forceinline__ bool stage_blocks(const CdefSbArgs &A) {
    int coded_blk = 0;
    if (t < 64) {
      const int bx = t & 7, by = t >> 3;
      const bool in = bx < g.bw8 && by < g.bh8;
      const size_t gb = (size_t)(((g.ay + g.y0) >> 3) + by) * A.w8 + ((g.ax + g.x0) >> 3) + bx;
      const bool skip = !in || (A.skip8 && A.skip8[gb]);
      s_skip[t] = skip;
      s_bias[t] = in && A.imp ? A.imp[gb] : (1u << 14);
      coded_blk = !skip;
    }
    const int coded = __syncthreads_or(coded_blk);
    sk = s_skip[b];
    return coded;
  }

  // rec (+ halo, sentinel outside the area) and, with `with_src`, src
  __device__ __forceinline__ void stage_pixels(const CdefSbArgs &A, bool with_src) {
#pragma unroll
    for (int p = 0; p < 3; p++) {
      if (p >= A.planes) break;
      const int xd = p ? XDEC : 0, yd = p ? YDEC : 0;
      const int tw = (64 >> xd) + 4, th = (64 >> yd) + 4, pitch = p ? L::CP : kLumaPitch;
      const int aw = g.wa >> xd, ah = g.ha >> yd, sx = g.x0 >> xd, sy = g.y0 >> yd;
      const T *rp = (const T *)A.rec[p].data + (long long)(g.ay >> yd) * A.rec[p].stride + (g.ax >> xd);
      short *tile = p ? ct[p - 1] : lt;
      for (int i = t; i < tw * th; i += kSbThreads) {
        const int r = i / tw, c = i - r * tw;
        const int x = sx + c - 2, y = sy + r - 2;
        short v = (short)0x8000;
        if (x >= 0 && x < aw && y >= 0 && y < ah) v = (short)rp[(long long)y * A.rec[p].stride + x];
        tile[r * pitch + c] = v;
      }
      if (with_src) {
        const T *sp = (const T *)A.src[p].data + (long long)(g.ay >> yd) * A.src[p].stride + (g.ax >> xd);
        short *dst = p ? cs[p - 1] : ls;
        const int sw = 64 >> xd, sh = 64 >> yd;
        for (int i = t; i < sw * sh; i += kSbThreads) {
          const int r = i / sw, c = i - r * sw;
          const int x = sx + c, y = sy + r;
          dst[i] = x < aw && y < ah ? (short)sp[(long long)y * A.src[p].stride + x] : (short)0;
        }
      }
    }
    __syncthreads();
  }

  // directions and variances (cdef_analyze_superblock, cdef.rs:340-374)
  __device__ __forceinline__ void analyze() {
    if (t < 64) {
      unsigned v = 0;
      int d = 0;
      if (!s_skip[t])
        d = find_dir_8x8<short>(lt + (2 + 8 * (t >> 3)) * kLumaPitch + 2 + 8 * (t & 7), kLumaPitch, coeff_shift, &v);
      s_dir[t] = (uint8_t)d;
      s_var[t] = (int)v;
    }
    __syncthreads();
  }

  // the pixel plane p's distortion measures at tile pixel `ctr` (sg[p][off] for a Sgrproj plane)
  __device__ __forceinline__ int test_px(bool sgr, int p, int off, const short *ctr, const CdefBlockTaps &tp) const {
    if constexpr (SGR) {
      if (sgr) return sg[p * kSbPx + off];
    }
    return sk ? (int)ctr[0] : cdef_filter_tile_px(ctr, tp);
  }

  // index i over the superblock: the per-plane distortions, err * dist_scale and the cost at `rate` (bits * 8).
  // Thread 0 stores err / cost at [i] where those are set and keeps the first minimum (rdo.rs:2531-2534) in
  // best / best_cost.  s_mode is read only with SGR.
  __device__ __forceinline__ void evaluate(const CdefSbArgs &A, int i, uint32_t rate, const int *s_mode,
                                           unsigned long long *err_out, double *cost_out, int &best,
                                           double &best_cost) {
    const int q = t & 3, warp = t >> 5, lane = t & 31;
    unsigned long long acc[3] = {0, 0, 0};
    {  // luma: cdef_dist_kernel(src, test, 8, 8) * bias
      bool sgr = false;
      if constexpr (SGR) sgr = s_mode[0] >= 0;
      const CdefBlockTaps tp = cdef_block_taps(A.ystr + i, 0, XDEC, YDEC, s_dir, s_var, b, A.damping, coeff_shift,
                                               kLumaPitch);
      uint32_t ss = 0, sd = 0, ss2 = 0, sd2 = 0, ssd = 0;
#pragma unroll
      for (int r = 0; r < 4; r++)
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const short *ctr = lt + (2 + ly + r) * kLumaPitch + 2 + lx + c;
          const uint32_t d = (uint32_t)test_px(sgr, 0, (ly + r) * 64 + lx + c, ctr, tp);
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
      bool sgr = false;
      if constexpr (SGR) sgr = s_mode[p] >= 0;
      const short *tile = ct[p - 1], *src = cs[p - 1];
      const CdefBlockTaps tp = cdef_block_taps(A.uvstr + i, p, XDEC, YDEC, s_dir, s_var, b, A.damping, coeff_shift,
                                               L::CP);
      uint32_t sse = 0;
#pragma unroll
      for (int r = 0; r < CROWS; r++)
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const short *ctr = tile + (2 + cy + r) * L::CP + 2 + cx + c;
          const int d = test_px(sgr, p, (cy + r) * 64 + cx + c, ctr, tp);
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
        for (int w = 0; w < kSbThreads / 32; w++) sum += s_red[w * 3 + p];
        err += ((unsigned long long)A.dist_scale[p] * sum + (1u << 13)) >> 14;  // err * fi.dist_scale[p]
      }
      const double cost = __fma_rn(A.lambda, (double)rate / 8.0, (double)err);
      if (err_out) err_out[i] = err;
      if (cost_out) cost_out[i] = cost;
      if (best_cost < 0. || cost < best_cost) {
        best_cost = cost;
        best = i;
      }
    }
    __syncthreads();
  }

  // this thread's pixels of plane p at index idx (rec for skipped blocks) into `dst`, addressed like the frame
  __device__ __forceinline__ void write(const CdefSbArgs &A, int p, int idx, void *dst, int stride) const {
    if (!inr) return;
    const int xd = p ? XDEC : 0, yd = p ? YDEC : 0;
    const int pitch = p ? L::CP : kLumaPitch, rows = p ? CROWS : 4, px0 = p ? cx : lx, py0 = p ? cy : ly;
    const short *tile = p ? ct[p - 1] : lt;
    const CdefBlockTaps tp = cdef_block_taps((p ? A.uvstr : A.ystr) + idx, p, XDEC, YDEC, s_dir, s_var, b, A.damping,
                                             coeff_shift, pitch);
    T *o = (T *)dst + (long long)(((g.ay + g.y0) >> yd) + py0) * stride + ((g.ax + g.x0) >> xd) + px0;
#pragma unroll
    for (int r = 0; r < rows; r++)
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const short *ctr = tile + (2 + py0 + r) * pitch + 2 + px0 + c;
        o[(long long)r * stride + c] = (T)(sk ? (int)ctr[0] : cdef_filter_tile_px(ctr, tp));
      }
  }
};

template <typename T, int XDEC, int YDEC>
struct SbKind {
  using Pixel = T;
  static constexpr int xdec = XDEC, ydec = YDEC;
};
// Launches kernel_of(SbKind<T, XDEC, YDEC>{}), the kernel for the pixel type and chroma layout (4:0:0 runs as
// 4:2:0), over n superblocks with its layout's dynamic shared memory.
template <bool SGR, typename KernelOf, typename... Args>
int cdef_sb_launch(b200_ctx *ctx, int bpp, int xdec, int ydec, int n, KernelOf kernel_of, const Args &...args) {
  auto launch = [&](auto k) {
    using K = decltype(k);
    constexpr size_t bytes = SbLayout<K::xdec, K::ydec, SGR>::BYTES;
    const auto kernel = kernel_of(k);
    if (int st = b200_smem_opt_in(ctx, (const void *)kernel, (int)bytes)) return st;
    kernel<<<n, kSbThreads, bytes, ctx->stream>>>(args...);
    B200_LAUNCH_CHECK(ctx);
    return (int)B200_OK;
  };
  if (bpp == 1) {
    if (xdec && ydec) return launch(SbKind<uint8_t, 1, 1>{});
    if (xdec) return launch(SbKind<uint8_t, 1, 0>{});
    return launch(SbKind<uint8_t, 0, 0>{});
  }
  if (xdec && ydec) return launch(SbKind<uint16_t, 1, 1>{});
  if (xdec) return launch(SbKind<uint16_t, 1, 0>{});
  return launch(SbKind<uint16_t, 0, 0>{});
}

}  // namespace
