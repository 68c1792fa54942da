// loop_decision.cu — rdo_loop_decision (rav1e src/rdo.rs:2104-2745) after its optional deblock, for many
// loop-restoration areas in one call: the CDEF / restoration pass loop, C, L, C, L, .. per area until a
// stage changes nothing.
//
// Launches, all on the context's stream:
//  - loop_flags / loop_areas / loop_init: which areas have CDEF work (a superblock that is not all-skip) and
//    restoration work, the initial unit state (None, cost -1) and a copy of rec into `work` over the
//    scratch rect of every area that runs a stage (cdef_work = rec_subset.clone(), rdo.rs:2329-2330).
//  - C stage: loop_cdef_kernel once per anti-diagonal of superblocks (sbx + sby = 0 .. 6), or once for all of
//    them where no unit can hold Sgrproj (the first pass, or no unit searched).  A superblock's
//    Sgrproj branch reads up to 4 columns to its left and 2 rows above from `work`, which must hold THIS
//    pass's winners of the left, upper and upper-left superblocks, as the reference's raster walk leaves
//    them; those lie on earlier diagonals, so stream order alone separates the writers from the readers.
//  - L stage: the restoration search's four kernels (lrf_search_dev.cuh), the incumbents carried on the
//    device and areas that already stopped masked out.
//  - loop_status: per area, was the stage a change; the areas still running are counted, and that count
//    is the one read back per stage.
#include <algorithm>
#include <vector>

#include "cdef_dev.cuh"
#include "host_stage.cuh"
#include "lrf_search_dev.cuh"

namespace {

constexpr int kLoopThreads = 256;
constexpr int kLumaPitch = 70;  // 68 staged columns; rows 35 words apart -> odd bank shift
constexpr int kSbPx = 64 * 64;  // one plane of a superblock's self-guided output

enum : uint8_t { kCdefWork = 1, kLrfWork = 2 };

struct LoopArgs {
  PlaneView rec[3], src[3];
  void *work[3];
  int work_stride[3];
  int planes, width, height, w8, bit_depth, damping, nidx, enable_cdef;
  uint8_t ystr[8], uvstr[8];
  const uint8_t *skip8;
  const uint32_t *imp;
  uint32_t dist_scale[3];
  double lambda;
  const b200_cdef_rdo_area *areas;
  uint32_t n_areas, n_units;
  const b200_loop_unit *units;
  const int32_t *sb_unit;
  uint32_t *flags;         // [area] kCdefWork | kLrfWork
  uint8_t *active;         // [area]
  uint8_t *changed;        // [area] set by the current stage
  int *area_stages;        // [area]
  int *status;             // [0] areas still running, [1] the longest area's stage count
  b200_lrf_unit *unit;     // [unit] the current filter (best_lrf)
  double *unit_cost;       // [unit] best_lrf_cost
  uint8_t *written;        // [unit]
  int8_t *best;            // [slot]
  unsigned long long *err;
  double *cost;
};

template <int XDEC, int YDEC>
struct LoopLayout {
  static constexpr int CW = 64 >> XDEC, CH = 64 >> YDEC;  // chroma superblock
  static constexpr int CP = CW + 6;                       // chroma tile pitch
  static constexpr int LT = 68 * kLumaPitch, CT = (CH + 4) * CP;
  // shorts: luma tile, 2 chroma tiles, luma source, 2 chroma sources, 3 self-guided outputs
  static constexpr int SHORTS = LT + 2 * CT + 64 * 64 + 2 * CW * CH + 3 * kSbPx;
  static constexpr size_t BYTES = SHORTS * 2 + 64 * (4 + 4 + 1 + 1) + 8 * 3 * 8 + 16;
};

// the superblock's rect inside its area: whether the 8x8 grid covers it, and its luma origin
struct SbGeo {
  int ax, ay, sb_w, sb_h, wa, ha, x0, y0, bw8, bh8;
};
__device__ __forceinline__ SbGeo sb_geo(const LoopArgs &A, uint32_t slot) {
  const b200_cdef_rdo_area r = A.areas[slot >> 4];
  SbGeo g;
  g.ax = r.sbx * 64, g.ay = r.sby * 64, g.sb_w = r.sb_w, g.sb_h = r.sb_h;
  // the scratch copy: the area cropped to the visible frame, rounded up to 8 (rdo.rs:2152-2157, 2281-2282)
  g.wa = (min(A.width - g.ax, g.sb_w * 64) + 7) & ~7, g.ha = (min(A.height - g.ay, g.sb_h * 64) + 7) & ~7;
  g.x0 = (slot & 3) * 64, g.y0 = ((slot >> 2) & 3) * 64;
  g.bw8 = min(64, g.wa - g.x0) >> 3, g.bh8 = min(64, g.ha - g.y0) >> 3;
  return g;
}

// per superblock: does CDEF run on it (rdo.rs:2189-2205); an area has CDEF work if one does
__global__ void loop_flags(const __grid_constant__ LoopArgs A, const uint32_t *slots) {
  const uint32_t slot = slots[blockIdx.x];
  const SbGeo g = sb_geo(A, slot);
  const int t = threadIdx.x;
  int coded = 0;
  if (t < 64 && A.enable_cdef) {
    const int bx = t & 7, by = t >> 3;
    if (bx < g.bw8 && by < g.bh8)
      coded = !(A.skip8 && A.skip8[(size_t)(((g.ay + g.y0) >> 3) + by) * A.w8 + ((g.ax + g.x0) >> 3) + bx]);
  }
  if (__syncthreads_or(coded) && t == 0) atomicOr(&A.flags[slot >> 4], (uint32_t)kCdefWork);
}

// per area: the areas that run a stage (rdo.rs:2267); per unit of those: None, cost -1, not written
__global__ void loop_areas(const __grid_constant__ LoopArgs A) {
  for (uint32_t a = threadIdx.x; a < A.n_areas; a += blockDim.x) {
    A.active[a] = A.flags[a] != 0;
    A.changed[a] = 0;
    A.area_stages[a] = 0;
  }
  for (uint32_t u = threadIdx.x; u < A.n_units; u += blockDim.x)
    if (A.flags[A.units[u].area]) {
      A.unit[u] = b200_lrf_unit{};
      A.unit_cost[u] = -1.;
      A.written[u] = 0;
    }
}

// per superblock of a running area: best_index = -1 and work = rec over its part of the scratch rect
template <typename T>
__global__ void loop_init(const __grid_constant__ LoopArgs A, const uint32_t *slots, int xdec, int ydec) {
  const uint32_t slot = slots[blockIdx.x];
  if (!A.active[slot >> 4]) return;
  const SbGeo g = sb_geo(A, slot);
  if (threadIdx.x == 0) A.best[slot] = -1;
  for (int p = 0; p < A.planes; p++) {
    const int xd = p ? xdec : 0, yd = p ? ydec : 0;
    const int w = min(64, g.wa - g.x0) >> xd, h = min(64, g.ha - g.y0) >> yd;
    const int ox = (g.ax + g.x0) >> xd, oy = (g.ay + g.y0) >> yd;
    const T *s = (const T *)A.rec[p].data;
    T *d = (T *)A.work[p];
    for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
      const int r = i / w, c = i - r * w;
      d[(long long)(oy + r) * A.work_stride[p] + ox + c] = s[(long long)(oy + r) * A.rec[p].stride + ox + c];
    }
  }
}

// one C stage over the superblocks of one anti-diagonal (rdo.rs:2373-2567): cdef_rdo.cu's superblock
// evaluation with the restoration branches of rdo.rs:2424-2527
template <typename T, int XDEC, int YDEC>
__global__ void __launch_bounds__(kLoopThreads) loop_cdef_kernel(const __grid_constant__ LoopArgs A,
                                                                const uint32_t *slots) {
  using L = LoopLayout<XDEC, YDEC>;
  constexpr int CW8 = 8 >> XDEC, CH8 = 8 >> YDEC;  // chroma block of one 8x8 luma block
  constexpr int CROWS = CW8 * CH8 / 16;            // rows of 4 pixels per thread: 4 / 2 / 1
  constexpr int LPC = 4 / (CW8 * CH8 / 16);        // lanes per 4x4 chunk: 1 / 2 / 4
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ uint16_t sp[kSP][kSP];
  __shared__ uint32_t box1[2][kAB][kAB], box2[2][kR2][kAB];
  __shared__ uint32_t a1[kAB][kAB], b1[kAB][kAB], a2[kR2][kAB], b2[kR2][kAB];
  __shared__ int s_mode[3];  // -1: CDEF output measured; else the Sgrproj unit
  __shared__ uint32_t s_rate;
  short *lt = (short *)smem;
  short *ct[2] = {lt + L::LT, lt + L::LT + L::CT};
  short *ls = lt + L::LT + 2 * L::CT;
  short *cs[2] = {ls + 64 * 64, ls + 64 * 64 + L::CW * L::CH};
  uint16_t *sg = (uint16_t *)(cs[1] + L::CW * L::CH);  // [3][64 * 64]: the self-guided outputs
  int *s_var = (int *)(smem + L::SHORTS * 2);
  uint32_t *s_bias = (uint32_t *)(s_var + 64);
  uint8_t *s_dir = (uint8_t *)(s_bias + 64);
  uint8_t *s_skip = s_dir + 64;
  unsigned long long *s_red = (unsigned long long *)(s_skip + 64);  // [8 warps][3 planes]
  int *s_best = (int *)(s_red + 24);

  const int t = threadIdx.x;
  const uint32_t slot = slots[blockIdx.x];
  const uint32_t area = slot >> 4;
  if (!A.active[area] || !(A.flags[area] & kCdefWork)) return;
  const SbGeo G = sb_geo(A, slot);
  const int ax = G.ax, ay = G.ay, x0 = G.x0, y0 = G.y0, wa = G.wa, ha = G.ha, bw8 = G.bw8, bh8 = G.bh8;
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
  if (t == 0) s_rate = 0;
  __syncthreads();
  if (t < 3) {  // the restoration branch of each plane (rdo.rs:2424-2431) and its rate
    int m = -1;
    const int32_t u = t < A.planes && (A.flags[area] & kLrfWork) ? A.sb_unit[slot * 3 + t] : -1;
    if (u >= 0) {
      const b200_lrf_unit f = A.unit[u];
      atomicAdd(&s_rate, lrf_rate(A.units[u], f.type, f.set, f.xqd[0], f.xqd[1]));
      if (f.type == 2) m = u;
    }
    s_mode[t] = m;
  }
  const int coded = __syncthreads_or(coded_blk);  // rdo.rs:2380: an all-skip superblock is not decided
  if (!coded) return;
  const bool any_sgr = s_mode[0] >= 0 || s_mode[1] >= 0 || s_mode[2] >= 0;

  // ---- stage rec (+ halo, sentinel outside the area) and src
#pragma unroll
  for (int p = 0; p < 3; p++) {
    if (p >= A.planes) break;
    const int xd = p ? XDEC : 0, yd = p ? YDEC : 0;
    const int tw = (64 >> xd) + 4, th = (64 >> yd) + 4, pitch = p ? L::CP : kLumaPitch;
    const int aw = wa >> xd, ah = ha >> yd, sx = x0 >> xd, sy = y0 >> yd;
    const T *rp = (const T *)A.rec[p].data + (long long)(ay >> yd) * A.rec[p].stride + (ax >> xd);
    short *tile = p ? ct[p - 1] : lt;
    for (int i = t; i < tw * th; i += kLoopThreads) {
      const int r = i / tw, c = i - r * tw;
      const int x = sx + c - 2, y = sy + r - 2;
      short v = (short)0x8000;
      if (x >= 0 && x < aw && y >= 0 && y < ah) v = (short)rp[(long long)y * A.rec[p].stride + x];
      tile[r * pitch + c] = v;
    }
    const T *srp = (const T *)A.src[p].data + (long long)(ay >> yd) * A.src[p].stride + (ax >> xd);
    short *dst = p ? cs[p - 1] : ls;
    const int sw = 64 >> xd, sh = 64 >> yd;
    for (int i = t; i < sw * sh; i += kLoopThreads) {
      const int r = i / sw, c = i - r * sw;
      const int x = sx + c, y = sy + r;
      dst[i] = x < aw && y < ah ? (short)srp[(long long)y * A.src[p].stride + x] : (short)0;
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

  // the index's CDEF output of this thread's pixels of plane p into the working copy
  auto write_cdef = [&](int p, int idx) {
    if (!inr) return;
    const int xd = p ? XDEC : 0, yd = p ? YDEC : 0;
    const int pitch = p ? L::CP : kLumaPitch, rows = p ? CROWS : 4, px0 = p ? cx : lx, py0 = p ? cy : ly;
    const short *tile = p ? ct[p - 1] : lt;
    const CdefBlockTaps tp = cdef_block_taps((p ? A.uvstr : A.ystr) + idx, p, XDEC, YDEC, s_dir, s_var, b, A.damping,
                                             coeff_shift, pitch);
    T *o = (T *)A.work[p] + (long long)(((ay + y0) >> yd) + py0) * A.work_stride[p] + ((ax + x0) >> xd) + px0;
    for (int r = 0; r < rows; r++)
#pragma unroll
      for (int c = 0; c < 4; c++) {
        const short *ctr = tile + (2 + py0 + r) * pitch + 2 + px0 + c;
        o[(long long)r * A.work_stride[p] + c] = (T)(sk ? (int)ctr[0] : cdef_filter_tile_px(ctr, tp));
      }
  };

  // the self-guided filter of plane p's part of the superblock, read from the working copy (rdo.rs:2458-2488)
  auto sgr_plane = [&](int p) {
    const int xd = p ? XDEC : 0, yd = p ? YDEC : 0;
    const b200_lrf_unit f = A.unit[s_mode[p]];
    const int po_x = x0 >> xd, po_y = y0 >> yd;
    const int vis_w = min(64 >> xd, ((A.width - ax) >> xd) - po_x), vis_h = min(64 >> yd, ((A.height - ay) >> yd) - po_y);
    const T *in = (const T *)A.work[p] + (long long)(ay >> yd) * A.work_stride[p] + (ax >> xd);
    const uint32_t s2 = kSgrS[f.set][0], s1 = kSgrS[f.set][1];
    const int w0 = f.xqd[0], w1 = f.xqd[1], w2 = 128 - w0 - w1;
    uint16_t *o = sg + p * kSbPx;
    for (int i = t; i < kSbPx; i += kLoopThreads) o[i] = B200_LRF_WORK_FILL;
    for (int ty = 0; ty < vis_h; ty += kT)
      for (int tx = 0; tx < vis_w; tx += kT) {
        __syncthreads();
        sgr_stage_tile<T>(sp, in, A.work_stride[p], po_x, po_y, vis_w, vis_h, tx, ty);
        __syncthreads();
        sgr_box_sums(sp, box1, box2);
        __syncthreads();
        sgr_ab(box1, box2, a1, b1, a2, b2, s1, s2, coeff_shift);
        __syncthreads();
        for (int i = t; i < kT * kT; i += kLoopThreads) {
          const int y = i / kT, x = i - y * kT;
          if (tx + x >= vis_w || ty + y >= vis_h) continue;
          uint32_t g1, g2;
          const uint32_t px = sgr_f(sp, a1, b1, a2, b2, s1, s2, y, x, g1, g2);
          o[(ty + y) * 64 + tx + x] = sgr_apply(w0, w1, w2, g1, g2, px, A.bit_depth);
        }
      }
  };

  int best = -1;
  double best_cost = -1.;
  for (int i = 0; i < A.nidx; i++) {
    if (any_sgr) {  // filter into the working copy, then the self-guided filter reads it
#pragma unroll
      for (int p = 0; p < 3; p++)
        if (p < A.planes && s_mode[p] >= 0) write_cdef(p, i);
      __syncthreads();
#pragma unroll
      for (int p = 0; p < 3; p++)
        if (p < A.planes && s_mode[p] >= 0) sgr_plane(p);
      __syncthreads();
    }
    unsigned long long acc[3] = {0, 0, 0};
    {  // luma: cdef_dist_kernel(src, test, 8, 8) * bias
      const bool sg0 = s_mode[0] >= 0;
      const CdefBlockTaps tp = cdef_block_taps(A.ystr + i, 0, XDEC, YDEC, s_dir, s_var, b, A.damping, coeff_shift,
                                               kLumaPitch);
      uint32_t ss = 0, sd = 0, ss2 = 0, sd2 = 0, ssd = 0;
#pragma unroll
      for (int r = 0; r < 4; r++)
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const short *ctr = lt + (2 + ly + r) * kLumaPitch + 2 + lx + c;
          const uint32_t d = sg0 ? (uint32_t)sg[(ly + r) * 64 + lx + c]
                                 : (uint32_t)(sk ? (int)ctr[0] : cdef_filter_tile_px(ctr, tp));
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
      const bool sgp = s_mode[p] >= 0;
      const short *tile = ct[p - 1], *src = cs[p - 1];
      const CdefBlockTaps tp = cdef_block_taps(A.uvstr + i, p, XDEC, YDEC, s_dir, s_var, b, A.damping, coeff_shift,
                                               L::CP);
      uint32_t sse = 0;
#pragma unroll
      for (int r = 0; r < CROWS; r++)
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const short *ctr = tile + (2 + cy + r) * L::CP + 2 + cx + c;
          const int d = sgp ? (int)sg[p * kSbPx + (cy + r) * 64 + cx + c]
                            : (sk ? (int)ctr[0] : cdef_filter_tile_px(ctr, tp));
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
        for (int w = 0; w < kLoopThreads / 32; w++) sum += s_red[w * 3 + p];
        err += ((unsigned long long)A.dist_scale[p] * sum + (1u << 13)) >> 14;  // err * fi.dist_scale[p]
      }
      const double cost = __fma_rn(A.lambda, (double)s_rate / 8.0, (double)err);
      if (A.err) A.err[slot * 8 + i] = err;
      if (A.cost) A.cost[slot * 8 + i] = cost;
      if (best_cost < 0. || cost < best_cost) {  // first minimum, rdo.rs:2531-2534
        best_cost = cost;
        best = i;
      }
    }
    __syncthreads();
  }
  if (t == 0) {
    if (best != A.best[slot]) A.changed[area] = 1;  // rdo.rs:2537-2542
    A.best[slot] = (int8_t)best;
    *s_best = best;
  }
  __syncthreads();
  // ---- keep the working copy up to date with the winner (rdo.rs:2554-2564)
  const int wi = *s_best;
#pragma unroll
  for (int p = 0; p < 3; p++)
    if (p < A.planes) write_cdef(p, wi);
}

// per area: was this stage a change; count the areas still running and the longest stage count
__global__ void loop_status(const __grid_constant__ LoopArgs A, int stage) {
  __shared__ int s_run, s_long;
  if (threadIdx.x == 0) s_run = 0, s_long = 0;
  __syncthreads();
  int run = 0, lng = 0;
  for (uint32_t a = threadIdx.x; a < A.n_areas; a += blockDim.x) {
    if (A.active[a]) {
      // the first C stage always counts as a change (cdef_change starts true, rdo.rs:2370)
      const bool ch = stage == 0 || A.changed[a];
      A.area_stages[a] = stage + 1;
      if (!ch) A.active[a] = 0;
    }
    A.changed[a] = 0;
    run += A.active[a];
    lng = max(lng, A.area_stages[a]);
  }
  atomicAdd(&s_run, run);
  atomicMax(&s_long, lng);
  __syncthreads();
  if (threadIdx.x == 0) A.status[0] = s_run, A.status[1] = s_long;
}

template <typename T, int XDEC, int YDEC>
int loop_cdef_launch(b200_ctx *ctx, const LoopArgs &a, const uint32_t *slots, int n) {
  constexpr size_t bytes = LoopLayout<XDEC, YDEC>::BYTES;
  if (int st = b200_smem_opt_in(ctx, (const void *)loop_cdef_kernel<T, XDEC, YDEC>, (int)bytes)) return st;
  loop_cdef_kernel<T, XDEC, YDEC><<<n, kLoopThreads, bytes, ctx->stream>>>(a, slots);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

int loop_cdef_dispatch(b200_ctx *ctx, int bpp, int xdec, int ydec, const LoopArgs &a, const uint32_t *slots, int n) {
  if (bpp == 1) {
    if (xdec && ydec) return loop_cdef_launch<uint8_t, 1, 1>(ctx, a, slots, n);
    if (xdec) return loop_cdef_launch<uint8_t, 1, 0>(ctx, a, slots, n);
    return loop_cdef_launch<uint8_t, 0, 0>(ctx, a, slots, n);
  }
  if (xdec && ydec) return loop_cdef_launch<uint16_t, 1, 1>(ctx, a, slots, n);
  if (xdec) return loop_cdef_launch<uint16_t, 1, 0>(ctx, a, slots, n);
  return loop_cdef_launch<uint16_t, 0, 0>(ctx, a, slots, n);
}

bool unit_size_ok(int s) { return s >= 32 && s <= 256 && (s & (s - 1)) == 0; }

bool overlaps(const b200_plane &a, const b200_plane &b) {
  const uint8_t *a0 = (const uint8_t *)a.data, *b0 = (const uint8_t *)b.data;
  const uint8_t *a1 = a0 + ((size_t)a.stride * (a.height - 1) + a.width) * a.bpp;
  const uint8_t *b1 = b0 + ((size_t)b.stride * (b.height - 1) + b.width) * b.bpp;
  return a0 < b1 && b0 < a1;
}

}  // namespace

extern "C" int b200_loop_decision_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src,
                                      const b200_plane *work, int planes, int xdec, int ydec, int frame_width,
                                      int frame_height, int bit_depth, int enable_cdef, int damping, int cdef_bits,
                                      const uint8_t y_strengths[8], const uint8_t uv_strengths[8],
                                      const uint8_t *d_skip8, int enable_restoration, const int unit_size[3],
                                      int reduced_sets, const uint32_t *d_imp_scales, const uint32_t dist_scale[3],
                                      double lambda, const b200_cdef_rdo_area *areas, size_t n_areas,
                                      const b200_loop_unit *units, size_t n_units, const int32_t *sb_unit,
                                      int8_t *d_best_index, b200_lrf_unit *d_unit, double *d_unit_cost,
                                      uint8_t *d_written, uint64_t *d_err, double *d_cost, int *stages) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, rec && src && work && dist_scale && stages && d_best_index,
               "NULL rec / src / work / dist_scale / stages / d_best_index");
  B200_REQUIRE(ctx, n_units == 0 || (d_unit && d_unit_cost && d_written), "NULL unit outputs");
  B200_REQUIRE(ctx, planes == 1 || planes == 3, "planes must be 1 or 3, got %d", planes);
  B200_REQUIRE(ctx, (xdec == 1 && ydec == 1) || (xdec == 1 && ydec == 0) || (xdec == 0 && ydec == 0),
               "chroma layout (xdec %d, ydec %d) is not 4:2:0, 4:2:2 or 4:4:4", xdec, ydec);
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  B200_REQUIRE(ctx, frame_width > 0 && frame_height > 0 && frame_width <= 65536 && frame_height <= 65536,
               "bad frame size %dx%d", frame_width, frame_height);
  const int nidx = enable_cdef ? 1 << cdef_bits : 0;
  if (enable_cdef) {
    B200_REQUIRE(ctx, y_strengths && uv_strengths, "NULL strengths");
    B200_REQUIRE(ctx, damping >= 3 && damping <= 6, "damping %d outside 3..6", damping);
    B200_REQUIRE(ctx, cdef_bits >= 0 && cdef_bits <= 3, "cdef_bits %d outside 0..3", cdef_bits);
    for (int i = 0; i < nidx; i++)
      B200_REQUIRE(ctx, y_strengths[i] <= 63 && uv_strengths[i] <= 63, "strength %d above 63 at index %d",
                   std::max(y_strengths[i], uv_strengths[i]), i);
  }
  const int bpp = bit_depth == 8 ? 1 : 2;
  const int w8px = (frame_width + 7) & ~7, h8px = (frame_height + 7) & ~7;
  for (int p = 0; p < planes; p++) {
    const int xd = p ? xdec : 0, yd = p ? ydec : 0;
    for (const b200_plane *pl : {rec, src, work}) {
      B200_REQUIRE(ctx, pl[p].data != nullptr, "NULL plane %d", p);
      B200_REQUIRE(ctx, pl[p].bpp == bpp, "plane %d: bpp %d does not match bit depth %d", p, pl[p].bpp, bit_depth);
      B200_REQUIRE(ctx, pl[p].width >= (w8px >> xd) && pl[p].height >= (h8px >> yd) && pl[p].stride >= pl[p].width,
                   "plane %d (%dx%d) smaller than the frame's 8x8 blocks (%dx%d)", p, pl[p].width, pl[p].height,
                   w8px >> xd, h8px >> yd);
    }
    for (int r = 0; r < planes; r++)
      B200_REQUIRE(ctx, !overlaps(work[p], rec[r]) && !overlaps(work[p], src[r]),
                   "work plane %d aliases rec or src plane %d", p, r);
    if (enable_restoration) {
      B200_REQUIRE(ctx, unit_size != nullptr, "NULL unit_size");
      const int us = unit_size[p];
      B200_REQUIRE(ctx, unit_size_ok(us) && ((us << xd) % 64) == 0 && ((us << yd) % 64) == 0 && (us << xd) <= 256 &&
                            (us << yd) <= 256,
                   "plane %d: unit size %d is not 32..256 in whole superblocks", p, us);
    }
  }
  if (n_areas == 0) {
    *stages = 0;
    return B200_OK;
  }
  B200_REQUIRE(ctx, areas != nullptr && sb_unit != nullptr, "NULL areas / sb_unit");
  B200_REQUIRE(ctx, n_units == 0 || units != nullptr, "NULL units");
  B200_REQUIRE(ctx, n_areas <= (1u << 20) && n_units <= (1u << 24), "%zu areas / %zu units: too many", n_areas,
               n_units);
  const int sbw = (frame_width + 63) >> 6, sbh = (frame_height + 63) >> 6;
  std::vector<uint8_t> used((size_t)sbw * sbh, 0);
  std::vector<uint32_t> flags(n_areas, 0);
  std::vector<uint32_t> diag[7];
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
    for (int y = 0; y < r.sb_h; y++)
      for (int x = 0; x < r.sb_w; x++) diag[x + y].push_back((uint32_t)(k * 16 + y * 4 + x));
  }
  // the restoration stage's items: the units with `search` set
  std::vector<b200_lrf_search_item> items;
  std::vector<Geo> geo;
  std::vector<Tile> tiles;
  std::vector<uint32_t> unit_of;
  for (size_t u = 0; u < n_units; u++) {
    const b200_loop_unit &un = units[u];
    B200_REQUIRE(ctx, un.area >= 0 && (size_t)un.area < n_areas, "unit %zu: area %d of %zu", u, un.area, n_areas);
    B200_REQUIRE(ctx, un.plane >= 0 && un.plane < planes, "unit %zu: plane %d", u, un.plane);
    B200_REQUIRE(ctx, un.sgrproj_ref[0] >= -96 && un.sgrproj_ref[0] <= 31 && un.sgrproj_ref[1] >= -32 &&
                          un.sgrproj_ref[1] <= 95,
                 "unit %zu: sgrproj_ref (%d, %d) out of range", u, un.sgrproj_ref[0], un.sgrproj_ref[1]);
    if (!enable_restoration) continue;
    const b200_cdef_rdo_area &r = areas[un.area];
    const int p = un.plane, xd = p ? xdec : 0, yd = p ? ydec : 0, us = unit_size[p];
    const int lsw = (us << xd) / 64, lsh = (us << yd) / 64;
    B200_REQUIRE(ctx, un.lru_x >= 0 && un.lru_y >= 0 && un.lru_x * lsw < r.sb_w && un.lru_y * lsh < r.sb_h,
                 "unit %zu: (%d, %d) outside its %dx%d area", u, un.lru_x, un.lru_y, r.sb_w, r.sb_h);
    const Geo g = lrf_unit_geo(r, p, xd, yd, us, un.lru_x, un.lru_y, frame_width, frame_height);
    B200_REQUIRE(ctx, g.vis_w > 0 && g.vis_h > 0, "unit %zu: (%d, %d) outside the visible frame", u, un.lru_x,
                 un.lru_y);
    if (!un.search) continue;
    flags[un.area] |= kLrfWork;
    b200_lrf_search_item it{};
    it.area = un.area, it.plane = p, it.lru_x = un.lru_x, it.lru_y = un.lru_y;
    it.none_bits = un.none_bits, it.sgr_bits = un.sgr_bits;
    it.sgrproj_ref[0] = un.sgrproj_ref[0], it.sgrproj_ref[1] = un.sgrproj_ref[1];
    it.incoming_cost = -1.;
    for (int ty = 0; ty < g.eh; ty += kT)
      for (int tx = 0; tx < g.ew; tx += kT) tiles.push_back(Tile{(uint32_t)items.size(), (uint16_t)tx, (uint16_t)ty});
    items.push_back(it);
    geo.push_back(g);
    unit_of.push_back((uint32_t)u);
  }
  for (size_t k = 0; k < n_areas; k++)
    for (int s = 0; s < 16; s++)
      for (int p = 0; p < 3; p++) {
        if ((s & 3) >= areas[k].sb_w || (s >> 2) >= areas[k].sb_h) continue;
        const int32_t u = p < planes ? sb_unit[(k * 16 + s) * 3 + p] : -1;
        B200_REQUIRE(ctx, u >= -1 && (int64_t)u < (int64_t)n_units, "sb_unit[%zu]: %d of %zu units",
                     (k * 16 + s) * 3 + p, u, n_units);
        B200_REQUIRE(ctx, u < 0 || ((size_t)units[u].area == k && units[u].plane == p),
                     "sb_unit[%zu]: unit %d belongs to area %d plane %d", (k * 16 + s) * 3 + p, u,
                     u < 0 ? -1 : units[u].area, u < 0 ? -1 : units[u].plane);
      }

  // ---- one upload: areas, map, units, flags, the diagonals' slot lists, the items, geometry and tiles
  size_t nslots = 0;
  for (auto &d : diag) nslots += d.size();
  std::vector<uint32_t> slots;
  slots.reserve(nslots);
  size_t doff[8] = {0};
  for (int d = 0; d < 7; d++) {
    doff[d] = slots.size();
    slots.insert(slots.end(), diag[d].begin(), diag[d].end());
  }
  doff[7] = slots.size();
  const size_t n_items = items.size();
  std::vector<std::pair<const void *, size_t>> parts = {
      {areas, n_areas * sizeof(b200_cdef_rdo_area)},  {sb_unit, n_areas * 48 * sizeof(int32_t)},
      {units, n_units * sizeof(b200_loop_unit)},     {flags.data(), n_areas * sizeof(uint32_t)},
      {slots.data(), slots.size() * sizeof(uint32_t)}, {items.data(), n_items * sizeof(b200_lrf_search_item)},
      {geo.data(), n_items * sizeof(Geo)},           {tiles.data(), tiles.size() * sizeof(Tile)},
      {unit_of.data(), n_items * sizeof(uint32_t)}};
  size_t up_bytes = 0, off[9];
  for (size_t i = 0; i < parts.size(); i++) {
    off[i] = up_bytes;
    up_bytes += b200_align_up(parts[i].second, 256);
  }
  std::vector<uint8_t> packed(up_bytes, 0);
  for (size_t i = 0; i < parts.size(); i++)
    if (parts[i].second) memcpy(packed.data() + off[i], parts[i].first, parts[i].second);
  const size_t b_area = b200_align_up(n_areas * 4, 256) * 3, b_status = 256;
  const size_t b_acc = std::max<size_t>(n_items, 1) * 16 * 5 * sizeof(long long);
  const size_t b_err = std::max<size_t>(n_items, 1) * kCands * sizeof(unsigned long long);
  const size_t b_item = std::max<size_t>(n_items, 1) * (32 + sizeof(b200_lrf_unit) + 8 + 1);
  HostStage s(ctx, up_bytes + b_area + b_status + 4 * 256 + b200_align_up(b_acc, 256) + b200_align_up(b_err, 256) +
                       b200_align_up(b_item, 256) + 3 * 256);
  uint8_t *d_up = s.take(up_bytes);
  uint8_t *d_active = s.take(n_areas), *d_changed = s.take(n_areas);
  int *d_area_stages = (int *)s.take(n_areas * 4);
  int *d_status = (int *)s.take(b_status);
  long long *d_acc = (long long *)s.take(b_acc);
  unsigned long long *d_cerr = (unsigned long long *)s.take(b_err);
  int8_t *d_xq = (int8_t *)s.take(std::max<size_t>(n_items, 1) * 32);
  b200_lrf_unit *d_ibest = (b200_lrf_unit *)s.take(std::max<size_t>(n_items, 1) * sizeof(b200_lrf_unit));
  double *d_icost = (double *)s.take(std::max<size_t>(n_items, 1) * 8);
  uint8_t *d_ichanged = s.take(std::max<size_t>(n_items, 1));
  s.up(d_up, packed.data(), up_bytes);
  if (!s.ok()) return s.finish(false);

  LoopArgs a{};
  for (int p = 0; p < planes; p++) {
    a.rec[p] = PlaneView{rec[p].data, rec[p].stride};
    a.src[p] = PlaneView{src[p].data, src[p].stride};
    a.work[p] = work[p].data;
    a.work_stride[p] = work[p].stride;
  }
  a.planes = planes, a.width = frame_width, a.height = frame_height, a.w8 = w8px >> 3, a.bit_depth = bit_depth;
  a.damping = damping, a.nidx = nidx, a.enable_cdef = enable_cdef != 0;
  for (int i = 0; i < 8; i++) {
    a.ystr[i] = i < nidx ? y_strengths[i] : 0;
    a.uvstr[i] = i < nidx ? uv_strengths[i] : 0;
  }
  a.skip8 = d_skip8, a.imp = d_imp_scales;
  for (int p = 0; p < 3; p++) a.dist_scale[p] = p < planes ? dist_scale[p] : 0;
  a.lambda = lambda;
  a.areas = (const b200_cdef_rdo_area *)(d_up + off[0]);
  a.sb_unit = (const int32_t *)(d_up + off[1]);
  a.units = (const b200_loop_unit *)(d_up + off[2]);
  a.flags = (uint32_t *)(d_up + off[3]);
  a.n_areas = (uint32_t)n_areas, a.n_units = (uint32_t)n_units;
  a.active = d_active, a.changed = d_changed, a.area_stages = d_area_stages, a.status = d_status;
  a.unit = d_unit, a.unit_cost = d_unit_cost, a.written = d_written;
  a.best = d_best_index, a.err = (unsigned long long *)d_err, a.cost = d_cost;
  const uint32_t *d_slots = (const uint32_t *)(d_up + off[4]);

  SearchArgs la{};
  for (int p = 0; p < planes; p++) {
    la.in[p] = PlaneView{work[p].data, work[p].stride};
    la.src[p] = PlaneView{src[p].data, src[p].stride};
  }
  la.xdec = xdec, la.ydec = ydec, la.bit_depth = bit_depth, la.w8 = w8px >> 3;
  la.reduced = reduced_sets != 0;
  la.nsets = la.reduced ? 8 : 16;
  la.imp = d_imp_scales;
  for (int p = 0; p < 3; p++) la.dist_scale[p] = a.dist_scale[p];
  la.lambda = lambda;
  la.items = (const b200_lrf_search_item *)(d_up + off[5]);
  la.geo = (const Geo *)(d_up + off[6]);
  la.tiles = (const Tile *)(d_up + off[7]);
  la.n_items = (uint32_t)n_items, la.n_tiles = (uint32_t)tiles.size();
  la.acc = d_acc, la.err = d_cerr, la.xq = d_xq;
  la.best = d_ibest, la.cost = d_icost, la.changed = d_ichanged;
  la.unit_of = (const uint32_t *)(d_up + off[8]);
  la.inc = d_unit, la.inc_cost = d_unit_cost, la.written = d_written;
  la.active = d_active, la.area_changed = d_changed;

  const unsigned n_all = (unsigned)slots.size();
  loop_flags<<<n_all, kLoopThreads, 0, ctx->stream>>>(a, d_slots);
  B200_LAUNCH_CHECK(ctx);
  loop_areas<<<1, 256, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  if (bpp == 1) loop_init<uint8_t><<<n_all, kLoopThreads, 0, ctx->stream>>>(a, d_slots, xdec, ydec);
  else loop_init<uint16_t><<<n_all, kLoopThreads, 0, ctx->stream>>>(a, d_slots, xdec, ydec);
  B200_LAUNCH_CHECK(ctx);

  const unsigned tile_grid = (unsigned)std::min<size_t>(tiles.size(), 8192);
  const unsigned solve_grid = (unsigned)std::min<size_t>((n_items * la.nsets + 255) / 256, 4096);
  const unsigned item_grid = (unsigned)std::min<size_t>((n_items + 255) / 256, 4096);
  int result = -1;
  for (int stage = 0; stage < B200_LOOP_MAX_STAGES; stage++) {
    if (!(stage & 1)) {  // C
      // No unit holds Sgrproj on the first pass (all start as None) or when no unit is searched, so no superblock
      // reads another's output: every slot goes in one launch.  Otherwise one launch per anti-diagonal.
      const bool one_launch = stage == 0 || n_items == 0;
      for (int d = 0; d < 7 && nidx; d++) {
        const size_t b = one_launch ? 0 : doff[d], e = one_launch ? doff[7] : doff[d + 1];
        if (e > b)
          if (int st = loop_cdef_dispatch(ctx, bpp, xdec, ydec, a, d_slots + b, (int)(e - b))) {
            s.run(st);
            return s.finish(false);
          }
        if (one_launch) break;
      }
    } else if (n_items) {  // L
      s.run(cudaMemsetAsync(d_acc, 0, b_acc, ctx->stream) == cudaSuccess ? B200_OK : B200_ERR_CUDA);
      s.run(cudaMemsetAsync(d_cerr, 0, b_err, ctx->stream) == cudaSuccess ? B200_OK : B200_ERR_CUDA);
      if (!s.ok()) return s.finish(false);
      if (bpp == 1) lrf_search_tiles<uint8_t, false><<<tile_grid, kThreads, 0, ctx->stream>>>(la);
      else lrf_search_tiles<uint16_t, false><<<tile_grid, kThreads, 0, ctx->stream>>>(la);
      B200_LAUNCH_CHECK(ctx);
      lrf_search_solve<<<solve_grid, 256, 0, ctx->stream>>>(la);
      B200_LAUNCH_CHECK(ctx);
      if (bpp == 1) lrf_search_tiles<uint8_t, true><<<tile_grid, kThreads, 0, ctx->stream>>>(la);
      else lrf_search_tiles<uint16_t, true><<<tile_grid, kThreads, 0, ctx->stream>>>(la);
      B200_LAUNCH_CHECK(ctx);
      lrf_search_decide<<<item_grid, 256, 0, ctx->stream>>>(la);
      B200_LAUNCH_CHECK(ctx);
    }
    loop_status<<<1, 256, 0, ctx->stream>>>(a, stage);
    B200_LAUNCH_CHECK(ctx);
    int st[2] = {0, 0};
    s.down(st, d_status, sizeof(st));  // the one synchronisation of the stage
    s.run(cudaStreamSynchronize(ctx->stream) == cudaSuccess ? B200_OK : B200_ERR_CUDA);
    if (!s.ok()) return s.finish(false);
    if (st[0] == 0) {
      result = st[1];
      break;
    }
  }
  *stages = result;
  return s.finish(false);
}
