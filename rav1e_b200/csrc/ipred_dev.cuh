// ipred_dev.cuh — the device form of dispatch_predict_intra (rav1e src/predict.rs:705-1505), shared by
// the batched predictor (ipred.cu), the intra mode screening (intra_screen.cu) and the CfL alpha search
// (cfl_alpha.cu, which also shares pred_cfl_ac with ipred.cu's cfl_ac_kernel).
//
// A prediction is split in two so that a kernel can evaluate any pixel of it anywhere:
//   - preparation, once per (block, mode) by a group of threads: the DC value (ipred_dc, one thread)
//     and, for directional modes with the intra edge filter on, the filtered / upsampled edges
//     (ipred_filter_edges, predict.rs:1203-1266, thread-parallel over the edge: each output tap reads
//     only the unfiltered copy);
//   - ipred_pixel(p, r, c), the predicted pixel at row r, column c, which any thread can evaluate from
//     the staged edge and the prepared state alone; ipred_pixel_k<kind> is the same for a predictor
//     kind fixed at compile time, for loops over many pixels of one prediction.
// All arithmetic is the reference's integer arithmetic, including its index quirks (saturating left
// index, the `base + offset == -2` special case in zone 2).
//
// Edges are staged as int: `edge` is the reference's IntraEdge buffer (partition.rs:600-637), 257
// entries, top-left at [128], left pixels bottom->top below it, above pixels after it.
#pragma once

#include <type_traits>

#include "common.cuh"

namespace ipred {

enum { DC_PRED = 0, V_PRED, H_PRED, D45_PRED, D135_PRED, D113_PRED, D157_PRED, D203_PRED, D67_PRED,
       SMOOTH_PRED, SMOOTH_V_PRED, SMOOTH_H_PRED, PAETH_PRED, UV_CFL_PRED };
enum { VAR_NONE = 0, VAR_LEFT, VAR_TOP, VAR_BOTH };
constexpr int kMaxTx = 64;
constexpr int kEdgeLen = 4 * kMaxTx + 1;

// predict.rs:603-624 (AV1 Sm_Weights_Tx_*), indexed [size + i]
static __constant__ uint8_t kSmWeights[2 * kMaxTx] = {
    0, 0, 255, 128, 255, 149, 85, 64, 255, 197, 146, 105, 73, 50, 37, 32,
    255, 225, 196, 170, 145, 123, 102, 84, 68, 54, 43, 33, 26, 20, 17, 16,
    255, 240, 225, 210, 196, 182, 169, 157, 145, 133, 122, 111, 101, 92, 83, 74,
    66, 59, 52, 45, 39, 34, 29, 25, 21, 17, 14, 12, 10, 9, 8, 8,
    255, 248, 240, 233, 225, 218, 210, 203, 196, 189, 182, 176, 169, 163, 156,
    150, 144, 138, 133, 127, 121, 116, 111, 106, 101, 96, 91, 86, 82, 77, 73, 69,
    65, 61, 57, 54, 50, 47, 44, 41, 38, 35, 32, 29, 27, 25, 22, 20, 18, 16, 15,
    13, 12, 10, 9, 8, 7, 6, 6, 5, 5, 4, 4, 4};

// predict.rs:1268-1299, indexed by angle (0 where undefined)
static __constant__ short kDrDerivative[91] = {
    0, 0, 0, 1023, 0, 0, 547, 0, 0, 372, 0, 0, 0, 0, 273, 0, 0, 215, 0, 0, 178, 0, 0, 151, 0, 0, 132,
    0, 0, 116, 0, 0, 102, 0, 0, 0, 90, 0, 0, 80, 0, 0, 71, 0, 0, 64, 0, 0, 57, 0, 0, 51, 0, 0, 45, 0,
    0, 0, 40, 0, 0, 35, 0, 0, 31, 0, 0, 27, 0, 0, 23, 0, 0, 19, 0, 0, 15, 0, 0, 0, 0, 11, 0, 0, 7, 0,
    0, 3, 0, 0, 0};

__device__ __forceinline__ int dr_derivative(int a) { return (a >= 0 && a <= 90) ? kDrDerivative[a] : 0; }

// predict.rs:1125-1186
__device__ __forceinline__ int ief_strength(int width, int height, int smooth, int angle_delta) {
  const int wh = width + height, d = abs(angle_delta);
  if (smooth) {
    if (wh <= 8) return d >= 64 ? 2 : d >= 40 ? 1 : 0;
    if (wh <= 16) return d >= 48 ? 2 : d >= 20 ? 1 : 0;
    if (wh <= 24) return d >= 4 ? 3 : 0;
    return 3;
  }
  if (wh <= 8) return d >= 56 ? 1 : 0;
  if (wh <= 16) return d >= 40 ? 1 : 0;
  if (wh <= 24) return d >= 32 ? 3 : d >= 16 ? 2 : d >= 8 ? 1 : 0;
  if (wh <= 32) return d >= 32 ? 3 : d >= 4 ? 2 : 1;
  return 3;
}
// predict.rs:1188-1201
__device__ __forceinline__ int ief_upsample(int width, int height, int smooth, int angle_delta) {
  const int wh = width + height, d = abs(angle_delta);
  if (d == 0 || d >= 40) return 0;
  return smooth ? wh <= 8 : wh <= 16;
}

// Thread groups the preparation step runs on: a whole CTA, or one warp.
struct CtaGroup {
  __device__ int rank() const { return threadIdx.x; }
  __device__ int size() const { return blockDim.x; }
  __device__ void sync() const { __syncthreads(); }
};
struct WarpGroup {
  __device__ int rank() const { return threadIdx.x & 31; }
  __device__ int size() const { return 32; }
  __device__ void sync() const { __syncwarp(); }
};

// filter_edge (predict.rs:1203-1232): dst[i] for i in 1..size from the unfiltered src; strength 0 copies.
template <class G>
__device__ void filter_edge_par(const G &g, const int *src, int *dst, int len, int size, int strength) {
  for (int i = g.rank(); i < len; i += g.size()) {
    int v = src[i];
    if (strength > 0 && i >= 1 && i < size) {
      const int k0 = strength == 3 ? 2 : 0, k1 = strength == 1 ? 4 : strength == 2 ? 5 : 4,
                k2 = strength == 1 ? 8 : strength == 2 ? 6 : 4;  // [0,4,8,4,0] [0,5,6,5,0] [2,4,4,4,2]
      const int kk[5] = {k0, k1, k2, k1, k0};
      unsigned s = 0;
#pragma unroll
      for (int j = 0; j < 5; j++) {
        const int k = min(max(i + j - 2, 0), size - 1);
        s += (unsigned)kk[j] * (unsigned)src[k];
      }
      v = (int)((s + 8) >> 4);
    }
    dst[i] = v;
  }
}

// upsample_edge (predict.rs:1234-1266): in-place semantics reproduced out of place: src holds
// edge[0..=size], dst receives edge[0..=2*size].
template <class G>
__device__ void upsample_edge_par(const G &g, const int *src, int *dst, int size, int maxv) {
  for (int i = g.rank(); i <= size; i += g.size()) {
    if (i == 0) dst[0] = src[0];
    if (i < size) {
      // dup = [e0, e0, e1, ..., e_size, e_size]
      const int d0 = src[max(i - 1, 0)], d1 = src[i], d2 = src[i + 1], d3 = src[min(i + 2, size)];
      int s = -d0 + 9 * d1 + 9 * d2 - d3;
      s = (s + 8) / 16;  // truncating division, as the reference
      dst[2 * i + 1] = min(max(s, 0), maxv);
      dst[2 * i + 2] = d2;
    }
  }
}

// The predictor a (block, mode) runs, decided once by ipred_setup: a kernel that evaluates many pixels
// of one prediction can dispatch on it once and run ipred_pixel_k<kind> in its inner loop.
enum { K_DC = 0, K_V, K_H, K_PAETH, K_SMOOTH, K_SMOOTH_V, K_SMOOTH_H, K_Z1, K_Z2, K_Z3 };

// Everything ipred_pixel reads for one (block, mode).  Built by ipred_setup, identically in every
// thread; `fa` / `fl` are read only for directional modes with the edge filter on.
struct IpredPix {
  const int *edge;     // staged IntraEdge buffer
  const int *fa, *fl;  // filtered / upsampled above and left edges (index 0 = top-left)
  int mode, kind, w, h, maxv, dc;
  int directional, angle, enable, smooth, up_above, up_left;
  int flen, llb_n, dx, dy;
};

// The per-(block, mode) scalars of dispatch_predict_intra.  mode / angle / ief as b200_intra_item
// (PAETH already remapped, angle = intra_mode_to_angle + 3 * angle_delta).
__device__ __forceinline__ IpredPix ipred_setup(const int *edge, int mode, int angle, int ief, int left_len, int w,
                                                int h, int bit_depth, const int *fa, const int *fl, int dc) {
  IpredPix p;
  p.edge = edge;
  p.fa = fa;
  p.fl = fl;
  p.mode = mode;
  p.w = w;
  p.h = h;
  p.maxv = (1 << bit_depth) - 1;
  p.dc = dc;
  p.directional = mode >= V_PRED && mode <= D67_PRED && !(mode == V_PRED && angle == 90) &&
                  !(mode == H_PRED && angle == 180);
  p.angle = angle;
  p.enable = ief >= 0;
  p.smooth = ief > 0;
  p.up_above = p.enable ? ief_upsample(w, h, p.smooth, angle - 90) : 0;
  p.up_left = p.enable ? ief_upsample(w, h, p.smooth, angle - 180) : 0;
  p.flen = (w + h) * 2 + 1;
  p.llb_n = min(left_len, w + h);  // left_and_left_below slice length
  p.dx = angle < 90 ? dr_derivative(angle) : (angle > 90 && angle < 180) ? dr_derivative(180 - angle) : 0;
  p.dy = (angle > 90 && angle < 180) ? dr_derivative(angle - 90) : angle > 180 ? dr_derivative(270 - angle) : 0;
  p.kind = (mode == DC_PRED || mode == UV_CFL_PRED) ? K_DC
           : p.directional ? (angle < 90 ? K_Z1 : angle < 180 ? K_Z2 : K_Z3)
           : mode == V_PRED ? K_V
           : mode == H_PRED ? K_H
           : mode == PAETH_PRED ? K_PAETH
           : mode == SMOOTH_PRED ? K_SMOOTH
           : mode == SMOOTH_H_PRED ? K_SMOOTH_H
                                   : K_SMOOTH_V;
  return p;
}

// DC value of the DC-like modes (predict.rs:795-858): one thread.
__device__ __forceinline__ int ipred_dc(const int *edge, int variant, int w, int h, int left_len, int bit_depth) {
  const int *above = edge + 2 * kMaxTx + 1;
  const int ls_n = min(left_len, h);  // left_slice length
  unsigned v;
  if (variant == VAR_NONE) {
    v = 128u << (bit_depth - 8);
  } else if (variant == VAR_LEFT) {  // predict.rs:815-827: whole slice, divided by height
    unsigned s = 0;
    for (int k = 0; k < ls_n; k++) s += (unsigned)edge[2 * kMaxTx - 1 - k];
    v = (s + (unsigned)(h >> 1)) / (unsigned)h;
  } else if (variant == VAR_TOP) {
    unsigned s = 0;
    for (int k = 0; k < w; k++) s += (unsigned)above[k];
    v = (s + (unsigned)(w >> 1)) / (unsigned)w;
  } else {
    unsigned s = 0;
    for (int k = 0; k < h; k++) s += (unsigned)edge[2 * kMaxTx - 1 - k];
    for (int k = 0; k < w; k++) s += (unsigned)above[k];
    v = (s + (unsigned)((w + h) >> 1)) / (unsigned)(w + h);
  }
  return (int)v;
}

// pred_directional's edge preparation (predict.rs:1335-1400) for p (directional, filter on): stages the
// edges into the scratch sa / sl (2(w+h)+1 ints each), filters them into fa / fl and upsamples there.
// (x, y) = dst.rect() in the plane, for the filter's num_px clipping.  Ends with g.sync().
template <class G>
__device__ void ipred_filter_edges(const G &g, const IpredPix &p, int above_len, int plane_w, int plane_h, int x,
                                   int y, int *sa, int *sl, int *fa, int *fl) {
  const int w = p.w, h = p.h, flen = p.flen, angle = p.angle;
  const int *above = p.edge + 2 * kMaxTx + 1;
  const int top_left = p.edge[2 * kMaxTx];
  // at 90 / 180 degrees the reference filters nothing and leaves entry 0 at zero
  const int filtering = angle != 90 && angle != 180;
  const int a_len = min(above_len, flen - 1), l_len = min(p.llb_n, flen - 1);
  for (int i = g.rank(); i < flen; i += g.size()) {
    sa[i] = i == 0 ? (filtering ? top_left : 0) : i <= a_len ? above[i - 1] : 0;
    sl[i] = i == 0 ? (filtering ? top_left : 0) : i <= l_len ? p.edge[2 * kMaxTx - i] : 0;
  }
  g.sync();
  const int aw = plane_w - x, ah = plane_h - y;
  const int num_above = min(w, aw) + (angle < 90 ? h : 0) + 1;
  const int num_left = min(h, ah) + (angle > 180 ? w : 0) + 1;
  filter_edge_par(g, sa, fa, flen, num_above, filtering ? ief_strength(w, h, p.smooth, angle - 90) : 0);
  filter_edge_par(g, sl, fl, flen, num_left, filtering ? ief_strength(w, h, p.smooth, angle - 180) : 0);
  g.sync();
  if (p.up_above | p.up_left) {
    // entries past 2n keep their filtered values in the reference (in-place update): the upsampler
    // reads a copy and overwrites [0, 2n] of the filtered edge
    for (int i = g.rank(); i < flen; i += g.size()) {
      if (p.up_above) sa[i] = fa[i];
      if (p.up_left) sl[i] = fl[i];
    }
    g.sync();
    if (p.up_above) upsample_edge_par(g, sa, fa, w + (angle < 90 ? h : 0), p.maxv);
    if (p.up_left) upsample_edge_par(g, sl, fl, h + (angle > 180 ? w : 0), p.maxv);
    g.sync();
  }
}

// The predicted pixel at row r, column c for a prediction of kind K = p.kind (predict.rs:860-944 and
// pred_directional :1401-1505); K_DC returns the DC value.
template <int K>
__device__ __forceinline__ int ipred_pixel_k(const IpredPix &p, int r, int c) {
  const int *edge = p.edge;
  const int *above = edge + 2 * kMaxTx + 1;
  const int top_left = edge[2 * kMaxTx];
  const int w = p.w, h = p.h;
  // left(k) for k = 0 at the row next to the top-left pixel, growing downwards:
  // the reference's bottom->top slice element left[len-1-k]
  auto leftv = [&](int k) { return edge[2 * kMaxTx - 1 - k]; };
  if constexpr (K == K_DC) return p.dc;
  if constexpr (K == K_V) return above[c];
  if constexpr (K == K_H) return leftv(r);
  if constexpr (K == K_PAETH) {  // predict.rs:860-887
    const int l = leftv(r), t = above[c];
    const int base = t + l - top_left;
    const int pl = abs(base - l), pt = abs(base - t), ptl = abs(base - top_left);
    return (pl <= pt && pl <= ptl) ? l : (pt <= ptl ? t : top_left);
  }
  if constexpr (K == K_SMOOTH) {  // predict.rs:889-944
    const unsigned below = (unsigned)leftv(h - 1), right = (unsigned)above[w - 1];
    const unsigned wh_ = kSmWeights[h + r], ww_ = kSmWeights[w + c];
    const unsigned s = wh_ * (unsigned)above[c] + (256u - wh_) * below + ww_ * (unsigned)leftv(r) +
                       (256u - ww_) * right;
    return (int)((s + 256u) >> 9);
  }
  if constexpr (K == K_SMOOTH_H) {
    const unsigned ww_ = kSmWeights[w + c];
    return (int)((ww_ * (unsigned)leftv(r) + (256u - ww_) * (unsigned)above[w - 1] + 128u) >> 8);
  }
  if constexpr (K == K_SMOOTH_V) {
    const unsigned wh_ = kSmWeights[h + r];
    return (int)((wh_ * (unsigned)above[c] + (256u - wh_) * (unsigned)leftv(h - 1) + 128u) >> 8);
  }
  if constexpr (K >= K_Z1) {
    // ---- pred_directional (predict.rs:1301-1505)
    const int enable = p.enable, up_above = p.up_above, up_left = p.up_left;
    const int dx = p.dx, dy = p.dy;
    // Edge accessors in the reference's index space.
    // above_edge[k]: filtered buffer when enabled, else the raw above slice.
    auto above_at = [&](int k) { return enable ? p.fa[k] : above[k]; };
    // left_edge is the REVERSED buffer: left_edge[l - m] == (enabled ? fl[m] : leftv(m)) with
    // l = len - 1; left_edge[0] / [1] are the far (bottom) end.
    const int lel = enable ? p.flen : p.llb_n;
    auto left_fwd = [&](int m) { return enable ? p.fl[m] : leftv(m); };  // m counted from the top
    auto left_rev = [&](int idx) { return left_fwd(lel - 1 - idx); };    // reference index
    const int off_a = enable << up_above, off_l = enable << up_left;
    const int i = r, j = c;
    int v;
    if constexpr (K == K_Z1) {  // p_angle < 90
      const int idx = (i + 1) * dx;
      const int base = (idx >> (6 - up_above)) + (j << up_above);
      const int shift = ((idx << up_above) >> 1) & 31;
      const int max_base_x = (h + w - 1) << up_above;
      if (base < max_base_x)
        v = (above_at(base + off_a) * (32 - shift) + above_at(base + 1 + off_a) * shift + 16) >> 5;
      else
        v = above_at(max_base_x + off_a);
    } else if constexpr (K == K_Z2) {  // 90 < p_angle < 180
      const int idx = (j << 6) - (i + 1) * dx;
      const int base = idx >> (6 - up_above);
      if (base >= -(1 << up_above)) {
        const int shift = ((idx * (1 << up_above)) >> 1) & 31;
        const int av = (!enable && base < 0) ? top_left : above_at(base + off_a);
        const int bv = above_at(base + 1 + off_a);
        v = (av * (32 - shift) + bv * shift + 16) >> 5;
      } else {
        const int idx2 = (i << 6) - (j + 1) * dy;
        const int base2 = idx2 >> (6 - up_left);
        const int shift = ((idx2 * (1 << up_left)) >> 1) & 31;
        const int l = lel - 1;
        int av, bv;
        if (!enable && base2 < 0)
          av = top_left;
        else if (base2 + off_l == -2)
          av = left_rev(0);
        else
          av = left_rev(l - (base2 + off_l));
        if (base2 + off_l == -2)
          bv = left_rev(1);
        else
          bv = left_rev(l - (base2 + off_l + 1));
        v = (av * (32 - shift) + bv * shift + 16) >> 5;
      }
    } else {  // p_angle > 180
      const int idx = (j + 1) * dy;
      const int base = (idx >> (6 - up_left)) + (i << up_left);
      const int shift = ((idx << up_left) >> 1) & 31;
      const int l = lel - 1;
      const int ia = max(l - (base + off_l), 0), ib = max(l - (base + off_l + 1), 0);  // saturating_sub
      v = (left_rev(ia) * (32 - shift) + left_rev(ib) * shift + 16) >> 5;
    }
    return min(max(v, 0), p.maxv);
  }
  return 0;
}

// Calls f(std::integral_constant<int, K>) with K = p.kind: one dispatch per prediction instead of one per pixel.
template <typename F>
__device__ __forceinline__ auto ipred_dispatch(const IpredPix &p, F &&f) {
  switch (p.kind) {
    case K_DC: return f(std::integral_constant<int, K_DC>{});
    case K_V: return f(std::integral_constant<int, K_V>{});
    case K_H: return f(std::integral_constant<int, K_H>{});
    case K_PAETH: return f(std::integral_constant<int, K_PAETH>{});
    case K_SMOOTH: return f(std::integral_constant<int, K_SMOOTH>{});
    case K_SMOOTH_V: return f(std::integral_constant<int, K_SMOOTH_V>{});
    case K_SMOOTH_H: return f(std::integral_constant<int, K_SMOOTH_H>{});
    case K_Z1: return f(std::integral_constant<int, K_Z1>{});
    case K_Z2: return f(std::integral_constant<int, K_Z2>{});
    default: return f(std::integral_constant<int, K_Z3>{});
  }
}

// The predicted pixel at row r, column c of any prediction.
__device__ __forceinline__ int ipred_pixel(const IpredPix &p, int r, int c) {
  return ipred_dispatch(p, [&](auto k) { return ipred_pixel_k<decltype(k)::value>(p, r, c); });
}

// ---- chroma from luma (shared by ipred.cu's CfL kernels and the CfL alpha search, cfl_alpha.cu)

// pred_cfl_inner (predict.rs:1065-1088) for one pixel of a non-zero alpha, with get_scaled_luma_q0
// (:626-635): the DC value plus the scaled luma AC, clamped to the bit depth.
__device__ __forceinline__ int cfl_pixel(int dc, int alpha, int ac, int maxv) {
  const int q6 = alpha * ac;
  const int q0 = (abs(q6) + 32) >> 6;
  return min(max(dc + (q6 < 0 ? -q0 : q0), 0), maxv);
}

// pred_cfl_ac (predict.rs:1020-1063) for a bw x bh chroma block with its padding: the clamp limits
// of the luma reads and the log2 area the average divides by.
struct CflAcShape {
  int bw, xdec, ydec, max_luma_x, max_luma_y, shift;
};
__device__ __forceinline__ CflAcShape cfl_ac_shape(int bw, int bh, int w_pad, int h_pad, int xdec, int ydec) {
  CflAcShape s;
  s.bw = bw;
  s.xdec = xdec;
  s.ydec = ydec;
  s.max_luma_x = max((bw - w_pad * 4) << xdec, 8) - (1 << xdec);
  s.max_luma_y = max((bh - h_pad * 4) << ydec, 8) - (1 << ydec);
  s.shift = 0;
  for (int v = bw; v > 1; v >>= 1) s.shift++;
  for (int v = bh; v > 1; v >>= 1) s.shift++;
  return s;
}
// Element i (raster order) of the block before the average is removed: the subsampled luma sum << 3 - xdec - ydec,
// in the reference's i16 arithmetic.  `luma` addresses the block's luma pixel (0, 0).
template <typename T>
__device__ __forceinline__ short cfl_ac_sample(const CflAcShape &s, const T *luma, int stride, int i) {
  const int sy = i / s.bw, sx = i - sy * s.bw;
  const int y = min(sy << s.ydec, s.max_luma_y), x = min(sx << s.xdec, s.max_luma_x);
  short v = (short)luma[(long long)y * stride + x];
  if (s.xdec) v = (short)(v + (short)luma[(long long)y * stride + x + 1]);
  if (s.ydec) v = (short)(v + (short)luma[(long long)(y + 1) * stride + x] + (short)luma[(long long)(y + 1) * stride + x + 1]);
  return (short)(v << (3 - s.xdec - s.ydec));
}
// The average the reference subtracts, from the i32 sum of the samples.
__device__ __forceinline__ short cfl_ac_average(const CflAcShape &s, int sum) {
  return (short)((sum + (1 << (s.shift - 1))) >> s.shift);
}

}  // namespace ipred
