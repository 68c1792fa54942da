// ipred.cu — batched AV1 intra prediction (rav1e src/predict.rs:705-1505) for sm_90a.
//
// One CTA per (block, mode) item: the RDO loop evaluates ~13 modes per block from the same
// neighbour pixels (rdo.rs:1470-1505), so a launch carries blocks x modes items that all read a
// small IntraEdge buffer (partition.rs:600-637) and write a packed w x h prediction.  The
// edge buffer is staged in shared memory; the intra-edge filter and the 2x edge upsampler
// (predict.rs:1203-1266) run thread-parallel over the edge (each output tap reads only the
// unfiltered copy), then every thread interpolates its pixels.  All arithmetic is the
// reference's integer arithmetic, including its index quirks (saturating left index, the
// `base + offset == -2` special case in zone 2).
#include "common.cuh"

namespace {

enum { DC_PRED = 0, V_PRED, H_PRED, D45_PRED, D135_PRED, D113_PRED, D157_PRED, D203_PRED, D67_PRED,
       SMOOTH_PRED, SMOOTH_V_PRED, SMOOTH_H_PRED, PAETH_PRED, UV_CFL_PRED };
enum { VAR_NONE = 0, VAR_LEFT, VAR_TOP, VAR_BOTH };
constexpr int kMaxTx = 64;
constexpr int kEdgeLen = 4 * kMaxTx + 1;

// predict.rs:603-624 (AV1 Sm_Weights_Tx_*), indexed [size + i]
__constant__ uint8_t kSmWeights[2 * kMaxTx] = {
    0, 0, 255, 128, 255, 149, 85, 64, 255, 197, 146, 105, 73, 50, 37, 32,
    255, 225, 196, 170, 145, 123, 102, 84, 68, 54, 43, 33, 26, 20, 17, 16,
    255, 240, 225, 210, 196, 182, 169, 157, 145, 133, 122, 111, 101, 92, 83, 74,
    66, 59, 52, 45, 39, 34, 29, 25, 21, 17, 14, 12, 10, 9, 8, 8,
    255, 248, 240, 233, 225, 218, 210, 203, 196, 189, 182, 176, 169, 163, 156,
    150, 144, 138, 133, 127, 121, 116, 111, 106, 101, 96, 91, 86, 82, 77, 73, 69,
    65, 61, 57, 54, 50, 47, 44, 41, 38, 35, 32, 29, 27, 25, 22, 20, 18, 16, 15,
    13, 12, 10, 9, 8, 7, 6, 6, 5, 5, 4, 4, 4};

// predict.rs:1268-1299, indexed by angle (0 where undefined)
__constant__ short kDrDerivative[91] = {
    0, 0, 0, 1023, 0, 0, 547, 0, 0, 372, 0, 0, 0, 0, 273, 0, 0, 215, 0, 0, 178, 0, 0, 151, 0, 0, 132,
    0, 0, 116, 0, 0, 102, 0, 0, 0, 90, 0, 0, 80, 0, 0, 71, 0, 0, 64, 0, 0, 57, 0, 0, 51, 0, 0, 45, 0,
    0, 0, 40, 0, 0, 35, 0, 0, 31, 0, 0, 27, 0, 0, 23, 0, 0, 19, 0, 0, 15, 0, 0, 0, 0, 11, 0, 0, 7, 0,
    0, 3, 0, 0, 0};

__device__ __forceinline__ int dr_derivative(int a) { return (a >= 0 && a <= 90) ? kDrDerivative[a] : 0; }

// predict.rs:1125-1186
__device__ int ief_strength(int width, int height, int smooth, int angle_delta) {
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
__device__ int ief_upsample(int width, int height, int smooth, int angle_delta) {
  const int wh = width + height, d = abs(angle_delta);
  if (d == 0 || d >= 40) return 0;
  return smooth ? wh <= 8 : wh <= 16;
}

struct IpredArgs {
  const void *edges;           // n_edges x kEdgeLen pixels
  const b200_intra_item *items;
  const short *ac;             // CfL ac blocks, w*h each
  void *out;                   // n x h x w pixels
  size_t n;
  int w, h, bit_depth;
  int plane_w, plane_h;
};

// filter_edge (predict.rs:1203-1232): dst[i] for i in 1..size from the unfiltered src.
__device__ void filter_edge_par(const int *src, int *dst, int len, int size, int strength) {
  for (int i = threadIdx.x; i < len; i += blockDim.x) {
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
__device__ void upsample_edge_par(const int *src, int *dst, int size, int maxv) {
  for (int i = threadIdx.x; i <= size; i += blockDim.x) {
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

template <typename T>
__global__ void __launch_bounds__(128) ipred_kernel(IpredArgs a) {
  __shared__ int s_edge[kEdgeLen];      // raw IntraEdge buffer, top-left at [128]
  __shared__ int s_af[2][kEdgeLen];     // above: filtered / upsampled
  __shared__ int s_lf[2][kEdgeLen];     // left (index 0 = top-left, growing downwards)
  __shared__ int s_dc;
  const int w = a.w, h = a.h;
  const int maxv = (1 << a.bit_depth) - 1;
  for (size_t it = blockIdx.x; it < a.n; it += gridDim.x) {
    const b200_intra_item item = a.items[it];
    const T *edge = (const T *)a.edges + (size_t)item.edge * kEdgeLen;
    __syncthreads();
    for (int i = threadIdx.x; i < kEdgeLen; i += blockDim.x) s_edge[i] = (int)edge[i];
    __syncthreads();
    const int left_len = item.left_len, above_len = item.above_len;
    const int *above = s_edge + 2 * kMaxTx + 1;
    const int top_left = s_edge[2 * kMaxTx];
    // left(k) for k = 0 at the row next to the top-left pixel, growing downwards:
    // the reference's bottom->top slice element left[len-1-k]
    auto leftv = [&](int k) { return s_edge[2 * kMaxTx - 1 - k]; };
    const int ls_n = min(left_len, h);  // left_slice length
    T *out = (T *)a.out + it * (size_t)w * h;
    const int mode = item.mode, variant = item.variant, angle = item.angle;

    const bool dc_like = mode == DC_PRED || mode == UV_CFL_PRED;
    if (dc_like) {
      if (threadIdx.x == 0) {
        unsigned v;
        if (variant == VAR_NONE) {
          v = 128u << (a.bit_depth - 8);
        } else if (variant == VAR_LEFT) {  // predict.rs:815-827: whole slice, divided by height
          unsigned s = 0;
          for (int k = 0; k < ls_n; k++) s += (unsigned)leftv(k);
          v = (s + (unsigned)(h >> 1)) / (unsigned)h;
        } else if (variant == VAR_TOP) {
          unsigned s = 0;
          for (int k = 0; k < w; k++) s += (unsigned)above[k];
          v = (s + (unsigned)(w >> 1)) / (unsigned)w;
        } else {
          unsigned s = 0;
          for (int k = 0; k < h; k++) s += (unsigned)leftv(k);
          for (int k = 0; k < w; k++) s += (unsigned)above[k];
          v = (s + (unsigned)((w + h) >> 1)) / (unsigned)(w + h);
        }
        s_dc = (int)(T)v;
      }
      __syncthreads();
      const int avg = s_dc;
      const short alpha = (short)angle;
      const short *ac = (mode == UV_CFL_PRED && alpha != 0) ? a.ac + (size_t)item.ac * w * h : nullptr;
      for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
        int v = avg;
        if (ac) {  // pred_cfl_inner, predict.rs:1065-1088 + get_scaled_luma_q0 :626-635
          const int q6 = (int)alpha * (int)ac[i];
          const int q0 = (abs(q6) + 32) >> 6;
          v = min(max(avg + (q6 < 0 ? -q0 : q0), 0), maxv);
        }
        out[i] = (T)v;
      }
      continue;
    }

    const bool directional = mode >= V_PRED && mode <= D67_PRED &&
                             !(mode == V_PRED && angle == 90) && !(mode == H_PRED && angle == 180);
    if (!directional) {
      for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
        const int r = i / w, c = i - r * w;
        int v;
        if (mode == V_PRED) {
          v = above[c];
        } else if (mode == H_PRED) {
          v = leftv(r);
        } else if (mode == PAETH_PRED) {  // predict.rs:860-887
          const int l = leftv(r), t = above[c];
          const int base = t + l - top_left;
          const int pl = abs(base - l), pt = abs(base - t), ptl = abs(base - top_left);
          v = (pl <= pt && pl <= ptl) ? l : (pt <= ptl ? t : top_left);
        } else if (mode == SMOOTH_PRED) {  // predict.rs:889-944
          const unsigned below = (unsigned)leftv(h - 1), right = (unsigned)above[w - 1];
          const unsigned wh_ = kSmWeights[h + r], ww_ = kSmWeights[w + c];
          const unsigned p = wh_ * (unsigned)above[c] + (256u - wh_) * below +
                             ww_ * (unsigned)leftv(r) + (256u - ww_) * right;
          v = (int)((p + 256u) >> 9);
        } else if (mode == SMOOTH_H_PRED) {
          const unsigned ww_ = kSmWeights[w + c];
          v = (int)((ww_ * (unsigned)leftv(r) + (256u - ww_) * (unsigned)above[w - 1] + 128u) >> 8);
        } else {  // SMOOTH_V_PRED
          const unsigned wh_ = kSmWeights[h + r];
          v = (int)((wh_ * (unsigned)above[c] + (256u - wh_) * (unsigned)leftv(h - 1) + 128u) >> 8);
        }
        out[i] = (T)v;
      }
      continue;
    }

    // ---- pred_directional (predict.rs:1301-1505)
    const int p_angle = angle;
    const int enable = item.ief >= 0;
    const int smooth = item.ief > 0;
    const int flen = (w + h) * 2 + 1;
    const int llb_n = min(left_len, w + h);  // left_and_left_below slice length
    int up_above = 0, up_left = 0;
    int cur_a = 0, cur_l = 0;  // which of the two scratch buffers holds the current edge
    if (enable) {
      const int a_len = min(above_len, flen - 1), l_len = min(llb_n, flen - 1);
      for (int i = threadIdx.x; i < flen; i += blockDim.x) {
        s_af[0][i] = (i >= 1 && i <= a_len) ? above[i - 1] : 0;
        s_lf[0][i] = (i >= 1 && i <= l_len) ? leftv(i - 1) : 0;
      }
      __syncthreads();
      if (p_angle != 90 && p_angle != 180) {
        if (threadIdx.x == 0) {
          s_af[0][0] = top_left;
          s_lf[0][0] = top_left;
        }
        __syncthreads();
        const int aw = a.plane_w - 1 - item.x + 1, ah = a.plane_h - 1 - item.y + 1;
        const int num_above = min(w, aw) + (p_angle < 90 ? h : 0) + 1;
        const int num_left = min(h, ah) + (p_angle > 180 ? w : 0) + 1;
        filter_edge_par(s_af[0], s_af[1], flen, num_above, ief_strength(w, h, smooth, p_angle - 90));
        filter_edge_par(s_lf[0], s_lf[1], flen, num_left, ief_strength(w, h, smooth, p_angle - 180));
        cur_a = cur_l = 1;
        __syncthreads();
      }
      up_above = ief_upsample(w, h, smooth, p_angle - 90);
      up_left = ief_upsample(w, h, smooth, p_angle - 180);
      if (up_above) {
        const int n = w + (p_angle < 90 ? h : 0);
        // entries past 2*n keep their previous values in the reference (in-place update)
        for (int i = threadIdx.x; i < flen; i += blockDim.x) s_af[cur_a ^ 1][i] = s_af[cur_a][i];
        __syncthreads();
        upsample_edge_par(s_af[cur_a], s_af[cur_a ^ 1], n, maxv);
        cur_a ^= 1;
      }
      if (up_left) {
        const int n = h + (p_angle > 180 ? w : 0);
        for (int i = threadIdx.x; i < flen; i += blockDim.x) s_lf[cur_l ^ 1][i] = s_lf[cur_l][i];
        __syncthreads();
        upsample_edge_par(s_lf[cur_l], s_lf[cur_l ^ 1], n, maxv);
        cur_l ^= 1;
      }
      __syncthreads();
    }
    const int *af = s_af[cur_a];
    const int *lf = s_lf[cur_l];
    // Edge accessors in the reference's index space.
    // above_edge[k]: filtered buffer when enabled, else the raw above slice.
    auto above_at = [&](int k) { return enable ? af[k] : above[k]; };
    // left_edge is the REVERSED buffer: left_edge[l - m] == (enabled ? lf[m] : leftv(m)) with
    // l = len - 1; left_edge[0] / [1] are the far (bottom) end.
    const int lel = enable ? flen : llb_n;
    auto left_fwd = [&](int m) { return enable ? lf[m] : leftv(m); };     // m counted from the top
    auto left_rev = [&](int idx) { return left_fwd(lel - 1 - idx); };      // reference index
    const int dx = p_angle < 90 ? dr_derivative(p_angle)
                   : (p_angle > 90 && p_angle < 180) ? dr_derivative(180 - p_angle) : 0;
    const int dy = (p_angle > 90 && p_angle < 180) ? dr_derivative(p_angle - 90)
                   : p_angle > 180 ? dr_derivative(270 - p_angle) : 0;
    const int off_a = enable << up_above, off_l = enable << up_left;
    for (int i2 = threadIdx.x; i2 < w * h; i2 += blockDim.x) {
      const int i = i2 / w, j = i2 - i * w;
      int v;
      if (p_angle < 90) {
        const int idx = (i + 1) * dx;
        const int base = (idx >> (6 - up_above)) + (j << up_above);
        const int shift = ((idx << up_above) >> 1) & 31;
        const int max_base_x = (h + w - 1) << up_above;
        if (base < max_base_x)
          v = (above_at(base + off_a) * (32 - shift) + above_at(base + 1 + off_a) * shift + 16) >> 5;
        else
          v = above_at(max_base_x + off_a);
      } else if (p_angle < 180) {
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
      } else {
        const int idx = (j + 1) * dy;
        const int base = (idx >> (6 - up_left)) + (i << up_left);
        const int shift = ((idx << up_left) >> 1) & 31;
        const int l = lel - 1;
        const int ia = max(l - (base + off_l), 0), ib = max(l - (base + off_l + 1), 0);  // saturating_sub
        v = (left_rev(ia) * (32 - shift) + left_rev(ib) * shift + 16) >> 5;
      }
      out[i2] = (T)min(max(v, 0), maxv);
    }
  }
}

// pred_cfl_ac (predict.rs:1020-1063): one CTA per block.
struct CflAcArgs {
  const void *luma;
  int stride;
  const b200_block *blocks;  // luma position of each block
  size_t n;
  int bw, bh, w_pad, h_pad, xdec, ydec;
  short *ac;
};

template <typename T>
__global__ void __launch_bounds__(128) cfl_ac_kernel(CflAcArgs a) {
  __shared__ int s_sum[4];
  __shared__ int s_avg;
  const int bw = a.bw, bh = a.bh, xdec = a.xdec, ydec = a.ydec;
  const int max_luma_x = max((bw - a.w_pad * 4) << xdec, 8) - (1 << xdec);
  const int max_luma_y = max((bh - a.h_pad * 4) << ydec, 8) - (1 << ydec);
  int shift = 0;
  for (int v = bw; v > 1; v >>= 1) shift++;
  for (int v = bh; v > 1; v >>= 1) shift++;
  for (size_t blk = blockIdx.x; blk < a.n; blk += gridDim.x) {
    const b200_block b = a.blocks[blk];
    const T *luma = (const T *)a.luma + (long long)b.y * a.stride + b.x;
    short *ac = a.ac + blk * (size_t)bw * bh;
    int local = 0;
    for (int i = threadIdx.x; i < bw * bh; i += blockDim.x) {
      const int sy = i / bw, sx = i - sy * bw;
      const int y = min(sy << ydec, max_luma_y), x = min(sx << xdec, max_luma_x);
      short s = (short)luma[(long long)y * a.stride + x];
      if (xdec) s = (short)(s + (short)luma[(long long)y * a.stride + x + 1]);
      if (ydec) s = (short)(s + (short)luma[(long long)(y + 1) * a.stride + x] + (short)luma[(long long)(y + 1) * a.stride + x + 1]);
      s = (short)(s << (3 - xdec - ydec));
      ac[i] = s;
      local += s;
    }
    local = (int)warp_sum_u32((uint32_t)local);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
      int sum = 0;
      for (int k = 0; k < (int)(blockDim.x >> 5); k++) sum += s_sum[k];
      s_avg = (short)((sum + (1 << (shift - 1))) >> shift);
    }
    __syncthreads();
    const short avg = (short)s_avg;
    for (int i = threadIdx.x; i < bw * bh; i += blockDim.x) ac[i] = (short)(ac[i] - avg);
  }
}

bool valid_tx_dim(int v) { return v == 4 || v == 8 || v == 16 || v == 32 || v == 64; }

}  // namespace

extern "C" int b200_predict_intra_dev(b200_ctx *ctx, const void *d_edges, const b200_intra_item *d_items,
                                      size_t nitems, const int16_t *d_ac, int w, int h, int bit_depth,
                                      int plane_w, int plane_h, void *d_out) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, valid_tx_dim(w) && valid_tx_dim(h), "tx block %dx%d not a TxSize", w, h);
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  if (nitems == 0) return B200_OK;
  B200_REQUIRE(ctx, d_edges && d_items && d_out, "NULL argument");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  IpredArgs a;
  a.edges = d_edges;
  a.items = d_items;
  a.ac = d_ac;
  a.out = d_out;
  a.n = nitems;
  a.w = w;
  a.h = h;
  a.bit_depth = bit_depth;
  a.plane_w = plane_w;
  a.plane_h = plane_h;
  const int grid = (int)std::min<size_t>(nitems, (size_t)ctx->num_sms * 32);
  if (bit_depth == 8)
    ipred_kernel<uint8_t><<<grid, 128, 0, ctx->stream>>>(a);
  else
    ipred_kernel<uint16_t><<<grid, 128, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_pred_cfl_ac_dev(b200_ctx *ctx, const b200_plane *luma, const b200_block *d_blocks,
                                    size_t nblocks, int bw, int bh, int w_pad, int h_pad, int xdec,
                                    int ydec, int16_t *d_ac) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, luma && luma->data, "bad luma plane");
  B200_REQUIRE(ctx, bw >= 4 && bh >= 4 && bw <= 32 && bh <= 32 && (bw & (bw - 1)) == 0 && (bh & (bh - 1)) == 0,
               "CfL block %dx%d out of range", bw, bh);
  B200_REQUIRE(ctx, (xdec == 0 || xdec == 1) && (ydec == 0 || ydec == 1) && !(ydec && !xdec), "bad decimation");
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && d_ac, "NULL argument");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  CflAcArgs a{luma->data, luma->stride, d_blocks, nblocks, bw, bh, w_pad, h_pad, xdec, ydec, d_ac};
  const int grid = (int)std::min<size_t>(nblocks, (size_t)ctx->num_sms * 32);
  if (luma->bpp == 1)
    cfl_ac_kernel<uint8_t><<<grid, 128, 0, ctx->stream>>>(a);
  else
    cfl_ac_kernel<uint16_t><<<grid, 128, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// Per-call form mirroring dispatch_predict_intra (predict.rs:705-784): host pointers, dst stride
// in BYTES; edge = the reference's IntraEdge buffer (4*64+1 pixels, top-left at [128]).
extern "C" void b200_predict_intra(int mode, int variant, void *dst, ptrdiff_t dst_stride, int w, int h,
                                   int bit_depth, const int16_t *ac, int angle, int ief,
                                   const void *edge, int left_len, int above_len, int plane_w,
                                   int plane_h, int dst_x, int dst_y) {
  b200_ctx *ctx = b200_default_ctx();
  const int bpp = bit_depth == 8 ? 1 : 2;
  const size_t edge_bytes = b200_align_up((size_t)kEdgeLen * bpp, 256);
  const size_t ac_bytes = b200_align_up((size_t)w * h * 2, 256);
  void *dbase = nullptr;
  int st = B200_OK;
  if (cudaSetDevice(ctx->device) != cudaSuccess ||
      cudaMallocAsync(&dbase, edge_bytes + ac_bytes + 256 + (size_t)w * h * bpp, ctx->stream) != cudaSuccess)
    st = b200_fail(ctx, B200_ERR_CUDA, "alloc failed");
  uint8_t *d_edge = (uint8_t *)dbase, *d_ac = d_edge + edge_bytes, *d_item = d_ac + ac_bytes,
          *d_out = d_item + 256;
  b200_intra_item item{};
  item.edge = 0;
  item.ac = 0;
  item.x = (int16_t)dst_x;
  item.y = (int16_t)dst_y;
  item.angle = (int16_t)angle;
  item.mode = (uint8_t)mode;
  item.variant = (uint8_t)variant;
  item.ief = (int8_t)ief;
  item.left_len = (uint8_t)left_len;
  item.above_len = (uint8_t)above_len;
  if (!st && (cudaMemcpyAsync(d_edge, edge, (size_t)kEdgeLen * bpp, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess ||
              cudaMemcpyAsync(d_item, &item, sizeof item, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess ||
              (ac && cudaMemcpyAsync(d_ac, ac, (size_t)w * h * 2, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess)))
    st = b200_fail(ctx, B200_ERR_CUDA, "H2D copy failed");
  if (!st)
    st = b200_predict_intra_dev(ctx, d_edge, (const b200_intra_item *)d_item, 1, (const int16_t *)d_ac, w, h,
                                bit_depth, plane_w, plane_h, d_out);
  if (!st && cudaMemcpy2DAsync(dst, (size_t)dst_stride, d_out, (size_t)w * bpp, (size_t)w * bpp, h,
                               cudaMemcpyDeviceToHost, ctx->stream) != cudaSuccess)
    st = b200_fail(ctx, B200_ERR_CUDA, "D2H copy failed");
  if (dbase) cudaFreeAsync(dbase, ctx->stream);
  if (!st && cudaStreamSynchronize(ctx->stream) != cudaSuccess) st = b200_fail(ctx, B200_ERR_CUDA, "sync failed");
  if (st) {
    fprintf(stderr, "b200rdo: FATAL: predict_intra failed: %s\n", b200_last_error(ctx));
    abort();
  }
}
