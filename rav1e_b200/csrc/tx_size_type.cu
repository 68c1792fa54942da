// tx_size_type.cu — the intra transform size and type decision for sm_90a: rdo_tx_size_type
// (src/rdo.rs:725-802) with rdo_tx_type_decision (:1701-1823) and the luma loop of write_tx_blocks /
// encode_tx_block (src/encoder.rs:2243-2311, :1404-1658) for a batch of (block, mode, quantizer) items.
// Contract and rules: include/b200rdo.h (b200_intra_tx_size_type_dev).
//
// Every candidate (ladder level, tx type) of an item starts from the same coefficient-context checkpoint,
// so all of them are evaluated in parallel and the decision rules run afterwards:
//   1. bucket: one thread per item appends each (item, level) of its size ladder to its TxSize's list;
//   2. one launch per TxSize (the transform stays compile-time, as in encode_tx.cu): one CTA per
//      (item, level, type) walks the candidate's transform blocks in raster order — edges
//      (intra_edges_dev.cuh; pixels inside the partition from the candidate's own reconstruction in
//      shared memory), prediction (ipred_dev.cuh), residual and forward transform (fwd_txfm_dev.cuh),
//      quantize (quantize_dev.cuh), the coefficient counter (coeff_rate_dev.cuh), the inverse transform
//      into the shared reconstruction (inv_txfm_dev.cuh) and the tx-domain distortion; then the
//      pixel-domain distortion (rdo_dist_dev.cuh) and the cost.  Nothing per transform block leaves
//      shared memory; the candidate's (rate, distortion, rd) goes to its record;
//   3. decide: one thread per item applies the early exit and the strict `<` rules in the reference's
//      order to the records.
#include <cfloat>

#include "coeff_rate_dev.cuh"
#include "fwd_txfm_dev.cuh"
#include "intra_edges_dev.cuh"
#include "inv_txfm_dev.cuh"
#include "ipred_dev.cuh"
#include "quantize_dev.cuh"
#include "rdo_dist_dev.cuh"

namespace {

using namespace ipred;
using intra_edges::EdgeLens;

constexpr int kThreads = 64;  // one thread per column / row of the largest transform
constexpr int kTypes = 7;     // RAV1E_TX_TYPES
constexpr int kCands = 3 * kTypes;
static_assert(sizeof(b200_tx_item) == 52 && sizeof(b200_tx_best) == 16 && sizeof(b200_tx_cand) == 24,
              "record layout");

// max_txsize_rect_lookup and sub_tx_size_map (context/transform_unit.rs:60-105), RAV1E_TX_TYPES
__constant__ uint8_t kMaxTxOf[22] = {0, 5, 6, 1, 7, 8, 2, 9, 10, 3, 11, 12, 4, 4, 4, 4, 13, 14, 15, 16, 17, 18};
__constant__ uint8_t kSubTx[19] = {0, 0, 1, 2, 3, 0, 0, 1, 1, 2, 2, 3, 3, 5, 6, 7, 8, 9, 10};
__constant__ uint8_t kTxTypes[kTypes] = {0, 1, 2, 3, 9, 10, 11};

struct TstArgs {
  intra_edges::EdgeGeom rec;  // the region of rec
  const void *src;            // src pixel at the region's (0, 0)
  int src_stride;
  int frame_w, frame_h, w_in_b, h_in_b, mi_w, mi_h;
  int dist_mode, reduced;
  double lambda;
  uint32_t dist_scale;
  const uint32_t *scale;  // per frame 4x4, NULL: default scales
  size_t scale_stride;
  const b200_coeff_cdfs *cdfs;
  size_t ncdfs;
  const b200_tx_item *items;
  size_t n;
  b200_tx_cand *cands;  // n x 21
  uint32_t *counts;     // per TxSize: entries of its list
  uint32_t *lists;      // 19 x n: item * 3 + level
  ScanTables st;
};
// per-launch (TxSize) tables, index = position in RAV1E_TX_TYPES
struct SizeArgs {
  int tx_size;
  const uint16_t *iscan[3];
  TxSetup tx[kTypes];
  InvArgs inv[kTypes];
};

__device__ __forceinline__ bool tx_item_valid(const b200_tx_item &it, const TstArgs &a) {
  if (it.bsize >= 22 || (it.bsize >= 13 && it.bsize <= 15) || it.mode >= 13) return false;
  if (it.x < 0 || it.y < 0 || it.x >= a.rec.rect_w || it.y >= a.rec.rect_h || (it.x & 3) || (it.y & 3)) return false;
  if (it.dc_quant < 1 || it.dc_quant > 65535 || it.ac_quant < 1 || it.ac_quant > 65535) return false;
  return it.snapshot < a.ncdfs;
}
// level l of the item's size ladder, -1 past its end
__device__ __forceinline__ int ladder_size(int bsize, int l) {
  int t = kMaxTxOf[bsize];
  for (int i = 0; i < l; i++) {
    const int nx = kSubTx[t];
    if (nx == t) return -1;
    t = nx;
  }
  return t;
}
// RAV1E_TX_TYPES[k] in the list rdo_tx_size_type passes for size t (rdo.rs:751-761, av1_tx_used)
__device__ __forceinline__ bool in_list(int t, int k, int skip, int reduced) {
  const int set = tx_set_of(t, 0, reduced);  // 0 DCTONLY, 2 INTRA_2, 3 INTRA_1
  if (set == 0 || skip) return k == 0;
  return set == 3 || k <= 4;
}
__device__ __forceinline__ uint32_t bias_at(const TstArgs &a, int fx4, int fy4) {  // distortion_scale
  return a.scale ? a.scale[(size_t)fy4 * a.scale_stride + fx4] : 1u << 14;
}
__device__ __forceinline__ unsigned long long scale_mul(uint32_t scale, unsigned long long d) {  // mul_u64
  return ((unsigned long long)scale * d + (1u << 13)) >> 14;
}

__global__ void tx_bucket_kernel(const __grid_constant__ TstArgs a) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (size_t)gridDim.x * blockDim.x) {
    const b200_tx_item it = a.items[i];
    if (!tx_item_valid(it, a)) continue;
    for (int l = 0; l < 3; l++) {
      const int t = ladder_size(it.bsize, l);
      if (t < 0) break;
      a.lists[(size_t)t * a.n + atomicAdd(&a.counts[t], 1u)] = (uint32_t)(i * 3 + l);
    }
  }
}

template <int W, int H, typename Px, typename CoefT>
struct TstSmem {
  static constexpr int PITCH = W + 1;
  static constexpr int CODED = (W < 32 ? W : 32) * (H < 32 ? H : 32);
  WarpSmem ws;  // the counter's CDFs, packed symbols, levels and context window
  int tile[H * PITCH];
  CoefT coef[W * H], q[CODED], r[CODED];
  int edge[kEdgeLen], fa[kEdgeLen], fl[kEdgeLen], sa[kEdgeLen], sl[kEdgeLen];
  Px rec[kMaxTx * kMaxTx];  // the partition's reconstruction, stride 64
  unsigned long long raw, acc;
  uint16_t eob;
  int dc;
};

template <int W, int H, typename Px>
__global__ void __launch_bounds__(kThreads, 1) tx_candidate_kernel(const __grid_constant__ TstArgs a,
                                                                const __grid_constant__ SizeArgs z) {
  using CoefT = typename std::conditional<sizeof(Px) == 1, int16_t, int32_t>::type;
  using S = TstSmem<W, H, Px, CoefT>;
  constexpr int PITCH = S::PITCH;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  S &s = *reinterpret_cast<S *>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int tsz = z.tx_size, bd = a.rec.bit_depth;
  const size_t nslots = (size_t)a.counts[tsz] * kTypes;
  const Px *reg = (const Px *)a.rec.data, *src = (const Px *)a.src;
  for (size_t slot = blockIdx.x; slot < nslots; slot += gridDim.x) {
    const uint32_t e = a.lists[(size_t)tsz * a.n + slot / kTypes];
    const int k = (int)(slot % kTypes), l = (int)(e % 3);
    const size_t i = e / 3;
    const b200_tx_item it = a.items[i];
    if (!in_list(tsz, k, it.skip, a.reduced)) continue;
    const int type = kTxTypes[k], kind = type < 10 ? 0 : ((type & 1) ? 2 : 1);
    const int x0 = it.x, y0 = it.y, bw = intra_edges::kBsW[it.bsize], bh = intra_edges::kBsH[it.bsize];
    const bool need_recon_pixel = W != bw || H != bh;
    QuantArgs q{};
    q.scan = a.st.p[tsz][kind];
    q.iscan = z.iscan[kind];
    quant_params(W, H, it.dc_quant, it.ac_quant, 1, sizeof(CoefT) == 4, q);
    InvArgs inv = z.inv[k];
    inv.dst_stride = kMaxTx;
    const TxSetup &tx = z.tx[k];
    const uint16_t *g = reinterpret_cast<const uint16_t *>(a.cdfs + it.snapshot);
    uint64_t m0 = 0, m1 = 0, m2 = 0;
    Coder w{32768u, 0};  // WriterCounter::new()
    unsigned long long txd = 0;
    __syncthreads();  // the previous candidate's readers are done with shared memory
    if (warp == 0) {  // the checkpoint: the item's context windows and a fresh copy of its snapshot
      if (lane < 16) {
        s.ws.above[0][lane] = it.above[lane];
        s.ws.left[0][lane] = it.left[lane];
      }
      __syncwarp();
      count_begin(m0, s.ws.cdf, g, lane);
    }
    // region pixels for the edges: inside the partition this candidate's own reconstruction
    auto PX = [&](int yy, int xx) -> unsigned {
      const int dx = xx - x0, dy = yy - y0;
      if (dx >= 0 && dx < bw && dy >= 0 && dy < bh) return (unsigned)s.rec[dy * kMaxTx + dx];
      return (unsigned)reg[(long long)yy * a.rec.stride + xx];
    };
    for (int by = 0; by < bh / H; by++)
      for (int bx = 0; bx < bw / W; bx++) {
        const int px = x0 + bx * W, py = y0 + by * H;
        if ((px >> 2) >= a.mi_w || (py >> 2) >= a.mi_h) continue;  // encoder.rs:2282
        // ---- get_intra_edges + predict_intra (encoder.rs:1468-1499, predict.rs:205-249)
        b200_edge_item ei{};
        ei.po_x = (int16_t)px;
        ei.po_y = (int16_t)py;
        ei.part_x = (int16_t)(x0 >> 2);
        ei.part_y = (int16_t)(y0 >> 2);
        ei.bx = (uint8_t)bx;
        ei.by = (uint8_t)by;
        ei.bsize = it.bsize;
        ei.tx_size = (uint8_t)tsz;
        ei.mode = it.mode;
        ei.enable_ief = it.ief >= 0;
        __syncthreads();  // the previous block's readers of the edges / tile are done
        const EdgeLens lens = intra_edges::gather_intra_edge_px(a.rec, ei, tid, kThreads, s.edge, PX);
        __syncthreads();
        const int variant = (px == 0 && py == 0) ? VAR_NONE : py == 0 ? VAR_LEFT : px == 0 ? VAR_TOP : VAR_BOTH;
        int mode = it.mode;
        if (mode == PAETH_PRED)
          mode = variant == VAR_NONE ? DC_PRED : variant == VAR_TOP ? V_PRED : variant == VAR_LEFT ? H_PRED : PAETH_PRED;
        const int angle = mode >= V_PRED && mode <= D67_PRED ? intra_edges::kModeAngle[mode] : 0;
        const int ief = it.mode >= V_PRED && it.mode <= D67_PRED ? it.ief : -1;
        if (tid == 0) s.dc = ipred_dc(s.edge, variant, W, H, lens.left, bd);
        IpredPix p = ipred_setup(s.edge, mode, angle, ief, lens.left, W, H, bd, s.fa, s.fl, 0);
        if (p.directional && p.enable)
          ipred_filter_edges(CtaGroup(), p, lens.above, a.rec.plane_w, a.rec.plane_h, a.rec.rect_x + px,
                             a.rec.rect_y + py, s.sa, s.sl, s.fa, s.fl);
        __syncthreads();
        p.dc = s.dc;
        Px *dst = s.rec + (py - y0) * kMaxTx + (px - x0);
        for (int idx = tid; idx < W * H; idx += kThreads) {
          const int r = idx / W, c = idx - r * W;
          dst[r * kMaxTx + c] = (Px)ipred_pixel(p, r, c);
        }
        __syncthreads();
        // ---- residual (zero when invisible) + forward transform (forward.rs:94-160), as encode_tx.cu
        const int fx = a.rec.rect_x + px, fy = a.rec.rect_y + py;
        const bool visible = fx < a.frame_w && fy < a.frame_h;
        if (tid < W) {
          TXV c[H];
#pragma unroll
          for (int r = 0; r < H; r++) {
            const int rr = tx.ud_flip ? H - 1 - r : r;
            const int d = visible ? (int)src[(long long)(py + rr) * a.src_stride + px + tid] - (int)dst[rr * kMaxTx + tid]
                                  : 0;
            c[r] = round_shift_bit(d, tx.bit0);
          }
          run_1d<H>(tx.col_type, c);
          const int cc = tx.lr_flip ? W - 1 - tid : tid;
#pragma unroll
          for (int r = 0; r < H; r++) s.tile[r * PITCH + cc] = round_shift_bit(c[r], tx.bit1);
        }
        __syncthreads();
        if (tid < H) {
          TXV c[W];
#pragma unroll
          for (int kk = 0; kk < W; kk++) c[kk] = s.tile[tid * PITCH + kk];
          run_1d<W>(tx.row_type, c);
          const int off0 = CoefOrder<W, H>::row(tid);
#pragma unroll
          for (int kk = 0; kk < W; kk++) s.coef[off0 + CoefOrder<W, H>::col(kk)] = (CoefT)round_shift_bit(c[kk], tx.bit2);
        }
        __syncthreads();
        // ---- quantize -> dequantize -> raw tx distortion, then write_coeffs_lv_map counted (warp 0)
        if (warp == 0) {
          quantize_block_warp<CoefT>(q, s.coef, s.q, s.r, &s.eob, &s.raw, lane);
          __syncwarp();
          b200_coeff_item ci{};
          ci.eob = s.eob;
          ci.tx_size = (uint8_t)tsz;
          ci.tx_type = (uint8_t)type;
          ci.plane_bsize = it.bsize;
          ci.mode = it.mode;
          ci.reduced_tx_set = (uint8_t)a.reduced;
          ci.x4 = (uint8_t)(bx * W / 4);
          ci.y4 = (uint8_t)(by * H / 4);
          ci.clip_w4 = (uint8_t)(min((a.w_in_b - (fx >> 2)) << 2, W) >> 2);  // frame_clipped_txw, encoder.rs:1561
          ci.clip_h4 = (uint8_t)(min((a.h_in_b - (fy >> 2)) << 2, H) >> 2);
          count_item<CoefT>(s.ws, m0, m1, m2, g, a.st, ci, s.q, w, nullptr, lane);
          if (lane == 0 && a.dist_mode == 0 && visible)  // RawDistortion * bias * dist_scale[0]
            txd += scale_mul(a.dist_scale, scale_mul(bias_at(a, fx >> 2, fy >> 2), s.raw));
        }
        __syncthreads();
        // ---- inverse_transform_add into the reconstruction (encoder.rs:1598-1609)
        if (s.eob > 0 && (need_recon_pixel || a.dist_mode != 0)) {
          if (tid < H) inv_row_pass_ptr<W, H, CoefT>(inv, s.r, tid, s.tile);
          __syncthreads();
          if (tid < W) inv_col_pass_ptr<W, H, Px>(inv, dst, tid, s.tile);
        }
      }
    __syncthreads();
    // ---- compute_distortion's luma term (rdo.rs:254-293) over the visible block
    unsigned long long dist = txd;
    if (a.dist_mode != 0) {
      const int fx0 = a.rec.rect_x + x0, fy0 = a.rec.rect_y + y0;
      const int vw = fx0 + bw <= a.frame_w ? bw : fx0 >= a.frame_w ? 0 : a.frame_w - fx0;
      const int vh = fy0 + bh <= a.frame_h ? bh : fy0 >= a.frame_h ? 0 : a.frame_h - fy0;
      if (tid == 0) s.acc = 0;
      __syncthreads();
      const Px *sb = src + (long long)y0 * a.src_stride + x0;
      if (a.dist_mode == 1) {  // sse_wxh: get_weighted_sse over whole 4x4 chunks, the bias per chunk
        const int nw = vw >> 2, nh = vh >> 2;
        for (int u = tid; u < nw * nh; u += kThreads) {
          const int cy = (u / nw) * 4, cx = (u % nw) * 4;
          uint32_t sum = 0;
          for (int yy = 0; yy < 4; yy++)
            for (int xx = 0; xx < 4; xx++) {
              const int d = (int)sb[(long long)(cy + yy) * a.src_stride + cx + xx] - (int)s.rec[(cy + yy) * kMaxTx + cx + xx];
              sum += (uint32_t)(d * d);
            }
          atomicAdd(&s.acc, wsse_chunk(sum, bias_at(a, (fx0 + cx) >> 2, (fy0 + cy) >> 2)));
        }
      } else {  // cdef_dist_wxh: 8x8 steps, each boosted and biased
        const int nw = (vw + 7) >> 3, nh = (vh + 7) >> 3;
        for (int u = tid; u < nw * nh; u += kThreads) {
          const int cy = (u / nw) * 8, cx = (u % nw) * 8;
          const int kw = min(vw - cx, 8), kh = min(vh - cy, 8);
          uint32_t ss = 0, sd = 0, ss2 = 0, sd2 = 0, ssd = 0;
          for (int yy = 0; yy < kh; yy++)
            for (int xx = 0; xx < kw; xx++) {
              const uint32_t sv = sb[(long long)(cy + yy) * a.src_stride + cx + xx], dv = s.rec[(cy + yy) * kMaxTx + cx + xx];
              ss += sv;
              sd += dv;
              ss2 += sv * sv;
              sd2 += dv * dv;
              ssd += sv * dv;
            }
          uint32_t svar, dvar;
          const uint32_t sse = cdef_dist_vars(ss, sd, ss2, sd2, ssd, kw * kh, &svar, &dvar);
          const uint32_t v = apply_ssim_boost(sse, svar, dvar, bd);
          atomicAdd(&s.acc, scale_mul(bias_at(a, (fx0 + cx) >> 2, (fy0 + cy) >> 2), v));
        }
      }
      __syncthreads();
      dist = scale_mul(a.dist_scale, a.dist_mode == 1 ? wsse_finish(s.acc) : s.acc);
    }
    if (tid == 0) {  // tell_frac(end) - tell_frac(start) (ec.rs:782-798)
      const uint32_t rate = frac(w.bits + 1, w.rng) - frac(1, 32768u);
      b200_tx_cand c;
      c.rd = rd_cost(a.lambda, rate, dist);
      c.dist = dist;
      c.rate = rate;
      c.state = B200_TX_EVALUATED;
      a.cands[i * kCands + l * kTypes + k] = c;
    }
  }
}

// rdo_tx_size_type's loop over the records (rdo.rs:766-801, :1806-1821)
__global__ void tx_decide_kernel(const __grid_constant__ TstArgs a, b200_tx_best *best) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (size_t)gridDim.x * blockDim.x) {
    const b200_tx_item it = a.items[i];
    b200_tx_cand *c = a.cands + i * kCands;
    const b200_tx_cand none{0.0, 0, 0, 0};
    if (!tx_item_valid(it, a)) {
      for (int j = 0; j < kCands; j++) {
        c[j] = none;
        c[j].state = B200_TX_INVALID;
      }
      best[i] = b200_tx_best{-1.0, 0xFF, 0xFF, {0}};
      continue;
    }
    double best_rd = DBL_MAX;
    int best_size = kMaxTxOf[it.bsize], best_type = 0;
    for (int l = 0; l < 3; l++) {
      const int t = ladder_size(it.bsize, l);
      bool first = true, cut = false;
      double size_rd = DBL_MAX;
      int size_type = 0;
      for (int k = 0; k < kTypes; k++) {
        b200_tx_cand &r = c[l * kTypes + k];
        const int state = t < 0                                ? B200_TX_NOT_IN_LADDER
                          : !in_list(t, k, it.skip, a.reduced) ? B200_TX_NOT_IN_SET
                          : cut                                ? B200_TX_CUT
                                                               : B200_TX_EVALUATED;
        if (state != B200_TX_EVALUATED) {
          r = none;
          r.state = (uint32_t)state;
          continue;
        }
        const double rd = r.rd;
        if (first) {
          first = false;
          if (rd > best_rd) {  // the size's first type loses to the best size so far: skip the rest
            cut = true;
            continue;
          }
        }
        if (rd < size_rd) {
          size_rd = rd;
          size_type = kTxTypes[k];
        }
      }
      if (t >= 0 && size_rd < best_rd) {
        best_rd = size_rd;
        best_size = t;
        best_type = size_type;
      }
    }
    best[i] = b200_tx_best{best_rd, (uint8_t)best_size, (uint8_t)best_type, {0}};
  }
}

template <int W, int H>
int launch_size(b200_ctx *ctx, const TstArgs &a, int tx_size, int grid) {
  SizeArgs z{};
  z.tx_size = tx_size;
  for (int kind = 0; kind < 3; kind++) {
    const uint16_t *scan;
    if (int st = scan_tables(ctx, tx_size, kind, &scan, &z.iscan[kind])) return st;
  }
  for (int k = 0; k < kTypes; k++) {
    static const int kTy[kTypes] = {0, 1, 2, 3, 9, 10, 11};
    if (!valid_transform(tx_size, kTy[k])) continue;  // never in the size's list
    z.tx[k] = tx_setup(tx_size, kTy[k], a.rec.bit_depth);
    inv_setup(tx_size, kTy[k], a.rec.bit_depth, &z.inv[k]);
  }
  const auto go = [&](auto tag) -> int {
    using Px = decltype(tag);
    using CoefT = typename std::conditional<sizeof(Px) == 1, int16_t, int32_t>::type;
    const int smem = (int)sizeof(TstSmem<W, H, Px, CoefT>);
    if (int st = b200_smem_opt_in(ctx, (const void *)tx_candidate_kernel<W, H, Px>, smem)) return st;
    tx_candidate_kernel<W, H, Px><<<grid, kThreads, smem, ctx->stream>>>(a, z);
    B200_LAUNCH_CHECK(ctx);
    return B200_OK;
  };
  return a.rec.bit_depth > 8 ? go(uint16_t{}) : go(uint8_t{});
}

}  // namespace

extern "C" int b200_intra_tx_size_type_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src, int rect_x,
                                           int rect_y, int rect_w, int rect_h, int frame_width, int frame_height,
                                           int bit_depth, int dist_mode, int reduced_tx_set, double lambda,
                                           uint32_t dist_scale, const uint32_t *d_scale4x4, size_t scale_stride,
                                           const b200_coeff_cdfs *d_cdfs, size_t ncdfs, const b200_tx_item *d_items,
                                           size_t nitems, b200_tx_best *d_best, b200_tx_cand *d_cands) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, rec && rec->data && src && src->data, "NULL plane");
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  B200_REQUIRE(ctx, rec->bpp == (bit_depth == 8 ? 1 : 2) && src->bpp == rec->bpp, "bpp %d / %d vs bit depth %d",
               rec->bpp, src->bpp, bit_depth);
  B200_REQUIRE(ctx, rec->width == src->width && rec->height == src->height, "rec %dx%d vs src %dx%d", rec->width,
               rec->height, src->width, src->height);
  B200_REQUIRE(ctx, rect_x >= 0 && rect_y >= 0 && rect_w > 0 && rect_h > 0 && rect_x + rect_w <= rec->width &&
                        rect_y + rect_h <= rec->height,
               "region (%d, %d, %d, %d) outside the %dx%d plane", rect_x, rect_y, rect_w, rect_h, rec->width,
               rec->height);
  B200_REQUIRE(ctx, frame_width > 0 && frame_height > 0 && frame_width <= rec->width && frame_height <= rec->height,
               "frame %dx%d not inside the %dx%d plane", frame_width, frame_height, rec->width, rec->height);
  const int w_in_b = 2 * ((frame_width + 7) >> 3), h_in_b = 2 * ((frame_height + 7) >> 3);
  B200_REQUIRE(ctx, rect_x + rect_w <= 4 * w_in_b && rect_y + rect_h <= 4 * h_in_b,
               "region (%d, %d, %d, %d) past the frame's %dx%d 4x4 blocks", rect_x, rect_y, rect_w, rect_h, w_in_b,
               h_in_b);
  B200_REQUIRE(ctx, rec->pad >= kMaxTx && src->pad >= kMaxTx, "plane padding %d / %d below %d", rec->pad, src->pad,
               kMaxTx);
  B200_REQUIRE(ctx, dist_mode >= 0 && dist_mode <= 2, "dist_mode %d not 0 / 1 / 2", dist_mode);
  B200_REQUIRE(ctx, reduced_tx_set == 0 || reduced_tx_set == 1, "reduced_tx_set %d not 0 / 1", reduced_tx_set);
  B200_REQUIRE(ctx, lambda >= 0.0 && lambda <= DBL_MAX, "lambda %g not finite and >= 0", lambda);
  B200_REQUIRE(ctx, d_scale4x4 == nullptr || scale_stride >= (size_t)w_in_b, "scale stride %zu below w_in_b %d",
               scale_stride, w_in_b);
  B200_REQUIRE(ctx, nitems < (1ull << 30), "nitems %zu >= 2^30", nitems);
  if (nitems == 0) return B200_OK;
  B200_REQUIRE(ctx, d_items && d_best && d_cdfs, "NULL items / best output / CDF snapshots");
  B200_REQUIRE(ctx, ncdfs > 0, "no CDF snapshot");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  // work: the 19 list counts, the 19 lists, the candidate records when the caller keeps none
  const size_t lists_off = 128, cands_off = b200_align_up(lists_off + 19 * nitems * sizeof(uint32_t), 256);
  const size_t need = d_cands ? cands_off : cands_off + nitems * kCands * sizeof(b200_tx_cand);
  if (int st = b200_reserve_dwork(ctx, need)) return st;
  unsigned char *work = (unsigned char *)ctx->dwork;
  TstArgs a{};
  a.rec.data = (const uint8_t *)rec->data + ((long long)rect_y * rec->stride + rect_x) * rec->bpp;
  a.rec.stride = rec->stride;
  a.rec.plane_w = rec->width;
  a.rec.plane_h = rec->height;
  a.rec.rect_x = rect_x, a.rec.rect_y = rect_y, a.rec.rect_w = rect_w, a.rec.rect_h = rect_h;
  a.rec.bit_depth = bit_depth;
  a.src = (const uint8_t *)src->data + ((long long)rect_y * src->stride + rect_x) * src->bpp;
  a.src_stride = src->stride;
  a.frame_w = frame_width, a.frame_h = frame_height, a.w_in_b = w_in_b, a.h_in_b = h_in_b;
  a.mi_w = (rect_w + 3) >> 2, a.mi_h = (rect_h + 3) >> 2;
  a.dist_mode = dist_mode, a.reduced = reduced_tx_set;
  a.lambda = lambda;
  a.dist_scale = dist_scale;
  a.scale = d_scale4x4;
  a.scale_stride = scale_stride;
  a.cdfs = d_cdfs, a.ncdfs = ncdfs;
  a.items = d_items, a.n = nitems;
  a.cands = d_cands ? d_cands : (b200_tx_cand *)(work + cands_off);
  a.counts = (uint32_t *)work;
  a.lists = (uint32_t *)(work + lists_off);
  for (int t = 0; t < 19; t++) {
    static const int kKindType[3] = {0, 10, 11};  // a tx_type of each scan kind
    for (int kk = 0; kk < 3; kk++)
      if (int e = b200_scan_table_internal(ctx, t, kKindType[kk], &a.st.p[t][kk])) return e;
  }
  B200_CUDA(ctx, cudaMemsetAsync(a.counts, 0, 19 * sizeof(uint32_t), ctx->stream));
  const int igrid = (int)std::min<size_t>((nitems + 255) / 256, (size_t)ctx->num_sms * 8);
  tx_bucket_kernel<<<igrid, 256, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  const int grid = (int)std::min<size_t>(nitems * kCands, (size_t)ctx->num_sms * 16);
  for (int t = 0; t < 19; t++) {
    int st = B200_OK;
    switch (t) {
#define B200_TST(ID, W_, H_)                    \
  case ID:                                      \
    st = launch_size<W_, H_>(ctx, a, ID, grid); \
    break;
      B200_TST(0, 4, 4)
      B200_TST(1, 8, 8)
      B200_TST(2, 16, 16)
      B200_TST(3, 32, 32)
      B200_TST(4, 64, 64)
      B200_TST(5, 4, 8)
      B200_TST(6, 8, 4)
      B200_TST(7, 8, 16)
      B200_TST(8, 16, 8)
      B200_TST(9, 16, 32)
      B200_TST(10, 32, 16)
      B200_TST(11, 32, 64)
      B200_TST(12, 64, 32)
      B200_TST(13, 4, 16)
      B200_TST(14, 16, 4)
      B200_TST(15, 8, 32)
      B200_TST(16, 32, 8)
      B200_TST(17, 16, 64)
      B200_TST(18, 64, 16)
#undef B200_TST
    }
    if (st) return st;
  }
  tx_decide_kernel<<<igrid, 256, 0, ctx->stream>>>(a, d_best);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
