// fwd_txfm.cu — batched 2-D forward transforms (rav1e src/transform/forward.rs:71-161) for sm_90a.
//
// One thread owns one whole column (pass 1) and then one whole row (pass 2) of a block in
// registers and runs the straight-line lifting network on it (txfm_networks.cuh); the
// transposition between the passes goes through a padded shared-memory tile, so both the
// int16 residual loads and the coefficient stores (the reference's transposed, 32x32-chunked
// order, forward.rs:135-159) are coalesced.  A CTA of 128 threads carries 128/max(W,H) blocks
// at a time.  Warp shuffles are deliberately NOT used for the butterflies: the Daala networks
// are irregular lifting ladders with per-node constants, so a lane-per-coefficient layout
// would diverge on every step, while a thread-per-vector layout needs no communication at all
// inside a 1-D pass.
#include "fwd_txfm_dev.cuh"
#include "host_stage.cuh"

namespace {

// Several (cur, ref) plane pairs per launch (see b200_me_candidates_multi_dev): pair k owns
// blocks [block_end[k-1], block_end[k]) of the launch.
constexpr int kTxMaxPairs = 32;
struct TxPairs {
  int n;  // <= 1: TxArgs::cur / ref
  uint32_t block_end[kTxMaxPairs];
  const void *cur[kTxMaxPairs], *ref[kTxMaxPairs];
  int cur_stride[kTxMaxPairs], ref_stride[kTxMaxPairs];
};

struct TxArgs {
  // fused residual source (PLANES variants): cur - ref displaced by the full-pel winner mv
  const void *cur, *ref;
  int cur_stride, ref_stride;
  TxPairs pr;
  const b200_block *blocks;
  const b200_me_result *mv_src;
  const void *pred_packed;  // PLANES variants: prediction given as packed W x H blocks instead of a plane
  const int16_t *in;
  void *out;
  size_t n;
  size_t in_block_stride;  // elements between consecutive blocks
  int in_row_stride;       // elements between rows of a block
  int col_type, row_type;
  int ud_flip, lr_flip;
  int bit0, bit1, bit2;    // av1_round_shift_array `bit` = -shift[k]: >0 round-shift right, <0 left
};

constexpr int kTxThreads = 128;

template <int W, int H, typename CoefT, bool PLANES>
__global__ void __launch_bounds__(kTxThreads) fwd_txfm_kernel(const __grid_constant__ TxArgs a) {
  constexpr int T = W > H ? W : H;       // threads per block-transform
  constexpr int PER = kTxThreads / T;    // transforms in flight per CTA
  constexpr int PITCH = W + 1;           // padded row pitch: conflict-free transposition
  constexpr int REGION = H * PITCH + ((H * PITCH) % 2 == 0 ? 1 : 0);
  __shared__ int buf[PER * REGION];
  const int slot = threadIdx.x / T, t = threadIdx.x - slot * T;
  int *tile = buf + slot * REGION;
  const size_t stride_blk = (size_t)gridDim.x * PER;
  for (size_t base = (size_t)blockIdx.x * PER; base < a.n; base += stride_blk) {
    const size_t blk = base + slot;
    const bool valid = blk < a.n;
    // ---- columns (forward.rs:95-126)
    if (valid && t < W) {
      TXV c[H];
      if constexpr (PLANES) {
        // residual computed on the fly (encoder.rs:1533 `diff`): u8 planes pair with i16
        // coefficients, u16 planes with i32 (T::Coeff)
        using Px = typename std::conditional<sizeof(CoefT) == 2, uint8_t, uint16_t>::type;
        const b200_block b = a.blocks[blk];
        int dx = 0, dy = 0;
        if (a.mv_src && a.mv_src[blk].cost != ~0ull) {
          dx = a.mv_src[blk].mv_col / 8;
          dy = a.mv_src[blk].mv_row / 8;
        }
        const void *cur_p = a.cur, *ref_p = a.ref;
        int cur_stride = a.cur_stride, ref_stride = a.ref_stride;
        if (a.pr.n > 1) {  // first pair whose block range holds blk
          int lo = 0, hi = a.pr.n - 1;
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if ((uint32_t)blk < a.pr.block_end[mid])
              hi = mid;
            else
              lo = mid + 1;
          }
          cur_p = a.pr.cur[lo], ref_p = a.pr.ref[lo];
          cur_stride = a.pr.cur_stride[lo], ref_stride = a.pr.ref_stride[lo];
        }
        const Px *pc = (const Px *)cur_p + (long long)b.y * cur_stride + b.x + t;
        const Px *pr;
        long long rstride;
        if (a.pred_packed) {
          pr = (const Px *)a.pred_packed + blk * (size_t)(W * H) + t;
          rstride = W;
        } else {
          pr = (const Px *)ref_p + (long long)(b.y + dy) * ref_stride + b.x + dx + t;
          rstride = ref_stride;
        }
#pragma unroll
        for (int r = 0; r < H; r++) {
          const int rr = a.ud_flip ? H - 1 - r : r;
          c[r] = round_shift_bit((int)pc[(long long)rr * cur_stride] - (int)pr[rr * rstride], a.bit0);
        }
      } else {
        const int16_t *src = a.in + blk * a.in_block_stride + t;
#pragma unroll
        for (int r = 0; r < H; r++) {
          const int rr = a.ud_flip ? H - 1 - r : r;
          c[r] = round_shift_bit((int)src[(size_t)rr * a.in_row_stride], a.bit0);
        }
      }
      run_1d<H>(a.col_type, c);
      const int cc = a.lr_flip ? W - 1 - t : t;
#pragma unroll
      for (int r = 0; r < H; r++) tile[r * PITCH + cc] = round_shift_bit(c[r], a.bit1);
    }
    __syncthreads();
    // ---- rows (forward.rs:131-160)
    if (valid && t < H) {
      TXV c[W];
#pragma unroll
      for (int k = 0; k < W; k++) c[k] = tile[t * PITCH + k];
      run_1d<W>(a.row_type, c);
      constexpr int HS = H < 32 ? H : 32, WC = W < 32 ? W : 32;
      CoefT *dst = (CoefT *)a.out + blk * (size_t)(W * H) + (t >= 32 ? HS * WC : 0) + (t & 31);
#pragma unroll
      for (int k = 0; k < W; k++)
        dst[(size_t)H * 32 * (k >= 32) + (k & 31) * HS] = (CoefT)round_shift_bit(c[k], a.bit2);
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- DCT_DCT from aligned planes
// The fused-residual forms on 8-bit planes at DCT_DCT with both sides in 8..32 take a kernel of their
// own: the 1-D kinds, the absence of flips and the three stage shifts (forward_shared.rs:22-64,
// classes A and B of kShiftClass) are compile-time, and each block row is read as whole 16-byte
// segments, one round of blocks ahead of the one being transformed.  A warp owns its blocks end to
// end, so it needs no __syncthreads:
//   rows:    lane t loads row t of cur and of the prediction (aligned 16-byte segments, the bytes
//            picked out with funnel shifts), forms the residual, stores it as a row of the tile;
//   columns: lane c runs the column transform on column c (forward.rs:95-126) in place;
//   rows:    lane t runs the row transform on row t (forward.rs:131-160) and stages its outputs in
//            the block's coefficient order dst[k * H + t] (forward.rs:135-159 for W, H <= 32);
//   store:   the lanes write the block's contiguous W * H coefficients with 16-byte stores.
// The block records, winner vectors and pair lookups of up to 32 blocks are resolved once, one
// block per lane, and handed to the lanes that transform the block by shuffles.
//
// forward_shared.rs:22-64 at 8 bit: av1_round_shift_array `bit` = -shift[k] (TxSetup::bit0..2)
template <int W, int H>
struct FastShift {
  static constexpr bool kClassB = W * H >= 512;  // 32x32, 16x32, 32x16
  static constexpr int bit0 = -4, bit1 = kClassB ? 2 : 1, bit2 = 0;
};

template <int BIT>
__device__ __forceinline__ int round_shift_c(int v) {
  if constexpr (BIT > 0) return (v + (1 << (BIT - 1))) >> BIT;
  else return (int)((unsigned)v << (-BIT));
}

template <int N>
__device__ __forceinline__ void fdct_1d(TXV (&c)[N]) {
  if constexpr (N == 8) tx_fdct8(c);
  else if constexpr (N == 16) tx_fdct16(c);
  else tx_fdct32(c);
}

// RB bytes from p (any alignment), read only through the 16-byte-aligned segments that hold them:
// such a segment lies inside the 16-byte granules of the row, so it stays in the allocation whenever
// the row's start and pitch are 16-byte aligned.  fetch() issues the loads, bytes() picks the row out
// of the segments once they have arrived, so a round's loads can be in flight during the previous one.
template <int RB>
struct RowSegs {
  static constexpr int NW = RB / 4, NSEG = RB >= 16 ? RB / 16 + 1 : 2;
  uint32_t w[NSEG * 4];
  int off;

  __device__ __forceinline__ void fetch(const uint8_t *p) {
    off = (int)((uintptr_t)p & 15);
    const uint4 *s = (const uint4 *)(p - off);
#pragma unroll
    for (int k = 0; k < NSEG; k++) {
      // the last segment is needed only when the row crosses into it
      const bool need = k < NSEG - 1 || off + RB > 16 * k;
      const uint4 v = need ? __ldg(s + k) : make_uint4(0, 0, 0, 0);
      w[4 * k] = v.x, w[4 * k + 1] = v.y, w[4 * k + 2] = v.z, w[4 * k + 3] = v.w;
    }
  }

  __device__ __forceinline__ void bytes(uint32_t (&o)[NW]) const {
    uint32_t v[NSEG * 4];
#pragma unroll
    for (int i = 0; i < NSEG * 4; i++) v[i] = w[i];
    if (off == 0) {
#pragma unroll
      for (int i = 0; i < NW; i++) o[i] = v[i];
      return;
    }
    // v[i] = w[i + q] for i <= NW (two select stages), then o[i] = bytes (off & 3) .. of v[i], v[i + 1]
    const int q = off >> 2;
#pragma unroll
    for (int i = 0; i < NW + 2; i++) v[i] = (q & 2) ? v[i + 2] : v[i];
#pragma unroll
    for (int i = 0; i < NW + 1; i++) v[i] = (q & 1) ? v[i + 1] : v[i];
#pragma unroll
    for (int i = 0; i < NW; i++) o[i] = __funnelshift_r(v[i], v[i + 1], (off & 3) * 8);
  }
};

__device__ __forceinline__ int byte_at(const uint32_t *w, int c) {
  return (int)__byte_perm(w[c >> 2], 0, 0x4440 | (c & 3));
}

constexpr int kFastThreads = 128;
// blocks with sides up to 16 fit 80 registers with the next round's rows in flight: 6 CTAs per SM
template <int W, int H>
constexpr int fast_min_ctas() { return W <= 16 && H <= 16 ? 6 : 1; }

template <int W, int H>
__global__ void __launch_bounds__(kFastThreads, fast_min_ctas<W, H>()) fwd_dct_fast_kernel(const __grid_constant__ TxArgs a) {
  using CoefT = int16_t;
  using S = FastShift<W, H>;
  constexpr int T = W > H ? W : H;  // lanes per block
  constexpr int SPW = 32 / T;       // blocks per warp round
  constexpr int PITCH = W + 4;      // keeps rows 16-byte aligned; row and column accesses conflict-free
  // slot s starts at bank 8s (8x8), 16s (16-wide) so the slots of a warp use disjoint banks
  constexpr int SLOT = (H * PITCH + 31) / 32 * 32 + (SPW > 1 ? T : 0);
  constexpr int WARPS = kFastThreads / 32;
  constexpr int RB = W;  // bytes per block row
  static_assert(W * H * sizeof(CoefT) <= H * PITCH * 4, "coefficients fit the tile");
  __shared__ __align__(16) int smem[WARPS][SPW * SLOT];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int slot = lane / T, t = lane - slot * T;
  int *tile = smem[warp] + slot * SLOT;
  const size_t coef_bytes = (size_t)W * H * sizeof(CoefT);
  // Round r of the launch is blocks [r * SPW, r * SPW + SPW); warp w of tw takes rounds w, w + tw, ...,
  // so the warps on the GPU at one time work on neighbouring blocks (and the same reference area).
  // A pass of a warp is its next RPP rounds, whose blocks are resolved one per lane up front.
  constexpr int RPP = 32 / SPW;
  // (32-bit indices: the host sends fewer than 2^31 blocks)
  const uint32_t n = (uint32_t)a.n, rounds = (n + SPW - 1) / SPW;
  const uint32_t tw = gridDim.x * WARPS, w = blockIdx.x * WARPS + warp;
  const uint32_t my_rounds = w < rounds ? (rounds - w + tw - 1) / tw : 0;
  const auto block_of = [&](uint32_t p0, int j) { return ((p0 + j / SPW) * tw + w) * SPW + j % SPW; };
  for (uint32_t p0 = 0; p0 < my_rounds; p0 += RPP) {
    const int nloc = (int)min((uint32_t)RPP, my_rounds - p0) * SPW;
    // lane j: where the rows of block block_of(p0, j) start (NULL: no such block)
    const uint8_t *cur_p = nullptr, *ref_p = nullptr;
    int cur_sb = 0, ref_sb = 0;  // row pitches, bytes
    if (lane < nloc && block_of(p0, lane) < n) {
      const uint32_t blk = block_of(p0, lane);
      const b200_block b = a.blocks[blk];
      int dx = 0, dy = 0;
      if (a.mv_src) {
        const b200_me_result m = a.mv_src[blk];
        if (m.cost != ~0ull) dx = m.mv_col / 8, dy = m.mv_row / 8;
      }
      const void *cp = a.cur, *rp = a.ref;
      int cs = a.cur_stride, rs = a.ref_stride;
      if (a.pr.n > 1) {  // first pair whose block range holds blk
        int lo = 0, hi = a.pr.n - 1;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if ((uint32_t)blk < a.pr.block_end[mid])
            hi = mid;
          else
            lo = mid + 1;
        }
        cp = a.pr.cur[lo], rp = a.pr.ref[lo];
        cs = a.pr.cur_stride[lo], rs = a.pr.ref_stride[lo];
      }
      cur_p = (const uint8_t *)cp + (long long)b.y * cs + b.x;
      cur_sb = cs;
      if (a.pred_packed) {
        ref_p = (const uint8_t *)a.pred_packed + (size_t)blk * (W * H);
        ref_sb = RB;
      } else {
        ref_p = (const uint8_t *)rp + (long long)(b.y + dy) * rs + b.x + dx;
        ref_sb = rs;
      }
    }
    // round i + SPW's rows are loaded while round i is transformed
    RowSegs<RB> next_cur, next_ref;
    const auto fetch = [&](int i) {
      const int j = i + slot;
      const uint8_t *cp = (const uint8_t *)__shfl_sync(~0u, (unsigned long long)cur_p, j);
      const uint8_t *rp = (const uint8_t *)__shfl_sync(~0u, (unsigned long long)ref_p, j);
      const int cs = __shfl_sync(~0u, cur_sb, j), rs = __shfl_sync(~0u, ref_sb, j);
      if (cp && t < H) {
        next_cur.fetch(cp + (long long)t * cs);
        next_ref.fetch(rp + (long long)t * rs);
      }
    };
    fetch(0);
    for (int i = 0; i < nloc; i += SPW) {
      const uint32_t blk = block_of(p0, i + slot);
      const bool valid = blk < n;
      const RowSegs<RB> row_cur = next_cur, row_ref = next_ref;
      if (i + SPW < nloc) fetch(i + SPW);
      // ---- residual rows (encoder.rs:1533 `diff`)
      if (valid && t < H) {
        uint32_t cw[RB / 4], rw[RB / 4];
        row_cur.bytes(cw);
        row_ref.bytes(rw);
        int d[W];
#pragma unroll
        for (int c = 0; c < W; c++) d[c] = round_shift_c<S::bit0>(byte_at(cw, c) - byte_at(rw, c));
#pragma unroll
        for (int c = 0; c < W; c += 4) *(int4 *)&tile[t * PITCH + c] = make_int4(d[c], d[c + 1], d[c + 2], d[c + 3]);
      }
      __syncwarp();
      // ---- columns (forward.rs:95-126)
      if (valid && t < W) {
        TXV v[H];
#pragma unroll
        for (int r = 0; r < H; r++) v[r] = tile[r * PITCH + t];
        fdct_1d<H>(v);
#pragma unroll
        for (int r = 0; r < H; r++) tile[r * PITCH + t] = round_shift_c<S::bit1>(v[r]);
      }
      __syncwarp();
      // ---- rows (forward.rs:131-160)
      TXV v[W];
      if (valid && t < H) {
#pragma unroll
        for (int k = 0; k < W; k += 4) {
          const int4 q = *(const int4 *)&tile[t * PITCH + k];
          v[k] = q.x, v[k + 1] = q.y, v[k + 2] = q.z, v[k + 3] = q.w;
        }
        fdct_1d<W>(v);
      }
      __syncwarp();
      if (valid && t < H) {
        CoefT *o = (CoefT *)tile;
#pragma unroll
        for (int k = 0; k < W; k++) o[k * H + t] = (CoefT)round_shift_c<S::bit2>(v[k]);
      }
      __syncwarp();
      if (valid) {
        constexpr int NCH = W * H * (int)sizeof(CoefT) / 16;
        uint4 *dst = (uint4 *)((uint8_t *)a.out + (size_t)blk * coef_bytes);
#pragma unroll
        for (int q = t; q < NCH; q += T) dst[q] = ((const uint4 *)tile)[q];
      }
      __syncwarp();
    }
  }
}

template <int W, int H>
int launch_fast(b200_ctx *ctx, const TxArgs &a) {
  constexpr int T = W > H ? W : H;
  constexpr int SPW = 32 / T;
  constexpr int WARPS = kFastThreads / 32;
  // As many CTAs as are resident at once (the rounds are spread over the warps, not the CTAs over
  // time), fewer when there are not enough rounds for them.
  static int per_sm[64];
  int &occ = per_sm[ctx->device & 63];
  if (!occ)
    B200_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fwd_dct_fast_kernel<W, H>, kFastThreads, 0));
  const size_t rounds = (a.n + SPW - 1) / SPW;
  const int grid = (int)std::max<size_t>(1, std::min<size_t>((rounds + WARPS - 1) / WARPS, (size_t)ctx->num_sms * occ));
  fwd_dct_fast_kernel<W, H><<<grid, kFastThreads, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

bool rows_16b_aligned(const void *p, long long pitch_bytes) {
  return (uintptr_t)p % 16 == 0 && pitch_bytes % 16 == 0;
}

// The fast kernel serves a fused-residual call on 8-bit planes at DCT_DCT, sides in 8..32, when every
// plane row and the output start on 16-byte boundaries; everything else runs fwd_txfm_kernel.  At 10
// and 12 bit the u16 rows and i32 coefficients need about 100 registers with a round of rows in
// flight, and fwd_txfm_kernel stayed faster there (16x16 on H100: 0.216 vs 0.291 ms per launch).
bool fast_path_ok(const TxArgs &a, int tx_type, int w, int h, int bpp) {
  if (!a.cur || bpp != 1 || tx_type != TX_DCT_DCT || w < 8 || h < 8 || w > 32 || h > 32) return false;
  if (a.n >= (1u << 31)) return false;
  if ((uintptr_t)a.out % 16) return false;
  // packed predictions: each block is W * H >= 64 bytes, so an aligned buffer keeps every segment inside it
  if (a.pred_packed) return rows_16b_aligned(a.pred_packed, 0) && rows_16b_aligned(a.cur, (long long)a.cur_stride * bpp);
  if (a.pr.n > 1) {
    for (int k = 0; k < a.pr.n; k++)
      if (!rows_16b_aligned(a.pr.cur[k], (long long)a.pr.cur_stride[k] * bpp) ||
          !rows_16b_aligned(a.pr.ref[k], (long long)a.pr.ref_stride[k] * bpp))
        return false;
    return true;
  }
  return rows_16b_aligned(a.cur, (long long)a.cur_stride * bpp) &&
         rows_16b_aligned(a.ref, (long long)a.ref_stride * bpp);
}

template <int W, int H>
int launch_txfm(b200_ctx *ctx, const TxArgs &a, int coeff_is_i32) {
  constexpr int T = W > H ? W : H;
  constexpr int PER = kTxThreads / T;
  const size_t ctas = (a.n + PER - 1) / PER;
  const int grid = (int)std::min<size_t>(ctas, (size_t)ctx->num_sms * 32);
  if (a.cur) {
    if (coeff_is_i32)
      fwd_txfm_kernel<W, H, int32_t, true><<<grid, kTxThreads, 0, ctx->stream>>>(a);
    else
      fwd_txfm_kernel<W, H, int16_t, true><<<grid, kTxThreads, 0, ctx->stream>>>(a);
  } else if (coeff_is_i32) {
    fwd_txfm_kernel<W, H, int32_t, false><<<grid, kTxThreads, 0, ctx->stream>>>(a);
  } else {
    fwd_txfm_kernel<W, H, int16_t, false><<<grid, kTxThreads, 0, ctx->stream>>>(a);
  }
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

}  // namespace

extern "C" int b200_valid_av1_transform(int tx_size, int tx_type) {
  return valid_transform(tx_size, tx_type) ? 1 : 0;
}
extern "C" int b200_tx_width(int tx_size) { return tx_size >= 0 && tx_size < 19 ? kTxW[tx_size] : 0; }
extern "C" int b200_tx_height(int tx_size) { return tx_size >= 0 && tx_size < 19 ? kTxH[tx_size] : 0; }

static int fwd_txfm_impl(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                         const TxPairs *pairs, const void *d_pred_packed, const b200_block *d_blocks,
                         const b200_me_result *d_mv_src,
                         const int16_t *d_input, size_t in_block_stride, size_t in_row_stride,
                         void *d_output, size_t nblocks, int tx_size, int tx_type, int bd,
                         int coeff_is_i32) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  // forward.rs:75: assert!(valid_av1_transform(tx_size, tx_type))
  B200_REQUIRE(ctx, valid_transform(tx_size, tx_type), "invalid transform: tx_size %d tx_type %d",
               tx_size, tx_type);
  B200_REQUIRE(ctx, bd == 8 || bd == 10 || bd == 12, "bit depth %d not in {8,10,12}", bd);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, (d_input || cur) && d_output, "NULL input/output");
  const int w = kTxW[tx_size], h = kTxH[tx_size];
  B200_REQUIRE(ctx, cur || in_row_stride >= (size_t)w, "row stride %zu < width %d", in_row_stride, w);
  (void)h;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const TxSetup ts = tx_setup(tx_size, tx_type, bd);
  TxArgs a;
  a.cur = cur ? cur->data : nullptr;
  a.ref = ref ? ref->data : nullptr;
  a.cur_stride = cur ? cur->stride : 0;
  a.ref_stride = ref ? ref->stride : 0;
  if (pairs)
    a.pr = *pairs;
  else
    a.pr.n = 0;
  a.blocks = d_blocks;
  a.mv_src = d_mv_src;
  a.pred_packed = d_pred_packed;
  a.in = d_input;
  a.out = d_output;
  a.n = nblocks;
  a.in_block_stride = in_block_stride;
  a.in_row_stride = (int)in_row_stride;
  a.col_type = ts.col_type;
  a.row_type = ts.row_type;
  a.ud_flip = ts.ud_flip;
  a.lr_flip = ts.lr_flip;
  a.bit0 = ts.bit0;
  a.bit1 = ts.bit1;
  a.bit2 = ts.bit2;
  if (fast_path_ok(a, tx_type, w, h, cur ? cur->bpp : 0)) {
    switch (tx_size) {
#define B200_TX(ID, W_, H_) \
  case ID:                  \
    return launch_fast<W_, H_>(ctx, a);
      B200_TX(1, 8, 8)
      B200_TX(2, 16, 16)
      B200_TX(3, 32, 32)
      B200_TX(7, 8, 16)
      B200_TX(8, 16, 8)
      B200_TX(9, 16, 32)
      B200_TX(10, 32, 16)
      B200_TX(15, 8, 32)
      B200_TX(16, 32, 8)
#undef B200_TX
    }
  }
  switch (tx_size) {
#define B200_TX(ID, W_, H_) \
  case ID:                  \
    return launch_txfm<W_, H_>(ctx, a, coeff_is_i32);
    B200_TX(0, 4, 4)
    B200_TX(1, 8, 8)
    B200_TX(2, 16, 16)
    B200_TX(3, 32, 32)
    B200_TX(4, 64, 64)
    B200_TX(5, 4, 8)
    B200_TX(6, 8, 4)
    B200_TX(7, 8, 16)
    B200_TX(8, 16, 8)
    B200_TX(9, 16, 32)
    B200_TX(10, 32, 16)
    B200_TX(11, 32, 64)
    B200_TX(12, 64, 32)
    B200_TX(13, 4, 16)
    B200_TX(14, 16, 4)
    B200_TX(15, 8, 32)
    B200_TX(16, 32, 8)
    B200_TX(17, 16, 64)
    B200_TX(18, 64, 16)
#undef B200_TX
  }
  return b200_fail(ctx, B200_ERR_ARG, "unreachable tx_size %d", tx_size);
}

extern "C" int b200_fwd_txfm_dev(b200_ctx *ctx, const int16_t *d_input, size_t in_block_stride,
                                 size_t in_row_stride, void *d_output, size_t nblocks, int tx_size,
                                 int tx_type, int bd, int coeff_is_i32) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, d_input || nblocks == 0, "NULL input");
  return fwd_txfm_impl(ctx, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, d_input, in_block_stride,
                       in_row_stride, d_output, nblocks, tx_size, tx_type, bd, coeff_is_i32);
}

// Fused `diff` + forward transform (encoder.rs:1533-1544): residual of each block against the
// reference displaced by the full-pel part of d_mv_src (NULL = zero motion), transformed without
// a round trip of the residual through HBM.  u8 planes give i16 coefficients, u16 planes i32.
extern "C" int b200_fwd_txfm_residual_dev(b200_ctx *ctx, const b200_plane *cur,
                                          const b200_plane *ref, const b200_block *d_blocks,
                                          size_t nblocks, const b200_me_result *d_mv_src,
                                          void *d_output, int tx_size, int tx_type, int bd) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && ref && cur->data && ref->data && cur->bpp == ref->bpp, "bad planes");
  B200_REQUIRE(ctx, (cur->bpp == 1) == (bd == 8), "bpp %d does not match bit depth %d", cur->bpp, bd);
  B200_REQUIRE(ctx, d_blocks || nblocks == 0, "NULL blocks");
  return fwd_txfm_impl(ctx, cur, ref, nullptr, nullptr, d_blocks, d_mv_src, nullptr, 0, 0, d_output,
                       nblocks, tx_size, tx_type, bd, cur->bpp == 2);
}

// The fused residual + transform over several plane pairs in one launch (block ranges as in
// b200_me_candidates_multi_dev; d_mv_src / d_output follow the concatenated block order).
extern "C" int b200_fwd_txfm_residual_multi_dev(b200_ctx *ctx, size_t npairs, const b200_plane *curs,
                                                const b200_plane *refs, const uint32_t *pair_block_end,
                                                const b200_block *d_blocks, size_t nblocks,
                                                const b200_me_result *d_mv_src, void *d_output,
                                                int tx_size, int tx_type, int bd) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, npairs >= 1 && curs && refs && pair_block_end, "NULL plane pair table");
  B200_REQUIRE(ctx, valid_transform(tx_size, tx_type), "invalid transform: tx_size %d tx_type %d",
               tx_size, tx_type);
  B200_REQUIRE(ctx, d_blocks || nblocks == 0, "NULL blocks");
  B200_REQUIRE(ctx, pair_block_end[npairs - 1] == nblocks && nblocks < (1ull << 32),
               "last pair must end at nblocks");
  for (size_t k = 0; k < npairs; k++) {
    B200_REQUIRE(ctx, curs[k].data && refs[k].data && curs[k].bpp == refs[k].bpp &&
                          curs[k].bpp == curs[0].bpp, "pair %zu: bad planes", k);
    B200_REQUIRE(ctx, pair_block_end[k] >= (k ? pair_block_end[k - 1] : 0),
                 "pair %zu: block ends must be non-decreasing", k);
  }
  B200_REQUIRE(ctx, (curs[0].bpp == 1) == (bd == 8), "bpp %d does not match bit depth %d", curs[0].bpp, bd);
  const size_t coef_bytes = (size_t)kTxW[tx_size] * kTxH[tx_size] * (curs[0].bpp == 2 ? 4 : 2);
  for (size_t k0 = 0; k0 < npairs; k0 += kTxMaxPairs) {
    const int n = (int)std::min<size_t>(kTxMaxPairs, npairs - k0);
    const uint32_t b0 = k0 ? pair_block_end[k0 - 1] : 0;
    TxPairs t;
    t.n = n;
    for (int k = 0; k < n; k++) {
      t.block_end[k] = pair_block_end[k0 + k] - b0;
      t.cur[k] = curs[k0 + k].data;
      t.ref[k] = refs[k0 + k].data;
      t.cur_stride[k] = curs[k0 + k].stride;
      t.ref_stride[k] = refs[k0 + k].stride;
    }
    const size_t nb = t.block_end[n - 1];
    if (nb == 0) continue;
    if (int st = fwd_txfm_impl(ctx, &curs[k0], &refs[k0], &t, nullptr, d_blocks + b0,
                               d_mv_src ? d_mv_src + b0 : nullptr, nullptr, 0, 0,
                               (uint8_t *)d_output + (size_t)b0 * coef_bytes, nb, tx_size, tx_type, bd,
                               curs[0].bpp == 2))
      return st;
  }
  return B200_OK;
}

// Residual against PACKED predictions (the output layout of b200_mc_blocks_dev /
// b200_predict_intra_dev): block i = cur(d_blocks[i]) - d_pred[i], then the forward transform.
// This is encode_tx_block's predict -> diff -> forward_transform chain (encoder.rs:1492-1544)
// for sub-pel inter or intra predictions.
extern "C" int b200_fwd_txfm_pred_dev(b200_ctx *ctx, const b200_plane *cur, const void *d_pred,
                                      const b200_block *d_blocks, size_t nblocks, void *d_output,
                                      int tx_size, int tx_type, int bd) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && cur->data && d_pred, "bad plane / prediction");
  B200_REQUIRE(ctx, (cur->bpp == 1) == (bd == 8), "bpp %d does not match bit depth %d", cur->bpp, bd);
  B200_REQUIRE(ctx, d_blocks || nblocks == 0, "NULL blocks");
  return fwd_txfm_impl(ctx, cur, cur, nullptr, d_pred, d_blocks, nullptr, nullptr, 0, 0, d_output, nblocks,
                       tx_size, tx_type, bd, cur->bpp == 2);
}

// Host-buffer form: packed residual blocks in, coefficients out.
extern "C" int b200_fwd_txfm_batch(b200_ctx *ctx, const int16_t *input, size_t in_block_stride,
                                   size_t in_row_stride, void *output, size_t nblocks, int tx_size,
                                   int tx_type, int bd, int coeff_is_i32) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, valid_transform(tx_size, tx_type), "invalid transform: tx_size %d tx_type %d",
               tx_size, tx_type);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, input && output, "NULL input/output");
  const int w = kTxW[tx_size], h = kTxH[tx_size];
  const size_t in_elems = (nblocks - 1) * in_block_stride + (size_t)(h - 1) * in_row_stride + w;
  const size_t out_bytes = nblocks * (size_t)w * h * (coeff_is_i32 ? 4 : 2);
  HostStage s(ctx, b200_align_up(in_elems * 2, 256) + out_bytes);
  int16_t *d_in = (int16_t *)s.take(in_elems * 2);
  uint8_t *d_out = s.take(out_bytes);
  s.up(d_in, input, in_elems * 2);
  if (s.ok())
    s.run(b200_fwd_txfm_dev(ctx, d_in, in_block_stride, in_row_stride, d_out, nblocks, tx_size, tx_type, bd,
                            coeff_is_i32));
  s.down(output, d_out, out_bytes);
  return s.finish(!ctx->async_batch);
}

extern "C" int b200_fwd_txfm_residual_resident(b200_ctx *ctx, const b200_plane *cur,
                                               const b200_plane *ref, const b200_block *blocks,
                                               size_t nblocks, const b200_me_result *mv_src,
                                               void *output, int tx_size, int tx_type, int bd) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, valid_transform(tx_size, tx_type), "invalid transform: tx_size %d tx_type %d",
               tx_size, tx_type);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, cur && ref && blocks && output, "NULL argument");
  const size_t area = (size_t)kTxW[tx_size] * kTxH[tx_size];
  const size_t out_bytes = nblocks * area * (cur->bpp == 2 ? 4 : 2);
  const size_t blk_bytes = b200_align_up(nblocks * sizeof(b200_block), 256);
  const size_t mv_bytes = mv_src ? b200_align_up(nblocks * sizeof(b200_me_result), 256) : 0;
  HostStage s(ctx, blk_bytes + mv_bytes + out_bytes);
  b200_block *d_blk = (b200_block *)s.take(nblocks * sizeof(b200_block));
  b200_me_result *d_mv = mv_src ? (b200_me_result *)s.take(nblocks * sizeof(b200_me_result)) : nullptr;
  uint8_t *d_out = s.take(out_bytes);
  s.up(d_blk, blocks, nblocks * sizeof(b200_block));
  if (mv_src) s.up(d_mv, mv_src, nblocks * sizeof(b200_me_result));
  if (s.ok()) s.run(b200_fwd_txfm_residual_dev(ctx, cur, ref, d_blk, nblocks, d_mv, d_out, tx_size, tx_type, bd));
  s.down(output, d_out, out_bytes);
  return s.finish(!ctx->async_batch);
}

// Per-call form with the reference's signature (asm/x86/transform/forward.rs:444-447):
// forward_transform(input: &[i16], output: &mut [T::Coeff], stride, tx_size, tx_type, bd, cpu).
extern "C" void b200_forward_transform(const int16_t *input, void *output, size_t stride,
                                       int tx_size, int tx_type, int bd, int coeff_is_i32) {
  b200_ctx *ctx = b200_default_ctx();
  // the reference panics on an invalid (size, type) pair (forward.rs:75)
  b200_percall_check(ctx, b200_fwd_txfm_batch(ctx, input, 0, stride, output, 1, tx_size, tx_type, bd, coeff_is_i32),
                     "forward_transform");
}
