// mc.cu — batched 8-tap sub-pel motion compensation (rav1e src/mc.rs:250-479) for sm_90a.
//
// One warp per predicted block (up to 8 blocks per CTA).  The (w+7) x (h+7) source footprint is
// staged once in shared memory; the separable filter then runs as the reference's four cases (copy / V only /
// H only with its double rounding / H into an i16 intermediate then V), all in exact integer
// arithmetic, with the 6 x 16 x 8 coefficient table in constant memory.  `put` writes pixels,
// `prep` writes the biased i16 intermediate used by compound prediction, `avg` blends two of
// those (mc.rs:454-479).  Blocks are addressed by (position, motion vector) through
// get_mv_params (predict.rs:284-297), so one launch predicts thousands of blocks.
#include "host_stage.cuh"
#include "mc_dev.cuh"

namespace {

struct McArgs {
  const void *ref;    // plane pixel (0,0)
  int ref_stride;     // elements
  const b200_block *blocks;
  const short *mvs;   // row, col per block (1/8 pel); null = zero motion
  const b200_cand *cands;  // optional: item i = (blocks[cands[i].block], cands[i].mv)
  size_t n;
  int w, h;
  int mode_x, mode_y;
  int bit_depth;
  int xdec, ydec;
  int kind;           // 0 put, 1 prep
  void *out;          // packed blocks: pixels (put) or int16 (prep)
  // per-call form: explicit fractions and no block list
  int explicit_frac;
  int col_frac, row_frac;
};

// One WARP per predicted block; a CTA carries `blockDim.x / 32` blocks, each with its own slice
// of shared memory (source tile + i16 intermediate).  Warp-level staging and passes need no
// block-wide barriers; filter taps sit in registers.
template <typename T>
__global__ void __launch_bounds__(256) mc_kernel(McArgs a, int smem_per_warp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int w = a.w, h = a.h;
  const int tw = w + 7, th = h + 7;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T *tile = (T *)(smem_raw + (size_t)wid * smem_per_warp);                       // [th][tw]
  short *inter = (short *)(tile + (size_t)th * tw + (((size_t)th * tw) & 1));     // [th][w]
  const int ib = 4 - (a.bit_depth == 12 ? 2 : 0);
  const int maxv = (1 << a.bit_depth) - 1;
  const int prep_bias = a.bit_depth == 8 ? 0 : 8192;
  const int xb = filter_bank(a.mode_x, w), yb = filter_bank(a.mode_y, h);
  const int wlog2 = 31 - __clz(w);

  for (size_t blk = (size_t)blockIdx.x * nw + wid; blk < a.n; blk += (size_t)gridDim.x * nw) {
    int x0 = 0, y0 = 0, col_frac = a.col_frac, row_frac = a.row_frac;
    if (!a.explicit_frac) {
      b200_block b;
      int mvr, mvc;
      if (a.cands) {
        const b200_cand c = a.cands[blk];
        b = a.blocks[c.block];
        mvr = c.mv_row;
        mvc = c.mv_col;
      } else {
        b = a.blocks[blk];
        mvr = a.mvs ? a.mvs[2 * blk] : 0;
        mvc = a.mvs ? a.mvs[2 * blk + 1] : 0;
      }
      // predict.rs:284-297 get_mv_params
      y0 = b.y + (mvr >> (3 + a.ydec));
      x0 = b.x + (mvc >> (3 + a.xdec));
      row_frac = (int)(((unsigned)mvr << (1 - a.ydec)) & 0xf);
      col_frac = (int)(((unsigned)mvc << (1 - a.xdec)) & 0xf);
    }
    const T *src = (const T *)a.ref + (long long)y0 * a.ref_stride + x0;
    int xf[8], yf[8];
#pragma unroll
    for (int k = 0; k < 8; k++) {
      xf[k] = kSubpel[xb][col_frac][k];
      yf[k] = kSubpel[yb][row_frac][k];
    }
    __syncwarp();
    for (int r = 0; r < th; r++) {
      const T *srow = src + (long long)(r - 3) * a.ref_stride - 3;
      for (int c = lane; c < tw; c += 32) tile[r * tw + c] = srow[c];
    }
    __syncwarp();
    T *outp = (T *)a.out + blk * (size_t)w * h;
    short *outs = (short *)a.out + blk * (size_t)w * h;
    if (col_frac != 0 && row_frac != 0) {
      // H pass into the i16 intermediate over h+7 rows (mc.rs:312-327): `as i16` truncates
      // flattened (row, col) index: w is a power of two, so all 32 lanes stay busy for any w
      for (int i = lane; i < th * w; i += 32) {
        const int r = i >> wlog2, c = i & (w - 1);
        int s = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) s += xf[k] * (int)tile[r * tw + c + k];
        inter[i] = (short)rshift_round(s, 7 - ib);
      }
      __syncwarp();
      for (int i = lane; i < h * w; i += 32) {
        int s = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) s += yf[k] * (int)inter[i + k * w];
        if (a.kind == 0)
          outp[i] = (T)min(max(rshift_round(s, 7 + ib), 0), maxv);
        else
          outs[i] = (short)(rshift_round(s, 7) - prep_bias);
      }
    } else {
      for (int i = lane; i < h * w; i += 32) {
          const int r = i >> wlog2, c = i & (w - 1);
          if (col_frac == 0 && row_frac == 0) {
            const int p = (int)tile[(r + 3) * tw + c + 3];
            if (a.kind == 0)
              outp[i] = (T)p;
            else
              outs[i] = (short)((short)((short)p << ib) - (short)prep_bias);
          } else if (col_frac == 0) {  // V only (mc.rs:277-296 / :387-403)
            int s = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) s += yf[k] * (int)tile[(r + k) * tw + c + 3];
            if (a.kind == 0)
              outp[i] = (T)min(max(rshift_round(s, 7), 0), maxv);
            else
              outs[i] = (short)(rshift_round(s, 7 - ib) - prep_bias);
          } else {  // H only, double rounding in `put` (mc.rs:297-311)
            int s = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) s += xf[k] * (int)tile[(r + 3) * tw + c + k];
            if (a.kind == 0)
              outp[i] = (T)min(max(rshift_round(rshift_round(s, 7 - ib), ib), 0), maxv);
            else
              outs[i] = (short)(rshift_round(s, 7 - ib) - prep_bias);
          }
        }
    }
    __syncwarp();
  }
}

template <typename T>
__global__ void mc_avg_kernel(const short *t1, const short *t2, T *dst, size_t total, int bit_depth) {
  const int ib = 4 - (bit_depth == 12 ? 2 : 0);
  const int maxv = (1 << bit_depth) - 1;
  const int bias = bit_depth == 8 ? 0 : 8192 * 2;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total;
       i += (size_t)gridDim.x * blockDim.x)
    dst[i] = (T)min(max(rshift_round((int)t1[i] + (int)t2[i] + bias, ib + 1), 0), maxv);
}

// `put` for the square sizes the RDO loop predicts most (8x8 .. 64x64): the packed-word path of
// mc_dev.cuh (IDP.4A / IDP.2A, four outputs per task), one warp per block, predictions written
// straight to their packed slots.
template <typename T, int W, int H>
__global__ void __launch_bounds__(256) mc_put_fast_kernel(McArgs a, int smem_per_warp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using ML = McLayout<T, W, H>;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  T *tile = (T *)(smem_raw + (size_t)wid * smem_per_warp);
  short *inter = (short *)((unsigned char *)tile + ML::TILE_BYTES);
  const int xb = filter_bank(a.mode_x, W), yb = filter_bank(a.mode_y, H);
  for (size_t blk = (size_t)blockIdx.x * nw + wid; blk < a.n; blk += (size_t)gridDim.x * nw) {
    b200_block b;
    int mvr, mvc;
    if (a.cands) {
      const b200_cand c = a.cands[blk];
      b = a.blocks[c.block];
      mvr = c.mv_row, mvc = c.mv_col;
    } else {
      b = a.blocks[blk];
      mvr = a.mvs ? a.mvs[2 * blk] : 0;
      mvc = a.mvs ? a.mvs[2 * blk + 1] : 0;
    }
    // predict.rs:284-297 get_mv_params
    const int y0 = b.y + (mvr >> (3 + a.ydec)), x0 = b.x + (mvc >> (3 + a.xdec));
    const int row_frac = (int)(((unsigned)mvr << (1 - a.ydec)) & 0xf), col_frac = (int)(((unsigned)mvc << (1 - a.xdec)) & 0xf);
    const T *src = (const T *)a.ref + (long long)(y0 - 3) * a.ref_stride + (x0 - 3);
    __syncwarp();
    mc_stage_tile<T, W, H>(tile, src, a.ref_stride, lane);
    __syncwarp();
    mc_put_warp<T, W, H>(tile, inter, (T *)a.out + blk * (size_t)(W * H), xb, col_frac, yb, row_frac, a.bit_depth, lane);
  }
}

template <typename T, int N>
int launch_mc_fast(b200_ctx *ctx, const McArgs &a) {
  using ML = McLayout<T, N, N>;
  const size_t per_warp = b200_align_up(ML::TILE_BYTES + ML::INTER_BYTES, 16);
  const int wpc = (int)std::min<size_t>(8, std::max<size_t>(1, (128 * 1024) / per_warp));
  if (int st = b200_smem_opt_in(ctx, (const void *)mc_put_fast_kernel<T, N, N>, 160 * 1024)) return st;
  const int grid = (int)std::min<size_t>((a.n + wpc - 1) / wpc, (size_t)ctx->num_sms * 16);
  mc_put_fast_kernel<T, N, N><<<grid, wpc * 32, per_warp * wpc, ctx->stream>>>(a, (int)per_warp);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

int check_mc(b200_ctx *ctx, int w, int h, int mode_x, int mode_y, int bit_depth) {
  // mc.rs:256-257: the asm only supports even heights and power-of-two widths 2..128
  B200_REQUIRE(ctx, (h & 1) == 0 && h > 0 && h <= 128, "height %d must be even and <= 128", h);
  B200_REQUIRE(ctx, w >= 2 && w <= 128 && (w & (w - 1)) == 0, "width %d must be a power of two in 2..128", w);
  B200_REQUIRE(ctx, mode_x >= 0 && mode_x <= 3 && mode_y >= 0 && mode_y <= 3, "bad FilterMode");
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  return B200_OK;
}

int launch_mc(b200_ctx *ctx, const McArgs &a, int bpp) {
  if (a.kind == 0 && !a.explicit_frac && a.w == a.h && !getenv("B200_MC_GENERIC")) {
#define B200_MCF(N) \
  if (a.w == N) return bpp == 1 ? launch_mc_fast<uint8_t, N>(ctx, a) : launch_mc_fast<uint16_t, N>(ctx, a);
    B200_MCF(8)
    B200_MCF(16)
    B200_MCF(32)
    B200_MCF(64)
#undef B200_MCF
  }
  const size_t tile_elems = (size_t)(a.w + 7) * (a.h + 7);
  const size_t per_warp = b200_align_up((tile_elems + (tile_elems & 1)) * bpp + (size_t)(a.h + 7) * a.w * 2, 16);
  // warps (= blocks in flight) per CTA: as many as fit ~96 KB, at most 8
  int wpc = (int)std::min<size_t>(8, std::max<size_t>(1, (96 * 1024) / per_warp));
  const size_t smem = per_warp * wpc;
  // 128 KB covers one 128x128 u16 block per warp slot
  if (int st = b200_smem_opt_in(ctx, bpp == 1 ? (const void *)mc_kernel<uint8_t> : (const void *)mc_kernel<uint16_t>,
                                128 * 1024))
    return st;
  const size_t ctas = (a.n + wpc - 1) / wpc;
  const int grid = (int)std::min<size_t>(ctas, (size_t)ctx->num_sms * 16);
  if (bpp == 1)
    mc_kernel<uint8_t><<<grid, wpc * 32, smem, ctx->stream>>>(a, (int)per_warp);
  else
    mc_kernel<uint16_t><<<grid, wpc * 32, smem, ctx->stream>>>(a, (int)per_warp);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

}  // namespace

extern "C" int b200_mc_blocks_dev(b200_ctx *ctx, const b200_plane *ref, const b200_block *d_blocks,
                                  const int16_t *d_mvs, size_t nblocks, int w, int h, int mode_x,
                                  int mode_y, int bit_depth, int xdec, int ydec, int kind,
                                  void *d_out) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, ref && ref->data, "bad reference plane");
  if (int st = check_mc(ctx, w, h, mode_x, mode_y, bit_depth)) return st;
  B200_REQUIRE(ctx, (ref->bpp == 1) == (bit_depth == 8), "plane bpp %d vs bit depth %d", ref->bpp, bit_depth);
  B200_REQUIRE(ctx, (xdec == 0 || xdec == 1) && (ydec == 0 || ydec == 1), "bad decimation");
  B200_REQUIRE(ctx, kind == 0 || kind == 1, "kind must be 0 (put) or 1 (prep)");
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && d_out, "NULL blocks/out");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  McArgs a{};
  a.ref = ref->data;
  a.ref_stride = ref->stride;
  a.blocks = d_blocks;
  a.mvs = d_mvs;
  a.n = nblocks;
  a.w = w;
  a.h = h;
  a.mode_x = mode_x;
  a.mode_y = mode_y;
  a.bit_depth = bit_depth;
  a.xdec = xdec;
  a.ydec = ydec;
  a.kind = kind;
  a.out = d_out;
  return launch_mc(ctx, a, ref->bpp);
}

// Internal (me_cand.cu): one `put` prediction per candidate, luma plane, packed w x h outputs.
int b200_mc_cands_internal(b200_ctx *ctx, const b200_plane *ref, const b200_block *d_blocks,
                           const b200_cand *d_cands, size_t ncands, int w, int h, int mode,
                           int bit_depth, void *d_out) {
  if (int st = check_mc(ctx, w, h, mode, mode, bit_depth)) return st;
  McArgs a{};
  a.ref = ref->data;
  a.ref_stride = ref->stride;
  a.blocks = d_blocks;
  a.cands = d_cands;
  a.n = ncands;
  a.w = w;
  a.h = h;
  a.mode_x = mode;
  a.mode_y = mode;
  a.bit_depth = bit_depth;
  a.kind = 0;
  a.out = d_out;
  return launch_mc(ctx, a, ref->bpp);
}

extern "C" int b200_mc_avg_dev(b200_ctx *ctx, const int16_t *d_tmp1, const int16_t *d_tmp2,
                               void *d_dst, size_t nblocks, int w, int h, int bit_depth) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (int st = check_mc(ctx, w, h, 0, 0, bit_depth)) return st;
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_tmp1 && d_tmp2 && d_dst, "NULL buffers");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t total = nblocks * (size_t)w * h;
  const int grid = (int)std::min<size_t>((total + 255) / 256, (size_t)ctx->num_sms * 32);
  if (bit_depth == 8)
    mc_avg_kernel<uint8_t><<<grid, 256, 0, ctx->stream>>>(d_tmp1, d_tmp2, (uint8_t *)d_dst, total, bit_depth);
  else
    mc_avg_kernel<uint16_t><<<grid, 256, 0, ctx->stream>>>(d_tmp1, d_tmp2, (uint16_t *)d_dst, total, bit_depth);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// ---- per-call forms with the argument order of the dav1d-style symbols rav1e binds
// (asm/x86/mc.rs:17-76): host pointers, BYTE strides, mx/my = col_frac/row_frac.  The filter
// pair that the reference encodes in the symbol name is passed as (mode_x, mode_y).
namespace {
int percall_mc(int kind, void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride,
               int w, int h, int col_frac, int row_frac, int mode_x, int mode_y, int bit_depth) {
  b200_ctx *ctx = b200_default_ctx();
  if (int st = check_mc(ctx, w, h, mode_x, mode_y, bit_depth)) return st;
  B200_REQUIRE(ctx, col_frac >= 0 && col_frac < 16 && row_frac >= 0 && row_frac < 16, "bad fraction");
  const int bpp = bit_depth == 8 ? 1 : 2;
  const int tw = w + 7, th = h + 7;
  const size_t out_bytes = (size_t)w * h * (kind == 0 ? bpp : 2);
  HostStage s(ctx, b200_align_up((size_t)tw * th * bpp, 256) + out_bytes);
  uint8_t *d_tile = s.take((size_t)tw * th * bpp);
  const uint8_t *h0 = (const uint8_t *)src - 3 * src_stride - 3 * bpp;  // asm/x86/mc.rs:122-123
  s.up2d(d_tile, (size_t)tw * bpp, h0, (size_t)src_stride, (size_t)tw * bpp, th);
  McArgs a{};
  a.ref = d_tile + ((size_t)3 * tw + 3) * bpp;
  a.ref_stride = tw;
  a.n = 1;
  a.w = w;
  a.h = h;
  a.mode_x = mode_x;
  a.mode_y = mode_y;
  a.bit_depth = bit_depth;
  a.kind = kind;
  a.out = s.take(out_bytes);
  a.explicit_frac = 1;
  a.col_frac = col_frac;
  a.row_frac = row_frac;
  if (s.ok()) s.run(launch_mc(ctx, a, bpp));
  if (kind == 0)
    s.down2d(dst, (size_t)dst_stride, a.out, (size_t)w * bpp, (size_t)w * bpp, h);
  else
    s.down(dst, a.out, out_bytes);
  return s.finish(true);
}
}  // namespace

extern "C" void b200_put_8tap(void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride,
                              int w, int h, int col_frac, int row_frac, int mode_x, int mode_y,
                              int bit_depth) {
  // the reference asserts (mc.rs:256-257) and has no error return
  const int st = percall_mc(0, dst, dst_stride, src, src_stride, w, h, col_frac, row_frac, mode_x, mode_y, bit_depth);
  b200_percall_check(b200_default_ctx(), st, "put_8tap");
}

extern "C" void b200_prep_8tap(int16_t *tmp, const void *src, ptrdiff_t src_stride, int w, int h,
                               int col_frac, int row_frac, int mode_x, int mode_y, int bit_depth) {
  const int st = percall_mc(1, tmp, 0, src, src_stride, w, h, col_frac, row_frac, mode_x, mode_y, bit_depth);
  b200_percall_check(b200_default_ctx(), st, "prep_8tap");
}

extern "C" void b200_mc_avg(void *dst, ptrdiff_t dst_stride, const int16_t *tmp1, const int16_t *tmp2,
                            int w, int h, int bit_depth) {
  b200_ctx *ctx = b200_default_ctx();
  const int bpp = bit_depth == 8 ? 1 : 2;
  const size_t n = (size_t)w * h;
  HostStage s(ctx, n * 4 + n * bpp + 512);
  int16_t *d1 = (int16_t *)s.take(n * 2), *d2 = (int16_t *)s.take(n * 2);
  uint8_t *dd = s.take(n * bpp);
  s.up(d1, tmp1, n * 2);
  s.up(d2, tmp2, n * 2);
  if (s.ok()) s.run(b200_mc_avg_dev(ctx, d1, d2, dd, 1, w, h, bit_depth));
  s.down2d(dst, (size_t)dst_stride, dd, (size_t)w * bpp, (size_t)w * bpp, h);
  b200_percall_check(ctx, s.finish(true), "mc_avg");
}
