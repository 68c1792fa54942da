// me_full_search.cu — full_search (src/me.rs:1464-1509) on the device for sm_90a, incl. its
// first-minimum argmin: b200_me_full_search_dev.
//
// Kernels
//   me_full_search_generic<T>  any size / depth, one CTA per block, warp per position.
//   me_full_search_u8<W,H>  8-bit fast path: window staged in smem so that every candidate
//                           column is word aligned; each thread evaluates NP adjacent positions
//                           sharing their loaded words.
#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"
#include "me_dev.cuh"

namespace {

struct FsArgs {
  PlaneView cur, ref;
  const b200_block *blocks;
  b200_me_result *out;
  size_t nblocks;
  int w, h;
  int w_in_b, h_in_b;
  uint32_t lambda;
  int allow_hp;
  int range_x, range_y, step;
};

struct FsWindow {
  int x_lo, x_hi, y_lo, y_hi, nx, ny;
};

// me.rs:822-846: window = po +- range, clamped to the mv range (in full pel, trunc /8).
__device__ __forceinline__ FsWindow fs_window(const FsArgs &a, b200_block b) {
  const MvRange r = b200_mv_range(a.w_in_b, a.h_in_b, b.x / MI_SIZE, b.y / MI_SIZE, a.w, a.h);
  FsWindow w;
  w.x_lo = b.x + max(-a.range_x, r.x_min / 8);
  w.x_hi = b.x + min(a.range_x, r.x_max / 8);
  w.y_lo = b.y + max(-a.range_y, r.y_min / 8);
  w.y_hi = b.y + min(a.range_y, r.y_max / 8);
  w.nx = w.x_hi >= w.x_lo ? (w.x_hi - w.x_lo) / a.step + 1 : 0;
  w.ny = w.y_hi >= w.y_lo ? (w.y_hi - w.y_lo) / a.step + 1 : 0;
  return w;
}

__device__ __forceinline__ void fs_write(const FsArgs &a, size_t blk, b200_block b,
                                         const FsWindow &w, CostIdx best, uint32_t sad_of_best) {
  b200_me_result res;
  res.cost = kEmptyCost;
  res.sad = kEmptySad;
  res.mv_row = 0;
  res.mv_col = 0;
  if (best.cost != kEmptyCost) {
    const int py = best.idx / w.nx, pxi = best.idx - py * w.nx;
    const int x = w.x_lo + pxi * a.step, y = w.y_lo + py * a.step;
    res.cost = best.cost;
    res.sad = sad_of_best;
    res.mv_row = (short)(8 * (short)(y - b.y));  // me.rs:1482-1485
    res.mv_col = (short)(8 * (short)(x - b.x));
  }
  a.out[blk] = res;
}

__device__ __forceinline__ uint32_t fs_sad_from_cost(const FsArgs &a, b200_block b,
                                                     const FsWindow &w, CostIdx best) {
  if (best.cost == kEmptyCost) return kEmptySad;
  const int py = best.idx / w.nx, pxi = best.idx - py * w.nx;
  const int mvr = (short)(8 * (short)(w.y_lo + py * a.step - b.y));
  const int mvc = (short)(8 * (short)(w.x_lo + pxi * a.step - b.x));
  uint32_t r1 = b200_mv_rate(mvr, mvc, 0, 0, a.allow_hp);
  uint32_t rate = r1 < r1 + 1 ? r1 : r1 + 1;  // min(rate1, rate2 + 1) with pmv0 == pmv1 == 0
  return (uint32_t)((best.cost - (unsigned long long)rate * a.lambda) >> 8);
}

template <typename T>
__global__ void __launch_bounds__(256) me_full_search_generic(FsArgs a) {
  __shared__ CostIdx s_red[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (size_t blk = blockIdx.x; blk < a.nblocks; blk += gridDim.x) {
    const b200_block b = a.blocks[blk];
    const FsWindow w = fs_window(a, b);
    CostIdx best{kEmptyCost, 0xffffffffu};
    const int npos = w.nx * w.ny;
    for (int p = wid; p < npos; p += nw) {
      const int py = p / w.nx, pxi = p - py * w.nx;
      const int x = w.x_lo + pxi * a.step, y = w.y_lo + py * a.step;
      const uint32_t sad = warp_block_dist<T>(px<T>(a.cur, b.x, b.y), a.cur.stride,
                                              px<T>(a.ref, x, y), a.ref.stride, a.w, a.h, 0, lane);
      const int mvr = (short)(8 * (short)(y - b.y)), mvc = (short)(8 * (short)(x - b.x));
      const unsigned long long cost =
          b200_mv_cost(sad, mvr, mvc, 0, 0, 0, 0, a.lambda, a.allow_hp);
      best = best_min(best, CostIdx{cost, (uint32_t)p});
    }
    best = block_best(best, s_red);
    if (threadIdx.x == 0) fs_write(a, blk, b, w, best, fs_sad_from_cost(a, b, w, best));
    __syncthreads();
  }
}

// 8-bit fast path.  The window is staged so that smem column 0 == x_lo: with the reference's
// step (4 at full resolution, me.rs:840-844) every candidate then starts on a word boundary
// and needs no byte shifting; other steps use the funnel-shift form.  Each thread evaluates
// NP horizontally adjacent positions per task, sharing the loaded reference words.
constexpr int kFsSmemBytes = 200 * 1024;

template <int W, int H, int NP>
__global__ void __launch_bounds__(256) me_full_search_u8(FsArgs a) {
  extern __shared__ __align__(128) uint32_t smem[];
  __shared__ uint32_t s_org[H * W / 4];
  __shared__ CostIdx s_red[32];
  const int step = a.step;
  for (size_t blk = blockIdx.x; blk < a.nblocks; blk += gridDim.x) {
    const b200_block b = a.blocks[blk];
    const FsWindow w = fs_window(a, b);
    __syncthreads();
    {
      const uint8_t *o = px<uint8_t>(a.cur, b.x, b.y);
      for (int i = threadIdx.x; i < H * W / 4; i += blockDim.x) {
        const int y = i / (W / 4), k = i - y * (W / 4);
        const uint8_t *p = o + (long long)y * a.cur.stride + 4 * k;
        s_org[i] = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) |
                   ((uint32_t)p[3] << 24);
      }
    }
    // stage [x_lo, x_hi + W + 4) x [y_lo, y_hi + H) with column 0 = x_lo (byte-realigned)
    const int npos = w.nx * w.ny;
    const int row_px = npos ? (w.x_hi - w.x_lo) + W : 0;
    // words per row incl. the NP-1 extra positions a task may touch, rounded to 16 bytes so
    // rows stay uint4-aligned (LDS.128); +4 words slack for the funnel-shift form
    const int row_words = ((row_px + 3) / 4 + NP + 4 + 3) & ~3;
    const int pitch_words = row_words;
    const int rows = npos ? (w.y_hi - w.y_lo) + H : 0;
    {
      const int mis = (int)((uintptr_t)a.ref.data & 3);
      const int ax = ((w.x_lo + mis) & ~3) - mis;  // word-aligned source column
      const int d = w.x_lo - ax;                   // byte realignment, 0..3
      const uint8_t *src = px<uint8_t>(a.ref, ax, w.y_lo);
      // Only the row_px bytes [x_lo, x_hi + W) are read: words past them feed only positions beyond
      // nx and are staged as zeros (the window is clamped to get_mv_range, so those bytes may lie
      // past the plane's pad).  Each source word loaded holds at least one byte of the row; its
      // other bytes (up to 3 before x_lo or after x_hi + W - 1, same aligned word) are shifted out.
      const int need = (row_px + 3) / 4;
      for (int i = threadIdx.x; i < rows * row_words; i += blockDim.x) {
        const int y = i / row_words, k = i - y * row_words;
        const uint32_t *s = (const uint32_t *)(src + (long long)y * a.ref.stride) + k;
        uint32_t v = 0u;
        if (k < need) {
          const uint32_t lo = __ldg(s);
          const uint32_t hi = d && 4 * k + 4 - d < row_px ? __ldg(s + 1) : 0u;
          v = __funnelshift_r(lo, hi, d * 8);
        }
        smem[y * pitch_words + k] = v;
      }
    }
    __syncthreads();
    CostIdx best{kEmptyCost, 0xffffffffu};
    const int groups_x = (w.nx + NP - 1) / NP;
    const int ntasks = groups_x * w.ny;
    for (int t = threadIdx.x; t < ntasks; t += blockDim.x) {
      const int py = t / groups_x, g = t - py * groups_x;
      const int px0 = g * NP;                      // first position index in this row
      const int off = px0 * step;                  // byte offset of that position
      const int word0 = off >> 2;
      const uint32_t *wrow = smem + (py * step) * pitch_words + word0;
      uint32_t acc[NP];
#pragma unroll
      for (int p = 0; p < NP; p++) acc[p] = 0;
      if (step == 4 && NP == 4) {
        // word0 = 4*g: 16-byte aligned -> the W/4 + 3 words come in as uint4 (LDS.128),
        // consecutive threads read consecutive 16-byte chunks (conflict free)
        constexpr int NV = (W / 4 + NP - 1 + 3) / 4;
#pragma unroll 2
        for (int y = 0; y < H; y++) {
          uint32_t rw[NV * 4];
          const uint4 *v = (const uint4 *)(wrow + y * pitch_words);
#pragma unroll
          for (int k = 0; k < NV; k++) {
            const uint4 q = v[k];
            rw[4 * k] = q.x, rw[4 * k + 1] = q.y, rw[4 * k + 2] = q.z, rw[4 * k + 3] = q.w;
          }
#pragma unroll
          for (int k = 0; k < W / 4; k++) {
            const uint32_t o = s_org[y * (W / 4) + k];
#pragma unroll
            for (int p = 0; p < NP; p++) acc[p] = sad4_acc(rw[k + p], o, acc[p]);
          }
        }
      } else {
#pragma unroll
        for (int p = 0; p < NP; p++) {
          const int o2 = (px0 + p) * step;
          const int w0 = (o2 >> 2) - word0, s2 = (o2 & 3) * 8;
          for (int y = 0; y < H; y++)
            acc[p] = row_sad_u8<W>(wrow + y * pitch_words, w0, s2, s_org + y * (W / 4), acc[p]);
        }
      }
#pragma unroll
      for (int p = 0; p < NP; p++) {
        if (px0 + p < w.nx) {
          const int x = w.x_lo + (px0 + p) * step, y = w.y_lo + py * step;
          const int mvr = (short)(8 * (short)(y - b.y)), mvc = (short)(8 * (short)(x - b.x));
          const unsigned long long cost =
              b200_mv_cost(acc[p], mvr, mvc, 0, 0, 0, 0, a.lambda, a.allow_hp);
          best = best_min(best, CostIdx{cost, (uint32_t)(py * w.nx + px0 + p)});
        }
      }
    }
    best = block_best(best, s_red);
    if (threadIdx.x == 0) fs_write(a, blk, b, w, best, fs_sad_from_cost(a, b, w, best));
  }
}
template <int W, int H>
int launch_fs_u8(b200_ctx *ctx, const FsArgs &a, size_t smem_bytes) {
  constexpr int NP = W >= 8 ? 4 : 2;
  if (int st = b200_smem_opt_in(ctx, (const void *)me_full_search_u8<W, H, NP>, kFsSmemBytes)) return st;
  const int grid = (int)std::min<size_t>(a.nblocks, (size_t)ctx->num_sms * 32);
  me_full_search_u8<W, H, NP><<<grid, 256, smem_bytes, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

}  // namespace

extern "C" int b200_me_full_search_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                       const b200_block *d_blocks, size_t nblocks,
                                       const b200_me_params *p, int range_x, int range_y, int step,
                                       b200_me_result *d_best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (int st = b200_me_check_planes(ctx, cur, ref, p)) return st;
  B200_REQUIRE(ctx, range_x >= 0 && range_y >= 0 && step >= 1, "bad range/step %d %d %d", range_x,
               range_y, step);
  B200_REQUIRE(ctx, !p->use_satd, "full_search always uses SAD (me.rs:1489)");
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && d_best, "NULL blocks/out");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));

  FsArgs a;
  a.cur = {cur->data, cur->stride};
  a.ref = {ref->data, ref->stride};
  a.blocks = d_blocks;
  a.out = d_best;
  a.nblocks = nblocks;
  a.w = p->w;
  a.h = p->h;
  a.w_in_b = p->frame_w_in_b;
  a.h_in_b = p->frame_h_in_b;
  a.lambda = p->lambda;
  a.allow_hp = p->allow_high_precision_mv;
  a.range_x = range_x;
  a.range_y = range_y;
  a.step = step;

  if (cur->bpp == 1 && (ref->stride & 3) == 0) {
    const int np = p->w >= 8 ? 4 : 2;  // must match launch_fs_u8 / the kernel's row_words
    const size_t row_words = (size_t)(((2 * range_x + p->w + 3) / 4 + np + 4 + 3) & ~3);
    const size_t smem_bytes = row_words * 4 * (size_t)(2 * range_y + p->h);
    if (smem_bytes <= (size_t)kFsSmemBytes) {
#define B200_CASE(W_, H_) \
  if (p->w == W_ && p->h == H_) return launch_fs_u8<W_, H_>(ctx, a, smem_bytes);
      B200_CASE(8, 8)
      B200_CASE(16, 16)
      B200_CASE(32, 32)
      B200_CASE(64, 64)
#undef B200_CASE
    }
  }
  const int grid = (int)std::min<size_t>(nblocks, (size_t)ctx->num_sms * 16);
  if (cur->bpp == 1)
    me_full_search_generic<uint8_t><<<grid, 256, 0, ctx->stream>>>(a);
  else
    me_full_search_generic<uint16_t><<<grid, 256, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
