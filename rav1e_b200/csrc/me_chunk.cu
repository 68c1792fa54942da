// me_chunk.cu — sparse candidate lists in 8x8 chunks for sm_90a: the staged chunk kernel behind
// b200_me_candidates_dev / _multi_dev for 8-bit SATD lists and 16-bit SAD / SATD lists (me_cand.cu
// routes them here).
//
// Kernels
//   me_chunk_lists<T,W,H,SATD>  a warp per block, candidates' footprints staged per warp with
//                           cp.async, thread per (candidate, 8x8 chunk).  Fused cost + argmin.
//
// The warp-per-block kernel (me_cand_warp_u8) gives every thread one 8x8 chunk of one candidate and
// lets it fetch its own 8 rows: 32 threads read 32 different places per load (32 cache lines per
// instruction, L1 tag bound, 120 registers).  This kernel keeps the
// thread-per-chunk arithmetic (no shuffles inside the transform) but separates fetching from
// evaluating and pipelines the two across blocks.  Per warp, for the blocks b0, b1, ... it owns:
//   header   (block position, candidate range)        loaded three blocks ahead        -> registers
//   record   (this lane's candidate)                  loaded two blocks ahead          -> registers
//   stage    the candidates' footprints, whole 16-byte aligned segments with lanes walking
//            (row, segment) so one instruction touches H cache lines instead of 32, and the block's
//            org rows, copied global -> shared with cp.async (LDGSTS: no registers, asynchronous)
//            one block ahead into the other half of a double buffer;
//   evaluate thread (candidate, chunk) reads its 8 rows from shared memory (3 words + funnel shift
//            per row), runs the horizontal pass as IDP.4A chains (t = H.org - H.ref, 4 dp4a per
//            output, nothing on the ALU pipe), the vertical pass as register butterflies whose last
//            stage is folded into the sum (|a+b| + |a-b| = 2 max(|a|,|b|)); the chunk sums of a
//            candidate meet by shuffle.
// No dependent global load is waited for inside a block: every wait is for data requested at least
// one block earlier.  Blocks with more than CPP = 32 / NCH candidates take their further batches
// in place (not pipelined).  Same results as get_satd (dist.rs:156-221): exact integer arithmetic,
// one final rounding.
#include <cuda_runtime.h>

#include "common.cuh"
#include "me_cand.cuh"
#include "me_dev.cuh"

#ifndef B200_SATD_SPARSE_MINBLOCKS
#define B200_SATD_SPARSE_MINBLOCKS 2
#endif

using namespace b200_me;

namespace {

template <typename T, int W, int H>
struct SatdSparseCfg {
  static constexpr int BPP = (int)sizeof(T);
  static constexpr int CW = W / 8, CH = H / 8, NCH = CW * CH;
  static constexpr int CPP = 32 / NCH;                    // candidates per batch
  static constexpr int NSEG = (W * BPP + 30) / 16;        // 16-byte segments covering a row + 15 bytes
  static constexpr int ROWW = NSEG * 4;                   // words per staged row
  static constexpr int CANDW0 = H * ROWW + 4 * CH;        // + one 16-byte pad per chunk row (bank spread)
  static constexpr int CANDW = CANDW0 + ((8 - CANDW0 % 32 + 32) % 32);  // == 8 (mod 32), 16-byte multiple
  static constexpr int CHW = 2 * BPP;                     // words of one chunk row (8 pixels)
  static constexpr int ORGW = NCH * 8 * CHW;              // org words: [chunk][row][CHW]
  static constexpr int BUFW = CPP * CANDW + ORGW;   // one half of the double buffer
  static constexpr int WARP_WORDS = 2 * BUFW;
  static constexpr int WARPS = 8;
  static constexpr size_t SMEM = (size_t)WARPS * WARP_WORDS * 4;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}

struct SatdHdr {   // what a stage needs to know about a block
  uint32_t lo, hi;  // candidate range
  b200_block b;
};
struct SatdLane {  // this lane's candidate of a batch and what staging derived from it
  b200_cand c;
  int mis;   // (reference address of the candidate's first pixel) & 15
  bool inr;  // in the block's mv range (evaluated and reported)
};

template <typename T, int W, int H, bool SATD>
__global__ void __launch_bounds__(256, B200_SATD_SPARSE_MINBLOCKS)
    me_chunk_lists(const __grid_constant__ MeArgs a) {
  using C = SatdSparseCfg<T, W, H>;
  constexpr int BPP = C::BPP, CHW = C::CHW;
  constexpr int CW = C::CW, NCH = C::NCH, CPP = C::CPP, NSEG = C::NSEG, ROWW = C::ROWW, CANDW = C::CANDW,
                BUFW = C::BUFW;
  extern __shared__ __align__(128) uint32_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t *const wbuf = smem + warp * C::WARP_WORDS;
  const uint32_t wbuf_s = smem_u32(wbuf);
  const int myc = lane / NCH, chunk = lane - myc * NCH;  // evaluation role: (candidate, chunk)
  const int cy = chunk / CW, cx = chunk - cy * CW;
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  const size_t blk_end = a.pr.block_end[a.pr.n - 1];
  const size_t blk0 = a.pr.block_begin + (size_t)blockIdx.x * (blockDim.x >> 5) + warp;

  auto fetch_hdr = [&](size_t blk) {
    SatdHdr h;
    h.lo = h.hi = 0;
    h.b.x = h.b.y = 0;
    if (blk < blk_end) {
      h.lo = __ldg(a.cand_offsets + blk);
      h.hi = __ldg(a.cand_offsets + blk + 1);
      h.b = a.blocks[blk];
    }
    return h;
  };
  auto fetch_cand = [&](const SatdHdr &h, uint32_t base) {
    b200_cand c;
    c.block = 0;
    c.mv_row = 0;
    c.mv_col = 0;
    if (base + myc < h.hi) c = a.cands[base + myc];
    return c;
  };
  // stage one batch (and, with_org, the block's org rows) into half `half` of the double buffer
  // staging roles, fixed per lane: unit u = u0 + lane = (candidate, row, segment) for every step u0
  constexpr int UPC = H * NSEG;  // units per candidate
  constexpr int NSTEP = CPP * UPC / 32;
  int st_src[NSTEP], st_dst[NSTEP], st_lane[NSTEP];  // per step: row * stride is added per block
  int st_row[NSTEP];
#pragma unroll
  for (int k = 0; k < NSTEP; k++) {
    const int u = k * 32 + lane;
    const int uc = u / UPC, rem = u - uc * UPC, R = rem / NSEG, seg = rem - R * NSEG;
    st_row[k] = R;
    st_src[k] = seg * 16;
    st_dst[k] = (uc * CANDW + R * ROWW + 4 * (R >> 3) + seg * 4) * 4;
    st_lane[k] = (uc * NCH) & 31;
  }
  constexpr int kNoCand = INT_MIN;
  auto stage = [&](size_t blk, int pi, const SatdHdr &h, uint32_t base, const b200_cand &c, int half,
                   bool with_org) {
    SatdLane L;
    L.c = c;
    L.mis = 0;
    L.inr = false;
    if (blk < blk_end) {
      const PlaneView cur = a.pr.cur[pi], ref = a.pr.ref[pi];
      const MvRange r = b200_mv_range(a.w_in_b, a.h_in_b, h.b.x / MI_SIZE, h.b.y / MI_SIZE, W, H);
      L.inr = base + myc < h.hi && !B200_MV_OUTSIDE(c.mv_row, c.mv_col, r);
      // byte offset of the candidate's first pixel from pixel (0,0) of the reference plane (planes
      // are far smaller than 2 GB), split into its 16-byte aligned part and the misalignment
      const int off = ((h.b.y + c.mv_row / 8) * ref.stride + h.b.x + c.mv_col / 8) * BPP;
      L.mis = (int)(((uintptr_t)ref.data + (unsigned)off) & 15);
      const int segoff = L.inr ? off - L.mis : kNoCand;
      const uint32_t dst0 = wbuf_s + (uint32_t)(half * BUFW) * 4u;
      const uint8_t *rbase = (const uint8_t *)ref.data;
#pragma unroll
      for (int k = 0; k < NSTEP; k++) {
        const int so = __shfl_sync(0xffffffffu, segoff, st_lane[k]);
        if (so != kNoCand) cp_async16(dst0 + (uint32_t)st_dst[k], rbase + (so + st_row[k] * ref.stride * BPP + st_src[k]));
      }
      if (with_org) {  // org rows as [chunk][row][8 pixels]
        const uint8_t *op = (const uint8_t *)px<T>(cur, h.b.x, h.b.y);
        const uint32_t odst = dst0 + (uint32_t)(CPP * CANDW) * 4u;
        const int al = (int)((uintptr_t)op | (uintptr_t)(unsigned)(cur.stride * BPP)) & (8 * BPP - 1);
#pragma unroll
        for (int t0 = 0; t0 < NCH * 8; t0 += 32) {
          const int t = t0 + lane;  // unit t = (chunk, row): 8 pixels
          if ((NCH * 8) % 32 == 0 || t < NCH * 8) {
            const int ch = t >> 3, row = t & 7;
            const int ocy = ch / CW, ocx = ch - ocy * CW;
            const uint8_t *q = op + ((ocy * 8 + row) * cur.stride + ocx * 8) * BPP;
            const uint32_t d = odst + (uint32_t)t * (8u * BPP);
            if (al == 0) {
              if (BPP == 1)
                asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(q) : "memory");
              else
                cp_async16(d, q);
            } else if ((al & 3) == 0) {
#pragma unroll
              for (int k = 0; k < CHW; k++) cp_async4(d + 4u * k, q + 4 * k);
            } else {  // rare: blocks on odd byte addresses take the synchronous way
              const int osh = (int)((uintptr_t)q & 3);
              const uint32_t *qw = (const uint32_t *)(q - osh);
              uint32_t *dw = wbuf + half * BUFW + CPP * CANDW + CHW * t;
              uint32_t lo = __ldg(qw);
#pragma unroll
              for (int k = 0; k < CHW; k++) {
                const uint32_t hi = __ldg(qw + k + 1);
                dw[k] = __funnelshift_r(lo, hi, osh * 8);
                lo = hi;
              }
            }
          }
        }
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    return L;
  };
  // evaluate this thread's chunk of its candidate from half `half`; every lane of a candidate
  // returns the candidate's SATD
  auto evaluate = [&](int half, int mis) -> uint32_t {
    const int off = mis + cx * 8 * BPP;
    const uint32_t *rowp = wbuf + half * BUFW + myc * CANDW + (cy * 8) * ROWW + 4 * cy + (off >> 2);
    const uint32_t *orgp = wbuf + half * BUFW + CPP * CANDW + chunk * 8 * CHW;
    const int sh = (off & 3) * 8;
    uint32_t acc;
    if constexpr (BPP == 1 && SATD) {
      int t[8][8];
#pragma unroll
      for (int y = 0; y < 8; y++) {
        const uint32_t w0 = rowp[y * ROWW], w1 = rowp[y * ROWW + 1], w2 = rowp[y * ROWW + 2];
        const uint32_t q0 = __funnelshift_r(w0, w1, sh), q1 = __funnelshift_r(w1, w2, sh);
        const uint2 o = ((const uint2 *)orgp)[y];
        // t = H.org - H.ref for the row: Hadamard rows on the org bytes, negated ones on the
        // reference bytes; outputs 4..7 take the second word of each with the opposite sign
        t[y][0] = dp4a_us(q1, 0xFFFFFFFFu, dp4a_us(q0, 0xFFFFFFFFu, dp4a_us(o.y, 0x01010101u, dp4a_us(o.x, 0x01010101u, 0))));
        t[y][1] = dp4a_us(q1, 0x01FF01FFu, dp4a_us(q0, 0x01FF01FFu, dp4a_us(o.y, 0xFF01FF01u, dp4a_us(o.x, 0xFF01FF01u, 0))));
        t[y][2] = dp4a_us(q1, 0x0101FFFFu, dp4a_us(q0, 0x0101FFFFu, dp4a_us(o.y, 0xFFFF0101u, dp4a_us(o.x, 0xFFFF0101u, 0))));
        t[y][3] = dp4a_us(q1, 0xFF0101FFu, dp4a_us(q0, 0xFF0101FFu, dp4a_us(o.y, 0x01FFFF01u, dp4a_us(o.x, 0x01FFFF01u, 0))));
        t[y][4] = dp4a_us(q1, 0x01010101u, dp4a_us(q0, 0xFFFFFFFFu, dp4a_us(o.y, 0xFFFFFFFFu, dp4a_us(o.x, 0x01010101u, 0))));
        t[y][5] = dp4a_us(q1, 0xFF01FF01u, dp4a_us(q0, 0x01FF01FFu, dp4a_us(o.y, 0x01FF01FFu, dp4a_us(o.x, 0xFF01FF01u, 0))));
        t[y][6] = dp4a_us(q1, 0xFFFF0101u, dp4a_us(q0, 0x0101FFFFu, dp4a_us(o.y, 0x0101FFFFu, dp4a_us(o.x, 0xFFFF0101u, 0))));
        t[y][7] = dp4a_us(q1, 0x01FFFF01u, dp4a_us(q0, 0xFF0101FFu, dp4a_us(o.y, 0xFF0101FFu, dp4a_us(o.x, 0x01FFFF01u, 0))));
      }
      uint32_t s = 0;
#pragma unroll
      for (int col = 0; col < 8; col++) {
        int v[8];
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = t[k][col];
        hadamard8<2>(v);
        // last stage pairs (k, k + 4): |x + y| + |x - y| = 2 max(|x|, |y|)
#pragma unroll
        for (int k = 0; k < 4; k++) s += (uint32_t)max(abs(v[k]), abs(v[k + 4]));
      }
      acc = 2u * s;
    } else if constexpr (SATD) {  // 16-bit pixels: differences unpacked, butterflies in both directions
      int t[8][8];
#pragma unroll
      for (int y = 0; y < 8; y++) {
        uint32_t w[5];
#pragma unroll
        for (int k = 0; k < 5; k++) w[k] = rowp[y * ROWW + k];
        const uint4 o = ((const uint4 *)orgp)[y];
        const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
        int d[8];
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const uint32_t r = __funnelshift_r(w[k], w[k + 1], sh);
          d[2 * k] = (int)(ow[k] & 0xffffu) - (int)(r & 0xffffu);
          d[2 * k + 1] = (int)(ow[k] >> 16) - (int)(r >> 16);
        }
        hadamard8(d);
#pragma unroll
        for (int k = 0; k < 8; k++) t[y][k] = d[k];
      }
      uint32_t s = 0;
#pragma unroll
      for (int col = 0; col < 8; col++) {
        int v[8];
#pragma unroll
        for (int k = 0; k < 8; k++) v[k] = t[k][col];
        hadamard8<2>(v);
#pragma unroll
        for (int k = 0; k < 4; k++) s += (uint32_t)max(abs(v[k]), abs(v[k + 4]));
      }
      acc = 2u * s;
    } else if constexpr (BPP == 1) {  // SAD, 8-bit: VABSDIFF4 with the accumulator fused
      acc = 0;
#pragma unroll
      for (int y = 0; y < 8; y++) {
        const uint32_t w0 = rowp[y * ROWW], w1 = rowp[y * ROWW + 1], w2 = rowp[y * ROWW + 2];
        const uint2 o = ((const uint2 *)orgp)[y];
        acc = sad4_acc(__funnelshift_r(w0, w1, sh), o.x, acc);
        acc = sad4_acc(__funnelshift_r(w1, w2, sh), o.y, acc);
      }
    } else {  // SAD, 16-bit: |a - b| per u16 lane = max - min, lanes summed packed (8 rows x 4095 < 2^16)
      uint32_t pk[4] = {0, 0, 0, 0};
#pragma unroll
      for (int y = 0; y < 8; y++) {
        uint32_t w[5];
#pragma unroll
        for (int k = 0; k < 5; k++) w[k] = rowp[y * ROWW + k];
        const uint4 o = ((const uint4 *)orgp)[y];
        const uint32_t ow[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const uint32_t r = __funnelshift_r(w[k], w[k + 1], sh);
          pk[k] += __vmaxu2(ow[k], r) - __vminu2(ow[k], r);
        }
      }
      acc = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) acc += (pk[k] & 0xffffu) + (pk[k] >> 16);
    }
#pragma unroll
    for (int o = NCH >> 1; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    return SATD ? (acc + 4u) >> 3 : acc;  // dist.rs:219-220: one final rounding (8x8 chunks: ln = 3)
  };

  // ---- prologue: headers of blocks 0..2, records of 0..1, block 0 staged
  size_t blk = blk0;
  SatdHdr h0 = fetch_hdr(blk), h1 = fetch_hdr(blk + nwarps), h2 = fetch_hdr(blk + 2 * nwarps);
  b200_cand c0 = fetch_cand(h0, h0.lo), c1 = fetch_cand(h1, h1.lo);
  // plane pair of a block: the warp's blocks come in ascending order, the pair index only grows
  uint32_t pair_end = a.pr.block_end[0];  // end of the pair the newest staged block belongs to
  auto advance_pair = [&](int pi, size_t b) {
    if ((uint32_t)b < pair_end) return pi;  // the usual case costs one compare
    while (pi + 1 < a.pr.n && (uint32_t)b >= a.pr.block_end[pi]) pi++;
    pair_end = a.pr.block_end[pi];
    return pi;
  };
  int pi0 = advance_pair(0, blk);
  SatdLane L0 = stage(blk, pi0, h0, h0.lo, c0, 0, true);
  int half = 0;
  for (; blk < blk_end; blk += nwarps) {
    // ---- look ahead: stage block k+1, request block k+2's records and block k+3's header
    const int pi1 = advance_pair(pi0, blk + nwarps);
    const SatdLane L1 = stage(blk + nwarps, pi1, h1, h1.lo, c1, half ^ 1, true);
    const b200_cand c2 = fetch_cand(h2, h2.lo);
    const SatdHdr h3 = fetch_hdr(blk + 3 * nwarps);
    const Pmv pm = load_pmv(a.pmv, blk);
    // ---- block k: its footprints were requested one block ago
    asm volatile("cp.async.wait_group 1;" ::: "memory");
    __syncwarp();
    unsigned long long best = ~0ull;
    uint32_t best_sad = kEmptySad;  // this lane's best candidate so far: the lane that owns the block's
    short best_row = 0, best_col = 0;  // first minimum writes the record itself
    SatdLane L = L0;
    for (uint32_t base = h0.lo;;) {
      const uint32_t i = base + myc;
      const uint32_t acc = evaluate(half, L.mis);
      uint32_t sad = kEmptySad;
      unsigned long long cost = kEmptyCost, key = ~0ull;
      if (L.inr && chunk == 0) {
        sad = acc;
        cost = b200_mv_cost(sad, L.c.mv_row, L.c.mv_col, pm.r0, pm.c0, pm.r1, pm.c1, a.lambda, a.allow_hp);
        key = pack_key(cost, i - h0.lo);
      }
      if (i < h0.hi && chunk == 0) {
        if (a.out_sad) a.out_sad[i] = sad;
        if (a.out_cost) a.out_cost[i] = cost;
      }
      if (key < best) best = key, best_sad = sad, best_row = L.c.mv_row, best_col = L.c.mv_col;
      base += CPP;
      if (base >= h0.hi) break;
      // further batches of a long list, in place: this half is free once every lane has evaluated
      __syncwarp();
      L = stage(blk, pi0, h0, base, fetch_cand(h0, base), half, false);
      asm volatile("cp.async.wait_group 0;" ::: "memory");
      __syncwarp();
    }
    if (a.out_best) {
      // keys are unique (they carry the candidate's index), so exactly one lane holds the minimum;
      // with no candidate in range every key is ~0 and lane 0 writes MotionSearchResult::empty()
      const unsigned long long key = warp_min_key(best);
      if (key == ~0ull ? lane == 0 : best == key) {
        b200_me_result res;
        res.cost = key == ~0ull ? kEmptyCost : key >> kKeyIdxBits;
        res.sad = best_sad;
        res.mv_row = best_row;
        res.mv_col = best_col;
        a.out_best[blk] = res;
      }
    }
    __syncwarp();  // every lane is done with this half before block k+2 is staged into it
    h0 = h1, h1 = h2, h2 = h3;
    c0 = c1, c1 = c2;
    L0 = L1;
    pi0 = pi1;
    half ^= 1;
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

template <typename T, int W, int H, bool SATD>
int launch_chunk_lists(b200_ctx *ctx, const MeArgs &a) {
  using C = SatdSparseCfg<T, W, H>;
  if (int st = b200_smem_opt_in(ctx, (const void *)me_chunk_lists<T, W, H, SATD>, (int)C::SMEM)) return st;
  const int wpc = C::WARPS;
  const int grid = (int)std::min<size_t>((a.nblocks + wpc - 1) / wpc, (size_t)ctx->num_sms * 16);
  me_chunk_lists<T, W, H, SATD><<<grid, wpc * 32, C::SMEM, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

}  // namespace

ChunkListsLaunch b200_me::chunk_lists_launcher(int bpp, int w, int h, bool satd) {
#define B200_U8(W_, H_) \
  if (w == W_ && h == H_) return launch_chunk_lists<uint8_t, W_, H_, true>;
#define B200_U16(W_, H_) \
  if (w == W_ && h == H_) return satd ? launch_chunk_lists<uint16_t, W_, H_, true> : launch_chunk_lists<uint16_t, W_, H_, false>;
  if (bpp == 1 && satd) {  // 8-bit SAD lists stay with the grouped and warp kernels
    B200_U8(8, 8)
    B200_U8(16, 16)
    B200_U8(32, 32)
    B200_U8(8, 16)
    B200_U8(16, 8)
    B200_U8(16, 32)
    B200_U8(32, 16)
    B200_U8(32, 64)
    B200_U8(64, 32)
  }
  if (bpp == 2) {
    B200_U16(8, 8)
    B200_U16(16, 16)
    B200_U16(32, 32)
    B200_U16(8, 16)
    B200_U16(16, 8)
    B200_U16(16, 32)
    B200_U16(32, 16)
  }
#undef B200_U8
#undef B200_U16
  return nullptr;
}
