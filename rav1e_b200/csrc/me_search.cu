// me_search.cu — the move-to-best search stages of rav1e's full_pixel_me on the device.
//
// Replaces, for every block of a frame (or of several (cur, ref) plane pairs) in one launch, the
// serial per-block chain of src/me.rs:
//   full_pixel_me            :692-856   (the `try_cands` closure, the extensive-search ladder)
//   get_best_predictor       :884-909
//   fullpel_diamond_search   :955-998   (4-point diamond, radius 2 then 1, move until no gain)
//   hexagon_search           :1055-1135 (6 / 3-point hexagon, then the 8-point square)
//   uneven_multi_hex_search  :1170-1303 (cross 24 + 12, 5x5, 16-point hexagons x 6 scales)
// The exhaustive grid that may follow (:822-846) is b200_me_full_search_dev.
//
// One WARP per block.  A stage's candidate set is evaluated four candidates at a time (8 lanes
// each, lane = row mod 8), straight from the planes through L1 (neighbouring candidates overlap
// almost entirely); every "if rd.cost < best.cost" chain of the reference is a first-minimum
// argmin over the set, so the winner is found with shuffles and the data-dependent control flow
// (move, shrink the radius, early exits) stays warp-uniform.  Predictor subsets come from the
// caller: get_subset_predictors (me.rs:381-533) reads neighbouring blocks' results of the same
// pass, a wavefront dependency that stays with the encoder's block order.
#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"

#ifndef B200_SEARCH_MINBLOCKS
#define B200_SEARCH_MINBLOCKS 6  // CTAs of 4 warps per SM the search kernel is register-capped for (80 regs)
#endif

namespace {

constexpr unsigned long long kEmptyCost = ~0ull;  // MVCandidateRD::empty(), me.rs:139-146
constexpr uint32_t kEmptySad = ~0u;
constexpr int kMaxPairs = 32;

struct PlaneRef {
  const void *data;  // pixel (0,0)
  int stride;        // elements
};

struct SearchArgs {
  int npairs;
  uint32_t block_end[kMaxPairs];  // pair k owns blocks [block_end[k-1], block_end[k])
  PlaneRef cur[kMaxPairs], ref[kMaxPairs];
  const b200_block *blocks;
  const b200_cand *preds;
  const uint32_t *subset_offsets;  // nblocks * nsubsets + 1
  const short *pmv;                // 4 shorts per block or null
  const uint32_t *thresh;          // per block (extensive ladder) or null
  b200_me_result *out;
  size_t nblocks;
  int nsubsets;  // 1: all_mvs (non-extensive); 3: median | subset_b | subset_c
  int w, h, w_in_b, h_in_b;
  uint32_t lambda;
  int allow_hp;
  int umh_range;
};

struct Best {  // MotionSearchResult (+ the index of the winner inside its candidate set)
  unsigned long long cost;
  uint32_t sad;
  int row, col;  // i16 values
  int idx;
};

__device__ __forceinline__ Best best_empty() {
  Best b;
  b.cost = kEmptyCost;
  b.sad = kEmptySad;
  b.row = 0;
  b.col = 0;
  b.idx = 0x7fffffff;
  return b;
}

__device__ __forceinline__ uint32_t sad4_acc(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t d;
  asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}

// search_pattern! tables (me.rs:944-947, :1022-1025, :1035-1038, :1153-1156), full pixels
__constant__ signed char kDiamond[4][2] = {{1, 0}, {0, 1}, {-1, 0}, {0, -1}};  // {row, col}
__constant__ signed char kHexagon[6][2] = {{-2, 0}, {-1, 2}, {1, 2}, {2, 0}, {1, -2}, {-1, -2}};
__constant__ signed char kSquare[8][2] = {{1, -1}, {1, 0}, {1, 1}, {0, -1}, {0, 1}, {-1, -1}, {-1, 0}, {-1, 1}};
__constant__ signed char kUmh[16][2] = {{4, -2}, {4, -1}, {4, 0},  {4, 1},   {4, 2},   {2, 3},  {0, 4},  {-2, 3},
                                        {-4, 2}, {-4, 1}, {-4, 0}, {-4, -1}, {-4, -2}, {-2, 3}, {0, -4}, {2, -3}};

constexpr int kOrgRegs = 16;  // org words a lane keeps in registers (blocks up to 512 bytes)

struct BlockCtx {
  const uint8_t *org;   // block pixel (0,0), bytes
  long long org_pitch;  // bytes
  const uint8_t *ref0;
  long long ref_pitch;  // bytes
  int po_x, po_y;
  MvRange rng;
  int p0r, p0c, p1r, p1c;
  int w, h;
  int log_nw;  // log2(words per block row)
  int total;   // words per block
  bool cached;  // the lane's org words are in orgw[]
  uint32_t orgw[kOrgRegs];
  uint32_t lambda;
  int allow_hp;
};

// word `i` (row-major, nw words per row) of the w x h area whose pixel (0,0) is at byte address
// `p0` (any alignment; the row pitch is a multiple of 4 bytes)
__device__ __forceinline__ uint32_t load_word(const uint8_t *p0, long long pitch, int y, int k) {
  const uint8_t *p = p0 + (long long)y * pitch + 4 * k;
  const int sh = (int)((uintptr_t)p & 3);
  const uint32_t *q = (const uint32_t *)(p - sh);
  const uint32_t lo = __ldg(q);
  return sh ? __funnelshift_r(lo, __ldg(q + 1), sh * 8) : lo;
}

template <typename T>
__device__ __forceinline__ uint32_t word_sad(uint32_t a, uint32_t b, uint32_t acc) {
  if (sizeof(T) == 1) return sad4_acc(a, b, acc);
  // |a - b| per u16 lane = max - min (VIMNMX.U16x2 twice; max >= min per lane, so the 32-bit subtraction
  // never borrows across lanes) - __vabsdiffu2 expands to ten instructions
  const uint32_t d = __vmaxu2(a, b) - __vminu2(a, b);
  return acc + (d & 0xffffu) + (d >> 16);
}

// The 8 lanes of a candidate's group walk the block's words 8 at a time (lane = word index mod 8:
// neighbouring lanes read neighbouring bytes, so one load touches few cache lines).  The word to the
// right - needed to realign an unaligned reference row - comes from the neighbouring lane by
// shuffle; only the last lane of a row segment loads it.  Called by all 32 lanes (candidates that
// are out of range evaluate the zero vector and are discarded by the caller).
template <typename T>
__device__ __forceinline__ uint32_t partial_sad(const BlockCtx &c, int dx, int dy, int sub) {
  const uint8_t *r0 = c.ref0 + (long long)(c.po_y + dy) * c.ref_pitch + (long long)(c.po_x + dx) * (long long)sizeof(T);
  const int rsh = (int)((uintptr_t)r0 & 3);
  const uint32_t *rw = (const uint32_t *)(r0 - rsh);
  const long long rpw = c.ref_pitch >> 2;
  const int nw = 1 << c.log_nw, seg = nw < 8 ? nw : 8;  // words of one row a group covers per step
  uint32_t acc = 0;
  if (c.cached) {
#pragma unroll
    for (int j = 0; j < kOrgRegs; j++) {
      const int i = sub + 8 * j;
      const bool on = i < c.total;  // uniform per step except in blocks smaller than 8 words
      const int y = i >> c.log_nw, k = i & (nw - 1);
      const uint32_t *q = rw + (on ? (long long)y * rpw + k : 0);
      const uint32_t w0 = __ldg(q);
      uint32_t w1 = __shfl_down_sync(0xffffffffu, w0, 1);
      if (rsh && ((k & (seg - 1)) == seg - 1 || !on)) w1 = __ldg(q + 1);
      if (on) acc = word_sad<T>(__funnelshift_r(w0, w1, rsh * 8), c.orgw[j], acc);
      if (8 * (j + 1) >= c.total) break;  // uniform
    }
  } else {
    // same row-end rule as the cached path (a 16x64 8-bit block has 4 words per row: two rows per
    // step); uniform trip count so every full-mask shuffle is executed by all 32 lanes
    for (int i0 = 0; i0 < c.total; i0 += 8) {
      const int i = i0 + sub;
      const bool on = i < c.total;
      const int y = i >> c.log_nw, k = i & (nw - 1);
      const uint32_t *q = rw + (on ? (long long)y * rpw + k : 0);
      const uint32_t w0 = __ldg(q);
      uint32_t w1 = __shfl_down_sync(0xffffffffu, w0, 1);
      if (rsh && ((k & (seg - 1)) == seg - 1 || !on)) w1 = __ldg(q + 1);
      if (on) acc = word_sad<T>(__funnelshift_r(w0, w1, rsh * 8), load_word(c.org, c.org_pitch, y, k), acc);
    }
  }
  return acc;
}

__device__ __forceinline__ int s16(int v) { return (int)(short)v; }  // i16 wrap (release builds)

// The stages as a state machine with ONE evaluation site: every stage is "evaluate a candidate
// set, keep its first minimum" (what `for cand { if rd.cost < best.cost { best = rd } }` leaves
// when started from empty(), me.rs:884-909 and every pattern loop), followed by a transition.
enum Stage {
  S_PRED,     // get_best_predictor over a subset                         me.rs:884-909
  S_DIAMOND,  // fullpel_diamond_search, radius 2 then 1                  me.rs:955-998
  S_CROSS,    // uneven_multi_hex_search: both lines of the cross         me.rs:1187-1234
  S_FIVE,     //   5x5 (raw eighth-pel offsets)                           me.rs:1237-1253
  S_UMH,      //   16-point hexagons x (me_range >> 2) scales             me.rs:1281-1296
  S_HEX6,     // hexagon_search: first iteration                          me.rs:1070-1083
  S_HEX3,     //   following iterations (3 new points)                    me.rs:1087-1115
  S_SQUARE,   //   square refinement                                      me.rs:1118-1132
  S_DONE
};

template <typename T>
__global__ void __launch_bounds__(128, B200_SEARCH_MINBLOCKS) me_search_kernel(const __grid_constant__ SearchArgs a) {
  const size_t warp0 = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  const int lane = threadIdx.x & 31, g = lane >> 3, sub = lane & 7;
  for (size_t blk = warp0; blk < a.nblocks; blk += nwarps) {
    int pi = 0;
    if (a.npairs > 1) {  // first pair with blk < block_end
      int lo = 0, hi = a.npairs - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if ((uint32_t)blk < a.block_end[mid])
          hi = mid;
        else
          lo = mid + 1;
      }
      pi = lo;
    }
    const b200_block bk = a.blocks[blk];
    BlockCtx c;
    c.org_pitch = (long long)a.cur[pi].stride * (long long)sizeof(T);
    c.ref_pitch = (long long)a.ref[pi].stride * (long long)sizeof(T);
    c.org = (const uint8_t *)a.cur[pi].data + (long long)bk.y * c.org_pitch + (long long)bk.x * (long long)sizeof(T);
    c.ref0 = (const uint8_t *)a.ref[pi].data;
    c.po_x = bk.x;
    c.po_y = bk.y;
    c.w = a.w;
    c.h = a.h;
    c.rng = b200_mv_range(a.w_in_b, a.h_in_b, bk.x / MI_SIZE, bk.y / MI_SIZE, a.w, a.h);
    c.p0r = c.p0c = c.p1r = c.p1c = 0;
    if (a.pmv) {
      const short *p = a.pmv + 4 * blk;
      c.p0r = p[0], c.p0c = p[1], c.p1r = p[2], c.p1c = p[3];
    }
    c.lambda = a.lambda;
    c.allow_hp = a.allow_hp;
    {
      const int nw = a.w * (int)sizeof(T) / 4;  // power of two (host-checked)
      c.log_nw = 31 - __clz(nw);
      c.total = nw * a.h;
      c.cached = c.total <= 8 * kOrgRegs;
      if (c.cached) {
#pragma unroll
        for (int j = 0; j < kOrgRegs; j++) {
          const int i = sub + 8 * j;
          c.orgw[j] = i < c.total ? load_word(c.org, c.org_pitch, i >> c.log_nw, i & (nw - 1)) : 0u;
        }
      }
    }
    const int n_row = (a.umh_range + 1) >> 1;         // cross, first line: i = 1, 3, ... <= me_range
    const int n_col = ((a.umh_range >> 1) + 1) >> 1;  // second line: i = 1, 3, ... <= me_range / 2
    const uint32_t thresh = a.nsubsets == 3 ? a.thresh[blk] : 0u;

    Best best = best_empty();  // full_pixel_me's `best`
    Best cur = best_empty();   // the running stage's `current` / `results`
    int subset = 0, radius_log2 = 1, center_idx = 0, best_idx = 0;
    int cr = 0, cc = 0;        // centre the running pattern is laid around
    uint32_t plo = 0;          // first predictor of the running subset
    int stage = S_DONE, n = 0;

    // pick the next predictor subset (or what follows the last one)
    auto next_subset = [&]() {
      while (subset < a.nsubsets) {
        const uint32_t lo = a.subset_offsets[blk * a.nsubsets + subset];
        const uint32_t hi = a.subset_offsets[blk * a.nsubsets + subset + 1];
        if (a.nsubsets == 3 && subset == 0 && lo == hi) {  // `if let Some(median)`, me.rs:774
          subset++;
          continue;
        }
        plo = lo;
        n = (int)(hi - lo);
        stage = S_PRED;
        return;
      }
      if (a.nsubsets == 3 && a.umh_range > 0 && best.cost != kEmptyCost) {  // me.rs:794-812
        cur = best;
        cr = cur.row, cc = cur.col;
        n = 2 * (n_row + n_col);
        stage = S_CROSS;
      } else {
        stage = S_DONE;
      }
    };
    next_subset();

    while (stage != S_DONE) {
      // ---- evaluate the stage's candidate set, four candidates at a time (8 lanes each)
      Best b = best_empty();
      for (int k0 = 0; k0 < n; k0 += 4) {
        const int k = k0 + g;
        int row = cr, col = cc;
        switch (stage) {
          case S_PRED:
            if (k < n) {
              const b200_cand q = a.preds[plo + k];
              row = q.mv_row, col = q.mv_col;
            }
            break;
          case S_DIAMOND:
            row = s16(cr + s16(kDiamond[k & 3][0] * (8 << radius_log2)));
            col = s16(cc + s16(kDiamond[k & 3][1] * (8 << radius_log2)));
            break;
          case S_CROSS:  // quirk kept: the first ("horizontal") line steps the ROW, me.rs:1195-1198
            if (k < 2 * n_row) {
              row = s16(cr + s16(((k & 1) ? 8 : -8) * (1 + 2 * (k >> 1))));
            } else {
              const int kk = k - 2 * n_row;
              col = s16(cc + s16(((kk & 1) ? 8 : -8) * (1 + 2 * (kk >> 1))));
            }
            break;
          case S_FIVE: {  // row-major 5x5 without its centre, raw {row, col} (me.rs:1240-1246)
            const int idx = k < 12 ? k : k + 1;
            row = s16(cr + idx / 5 - 2);
            col = s16(cc + idx % 5 - 2);
            break;
          }
          case S_UMH:
            row = s16(cr + s16(kUmh[k & 15][0] * 8 * (1 + (k >> 4))));
            col = s16(cc + s16(kUmh[k & 15][1] * 8 * (1 + (k >> 4))));
            break;
          case S_HEX6:
            row = s16(cr + kHexagon[k % 6][0] * 8);
            col = s16(cc + kHexagon[k % 6][1] * 8);
            break;
          case S_HEX3: {
            const int i = (center_idx + 5 + k) % 6;
            row = s16(cr + kHexagon[i][0] * 8);
            col = s16(cc + kHexagon[i][1] * 8);
            break;
          }
          default:  // S_SQUARE
            row = s16(cr + kSquare[k & 7][0] * 8);
            col = s16(cc + kSquare[k & 7][1] * 8);
            break;
        }
        // get_fullpel_mv_rd, me.rs:1386-1409
        const bool inr = k < n && !(col < c.rng.x_min || col > c.rng.x_max || row < c.rng.y_min || row > c.rng.y_max);
        uint32_t acc = partial_sad<T>(c, inr ? col / 8 : 0, inr ? row / 8 : 0, sub);  // trunc toward zero
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        acc += __shfl_xor_sync(0xffffffffu, acc, 4);
        if (inr) {
          const unsigned long long cost =
              b200_mv_cost(acc, row, col, c.p0r, c.p0c, c.p1r, c.p1c, c.lambda, c.allow_hp);
          if (cost < b.cost) {
            b.cost = cost;
            b.sad = acc;
            b.row = row;
            b.col = col;
            b.idx = k;
          }
        }
      }
      // the four groups: lowest cost, ties to the lowest index (the serial scan's strict `<`)
#pragma unroll
      for (int o = 8; o <= 16; o <<= 1) {
        Best q;
        q.cost = __shfl_xor_sync(0xffffffffu, b.cost, o);
        q.sad = __shfl_xor_sync(0xffffffffu, b.sad, o);
        q.row = __shfl_xor_sync(0xffffffffu, b.row, o);
        q.col = __shfl_xor_sync(0xffffffffu, b.col, o);
        q.idx = __shfl_xor_sync(0xffffffffu, b.idx, o);
        if (q.cost < b.cost || (q.cost == b.cost && q.idx < b.idx)) b = q;
      }

      // ---- transition (warp-uniform: every lane holds the same b / cur / best)
      switch (stage) {
        case S_PRED:
          cur = b;
          radius_log2 = 1;
          stage = S_DIAMOND;
          n = 4;
          break;
        case S_DIAMOND:
          if (cur.cost <= b.cost) {
            if (radius_log2 == 0) {                                  // end of try_cands, me.rs:750-752
              if (cur.cost < best.cost) best = cur;
              if (a.nsubsets == 3 && best.sad < thresh) {            // me.rs:777-790
                stage = S_DONE;
              } else {
                subset++;
                next_subset();
              }
            } else {
              radius_log2--;
            }
          } else {
            cur = b;
          }
          break;
        case S_CROSS:
          if (b.cost < cur.cost) cur = b;
          stage = S_FIVE;
          n = 24;
          break;
        case S_FIVE:
          if (b.cost < cur.cost) cur = b;
          stage = S_UMH;
          n = 16 * (a.umh_range >> 2);
          break;
        case S_UMH:
          if (b.cost < cur.cost) cur = b;
          stage = S_HEX6;
          n = 6;
          break;
        case S_HEX6:
        case S_HEX3:
          if (b.cost != kEmptyCost) best_idx = stage == S_HEX6 ? b.idx : (center_idx + 5 + b.idx) % 6;
          if (b.cost < cur.cost) {
            cur = b;
            center_idx = best_idx;
            stage = S_HEX3;
            n = 3;
          } else {
            stage = S_SQUARE;
            n = 8;
          }
          break;
        default:  // S_SQUARE: end of hexagon_search = end of uneven_multi_hex_search
          if (b.cost < cur.cost) cur = b;
          best = cur;
          stage = S_DONE;
          break;
      }
      cr = cur.row, cc = cur.col;
    }
    if (lane == 0) {
      b200_me_result res;
      res.cost = best.cost;
      res.sad = best.sad;
      res.mv_row = (int16_t)best.row;
      res.mv_col = (int16_t)best.col;
      a.out[blk] = res;
    }
  }
}

int search_pairs(b200_ctx *ctx, size_t npairs, const b200_plane *curs, const b200_plane *refs,
                 const uint32_t *block_end, const b200_block *d_blocks, size_t nblocks,
                 const b200_cand *d_preds, const uint32_t *d_subset_offsets, int nsubsets,
                 const int16_t *d_pmv, const uint32_t *d_thresh, const b200_me_params *p, int umh_range,
                 b200_me_result *d_best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, p != nullptr && npairs >= 1 && curs && refs && block_end, "NULL params / plane pair table");
  B200_REQUIRE(ctx, nsubsets == 1 || nsubsets == 3, "nsubsets must be 1 (all_mvs) or 3 (median|b|c), got %d", nsubsets);
  B200_REQUIRE(ctx, nsubsets == 1 || d_thresh != nullptr, "the extensive ladder needs per-block thresholds");
  B200_REQUIRE(ctx, p->w >= 4 && p->h > 0 && p->w <= 128 && p->h <= 128 && (p->w & (p->w - 1)) == 0,
               "block size %dx%d out of range (<= 128, width a power of two >= 4)", p->w, p->h);
  B200_REQUIRE(ctx, umh_range >= 0 && umh_range <= 64, "umh_range %d out of range", umh_range);
  B200_REQUIRE(ctx, nblocks < (1ull << 32), "nblocks must fit 32 bits");
  for (size_t k = 0; k < npairs; k++) {
    B200_REQUIRE(ctx, curs[k].data && refs[k].data, "pair %zu: plane has no device memory", k);
    B200_REQUIRE(ctx, curs[k].bpp == refs[k].bpp && curs[k].bpp == curs[0].bpp && (curs[0].bpp == 1 || curs[0].bpp == 2),
                 "plane pairs must share bpp (1 or 2)");
    B200_REQUIRE(ctx, ((curs[k].stride * curs[0].bpp) & 3) == 0 && ((refs[k].stride * curs[0].bpp) & 3) == 0,
                 "planes need a row pitch that is a multiple of 4 bytes");
    B200_REQUIRE(ctx, block_end[k] >= (k ? block_end[k - 1] : 0), "pair %zu: block ends must be non-decreasing", k);
  }
  B200_REQUIRE(ctx, block_end[npairs - 1] == nblocks, "last pair must end at nblocks");
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && d_subset_offsets && d_best, "NULL blocks / offsets / output");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  for (size_t k0 = 0; k0 < npairs; k0 += kMaxPairs) {
    const int n = (int)std::min<size_t>(kMaxPairs, npairs - k0);
    const uint32_t b0 = k0 ? block_end[k0 - 1] : 0;
    SearchArgs a{};
    a.npairs = n;
    for (int k = 0; k < n; k++) {
      a.block_end[k] = block_end[k0 + k] - b0;
      a.cur[k] = {curs[k0 + k].data, curs[k0 + k].stride};
      a.ref[k] = {refs[k0 + k].data, refs[k0 + k].stride};
    }
    a.nblocks = a.block_end[n - 1];
    if (a.nblocks == 0) continue;
    a.blocks = d_blocks + b0;
    a.preds = d_preds;                                          // offsets are global
    a.subset_offsets = d_subset_offsets + (size_t)b0 * nsubsets;
    a.pmv = d_pmv ? d_pmv + 4 * (size_t)b0 : nullptr;
    a.thresh = d_thresh ? d_thresh + b0 : nullptr;
    a.out = d_best + b0;
    a.nsubsets = nsubsets;
    a.w = p->w;
    a.h = p->h;
    a.w_in_b = p->frame_w_in_b;
    a.h_in_b = p->frame_h_in_b;
    a.lambda = p->lambda;
    a.allow_hp = p->allow_high_precision_mv;
    a.umh_range = umh_range;
    const int wpc = 4;
    const int grid = (int)std::min<size_t>((a.nblocks + wpc - 1) / wpc, (size_t)ctx->num_sms * 64);
    if (curs[0].bpp == 1)
      me_search_kernel<uint8_t><<<grid, wpc * 32, 0, ctx->stream>>>(a);
    else
      me_search_kernel<uint16_t><<<grid, wpc * 32, 0, ctx->stream>>>(a);
    B200_LAUNCH_CHECK(ctx);
  }
  return B200_OK;
}

}  // namespace

extern "C" int b200_me_search_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                  const b200_block *d_blocks, size_t nblocks, const b200_cand *d_preds,
                                  const uint32_t *d_subset_offsets, int nsubsets, const int16_t *d_pmv,
                                  const uint32_t *d_thresh, const b200_me_params *params, int umh_range,
                                  b200_me_result *d_best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && ref && nblocks < (1ull << 32), "NULL planes / nblocks must fit 32 bits");
  const uint32_t be = (uint32_t)nblocks;
  return search_pairs(ctx, 1, cur, ref, &be, d_blocks, nblocks, d_preds, d_subset_offsets, nsubsets, d_pmv,
                      d_thresh, params, umh_range, d_best);
}

extern "C" int b200_me_search_multi_dev(b200_ctx *ctx, size_t npairs, const b200_plane *curs,
                                        const b200_plane *refs, const uint32_t *pair_block_end,
                                        const b200_block *d_blocks, size_t nblocks,
                                        const b200_cand *d_preds, const uint32_t *d_subset_offsets,
                                        int nsubsets, const int16_t *d_pmv, const uint32_t *d_thresh,
                                        const b200_me_params *params, int umh_range,
                                        b200_me_result *d_best) {
  return search_pairs(ctx, npairs, curs, refs, pair_block_end, d_blocks, nblocks, d_preds, d_subset_offsets,
                      nsubsets, d_pmv, d_thresh, params, umh_range, d_best);
}
