// me_search_dev.cuh — the block state machine of full_pixel_me's search stages (me.rs:692-1303), one
// warp per block, shared by the candidate-list search (me_search.cu) and the lookahead's motion
// estimation (lookahead_me.cu).  See me_search.cu for the evaluation scheme.
#pragma once

#include <cuda_runtime.h>

#include "common.cuh"
#include "me_dev.cuh"

namespace {

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
// Read footprint: with rsh != 0 the aligned-down word of a row starts rsh bytes before the candidate's
// first column and the extra word ends 4 - rsh bytes past its last, so a candidate on get_mv_range's
// x_min / x_max touches up to 3 bytes outside min_pad.  Every word loaded still holds a byte of the
// candidate's row (rsh >= 1 puts the extra word's first byte at or before the row's last byte), so the
// load stays inside an aligned 4-byte word that is partly readable, and the funnel shift drops the
// outside bytes: no value outside the footprint reaches a SAD.
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

// A block of any w x h (the lookahead's edge crops, of any width): lane `sub` of a candidate's group
// sums rows sub, sub + 8, ..., pixel by pixel through L1.  No shuffles: callable per lane.
template <typename T>
__device__ __forceinline__ uint32_t crop_sad(const BlockCtx &c, int dx, int dy, int sub) {
  uint32_t acc = 0;
  for (int y = sub; y < c.h; y += 8) {
    const T *o = (const T *)(c.org + (long long)y * c.org_pitch);
    const T *r = (const T *)(c.ref0 + (long long)(c.po_y + dy + y) * c.ref_pitch) + (c.po_x + dx);
    for (int x = 0; x < c.w; x++) acc += (uint32_t)abs((int)__ldg(o + x) - (int)__ldg(r + x));
  }
  return acc;
}

// Predictor subsets as CSR lists in device memory: offs = the block's nsubsets + 1 offsets into preds.
struct ListPreds {
  const b200_cand *preds;
  const uint32_t *offs;
  __device__ __forceinline__ void span(int s, uint32_t &lo, uint32_t &hi) const {
    lo = offs[s];
    hi = offs[s + 1];
  }
  __device__ __forceinline__ void mv(uint32_t i, int &row, int &col) const {
    const b200_cand q = preds[i];
    row = q.mv_row, col = q.mv_col;
  }
};

// Predictor subsets gathered into shared memory: offs = nsubsets + 1 offsets into list.
struct SmemPreds {
  const short2 *list;  // (row, col)
  const uint32_t *offs;
  __device__ __forceinline__ void span(int s, uint32_t &lo, uint32_t &hi) const {
    lo = offs[s];
    hi = offs[s + 1];
  }
  __device__ __forceinline__ void mv(uint32_t i, int &row, int &col) const {
    const short2 q = list[i];
    row = q.x, col = q.y;
  }
};

// get_subset_predictors' steps (me.rs:386-534) shared by the lookahead (lookahead_me.cu) and the encode-time
// search (encode_me.cu).  Every lane gathers the same values.
struct Gather {
  uint32_t min_sad;
  const BlockCtx *c;
  __device__ __forceinline__ short2 proc(const b200_me_stats st) {  // process_cand, me.rs:405-412
    min_sad = min(min_sad, st.normalized_sad);
    const int col = min(max((st.mv_col / 8) * 8, c->rng.x_min), c->rng.x_max);
    const int row = min(max((st.mv_row / 8) * 8, c->rng.y_min), c->rng.y_max);
    return make_short2((short)row, (short)col);
  }
  // subset C (me.rs:477-515): LAST's stats grid P (W x H cells) around the block at frame 4x4 offset (bx, by),
  // wb x hb cells; appends left, top, right, bottom (those inside the frame) and the centre to cc
  __device__ __forceinline__ int subset_c(const b200_me_stats *P, int W, int H, int bx, int by, int wb, int hb,
                                          short2 *cc) {
    int nc = 0;
    const int hw = min(wb >> 1, W - 1 - bx), hh = min(hb >> 1, H - 1 - by);
    if (bx > 0) cc[nc++] = proc(P[(size_t)(by + hh) * W + bx - 1]);
    if (by > 0) cc[nc++] = proc(P[(size_t)(by - 1) * W + bx + hw]);
    if (bx + wb < W) cc[nc++] = proc(P[(size_t)(by + hh) * W + bx + wb]);
    if (by + hb < H) cc[nc++] = proc(P[(size_t)(by + hb) * W + bx + hw]);
    cc[nc++] = proc(P[(size_t)(by + hh) * W + bx + hw]);
    return nc;
  }
};

// full_pixel_me without the exhaustive grid for the block of `c`, called by all 32 lanes (g = lane / 8,
// sub = lane % 8); returns the same Best in every lane.  nsubsets 1: all_mvs (non-extensive); 3: median |
// subset_b | subset_c with the `sad < thresh` exits and UMH over umh_range.  Preds: span(subset, lo, hi)
// and mv(i, row, col), warp-uniform.  kCrop: the block is any w x h (crop_sad), else partial_sad's
// power-of-two rows.
template <typename T, bool kCrop, typename Preds>
__device__ __forceinline__ Best search_block(const BlockCtx &c, const Preds &P, int nsubsets, uint32_t thresh,
                                             int umh_range, int g, int sub) {
  const int n_row = (umh_range + 1) >> 1;         // cross, first line: i = 1, 3, ... <= me_range
  const int n_col = ((umh_range >> 1) + 1) >> 1;  // second line: i = 1, 3, ... <= me_range / 2
  
  Best best = best_empty();  // full_pixel_me's `best`
  Best cur = best_empty();   // the running stage's `current` / `results`
  int subset = 0, radius_log2 = 1, center_idx = 0, best_idx = 0;
  int cr = 0, cc = 0;        // centre the running pattern is laid around
  uint32_t plo = 0;          // first predictor of the running subset
  int stage = S_DONE, n = 0;

  // pick the next predictor subset (or what follows the last one)
  auto next_subset = [&]() {
    while (subset < nsubsets) {
      uint32_t lo, hi;
      P.span(subset, lo, hi);
      if (nsubsets == 3 && subset == 0 && lo == hi) {  // `if let Some(median)`, me.rs:774
        subset++;
        continue;
      }
      plo = lo;
      n = (int)(hi - lo);
      stage = S_PRED;
      return;
    }
    if (nsubsets == 3 && umh_range > 0 && best.cost != kEmptyCost) {  // me.rs:794-812
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
            P.mv(plo + k, row, col);
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
      const bool inr = k < n && !B200_MV_OUTSIDE(row, col, c.rng);
      uint32_t acc = kCrop ? crop_sad<T>(c, inr ? col / 8 : 0, inr ? row / 8 : 0, sub)  // trunc toward zero
                          : partial_sad<T>(c, inr ? col / 8 : 0, inr ? row / 8 : 0, sub);
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
            if (nsubsets == 3 && best.sad < thresh) {            // me.rs:777-790
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
        n = 16 * (umh_range >> 2);
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
  return best;
}

}  // namespace
