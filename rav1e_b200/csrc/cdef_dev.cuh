// cdef_dev.cuh — the CDEF device primitives (rav1e src/cdef.rs): direction search of one 8x8 block,
// the constrain / adjust_strength helpers, the per-block strength and direction set-up of
// cdef_filter_superblock and the per-pixel filter over an int16 tile that carries the sentinel.
// Used by the frame-level kernels (cdef.cu) and the loop-filter RDO superblock (cdef_sb_dev.cuh).
#pragma once
#include "common.cuh"

namespace {

constexpr int kVeryLarge = 0x8000;  // CDEF_VERY_LARGE, cdef.rs:30
enum { HAVE_LEFT = 1, HAVE_RIGHT = 2, HAVE_TOP = 4, HAVE_BOTTOM = 8 };

__constant__ int kDivTable[9] = {0, 840, 420, 280, 210, 168, 140, 120, 105};  // cdef.rs:54

template <typename T>
__device__ int find_dir_8x8(const T *img, int stride, int coeff_shift, unsigned *var_out) {
  int partial[8][15];
#pragma unroll
  for (int d = 0; d < 8; d++)
#pragma unroll
    for (int k = 0; k < 15; k++) partial[d][k] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
#pragma unroll
    for (int j = 0; j < 8; j++) {
      const int x = ((int)img[(long long)i * stride + j] >> coeff_shift) - 128;
      partial[0][i + j] += x;
      partial[1][i + j / 2] += x;
      partial[2][i] += x;
      partial[3][3 + i - j / 2] += x;
      partial[4][7 + i - j] += x;
      partial[5][3 - i / 2 + j] += x;
      partial[6][j] += x;
      partial[7][i / 2 + j] += x;
    }
  }
  int cost[8];
#pragma unroll
  for (int d = 0; d < 8; d++) cost[d] = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    cost[2] += partial[2][i] * partial[2][i];
    cost[6] += partial[6][i] * partial[6][i];
  }
  cost[2] *= 105;
  cost[6] *= 105;
#pragma unroll
  for (int i = 0; i < 7; i++) {
    cost[0] += (partial[0][i] * partial[0][i] + partial[0][14 - i] * partial[0][14 - i]) * kDivTable[i + 1];
    cost[4] += (partial[4][i] * partial[4][i] + partial[4][14 - i] * partial[4][14 - i]) * kDivTable[i + 1];
  }
  cost[0] += partial[0][7] * partial[0][7] * 105;
  cost[4] += partial[4][7] * partial[4][7] * 105;
#pragma unroll
  for (int i = 1; i < 8; i += 2) {
#pragma unroll
    for (int j = 0; j < 5; j++) cost[i] += partial[i][3 + j] * partial[i][3 + j];
    cost[i] *= 105;
#pragma unroll
    for (int j = 0; j < 3; j++)
      cost[i] += (partial[i][j] * partial[i][j] + partial[i][10 - j] * partial[i][10 - j]) * kDivTable[2 * j + 2];
  }
  int best = 0, best_cost = cost[0];
#pragma unroll
  for (int d = 1; d < 8; d++)
    if (cost[d] > best_cost) {  // strict: first maximum wins (cdef.rs:66-76)
      best = d;
      best_cost = cost[d];
    }
  int ortho = 0;
#pragma unroll
  for (int d = 0; d < 8; d++)
    if (d == ((best + 4) & 7)) ortho = cost[d];
  *var_out = (unsigned)((best_cost - ortho) >> 10);
  return best;
}

// cdef.rs:146-159, with `shift = max(0, damping - msb(threshold))` hoisted out of the tap loop
// (it only depends on the block's strength).  threshold == 0 gives 0 for any shift.
__device__ __forceinline__ int constrain_shift(int threshold, int damping) {
  return threshold ? max(0, damping - (31 - __clz(threshold))) : 0;
}
__device__ __forceinline__ int constrain(int diff, int threshold, int shift) {
  const int ad = abs(diff);
  const int mag = min(max(threshold - (ad >> shift), 0), ad);  // threshold == 0 -> 0
  return diff < 0 ? -mag : mag;
}

// cdef.rs:315-322
__device__ __forceinline__ int adjust_strength(int strength, int var) {
  const int i = (var >> 6) != 0 ? min(31 - __clz(var >> 6), 12) : 0;
  return var != 0 ? (strength * (4 + i) + 8) >> 4 : 0;
}

// direction offsets (dy, dx) for k = 0, 1  (cdef.rs:242-251)
__constant__ signed char kDirs[8][2][2] = {{{-1, 1}, {-2, 2}}, {{0, 1}, {-1, 2}}, {{0, 1}, {0, 2}},
                                           {{0, 1}, {1, 2}},   {{1, 1}, {2, 2}},  {{1, 0}, {2, 1}},
                                           {{1, 0}, {2, 0}},   {{1, 0}, {2, -1}}};

// One output pixel of cdef_filter_block (cdef.rs:253-296).  `load(dy, dx)` returns the input at
// (i+dy, j+dx) relative to the block, or CDEF_VERY_LARGE where the reference's padded scratch
// would hold the sentinel.
template <typename Load>
__device__ __forceinline__ int cdef_pixel(Load load, int pri_strength, int sec_strength, int dir,
                                          int damping, int coeff_shift) {
  const int x = load(0, 0);
  const int pri_shift = constrain_shift(pri_strength, damping);
  const int sec_shift = constrain_shift(sec_strength, damping);
  const int sel = (pri_strength >> coeff_shift) & 1;
  const int pri_taps[2] = {sel ? 3 : 4, sel ? 3 : 2};
  const int sec_taps[2] = {2, 1};
  int sum = 0, mx = x, mn = x;
#pragma unroll
  for (int k = 0; k < 2; k++) {
    const int d0y = kDirs[dir][k][0], d0x = kDirs[dir][k][1];
    const int d1y = kDirs[(dir + 2) & 7][k][0], d1x = kDirs[(dir + 2) & 7][k][1];
    const int d2y = kDirs[(dir + 6) & 7][k][0], d2x = kDirs[(dir + 6) & 7][k][1];
    const int p[2] = {load(d0y, d0x), load(-d0y, -d0x)};
#pragma unroll
    for (int t = 0; t < 2; t++) {
      sum += pri_taps[k] * constrain(p[t] - x, pri_strength, pri_shift);
      if (p[t] != kVeryLarge) mx = max(p[t], mx);
      mn = min(p[t], mn);
    }
    const int s[4] = {load(d1y, d1x), load(-d1y, -d1x), load(d2y, d2x), load(-d2y, -d2x)};
#pragma unroll
    for (int t = 0; t < 4; t++) {
      if (s[t] != kVeryLarge) mx = max(s[t], mx);
      mn = min(s[t], mn);
      sum += sec_taps[k] * constrain(s[t] - x, sec_strength, sec_shift);
    }
  }
  const int v = x + ((8 + sum - (sum < 0)) >> 4);
  return min(max(v, mn), mx);
}

// The filter parameters of one 8x8 block of cdef_filter_superblock (cdef.rs:406-516) over an int16
// tile of row pitch `pitch`: the 6-bit strength (pri * 4 + sec) split with sec == 3 -> 4, luma's
// adjust_strength by the block's variance, chroma's damping - 1 and 4:2:2 direction remap, the two
// constrain shifts and the tile offsets of the twelve taps.
struct CdefBlockTaps {
  int pri, sec, pri_shift, sec_shift, pt0, pt1;
  int off[6];  // primary k = 0, 1; secondary (dir + 2) k = 0, 1; (dir + 6) k = 0, 1
};

// `strength` (pri * 4 + sec) and the block's dirs[b] / vars[b] are read here, in the reference's order;
// vars only for luma.
__device__ __forceinline__ CdefBlockTaps cdef_block_taps(const uint8_t *strength_p, int plane, int xdec, int ydec,
                                                         const uint8_t *dirs, const int *vars, int b, int damping,
                                                         int coeff_shift, int pitch) {
  const int strength = *strength_p;
  const int pri = strength >> 2;
  int sec = strength & 3;
  if (sec == 3) sec = 4;  // cdef.rs:421-426
  const int d = dirs[b];
  int local_pri, local_dir, local_damping = damping + coeff_shift;
  const int local_sec = sec << coeff_shift;
  if (plane == 0) {
    local_pri = adjust_strength(pri << coeff_shift, vars[b]);
    local_dir = pri != 0 ? d : 0;
  } else {
    local_pri = pri << coeff_shift;
    local_damping -= 1;
    const int remap = (0x66654207 >> (4 * d)) & 7;  // [7,0,2,4,5,6,6,6], cdef.rs:505-509
    local_dir = pri != 0 ? (xdec != ydec ? remap : d) : 0;
  }
  CdefBlockTaps t;
  t.pri = local_pri;
  t.sec = local_sec;
  t.pri_shift = constrain_shift(local_pri, local_damping);
  t.sec_shift = constrain_shift(local_sec, local_damping);
  const int sel = (local_pri >> coeff_shift) & 1;
  t.pt0 = sel ? 3 : 4;
  t.pt1 = sel ? 3 : 2;
#pragma unroll
  for (int k = 0; k < 2; k++) {
    t.off[k] = kDirs[local_dir][k][0] * pitch + kDirs[local_dir][k][1];
    t.off[2 + k] = kDirs[(local_dir + 2) & 7][k][0] * pitch + kDirs[(local_dir + 2) & 7][k][1];
    t.off[4 + k] = kDirs[(local_dir + 6) & 7][k][0] * pitch + kDirs[(local_dir + 6) & 7][k][1];
  }
  return t;
}

// One output pixel at `c` in the int16 tile.  Sentinel handling without a compare per tap: the
// sentinel is stored as int16 0x8000 = -32768, so `max` ignores it on its own (every real pixel is
// >= 0) and `min` runs on the value reinterpreted as unsigned (0xffff8000: larger than any pixel);
// its difference to the centre is so large that constrain() returns 0 for it, exactly like the
// reference's 0x8000 does.  That holds up to a final damping of 13 at 12 bit and 14 at 8 / 10 bit
// (tests/test_oracle_cdef.py derives it); the largest the drivers pass is 6 + coeff_shift.
__device__ __forceinline__ int cdef_filter_tile_px(const short *c, const CdefBlockTaps &b) {
  const int xv = c[0];
  int sum = 0, mx = xv;
  unsigned mn = (unsigned)xv;
  auto tap = [&](int o, int thr, int shift, int w) {
    const int p0 = c[o], p1 = c[-o];
    sum += w * (constrain(p0 - xv, thr, shift) + constrain(p1 - xv, thr, shift));
    mx = max(mx, max(p0, p1));
    mn = min(mn, min((unsigned)p0, (unsigned)p1));
  };
  tap(b.off[0], b.pri, b.pri_shift, b.pt0);
  tap(b.off[1], b.pri, b.pri_shift, b.pt1);
  tap(b.off[2], b.sec, b.sec_shift, 2);
  tap(b.off[3], b.sec, b.sec_shift, 1);
  tap(b.off[4], b.sec, b.sec_shift, 2);
  tap(b.off[5], b.sec, b.sec_shift, 1);
  const int v = xv + ((8 + sum - (sum < 0)) >> 4);
  return min(max(v, (int)mn), mx);
}

}  // namespace
