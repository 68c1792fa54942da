// fwd_txfm_dev.cuh — what every kernel that runs rav1e's forward transform shares: the per-TxType 1-D
// kinds, flips and per-stage shifts (forward_shared.rs:22-164, transform/mod.rs:364-417) and the
// dispatch from a register vector to the generated 1-D networks (txfm_networks.cuh).  Included by
// fwd_txfm.cu (batched transform) and subpel_rdo.cu (sub-pel refinement fused with the transform).
#pragma once
#include "common.cuh"
#include "txfm_networks.cuh"

namespace {

enum { T1_DCT = 0, T1_ADST = 1, T1_FLIPADST = 2, T1_IDTX = 3, T1_WHT = 4 };
enum { TX_DCT_DCT = 0, TX_IDTX = 9, TX_WHT_WHT = 16 };

// transform/mod.rs:101-123 (declaration order)
const uint8_t kTxW[19] = {4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64};
const uint8_t kTxH[19] = {4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16};
// transform/mod.rs:364-402
const uint8_t kVtx[17] = {T1_DCT, T1_ADST, T1_DCT, T1_ADST, T1_FLIPADST, T1_DCT, T1_FLIPADST,
                          T1_ADST, T1_FLIPADST, T1_IDTX, T1_DCT, T1_IDTX, T1_ADST, T1_IDTX,
                          T1_FLIPADST, T1_IDTX, T1_WHT};
const uint8_t kHtx[17] = {T1_DCT, T1_DCT, T1_ADST, T1_ADST, T1_DCT, T1_FLIPADST, T1_FLIPADST,
                          T1_FLIPADST, T1_ADST, T1_IDTX, T1_IDTX, T1_DCT, T1_IDTX, T1_ADST,
                          T1_IDTX, T1_FLIPADST, T1_WHT};
// forward_shared.rs:22-64, indexed [class][(bd-8)/2][stage]
const int8_t kShift4x4[3][3] = {{3, 0, 0}, {2, 0, 1}, {0, 0, 3}};
const int8_t kShiftA[3][3] = {{4, -1, 0}, {2, 0, 1}, {0, 0, 3}};    // 8x8,16x16,4x8,...,32x8
const int8_t kShiftB[3][3] = {{4, -2, 0}, {2, 0, 0}, {0, 0, 2}};    // 32x32,16x32,32x16,16x64,64x16
const int8_t kShiftC[3][3] = {{4, -1, -2}, {2, 0, -1}, {0, 0, 1}};  // 64x64,32x64,64x32
const int8_t kShiftWht[3] = {0, 0, 2};
// class per TxSize: 0 = 4x4, 1 = A, 2 = B, 3 = C
const uint8_t kShiftClass[19] = {0, 1, 1, 2, 3, 1, 1, 1, 1, 2, 2, 3, 3, 1, 1, 1, 1, 2, 2};

int size_index(int n) { return n == 4 ? 0 : n == 8 ? 1 : n == 16 ? 2 : n == 32 ? 3 : 4; }

// mod.rs:405-417 plus the `.unwrap()`s of Txfm2DFlipCfg::fwd (forward_shared.rs:128-134)
bool valid_transform(int tx_size, int tx_type) {
  if (tx_size < 0 || tx_size >= 19 || tx_type < 0 || tx_type > 16) return false;
  const int w = kTxW[tx_size], h = kTxH[tx_size], m = w > h ? w : h;
  if (m == 64 && tx_type != TX_DCT_DCT) return false;
  if (m == 32 && tx_type != TX_DCT_DCT && tx_type != TX_IDTX) return false;
  const int t1[2] = {kVtx[tx_type], kHtx[tx_type]}, n[2] = {h, w};
  for (int k = 0; k < 2; k++) {
    const int idx = size_index(n[k]);
    if (t1[k] == T1_WHT && idx != 0) return false;
    if ((t1[k] == T1_ADST || t1[k] == T1_FLIPADST) && idx > 2) return false;
    if (t1[k] == T1_IDTX && idx > 3) return false;
  }
  return true;
}

// mod.rs:320-336
__device__ __forceinline__ int round_shift_bit(int v, int bit) {
  if (bit > 0) return (v + ((1 << bit) >> 1)) >> bit;
  return (int)((unsigned)v << (-bit));
}

template <int N>
__device__ __forceinline__ void run_1d(int type, TXV (&c)[N]) {
  if (type == T1_IDTX) return;  // fidentity, forward_shared.rs:1775
  if constexpr (N == 4) {
    if (type == T1_DCT) tx_fdct4(c);
    else if (type == T1_WHT) tx_fwht4(c);
    else tx_fdst_vii_4(c);
  } else if constexpr (N == 8) {
    if (type == T1_DCT) tx_fdct8(c);
    else tx_fdst8(c);
  } else if constexpr (N == 16) {
    if (type == T1_DCT) tx_fdct16(c);
    else tx_fdst16(c);
  } else if constexpr (N == 32) {
    tx_fdct32(c);
  } else {
    tx_fdct64(c);
  }
}

// Where the transform's output row t, coefficient k goes: the reference's transposed, 32x32-chunked order
// (forward.rs:135-159; rows 32.. after the first chunk of columns, columns 32.. after all rows of the first
// 32 columns).  dst[row(t) + col(k)]; for W, H <= 32 that is dst[k * H + t].
template <int W, int H>
struct CoefOrder {
  static constexpr int HS = H < 32 ? H : 32, WC = W < 32 ? W : 32;
  __device__ __forceinline__ static int row(int t) { return (t >= 32 ? HS * WC : 0) + (t & 31); }
  __device__ __forceinline__ static int col(int k) { return H * 32 * (k >= 32) + (k & 31) * HS; }
};

// Everything a kernel needs to know about one (tx_size, tx_type, bit depth): set up on the host.
struct TxSetup {
  int col_type, row_type;
  int ud_flip, lr_flip;
  int bit0, bit1, bit2;  // av1_round_shift_array `bit` = -shift[k]: >0 round-shift right, <0 left
};
inline TxSetup tx_setup(int tx_size, int tx_type, int bd) {
  const int8_t *sh;
  if (tx_type == TX_WHT_WHT) {
    sh = kShiftWht;
  } else {
    const int cls = kShiftClass[tx_size], b = (bd - 8) / 2;
    sh = cls == 0 ? kShift4x4[b] : cls == 1 ? kShiftA[b] : cls == 2 ? kShiftB[b] : kShiftC[b];
  }
  TxSetup t;
  t.col_type = kVtx[tx_type];
  t.row_type = kHtx[tx_type];
  t.ud_flip = t.col_type == T1_FLIPADST;  // forward_shared.rs:155-164
  t.lr_flip = t.row_type == T1_FLIPADST;
  t.bit0 = -sh[0];
  t.bit1 = -sh[1];
  t.bit2 = -sh[2];
  return t;
}

}  // namespace
