// me_cand.cu — batched motion-estimation distortion over candidate lists for sm_90a.
//
// Replaces, for thousands of candidates per launch, the serial loop
//   get_fullpel_mv_rd -> compute_mv_rd -> get_sad / get_satd     (rav1e src/me.rs:1386-1461,
//                                                                  src/dist.rs:31-52, :156-221)
// incl. its first-minimum argmin: b200_me_candidates_dev / _multi_dev (the dispatcher below picks a
// kernel per launch), the packed-prediction form b200_me_subpel_candidates_dev and the full-pel
// residual b200_block_residual_dev.
//
// Kernels
//   me_cand_generic<T>      any w x h <= 128, u8/u16, SAD or SATD.  One warp per candidate.
//   me_cand_group_u8<W,H,SATD>  8-bit fast path: a CTA takes a group of consecutive blocks, stages
//                           one shared-memory window covering all their candidates with 16-byte
//                           loads, then evaluates candidates from smem (SAD: VABSDIFF4.ACC;
//                           SATD: IDP.4A Hadamard rows + butterflies).  Fused cost + argmin.
//   me_cand_warp_u8<W,H,SATD>  8-bit sparse lists: a warp per block, straight from the planes.
//   me_best_from_cost       segmented first-min argmin over a CSR candidate list.
//   me_dist_packed_kernel<T>  distortion of packed predictions (the sub-pel form).
//   block_residual_kernel<T>  residual against the reference displaced by the full-pel winner.
// The staged chunk kernel for sparse 8-bit SATD and 16-bit lists is me_chunk.cu.
#include <cuda.h>  // CUtensorMap (types only: the encoder is fetched through the runtime)
#include <cuda_runtime.h>

#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "me_cand.cuh"
#include "me_dev.cuh"

#ifndef B200_WARP_SATD_MINBLOCKS
#define B200_WARP_SATD_MINBLOCKS 1  // register cap of the warp-per-block SATD kernel (CTAs of 8 warps per SM)
#endif
#ifndef B200_SAD_THREADS
#define B200_SAD_THREADS 256  // CTA size of the SAD instantiations of the grouped kernel
#endif
#ifndef B200_SAD16_MINBLOCKS
// Resident CTAs per SM the 16x16 SAD kernel is register-capped for: 4 (64 registers, no spills).
#define B200_SAD16_MINBLOCKS 4
#endif

using namespace b200_me;

namespace {

// first k with v < ends[k] (v < ends[n-1] is the caller's invariant)
__device__ __forceinline__ int pair_lookup(const uint32_t *ends, int n, uint32_t v) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (v < ends[mid])
      hi = mid;
    else
      lo = mid + 1;
  }
  return lo;
}

// Tensor maps (TMA descriptors) of the reference planes of one launch: the grouped SAD kernel
// fetches its search window with ONE cp.async.bulk.tensor per group (box_w bytes x box_h rows,
// dense rows in shared memory, out-of-plane parts zero-filled) instead of load/store loops.
// Coordinates are pixels relative to the tensor origin (-ox, -oy) of each plane.
struct MeTma {
  int enabled;
  int box_w, box_h;
  short ox[kMaxPairs], oy[kMaxPairs];
  alignas(64) CUtensorMap map[kMaxPairs];
};

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// One thread: order the CTA's earlier generic-proxy reads of the window before the async-proxy
// write, arm the barrier with the box size and start the copy.
__device__ __forceinline__ void tma_load_window(uint32_t dst, const CUtensorMap *map, int x, int y,
                                                uint32_t bar, uint32_t bytes) {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(map), "r"(x), "r"(y), "r"(bar)
      : "memory");
}

// All threads: wait for the copy armed with parity `parity`.  Bounded: a copy that never lands
// (a descriptor / byte-count bug) traps instead of hanging the device.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  for (uint32_t spin = 0;; spin++) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) return;
    if (spin > (1u << 24)) __trap();
  }
}

// ---------------------------------------------------------------- generic candidate list
template <typename T>
__global__ void __launch_bounds__(256) me_cand_generic(MeArgs a) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t i = warp0; i < a.ncands; i += nwarps) {
    const b200_cand c = a.cands[i];
    const b200_block b = a.blocks[c.block];
    const MvRange r = b200_mv_range(a.w_in_b, a.h_in_b, b.x / MI_SIZE, b.y / MI_SIZE, a.w, a.h);
    uint32_t sad = kEmptySad;
    unsigned long long cost = kEmptyCost;
    if (!B200_MV_OUTSIDE(c.mv_row, c.mv_col, r)) {
      const int rx = b.x + c.mv_col / 8, ry = b.y + c.mv_row / 8;  // trunc toward zero
      sad = warp_block_dist<T>(px<T>(a.cur, b.x, b.y), a.cur.stride, px<T>(a.ref, rx, ry),
                               a.ref.stride, a.w, a.h, a.use_satd, lane);
      const Pmv pm = load_pmv(a.pmv, c.block);
      cost = b200_mv_cost(sad, c.mv_row, c.mv_col, pm.r0, pm.c0, pm.r1, pm.c1, a.lambda, a.allow_hp);
    }
    if (lane == 0) {
      if (a.out_sad) a.out_sad[i] = sad;
      if (a.out_cost) a.out_cost[i] = cost;
    }
  }
}
// One warp per block: first-min over its CSR range of precomputed costs.
__global__ void me_best_from_cost(const unsigned long long *cost, const uint32_t *sad,
                                  const b200_cand *cands, const uint32_t *offs, size_t nblocks,
                                  b200_me_result *out) {
  const int lane = threadIdx.x & 31;
  const size_t blk = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (blk >= nblocks) return;
  const uint32_t lo = offs[blk], hi = offs[blk + 1];
  CostIdx v{kEmptyCost, 0xffffffffu};
  for (uint32_t i = lo + lane; i < hi; i += 32) v = best_min(v, CostIdx{cost[i], i});
  v = warp_best(v);
  if (lane == 0) {
    b200_me_result r;
    r.cost = kEmptyCost;
    r.sad = kEmptySad;
    r.mv_row = 0;
    r.mv_col = 0;  // MotionSearchResult::empty(), me.rs:111-116
    if (v.cost != kEmptyCost) {
      r.cost = v.cost;
      r.sad = sad[v.idx];
      r.mv_row = cands[v.idx].mv_row;
      r.mv_col = cands[v.idx].mv_col;
    }
    out[blk] = r;
  }
}

// ---------------------------------------------------------------- 8-bit fast paths
// Stage `rows` x `row_bytes` (row_bytes multiple of 16, src and smem rows 16-byte aligned) into
// smem.  Half-warps own rows (16 lanes x 16 bytes = one 256-byte row segment per step); each
// thread walks its (row, vector) column with pointer increments only, three rows in flight.
// (A per-row cp.async.bulk / UBLKCP version needs 144 small bulk copies per window, which serialise
// in the copy engine while the whole CTA waits on the mbarrier.)
__device__ __forceinline__ void stage_window(uint32_t *smem, int pitch_words, const uint8_t *src,
                                             long long src_stride, int rows, int row_bytes) {
  const int vpr = row_bytes >> 4;
  const int nhw = blockDim.x >> 4;  // rows per sweep
  for (int v = threadIdx.x & 15; v < vpr; v += 16) {
    int y = threadIdx.x >> 4;
    const uint4 *s = (const uint4 *)(src + (long long)y * src_stride) + v;
    uint4 *d = (uint4 *)(smem + y * pitch_words) + v;
    const long long sstep = (long long)nhw * src_stride / 16;  // in uint4 units (stride % 16 == 0)
    const int dstep = nhw * pitch_words / 4;
    for (; y + 2 * nhw < rows; y += 3 * nhw) {
      const uint4 q0 = __ldg(s), q1 = __ldg(s + sstep), q2 = __ldg(s + 2 * sstep);
      d[0] = q0;
      d[dstep] = q1;
      d[2 * dstep] = q2;
      s += 3 * sstep;
      d += 3 * dstep;
    }
    for (; y < rows; y += nhw) {
      *d = __ldg(s);
      s += sstep;
      d += dstep;
    }
  }
}

// ---- SATD of one S x S chunk straight from packed bytes (dist.rs:55-149 restated for dp4a).
// The 2-D Hadamard is exact integer and separable, and only sum|coeff| is consumed, so the
// pass order (reference: vertical then horizontal) and the order of outputs inside a vector
// do not change the result.  Horizontal pass: rows of 4 packed u8 times the +-1 rows of H4 as
// signed-byte dot products (IDP.4A), org minus ref folded in by negating the coefficients.
__device__ __forceinline__ void h4_rows_dp4a(uint32_t o, uint32_t r, int (&out)[4]) {
  out[0] = dp4a_us(o, 0x01010101u, dp4a_us(r, 0xFFFFFFFFu, 0));  // + + + +
  out[1] = dp4a_us(o, 0xFF01FF01u, dp4a_us(r, 0x01FF01FFu, 0));  // + - + -
  out[2] = dp4a_us(o, 0xFFFF0101u, dp4a_us(r, 0x0101FFFFu, 0));  // + + - -
  out[3] = dp4a_us(o, 0x01FFFF01u, dp4a_us(r, 0xFF0101FFu, 0));  // + - - +
}

__device__ __forceinline__ uint32_t abs_acc(int v, uint32_t acc) { return acc + (uint32_t)abs(v); }

// wrow: window row 0 of the chunk; word0/sh locate the chunk's first pixel; orow: org chunk
// row 0 (word aligned), org pitch in words.
template <int S>
__device__ __forceinline__ uint32_t chunk_satd_u8(const uint32_t *wrow, int pitch_words, int word0,
                                                  int sh, const uint32_t *orow, int org_pitch) {
  if (S == 4) {
    int t[4][4];
#pragma unroll
    for (int y = 0; y < 4; y++) {
      const uint32_t *w = wrow + y * pitch_words + word0;
      const uint32_t r = __funnelshift_r(w[0], w[1], sh);
      h4_rows_dp4a(orow[y * org_pitch], r, t[y]);
    }
    uint32_t s = 0;
#pragma unroll
    for (int c = 0; c < 4; c++) {
      int a[4] = {t[0][c], t[1][c], t[2][c], t[3][c]};
      hadamard4(a);
      s = abs_acc(a[0], abs_acc(a[1], abs_acc(a[2], abs_acc(a[3], s))));
    }
    return s;
  } else {
    int t[8][8];
#pragma unroll
    for (int y = 0; y < 8; y++) {
      const uint32_t *w = wrow + y * pitch_words + word0;
      const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
      const uint32_t r0 = __funnelshift_r(w0, w1, sh), r1 = __funnelshift_r(w1, w2, sh);
      int A[4], B[4];
      h4_rows_dp4a(orow[y * org_pitch], r0, A);
      h4_rows_dp4a(orow[y * org_pitch + 1], r1, B);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        t[y][j] = A[j] + B[j];
        t[y][j + 4] = A[j] - B[j];
      }
    }
    uint32_t s = 0;
#pragma unroll
    for (int c = 0; c < 8; c++) {
      int a[8];
#pragma unroll
      for (int k = 0; k < 8; k++) a[k] = t[k][c];
      hadamard8(a);
#pragma unroll
      for (int k = 0; k < 8; k++) s = abs_acc(a[k], s);
    }
    return s;
  }
}

// sad = tot on lane `which`, one compare + one predicated move where they stand: written as `if (lane ==
// sidx) sad = tot` in a fully unrolled loop the compiler hoists all 32 compares out of the loop and packs
// the predicates into a bit mask
__device__ __forceinline__ void keep_if_lane(uint32_t &sad, uint32_t tot, int lane, int which) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.eq.s32 p, %1, %2;\n\t@p mov.u32 %0, %3;\n\t}"
      : "+r"(sad)
      : "r"(lane), "r"(which), "r"(tot));
}

constexpr int kCandSmemBytes = 160 * 1024;  // upper bound of the dynamic smem (window + org)
constexpr int kMaxGroup = 16;               // blocks sharing one staged window

// Fold the warp's packed keys into the per-block minima s_key[lb] (lb = -1: a lane without a
// candidate, its key is ~0).  A warp that holds one block takes its minimum by REDUX and makes one
// shared atomic; a warp that straddles blocks makes one per lane.
__device__ __forceinline__ void warp_keys_into(unsigned long long *s_key, unsigned long long key, int lb, int lane) {
  const int lb0 = __shfl_sync(0xffffffffu, lb, 0);
  if (__all_sync(0xffffffffu, lb == lb0 || key == ~0ull)) {
    const unsigned long long kmin = warp_min_key(key);
    // the owner block: any lane with a real key
    const int owner = __reduce_max_sync(0xffffffffu, key == ~0ull ? -1 : lb);
    if (lane == 0 && owner >= 0) atomicMin(&s_key[owner], kmin);
  } else if (key != ~0ull) {
    atomicMin(&s_key[lb], key);
  }
}

// 8-bit candidate-list kernel.  A CTA takes `G` consecutive blocks of the (block-grouped)
// candidate list, stages ONE window covering all their in-range candidates (neighbouring
// blocks overlap almost completely) plus their org pixels, then evaluates candidates from
// shared memory: SAD = one thread per candidate (aligned LDS.32 + funnel shift + VABSDIFF4.ACC),
// SATD = TPC threads per candidate, one Hadamard chunk each.  Cost (me.rs:1455-1460) and the
// per-block first-minimum (me.rs:898) are fused: REDUX over a packed (cost, index) key, one
// shared atomicMin per warp.  Windows that do not fit fall back to one block per pass, and a
// single block that still does not fit reads the reference plane directly.
template <int W, int H, bool SATD>
__global__ void __launch_bounds__(SATD ? 128 : B200_SAD_THREADS, (!SATD && W >= 16 && W * H <= 256) ? B200_SAD16_MINBLOCKS : 1)
    me_cand_group_u8(const __grid_constant__ MeArgs a, int G, const __grid_constant__ MeTma tm) {
  extern __shared__ __align__(128) uint32_t smem[];
  __shared__ int s_box[5];  // x0, x1, y0, y1 of the window's block origins; [4]: fetched by TMA
  __shared__ __align__(8) unsigned long long s_mbar;
  __shared__ unsigned long long s_key[kMaxGroup];
  __shared__ b200_block s_blk[kMaxGroup];
  __shared__ MvRange s_rng[kMaxGroup];
  __shared__ uint32_t s_off[kMaxGroup + 1];
  __shared__ short s_pmv[kMaxGroup][4];

  constexpr int S = (W < 8 || H < 8) ? 4 : 8;                 // dist.rs:166
  constexpr int NCH = SATD ? (W / S) * (H / S) : 1;           // chunks per candidate
  constexpr int TPC = NCH < 32 ? NCH : 32;                    // threads per candidate
  constexpr int ORGW = H * W / 4;                             // org words per block
  // COOP = cooperative SAD evaluation: a warp evaluates its 32 candidates one after the other,
  // lane = (row % RPP, word), so every LDS touches RPP rows x LPR words on 32 distinct banks
  // (pitch == LPR mod 32) instead of 32 randomly placed rows (3.4-way conflicts).
  constexpr int LPR = W / 4;
  constexpr bool COOP = !SATD && W >= 16 && W <= 64 && (LPR * H) >= 32 && (LPR * H) % 32 == 0;
  constexpr int RPP = COOP ? 32 / LPR : 1;
  constexpr int P = COOP ? H / RPP : 1;
  constexpr int nthr = SATD ? 128 : B200_SAD_THREADS;  // must match launch_cand_group
  const int lane = threadIdx.x & 31;
  uint32_t *const s_org = smem;                               // [G][ORGW]
  uint32_t *const win = smem + G * ORGW;
  const int win_bytes = a.smem_bytes - G * ORGW * 4;
  const size_t ngroups = a.ngroups;  // host-computed: no 64-bit division per thread
  const bool tma_on = COOP && tm.enabled;
  const uint32_t mbar = smem_u32(&s_mbar);
  uint32_t tma_parity = 0;
  __shared__ uint32_t s_gend[kMaxPairs];
  if (threadIdx.x < a.pr.n) s_gend[threadIdx.x] = a.pr.group_end[threadIdx.x];
  if (tma_on && threadIdx.x == 0) mbar_init(mbar, 1);
  __syncthreads();

  for (size_t grp = blockIdx.x; grp < ngroups; grp += gridDim.x) {
    int pi = 0;
    uint32_t g0 = 0, pb0 = a.pr.block_begin;
    if (a.pr.n > 1) {
      // first pair whose group_end exceeds grp: one lane per pair, a ballot instead of a search
      const uint32_t e = lane < a.pr.n ? s_gend[lane] : 0xffffffffu;
      pi = __ffs(__ballot_sync(0xffffffffu, (uint32_t)grp < e)) - 1;
      if (pi) g0 = s_gend[pi - 1], pb0 = a.pr.block_end[pi - 1];
    }
    const PlaneView cur = a.pr.cur[pi], ref = a.pr.ref[pi];
    const size_t gb0 = pb0 + (grp - g0) * G, gb1 = min(gb0 + (size_t)G, (size_t)a.pr.block_end[pi]);
    // A pass takes `chunk` blocks; it starts as the whole group and halves whenever a window does not
    // fit (e.g. a group that straddles the end of a block row), down to single blocks.
    int chunk = G;
    bool force_bbox = false;  // set when a hinted window does not fit in shared memory
    size_t b0 = gb0, b1 = gb1;
    while (b0 < gb1) {
      const int nb = (int)(b1 - b0);
      __syncthreads();  // previous pass is done with shared memory
      bool pmv_eq = true;  // this thread's block has p0 == p1
      if (threadIdx.x < nb) {
        const size_t blk = b0 + threadIdx.x;
        const b200_block b = a.blocks[blk];
        s_blk[threadIdx.x] = b;
        s_rng[threadIdx.x] =
            b200_mv_range(a.w_in_b, a.h_in_b, b.x / MI_SIZE, b.y / MI_SIZE, W, H);
        s_key[threadIdx.x] = ~0ull;
        s_off[threadIdx.x] = a.cand_offsets[blk];
        if (threadIdx.x == nb - 1) s_off[nb] = a.cand_offsets[blk + 1];
        short pv[4];
#pragma unroll
        for (int k = 0; k < 4; k++) s_pmv[threadIdx.x][k] = pv[k] = a.pmv ? a.pmv[4 * blk + k] : (short)0;
        pmv_eq = pv[0] == pv[2] && pv[1] == pv[3];
      }
      if (threadIdx.x == 32) {
        s_box[0] = INT_MAX;
        s_box[1] = INT_MIN;
        s_box[2] = INT_MAX;
        s_box[3] = INT_MIN;
      }
      // every block of the pass has p0 == p1 (always without a predictor table): the second rate of
      // b200_mv_cost is then r1 + 1 > r1, and the cooperative path skips it for the whole pass
      const bool same_pmv = __syncthreads_and(pmv_eq);
      const uint32_t lo = s_off[0], hi = s_off[nb];
      // ---- window extent.  With a search-range hint (cooperative path only) the window is the
      // union of the group's blocks grown by the hint: no pass over the candidates, and staging
      // can start right away; pass 1 checks every candidate against it, and a candidate the hint
      // does not cover is evaluated by its own lane from the reference plane.  Otherwise: bounding box of
      // the in-range candidates (reference coordinates of the block top-left).
      const bool hinted = COOP && a.hint_px > 0 && !force_bbox;
      // hinted: the first round's candidate is fetched now, under the window staging
      b200_cand pre;
      pre.block = 0;
      pre.mv_row = 0;
      pre.mv_col = 0;
      if (hinted && lo + threadIdx.x < hi) pre = a.cands[lo + threadIdx.x];
      if (hinted) {
        if (threadIdx.x < 32) {  // warp 0: a lane per block, never beyond what get_mv_range allows (plane padding)
          int x0 = INT_MAX, x1 = INT_MIN, y0 = INT_MAX, y1 = INT_MIN;
          if (lane < nb) {
            const MvRange r = s_rng[lane];
            x0 = s_blk[lane].x + max(-a.hint_px, r.x_min / 8);
            x1 = s_blk[lane].x + min(a.hint_px, r.x_max / 8);
            y0 = s_blk[lane].y + max(-a.hint_px, r.y_min / 8);
            y1 = s_blk[lane].y + min(a.hint_px, r.y_max / 8);
          }
          x0 = __reduce_min_sync(0xffffffffu, x0);
          x1 = __reduce_max_sync(0xffffffffu, x1);
          y0 = __reduce_min_sync(0xffffffffu, y0);
          y1 = __reduce_max_sync(0xffffffffu, y1);
          if (lane == 0) {
            s_box[0] = x0;
            s_box[1] = x1;
            s_box[2] = y0;
            s_box[3] = y1;
            // TMA: the fixed box must cover the extent, and the set must be dense enough to stage
            int by_tma = 0;
            if (tma_on) {
              const bool dense0 = (long long)(hi - lo) * (W * H) * 2 >= (long long)tm.box_h * tm.box_w;
              // the box starts on a 16-byte column of the tensor
              const int cx = (x0 + tm.ox[pi]) & ~15;
              const int wx = cx - tm.ox[pi];
              by_tma = dense0 && x1 - wx + W + 4 <= tm.box_w && y1 - y0 + H <= tm.box_h;
              if (by_tma) {
                tma_load_window(smem_u32(win), &tm.map[pi], cx >> 2, y0 + tm.oy[pi], mbar,
                                (uint32_t)(tm.box_w * tm.box_h));
                s_box[0] = wx;
              }
            }
            s_box[4] = by_tma;
          }
        }
      } else {
        int bx0 = INT_MAX, bx1 = INT_MIN, by0 = INT_MAX, by1 = INT_MIN;
        for (uint32_t i = lo + threadIdx.x; i < hi; i += nthr) {
          const b200_cand c = a.cands[i];
          const int lb = (int)(c.block - (uint32_t)b0);
          const MvRange r = s_rng[lb];
          if (B200_MV_OUTSIDE(c.mv_row, c.mv_col, r)) continue;
          const int rx = s_blk[lb].x + c.mv_col / 8, ry = s_blk[lb].y + c.mv_row / 8;
          bx0 = min(bx0, rx), bx1 = max(bx1, rx), by0 = min(by0, ry), by1 = max(by1, ry);
        }
        bx0 = __reduce_min_sync(0xffffffffu, bx0);
        bx1 = __reduce_max_sync(0xffffffffu, bx1);
        by0 = __reduce_min_sync(0xffffffffu, by0);
        by1 = __reduce_max_sync(0xffffffffu, by1);
        if (lane == 0 && bx0 != INT_MAX) {
          atomicMin(&s_box[0], bx0);
          atomicMax(&s_box[1], bx1);
          atomicMin(&s_box[2], by0);
          atomicMax(&s_box[3], by1);
        }
      }
      __syncthreads();
      const bool have = s_box[0] != INT_MAX;
      const bool by_tma = hinted && tma_on && s_box[4];
      // 16-byte aligned window origin whatever the alignment of pixel (0,0) (TMA: any origin)
      const int mis = (int)((uintptr_t)ref.data & 15);
      const int wx0 = by_tma ? s_box[0] : have ? (((s_box[0] + mis) & ~15) - mis) : 0;
      const int wy0 = have ? s_box[2] : 0;
      // +4 bytes: the funnel shift reads one word past the last pixel
      const int row_bytes = by_tma ? tm.box_w : have ? (int)b200_align_up((size_t)(s_box[1] + W + 4 - wx0), 16) : 0;
      const int rows = by_tma ? tm.box_h : have ? s_box[3] - wy0 + H : 0;
      int pitch_words;
      if (by_tma) {       // dense box rows; the host picked box_w / 4 == LPR * odd (conflict-free)
        pitch_words = row_bytes >> 2;
      } else if (COOP) {  // LPR * odd: conflict-free cooperative loads, rows stay 16-byte aligned
        pitch_words = ((row_bytes >> 2) + LPR - 1) & ~(LPR - 1);
        if (((pitch_words / LPR) & 1) == 0) pitch_words += LPR;
      } else {     // 16-byte aligned rows, odd multiple of 4 words
        pitch_words = (row_bytes >> 2) | 4;
      }
      const bool fits = (long long)rows * pitch_words * 4 <= (long long)win_bytes;
      if (!fits && nb > 1) {  // uniform: derived from shared state
        // a group that runs over the end of a block row: split it there (each part is a compact window again)
        int brk = nb;
        for (int k = nb - 1; k >= 1; k--)
          if (s_blk[k].y != s_blk[0].y) brk = k;
        if (brk < nb) {
          b1 = b0 + brk;
          force_bbox = false;
          continue;
        }
      }
      if (!fits && hinted) {  // a hint wider than shared memory: the exact bounding box may still fit
        force_bbox = true;
        continue;
      }
      if (!fits && nb > 1) {
        chunk = (nb + 1) >> 1;
        b1 = b0 + chunk;
        force_bbox = false;
        continue;
      }
      // Sparse candidate sets (few candidates per block, e.g. the sub-pel / mode-pruning SATD
      // lists) read fewer bytes straight from L1/L2 than staging the whole bounding window would
      // move: stage only when the candidates' own footprints exceed half the window.
      const bool dense = (long long)(hi - lo) * (W * H) * 2 >= (long long)rows * row_bytes;
      const bool staged = have && fits && dense;
      if (staged && !by_tma)
        stage_window(win, pitch_words, px<uint8_t>(ref, wx0, wy0), ref.stride, rows, row_bytes);
      // org blocks -> packed words
      for (int i = threadIdx.x; i < nb * ORGW; i += nthr) {
        const int lb = i / ORGW, wi = i - lb * ORGW;
        const int y = wi / (W / 4), k = wi - y * (W / 4);
        const uint8_t *p = px<uint8_t>(cur, s_blk[lb].x + 4 * k, s_blk[lb].y + y);
        uint32_t v;
        if (((uintptr_t)p & 3) == 0)
          v = __ldg((const uint32_t *)p);
        else
          v = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
        s_org[i] = v;
      }
      __syncthreads();

      if (COOP && staged) {
        // Pass 1 (thread per candidate): range check and addresses -> one 8-byte record per candidate:
        //   {shared address of the candidate's first footprint word, shared address of its block's org
        //    words << 3 | funnel shift}.  The funnel shift reads the low 5 bits of the second word, and an
        //   org address is a multiple of 4, so the shift needs no word of its own.  Out-of-range
        //   candidates, and in-range ones the hinted window does not cover, point at the window origin:
        //   the loop evaluates them like the others (no divergence) and the result is discarded.
        // Pass 2 (warp per 32 candidates, fully unrolled): one broadcast LDS.64 fetches the
        //   parameters, each lane loads its (row, word) of the footprint and of org with plain
        //   32-bit shared addresses, REDUX.SUM hands the SAD to the owner lane.  s_par is per warp,
        //   so a round needs no CTA barrier.
        // A candidate outside the hinted window takes its SAD from the reference plane in its own
        // lane after the loop.
        __shared__ uint2 s_par[nthr];
        const int warp = threadIdx.x >> 5;
        const int lrow = lane / LPR, lword = lane - lrow * LPR;
        const uint32_t win_s = smem_u32(win), org_s = smem_u32(s_org);
        const uint32_t lane_win = (uint32_t)(lrow * pitch_words + lword) * 4u;
        const uint32_t lane_org = (uint32_t)(lrow * (W / 4) + lword) * 4u;
        const uint32_t pstep = (uint32_t)(RPP * pitch_words) * 4u;
        for (uint32_t base = lo; base < hi; base += nthr) {
          const uint32_t i = base + threadIdx.x;
          const bool valid = i < hi;
          bool inr = false, outside = false;
          b200_cand cd;
          cd.block = 0;
          cd.mv_row = 0;
          cd.mv_col = 0;
          int lb = 0;
          uint2 par = make_uint2(win_s, org_s << 3);
          if (valid) {
            cd = (hinted && base == lo) ? pre : a.cands[i];
            lb = (int)(cd.block - (uint32_t)b0);
            const MvRange r = s_rng[lb];
            inr = !B200_MV_OUTSIDE(cd.mv_row, cd.mv_col, r);
            if (inr) {
              const b200_block b = s_blk[lb];
              const int off = b.x + cd.mv_col / 8 - wx0;
              const int roff = b.y + cd.mv_row / 8 - wy0;
              outside = off < 0 || off + W + 4 > row_bytes || roff < 0 || roff + H > rows;
              if (!outside) {
                par.x = win_s + (uint32_t)(roff * pitch_words + (off >> 2)) * 4u;
                par.y = ((org_s + (uint32_t)(lb * ORGW) * 4u) << 3) | (uint32_t)(off & 3) * 8u;
              }
            }
          }
          __syncwarp();  // the warp's previous round has read its s_par slots
          s_par[threadIdx.x] = par;
          __syncwarp();
          if (by_tma && base == lo) {  // window bytes arrive here, behind pass 1
            mbar_wait(mbar, tma_parity);
            tma_parity ^= 1;
          }
          uint32_t sad = 0;
          const uint32_t par_s = smem_u32(s_par + warp * 32);
          // When the warp's 32 candidates belong to one block (the usual case: lists are grouped
          // by block) its org words are loaded into registers once instead of per candidate, and
          // its first minimum is one 32-bit REDUX.
          // (out-of-range / padding lanes are ignored: their result is discarded anyway)
          const unsigned live = __ballot_sync(0xffffffffu, inr);
          const int lb0 = __shfl_sync(0xffffffffu, lb, live ? __ffs(live) - 1 : 0);
          const bool one_block = __all_sync(0xffffffffu, !inr || lb == lb0);
          if (!live) {
            // nothing in range in this warp's 32 slots (the tail of a group's last round): skip the evaluation
          } else if (one_block) {
            const uint32_t org0 = org_s + (uint32_t)(lb0 * ORGW) * 4u;
            uint32_t orgr[P];
#pragma unroll
            for (int p = 0; p < P; p++)
              asm volatile("ld.shared.u32 %0, [%1];"
                           : "=r"(orgr[p])
                           : "r"(org0 + lane_org + (uint32_t)(p * RPP * (W / 4)) * 4u));
#pragma unroll
            for (int sidx = 0; sidx < 32; sidx++) {
              uint32_t qa, qs;
              asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(qa), "=r"(qs) : "r"(par_s + (uint32_t)sidx * 8u));
              uint32_t wa = qa + lane_win;
              uint32_t part = 0;
#pragma unroll
              for (int p = 0; p < P; p++) {
                uint32_t w0, w1;
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w0) : "r"(wa));
                asm volatile("ld.shared.u32 %0, [%1+4];" : "=r"(w1) : "r"(wa));
                part = sad4_acc(__funnelshift_r(w0, w1, qs), orgr[p], part);
                wa += pstep;
              }
              const uint32_t tot = __reduce_add_sync(0xffffffffu, part);
              keep_if_lane(sad, tot, lane, sidx);
            }
          } else {
#pragma unroll
            for (int sidx = 0; sidx < 32; sidx++) {
              uint32_t qa, qs;
              asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(qa), "=r"(qs) : "r"(par_s + (uint32_t)sidx * 8u));
              uint32_t wa = qa + lane_win;
              const uint32_t oa = ((qs >> 3) & ~3u) + lane_org;  // drop the shift's (off & 3)
              uint32_t part = 0;
#pragma unroll
              for (int p = 0; p < P; p++) {
                uint32_t w0, w1, o;
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w0) : "r"(wa));
                asm volatile("ld.shared.u32 %0, [%1+4];" : "=r"(w1) : "r"(wa));
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(o) : "r"(oa + (uint32_t)(p * RPP * (W / 4)) * 4u));
                part = sad4_acc(__funnelshift_r(w0, w1, qs), o, part);
                wa += pstep;
              }
              const uint32_t tot = __reduce_add_sync(0xffffffffu, part);
              keep_if_lane(sad, tot, lane, sidx);
            }
          }
          if (outside) {  // in range, beyond the hinted window: the non-staged form, from the plane
            const b200_block b = s_blk[lb];
            const uint8_t *rp = px<uint8_t>(ref, b.x + cd.mv_col / 8, b.y + cd.mv_row / 8);
            const int gsh = (int)((uintptr_t)rp & 3);
            const uint32_t *gw = (const uint32_t *)(rp - gsh);
            const uint32_t *org = s_org + lb * ORGW;
            sad = 0;
            for (int y = 0; y < H; y++)
              sad = row_sad_u8<W>(gw + (long long)y * (ref.stride >> 2), 0, gsh * 8, org + y * (W / 4), sad);
          }
          unsigned long long cost = kEmptyCost;
          if (inr) {
            uint32_t rate = b200_mv_rate(cd.mv_row, cd.mv_col, s_pmv[lb][0], s_pmv[lb][1], a.allow_hp);
            if (!same_pmv) {
              const uint32_t r2 = b200_mv_rate(cd.mv_row, cd.mv_col, s_pmv[lb][2], s_pmv[lb][3], a.allow_hp) + 1;
              rate = r2 < rate ? r2 : rate;
            }
            cost = 256ull * sad + (unsigned long long)rate * a.lambda;  // b200_mv_cost
          } else {
            sad = kEmptySad;
            lb = -1;
          }
          if (valid) {
            if (a.out_sad) a.out_sad[i] = sad;
            if (a.out_cost) a.out_cost[i] = cost;
          }
          if (a.out_best) {
            if (one_block && a.key32) {
              // (cost, lane) in 32 bits orders like (cost, index) inside the warp; the winning lane
              // folds its 64-bit key into the block's minimum
              const uint32_t k = inr ? ((uint32_t)cost << 5) | (uint32_t)lane : ~0u;
              const uint32_t kmin = __reduce_min_sync(0xffffffffu, k);
              if (k == kmin && inr) atomicMin(&s_key[lb], pack_key(cost, i - s_off[lb]));
            } else {
              warp_keys_into(s_key, inr ? pack_key(cost, i - s_off[lb]) : ~0ull, lb, lane);
            }
          }
        }
      } else {
      // ---- evaluate: each slot of TPC threads takes candidates lo+slot, lo+slot+nslots, ...
      const int nslots = nthr / TPC;
      const int slot = threadIdx.x / TPC, sub = threadIdx.x - slot * TPC;
      const uint32_t ntrip = (hi - lo + nslots - 1) / nslots;
      for (uint32_t t = 0; t < ntrip; t++) {
        const uint32_t i = lo + t * nslots + slot;
        const bool valid = i < hi;
        uint32_t sad = kEmptySad;
        unsigned long long cost = kEmptyCost;
        int lb = -1;
        b200_cand c;
        c.block = 0;
        c.mv_row = 0;
        c.mv_col = 0;
        bool inr = false;
        if (valid) {
          c = a.cands[i];
          lb = (int)(c.block - (uint32_t)b0);
          const MvRange r = s_rng[lb];
          inr = !B200_MV_OUTSIDE(c.mv_row, c.mv_col, r);
        }
        uint32_t acc = 0;
        if (inr) {
          const int rx = s_blk[lb].x + c.mv_col / 8, ry = s_blk[lb].y + c.mv_row / 8;
          const uint32_t *org = s_org + lb * ORGW;
          if (staged) {
            const int off = rx - wx0;
            const uint32_t *wrow = win + (ry - wy0) * pitch_words;
            if (!SATD) {
              const int word0 = off >> 2, sh = (off & 3) * 8;
#pragma unroll 4
              for (int y = 0; y < H; y++)
                acc = row_sad_u8<W>(wrow + y * pitch_words, word0, sh, org + y * (W / 4), acc);
            } else {
              for (int ch = sub; ch < NCH; ch += TPC) {
                const int cy = (ch / (W / S)) * S, cx = (ch % (W / S)) * S;
                const int o2 = off + cx;
                acc += chunk_satd_u8<S>(wrow + cy * pitch_words, pitch_words, o2 >> 2, (o2 & 3) * 8,
                                        org + cy * (W / 4) + cx / 4, W / 4);
              }
            }
          } else {
            // not staged (sparse set, or a window too large for shared memory): the same word /
            // funnel-shift arithmetic straight from the plane through L1/L2.  Rows are word
            // addressed from a 4-byte aligned base (the row pitch is a multiple of 16 bytes).
            const uint8_t *rp = px<uint8_t>(ref, rx, ry);
            const int gsh = (int)((uintptr_t)rp & 3);
            const uint32_t *gw = (const uint32_t *)(rp - gsh);
            const int gpitch = ref.stride >> 2;
            if (!SATD) {
#pragma unroll 4
              for (int y = 0; y < H; y++)
                acc = row_sad_u8<W>(gw + (long long)y * gpitch, 0, gsh * 8, org + y * (W / 4), acc);
            } else {
              for (int ch = sub; ch < NCH; ch += TPC) {
                const int cy = (ch / (W / S)) * S, cx = (ch % (W / S)) * S;
                const int o2 = gsh + cx;
                acc += chunk_satd_u8<S>(gw + (long long)cy * gpitch, gpitch, o2 >> 2, (o2 & 3) * 8,
                                        org + cy * (W / 4) + cx / 4, W / 4);
              }
            }
          }
        }
        if (SATD) {
#pragma unroll
          for (int o = TPC >> 1; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
          constexpr int ln = S == 4 ? 2 : 3;
          acc = (acc + ((1u << ln) >> 1)) >> ln;  // dist.rs:219-220, single final rounding
        }
        unsigned long long key = ~0ull;
        if (inr && sub == 0) {
          sad = acc;
          cost = b200_mv_cost(sad, c.mv_row, c.mv_col, s_pmv[lb][0], s_pmv[lb][1], s_pmv[lb][2],
                              s_pmv[lb][3], a.lambda, a.allow_hp);
          key = pack_key(cost, i - s_off[lb]);
        }
        if (valid && sub == 0) {
          if (a.out_sad) a.out_sad[i] = sad;
          if (a.out_cost) a.out_cost[i] = cost;
        }
        if (a.out_best) warp_keys_into(s_key, key, lb, lane);
      }
      }  // cooperative / generic evaluation
      if (a.out_best) {
        __syncthreads();
        if (threadIdx.x < nb) {
          const int lb = threadIdx.x;
          const unsigned long long key = s_key[lb];
          b200_me_result res;
          res.cost = kEmptyCost;
          res.sad = kEmptySad;
          res.mv_row = 0;
          res.mv_col = 0;  // MotionSearchResult::empty(), me.rs:111-116
          if (key != ~0ull) {
            const uint32_t idx = (uint32_t)(key & ((1u << kKeyIdxBits) - 1));
            const unsigned long long cost = key >> kKeyIdxBits;
            const b200_cand c = a.cands[s_off[lb] + idx];
            const uint32_t r1 = b200_mv_rate(c.mv_row, c.mv_col, s_pmv[lb][0], s_pmv[lb][1], a.allow_hp);
            const uint32_t r2 =
                b200_mv_rate(c.mv_row, c.mv_col, s_pmv[lb][2], s_pmv[lb][3], a.allow_hp) + 1;
            const uint32_t rate = r1 < r2 ? r1 : r2;
            res.cost = cost;
            res.sad = (uint32_t)((cost - (unsigned long long)rate * a.lambda) >> 8);
            res.mv_row = c.mv_row;
            res.mv_col = c.mv_col;
          }
          a.out_best[b0 + lb] = res;
        }
      }
      // next pass
      b0 = b1;
      b1 = min(b0 + (size_t)chunk, gb1);
      force_bbox = false;
    }
  }
}

// ---------------------------------------------------------------- sparse candidate lists
// Few candidates per block (sub-pel refinement, mode pruning: ~4-16): staging a window per group
// costs more than the candidates read, and a CTA-wide pipeline has nothing to amortise.  One WARP
// per block instead: TPC lanes per candidate (SATD: one Hadamard chunk each; SAD: TPC = 1), the
// reference and org words come straight from the planes through L1 (all lanes of a warp share the
// block, so org reads are broadcasts), cost + first-min argmin by REDUX over the packed key.  No
// shared memory, no barriers.
template <int W, int H, bool SATD>
__global__ void __launch_bounds__(256, SATD ? B200_WARP_SATD_MINBLOCKS : 1) me_cand_warp_u8(const __grid_constant__ MeArgs a) {
  constexpr int S = (W < 8 || H < 8) ? 4 : 8;
  constexpr int NCH = SATD ? (W / S) * (H / S) : 1;
  constexpr int TPC = NCH < 32 ? NCH : 32;
  constexpr int SLOTS = 32 / TPC;
  const int lane = threadIdx.x & 31;
  const int slot = lane / TPC, sub = lane - slot * TPC;
  const size_t warp0 = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  const size_t blk_end = a.pr.block_end[a.pr.n - 1];
  for (size_t blk = a.pr.block_begin + warp0; blk < blk_end; blk += nwarps) {
    const int pi = a.pr.n > 1 ? pair_lookup(a.pr.block_end, a.pr.n, (uint32_t)blk) : 0;
    const PlaneView cur = a.pr.cur[pi], ref = a.pr.ref[pi];
    const int cpitch = cur.stride >> 2, rpitch = ref.stride >> 2;
    const uint32_t lo = a.cand_offsets[blk], hi = a.cand_offsets[blk + 1];
    const b200_block b = a.blocks[blk];
    const MvRange r = b200_mv_range(a.w_in_b, a.h_in_b, b.x / MI_SIZE, b.y / MI_SIZE, W, H);
    const Pmv pm = load_pmv(a.pmv, blk);
    // org block: word-addressed from a 4-byte aligned base
    const uint8_t *op = px<uint8_t>(cur, b.x, b.y);
    const int osh = (int)((uintptr_t)op & 3);
    const uint32_t *ow = (const uint32_t *)(op - osh);
    unsigned long long best = ~0ull;
    for (uint32_t base = lo; base < hi; base += SLOTS) {
      const uint32_t i = base + slot;
      const bool valid = i < hi;
      b200_cand c;
      c.block = 0;
      c.mv_row = 0;
      c.mv_col = 0;
      if (valid) c = a.cands[i];
      const bool inr = valid && !B200_MV_OUTSIDE(c.mv_row, c.mv_col, r);
      uint32_t acc = 0;
      if (inr) {
        const uint8_t *rp = px<uint8_t>(ref, b.x + c.mv_col / 8, b.y + c.mv_row / 8);
        const int gsh = (int)((uintptr_t)rp & 3);
        const uint32_t *gw = (const uint32_t *)(rp - gsh);
        if (!SATD) {
          for (int y = 0; y < H; y++) {
            uint32_t orow[W / 4];
            const uint32_t *os = ow + (long long)y * cpitch;
            uint32_t olo = __ldg(os);
#pragma unroll
            for (int k = 0; k < W / 4; k++) {
              const uint32_t ohi = __ldg(os + k + 1);
              orow[k] = __funnelshift_r(olo, ohi, osh * 8);
              olo = ohi;
            }
            acc = row_sad_u8<W>(gw + (long long)y * rpitch, 0, gsh * 8, orow, acc);
          }
        } else {
          for (int ch = sub; ch < NCH; ch += TPC) {
            const int cy = (ch / (W / S)) * S, cx = (ch % (W / S)) * S;
            uint32_t ochunk[S * (S / 4)];  // this chunk's org rows, realigned to words
#pragma unroll
            for (int y = 0; y < S; y++) {
              const int oo = osh + cx;
              const uint32_t *os = ow + (long long)(cy + y) * cpitch + (oo >> 2);
              uint32_t olo = __ldg(os);
#pragma unroll
              for (int k = 0; k < S / 4; k++) {
                const uint32_t ohi = __ldg(os + k + 1);
                ochunk[y * (S / 4) + k] = __funnelshift_r(olo, ohi, (oo & 3) * 8);
                olo = ohi;
              }
            }
            const int o2 = gsh + cx;
            acc += chunk_satd_u8<S>(gw + (long long)cy * rpitch, rpitch, o2 >> 2, (o2 & 3) * 8, ochunk, S / 4);
          }
        }
      }
      if (SATD) {
#pragma unroll
        for (int o = TPC >> 1; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        constexpr int ln = S == 4 ? 2 : 3;
        acc = (acc + ((1u << ln) >> 1)) >> ln;
      }
      uint32_t sad = kEmptySad;
      unsigned long long cost = kEmptyCost, key = ~0ull;
      if (inr && sub == 0) {
        sad = acc;
        cost = b200_mv_cost(sad, c.mv_row, c.mv_col, pm.r0, pm.c0, pm.r1, pm.c1, a.lambda, a.allow_hp);
        key = pack_key(cost, i - lo);
      }
      if (valid && sub == 0) {
        if (a.out_sad) a.out_sad[i] = sad;
        if (a.out_cost) a.out_cost[i] = cost;
      }
      best = key < best ? key : best;
    }
    if (a.out_best) {
      const unsigned long long key = warp_min_key(best);
      // key -> result as in me_cand_group_u8; written out in both kernels because a shared helper
      // costs the grouped kernels instructions and this one registers
      if (lane == 0) {
        b200_me_result res;
        res.cost = kEmptyCost;
        res.sad = kEmptySad;
        res.mv_row = 0;
        res.mv_col = 0;
        if (key != ~0ull) {
          const uint32_t idx = (uint32_t)(key & ((1u << kKeyIdxBits) - 1));
          const unsigned long long cost = key >> kKeyIdxBits;
          const b200_cand c = a.cands[lo + idx];
          const uint32_t r1 = b200_mv_rate(c.mv_row, c.mv_col, pm.r0, pm.c0, a.allow_hp);
          const uint32_t r2 = b200_mv_rate(c.mv_row, c.mv_col, pm.r1, pm.c1, a.allow_hp) + 1;
          const uint32_t rate = r1 < r2 ? r1 : r2;
          res.cost = cost;
          res.sad = (uint32_t)((cost - (unsigned long long)rate * a.lambda) >> 8);
          res.mv_row = c.mv_row;
          res.mv_col = c.mv_col;
        }
        a.out_best[blk] = res;
      }
    }
  }
}

// ---------------------------------------------------------------- host-side dispatch
// ---- tensor maps of reference planes (host).  cuTensorMapEncodeTiled comes from the driver
// through the runtime (no link-time dependency on libcuda); encoded maps are cached by geometry.
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *,
                                  const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn tma_encoder() {
  static EncodeTiledFn fn = [] {
    void *f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      f = nullptr;
    (void)cudaGetLastError();
    return (EncodeTiledFn)f;
  }();
  return fn;
}

struct TmaKey {
  const void *base;
  uint64_t w, h, stride;
  uint32_t bw, bh;
  bool operator==(const TmaKey &o) const {
    return base == o.base && w == o.w && h == o.h && stride == o.stride && bw == o.bw && bh == o.bh;
  }
};
struct TmaKeyHash {
  size_t operator()(const TmaKey &k) const {
    size_t x = (size_t)k.base;
    for (uint64_t v : {k.w, k.h, k.stride, (uint64_t)k.bw, (uint64_t)k.bh})
      x = x * 1099511628211ull ^ (size_t)v;
    return x;
  }
};

// Tensor map of an 8-bit plane's readable area (pixels [-pad, dim + pad)) with a bw x bh box.
// False when the plane cannot be described (unaligned base / pitch): the caller stages by hand.
bool tma_plane_map(const b200_plane &p, uint32_t bw, uint32_t bh, CUtensorMap *out, short *ox, short *oy) {
  EncodeTiledFn enc = tma_encoder();
  // the map counts 4-byte elements (box dimensions are limited to 256 ELEMENTS: a byte map would cap the
  // window at 256 pixels), so x coordinates are pixel columns / 4
  if (!enc || p.bpp != 1 || p.pad < 0 || p.pad > 16384 || (p.stride & 15) || bw > 1024 || bh > 256 ||
      (bw & 15))
    return false;
  // origin: the allocation's first column when known (b200_plane_alloc keeps it 256-byte
  // aligned), else pixel (-pad, -pad)
  long long lead = p.pad;
  if (p.alloc) {
    const long long off = (const uint8_t *)p.data - (const uint8_t *)p.alloc - (long long)p.pad * p.stride;
    if (off >= p.pad && off < p.stride) lead = off;
  }
  const uint8_t *base = (const uint8_t *)p.data - (long long)p.pad * p.stride - lead;
  if ((uintptr_t)base & 15) return false;
  TmaKey key{base, (uint64_t)(lead + p.width + p.pad), (uint64_t)(p.height + 2 * p.pad), (uint64_t)p.stride, bw, bh};
  static std::mutex mu;
  static std::unordered_map<TmaKey, CUtensorMap, TmaKeyHash> cache;
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it == cache.end()) {
    CUtensorMap m;
    const cuuint64_t dims[2] = {(key.w + 3) / 4, key.h};  // the row pitch is a multiple of 16: still inside the row
    const cuuint64_t strides[1] = {key.stride};
    const cuuint32_t box[2] = {bw / 4, bh};
    const cuuint32_t estr[2] = {1, 1};
    if (key.w > key.stride ||
        enc(&m, CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void *)base, dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return false;
    if (cache.size() > 8192) cache.clear();
    it = cache.emplace(key, m).first;
  }
  *out = it->second;
  *ox = (short)lead;
  *oy = (short)p.pad;
  return true;
}

// The staged chunk kernel needs 16-byte aligned reference rows (whole aligned segments are copied).
bool chunk_lists_ok(const MeArgs &a) {
  for (int k = 0; k < a.pr.n; k++)
    if ((a.pr.ref[k].stride & 15) || ((uintptr_t)a.pr.ref[k].data & 15)) return false;
  return true;
}

template <int W, int H, bool SATD>
int launch_cand_group(b200_ctx *ctx, MeArgs a, int window_hint_px, const b200_plane *refs) {
  // opt in to the largest dynamic shared memory this kernel may be launched with
  if (int st = b200_smem_opt_in(ctx, (const void *)me_cand_group_u8<W, H, SATD>, kCandSmemBytes)) return st;
  bool cur_word_pitch = true;
  for (int k = 0; k < a.pr.n; k++) cur_word_pitch = cur_word_pitch && (a.pr.cur[k].stride & 3) == 0;
  {
    // Sparse lists: when a block's candidates cover less than a quarter of the window the
    // grouped kernel would stage for it, take the warp-per-block kernel (no staging at all).
    const int hint0 = window_hint_px > 0 ? window_hint_px : 32;
    const double win_bytes = (double)(2 * hint0 + W) * (2 * hint0 + H);
    const double avg0 = a.nblocks ? (double)a.ncands / (double)a.nblocks : 0.0;
    if (avg0 * W * H * 4 < win_bytes && cur_word_pitch) {
      const int wpc = 8;
      if constexpr (SATD && W >= 8 && H >= 8 && (W / 8) * (H / 8) <= 32) {
        // 8x8-chunk SATD: footprints staged per warp with cp.async, thread per (candidate, chunk)
        const ChunkListsLaunch chunk = chunk_lists_launcher(1, W, H, true);  // null: falls through to the warp kernel
        if (chunk && chunk_lists_ok(a) && !getenv("B200_OLD_SATD")) return chunk(ctx, a);
      }
      const int grid = (int)std::min<size_t>((a.nblocks + wpc - 1) / wpc, (size_t)ctx->num_sms * 16);
      me_cand_warp_u8<W, H, SATD><<<grid, wpc * 32, 0, ctx->stream>>>(a);
      B200_LAUNCH_CHECK(ctx);
      return B200_OK;
    }
  }
  // Group size: enough candidates to fill a CTA, bounded by the org tile budget.
  const size_t avg = a.nblocks ? a.ncands / a.nblocks : 0;
  constexpr int S = (W < 8 || H < 8) ? 4 : 8;
  constexpr int NCH = SATD ? (W / S) * (H / S) : 1;
  constexpr int TPC = NCH < 32 ? NCH : 32;
  const int threads = SATD ? 128 : B200_SAD_THREADS;  // SATD holds a 64-entry chunk per thread: smaller CTAs, more of them
  int G = (int)std::min<size_t>(kMaxGroup, std::max<size_t>(1, (threads / TPC) / std::max<size_t>(avg, 1)));
  // Cooperative SAD: the per-group work (descriptors, window geometry, TMA issue, barriers) is paid per
  // group whatever its size, and a wider group re-uses more of its window: take more blocks per group
  // than one round of the CTA needs (B200_SAD_GROUP overrides, for A/B runs).
  if (!SATD && W >= 16 && W <= 64 && window_hint_px > 0) {
    static const int env_g = getenv("B200_SAD_GROUP") ? atoi(getenv("B200_SAD_GROUP")) : 0;
    int want = env_g > 0 ? std::min(env_g, kMaxGroup) : 0;
    if (!want) {
      // the widest group (<= 12 blocks) whose window + org tiles leave room for three CTAs per SM (227 KB of
      // shared memory, 1 KB reserved + ~5 KB static per CTA); on an H100 at 400 W, 16x16 / +-64 px, ms per 32-pair
      // launch: 4: 0.94, 8: 0.79, 12: 0.75-0.76, 16: 0.82 (profiles/sad_group_sweep_h100.jsonl)
      const size_t budget = (size_t)227 * 1024 / 3 - 6 * 1024;
      for (want = 12; want > 1; want--) {
        const size_t bw = b200_align_up((size_t)(2 * window_hint_px + want * W + 4 + 15), 16) + 16;
        if (bw * (size_t)(2 * window_hint_px + H) + (size_t)want * W * H <= budget) break;
      }
    }
    G = std::max(G, want);
  }
  G = std::max(1, std::min(G, 16384 / (W * H)));  // org tiles <= 16 KB
  // Shared window sized from the caller's search-range hint (+ the group's extent along x);
  // groups/blocks that do not fit degrade inside the kernel, never fail.
  const int hint = window_hint_px > 0 ? window_hint_px : 32;
  constexpr int LPR = W / 4;
  constexpr bool COOP = !SATD && W >= 16 && W <= 64 && (LPR * H) >= 32 && (LPR * H) % 32 == 0;
  // Window by TMA (cooperative SAD with a search-range hint): box = the hint window, widened to
  // a multiple of 16 bytes whose word pitch is LPR * odd (conflict-free like the padded pitch).
  static thread_local MeTma tm;
  tm.enabled = 0;
  size_t smem = 0;
  if (COOP && window_hint_px > 0 && !getenv("B200_NO_TMA")) {
    // + up to 15 bytes in front of the window to start the box on a 16-byte column; none when
    // hint and block width keep every window origin aligned (groups that are not fall back to
    // staging by hand inside the kernel)
    const int slack = (hint % 16 == 0 && W % 16 == 0) ? 0 : 15;
    uint32_t bw = (uint32_t)b200_align_up((size_t)(2 * hint + G * W + 4 + slack), 16);
    while (((bw / 4) / LPR) % 2 == 0 || (bw / 4) % LPR) bw += 16;
    const uint32_t bh = (uint32_t)(2 * hint + H);
    smem = (size_t)bw * bh + (size_t)G * W * H;
    if (smem <= (size_t)kCandSmemBytes) {
      bool ok = true;
      for (int k = 0; k < a.pr.n && ok; k++) ok = tma_plane_map(refs[k], bw, bh, &tm.map[k], &tm.ox[k], &tm.oy[k]);
      if (ok) {
        tm.enabled = 1;
        tm.box_w = (int)bw;
        tm.box_h = (int)bh;
      }
    }
  }
  if (!tm.enabled) {
    // mirror the kernel's pitch choice for the widest hand-staged window the hint allows
    const size_t words = b200_align_up((size_t)(2 * hint + G * W + 4 + 15), 16) >> 2;
    size_t pitch;
    if (COOP) {
      pitch = (words + LPR - 1) & ~(size_t)(LPR - 1);
      if (((pitch / LPR) & 1) == 0) pitch += LPR;
    } else {
      pitch = words | 4;
    }
    smem = pitch * 4 * (size_t)(2 * hint + H) + (size_t)G * W * H;
  }
  smem = std::min<size_t>(std::max<size_t>(smem, 16 * 1024), (size_t)kCandSmemBytes);
  a.smem_bytes = (int)smem;
  // 32-bit warp keys when the largest possible cost, 256 * 255 * W * H + 64 * lambda (a rate is two
  // b200_diff_to_rate terms of at most 2 * 16), leaves (cost << 5 | 31) below ~0u; the 64-bit key is
  // the only exact form above that
  a.key32 = 256ull * 255 * W * H + 64ull * a.lambda < (1ull << 27) - 1;
  // groups never straddle a plane pair
  size_t ngroups = 0;
  uint32_t b0 = a.pr.block_begin;
  for (int k = 0; k < a.pr.n; k++) {
    ngroups += (a.pr.block_end[k] - b0 + G - 1) / G;
    a.pr.group_end[k] = (uint32_t)ngroups;
    b0 = a.pr.block_end[k];
  }
  a.ngroups = ngroups;
  if (ngroups == 0) return B200_OK;
  const int grid = (int)std::min<size_t>(ngroups, (size_t)ctx->num_sms * 32);
  me_cand_group_u8<W, H, SATD><<<grid, threads, smem, ctx->stream>>>(a, G, tm);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

}  // namespace

int b200_me_check_planes(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref, const b200_me_params *p) {
  B200_REQUIRE(ctx, cur && ref && p, "NULL plane/params");
  B200_REQUIRE(ctx, cur->data && ref->data, "plane has no device memory");
  B200_REQUIRE(ctx, cur->bpp == ref->bpp && (cur->bpp == 1 || cur->bpp == 2),
               "planes must share bpp (1 or 2), got %d / %d", cur->bpp, ref->bpp);
  // dist.rs:35 / :160: w and h can be at most 128
  B200_REQUIRE(ctx, p->w > 0 && p->h > 0 && p->w <= 128 && p->h <= 128,
               "block size %dx%d out of range (<= 128)", p->w, p->h);
  // dist.rs:166-167: the transform is 4x4 iff min(w,h) == 4, else 8x8; any other minimum < 8
  // makes the reference run an 8x8 transform over a short buffer (UB) - reject it.
  B200_REQUIRE(ctx, !p->use_satd || std::min(p->w, p->h) >= 8 || std::min(p->w, p->h) == 4,
               "get_satd: min(w,h) must be 4 or >= 8, got %dx%d", p->w, p->h);
  return B200_OK;
}

namespace {

// Candidate-list evaluation over `npairs` plane pairs.  Pair k owns blocks
// [block_end[k-1], block_end[k]) and candidates [cand_end[k-1], cand_end[k]) of the concatenated
// arrays (candidates carry global block indices).
int me_candidates_pairs(b200_ctx *ctx, size_t npairs, const b200_plane *curs, const b200_plane *refs,
                        const uint32_t *block_end, const uint32_t *cand_end,
                        const b200_block *d_blocks, size_t nblocks, const b200_cand *d_cands,
                        size_t ncands, const uint32_t *d_cand_offsets, const int16_t *d_pmv,
                        const b200_me_params *p, uint32_t *d_sad, uint64_t *d_cost,
                        b200_me_result *d_best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, npairs >= 1 && curs && refs && block_end && cand_end, "NULL plane pair table");
  bool fast_planes = true;
  for (size_t k = 0; k < npairs; k++) {
    if (int st = b200_me_check_planes(ctx, &curs[k], &refs[k], p)) return st;
    B200_REQUIRE(ctx, curs[k].bpp == curs[0].bpp, "plane pairs must share bpp");
    B200_REQUIRE(ctx, block_end[k] >= (k ? block_end[k - 1] : 0) && cand_end[k] >= (k ? cand_end[k - 1] : 0),
                 "pair %zu: block/candidate ends must be non-decreasing", k);
    fast_planes = fast_planes && (refs[k].stride & 15) == 0;
  }
  B200_REQUIRE(ctx, block_end[npairs - 1] == nblocks && cand_end[npairs - 1] == ncands,
               "last pair must end at nblocks / ncands");
  B200_REQUIRE(ctx, d_best == nullptr || d_cand_offsets != nullptr,
               "d_best needs CSR d_cand_offsets (candidates grouped by block)");
  B200_REQUIRE(ctx, ncands < (1ull << 32) && nblocks < (1ull << 32), "ncands / nblocks must fit 32 bits");
  if (ncands == 0 && (nblocks == 0 || !d_best)) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && (d_cands || ncands == 0), "NULL blocks/cands");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));

  MeArgs a{};
  a.cur = {curs[0].data, curs[0].stride};
  a.ref = {refs[0].data, refs[0].stride};
  a.blocks = d_blocks;
  a.cands = d_cands;
  a.cand_offsets = d_cand_offsets;
  a.pmv = d_pmv;
  a.out_sad = d_sad;
  a.out_cost = (unsigned long long *)d_cost;
  a.out_best = d_best;
  a.ncands = ncands;
  a.nblocks = nblocks;
  a.w = p->w;
  a.h = p->h;
  a.w_in_b = p->frame_w_in_b;
  a.h_in_b = p->frame_h_in_b;
  a.lambda = p->lambda;
  a.allow_hp = p->allow_high_precision_mv;
  a.use_satd = p->use_satd;
  a.smem_bytes = 0;
  a.ngroups = 0;
  a.hint_px = p->window_hint_px;

  // Fast paths, candidates grouped by block (CSR), kMaxPairs plane pairs per launch:
  //   8-bit, block sizes up to 64x64: the grouped, warp and chunk kernels (launch_cand_group);
  //   high bit depth, block sides multiples of 8 (at most 32 8x8 chunks): the staged chunk kernel
  //   (16-bit lanes: max - min absolute differences, unpacked Hadamard).  The reference's counterpart
  //   is its AVX2 HBD SAD / SATD (asm/x86/dist/mod.rs:96-182, satd16_avx2.asm).
  // (the packed argmin key holds a candidate's index INSIDE its block in kKeyIdxBits = 24 bits: a
  // precondition on the lists - no block has 2^24 candidates - not on their total)
  int (*group)(b200_ctx *, MeArgs, int, const b200_plane *) = nullptr;
  ChunkListsLaunch chunk = nullptr;
  if (curs[0].bpp == 1 && d_cand_offsets && nblocks > 0 && fast_planes) {
#define B200_CASE(W_, H_)            \
  if (p->w == W_ && p->h == H_)      \
    group = p->use_satd ? launch_cand_group<W_, H_, true> : launch_cand_group<W_, H_, false>;
    B200_CASE(4, 4)
    B200_CASE(8, 8)
    B200_CASE(16, 16)
    B200_CASE(32, 32)
    B200_CASE(64, 64)
    B200_CASE(4, 8)
    B200_CASE(8, 4)
    B200_CASE(8, 16)
    B200_CASE(16, 8)
    B200_CASE(16, 32)
    B200_CASE(32, 16)
    B200_CASE(32, 64)
    B200_CASE(64, 32)
#undef B200_CASE
  }
  if (curs[0].bpp == 2 && d_cand_offsets && nblocks > 0 && !getenv("B200_HBD_GENERIC")) {
    bool ok = true;
    for (size_t k = 0; k < npairs; k++)
      ok = ok && (refs[k].stride * 2 % 16 == 0) && ((uintptr_t)refs[k].data & 15) == 0 && (curs[k].stride & 1) == 0;
    if (ok) chunk = chunk_lists_launcher(2, p->w, p->h, p->use_satd);
  }
  if (group || chunk) {
    for (size_t k0 = 0; k0 < npairs; k0 += kMaxPairs) {
      const int n = (int)std::min<size_t>(kMaxPairs, npairs - k0);
      a.pr.n = n;
      a.pr.block_begin = k0 ? block_end[k0 - 1] : 0;
      for (int k = 0; k < n; k++) {
        a.pr.block_end[k] = block_end[k0 + k];
        a.pr.cur[k] = {curs[k0 + k].data, curs[k0 + k].stride};
        a.pr.ref[k] = {refs[k0 + k].data, refs[k0 + k].stride};
      }
      // per-launch totals steer the kernel choice and the group size
      a.nblocks = a.pr.block_end[n - 1] - a.pr.block_begin;
      a.ncands = cand_end[k0 + n - 1] - (k0 ? cand_end[k0 - 1] : 0);
      if (a.nblocks == 0) continue;
      if (int st = group ? group(ctx, a, p->window_hint_px, refs + k0) : chunk(ctx, a)) return st;
    }
    return B200_OK;
  }

  // Generic path: per-candidate values pair by pair, then (optionally) the segmented argmin.
  unsigned long long *cost_buf = a.out_cost;
  uint32_t *sad_buf = a.out_sad;
  if (d_best && ncands) {
    size_t need = 0;
    if (!cost_buf) need += ncands * 8;
    if (!sad_buf) need += ncands * 4;
    if (need) {
      if (int st = b200_reserve_dwork(ctx, need)) return st;
      uint8_t *wsp = (uint8_t *)ctx->dwork;
      if (!cost_buf) {
        cost_buf = (unsigned long long *)wsp;
        wsp += ncands * 8;
      }
      if (!sad_buf) sad_buf = (uint32_t *)wsp;
    }
  }
  for (size_t k = 0; k < npairs; k++) {
    const size_t c0 = k ? cand_end[k - 1] : 0, c1 = cand_end[k];
    if (c1 == c0) continue;
    a.cur = {curs[k].data, curs[k].stride};
    a.ref = {refs[k].data, refs[k].stride};
    a.cands = d_cands + c0;
    a.ncands = c1 - c0;
    a.out_cost = cost_buf ? cost_buf + c0 : nullptr;
    a.out_sad = sad_buf ? sad_buf + c0 : nullptr;
    const int warps_per_cta = 8;
    const size_t want = (a.ncands + warps_per_cta - 1) / warps_per_cta;
    const int grid = (int)std::min<size_t>(want, (size_t)ctx->num_sms * 16);
    if (curs[0].bpp == 1)
      me_cand_generic<uint8_t><<<grid, warps_per_cta * 32, 0, ctx->stream>>>(a);
    else
      me_cand_generic<uint16_t><<<grid, warps_per_cta * 32, 0, ctx->stream>>>(a);
    B200_LAUNCH_CHECK(ctx);
  }
  if (d_best && nblocks) {
    const int wpc = 8;
    const int grid = (int)((nblocks + wpc - 1) / wpc);
    me_best_from_cost<<<grid, wpc * 32, 0, ctx->stream>>>(cost_buf, sad_buf, d_cands,
                                                          d_cand_offsets, nblocks, d_best);
    B200_LAUNCH_CHECK(ctx);
  }
  return B200_OK;
}

}  // namespace

extern "C" int b200_me_candidates_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                      const b200_block *d_blocks, size_t nblocks,
                                      const b200_cand *d_cands, size_t ncands,
                                      const uint32_t *d_cand_offsets, const int16_t *d_pmv,
                                      const b200_me_params *p, uint32_t *d_sad, uint64_t *d_cost,
                                      b200_me_result *d_best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && ref && p, "NULL plane/params");
  B200_REQUIRE(ctx, ncands < (1ull << 32) && nblocks < (1ull << 32), "ncands / nblocks must fit 32 bits");
  const uint32_t be = (uint32_t)nblocks, ce = (uint32_t)ncands;
  return me_candidates_pairs(ctx, 1, cur, ref, &be, &ce, d_blocks, nblocks, d_cands, ncands,
                             d_cand_offsets, d_pmv, p, d_sad, d_cost, d_best);
}

extern "C" int b200_me_candidates_multi_dev(b200_ctx *ctx, size_t npairs, const b200_plane *curs,
                                            const b200_plane *refs, const uint32_t *pair_block_end,
                                            const uint32_t *pair_cand_end, const b200_block *d_blocks,
                                            size_t nblocks, const b200_cand *d_cands, size_t ncands,
                                            const uint32_t *d_cand_offsets, const int16_t *d_pmv,
                                            const b200_me_params *p, uint32_t *d_sad,
                                            uint64_t *d_cost, b200_me_result *d_best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, p != nullptr, "NULL params");
  return me_candidates_pairs(ctx, npairs, curs, refs, pair_block_end, pair_cand_end, d_blocks, nblocks,
                             d_cands, ncands, d_cand_offsets, d_pmv, p, d_sad, d_cost, d_best);
}

// Residual of each block against the reference displaced by a full-pel motion vector:
// the `diff` step of encode_tx_block (encoder.rs:1533) for the full-pel winners of the ME
// stage; feeds forward_transform.  out[i][r][c] = cur(bx+c, by+r) - ref(bx+mvx+c, by+mvy+r).
template <typename T>
__global__ void block_residual_kernel(PlaneView cur, PlaneView ref, const b200_block *blocks,
                                      const b200_me_result *mv_src, size_t n, int w, int h,
                                      int16_t *out) {
  const size_t area = (size_t)w * h;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n * area;
       i += (size_t)gridDim.x * blockDim.x) {
    const size_t blk = i / area;
    const int rem = (int)(i - blk * area), r = rem / w, c = rem - r * w;
    const b200_block b = blocks[blk];
    int dx = 0, dy = 0;
    if (mv_src && mv_src[blk].cost != kEmptyCost) {
      dx = mv_src[blk].mv_col / 8;
      dy = mv_src[blk].mv_row / 8;
    }
    out[i] = (int16_t)((int)*px<T>(cur, b.x + c, b.y + r) - (int)*px<T>(ref, b.x + dx + c, b.y + dy + r));
  }
}

extern "C" int b200_block_residual_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                       const b200_block *d_blocks, size_t nblocks,
                                       const b200_me_result *d_mv_src, int w, int h,
                                       int16_t *d_out) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && ref && cur->data && ref->data && cur->bpp == ref->bpp, "bad planes");
  B200_REQUIRE(ctx, w > 0 && h > 0 && w <= 128 && h <= 128, "bad block size %dx%d", w, h);
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && d_out, "NULL blocks/out");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t total = nblocks * (size_t)w * h;
  const int grid = (int)std::min<size_t>((total + 255) / 256, (size_t)ctx->num_sms * 32);
  PlaneView c{cur->data, cur->stride}, r{ref->data, ref->stride};
  if (cur->bpp == 1)
    block_residual_kernel<uint8_t><<<grid, 256, 0, ctx->stream>>>(c, r, d_blocks, d_mv_src, nblocks, w, h, d_out);
  else
    block_residual_kernel<uint16_t><<<grid, 256, 0, ctx->stream>>>(c, r, d_blocks, d_mv_src, nblocks, w, h, d_out);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// Distortion of each candidate's PACKED prediction (mc output, stride = pw) against the source
// block: the compute_mv_rd half of get_subpel_mv_rd (me.rs:1434-1441).  One warp per candidate.
template <typename T>
__global__ void __launch_bounds__(256) me_dist_packed_kernel(MeArgs a, const T *pred, int pw, int ph) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t i = warp0; i < a.ncands; i += nwarps) {
    const b200_cand c = a.cands[i];
    const b200_block b = a.blocks[c.block];
    const MvRange r = b200_mv_range(a.w_in_b, a.h_in_b, b.x / MI_SIZE, b.y / MI_SIZE, a.w, a.h);
    uint32_t sad = kEmptySad;
    unsigned long long cost = kEmptyCost;
    if (!B200_MV_OUTSIDE(c.mv_row, c.mv_col, r)) {
      sad = warp_block_dist<T>(px<T>(a.cur, b.x, b.y), a.cur.stride, pred + i * (size_t)pw * ph, pw,
                               a.w, a.h, a.use_satd, lane);
      const Pmv pm = load_pmv(a.pmv, c.block);
      cost = b200_mv_cost(sad, c.mv_row, c.mv_col, pm.r0, pm.c0, pm.r1, pm.c1, a.lambda, a.allow_hp);
    }
    if (lane == 0) {
      if (a.out_sad) a.out_sad[i] = sad;
      if (a.out_cost) a.out_cost[i] = cost;
    }
  }
}

// get_subpel_mv_rd (me.rs:1411-1442) over a candidate list: predict_inter_single (8-tap put with
// `filter_mode`, the frame's default_filter) into a scratch of next_power_of_two(w) x ((h+1)&~1)
// per candidate (me.rs:1322-1324), distortion against the source block, cost, per-block
// first-minimum.  Out-of-range vectors give the empty result, exactly like the full-pel form.
extern "C" int b200_me_subpel_candidates_dev(b200_ctx *ctx, const b200_plane *cur,
                                             const b200_plane *ref, const b200_block *d_blocks,
                                             size_t nblocks, const b200_cand *d_cands, size_t ncands,
                                             const uint32_t *d_cand_offsets, const int16_t *d_pmv,
                                             const b200_me_params *p, int filter_mode,
                                             uint32_t *d_sad, uint64_t *d_cost,
                                             b200_me_result *d_best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (int st = b200_me_check_planes(ctx, cur, ref, p)) return st;
  B200_REQUIRE(ctx, d_best == nullptr || d_cand_offsets != nullptr, "d_best needs CSR d_cand_offsets");
  B200_REQUIRE(ctx, filter_mode >= 0 && filter_mode <= 3, "bad FilterMode %d", filter_mode);
  B200_REQUIRE(ctx, (cur->bpp == 1) == (p->bit_depth == 8), "bpp %d vs bit depth %d", cur->bpp, p->bit_depth);
  if (ncands == 0 && (nblocks == 0 || !d_best)) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && (d_cands || ncands == 0), "NULL blocks/cands");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  int mc_w = 1;
  while (mc_w < p->w) mc_w <<= 1;
  const int mc_h = (p->h + 1) & ~1;
  const size_t pred_bytes = b200_align_up(ncands * (size_t)mc_w * mc_h * cur->bpp, 256);
  const size_t need = pred_bytes + (d_cost ? 0 : ncands * 8) + (d_sad ? 0 : ncands * 4) + 512;
  if (int st = b200_reserve_dwork(ctx, need)) return st;
  uint8_t *wsp = (uint8_t *)ctx->dwork;
  void *d_pred = wsp;
  wsp += pred_bytes;
  unsigned long long *cost_buf = (unsigned long long *)d_cost;
  uint32_t *sad_buf = d_sad;
  if (!cost_buf) {
    cost_buf = (unsigned long long *)wsp;
    wsp += b200_align_up(ncands * 8, 256);
  }
  if (!sad_buf) sad_buf = (uint32_t *)wsp;
  if (ncands) {
    if (int st = b200_mc_cands_internal(ctx, ref, d_blocks, d_cands, ncands, mc_w, mc_h, filter_mode,
                                        p->bit_depth, d_pred))
      return st;
    MeArgs a{};
    a.cur = {cur->data, cur->stride};
    a.ref = {ref->data, ref->stride};
    a.blocks = d_blocks;
    a.cands = d_cands;
    a.pmv = d_pmv;
    a.out_sad = sad_buf;
    a.out_cost = cost_buf;
    a.ncands = ncands;
    a.nblocks = nblocks;
    a.w = p->w;
    a.h = p->h;
    a.w_in_b = p->frame_w_in_b;
    a.h_in_b = p->frame_h_in_b;
    a.lambda = p->lambda;
    a.allow_hp = p->allow_high_precision_mv;
    a.use_satd = p->use_satd;
    const int wpc = 8;
    const int grid = (int)std::min<size_t>((ncands + wpc - 1) / wpc, (size_t)ctx->num_sms * 16);
    if (cur->bpp == 1)
      me_dist_packed_kernel<uint8_t><<<grid, wpc * 32, 0, ctx->stream>>>(a, (const uint8_t *)d_pred, mc_w, mc_h);
    else
      me_dist_packed_kernel<uint16_t><<<grid, wpc * 32, 0, ctx->stream>>>(a, (const uint16_t *)d_pred, mc_w, mc_h);
    B200_LAUNCH_CHECK(ctx);
  }
  if (d_best && nblocks) {
    const int wpc = 8;
    me_best_from_cost<<<(int)((nblocks + wpc - 1) / wpc), wpc * 32, 0, ctx->stream>>>(
        cost_buf, sad_buf, d_cands, d_cand_offsets, nblocks, d_best);
    B200_LAUNCH_CHECK(ctx);
  }
  return B200_OK;
}
