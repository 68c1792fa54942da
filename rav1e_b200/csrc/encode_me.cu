// encode_me.cu — encode-time motion search on the device: estimate_motion (me.rs:536-632) as
// inter_frame_rdo_mode_decision calls it for every block and reference (rdo.rs:1164-1196), for batches of
// (block, reference slot) items of every block size:
//   get_mv_range               me.rs:339-362
//   get_subset_predictors      me.rs:386-534, CORNER { right: true, bottom: true }, ssdec 0
//   full_pixel_me (all_mvs)    me.rs:692-764: get_best_predictor + fullpel_diamond_search
//   get_fullpel_mv_rd (SATD)   me.rs:590-607, with use_satd_subpel
//   sub_pixel_me               me.rs:857-882 -> subpel_diamond_search
//
// Every input is final before the encode pass starts: the frame's own stats grids and LAST's are filled by
// the lookahead (compute_motion_vectors), and nothing in the encode pass writes them (save_me_stats runs only
// in estimate_sb_motion).  So once a block's mv stack is known its items are independent of every other item.
//
// One warp per item.  The warp gathers the item's predictors from the grids into shared memory, runs
// me_search_dev.cuh's search_block over them as one subset, re-measures the winner with SATD from a staged
// copy of its reference block, and runs subpel_dev.cuh's sub-pel diamond with the predictions in shared
// memory.  One launch per non-empty block-size group (the prediction and transform shapes are compile-time).
#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"
#include "me_search_dev.cuh"
#include "subpel_dev.cuh"

namespace {

constexpr int kMaxSlots = 7;  // INTER_REFS_PER_FRAME
constexpr int kMaxPreds = 11;  // all_mvs: median + 5 of subset B + 5 of subset C

constexpr size_t align16(size_t v) { return (v + 15) / 16 * 16; }

// A warp's slice of shared memory: the MC tile and intermediate, one prediction, the predictor list.
template <typename T, int W, int H>
struct EncLayout {
  using ML = McLayout<T, W, H>;
  static constexpr size_t INTER = ML::TILE_BYTES;
  static constexpr size_t PRED = align16(ML::TILE_BYTES + ML::INTER_BYTES);
  static constexpr size_t LIST = align16(PRED + (size_t)W * H * sizeof(T));
  static constexpr size_t OFFS = LIST + kMaxPreds * sizeof(short2);
  static constexpr size_t BYTES = align16(OFFS + 2 * sizeof(uint32_t));
};

struct EncMeArgs {
  PlaneView src;
  PlaneView refs[kMaxSlots];
  const b200_me_stats *stats;  // nslots grids of this frame
  const b200_me_stats *prev;   // nslots grids of LAST, or null
  uint32_t prev_mask;          // bit k: slot k reads prev
  int nslots;
  size_t ncells;
  int w_in_b, h_in_b;
  int tile_w4, tile_h4;  // tile size in 4x4 units
  uint32_t lambda;
  int allow_hp, use_satd, mode, bit_depth;
  const b200_enc_me_item *items;  // this size group
  size_t nitems;
  b200_me_result *out;
};

template <typename T, int W, int H>
__global__ void __launch_bounds__(256, 1) encode_me_kernel(const __grid_constant__ EncMeArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using L = EncLayout<T, W, H>;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5, g = lane >> 3, sub = lane & 7;
  unsigned char *base = smem_raw + (size_t)wid * L::BYTES;
  T *tile = (T *)base;
  short *inter = (short *)(base + L::INTER);
  T *pred = (T *)(base + L::PRED);
  short2 *s_mv = (short2 *)(base + L::LIST);
  uint32_t *s_offs = (uint32_t *)(base + L::OFFS);
  const int xb = filter_bank(a.mode, W), yb = filter_bank(a.mode, H);
  constexpr int wb = W / MI_SIZE, hb = H / MI_SIZE;  // the block in 4x4 units

  for (size_t it = (size_t)blockIdx.x * nw + wid; it < a.nitems; it += (size_t)gridDim.x * nw) {
    const b200_enc_me_item item = a.items[it];
    const int bx = item.x4, by = item.y4, slot = item.slot;
    unsigned long long cost = kEmptyCost;
    uint32_t sad = kEmptySad;
    int row = 0, col = 0;
    if (slot < a.nslots && bx < a.w_in_b && by < a.h_in_b) {  // warp-uniform; an invalid item reads nothing
      const int x = bx * MI_SIZE, y = by * MI_SIZE;
      BlockCtx c;
      c.org_pitch = (long long)a.src.stride * (long long)sizeof(T);
      c.ref_pitch = (long long)a.refs[slot].stride * (long long)sizeof(T);
      c.org = (const uint8_t *)a.src.data + (long long)y * c.org_pitch + (long long)x * (long long)sizeof(T);
      c.ref0 = (const uint8_t *)a.refs[slot].data;
      c.po_x = x;
      c.po_y = y;
      c.w = W;
      c.h = H;
      c.rng = b200_mv_range(a.w_in_b, a.h_in_b, bx, by, W, H);
      c.p0r = item.pmv[0][0], c.p0c = item.pmv[0][1], c.p1r = item.pmv[1][0], c.p1c = item.pmv[1][1];
      c.lambda = a.lambda;
      c.allow_hp = a.allow_hp;
      {
        constexpr int nwords = W * (int)sizeof(T) / 4;
        c.log_nw = 31 - __clz(nwords);
        c.total = nwords * H;
        c.cached = c.total <= 8 * kOrgRegs;
        if (c.cached) {
#pragma unroll
          for (int j = 0; j < kOrgRegs; j++) {
            const int i = sub + 8 * j;
            c.orgw[j] = i < c.total ? load_word(c.org, c.org_pitch, i >> c.log_nw, i & (nwords - 1)) : 0u;
          }
        }
      }

      // ---- get_subset_predictors (me.rs:386-534), CORNER { right, bottom }: subset B and the centre in the
      // block's tile (tile-local offsets, the tile cropped at the frame), subset C from LAST in frame coordinates
      const int tx0 = bx / a.tile_w4 * a.tile_w4, ty0 = by / a.tile_h4 * a.tile_h4;
      const int cols = min(a.tile_w4, a.w_in_b - tx0), rows = min(a.tile_h4, a.h_in_b - ty0);
      const int tbx = bx - tx0, tby = by - ty0;
      const int chw = min(wb >> 1, cols - 1 - tbx), chh = min(hb >> 1, rows - 1 - tby);
      const b200_me_stats *S = a.stats + (size_t)slot * a.ncells;
      auto at = [&](int tx, int ty) { return S[(size_t)(ty0 + ty) * a.w_in_b + tx0 + tx]; };
      Gather G;
      G.min_sad = 0xffffffffu;
      G.c = &c;
      // all_mvs: median | subset_b | subset_c, stored by every lane (the same values) straight into the list
      int n = 0;
      s_mv[n++] = G.proc(at(tbx + chw, tby + chh));  // the centre sample is the median
      if (tbx > 0) s_mv[n++] = G.proc(at(tbx - 1, tby + chh));
      if (tby > 0) s_mv[n++] = G.proc(at(tbx + chw, tby - 1));
      if (tbx + wb < cols) s_mv[n++] = G.proc(at(tbx + wb, tby + chh));
      if (tby + hb < rows) s_mv[n++] = G.proc(at(tbx + chw, tby + hb));
      s_mv[n++] = make_short2(0, 0);
      if (a.prev && ((a.prev_mask >> slot) & 1u))
        n += G.subset_c(a.prev + (size_t)slot * a.ncells, a.w_in_b, a.h_in_b, bx, by, wb, hb, s_mv + n);
      if (lane == 0) {
        s_offs[0] = 0;
        s_offs[1] = n;
      }
      __syncwarp();

      // ---- full_pixel_me, non-extensive: get_best_predictor + fullpel_diamond_search
      const Best best = search_block<T, false>(c, SmemPreds{s_mv, s_offs}, 1, 0u, 0, g, sub);
      cost = best.cost, sad = best.sad, row = best.row, col = best.col;
      if (cost != kEmptyCost) {
        const T *org = (const T *)c.org;
        const SubpelBlock<T, W, H> sp{org, a.src.stride, (const T *)a.refs[slot].data, a.refs[slot].stride, x, y,
                                      c.rng, Pmv{c.p0r, c.p0c, c.p1r, c.p1c}, a.lambda, a.allow_hp, a.use_satd,
                                      a.bit_depth, xb, yb, tile, inter};
        if (a.use_satd) {  // best.rd = get_fullpel_mv_rd(.., use_satd, .., best.mv), me.rs:596-616
          const T *r = px<T>(a.refs[slot], x + col / 8, y + row / 8);
          __syncwarp();
          for (int i = lane; i < W * H; i += 32) pred[i] = r[(long long)(i / W) * a.refs[slot].stride + i % W];
          __syncwarp();
          sad = block_satd<T, W, H>(org, a.src.stride, pred, lane);
          cost = b200_mv_cost(sad, row, col, c.p0r, c.p0c, c.p1r, c.p1c, a.lambda, a.allow_hp);
        }
        sp.diamond(cost, sad, row, col, pred, lane);  // sub_pixel_me, me.rs:857-882
      }
    }
    if (lane == 0) {
      b200_me_result res;
      res.cost = cost;
      res.sad = sad;
      res.mv_row = (int16_t)row;
      res.mv_col = (int16_t)col;
      a.out[it] = res;
    }
    __syncwarp();  // the shared list and buffers are rewritten by this warp's next item
  }
}

template <typename T, int W, int H>
int launch_group(b200_ctx *ctx, const EncMeArgs &a) {
  constexpr size_t per_warp = EncLayout<T, W, H>::BYTES;
  const int wpc = (int)std::min<size_t>(8, std::max<size_t>(1, (160 * 1024) / per_warp));
  if (int st = b200_smem_opt_in(ctx, (const void *)encode_me_kernel<T, W, H>, (int)(per_warp * wpc))) return st;
  const int grid = (int)std::min<size_t>((a.nitems + wpc - 1) / wpc, (size_t)ctx->num_sms * 16);
  encode_me_kernel<T, W, H><<<grid, wpc * 32, per_warp * wpc, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

template <typename T>
int launch_size(b200_ctx *ctx, int s, const EncMeArgs &a) {
  switch (s) {  // TxSize order, the sizes b200_subpel_search_dev takes
    case 0: return launch_group<T, 4, 4>(ctx, a);
    case 1: return launch_group<T, 8, 8>(ctx, a);
    case 2: return launch_group<T, 16, 16>(ctx, a);
    case 3: return launch_group<T, 32, 32>(ctx, a);
    case 4: return launch_group<T, 64, 64>(ctx, a);
    case 5: return launch_group<T, 4, 8>(ctx, a);
    case 6: return launch_group<T, 8, 4>(ctx, a);
    case 7: return launch_group<T, 8, 16>(ctx, a);
    case 8: return launch_group<T, 16, 8>(ctx, a);
    case 9: return launch_group<T, 16, 32>(ctx, a);
    case 10: return launch_group<T, 32, 16>(ctx, a);
    case 11: return launch_group<T, 32, 64>(ctx, a);
    case 12: return launch_group<T, 64, 32>(ctx, a);
    case 13: return launch_group<T, 4, 16>(ctx, a);
    case 14: return launch_group<T, 16, 4>(ctx, a);
    case 15: return launch_group<T, 8, 32>(ctx, a);
    case 16: return launch_group<T, 32, 8>(ctx, a);
    case 17: return launch_group<T, 16, 64>(ctx, a);
    case 18: return launch_group<T, 64, 16>(ctx, a);
  }
  return b200_fail(ctx, B200_ERR_ARG, "unreachable block size");
}

}  // namespace

extern "C" int b200_estimate_motion_dev(b200_ctx *ctx, const b200_plane *src, size_t nslots, const b200_plane *refs,
                                        const b200_me_stats *d_stats, const b200_me_stats *d_prev,
                                        const uint8_t *has_prev, const b200_enc_me_params *p,
                                        const uint32_t size_end[19], const b200_enc_me_item *d_items, size_t nitems,
                                        b200_me_result *d_out) {
  static const int kW[19] = {4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64};
  static const int kH[19] = {4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16};
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, src && refs && p && size_end && d_stats, "NULL source / references / params / size_end / stats");
  B200_REQUIRE(ctx, nslots >= 1 && nslots <= (size_t)kMaxSlots, "nslots %zu out of 1..7", nslots);
  B200_REQUIRE(ctx, (d_prev == nullptr) == (has_prev == nullptr), "d_prev and the host has_prev flags go together");
  B200_REQUIRE(ctx, p->tile_w_sb >= 1 && p->tile_h_sb >= 1, "tile size %dx%d SBs must be >= 1", p->tile_w_sb,
               p->tile_h_sb);
  B200_REQUIRE(ctx, p->filter_mode >= 0 && p->filter_mode <= 3, "bad FilterMode %d", p->filter_mode);
  const int bpp = src->bpp, width = src->width, height = src->height;
  B200_REQUIRE(ctx, bpp == 1 || bpp == 2, "bpp must be 1 or 2");
  B200_REQUIRE(ctx, bpp == 1 ? p->bit_depth == 8 : (p->bit_depth == 10 || p->bit_depth == 12),
               "bit_depth %d does not fit bpp %d", p->bit_depth, bpp);
  B200_REQUIRE(ctx, width >= 1 && height >= 1 && width <= 8192 && height <= 8192, "frame %dx%d out of range", width,
               height);
  for (size_t k = 0; k <= nslots; k++) {
    const b200_plane *pl = k ? refs + (k - 1) : src;
    B200_REQUIRE(ctx, pl->data != nullptr, "plane %zu has no device memory", k);
    B200_REQUIRE(ctx, pl->bpp == bpp, "planes must share bpp");
    B200_REQUIRE(ctx, pl->width == width && pl->height == height, "plane %zu is %dx%d, the source %dx%d", k,
                 pl->width, pl->height, width, height);
    B200_REQUIRE(ctx, ((pl->stride * bpp) & 3) == 0, "planes need a row pitch that is a multiple of 4 bytes");
  }
  uint32_t prev_end = 0;
  for (int s = 0; s < 19; s++) {
    B200_REQUIRE(ctx, size_end[s] >= prev_end, "size_end must be non-decreasing (size %d)", s);
    prev_end = size_end[s];
  }
  B200_REQUIRE(ctx, (size_t)size_end[18] == nitems, "size_end[18] = %u, want nitems = %zu", size_end[18], nitems);
  B200_REQUIRE(ctx, nitems == 0 || (d_items && d_out), "NULL items / output");
  // padding (see the header): the mv range of the largest non-empty group plus the 8-tap footprint
  const int W8 = (width + 7) & ~7, H8 = (height + 7) & ~7;
  int need = 0;
  for (int s = 0; s < 19; s++) {
    if (size_end[s] == (s ? size_end[s - 1] : 0)) continue;
    need = std::max({need, kW[s] + 19, W8 - width + kW[s] + 20, kH[s] + 19, H8 - height + kH[s] + 20});
  }
  for (size_t k = 0; k <= nslots; k++) {
    const b200_plane *pl = k ? refs + (k - 1) : src;
    B200_REQUIRE(ctx, pl->pad >= need, "plane %zu needs pad >= %d (has %d)", k, need, pl->pad);
  }
  if (nitems == 0) return B200_OK;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));

  EncMeArgs a{};
  a.src = {src->data, src->stride};
  for (size_t k = 0; k < nslots; k++) a.refs[k] = {refs[k].data, refs[k].stride};
  a.stats = d_stats;
  a.prev = d_prev;
  for (size_t k = 0; d_prev && k < nslots; k++) a.prev_mask |= has_prev[k] ? 1u << k : 0u;
  a.nslots = (int)nslots;
  a.w_in_b = W8 >> 2, a.h_in_b = H8 >> 2;
  a.ncells = (size_t)a.w_in_b * a.h_in_b;
  a.tile_w4 = p->tile_w_sb * 16, a.tile_h4 = p->tile_h_sb * 16;
  // me.rs:549-552: (fi.me_lambda * 256.0 * 0.5) as u32, saturating
  const double l = p->me_lambda * 256.0 * 0.5;
  a.lambda = !(l > 0.0) ? 0u : l >= 4294967295.0 ? 0xffffffffu : (uint32_t)l;
  a.allow_hp = p->allow_high_precision_mv != 0;
  a.use_satd = p->use_satd_subpel != 0;
  a.mode = p->filter_mode;
  a.bit_depth = p->bit_depth;
  for (int s = 0; s < 19; s++) {
    const uint32_t lo = s ? size_end[s - 1] : 0, hi = size_end[s];
    if (hi == lo) continue;
    a.items = d_items + lo;
    a.nitems = hi - lo;
    a.out = d_out + lo;
    const int st = bpp == 1 ? launch_size<uint8_t>(ctx, s, a) : launch_size<uint16_t>(ctx, s, a);
    if (st != B200_OK) return st;
  }
  return B200_OK;
}
