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
// caller here; the lookahead's own pass gathers them in lookahead_me.cu and the encode-time search
// (estimate_motion with a pmv) in encode_me.cu.  The state machine itself is in me_search_dev.cuh.
#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"
#include "me_search_dev.cuh"

#ifndef B200_SEARCH_MINBLOCKS
#define B200_SEARCH_MINBLOCKS 6  // CTAs of 4 warps per SM the search kernel is register-capped for (80 regs)
#endif

namespace {

constexpr int kMaxPairs = 32;

struct SearchArgs {
  int npairs;
  uint32_t block_end[kMaxPairs];  // pair k owns blocks [block_end[k-1], block_end[k])
  PlaneView cur[kMaxPairs], ref[kMaxPairs];
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
    const uint32_t thresh = a.nsubsets == 3 ? a.thresh[blk] : 0u;
    const ListPreds P{a.preds, a.subset_offsets + blk * a.nsubsets};
    const Best best = search_block<T, false>(c, P, a.nsubsets, thresh, a.umh_range, g, sub);
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
