// lookahead_me.cu — the lookahead's motion vectors on the device: estimate_tile_motion (me.rs:153-337)
// with its predictor gathering (get_subset_predictors, :386-534), for whole frames.
//
// Three levels per (frame, reference slot) pair: 64 px blocks on the quarter resolution plane (extensive
// search, then the optional exhaustive grid), 32 px on the half and 16 px on the full resolution plane.
// Each later level starts every superblock by re-searching the previous level's blocks of that superblock
// (refine_subsampled_sb_motion, :284-322); the reference interleaves refinement and estimation SB by SB.
//
// Estimation reads the left and top neighbours' results of the same level, so it runs as a wavefront:
// one launch per tile-local anti-diagonal d = bx + by of blocks (all tiles and pairs in each launch; no
// block waits on another inside a launch).  The right, bottom and centre predictors read the previous
// level, and in the reference's serial order that value is refined inside the block's own superblock
// (its refinement ran first) but not yet refined in the next superblock or superblock row.  So each
// level first runs ONE refinement launch over every block, which writes the refined grid and keeps the
// unrefined one, and the wavefront picks between them by superblock membership.  The search itself is
// me_search_dev.cuh's state machine, one warp per block, with crop-size SADs.
//
// Launches per call: 2 + sum over the levels of (tile_bx + tile_by - 1), tile_bx / tile_by = the blocks
// of the largest (first) tile at that level's block size; 328 for a 1080p frame in one tile.
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "me_search_dev.cuh"

namespace {

struct LaPair {
  PlaneView cur[3], ref[3];  // full, half, quarter resolution
  int has_prev;
};

struct LaArgs {
  const LaPair *pairs;
  int npairs;
  b200_me_stats *stats;        // npairs x ncells: the output, current level
  b200_me_stats *refined;      // the previous level after refinement
  b200_me_stats *unrefined;    // the previous level as it ended
  const b200_me_stats *prev;   // LAST's final stats per pair, or null
  size_t ncells;
  int w_in_b, h_in_b, W8, H8;  // 4x4 grid; 8-aligned frame (px)
  int tile_w, tile_h;          // full tile size (px)
  int log2, ssdec;             // block = 4 << log2 px; plane = full >> ssdec
  uint32_t lambda;
  int allow_hp, bit_depth, full_search, range_scale;
  int nbx, nby;                // blocks of the frame at this block size
  int tbw, tbh;                // blocks per full tile
  int ntr;                     // tile rows
  int diag;
};

__device__ __forceinline__ int crop(int mv_size, int rest, int ssdec) {  // me.rs:250-251
  return min(mv_size, rest + (1 << ssdec) - 1) >> ssdec;
}

// geometry of a block at level resolution: org, ref, po, range >> ssdec (estimate_motion, me.rs:542-573)
template <typename T>
__device__ __forceinline__ void block_ctx(const LaArgs &a, const LaPair &pp, int bx, int by, int w, int h,
                                          BlockCtx &c) {
  const int s = a.ssdec;
  c.org_pitch = (long long)pp.cur[s].stride * (long long)sizeof(T);
  c.ref_pitch = (long long)pp.ref[s].stride * (long long)sizeof(T);
  c.po_x = (bx * MI_SIZE) >> s;
  c.po_y = (by * MI_SIZE) >> s;
  c.org = (const uint8_t *)pp.cur[s].data + (long long)c.po_y * c.org_pitch + (long long)c.po_x * (long long)sizeof(T);
  c.ref0 = (const uint8_t *)pp.ref[s].data;
  c.w = w;
  c.h = h;
  MvRange r = b200_mv_range(a.w_in_b, a.h_in_b, bx, by, w << s, h << s);
  c.rng.x_min = r.x_min >> s, c.rng.x_max = r.x_max >> s, c.rng.y_min = r.y_min >> s, c.rng.y_max = r.y_max >> s;
  c.p0r = c.p0c = c.p1r = c.p1c = 0;
  c.lambda = a.lambda;
  c.allow_hp = a.allow_hp;
  c.log_nw = 0;
  c.total = 0;
  c.cached = false;
}

// the first minimum of the four candidate groups (the serial scan's strict `<`)
__device__ __forceinline__ Best group_min(Best b) {
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
  return b;
}

// full_search (me.rs:1464-1509): rows y_lo.., columns x_lo.., `step` apart, first minimum in scan order,
// pmv zero.  An empty window leaves the result empty.
template <typename T>
__device__ Best full_search_warp(const BlockCtx &c, int x_lo, int x_hi, int y_lo, int y_hi, int step, int g,
                                 int sub) {
  const int nx = x_hi >= x_lo ? (x_hi - x_lo) / step + 1 : 0;
  const int ny = y_hi >= y_lo ? (y_hi - y_lo) / step + 1 : 0;
  const int n = nx * ny;
  Best b = best_empty();
  for (int k0 = 0; k0 < n; k0 += 4) {
    const int k = k0 + g;
    const bool on = k < n;
    const int y = on ? y_lo + (k / nx) * step : c.po_y, x = on ? x_lo + (k % nx) * step : c.po_x;
    uint32_t acc = on ? crop_sad<T>(c, x - c.po_x, y - c.po_y, sub) : 0u;
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if (on) {
      const int row = s16(8 * s16(y - c.po_y)), col = s16(8 * s16(x - c.po_x));
      const unsigned long long cost = b200_mv_cost(acc, row, col, 0, 0, 0, 0, c.lambda, c.allow_hp);
      if (cost < b.cost) {
        b.cost = cost;
        b.sad = acc;
        b.row = row;
        b.col = col;
        b.idx = k;
      }
    }
  }
  return group_min(b);
}

// save_me_stats (me.rs:324-337): {mv << ssdec, (sad << 14) / (w * h)} into every cell of the block
// (size 4 << log2 px) inside the frame; a block never crosses a tile edge.  All lanes share the stores.
__device__ __forceinline__ void save(b200_me_stats *grid, const LaArgs &a, int log2, int bx, int by, const Best &b,
                                     int w, int h, int lane) {
  b200_me_stats st;
  st.mv_row = (int16_t)(b.row * (1 << a.ssdec));
  st.mv_col = (int16_t)(b.col * (1 << a.ssdec));
  st.normalized_sad = (uint32_t)(((unsigned long long)b.sad << 14) / (unsigned long long)(w * h));
  const int n = 1 << log2, xe = min(bx + n, a.w_in_b), ye = min(by + n, a.h_in_b);
  for (int i = lane; i < (xe - bx) * (ye - by); i += 32) grid[(size_t)(by + i / (xe - bx)) * a.w_in_b + bx + i % (xe - bx)] = st;
}

// refine_subsampled_motion_estimate (me.rs:633-690) for every block of the previous level (log2 + 1):
// a 4x4 full search around the stored vector >> ssdec, into `refined`; `unrefined` keeps the old cells.
template <typename T>
__global__ void __launch_bounds__(128) refine_kernel(const __grid_constant__ LaArgs a) {
  const int lane = threadIdx.x & 31, g = lane >> 3, sub = lane & 7;
  const int log2 = a.log2 + 1, mv_size = MI_SIZE << log2;
  const int nbx = (a.W8 + mv_size - 1) / mv_size, nby = (a.H8 + mv_size - 1) / mv_size;
  const size_t nitems = (size_t)a.npairs * nbx * nby;
  for (size_t it = (size_t)blockIdx.x * 4 + (threadIdx.x >> 5); it < nitems; it += (size_t)gridDim.x * 4) {
    const int pi = (int)(it / ((size_t)nbx * nby));
    const int rem = (int)(it % ((size_t)nbx * nby));
    const int X = (rem % nbx) * mv_size, Y = (rem / nbx) * mv_size;
    const int bx = X >> 2, by = Y >> 2;
    const int w = crop(mv_size, a.W8 - X, a.ssdec), h = crop(mv_size, a.H8 - Y, a.ssdec);
    const LaPair &pp = a.pairs[pi];
    b200_me_stats *stats = a.stats + pi * a.ncells;
    BlockCtx c;
    block_ctx<T>(a, pp, bx, by, w, h, c);
    const b200_me_stats st = stats[(size_t)by * a.w_in_b + bx];
    const int mc = s16(st.mv_col >> a.ssdec) / 8, mr = s16(st.mv_row >> a.ssdec) / 8;
    const Best b = full_search_warp<T>(c, c.po_x + max(mc - 1, c.rng.x_min / 8), c.po_x + min(mc + 2, c.rng.x_max / 8),
                                       c.po_y + max(mr - 1, c.rng.y_min / 8), c.po_y + min(mr + 2, c.rng.y_max / 8), 1,
                                       g, sub);
    const int n = 1 << log2, xe = min(bx + n, a.w_in_b), ye = min(by + n, a.h_in_b);
    b200_me_stats *un = a.unrefined + pi * a.ncells;
    for (int i = lane; i < (xe - bx) * (ye - by); i += 32) {
      const size_t o = (size_t)(by + i / (xe - bx)) * a.w_in_b + bx + i % (xe - bx);
      un[o] = stats[o];
    }
    save(a.refined + pi * a.ncells, a, log2, bx, by, b, w, h, lane);
  }
}

// One anti-diagonal of one level: get_subset_predictors + full_pixel_me (+ the exhaustive grid) per block.
template <typename T>
__global__ void __launch_bounds__(128) diag_kernel(const __grid_constant__ LaArgs a) {
  __shared__ short2 s_mv[4][12];
  __shared__ uint32_t s_offs[4][4];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 3, sub = lane & 7;
  const int mv_size = MI_SIZE << a.log2, s = a.ssdec;
  const bool init = a.log2 == 4;
  const size_t nitems = (size_t)a.npairs * a.nbx * a.ntr;
  for (size_t it = (size_t)blockIdx.x * 4 + wid; it < nitems; it += (size_t)gridDim.x * 4) {
    const int pi = (int)(it / ((size_t)a.nbx * a.ntr));
    const int rem = (int)(it % ((size_t)a.nbx * a.ntr));
    const int I = rem % a.nbx, tr = rem / a.nbx, tc = I / a.tbw;
    const int i = I - tc * a.tbw, j = a.diag - i;
    if (j < 0 || j >= min(a.tbh, a.nby - tr * a.tbh)) continue;  // warp-uniform
    const int X = I * mv_size, Y = (tr * a.tbh + j) * mv_size;
    const int bx = X >> 2, by = Y >> 2;
    const int tx0 = tc * (a.tile_w >> 2), ty0 = tr * (a.tile_h >> 2);
    const int cols = (min(a.tile_w, a.W8 - tc * a.tile_w)) >> 2, rows = (min(a.tile_h, a.H8 - tr * a.tile_h)) >> 2;
    const int tbx = bx - tx0, tby = by - ty0;  // tile-local
    const int w = crop(mv_size, a.W8 - X, s), h = crop(mv_size, a.H8 - Y, s);
    const LaPair &pp = a.pairs[pi];
    const size_t base = (size_t)pi * a.ncells;
    BlockCtx c;
    block_ctx<T>(a, pp, bx, by, w, h, c);

    // ---- get_subset_predictors (me.rs:386-534), in tile coordinates
    const int wb = ((w << s) + MI_SIZE - 1) >> 2, hb = ((h << s) + MI_SIZE - 1) >> 2;
    const int chw = min(wb >> 1, cols - 1 - tbx), chh = min(hb >> 1, rows - 1 - tby);
    // the current level (left, top) / the previous one, refined inside this superblock (right, bottom, centre)
    auto cur_at = [&](int x, int y) { return a.stats[base + (size_t)(ty0 + y) * a.w_in_b + tx0 + x]; };
    auto prev_level_at = [&](int x, int y) {
      const int gx = tx0 + x, gy = ty0 + y;
      const bool same_sb = (gx >> 4) == (bx >> 4) && (gy >> 4) == (by >> 4);
      return (same_sb ? a.refined : a.unrefined)[base + (size_t)gy * a.w_in_b + gx];
    };
    Gather G;
    G.min_sad = 0xffffffffu;
    G.c = &c;
    short2 b[5], cc[5], median = make_short2(0, 0);
    int nb = 0, nc = 0;
    bool has_median = false;
    if (tbx > 0) b[nb++] = G.proc(cur_at(tbx - 1, tby + chh));
    if (tby > 0) b[nb++] = G.proc(cur_at(tbx + chw, tby - 1));
    if (!init) {
      if ((X & mv_size) && tbx + wb < cols) b[nb++] = G.proc(prev_level_at(tbx + wb, tby + chh));
      if ((Y & mv_size) && tby + hb < rows) b[nb++] = G.proc(prev_level_at(tbx + chw, tby + hb));
      median = G.proc(prev_level_at(tbx + chw, tby + chh));
      has_median = true;
    } else if (nb == 3) {  // kept for fidelity: INIT samples only left and top, so never taken
      const short r0 = b[0].x, r1 = b[1].x, r2 = b[2].x, c0 = b[0].y, c1 = b[1].y, c2 = b[2].y;
      median = make_short2((short)max(min(r0, r1), min(max(r0, r1), r2)), (short)max(min(c0, c1), min(max(c0, c1), c2)));
      has_median = true;
    }
    b[nb++] = make_short2(0, 0);
    if (a.prev && pp.has_prev)  // subset C: LAST's final stats for this slot, frame coordinates
      nc = G.subset_c(a.prev + base, a.w_in_b, a.h_in_b, bx, by, wb, hb, cc);
    const uint32_t min_sad = (uint32_t)(((unsigned long long)G.min_sad * (unsigned long long)(w * h)) >> 14);
    auto dec = [&](short2 v) { return make_short2((short)(v.x >> s), (short)(v.y >> s)); };
    // all_mvs (one list) or median | subset_b | subset_c
    int n = 0;
    if (lane == 0) {
      s_offs[wid][0] = 0;
      if (has_median) s_mv[wid][n++] = dec(median);
      if (init) s_offs[wid][1] = n;
      for (int k = 0; k < nb; k++) s_mv[wid][n++] = dec(b[k]);
      if (init) s_offs[wid][2] = n;
      for (int k = 0; k < nc; k++) s_mv[wid][n++] = dec(cc[k]);
      s_offs[wid][init ? 3 : 1] = n;
    }
    __syncwarp();
    const SmemPreds P{s_mv[wid], s_offs[wid]};
    Best best;
    if (!init) {
      best = search_block<T, true>(c, P, 1, 0u, 0, g, sub);
    } else {
      // thresh, me.rs:771-772: the f32 product, then a saturating `as u32`
      const float t = __fmul_rn((float)min_sad, 1.2f);
      const uint32_t thresh = (t >= 4294967296.0f ? 0xffffffffu : (uint32_t)t) + ((uint32_t)(w * h) << (a.bit_depth - 8));
      best = search_block<T, true>(c, P, 3, thresh, 24, g, sub);
      if (a.full_search && best.sad >= thresh) {  // me.rs:815-853
        const int range_x = (192 * a.range_scale) >> s, range_y = (64 * a.range_scale) >> s;
        const Best f = full_search_warp<T>(c, c.po_x + max(-range_x, c.rng.x_min / 8), c.po_x + min(range_x, c.rng.x_max / 8),
                                           c.po_y + max(-range_y, c.rng.y_min / 8), c.po_y + min(range_y, c.rng.y_max / 8),
                                           4 >> s, g, sub);
        if (f.cost < best.cost) best = f;
      }
    }
    save(a.stats + base, a, a.log2, bx, by, best, w, h, lane);
    __syncwarp();  // the shared lists are rewritten by this warp's next block
  }
}

int grid_for(const b200_ctx *ctx, size_t items) {
  return (int)std::max<size_t>(1, std::min<size_t>((items + 3) / 4, (size_t)ctx->num_sms * 32));
}

}  // namespace

extern "C" int b200_lookahead_motion_dev(b200_ctx *ctx, size_t npairs, const b200_plane *curs, const b200_plane *refs,
                                         const b200_lookahead_me_params *p, const b200_me_stats *d_prev,
                                         const uint8_t *has_prev, b200_me_stats *d_stats) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, p && curs && refs && d_stats && npairs >= 1, "NULL params / planes / output, or no pair");
  B200_REQUIRE(ctx, !d_prev || has_prev, "d_prev needs the host has_prev flags");
  B200_REQUIRE(ctx, p->tile_w_sb >= 1 && p->tile_h_sb >= 1, "tile size %dx%d SBs must be >= 1", p->tile_w_sb,
               p->tile_h_sb);
  B200_REQUIRE(ctx, p->me_range_scale >= 1 && p->me_range_scale <= 16, "me_range_scale %d out of 1..16",
               p->me_range_scale);
  const int bpp = curs[0].bpp, width = curs[0].width, height = curs[0].height;
  B200_REQUIRE(ctx, bpp == 1 || bpp == 2, "bpp must be 1 or 2");
  B200_REQUIRE(ctx, bpp == 1 ? p->bit_depth == 8 : (p->bit_depth > 8 && p->bit_depth <= 12),
               "bit_depth %d does not fit bpp %d", p->bit_depth, bpp);
  B200_REQUIRE(ctx, width >= 1 && height >= 1 && width <= 8192 && height <= 8192, "frame %dx%d out of range", width,
               height);
  const int W8 = (width + 7) & ~7, H8 = (height + 7) & ~7;
  for (size_t k = 0; k < npairs; k++) {
    for (int side = 0; side < 2; side++) {
      const b200_plane *pl = (side ? refs : curs) + 3 * k;
      for (int s = 0; s < 3; s++) {
        const int pw = (width + (1 << s) - 1) >> s, ph = (height + (1 << s) - 1) >> s;
        B200_REQUIRE(ctx, pl[s].data != nullptr, "pair %zu: plane %d has no device memory", k, s);
        B200_REQUIRE(ctx, pl[s].bpp == bpp, "pair %zu: planes must share bpp", k);
        B200_REQUIRE(ctx, pl[s].width == pw && pl[s].height == ph,
                     "pair %zu: plane %d is %dx%d, want %dx%d (full, (w+1)/2, (w+3)/4)", k, s, pl[s].width,
                     pl[s].height, pw, ph);
      }
    }
  }
  // padding (see the header): the widest block searched at each resolution, within get_mv_range
  for (int s = 0; s < 3; s++) {
    const int mv_full = s == 0 ? 32 : 64;  // full-res px: the refinement re-searches the previous level's blocks
    const int wm = std::min(mv_full, W8 + (1 << s) - 1) >> s, hm = std::min(mv_full, H8 + (1 << s) - 1) >> s;
    const int pw = (width + (1 << s) - 1) >> s, ph = (height + (1 << s) - 1) >> s;
    const int need = std::max({(16 >> s) + wm, (16 >> s) + hm, ((W8 + 16) >> s) + wm - pw, ((H8 + 16) >> s) + hm - ph});
    for (size_t k = 0; k < npairs; k++)
      B200_REQUIRE(ctx, curs[3 * k + s].pad >= need && refs[3 * k + s].pad >= need,
                   "pair %zu: plane %d needs pad >= %d", k, s, need);
  }
  B200_CUDA(ctx, cudaSetDevice(ctx->device));

  const int w_in_b = W8 >> 2, h_in_b = H8 >> 2;
  const size_t ncells = (size_t)w_in_b * h_in_b;
  const size_t table = b200_align_up(npairs * sizeof(LaPair), 256);
  const size_t grid_bytes = npairs * ncells * sizeof(b200_me_stats);
  int st = b200_reserve_dwork(ctx, table + 2 * grid_bytes);
  if (st != B200_OK) return st;
  std::vector<LaPair> host(npairs);
  for (size_t k = 0; k < npairs; k++) {
    for (int s = 0; s < 3; s++) {
      host[k].cur[s] = {curs[3 * k + s].data, curs[3 * k + s].stride};
      host[k].ref[s] = {refs[3 * k + s].data, refs[3 * k + s].stride};
    }
    host[k].has_prev = d_prev && has_prev[k];
  }
  uint8_t *work = (uint8_t *)ctx->dwork;
  B200_CUDA(ctx, cudaMemcpyAsync(work, host.data(), npairs * sizeof(LaPair), cudaMemcpyHostToDevice, ctx->stream));

  LaArgs a{};
  a.pairs = (const LaPair *)work;
  a.npairs = (int)npairs;
  a.stats = d_stats;
  a.refined = (b200_me_stats *)(work + table);
  a.unrefined = (b200_me_stats *)(work + table + grid_bytes);
  a.prev = d_prev;
  a.ncells = ncells;
  a.w_in_b = w_in_b, a.h_in_b = h_in_b, a.W8 = W8, a.H8 = H8;
  a.tile_w = p->tile_w_sb * 64, a.tile_h = p->tile_h_sb * 64;
  a.allow_hp = p->allow_high_precision_mv, a.bit_depth = p->bit_depth;
  a.full_search = p->me_allow_full_search, a.range_scale = p->me_range_scale;
  a.ntr = (H8 + a.tile_h - 1) / a.tile_h;
  for (int log2 = 4; log2 >= 2; log2--) {
    const int s = log2 - 2, mv_size = MI_SIZE << log2;  // ssdec 2, 1, 0
    // me.rs:175-176 in f64, then a saturating `as u32`
    const double l = p->me_lambda * 256.0 / (double)(1 << (2 * s)) * (s == 0 ? 0.5 : 0.125);
    a.lambda = !(l > 0.0) ? 0u : l >= 4294967295.0 ? 0xffffffffu : (uint32_t)l;
    a.log2 = log2, a.ssdec = s;
    if (log2 < 4) {
      const int pm = mv_size * 2;
      const size_t items = npairs * (size_t)((W8 + pm - 1) / pm) * ((H8 + pm - 1) / pm);
      if (bpp == 1)
        refine_kernel<uint8_t><<<grid_for(ctx, items), 128, 0, ctx->stream>>>(a);
      else
        refine_kernel<uint16_t><<<grid_for(ctx, items), 128, 0, ctx->stream>>>(a);
      B200_LAUNCH_CHECK(ctx);
    }
    a.nbx = (W8 + mv_size - 1) / mv_size, a.nby = (H8 + mv_size - 1) / mv_size;
    a.tbw = a.tile_w / mv_size, a.tbh = a.tile_h / mv_size;
    const int ndiag = std::min(a.tbw, a.nbx) + std::min(a.tbh, a.nby) - 1;
    const size_t items = npairs * (size_t)a.nbx * a.ntr;
    for (int d = 0; d < ndiag; d++) {
      a.diag = d;
      if (bpp == 1)
        diag_kernel<uint8_t><<<grid_for(ctx, items), 128, 0, ctx->stream>>>(a);
      else
        diag_kernel<uint16_t><<<grid_for(ctx, items), 128, 0, ctx->stream>>>(a);
      B200_LAUNCH_CHECK(ctx);
    }
  }
  return B200_OK;
}
