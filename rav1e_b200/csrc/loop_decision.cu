// loop_decision.cu — rdo_loop_decision (rav1e src/rdo.rs:2104-2745) after its optional deblock, for many
// loop-restoration areas in one call: the CDEF / restoration pass loop, C, L, C, L, .. per area until a
// stage changes nothing.
//
// Launches, all on the context's stream:
//  - loop_flags / loop_areas / loop_init: which areas have CDEF work (a superblock that is not all-skip) and
//    restoration work, the initial unit state (None, cost -1) and a copy of rec into `work` over the
//    scratch rect of every area that runs a stage (cdef_work = rec_subset.clone(), rdo.rs:2329-2330).
//  - C stage: loop_cdef_kernel once per anti-diagonal of superblocks (sbx + sby = 0 .. 6), or once for all of
//    them where no unit can hold Sgrproj (the first pass, or no unit searched).  A superblock's
//    Sgrproj branch reads up to 4 columns to its left and 2 rows above from `work`, which must hold THIS
//    pass's winners of the left, upper and upper-left superblocks, as the reference's raster walk leaves
//    them; those lie on earlier diagonals, so stream order alone separates the writers from the readers.
//  - L stage: the restoration search's four kernels (lrf_search_launch, lrf_search.cu), the incumbents
//    carried on the device and areas that already stopped masked out.
//  - loop_status: per area, was the stage a change; the areas still running are counted, and that count
//    is the one read back per stage.
#include <algorithm>
#include <vector>

#include "cdef_sb_dev.cuh"
#include "loop_filter_checks.cuh"
#include "lrf_search_dev.cuh"

namespace {

enum : uint8_t { kCdefWork = 1, kLrfWork = 2 };

struct LoopArgs {
  CdefSbArgs sb;
  void *work[3];
  int work_stride[3];
  int enable_cdef;
  const b200_cdef_rdo_area *areas;
  uint32_t n_areas, n_units;
  const b200_loop_unit *units;
  const int32_t *sb_unit;
  uint32_t *flags;         // [area] kCdefWork | kLrfWork
  uint8_t *active;         // [area]
  uint8_t *changed;        // [area] set by the current stage
  int *area_stages;        // [area]
  int *status;             // [0] areas still running, [1] the longest area's stage count
  b200_lrf_unit *unit;     // [unit] the current filter (best_lrf)
  double *unit_cost;       // [unit] best_lrf_cost
  uint8_t *written;        // [unit]
  int8_t *best;            // [slot]
  unsigned long long *err;
  double *cost;
};

// slot = area << 4 | sby << 2 | sbx
__device__ __forceinline__ SbGeo sb_geo(const LoopArgs &A, uint32_t slot) {
  const b200_cdef_rdo_area r = A.areas[slot >> 4];
  return sb_geo(A.sb, r.sbx, r.sby, r.sb_w, r.sb_h, slot);
}

// per superblock: does CDEF run on it (rdo.rs:2189-2205); an area has CDEF work if one does
__global__ void loop_flags(const __grid_constant__ LoopArgs A, const uint32_t *slots) {
  const uint32_t slot = slots[blockIdx.x];
  const SbGeo g = sb_geo(A, slot);
  const int t = threadIdx.x;
  int coded = 0;
  if (t < 64 && A.enable_cdef) {
    const int bx = t & 7, by = t >> 3;
    if (bx < g.bw8 && by < g.bh8)
      coded = !(A.sb.skip8 && A.sb.skip8[(size_t)(((g.ay + g.y0) >> 3) + by) * A.sb.w8 + ((g.ax + g.x0) >> 3) + bx]);
  }
  if (__syncthreads_or(coded) && t == 0) atomicOr(&A.flags[slot >> 4], (uint32_t)kCdefWork);
}

// per area: the areas that run a stage (rdo.rs:2267); per unit of those: None, cost -1, not written
__global__ void loop_areas(const __grid_constant__ LoopArgs A) {
  for (uint32_t a = threadIdx.x; a < A.n_areas; a += blockDim.x) {
    A.active[a] = A.flags[a] != 0;
    A.changed[a] = 0;
    A.area_stages[a] = 0;
  }
  for (uint32_t u = threadIdx.x; u < A.n_units; u += blockDim.x)
    if (A.flags[A.units[u].area]) {
      A.unit[u] = b200_lrf_unit{};
      A.unit_cost[u] = -1.;
      A.written[u] = 0;
    }
}

// per superblock of a running area: best_index = -1 and work = rec over its part of the scratch rect
template <typename T>
__global__ void loop_init(const __grid_constant__ LoopArgs A, const uint32_t *slots, int xdec, int ydec) {
  const uint32_t slot = slots[blockIdx.x];
  if (!A.active[slot >> 4]) return;
  const SbGeo g = sb_geo(A, slot);
  if (threadIdx.x == 0) A.best[slot] = -1;
  for (int p = 0; p < A.sb.planes; p++) {
    const int xd = p ? xdec : 0, yd = p ? ydec : 0;
    const int w = min(64, g.wa - g.x0) >> xd, h = min(64, g.ha - g.y0) >> yd;
    const int ox = (g.ax + g.x0) >> xd, oy = (g.ay + g.y0) >> yd;
    const T *s = (const T *)A.sb.rec[p].data;
    T *d = (T *)A.work[p];
    for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
      const int r = i / w, c = i - r * w;
      d[(long long)(oy + r) * A.work_stride[p] + ox + c] = s[(long long)(oy + r) * A.sb.rec[p].stride + ox + c];
    }
  }
}

// one C stage over the superblocks of one anti-diagonal (rdo.rs:2373-2567): cdef_sb_dev.cuh's superblock
// evaluation with the restoration branches of rdo.rs:2424-2527
template <typename T, int XDEC, int YDEC>
__global__ void __launch_bounds__(kSbThreads) loop_cdef_kernel(const __grid_constant__ LoopArgs A,
                                                              const uint32_t *slots) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ uint16_t sp[kSP][kSP];
  __shared__ uint32_t box1[2][kAB][kAB], box2[2][kR2][kAB];
  __shared__ uint32_t a1[kAB][kAB], b1[kAB][kAB], a2[kR2][kAB], b2[kR2][kAB];
  __shared__ int s_mode[3];  // -1: CDEF output measured; else the Sgrproj unit
  __shared__ uint32_t s_rate;

  const int t = threadIdx.x;
  const uint32_t slot = slots[blockIdx.x];
  const uint32_t area = slot >> 4;
  if (!A.active[area] || !(A.flags[area] & kCdefWork)) return;
  CdefSb<T, XDEC, YDEC, true> sb(smem, sb_geo(A, slot), A.sb.bit_depth);
  const SbGeo &G = sb.g;
  const int planes = A.sb.planes, bit_depth = A.sb.bit_depth;

  if (t == 0) s_rate = 0;
  __syncthreads();
  if (t < 3) {  // the restoration branch of each plane (rdo.rs:2424-2431) and its rate
    int m = -1;
    const int32_t u = t < planes && (A.flags[area] & kLrfWork) ? A.sb_unit[slot * 3 + t] : -1;
    if (u >= 0) {
      const b200_lrf_unit f = A.unit[u];
      atomicAdd(&s_rate, lrf_rate(A.units[u], f.type, f.set, f.xqd[0], f.xqd[1]));
      if (f.type == 2) m = u;
    }
    s_mode[t] = m;
  }
  if (!sb.stage_blocks(A.sb)) return;  // rdo.rs:2380: an all-skip superblock is not decided
  const bool any_sgr = s_mode[0] >= 0 || s_mode[1] >= 0 || s_mode[2] >= 0;
  sb.stage_pixels(A.sb, true);
  sb.analyze();

  // the self-guided filter of plane p's part of the superblock, read from the working copy (rdo.rs:2458-2488)
  auto sgr_plane = [&](int p) {
    const int xd = p ? XDEC : 0, yd = p ? YDEC : 0;
    const b200_lrf_unit f = A.unit[s_mode[p]];
    const int po_x = G.x0 >> xd, po_y = G.y0 >> yd;
    const int vis_w = min(64 >> xd, ((A.sb.width - G.ax) >> xd) - po_x);
    const int vis_h = min(64 >> yd, ((A.sb.height - G.ay) >> yd) - po_y);
    const T *in = (const T *)A.work[p] + (long long)(G.ay >> yd) * A.work_stride[p] + (G.ax >> xd);
    const uint32_t s2 = kSgrS[f.set][0], s1 = kSgrS[f.set][1];
    const int w0 = f.xqd[0], w1 = f.xqd[1], w2 = 128 - w0 - w1;
    uint16_t *o = sb.sg + p * kSbPx;
    for (int i = t; i < kSbPx; i += kSbThreads) o[i] = B200_LRF_WORK_FILL;
    for (int ty = 0; ty < vis_h; ty += kT)
      for (int tx = 0; tx < vis_w; tx += kT) {
        __syncthreads();
        sgr_stage_tile<T>(sp, in, A.work_stride[p], po_x, po_y, vis_w, vis_h, tx, ty);
        __syncthreads();
        sgr_box_sums(sp, box1, box2);
        __syncthreads();
        sgr_ab(box1, box2, a1, b1, a2, b2, s1, s2, bit_depth - 8);
        __syncthreads();
        for (int i = t; i < kT * kT; i += kSbThreads) {
          const int y = i / kT, x = i - y * kT;
          if (tx + x >= vis_w || ty + y >= vis_h) continue;
          uint32_t g1, g2;
          const uint32_t px = sgr_f(sp, a1, b1, a2, b2, s1, s2, y, x, g1, g2);
          o[(ty + y) * 64 + tx + x] = sgr_apply(w0, w1, w2, g1, g2, px, bit_depth);
        }
      }
  };

  int best = -1;
  double best_cost = -1.;
  for (int i = 0; i < A.sb.nidx; i++) {
    if (any_sgr) {  // filter into the working copy, then the self-guided filter reads it
#pragma unroll
      for (int p = 0; p < 3; p++)
        if (p < planes && s_mode[p] >= 0) sb.write(A.sb, p, i, A.work[p], A.work_stride[p]);
      __syncthreads();
#pragma unroll
      for (int p = 0; p < 3; p++)
        if (p < planes && s_mode[p] >= 0) sgr_plane(p);
      __syncthreads();
    }
    sb.evaluate(A.sb, i, s_rate, s_mode, A.err ? A.err + slot * 8 : nullptr, A.cost ? A.cost + slot * 8 : nullptr,
                best, best_cost);
  }
  if (t == 0) {
    if (best != A.best[slot]) A.changed[area] = 1;  // rdo.rs:2537-2542
    A.best[slot] = (int8_t)best;
    *sb.s_best = best;
  }
  __syncthreads();
  // ---- keep the working copy up to date with the winner (rdo.rs:2554-2564)
  const int wi = *sb.s_best;
#pragma unroll
  for (int p = 0; p < 3; p++)
    if (p < planes) sb.write(A.sb, p, wi, A.work[p], A.work_stride[p]);
}

// per area: was this stage a change; count the areas still running and the longest stage count
__global__ void loop_status(const __grid_constant__ LoopArgs A, int stage) {
  __shared__ int s_run, s_long;
  if (threadIdx.x == 0) s_run = 0, s_long = 0;
  __syncthreads();
  int run = 0, lng = 0;
  for (uint32_t a = threadIdx.x; a < A.n_areas; a += blockDim.x) {
    if (A.active[a]) {
      // the first C stage always counts as a change (cdef_change starts true, rdo.rs:2370)
      const bool ch = stage == 0 || A.changed[a];
      A.area_stages[a] = stage + 1;
      if (!ch) A.active[a] = 0;
    }
    A.changed[a] = 0;
    run += A.active[a];
    lng = max(lng, A.area_stages[a]);
  }
  atomicAdd(&s_run, run);
  atomicMax(&s_long, lng);
  __syncthreads();
  if (threadIdx.x == 0) A.status[0] = s_run, A.status[1] = s_long;
}

bool overlaps(const b200_plane &a, const b200_plane &b) {
  const uint8_t *a0 = (const uint8_t *)a.data, *b0 = (const uint8_t *)b.data;
  const uint8_t *a1 = a0 + ((size_t)a.stride * (a.height - 1) + a.width) * a.bpp;
  const uint8_t *b1 = b0 + ((size_t)b.stride * (b.height - 1) + b.width) * b.bpp;
  return a0 < b1 && b0 < a1;
}

}  // namespace

extern "C" int b200_loop_decision_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src,
                                      const b200_plane *work, int planes, int xdec, int ydec, int frame_width,
                                      int frame_height, int bit_depth, int enable_cdef, int damping, int cdef_bits,
                                      const uint8_t y_strengths[8], const uint8_t uv_strengths[8],
                                      const uint8_t *d_skip8, int enable_restoration, const int unit_size[3],
                                      int reduced_sets, const uint32_t *d_imp_scales, const uint32_t dist_scale[3],
                                      double lambda, const b200_cdef_rdo_area *areas, size_t n_areas,
                                      const b200_loop_unit *units, size_t n_units, const int32_t *sb_unit,
                                      int8_t *d_best_index, b200_lrf_unit *d_unit, double *d_unit_cost,
                                      uint8_t *d_written, uint64_t *d_err, double *d_cost, int *stages) {
  if (int st = lf_check_frame(ctx, planes, xdec, ydec, bit_depth, frame_width, frame_height)) return st;
  B200_REQUIRE(ctx, rec && src && work && dist_scale && stages && d_best_index,
               "NULL rec / src / work / dist_scale / stages / d_best_index");
  B200_REQUIRE(ctx, n_units == 0 || (d_unit && d_unit_cost && d_written), "NULL unit outputs");
  if (enable_cdef)
    if (int st = lf_check_cdef(ctx, damping, cdef_bits, y_strengths, uv_strengths)) return st;
  const int nidx = enable_cdef ? 1 << cdef_bits : 0;
  for (const b200_plane *pl : {rec, src, work})
    if (int st = lf_check_planes(ctx, pl, planes, xdec, ydec, bit_depth, frame_width, frame_height)) return st;
  for (int p = 0; p < planes; p++)
    for (int r = 0; r < planes; r++)
      B200_REQUIRE(ctx, !overlaps(work[p], rec[r]) && !overlaps(work[p], src[r]),
                   "work plane %d aliases rec or src plane %d", p, r);
  if (enable_restoration)
    if (int st = lf_check_unit_sizes(ctx, unit_size, planes, xdec, ydec)) return st;
  if (n_areas == 0) {
    *stages = 0;
    return B200_OK;
  }
  B200_REQUIRE(ctx, sb_unit != nullptr, "NULL sb_unit");
  B200_REQUIRE(ctx, n_units == 0 || units != nullptr, "NULL units");
  B200_REQUIRE(ctx, n_areas <= (1u << 20) && n_units <= (1u << 24), "%zu areas / %zu units: too many", n_areas,
               n_units);
  if (int st = lf_check_areas(ctx, areas, n_areas, frame_width, frame_height, true)) return st;
  const int bpp = bit_depth == 8 ? 1 : 2;
  std::vector<uint32_t> flags(n_areas, 0);
  std::vector<uint32_t> diag[7];
  for (size_t k = 0; k < n_areas; k++)
    for (int y = 0; y < areas[k].sb_h; y++)
      for (int x = 0; x < areas[k].sb_w; x++) diag[x + y].push_back((uint32_t)(k * 16 + y * 4 + x));
  // the restoration stage's items: the units with `search` set
  std::vector<b200_lrf_search_item> items;
  std::vector<Geo> geo;
  std::vector<Tile> tiles;
  std::vector<uint32_t> unit_of;
  for (size_t u = 0; u < n_units; u++) {
    const b200_loop_unit &un = units[u];
    B200_REQUIRE(ctx, un.area >= 0 && (size_t)un.area < n_areas, "unit %zu: area %d of %zu", u, un.area, n_areas);
    B200_REQUIRE(ctx, un.plane >= 0 && un.plane < planes, "unit %zu: plane %d", u, un.plane);
    B200_REQUIRE(ctx, sgrproj_xqd_ok(un.sgrproj_ref[0], un.sgrproj_ref[1]), "unit %zu: sgrproj_ref (%d, %d) out of range",
                 u, un.sgrproj_ref[0], un.sgrproj_ref[1]);
    if (!enable_restoration) continue;
    Geo g;
    if (int st = lrf_item_geo(ctx, u, areas[un.area], un.plane, xdec, ydec, unit_size[un.plane], un.lru_x, un.lru_y,
                              frame_width, frame_height, g))
      return st;
    if (!un.search) continue;
    flags[un.area] |= kLrfWork;
    b200_lrf_search_item it{};
    it.area = un.area, it.plane = un.plane, it.lru_x = un.lru_x, it.lru_y = un.lru_y;
    it.none_bits = un.none_bits, it.sgr_bits = un.sgr_bits;
    it.sgrproj_ref[0] = un.sgrproj_ref[0], it.sgrproj_ref[1] = un.sgrproj_ref[1];
    it.incoming_cost = -1.;
    lrf_item_tiles(g, (uint32_t)items.size(), tiles);
    items.push_back(it);
    geo.push_back(g);
    unit_of.push_back((uint32_t)u);
  }
  for (size_t k = 0; k < n_areas; k++)
    for (int s = 0; s < 16; s++)
      for (int p = 0; p < 3; p++) {
        if ((s & 3) >= areas[k].sb_w || (s >> 2) >= areas[k].sb_h) continue;
        const int32_t u = p < planes ? sb_unit[(k * 16 + s) * 3 + p] : -1;
        B200_REQUIRE(ctx, u >= -1 && (int64_t)u < (int64_t)n_units, "sb_unit[%zu]: %d of %zu units",
                     (k * 16 + s) * 3 + p, u, n_units);
        B200_REQUIRE(ctx, u < 0 || ((size_t)units[u].area == k && units[u].plane == p),
                     "sb_unit[%zu]: unit %d belongs to area %d plane %d", (k * 16 + s) * 3 + p, u,
                     u < 0 ? -1 : units[u].area, u < 0 ? -1 : units[u].plane);
      }

  // ---- one upload: areas, map, units, flags, the diagonals' slot lists, the items, geometry and tiles
  size_t nslots = 0;
  for (auto &d : diag) nslots += d.size();
  std::vector<uint32_t> slots;
  slots.reserve(nslots);
  size_t doff[8] = {0};
  for (int d = 0; d < 7; d++) {
    doff[d] = slots.size();
    slots.insert(slots.end(), diag[d].begin(), diag[d].end());
  }
  doff[7] = slots.size();
  const size_t n_items = items.size();
  std::vector<std::pair<const void *, size_t>> parts = {
      {areas, n_areas * sizeof(b200_cdef_rdo_area)},  {sb_unit, n_areas * 48 * sizeof(int32_t)},
      {units, n_units * sizeof(b200_loop_unit)},     {flags.data(), n_areas * sizeof(uint32_t)},
      {slots.data(), slots.size() * sizeof(uint32_t)}, {items.data(), n_items * sizeof(b200_lrf_search_item)},
      {geo.data(), n_items * sizeof(Geo)},           {tiles.data(), tiles.size() * sizeof(Tile)},
      {unit_of.data(), n_items * sizeof(uint32_t)}};
  size_t up_bytes = 0, off[9];
  for (size_t i = 0; i < parts.size(); i++) {
    off[i] = up_bytes;
    up_bytes += b200_align_up(parts[i].second, 256);
  }
  std::vector<uint8_t> packed(up_bytes, 0);
  for (size_t i = 0; i < parts.size(); i++)
    if (parts[i].second) memcpy(packed.data() + off[i], parts[i].first, parts[i].second);
  const size_t b_area = b200_align_up(n_areas * 4, 256) * 3, b_status = 256;
  const size_t b_acc = std::max<size_t>(n_items, 1) * 16 * 5 * sizeof(long long);
  const size_t b_err = std::max<size_t>(n_items, 1) * kCands * sizeof(unsigned long long);
  const size_t b_item = std::max<size_t>(n_items, 1) * (32 + sizeof(b200_lrf_unit) + 8 + 1);
  HostStage s(ctx, up_bytes + b_area + b_status + 4 * 256 + b200_align_up(b_acc, 256) + b200_align_up(b_err, 256) +
                       b200_align_up(b_item, 256) + 3 * 256);
  uint8_t *d_up = s.take(up_bytes);
  uint8_t *d_active = s.take(n_areas), *d_changed = s.take(n_areas);
  int *d_area_stages = (int *)s.take(n_areas * 4);
  int *d_status = (int *)s.take(b_status);
  long long *d_acc = (long long *)s.take(b_acc);
  unsigned long long *d_cerr = (unsigned long long *)s.take(b_err);
  int8_t *d_xq = (int8_t *)s.take(std::max<size_t>(n_items, 1) * 32);
  b200_lrf_unit *d_ibest = (b200_lrf_unit *)s.take(std::max<size_t>(n_items, 1) * sizeof(b200_lrf_unit));
  double *d_icost = (double *)s.take(std::max<size_t>(n_items, 1) * 8);
  uint8_t *d_ichanged = s.take(std::max<size_t>(n_items, 1));
  s.up(d_up, packed.data(), up_bytes);
  if (!s.ok()) return s.finish(false);

  LoopArgs a{};
  a.sb = cdef_sb_args(rec, src, planes, frame_width, frame_height, bit_depth, damping, nidx, y_strengths,
                      uv_strengths, d_skip8, d_imp_scales, dist_scale, lambda);
  for (int p = 0; p < planes; p++) {
    a.work[p] = work[p].data;
    a.work_stride[p] = work[p].stride;
  }
  a.enable_cdef = enable_cdef != 0;
  a.areas = (const b200_cdef_rdo_area *)(d_up + off[0]);
  a.sb_unit = (const int32_t *)(d_up + off[1]);
  a.units = (const b200_loop_unit *)(d_up + off[2]);
  a.flags = (uint32_t *)(d_up + off[3]);
  a.n_areas = (uint32_t)n_areas, a.n_units = (uint32_t)n_units;
  a.active = d_active, a.changed = d_changed, a.area_stages = d_area_stages, a.status = d_status;
  a.unit = d_unit, a.unit_cost = d_unit_cost, a.written = d_written;
  a.best = d_best_index, a.err = (unsigned long long *)d_err, a.cost = d_cost;
  const uint32_t *d_slots = (const uint32_t *)(d_up + off[4]);

  SearchArgs la = search_args(work, src, planes, xdec, ydec, bit_depth, frame_width, reduced_sets, d_imp_scales,
                              dist_scale, lambda);
  la.items = (const b200_lrf_search_item *)(d_up + off[5]);
  la.geo = (const Geo *)(d_up + off[6]);
  la.tiles = (const Tile *)(d_up + off[7]);
  la.n_items = (uint32_t)n_items, la.n_tiles = (uint32_t)tiles.size();
  la.acc = d_acc, la.err = d_cerr, la.xq = d_xq;
  la.best = d_ibest, la.cost = d_icost, la.changed = d_ichanged;
  la.unit_of = (const uint32_t *)(d_up + off[8]);
  la.inc = d_unit, la.inc_cost = d_unit_cost, la.written = d_written;
  la.active = d_active, la.area_changed = d_changed;

  const unsigned n_all = (unsigned)slots.size();
  loop_flags<<<n_all, kSbThreads, 0, ctx->stream>>>(a, d_slots);
  B200_LAUNCH_CHECK(ctx);
  loop_areas<<<1, 256, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  if (bpp == 1) loop_init<uint8_t><<<n_all, kSbThreads, 0, ctx->stream>>>(a, d_slots, xdec, ydec);
  else loop_init<uint16_t><<<n_all, kSbThreads, 0, ctx->stream>>>(a, d_slots, xdec, ydec);
  B200_LAUNCH_CHECK(ctx);

  int result = -1;
  for (int stage = 0; stage < B200_LOOP_MAX_STAGES; stage++) {
    if (!(stage & 1)) {  // C
      // No unit holds Sgrproj on the first pass (all start as None) or when no unit is searched, so no superblock
      // reads another's output: every slot goes in one launch.  Otherwise one launch per anti-diagonal.
      const bool one_launch = stage == 0 || n_items == 0;
      for (int d = 0; d < 7 && nidx; d++) {
        const size_t b = one_launch ? 0 : doff[d], e = one_launch ? doff[7] : doff[d + 1];
        if (e > b) {
          const int st = cdef_sb_launch<true>(ctx, bpp, xdec, ydec, (int)(e - b), [](auto k) {
            using K = decltype(k);
            return loop_cdef_kernel<typename K::Pixel, K::xdec, K::ydec>;
          }, a, d_slots + b);
          if (st) {
            s.run(st);
            return s.finish(false);
          }
        }
        if (one_launch) break;
      }
    } else if (n_items) {  // L
      if (int st = lrf_search::lrf_search_launch(ctx, s, la)) return st;
    }
    loop_status<<<1, 256, 0, ctx->stream>>>(a, stage);
    B200_LAUNCH_CHECK(ctx);
    int st[2] = {0, 0};
    s.down(st, d_status, sizeof(st));  // the one synchronisation of the stage
    s.run(cudaStreamSynchronize(ctx->stream) == cudaSuccess ? B200_OK : B200_ERR_CUDA);
    if (!s.ok()) return s.finish(false);
    if (st[0] == 0) {
      result = st[1];
      break;
    }
  }
  *stages = result;
  return s.finish(false);
}
