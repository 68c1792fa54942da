// cdef_rdo.cu — the CDEF pass of rdo_loop_decision (rav1e src/rdo.rs:2104-2567, RestorationFilter::None
// and no-LRU branches) for many loop-restoration areas in one call: every superblock of every area at every
// cdef index 0 .. 1 << cdef_bits, evaluated by cdef_sb_dev.cuh; the first minimum wins and, on request, the
// winner's pixels are written.  One CTA per area superblock; only distortions, costs, the winner and the
// winner's pixels leave the chip.
#include <vector>

#include "cdef_sb_dev.cuh"
#include "loop_filter_checks.cuh"

namespace {

constexpr int kRdoMaxAreas = 256;   // areas per launch (kernel-parameter table)
constexpr int kRdoMaxSlots = 1024;  // superblocks per launch

struct CdefRdoArgs {
  CdefSbArgs sb;
  void *out[3];
  int out_stride[3];
  const uint32_t *rate;
  unsigned long long *err;
  double *cost;
  int8_t *best;
};

// The areas and superblocks of one launch.  slot[k] = local area index << 4 | sby << 2 | sbx.
struct CdefRdoSlots {
  uint32_t area0;  // index of local area 0 in the caller's array
  uint16_t ax[kRdoMaxAreas], ay[kRdoMaxAreas];
  uint8_t wh[kRdoMaxAreas];  // sb_w | sb_h << 4
  uint16_t slot[kRdoMaxSlots];
};
static_assert(sizeof(CdefRdoArgs) + sizeof(CdefRdoSlots) <= 4096, "kernel parameters over 4 KB");

template <typename T, int XDEC, int YDEC>
__global__ void __launch_bounds__(kSbThreads, 2)
    cdef_rdo_kernel(const __grid_constant__ CdefRdoArgs A, const __grid_constant__ CdefRdoSlots S) {
  extern __shared__ __align__(16) unsigned char smem[];
  const uint32_t e = S.slot[blockIdx.x];
  const int la = e >> 4;
  const size_t slot = (size_t)(S.area0 + la) * 16 + (e & 15);
  CdefSb<T, XDEC, YDEC, false> sb(smem, sb_geo(A.sb, S.ax[la], S.ay[la], S.wh[la] & 15, S.wh[la] >> 4, e),
                                  A.sb.bit_depth);
  const bool coded = sb.stage_blocks(A.sb);
  sb.stage_pixels(A.sb, coded);
  sb.analyze();

  int best = -1;
  double best_cost = -1.;
  if (coded) {
    const uint32_t rate = A.rate ? A.rate[slot] : 0u;
    for (int i = 0; i < A.sb.nidx; i++)
      sb.evaluate(A.sb, i, rate, nullptr, A.err + slot * 8, A.cost + slot * 8, best, best_cost);
  }
  if (threadIdx.x == 0) {
    A.best[slot] = (int8_t)best;
    *sb.s_best = best;
  }
  if (!A.out[0]) return;
  __syncthreads();
  // ---- the area's CDEF output: the winner, or a copy of rec for skipped blocks and superblocks
  const int wi = max(*sb.s_best, 0);
#pragma unroll
  for (int p = 0; p < 3; p++)
    if (p < A.sb.planes) sb.write(A.sb, p, wi, A.out[p], A.out_stride[p]);
}

}  // namespace

extern "C" int b200_cdef_rdo_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src, const b200_plane *out,
                                 int planes, int xdec, int ydec, int frame_width, int frame_height, int bit_depth,
                                 int damping, int cdef_bits, const uint8_t y_strengths[8],
                                 const uint8_t uv_strengths[8], const uint8_t *d_skip8, const uint32_t *d_imp_scales,
                                 const uint32_t dist_scale[3], double lambda, const b200_cdef_rdo_area *areas,
                                 size_t n_areas, const uint32_t *d_rate, uint64_t *d_err, double *d_cost,
                                 int8_t *d_best) {
  if (int st = lf_check_frame(ctx, planes, xdec, ydec, bit_depth, frame_width, frame_height)) return st;
  B200_REQUIRE(ctx, rec && src && dist_scale && d_err && d_cost && d_best, "NULL rec / src / dist_scale / outputs");
  if (int st = lf_check_cdef(ctx, damping, cdef_bits, y_strengths, uv_strengths)) return st;
  for (const b200_plane *pl : {rec, src, out})
    if (pl)
      if (int st = lf_check_planes(ctx, pl, planes, xdec, ydec, bit_depth, frame_width, frame_height)) return st;
  if (out)
    for (int p = 0; p < planes; p++)
      for (int r = 0; r < planes; r++)
        B200_REQUIRE(ctx, out[p].data != rec[r].data, "out plane %d aliases rec plane %d", p, r);
  if (n_areas == 0) return B200_OK;
  if (int st = lf_check_areas(ctx, areas, n_areas, frame_width, frame_height, true)) return st;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));

  CdefRdoArgs a{};
  a.sb = cdef_sb_args(rec, src, planes, frame_width, frame_height, bit_depth, damping, 1 << cdef_bits, y_strengths,
                      uv_strengths, d_skip8, d_imp_scales, dist_scale, lambda);
  for (int p = 0; p < planes; p++) {
    a.out[p] = out ? out[p].data : nullptr;
    a.out_stride[p] = out ? out[p].stride : 0;
  }
  a.rate = d_rate;
  a.err = (unsigned long long *)d_err;
  a.cost = d_cost;
  a.best = d_best;

  // areas in launch-sized groups: up to kRdoMaxAreas areas and kRdoMaxSlots superblocks each
  CdefRdoSlots s;
  size_t k = 0;
  while (k < n_areas) {
    s.area0 = (uint32_t)k;
    int na = 0, ns = 0;
    while (k < n_areas && na < kRdoMaxAreas && ns + areas[k].sb_w * areas[k].sb_h <= kRdoMaxSlots) {
      const b200_cdef_rdo_area &r = areas[k];
      s.ax[na] = (uint16_t)r.sbx;
      s.ay[na] = (uint16_t)r.sby;
      s.wh[na] = (uint8_t)(r.sb_w | r.sb_h << 4);
      for (int y = 0; y < r.sb_h; y++)
        for (int x = 0; x < r.sb_w; x++) s.slot[ns++] = (uint16_t)(na << 4 | y << 2 | x);
      na++, k++;
    }
    const int st = cdef_sb_launch<false>(ctx, bit_depth == 8 ? 1 : 2, xdec, ydec, ns, [](auto k) {
      using K = decltype(k);
      return cdef_rdo_kernel<typename K::Pixel, K::xdec, K::ydec>;
    }, a, s);
    if (st) return st;
  }
  return B200_OK;
}
