// me_host.cu — host-buffer (`*_batch`) and per-call reference-signature entry points of the
// SAD/SATD/ME path.  They copy the caller's host buffers (pinned or pageable) to a stream-
// ordered device allocation, run the same device kernels as the `_dev` forms (me_cand.cu, me_full_search.cu) and copy results back before returning.
#include "host_stage.cuh"

namespace {

size_t host_plane_span(const b200_host_plane *hp, size_t *row_bytes, size_t *rows) {
  *row_bytes = (size_t)(hp->width + 2 * hp->pad) * hp->bpp;
  *rows = (size_t)hp->height + 2 * (size_t)hp->pad;
  return *row_bytes * *rows;
}

// Device layout for a staged plane: pixel (0,0) and every row start 128-byte aligned.
size_t staged_lead(const b200_host_plane *hp) { return b200_align_up((size_t)hp->pad * hp->bpp, 128); }
size_t staged_pitch(const b200_host_plane *hp) {
  return b200_align_up(staged_lead(hp) + (size_t)(hp->width + hp->pad) * hp->bpp + 64, 128);
}

void upload_host_plane(HostStage &s, const b200_host_plane *hp, uint8_t *dbase, b200_plane *out) {
  const size_t pitch = staged_pitch(hp);
  size_t row_bytes, rows;
  host_plane_span(hp, &row_bytes, &rows);
  const uint8_t *h0 = (const uint8_t *)hp->data - (ptrdiff_t)hp->pad * hp->stride -
                      (ptrdiff_t)hp->pad * hp->bpp;
  const size_t lead = staged_lead(hp);
  s.up2d(dbase + lead - (size_t)hp->pad * hp->bpp, pitch, h0, (size_t)hp->stride, row_bytes, rows);
  out->alloc = nullptr;
  out->data = dbase + (size_t)hp->pad * pitch + lead;
  out->stride = (int32_t)(pitch / hp->bpp);
  out->width = hp->width;
  out->height = hp->height;
  out->pad = hp->pad;
  out->bpp = hp->bpp;
}

int check_host_plane(b200_ctx *ctx, const b200_host_plane *hp) {
  B200_REQUIRE(ctx, hp && hp->data, "NULL host plane");
  B200_REQUIRE(ctx, (hp->bpp == 1 || hp->bpp == 2) && hp->width > 0 && hp->height > 0 && hp->pad >= 0,
               "bad host plane geometry");
  B200_REQUIRE(ctx, hp->stride >= (ptrdiff_t)(hp->width + 2 * hp->pad) * hp->bpp,
               "host stride smaller than width + 2*pad");
  return B200_OK;
}

}  // namespace

// Host descriptors in / host results out; planes either host (copied) or device-resident.
// MotionVector lists (4 bytes per candidate, the block implied by the CSR) -> b200_cand records.
__global__ void expand_mvs_kernel(const short2 *mvs, const uint32_t *offs, size_t nblocks, b200_cand *out) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t b = warp0; b < nblocks; b += nwarps) {
    const uint32_t lo = offs[b], hi = offs[b + 1];
    for (uint32_t i = lo + lane; i < hi; i += 32) {
      const short2 m = mvs[i];  // {row, col}
      b200_cand c;
      c.block = (uint32_t)b;
      c.mv_row = m.x;
      c.mv_col = m.y;
      out[i] = c;
    }
  }
}

static int me_candidates_host_impl(b200_ctx *ctx, const b200_host_plane *cur,
                                   const b200_host_plane *ref, const b200_plane *rcur,
                                   const b200_plane *rref, const b200_block *blocks,
                                   size_t nblocks, const b200_cand *cands, const int16_t *mvs, size_t ncands,
                                   const uint32_t *cand_offsets, const int16_t *pmv,
                                   const b200_me_params *params, uint32_t *sad,
                                   uint64_t *cost, b200_me_result *best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (!rcur) {
    if (int st = check_host_plane(ctx, cur)) return st;
    if (int st = check_host_plane(ctx, ref)) return st;
  } else {
    B200_REQUIRE(ctx, rcur->data && rref && rref->data, "bad resident planes");
  }
  B200_REQUIRE(ctx, params && blocks && (cands || mvs || !ncands), "NULL params/blocks/cands");
  B200_REQUIRE(ctx, !mvs || cand_offsets, "MotionVector lists need cand_offsets (the CSR names the block)");
  B200_REQUIRE(ctx, best == nullptr || cand_offsets != nullptr, "best needs cand_offsets");
  size_t rb, rows;
  const size_t cur_bytes = rcur ? 0 : staged_pitch(cur) * (host_plane_span(cur, &rb, &rows), rows) + 512;
  const size_t ref_bytes = rcur ? 0 : staged_pitch(ref) * (host_plane_span(ref, &rb, &rows), rows) + 512;
  size_t total = cur_bytes + ref_bytes + nblocks * sizeof(b200_block) + ncands * sizeof(b200_cand) +
                 (cand_offsets ? (nblocks + 1) * 4 : 0) + (pmv ? nblocks * 8 : 0) +
                 (sad ? ncands * 4 : 0) + (cost ? ncands * 8 : 0) +
                 (best ? nblocks * sizeof(b200_me_result) : 0) + (mvs ? ncands * 4 : 0) + 16 * 256;
  // leave room for the generic path's internal cost/sad scratch (b200_reserve_dwork is
  // grow-only and shared): carve our buffers from a private allocation instead.
  HostStage s(ctx, total);
  b200_plane dcur, dref;
  if (rcur) {
    dcur = *rcur;
    dref = *rref;
  } else {
    upload_host_plane(s, cur, s.take(cur_bytes), &dcur);
    upload_host_plane(s, ref, s.take(ref_bytes), &dref);
  }
  b200_block *d_blocks = (b200_block *)s.take(nblocks * sizeof(b200_block));
  b200_cand *d_cands = (b200_cand *)s.take(ncands * sizeof(b200_cand));
  short2 *d_mvs = mvs ? (short2 *)s.take(ncands * 4) : nullptr;
  uint32_t *d_offs = cand_offsets ? (uint32_t *)s.take((nblocks + 1) * 4) : nullptr;
  int16_t *d_pmv = pmv ? (int16_t *)s.take(nblocks * 8) : nullptr;
  uint32_t *d_sad = sad ? (uint32_t *)s.take(ncands * 4) : nullptr;
  uint64_t *d_cost = cost ? (uint64_t *)s.take(ncands * 8) : nullptr;
  b200_me_result *d_best = best ? (b200_me_result *)s.take(nblocks * sizeof(b200_me_result)) : nullptr;
  s.up(d_blocks, blocks, nblocks * sizeof(b200_block));
  if (d_mvs) {
    s.up(d_mvs, mvs, ncands * 4);
  } else {
    s.up(d_cands, cands, ncands * sizeof(b200_cand));
  }
  if (d_offs) s.up(d_offs, cand_offsets, (nblocks + 1) * 4);
  if (s.ok() && d_mvs && ncands) {
    const int grid = (int)std::min<size_t>((nblocks + 7) / 8, (size_t)ctx->num_sms * 16);
    expand_mvs_kernel<<<grid, 256, 0, ctx->stream>>>(d_mvs, d_offs, nblocks, d_cands);
    ctx->launches++;
  }
  if (d_pmv) s.up(d_pmv, pmv, nblocks * 8);
  if (s.ok())
    s.run(b200_me_candidates_dev(ctx, &dcur, &dref, d_blocks, nblocks, d_cands, ncands, d_offs, d_pmv, params,
                                 d_sad, d_cost, d_best));
  if (sad) s.down(sad, d_sad, ncands * 4);
  if (cost) s.down(cost, d_cost, ncands * 8);
  if (best) s.down(best, d_best, nblocks * sizeof(b200_me_result));
  return s.finish(!ctx->async_batch);
}

extern "C" int b200_me_candidates_batch(b200_ctx *ctx, const b200_host_plane *cur,
                                        const b200_host_plane *ref, const b200_block *blocks,
                                        size_t nblocks, const b200_cand *cands, size_t ncands,
                                        const uint32_t *cand_offsets, const int16_t *pmv,
                                        const b200_me_params *params, uint32_t *sad,
                                        uint64_t *cost, b200_me_result *best) {
  return me_candidates_host_impl(ctx, cur, ref, nullptr, nullptr, blocks, nblocks, cands, nullptr, ncands,
                                 cand_offsets, pmv, params, sad, cost, best);
}

extern "C" int b200_me_candidates_resident(b200_ctx *ctx, const b200_plane *cur,
                                           const b200_plane *ref, const b200_block *blocks,
                                           size_t nblocks, const b200_cand *cands, size_t ncands,
                                           const uint32_t *cand_offsets, const int16_t *pmv,
                                           const b200_me_params *params, uint32_t *sad,
                                           uint64_t *cost, b200_me_result *best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && ref, "NULL planes");
  return me_candidates_host_impl(ctx, nullptr, nullptr, cur, ref, blocks, nblocks, cands, nullptr, ncands,
                                 cand_offsets, pmv, params, sad, cost, best);
}

extern "C" int b200_me_mvs_resident(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                    const b200_block *blocks, size_t nblocks, const int16_t *mvs,
                                    size_t ncands, const uint32_t *cand_offsets, const int16_t *pmv,
                                    const b200_me_params *params, uint32_t *sad, uint64_t *cost,
                                    b200_me_result *best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, cur && ref, "NULL planes");
  B200_REQUIRE(ctx, mvs || !ncands, "NULL mvs");
  return me_candidates_host_impl(ctx, nullptr, nullptr, cur, ref, blocks, nblocks, nullptr, mvs, ncands,
                                 cand_offsets, pmv, params, sad, cost, best);
}

extern "C" int b200_me_full_search_batch(b200_ctx *ctx, const b200_host_plane *cur,
                                         const b200_host_plane *ref, const b200_block *blocks,
                                         size_t nblocks, const b200_me_params *params, int range_x,
                                         int range_y, int step, b200_me_result *best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (int st = check_host_plane(ctx, cur)) return st;
  if (int st = check_host_plane(ctx, ref)) return st;
  B200_REQUIRE(ctx, params && blocks && best, "NULL params/blocks/best");
  size_t rb, rows;
  const size_t cur_bytes = staged_pitch(cur) * (host_plane_span(cur, &rb, &rows), rows) + 512;
  const size_t ref_bytes = staged_pitch(ref) * (host_plane_span(ref, &rb, &rows), rows) + 512;
  HostStage s(ctx, cur_bytes + ref_bytes + nblocks * (sizeof(b200_block) + sizeof(b200_me_result)) + 8 * 256);
  b200_plane dcur, dref;
  upload_host_plane(s, cur, s.take(cur_bytes), &dcur);
  upload_host_plane(s, ref, s.take(ref_bytes), &dref);
  b200_block *d_blocks = (b200_block *)s.take(nblocks * sizeof(b200_block));
  b200_me_result *d_best = (b200_me_result *)s.take(nblocks * sizeof(b200_me_result));
  s.up(d_blocks, blocks, nblocks * sizeof(b200_block));
  if (s.ok())
    s.run(b200_me_full_search_dev(ctx, &dcur, &dref, d_blocks, nblocks, params, range_x, range_y, step, d_best));
  s.down(best, d_best, nblocks * sizeof(b200_me_result));
  return s.finish(true);
}

// ------------------------------------------------------------------ per-call forms
// One block pair per call: the signature rav1e's tables expect.  Latency-bound by design
// (two tiny H2D copies + one launch + one D2H); the batched forms are the product path.
namespace {

uint32_t percall_dist(const void *org, ptrdiff_t org_stride, const void *ref, ptrdiff_t ref_stride,
                      int w, int h, int bpp, int use_satd) {
  b200_ctx *ctx = b200_default_ctx();
  b200_host_plane hc{org, org_stride, w, h, 0, bpp};
  b200_host_plane hr{ref, ref_stride, w, h, 0, bpp};
  b200_block blk{0, 0};
  b200_cand cand{0, 0, 0};
  b200_me_params p{};
  p.w = w;
  p.h = h;
  p.frame_w_in_b = 1 << 20;  // a single block pair: the mv (0,0) is always in range
  p.frame_h_in_b = 1 << 20;
  p.lambda = 0;
  p.use_satd = use_satd;
  p.bit_depth = bpp == 1 ? 8 : 10;
  uint32_t out = 0;
  b200_percall_check(ctx,
                     b200_me_candidates_batch(ctx, &hc, &hr, &blk, 1, &cand, 1, nullptr, nullptr, &p, &out, nullptr,
                                              nullptr),
                     "per-call distortion");
  return out;
}

}  // namespace

extern "C" uint32_t b200_get_sad(const void *org, ptrdiff_t org_stride, const void *ref,
                                 ptrdiff_t ref_stride, int w, int h, int bpp) {
  return percall_dist(org, org_stride, ref, ref_stride, w, h, bpp, 0);
}

extern "C" uint32_t b200_get_satd(const void *org, ptrdiff_t org_stride, const void *ref,
                                  ptrdiff_t ref_stride, int w, int h, int bpp) {
  return percall_dist(org, org_stride, ref, ref_stride, w, h, bpp, 1);
}

#define B200_DEF_DIST(W, H)                                                                   \
  extern "C" uint32_t rav1e_sad##W##x##H##_cuda(const uint8_t *src, ptrdiff_t ss,             \
                                                const uint8_t *dst, ptrdiff_t ds) {           \
    return percall_dist(src, ss, dst, ds, W, H, 1, 0);                                        \
  }                                                                                           \
  extern "C" uint32_t rav1e_sad_##W##x##H##_hbd_cuda(const uint16_t *src, ptrdiff_t ss,       \
                                                     const uint16_t *dst, ptrdiff_t ds) {     \
    return percall_dist(src, ss, dst, ds, W, H, 2, 0);                                        \
  }                                                                                           \
  extern "C" uint32_t rav1e_satd_##W##x##H##_cuda(const uint8_t *src, ptrdiff_t ss,           \
                                                  const uint8_t *dst, ptrdiff_t ds) {         \
    return percall_dist(src, ss, dst, ds, W, H, 1, 1);                                        \
  }                                                                                           \
  extern "C" uint32_t rav1e_satd_##W##x##H##_hbd_cuda(const uint16_t *src, ptrdiff_t ss,      \
                                                      const uint16_t *dst, ptrdiff_t ds,      \
                                                      uint32_t bdmax) {                       \
    (void)bdmax;                                                                              \
    return percall_dist(src, ss, dst, ds, W, H, 2, 1);                                        \
  }
B200_FOR_EACH_BLOCK_SIZE(B200_DEF_DIST)
#undef B200_DEF_DIST
