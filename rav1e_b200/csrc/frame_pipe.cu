// frame_pipe.cu — the frame-level host-buffer entry point: what an encoder thread calls once per frame
// to run the ME / transform legs of the RDO inner loop for every block of that frame.
//
// Why it exists: the per-list host-buffer forms (b200_me_mvs_resident, b200_fwd_txfm_residual_resident)
// re-send what does not change (block grid, CSR offsets), send every frame twice (once as `cur`, once as
// the next pair's `ref`), allocate per call and bounce the winners through the host between the ME and
// the transform leg.  A pipe keeps the state an encoder keeps per tile thread:
//   * two resident planes: pushing a frame uploads it ONCE (one linear copy + on-device unpack / border
//     replication, v_frame Plane::pad semantics) and the previously pushed frame becomes the reference
//     (rav1e: the reconstructed / source frame stays in the reference slots, src/encoder.rs:476-477);
//   * the block grid, the CSR offsets of the (uniform) candidate lists and every intermediate on the
//     device, allocated once;
//   * candidate lists travel as 2 bytes per candidate: (row, col) full-pel offsets relative to a
//     per-block centre MotionVector - the shape of rav1e's search stages, which evaluate a predictor plus
//     a pattern around it (me.rs:884-1303); the device expands them to MotionVectors
//     (centre + 8 * offset, i16 wrapping like the reference's MotionVector arithmetic);
//   * the winners of the SAD list feed the fused residual + forward transform (+ quantize chain) on the
//     device; only results cross PCIe: winners, coefficients (or qcoeffs + eob + tx-domain distortion).
//   * b200_frame_pipe_set_lists keeps the candidate lists on the device (a search pattern is an encoder
//     constant): a push then moves only the frame; b200_frame_pipe_push_packed returns, instead of the dense
//     coefficient block, what the entropy coder reads: coeffs[scan[0 .. eob)] of every block, packed.
// Everything is enqueued on the context's stream; with b200_ctx_set_async the call returns at once and
// the host buffers are valid after b200_ctx_synchronize, so frames pipeline over several contexts.
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include "common.cuh"

struct b200_frame_pipe {
  b200_ctx *ctx = nullptr;
  b200_frame_pipe_cfg cfg{};
  b200_plane planes[2]{};
  int cur = -1;          // index of the most recently pushed frame (-1: none yet)
  size_t nblocks = 0;
  void *dbase = nullptr;  // one allocation carved into the buffers below
  b200_block *d_blocks = nullptr;
  uint32_t *d_offs_sad = nullptr, *d_offs_satd = nullptr;
  // one staging area for everything a push sends: [frame (packed rows) | sad offsets | satd offsets |
  // centres]; inputs that lie back to back in host memory travel as ONE copy
  uint8_t *d_stage = nullptr;
  size_t frame_bytes = 0;
  int8_t *d_o8_sad = nullptr, *d_o8_satd = nullptr;
  int16_t *d_centers = nullptr;
  b200_cand *d_cand_sad = nullptr, *d_cand_satd = nullptr;
  // outputs, contiguous in this order so that host buffers laid out the same way take one copy:
  // [best_sad | best_satd | coefficients (raw, or quantized) | eob | tx_dist]
  b200_me_result *d_best_sad = nullptr, *d_best_satd = nullptr;
  void *d_coef = nullptr, *d_q = nullptr;  // d_coef is scratch when the quantize chain is on
  void *d_cout = nullptr;                  // what travels: d_coef (raw) or d_q
  uint16_t *d_eob = nullptr;
  uint64_t *d_dist = nullptr;
  size_t coef_bytes = 0, q_bytes = 0;
  // resident lists (b200_frame_pipe_set_lists) and packed output (b200_frame_pipe_push_packed)
  bool lists_resident = false, centers_resident = false;
  uint32_t *d_pack_offs = nullptr;  // [nblocks + 1] exclusive scan of eob; [nblocks] = total
  void *d_packed = nullptr;         // worst case: every coefficient of every block
  uint32_t *h_total = nullptr;      // pinned: the total, read by the host once per packed push
};

namespace {

// candidate k of block b = centre_b + 8 * (offset_row, offset_col); lists have `per` entries per block
// both lists of a push in one launch
__global__ void expand_offsets_kernel(const char2 *offs1, int per1, b200_cand *out1, const char2 *offs2, int per2,
                                      b200_cand *out2, const short2 *centers, size_t nblocks) {
  const size_t n1 = nblocks * (size_t)per1, n = n1 + nblocks * (size_t)per2;
  for (size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x; k < n; k += (size_t)gridDim.x * blockDim.x) {
    const bool first = k < n1;
    const size_t i = first ? k : k - n1;
    const size_t b = i / (size_t)(first ? per1 : per2);
    const char2 o = (first ? offs1 : offs2)[i];  // {row, col}, full pel
    short2 c = make_short2(0, 0);
    if (centers) c = centers[b];
    b200_cand r;
    r.block = (uint32_t)b;
    r.mv_row = (short)(c.x + (short)(8 * o.x));
    r.mv_col = (short)(c.y + (short)(8 * o.y));
    (first ? out1 : out2)[i] = r;
  }
}

// offs[i] = eob[0] + ... + eob[i - 1], offs[n] = total: one CTA walks the blocks 1024 at a time (a frame has
// a few thousand transform blocks; the scan is a few microseconds)
__global__ void __launch_bounds__(1024) eob_scan_kernel(const uint16_t *eob, uint32_t *offs, size_t n) {
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (size_t base = 0; base < n; base += blockDim.x) {
    const size_t i = base + threadIdx.x;
    const uint32_t v = i < n ? eob[i] : 0u;
    uint32_t x = v;  // inclusive scan inside the warp
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    if (warp == 0) {  // exclusive scan of the warp totals
      const uint32_t w = s_warp[lane];
      uint32_t z = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, z, o);
        if (lane >= o) z += y;
      }
      s_warp[lane] = z - w;
    }
    __syncthreads();
    const uint32_t excl = s_carry + s_warp[warp] + x - v;
    if (i < n) offs[i] = excl;
    __syncthreads();  // every thread has read s_carry and s_warp
    if (threadIdx.x == blockDim.x - 1) s_carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) offs[n] = s_carry;
}

// packed[offs[b] + k] = q[b * coded + scan[k]] for k < eob[b]: a warp per block
template <typename CoefT>
__global__ void __launch_bounds__(256) pack_gather_kernel(const CoefT *q, const uint16_t *eob, const uint32_t *offs,
                                                          const uint16_t *scan, int coded, size_t n, CoefT *packed) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t b = warp0; b < n; b += nwarps) {
    const int e = eob[b];
    const CoefT *src = q + b * (size_t)coded;
    CoefT *dst = packed + offs[b];
    for (int k = lane; k < e; k += 32) dst[k] = src[scan[k]];
  }
}

struct Carve {
  uint8_t *p;
  size_t used = 0;
  void *take(size_t bytes) {
    void *r = p ? p + used : nullptr;
    used += b200_align_up(bytes, 256);
    return r;
  }
};

}  // namespace

extern "C" int b200_frame_pipe_create(b200_ctx *ctx, const b200_frame_pipe_cfg *cfg, b200_frame_pipe **out) {
  B200_REQUIRE(ctx, ctx && cfg && out, "b200_frame_pipe_create: NULL argument");
  *out = nullptr;
  B200_REQUIRE(ctx, cfg->width > 0 && cfg->height > 0 && cfg->pad >= 0 && (cfg->bpp == 1 || cfg->bpp == 2),
               "bad frame geometry");
  B200_REQUIRE(ctx, (cfg->bpp == 1) == (cfg->bit_depth == 8), "bpp %d vs bit depth %d", cfg->bpp, cfg->bit_depth);
  B200_REQUIRE(ctx, cfg->block_w >= 4 && cfg->block_h >= 4 && cfg->block_w <= 128 && cfg->block_h <= 128 &&
                        cfg->block_w <= cfg->width && cfg->block_h <= cfg->height,
               "bad block size %dx%d", cfg->block_w, cfg->block_h);
  B200_REQUIRE(ctx, cfg->sad_per_block >= 0 && cfg->satd_per_block >= 0, "negative list length");
  B200_REQUIRE(ctx, cfg->tx_size < 0 || (b200_valid_av1_transform(cfg->tx_size, cfg->tx_type) &&
                                         b200_tx_width(cfg->tx_size) == cfg->block_w &&
                                         b200_tx_height(cfg->tx_size) == cfg->block_h),
               "transform %d/%d does not match the %dx%d blocks", cfg->tx_size, cfg->tx_type, cfg->block_w,
               cfg->block_h);
  // as b200_quantize_dev, here so that a bad quantizer fails before a push has enqueued anything
  B200_REQUIRE(ctx, cfg->tx_size < 0 || cfg->ac_quant == 0 ||
                        (cfg->dc_quant >= 1 && cfg->dc_quant <= 65535 && cfg->ac_quant <= 65535),
               "quantizer step sizes must be NonZeroU16 (dc %u, ac %u)", cfg->dc_quant, cfg->ac_quant);
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  b200_frame_pipe *p = new b200_frame_pipe();
  p->ctx = ctx;
  p->cfg = *cfg;
  const int nbx = cfg->width / cfg->block_w, nby = cfg->height / cfg->block_h;
  p->nblocks = (size_t)nbx * nby;
  const size_t nb = p->nblocks, ns = nb * (size_t)cfg->sad_per_block, nt = nb * (size_t)cfg->satd_per_block;
  const size_t area = (size_t)cfg->block_w * cfg->block_h;
  p->coef_bytes = cfg->tx_size >= 0 ? nb * area * (cfg->bpp == 1 ? 2 : 4) : 0;
  p->q_bytes = (cfg->tx_size >= 0 && cfg->ac_quant) ? nb * (size_t)b200_coded_tx_area(cfg->tx_size) * (cfg->bpp == 1 ? 2 : 4) : 0;
  for (int pass = 0; pass < 2; pass++) {  // pass 0 sizes the allocation, pass 1 carves it
    Carve c{(uint8_t *)p->dbase};
    p->d_blocks = (b200_block *)c.take(nb * sizeof(b200_block));
    p->d_offs_sad = (uint32_t *)c.take((nb + 1) * 4);
    p->d_offs_satd = (uint32_t *)c.take((nb + 1) * 4);
    p->frame_bytes = (size_t)cfg->width * cfg->height * cfg->bpp;
    // dense: mirrors the host layout.  It starts `lead` bytes into its carve so that the centres (read as short2)
    // are 4-aligned whatever the frame size; then the offsets (char2) are 2-aligned, 2 * ns + 2 * nt being even,
    // and an HBD frame stays 2-aligned, its frame_bytes and so `lead` being even.
    const size_t lead = (4 - (p->frame_bytes + ns * 2 + nt * 2) % 4) % 4;
    uint8_t *stage = (uint8_t *)c.take(p->frame_bytes + ns * 2 + nt * 2 + nb * 4 + 4);
    p->d_stage = stage ? stage + lead : nullptr;
    p->d_o8_sad = p->d_stage ? (int8_t *)(p->d_stage + p->frame_bytes) : nullptr;
    p->d_o8_satd = p->d_stage ? p->d_o8_sad + ns * 2 : nullptr;
    p->d_centers = p->d_stage ? (int16_t *)(p->d_o8_satd + nt * 2) : nullptr;
    p->d_cand_sad = (b200_cand *)c.take(ns * sizeof(b200_cand));
    p->d_cand_satd = (b200_cand *)c.take(nt * sizeof(b200_cand));
    const bool quant = p->q_bytes != 0;
    if (quant) p->d_coef = c.take(p->coef_bytes);  // scratch: only the quantized coefficients travel
    // dense output block (16-byte multiples keep every member aligned)
    uint8_t *ob = (uint8_t *)c.take(2 * nb * sizeof(b200_me_result) + (quant ? p->q_bytes : p->coef_bytes) + nb * 2 + 16 + nb * 8);
    p->d_best_sad = (b200_me_result *)ob;
    p->d_best_satd = ob ? p->d_best_sad + nb : nullptr;
    p->d_cout = ob ? (void *)(p->d_best_satd + nb) : nullptr;
    if (quant) p->d_q = p->d_cout; else p->d_coef = p->d_cout;
    p->d_eob = ob ? (uint16_t *)((uint8_t *)p->d_cout + (quant ? p->q_bytes : p->coef_bytes)) : nullptr;
    p->d_dist = ob ? (uint64_t *)((uint8_t *)p->d_eob + b200_align_up(nb * 2, 8)) : nullptr;
    if (quant) {
      p->d_pack_offs = (uint32_t *)c.take((nb + 1) * 4);
      p->d_packed = c.take(p->q_bytes);
    }
    if (pass == 0) {
      const cudaError_t e = cudaMalloc(&p->dbase, c.used + 256);
      if (e != cudaSuccess) {
        delete p;
        B200_CUDA(ctx, e);
      }
    }
  }
  int st = b200_plane_alloc(ctx, cfg->width, cfg->height, cfg->pad, cfg->bpp, &p->planes[0]);
  if (!st) st = b200_plane_alloc(ctx, cfg->width, cfg->height, cfg->pad, cfg->bpp, &p->planes[1]);
  if (!st) {  // the block grid and the CSR offsets never change
    std::vector<b200_block> hb(nb);
    for (int y = 0; y < nby; y++)
      for (int x = 0; x < nbx; x++) hb[(size_t)y * nbx + x] = b200_block{(int16_t)(x * cfg->block_w), (int16_t)(y * cfg->block_h)};
    std::vector<uint32_t> o1(nb + 1), o2(nb + 1);
    for (size_t i = 0; i <= nb; i++) o1[i] = (uint32_t)(i * cfg->sad_per_block), o2[i] = (uint32_t)(i * cfg->satd_per_block);
    // the alignment gap between eob and tx_dist travels with the one-copy result block: zero, not stale bytes
    const size_t gap = b200_align_up(nb * 2, 8) - nb * 2;
    if (cudaMemcpy(p->d_blocks, hb.data(), nb * sizeof(b200_block), cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(p->d_offs_sad, o1.data(), (nb + 1) * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(p->d_offs_satd, o2.data(), (nb + 1) * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
        (gap && cudaMemset((uint8_t *)p->d_eob + nb * 2, 0, gap) != cudaSuccess) ||
        cudaDeviceSynchronize() != cudaSuccess)
      st = b200_fail(ctx, B200_ERR_CUDA, "b200_frame_pipe_create: descriptor upload failed");
  }
  if (!st && p->q_bytes && cudaHostAlloc((void **)&p->h_total, 8, cudaHostAllocDefault) != cudaSuccess)
    st = b200_fail(ctx, B200_ERR_CUDA, "b200_frame_pipe_create: pinned scalar");
  if (st) {
    b200_frame_pipe_destroy(p);
    return st;
  }
  *out = p;
  return B200_OK;
}

extern "C" void b200_frame_pipe_destroy(b200_frame_pipe *p) {
  if (!p) return;
  cudaSetDevice(p->ctx->device);
  cudaStreamSynchronize(p->ctx->stream);
  for (auto &pl : p->planes)
    if (pl.alloc) cudaFree(pl.alloc);
  if (p->dbase) cudaFree(p->dbase);
  if (p->h_total) cudaFreeHost(p->h_total);
  delete p;
}

extern "C" size_t b200_frame_pipe_nblocks(const b200_frame_pipe *p) { return p ? p->nblocks : 0; }

extern "C" int b200_frame_pipe_push(b200_frame_pipe *p, const void *frame, ptrdiff_t frame_stride_bytes,
                                    const int8_t *sad_offsets, const int8_t *satd_offsets, const int16_t *centers,
                                    b200_me_result *best_sad, b200_me_result *best_satd, void *coeffs,
                                    uint16_t *eob, uint64_t *tx_dist) {
  if (!p) return b200_fail(nullptr, B200_ERR_ARG, "b200_frame_pipe_push: pipe is NULL");
  b200_ctx *ctx = p->ctx;
  const b200_frame_pipe_cfg &cfg = p->cfg;
  B200_REQUIRE(ctx, frame != nullptr, "frame is NULL");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t nb = p->nblocks, ns = nb * (size_t)cfg.sad_per_block, nt = nb * (size_t)cfg.satd_per_block;
  // ---- inputs -> the device staging area.  The frame is uploaded once (the previous one becomes the
  // reference); a dense frame followed in host memory by its lists travels as ONE copy.
  const int nxt = p->cur < 0 ? 0 : p->cur ^ 1;
  const bool first = p->cur < 0;
  const size_t row_bytes = (size_t)cfg.width * cfg.bpp;
  const bool resident = p->lists_resident && !sad_offsets && !satd_offsets && !centers;
  B200_REQUIRE(ctx, first || resident || ((ns == 0 || sad_offsets) && (nt == 0 || satd_offsets)),
               "NULL candidate offsets (and no resident lists: b200_frame_pipe_set_lists)");
  const uint8_t *fend = (const uint8_t *)frame + p->frame_bytes;
  const bool dense = (size_t)frame_stride_bytes == row_bytes;
  size_t one = 0;  // bytes covered by the first (possibly only) copy
  if (dense) {
    one = p->frame_bytes;
    if (!first && (ns == 0 || (const uint8_t *)sad_offsets == fend)) {
      one += ns * 2;
      if (nt == 0 || (const uint8_t *)satd_offsets == fend + ns * 2) {
        one += nt * 2;
        if (centers && (const uint8_t *)centers == fend + ns * 2 + nt * 2) one += nb * 4;
      }
    }
    B200_CUDA(ctx, cudaMemcpyAsync(p->d_stage, frame, one, cudaMemcpyHostToDevice, ctx->stream));
  } else {
    B200_CUDA(ctx, cudaMemcpy2DAsync(p->d_stage, row_bytes, frame, (size_t)frame_stride_bytes, row_bytes, cfg.height,
                                     cudaMemcpyHostToDevice, ctx->stream));
    one = p->frame_bytes;
  }
  if (int st = b200_plane_unpack_internal(ctx, &p->planes[nxt], p->d_stage)) return st;
  p->cur = nxt;
  if (first) {  // nothing to search against yet
    if (!ctx->async_batch) B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B200_OK;
  }
  if (!resident) {
    if (ns && one < p->frame_bytes + ns * 2)
      B200_CUDA(ctx, cudaMemcpyAsync(p->d_o8_sad, sad_offsets, ns * 2, cudaMemcpyHostToDevice, ctx->stream));
    if (nt && one < p->frame_bytes + ns * 2 + nt * 2)
      B200_CUDA(ctx, cudaMemcpyAsync(p->d_o8_satd, satd_offsets, nt * 2, cudaMemcpyHostToDevice, ctx->stream));
    if (centers && one < p->frame_bytes + ns * 2 + nt * 2 + nb * 4)
      B200_CUDA(ctx, cudaMemcpyAsync(p->d_centers, centers, nb * 4, cudaMemcpyHostToDevice, ctx->stream));
    p->lists_resident = false;  // per-push lists replace whatever was resident
  }
  const b200_plane *cur = &p->planes[nxt], *ref = &p->planes[nxt ^ 1];
  b200_me_params mp{};
  mp.w = cfg.block_w, mp.h = cfg.block_h;
  mp.frame_w_in_b = 2 * ((cfg.width + 7) >> 3);  // encoder.rs:852
  mp.frame_h_in_b = 2 * ((cfg.height + 7) >> 3);
  mp.lambda = cfg.lambda;
  mp.bit_depth = cfg.bit_depth;
  mp.window_hint_px = cfg.window_hint_px;
  if ((ns + nt) && !resident) {  // (resident lists were expanded once, by b200_frame_pipe_set_lists)
    expand_offsets_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(
        (const char2 *)p->d_o8_sad, cfg.sad_per_block, p->d_cand_sad, (const char2 *)p->d_o8_satd, cfg.satd_per_block,
        p->d_cand_satd, centers ? (const short2 *)p->d_centers : nullptr, nb);
    B200_LAUNCH_CHECK(ctx);
  }
  if (ns) {
    mp.use_satd = 0;
    if (int st = b200_me_candidates_dev(ctx, cur, ref, p->d_blocks, nb, p->d_cand_sad, ns, p->d_offs_sad, nullptr, &mp,
                                        nullptr, nullptr, p->d_best_sad))
      return st;
  }
  if (nt) {
    mp.use_satd = 1;
    if (int st = b200_me_candidates_dev(ctx, cur, ref, p->d_blocks, nb, p->d_cand_satd, nt, p->d_offs_satd, nullptr, &mp,
                                        nullptr, nullptr, p->d_best_satd))
      return st;
  }
  const bool quant = cfg.tx_size >= 0 && cfg.ac_quant;
  if (cfg.tx_size >= 0) {
    // residual of every block against the reference displaced by its SAD winner -> forward transform
    // (-> quantize chain), all on the device
    if (int st = b200_fwd_txfm_residual_dev(ctx, cur, ref, p->d_blocks, nb, ns ? p->d_best_sad : nullptr, p->d_coef,
                                            cfg.tx_size, cfg.tx_type, cfg.bit_depth))
      return st;
    if (quant)
      if (int st = b200_quantize_dev(ctx, p->d_coef, nb, cfg.tx_size, cfg.tx_type, cfg.dc_quant, cfg.ac_quant, 0,
                                     cfg.bpp == 2, p->d_q, nullptr, p->d_eob, p->d_dist))
        return st;
  }
  // ---- results -> host.  Buffers laid out like the device's output block
  // ([best_sad | best_satd | coefficients | eob | tx_dist], each directly behind the other) take one copy.
  const size_t cbytes = cfg.tx_size < 0 ? 0 : quant ? p->q_bytes : p->coef_bytes;
  const size_t rb = nb * sizeof(b200_me_result);
  const bool out_dense = ns && nt && best_sad && best_satd == best_sad + nb &&
                         (cbytes == 0 || (coeffs && (uint8_t *)coeffs == (uint8_t *)(best_satd + nb)));
  if (out_dense) {
    size_t bytes = 2 * rb + cbytes;
    if (quant && eob && (uint8_t *)eob == (uint8_t *)coeffs + cbytes) {
      bytes += nb * 2;
      eob = nullptr;  // travelled with the block
      if (tx_dist && (uint8_t *)tx_dist == (uint8_t *)coeffs + cbytes + b200_align_up(nb * 2, 8)) {
        bytes = 2 * rb + cbytes + b200_align_up(nb * 2, 8) + nb * 8;
        tx_dist = nullptr;
      }
    }
    B200_CUDA(ctx, cudaMemcpyAsync(best_sad, p->d_best_sad, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  } else {
    if (ns && best_sad) B200_CUDA(ctx, cudaMemcpyAsync(best_sad, p->d_best_sad, rb, cudaMemcpyDeviceToHost, ctx->stream));
    if (nt && best_satd) B200_CUDA(ctx, cudaMemcpyAsync(best_satd, p->d_best_satd, rb, cudaMemcpyDeviceToHost, ctx->stream));
    if (cbytes && coeffs) B200_CUDA(ctx, cudaMemcpyAsync(coeffs, p->d_cout, cbytes, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (quant && eob) B200_CUDA(ctx, cudaMemcpyAsync(eob, p->d_eob, nb * 2, cudaMemcpyDeviceToHost, ctx->stream));
  if (quant && tx_dist) B200_CUDA(ctx, cudaMemcpyAsync(tx_dist, p->d_dist, nb * 8, cudaMemcpyDeviceToHost, ctx->stream));
  if (!ctx->async_batch) B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

extern "C" int b200_frame_pipe_set_lists(b200_frame_pipe *p, const int8_t *sad_offsets, const int8_t *satd_offsets,
                                         const int16_t *centers) {
  if (!p) return b200_fail(nullptr, B200_ERR_ARG, "b200_frame_pipe_set_lists: pipe is NULL");
  b200_ctx *ctx = p->ctx;
  const b200_frame_pipe_cfg &cfg = p->cfg;
  const size_t nb = p->nblocks, ns = nb * (size_t)cfg.sad_per_block, nt = nb * (size_t)cfg.satd_per_block;
  B200_REQUIRE(ctx, (ns == 0 || sad_offsets) && (nt == 0 || satd_offsets), "NULL candidate offsets");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  if (ns) B200_CUDA(ctx, cudaMemcpyAsync(p->d_o8_sad, sad_offsets, ns * 2, cudaMemcpyHostToDevice, ctx->stream));
  if (nt) B200_CUDA(ctx, cudaMemcpyAsync(p->d_o8_satd, satd_offsets, nt * 2, cudaMemcpyHostToDevice, ctx->stream));
  if (centers) B200_CUDA(ctx, cudaMemcpyAsync(p->d_centers, centers, nb * 4, cudaMemcpyHostToDevice, ctx->stream));
  if (ns + nt) {
    expand_offsets_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(
        (const char2 *)p->d_o8_sad, cfg.sad_per_block, p->d_cand_sad, (const char2 *)p->d_o8_satd, cfg.satd_per_block,
        p->d_cand_satd, centers ? (const short2 *)p->d_centers : nullptr, nb);
    B200_LAUNCH_CHECK(ctx);
  }
  B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the host lists may be reused at once
  p->lists_resident = true;
  p->centers_resident = centers != nullptr;
  return B200_OK;
}

extern "C" int b200_frame_pipe_push_packed(b200_frame_pipe *p, const void *frame, ptrdiff_t frame_stride_bytes,
                                           b200_me_result *best_sad, b200_me_result *best_satd, uint16_t *eob,
                                           uint64_t *tx_dist, void *packed, size_t packed_capacity,
                                           size_t *packed_count) {
  if (!p) return b200_fail(nullptr, B200_ERR_ARG, "b200_frame_pipe_push_packed: pipe is NULL");
  b200_ctx *ctx = p->ctx;
  const b200_frame_pipe_cfg &cfg = p->cfg;
  B200_REQUIRE(ctx, p->q_bytes != 0, "packed output needs a quantizing pipe (tx_size >= 0 and ac_quant != 0)");
  B200_REQUIRE(ctx, p->lists_resident, "packed pushes use resident lists: call b200_frame_pipe_set_lists first");
  B200_REQUIRE(ctx, packed_count != nullptr && (packed != nullptr || packed_capacity == 0), "NULL packed buffer");
  const bool first = p->cur < 0;
  const int was_async = ctx->async_batch;
  // the frame, the kernels up to the quantize chain; nothing comes back yet
  ctx->async_batch = 1;
  const int st = b200_frame_pipe_push(p, frame, frame_stride_bytes, nullptr, nullptr, nullptr, nullptr, nullptr,
                                      nullptr, nullptr, nullptr);
  ctx->async_batch = was_async;
  if (st) return st;
  *packed_count = 0;
  if (first) {
    if (!was_async) B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B200_OK;
  }
  const size_t nb = p->nblocks;
  const int coded = b200_coded_tx_area(cfg.tx_size);
  const uint16_t *d_scan = nullptr;
  if (int s2 = b200_scan_table_internal(ctx, cfg.tx_size, cfg.tx_type, &d_scan)) return s2;
  eob_scan_kernel<<<1, 1024, 0, ctx->stream>>>(p->d_eob, p->d_pack_offs, nb);
  B200_LAUNCH_CHECK(ctx);
  const int grid = (int)std::min<size_t>((nb + 7) / 8, (size_t)ctx->num_sms * 8);
  if (cfg.bpp == 1)
    pack_gather_kernel<int16_t><<<grid, 256, 0, ctx->stream>>>((const int16_t *)p->d_q, p->d_eob, p->d_pack_offs, d_scan,
                                                               coded, nb, (int16_t *)p->d_packed);
  else
    pack_gather_kernel<int32_t><<<grid, 256, 0, ctx->stream>>>((const int32_t *)p->d_q, p->d_eob, p->d_pack_offs, d_scan,
                                                               coded, nb, (int32_t *)p->d_packed);
  B200_LAUNCH_CHECK(ctx);
  // the small fixed-size results and the total (the winners of a leg that is off are not written, as in a push)
  const size_t rb = nb * sizeof(b200_me_result);
  const bool sad_leg = cfg.sad_per_block > 0, satd_leg = cfg.satd_per_block > 0;
  if (sad_leg && satd_leg && best_sad && best_satd == best_sad + nb) {
    B200_CUDA(ctx, cudaMemcpyAsync(best_sad, p->d_best_sad, 2 * rb, cudaMemcpyDeviceToHost, ctx->stream));
  } else {
    if (sad_leg && best_sad) B200_CUDA(ctx, cudaMemcpyAsync(best_sad, p->d_best_sad, rb, cudaMemcpyDeviceToHost, ctx->stream));
    if (satd_leg && best_satd)
      B200_CUDA(ctx, cudaMemcpyAsync(best_satd, p->d_best_satd, rb, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (eob) B200_CUDA(ctx, cudaMemcpyAsync(eob, p->d_eob, nb * 2, cudaMemcpyDeviceToHost, ctx->stream));
  if (tx_dist) B200_CUDA(ctx, cudaMemcpyAsync(tx_dist, p->d_dist, nb * 8, cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(ctx, cudaMemcpyAsync(p->h_total, p->d_pack_offs + nb, 4, cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the size of the packed copy is a result
  const size_t total = *p->h_total;
  *packed_count = total;
  const size_t ncopy = std::min(total, packed_capacity);
  if (ncopy)
    B200_CUDA(ctx, cudaMemcpyAsync(packed, p->d_packed, ncopy * (cfg.bpp == 1 ? 2 : 4), cudaMemcpyDeviceToHost, ctx->stream));
  if (!was_async) B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}
