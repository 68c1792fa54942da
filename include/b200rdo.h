/*
 * b200rdo.h — C ABI of the H100-native (sm_90a) backend for rav1e's RDO inner loop.
 *
 * Drop-in boundary: rav1e selects a kernel backend per file with a `cfg_if!` module swap
 * (src/dist.rs:10-18, src/mc.rs:10-18, src/predict.rs:16-24, src/cdef.rs:20-28,
 * src/transform/forward.rs:15-23) and, inside the wrapper module, a per-CpuFeatureLevel
 * table of `unsafe extern fn` pointers (src/cpu_features/x86.rs:97-158,
 * src/asm/x86/dist/mod.rs:483-729).  This header declares what such a wrapper module
 * (`asm::cuda::*`, see INTEGRATION.md) binds:
 *
 *   (1) per-call entry points with EXACTLY the signatures of the x86 asm symbols
 *       (`rav1e_sad16x16_avx2(src, src_stride_bytes, dst, dst_stride_bytes) -> u32` ...),
 *       suffix `_cuda`, host pointers in / scalar out — so they slot into the existing
 *       SAD_FNS/SATD_FNS/... tables unchanged; and
 *   (2) batched entry points (`*_batch` = host buffers, `*_dev` = device-resident) that
 *       evaluate thousands of candidate blocks per launch — the form the north star asks
 *       for, which the reference's one-block-per-call ABI cannot express.
 *
 * Conventions (same as the asm ABI, src/asm/x86/dist/mod.rs:130-133): per-call entry
 * points take BYTE strides (ptrdiff_t); batched entry points take ELEMENT strides inside
 * b200_plane.  No torch types.  Every function returning int returns a b200_status;
 * b200_last_error() gives the message.  No entry point ever falls back to CPU code: if no
 * CUDA device is usable the call fails with B200_ERR_NODEV (per-call scalar forms abort,
 * mirroring the reference where a bad table entry is UB, not a silent wrong answer).
 */
#ifndef B200RDO_H
#define B200RDO_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200RDO_ABI_VERSION 1

typedef enum {
  B200_OK = 0,
  B200_ERR_CUDA = 1,  /* a CUDA runtime call failed */
  B200_ERR_ARG = 2,   /* precondition violated (the reference would assert!/panic) */
  B200_ERR_NODEV = 3, /* no usable CUDA device */
  B200_ERR_OOM = 4
} b200_status;

typedef struct b200_ctx b200_ctx; /* one per host thread / rayon worker (encoder.rs:3253) */

int b200_abi_version(void);
int b200_device_count(void);
int b200_ctx_create(int device, b200_ctx **out);
void b200_ctx_destroy(b200_ctx *ctx);
const char *b200_last_error(const b200_ctx *ctx); /* ctx may be NULL: global last error */
/* Enqueue on an externally owned cudaStream_t (e.g. the host framework's current stream;
 * NULL = the CUDA default stream).  b200_ctx_reset_stream returns to the ctx's own stream.
 * ORDERING CONTRACT: every `*_dev` entry point only enqueues work on the ctx's stream.  The ctx's
 * own stream is created cudaStreamNonBlocking, i.e. it does NOT synchronise with the legacy default
 * stream: device buffers a caller fills on another stream (a framework's zero-fill, an upload) must
 * be complete - or that stream must be the one given to b200_ctx_set_stream - before they are
 * handed to a `*_dev` call, and results must be read after b200_ctx_synchronize() or on the same
 * stream. */
int b200_ctx_set_stream(b200_ctx *ctx, void *cuda_stream);
int b200_ctx_reset_stream(b200_ctx *ctx);
void *b200_ctx_get_stream(b200_ctx *ctx);
int b200_ctx_synchronize(b200_ctx *ctx);
/* Asynchronous host-buffer mode: when enabled, the `*_batch` / `*_resident` entry points enqueue
 * their copies and kernels and return without waiting; output buffers are valid after
 * b200_ctx_synchronize().  Host input/output buffers must stay alive (and should be pinned) until
 * then.  Lets a caller pipeline frames over several contexts so PCIe copies overlap kernels. */
int b200_ctx_set_async(b200_ctx *ctx, int enable);
/* Number of kernels this ctx has launched since creation (bench.py's gpu_launches). */
uint64_t b200_ctx_launch_count(const b200_ctx *ctx);

/* Raw device memory helpers so non-torch hosts (the Rust shim) can keep data resident. */
int b200_malloc(b200_ctx *ctx, size_t bytes, void **dptr);
int b200_free(b200_ctx *ctx, void *dptr);
int b200_memcpy_h2d(b200_ctx *ctx, void *dptr, const void *host, size_t bytes);
int b200_memcpy_d2h(b200_ctx *ctx, void *host, const void *dptr, size_t bytes);

/* ------------------------------------------------------------------ planes
 * Device image of v_frame::Plane<T> as seen through PlaneRegion (tiling/plane_region.rs:
 * 116-135): `data` addresses pixel (0,0); [-pad, width+pad) x [-pad, height+pad) is
 * readable (frame/mod.rs:22-23 pads 88 luma px; regions may address the padding,
 * plane_region.rs:164-172). */
typedef struct {
  void *data;     /* DEVICE pointer to pixel (0,0) */
  int32_t stride; /* elements */
  int32_t width, height;
  int32_t pad; /* readable border on all four sides, pixels */
  int32_t bpp; /* bytes per pixel: 1 (u8) or 2 (u16) */
  void *alloc; /* allocation base (owned by b200_plane_alloc) */
} b200_plane;

int b200_plane_alloc(b200_ctx *ctx, int width, int height, int pad, int bpp, b200_plane *out);
int b200_plane_free(b200_ctx *ctx, b200_plane *p);
/* Upload the visible width x height area from host (row pitch host_stride_bytes) and
 * replicate edges into the padding on-device (v_frame Plane::pad semantics). */
int b200_plane_upload(b200_ctx *ctx, const b200_plane *p, const void *host,
                      ptrdiff_t host_stride_bytes);
int b200_plane_download(b200_ctx *ctx, const b200_plane *p, void *host,
                        ptrdiff_t host_stride_bytes);

/* --------------------------------------------------- SAD / SATD / ME (dist.rs, me.rs)
 * Per-call, reference-signature entry points.  Replaces rav1e_sad{W}x{H}_{sse2,avx2},
 * rav1e_satd_{W}x{H}_{ssse3,sse4,avx2} and the _hbd variants (asm/x86/dist/mod.rs:21-43,
 * tables :483-729).  22 block sizes each: see B200_FOR_EACH_BLOCK_SIZE below. */
#define B200_FOR_EACH_BLOCK_SIZE(X)                                                      \
  X(4, 4) X(4, 8) X(4, 16) X(8, 4) X(8, 8) X(8, 16) X(8, 32) X(16, 4) X(16, 8) X(16, 16) \
  X(16, 32) X(16, 64) X(32, 8) X(32, 16) X(32, 32) X(32, 64) X(64, 16) X(64, 32)         \
  X(64, 64) X(64, 128) X(128, 64) X(128, 128)

#define B200_DECL_DIST(W, H)                                                              \
  uint32_t rav1e_sad##W##x##H##_cuda(const uint8_t *src, ptrdiff_t src_stride,            \
                                     const uint8_t *dst, ptrdiff_t dst_stride);           \
  uint32_t rav1e_sad_##W##x##H##_hbd_cuda(const uint16_t *src, ptrdiff_t src_stride,      \
                                          const uint16_t *dst, ptrdiff_t dst_stride);     \
  uint32_t rav1e_satd_##W##x##H##_cuda(const uint8_t *src, ptrdiff_t src_stride,          \
                                       const uint8_t *dst, ptrdiff_t dst_stride);         \
  uint32_t rav1e_satd_##W##x##H##_hbd_cuda(const uint16_t *src, ptrdiff_t src_stride,     \
                                           const uint16_t *dst, ptrdiff_t dst_stride,     \
                                           uint32_t bdmax);
B200_FOR_EACH_BLOCK_SIZE(B200_DECL_DIST)
#undef B200_DECL_DIST

/* Generic w x h (the `rust::get_sad` fallback for non-canonical crops,
 * asm/x86/dist/mod.rs:299) — host pointers, byte strides, bpp 1|2. */
uint32_t b200_get_sad(const void *org, ptrdiff_t org_stride, const void *ref,
                      ptrdiff_t ref_stride, int w, int h, int bpp);
uint32_t b200_get_satd(const void *org, ptrdiff_t org_stride, const void *ref,
                       ptrdiff_t ref_stride, int w, int h, int bpp);

/* Batched motion-estimation distortion.  One launch = all candidates of all blocks. */
typedef struct {
  int16_t x, y; /* luma px of the block's top-left (PlaneBlockOffset << 2) */
} b200_block;

typedef struct {
  uint32_t block;         /* index into blocks[] */
  int16_t mv_row, mv_col; /* MotionVector, 1/8 pel (mc.rs:29-32); fullpel offset = mv/8 */
} b200_cand;

typedef struct {
  uint64_t cost; /* 256*sad + rate*lambda (me.rs:1460); UINT64_MAX = empty (me.rs:139-146) */
  uint32_t sad;
  int16_t mv_row, mv_col;
} b200_me_result;

typedef struct {
  int32_t w, h;                       /* block size in px (<= 128) */
  int32_t frame_w_in_b, frame_h_in_b; /* fi.w_in_b / fi.h_in_b (4x4 units), for get_mv_range */
  uint32_t lambda;                    /* me.rs:549-552 */
  int32_t allow_high_precision_mv;
  int32_t use_satd; /* 0: get_sad, 1: get_satd (me.rs:1450-1454) */
  int32_t bit_depth;
  int32_t window_hint_px; /* 0 = unknown; else bound on |mv|/8 of the candidates, used only to
                             size the shared-memory window (wrong hints cost speed, not results) */
} b200_me_params;

/* get_fullpel_mv_rd (me.rs:1386-1409) over a candidate list, device-resident.
 * d_pmv: NULL (both predictors zero) or 2 MotionVectors (row,col int16) per block.
 * d_cand_offsets: NULL, or nblocks+1 CSR offsets when cands are grouped by block in
 *   ascending block order — required for d_best (per-block first-minimum winner in list
 *   order, the serial scan's tie-break, me.rs:898,974).  A block's list holds fewer than 2^24
 *   candidates (the winner's index inside its block is packed into 24 bits).
 * Outputs (each may be NULL): d_sad[ncands], d_cost[ncands], d_best[nblocks].
 * Padding contract (the reference's, frame/mod.rs:22-23 + me.rs:339-362): candidates are accepted
 * up to get_mv_range's border, 16 + block size pixels outside the 8-aligned frame (4 * frame_w_in_b
 * x 4 * frame_h_in_b, which exceeds width x height when they are not multiples of 8), so both planes
 * must be readable that far: pad >= 4 * frame_w_in_b - width + 16 + w, and likewise for y
 * (b200_plane.pad); nothing checks it per candidate. */
int b200_me_candidates_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                           const b200_block *d_blocks, size_t nblocks, const b200_cand *d_cands,
                           size_t ncands, const uint32_t *d_cand_offsets, const int16_t *d_pmv,
                           const b200_me_params *params, uint32_t *d_sad, uint64_t *d_cost,
                           b200_me_result *d_best);

/* The same over `npairs` (cur, ref) plane pairs in ONE launch — the reference evaluates every
 * allowed reference frame of every superblock in turn (estimate_tile_motion, me.rs:178-212) and
 * runs tiles and frames concurrently; a launch per pair leaves the GPU mostly ramping up and
 * draining, so the pairs share a grid.  Blocks, candidates, offsets, pmv and the outputs are the
 * concatenation pair after pair: pair k owns blocks [pair_block_end[k-1], pair_block_end[k]) and
 * candidates [pair_cand_end[k-1], pair_cand_end[k]) (HOST arrays, npairs entries; the last entries
 * equal nblocks / ncands); b200_cand.block and d_cand_offsets index the concatenated arrays.
 * curs/refs: HOST arrays of npairs plane descriptors sharing bpp and the frame size in `params`.
 * Results are identical to npairs calls of b200_me_candidates_dev. */
int b200_me_candidates_multi_dev(b200_ctx *ctx, size_t npairs, const b200_plane *curs,
                                 const b200_plane *refs, const uint32_t *pair_block_end,
                                 const uint32_t *pair_cand_end, const b200_block *d_blocks,
                                 size_t nblocks, const b200_cand *d_cands, size_t ncands,
                                 const uint32_t *d_cand_offsets, const int16_t *d_pmv,
                                 const b200_me_params *params, uint32_t *d_sad, uint64_t *d_cost,
                                 b200_me_result *d_best);

/* The move-to-best search stages of full_pixel_me (me.rs:692-856) for every block, on the device:
 * per predictor subset get_best_predictor (:884-909) + fullpel_diamond_search (:955-998), the
 * extensive ladder's early exits (`best.rd.sad < thresh`, :777-790) and uneven_multi_hex_search
 * (:1170-1303, ends in hexagon_search :1055-1135).  The exhaustive grid that may follow
 * (:822-846) is b200_me_full_search_dev.
 *   nsubsets 1: non-extensive search, d_preds holds `subsets.all_mvs()` per block (:757-759);
 *   nsubsets 3: extensive search, subsets = {median (skipped when empty), subset_b, subset_c},
 *               d_thresh[nblocks] = the caller's `thresh` (:771-772), umh_range = 24 (:806) or 0
 *               to stop before the UMH stage.
 * d_subset_offsets: nblocks * nsubsets + 1 offsets into d_preds (b200_cand.block is ignored).
 * Predictor gathering (get_subset_predictors, :381-533) stays with the caller of this call.  For
 * encode-time motion search (estimate_motion with a pmv) use b200_estimate_motion_dev, which gathers the
 * predictors from the lookahead's stats grids on the device and adds the SATD re-measure and the sub-pel
 * stage.  A block whose candidates are all out of range (where the reference would assert) yields the
 * empty result. */
int b200_me_search_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                       const b200_block *d_blocks, size_t nblocks, const b200_cand *d_preds,
                       const uint32_t *d_subset_offsets, int nsubsets, const int16_t *d_pmv,
                       const uint32_t *d_thresh, const b200_me_params *params, int umh_range,
                       b200_me_result *d_best);
/* The same over `npairs` plane pairs in one launch (block ranges as in
 * b200_me_candidates_multi_dev; offsets, pmv, thresh and results follow the concatenated blocks). */
int b200_me_search_multi_dev(b200_ctx *ctx, size_t npairs, const b200_plane *curs,
                             const b200_plane *refs, const uint32_t *pair_block_end,
                             const b200_block *d_blocks, size_t nblocks, const b200_cand *d_preds,
                             const uint32_t *d_subset_offsets, int nsubsets, const int16_t *d_pmv,
                             const uint32_t *d_thresh, const b200_me_params *params, int umh_range,
                             b200_me_result *d_best);

/* get_subpel_mv_rd (me.rs:1411-1442) over a candidate list of SUB-PEL vectors: each candidate is
 * predicted with the 8-tap filter `filter_mode` (fi.default_filter; predict_inter_single,
 * predict.rs:304-336) and measured with SAD or SATD against the source block — the unit of work
 * of subpel_diamond_search (me.rs:1311-1383).  Same outputs and tie-break as the full-pel form. */
int b200_me_subpel_candidates_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                  const b200_block *d_blocks, size_t nblocks,
                                  const b200_cand *d_cands, size_t ncands,
                                  const uint32_t *d_cand_offsets, const int16_t *d_pmv,
                                  const b200_me_params *params, int filter_mode, uint32_t *d_sad,
                                  uint64_t *d_cost, b200_me_result *d_best);

/* Sub-pel refinement FUSED with the winner's residual and forward transform (BASELINE configs[3]): per
 * block, every candidate of its list is predicted (8-tap `filter_mode`), measured (SAD / SATD + mv cost)
 * and the first minimum kept, exactly like b200_me_subpel_candidates_dev; then the winner's prediction -
 * still in shared memory - is subtracted from the source and run through the forward transform
 * (tx_size / tx_type; block size = transform size; tx_size < 0: no transform), like
 * b200_mc_blocks_dev + b200_fwd_txfm_pred_dev would, without any prediction touching HBM.
 * Every AV1 block size from 4x4 to 64x64 (the 19 TxSize shapes: squares, 1:2 and 1:4 rectangles); any other
 * params->w x h is B200_ERR_ARG before any launch.  SATD uses 4x4 Hadamard chunks when a side is 4, 8x8
 * otherwise (get_satd).  d_cand_offsets required.  d_coeffs: nblocks x w*h (i16 for 8-bit planes, i32 for
 * HBD) in b200_fwd_txfm_pred_dev's layout for tx_size (the 32x32-chunked order when a side is 64); blocks
 * whose candidates are all out of range get zeros. */
int b200_subpel_rdo_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref, const b200_block *d_blocks,
                        size_t nblocks, const b200_cand *d_cands, size_t ncands, const uint32_t *d_cand_offsets,
                        const int16_t *d_pmv, const b200_me_params *params, int filter_mode, int tx_size,
                        int tx_type, uint32_t *d_sad, uint64_t *d_cost, b200_me_result *d_best, void *d_coeffs);

/* subpel_diamond_search (me.rs:1311-1383) for every block, the move-to-best loop on the device: starting
 * from d_start[i] (the full-pel stage's MotionSearchResult: vector, cost, sad - blocks whose start is the
 * empty result are undefined upstream, `assert!(!current.is_empty())`), the four diamond points at 1/2 pel
 * are evaluated with get_subpel_mv_rd (8-tap prediction + SAD / SATD + mv cost), the centre moves while a
 * point is strictly better, then the radius halves down to 1/4 pel (1/8 with allow_high_precision_mv).
 * d_best[i] = the final result (d_start may equal d_best); with tx_size >= 0 the final vector's prediction
 * is subtracted from the source and transformed like b200_subpel_rdo_dev does.  Same block sizes. */
int b200_subpel_search_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref, const b200_block *d_blocks,
                           size_t nblocks, const b200_me_result *d_start, const int16_t *d_pmv,
                           const b200_me_params *params, int filter_mode, int tx_size, int tx_type,
                           b200_me_result *d_best, void *d_coeffs);

/* full_search (me.rs:1464-1509) as called from full_pixel_me (me.rs:822-846) for every
 * block: window po +- (range_x, range_y) px clamped to get_mv_range, positions every
 * `step` px, pmv = 0, first-minimum winner in row-major scan order. */
int b200_me_full_search_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                            const b200_block *d_blocks, size_t nblocks,
                            const b200_me_params *params, int range_x, int range_y, int step,
                            b200_me_result *d_best);

/* Residual of every block against the reference displaced by the full-pel part of the
 * winners' motion vectors (the `diff` of encode_tx_block, encoder.rs:1533); d_mv_src may be
 * NULL (zero motion).  d_out: nblocks packed w x h int16 blocks, the input layout of
 * b200_fwd_txfm_dev with in_block_stride = w*h, in_row_stride = w. */
int b200_block_residual_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                            const b200_block *d_blocks, size_t nblocks,
                            const b200_me_result *d_mv_src, int w, int h, int16_t *d_out);

/* Host-buffer forms (what a Rust caller holding Plane<T> memory calls): planes are given
 * as host pointers to pixel (0,0) + byte strides and must be readable over the padding the
 * candidates can reach; everything is copied H2D, computed, and copied back before return. */
typedef struct {
  const void *data;    /* HOST pointer to pixel (0,0) */
  ptrdiff_t stride;    /* bytes */
  int32_t width, height;
  int32_t pad;         /* readable border present in host memory, pixels */
  int32_t bpp;
} b200_host_plane;

int b200_me_candidates_batch(b200_ctx *ctx, const b200_host_plane *cur,
                             const b200_host_plane *ref, const b200_block *blocks,
                             size_t nblocks, const b200_cand *cands, size_t ncands,
                             const uint32_t *cand_offsets, const int16_t *pmv,
                             const b200_me_params *params, uint32_t *sad, uint64_t *cost,
                             b200_me_result *best);
/* Same as b200_me_candidates_batch but with the planes already resident on the device
 * (b200_plane_alloc + b200_plane_upload once per frame, reused by every call of the frame): only
 * descriptors travel host->device and results device->host. */
int b200_me_candidates_resident(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                const b200_block *blocks, size_t nblocks, const b200_cand *cands,
                                size_t ncands, const uint32_t *cand_offsets, const int16_t *pmv,
                                const b200_me_params *params, uint32_t *sad, uint64_t *cost,
                                b200_me_result *best);
/* The same with the candidates as plain MotionVector lists: mvs[2*i] = row, mvs[2*i+1] = col of
 * candidate i (1/8 pel), the lists of consecutive blocks concatenated and delimited by
 * cand_offsets (required) — the `&[MotionVector]` a search stage holds per block, 4 bytes per
 * candidate over PCIe instead of 8. */
int b200_me_mvs_resident(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                         const b200_block *blocks, size_t nblocks, const int16_t *mvs, size_t ncands,
                         const uint32_t *cand_offsets, const int16_t *pmv,
                         const b200_me_params *params, uint32_t *sad, uint64_t *cost,
                         b200_me_result *best);
int b200_me_full_search_batch(b200_ctx *ctx, const b200_host_plane *cur,
                              const b200_host_plane *ref, const b200_block *blocks,
                              size_t nblocks, const b200_me_params *params, int range_x,
                              int range_y, int step, b200_me_result *best);

/* ---------------------------------------------------------------- RDO distortion kernels
 * get_weighted_sse (dist.rs:234-283; asm `rav1e_weighted_sse_{W}x{H}`, asm/x86/dist/sse.rs:18-35)
 * and cdef_dist_kernel (dist.rs:302-372; asm `rav1e_cdef_dist_kernel_{W}x{H}`,
 * asm/x86/dist/cdef_dist.rs:18-52) — the distortion terms of compute_distortion / sse_wxh /
 * cdef_dist_wxh (rdo.rs:142-330).
 *
 * Per-call forms: HOST pointers, BYTE strides, like the asm symbols.  `scale`: one Q14
 * DistortionScale per 4x4 chunk, rows `scale_stride_bytes` apart.  b200_cdef_dist_kernel returns
 * apply_ssim_boost(sse, svar, dvar) (activity.rs:159-186) and, when ret != NULL, the asm kernels'
 * raw triple {svar, dvar, sse}. */
uint64_t b200_weighted_sse(const void *src, ptrdiff_t src_stride, const void *dst, ptrdiff_t dst_stride,
                           const uint32_t *scale, ptrdiff_t scale_stride_bytes, int w, int h, int bpp);
uint32_t b200_cdef_dist_kernel(const void *src, ptrdiff_t src_stride, const void *dst, ptrdiff_t dst_stride,
                               int w, int h, int bit_depth, uint32_t ret[3]);
/* Batched, device-resident: block i = the w x h area at d_blocks[i] of both planes.
 * d_scale: one DistortionScale per 4x4 chunk of the PLANE (chunk (cx, cy) at
 * d_scale[cy * scale_stride + cx], entries); blocks sit on multiples of 4 pixels.
 * d_out[i] = get_weighted_sse of block i. */
int b200_weighted_sse_dev(b200_ctx *ctx, const b200_plane *src1, const b200_plane *src2,
                          const b200_block *d_blocks, size_t nblocks, int w, int h,
                          const uint32_t *d_scale, size_t scale_stride, uint64_t *d_out);
/* cdef_dist_kernel for many blocks (w, h <= 8; cdef_dist_wxh walks a block in 8x8 steps,
 * rdo.rs:152-170).  d_out[i] (may be NULL) = the boosted distortion, d_raw[3*i..] (may be NULL) =
 * {svar, dvar, sse}. */
int b200_cdef_dist_dev(b200_ctx *ctx, const b200_plane *src, const b200_plane *dst,
                       const b200_block *d_blocks, size_t nblocks, int w, int h, int bit_depth,
                       uint32_t *d_out, uint32_t *d_raw);

/* ---------------------------------------------------------------- RDO cost (rdo.rs)
 * compute_rd_cost (rdo.rs:718-723): fi.lambda.mul_add(rate as f64 / 8.0, distortion.0 as f64) - the
 * only floating-point value on the path.  Device DFMA + round-to-nearest conversions: bit-identical
 * to f64::mul_add (0 ULP; the north star allows 1).
 * Batched: d_cost[i] (may be NULL when d_best is asked for) for n (rate, distortion) pairs; with
 * d_group_offsets (ngroups + 1 CSR offsets) d_best[g] = index inside group g of its first minimum
 * (the RDO loops' strict `rd < best.rd_cost`, e.g. rdo.rs:1003-1009), 0xffffffff for an empty group. */
int b200_compute_rd_cost_dev(b200_ctx *ctx, double lambda, const uint32_t *d_rate,
                             const uint64_t *d_distortion, size_t n, const uint32_t *d_group_offsets,
                             size_t ngroups, double *d_cost, uint32_t *d_best);
/* Per-call form (host scalars in, cost out; one launch on the calling thread's context). */
double b200_compute_rd_cost(double lambda, uint32_t rate, uint64_t distortion);

/* ------------------------------------------------ forward transform (transform/forward.rs)
 * The reference has no extern-C symbol here: the boundary is the generic Rust fn
 *   forward_transform<T: Coefficient>(input: &[i16], output: &mut [MaybeUninit<T>],
 *                                     stride, tx_size: TxSize, tx_type: TxType, bd, cpu)
 * (asm/x86/transform/forward.rs:444-447).  tx_size / tx_type are the enum discriminants
 * (transform/mod.rs:56-74 and :101-123); coeff_is_i32 selects T::Coeff (0: i16 for 8-bit
 * pixels, 1: i32 for HBD).  Output order is the reference's: column-major within 32x32
 * chunks (forward.rs:135-159).  Invalid (size, type) pairs: the reference panics
 * (forward.rs:75); the status-returning forms return B200_ERR_ARG, the per-call form aborts. */
int b200_valid_av1_transform(int tx_size, int tx_type);
int b200_tx_width(int tx_size);
int b200_tx_height(int tx_size);
void b200_forward_transform(const int16_t *input, void *output, size_t stride, int tx_size,
                            int tx_type, int bd, int coeff_is_i32);
/* Batched: block i reads input[i*in_block_stride + r*in_row_stride + c] and writes
 * output[i*w*h ...].  `_dev`: device pointers, asynchronous on the ctx stream. */
int b200_fwd_txfm_dev(b200_ctx *ctx, const int16_t *d_input, size_t in_block_stride,
                      size_t in_row_stride, void *d_output, size_t nblocks, int tx_size,
                      int tx_type, int bd, int coeff_is_i32);
/* Fused residual (`diff`, encoder.rs:1533) + forward transform: block i = cur(block) minus ref
 * displaced by the full-pel part of d_mv_src[i] (NULL: zero motion).  u8 planes produce i16
 * coefficients, u16 planes i32; bd must match the planes' depth. */
int b200_fwd_txfm_residual_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                               const b200_block *d_blocks, size_t nblocks,
                               const b200_me_result *d_mv_src, void *d_output, int tx_size,
                               int tx_type, int bd);
/* The same over `npairs` plane pairs in one launch; pair k owns blocks
 * [pair_block_end[k-1], pair_block_end[k]) (HOST array) of the concatenated d_blocks / d_mv_src /
 * d_output, as in b200_me_candidates_multi_dev. */
int b200_fwd_txfm_residual_multi_dev(b200_ctx *ctx, size_t npairs, const b200_plane *curs,
                                     const b200_plane *refs, const uint32_t *pair_block_end,
                                     const b200_block *d_blocks, size_t nblocks,
                                     const b200_me_result *d_mv_src, void *d_output, int tx_size,
                                     int tx_type, int bd);
/* ActivityMask::from_plane + fill_scales (activity.rs:21-100): d_variances[by * wb + bx] =
 * variance_8x8 of luma block (bx, by), wb = ceil(width / 8), hb = ceil(height / 8) (the plane's
 * padding must cover the rounding up); d_scales (may be NULL) = ssim_boost(var, var, bit_depth),
 * the Q14 DistortionScale per importance block.  An empty plane launches nothing. */
int b200_activity_mask_dev(b200_ctx *ctx, const b200_plane *luma, int bit_depth, uint32_t *d_variances,
                           uint32_t *d_scales);

/* ---------------------------------------------------------------- frame pipe (host buffers, per frame)
 * One call per frame runs the ME and transform legs of the RDO inner loop for every block of the frame
 * with the state an encoder thread keeps per tile: pushing a frame uploads it ONCE (the previously
 * pushed frame is the reference, like the reference slots rav1e searches, me.rs:178-212), the block
 * grid and every intermediate stay on the device, candidate lists travel as 2 bytes per candidate
 * ((row, col) full-pel offsets around a per-block centre MotionVector: a search stage's pattern around
 * its predictor, me.rs:884-1303; candidate = centre + 8 * offset with i16 wrapping), the SAD winners
 * feed the fused residual + forward transform (+ quantize chain, when ac_quant != 0) on the device and
 * only results cross PCIe.  Asynchronous like the other host-buffer forms under b200_ctx_set_async:
 * host buffers (pinned for speed) are valid after b200_ctx_synchronize. */
typedef struct b200_frame_pipe b200_frame_pipe;
typedef struct {
  int32_t width, height, pad, bpp, bit_depth;
  int32_t block_w, block_h; /* the blocks tile the frame (full blocks only), row-major */
  uint32_t lambda;
  int32_t sad_per_block, satd_per_block; /* list lengths (uniform over the blocks; 0 = leg off) */
  int32_t window_hint_px;                /* bound on the offsets' reach, as in b200_me_params */
  int32_t tx_size, tx_type; /* transform of the SAD winner's residual (block size = transform size); tx_size < 0: off */
  uint32_t dc_quant, ac_quant; /* ac_quant 0: raw coefficients out; else qcoeffs + eob + tx-domain distortion */
} b200_frame_pipe_cfg;
/* Rejects with B200_ERR_ARG: a bad geometry, bpp that does not match bit_depth, a transform that is invalid or
 * not of the block size and, when the quantize chain is on (tx_size >= 0, ac_quant != 0), step sizes outside
 * 1..65535 (as b200_quantize_dev), so that a bad quantizer fails here rather than in a push. */
int b200_frame_pipe_create(b200_ctx *ctx, const b200_frame_pipe_cfg *cfg, b200_frame_pipe **out);
void b200_frame_pipe_destroy(b200_frame_pipe *pipe);
size_t b200_frame_pipe_nblocks(const b200_frame_pipe *pipe);
/* frame: HOST pointer to the visible width x height area.  sad_offsets / satd_offsets: nblocks x
 * per_block (row, col) int8 pairs; centers: nblocks (row, col) int16 MotionVectors in 1/8 pel or NULL
 * (zero).  Outputs (each may be NULL): best_sad / best_satd [nblocks]; coeffs: nblocks x w*h raw
 * coefficients, or nblocks x b200_coded_tx_area() quantized ones with eob [nblocks] and tx_dist
 * [nblocks] (i16 for 8-bit frames, i32 for HBD).  The first push only uploads (there is no reference
 * yet) and leaves the outputs untouched.
 * Copies: inputs that lie back to back in host memory in the order [frame (dense rows) | sad_offsets |
 * satd_offsets | centers] travel as ONE host->device copy, outputs laid out [best_sad | best_satd |
 * coeffs | eob | (8-byte aligned) tx_dist] as ONE device->host copy (which writes zeros into the alignment
 * gap in front of tx_dist); any other layout works with a copy per buffer, and nothing outside the
 * buffers themselves is written. */
int b200_frame_pipe_push(b200_frame_pipe *pipe, const void *frame, ptrdiff_t frame_stride_bytes,
                         const int8_t *sad_offsets, const int8_t *satd_offsets, const int16_t *centers,
                         b200_me_result *best_sad, b200_me_result *best_satd, void *coeffs, uint16_t *eob,
                         uint64_t *tx_dist);
/* Resident candidate lists.  A search stage's pattern is an encoder constant, not per-frame data: upload the
 * lists (same layout as for b200_frame_pipe_push; centers may be NULL) ONCE; the device keeps them expanded, and
 * later pushes may pass NULL for sad_offsets / satd_offsets / centers - then only the frame crosses PCIe.
 * Synchronous. */
int b200_frame_pipe_set_lists(b200_frame_pipe *pipe, const int8_t *sad_offsets, const int8_t *satd_offsets,
                              const int16_t *centers);
/* A push whose results come back PACKED: what the entropy coder reads from a transform block is
 * coeffs[scan[0 .. eob)] (src/context/block_unit.rs write_coeffs_lv_map walks the scan order up to eob), so
 * a quantizing pipe (tx_size >= 0, ac_quant != 0) with resident lists returns, per block, its eob and tx-domain
 * distortion and - block after block in `packed` - only those eob quantized coefficients in scan order
 * (i16 for 8-bit frames, i32 for HBD).  *packed_count = total number of coefficients; when it exceeds
 * packed_capacity (in coefficients) only the first packed_capacity were copied (the call still succeeds: the
 * caller retries with a larger buffer).  best_sad / best_satd / eob / tx_dist may be NULL; as in a push, the
 * winners of a leg whose list length is 0 are not written.  The call waits
 * once for the device (the size of the packed copy is a result); in asynchronous mode the packed copy itself is
 * still in flight when it returns.  The first push of a pipe only uploads: *packed_count = 0. */
int b200_frame_pipe_push_packed(b200_frame_pipe *pipe, const void *frame, ptrdiff_t frame_stride_bytes,
                                b200_me_result *best_sad, b200_me_result *best_satd, uint16_t *eob,
                                uint64_t *tx_dist, void *packed, size_t packed_capacity, size_t *packed_count);

/* ---------------------------------------------------------------- lookahead (api/lookahead.rs)
 * Plane::downsampled (v_frame 0.3.9; encoder.rs:476-477 builds the half / quarter resolution planes of
 * the ME pyramid): dst(c, r) = (src(2c, 2r) + src(2c+1, 2r) + src(2c, 2r+1) + src(2c+1, 2r+1) + 2) >> 2,
 * dst is ((src.width + 1) / 2) x ((src.height + 1) / 2), followed by Plane::pad(frame_w, frame_h):
 * everything outside [0, pad_w) x [0, pad_h) is a replica of the nearest pixel inside, with
 * pad_w = (frame_w + xdec) >> xdec, pad_h = (frame_h + ydec) >> ydec of the NEW plane (xdec = 1 for
 * the half, 2 for the quarter resolution plane).  The whole padded area of dst is written.  Both planes
 * must share bpp 1 or 2. */
int b200_plane_downsample_dev(b200_ctx *ctx, const b200_plane *src, const b200_plane *dst, int pad_w, int pad_h);
/* estimate_intra_costs (lookahead.rs:30-128): for every 8x8 importance block of the source luma,
 * get_intra_edges(DC_PRED, TX_8X8) -> DC prediction -> get_satd against the source, fused;
 * d_costs[(y / 8) * (width / 8) + x / 8].  bit_depth must be 8 (bpp 1), 10 or 12 (bpp 2); a plane
 * narrower or shorter than 8 pixels has no block and launches nothing. */
int b200_estimate_intra_costs_dev(b200_ctx *ctx, const b200_plane *luma, int bit_depth, uint32_t *d_costs);
/* The cost part of estimate_inter_costs (lookahead.rs:238-270): SATD between every importance block and
 * the reference block displaced by its motion vector (d_mvs: (row, col) int16 per importance block =
 * stats[y * 2][x * 2].mv of the reference, e.g. the winners of b200_me_search_dev) -> d_costs (may be
 * NULL) and *d_mean = sum / count as f64 (one correctly rounded division, bit-identical to the
 * reference's).  d_scratch: 8 bytes of device memory.  The reference plane must be readable wherever
 * the vectors point (padding). */
int b200_estimate_inter_costs_dev(b200_ctx *ctx, const b200_plane *org, const b200_plane *ref, const int16_t *d_mvs,
                                  uint32_t *d_costs, uint64_t *d_scratch, double *d_mean);
/* estimate_importance_block_difference (lookahead.rs:131-180): mean over the importance blocks of
 * |round(mean(org block)) - round(mean(ref block))| as f64. */
int b200_importance_block_difference_dev(b200_ctx *ctx, const b200_plane *org, const b200_plane *ref,
                                         uint64_t *d_scratch, double *d_mean);

/* ---------------------------------------------------------------- lookahead motion (me.rs:153-337)
 * compute_motion_vectors (api/lookahead.rs:271-284) -> estimate_tile_motion for every tile: the
 * three-level search (64 px blocks on the quarter, 32 px on the half, 16 px on the full resolution plane,
 * each later level refining the previous one superblock by superblock) with get_subset_predictors'
 * predictor gathering, bit-identical to the reference's serial order.  No sub-pel stage.
 *
 * A pair is one (frame, reference slot); pairs are independent and share every launch.  curs / refs:
 * HOST arrays of npairs x {full, half, quarter} planes (b200_plane_downsample_dev builds the other two),
 * all pairs the same size and bpp.  The result d_stats is npairs grids of w_in_b x h_in_b b200_me_stats,
 * row-major, w_in_b = 2 * ceil(width / 8), h_in_b = 2 * ceil(height / 8) (FrameMEStats): every cell is
 * written.  The lookahead reads it at stride 2: importance block (x, y)'s vector is cell (2x, 2y), the
 * d_mvs entry of b200_estimate_inter_costs_dev and b200_block_importances_dev; in the other direction, a
 * frame's d_stats grid is its successor's d_prev (subset C reads LAST's final stats for the same slot, in
 * frame coordinates).  d_prev: NULL, or npairs grids; has_prev: HOST flags per pair (required with d_prev).
 * Tiles: the uniform grid of tile_w_sb x tile_h_sb superblocks of TilingInfo over the 8-aligned frame, the
 * last ones cropped; predictors never cross a tile edge.
 *
 * Rejected with B200_ERR_ARG before anything is enqueued: plane sizes other than w x h, (w + 1) / 2 x
 * (h + 1) / 2 and (w + 3) / 4 x (h + 3) / 4; mixed bpp or sizes; a tile size of 0; bit_depth not 8 for
 * bpp 1 or outside 9..12 for bpp 2; me_range_scale outside 1..16; and a pad on any plane below what the mv
 * range needs.  With W8 = width rounded up to 8 and, at resolution level s (0 full, 1 half, 2 quarter),
 * bw = min(s == 0 ? 32 : 64, W8 + 2^s - 1) >> s (the widest block searched there: the refinement re-searches
 * the previous level's 64 / 32 px blocks), the pad of both level-s planes must be at least
 *   max((16 >> s) + bw, (W8 + 16) / 2^s + bw - plane width), and likewise for heights;
 * 20 / 40 / 48 px left and top on the quarter / half / full plane.
 *
 * Launches: 2 + sum over the three levels of (tbx + tby - 1), tbx x tby = the first tile's blocks at that
 * level (min(64 * tile_w_sb, W8) / block size, rounded up): one refinement launch per later level, then one
 * per tile-local anti-diagonal.  328 for a 1080p frame in one tile. */
typedef struct {
  int16_t mv_row, mv_col;  /* MEStats.mv, 1/8 pel */
  uint32_t normalized_sad; /* sad scaled to a 128x128 block */
} b200_me_stats;
typedef struct {
  int32_t bit_depth, allow_high_precision_mv;
  double me_lambda; /* fi.me_lambda; the levels' lambdas are derived as me.rs:175-176 */
  int32_t me_allow_full_search, me_range_scale;
  int32_t tile_w_sb, tile_h_sb; /* TilingInfo tile size in 64 px superblocks */
} b200_lookahead_me_params;
int b200_lookahead_motion_dev(b200_ctx *ctx, size_t npairs, const b200_plane *curs, const b200_plane *refs,
                              const b200_lookahead_me_params *p, const b200_me_stats *d_prev,
                              const uint8_t *has_prev, b200_me_stats *d_stats);

/* ---------------------------------------------------------------- encode-time motion search (me.rs:536-632)
 * estimate_motion(fi, ts, w, h, tile_bo, ref, Some(pmv), CORNER { right: true, bottom: true }, false, 0, None) as
 * inter_frame_rdo_mode_decision calls it (rdo.rs:1164-1196), for a batch of (block, reference slot) items of any
 * of the 19 block sizes 4x4 .. 64x64, in one call:
 *   - get_mv_range (me.rs:339-362) of the w x h block at frame 4x4 offset (x4, y4);
 *   - get_subset_predictors (me.rs:386-534) in CORNER mode: left, top, right and bottom neighbours and the centre
 *     from d_stats[slot] in the block's tile (tile-local offsets; the uniform grid of tile_w_sb x tile_h_sb
 *     superblocks over the 8-aligned frame, the last tiles cropped; right / bottom only inside the tile), the zero
 *     vector, and subset C from d_prev[slot] in frame coordinates when has_prev[slot]; each through process_cand
 *     (quantize_to_fullpel, then clamp to the range);
 *   - full_pixel_me's non-extensive branch over all_mvs() (get_best_predictor + fullpel_diamond_search);
 *   - with use_satd_subpel, best.rd = get_fullpel_mv_rd with SATD at best.mv (me.rs:596-616);
 *   - sub_pixel_me (me.rs:857-882): subpel_diamond_search with fi.default_filter = filter_mode, to 1/8 pel with
 *     allow_high_precision_mv, SATD or SAD by use_satd_subpel.
 * lambda = (me_lambda * 256.0 * 0.5) as u32 (me.rs:549-552).  d_out[i] = the MotionSearchResult of item i.
 *
 * Every input is final before the encode pass: both stats grids are filled by compute_motion_vectors and the
 * encode pass never writes them, so once a block's mv stack (find_mvrefs) is known its items are independent.
 * Which blocks share a call is the caller's business.
 *
 * src: the full-resolution source luma; refs: HOST array of nslots (1..7) reconstructed luma planes (fi.rec_buffer
 * slots, indexed by ref_frame.to_index()), all of src's size and bpp.  d_stats: nslots grids of this frame in
 * b200_lookahead_motion_dev's layout (its output passed unchanged); d_prev: NULL, or nslots grids of LAST's stats;
 * has_prev: HOST flags per slot, required with d_prev and only with it.  Items are grouped by block size in TxSize
 * order (4x4, 8x8, 16x16, 32x32, 64x64, 4x8, 8x4, 8x16, 16x8, 16x32, 32x16, 32x64, 64x32, 4x16, 16x4, 8x32, 32x8,
 * 16x64, 64x16): size s owns items [size_end[s-1], size_end[s]) (HOST array; size_end[18] = nitems).  One launch per
 * non-empty size group; no host synchronisation.
 *
 * Rejected with B200_ERR_ARG before anything is enqueued: nslots outside 1..7; mixed bpp or plane sizes; bit_depth
 * not 8 for bpp 1 or not 10 / 12 for bpp 2; a row pitch that is not a multiple of 4 bytes; a tile size of 0;
 * filter_mode outside 0..3; d_prev without has_prev or has_prev without d_prev; size_end decreasing or not ending
 * at nitems; and a pad on any plane below what the mv range plus the 8-tap footprint (-3 .. +4) needs.  With W8 /
 * H8 = width / height rounded up to 8, every plane's pad must be at least
 *   max(w + 19, W8 - width + w + 20, h + 19, H8 - height + h + 20)
 * for the largest w and h of the non-empty size groups (e.g. 84 for 64x64 blocks of a 1920x1080 frame).  Above that
 * pad no footprint reaches past the readable border, so PlaneSlice::clamp (predict.rs:296) never moves one.
 * An item whose slot is >= nslots or whose (x4, y4) lies outside the frame's 4x4 grid (2 * ceil(width / 8) x
 * 2 * ceil(height / 8)) gets the empty result {UINT64_MAX, UINT32_MAX, 0, 0} and reads nothing; so does an item whose
 * candidates are all out of range (never the case for a valid item: the zero vector is always in range). */
typedef struct {
  uint16_t x4, y4;   /* frame block offset in 4x4 units (PlaneBlockOffset) */
  uint8_t slot;      /* reference slot index, 0 .. nslots-1 (ref_frame.to_index()) */
  uint8_t pad_;
  int16_t pmv[2][2]; /* (row, col) of mv_stack[0].this_mv, mv_stack[1].this_mv, 1/8 pel (rdo.rs:1174-1180) */
} b200_enc_me_item;  /* 14 B */
typedef struct {
  int32_t bit_depth, allow_high_precision_mv;
  double me_lambda;         /* fi.me_lambda */
  int32_t use_satd_subpel;  /* speed_settings.motion.use_satd_subpel */
  int32_t filter_mode;      /* fi.default_filter, as b200_subpel_search_dev takes it */
  int32_t tile_w_sb, tile_h_sb;
} b200_enc_me_params;
int b200_estimate_motion_dev(b200_ctx *ctx, const b200_plane *src, size_t nslots, const b200_plane *refs,
                             const b200_me_stats *d_stats, const b200_me_stats *d_prev, const uint8_t *has_prev,
                             const b200_enc_me_params *p, const uint32_t size_end[19],
                             const b200_enc_me_item *d_items, size_t nitems, b200_me_result *d_out);

/* ---------------------------------------------------------------- temporal RDO (api/internal.rs, rdo.rs)
 * compute_block_importances (internal.rs:1075-1230): the mbtree-style propagation of block importances
 * backwards through the RDO lookahead window, then the distortion scales of the frame being coded and
 * their normalisation (compute_{spatio,}temporal_scores, encoder.rs:744-777).  Importance blocks are
 * 8x8 on the CEIL grid: w_imp = ceil(W / 8), h_imp = ceil(H / 8), n_imp = w_imp * h_imp; the intra-cost
 * maps are b200_estimate_intra_costs_dev's floor(W / 8) x floor(H / 8) maps, read flat in rows of w_imp
 * as the reference does (so only rows y < floor(n_intra / w_imp) propagate).  Results are bit-identical
 * to the reference's f32 / integer arithmetic; the one exception is stated at b200_distortion_scales_dev.
 *
 * One propagation step = update_block_importances (internal.rs:912-1071) of frame `src` into its
 * reference `dst`, `len` = the number of unique references of `src` (1..3), motion vectors = the map
 * number `mv_index` of d_mvs (me_stats[2y][2x].mv of that reference, (row, col) i16 per importance block).
 * Steps run in the order given: the reference's reverse frame order (key frames contribute none), each
 * frame's references in ref_frames order.  Rejected with B200_ERR_ARG before anything is enqueued: a
 * frame index outside the window, src == dst, len outside 1..3, and a step whose src is the dst of a
 * LATER step (its importances would not be final yet). */
typedef struct {
  uint32_t src, dst; /* frame indices inside the window */
  uint32_t len;      /* divisor: unique references of src */
  uint32_t mv_index; /* which n_imp-entry vector map of d_mvs */
} b200_imp_step;
/* frames: HOST array of nframes source luma planes (same size and bpp; padding covers the ceil grid
 * and wherever the vectors point, as for b200_estimate_inter_costs_dev); d_intra_costs: nframes x
 * floor(W/8)*floor(H/8); d_importances: nframes x n_imp f32, zeroed by the call, then propagated.
 * bit_depth must be 8 (bpp 1), 10 or 12 (bpp 2). */
int b200_block_importances_dev(b200_ctx *ctx, size_t nframes, const b200_plane *frames, int bit_depth,
                               const uint32_t *d_intra_costs, const int16_t *d_mvs, size_t nsteps,
                               const b200_imp_step *steps, float *d_importances);
/* distortion_scale_for (rdo.rs:506-553) per importance block of `frame` (only its size is read):
 * d_scales[i] = Q14 DistortionScale of pow((intra + imp) / intra, 1/3) (16384 where intra == 0 and for
 * i >= n_intra, where the reference's zip stops).  The device's double pow is within 2 ULP where glibc's
 * is within 1, so a scale can differ from the reference's only where 32768 * s lies within a few ULP of
 * an odd integer (DESIGN §2). */
int b200_distortion_scales_dev(b200_ctx *ctx, const b200_plane *frame, const float *d_importances,
                               const uint32_t *d_intra_costs, uint32_t *d_scales);
/* d_activity NULL: compute_temporal_scores (d_spatiotemporal, may be NULL, receives the scaled
 * distortion scales); else compute_spatiotemporal_scores (d_activity = the activity scales of
 * b200_activity_mask_dev; d_spatiotemporal required).  d_scales is scaled in place;
 * *d_log_isqrt_mean_scale (may be NULL) = the returned inv_mean.blog64() >> 1; d_scale4x4 (may be NULL)
 * = sse_wxh's per-4x4-chunk luma map (rdo.rs:177-224): 2*w_imp x 2*h_imp entries, rows scale4x4_stride
 * apart, ready for b200_weighted_sse_dev.  w_imp * h_imp must be below 2^30. */
int b200_temporal_scores_dev(b200_ctx *ctx, size_t w_imp, size_t h_imp, uint32_t *d_scales,
                             const uint32_t *d_activity, uint32_t *d_spatiotemporal,
                             int64_t *d_log_isqrt_mean_scale, uint32_t *d_scale4x4, size_t scale4x4_stride);

/* ---------------------------------------------------------------- segmentation (segmentation.rs, rdo.rs)
 * rav1e's adaptive quantization.  A frame step, segmentation_optimize (segmentation.rs:23-160, called at
 * encoder.rs:3776-3779 after get_initial_segmentation), fits k-means (util/kmeans.rs, k = 3..8) to the
 * binary logarithms of the frame's spatiotemporal scores and turns the centroids into per-segment q-index
 * deltas and distortion thresholds; a block step, select_segment (segmentation.rs:163-196, called per skip
 * choice at rdo.rs:855-861), places a block's spatiotemporal_scale (rdo.rs:464-504) among those thresholds.
 * Both read and write device memory only; results are bit-identical to the reference.
 *
 * b200_segmentation mirrors SegmentationState (encoder.rs:550-562) field for field (bools as 0 / 1,
 * SegLvl::SEG_LVL_ALT_Q = feature 0, threshold[] = Q14 DistortionScale) and adds:
 *   qidx[s]  get_qidx (encoder.rs:1383-1394) of segment s: clamp(base_q_idx + data[s][0], 0, 255) where
 *            features[s][0] is set (the i16 sum wraps as in a release build), else base_q_idx;
 *   status   0, or where the reference panics: 1 = update_data == 0 and no segment has ALT_Q set with
 *            data >= 1 - base_q_idx (segmentation.rs:52); 2 = update_data == 0 and the previous
 *            max_segment > 7 (update_threshold's slice).  With a non-zero status the record holds the
 *            previous state with enabled / update_map / update_data set and qidx filled; select_segment
 *            treats every item as invalid. */
typedef struct {
  uint8_t enabled, update_data, update_map, preskip;
  uint8_t last_active_segid, min_segment, max_segment, pad_;
  uint8_t features[8][8]; /* [segment][SegLvl] */
  int16_t data[8][8];     /* [segment][SegLvl] */
  uint32_t threshold[7];  /* DistortionScale, Q14 */
  uint8_t qidx[8];
  int32_t status;
} b200_segmentation; /* 240 B */
/* segmentation_optimize for one frame.  d_spatiotemporal: the w_imp x h_imp score map that
 * b200_temporal_scores_dev leaves (either form; w_imp = w_in_b / 2 on the ceil grid, as CodedFrameData),
 * read only when update_data is 1.  ac_q: HOST copy of the caller's 256-entry ac_qlookup table for
 * bit_depth (ac_qlookup_Q3 / _10_ / _12_, quantize/tables.rs); the library holds no quantizer tables.
 * update_data = (primary_ref_frame == PRIMARY_REF_NONE).  d_prev: the previous state
 * (get_initial_segmentation: the primary reference's record) or NULL for SegmentationState::default();
 * it may equal d_out.  update_data 0: min_segment search and update_threshold with the previous
 * max_segment, preskip / last_active_segid kept; 1: the k-means fit, then preskip / last_active_segid over
 * all eight segments (entries past the chosen k keep the previous state's values, as in the reference).
 * Thresholds use ac_q(base, data as i8): a delta outside -128..127 wraps there (not in data or qidx),
 * and the thresholds then need not be monotone (see b200_select_segment_dev).
 * Rejected with B200_ERR_ARG before anything is enqueued: NULL ctx / ac_q / d_out, NULL d_spatiotemporal
 * with update_data 1, a bit depth other than 8 / 10 / 12, base_q_idx outside 0..255, update_data not 0 / 1,
 * a map size of 0 or w_imp * h_imp >= 2^30, and a table with a zero or that is not strictly increasing
 * (select_qi's binary search needs it).  With update_data 1: a histogram clear (cudaMemsetAsync) and two
 * launches (the histogram, one 512-thread CTA); otherwise one launch.  Context scratch holds the histogram
 * and its prefix sums (786 KB). */
int b200_segmentation_optimize_dev(b200_ctx *ctx, const uint32_t *d_spatiotemporal, size_t w_imp, size_t h_imp,
                                   int base_q_idx, int bit_depth, const uint16_t *ac_q, int update_data,
                                   const b200_segmentation *d_prev, b200_segmentation *d_out);
/* select_segment for a batch of blocks, each with its skip choice.  Per item: skip gives 0..=0; level Full
 * gives min_segment..=max_segment; otherwise spatiotemporal_scale of the block (x0 = x >> 3,
 * x1 = min(x0 + max(w >> 3, 1), w_imp), likewise y; the u64 sum of distortion x activity over at most
 * MAX_SB_IN_IMP_B = 16 columns per row, wrapping; (sum + den / 2) / den with den = (x1 - x0)(y1 - y0) << 14,
 * truncated to u32), its segment by segment_idx_from_distortion, raised to min_segment; Complex then gives
 * sidx..=min(max_segment, sidx + 1), Simple sidx..=sidx.  segment_idx_from_distortion is
 * threshold.partition_point(|t| s < t), restated as the branchless binary search of Rust 1.83's
 * core::slice::binary_search_by (the reference's MSRV; the form since Rust 1.82): for monotone thresholds it
 * has the one answer any search has; for the non-monotone ones an i8-wrapped delta can produce it follows
 * that probe order.
 * d_scales / d_activity: the distortion and activity scale maps (w_imp x h_imp; d_activity NULL = 1 << 14
 * everywhere).  scales_off != 0: the block scale is DistortionScale::default() (rdo.rs:467-469: temporal RDO
 * off and tune not Psychovisual); the maps are then not read and may be NULL.  level: SegmentationLevel
 * discriminant 1 Simple, 2 Complex, 3 Full.  d_seg: the record of b200_segmentation_optimize_dev.
 * d_sidx: nitems x 2 (sidx_lo, sidx_hi); d_scale (may be NULL): the block's Q14 spatiotemporal_scale
 * (computed for every valid item, whatever its skip and the level).  Rejected with B200_ERR_ARG before any
 * launch: NULL ctx / d_seg / d_sidx, NULL d_items with nitems > 0, NULL d_scales unless scales_off, a level
 * outside 1..3, a map size of 0 or w_imp * h_imp >= 2^30.  An invalid item gets {255, 255} in d_sidx and
 * UINT32_MAX in d_scale, and nothing is read for it: bsize >= 22, x or y negative or not a multiple of 4,
 * x >> 3 >= w_imp or y >> 3 >= h_imp; so does every item when the record's status is non-zero.  One
 * launch, a thread per item in a grid-stride loop; nitems == 0 launches nothing. */
typedef struct {
  int16_t x, y;  /* block's top-left in the frame, luma px, multiples of 4 (frame_bo.to_luma_plane_offset) */
  uint8_t bsize; /* BlockSize 0..21 (partition.rs:130-153) */
  uint8_t skip;  /* the skip choice select_segment is called with */
  uint8_t pad_[2];
} b200_segment_item; /* 8 B */
int b200_select_segment_dev(b200_ctx *ctx, const b200_segment_item *d_items, size_t nitems,
                            const uint32_t *d_scales, const uint32_t *d_activity, size_t w_imp, size_t h_imp,
                            int scales_off, int level, const b200_segmentation *d_seg, uint8_t *d_sidx,
                            uint32_t *d_scale);

/* ---------------------------------------------------------------- quantize chain
 * The steps of encode_tx_block after the forward transform (encoder.rs:1556-1655) for nblocks
 * transform blocks of one (tx_size, tx_type), device-resident:
 *   QuantizationContext::quantize (quantize/mod.rs:269-361)  -> d_qcoeffs, d_eob
 *   dequantize (quantize/mod.rs:368-392)                     -> d_rcoeffs   (may be NULL)
 *   raw transform-domain distortion (encoder.rs:1611-1640)   -> d_tx_dist   (may be NULL)
 * d_coeffs: nblocks x (w*h) coefficients exactly as b200_fwd_txfm_* writes them (i16, or i32 when
 * coeff_is_i32); d_qcoeffs / d_rcoeffs: nblocks x b200_coded_tx_area(tx_size) (64-point dimensions
 * code 32, av1_get_coded_tx_size).  dc_quant / ac_quant are the caller's dc_q() / ac_q() of the
 * block's qindex (quantize/mod.rs:36-48; the lookup is control plane).  tx_type 0..15 (WHT_WHT is
 * lossless-only and has no scan order).  The rate estimate and the bias multiplications that
 * follow (encoder.rs:1642-1652) consume d_tx_dist on the host. */
int b200_coded_tx_area(int tx_size);
int b200_quantize_dev(b200_ctx *ctx, const void *d_coeffs, size_t nblocks, int tx_size, int tx_type,
                      uint32_t dc_quant, uint32_t ac_quant, int is_intra, int coeff_is_i32,
                      void *d_qcoeffs, void *d_rcoeffs, uint16_t *d_eob, uint64_t *d_tx_dist);

/* inverse_transform_add (transform/inverse.rs:1637-1704) for nblocks blocks of one (tx_size,
 * tx_type): dst(block i) += inverse(coefficients i), clamped to bd bits — the reconstruction step
 * of encode_tx_block (encoder.rs:1600-1609).  d_coeffs: b200_coded_tx_area(tx_size) coefficients
 * per block in the forward transform's layout (i16 for 8-bit planes, i32 for HBD), e.g. the
 * d_rcoeffs of b200_quantize_dev.  Blocks of one call must not overlap.  tx_type 0..16; pairs the
 * reference leaves `unimplemented!()` (INV_TXFM_FNS :1593-1623) are rejected. */
int b200_inverse_transform_add_dev(b200_ctx *ctx, const void *d_coeffs, const b200_plane *dst,
                                   const b200_block *d_blocks, size_t nblocks, int tx_size, int tx_type,
                                   int bd);

/* encode_tx_block's numeric core (encoder.rs:1492-1655) for nblocks transform blocks in ONE kernel - the
 * coefficients of a block stay in shared memory from the forward transform to the reconstruction:
 * residual against `ref` displaced by d_mv_src (NULL: zero motion) -> forward transform -> quantize ->
 * dequantize -> raw tx-domain distortion, and, when need_recon_pixel, the inverse transform added into
 * `rec` (which must already hold the prediction in the blocks' areas).
 * d_qcoeffs: nblocks x b200_coded_tx_area(tx_size) (required; i16, or i32 for HBD).  Optional outputs (each
 * may be NULL): d_coeffs nblocks x w*h raw coefficients, d_rcoeffs dequantized ones (coded area), d_eob,
 * d_tx_dist.  Entropy coding of d_qcoeffs and the rate / bias terms stay with the caller.  Results are
 * identical to b200_fwd_txfm_residual_dev + b200_quantize_dev + b200_inverse_transform_add_dev. */
int b200_encode_tx_blocks_dev(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                              const b200_plane *rec, const b200_block *d_blocks, size_t nblocks,
                              const b200_me_result *d_mv_src, int tx_size, int tx_type, int bd,
                              uint32_t dc_quant, uint32_t ac_quant, int is_intra, int need_recon_pixel,
                              void *d_coeffs, void *d_qcoeffs, void *d_rcoeffs, uint16_t *d_eob,
                              uint64_t *d_tx_dist);

/* ---------------------------------------------------------------- coefficient rate
 * The rate term of every transform candidate: what rav1e's WriterCounter reports for the symbols
 * write_coeffs_lv_map (context/block_unit.rs:1783-2016) codes, counted from a CDF snapshot the caller
 * provides.  One CHAIN is the ordered list of transform blocks one write_tx_blocks / write_tx_tree call
 * (or one plane of it) writes through one writer; its items share the writer state (rng), the adapting
 * CDFs and a window of coefficient contexts.  Per item, in the reference's symbol order:
 *   txb_skip (get_txb_ctx :442-526) -> eob 0 ends the item with cul_level 0;
 *   write_tx_type (transform_unit.rs:530-574, luma only) -> encode_eob -> encode_coeffs (reverse scan,
 *   the base symbol then its br loop) -> encode_coeff_signs (forward: dc_sign, bypass sign bits,
 *   write_golomb) -> set_coeff_context (:333-348) writes cul_level over the tx block's width_mi /
 *   height_mi window entries.
 * Every symbol_with_update adapts the chain's private copy of its snapshot (update_cdf, ec.rs:935-955);
 * nothing is written back.  d_rate[c] = tell_frac(end) - tell_frac(start) in 1/8 bit (OD_BITRES 3) of a
 * counter whose rng is chain.init_rng at the start (0x8000 for WriterCounter::new(); a writer that has
 * already coded mode symbols passes its rng and gets the exact increment, since frac_compute is linear
 * in the bit count).  It plugs into b200_compute_rd_cost_dev's d_rate unchanged.
 *
 * b200_coeff_cdfs holds the coefficient and tx-type fields of CDFContext (context/cdf_context.rs:28-93)
 * with rav1e's array shapes and element form: u16 inverse CDFs, N slots for N symbols, the adaptation
 * count in the last slot.  The Rust side copies the fields across unchanged.
 *
 * Rules of one call:
 *  - d_qcoeffs: ncoeffs coefficients, i16 or i32 (coeff_is_i32), holding coded blocks in the layout
 *    b200_quantize_dev / b200_encode_tx_blocks_dev write.  An item's block starts at coefficient
 *    item.block * b200_coded_tx_area(item.tx_size): the d_qcoeffs of one such call for the item's size.
 *    The levels and contexts read the whole coded block (txb_init_levels), not only its first eob.
 *  - The scan is av1_scan_orders[tx_size][tx_type] (the context's tables, as b200_quantize_dev).
 *  - Window: above[plane][x4 ..] / left[plane][y4 ..] are the entries get_txb_ctx reads
 *    (clip_w4 / clip_h4 of them) and set_coeff_context writes (width_mi / height_mi of them).  An
 *    entry's sign field (bits 6-7) of 3, which set_coeff_context never writes, counts as no sign.
 * A chain is INVALID - d_rate[c] = UINT32_MAX, no symbol counted, its items' d_cul_level untouched -
 * when its snapshot >= ncdfs, init_rng outside 32768..65535, its item range leaves [0, nitems), or any
 * item has: tx_size >= 19; tx_type >= 16 (WHT_WHT has no scan); plane > 2; plane_bsize >= 22; mode > 33
 * (NEW_NEWMV), or UV_CFL_PRED (13) on luma; a block reaching past ncoeffs; eob > the coded area; eob > 0 with a zero
 * coefficient at scan[eob - 1] (get_eob_pos_token would underflow); a coefficient of the coded block equal
 * to INT16_MIN / INT32_MIN (whose abs() overflows); a luma tx_type its set does not use when eob > 0 and
 * the set has more than one type (write_tx_type asserts); clip_w4 or clip_h4 of 0; or x4 + max(width_mi,
 * clip_w4) > 16 or y4 + max(height_mi, clip_h4) > 16.
 * Rejected with B200_ERR_ARG before any launch, outputs untouched: NULL ctx; nchains > 0 with NULL
 * d_chains / d_cdfs / d_rate; nitems > 0 with NULL d_items or d_qcoeffs; ncdfs == 0 with nchains > 0;
 * coeff_is_i32 not 0 / 1; nchains or nitems >= 2^31.  d_cul_level may be NULL: else
 * d_cul_level[i] is the byte set_coeff_context wrote for item i (0 for eob 0), for the caller to commit
 * for the candidate it keeps.  Inputs are only read. */
typedef struct {
  uint16_t txb_skip[5][13][2];
  uint16_t dc_sign[2][3][2];
  uint16_t eob_extra[5][2][9][2];
  uint16_t eob_flag16[2][2][5];
  uint16_t eob_flag32[2][2][6];
  uint16_t eob_flag64[2][2][7];
  uint16_t eob_flag128[2][2][8];
  uint16_t eob_flag256[2][2][9];
  uint16_t eob_flag512[2][2][10];
  uint16_t eob_flag1024[2][2][11];
  uint16_t coeff_base_eob[5][2][4][3];
  uint16_t coeff_base[5][2][42][4];
  uint16_t coeff_br[5][2][21][4];
  uint16_t intra_tx_1[4][13][7];
  uint16_t intra_tx_2[4][13][5];
  uint16_t inter_tx_1[4][16];
  uint16_t inter_tx_2[4][12];
  uint16_t inter_tx_3[4][2];
} b200_coeff_cdfs; /* 3930 x u16 = 7860 B */
typedef struct {
  uint32_t snapshot;   /* index into d_cdfs */
  uint32_t init_rng;   /* the counter's rng when the chain starts, 32768..65535 */
  uint32_t item_begin; /* the chain's items are d_items[item_begin .. item_begin + item_count) */
  uint32_t item_count;
  uint8_t above[3][16]; /* above_coeff_context window per plane, 4-px units of that plane */
  uint8_t left[3][16];  /* left_coeff_context window per plane */
} b200_coeff_chain;     /* 112 B */
typedef struct {
  uint32_t block;     /* coded block index in d_qcoeffs */
  uint16_t eob;       /* 0 ..= coded area */
  uint8_t tx_size;    /* TxSize 0..18 */
  uint8_t tx_type;    /* TxType 0..15 */
  uint8_t plane;      /* 0..2 */
  uint8_t plane_bsize; /* BlockSize 0..21 of the block in this plane */
  uint8_t mode;       /* PredictionMode 0..33: inter when >= NEARESTMV (14); the intra direction for luma */
  uint8_t reduced_tx_set;
  uint8_t x4, y4;     /* the tx block's first above / left entry in the chain's window */
  uint8_t clip_w4, clip_h4; /* frame_clipped_txw >> 2, frame_clipped_txh >> 2 (encoder.rs:1561-1566) */
} b200_coeff_item; /* 16 B */
int b200_coeff_rate_dev(b200_ctx *ctx, const b200_coeff_cdfs *d_cdfs, size_t ncdfs, const b200_coeff_chain *d_chains,
                        size_t nchains, const b200_coeff_item *d_items, size_t nitems, const void *d_qcoeffs,
                        size_t ncoeffs, int coeff_is_i32, uint32_t *d_rate, uint8_t *d_cul_level);

/* ---------------------------------------------------------------- intra transform size and type decision
 * rdo_tx_size_type (rdo.rs:725-802) for intra luma modes with rdo_tx_decision on (speeds 0-5; that setting
 * is also tx_mode_select, so the size ladder always runs), with rdo_tx_type_decision (rdo.rs:1701-1823) and
 * write_tx_blocks' luma loop (encoder.rs:2243-2311 -> encode_tx_block :1404-1658), for a batch of items of
 * one PlaneRegion (tile).  An item is what luma_chroma_mode_rdo / encode_block call it with: a block, a luma
 * mode and the quantizers of one segment.  Per item:
 *  - Size ladder: max_txsize_rect_lookup[bsize], then sub_tx_size_map twice, stopping where the size no
 *    longer changes.  Per size, the types are RAV1E_TX_TYPES (DCT_DCT, ADST_DCT, DCT_ADST, ADST_ADST, IDTX,
 *    V_DCT, H_DCT) that av1_tx_used[get_tx_set(size, intra, reduced_tx_set)] keeps; DCT_DCT only for
 *    TX_SET_DCTONLY or a skip item.  A skip item still codes its coefficients (the reference passes
 *    skip = false to write_tx_blocks).
 *  - One candidate (size, type) starts from the item's coefficient-context checkpoint (its above / left
 *    windows, a private copy of CDF snapshot d_cdfs[snapshot], a WriterCounter at rng 0x8000) and walks the
 *    size's transform blocks in raster order, skipping a block whose first 4x4 lies at or past the region's
 *    4x4 extent (ceil(rect_w / 4) x ceil(rect_h / 4)).  Per transform block: get_intra_edges at (bx, by)
 *    (pixels inside the partition from this candidate's own reconstruction, others from rec),
 *    predict_intra (angle delta 0, the item's ief, PredictionVariant and the PAETH remap from the transform
 *    block's tile-relative position), the residual against src (zero when the block is invisible in the
 *    frame), forward_transform, quantize, write_coeffs_lv_map counted with frame_clipped_txw / txh,
 *    dequantize, inverse_transform_add when eob > 0 and (the size is not the block's or the distortion is
 *    pixel-domain), and the tx-domain distortion.
 *  - Distortion (dist_mode): 0 = tx-domain (Tune::Psnr with tx_domain_distortion): per visible transform
 *    block its rounded raw distortion times distortion_scale at the block times dist_scale; 1 = sse_wxh
 *    (Tune::Psnr) and 2 = cdef_dist_wxh (Tune::Psychovisual) over the block's visible area
 *    (clip_visible_bsize), each chunk times its distortion_scale, the sum times dist_scale.  dist_scale is
 *    fi.dist_scale[0] (Q14 DistortionScale); d_scale4x4 the per-4x4 luma map b200_weighted_sse_dev takes,
 *    addressed by frame 4x4 position with scale_stride entries per row; NULL means every distortion_scale is
 *    the default (temporal RDO off).
 *  - Cost: rd = compute_rd_cost(lambda, rate, distortion) (f64 fma, as b200_compute_rd_cost_dev).
 *  - Decision, exactly the reference's: within a size, a first type whose rd > the best rd so far ends the
 *    size, which then contributes (DCT_DCT, f64::MAX) while the ladder continues; a type replaces the size's
 *    best only if its rd is strictly less; a size replaces the best only if its rd is strictly less (ties
 *    keep the larger size).
 * Every candidate starts from the same checkpoint, so the call evaluates them in parallel and applies the
 * rules afterwards.  rec is only read: as with b200_cfl_alpha_dev, the caller re-encodes the candidate it
 * keeps.  What may share a call is the caller's business: each block's neighbours must be final in rec.
 *
 * frame_width / frame_height are fi.width / fi.height (clip_visible_bsize, w_in_b / h_in_b).  Outputs:
 * d_best[i] = the best (tx_size, tx_type) and its rd; d_cands (may be NULL) nitems x 21 records
 * [item][level * 7 + position in RAV1E_TX_TYPES]: rate (1/8 bit), scaled distortion and rd of every
 * candidate the reference evaluates, and only the state for the others.
 * An INVALID item gets {rd -1.0, tx_size 0xFF, tx_type 0xFF} and 21 records of state B200_TX_INVALID, and
 * nothing is read for it: bsize >= 22 or of the 128 class (13 / 14 / 15), mode >= 13, (x, y) outside the
 * region or not a multiple of 4, dc_quant or ac_quant outside 1 .. 65535, snapshot >= ncdfs.  (The 16-entry
 * context windows cover every block up to 64x64, so no window can overflow.)
 * Rejected with B200_ERR_ARG before any launch, outputs untouched: NULL ctx or planes; a bit depth other
 * than 8 / 10 / 12 or a bpp that does not match it; rec and src of different sizes; a region outside the
 * plane or past the frame's 4x4 blocks (4 * w_in_b); a frame larger than the plane; rec->pad or src->pad
 * below 64 (encode_tx_block's diff reads the whole transform block past the visible frame); dist_mode
 * outside 0 .. 2; reduced_tx_set not 0 / 1; lambda negative or not finite; a scale map whose stride is below
 * w_in_b; nitems >= 2^30; with nitems > 0, NULL d_items / d_best / d_cdfs or ncdfs == 0.  nitems == 0
 * launches nothing.  Context scratch holds the per-size lists (and the records when d_cands is NULL). */
typedef struct {
  int16_t x, y;       /* block's top-left inside the region, luma px, multiples of 4 */
  uint8_t bsize;      /* BlockSize 0..21 without the 128 class */
  uint8_t mode;       /* luma PredictionMode 0..12 */
  int8_t ief;         /* -1: enable_intra_edge_filter off; else IntraEdgeFilterParameters::use_smooth_filter() */
  uint8_t skip;       /* the skip choice the block is evaluated with */
  uint32_t dc_quant;  /* dc_q / ac_q of get_qidx's qindex, 1..65535 */
  uint32_t ac_quant;
  uint32_t snapshot;  /* index into d_cdfs: the CDFs at the block's checkpoint */
  uint8_t above[16];  /* luma above / left coefficient contexts from the block's first 4x4 */
  uint8_t left[16];
} b200_tx_item; /* 52 B */
typedef struct {
  double rd;
  uint8_t tx_size, tx_type; /* TxSize / TxType discriminants */
  uint8_t pad_[6];
} b200_tx_best; /* 16 B */
#define B200_TX_EVALUATED 0
#define B200_TX_NOT_IN_SET 1    /* av1_tx_used or the DCT-only rule leaves the type out */
#define B200_TX_CUT 2           /* after the size's first type lost to the best size so far */
#define B200_TX_NOT_IN_LADDER 3 /* the ladder stopped before this level */
#define B200_TX_INVALID 255
typedef struct {
  double rd;
  uint64_t dist;  /* ScaledDistortion */
  uint32_t rate;  /* 1/8 bit */
  uint32_t state; /* B200_TX_*; rate / dist / rd are 0 unless EVALUATED */
} b200_tx_cand; /* 24 B */
int b200_intra_tx_size_type_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src, int rect_x, int rect_y,
                                int rect_w, int rect_h, int frame_width, int frame_height, int bit_depth,
                                int dist_mode, int reduced_tx_set, double lambda, uint32_t dist_scale,
                                const uint32_t *d_scale4x4, size_t scale_stride, const b200_coeff_cdfs *d_cdfs,
                                size_t ncdfs, const b200_tx_item *d_items, size_t nitems, b200_tx_best *d_best,
                                b200_tx_cand *d_cands);

/* Fused residual + transform with resident planes and HOST descriptors / outputs. */
int b200_fwd_txfm_residual_resident(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref,
                                    const b200_block *blocks, size_t nblocks,
                                    const b200_me_result *mv_src, void *output, int tx_size,
                                    int tx_type, int bd);
/* Residual against PACKED predictions (nblocks x h x w pixels, the output of b200_mc_blocks_dev or
 * b200_predict_intra_dev) + forward transform: predict -> diff -> forward_transform of
 * encode_tx_block (encoder.rs:1492-1544) without the residual touching HBM. */
int b200_fwd_txfm_pred_dev(b200_ctx *ctx, const b200_plane *cur, const void *d_pred,
                           const b200_block *d_blocks, size_t nblocks, void *d_output, int tx_size,
                           int tx_type, int bd);
int b200_fwd_txfm_batch(b200_ctx *ctx, const int16_t *input, size_t in_block_stride,
                        size_t in_row_stride, void *output, size_t nblocks, int tx_size,
                        int tx_type, int bd, int coeff_is_i32);

/* ------------------------------------------------ motion compensation (mc.rs, predict.rs)
 * Per-call forms: the argument order of the dav1d-style symbols rav1e binds
 * (`rav1e_put_8tap_regular_smooth_8bpc_avx2(dst, dst_stride, src, src_stride, w, h, mx, my)`,
 * asm/x86/mc.rs:17-76, table index (fx + 4*fy)&15 :80-82) with the filter pair passed as
 * arguments instead of being baked into the symbol name.  Host pointers, BYTE strides; src must
 * be readable over [-3, w+4) x [-3, h+4) (asm/x86/mc.rs:122-123).  FilterMode: 0 REGULAR,
 * 1 SMOOTH, 2 SHARP, 3 BILINEAR (mc.rs:98-106).  Preconditions as the reference asserts
 * (mc.rs:256-257): even height, power-of-two width in 2..128; violations abort. */
void b200_put_8tap(void *dst, ptrdiff_t dst_stride, const void *src, ptrdiff_t src_stride, int w,
                   int h, int col_frac, int row_frac, int mode_x, int mode_y, int bit_depth);
void b200_prep_8tap(int16_t *tmp, const void *src, ptrdiff_t src_stride, int w, int h,
                    int col_frac, int row_frac, int mode_x, int mode_y, int bit_depth);
void b200_mc_avg(void *dst, ptrdiff_t dst_stride, const int16_t *tmp1, const int16_t *tmp2, int w,
                 int h, int bit_depth);
/* Batched predict_inter_single (predict.rs:304-336): block i is predicted from `ref` at
 * d_blocks[i] displaced by d_mvs[2i] (row), d_mvs[2i+1] (col) in 1/8 pel through get_mv_params
 * (predict.rs:284-297; xdec/ydec = plane decimation).  kind 0 = put (packed w*h pixels per block),
 * kind 1 = prep (packed w*h int16 per block, for b200_mc_avg_dev). */
int b200_mc_blocks_dev(b200_ctx *ctx, const b200_plane *ref, const b200_block *d_blocks,
                       const int16_t *d_mvs, size_t nblocks, int w, int h, int mode_x, int mode_y,
                       int bit_depth, int xdec, int ydec, int kind, void *d_out);
int b200_mc_avg_dev(b200_ctx *ctx, const int16_t *d_tmp1, const int16_t *d_tmp2, void *d_dst,
                    size_t nblocks, int w, int h, int bit_depth);

/* ------------------------------------------------------------------ CDEF (cdef.rs)
 * Per-call forms with the asm signatures rav1e binds (asm/x86/cdef.rs:16-37, :184-191):
 *   rav1e_cdef_dir_{8,16}bpc(img, stride_bytes, &var[, bitdepth_max]) -> dir
 *   rav1e_cdef_filter_{4x4,4x8,8x8}(dst, dst_stride, tmp_u16, tmp_stride, pri, sec, dir, damping)
 * `tmp` addresses the block's top-left inside the caller-built padded u16 tile (2 px border,
 * CDEF_VERY_LARGE = 0x8000 where pixels are unavailable, cdef.rs:161-194); strides in BYTES. */
int32_t b200_cdef_dir(const void *img, ptrdiff_t stride, uint32_t *var, int bit_depth);
void b200_cdef_filter_block(void *dst, ptrdiff_t dst_stride, const uint16_t *tmp,
                            ptrdiff_t tmp_stride, int pri_strength, int sec_strength, int dir,
                            int damping, int bit_depth, int xdec, int ydec);
/* Frame-level batch = cdef_filter_tile (cdef.rs:597-625) with the tile rect equal to the frame.
 * b200_cdef_find_dir_dev: cdef_analyze_superblock for every 8x8 luma block (d_skip8: one byte
 * per 8x8 block = AND of its four 4x4 `skip` flags, row-major, may be NULL); writes dir/var
 * (0 where skipped).  b200_cdef_filter_plane_dev: cdef_filter_superblock for one plane; `in`
 * and `out` are distinct planes of the same geometry; d_strength_sb holds the 6-bit strength
 * (pri*4+sec; fi.cdef_y_strengths / cdef_uv_strengths[cdef_index]) per 64x64 superblock,
 * row-major with ceil(luma_width/64) entries per row; damping = fi.cdef_damping. */
int b200_cdef_find_dir_dev(b200_ctx *ctx, const b200_plane *luma, int bit_depth,
                           const uint8_t *d_skip8, uint8_t *d_dir, int32_t *d_var);
int b200_cdef_filter_plane_dev(b200_ctx *ctx, const b200_plane *in, const b200_plane *out,
                               int plane, int xdec, int ydec, int luma_width, int luma_height,
                               int bit_depth, int damping, const uint8_t *d_skip8,
                               const uint8_t *d_dir, const int32_t *d_var,
                               const uint8_t *d_strength_sb);

/* The same restricted to the luma 8x8 blocks [rx8, rx8 + rw8) x [ry8, ry8 + rh8) of the frame (a tile of
 * cdef_filter_tile, cdef.rs:597-625: tiles run concurrently, taps still read across tile borders and
 * see the sentinel only outside the FRAME); dir / var / skip / strength arrays stay frame-indexed. */
int b200_cdef_find_dir_rect_dev(b200_ctx *ctx, const b200_plane *luma, int bit_depth, const uint8_t *d_skip8,
                                uint8_t *d_dir, int32_t *d_var, int rx8, int ry8, int rw8, int rh8);
int b200_cdef_filter_rect_dev(b200_ctx *ctx, const b200_plane *in, const b200_plane *out, int plane, int xdec,
                              int ydec, int luma_width, int luma_height, int bit_depth, int damping,
                              const uint8_t *d_skip8, const uint8_t *d_dir, const int32_t *d_var,
                              const uint8_t *d_strength_sb, int rx8, int ry8, int rw8, int rh8);

/* Many (plane, tile) items per call - the tiles a rank owns across the frames of a batch - served by
 * as few launches as possible (32 items per launch): with find_dir the directions / variances of every
 * item's blocks are (re)computed from `in` (luma only), with filter every item's rect of `in` is
 * filtered into `out`.  `items` is a HOST array; the arrays an item points to are frame-indexed.
 * This call and the four above check every argument and every item before the first launch, and
 * reject with B200_ERR_ARG (nothing launched, nothing written): a luma size that is not a positive
 * multiple of 8, a bit depth other than 8 / 10 / 12, a chroma layout other than 4:4:4 / 4:2:2 / 4:2:0,
 * plane 0 with xdec or ydec set, find_dir on a chroma plane; with filter, damping outside 3..6
 * (fi.cdef_damping) or NULL strengths; per item, a NULL in / dir / var, an `in` (or with filter `out`)
 * whose bpp does not match the bit depth or that is smaller than (luma_width >> xdec) x
 * (luma_height >> ydec) or has a stride below its width, with filter an `out` that is NULL or is `in`,
 * and a rect outside the luma 8x8 grid.  nitems == 0 launches nothing. */
typedef struct {
  const b200_plane *in, *out; /* out may be NULL when only the directions are wanted */
  const uint8_t *d_skip8;     /* may be NULL */
  uint8_t *d_dir;
  int32_t *d_var;
  int32_t rx8, ry8, rw8, rh8; /* the tile in 8x8 luma blocks */
} b200_cdef_item;
int b200_cdef_tiles_dev(b200_ctx *ctx, const b200_cdef_item *items, size_t nitems, int plane, int xdec, int ydec,
                        int luma_width, int luma_height, int bit_depth, int damping, const uint8_t *d_strength_sb,
                        int find_dir, int filter);

/* The CDEF pass of rdo_loop_decision (rdo.rs:2104-2567; the RestorationFilter::None and no-LRU branches,
 * i.e. the whole first pass and every pass when restoration is off) for many loop-restoration areas in one
 * asynchronous call on the context's stream, without host synchronisation.  Per area the reference takes a
 * scratch copy of the area cropped to the visible frame and rounded up to 8 (rdo.rs:2152-2157, 2277-2284),
 * so CDEF's edge flags treat everything outside the AREA as unavailable, even where the frame continues.
 * For each superblock of an area that has a coded 8x8 block (rdo.rs:2185-2205) and each cdef index
 * 0 .. 1 << cdef_bits: cdef_filter_superblock with that index's strengths (skipped 8x8 blocks copied), then
 * rdo_loop_plane_error per plane (luma cdef_dist_kernel 8x8 times the 8x8 block's frame-absolute
 * distortion_scale; chroma sse_wxh with that bias per 4x4 chunk; the plane's sum times dist_scale[p]),
 * summed over planes; then compute_rd_cost (an fma in f64) with the slot's rate; the first minimum wins.
 *
 * rec / src / out: HOST arrays of `planes` (1 = 4:0:0, or 3) frame planes: the deblocked reconstruction,
 * the input, and (out may be NULL) the area's CDEF output after the pass, written over each area's scratch
 * rect only: the winner's filter output for decided superblocks, a copy of rec for CDEF-skipped ones.
 * Planes cover at least the frame rounded up to 8 luma pixels; out must not alias rec.
 * frame_width / frame_height = fi.width / fi.height.  d_skip8: one byte per 8x8 luma block of the frame
 * (AND of its four 4x4 skips), ceil(W/8) per row, as b200_cdef_find_dir_dev; NULL = none skipped.
 * d_imp_scales: the Q14 distortion scale per 8x8 importance block (b200_distortion_scales_dev's ceil
 * grid); NULL = the default scale (no temporal RDO).  dist_scale = fi.dist_scale (Q14, host).
 * areas: HOST array; slot area * 16 + sby * 4 + sbx addresses a superblock inside its area.
 * d_rate: one rate (1/8 bit) per slot, NULL = 0.  Outputs per slot: d_err[slot * 8 + i] (ScaledDistortion
 * summed over planes) and d_cost[slot * 8 + i] for i < 1 << cdef_bits, written for decided superblocks
 * only; d_best[slot] = the winning index, or -1 for a CDEF-skipped superblock.  Slots outside an area are
 * not written.  Rejected with B200_ERR_ARG before any launch: NULL pointers, a bpp that does not match
 * bit_depth (8 / 10 / 12), planes other than 1 / 3, a chroma layout other than 4:2:0 / 4:2:2 / 4:4:4,
 * cdef_bits outside 0..3, a used strength above 63, damping outside 3..6 (fi.cdef_damping =
 * 3 + (base_q_idx >> 6)), planes smaller than the frame, areas outside the frame, larger than 4x4
 * superblocks or overlapping each other, out aliasing rec.  n_areas == 0 launches nothing. */
typedef struct {
  int32_t sbx, sby;   /* frame-absolute superblock of the area's top-left (tile sbo + base_sbo) */
  int32_t sb_w, sb_h; /* 1..4 each, already trimmed to the tile as rdo.rs:2146-2147 does */
} b200_cdef_rdo_area;
int b200_cdef_rdo_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src, const b200_plane *out, int planes,
                      int xdec, int ydec, int frame_width, int frame_height, int bit_depth, int damping, int cdef_bits,
                      const uint8_t y_strengths[8], const uint8_t uv_strengths[8], const uint8_t *d_skip8,
                      const uint32_t *d_imp_scales, const uint32_t dist_scale[3], double lambda,
                      const b200_cdef_rdo_area *areas, size_t n_areas, const uint32_t *d_rate, uint64_t *d_err,
                      double *d_cost, int8_t *d_best);

/* ------------------------------------------------------- deblocking (deblock.rs)
 * The deblocking filter's level search (deblock_filter_optimize without fast_deblock, i.e. sse_optimize,
 * deblock.rs:1461-1618) and the filter itself (deblock_filter_frame -> deblock_plane, deblock.rs:1294-1551)
 * for a HOST list of items, each asynchronous on the context's stream.  An item is the TileBlocks rect one
 * of the reference's call sites passes: the whole frame (encoder.rs:3263-3290), a tile (the delayed
 * loop-filter RDO, encoder.rs:3586-3625) or a loop-restoration area (rdo.rs:2297-2331).  Edges are found on
 * the item's own grid: nothing is filtered across its left or top border.  Levels stay on the device
 * between the two calls, so "levels, filter, b200_cdef_rdo_dev" needs no host synchronisation.
 *
 * d_mi: one b200_deblock_mi per 4x4 luma block of the frame, mi_stride records per row, covering every
 * item's mi rect.  It is device data, so it is not checked: every table lookup is bounded for any byte
 * value, and for a record the reference would panic on (bsize >= 22, txsize >= 19, a bsize without a
 * subsampled_size in 4:2:2) the item's results are unspecified.  The grid must be consistent as an
 * encoder writes it (one bsize and txsize per block, transforms tiling the block): the filter runs all
 * edges of one direction in parallel, which equals the reference's order only when no two edges of one
 * direction touch the same pixels.
 *
 * The working rect of an item is the region the reference's scratch copy covers: luma pixels
 * [4 mi_x, 4 mi_x + min(4 mi_w, vis_w rounded up to 8)) and likewise vertically; chroma planes take it
 * decimated.  The filter reads `in` and writes `out` there and nowhere else: pixels are filtered where an
 * edge is filtered and copied from `in` everywhere else, so a caller needs no "deblock in place, then
 * restore" (encoder.rs:3598-3647).  An item whose luma levels are both 0 gets a copy of `in` in every plane,
 * as every call site skips deblock_filter_frame then (encoder.rs:3280, :3598, rdo.rs:2311); a chroma plane
 * whose own level is 0 gets a copy (deblock.rs:1302-1319).  The level search reads rec and src over the
 * working rect and, because sse_h_edge sizes horizontal edges by the transform WIDTH (deblock.rs:1257, kept
 * as is), up to 4 rows above and below it.
 *
 * rec / src / in / out: HOST arrays of `planes` (1 = 4:0:0, or 3) device planes.  d_levels: 4 per item
 * (Y vertical, Y horizontal, U, V); the level search writes them (0 for U and V in 4:0:0), the filter reads
 * them.  d_tally (may be NULL): per item x plane (3, zeros for absent planes) x {vertical, horizontal}, the
 * 64 prefix-summed i64 tallies (levels 0..63) the argmin reads: d_tally[((item * 3 + p) * 2 + dir) * 64 + l].
 * Rejected with B200_ERR_ARG before any launch, with nothing written: NULL pointers, a bpp that does not
 * match bit_depth (8 / 10 / 12), planes other than 1 / 3, a layout other than 4:2:0 / 4:2:2 / 4:4:4, an
 * item whose origin is not on the 64x64 superblock grid, that is empty, has an odd mi_w / mi_h (FrameBlocks
 * are always an even number of 4x4 blocks, encoder.rs:852-853), reaches past mi_stride, or overlaps
 * another item, vis_w / vis_h <= 0, a working rect (for the level search extended by 4 rows above and
 * below) outside a plane's readable area [-pad, width + pad) x [-pad, height + pad), with the filter `out`
 * aliasing `in`, and a state with block_delta_shift above 3 (delta_lf_res is two bits).
 * n_items == 0 launches nothing. */
typedef struct {   /* one per 4x4 luma block: the fields of Block (context/block_unit.rs:165-183) deblocking reads */
  uint8_t bsize;   /* BlockSize 0..21 (n4_w / n4_h and the chroma tx size derive from it) */
  uint8_t txsize;  /* luma TxSize 0..18 */
  uint8_t mode;    /* PredictionMode discriminant (mode_deltas' mode type, deblock.rs:48-53) */
  uint8_t skip;    /* 0 / 1 */
  int8_t ref0;     /* ref_frames[0].to_index(); 0 = INTRA_FRAME */
  int8_t deltas[4]; /* Block::deblock_deltas */
  uint8_t pad_[3];
} b200_deblock_mi; /* 12 B */
typedef struct {
  int32_t mi_x, mi_y; /* origin in 4x4 luma units, frame-absolute, multiples of 16 (a superblock) */
  int32_t mi_w, mi_h; /* the item's TileBlocks cols() / rows() */
  int32_t vis_w, vis_h; /* visible luma pixels from the origin: crop_w - rect.x, crop_h - rect.y */
} b200_deblock_item;
typedef struct {       /* DeblockState (encoder.rs:522-532) without levels; sharpness is not read */
  uint8_t deltas_enabled;
  int8_t ref_deltas[8];
  int8_t mode_deltas[2];
  uint8_t block_deltas_enabled, block_delta_shift, block_delta_multi;
  uint8_t pad_[2];
} b200_deblock_state; /* 16 B */
int b200_deblock_levels_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src, int planes, int xdec,
                            int ydec, int bit_depth, const b200_deblock_mi *d_mi, int mi_stride,
                            const b200_deblock_item *items, size_t n_items, uint8_t *d_levels, int64_t *d_tally);
int b200_deblock_filter_dev(b200_ctx *ctx, const b200_plane *in, const b200_plane *out, int planes, int xdec,
                            int ydec, int bit_depth, const b200_deblock_state *state, const uint8_t *d_levels,
                            const b200_deblock_mi *d_mi, int mi_stride, const b200_deblock_item *items,
                            size_t n_items);

/* ------------------------------------------------------- loop restoration (lrf.rs)
 * RestorationState::lrf_filter_frame (lrf.rs:1482-1585), asynchronous on the context's stream: Wiener
 * (wiener_stripe_filter, :1099-1207) and self-guided (setup_integral_image + sgrproj_stripe_filter,
 * :529-830) units over whole frames, stripe by stripe, reading the CDEF output `cdeffed` and the deblocked
 * frame `deblocked` through the reference's stripe source rules.  Planes: 1 (4:0:0) or 3; the crop of plane
 * p is ((frame_width + (1 << xd >> 1)) >> xd) x ((frame_height + (1 << yd >> 1)) >> yd).
 *
 * Every pixel of every plane's crop is written to `out`, filtered or copied from `cdeffed` (None units, and
 * Sgrproj units when enable_cdef == 0, as lrf.rs:1545-1547 skips them); nothing else is written, so a
 * caller needs no "copy, then filter in place".  Where the frame is shorter than stripe 0 (crop_h < 56 >>
 * ydec) the reference also writes Sgrproj rows below the crop; this call does not.  `cdeffed` may be the
 * same plane as `deblocked`; `out` may alias neither.
 *
 * units[p]: a HOST array of cols x rows records for plane p, row-major, with cols = max(1, (crop_w +
 * unit_size[p] / 2) / unit_size[p]) and rows likewise (lrf.rs:1431-1440).  A stripe's unit row is
 * min(stripe * stripe_height / unit_size, rows - 1), with stripe_height 32 for 4:2:0 chroma and 64
 * otherwise (lrf.rs:1295-1312); the last unit column stretches to the crop.  All records go up in one copy.
 * Rejected with B200_ERR_ARG before any launch, with nothing written: NULL pointers, a bpp that does not
 * match bit_depth (8 / 10 / 12), planes other than 1 / 3, a layout other than 4:2:0 / 4:2:2 / 4:4:4, a frame
 * under 32x32 (enable_restoration_filters, encoder.rs:232), a unit_size that is not a power of two in
 * 32..256, a plane smaller than its crop, an `out` plane's crop overlapping an input plane's crop, and a
 * record out of range (lrf.rs:39-48): type above 2, or for Sgrproj a set above 15 or xqd outside
 * SGRPROJ_XQD_MIN..MAX, or for Wiener a tap outside WIENER_TAPS_MIN..MAX. */
typedef struct {      /* RestorationFilter (lrf.rs:126-136) */
  uint8_t type;       /* 0 None, 1 Wiener, 2 Sgrproj */
  uint8_t set;        /* Sgrproj: SGRPROJ_PARAMS_S index */
  int8_t xqd[2];      /* Sgrproj */
  int8_t coeffs[2][3]; /* Wiener: [0] vertical, [1] horizontal */
  uint8_t pad_[2];
} b200_lrf_unit;      /* 12 B */
int b200_lrf_filter_dev(b200_ctx *ctx, const b200_plane *cdeffed, const b200_plane *deblocked,
                        const b200_plane *out, int planes, int xdec, int ydec, int frame_width, int frame_height,
                        int bit_depth, int enable_cdef, const int unit_size[3],
                        const b200_lrf_unit *const units[3]);

/* The restoration search of one rdo_loop_decision pass (rdo.rs:2575-2740) for a HOST list of items,
 * asynchronous on the context's stream with a fixed number of launches and no host synchronisation.  An
 * item is one (area, plane, unit) the reference reaches at rdo.rs:2607-2611: the caller builds the list
 * where rdo.rs:2585-2611 loops, so lru_skip / lru_on_skip and has_restoration_unit(.., false) stay with it.
 *
 * Per item, in the plane's pixels: the unit's origin inside the area is lrf_po = (lru_x * lru_sb_w,
 * lru_y * lru_sb_h) superblocks with lru_sb_w = (unit_size << xdec) / 64, and its visible rect is
 * vis_w = min(unit_size, ((frame_width - area_x) >> xdec) - lrf_po.x), vis_h likewise (rdo.rs:2651-2658;
 * a floor shift, so an odd luma crop's last 4:2:0 chroma column is outside it).
 *  1. None: rdo_loop_plane_error (rdo.rs:2027-2093) of lrf_in over the unit's superblocks (luma
 *     cdef_dist_kernel 8x8, chroma sse_wxh, each times the 8x8 block's frame-absolute distortion_scale,
 *     blocks inside the area's 8x8 grid only, the sum times dist_scale[p]).  Its rate is
 *     count_lrf_switchable of the INCOMING filter, as the reference passes best_new_lrf (rdo.rs:2633-2638):
 *     an Sgrproj incumbent charges None its own rate.  Taken if incoming_cost < 0 or cost < incoming_cost.
 *  2. The integral image of lrf_in over vis (setup_integral_image, lrf.rs:529-627) in the area's scratch
 *     copy: 4 real columns on the left unless the unit starts at the area's left edge, the last column
 *     repeated on the right, real rows down to 2 above the unit (clamped to the area's row 0), the last row
 *     repeated below.  All reads stay inside the area.
 *  3. For each set of get_sgr_sets (all 16, or 1, 3, .. 15 with reduced_sets): sgrproj_solve
 *     (lrf.rs:846-1096), sgrproj_stripe_filter over vis, rdo_loop_plane_error with the filtered pixels
 *     inside vis and B200_LRF_WORK_FILL outside it, the rate sgr_bits + (4 << 3) + the signed subexp bits
 *     of xqd against sgrproj_ref (context/frame_header.rs:14-45, ec.rs:639-773), compute_rd_cost; taken
 *     on a strict `<`.
 * The solve's sums are exact: every term is below 2^34 in magnitude and a 256x256 unit's total below
 * 2^50, so the reference's f64 accumulation of i64 line sums equals one i64 total, and the rest of the
 * solve runs the reference's f64 operations one for one; results are bit exact.
 *
 * lrf_in / src: HOST arrays of `planes` planes: the pass's lrf_input (the `out` of b200_cdef_rdo_dev, or the
 * deblocked frame with CDEF off) and the input, covering at least the frame rounded up to 8 luma pixels.
 * unit_size[p]: RestorationPlaneConfig::unit_size, whole superblocks (unit_size << dec a multiple of 64),
 * 32..256.  d_imp_scales / dist_scale / lambda as b200_cdef_rdo_dev.  areas: HOST, as b200_cdef_rdo_dev.
 * Outputs on the device, per item i: d_best[i] (the winner: the incoming filter when nothing beat it),
 * d_cost[i] (its cost, the incoming cost when nothing improved), d_changed[i] = incoming.notequal(best)
 * (lrf.rs:139-160).  Optional (NULL = not wanted): d_xqd[(i * 16 + set) * 2 + k], d_err[i * 17 + c] and
 * d_cand_cost[i * 17 + c] with c = 0 for None and 1 + set for each set searched; other slots untouched.
 * Rejected with B200_ERR_ARG before any launch, with nothing written: NULL pointers, a bpp that does not
 * match bit_depth (8 / 10 / 12), planes other than 1 / 3, a layout other than 4:2:0 / 4:2:2 / 4:4:4, bad
 * frame sizes, planes smaller than the frame's 8x8 blocks, a unit size that is not a power of two in
 * 32..256 made of whole superblocks, an area outside the frame or larger than 4x4 superblocks, an item
 * whose area or plane index is out of range or whose unit starts outside its area or its visible crop, an
 * incoming record that is Wiener (the reference has no rate for it) or out of range, and a sgrproj_ref out
 * of SGRPROJ_XQD_MIN..MAX.  n_items == 0 launches nothing. */
/* The pixels of the reference's lrf_work outside each unit's visible rect: Plane::new's fill (v_frame
 * 0.3.9, off disk upstream; restated as T::cast_from(128) and parity-unpinned). */
#define B200_LRF_WORK_FILL 128
typedef struct {
  int32_t area;            /* index into areas */
  int32_t plane;           /* 0..planes-1 */
  int32_t lru_x, lru_y;    /* the unit inside the area, in units of this plane */
  b200_lrf_unit incoming;  /* best_lrf of the unit on entry: None or Sgrproj */
  uint32_t none_bits;      /* symbol_bits(0, lrf_switchable_cdf) */
  double incoming_cost;    /* best_lrf_cost on entry; < 0 = none yet */
  uint32_t sgr_bits;       /* symbol_bits(2, lrf_switchable_cdf) */
  int8_t sgrproj_ref[2];   /* the plane's TileRestorationPlane::sgrproj_ref */
  uint8_t pad_[2];
} b200_lrf_search_item;    /* 48 B */
int b200_lrf_search_dev(b200_ctx *ctx, const b200_plane *lrf_in, const b200_plane *src, int planes, int xdec,
                        int ydec, int frame_width, int frame_height, int bit_depth, const int unit_size[3],
                        int reduced_sets, const uint32_t *d_imp_scales, const uint32_t dist_scale[3],
                        double lambda, const b200_cdef_rdo_area *areas, size_t n_areas,
                        const b200_lrf_search_item *items, size_t n_items, b200_lrf_unit *d_best,
                        double *d_cost, uint8_t *d_changed, int8_t *d_xqd, uint64_t *d_err,
                        double *d_cand_cost);

/* rdo_loop_decision (rdo.rs:2104-2745) from the point after its optional deblock, for a HOST list of
 * loop-restoration areas in one call: the CDEF analysis, then the pass loop of CDEF stages (C) and
 * restoration stages (L), C, L, C, L, .., per area until a stage changes nothing.  Unlike its neighbours this
 * call SYNCHRONISES the context's stream: the number of stages depends on the data, so after every stage it
 * reads back one small status record (the count of areas still changing); nothing else comes back.  Areas
 * are independent, as in the reference (each has its own scratch copy).
 *
 * Per area: it has CDEF work when enable_cdef and some 8x8 block of it is not skipped (!cdef_skip_all), and
 * restoration work (lrf_work) when enable_restoration and some unit of it has `search` set.  An area with
 * neither gets no stage (rdo.rs:2267).  A C stage counts as changed on the first pass whatever it does
 * (cdef_change starts true) and afterwards when some superblock's index changed; without CDEF work it does
 * nothing.  An L stage counts as changed when some unit's filter changed; without lrf_work it does nothing
 * and is unchanged.  An area stops after its first unchanged stage; its stage count includes that stage.
 *  C: every superblock that is not CDEF-skipped, in raster order, tries every index 0 .. 1 << cdef_bits as
 *     b200_cdef_rdo_dev does, except for the restoration terms of each plane p whose map entry u =
 *     sb_unit[(area * 16 + sby * 4 + sbx) * 3 + p] is not -1, when the area has lrf_work:
 *     - the rate adds count_lrf_switchable of unit u's current filter: none_bits for None, sgr_bits +
 *       (4 << 3) + the signed subexp bits of xqd against sgrproj_ref for Sgrproj (rdo.rs:2446-2506);
 *     - for Sgrproj, the plane's distortion is measured after the self-guided filter (rdo.rs:2458-2500):
 *       the integral image of the CDEF working copy over the superblock's visible rect with crop = stripe
 *       = vis (4 real columns on the left unless the superblock is in the area's column 0, 2 real rows
 *       above clamped to the area's row 0, nothing real right or below), sgrproj_stripe_filter with the
 *       unit's set and xqd, then rdo_loop_plane_error with the filtered pixels inside vis and
 *       B200_LRF_WORK_FILL outside it.  Those left / upper pixels are THIS pass's winners of the left, upper
 *       and upper-left superblocks (rdo.rs:2554-2564 re-filters every winner in raster order), so the
 *       device runs each C stage one anti-diagonal of superblocks at a time.
 *     Without lrf_work the rate is 0 and the distortion is the CDEF output's (the no-LRU branch).  The
 *     first minimum wins; the winner is filtered into the working copy.
 *  L: b200_lrf_search_dev's computation over the units with `search` set, reading the working copy (rec for
 *     an area without CDEF work), with the incumbent filter and best_lrf_cost carried from the previous L
 *     stage (None and -1 on the first).
 *
 * rec: HOST array of `planes` planes, the deblocked reconstruction (b200_deblock_filter_dev's `out` over the
 * same areas, or the reconstruction when deblocking is off).  src: the input.  work: the caller's CDEF
 * working copy (the reference's cdef_work), aliasing neither rec nor src; every area that runs a stage gets
 * a copy of rec over its scratch rect first, and holds afterwards the last C stage's output there (rec
 * itself for an area without CDEF work).  Nothing outside those rects is written.  Planes cover at least
 * the frame rounded up to 8 luma pixels.  enable_cdef / damping / cdef_bits / strengths / d_skip8 as
 * b200_cdef_rdo_dev (the strengths are not read with enable_cdef == 0); enable_restoration / unit_size /
 * reduced_sets as b200_lrf_search_dev (unit_size is not read with enable_restoration == 0);
 * d_imp_scales / dist_scale / lambda as both.
 *
 * units: HOST array of n_units records, one per restoration unit of an area and plane the caller tracks
 * (TileRestorationState's units, which stay with the caller); sb_unit: HOST, n_areas * 16 * 3 entries,
 * each an index into units or -1, mirroring restoration_unit_offset(base_sbo, loop_sbo, false) for every
 * superblock slot of every area (entries of slots outside an area are not read).
 * Outputs on the device: d_best_index[slot] (area * 16 + sby * 4 + sbx): the final index, -1 for
 * CDEF-skipped superblocks and every superblock of an area without CDEF work (set_cdef reads it); per unit
 * d_unit[u], d_unit_cost[u] (best_lrf_cost) and d_written[u] = 1 when the unit's filter changed at some
 * stage of the call, so the caller can apply rdo.rs:2730-2741's conditional `ru.filter = ..` exactly.
 * Optional (NULL = not wanted): d_err / d_cost of the LAST C stage that evaluated a superblock, laid out as
 * b200_cdef_rdo_dev's.  Slots and units of areas that run no stage, and slots outside the areas, are not
 * written.  *stages: the number of stages of the longest area (0 when no area runs one), or -1 when an
 * area was still changing after B200_LOOP_MAX_STAGES stages, where the call stops.
 * Rejected with B200_ERR_ARG before any launch, with nothing written: a NULL ctx / rec / src / work /
 * dist_scale / stages / d_best_index, or NULL unit outputs with n_units > 0; a bpp that does not match
 * bit_depth (8 / 10 / 12); planes other than 1 / 3; a layout other than 4:2:0 / 4:2:2 / 4:4:4; bad frame
 * sizes; planes smaller than the frame's 8x8 blocks; work aliasing rec or src; with enable_cdef, NULL
 * strengths, cdef_bits outside 0..3, a used strength above 63 or damping outside 3..6; with
 * enable_restoration, a NULL unit_size or a unit size as b200_lrf_search_dev rejects it; areas outside
 * the frame, larger than 4x4 superblocks or overlapping each other; n_areas > 0 with NULL areas / sb_unit;
 * n_units > 0 with NULL units; a unit whose area or plane is out of range, which starts outside its area
 * or its visible crop, or whose sgrproj_ref is out of SGRPROJ_XQD_MIN..MAX; a map entry outside -1 ..
 * n_units - 1 or naming a unit of another area or plane.  n_areas == 0 launches nothing. */
#define B200_LOOP_MAX_STAGES 64
typedef struct {
  int32_t area;            /* index into areas */
  int32_t plane;           /* 0..planes-1 */
  int32_t lru_x, lru_y;    /* the unit inside the area, in units of this plane */
  uint32_t none_bits;      /* symbol_bits(0, lrf_switchable_cdf) */
  uint32_t sgr_bits;       /* symbol_bits(2, lrf_switchable_cdf) */
  int8_t sgrproj_ref[2];   /* the plane's TileRestorationPlane::sgrproj_ref */
  uint8_t search;          /* !lru_skip && has_restoration_unit(.., false) (rdo.rs:2212-2263, 2593-2611) */
  uint8_t pad_;
} b200_loop_unit;          /* 28 B */
int b200_loop_decision_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src, const b200_plane *work,
                           int planes, int xdec, int ydec, int frame_width, int frame_height, int bit_depth,
                           int enable_cdef, int damping, int cdef_bits, const uint8_t y_strengths[8],
                           const uint8_t uv_strengths[8], const uint8_t *d_skip8, int enable_restoration,
                           const int unit_size[3], int reduced_sets, const uint32_t *d_imp_scales,
                           const uint32_t dist_scale[3], double lambda, const b200_cdef_rdo_area *areas,
                           size_t n_areas, const b200_loop_unit *units, size_t n_units, const int32_t *sb_unit,
                           int8_t *d_best_index, b200_lrf_unit *d_unit, double *d_unit_cost, uint8_t *d_written,
                           uint64_t *d_err, double *d_cost, int *stages);

/* ------------------------------------------------------- intra prediction (predict.rs)
 * Boundary = rust::dispatch_predict_intra(mode, variant, dst, tx_size, bit_depth, ac, angle,
 * ief_params, edge_buf, cpu) (predict.rs:705-784; the asm wrappers, asm/x86/predict.rs:239-873,
 * have the same Rust signature).  `edge` is the reference's IntraEdge buffer (partition.rs:
 * 600-637): 4*64+1 pixels, top-left at index 128, left pixels bottom->top in [128-left_len, 128),
 * above pixels in [129, 129+above_len).  mode = PredictionMode discriminant 0..13
 * (predict.rs:73-87); variant 0 NONE, 1 LEFT, 2 TOP, 3 BOTH (:112-118); angle = prediction angle
 * in degrees (intra_mode_to_angle + 3*angle_delta) or the CfL alpha; ief = -1 for None, else
 * IntraEdgeFilterParameters::use_smooth_filter() as 0/1 (:574-596); plane_w/plane_h/dst_x/dst_y =
 * dst.plane_cfg.{width,height} and dst.rect().{x,y} (edge-filter clipping, :1357-1364). */
void b200_predict_intra(int mode, int variant, void *dst, ptrdiff_t dst_stride, int w, int h,
                        int bit_depth, const int16_t *ac, int angle, int ief, const void *edge,
                        int left_len, int above_len, int plane_w, int plane_h, int dst_x, int dst_y);

typedef struct {
  uint32_t edge;    /* index of the IntraEdge buffer inside d_edges (257 pixels each) */
  uint32_t ac;      /* index of the w*h int16 CfL ac block inside d_ac (UV_CFL_PRED only) */
  int16_t x, y;     /* dst.rect().x / .y */
  int16_t angle;    /* degrees, or CfL alpha */
  uint8_t mode;     /* PredictionMode 0..13 */
  uint8_t variant;  /* PredictionVariant */
  int8_t ief;       /* -1 none, 0/1 = Some(use_smooth_filter) */
  uint8_t left_len, above_len;
  uint8_t pad_;
} b200_intra_item;

/* get_intra_edges (partition.rs:639-898) for a batch of transform blocks of one PlaneRegion: builds
 * the IntraEdge buffers b200_predict_intra_dev consumes, with the reference's availability rules
 * (has_top_right / has_bottom_left, recon_intra.rs:174-452), border constants and replication.
 * `plane` with (rect_x, rect_y, rect_w, rect_h) is the `dst` region (tile) the offsets are relative
 * to; plane->width / height are plane_cfg.width / height; xdec / ydec the plane's decimation.
 * d_edges: nitems x 257 pixels (top-left at [128]); entries outside
 * [128 - init_left, 129 + init_above) are zero (uninitialised upstream); d_lens (may be NULL):
 * {init_left, init_above} per item = the slice lengths IntraEdge::new records.  What may share a
 * batch is the caller's business: blocks whose neighbours are final (all of a frame in the lookahead,
 * one wavefront of the encode loop). */
typedef struct {
  int16_t po_x, po_y;     /* PlaneOffset of the transform block inside the region, pixels */
  int16_t part_x, part_y; /* partition_bo (TileBlockOffset), 4x4 luma units */
  uint8_t bx, by;         /* transform-block index inside the partition */
  uint8_t bsize;          /* partition BlockSize discriminant 0..21 (partition.rs:130-153) */
  uint8_t tx_size;        /* TxSize discriminant 0..18 */
  uint8_t mode;           /* PredictionMode 0..13, 255 = None (every edge wanted) */
  int8_t angle_delta;     /* IntraParam::AngleDelta, else 0 */
  uint8_t enable_ief;     /* enable_intra_edge_filter */
  uint8_t pad_;
} b200_edge_item;
int b200_get_intra_edges_dev(b200_ctx *ctx, const b200_plane *plane, int rect_x, int rect_y, int rect_w,
                             int rect_h, int xdec, int ydec, int bit_depth, const b200_edge_item *d_items,
                             size_t nitems, void *d_edges, uint8_t *d_lens);

/* Batched: one prediction per item (typically blocks x candidate modes sharing edge buffers);
 * d_out receives nitems packed w x h blocks (pixels). */
int b200_predict_intra_dev(b200_ctx *ctx, const void *d_edges, const b200_intra_item *d_items,
                           size_t nitems, const int16_t *d_ac, int w, int h, int bit_depth,
                           int plane_w, int plane_h, void *d_out);
/* Intra mode screening, the pruning metric of intra_frame_rdo_mode_decision (rdo.rs:1433-1511) for a
 * batch of luma blocks of one PlaneRegion (tile): per item, get_intra_edges (mode None) from `rec`,
 * then every mode in positions num_modes_rdo / 2 .. 13 of `modes` predicted at bsize.tx_size()
 * (partition.rs:306-328; TX_64X64 for the 128-class sizes) through PredictionMode::predict_intra
 * (predict.rs:205-249: PredictionVariant from the tile-relative position, PAETH_PRED remapped to
 * DC / V / H at the tile's top / left edges, intra_mode_to_angle, `ief` for directional modes only),
 * get_satd of each prediction against `src` at the tx size, and the tail of `modes` stable-sorted by
 * SATD (ties keep the CDF order).  One launch; the edges and the source block are staged once per
 * block, predictions exist only in registers, `rec` is not written.
 *
 * `rec` / `src` with (rect_x, rect_y, rect_w, rect_h) are the tile's reconstruction and input; the
 * region must lie inside the plane.  What may share a call is the caller's business: every block's
 * neighbours must be final in `rec` (a whole frame in the lookahead, one wavefront of the encode
 * loop); tiles run on their own threads and contexts (encoder.rs:3253).
 *
 * d_satd (nitems x 13, by PredictionMode discriminant: satds_all, 0 = not screened) and d_modes
 * (nitems x 13: `modes` after the tail sort) may each be NULL, not both.  Rejected with B200_ERR_ARG
 * before any launch: num_modes_rdo other than 3 / 7, a bpp that does not match bit_depth (8 / 10 /
 * 12), rec and src of different sizes, a region outside the plane, rec->pad or src->pad below 64 (the
 * SATD reads the whole tx block past the visible frame, as the reference does), both outputs NULL,
 * NULL items with nitems > 0.  An item with bsize >= 22, a list entry >= 13 or repeated, or (x, y)
 * outside the region or not a multiple of 4 gets UINT32_MAX in its 13 d_satd entries and its list
 * copied unchanged; nothing is read or written out of bounds for it. */
typedef struct {
  int16_t x, y;      /* block's top-left inside the region, luma px, multiples of 4 (tile_bo.plane_offset) */
  uint8_t bsize;     /* BlockSize 0..21 (partition.rs:130-153) */
  int8_t ief;        /* -1: enable_intra_edge_filter off; else IntraEdgeFilterParameters::use_smooth_filter() */
  uint8_t modes[13]; /* RAV1E_INTRA_MODES after the CDF sort (rdo.rs:1416-1428), PredictionMode discriminants */
  uint8_t pad_;
} b200_intra_screen_item;
int b200_intra_mode_screen_dev(b200_ctx *ctx, const b200_plane *rec, const b200_plane *src, int rect_x, int rect_y,
                               int rect_w, int rect_h, int bit_depth, int num_modes_rdo,
                               const b200_intra_screen_item *d_items, size_t nitems, uint32_t *d_satd,
                               uint8_t *d_modes);

/* Inter mode screening, the SATD pruning of inter_frame_rdo_mode_decision (rdo.rs:1281-1363) for a batch
 * of luma blocks of one PlaneRegion (tile): per item, every entry of its resolved mode list predicted at
 * the full block size through PredictionMode::predict_inter (predict.rs:284-421): put_8tap for a single
 * reference, prep_8tap of both references then mc_avg for a compound pair, both with FilterMode
 * `filter_mode` (fi.default_filter) in both directions; the source position is get_mv_params', including
 * PlaneSlice::clamp to [-xorigin, width] x [-yorigin, height] (a rav1e caller passes its luma plane's
 * cfg.xorigin / cfg.yorigin); get_satd of each prediction against `src`; the entries stable-sorted by SATD
 * (sort_by_key, ties keep list order).  Predictions exist only in shared memory.
 *
 * The mode list itself (rdo.rs:1158-1318, find_mvrefs' stacks) stays with the caller, and so do two of
 * its quirks: rdo.rs computes and sorts the SATDs only when num_modes_rdo != the list's length (lists
 * shorter than 9 included), and a missing reference frame (`if let Some(ref rec)`) leaves a stale
 * prediction there; call this only for lists the reference screens, over present references.
 *
 * `src` with (rect_x, rect_y, rect_w, rect_h) is the tile's input and region (inside the plane);
 * refs[0 .. nrefs) are whole reference frames (fi.rec_buffer slots, 1 <= nrefs <= 8) of src's size and
 * bpp, addressed by the entries' `ref` indices.  Up to four launches (a validation / bucketing pass by
 * size class, then one per class); no host synchronisation; context scratch holds the buckets.
 *
 * d_satd (nitems x 20, list order, UINT32_MAX at positions >= n) and d_order (nitems x 20: the stable
 * ascending sort of entries 0 .. n by SATD followed by n .. 19, a permutation of 0 .. 19) may each be
 * NULL, not both.  Rejected with B200_ERR_ARG before any launch: a bit depth other than 8 / 10 / 12 or a
 * bpp that does not match it, nrefs outside 1 .. 8 or a reference whose size or bpp differs from src, a
 * region outside the plane, filter_mode outside 0 .. 3, src->pad below 64, a negative xorigin / yorigin, a
 * reference pad below max(xorigin, yorigin, 71) (the clamped footprint spans [-origin, size + 70]), both
 * outputs NULL, NULL items with nitems > 0.  An item with bsize >= 22 or 128-sided (13 / 14 / 15), n > 20,
 * a ref index >= nrefs in one of its n entries, or (x, y) outside the region or not a multiple of 4 gets
 * UINT32_MAX in its 20 d_satd entries and the identity order; nothing is read or written out of bounds
 * for it.  nitems == 0 launches nothing. */
typedef struct {
  int16_t mv[2][2]; /* mv[k] = {row, col}, 1/8 pel (MotionVector); mv[1] ignored for a single reference */
  uint8_t ref[2];   /* index into refs[]; ref[1] = 0xFF: single reference (NONE_FRAME) */
  uint8_t pad_[2];
} b200_inter_screen_cand; /* 12 B */
typedef struct {
  int16_t x, y;  /* block's top-left inside the region, luma px, multiples of 4 */
  uint8_t bsize; /* BlockSize 0..21 (partition.rs:130-153) */
  uint8_t n;     /* entries used, 0..20 (ArrayVec<_, 20>, rdo.rs:1158) */
  uint8_t pad_[2];
  b200_inter_screen_cand cands[20];
} b200_inter_screen_item; /* 248 B */
int b200_inter_mode_screen_dev(b200_ctx *ctx, const b200_plane *src, int rect_x, int rect_y, int rect_w,
                               int rect_h, const b200_plane *refs, int nrefs, int xorigin, int yorigin,
                               int filter_mode, int bit_depth, const b200_inter_screen_item *d_items,
                               size_t nitems, uint32_t *d_satd, uint8_t *d_order);

/* pred_cfl_ac (predict.rs:1020-1063; asm cfl_ac_{420,422,444}, asm/x86/predict.rs:142-186):
 * bw x bh = chroma block size; d_blocks[i] = LUMA position of block i. */
int b200_pred_cfl_ac_dev(b200_ctx *ctx, const b200_plane *luma, const b200_block *d_blocks,
                         size_t nblocks, int bw, int bh, int w_pad, int h_pad, int xdec, int ydec,
                         int16_t *d_ac);

/* The CfL alpha search of rdo_mode_decision (rdo.rs:1013-1041): rdo_cfl_alpha (rdo.rs:1593-1689) for a batch
 * of blocks of one tile in one asynchronous call on the context's stream, without host synchronisation.  Per
 * item: uv_tx_size = bsize.largest_chroma_tx_size; the visible chroma area from clip_visible_bsize
 * (rdo.rs:228-253) at the frame block offset, i.e. ((x + rect_x) >> xdec, (y + rect_y) >> ydec), which for a
 * sub-8x8 block at an odd 4x4 position is 2 (mod 4), not the 4-aligned chroma origin; luma_ac
 * (predict.rs:644-698: the luma of tile_bo + sub8x8_offset, frame_clipped_bw / bh against fi.w_in_b /
 * fi.h_in_b, the frame rounded up to 8, max_luma_w / h rounded up to the luma tx size for sides above 8,
 * per-block w_pad / h_pad); per chroma plane get_intra_edges (UV_CFL_PRED, po = tile_bo.plane_offset),
 * predict_intra at each alpha -16 ..= 16 (alpha 0 = DC_PRED, else DC + get_scaled_luma_q0) and sse_wxh over
 * the visible area at the default DistortionScale (whole 4x4 chunks only); then the reference's early exit:
 * best = (cost(0), 0), count = 2, for alpha 1..=16 +alpha then -alpha against the updated best, each strict
 * improvement adds 2 to count, break when count < alpha.  Predictions exist only in registers; `rec` is not
 * written (the reference's last write there is dead: its caller re-predicts chroma, rdo.rs:1054-1075).
 *
 * rec / src: HOST arrays of the three frame planes (src[0] is not read).  (rect_x, rect_y, rect_w, rect_h) is
 * the tile in luma pixels, origin a multiple of 8, inside the frame's 8x8 blocks; the chroma region is that
 * rect decimated (TileRect::decimated).  frame_width / frame_height = fi.width / fi.height.  What may share a
 * call is the caller's business: each block's luma reconstruction and its chroma neighbours must be final in
 * rec (one wavefront of the encode loop); tiles run on their own threads and contexts (encoder.rs:3253).
 *
 * d_alpha (nitems x 2: best_alpha of planes 1 and 2; the caller forms None when both are 0, else
 * CFLParams::from_alpha) and d_sse (nitems x 2 x 33, [item][plane - 1][alpha + 16]: the sse_wxh of every alpha
 * the reference evaluates, UINT64_MAX for the alphas its loop never reaches) may each be NULL, not both.
 * Rejected with B200_ERR_ARG before any launch: NULL pointers, a bit depth other than 8 / 10 / 12 or a bpp
 * that does not match it, a layout other than 4:2:0 / 4:2:2 / 4:4:4, planes smaller than the frame (chroma:
 * (fi.width + xdec) >> xdec by (fi.height + ydec) >> ydec), src and rec chroma of different sizes, a region
 * outside the frame's 8x8 blocks or not 8-aligned, and a luma rec that does not reach 31 pixels past the
 * frame in each direction (rec[0].width + rec[0].pad >= frame_width + 31, likewise the height: luma_ac reads
 * up to that far past the visible frame, as the reference does).  nitems == 0 launches nothing.
 * An invalid item gets {0, 0} in d_alpha and UINT64_MAX in its 66 d_sse entries, and nothing is read for it:
 * bsize > BLOCK_32X32 (cfl_allowed; 4x16 / 16x4 / 8x32 / 32x8 included), a size with no subsampled_size for
 * the layout (4:2:2: 4x8, 8x16, 16x32), a block without chroma (has_chroma), tx_size >= 19 or larger than
 * the block, (x, y) outside the region or not a multiple of 4.  A valid item whose visible area is 0 gets the
 * same outputs (the reference returns None without evaluating anything). */
typedef struct {
  int16_t x, y;    /* block's top-left inside the region, luma px, multiples of 4 (tile_bo.to_luma_plane_offset) */
  uint8_t bsize;   /* BlockSize 0..21; only cfl_allowed() sizes (discriminant <= BLOCK_32X32) are valid */
  uint8_t tx_size; /* the block's luma TxSize (rdo_mode_decision's best.tx_size) */
  uint8_t pad_[2];
} b200_cfl_item; /* 8 B */
int b200_cfl_alpha_dev(b200_ctx *ctx, const b200_plane rec[3], const b200_plane src[3], int xdec, int ydec,
                       int rect_x, int rect_y, int rect_w, int rect_h, int frame_width, int frame_height,
                       int bit_depth, const b200_cfl_item *d_items, size_t nitems, int8_t *d_alpha,
                       uint64_t *d_sse);

/* ------------------------------------------------ reference-signature symbols (MC / intra / CDEF)
 * The reference's own extern "C" prototypes, symbol for symbol, with the ISA suffix replaced by
 * `_cuda`: they slot into PUT_FNS / PUT_HBD_FNS / PREP_FNS / PREP_HBD_FNS / AVG_FNS / AVG_HBD_FNS
 * (asm/x86/mc.rs:322-620), the per-mode calls of asm::x86::predict::dispatch_predict_intra and
 * pred_cfl_ac (asm/x86/predict.rs:239-960), CDEF_FILTER_FNS and CDEF_DIR_{LBD,HBD}_FNS
 * (asm/x86/cdef.rs:161-176, :236-260) unchanged.  Host pointers, BYTE strides, exactly the
 * reference's argument lists (defined in rav1e_b200/csrc/ref_abi.cu over the per-call forms above).
 * Re-entrant: each host thread runs on its own context (one rayon worker per tile, encoder.rs:3253). */
/* X(name, FilterMode x, FilterMode y): table slot (x + 4 y) & 15, asm/x86/mc.rs:80-82, :394-405 */
#define B200_FOR_EACH_MC_FILTER(X)                                                              \
  X(8tap_regular, 0, 0) X(8tap_regular_smooth, 0, 1) X(8tap_regular_sharp, 0, 2)                \
  X(8tap_smooth_regular, 1, 0) X(8tap_smooth, 1, 1) X(8tap_smooth_sharp, 1, 2)                  \
  X(8tap_sharp_regular, 2, 0) X(8tap_sharp_smooth, 2, 1) X(8tap_sharp, 2, 2) X(bilin, 3, 3)
#define B200_DECL_MC(NAME, MX, MY)                                                                            \
  void rav1e_put_##NAME##_8bpc_cuda(uint8_t *dst, ptrdiff_t dst_stride, const uint8_t *src,                   \
                                    ptrdiff_t src_stride, int w, int h, int mx, int my);                      \
  void rav1e_put_##NAME##_16bpc_cuda(uint16_t *dst, ptrdiff_t dst_stride, const uint16_t *src,                \
                                     ptrdiff_t src_stride, int w, int h, int mx, int my, int bitdepth_max);   \
  void rav1e_prep_##NAME##_8bpc_cuda(int16_t *tmp, const uint8_t *src, ptrdiff_t src_stride, int w, int h,    \
                                     int mx, int my);                                                         \
  void rav1e_prep_##NAME##_16bpc_cuda(int16_t *tmp, const uint16_t *src, ptrdiff_t src_stride, int w, int h,  \
                                      int mx, int my, int bitdepth_max);
B200_FOR_EACH_MC_FILTER(B200_DECL_MC)
#undef B200_DECL_MC
void rav1e_avg_8bpc_cuda(uint8_t *dst, ptrdiff_t dst_stride, const int16_t *tmp1, const int16_t *tmp2, int w,
                         int h);
void rav1e_avg_16bpc_cuda(uint16_t *dst, ptrdiff_t dst_stride, const int16_t *tmp1, const int16_t *tmp2, int w,
                          int h, int bitdepth_max);

/* X(name, PredictionMode, PredictionVariant): asm/x86/predict.rs:21-120.  `topleft` = IntraEdge::
 * top_left_ptr() (element 128 of the 257-pixel buffer, partition.rs:600-627). */
#define B200_FOR_EACH_IPRED(X)                                                              \
  X(dc, 0, 3) X(dc_128, 0, 0) X(dc_left, 0, 1) X(dc_top, 0, 2) X(v, 1, 3) X(h, 2, 3)        \
  X(smooth, 9, 3) X(smooth_v, 10, 3) X(smooth_h, 11, 3) X(paeth, 12, 3)
#define B200_DECL_IPRED(NAME, MODE, VAR)                                                                      \
  void rav1e_ipred_##NAME##_8bpc_cuda(uint8_t *dst, ptrdiff_t stride, const uint8_t *topleft, int width,      \
                                      int height, int angle);                                                 \
  void rav1e_ipred_##NAME##_16bpc_cuda(uint16_t *dst, ptrdiff_t stride, const uint16_t *topleft, int width,   \
                                       int height, int angle, int max_width, int max_height,                  \
                                       int bitdepth_max);
B200_FOR_EACH_IPRED(B200_DECL_IPRED)
#undef B200_DECL_IPRED
/* directional zones; `angle` = degrees | enable_ief << 10 | smooth << 9 (asm/x86/predict.rs:287-322);
 * z2: dx, dy = distance from the block to the frame edge rounded up to 8 (:304-313) */
void rav1e_ipred_z1_8bpc_cuda(uint8_t *dst, ptrdiff_t stride, const uint8_t *topleft, int width, int height,
                              int angle);
void rav1e_ipred_z2_8bpc_cuda(uint8_t *dst, ptrdiff_t stride, const uint8_t *topleft, int width, int height,
                              int angle, int dx, int dy);
void rav1e_ipred_z3_8bpc_cuda(uint8_t *dst, ptrdiff_t stride, const uint8_t *topleft, int width, int height,
                              int angle);
void rav1e_ipred_z1_16bpc_cuda(uint16_t *dst, ptrdiff_t stride, const uint16_t *topleft, int width, int height,
                               int angle, int max_width, int max_height, int bitdepth_max);
void rav1e_ipred_z2_16bpc_cuda(uint16_t *dst, ptrdiff_t stride, const uint16_t *topleft, int width, int height,
                               int angle, int dx, int dy, int bitdepth_max);
void rav1e_ipred_z3_16bpc_cuda(uint16_t *dst, ptrdiff_t stride, const uint16_t *topleft, int width, int height,
                               int angle, int max_width, int max_height, int bitdepth_max);
/* X(name, PredictionVariant): asm/x86/predict.rs:188-234 */
#define B200_FOR_EACH_CFL(X) X(cfl, 3) X(cfl_128, 0) X(cfl_left, 1) X(cfl_top, 2)
#define B200_DECL_CFL(NAME, VAR)                                                                              \
  void rav1e_ipred_##NAME##_8bpc_cuda(uint8_t *dst, ptrdiff_t stride, const uint8_t *topleft, int width,      \
                                      int height, const int16_t *ac, int alpha);                              \
  void rav1e_ipred_##NAME##_16bpc_cuda(uint16_t *dst, ptrdiff_t stride, const uint16_t *topleft, int width,   \
                                       int height, const int16_t *ac, int alpha, int bitdepth_max);
B200_FOR_EACH_CFL(B200_DECL_CFL)
#undef B200_DECL_CFL
/* X(layout, xdec, ydec): asm/x86/predict.rs:142-186 */
#define B200_FOR_EACH_CFL_AC(X) X(420, 1, 1) X(422, 1, 0) X(444, 0, 0)
#define B200_DECL_CFL_AC(NAME, XDEC, YDEC)                                                                    \
  void rav1e_ipred_cfl_ac_##NAME##_8bpc_cuda(int16_t *ac, const uint8_t *src, ptrdiff_t stride, int w_pad,    \
                                             int h_pad, int width, int height);                               \
  void rav1e_ipred_cfl_ac_##NAME##_16bpc_cuda(int16_t *ac, const uint16_t *src, ptrdiff_t stride, int w_pad,  \
                                              int h_pad, int width, int height);
B200_FOR_EACH_CFL_AC(B200_DECL_CFL_AC)
#undef B200_DECL_CFL_AC

/* X(size, xdec, ydec): CdefFilterFn, slot decimate_index(xdec, ydec) (asm/x86/cdef.rs:16-42, :146-167).
 * The reference has no HBD filter asm (its CDEF_FILTER_HBD_FNS table is empty, :174-178): the
 * `_16bpc` forms take CdefFilterHBDFn's argument list (:27-37) over the same padded u16 tile. */
#define B200_FOR_EACH_CDEF_SIZE(X) X(4x4, 1, 1) X(4x8, 1, 0) X(8x8, 0, 0)
#define B200_DECL_CDEF(NAME, XDEC, YDEC)                                                                      \
  void rav1e_cdef_filter_##NAME##_cuda(uint8_t *dst, ptrdiff_t dst_stride, const uint16_t *tmp,               \
                                       ptrdiff_t tmp_stride, int pri_strength, int sec_strength, int dir,     \
                                       int damping);                                                          \
  void rav1e_cdef_filter_##NAME##_16bpc_cuda(uint16_t *dst, ptrdiff_t dst_stride, const uint16_t *tmp,        \
                                             ptrdiff_t tmp_stride, int pri_strength, int sec_strength,        \
                                             int dir, int damping, int bitdepth_max);
B200_FOR_EACH_CDEF_SIZE(B200_DECL_CDEF)
#undef B200_DECL_CDEF
int32_t rav1e_cdef_dir_8bpc_cuda(const uint8_t *img, ptrdiff_t stride, uint32_t *var);
int32_t rav1e_cdef_dir_16bpc_cuda(const uint16_t *img, ptrdiff_t stride, uint32_t *var, int bitdepth_max);

#ifdef __cplusplus
}
#endif
#endif /* B200RDO_H */
