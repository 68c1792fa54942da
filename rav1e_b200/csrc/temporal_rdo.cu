// temporal_rdo.cu — temporal RDO on the device (sm_90a): block importances propagated across the
// lookahead window, the distortion scales derived from them, and their normalisation.
//
//   update_block_importances        src/api/internal.rs:912-1071
//   compute_block_importances       src/api/internal.rs:1075-1230
//   distortion_scale_for            src/rdo.rs:506-553 (+ DistortionScale::new / From<f64>, :579-583, :652-658)
//   compute_{spatio,}temporal_scores  src/encoder.rs:744-777 (inv_mean, Mul, blog64: rdo.rs:585-630)
//   blog32_q11 / bexp64 / blog64    src/util/logexp.rs (restated in logexp_dev.cuh)
//
// The propagation is a scatter: every source block splits its amount over the four blocks its
// motion-compensated position overlaps, and the reference adds into each destination in source
// raster order.  f32 addition does not reassociate, so the device reproduces that order exactly
// and uses no atomics:
//   pass A (one launch over every step x source block): SATD, inter cost, sub-block offsets and a
//           bucket key = the top-left destination on the ring grid [-1, w_imp) x [-1, h_imp), or
//           "none" when all four destinations fall outside;
//   a stable radix sort of source indices by (step, key) (CUB), then the bucket boundaries;
//   pass B (one launch per step, in the caller's order): one thread per destination merges the four
//           buckets that can reach it by source index and adds the amounts in that order.
// Every f32 operation is an explicit _rn intrinsic: nvcc would otherwise contract a*b+c into an FMA,
// which the reference never does.
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "hadamard.cuh"
#include "logexp_dev.cuh"

namespace {

constexpr uint32_t DS_SHIFT = 14;
constexpr uint32_t DS_MAX = (1u << 28) - 1;

struct StepDesc {
  PlaneView src, dst;
  const short *mvs;         // (row, col) per importance block of the source frame
  const uint32_t *intra;    // the source frame's intra-cost map, read flat
  const float *future;      // the source frame's importances (final when the step runs)
  float *imp_dst;           // the reference frame's importances
  float len;                // number of unique references of the source frame
  int rows;                 // min(h_imp, n_intra / w_imp): rows that propagate
};

// floor(v / 64) for the split (internal.rs:1010-1017), v in MV units
__device__ __forceinline__ int floor_div64(int v) { return v >> 6; }

// ---- pass A
template <typename T>
__global__ void __launch_bounds__(128) imp_pass_a(const StepDesc *steps, int nsteps, int w_imp, int h_imp,
                                                  uint32_t *keys, uint32_t *vals, uint32_t *inter,
                                                  uint16_t *fxy) {
  const int n_imp = w_imp * h_imp, w1 = w_imp + 1, nk = w1 * (h_imp + 1);
  const long long total = (long long)nsteps * n_imp;
  for (long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x; g < total;
       g += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(g / n_imp), i = (int)(g - (long long)s * n_imp);
    const int y = i / w_imp, x = i - y * w_imp;
    const StepDesc &st = steps[s];
    uint32_t key = nk, satd = 0, f = 0;
    if (y < st.rows) {
      const int rx = 64 * x + (int)st.mvs[2 * i + 1], ry = 64 * y + (int)st.mvs[2 * i];
      const int sx = rx / 8, sy = ry / 8;  // truncating toward zero, as `isize / 8`
      int d[64];
#pragma unroll
      for (int r = 0; r < 8; r++)
#pragma unroll
        for (int c = 0; c < 8; c++) d[r * 8 + c] = *px<T>(st.src, 8 * x + c, 8 * y + r) - *px<T>(st.dst, sx + c, sy + r);
      satd = satd8x8(d);
      const int bx = floor_div64(rx), by = floor_div64(ry);
      f = (uint32_t)(rx - 64 * bx) | (uint32_t)(ry - 64 * by) << 8;
      if (bx >= -1 && by >= -1 && bx < w_imp && by < h_imp) key = (uint32_t)((by + 1) * w1 + bx + 1);
    }
    keys[g] = (uint32_t)s * (uint32_t)(nk + 1) + key;
    vals[g] = (uint32_t)i;
    inter[g] = satd;
    fxy[g] = (uint16_t)f;
  }
}

// begin[k] / end[k] of every non-empty bucket of the sorted keys (the arrays start zeroed = empty)
__global__ void bucket_bounds(const uint32_t *keys, long long n, uint32_t *begin, uint32_t *end) {
  for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < n; j += (long long)gridDim.x * blockDim.x) {
    const uint32_t k = keys[j];
    if (j == 0 || keys[j - 1] != k) begin[k] = (uint32_t)j;
    if (j == n - 1 || keys[j + 1] != k) end[k] = (uint32_t)(j + 1);
  }
}

// ---- pass B: step s, one thread per destination block
__global__ void __launch_bounds__(128) imp_pass_b(const StepDesc *steps, int s, int w_imp, int h_imp,
                                                  const uint32_t *sorted_src, const uint32_t *begin,
                                                  const uint32_t *end, const uint32_t *inter, const uint16_t *fxy) {
  const int n_imp = w_imp * h_imp, w1 = w_imp + 1, nk = w1 * (h_imp + 1);
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n_imp) return;
  const StepDesc st = steps[s];
  const int dy = d / w_imp, dx = d - dy * w_imp;
  // buckets whose top-left destination is d, d - (1, 0), d - (0, 1), d - (1, 1): d is their TL, TR, BL, BR
  const uint32_t base = (uint32_t)s * (uint32_t)(nk + 1);
  const uint32_t k[4] = {base + (uint32_t)((dy + 1) * w1 + dx + 1), base + (uint32_t)((dy + 1) * w1 + dx),
                         base + (uint32_t)(dy * w1 + dx + 1), base + (uint32_t)(dy * w1 + dx)};
  uint32_t p[4], e[4];
#pragma unroll
  for (int c = 0; c < 4; c++) {
    p[c] = begin[k[c]];
    e[c] = end[k[c]];
  }
  const long long gbase = (long long)s * n_imp;
  float acc = st.imp_dst[d];
  for (;;) {
    int c = -1;
    uint32_t best = 0xffffffffu;
#pragma unroll
    for (int q = 0; q < 4; q++)
      if (p[q] < e[q] && sorted_src[p[q]] < best) {
        best = sorted_src[p[q]];
        c = q;
      }
    if (c < 0) break;
    p[c]++;
    const long long g = gbase + best;
    const float inter_c = __uint2float_rn(inter[g]), intra_c = __uint2float_rn(st.intra[best]);
    const float frac = intra_c <= inter_c ? 0.f : __fsub_rn(1.f, __fdiv_rn(inter_c, intra_c));
    const float amount = __fdiv_rn(__fmul_rn(__fadd_rn(intra_c, st.future[best]), frac), st.len);
    const int fx = fxy[g] & 0xff, fy = fxy[g] >> 8;
    const int wx = (c & 1) ? fx : 64 - fx, wy = (c & 2) ? fy : 64 - fy;
    const float weight = __fdiv_rn(__int2float_rn(wx * wy), 4096.f);
    acc = __fadd_rn(acc, __fmul_rn(amount, weight));
  }
  st.imp_dst[d] = acc;
}

// DistortionScale's Mul (rdo.rs:618-630)
__device__ __forceinline__ uint32_t ds_mul(uint32_t a, uint32_t b) {
  const unsigned long long v = ((unsigned long long)a * b + (1u << (DS_SHIFT - 1))) >> DS_SHIFT;
  return v < 1 ? 1u : v > DS_MAX ? DS_MAX : (uint32_t)v;
}

// ---- distortion_scale_for per importance block (internal.rs:1219-1230)
__global__ void distortion_scales_kernel(const float *imp, const uint32_t *intra, int n_imp, int n_intra,
                                         uint32_t *scales) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_imp) return;
  uint32_t out = 1u << DS_SHIFT;
  if (i < n_intra && intra[i] != 0) {
    const double ic = __uint2double_rn(intra[i]);
    const double s = pow(__ddiv_rn(__dadd_rn(ic, (double)imp[i]), ic), 1.0 / 3.0);
    // From<f64>: (s * 32768) as u64 (s >= 1: no saturation), then DistortionScale::new(num, 32768)
    const unsigned long long num = __double2ull_rz(__dmul_rn(s, 32768.0));
    const unsigned long long sh = num << DS_SHIFT;
    const unsigned long long raw = (sh > ~0ull - 16384 ? ~0ull : sh + 16384) / 32768;
    out = raw <= DS_MAX ? (uint32_t)raw : DS_MAX;
  }
  scales[i] = out;
}

// ---- scores: sum of blog32_q11 (exact i64, order-free), inv_mean, then the scaling
__global__ void scores_log_sum(const uint32_t *scales, const uint32_t *activity, uint32_t *spatio, int n,
                               unsigned long long *sum) {
  long long mine = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    uint32_t v = scales[i];
    if (activity) {
      v = ds_mul(v, activity[i]);
      spatio[i] = v;
    }
    mine += blog32_q11(v);
  }
  unsigned long long u = (unsigned long long)mine;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) u += __shfl_xor_sync(0xffffffffu, u, o);
  if ((threadIdx.x & 31) == 0 && u) atomicAdd(sum, u);
}

__global__ void scores_inv_mean(const unsigned long long *sum, int n, uint32_t *inv_mean, long long *log_isqrt) {
  // DistortionScale::inv_mean (rdo.rs:585-594)
  const long long log_inv_mean_q11 = ((long long)DS_SHIFT << 11) - (long long)*sum / n;
  const long long e = bexp64((long long)((unsigned long long)(log_inv_mean_q11 + ((long long)DS_SHIFT << 11)) << 46));
  const uint32_t inv = e < 1 ? 1u : e > (long long)DS_MAX ? DS_MAX : (uint32_t)e;
  *inv_mean = inv;
  if (log_isqrt) *log_isqrt = (blog64((long long)inv) - q57(DS_SHIFT)) >> 1;  // DistortionScale::blog64() >> 1
}

__global__ void scores_apply(uint32_t *scales, uint32_t *spatio, int spatio_is_product, int w_imp, int h_imp,
                             const uint32_t *inv_mean, uint32_t *scale4x4, size_t stride4) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w_imp * h_imp) return;
  const uint32_t inv = *inv_mean;
  const uint32_t d = ds_mul(scales[i], inv);
  scales[i] = d;
  if (spatio) spatio[i] = spatio_is_product ? ds_mul(spatio[i], inv) : d;
  if (scale4x4) {
    // sse_wxh's bias per 4x4 luma chunk (rdo.rs:177-224): distortion_scale() of the importance block
    // holding the chunk (rdo.rs:443-459, IMPORTANCE_BLOCK_TO_BLOCK_SHIFT = 1)
    const int y = i / w_imp, x = i - y * w_imp;
    uint32_t *row = scale4x4 + (size_t)(2 * y) * stride4 + 2 * x;
    row[0] = row[1] = row[stride4] = row[stride4 + 1] = d;
  }
}

int check_planes(b200_ctx *ctx, size_t nframes, const b200_plane *frames, int bit_depth) {
  B200_REQUIRE(ctx, frames != nullptr && nframes > 0, "no frames");
  const b200_plane &f0 = frames[0];
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bit depth %d not in {8,10,12}", bit_depth);
  B200_REQUIRE(ctx, (f0.bpp == 1) == (bit_depth == 8) && (f0.bpp == 1 || f0.bpp == 2), "bpp %d vs bit depth %d",
               f0.bpp, bit_depth);
  B200_REQUIRE(ctx, f0.width > 0 && f0.height > 0, "empty frame");
  const int w_imp = (f0.width + 7) / 8, h_imp = (f0.height + 7) / 8;
  for (size_t f = 0; f < nframes; f++) {
    const b200_plane &p = frames[f];
    B200_REQUIRE(ctx, p.data != nullptr, "frame %zu: NULL plane", f);
    B200_REQUIRE(ctx, p.width == f0.width && p.height == f0.height && p.bpp == f0.bpp,
                 "frame %zu: %dx%d bpp %d differs from frame 0 (%dx%d bpp %d)", f, p.width, p.height, p.bpp,
                 f0.width, f0.height, f0.bpp);
    // blocks of the ceil grid past the frame edge read the padding
    B200_REQUIRE(ctx, p.pad >= 8 * w_imp - p.width && p.pad >= 8 * h_imp - p.height,
                 "frame %zu: padding %d does not cover the last importance block", f, p.pad);
  }
  return B200_OK;
}

}  // namespace

extern "C" int b200_block_importances_dev(b200_ctx *ctx, size_t nframes, const b200_plane *frames, int bit_depth,
                                          const uint32_t *d_intra_costs, const int16_t *d_mvs, size_t nsteps,
                                          const b200_imp_step *steps, float *d_importances) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (int st = check_planes(ctx, nframes, frames, bit_depth)) return st;
  B200_REQUIRE(ctx, d_importances != nullptr, "NULL importances");
  B200_REQUIRE(ctx, nsteps == 0 || (steps && d_intra_costs && d_mvs), "NULL steps / intra costs / motion vectors");
  const int W = frames[0].width, H = frames[0].height;
  const int w_imp = (W + 7) / 8, h_imp = (H + 7) / 8, n_imp = w_imp * h_imp;
  const size_t n_intra = (size_t)(W / 8) * (H / 8);
  const long long nk1 = (long long)(w_imp + 1) * (h_imp + 1) + 1;  // ring-grid keys + "none", per step
  B200_REQUIRE(ctx, (long long)nsteps * nk1 < (1ll << 32) && (long long)nsteps * n_imp < (1ll << 31),
               "window too large (%zu steps of %d blocks)", nsteps, n_imp);
  // the reference's preconditions: no frame is its own reference (internal.rs:1181); a step reads its
  // source's importances, which must be final (every step into that frame comes earlier)
  std::vector<long long> last_into(nframes, -1);
  for (size_t k = 0; k < nsteps; k++) {
    const b200_imp_step &s = steps[k];
    B200_REQUIRE(ctx, s.src < nframes && s.dst < nframes, "step %zu: frame index outside the window of %zu", k,
                 nframes);
    B200_REQUIRE(ctx, s.src != s.dst, "step %zu: frame %u references itself", k, s.src);
    B200_REQUIRE(ctx, s.len >= 1 && s.len <= 3, "step %zu: len %u outside 1..3", k, s.len);
    last_into[s.dst] = (long long)k;
  }
  for (size_t k = 0; k < nsteps; k++)
    B200_REQUIRE(ctx, last_into[steps[k].src] < (long long)k,
                 "step %zu reads frame %u, which a later step (%lld) still propagates into", k, steps[k].src,
                 last_into[steps[k].src]);
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  B200_CUDA(ctx, cudaMemsetAsync(d_importances, 0, nframes * (size_t)n_imp * sizeof(float), ctx->stream));
  if (nsteps == 0) return B200_OK;

  const size_t N = nsteps * (size_t)n_imp, nkeys = nsteps * (size_t)nk1;
  int end_bit = 1;
  while ((1ull << end_bit) < (unsigned long long)nkeys) end_bit++;
  size_t sort_bytes = 0;
  B200_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                                 (const uint32_t *)nullptr, (uint32_t *)nullptr, N, 0, end_bit,
                                                 ctx->stream));
  // workspace: descriptors | keys in/out | vals in/out | inter | fxy | begin | end | sort temp
  size_t off = 0;
  auto carve = [&](size_t bytes) {
    const size_t o = off;
    off = b200_align_up(off + bytes, 256);
    return o;
  };
  const size_t o_desc = carve(nsteps * sizeof(StepDesc)), o_kin = carve(4 * N), o_kout = carve(4 * N),
               o_vin = carve(4 * N), o_vout = carve(4 * N), o_inter = carve(4 * N), o_fxy = carve(2 * N),
               o_begin = carve(4 * nkeys), o_end = carve(4 * nkeys), o_sort = carve(sort_bytes);
  if (int st = b200_reserve_dwork(ctx, off)) return st;
  uint8_t *ws = (uint8_t *)ctx->dwork;
  StepDesc *d_desc = (StepDesc *)(ws + o_desc);
  uint32_t *kin = (uint32_t *)(ws + o_kin), *kout = (uint32_t *)(ws + o_kout), *vin = (uint32_t *)(ws + o_vin),
           *vout = (uint32_t *)(ws + o_vout), *inter = (uint32_t *)(ws + o_inter), *begin = (uint32_t *)(ws + o_begin),
           *end = (uint32_t *)(ws + o_end);
  uint16_t *fxy = (uint16_t *)(ws + o_fxy);

  std::vector<StepDesc> desc(nsteps);
  const int rows = (int)std::min<size_t>((size_t)h_imp, n_intra / (size_t)w_imp);
  for (size_t k = 0; k < nsteps; k++) {
    const b200_imp_step &s = steps[k];
    desc[k].src = PlaneView{frames[s.src].data, frames[s.src].stride};
    desc[k].dst = PlaneView{frames[s.dst].data, frames[s.dst].stride};
    desc[k].mvs = (const short *)d_mvs + (size_t)s.mv_index * 2 * n_imp;
    desc[k].intra = d_intra_costs + (size_t)s.src * n_intra;
    desc[k].future = d_importances + (size_t)s.src * n_imp;
    desc[k].imp_dst = d_importances + (size_t)s.dst * n_imp;
    desc[k].len = (float)s.len;
    desc[k].rows = rows;
  }
  // pageable source: the call returns once the descriptors are staged, so `desc` may go out of scope
  B200_CUDA(ctx, cudaMemcpyAsync(d_desc, desc.data(), nsteps * sizeof(StepDesc), cudaMemcpyHostToDevice, ctx->stream));
  B200_CUDA(ctx, cudaMemsetAsync(begin, 0, 4 * nkeys, ctx->stream));
  B200_CUDA(ctx, cudaMemsetAsync(end, 0, 4 * nkeys, ctx->stream));

  const int grid_a = (int)std::min<size_t>((N + 127) / 128, (size_t)ctx->num_sms * 16);
  if (frames[0].bpp == 1)
    imp_pass_a<uint8_t><<<grid_a, 128, 0, ctx->stream>>>(d_desc, (int)nsteps, w_imp, h_imp, kin, vin, inter, fxy);
  else
    imp_pass_a<uint16_t><<<grid_a, 128, 0, ctx->stream>>>(d_desc, (int)nsteps, w_imp, h_imp, kin, vin, inter, fxy);
  B200_LAUNCH_CHECK(ctx);
  // LSD radix sort: stable, so every bucket keeps its sources in raster order
  B200_CUDA(ctx, cub::DeviceRadixSort::SortPairs(ws + o_sort, sort_bytes, kin, kout, vin, vout, N, 0, end_bit,
                                                 ctx->stream));
  B200_LAUNCH_CHECK(ctx);
  const int grid_n = (int)std::min<size_t>((N + 255) / 256, (size_t)ctx->num_sms * 16);
  bucket_bounds<<<grid_n, 256, 0, ctx->stream>>>(kout, (long long)N, begin, end);
  B200_LAUNCH_CHECK(ctx);
  for (size_t k = 0; k < nsteps; k++) {
    imp_pass_b<<<(n_imp + 127) / 128, 128, 0, ctx->stream>>>(d_desc, (int)k, w_imp, h_imp, vout, begin, end, inter, fxy);
    B200_LAUNCH_CHECK(ctx);
  }
  return B200_OK;
}

extern "C" int b200_distortion_scales_dev(b200_ctx *ctx, const b200_plane *frame, const float *d_importances,
                                          const uint32_t *d_intra_costs, uint32_t *d_scales) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, frame && frame->width > 0 && frame->height > 0, "NULL / empty frame");
  const int w_imp = (frame->width + 7) / 8, h_imp = (frame->height + 7) / 8, n_imp = w_imp * h_imp;
  const int n_intra = (frame->width / 8) * (frame->height / 8);
  B200_REQUIRE(ctx, d_importances && d_scales && (n_intra == 0 || d_intra_costs), "NULL importances / costs / scales");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  distortion_scales_kernel<<<(n_imp + 127) / 128, 128, 0, ctx->stream>>>(d_importances, d_intra_costs, n_imp, n_intra,
                                                                         d_scales);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_temporal_scores_dev(b200_ctx *ctx, size_t w_imp, size_t h_imp, uint32_t *d_scales,
                                        const uint32_t *d_activity, uint32_t *d_spatiotemporal,
                                        int64_t *d_log_isqrt_mean_scale, uint32_t *d_scale4x4,
                                        size_t scale4x4_stride) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  // each side bounded first, so that the product cannot wrap
  B200_REQUIRE(ctx, w_imp > 0 && h_imp > 0 && w_imp < (1u << 30) && h_imp < (1u << 30) && w_imp * h_imp < (1u << 30),
               "bad map size %zu x %zu", w_imp, h_imp);
  B200_REQUIRE(ctx, d_scales != nullptr, "NULL scales");
  B200_REQUIRE(ctx, !d_activity || d_spatiotemporal, "the spatiotemporal form needs d_spatiotemporal");
  B200_REQUIRE(ctx, !d_scale4x4 || scale4x4_stride >= 2 * w_imp, "4x4 map stride %zu < %zu", scale4x4_stride,
               2 * w_imp);
  const int n = (int)(w_imp * h_imp);
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  if (int st = b200_reserve_dwork(ctx, 16)) return st;
  unsigned long long *d_sum = (unsigned long long *)ctx->dwork;
  uint32_t *d_inv = (uint32_t *)((uint8_t *)ctx->dwork + 8);
  B200_CUDA(ctx, cudaMemsetAsync(d_sum, 0, 8, ctx->stream));
  const int grid = std::min((n + 255) / 256, ctx->num_sms * 8);
  scores_log_sum<<<grid, 256, 0, ctx->stream>>>(d_scales, d_activity, d_spatiotemporal, n, d_sum);
  B200_LAUNCH_CHECK(ctx);
  scores_inv_mean<<<1, 1, 0, ctx->stream>>>(d_sum, n, d_inv, (long long *)d_log_isqrt_mean_scale);
  B200_LAUNCH_CHECK(ctx);
  scores_apply<<<(n + 127) / 128, 128, 0, ctx->stream>>>(d_scales, d_spatiotemporal, d_activity != nullptr, (int)w_imp,
                                                         (int)h_imp, d_inv, d_scale4x4, scale4x4_stride);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
