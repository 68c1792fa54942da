// segmentation.cu — rav1e's adaptive quantization on the device (sm_90a): segmentation_optimize's k-means
// of the frame's log-domain spatiotemporal scores, the segment quantizers and thresholds, and select_segment
// for batches of blocks.
//
//   segmentation_optimize{,_inner}   src/segmentation.rs:23-160
//   kmeans / scan                    src/util/kmeans.rs:11-102
//   select_ac_qi / select_qi / ac_q  src/quantize/mod.rs:44-97
//   update_threshold                 src/encoder.rs:564-580
//   get_qidx                         src/encoder.rs:1383-1394
//   select_segment                   src/segmentation.rs:163-196
//   spatiotemporal_scale             src/rdo.rs:464-504
//   DistortionScale::{new, blog16}   src/rdo.rs:578-601
//
// The k-means runs on a histogram of the i16 log values instead of the sorted vector.  The reference's
// incremental `scan` leaves high[i] = upper_bound(t_i) and low[i + 1] = lower_bound(t_i) whatever they were
// before, and keeps sum[i] = P[high[i]] - P[low[i]] for the prefix sums P of the sorted data (the walks add
// and remove exactly the elements between the old and the new bound).  Both bounds fall on value
// boundaries, where the exclusive prefix sums of the histogram's counts and of value x count are P's
// indices and values, so one iteration is a pair of table reads per cluster.  The initial means
// data[(i * (n - 1)) / (K - 1)] are found by rank with a binary search over the count prefix sums.
#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"
#include "logexp_dev.cuh"

namespace {

constexpr int kBins = 1 << 16;  // every i16 value: blog16 wraps for scores past 2^28, as `as i16` does
constexpr int kScanThreads = 512;
constexpr int kBinsPerWarp = kBins / (kScanThreads / 32);
constexpr uint32_t DS_SHIFT = 14, DS_MAX = (1u << 28) - 1;
constexpr int ALT_Q = 0, SEG_LVL_REF_FRAME = 5;

struct AcTable {
  uint16_t q[256];
};

// BlockSize::width_imp_b() / height_imp_b() (partition.rs:267-303) by BlockSize discriminant
__constant__ uint8_t kImpW[22] = {1, 1, 1, 1, 1, 2, 2, 2, 4, 4, 4, 8, 8, 8, 16, 16, 1, 2, 1, 4, 2, 8};
__constant__ uint8_t kImpH[22] = {1, 1, 1, 1, 2, 1, 2, 4, 2, 4, 8, 4, 8, 16, 8, 16, 2, 1, 4, 1, 8, 2};

// DistortionScale::blog16: blog32_q11(s) - (14 << 11), as i16; its histogram bin
__device__ __forceinline__ int log_bin(uint32_t s) {
  return (uint16_t)(int16_t)(blog32_q11(s) - (int)(DS_SHIFT << 11)) ^ 0x8000u;
}

__global__ void __launch_bounds__(256) seg_histogram(const uint32_t *scores, int n, uint32_t *hist) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    atomicAdd(&hist[log_bin(scores[i])], 1u);
}

// DistortionScale::new (rdo.rs:578-583)
__device__ __forceinline__ uint32_t ds_new(unsigned long long num, unsigned long long den) {
  const unsigned long long sh = num << DS_SHIFT;
  const unsigned long long raw = (sh > ~0ull - den / 2 ? ~0ull : sh + den / 2) / den;
  return raw <= DS_MAX ? (uint32_t)raw : DS_MAX;
}

// select_qi (quantize/mod.rs:52-77) over a strictly increasing table: binary_search's Ok / Err index is
// the lower bound; the i32 products wrap as in a release build
__device__ int select_qi(long long quantizer, const uint16_t *t) {
  if (quantizer < t[0]) return 0;
  if (quantizer >= t[255]) return 255;
  int lo = 0, hi = 255;  // t[lo] <= quantizer < t[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (t[mid] <= quantizer) lo = mid; else hi = mid;
  }
  if (t[lo] == quantizer) return lo;
  const int32_t qthresh = (int32_t)((uint32_t)t[hi - 1] * (uint32_t)t[hi]);
  const int32_t q2 = (int32_t)((uint32_t)quantizer * (uint32_t)quantizer);
  return q2 < qthresh ? hi - 1 : hi;
}

// SegmentationState::update_threshold (encoder.rs:566-580); max_segment <= 7
__device__ void update_threshold(b200_segmentation &s, int base, const uint16_t *ac) {
  const unsigned long long base_ac_q = ac[base];
  for (int i = 0; i < 7; i++) s.threshold[i] = 0;
  // real_ac_q[i] = ac_q(base, data[i] as i8, bd)
  unsigned long long q1 = ac[min(max(base + (int)(int8_t)s.data[0][ALT_Q], 0), 255)];
  for (int i = 0; i < s.max_segment; i++) {
    const unsigned long long q2 = ac[min(max(base + (int)(int8_t)s.data[i + 1][ALT_Q], 0), 255)];
    s.threshold[i] = ds_new(base_ac_q * base_ac_q, q2 * q1);
    q1 = q2;
  }
}

// One CTA: the exclusive prefix sums of the histogram (counts -> cex, value x count -> sex, kBins + 1
// entries each; coalesced, a warp scan per 128 bins), one warp per k = 8 - warp for the k-means, then
// thread 0 for the rest of segmentation_optimize.  update_data == 0 needs none of the tables.
__global__ void __launch_bounds__(kScanThreads) seg_optimize_kernel(const uint32_t *hist, uint32_t *cex,
                                                                    long long *sex, int base, AcTable ac,
                                                                    int update_data,
                                                                    const b200_segmentation *prev,
                                                                    b200_segmentation *out) {
  __shared__ uint32_t wc[32];
  __shared__ long long ws[32];
  __shared__ int16_t cent[6][8];
  __shared__ uint16_t acq[256];
  __shared__ b200_segmentation s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 256; i += blockDim.x) acq[i] = ac.q[i];
  if (tid == 0) {
    if (prev)
      s = *prev;
    else
      memset(&s, 0, sizeof s);  // SegmentationState::default()
  }
  __syncthreads();
  if (update_data) {
    // ---- scan: warp w owns bins [4096 w, 4096 w + 4096), lane l bins 4 l .. 4 l + 3 of every 128
    const int wb0 = warp * kBinsPerWarp;
    uint32_t c = 0;
    long long sv = 0;
    for (int k = 4 * lane; k < kBinsPerWarp; k += 128) {
      const uint4 h = *(const uint4 *)(hist + wb0 + k);
      const long long v = wb0 + k - 32768;
      c += h.x + h.y + h.z + h.w;
      sv += (long long)h.x * v + (long long)h.y * (v + 1) + (long long)h.z * (v + 2) + (long long)h.w * (v + 3);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      c += __shfl_xor_sync(0xffffffffu, c, o);
      sv += __shfl_xor_sync(0xffffffffu, sv, o);
    }
    if (lane == 0) {
      wc[warp] = c;
      ws[warp] = sv;
    }
    __syncthreads();
    if (tid == 0) {  // exclusive prefix over the warps
      uint32_t rc = 0;
      long long rs = 0;
      for (int w = 0; w < kScanThreads / 32; w++) {
        const uint32_t tc = wc[w];
        const long long ts = ws[w];
        wc[w] = rc;
        ws[w] = rs;
        rc += tc;
        rs += ts;
      }
    }
    __syncthreads();
    uint32_t carry_c = wc[warp];
    long long carry_s = ws[warp];
    for (int k = 4 * lane; k < kBinsPerWarp; k += 128) {
      const uint4 h = *(const uint4 *)(hist + wb0 + k);
      const long long v = wb0 + k - 32768;
      const uint32_t lc = h.x + h.y + h.z + h.w;
      const long long ls =
          (long long)h.x * v + (long long)h.y * (v + 1) + (long long)h.z * (v + 2) + (long long)h.w * (v + 3);
      uint32_t ic = lc;
      long long is = ls;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t uc = __shfl_up_sync(0xffffffffu, ic, o);
        const long long us = __shfl_up_sync(0xffffffffu, is, o);
        if (lane >= o) {
          ic += uc;
          is += us;
        }
      }
      const uint32_t e0 = carry_c + ic - lc, e1 = e0 + h.x, e2 = e1 + h.y, e3 = e2 + h.z;
      const long long s0 = carry_s + is - ls, s1 = s0 + (long long)h.x * v, s2 = s1 + (long long)h.y * (v + 1),
                      s3 = s2 + (long long)h.z * (v + 2);
      *(uint4 *)(cex + wb0 + k) = make_uint4(e0, e1, e2, e3);
      *(longlong2 *)(sex + wb0 + k) = make_longlong2(s0, s1);
      *(longlong2 *)(sex + wb0 + k + 2) = make_longlong2(s2, s3);
      carry_c += __shfl_sync(0xffffffffu, ic, 31);
      carry_s += __shfl_sync(0xffffffffu, is, 31);
    }
    if (tid == kScanThreads - 1) {
      cex[kBins] = carry_c;
      sex[kBins] = carry_s;
    }
    __syncthreads();

    // ---- kmeans::<i16, K> (kmeans.rs:11-66), K = 8 - warp; lane i < K holds cluster i
    if (warp < 6) {
      const int K = 8 - warp;
      const uint32_t n = cex[kBins];
      const unsigned act = (1u << K) - 1;
      int m = 0;
      if (lane < K) {
        // means[i] = data[(i * (n - 1)) / (K - 1)]: the bin holding that rank
        const uint32_t idx = (uint32_t)(((unsigned long long)lane * (n - 1)) / (K - 1));
        int lo = 0, hi = kBins;
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (cex[mid] <= idx) lo = mid; else hi = mid;
        }
        m = lo - 32768;
      }
      const int limit = 2 * (32 - __clz(n));
      for (int it = 0; it < limit; it++) {
        const int m_next = __shfl_down_sync(0xffffffffu, m, 1);
        const int t = (m_next + m + 1) >> 1;  // threshold between clusters lane and lane + 1
        const int t_prev = __shfl_up_sync(0xffffffffu, t, 1);
        bool changed = false;
        if (lane < K) {
          const int hb = lane == K - 1 ? kBins : t + 32768 + 1;  // high[i] = upper_bound(t_i)
          const int lb = lane == 0 ? 0 : t_prev + 32768;         // low[i] = lower_bound(t_{i-1})
          const long long count = (long long)cex[hb] - (long long)cex[lb];
          if (count != 0) {
            const long long sum = sex[hb] - sex[lb];
            const int nm = (int16_t)((sum + (count >> 1)) / count);
            changed = nm != m;
            m = nm;
          }
        }
        if (!(__ballot_sync(0xffffffffu, changed) & act)) break;
      }
      if (lane < K) cent[warp][lane] = (int16_t)m;
    }
    __syncthreads();
  }
  if (tid != 0) return;
  s.enabled = 1;
  s.update_map = 1;
  s.update_data = (uint8_t)update_data;
  s.pad_ = 0;
  s.status = 0;
  const int offset_lower_limit = 1 - base;
  if (!update_data) {
    int min_segment = 8;
    for (int i = 0; i < 8; i++)
      if (s.features[i][ALT_Q] && s.data[i][ALT_Q] >= offset_lower_limit) {
        min_segment = i;
        break;
      }
    if (min_segment == 8) {
      s.status = 1;
    } else {
      s.min_segment = (uint8_t)min_segment;
      if (s.max_segment > 7)
        s.status = 2;
      else
        update_threshold(s, base, acq);
    }
  } else {
    // variance in spacing of each k's centroids; rposition of the minimum (ties go to the smaller k)
    int position = 0;
    unsigned long long best = ~0ull;
    for (int p = 0; p < 6; p++) {
      const int K = 8 - p;
      long long tot = 0;  // delta[j] = c[j] - c[j + 1]
      for (int j = 0; j < K - 1; j++) tot += (long long)cent[p][j] - cent[p][j + 1];
      const long long mean = tot / (K - 1);
      unsigned long long var = 0;
      for (int j = 0; j < K - 1; j++) {
        const long long d = (long long)cent[p][j] - cent[p][j + 1] - mean;
        var += (unsigned long long)(d * d);
      }
      if (var <= best) {
        best = var;
        position = p;
      }
    }
    // compute_delta: centroids from the largest down, q = base_ac_q / sqrt(scale) in the log domain
    const int K = 8 - position;
    const long long log2_base_ac_q_q57 = blog64((long long)acq[base]);
    s.min_segment = 0;
    s.max_segment = (uint8_t)(K - 1);
    for (int j = 0; j < K; j++) {
      const long long c = cent[position][K - 1 - j];
      const long long q = bexp64(log2_base_ac_q_q57 - (long long)((unsigned long long)c << (57 - 11 - 1)));
      const int delta = max(select_qi(q, acq), 1) - base;
      s.features[j][ALT_Q] = 1;
      s.data[j][ALT_Q] = (int16_t)max(delta, offset_lower_limit);
    }
    update_threshold(s, base, acq);
    s.preskip = 0;
    s.last_active_segid = 0;
    for (int i = 0; i < 8; i++)
      for (int j = 0; j < 8; j++)
        if (s.features[i][j]) {
          s.last_active_segid = (uint8_t)i;
          if (j >= SEG_LVL_REF_FRAME) s.preskip = 1;
        }
  }
  // get_qidx per segment: (qidx as i16) + delta wraps in a release build, then the clamp
  for (int i = 0; i < 8; i++)
    s.qidx[i] = s.features[i][ALT_Q] ? (uint8_t)min(max((int)(int16_t)(base + s.data[i][ALT_Q]), 0), 255)
                                     : (uint8_t)base;
  *out = s;
}

// segment_idx_from_distortion: threshold.partition_point(|&t| s < t) as Rust 1.83's branchless
// binary_search_by runs it over 7 entries (probes 3, then base + 2, base + 1, then base)
__device__ __forceinline__ int segment_idx(const uint32_t *thr, uint32_t s) {
  int size = 7, base = 0;
  while (size > 1) {
    const int half = size / 2, mid = base + half;
    base = s < thr[mid] ? mid : base;
    size -= half;
  }
  return base + (s < thr[base] ? 1 : 0);
}

__global__ void __launch_bounds__(256) select_segment_kernel(const b200_segment_item *items, long long n,
                                                             const uint32_t *scales, const uint32_t *activity,
                                                             int w_imp, int h_imp, int scales_off, int level,
                                                             const b200_segmentation *seg, uint8_t *sidx,
                                                             uint32_t *scale_out) {
  __shared__ uint32_t thr[7];
  if (threadIdx.x < 7) thr[threadIdx.x] = seg->threshold[threadIdx.x];
  __syncthreads();
  const int status = seg->status, min_seg = seg->min_segment, max_seg = seg->max_segment;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const b200_segment_item it = items[i];
    const int x = it.x, y = it.y, bs = it.bsize;
    if (status != 0 || bs >= 22 || x < 0 || y < 0 || (x & 3) || (y & 3) || (x >> 3) >= w_imp || (y >> 3) >= h_imp) {
      sidx[2 * i] = sidx[2 * i + 1] = 0xFF;
      if (scale_out) scale_out[i] = 0xFFFFFFFFu;
      continue;
    }
    uint32_t scale = 1u << DS_SHIFT;
    if (!scales_off) {
      const int x0 = x >> 3, y0 = y >> 3;
      const int x1 = min(x0 + (int)kImpW[bs], w_imp), y1 = min(y0 + (int)kImpH[bs], h_imp);
      const int cols = min(x1 - x0, 16);  // take_slice(.., MAX_SB_IN_IMP_B)
      unsigned long long sum = 0;
      for (int r = y0; r < y1; r++) {
        const size_t row = (size_t)r * w_imp + x0;
        for (int c = 0; c < cols; c++)
          sum += (unsigned long long)scales[row + c] * (activity ? activity[row + c] : 1u << DS_SHIFT);
      }
      const unsigned long long den = (unsigned long long)((x1 - x0) * (y1 - y0)) << DS_SHIFT;
      scale = (uint32_t)((sum + (den >> 1)) / den);
    }
    if (scale_out) scale_out[i] = scale;
    int lo = 0, hi = 0;
    if (!it.skip) {
      if (level == 3) {
        lo = min_seg;
        hi = max_seg;
      } else {
        lo = max(segment_idx(thr, scale), min_seg);
        hi = level == 2 ? min(max_seg, lo + 1) : lo;  // sidx.saturating_add(1): sidx <= 8
      }
    }
    sidx[2 * i] = (uint8_t)lo;
    sidx[2 * i + 1] = (uint8_t)hi;
  }
}

}  // namespace

extern "C" int b200_segmentation_optimize_dev(b200_ctx *ctx, const uint32_t *d_spatiotemporal, size_t w_imp,
                                              size_t h_imp, int base_q_idx, int bit_depth, const uint16_t *ac_q,
                                              int update_data, const b200_segmentation *d_prev,
                                              b200_segmentation *d_out) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, ac_q != nullptr && d_out != nullptr, "NULL ac_q table / output record");
  B200_REQUIRE(ctx, update_data == 0 || update_data == 1, "update_data %d not 0 / 1", update_data);
  B200_REQUIRE(ctx, !update_data || d_spatiotemporal != nullptr, "NULL score map with update_data 1");
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bit depth %d not in {8,10,12}", bit_depth);
  B200_REQUIRE(ctx, base_q_idx >= 0 && base_q_idx <= 255, "base_q_idx %d outside 0..255", base_q_idx);
  B200_REQUIRE(ctx, w_imp > 0 && h_imp > 0 && w_imp < (1u << 30) && h_imp < (1u << 30) && w_imp * h_imp < (1u << 30),
               "bad map size %zu x %zu", w_imp, h_imp);
  AcTable ac;
  B200_REQUIRE(ctx, ac_q[0] != 0, "ac_q[0] is 0");
  for (int i = 0; i < 256; i++) {
    B200_REQUIRE(ctx, i == 0 || ac_q[i] > ac_q[i - 1], "ac_q not strictly increasing at %d (%u after %u)", i,
                 ac_q[i], i ? ac_q[i - 1] : 0);
    ac.q[i] = ac_q[i];
  }
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  uint32_t *hist = nullptr, *cex = nullptr;
  long long *sex = nullptr;
  if (update_data) {
    const size_t o_cex = b200_align_up(4 * (size_t)kBins, 256), o_sex = b200_align_up(o_cex + 4 * (size_t)(kBins + 1), 256);
    if (int st = b200_reserve_dwork(ctx, o_sex + 8 * (size_t)(kBins + 1))) return st;
    uint8_t *ws = (uint8_t *)ctx->dwork;
    hist = (uint32_t *)ws;
    cex = (uint32_t *)(ws + o_cex);
    sex = (long long *)(ws + o_sex);
    const int n = (int)(w_imp * h_imp);
    B200_CUDA(ctx, cudaMemsetAsync(hist, 0, 4 * (size_t)kBins, ctx->stream));
    const int grid = std::min((n + 255) / 256, ctx->num_sms * 8);
    seg_histogram<<<grid, 256, 0, ctx->stream>>>(d_spatiotemporal, n, hist);
    B200_LAUNCH_CHECK(ctx);
  }
  seg_optimize_kernel<<<1, update_data ? kScanThreads : 32, 0, ctx->stream>>>(hist, cex, sex, base_q_idx, ac,
                                                                             update_data, d_prev, d_out);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_select_segment_dev(b200_ctx *ctx, const b200_segment_item *d_items, size_t nitems,
                                       const uint32_t *d_scales, const uint32_t *d_activity, size_t w_imp,
                                       size_t h_imp, int scales_off, int level, const b200_segmentation *d_seg,
                                       uint8_t *d_sidx, uint32_t *d_scale) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, d_seg != nullptr && d_sidx != nullptr, "NULL segmentation record / sidx output");
  B200_REQUIRE(ctx, nitems == 0 || d_items != nullptr, "NULL items");
  B200_REQUIRE(ctx, scales_off || d_scales != nullptr, "NULL distortion scales");
  B200_REQUIRE(ctx, level >= 1 && level <= 3, "segmentation level %d not Simple (1) / Complex (2) / Full (3)", level);
  B200_REQUIRE(ctx, w_imp > 0 && h_imp > 0 && w_imp < (1u << 30) && h_imp < (1u << 30) && w_imp * h_imp < (1u << 30),
               "bad map size %zu x %zu", w_imp, h_imp);
  if (nitems == 0) return B200_OK;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const int grid = (int)std::min<size_t>((nitems + 255) / 256, (size_t)ctx->num_sms * 4);
  select_segment_kernel<<<grid, 256, 0, ctx->stream>>>(d_items, (long long)nitems, d_scales, d_activity, (int)w_imp,
                                                       (int)h_imp, scales_off, level, d_seg, d_sidx, d_scale);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
