/*
 * segmentation.c — literal restatement of rav1e's segmentation (see segmentation.h):
 *   segmentation_optimize{,_inner}   src/segmentation.rs:23-160
 *   select_segment / segment_idx     src/segmentation.rs:163-196
 *   kmeans / scan                    src/util/kmeans.rs:11-102 (on the sorted data, the incremental walks)
 *   ac_q / select_qi                 src/quantize/mod.rs:44-77
 *   update_threshold                 src/encoder.rs:566-580
 *   get_qidx                         src/encoder.rs:1383-1394
 *   spatiotemporal_scale             src/rdo.rs:464-504
 *   DistortionScale::{new, blog16}   src/rdo.rs:578-601
 * Integer semantics are a release build's: i16 / i32 / u64 arithmetic wraps where the reference's would.
 */
#include "segmentation.h"

#include <stdlib.h>
#include <string.h>

#include "temporal_rdo.h"

enum { MAX_SEGMENTS = 8, ALT_Q = 0, SEG_LVL_REF_FRAME = 5, SEG_LVL_MAX = 8, MAX_SB_IN_IMP_B = 16 };
#define DS_SHIFT 14
#define DS_MAX ((1u << 28) - 1)

/* kmeans.rs:68-102; len bounds the forward walks as the slices `data[n..]` do */
static void scan(size_t *high, size_t *low, int64_t *sum, const int16_t *data, size_t len, int16_t t) {
  size_t n = *high;
  int64_t s = sum[0];
  while (n > 0 && data[n - 1] > t) {
    s -= data[n - 1];
    n--;
  }
  while (n < len && data[n] <= t) {
    s += data[n];
    n++;
  }
  *high = n;
  sum[0] = s;

  n = *low;
  s = sum[1];
  while (n < len && data[n] < t) {
    s -= data[n];
    n++;
  }
  while (n > 0 && data[n - 1] >= t) {
    s += data[n - 1];
    n--;
  }
  *low = n;
  sum[1] = s;
}

/* kmeans.rs:11-66 */
void orc_kmeans_i16(const int16_t *data, size_t len, int K, int16_t *means_out) {
  size_t low[MAX_SEGMENTS], high[MAX_SEGMENTS];
  int64_t sum[MAX_SEGMENTS] = {0};
  int16_t means[MAX_SEGMENTS];
  for (int i = 0; i < K; i++) low[i] = ((size_t)i * (len - 1)) / (size_t)(K - 1);
  for (int i = 0; i < K; i++) means[i] = data[low[i]];
  for (int i = 0; i < K; i++) high[i] = low[i];
  high[K - 1] = len;
  sum[K - 1] = means[K - 1];
  int bits = 0; /* usize::BITS - len.leading_zeros() */
  while (bits < 64 && (len >> bits)) bits++;
  const int limit = 2 * bits;
  for (int it = 0; it < limit; it++) {
    for (int i = 0; i + 1 < K; i++) {
      const int16_t threshold = (int16_t)(((int64_t)means[i + 1] + (int64_t)means[i] + 1) >> 1);
      scan(&high[i], &low[i + 1], &sum[i], data, len, threshold);
    }
    int changed = 0;
    for (int i = 0; i < K; i++) {
      const int64_t count = (int64_t)(high[i] - low[i]); /* usize subtraction wraps, then `as i64` */
      if (count == 0) continue;
      const int16_t new_mean = (int16_t)((sum[i] + (count >> 1)) / count);
      changed |= means[i] != new_mean;
      means[i] = new_mean;
    }
    if (!changed) break;
  }
  memcpy(means_out, means, (size_t)K * sizeof *means);
}

/* quantize/mod.rs:52-77 (MINQ 0, MAXQ 255); binary_search on a strictly increasing table */
int orc_select_qi(int64_t quantizer, const uint16_t *q) {
  if (quantizer < q[0]) return 0;
  if (quantizer >= q[255]) return 255;
  size_t lo = 0, hi = 256; /* first index with q[i] >= quantizer */
  while (lo < hi) {
    const size_t mid = (lo + hi) / 2;
    if (q[mid] < quantizer) lo = mid + 1; else hi = mid;
  }
  if (q[lo] == quantizer) return (int)lo;
  const int32_t qthresh = (int32_t)((uint32_t)q[lo - 1] * (uint32_t)q[lo]);
  const int32_t q2 = (int32_t)((uint32_t)(int32_t)quantizer * (uint32_t)(int32_t)quantizer);
  return q2 < qthresh ? (int)lo - 1 : (int)lo;
}

/* quantize/mod.rs:44-49 */
static uint64_t ac_q(int qindex, int8_t delta_q, const uint16_t *table) {
  int i = qindex + delta_q;
  if (i < 0) i = 0;
  if (i > 255) i = 255;
  return table[i];
}

/* rdo.rs:578-583 */
static uint32_t ds_new(uint64_t num, uint64_t den) {
  const uint64_t sh = num << DS_SHIFT;
  const uint64_t raw = (sh > UINT64_MAX - den / 2 ? UINT64_MAX : sh + den / 2) / den;
  return raw <= DS_MAX ? (uint32_t)raw : DS_MAX;
}

/* encoder.rs:566-580 */
static void update_threshold(orc_segmentation *s, int base_q_idx, const uint16_t *table) {
  const uint64_t base_ac_q = ac_q(base_q_idx, 0, table);
  uint64_t real_ac_q[MAX_SEGMENTS];
  for (int i = 0; i <= s->max_segment; i++) real_ac_q[i] = ac_q(base_q_idx, (int8_t)s->data[i][ALT_Q], table);
  for (int i = 0; i < MAX_SEGMENTS - 1; i++) s->threshold[i] = 0;
  for (int i = 0; i < s->max_segment; i++)
    s->threshold[i] = ds_new(base_ac_q * base_ac_q, real_ac_q[i + 1] * real_ac_q[i]);
}

static int cmp_i16(const void *a, const void *b) {
  const int16_t x = *(const int16_t *)a, y = *(const int16_t *)b;
  return (x > y) - (x < y);
}

/* segmentation.rs:77-160 */
static void optimize_inner(const uint32_t *scores, size_t n, int base_q_idx, const uint16_t *table,
                           int offset_lower_limit, orc_segmentation *s) {
  int16_t *log2_scale_q11 = malloc(n * sizeof *log2_scale_q11);
  for (size_t i = 0; i < n; i++) log2_scale_q11[i] = (int16_t)(orc_blog32_q11(scores[i]) - (DS_SHIFT << 11));
  qsort(log2_scale_q11, n, sizeof *log2_scale_q11, cmp_i16);
  int16_t c[6][MAX_SEGMENTS]; /* c.0 .. c.5: k = 8 .. 3 */
  for (int p = 0; p < 6; p++) orc_kmeans_i16(log2_scale_q11, n, 8 - p, c[p]);
  free(log2_scale_q11);

  uint64_t variance[6];
  for (int p = 0; p < 6; p++) {
    const int K = 8 - p;
    int64_t delta[MAX_SEGMENTS], tot = 0;
    for (int j = 0; j + 1 < K; j++) tot += delta[j] = (int64_t)c[p][j] - (int64_t)c[p][j + 1];
    const int64_t mean = tot / (K - 1);
    int64_t v = 0;
    for (int j = 0; j + 1 < K; j++) v += (delta[j] - mean) * (delta[j] - mean);
    variance[p] = (uint64_t)v;
  }
  uint64_t min_variance = variance[0];
  for (int p = 1; p < 6; p++)
    if (variance[p] < min_variance) min_variance = variance[p];
  int position = 0;
  for (int p = 5; p >= 0; p--)
    if (variance[p] == min_variance) {
      position = p; /* rposition */
      break;
    }

  const int K = 8 - position;
  const int64_t log2_base_ac_q_q57 = orc_blog64((int64_t)ac_q(base_q_idx, 0, table));
  int16_t seg_delta[MAX_SEGMENTS];
  for (int j = 0; j < K; j++) {
    const int16_t log2_scale = c[position][K - 1 - j]; /* .rev() */
    const int64_t q = orc_bexp64(log2_base_ac_q_q57 - (int64_t)((uint64_t)(int64_t)log2_scale << (57 - 11 - 1)));
    int qi = orc_select_qi(q, table);
    if (qi < 1) qi = 1;
    seg_delta[j] = (int16_t)(qi - base_q_idx);
  }
  s->min_segment = 0;
  s->max_segment = (uint8_t)(K - 1);
  for (int j = 0; j < K; j++) {
    s->features[j][ALT_Q] = 1;
    s->data[j][ALT_Q] = seg_delta[j] > offset_lower_limit ? seg_delta[j] : (int16_t)offset_lower_limit;
  }
  update_threshold(s, base_q_idx, table);
}

/* segmentation.rs:23-74 (the state from get_initial_segmentation in *prev), then get_qidx per segment */
int orc_segmentation_optimize(const uint32_t *scores, size_t n, int base_q_idx, int bit_depth, const uint16_t *table,
                              int update_data, const orc_segmentation *prev, orc_segmentation *out) {
  (void)bit_depth; /* the caller's table is the one for bit_depth */
  orc_segmentation s;
  if (prev)
    s = *prev;
  else
    memset(&s, 0, sizeof s);
  s.pad_ = 0;
  s.status = 0;
  s.enabled = 1;
  s.update_map = 1;
  s.update_data = update_data ? 1 : 0;
  const int offset_lower_limit = 1 - base_q_idx;
  if (!s.update_data) {
    int min_segment = MAX_SEGMENTS;
    for (int i = 0; i < MAX_SEGMENTS; i++)
      if (s.features[i][ALT_Q] && s.data[i][ALT_Q] >= offset_lower_limit) {
        min_segment = i;
        break;
      }
    if (min_segment == MAX_SEGMENTS) {
      s.status = 1; /* assert_ne!(min_segment, MAX_SEGMENTS) */
    } else {
      s.min_segment = (uint8_t)min_segment;
      if (s.max_segment >= MAX_SEGMENTS)
        s.status = 2; /* self.data[..=self.max_segment] */
      else
        update_threshold(&s, base_q_idx, table);
    }
  } else {
    optimize_inner(scores, n, base_q_idx, table, offset_lower_limit, &s);
    s.preskip = 0;
    s.last_active_segid = 0;
    for (int i = 0; i < MAX_SEGMENTS; i++)
      for (int j = 0; j < SEG_LVL_MAX; j++)
        if (s.features[i][j]) {
          s.last_active_segid = (uint8_t)i;
          if (j >= SEG_LVL_REF_FRAME) s.preskip = 1;
        }
  }
  for (int i = 0; i < MAX_SEGMENTS; i++) {
    int q = base_q_idx;
    if (s.features[i][ALT_Q]) {
      q = (int16_t)(uint16_t)((uint16_t)base_q_idx + (uint16_t)s.data[i][ALT_Q]); /* i16 add, wrapping */
      q = q < 0 ? 0 : q > 255 ? 255 : q;
    }
    s.qidx[i] = (uint8_t)q;
  }
  *out = s;
  return s.status;
}

/* BlockSize::width() / height() by discriminant (partition.rs:130-153) */
static const int kBw[22] = {4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 64, 128, 128, 4, 16, 8, 32, 16, 64};
static const int kBh[22] = {4, 8, 4, 8, 16, 8, 16, 32, 16, 32, 64, 32, 64, 128, 64, 128, 16, 4, 32, 8, 64, 16};

/* rdo.rs:464-504 */
uint32_t orc_spatiotemporal_scale(const uint32_t *scales, const uint32_t *activity, size_t w_imp, size_t h_imp,
                                  int x, int y, int bsize, int scales_off) {
  if (scales_off) return 1u << DS_SHIFT;
  const size_t x0 = (size_t)(x >> 2) >> 1, y0 = (size_t)(y >> 2) >> 1; /* frame_bo >> IMPORTANCE_BLOCK_TO_BLOCK_SHIFT */
  const size_t wb = kBw[bsize] >> 3 ? kBw[bsize] >> 3 : 1, hb = kBh[bsize] >> 3 ? kBh[bsize] >> 3 : 1;
  const size_t x1 = x0 + wb < w_imp ? x0 + wb : w_imp, y1 = y0 + hb < h_imp ? y0 + hb : h_imp;
  const uint64_t den = (uint64_t)((x1 - x0) * (y1 - y0)) << DS_SHIFT;
  uint64_t sum = 0;
  for (size_t r = y0; r < y1; r++) {
    const uint32_t *d = scales + r * w_imp + x0;
    size_t len = x1 - x0;
    if (len > MAX_SB_IN_IMP_B) len = MAX_SB_IN_IMP_B; /* take_slice */
    for (size_t i = 0; i < len; i++) sum += (uint64_t)d[i] * (activity ? activity[r * w_imp + x0 + i] : 1u << DS_SHIFT);
  }
  return (uint32_t)((sum + (den >> 1)) / den);
}

/* segmentation.rs:192-196: threshold.partition_point(|&t| s < t), i.e. binary_search_by as Rust 1.83's
 * core::slice implements it (branchless: the probe order depends only on the length) */
static int segment_idx_from_distortion(const uint32_t *threshold, uint32_t s) {
  size_t size = MAX_SEGMENTS - 1, base = 0;
  while (size > 1) {
    const size_t half = size / 2, mid = base + half;
    const int less = s < threshold[mid]; /* the predicate holds: Ordering::Less */
    base = less ? mid : base;            /* `if cmp == Greater { base } else { mid }` */
    size -= half;
  }
  return (int)base + (s < threshold[base] ? 1 : 0); /* Err(base + (cmp == Less)) */
}

/* segmentation.rs:163-190 per item */
void orc_select_segment(const orc_segment_item *items, size_t n, const uint32_t *scales, const uint32_t *activity,
                        size_t w_imp, size_t h_imp, int scales_off, int level, const orc_segmentation *seg,
                        uint8_t *sidx, uint32_t *scale) {
  for (size_t i = 0; i < n; i++) {
    const orc_segment_item *it = &items[i];
    if (seg->status != 0 || it->bsize >= 22 || it->x < 0 || it->y < 0 || (it->x & 3) || (it->y & 3) ||
        (size_t)(it->x >> 3) >= w_imp || (size_t)(it->y >> 3) >= h_imp) {
      sidx[2 * i] = sidx[2 * i + 1] = 0xFF;
      if (scale) scale[i] = UINT32_MAX;
      continue;
    }
    const uint32_t s = orc_spatiotemporal_scale(scales, activity, w_imp, h_imp, it->x, it->y, it->bsize, scales_off);
    if (scale) scale[i] = s;
    int lo, hi;
    if (it->skip) {
      lo = hi = 0;
    } else if (level == 3) { /* SegmentationLevel::Full */
      lo = seg->min_segment;
      hi = seg->max_segment;
    } else {
      int sid = segment_idx_from_distortion(seg->threshold, s);
      if (sid < seg->min_segment) sid = seg->min_segment;
      lo = sid;
      if (level == 2) { /* Complex */
        const int up = sid + 1 > 255 ? 255 : sid + 1;
        hi = seg->max_segment < up ? seg->max_segment : up;
      } else {
        hi = sid;
      }
    }
    sidx[2 * i] = (uint8_t)lo;
    sidx[2 * i + 1] = (uint8_t)hi;
  }
}
