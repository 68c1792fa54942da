// rdo_dist_dev.cuh — the integer cores of rav1e's RDO distortion terms, shared by the batched
// distortion kernels (rdo_dist.cu) and the fused loop-filter RDO (cdef_rdo.cu):
//   get_weighted_sse   src/dist.rs:234-283: one 4x4 chunk's scaled sum, and the final division
//   cdef_dist_kernel   src/dist.rs:302-372: the five sums -> sse, svar, dvar
//   apply_ssim_boost   src/activity.rs:159-186 (+ ssim_boost_rsqrt :107-143)
//   compute_rd_cost    src/rdo.rs:718-723 (see rd_cost.cu)
#pragma once
#include "common.cuh"

namespace {

constexpr int kWsseShift = 8;  // GET_WEIGHTED_SSE_SHIFT, dist.rs:223

// one 4x4 chunk's term of get_weighted_sse: its SSE times its Q14 scale, rounded >> 8
__device__ __forceinline__ unsigned long long wsse_chunk(uint32_t sum, uint32_t scale) {
  const unsigned long long s = scale;
  return ((unsigned long long)sum * s + ((1u << kWsseShift) >> 1)) >> kWsseShift;
}

// the sum of a block's chunk terms -> get_weighted_sse's result
__device__ __forceinline__ unsigned long long wsse_finish(unsigned long long acc) {
  // den = DistortionScale::new(1, 1 << 8).0 = ((1 << 14) + 128) / 256 = 64 (rdo.rs:579-583)
  constexpr unsigned long long den = ((1ull << 14) + ((1u << kWsseShift) / 2)) >> kWsseShift;
  return (acc + (den >> 1)) / den;
}

// round(2^14 / (1 + x)), dist.rs:288-297
__constant__ unsigned short kAreaDivisors[64] = {
    16384, 8192, 5461, 4096, 3277, 2731, 2341, 2048, 1820, 1638, 1489, 1365, 1260, 1170, 1092, 1024,
    964,   910,  862,  819,  780,  745,  712,  683,  655,  630,  607,  585,  565,  546,  529,  512,
    496,   482,  468,  455,  443,  431,  420,  410,  400,  390,  381,  372,  364,  356,  349,  341,
    334,   328,  321,  315,  309,  303,  298,  293,  287,  282,  278,  273,  269,  264,  260,  256};

// activity.rs:159-186 with ssim_boost_rsqrt :107-143 inlined
__device__ __forceinline__ uint32_t apply_ssim_boost(uint32_t input, uint32_t svar, uint32_t dvar, int bit_depth) {
  const int coeff_shift = bit_depth - 8;
  const unsigned long long sv = svar >> (2 * coeff_shift), dv = dvar >> (2 * coeff_shift);
  constexpr unsigned long long C1 = 3355, C2 = 16128, C3 = 12338;
  constexpr int RATIO_SHIFT = 14;
  constexpr unsigned long long RATIO = (((C1 << (RATIO_SHIFT + 1)) / C3) + 1) >> 1;
  const unsigned long long x = C1 * C1 + sv * dv;
  const int k = (63 - __clzll((long long)x)) >> 1;
  const int s = 2 * k - (16 - 2);
  const uint32_t t = (uint32_t)(s > 0 ? x >> s : x << -s) & 0xffffu;  // `as u16`
  const int shift = 14 + ((s + 16) >> 1);
  const int nn = (int)t - 32768;
  const int inner = -13490 + ((nn * 6711) >> 15);
  const uint32_t norm = (uint32_t)(23557 + ((nn * inner) >> 15)) & 0xffffu;
  return (uint32_t)(((unsigned long long)input * (((RATIO * (sv + dv + C2)) * (unsigned long long)norm) >> RATIO_SHIFT)) >> shift);
}

// cdef_dist_kernel after its loop (dist.rs:340-371): the five u32 sums (wrapping like the
// reference) of a w x h block with w * h = area -> sse, and svar / dvar scaled to an 8x8 area
__device__ __forceinline__ uint32_t cdef_dist_vars(uint32_t sum_s, uint32_t sum_d, uint32_t sum_s2, uint32_t sum_d2,
                                                   uint32_t sum_sd, int area, uint32_t *svar_out,
                                                   uint32_t *dvar_out) {
  const uint32_t sse = sum_d2 + sum_s2 - 2 * sum_sd;
  const unsigned long long S = sum_s, D = sum_d, div = kAreaDivisors[area - 1];
  const uint32_t ms = (uint32_t)((S * S * div + (1u << 13)) >> 14);
  const uint32_t md = (uint32_t)((D * D * div + (1u << 13)) >> 14);
  uint32_t svar = sum_s2 > ms ? sum_s2 - ms : 0u;  // saturating_sub
  uint32_t dvar = sum_d2 > md ? sum_d2 - md : 0u;
  *svar_out = (uint32_t)(((unsigned long long)svar * div + (1u << 7)) >> 8);  // scale to an 8x8 area
  *dvar_out = (uint32_t)(((unsigned long long)dvar * div + (1u << 7)) >> 8);
  return sse;
}

__device__ __forceinline__ double rd_cost(double lambda, uint32_t rate, unsigned long long dist) {
  const double rate_in_bits = (double)rate / 8.0;             // rdo.rs:721 (exact)
  return fma(lambda, rate_in_bits, __ull2double_rn(dist));    // rdo.rs:722
}

}  // namespace
