// lrf_dev.cuh — the self-guided filter's integer pieces shared by the frame filter (lrf.cu) and the
// restoration search (lrf_search.cu): the parameter table, sgrproj_sum_finish and the radius-1 / radius-2
// neighbourhood weightings of the box filter outputs.
#pragma once
#include "common.cuh"

namespace {

// SGRPROJ_PARAMS_S (lrf.rs:56-73): s for radius 2, s for radius 1
__constant__ uint16_t kSgrS[16][2] = {{140, 3236}, {112, 2158}, {93, 1618}, {80, 1438}, {70, 1295}, {58, 1177},
                                      {47, 1079},  {37, 996},   {30, 925},  {25, 863},  {0, 2589},  {0, 1618},
                                      {0, 1177},   {0, 925},    {56, 0},    {22, 0}};

// sgrproj_sum_finish (lrf.rs:344-362), u32 arithmetic as the reference
__device__ __forceinline__ void sum_finish(uint32_t ssq, uint32_t sum, uint32_t n, uint32_t one_over_n, uint32_t s,
                                           int bdm8, uint32_t &ra, uint32_t &rb) {
  const uint32_t scaled_ssq = (ssq + ((1u << (2 * bdm8)) >> 1)) >> (2 * bdm8);
  const uint32_t scaled_sum = (sum + ((1u << bdm8) >> 1)) >> bdm8;
  const uint32_t t0 = scaled_ssq * n, t1 = scaled_sum * scaled_sum;
  const uint32_t p = t0 > t1 ? t0 - t1 : 0;
  const uint32_t z = (p * s + (1u << 19)) >> 20;
  const uint32_t a = z >= 255 ? 256 : z == 0 ? 1 : ((z << 8) + z / 2) / (z + 1);
  ra = a;
  rb = ((256 - a) * sum * one_over_n + (1u << 11)) >> 12;
}

// sgrproj_box_f_r2 (lrf.rs:300-342): one radius-2 a / b row weighted 5 6 5 around column l + 1
__device__ __forceinline__ uint32_t r2_row(const uint32_t *row, int l) {
  return 5 * (row[l] + row[l + 2]) + 6 * row[l + 1];
}

// sgrproj_box_f_r1 (lrf.rs:266-291): the 3x3 neighbourhood of rows y .. y + 2, columns l .. l + 2, corners
// weighted 3 and the cross 4
template <int P>
__device__ __forceinline__ uint32_t r1_weigh(const uint32_t (*A)[P], int y, int l) {
  return 3 * (A[y][l] + A[y + 2][l] + A[y][l + 2] + A[y + 2][l + 2]) +
         4 * (A[y + 1][l] + A[y][l + 1] + A[y + 1][l + 1] + A[y + 2][l + 1] + A[y + 1][l + 2]);
}

}  // namespace
