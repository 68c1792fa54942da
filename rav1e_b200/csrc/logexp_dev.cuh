// logexp_dev.cuh — util/logexp.rs restated for the device: blog32_q11, bexp64 and blog64, shared by
// temporal RDO (temporal_rdo.cu: the score normalisation) and segmentation (segmentation.cu: the
// log-domain scores and the segment quantizers).
#pragma once
#include <cstdint>

namespace {

__device__ const long long ATANH_Q62[32] = {
    0x32B803473F7AD0F4, 0x2F2A71BD4E25E916, 0x2E68B244BB93BA06, 0x2E39FB9198CE62E4, 0x2E2E683F68565C8F,
    0x2E2B850BE2077FC1, 0x2E2ACC58FE7B78DB, 0x2E2A9E2DE52FD5F2, 0x2E2A92A338D53EEC, 0x2E2A8FC08F5E19B6,
    0x2E2A8F07E51A485E, 0x2E2A8ED9BA8AF388, 0x2E2A8ECE2FE7384A, 0x2E2A8ECB4D3E4B1A, 0x2E2A8ECA94940FE8,
    0x2E2A8ECA6669811D, 0x2E2A8ECA5ADEDD6A, 0x2E2A8ECA57FC347E, 0x2E2A8ECA57438A43, 0x2E2A8ECA57155FB4,
    0x2E2A8ECA5709D510, 0x2E2A8ECA5706F267, 0x2E2A8ECA570639BD, 0x2E2A8ECA57060B92, 0x2E2A8ECA57060008,
    0x2E2A8ECA5705FD25, 0x2E2A8ECA5705FC6C, 0x2E2A8ECA5705FC3E, 0x2E2A8ECA5705FC33, 0x2E2A8ECA5705FC30,
    0x2E2A8ECA5705FC2F, 0x2E2A8ECA5705FC2F};

__device__ __forceinline__ long long q57(int v) { return (long long)((unsigned long long)(long long)v << 57); }
// (v + m) ^ m with m = 0 or -1: v or -v, in wrapping arithmetic
__device__ __forceinline__ long long flip(long long v, long long m) {
  return (long long)(((unsigned long long)v + (unsigned long long)m) ^ (unsigned long long)m);
}
__device__ __forceinline__ long long twice(long long v) { return (long long)((unsigned long long)v << 1); }

__device__ int blog32_q11(uint32_t w) {
  if (w == 0) return -1;
  const int ipart = 32 - __clz(w);
  const int n = (int)(ipart > 16 ? w >> (ipart - 16) : w << (16 - ipart)) - 49152;
  int p = ((n * -1402) >> 15) + 2546;
  p = ((n * p) >> 15) - 5216;
  p = ((n * p) >> 15) + 15745;
  p = ((n * p) >> 15) - 6797;
  return (ipart << 11) + (p >> 3);
}

__device__ long long bexp64(long long logq57) {
  const int ipart = (int)(logq57 >> 57);
  if (ipart < 0) return 0;
  if (ipart >= 63) return 0x7FFFFFFFFFFFFFFFll;
  long long z = logq57 - q57(ipart), w;
  if (z == 0) {
    w = 1ll << 62;
  } else {
    z = (long long)((unsigned long long)z << 5);
    w = 0x26A3D0E401DD846Dll;
    int i = 0, again = 3;  // iterations 3, 12 and 39 run twice (hyperbolic CORDIC convergence)
    for (; i < 32;) {
      const long long m = z < 0 ? -1 : 0;
      w += flip(w >> (i + 1), m);
      z -= flip(ATANH_Q62[i], m);
      if (i == again) {
        again = 3 * again + 3;
      } else {
        z = twice(z);
        i++;
      }
    }
    int wlo = 0;
    if (ipart > 30)
      for (; i < 61;) {
        const long long m = z < 0 ? -1 : 0;
        wlo += (int)flip(w >> i, m);
        z -= flip(ATANH_Q62[31], m);
        if (i == again) {
          again = 3 * again + 3;
        } else {
          z = twice(z);
          i++;
        }
      }
    w = twice(w) + wlo;
  }
  if (ipart < 62) w = ((w >> (61 - ipart)) + 1) >> 1;
  return w;
}

__device__ long long blog64(long long n) {
  if (n <= 0) return -1;
  const int ipart = 63 - __clzll(n);
  const long long w = ipart > 61 ? n >> (ipart - 61) : (long long)((unsigned long long)n << (61 - ipart));
  if ((w & (w - 1)) == 0) return q57(ipart);
  long long z = 0, x = w + (1ll << 61), y = w - (1ll << 61);
  for (int i = 0, again = 3; i <= 61;) {
    const long long m = y < 0 ? -1 : 0;
    z += flip(ATANH_Q62[i < 31 ? i : 31] >> i, m);
    const long long u = x >> (i + 1);
    x -= flip(y >> (i + 1), m);
    y -= flip(u, m);
    if (i == again)
      again = 3 * again + 3;
    else
      i++;
  }
  return q57(ipart) + ((z + 8) >> 4);
}

}  // namespace
