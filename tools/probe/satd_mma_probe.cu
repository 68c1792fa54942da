// satd_mma_probe.cu — the experiment BASELINE.json's north star names: "tensor cores only if 8-bit SATD's
// Hadamard is cast as an i8 MMA and ncu shows a win".  Stand-alone micro-benchmark (not part of the
// library): the 8x8 SATD of 32 chunk pairs per warp, operands resident in shared memory, computed
//   (A) the way the product kernels do: thread per chunk, horizontal pass as IDP.4A chains, vertical pass
//       as register butterflies (me_chunk.cu, me_chunk_lists);
//   (B) with mma.sync.m16n8k32.s32.u8.s8: pixels as the A operand (16 rows x 32 bytes = 8 chunks, natural
//       row-major bytes, no transposes), the +-1 Hadamard matrix of one chunk column group as B (zeros
//       elsewhere: the 8 outputs of a row are all a m16n8 tile can hold), org and -ref accumulated into the
//       same tile; the VERTICAL pass then has to run on the s32 accumulator fragments, whose rows live in
//       different lanes: three shfl.xor butterfly stages, then |.| and the sum.
// Both must produce the same 32 sums.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o
// satd_mma_probe satd_mma_probe.cu ; run on the GPU; timings are per warp-iteration (32 chunks).
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

__device__ __forceinline__ int dp4a_us(uint32_t a, uint32_t b, int c) {
  int d;
  asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
}
__device__ __forceinline__ void bfly(int &a, int &b) {
  const int s = a + b, t = a - b;
  a = s;
  b = t;
}

// layout per warp: org[4 tiles][16 rows][32 bytes], ref likewise; chunk c = (tile, row half, column group)
constexpr int kTileBytes = 16 * 32;

// ---- (A) thread per chunk
__device__ uint32_t satd_alu(const uint32_t *org, const uint32_t *ref, int lane) {
  const int tile = lane >> 3, rh = (lane >> 2) & 1, cg = lane & 3;
  const uint32_t *o = org + tile * (kTileBytes / 4) + rh * 8 * 8 + cg * 2;
  const uint32_t *r = ref + tile * (kTileBytes / 4) + rh * 8 * 8 + cg * 2;
  int t[8][8];
#pragma unroll
  for (int y = 0; y < 8; y++) {
    const uint32_t o0 = o[y * 8], o1 = o[y * 8 + 1], q0 = r[y * 8], q1 = r[y * 8 + 1];
    t[y][0] = dp4a_us(q1, 0xFFFFFFFFu, dp4a_us(q0, 0xFFFFFFFFu, dp4a_us(o1, 0x01010101u, dp4a_us(o0, 0x01010101u, 0))));
    t[y][1] = dp4a_us(q1, 0x01FF01FFu, dp4a_us(q0, 0x01FF01FFu, dp4a_us(o1, 0xFF01FF01u, dp4a_us(o0, 0xFF01FF01u, 0))));
    t[y][2] = dp4a_us(q1, 0x0101FFFFu, dp4a_us(q0, 0x0101FFFFu, dp4a_us(o1, 0xFFFF0101u, dp4a_us(o0, 0xFFFF0101u, 0))));
    t[y][3] = dp4a_us(q1, 0xFF0101FFu, dp4a_us(q0, 0xFF0101FFu, dp4a_us(o1, 0x01FFFF01u, dp4a_us(o0, 0x01FFFF01u, 0))));
    t[y][4] = dp4a_us(q1, 0x01010101u, dp4a_us(q0, 0xFFFFFFFFu, dp4a_us(o1, 0xFFFFFFFFu, dp4a_us(o0, 0x01010101u, 0))));
    t[y][5] = dp4a_us(q1, 0xFF01FF01u, dp4a_us(q0, 0x01FF01FFu, dp4a_us(o1, 0x01FF01FFu, dp4a_us(o0, 0xFF01FF01u, 0))));
    t[y][6] = dp4a_us(q1, 0xFFFF0101u, dp4a_us(q0, 0x0101FFFFu, dp4a_us(o1, 0x0101FFFFu, dp4a_us(o0, 0xFFFF0101u, 0))));
    t[y][7] = dp4a_us(q1, 0x01FFFF01u, dp4a_us(q0, 0xFF0101FFu, dp4a_us(o1, 0xFF0101FFu, dp4a_us(o0, 0x01FFFF01u, 0))));
  }
  uint32_t s = 0;
#pragma unroll
  for (int col = 0; col < 8; col++) {
    int v[8];
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] = t[k][col];
    bfly(v[0], v[1]);
    bfly(v[2], v[3]);
    bfly(v[4], v[5]);
    bfly(v[6], v[7]);
    bfly(v[0], v[2]);
    bfly(v[1], v[3]);
    bfly(v[4], v[6]);
    bfly(v[5], v[7]);
#pragma unroll
    for (int k = 0; k < 4; k++) s += (uint32_t)max(abs(v[k]), abs(v[k + 4]));
  }
  return 2u * s;  // sum |H d H^T| of this lane's chunk
}

// ---- (B) mma.sync
__device__ __forceinline__ void mma_u8s8(int (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// B fragment of column group cg: B[k][n] = H8[n][k - 8 cg] for k in [8 cg, 8 cg + 8), else 0 (sign flips it for
// the reference).  Fragment: b0 = B[4t .. 4t+3][g], b1 = B[16 + 4t ..][g], t = lane % 4, g = lane / 4.
__device__ uint32_t hfrag(int cg, int reg, int lane, int sign) {
  const int t = lane & 3, g = lane >> 2;
  uint32_t w = 0;
  for (int j = 0; j < 4; j++) {
    const int k = reg * 16 + 4 * t + j, kk = k - 8 * cg;
    int v = 0;
    if (kk >= 0 && kk < 8) v = (__popc(g & kk) & 1) ? -sign : sign;  // Sylvester H8[g][kk] = (-1)^popc(g & kk)
    w |= ((uint32_t)v & 0xffu) << (8 * j);
  }
  return w;
}

__device__ uint32_t satd_mma(const uint32_t *org, const uint32_t *ref, int lane, const uint32_t (&hb)[4][2][2]) {
  const int t = lane & 3, g = lane >> 2;
  uint32_t mine = 0;  // this lane's share of the sums; chunk sums are recovered by the caller's reduction
#pragma unroll
  for (int tile = 0; tile < 4; tile++) {
    const uint32_t *o = org + tile * (kTileBytes / 4), *r = ref + tile * (kTileBytes / 4);
    const uint32_t ao[4] = {o[g * 8 + t], o[(g + 8) * 8 + t], o[g * 8 + 4 + t], o[(g + 8) * 8 + 4 + t]};
    const uint32_t ar[4] = {r[g * 8 + t], r[(g + 8) * 8 + t], r[g * 8 + 4 + t], r[(g + 8) * 8 + 4 + t]};
#pragma unroll
    for (int cg = 0; cg < 4; cg++) {
      int c[4] = {0, 0, 0, 0};  // rows g / g+8, output coefficients 2t, 2t+1 of column group cg
      mma_u8s8(c, ao, hb[cg][0]);
      mma_u8s8(c, ar, hb[cg][1]);
      // vertical 8-point Hadamard over the rows g = 0..7 (c[0], c[1]) and 8..15 (c[2], c[3]): rows are lanes
#pragma unroll
      for (int s = 4; s < 32; s <<= 1) {
        const bool hi = (lane & s) != 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const int other = __shfl_xor_sync(0xffffffffu, c[k], s);
          c[k] = hi ? other - c[k] : c[k] + other;
        }
      }
      // chunk (tile, row half 0, cg) collects |c0| + |c1| over all lanes, (tile, 1, cg) |c2| + |c3|;
      // pack both into one word (sums < 2^16 each per lane: 2 * 16320)
      mine += ((uint32_t)(abs(c[0]) + abs(c[1]))) << (0) ;
      mine += 0;  // (kept simple: the probe compares the grand total of all 32 chunks)
      mine += (uint32_t)(abs(c[2]) + abs(c[3]));
    }
  }
  return mine;
}

template <int MODE>
__global__ void __launch_bounds__(256) probe(const uint8_t *data, int iters, unsigned long long *out, long long *clk) {
  extern __shared__ uint32_t sm[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t *org = sm + warp * (2 * 4 * kTileBytes / 4), *ref = org + 4 * kTileBytes / 4;
  for (int i = lane; i < 2 * 4 * kTileBytes / 4; i += 32) org[i] = ((const uint32_t *)data)[(blockIdx.x * 8 + warp) * 1024 + i];
  uint32_t hb[4][2][2];
  for (int cg = 0; cg < 4; cg++)
    for (int reg = 0; reg < 2; reg++) {
      hb[cg][0][reg] = hfrag(cg, reg, lane, 1);
      hb[cg][1][reg] = hfrag(cg, reg, lane, -1);
    }
  __syncwarp();
  unsigned long long total = 0;
  const long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
    uint32_t v = MODE == 0 ? satd_alu(org, ref, lane) : satd_mma(org, ref, lane, hb);
    total += v;
    if (it == iters - 2) org[lane] ^= 0x01010101u;  // keep the loads inside the loop
    __syncwarp();
  }
  const long long t1 = clock64();
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
  if (lane == 0) {
    out[blockIdx.x * 8 + warp] = total;
    if (threadIdx.x == 0 && blockIdx.x == 0) *clk = t1 - t0;
  }
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  const int ctas = sms * 2, iters = 2000;
  std::vector<uint8_t> h((size_t)ctas * 8 * 4096);
  srand(1);
  for (auto &b : h) b = (uint8_t)rand();
  uint8_t *d;
  unsigned long long *o0, *o1;
  long long *clk;
  cudaMalloc(&d, h.size());
  cudaMalloc(&o0, ctas * 8 * 8);
  cudaMalloc(&o1, ctas * 8 * 8);
  cudaMalloc(&clk, 16);
  cudaMemcpy(d, h.data(), h.size(), cudaMemcpyHostToDevice);
  const size_t smem = 8 * 2 * 4 * kTileBytes;
  float ms[2];
  long long cyc[2];
  for (int mode = 0; mode < 2; mode++) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    for (int rep = 0; rep < 2; rep++) {  // first launch warms up
      cudaEventRecord(e0);
      if (mode == 0)
        probe<0><<<ctas, 256, smem>>>(d, iters, o0, clk);
      else
        probe<1><<<ctas, 256, smem>>>(d, iters, o1, clk + 1);
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      cudaEventElapsedTime(&ms[mode], e0, e1);
    }
  }
  cudaMemcpy(cyc, clk, 16, cudaMemcpyDeviceToHost);
  std::vector<unsigned long long> a(ctas * 8), b(ctas * 8);
  cudaMemcpy(a.data(), o0, a.size() * 8, cudaMemcpyDeviceToHost);
  cudaMemcpy(b.data(), o1, b.size() * 8, cudaMemcpyDeviceToHost);
  size_t bad = 0;
  for (size_t i = 0; i < a.size(); i++) bad += a[i] != b[i];
  const cudaError_t e = cudaGetLastError();
  const double chunks = (double)ctas * 8 * 32 * iters;
  printf("{\"probe\": \"satd 8x8: dp4a+butterflies vs mma.sync m16n8k32 u8xs8\", \"cuda\": \"%s\", \"mismatching_warps\": %zu, "
         "\"alu_ms\": %.3f, \"mma_ms\": %.3f, \"alu_Gchunks_per_s\": %.2f, \"mma_Gchunks_per_s\": %.2f, "
         "\"alu_cycles_per_warp_iteration\": %.1f, \"mma_cycles_per_warp_iteration\": %.1f}\n",
         cudaGetErrorString(e), bad, ms[0], ms[1], chunks / ms[0] / 1e6, chunks / ms[1] / 1e6, (double)cyc[0] / iters,
         (double)cyc[1] / iters);
  return bad != 0;
}
