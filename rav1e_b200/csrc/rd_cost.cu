// rd_cost.cu — the one floating-point value on the RDO path (sm_90a).
//
//   compute_rd_cost   src/rdo.rs:718-723
//       rate_in_bits = (rate as f64) / ((1 << OD_BITRES) as f64)          OD_BITRES = 3, ec.rs:25
//       fi.lambda.mul_add(rate_in_bits, distortion.0 as f64)
//
// f64::mul_add is the IEEE-754 fused multiply-add; `fma()` in device code is DFMA with round to
// nearest even, u32 -> f64 and the division by 8 are exact, u64 -> f64 (`as f64`) rounds to nearest
// even like __ull2double_rn: the result is bit-identical to the reference (0 ULP, inside the
// north star's 1-ULP rule).  The RDO loops that consume it keep the candidate with the smallest cost
// under a strict `<` (rdo.rs `if rd < best.rd_cost`): the batched form can also return, per group of
// candidates, the index of that first minimum.
#include <cuda_runtime.h>

#include <algorithm>

#include "host_stage.cuh"
#include "rdo_dist_dev.cuh"

namespace {


__global__ void rd_cost_kernel(double lambda, const uint32_t *rate, const unsigned long long *dist, size_t n,
                               double *out) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = rd_cost(lambda, rate[i], dist[i]);
}

// one warp per group: cost of every candidate (optionally stored) and the first minimum
__global__ void rd_best_kernel(double lambda, const uint32_t *rate, const unsigned long long *dist,
                               const uint32_t *offs, size_t ngroups, double *out_cost, uint32_t *out_best) {
  const int lane = threadIdx.x & 31;
  const size_t g = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (g >= ngroups) return;
  const uint32_t lo = offs[g], hi = offs[g + 1];
  double best = 0.0;
  uint32_t bi = 0xffffffffu;  // empty group
  for (uint32_t i = lo + lane; i < hi; i += 32) {
    const double c = rd_cost(lambda, rate[i], dist[i]);
    if (out_cost) out_cost[i] = c;
    if (bi == 0xffffffffu || c < best) best = c, bi = i;  // ascending i per lane: strict < keeps the first
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
    const uint32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi != 0xffffffffu && (bi == 0xffffffffu || ob < best || (ob == best && oi < bi))) best = ob, bi = oi;
  }
  if (lane == 0) out_best[g] = bi == 0xffffffffu ? bi : bi - lo;
}

}  // namespace

extern "C" int b200_compute_rd_cost_dev(b200_ctx *ctx, double lambda, const uint32_t *d_rate,
                                        const uint64_t *d_distortion, size_t n, const uint32_t *d_group_offsets,
                                        size_t ngroups, double *d_cost, uint32_t *d_best) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, d_best == nullptr || d_group_offsets != nullptr, "d_best needs d_group_offsets");
  if (n == 0 && (ngroups == 0 || !d_best)) return B200_OK;
  B200_REQUIRE(ctx, (d_rate && d_distortion) || n == 0, "NULL rate / distortion");
  B200_REQUIRE(ctx, d_cost || d_best, "no output requested");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  if (d_best) {
    const int wpc = 8;
    rd_best_kernel<<<(int)((ngroups + wpc - 1) / wpc), wpc * 32, 0, ctx->stream>>>(
        lambda, d_rate, (const unsigned long long *)d_distortion, d_group_offsets, ngroups, d_cost, d_best);
  } else {
    const int grid = (int)std::min<size_t>((n + 255) / 256, (size_t)ctx->num_sms * 16);
    rd_cost_kernel<<<grid, 256, 0, ctx->stream>>>(lambda, d_rate, (const unsigned long long *)d_distortion, n, d_cost);
  }
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// Per-call form: compute_rd_cost(fi, rate, distortion) with fi.lambda passed in.  One launch on the
// calling thread's context; exists for drop-in completeness and `check_asm`-style cross-checks (a host
// fma() would be the same bits, but nothing in this library computes on the CPU).
extern "C" double b200_compute_rd_cost(double lambda, uint32_t rate, uint64_t distortion) {
  b200_ctx *ctx = b200_default_ctx();
  struct {
    unsigned long long dist;
    double cost;
    uint32_t rate;
  } h{distortion, 0.0, rate};
  HostStage s(ctx, sizeof h);
  auto *d = (decltype(h) *)s.take(sizeof h);
  s.up(d, &h, sizeof h);
  if (s.ok())
    s.run(b200_compute_rd_cost_dev(ctx, lambda, &d->rate, (const uint64_t *)&d->dist, 1, nullptr, 0, &d->cost,
                                   nullptr));
  s.down(&h.cost, &d->cost, sizeof(double));
  b200_percall_check(ctx, s.finish(true), "compute_rd_cost");
  return h.cost;
}
