// common.cuh — context, error handling and device helpers shared by every kernel file.
#pragma once

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200rdo.h"

#define B200_NUM_SMS 132  /* H100 SXM; replaced by the device's count at context creation */

struct b200_ctx {
  int device = 0;
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;  // the stream kernels are enqueued on
  uint64_t launches = 0;
  int num_sms = B200_NUM_SMS;
  // grow-only device workspace (generic path scratch, sub-pel predictions)
  void *dwork = nullptr;
  size_t dwork_bytes = 0;
  int async_batch = 0;  // host-buffer forms skip their final synchronize (b200_ctx_set_async)
  // device copies of the coefficient scan tables, key = tx_size * 4 + kind (quantize.cu); owned
  // by the context and freed with it.  The host images stay alive with them (the upload is
  // stream-ordered on `stream`).
  std::map<int, uint16_t *> scan_dev;
  std::map<int, std::vector<uint16_t>> scan_host;
  // dynamic shared memory each kernel has been opted in to on this context's device (b200_smem_opt_in)
  std::unordered_map<const void *, int> smem_opt_in;
  char err[512] = {0};
};

extern char g_b200_last_error[512];

inline int b200_fail(b200_ctx *ctx, int status, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (ctx) memcpy(ctx->err, buf, sizeof buf);
  memcpy(g_b200_last_error, buf, sizeof buf);
  return status;
}

#define B200_CUDA(ctx, expr)                                                              \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      (void)cudaGetLastError(); /* reported here: do not leave it for a later launch check */ \
      return b200_fail((ctx), _e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA, \
                       "%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
    }                                                                                     \
  } while (0)

#define B200_REQUIRE(ctx, cond, ...)                              \
  do {                                                            \
    if (!(cond)) return b200_fail((ctx), B200_ERR_ARG, __VA_ARGS__); \
  } while (0)

#define B200_LAUNCH_CHECK(ctx)          \
  do {                                  \
    (ctx)->launches++;                  \
    B200_CUDA((ctx), cudaGetLastError()); \
  } while (0)

// Opt `kernel` in to `bytes` of dynamic shared memory on the context's device (the current device
// of every `_dev` call).  The attribute belongs to the device, so it is remembered per context,
// which serves one device and one host thread.
inline int b200_smem_opt_in(b200_ctx *ctx, const void *kernel, int bytes) {
  int &set = ctx->smem_opt_in[kernel];
  if (set >= bytes) return B200_OK;
  B200_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  set = bytes;
  return B200_OK;
}

// Per-call (reference-signature) forms have no error return (the reference asserts or panics; never
// silently wrong): a failed status prints the failing step and the context's last error, then aborts.
inline void b200_percall_check(const b200_ctx *ctx, int st, const char *what) {
  if (st == B200_OK) return;
  fprintf(stderr, "b200rdo: FATAL: %s failed: %s\n", what, b200_last_error(ctx));
  abort();
}

// Grow-only device scratch.
int b200_reserve_dwork(b200_ctx *ctx, size_t bytes);
int b200_mc_cands_internal(b200_ctx *ctx, const b200_plane *ref, const b200_block *d_blocks,
                           const b200_cand *d_cands, size_t ncands, int w, int h, int mode,
                           int bit_depth, void *d_out);
int b200_plane_unpack_internal(b200_ctx *ctx, const b200_plane *p, const void *d_packed);
// device copy of the scan order of (tx_size, tx_type) (scan_order.rs; owned by the context), quantize.cu
int b200_scan_table_internal(b200_ctx *ctx, int tx_size, int tx_type, const uint16_t **d_scan);
b200_ctx *b200_default_ctx();  // lazily created; aborts loudly if no device (no CPU fallback)
// the plane pair and block size a motion-estimation call may take (get_sad / get_satd), me_cand.cu
int b200_me_check_planes(b200_ctx *ctx, const b200_plane *cur, const b200_plane *ref, const b200_me_params *p);

#ifdef __CUDACC__
#define B200_HD __host__ __device__
#else
#define B200_HD
#endif
B200_HD static inline size_t b200_align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---------------------------------------------------------------- device helpers
#ifdef __CUDACC__

#define MI_SIZE 4
#define MV_LOW (-(1 << 14))
#define MV_UPP (1 << 14)

// A plane as the kernels see it: pixel (0,0) and the row pitch, both in elements of the pixel type.
struct PlaneView {
  const void *data;  // pixel (0,0)
  int stride;        // elements
};

template <typename T>
__device__ __forceinline__ const T *px(const PlaneView &p, int x, int y) {
  return (const T *)p.data + (long long)y * p.stride + x;
}

struct MvRange {
  int x_min, x_max, y_min, y_max;
};

// me.rs:339-362 get_mv_range (bo in 4x4 units, blk dims in px, result in 1/8 pel)
__host__ __device__ inline MvRange b200_mv_range(int w_in_b, int h_in_b, int bo_x, int bo_y,
                                                 int blk_w, int blk_h) {
  const int border_w = 128 + blk_w * 8;
  const int border_h = 128 + blk_h * 8;
  int x_min = -bo_x * (8 * MI_SIZE) - border_w;
  int x_max = ((w_in_b - bo_x) - (blk_w / MI_SIZE)) * (8 * MI_SIZE) + border_w;
  int y_min = -bo_y * (8 * MI_SIZE) - border_h;
  int y_max = ((h_in_b - bo_y) - (blk_h / MI_SIZE)) * (8 * MI_SIZE) + border_h;
  MvRange r;
  r.x_min = x_min > MV_LOW + 1 ? x_min : MV_LOW + 1;
  r.x_max = x_max < MV_UPP - 1 ? x_max : MV_UPP - 1;
  r.y_min = y_min > MV_LOW + 1 ? y_min : MV_LOW + 1;
  r.y_max = y_max < MV_UPP - 1 ? y_max : MV_UPP - 1;
  return r;
}

// me.rs:1512-1523 get_mv_rate.  ilog(x) = 32 - clz(x) for x > 0, else 0.
__device__ __forceinline__ uint32_t b200_diff_to_rate(int diff16, int allow_hp) {
  int d = (int)(short)diff16;          // i16 subtraction wraps like Rust release builds
  d = allow_hp ? d : (d >> 1);         // arithmetic shift
  // i16::abs wraps for i16::MIN in release builds and ILog::ilog counts the bits of the i16
  // pattern: |-32768| -> 0x8000 -> ilog 16 (v_frame 0.3.9 math.rs)
  const uint32_t a = (uint32_t)(uint16_t)(d < 0 ? -d : d);
  return a ? 2u * (32u - (uint32_t)__clz(a)) : 0u;
}

__device__ __forceinline__ uint32_t b200_mv_rate(int a_row, int a_col, int b_row, int b_col,
                                                 int allow_hp) {
  return b200_diff_to_rate(a_row - b_row, allow_hp) + b200_diff_to_rate(a_col - b_col, allow_hp);
}

// me.rs:1455-1460
__device__ __forceinline__ unsigned long long b200_mv_cost(uint32_t sad, int mv_row, int mv_col,
                                                           int p0_row, int p0_col, int p1_row,
                                                           int p1_col, uint32_t lambda,
                                                           int allow_hp) {
  // (no skipping of the second rate when the predictors are equal: that puts a branch in every
  // candidate's cost)
  const uint32_t r1 = b200_mv_rate(mv_row, mv_col, p0_row, p0_col, allow_hp);
  const uint32_t r2 = b200_mv_rate(mv_row, mv_col, p1_row, p1_col, allow_hp) + 1;
  const uint32_t rate = r1 < r2 ? r1 : r2;
  return 256ull * sad + (unsigned long long)rate * lambda;
}

__device__ __forceinline__ uint32_t warp_sum_u32(uint32_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

#endif  // __CUDACC__
