// host_stage.cuh — staging of host buffers for the host-buffer (`*_batch` / `*_resident`) and
// per-call entry points: one stream-ordered device arena per call, carved into 256-byte aligned
// slices, with the copies up and down on the context's stream.
#pragma once

#include "common.cuh"

// Binds one call's staging to a context.  The first failing step records its status and message
// (b200_fail); every later copy is skipped, and the caller skips its `_dev` step with ok().  The
// arena is freed on the stream by finish() or, on an early return, by the destructor.
class HostStage {
 public:
  // cudaSetDevice, then one cudaMallocAsync of `bytes` (the sum of the caller's slices, each
  // rounded up to 256 except the last)
  HostStage(b200_ctx *ctx, size_t bytes) : ctx_(ctx) {
    check(cudaSetDevice(ctx->device), "cudaSetDevice");
    if (ok()) check(cudaMallocAsync((void **)&base_, bytes, ctx->stream), "cudaMallocAsync");
  }
  ~HostStage() { release(); }
  HostStage(const HostStage &) = delete;
  HostStage &operator=(const HostStage &) = delete;

  bool ok() const { return st_ == B200_OK; }

  // the next slice of the arena, 256-byte aligned
  uint8_t *take(size_t bytes) {
    uint8_t *r = base_ ? base_ + used_ : nullptr;
    used_ += b200_align_up(bytes, 256);
    return r;
  }

  void up(void *dst, const void *src, size_t bytes) { copy(dst, src, bytes, cudaMemcpyHostToDevice, "H2D copy"); }
  void down(void *dst, const void *src, size_t bytes) { copy(dst, src, bytes, cudaMemcpyDeviceToHost, "D2H copy"); }
  void up2d(void *dst, size_t dpitch, const void *src, size_t spitch, size_t row_bytes, size_t rows) {
    copy2d(dst, dpitch, src, spitch, row_bytes, rows, cudaMemcpyHostToDevice, "H2D copy");
  }
  void down2d(void *dst, size_t dpitch, const void *src, size_t spitch, size_t row_bytes, size_t rows) {
    copy2d(dst, dpitch, src, spitch, row_bytes, rows, cudaMemcpyDeviceToHost, "D2H copy");
  }

  // records the status of a step the caller ran on the staged buffers (a `_dev` call, a launch)
  void run(int status) {
    if (ok()) st_ = status;
  }

  // frees the arena and, when `wait` is set and nothing failed, synchronises the stream
  int finish(bool wait) {
    release();
    if (ok() && wait) check(cudaStreamSynchronize(ctx_->stream), "cudaStreamSynchronize");
    return st_;
  }

 private:
  void check(cudaError_t e, const char *what) {
    if (e == cudaSuccess || !ok()) return;
    (void)cudaGetLastError();  // reported here: do not leave it for a later launch check
    st_ = b200_fail(ctx_, e == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA, "%s failed: %s", what,
                    cudaGetErrorString(e));
  }
  void copy(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind, const char *what) {
    if (ok() && bytes) check(cudaMemcpyAsync(dst, src, bytes, kind, ctx_->stream), what);
  }
  void copy2d(void *dst, size_t dpitch, const void *src, size_t spitch, size_t row_bytes, size_t rows,
              cudaMemcpyKind kind, const char *what) {
    if (ok() && row_bytes && rows)
      check(cudaMemcpy2DAsync(dst, dpitch, src, spitch, row_bytes, rows, kind, ctx_->stream), what);
  }
  void release() {
    if (base_) cudaFreeAsync(base_, ctx_->stream);
    base_ = nullptr;
  }

  b200_ctx *ctx_;
  uint8_t *base_ = nullptr;
  size_t used_ = 0;
  int st_ = B200_OK;
};
