// capi.cu — context, memory and plane management of the C ABI (include/b200rdo.h).
#include <mutex>

#include "host_stage.cuh"

char g_b200_last_error[512] = {0};

extern "C" int b200_abi_version(void) { return B200RDO_ABI_VERSION; }

extern "C" int b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

extern "C" const char *b200_last_error(const b200_ctx *ctx) {
  return ctx ? ctx->err : g_b200_last_error;
}

extern "C" int b200_ctx_create(int device, b200_ctx **out) {
  if (!out) return b200_fail(nullptr, B200_ERR_ARG, "b200_ctx_create: out is NULL");
  *out = nullptr;
  int n = b200_device_count();
  if (n <= 0 || device < 0 || device >= n)
    return b200_fail(nullptr, B200_ERR_NODEV,
                     "b200_ctx_create: CUDA device %d not available (%d devices); there is no "
                     "CPU fallback in this backend",
                     device, n);
  b200_ctx *ctx = new b200_ctx();
  ctx->device = device;
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) {
    int st = b200_fail(nullptr, B200_ERR_CUDA, "b200_ctx_create: %s", cudaGetErrorString(e));
    delete ctx;
    return st;
  }
  ctx->stream = ctx->own_stream;
  {  // keep stream-ordered allocations cached across calls (the host-buffer entry points
     // allocate per call; the default threshold of 0 would hand memory back at every sync)
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
      uint64_t thr = UINT64_MAX;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
  }
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && sms > 0)
    ctx->num_sms = sms;
  *out = ctx;
  return B200_OK;
}

extern "C" void b200_ctx_destroy(b200_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->dwork) cudaFree(ctx->dwork);
  for (auto &kv : ctx->scan_dev) cudaFree(kv.second);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  delete ctx;
}

extern "C" int b200_ctx_set_stream(b200_ctx *ctx, void *cuda_stream) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  ctx->stream = (cudaStream_t)cuda_stream;  // NULL is the CUDA default stream, a valid choice
  return B200_OK;
}

extern "C" int b200_ctx_reset_stream(b200_ctx *ctx) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  ctx->stream = ctx->own_stream;
  return B200_OK;
}

extern "C" int b200_ctx_set_async(b200_ctx *ctx, int enable) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  ctx->async_batch = enable ? 1 : 0;
  return B200_OK;
}

extern "C" void *b200_ctx_get_stream(b200_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

extern "C" int b200_ctx_synchronize(b200_ctx *ctx) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

extern "C" uint64_t b200_ctx_launch_count(const b200_ctx *ctx) { return ctx ? ctx->launches : 0; }

extern "C" int b200_malloc(b200_ctx *ctx, size_t bytes, void **dptr) {
  B200_REQUIRE(ctx, ctx && dptr, "b200_malloc: NULL argument");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  B200_CUDA(ctx, cudaMalloc(dptr, bytes ? bytes : 1));
  return B200_OK;
}

extern "C" int b200_free(b200_ctx *ctx, void *dptr) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  if (dptr) B200_CUDA(ctx, cudaFree(dptr));
  return B200_OK;
}

extern "C" int b200_memcpy_h2d(b200_ctx *ctx, void *dptr, const void *host, size_t bytes) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_CUDA(ctx, cudaMemcpyAsync(dptr, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
  B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

extern "C" int b200_memcpy_d2h(b200_ctx *ctx, void *host, const void *dptr, size_t bytes) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_CUDA(ctx, cudaMemcpyAsync(host, dptr, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

int b200_reserve_dwork(b200_ctx *ctx, size_t bytes) {
  if (bytes <= ctx->dwork_bytes) return B200_OK;
  if (ctx->dwork) {
    B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    B200_CUDA(ctx, cudaFree(ctx->dwork));
    ctx->dwork = nullptr;
    ctx->dwork_bytes = 0;
  }
  size_t want = b200_align_up(bytes + bytes / 4, 1 << 20);
  B200_CUDA(ctx, cudaMalloc(&ctx->dwork, want));
  ctx->dwork_bytes = want;
  return B200_OK;
}

// The context behind the per-call (reference-signature) entry points: ONE PER HOST THREAD, created
// on first use and destroyed with the thread.  rav1e calls its kernels concurrently from one rayon
// worker per tile (encoder.rs:3253) and the asm functions are re-entrant; a thread-local context
// (own stream, own scratch) keeps the per-call forms re-entrant too, with no lock anywhere.
namespace {
struct TlsCtx {
  b200_ctx *ctx = nullptr;
  ~TlsCtx() {
    if (ctx) b200_ctx_destroy(ctx);
  }
};
}  // namespace

b200_ctx *b200_default_ctx() {
  static thread_local TlsCtx t;
  if (!t.ctx) {
    int dev = 0;
    if (const char *e = getenv("B200RDO_DEVICE")) dev = atoi(e);
    // no CPU fallback, by design; the failure is recorded in the global last error
    b200_percall_check(nullptr, b200_ctx_create(dev, &t.ctx), "context creation");
  }
  return t.ctx;
}

// ------------------------------------------------------------------ planes

extern "C" int b200_plane_alloc(b200_ctx *ctx, int width, int height, int pad, int bpp,
                                b200_plane *out) {
  B200_REQUIRE(ctx, ctx && out, "b200_plane_alloc: NULL argument");
  B200_REQUIRE(ctx, width > 0 && height > 0 && pad >= 0 && (bpp == 1 || bpp == 2),
               "b200_plane_alloc: bad geometry %dx%d pad %d bpp %d", width, height, pad, bpp);
  // Row pitch: a multiple of 128 bytes, and pixel (0,0) 128-byte aligned, so 16-byte
  // vector loads of aligned columns and TMA boxes are legal.
  size_t lead = b200_align_up((size_t)pad * bpp, 128) / bpp;  // elements left of x = 0
  size_t stride = b200_align_up((lead + width + pad) * bpp, 128) / bpp;
  size_t rows = (size_t)height + 2 * (size_t)pad;
  size_t bytes = stride * rows * bpp + 256;
  void *base = nullptr;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  B200_CUDA(ctx, cudaMalloc(&base, bytes));
  B200_CUDA(ctx, cudaMemsetAsync(base, 0, bytes, ctx->stream));
  out->alloc = base;
  out->data = (uint8_t *)base + ((size_t)pad * stride + lead) * bpp;
  out->stride = (int32_t)stride;
  out->width = width;
  out->height = height;
  out->pad = pad;
  out->bpp = bpp;
  return B200_OK;
}

extern "C" int b200_plane_free(b200_ctx *ctx, b200_plane *p) {
  B200_REQUIRE(ctx, ctx && p, "b200_plane_free: NULL argument");
  if (p->alloc) B200_CUDA(ctx, cudaFree(p->alloc));
  memset(p, 0, sizeof *p);
  return B200_OK;
}

// Replicate the visible area's edges into the padding (v_frame Plane::pad).
template <typename T>
__global__ void pad_plane_kernel(T *p0, int stride, int width, int height, int pad) {
  const int total_w = width + 2 * pad;
  const int total_h = height + 2 * pad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
       i < (long long)total_w * total_h; i += (long long)gridDim.x * blockDim.x) {
    int y = (int)(i / total_w) - pad;
    int x = (int)(i % total_w) - pad;
    if (x >= 0 && x < width && y >= 0 && y < height) continue;
    int sx = min(max(x, 0), width - 1);
    int sy = min(max(y, 0), height - 1);
    p0[(long long)y * stride + x] = p0[(long long)sy * stride + sx];
  }
}

// The same from a packed copy of the visible area (row pitch = width): every pixel of the padded
// plane, border included, is written from `packed` in one pass.
template <typename T>
__global__ void unpack_pad_plane_kernel(T *p0, int stride, int width, int height, int pad, const T *packed) {
  const int total_w = width + 2 * pad;
  const int total_h = height + 2 * pad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
       i < (long long)total_w * total_h; i += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(i / total_w) - pad;
    const int x = (int)(i % total_w) - pad;
    const int sx = min(max(x, 0), width - 1);
    const int sy = min(max(y, 0), height - 1);
    p0[(long long)y * stride + x] = packed[(long long)sy * width + sx];
  }
}

// Internal (frame_pipe.cu): fill plane `p` (border included) from a packed device copy of its visible area.
int b200_plane_unpack_internal(b200_ctx *ctx, const b200_plane *p, const void *d_packed) {
  if (p->bpp == 1)
    unpack_pad_plane_kernel<uint8_t><<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(
        (uint8_t *)p->data, p->stride, p->width, p->height, p->pad, (const uint8_t *)d_packed);
  else
    unpack_pad_plane_kernel<uint16_t><<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(
        (uint16_t *)p->data, p->stride, p->width, p->height, p->pad, (const uint16_t *)d_packed);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_plane_upload(b200_ctx *ctx, const b200_plane *p, const void *host,
                                 ptrdiff_t host_stride_bytes) {
  B200_REQUIRE(ctx, ctx && p && host && p->data, "b200_plane_upload: NULL argument");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t row_bytes = (size_t)p->width * p->bpp;
  if ((size_t)host_stride_bytes == row_bytes) {
    // contiguous source: ONE linear copy (a pitched copy is a DMA descriptor per row and reaches a
    // fraction of the link rate), then unpack + replicate the border on the device
    const size_t bytes = row_bytes * p->height;
    HostStage s(ctx, bytes);
    uint8_t *packed = s.take(bytes);
    s.up(packed, host, bytes);
    if (s.ok()) s.run(b200_plane_unpack_internal(ctx, p, packed));
    if (int st = s.finish(false)) return st;
  } else {
    B200_CUDA(ctx, cudaMemcpy2DAsync(p->data, (size_t)p->stride * p->bpp, host,
                                     (size_t)host_stride_bytes, row_bytes, p->height,
                                     cudaMemcpyHostToDevice, ctx->stream));
    if (p->pad > 0) {
      if (p->bpp == 1)
        pad_plane_kernel<uint8_t><<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(
            (uint8_t *)p->data, p->stride, p->width, p->height, p->pad);
      else
        pad_plane_kernel<uint16_t><<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(
            (uint16_t *)p->data, p->stride, p->width, p->height, p->pad);
      B200_LAUNCH_CHECK(ctx);
    }
  }
  if (!ctx->async_batch) B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}

extern "C" int b200_plane_download(b200_ctx *ctx, const b200_plane *p, void *host,
                                   ptrdiff_t host_stride_bytes) {
  B200_REQUIRE(ctx, ctx && p && host && p->data, "b200_plane_download: NULL argument");
  B200_CUDA(ctx, cudaMemcpy2DAsync(host, (size_t)host_stride_bytes, p->data,
                                   (size_t)p->stride * p->bpp, (size_t)p->width * p->bpp,
                                   p->height, cudaMemcpyDeviceToHost, ctx->stream));
  B200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return B200_OK;
}
