// ipred.cu — batched AV1 intra prediction (rav1e src/predict.rs:705-1505) for sm_90a.
//
// One CTA per (block, mode) item: the RDO loop evaluates ~13 modes per block from the same
// neighbour pixels (rdo.rs:1470-1505), so a launch carries blocks x modes items that all read a
// small IntraEdge buffer (partition.rs:600-637) and write a packed w x h prediction.  The
// edge buffer is staged in shared memory, the CTA runs the preparation step of ipred_dev.cuh
// (DC value, edge filter and upsampler) and then every thread evaluates its pixels.
#include "host_stage.cuh"
#include "ipred_dev.cuh"

namespace {

using namespace ipred;

struct IpredArgs {
  const void *edges;           // n_edges x kEdgeLen pixels
  const b200_intra_item *items;
  const short *ac;             // CfL ac blocks, w*h each
  void *out;                   // n x h x w pixels
  size_t n;
  int w, h, bit_depth;
  int plane_w, plane_h;
};

template <typename T>
__global__ void __launch_bounds__(128) ipred_kernel(IpredArgs a) {
  __shared__ int s_edge[kEdgeLen];      // raw IntraEdge buffer, top-left at [128]
  __shared__ int s_af[2][kEdgeLen];     // above: staging scratch, filtered / upsampled
  __shared__ int s_lf[2][kEdgeLen];     // left (index 0 = top-left, growing downwards)
  __shared__ int s_dc;
  const CtaGroup g;
  const int w = a.w, h = a.h;
  const int maxv = (1 << a.bit_depth) - 1;
  for (size_t it = blockIdx.x; it < a.n; it += gridDim.x) {
    const b200_intra_item item = a.items[it];
    const T *edge = (const T *)a.edges + (size_t)item.edge * kEdgeLen;
    __syncthreads();
    for (int i = threadIdx.x; i < kEdgeLen; i += blockDim.x) s_edge[i] = (int)edge[i];
    __syncthreads();
    const int mode = item.mode;
    const bool dc_like = mode == DC_PRED || mode == UV_CFL_PRED;
    if (dc_like) {
      if (threadIdx.x == 0) s_dc = ipred_dc(s_edge, item.variant, w, h, item.left_len, a.bit_depth);
      __syncthreads();
    }
    IpredPix p = ipred_setup(s_edge, mode, item.angle, item.ief, item.left_len, w, h, a.bit_depth, s_af[1], s_lf[1],
                             dc_like ? s_dc : 0);
    if (p.directional && p.enable)
      ipred_filter_edges(g, p, item.above_len, a.plane_w, a.plane_h, item.x, item.y, s_af[0], s_lf[0], s_af[1],
                         s_lf[1]);
    T *out = (T *)a.out + it * (size_t)w * h;
    const short alpha = (short)item.angle;
    const short *ac = (mode == UV_CFL_PRED && alpha != 0) ? a.ac + (size_t)item.ac * w * h : nullptr;
    for (int i = threadIdx.x; i < w * h; i += blockDim.x) {
      const int r = i / w, c = i - r * w;
      int v = ipred_pixel(p, r, c);
      if (ac) v = cfl_pixel(v, alpha, ac[i], maxv);  // pred_cfl_inner, predict.rs:1065-1088
      out[i] = (T)v;
    }
  }
}

// pred_cfl_ac (predict.rs:1020-1063): one CTA per block.
struct CflAcArgs {
  const void *luma;
  int stride;
  const b200_block *blocks;  // luma position of each block
  size_t n;
  int bw, bh, w_pad, h_pad, xdec, ydec;
  short *ac;
};

template <typename T>
__global__ void __launch_bounds__(128) cfl_ac_kernel(CflAcArgs a) {
  __shared__ int s_sum[4];
  __shared__ int s_avg;
  const int bw = a.bw, bh = a.bh;
  const CflAcShape shape = cfl_ac_shape(bw, bh, a.w_pad, a.h_pad, a.xdec, a.ydec);
  for (size_t blk = blockIdx.x; blk < a.n; blk += gridDim.x) {
    const b200_block b = a.blocks[blk];
    const T *luma = (const T *)a.luma + (long long)b.y * a.stride + b.x;
    short *ac = a.ac + blk * (size_t)bw * bh;
    int local = 0;
    for (int i = threadIdx.x; i < bw * bh; i += blockDim.x) {
      const short s = cfl_ac_sample(shape, luma, a.stride, i);
      ac[i] = s;
      local += s;
    }
    local = (int)warp_sum_u32((uint32_t)local);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
      int sum = 0;
      for (int k = 0; k < (int)(blockDim.x >> 5); k++) sum += s_sum[k];
      s_avg = cfl_ac_average(shape, sum);
    }
    __syncthreads();
    const short avg = (short)s_avg;
    for (int i = threadIdx.x; i < bw * bh; i += blockDim.x) ac[i] = (short)(ac[i] - avg);
  }
}

bool valid_tx_dim(int v) { return v == 4 || v == 8 || v == 16 || v == 32 || v == 64; }

}  // namespace

extern "C" int b200_predict_intra_dev(b200_ctx *ctx, const void *d_edges, const b200_intra_item *d_items,
                                      size_t nitems, const int16_t *d_ac, int w, int h, int bit_depth,
                                      int plane_w, int plane_h, void *d_out) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, valid_tx_dim(w) && valid_tx_dim(h), "tx block %dx%d not a TxSize", w, h);
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  if (nitems == 0) return B200_OK;
  B200_REQUIRE(ctx, d_edges && d_items && d_out, "NULL argument");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  IpredArgs a;
  a.edges = d_edges;
  a.items = d_items;
  a.ac = d_ac;
  a.out = d_out;
  a.n = nitems;
  a.w = w;
  a.h = h;
  a.bit_depth = bit_depth;
  a.plane_w = plane_w;
  a.plane_h = plane_h;
  const int grid = (int)std::min<size_t>(nitems, (size_t)ctx->num_sms * 32);
  if (bit_depth == 8)
    ipred_kernel<uint8_t><<<grid, 128, 0, ctx->stream>>>(a);
  else
    ipred_kernel<uint16_t><<<grid, 128, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

extern "C" int b200_pred_cfl_ac_dev(b200_ctx *ctx, const b200_plane *luma, const b200_block *d_blocks,
                                    size_t nblocks, int bw, int bh, int w_pad, int h_pad, int xdec,
                                    int ydec, int16_t *d_ac) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, luma && luma->data, "bad luma plane");
  B200_REQUIRE(ctx, bw >= 4 && bh >= 4 && bw <= 32 && bh <= 32 && (bw & (bw - 1)) == 0 && (bh & (bh - 1)) == 0,
               "CfL block %dx%d out of range", bw, bh);
  B200_REQUIRE(ctx, (xdec == 0 || xdec == 1) && (ydec == 0 || ydec == 1) && !(ydec && !xdec), "bad decimation");
  if (nblocks == 0) return B200_OK;
  B200_REQUIRE(ctx, d_blocks && d_ac, "NULL argument");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  CflAcArgs a{luma->data, luma->stride, d_blocks, nblocks, bw, bh, w_pad, h_pad, xdec, ydec, d_ac};
  const int grid = (int)std::min<size_t>(nblocks, (size_t)ctx->num_sms * 32);
  if (luma->bpp == 1)
    cfl_ac_kernel<uint8_t><<<grid, 128, 0, ctx->stream>>>(a);
  else
    cfl_ac_kernel<uint16_t><<<grid, 128, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}

// Per-call form mirroring dispatch_predict_intra (predict.rs:705-784): host pointers, dst stride
// in BYTES; edge = the reference's IntraEdge buffer (4*64+1 pixels, top-left at [128]).
extern "C" void b200_predict_intra(int mode, int variant, void *dst, ptrdiff_t dst_stride, int w, int h,
                                   int bit_depth, const int16_t *ac, int angle, int ief,
                                   const void *edge, int left_len, int above_len, int plane_w,
                                   int plane_h, int dst_x, int dst_y) {
  b200_ctx *ctx = b200_default_ctx();
  const int bpp = bit_depth == 8 ? 1 : 2;
  const size_t edge_bytes = b200_align_up((size_t)kEdgeLen * bpp, 256);
  const size_t ac_bytes = b200_align_up((size_t)w * h * 2, 256);
  HostStage s(ctx, edge_bytes + ac_bytes + 256 + (size_t)w * h * bpp);
  uint8_t *d_edge = s.take((size_t)kEdgeLen * bpp), *d_ac = s.take((size_t)w * h * 2);
  uint8_t *d_item = s.take(sizeof(b200_intra_item)), *d_out = s.take((size_t)w * h * bpp);
  b200_intra_item item{};
  item.edge = 0;
  item.ac = 0;
  item.x = (int16_t)dst_x;
  item.y = (int16_t)dst_y;
  item.angle = (int16_t)angle;
  item.mode = (uint8_t)mode;
  item.variant = (uint8_t)variant;
  item.ief = (int8_t)ief;
  item.left_len = (uint8_t)left_len;
  item.above_len = (uint8_t)above_len;
  s.up(d_edge, edge, (size_t)kEdgeLen * bpp);
  s.up(d_item, &item, sizeof item);
  if (ac) s.up(d_ac, ac, (size_t)w * h * 2);
  if (s.ok())
    s.run(b200_predict_intra_dev(ctx, d_edge, (const b200_intra_item *)d_item, 1, (const int16_t *)d_ac, w, h,
                                 bit_depth, plane_w, plane_h, d_out));
  s.down2d(dst, (size_t)dst_stride, d_out, (size_t)w * bpp, (size_t)w * bpp, h);
  b200_percall_check(ctx, s.finish(true), "predict_intra");
}
