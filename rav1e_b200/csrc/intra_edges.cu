// intra_edges.cu — get_intra_edges for batches of transform blocks (sm_90a).
//
//   get_intra_edges                     src/partition.rs:639-898
//   has_top_right / has_bottom_left     src/recon_intra.rs:174-255, :374-452
//   supersample_chroma_bsize            src/partition.rs:559-598
//
// One warp builds one 257-pixel IntraEdge buffer with the gather of intra_edges_dev.cuh.
//
// What is batched is the caller's choice: in the encode loop a block's edges depend on its
// neighbours' reconstruction (a wavefront), in the lookahead (estimate_intra_costs, lookahead.rs:30)
// every block of a frame is independent - see lookahead.cu for that fused consumer.
#include <cuda_runtime.h>

#include <algorithm>

#include "common.cuh"
#include "intra_edges_dev.cuh"

namespace {

using namespace intra_edges;

struct EdgeArgs {
  EdgeGeom g;
  const b200_edge_item *items;
  size_t n;
  void *edges;            // n x 257 pixels
  unsigned char *lens;    // n x {init_left, init_above}
};

template <typename T>
__global__ void __launch_bounds__(256) intra_edges_kernel(const __grid_constant__ EdgeArgs a) {
  const int lane = threadIdx.x & 31;
  const size_t warp0 = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const size_t nwarps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t it = warp0; it < a.n; it += nwarps) {
    const EdgeLens l = gather_intra_edge<T>(a.g, a.items[it], lane, 32, (T *)a.edges + it * 257);
    if (lane == 0 && a.lens) {
      a.lens[2 * it] = (unsigned char)l.left;
      a.lens[2 * it + 1] = (unsigned char)l.above;
    }
  }
}

}  // namespace

extern "C" int b200_get_intra_edges_dev(b200_ctx *ctx, const b200_plane *plane, int rect_x, int rect_y,
                                        int rect_w, int rect_h, int xdec, int ydec, int bit_depth,
                                        const b200_edge_item *d_items, size_t nitems, void *d_edges,
                                        uint8_t *d_lens) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, plane && plane->data && (plane->bpp == 1 || plane->bpp == 2), "bad plane");
  B200_REQUIRE(ctx, (plane->bpp == 1) == (bit_depth == 8) && bit_depth >= 8 && bit_depth <= 12,
               "bpp %d vs bit depth %d", plane->bpp, bit_depth);
  B200_REQUIRE(ctx, rect_x >= 0 && rect_y >= 0 && rect_w > 0 && rect_h > 0 && rect_x < plane->width &&
                        rect_y < plane->height,
               "bad region rect (%d, %d, %d, %d)", rect_x, rect_y, rect_w, rect_h);
  B200_REQUIRE(ctx, (xdec == 0 || xdec == 1) && (ydec == 0 || ydec == 1), "bad decimation");
  if (nitems == 0) return B200_OK;
  B200_REQUIRE(ctx, d_items && d_edges, "NULL items / output");
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  EdgeArgs a{};
  a.g.data = (const uint8_t *)plane->data + ((long long)rect_y * plane->stride + rect_x) * plane->bpp;
  a.g.stride = plane->stride;
  a.g.plane_w = plane->width;
  a.g.plane_h = plane->height;
  a.g.rect_x = rect_x, a.g.rect_y = rect_y, a.g.rect_w = rect_w, a.g.rect_h = rect_h;
  a.g.xdec = xdec, a.g.ydec = ydec, a.g.bit_depth = bit_depth;
  a.items = d_items;
  a.n = nitems;
  a.edges = d_edges;
  a.lens = d_lens;
  const int wpc = 8;
  const int grid = (int)std::min<size_t>((nitems + wpc - 1) / wpc, (size_t)ctx->num_sms * 16);
  if (plane->bpp == 1)
    intra_edges_kernel<uint8_t><<<grid, wpc * 32, 0, ctx->stream>>>(a);
  else
    intra_edges_kernel<uint16_t><<<grid, wpc * 32, 0, ctx->stream>>>(a);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
