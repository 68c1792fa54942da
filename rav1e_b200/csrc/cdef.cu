// cdef.cu — CDEF direction search and constrained directional filter (rav1e src/cdef.rs) for
// sm_90a, batched over every 8x8 block of a frame plane.
//
//   cdef_find_dir_kernel   one thread per 8x8 luma block: the 8 directional partial-sum costs
//                          (cdef.rs:84-143) held in registers, first-max direction, variance.
//   cdef_filter_kernel     a CTA stages a 64 x 16 tile + halo once (sentinels where the reference's
//                          padded scratch has them, cdef.rs:161-231), a thread filters 4 pixels of
//                          one block row with the block's parameters computed once.
// The frame-level driver reproduces cdef_filter_superblock (cdef.rs:401-570): edge flags from
// the block's position in the frame, skip -> copy, strength split, adjust_strength on luma,
// chroma damping - 1 and the 4:2:2 direction remap.
#include <algorithm>

#include "cdef_dev.cuh"
#include "host_stage.cuh"

namespace {

// Up to kCdefMaxItems (plane, tile rect) items per launch: tiles of several frames share a grid
// (blockIdx.z / the item table in the kernel parameters), so tile-sized launches are not all ramp.
constexpr int kCdefMaxItems = 32;
struct CdefItems {
  int n;
  const void *in[kCdefMaxItems];
  void *out[kCdefMaxItems];
  int in_stride[kCdefMaxItems], out_stride[kCdefMaxItems];
  const uint8_t *skip8[kCdefMaxItems];
  uint8_t *dir[kCdefMaxItems];
  int *var[kCdefMaxItems];
  short rx8[kCdefMaxItems], ry8[kCdefMaxItems], rw8[kCdefMaxItems], rh8[kCdefMaxItems];
};

template <typename T>
__global__ void cdef_find_dir_kernel(const __grid_constant__ CdefItems it, int w8, int coeff_shift) {
  const int k = blockIdx.y;
  const T *luma = (const T *)it.in[k];
  const int stride = it.in_stride[k], rw8 = it.rw8[k], rh8 = it.rh8[k];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < rw8 * rh8; i += gridDim.x * blockDim.x) {
    const int by = it.ry8[k] + i / rw8, bx = it.rx8[k] + i % rw8;
    const int b = by * w8 + bx;
    unsigned v = 0;
    int d = 0;
    if (!(it.skip8[k] && it.skip8[k][b]))
      d = find_dir_8x8<T>(luma + (long long)(8 * by) * stride + 8 * bx, stride, coeff_shift, &v);
    it.dir[k][b] = (uint8_t)d;
    it.var[k][b] = (int)v;
  }
}


struct CdefPlaneArgs {
  int plane, xdec, ydec;
  int w8, h8, sbw;  // luma 8x8 grid and superblocks per row
  int bit_depth, damping;
  const uint8_t *strength_sb;
};

// Frame-level filter.  A CTA owns a 64 x 16 pixel tile of the plane (8 x 2 luma blocks): the tile and
// its 2-pixel halo are staged ONCE into shared memory as int16, with CDEF_VERY_LARGE written wherever
// the reference's padded scratch would hold the sentinel (outside the frame: cdef.rs:161-231,
// :446-466), so the taps are plain LDS.S16 and no tap tests availability.  A thread filters 4
// horizontally adjacent pixels of one block row: strength split, adjust_strength, direction remap
// and the constrain shifts are computed once per thread, the twelve tap offsets once per thread
// (cdef_block_taps; the sentinel handling is cdef_filter_tile_px's, cdef_dev.cuh).
constexpr int kCdefTW = 64, kCdefTH = 16, kCdefPitch = 70;  // pitch: rows 35 words apart -> odd bank shift

template <typename T>
__global__ void __launch_bounds__(256) cdef_filter_kernel(const __grid_constant__ CdefPlaneArgs a,
                                                          const __grid_constant__ CdefItems it) {
  __shared__ short s_tile[(kCdefTH + 4) * kCdefPitch];
  const int item = blockIdx.z;
  const int rx8 = it.rx8[item], ry8 = it.ry8[item], rw8 = it.rw8[item], rh8 = it.rh8[item];
  const int in_stride = it.in_stride[item], out_stride = it.out_stride[item];
  const uint8_t *skip8 = it.skip8[item];
  const uint8_t *dirs = it.dir[item];
  const int *vars = it.var[item];
  const int xs_log2 = 3 - a.xdec, ys_log2 = 3 - a.ydec;
  const int pw = a.w8 << xs_log2, ph = a.h8 << ys_log2;
  const int coeff_shift = a.bit_depth - 8;
  const T *in = (const T *)it.in[item];
  T *out = (T *)it.out[item];
  const int rx1 = (rx8 + rw8) << xs_log2, ry1 = (ry8 + rh8) << ys_log2;
  const int tx0 = (rx8 << xs_log2) + blockIdx.x * kCdefTW, ty0 = (ry8 << ys_log2) + blockIdx.y * kCdefTH;
  if (tx0 >= rx1 || ty0 >= ry1) return;  // the grid covers the largest item of the launch
  // ---- stage the tile + halo
  for (int i = threadIdx.x; i < (kCdefTH + 4) * (kCdefTW + 4); i += 256) {
    const int r = i / (kCdefTW + 4), c = i - r * (kCdefTW + 4);
    const int y = ty0 + r - 2, x = tx0 + c - 2;
    short v = (short)0x8000;
    if (x >= 0 && x < pw && y >= 0 && y < ph) v = (short)in[(long long)y * in_stride + x];
    s_tile[r * kCdefPitch + c] = v;
  }
  __syncthreads();
  // ---- 4 pixels per thread
  const int row = threadIdx.x >> 4, col = (threadIdx.x & 15) * 4;
  const int x = tx0 + col, y = ty0 + row;
  if (x >= rx1 || y >= ry1) return;
  const int gy = y >> ys_log2, gx = x >> xs_log2;
  const int b = gy * a.w8 + gx;
  const short *ctr = s_tile + (row + 2) * kCdefPitch + col + 2;
  int res[4];
  if (skip8 && skip8[b]) {  // cdef.rs:557-564
#pragma unroll
    for (int j = 0; j < 4; j++) res[j] = ctr[j];
  } else {
    const CdefBlockTaps bt = cdef_block_taps(a.strength_sb + ((gy >> 3) * a.sbw + (gx >> 3)), a.plane, a.xdec, a.ydec,
                                             dirs, vars, b, a.damping, coeff_shift, kCdefPitch);
#pragma unroll
    for (int j = 0; j < 4; j++) res[j] = cdef_filter_tile_px(ctr + j, bt);
  }
  T *o = out + (long long)y * out_stride + x;
  if (x + 4 <= rx1 && ((uintptr_t)o & (4 * sizeof(T) - 1)) == 0) {
    if (sizeof(T) == 1)
      *(uchar4 *)o = make_uchar4((unsigned char)res[0], (unsigned char)res[1], (unsigned char)res[2], (unsigned char)res[3]);
    else
      *(ushort4 *)o = make_ushort4((unsigned short)res[0], (unsigned short)res[1], (unsigned short)res[2], (unsigned short)res[3]);
  } else {
#pragma unroll
    for (int j = 0; j < 4; j++)
      if (x + j < rx1) o[j] = (T)res[j];
  }
}

// Asm-facing single block: padded u16 tile in, pixels out (asm/x86/cdef.rs:16-37).
template <typename T>
__global__ void cdef_filter_tmp16_kernel(T *dst, int dst_stride, const uint16_t *tmp, int tmp_stride,
                                         int pri, int sec, int dir, int damping, int bit_depth,
                                         int xsize, int ysize) {
  const int t = threadIdx.x;
  if (t >= xsize * ysize) return;
  const int i = t / xsize, j = t - i * xsize;
  auto load = [&](int dy, int dx) -> int { return (int)tmp[(i + dy) * tmp_stride + (j + dx)]; };
  dst[i * dst_stride + j] = (T)cdef_pixel(load, pri, sec, dir, damping, bit_depth - 8);
}

}  // namespace

namespace {

int check_rect(b200_ctx *ctx, int w8, int h8, int rx8, int ry8, int rw8, int rh8) {
  B200_REQUIRE(ctx, rx8 >= 0 && ry8 >= 0 && rw8 > 0 && rh8 > 0 && rx8 + rw8 <= w8 && ry8 + rh8 <= h8,
               "block rect (%d, %d, %d, %d) outside the %d x %d grid", rx8, ry8, rw8, rh8, w8, h8);
  return B200_OK;
}

// The filter reads (and writes) the plane's (luma >> dec) area and nothing outside it, so a smaller
// plane would give wrong pixels without any fault: it is rejected.
int check_plane(b200_ctx *ctx, const b200_plane *p, size_t k, const char *what, int width, int height, int bpp) {
  B200_REQUIRE(ctx, p->bpp == bpp, "item %zu: %s bpp %d, expected %d", k, what, p->bpp, bpp);
  B200_REQUIRE(ctx, p->width >= width && p->height >= height && p->stride >= p->width,
               "item %zu: %s plane %dx%d (stride %d) smaller than the %dx%d the filter covers", k, what, p->width,
               p->height, p->stride, width, height);
  return B200_OK;
}

int check_item(b200_ctx *ctx, const b200_cdef_item &q, size_t k, int xdec, int ydec, int luma_width, int luma_height,
               int bit_depth, int do_filter) {
  B200_REQUIRE(ctx, q.in && q.in->data && q.d_dir && q.d_var, "item %zu: NULL plane / dir / var", k);
  const int bpp = bit_depth == 8 ? 1 : 2;
  if (int st = check_plane(ctx, q.in, k, "in", luma_width >> xdec, luma_height >> ydec, bpp)) return st;
  if (do_filter) {
    B200_REQUIRE(ctx, q.out && q.out->data && q.out->data != q.in->data,
                 "item %zu: the filter needs a distinct output plane (taps read unfiltered neighbours)", k);
    if (int st = check_plane(ctx, q.out, k, "out", luma_width >> xdec, luma_height >> ydec, bpp)) return st;
  }
  return check_rect(ctx, luma_width >> 3, luma_height >> 3, q.rx8, q.ry8, q.rw8, q.rh8);
}

// items [k0, k0 + n) of a host item array, already checked -> one launch of each requested kernel
int cdef_launch(b200_ctx *ctx, const b200_cdef_item *items, int n, int plane, int xdec, int ydec, int luma_width,
                int luma_height, int bit_depth, int damping, const uint8_t *d_strength_sb, int do_dir, int do_filter) {
  CdefItems it{};
  it.n = n;
  int max_w8 = 0, max_h8 = 0;
  const int bpp = bit_depth == 8 ? 1 : 2;
  for (int k = 0; k < n; k++) {
    const b200_cdef_item &q = items[k];
    it.in[k] = q.in->data;
    it.in_stride[k] = q.in->stride;
    it.out[k] = do_filter ? q.out->data : nullptr;
    it.out_stride[k] = do_filter ? q.out->stride : 0;
    it.skip8[k] = q.d_skip8;
    it.dir[k] = q.d_dir;
    it.var[k] = q.d_var;
    it.rx8[k] = (short)q.rx8, it.ry8[k] = (short)q.ry8, it.rw8[k] = (short)q.rw8, it.rh8[k] = (short)q.rh8;
    max_w8 = std::max(max_w8, q.rw8);
    max_h8 = std::max(max_h8, q.rh8);
  }
  if (do_dir) {
    const dim3 grid(std::max(1, std::min((max_w8 * max_h8 + 127) / 128, ctx->num_sms * 16 / n)), n);
    if (bpp == 1)
      cdef_find_dir_kernel<uint8_t><<<grid, 128, 0, ctx->stream>>>(it, luma_width >> 3, bit_depth - 8);
    else
      cdef_find_dir_kernel<uint16_t><<<grid, 128, 0, ctx->stream>>>(it, luma_width >> 3, bit_depth - 8);
    B200_LAUNCH_CHECK(ctx);
  }
  if (do_filter) {
    CdefPlaneArgs a;
    a.plane = plane;
    a.xdec = xdec;
    a.ydec = ydec;
    a.w8 = luma_width >> 3;
    a.h8 = luma_height >> 3;
    a.sbw = (luma_width + 63) >> 6;
    a.bit_depth = bit_depth;
    a.damping = damping;
    a.strength_sb = d_strength_sb;
    const dim3 grid((((max_w8 * 8) >> xdec) + kCdefTW - 1) / kCdefTW, (((max_h8 * 8) >> ydec) + kCdefTH - 1) / kCdefTH, n);
    if (bpp == 1)
      cdef_filter_kernel<uint8_t><<<grid, 256, 0, ctx->stream>>>(a, it);
    else
      cdef_filter_kernel<uint16_t><<<grid, 256, 0, ctx->stream>>>(a, it);
    B200_LAUNCH_CHECK(ctx);
  }
  return B200_OK;
}

int cdef_items(b200_ctx *ctx, const b200_cdef_item *items, size_t nitems, int plane, int xdec, int ydec,
               int luma_width, int luma_height, int bit_depth, int damping, const uint8_t *d_strength_sb, int do_dir,
               int do_filter) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, (luma_width & 7) == 0 && (luma_height & 7) == 0 && luma_width > 0 && luma_height > 0,
               "luma %dx%d must be a multiple of 8 (rav1e pads frames to 8)", luma_width, luma_height);
  B200_REQUIRE(ctx, plane >= 0 && plane < 3, "bad plane %d", plane);
  B200_REQUIRE(ctx, (xdec == 0 && ydec == 0) || (xdec == 1 && ydec == 0) || (xdec == 1 && ydec == 1),
               "chroma layout (xdec %d, ydec %d) is not 4:4:4, 4:2:2 or 4:2:0", xdec, ydec);
  B200_REQUIRE(ctx, plane != 0 || (xdec == 0 && ydec == 0), "luma with xdec %d, ydec %d", xdec, ydec);
  B200_REQUIRE(ctx, !do_dir || plane == 0, "directions are searched on the luma plane");
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  if (do_filter) {
    // fi.cdef_damping = 3 + (base_q_idx >> 6) (encoder.rs:1221); the direction-only calls pass none
    B200_REQUIRE(ctx, damping >= 3 && damping <= 6, "damping %d outside 3..6", damping);
    B200_REQUIRE(ctx, d_strength_sb, "NULL strengths");
  }
  if (nitems == 0) return B200_OK;
  B200_REQUIRE(ctx, items != nullptr, "NULL items");
  // every item of every phase is checked before the first launch: a rejected call launches nothing
  for (size_t k = 0; k < nitems; k++)
    if (int st = check_item(ctx, items[k], k, xdec, ydec, luma_width, luma_height, bit_depth, do_filter)) return st;
  B200_CUDA(ctx, cudaSetDevice(ctx->device));
  // all the directions first: a tile's filter reads only its own blocks' directions, but keeping the
  // two phases apart lets one call serve callers that filter several planes from one analysis
  for (int phase = 0; phase < 2; phase++) {
    if (!(phase == 0 ? do_dir : do_filter)) continue;
    for (size_t k0 = 0; k0 < nitems; k0 += kCdefMaxItems) {
      const int n = (int)std::min<size_t>(kCdefMaxItems, nitems - k0);
      if (int st = cdef_launch(ctx, items + k0, n, plane, xdec, ydec, luma_width, luma_height, bit_depth, damping,
                               d_strength_sb, phase == 0, phase == 1))
        return st;
    }
  }
  return B200_OK;
}

}  // namespace

extern "C" int b200_cdef_find_dir_dev(b200_ctx *ctx, const b200_plane *luma, int bit_depth,
                                      const uint8_t *d_skip8, uint8_t *d_dir, int32_t *d_var) {
  B200_REQUIRE(ctx, ctx != nullptr && luma != nullptr, "NULL argument");
  const b200_cdef_item q{luma, nullptr, d_skip8, d_dir, d_var, 0, 0, luma->width >> 3, luma->height >> 3};
  return cdef_items(ctx, &q, 1, 0, 0, 0, luma->width, luma->height, bit_depth, 0, nullptr, 1, 0);
}

extern "C" int b200_cdef_find_dir_rect_dev(b200_ctx *ctx, const b200_plane *luma, int bit_depth,
                                           const uint8_t *d_skip8, uint8_t *d_dir, int32_t *d_var, int rx8, int ry8,
                                           int rw8, int rh8) {
  B200_REQUIRE(ctx, ctx != nullptr && luma != nullptr, "NULL argument");
  const b200_cdef_item q{luma, nullptr, d_skip8, d_dir, d_var, rx8, ry8, rw8, rh8};
  return cdef_items(ctx, &q, 1, 0, 0, 0, luma->width, luma->height, bit_depth, 0, nullptr, 1, 0);
}

extern "C" int b200_cdef_filter_plane_dev(b200_ctx *ctx, const b200_plane *in, const b200_plane *out,
                                          int plane, int xdec, int ydec, int luma_width,
                                          int luma_height, int bit_depth, int damping,
                                          const uint8_t *d_skip8, const uint8_t *d_dir,
                                          const int32_t *d_var, const uint8_t *d_strength_sb) {
  const b200_cdef_item q{in, out, d_skip8, (uint8_t *)d_dir, (int32_t *)d_var, 0, 0, luma_width >> 3, luma_height >> 3};
  return cdef_items(ctx, &q, 1, plane, xdec, ydec, luma_width, luma_height, bit_depth, damping, d_strength_sb, 0, 1);
}

extern "C" int b200_cdef_filter_rect_dev(b200_ctx *ctx, const b200_plane *in, const b200_plane *out, int plane,
                                         int xdec, int ydec, int luma_width, int luma_height, int bit_depth,
                                         int damping, const uint8_t *d_skip8, const uint8_t *d_dir,
                                         const int32_t *d_var, const uint8_t *d_strength_sb, int rx8, int ry8,
                                         int rw8, int rh8) {
  const b200_cdef_item q{in, out, d_skip8, (uint8_t *)d_dir, (int32_t *)d_var, rx8, ry8, rw8, rh8};
  return cdef_items(ctx, &q, 1, plane, xdec, ydec, luma_width, luma_height, bit_depth, damping, d_strength_sb, 0, 1);
}

extern "C" int b200_cdef_tiles_dev(b200_ctx *ctx, const b200_cdef_item *items, size_t nitems, int plane, int xdec,
                                   int ydec, int luma_width, int luma_height, int bit_depth, int damping,
                                   const uint8_t *d_strength_sb, int find_dir, int filter) {
  return cdef_items(ctx, items, nitems, plane, xdec, ydec, luma_width, luma_height, bit_depth, damping, d_strength_sb,
                    find_dir, filter);
}

// ---- per-call forms with the reference's asm signatures (asm/x86/cdef.rs:16-37, :184-191)
extern "C" int32_t b200_cdef_dir(const void *img, ptrdiff_t stride, uint32_t *var, int bit_depth) {
  b200_ctx *ctx = b200_default_ctx();
  const int bpp = bit_depth == 8 ? 1 : 2;
  HostStage s(ctx, 3 * 256);
  uint8_t *d_img = s.take(64 * bpp), *d_dir = s.take(1);
  int32_t *d_var = (int32_t *)s.take(4);
  s.up2d(d_img, 8 * bpp, img, (size_t)stride, 8 * bpp, 8);
  if (s.ok()) {
    b200_plane p{d_img, 8, 8, 8, 0, bpp, nullptr};
    s.run(b200_cdef_find_dir_dev(ctx, &p, bit_depth, nullptr, d_dir, d_var));
  }
  uint8_t dir = 0;
  int32_t v = 0;
  s.down(&dir, d_dir, 1);
  s.down(&v, d_var, 4);
  b200_percall_check(ctx, s.finish(true), "cdef_dir");
  *var = (uint32_t)v;
  return dir;
}

namespace {
int cdef_filter_tmp16(b200_ctx *ctx, void *d_dst, const uint16_t *d_tmp, int tw, int pri_strength, int sec_strength,
                      int dir, int damping, int bit_depth, int xsize, int ysize) {
  if (bit_depth == 8)
    cdef_filter_tmp16_kernel<uint8_t><<<1, 64, 0, ctx->stream>>>((uint8_t *)d_dst, xsize, d_tmp, tw, pri_strength,
                                                                 sec_strength, dir, damping, bit_depth, xsize, ysize);
  else
    cdef_filter_tmp16_kernel<uint16_t><<<1, 64, 0, ctx->stream>>>((uint16_t *)d_dst, xsize, d_tmp, tw, pri_strength,
                                                                  sec_strength, dir, damping, bit_depth, xsize, ysize);
  B200_LAUNCH_CHECK(ctx);
  return B200_OK;
}
}  // namespace

extern "C" void b200_cdef_filter_block(void *dst, ptrdiff_t dst_stride, const uint16_t *tmp,
                                       ptrdiff_t tmp_stride, int pri_strength, int sec_strength,
                                       int dir, int damping, int bit_depth, int xdec, int ydec) {
  b200_ctx *ctx = b200_default_ctx();
  const int bpp = bit_depth == 8 ? 1 : 2;
  const int xsize = 8 >> xdec, ysize = 8 >> ydec;
  const int tw = xsize + 4, th = ysize + 4;
  HostStage s(ctx, 512 + 64 * bpp);
  uint16_t *d_tile = (uint16_t *)s.take((size_t)tw * th * 2);
  uint8_t *d_dst = s.take(64 * bpp);
  // the caller's pointer addresses the block's top-left inside the padded tile (2 px border);
  // tmp_stride is in BYTES like every asm-ABI stride
  const uint8_t *h0 = (const uint8_t *)tmp - 2 * tmp_stride - 2 * 2;
  s.up2d(d_tile, tw * 2, h0, (size_t)tmp_stride, tw * 2, th);
  if (s.ok())
    s.run(cdef_filter_tmp16(ctx, d_dst, d_tile + 2 * tw + 2, tw, pri_strength, sec_strength, dir, damping, bit_depth,
                            xsize, ysize));
  s.down2d(dst, (size_t)dst_stride, d_dst, xsize * bpp, xsize * bpp, ysize);
  b200_percall_check(ctx, s.finish(true), "cdef_filter_block");
}
