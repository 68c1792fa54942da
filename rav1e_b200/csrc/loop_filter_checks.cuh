// loop_filter_checks.cuh — the host checks the loop-filter RDO entry points (b200_cdef_rdo_dev,
// b200_lrf_search_dev, b200_loop_decision_dev) share, and the loop-restoration range predicates the
// restoration filter (lrf.cu) checks its records with.  Each check returns B200_OK or the failure status.
#pragma once
#include <algorithm>
#include <vector>

#include "common.cuh"

namespace {

// a restoration unit size: a power of two in 32..256
inline bool lrf_unit_size_ok(int s) { return s >= 32 && s <= 256 && (s & (s - 1)) == 0; }

// a self-guided filter's xqd pair (SGRPROJ_XQD_MIN / MAX, lrf.rs:39-48)
inline bool sgrproj_xqd_ok(int x0, int x1) { return x0 >= -96 && x0 <= 31 && x1 >= -32 && x1 <= 95; }

// the context, plane count, chroma layout, bit depth and frame size
inline int lf_check_frame(b200_ctx *ctx, int planes, int xdec, int ydec, int bit_depth, int frame_width,
                          int frame_height) {
  B200_REQUIRE(ctx, ctx != nullptr, "ctx is NULL");
  B200_REQUIRE(ctx, planes == 1 || planes == 3, "planes must be 1 or 3, got %d", planes);
  B200_REQUIRE(ctx, (xdec == 1 && ydec == 1) || (xdec == 1 && ydec == 0) || (xdec == 0 && ydec == 0),
               "chroma layout (xdec %d, ydec %d) is not 4:2:0, 4:2:2 or 4:4:4", xdec, ydec);
  B200_REQUIRE(ctx, bit_depth == 8 || bit_depth == 10 || bit_depth == 12, "bad bit depth %d", bit_depth);
  B200_REQUIRE(ctx, frame_width > 0 && frame_height > 0 && frame_width <= 65536 && frame_height <= 65536,
               "bad frame size %dx%d", frame_width, frame_height);
  return B200_OK;
}

// one plane list: every plane set, of the bit depth's pixel size and covering the frame's 8x8 blocks
inline int lf_check_planes(b200_ctx *ctx, const b200_plane *pl, int planes, int xdec, int ydec, int bit_depth,
                           int frame_width, int frame_height) {
  const int bpp = bit_depth == 8 ? 1 : 2;
  const int w8px = (frame_width + 7) & ~7, h8px = (frame_height + 7) & ~7;
  for (int p = 0; p < planes; p++) {
    const int xd = p ? xdec : 0, yd = p ? ydec : 0;
    B200_REQUIRE(ctx, pl[p].data != nullptr, "NULL plane %d", p);
    B200_REQUIRE(ctx, pl[p].bpp == bpp, "plane %d: bpp %d does not match bit depth %d", p, pl[p].bpp, bit_depth);
    B200_REQUIRE(ctx, pl[p].width >= (w8px >> xd) && pl[p].height >= (h8px >> yd) && pl[p].stride >= pl[p].width,
                 "plane %d (%dx%d) smaller than the frame's 8x8 blocks (%dx%d)", p, pl[p].width, pl[p].height,
                 w8px >> xd, h8px >> yd);
  }
  return B200_OK;
}

// the CDEF parameters: fi.cdef_damping = 3 + (base_q_idx >> 6) (encoder.rs:1221), cdef_bits, 6-bit strengths
inline int lf_check_cdef(b200_ctx *ctx, int damping, int cdef_bits, const uint8_t *y_strengths,
                         const uint8_t *uv_strengths) {
  B200_REQUIRE(ctx, y_strengths && uv_strengths, "NULL strengths");
  B200_REQUIRE(ctx, damping >= 3 && damping <= 6, "damping %d outside 3..6", damping);
  B200_REQUIRE(ctx, cdef_bits >= 0 && cdef_bits <= 3, "cdef_bits %d outside 0..3", cdef_bits);
  for (int i = 0; i < 1 << cdef_bits; i++)
    B200_REQUIRE(ctx, y_strengths[i] <= 63 && uv_strengths[i] <= 63, "strength %d above 63 at index %d",
                 std::max(y_strengths[i], uv_strengths[i]), i);
  return B200_OK;
}

// each plane's restoration unit size: whole superblocks, at most the 4x4 of an area (rdo.rs:2160-2162)
inline int lf_check_unit_sizes(b200_ctx *ctx, const int *unit_size, int planes, int xdec, int ydec) {
  B200_REQUIRE(ctx, unit_size != nullptr, "NULL unit_size");
  for (int p = 0; p < planes; p++) {
    const int xd = p ? xdec : 0, yd = p ? ydec : 0, us = unit_size[p];
    B200_REQUIRE(ctx, lrf_unit_size_ok(us) && ((us << xd) % 64) == 0 && ((us << yd) % 64) == 0 && (us << xd) <= 256 &&
                          (us << yd) <= 256,
                 "plane %d: unit size %d is not 32..256 in whole superblocks", p, us);
  }
  return B200_OK;
}

// the areas: 1..4 superblocks a side inside the frame's superblock grid and, with `disjoint`, no superblock twice
inline int lf_check_areas(b200_ctx *ctx, const b200_cdef_rdo_area *areas, size_t n_areas, int frame_width,
                          int frame_height, bool disjoint) {
  B200_REQUIRE(ctx, areas != nullptr, "NULL areas");
  const int sbw = (frame_width + 63) >> 6, sbh = (frame_height + 63) >> 6;
  std::vector<uint8_t> used(disjoint ? (size_t)sbw * sbh : 0, 0);
  for (size_t k = 0; k < n_areas; k++) {
    const b200_cdef_rdo_area &r = areas[k];
    B200_REQUIRE(ctx, r.sb_w >= 1 && r.sb_w <= 4 && r.sb_h >= 1 && r.sb_h <= 4, "area %zu: %dx%d superblocks", k,
                 r.sb_w, r.sb_h);
    B200_REQUIRE(ctx, r.sbx >= 0 && r.sby >= 0 && r.sbx + r.sb_w <= sbw && r.sby + r.sb_h <= sbh,
                 "area %zu (%d, %d, %dx%d) outside the %dx%d superblock frame", k, r.sbx, r.sby, r.sb_w, r.sb_h, sbw,
                 sbh);
    if (disjoint)
      for (int y = r.sby; y < r.sby + r.sb_h; y++)
        for (int x = r.sbx; x < r.sbx + r.sb_w; x++) {
          B200_REQUIRE(ctx, !used[(size_t)y * sbw + x], "area %zu overlaps an earlier area at superblock (%d, %d)",
                       k, x, y);
          used[(size_t)y * sbw + x] = 1;
        }
  }
  return B200_OK;
}

}  // namespace
