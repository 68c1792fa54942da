// ref_abi.cu — the reference's own extern "C" signatures for motion compensation, intra prediction
// and CDEF, symbol for symbol, suffix `_cuda` in place of the ISA (`_avx2`, `_ssse3`, ...):
//
//   rav1e_put_8tap_<fx>[_<fy>]_{8,16}bpc, rav1e_put_bilin_*      PutFn / PutHBDFn   asm/x86/mc.rs:17-38, :322-443
//   rav1e_prep_8tap_<fx>[_<fy>]_{8,16}bpc, rav1e_prep_bilin_*    PrepFn / PrepHBDFn asm/x86/mc.rs:40-59
//   rav1e_avg_{8,16}bpc                                           AvgFn / AvgHBDFn   asm/x86/mc.rs:61-76
//   rav1e_ipred_<mode>_{8,16}bpc, rav1e_ipred_z{1,2,3}_*          asm/x86/predict.rs:21-141
//   rav1e_ipred_cfl[_128|_left|_top]_*, rav1e_ipred_cfl_ac_4xx_*  asm/x86/predict.rs:142-234
//   rav1e_cdef_filter_{4x4,4x8,8x8}, rav1e_cdef_dir_{8,16}bpc     asm/x86/cdef.rs:16-37, :184-191
//
// They slot into PUT_FNS / PREP_FNS / AVG_FNS / CDEF_FILTER_FNS / CDEF_DIR_*_FNS and the `match mode`
// of asm::x86::predict::dispatch_predict_intra unchanged (INTEGRATION.md).  Each one is a thin shim
// over the per-call forms (host pointers in, one launch on the calling thread's context, result
// copied back): latency-bound by construction, they exist for drop-in completeness and check_asm-style
// cross-checks; the batched `_dev` entry points are the product path.
#include <cuda_runtime.h>

#include "host_stage.cuh"

namespace {

inline int bd_of(int bitdepth_max) { return 32 - __builtin_clz((unsigned)bitdepth_max); }  // 1023 -> 10

// PredictionMode discriminants, predict.rs:73-87
enum { M_DC = 0, M_V = 1, M_H = 2, M_D45 = 3, M_SMOOTH = 9, M_SMOOTH_V = 10, M_SMOOTH_H = 11, M_PAETH = 12, M_CFL = 13 };
enum { V_NONE = 0, V_LEFT = 1, V_TOP = 2, V_BOTH = 3 };  // PredictionVariant, predict.rs:112-118

// `topleft` addresses element 2 * MAX_TX_SIZE = 128 of the caller's IntraEdge buffer
// (IntraEdge::top_left_ptr, partition.rs:625-627); the lengths are what get_intra_edges
// initialises for the mode (partition.rs:698-705).
void ipred(int mode, int variant, void *dst, ptrdiff_t stride, const void *topleft, int bpp, int w, int h, int bd,
           const int16_t *ac, int angle, int ief, int left_len, int above_len, int plane_w, int plane_h) {
  b200_predict_intra(mode, variant, dst, stride, w, h, bd, ac, angle, ief, (const uint8_t *)topleft - 128 * bpp,
                     left_len, above_len, plane_w, plane_h, 0, 0);
}

// z1 / z2 / z3: `angle` carries enable_ief << 10 | smooth << 9 (asm/x86/predict.rs:296-302)
void ipred_z(int zone, void *dst, ptrdiff_t stride, const void *topleft, int bpp, int w, int h, int bd, int angle_arg,
             int dx, int dy) {
  const int angle = angle_arg & 511;
  const int ief = (angle_arg >> 10) & 1 ? ((angle_arg >> 9) & 1) : -1;
  // z2 clips the filtered edge at the frame (dx, dy = distance to the frame edge, :304-313); z1 / z3
  // have no frame information in their signature: beyond the frame the caller's edge is replicated,
  // so clipping changes nothing there.
  const int pw = zone == 2 ? dx : (1 << 20), ph = zone == 2 ? dy : (1 << 20);
  const int left_len = zone == 3 ? w + h : h, above_len = zone == 1 ? w + h : w;
  ipred(M_D45, V_BOTH, dst, stride, topleft, bpp, w, h, bd, nullptr, angle, ief, left_len > 128 ? 128 : left_len,
        above_len > 128 ? 128 : above_len, pw, ph);
}

void cfl_ac(int16_t *ac, const void *src, ptrdiff_t stride, int bpp, int w_pad, int h_pad, int w, int h, int xdec,
            int ydec) {
  b200_ctx *ctx = b200_default_ctx();
  const int lw = w << xdec, lh = h << ydec;
  const size_t luma_bytes = b200_align_up((size_t)lw * lh * bpp, 256);
  HostStage s(ctx, luma_bytes + 256 + (size_t)w * h * 2);
  uint8_t *d_luma = s.take((size_t)lw * lh * bpp);
  b200_block *d_blk = (b200_block *)s.take(sizeof(b200_block));
  int16_t *d_ac = (int16_t *)s.take((size_t)w * h * 2);
  const b200_block blk{0, 0};
  s.up2d(d_luma, (size_t)lw * bpp, src, (size_t)stride, (size_t)lw * bpp, lh);
  s.up(d_blk, &blk, sizeof blk);
  if (s.ok()) {
    const b200_plane p{d_luma, lw, lw, lh, 0, bpp, nullptr};
    s.run(b200_pred_cfl_ac_dev(ctx, &p, d_blk, 1, w, h, w_pad, h_pad, xdec, ydec, d_ac));
  }
  s.down(ac, d_ac, (size_t)w * h * 2);
  b200_percall_check(ctx, s.finish(true), "cfl_ac");
}

}  // namespace

// ------------------------------------------------------------------ motion compensation
// name, FilterMode x, FilterMode y (REGULAR 0, SMOOTH 1, SHARP 2, BILINEAR 3; mc.rs:98-106); the table
// slot is (x + 4 y) & 15 (asm/x86/mc.rs:80-82)
#define B200_DEF_MC(NAME, MX, MY)                                                                              \
  extern "C" void rav1e_put_##NAME##_8bpc_cuda(uint8_t *dst, ptrdiff_t ds, const uint8_t *src, ptrdiff_t ss,   \
                                               int w, int h, int mx, int my) {                                 \
    b200_put_8tap(dst, ds, src, ss, w, h, mx, my, MX, MY, 8);                                                  \
  }                                                                                                            \
  extern "C" void rav1e_put_##NAME##_16bpc_cuda(uint16_t *dst, ptrdiff_t ds, const uint16_t *src,              \
                                                ptrdiff_t ss, int w, int h, int mx, int my, int bdmax) {       \
    b200_put_8tap(dst, ds, src, ss, w, h, mx, my, MX, MY, bd_of(bdmax));                                       \
  }                                                                                                            \
  extern "C" void rav1e_prep_##NAME##_8bpc_cuda(int16_t *tmp, const uint8_t *src, ptrdiff_t ss, int w, int h,  \
                                                int mx, int my) {                                              \
    b200_prep_8tap(tmp, src, ss, w, h, mx, my, MX, MY, 8);                                                     \
  }                                                                                                            \
  extern "C" void rav1e_prep_##NAME##_16bpc_cuda(int16_t *tmp, const uint16_t *src, ptrdiff_t ss, int w,       \
                                                 int h, int mx, int my, int bdmax) {                           \
    b200_prep_8tap(tmp, src, ss, w, h, mx, my, MX, MY, bd_of(bdmax));                                          \
  }
B200_FOR_EACH_MC_FILTER(B200_DEF_MC)
#undef B200_DEF_MC

extern "C" void rav1e_avg_8bpc_cuda(uint8_t *dst, ptrdiff_t ds, const int16_t *tmp1, const int16_t *tmp2, int w,
                                    int h) {
  b200_mc_avg(dst, ds, tmp1, tmp2, w, h, 8);
}
extern "C" void rav1e_avg_16bpc_cuda(uint16_t *dst, ptrdiff_t ds, const int16_t *tmp1, const int16_t *tmp2, int w,
                                     int h, int bdmax) {
  b200_mc_avg(dst, ds, tmp1, tmp2, w, h, bd_of(bdmax));
}

// ------------------------------------------------------------------ intra prediction
// name, PredictionMode, PredictionVariant
#define B200_DEF_IPRED(NAME, MODE, VAR)                                                                        \
  extern "C" void rav1e_ipred_##NAME##_8bpc_cuda(uint8_t *dst, ptrdiff_t stride, const uint8_t *topleft,       \
                                                 int w, int h, int angle) {                                    \
    ipred(MODE, VAR, dst, stride, topleft, 1, w, h, 8, nullptr, angle, -1, h, w, 1 << 20, 1 << 20);            \
  }                                                                                                            \
  extern "C" void rav1e_ipred_##NAME##_16bpc_cuda(uint16_t *dst, ptrdiff_t stride, const uint16_t *topleft,    \
                                                  int w, int h, int angle, int max_w, int max_h, int bdmax) {  \
    (void)max_w, (void)max_h;                                                                                  \
    ipred(MODE, VAR, dst, stride, topleft, 2, w, h, bd_of(bdmax), nullptr, angle, -1, h, w, 1 << 20, 1 << 20); \
  }
B200_FOR_EACH_IPRED(B200_DEF_IPRED)
#undef B200_DEF_IPRED

extern "C" void rav1e_ipred_z1_8bpc_cuda(uint8_t *dst, ptrdiff_t stride, const uint8_t *topleft, int w, int h,
                                         int angle) {
  ipred_z(1, dst, stride, topleft, 1, w, h, 8, angle, 0, 0);
}
extern "C" void rav1e_ipred_z3_8bpc_cuda(uint8_t *dst, ptrdiff_t stride, const uint8_t *topleft, int w, int h,
                                         int angle) {
  ipred_z(3, dst, stride, topleft, 1, w, h, 8, angle, 0, 0);
}
extern "C" void rav1e_ipred_z2_8bpc_cuda(uint8_t *dst, ptrdiff_t stride, const uint8_t *topleft, int w, int h,
                                         int angle, int dx, int dy) {
  ipred_z(2, dst, stride, topleft, 1, w, h, 8, angle, dx, dy);
}
extern "C" void rav1e_ipred_z1_16bpc_cuda(uint16_t *dst, ptrdiff_t stride, const uint16_t *topleft, int w, int h,
                                          int angle, int max_w, int max_h, int bdmax) {
  (void)max_w, (void)max_h;
  ipred_z(1, dst, stride, topleft, 2, w, h, bd_of(bdmax), angle, 0, 0);
}
extern "C" void rav1e_ipred_z3_16bpc_cuda(uint16_t *dst, ptrdiff_t stride, const uint16_t *topleft, int w, int h,
                                          int angle, int max_w, int max_h, int bdmax) {
  (void)max_w, (void)max_h;
  ipred_z(3, dst, stride, topleft, 2, w, h, bd_of(bdmax), angle, 0, 0);
}
extern "C" void rav1e_ipred_z2_16bpc_cuda(uint16_t *dst, ptrdiff_t stride, const uint16_t *topleft, int w, int h,
                                          int angle, int dx, int dy, int bdmax) {
  ipred_z(2, dst, stride, topleft, 2, w, h, bd_of(bdmax), angle, dx, dy);
}

// name, PredictionVariant; `alpha` travels in the angle slot (asm/x86/predict.rs:365-373)
#define B200_DEF_CFL(NAME, VAR)                                                                                \
  extern "C" void rav1e_ipred_##NAME##_8bpc_cuda(uint8_t *dst, ptrdiff_t stride, const uint8_t *topleft,       \
                                                 int w, int h, const int16_t *ac, int alpha) {                 \
    ipred(M_CFL, VAR, dst, stride, topleft, 1, w, h, 8, ac, alpha, -1, h, w, 1 << 20, 1 << 20);                \
  }                                                                                                            \
  extern "C" void rav1e_ipred_##NAME##_16bpc_cuda(uint16_t *dst, ptrdiff_t stride, const uint16_t *topleft,    \
                                                  int w, int h, const int16_t *ac, int alpha, int bdmax) {     \
    ipred(M_CFL, VAR, dst, stride, topleft, 2, w, h, bd_of(bdmax), ac, alpha, -1, h, w, 1 << 20, 1 << 20);     \
  }
B200_FOR_EACH_CFL(B200_DEF_CFL)
#undef B200_DEF_CFL

// layout name, xdec, ydec
#define B200_DEF_CFL_AC(NAME, XDEC, YDEC)                                                                      \
  extern "C" void rav1e_ipred_cfl_ac_##NAME##_8bpc_cuda(int16_t *ac, const uint8_t *src, ptrdiff_t stride,     \
                                                        int w_pad, int h_pad, int w, int h) {                  \
    cfl_ac(ac, src, stride, 1, w_pad, h_pad, w, h, XDEC, YDEC);                                                \
  }                                                                                                            \
  extern "C" void rav1e_ipred_cfl_ac_##NAME##_16bpc_cuda(int16_t *ac, const uint16_t *src, ptrdiff_t stride,   \
                                                         int w_pad, int h_pad, int w, int h) {                 \
    cfl_ac(ac, src, stride, 2, w_pad, h_pad, w, h, XDEC, YDEC);                                                \
  }
B200_FOR_EACH_CFL_AC(B200_DEF_CFL_AC)
#undef B200_DEF_CFL_AC

// ------------------------------------------------------------------ CDEF
// size name, xdec, ydec: the table slot is decimate_index(xdec, ydec) (asm/x86/cdef.rs:40-42, :161-167)
#define B200_DEF_CDEF(NAME, XDEC, YDEC)                                                                        \
  extern "C" void rav1e_cdef_filter_##NAME##_cuda(uint8_t *dst, ptrdiff_t ds, const uint16_t *tmp,             \
                                                  ptrdiff_t ts, int pri, int sec, int dir, int damping) {      \
    b200_cdef_filter_block(dst, ds, tmp, ts, pri, sec, dir, damping, 8, XDEC, YDEC);                           \
  }                                                                                                            \
  extern "C" void rav1e_cdef_filter_##NAME##_16bpc_cuda(uint16_t *dst, ptrdiff_t ds, const uint16_t *tmp,      \
                                                        ptrdiff_t ts, int pri, int sec, int dir, int damping,  \
                                                        int bdmax) {                                           \
    b200_cdef_filter_block(dst, ds, tmp, ts, pri, sec, dir, damping, bd_of(bdmax), XDEC, YDEC);                \
  }
B200_FOR_EACH_CDEF_SIZE(B200_DEF_CDEF)
#undef B200_DEF_CDEF

extern "C" int32_t rav1e_cdef_dir_8bpc_cuda(const uint8_t *img, ptrdiff_t stride, uint32_t *var) {
  return b200_cdef_dir(img, stride, var, 8);
}
extern "C" int32_t rav1e_cdef_dir_16bpc_cuda(const uint16_t *img, ptrdiff_t stride, uint32_t *var, int bdmax) {
  return b200_cdef_dir(img, stride, var, bd_of(bdmax));
}
