"""Temporal RDO in the oracle (oracle/temporal_rdo.c): the logexp helpers against the reference's own
known answers and round-trip tests (util/logexp.rs:292-358), the importance propagation of
compute_block_importances / update_block_importances (api/internal.rs:912-1230) against an independent
float32 numpy model (nothing upstream pins it), distortion_scale_for (rdo.rs:506-553) against
math.pow, and compute_{spatio,}temporal_scores (encoder.rs:744-777) against a Python restatement.
The window builders here are shared with tests/test_temporal_rdo_gpu.py and bench_kernels.py."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

from tests import oracle_lib as O
from tests.test_oracle_lookahead import satd8

KATS = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "logexp_kats.json")))
I64 = C.c_int64


def T():
    l = O.lib()
    vp, pd, sz, i32, u32 = C.c_void_p, C.c_ssize_t, C.c_size_t, C.c_int, C.c_uint32
    l.orc_bexp64.restype, l.orc_bexp64.argtypes = I64, [I64]
    l.orc_blog64.restype, l.orc_blog64.argtypes = I64, [I64]
    l.orc_blog32_q11.restype, l.orc_blog32_q11.argtypes = C.c_int32, [u32]
    l.orc_dscale_mul.restype, l.orc_dscale_mul.argtypes = u32, [u32, u32]
    l.orc_distortion_scale_for.restype, l.orc_distortion_scale_for.argtypes = u32, [C.c_double, C.c_double]
    l.orc_distortion_scales.restype, l.orc_distortion_scales.argtypes = None, [vp, sz, vp, sz, vp]
    l.orc_temporal_scores.restype, l.orc_temporal_scores.argtypes = I64, [vp, sz, vp, vp, vp]
    l.orc_block_importances.restype = None
    l.orc_block_importances.argtypes = [sz, vp, pd, i32, i32, i32, vp, vp, sz, vp, vp]
    return l


# ---------------------------------------------------------------- windows
class Window:
    """nframes source luma planes + intra-cost maps + vector maps + a step list (src, dst, len, mv_index)."""

    def __init__(self, imgs, pad, intra, mvs, steps, bd):
        self.imgs, self.pad, self.intra, self.mvs, self.steps, self.bd = imgs, pad, intra, mvs, steps, bd
        self.H, self.W = imgs[0].shape
        self.w_imp, self.h_imp = (self.W + 7) // 8, (self.H + 7) // 8
        self.n_imp, self.n_intra = self.w_imp * self.h_imp, (self.W // 8) * (self.H // 8)
        self.planes = []
        for im in imgs:
            p = O.Plane(self.W, self.H, pad, dtype=im.dtype)
            p.fill_from(im)
            self.planes.append(p)


def _frames(n, W, H, dtype, bd, rng, drift=(5, -3)):
    """low-passed noise drifting by `drift` px per frame, plus noise: real minima for the vectors"""
    maxv = (1 << bd) - 1
    m = 8 * n + 64
    base = rng.integers(0, maxv + 1, (H + 2 * m, W + 2 * m)).astype(np.float64)
    k = np.ones(5) / 5.0
    base = np.apply_along_axis(lambda r: np.convolve(r, k, mode="same"), 1, base)
    base = np.apply_along_axis(lambda c: np.convolve(c, k, mode="same"), 0, base)
    base = (base - base.min()) / (base.max() - base.min()) * maxv
    out = []
    for f in range(n):
        oy, ox = m + f * drift[1], m + f * drift[0]
        im = base[oy:oy + H, ox:ox + W] + rng.normal(0, 3 << (bd - 8), (H, W))
        out.append(np.ascontiguousarray(np.clip(np.rint(im), 0, maxv).astype(dtype)))
    return out


def _intra(n, n_intra, rng, bd, zero_frac=0.1):
    c = rng.integers(0, 6000 << (bd - 8), (n, n_intra)).astype(np.uint32)
    c[rng.random((n, n_intra)) < zero_frac] = 0
    return c


def small_window(dtype=np.uint8, bd=8, seed=1):
    """350x202 (neither a multiple of 8: ceil grid 44x26, intra map 43x25 -> 24 propagating rows);
    5 frames; len 1..3; frame 3 references frame 2 twice (two steps sharing a destination); vectors of
    both signs with sub-pel parts; ~10% zero intra costs."""
    rng = np.random.default_rng(seed)
    W, H, PAD = 350, 202, 64
    imgs = _frames(5, W, H, dtype, bd, rng)
    w_imp, h_imp = (W + 7) // 8, (H + 7) // 8
    steps = [(4, 3, 3, 0), (4, 2, 3, 1), (4, 1, 3, 2), (3, 2, 2, 3), (3, 2, 2, 4), (2, 1, 1, 5), (1, 0, 1, 6)]
    reach = (PAD - 16) * 8
    mvs = rng.integers(-reach, reach + 1, (7, w_imp * h_imp, 2)).astype(np.int16)
    mvs[::2] = (np.array([-3, 5]) * 8 + rng.integers(-20, 21, (4, w_imp * h_imp, 2))).astype(np.int16)
    return Window(imgs, PAD, _intra(5, (W // 8) * (H // 8), rng, bd), mvs, steps, bd)


def focus_window(dtype=np.uint8, bd=8, seed=2, target=(5 * 64 + 13, 3 * 64 + 40)):
    """every source block of frame 1 aimed at ONE position (one bucket holds the whole frame); the
    second step aims everything at (-30, -20): top-left destination on the ring, only BR inside"""
    rng = np.random.default_rng(seed)
    W, H, PAD = 96, 72, 64
    imgs = _frames(3, W, H, dtype, bd, rng)
    w_imp, h_imp = W // 8, H // 8
    ys, xs = np.divmod(np.arange(w_imp * h_imp), w_imp)
    mvs = np.zeros((2, w_imp * h_imp, 2), np.int16)
    mvs[0, :, 0], mvs[0, :, 1] = target[1] - 64 * ys, target[0] - 64 * xs
    mvs[1, :, 0], mvs[1, :, 1] = -20 - 64 * ys, -30 - 64 * xs
    steps = [(2, 1, 1, 1), (1, 0, 1, 0)]
    return Window(imgs, PAD, _intra(3, w_imp * h_imp, rng, bd, 0.0) + 4000, mvs, steps, bd)


def window_1080p(seed=7, nframes=21, W=1920, H=1080, PAD=96):
    """speed 6's RDO window at 1080p 8 bit: nframes frames, frame k references k-1, k-2, k-3 where they
    exist (57 steps for 21 frames), walked from the last frame back; smooth seeded motion plus
    per-block noise within +-48 px."""
    rng = np.random.default_rng(seed)
    imgs = _frames(nframes, W, H, np.uint8, 8, rng, drift=(2, -1))
    w_imp, h_imp = (W + 7) // 8, (H + 7) // 8
    ys, xs = np.divmod(np.arange(w_imp * h_imp), w_imp)
    steps, maps = [], []
    for k in range(nframes - 1, 0, -1):
        refs = [r for r in (k - 1, k - 2, k - 3) if r >= 0]
        for r in refs:
            d = k - r
            smooth = np.stack([8 * d * (-1 + 2 * np.sin(xs / 37.0 + k)), 8 * d * (2 + 3 * np.cos(ys / 23.0 + r))], 1)
            mv = np.clip(np.rint(smooth + rng.integers(-64, 65, (w_imp * h_imp, 2))), -48 * 8, 48 * 8)
            steps.append((k, r, len(refs), len(maps)))
            maps.append(mv.astype(np.int16))
    intra = np.zeros((nframes, (W // 8) * (H // 8)), np.uint32)
    return Window(imgs, PAD, intra, np.stack(maps), steps, 8)


def oracle_intra_costs(win):
    l = O.lib()
    l.orc_estimate_intra_costs.restype = None
    l.orc_estimate_intra_costs.argtypes = [C.c_void_p, C.c_ssize_t] + [C.c_int] * 4 + [C.c_void_p]
    for f, p in enumerate(win.planes):
        l.orc_estimate_intra_costs(p.at(0, 0), p.stride, win.W, win.H, p.bpp, win.bd, win.intra[f].ctypes.data)


def oracle_importances(win):
    imp = np.zeros((len(win.imgs), win.n_imp), np.float32)
    frames = (C.c_void_p * len(win.planes))(*[p.at(0, 0) for p in win.planes])
    steps = np.ascontiguousarray(np.array(win.steps, np.uint32).reshape(-1, 4))
    mvs = np.ascontiguousarray(win.mvs)
    intra = np.ascontiguousarray(win.intra)
    T().orc_block_importances(len(win.planes), C.addressof(frames), win.planes[0].stride, win.planes[0].bpp, win.W,
                              win.H, intra.ctypes.data, mvs.ctypes.data, len(win.steps), steps.ctypes.data,
                              imp.ctypes.data)
    return imp


# ---------------------------------------------------------------- independent model
def model_importances(win):
    """internal.rs:912-1206 in float32 scalars, in the reference's loop order"""
    imp = np.zeros((len(win.imgs), win.n_imp), np.float32)
    f32 = np.float32
    rows = min(win.h_imp, win.n_intra // win.w_imp)
    for src, dst, ln, mi in win.steps:
        org, ref, pad = win.planes[src].data, win.planes[dst].data, win.pad
        for y in range(rows):
            for x in range(win.w_imp):
                i = y * win.w_imp + x
                rx, ry = 64 * x + int(win.mvs[mi, i, 1]), 64 * y + int(win.mvs[mi, i, 0])
                sx, sy = math.trunc(rx / 8), math.trunc(ry / 8)
                inter = f32(satd8(org[pad + 8 * y:pad + 8 * y + 8, pad + 8 * x:pad + 8 * x + 8],
                                  ref[pad + sy:pad + sy + 8, pad + sx:pad + sx + 8]))
                intra = f32(int(win.intra[src, i]))
                frac = f32(0) if intra <= inter else f32(1) - inter / intra
                amount = (intra + imp[src, i]) * frac / f32(ln)
                bx, by = rx // 64, ry // 64                         # floor
                fx, fy = rx - 64 * bx, ry - 64 * by
                for dx, dy, wgt in ((0, 0, (64 - fx) * (64 - fy)), (1, 0, fx * (64 - fy)), (0, 1, (64 - fx) * fy),
                                    (1, 1, fx * fy)):
                    tx, ty = bx + dx, by + dy
                    if 0 <= tx < win.w_imp and 0 <= ty < win.h_imp:
                        imp[dst, ty * win.w_imp + tx] = imp[dst, ty * win.w_imp + tx] + amount * (f32(wgt) / f32(4096))
    return imp


def py_blog32_q11(w):
    if w == 0:
        return -1
    ipart = w.bit_length()
    n = (w >> (ipart - 16) if ipart > 16 else w << (16 - ipart)) - 49152
    p = -1402
    for c in (2546, -5216, 15745, -6797):
        p = ((n * p) >> 15) + c
    return (ipart << 11) + (p >> 3)


def py_bexp32_q10(z):
    """logexp.rs:254-267, restated (u32 arithmetic never wraps for these inputs)"""
    ipart = z >> 10
    n = (z & 1023) << 4
    p = 3548
    for c in (6817, 15823, 22708):
        p = ((n * p) >> 15) + c
    n = ((n * p) >> 15) + 16384
    return (n + (1 << (13 - ipart))) >> (14 - ipart) if 14 - ipart > 0 else n << (ipart - 14)


def py_mul(a, b):
    return min(max((a * b + 8192) >> 14, 1), (1 << 28) - 1)


def py_inv_mean(s):
    l = T()
    tot = sum(py_blog32_q11(int(v)) for v in s)
    q = abs(tot) // len(s) * (1 if tot >= 0 else -1)                   # i64 division truncates
    log_inv = (14 << 11) - q
    arg = I64(((log_inv + (14 << 11)) << 46) & ((1 << 64) - 1)).value
    return min(max(l.orc_bexp64(arg), 1), (1 << 28) - 1)


def py_scores(d, a=None):
    """encoder.rs:744-777 -> (distortion scales, spatiotemporal scores, log_isqrt_mean_scale)"""
    d = [int(v) for v in d]
    if a is None:
        inv = py_inv_mean(d)
        d = [py_mul(v, inv) for v in d]
        st = list(d)
    else:
        st = [py_mul(x, int(y)) for x, y in zip(d, a)]
        inv = py_inv_mean(st)
        st = [py_mul(v, inv) for v in st]
        d = [py_mul(v, inv) for v in d]
    return np.array(d, np.uint32), np.array(st, np.uint32), (T().orc_blog64(inv) - (14 << 57)) >> 1


def py_distortion_scale_for(imp, intra):
    if intra == 0.0:
        return 1 << 14
    s = math.pow((intra + imp) / intra, 1.0 / 3.0)
    num = int(s * 32768.0)
    raw = min((num << 14) + 16384, (1 << 64) - 1) // 32768
    return raw if raw <= (1 << 28) - 1 else (1 << 28) - 1


def oracle_scales(win, imp0, intra0):
    sc = np.zeros(win.n_imp, np.uint32)
    imp0, intra0 = np.ascontiguousarray(imp0, np.float32), np.ascontiguousarray(intra0, np.uint32)
    T().orc_distortion_scales(imp0.ctypes.data, win.n_imp, intra0.ctypes.data, win.n_intra, sc.ctypes.data)
    return sc


def oracle_scores(scales, activity=None):
    d = np.array(scales, np.uint32)
    st = np.zeros_like(d)
    a = None if activity is None else np.ascontiguousarray(activity, np.uint32)
    r = T().orc_temporal_scores(d.ctypes.data, len(d), None if a is None else a.ctypes.data, st.ctypes.data, None)
    return d, st, r


# ---------------------------------------------------------------- tests
def test_logexp_reference_kats():
    l = T()
    k = KATS
    for n, want in k["blog64"]:
        assert l.orc_blog64(n) == want
    for x, want, tol in k["bexp64"]:
        got = l.orc_bexp64(x)
        assert got == want if tol == 0 else abs(got - want) < tol
    assert l.orc_blog64(0) == -1 and l.orc_blog32_q11(0) == -1 and l.orc_bexp64(-1) == 0
    assert l.orc_bexp64(63 << 57) == (1 << 63) - 1


def test_blog64_bexp64_round_trip():
    """logexp.rs:304-314, every a in 1..=u16::MAX"""
    l = T()
    imax = (1 << 63) - 1
    for a in range(1, 1 << 16):
        b = imax // a
        la, lb, lab = l.orc_blog64(a), l.orc_blog64(b), l.orc_blog64(a * b)
        assert abs(la + lb - lab) < 4
        assert l.orc_bexp64(la) == a
        assert abs(l.orc_bexp64(lb) - b) < 128
        assert abs(l.orc_bexp64(lab) - a * b) < 128


def test_blog32_q11_round_trip_and_python_restatement():
    """logexp.rs:345-358 with bexp32_q10 restated here; the oracle's blog32_q11 equals the Python one"""
    l = T()
    for a in range(1, 1 << 15):
        b = 32767 // a
        la, lb, lab = l.orc_blog32_q11(a), l.orc_blog32_q11(b), l.orc_blog32_q11(a * b)
        assert (la, lb, lab) == (py_blog32_q11(a), py_blog32_q11(b), py_blog32_q11(a * b))
        assert abs(la + lb - lab) < 4
        assert abs(py_bexp32_q10((la + 1) >> 1) - a) < 18
        assert abs(py_bexp32_q10((lb + 1) >> 1) - b) < 2
        assert abs(py_bexp32_q10((lab + 1) >> 1) - a * b) < 18
    rng = np.random.default_rng(3)
    for w in rng.integers(1, 1 << 32, 2000, dtype=np.uint64):
        assert l.orc_blog32_q11(int(w)) == py_blog32_q11(int(w))


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10)])
@pytest.mark.parametrize("make", [small_window, focus_window])
def test_propagation_equals_the_float32_model(make, dtype, bd):
    win = make(dtype, bd)
    got = oracle_importances(win)
    want = model_importances(win)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    assert (got[:-1] > 0).any()                                      # something propagated
    if make is small_window:
        # rows past floor(n_intra / w_imp) = 24 never propagate: frame 0 only receives, from frame 1's rows < 24
        assert win.n_intra // win.w_imp == 24 and win.h_imp == 26
        assert (got[4] == 0).all()                                    # the last frame is nobody's reference


def test_focus_window_concentrates_on_four_blocks():
    win = focus_window()
    imp = oracle_importances(win)
    nz = np.flatnonzero(imp[0])
    assert set(nz) <= {3 * win.w_imp + 5, 3 * win.w_imp + 6, 4 * win.w_imp + 5, 4 * win.w_imp + 6}
    assert np.flatnonzero(imp[1]).tolist() == [0]                   # ring corner: only BR lands inside


def test_distortion_scale_for_equals_math_pow():
    l = T()
    win = small_window()
    imp = oracle_importances(win)
    rng = np.random.default_rng(4)
    pairs = [(float(imp[0, i]), float(win.intra[0, i])) for i in range(win.n_intra)]
    pairs += [(float(a), float(b)) for a, b in zip(rng.random(3000) * 1e6, rng.integers(0, 1 << 22, 3000))]
    pairs += [(0.0, 0.0), (5.0, 0.0), (0.0, 7.0), (1e30, 1.0)]
    for imp_v, intra_v in pairs:
        assert l.orc_distortion_scale_for(imp_v, intra_v) == py_distortion_scale_for(imp_v, intra_v), (imp_v, intra_v)
    sc = oracle_scales(win, imp[0], win.intra[0])
    assert (sc[win.n_intra:] == 16384).all()                        # the zip stops at the intra map's length
    assert sc[0] == py_distortion_scale_for(float(imp[0, 0]), float(win.intra[0, 0]))


def test_scores_equal_the_python_restatement():
    win = small_window()
    imp = oracle_importances(win)
    d = oracle_scales(win, imp[0], win.intra[0])
    rng = np.random.default_rng(5)
    act = rng.integers(1 << 12, 1 << 16, win.n_imp).astype(np.uint32)
    for a in (None, act):
        gd, gs, gr = oracle_scores(d, a)
        wd, ws, wr = py_scores(d, a)
        np.testing.assert_array_equal(gd, wd)
        np.testing.assert_array_equal(gs, ws)
        assert gr == wr
