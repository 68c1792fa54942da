"""CPU tests of the oracle's RDO distortion kernels (oracle/rdo_dist.c) — get_weighted_sse,
cdef_dist_kernel, apply_ssim_boost — against the float cross-checks the reference's own tests use
(activity.rs:204-252) and against plain numpy restatements."""
import ctypes as C
import math

import numpy as np

from tests import oracle_lib as O


def L():
    l = O.lib()
    l.orc_apply_ssim_boost.restype = C.c_uint32
    l.orc_apply_ssim_boost.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_int]
    for n, t in (("orc_weighted_sse_u8", None), ("orc_weighted_sse_u16", None)):
        f = getattr(l, n)
        f.restype = C.c_uint64
        f.argtypes = [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_size_t, C.c_int, C.c_int]
    for n in ("orc_cdef_dist_kernel_u8", "orc_cdef_dist_kernel_u16"):
        f = getattr(l, n)
        f.restype = C.c_uint32
        f.argtypes = [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_void_p]
    l.orc_distortion_scale_mul.restype = C.c_uint64
    l.orc_distortion_scale_mul.argtypes = [C.c_uint32, C.c_uint64]
    return l


def reference_ssim_boost(svar, dvar, bd):      # activity.rs:204-217 (floating point reference)
    vs = 1.0 / (1 << (2 * (bd - 8)))
    s, d = svar * vs, dvar * vs
    c1, c2, c3 = 3355.0, 16128.0, 12338.0
    return (c1 / c3) * (s + d + c2) / math.sqrt(c1 * c1 + s * d)


def test_ssim_boost_accuracy_like_the_reference_test():
    """activity.rs:220-252: max relative error against the float formula < 5 %."""
    l = L()
    rng = np.random.default_rng(0)
    worst = 0.0
    for scale in range(0, 12 + 3 * 2 - 2):
        for _ in range(40):
            sv, dv = int(rng.integers(0, 1 << scale)), int(rng.integers(0, 1 << scale))
            fixed = l.orc_apply_ssim_boost(1 << 23, sv, dv, 12) / float(1 << 23)
            worst = max(worst, abs(1.0 - fixed / reference_ssim_boost(sv, dv, 12)))
    assert worst < 0.05, worst


def test_ssim_boost_overflow_case():
    """activity.rs:195-201: the extreme 12-bit input must not wrap to nonsense."""
    l = L()
    d = (1 << 12) - 1
    v = l.orc_apply_ssim_boost(d * d * 64, d * 64 // 4, d * 64 // 4, 12)
    assert 0 < v < 2**32


def test_ssim_boost_reciprocal_cube_root_shape():
    """activity.rs:254-283: with equal variances the boost follows (x/2)^(-1/3)."""
    l = L()
    for bd in (8, 10, 12):
        scale = ((1 << bd) - 1) << (6 - 2 + bd - 8)
        worst = 0.0
        for svar in np.linspace(scale, (scale << 2) - 1, 200).astype(np.int64):
            want = ((scale << 1) / float(svar)) ** (1.0 / 3.0)
            got = l.orc_apply_ssim_boost(1 << 23, int(svar), int(svar), bd) / float(1 << 23)
            worst = max(worst, abs(1.0 - got / want))
        assert worst < 0.065, (bd, worst)     # the reference asserts < 0.065


def numpy_weighted_sse(a, b, scale):
    h, w = a.shape
    tot = 0
    for cy in range(0, h - 3, 4):
        for cx in range(0, w - 3, 4):
            d = a[cy:cy + 4, cx:cx + 4].astype(np.int64) - b[cy:cy + 4, cx:cx + 4].astype(np.int64)
            tot += (int((d * d).sum()) * int(scale[cy // 4, cx // 4]) + 128) >> 8
    return (tot + 32) // 64


def test_weighted_sse_matches_numpy_and_unit_scale_is_plain_sse():
    l = L()
    rng = np.random.default_rng(1)
    for dtype, maxv, fn in ((np.uint8, 255, l.orc_weighted_sse_u8), (np.uint16, 4095, l.orc_weighted_sse_u16)):
        for w, h in ((4, 4), (8, 8), (16, 16), (64, 32), (128, 128), (16, 4), (4, 16)):
            a = rng.integers(0, maxv + 1, (h, w + 5)).astype(dtype)
            b = rng.integers(0, maxv + 1, (h, w + 9)).astype(dtype)
            scale = rng.integers(1, 1 << 18, (h // 4, w // 4 + 2)).astype(np.uint32)
            got = fn(a.ctypes.data, a.shape[1], b.ctypes.data, b.shape[1], scale.ctypes.data, scale.shape[1], w, h)
            assert got == numpy_weighted_sse(a[:, :w], b[:, :w], scale)
            unit = np.full_like(scale, 1 << 14)
            got = fn(a.ctypes.data, a.shape[1], b.ctypes.data, b.shape[1], unit.ctypes.data, unit.shape[1], w, h)
            d = a[:, :w].astype(np.int64) - b[:, :w].astype(np.int64)
            # per-chunk rounding of sum*2^14 >> 8 is exact, the final /64 rounds to nearest
            assert got == (int((d * d).sum()) * 64 + 32) // 64


def test_cdef_dist_kernel_pieces():
    l = L()
    rng = np.random.default_rng(2)
    raw = (C.c_uint32 * 3)()
    for dtype, bd, fn in ((np.uint8, 8, l.orc_cdef_dist_kernel_u8), (np.uint16, 10, l.orc_cdef_dist_kernel_u16)):
        maxv = (1 << bd) - 1
        for w, h in ((8, 8), (4, 4), (8, 4), (4, 8), (6, 8), (8, 3)):
            s = rng.integers(0, maxv + 1, (8, 12)).astype(dtype)
            d = np.clip(s.astype(np.int64) + rng.integers(-9, 10, s.shape), 0, maxv).astype(dtype)
            v = fn(s.ctypes.data, 12, d.ctypes.data, 12, w, h, bd, raw)
            S, D = s[:h, :w].astype(np.int64), d[:h, :w].astype(np.int64)
            sse = int(((S - D) ** 2).sum())
            assert raw[2] == sse
            n = w * h
            # variance * area scaled to an 8x8 area: integer restatement with round(2^14 / n) as the
            # divisor (dist.rs:288-297), and - for power-of-two areas, where that divisor is exact -
            # the textbook float value
            div = int(round(16384.0 / n))
            for got, X in ((raw[0], S), (raw[1], D)):
                var = max(int((X * X).sum()) - ((int(X.sum()) ** 2 * div + 8192) >> 14), 0)
                assert got == (var * div + 128) >> 8, (w, h)
                if n & (n - 1) == 0:
                    exact = (float((X * X).sum()) - float(X.sum()) ** 2 / n) * 64.0 / n
                    assert abs(got - exact) <= 64.0 / n + 1, (w, h, got, exact)
            assert v == l.orc_apply_ssim_boost(sse, raw[0], raw[1], bd)
            # identical blocks: zero distortion whatever the variance
            assert fn(s.ctypes.data, 12, s.ctypes.data, 12, w, h, bd, None) == 0


M64 = (1 << 64) - 1
SSIM_RATIO = (((3355 << 15) // 12338) + 1) >> 1                 # activity.rs:179


def py_ssim_boost_rsqrt(x):
    """activity.rs:107-143 in Python integers: ilog2, i16 k / s, the `as u16` cast, i32 arithmetic shifts
    (Python's >> on negative ints is the arithmetic shift Rust's i32 >> is) -> (norm, shift)"""
    k = (x.bit_length() - 1) >> 1
    s = 2 * k - (16 - 2)
    t = (x >> s if s > 0 else x << -s) & 0xFFFF
    shift = (14 + ((s + 16) >> 1)) & 0xFF
    n = t - 32768
    rsqrt = 23557 + ((n * (-13490 + ((n * 6711) >> 15))) >> 15)
    return rsqrt & 0xFFFF, shift


def py_apply_ssim_boost(inp, svar, dvar, bd):
    """activity.rs:159-186 in Python integers, wrapping u64 products and the final `as u32` like a release
    build"""
    cs = bd - 8
    sv, dv = svar >> (2 * cs), dvar >> (2 * cs)
    c1, c2, c3 = 3355, 16128, 12338
    ratio = (((c1 << 15) // c3) + 1) >> 1
    assert ratio == SSIM_RATIO
    norm, shift = py_ssim_boost_rsqrt(c1 * c1 + sv * dv)
    inner = (((ratio * (sv + dv + c2)) & M64) * norm & M64) >> 14
    return (((inp * inner) & M64) >> shift) & 0xFFFFFFFF


def test_apply_ssim_boost_python_restatement_equals_the_oracle():
    """Both ends of every input: input, svar, dvar in {0, 1, ..., 2^32 - 1}, every bit depth, plus a random
    sweep; the inputs whose u64 product wraps are among them."""
    l = L()
    u32_edges = [0, 1, 2, 3, 255, 256, 4095, 16128, 65535, 1 << 16, (1 << 20) - 1, 1 << 24, 268304400,
                 (1 << 31) - 1, 1 << 31, (1 << 32) - 2, (1 << 32) - 1]
    inputs = [0, 1, 1 << 14, (1 << 14) + 1, 268304400, (1 << 32) - 1]
    wrapped = 0
    for bd in (8, 10, 12):
        for inp in inputs:
            for sv in u32_edges:
                for dv in u32_edges:
                    want = l.orc_apply_ssim_boost(inp, sv, dv, bd)
                    assert py_apply_ssim_boost(inp, sv, dv, bd) == want, (inp, sv, dv, bd)
                    cs = bd - 8
                    a, b = sv >> 2 * cs, dv >> 2 * cs
                    norm, _ = py_ssim_boost_rsqrt(3355 * 3355 + a * b)
                    wrapped += inp * (((SSIM_RATIO * (a + b + 16128)) * norm) >> 14) > M64
    assert wrapped > 0
    rng = np.random.default_rng(11)
    for _ in range(20000):
        bd = int(rng.choice([8, 10, 12]))
        inp, sv, dv = (int(v) for v in rng.integers(0, 1 << 32, 3, dtype=np.uint64) >> rng.integers(0, 32, 3).astype(np.uint64))
        assert py_apply_ssim_boost(inp, sv, dv, bd) == l.orc_apply_ssim_boost(inp, sv, dv, bd), (inp, sv, dv, bd)


def parse_area_divisors(path, name):
    """the 64 initialisers of the array `name` in a C / CUDA source"""
    import os
    import re
    src = open(os.path.join(O.ROOT, path)).read()
    body = re.search(name + r"\[64\]\s*=\s*\{(.*?)\};", re.sub(r"/\*.*?\*/", "", src, flags=re.S), re.S).group(1)
    return [int(v) for v in re.findall(r"\d+", body)]


def test_area_divisors_are_round_2_14_over_area_in_both_tables():
    """kAreaDivisors (rdo_dist_dev.cuh) and the oracle's AREA_DIVISORS (rdo_dist.c) against
    round(2^14 / (1 + x)) (dist.rs:288-297), exactly: a w x h <= 8x8 block reaches only 30 of the 64
    entries, so this pins the rest.  No entry is a tie, so the rounding direction does not matter."""
    from fractions import Fraction
    want = []
    for x in range(64):
        q = Fraction(1 << 14, 1 + x)
        assert q - int(q) != Fraction(1, 2)
        want.append(int(q + Fraction(1, 2)))
    assert parse_area_divisors("rav1e_b200/csrc/rdo_dist_dev.cuh", "kAreaDivisors") == want
    assert parse_area_divisors("oracle/rdo_dist.c", "AREA_DIVISORS") == want
    assert len({w * h for w in range(1, 9) for h in range(1, 9)}) == 30


def test_distortion_scale_mul_rounds_to_nearest():
    l = L()
    assert l.orc_distortion_scale_mul(1 << 14, 12345) == 12345
    assert l.orc_distortion_scale_mul(3 << 13, 3) == 5       # 4.5 -> 5 (round half up)
    assert l.orc_distortion_scale_mul(1, (1 << 13) - 1) == 0
    assert l.orc_distortion_scale_mul(1, 1 << 13) == 1
