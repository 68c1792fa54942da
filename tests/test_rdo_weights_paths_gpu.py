"""The RDO weighting chain on every kernel path, bit exact against the oracle and against independent exact models
(Python integers, numpy u64 with explicit wrapping, float32 scalars).

The kernels:
- rdo_dist.cu on rdo_dist_dev.cuh: `weighted_sse_kernel` (one warp per block, a lane per 4x4 chunk),
  `cdef_dist_kernel` (one thread per <= 8x8 block), `activity_mask_kernel` (one thread per 8x8 block), and the
  per-call b200_weighted_sse / b200_cdef_dist_kernel;
- lookahead.cu: `downsample_kernel`, `intra_cost_kernel`, `inter_cost_kernel`, `imp_diff_kernel`, `mean_kernel`;
- temporal_rdo.cu: `imp_pass_a`, the stable radix sort, `bucket_bounds`, `imp_pass_b`, `distortion_scales_kernel`,
  `scores_log_sum`, `scores_inv_mean`, `scores_apply`.
The sections:
1. weighted SSE: all 22 block sizes and sizes that are not multiples of 4, 1 / 31 / 32 / 33 / 1024 chunks, every
   4-pixel column phase, scales 1 .. 0xFFFFFFFF, u64 wrap, a ragged second grid-stride trip, the per-call form;
2. cdef_dist: every w x h in 1..8 x 1..8 on random / flat / 0-max checkerboard / 0-max step blocks at 8 / 10 / 12
   bit, the variance clamp, every output combination, the per-call form, a second grid-stride trip;
3. the activity mask: every frame size remainder mod 8 in both axes, flat and maximum-variance blocks, no scales,
   a second grid-stride trip;
4. the lookahead maps: the downsample at pad sizes 1 and full, intra costs with all four DC variants, inter costs on
   a vector table that proves truncation toward zero and at the far edge of the padding, the importance
   difference, both f64 means, a second grid-stride trip;
5. block importances on windows built to reach zero weights, off-grid sources, floor != truncation and long
   buckets, against the oracle and the float32 model;
6. distortion scales (the DS_MAX clamp, the u64 wrap of num << 14, the saturating add, inf) and both score forms
   (both ds_mul clamps, every optional output, a wide 4x4 map stride, a second trip of scores_log_sum);
7. every rejected argument of the ten _dev entry points launches nothing and writes nothing.
Each section asserts that it reached what it claims, computed from the models and the launch geometry below."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_activity import oracle_mask
from tests.test_lookahead_gpu import download_padded
from tests.test_oracle_lookahead import H8, L as LL, downsample as oracle_downsample
from tests.test_oracle_rdo_dist import L as OL, py_apply_ssim_boost
from tests.test_oracle_temporal_rdo import (T, Window, _frames, model_importances, oracle_importances, oracle_scores,
                                            py_blog32_q11, py_scores)

pytestmark = pytest.mark.gpu

BDS = [8, 10, 12]
M32, M64 = (1 << 32) - 1, (1 << 64) - 1
DS_MAX = (1 << 28) - 1                  # temporal_rdo.cu:35
CANARY = 0xA5

# Launch geometry mirrored from the sources: grid = min(ceil(work / per_cta), num_sms * ctas_per_sm), then a
# grid-stride loop.
WSSE_WARPS, WSSE_CTAS = 8, 32           # rdo_dist.cu:131-132  8 warps (blocks) per CTA
CDEF_DIST_THREADS, CDEF_DIST_CTAS = 128, 32   # rdo_dist.cu:158
ACT_THREADS, ACT_CTAS = 128, 32         # rdo_dist.cu:277
LA_THREADS, LA_CTAS = 128, 8            # lookahead.cu:179, :199, :220 (intra, inter, importance difference)
SCORES_THREADS, SCORES_CTAS = 256, 8    # temporal_rdo.cu:443  scores_log_sum

BLOCK_SIZES = B.BLOCK_SIZES             # the 22 sizes 4x4 .. 128x128
ODD_SIZES = [(5, 5), (6, 7), (7, 6), (5, 4), (4, 7), (14, 14), (126, 126), (127, 9), (9, 127), (126, 5),
             (124, 4), (124, 6), (44, 12), (47, 15), (13, 128), (128, 13)]


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pxdt(bd):
    return np.uint8 if bd == 8 else np.uint16


def canary(nbytes):
    return torch.full((max(nbytes, 1),), CANARY, dtype=torch.uint8, device="cuda")


def area_divisor(a):
    """round(2^14 / a), exactly (dist.rs:288-297; no entry is a tie)"""
    return int(Fraction(1 << 14, a) + Fraction(1, 2))


def assert_mean(got, total, count):
    """`total as f64 / count as f64` (total < 2^53: also the correctly rounded quotient of the integers)"""
    assert total < 1 << 53 and count < 1 << 53
    want = float(total) / float(count)
    assert want == total / count
    assert got == want, (got, want, total, count)


# ================================================================ 1. weighted SSE
def wsse_model(a, b, scale, blocks, w, h):
    """get_weighted_sse per block in numpy u64: u32 chunk sums, wrapping products and sums, (acc + 32) / 64.
    scale: a (rows, stride) map, chunk (cx, cy) of the plane at scale[cy, cx]."""
    H, W = a.shape
    d = a.astype(np.int64) - b.astype(np.int64)
    cs = (d * d)[:H // 4 * 4, :W // 4 * 4].reshape(H // 4, 4, W // 4, 4).sum((1, 3)) & M32
    terms = (cs.astype(np.uint64) * scale[:H // 4, :W // 4].astype(np.uint64) + np.uint64(128)) >> np.uint64(8)
    I = np.zeros((H // 4 + 1, W // 4 + 1), np.uint64)
    I[1:, 1:] = terms.cumsum(0, dtype=np.uint64).cumsum(1, dtype=np.uint64)
    x0, y0 = blocks["x"].astype(np.int64) // 4, blocks["y"].astype(np.int64) // 4
    x1, y1 = x0 + w // 4, y0 + h // 4
    acc = I[y1, x1] - I[y0, x1] - I[y1, x0] + I[y0, x0]
    return (acc + np.uint64(32)) // np.uint64(64)


def wsse_oracle(a, b, scale, blk, w, h):
    ol = OL()
    fn = ol.orc_weighted_sse_u8 if a.itemsize == 1 else ol.orc_weighted_sse_u16
    W, isz, x, y = a.shape[1], a.itemsize, int(blk["x"]), int(blk["y"])
    return fn(a.ctypes.data + (y * W + x) * isz, W, b.ctypes.data + (y * W + x) * isz, W,
              scale.ctypes.data + ((y // 4) * scale.shape[1] + x // 4) * 4, scale.shape[1], w, h)


def wsse_device(a, b, scale, blocks, w, h):
    c = G.ctx()
    pa, pb = c.plane_from_host(a, 0), c.plane_from_host(b, 0)
    n = len(blocks)
    d_out = canary(8 * n + 64)
    c.weighted_sse_dev(pa, pb, G.to_dev(blocks), n, w, h, G.to_dev(scale), scale.shape[1], d_out)
    c.synchronize()
    raw = d_out.cpu().numpy()
    assert (raw[8 * n:] == CANARY).all()                          # nothing past the last block
    for p in (pa, pb):
        c.plane_free(p)
    return raw[:8 * n].view(np.uint64)


def wsse_scales(rng, rows, cols):
    """a mix of the ends (1, 1 << 14, DS_MAX, 0xFFFFFFFF) and random Q14 scales"""
    pick = rng.integers(0, 6, (rows, cols))
    s = np.choose(pick, [np.full((rows, cols), 1), np.full((rows, cols), 1 << 14), np.full((rows, cols), DS_MAX),
                         np.full((rows, cols), M32), rng.integers(1, 1 << 20, (rows, cols)),
                         rng.integers(0, 1 << 32, (rows, cols), dtype=np.uint64)])
    return np.ascontiguousarray(s.astype(np.uint32))


@pytest.mark.parametrize("bd", BDS)
def test_weighted_sse_every_size_phase_and_scale(bd):
    rng = np.random.default_rng(100 + bd)
    W, H, maxv = 512, 384, (1 << bd) - 1
    a = rng.integers(0, maxv + 1, (H, W)).astype(pxdt(bd))
    b = np.clip(a.astype(np.int64) + rng.integers(-40, 41, a.shape), 0, maxv).astype(pxdt(bd))
    b[:, W // 2:] = rng.integers(0, maxv + 1, (H, W // 2))                # large errors on the right half
    a[:128, :128], b[:128, :128] = 0, maxv                                 # maximum error in one corner
    scale = wsse_scales(rng, H // 4, W // 4 + 3)
    chunks, phases, odd_w, odd_h = set(), set(), set(), set()
    for w, h in BLOCK_SIZES + ODD_SIZES:
        n = 40
        blocks = np.zeros(n, B.BLOCK_DTYPE)
        blocks["x"] = 4 * rng.integers(0, (W - w) // 4 + 1, n)
        blocks["y"] = 4 * rng.integers(0, (H - h) // 4 + 1, n)
        blocks[0] = (0, 0)
        got = wsse_device(a, b, scale, blocks, w, h)
        want = wsse_model(a, b, scale, blocks, w, h)
        np.testing.assert_array_equal(got, want, err_msg=f"{w}x{h}")
        for i, blk in enumerate(blocks):
            assert wsse_oracle(a, b, scale, blk, w, h) == int(want[i]), (w, h, i)
        chunks.add((w // 4) * (h // 4))
        phases |= set((blocks["x"] // 4 % 32).tolist())
        odd_w |= {w % 4} - {0}
        odd_h |= {h % 4} - {0}
    assert {1, 31, 32, 33, 1024} <= chunks
    assert phases == set(range(32)) and odd_w == {1, 2, 3} and odd_h == {1, 2, 3}
    assert {1, 1 << 14, DS_MAX, M32} <= set(np.unique(scale[:H // 4, :W // 4]).tolist())


def test_weighted_sse_at_the_u64_limit():
    """The largest 12-bit block, 128x128 of 0 against 4095, at DS_MAX and at 0xFFFFFFFF: each chunk term is rounded
    >> 8 before the sum, so even this stays below 2^64 (at most ~2^62).  The u64 sum does wrap with 14-bit values
    in a u16 plane (the kernel takes no bit depth): 16383 against 0 at 0xFFFFFFFF, a big-integer sum above 2^64
    that the kernel, the oracle and the model must all reduce mod 2^64."""
    for hi, s, wraps in ((4095, DS_MAX, False), (4095, M32, False), (16383, DS_MAX, False), (16383, M32, True)):
        a = np.zeros((128, 128), np.uint16)
        b = np.full((128, 128), hi, np.uint16)
        scale = np.full((32, 32), s, np.uint32)
        chunk = 16 * hi * hi
        assert chunk <= M32
        big = 1024 * ((chunk * s + 128) >> 8)
        assert (big > M64) == wraps
        want = (((big & M64) + 32) & M64) // 64
        blocks = np.zeros(1, B.BLOCK_DTYPE)
        assert int(wsse_device(a, b, scale, blocks, 128, 128)[0]) == want
        assert int(wsse_model(a, b, scale, blocks, 128, 128)[0]) == want
        assert wsse_oracle(a, b, scale, blocks[0], 128, 128) == want


def test_weighted_sse_second_grid_stride_trip():
    cap = num_sms() * WSSE_CTAS * WSSE_WARPS
    n = cap + cap // 3 + 7
    assert cap < n < 2 * cap
    rng = np.random.default_rng(7)
    W, H = 1024, 512
    a = rng.integers(0, 256, (H, W)).astype(np.uint8)
    b = rng.integers(0, 256, (H, W)).astype(np.uint8)
    scale = wsse_scales(rng, H // 4, W // 4)
    blocks = np.zeros(n, B.BLOCK_DTYPE)
    blocks["x"] = 4 * rng.integers(0, (W - 8) // 4 + 1, n)
    blocks["y"] = 4 * rng.integers(0, (H - 8) // 4 + 1, n)
    got = wsse_device(a, b, scale, blocks, 8, 8)
    want = wsse_model(a, b, scale, blocks, 8, 8)
    np.testing.assert_array_equal(got, want)
    for i in np.concatenate([rng.integers(0, cap, 300), rng.integers(cap, n, 700)]):
        assert wsse_oracle(a, b, scale, blocks[i], 8, 8) == int(want[i])


def test_weighted_sse_percall_byte_strides():
    """b200_weighted_sse with pixel strides of an odd number of bytes (u8) and of 2 mod 4 bytes (u16)"""
    lib, rng = B.lib(), np.random.default_rng(9)
    for bd in BDS:
        maxv = (1 << bd) - 1
        sa, sb = (131, 137) if bd == 8 else (133, 141)
        a = rng.integers(0, maxv + 1, (128, sa)).astype(pxdt(bd))
        b = rng.integers(0, maxv + 1, (128, sb)).astype(pxdt(bd))
        scale = wsse_scales(rng, 32, 37)
        for w, h in ((4, 4), (7, 9), (16, 16), (126, 5), (44, 12), (128, 128)):
            isz = a.itemsize
            assert (sa * isz) % 4 != 0 and (sb * isz) % 4 != 0
            got = lib.b200_weighted_sse(a.ctypes.data, sa * isz, b.ctypes.data, sb * isz, scale.ctypes.data, 37 * 4,
                                        w, h, isz)
            blk = np.zeros(1, B.BLOCK_DTYPE)
            want = int(wsse_model(np.ascontiguousarray(a[:, :124]), np.ascontiguousarray(b[:, :124]), scale, blk, w,
                                  h)[0]) if w <= 124 else None
            ol = OL()
            fn = ol.orc_weighted_sse_u8 if isz == 1 else ol.orc_weighted_sse_u16
            orc = fn(a.ctypes.data, sa, b.ctypes.data, sb, scale.ctypes.data, 37, w, h)
            assert got == orc and (want is None or want == orc), (bd, w, h)


# ================================================================ 2. cdef_dist
def cdef_dist_model(S, D, bd):
    """cdef_dist_kernel on (n, h, w) blocks: u32 sums, the exact round(2^14 / area) divisor, saturating_sub, the
    8x8 rescale, then the Python apply_ssim_boost -> (out, raw (n, 3), clamp hit per block)"""
    n, h, w = S.shape
    S, D = S.astype(np.int64), D.astype(np.int64)
    ss, sd = S.sum((1, 2)) & M32, D.sum((1, 2)) & M32
    s2, d2, sxd = (S * S).sum((1, 2)) & M32, (D * D).sum((1, 2)) & M32, (S * D).sum((1, 2)) & M32
    sse = (d2 + s2 - 2 * sxd) & M32
    div = area_divisor(w * h)
    ms, md = ((ss * ss * div + 8192) >> 14) & M32, ((sd * sd * div + 8192) >> 14) & M32
    sv, dv = np.where(s2 > ms, s2 - ms, 0), np.where(d2 > md, d2 - md, 0)
    sv, dv = ((sv * div + 128) >> 8) & M32, ((dv * div + 128) >> 8) & M32
    raw = np.stack([sv, dv, sse], 1).astype(np.uint32)
    out = np.array([py_apply_ssim_boost(int(e), int(x), int(y), bd) for x, y, e in raw.tolist()], np.uint32)
    return out, raw, (s2 < ms) | (d2 < md)


def tile_kinds(rng, kinds, maxv):
    """8x8 tiles: 0 random, 1 flat, 2 0/max checkerboard, 3 0/max step edge"""
    out = np.empty((len(kinds), 8, 8), np.int64)
    I, J = np.mgrid[0:8, 0:8]
    for t, k in enumerate(kinds):
        if k == 0:
            out[t] = rng.integers(0, maxv + 1, (8, 8))
        elif k == 1:
            out[t] = rng.integers(0, maxv + 1)
        elif k == 2:
            out[t] = maxv * ((I + J + t) % 2)
        else:
            out[t] = maxv * ((I if t % 2 else J) >= rng.integers(1, 8))
    return out


def tiles_plane(tiles, cols):
    rows = len(tiles) // cols
    return np.ascontiguousarray(tiles.reshape(rows, cols, 8, 8).transpose(0, 2, 1, 3).reshape(rows * 8, cols * 8))


def gather(img, xs, ys, w, h):
    yy = ys[:, None, None] + np.arange(h)[None, :, None]
    xx = xs[:, None, None] + np.arange(w)[None, None, :]
    return img[yy, xx]


@pytest.mark.parametrize("bd", BDS)
def test_cdef_dist_every_shape_and_output(bd):
    c, rng, maxv = G.ctx(), np.random.default_rng(200 + bd), (1 << bd) - 1
    cols, ntile = 16, 128
    sk, dk = rng.integers(0, 4, ntile), rng.integers(0, 4, ntile)
    sk[:16], dk[:16] = np.repeat(np.arange(4), 4), np.tile(np.arange(4), 4)      # every (src, dst) kind pair
    src = tiles_plane(tile_kinds(rng, sk, maxv), cols).astype(pxdt(bd))
    dst = tiles_plane(tile_kinds(rng, dk, maxv), cols).astype(pxdt(bd))
    dst[:, 8 * 8:] = np.where(rng.random(dst[:, 64:].shape) < 0.5, src[:, 64:], dst[:, 64:])   # mixed pairs
    ps, pd = c.plane_from_host(src, 0), c.plane_from_host(dst, 0)
    ol = OL()
    fn = ol.orc_cdef_dist_kernel_u8 if bd == 8 else ol.orc_cdef_dist_kernel_u16
    r3, clamped, modes = (C.c_uint32 * 3)(), set(), set()
    for w in range(1, 9):
        for h in range(1, 9):
            t = np.arange(ntile)
            xs = 8 * (t % cols) + rng.integers(0, 9 - w, ntile)
            ys = 8 * (t // cols) + rng.integers(0, 9 - h, ntile)
            blocks = np.zeros(ntile, B.BLOCK_DTYPE)
            blocks["x"], blocks["y"] = xs, ys
            mode = (w * 8 + h) % 3                                   # 0 both, 1 d_out only, 2 d_raw only
            modes.add(mode)
            d_out, d_raw = canary(4 * ntile + 16), canary(12 * ntile + 16)
            c.cdef_dist_dev(ps, pd, G.to_dev(blocks), ntile, w, h, bd, d_out if mode != 2 else None,
                            d_raw if mode != 1 else None)
            c.synchronize()
            out, raw, hit = cdef_dist_model(gather(src, xs, ys, w, h), gather(dst, xs, ys, w, h), bd)
            go, gr = d_out.cpu().numpy(), d_raw.cpu().numpy()
            if mode != 2:
                np.testing.assert_array_equal(go[:4 * ntile].view(np.uint32), out, err_msg=f"{w}x{h}")
            if mode != 1:
                np.testing.assert_array_equal(gr[:12 * ntile].view(np.uint32).reshape(-1, 3), raw,
                                              err_msg=f"{w}x{h}")
            assert (go[4 * ntile if mode != 2 else 0:] == CANARY).all()
            assert (gr[12 * ntile if mode != 1 else 0:] == CANARY).all()
            isz = src.itemsize
            for i in range(0, ntile, 3):
                x, y = int(xs[i]), int(ys[i])
                v = fn(src.ctypes.data + (y * src.shape[1] + x) * isz, src.shape[1],
                       dst.ctypes.data + (y * dst.shape[1] + x) * isz, dst.shape[1], w, h, bd, r3)
                assert (v, tuple(r3)) == (int(out[i]), tuple(int(e) for e in raw[i])), (w, h, i)
            if hit.any():
                clamped.add(w * h)
    for p in (ps, pd):
        c.plane_free(p)
    assert modes == {0, 1, 2}
    assert len({a for a in clamped if a & (a - 1)}) >= 3, clamped          # saturating_sub at non-power-of-two areas


def test_cdef_dist_percall_forms():
    """b200_cdef_dist_kernel at every shape, with odd byte strides, with and without `ret`"""
    lib, ol, rng = B.lib(), OL(), np.random.default_rng(21)
    g3, r3 = (C.c_uint32 * 3)(), (C.c_uint32 * 3)()
    for bd in BDS:
        maxv = (1 << bd) - 1
        s = rng.integers(0, maxv + 1, (8, 13)).astype(pxdt(bd))
        d = np.clip(s.astype(np.int64) + rng.integers(-30, 31, s.shape), 0, maxv).astype(pxdt(bd))
        s[:4, :4], d[4:, :] = maxv, 0
        fn = ol.orc_cdef_dist_kernel_u8 if bd == 8 else ol.orc_cdef_dist_kernel_u16
        isz = s.itemsize
        for w in range(1, 9):
            for h in range(1, 9):
                want = fn(s.ctypes.data, 13, d.ctypes.data, 13, w, h, bd, r3)
                assert lib.b200_cdef_dist_kernel(s.ctypes.data, 13 * isz, d.ctypes.data, 13 * isz, w, h, bd, g3) == want
                assert tuple(g3) == tuple(r3)
                assert lib.b200_cdef_dist_kernel(s.ctypes.data, 13 * isz, d.ctypes.data, 13 * isz, w, h, bd,
                                                 None) == want


def test_cdef_dist_second_grid_stride_trip():
    c = G.ctx()
    cap = num_sms() * CDEF_DIST_CTAS * CDEF_DIST_THREADS
    n = cap + 12345
    rng = np.random.default_rng(31)
    src = rng.integers(0, 4096, (256, 512)).astype(np.uint16)
    dst = np.clip(src.astype(np.int64) + rng.integers(-50, 51, src.shape), 0, 4095).astype(np.uint16)
    xs, ys = rng.integers(0, 512 - 4, n), rng.integers(0, 256 - 4, n)
    blocks = np.zeros(n, B.BLOCK_DTYPE)
    blocks["x"], blocks["y"] = xs, ys
    ps, pd = c.plane_from_host(src, 0), c.plane_from_host(dst, 0)
    d_out, d_raw = canary(4 * n), canary(12 * n)
    c.cdef_dist_dev(ps, pd, G.to_dev(blocks), n, 4, 4, 12, d_out, d_raw)
    c.synchronize()
    go, gr = G.from_dev(d_out, np.uint32), G.from_dev(d_raw, np.uint32).reshape(-1, 3)
    for lo in range(0, n, 200000):
        sl = slice(lo, min(lo + 200000, n))
        S, D = gather(src, xs[sl], ys[sl], 4, 4).astype(np.int64), gather(dst, xs[sl], ys[sl], 4, 4).astype(np.int64)
        ss, s2 = S.sum((1, 2)), (S * S).sum((1, 2))
        sd, d2, sxd = D.sum((1, 2)), (D * D).sum((1, 2)), (S * D).sum((1, 2))
        div = area_divisor(16)
        sv = np.maximum(s2 - ((ss * ss * div + 8192) >> 14), 0)
        dv = np.maximum(d2 - ((sd * sd * div + 8192) >> 14), 0)
        np.testing.assert_array_equal(gr[sl], np.stack([(sv * div + 128) >> 8, (dv * div + 128) >> 8,
                                                        (d2 + s2 - 2 * sxd) & M32], 1))
    ol, r3 = OL(), (C.c_uint32 * 3)()
    for i in np.concatenate([rng.integers(0, cap, 500), rng.integers(cap, n, 1500)]):
        x, y = int(xs[i]), int(ys[i])
        want = ol.orc_cdef_dist_kernel_u16(src.ctypes.data + (y * 512 + x) * 2, 512, dst.ctypes.data + (y * 512 + x) * 2,
                                           512, 4, 4, 12, r3)
        assert int(go[i]) == want == py_apply_ssim_boost(r3[2], r3[0], r3[1], 12)
    for p in (ps, pd):
        c.plane_free(p)


# ================================================================ 3. activity mask
def activity_model(img, bd):
    """variance_8x8 of the edge-replicated plane rounded up to 8 (u16 column sums cannot wrap at <= 12 bit), and
    ssim_boost(var, var) in Python integers"""
    h, w = img.shape
    hb, wb = (h + 7) // 8, (w + 7) // 8
    p = np.pad(img, ((0, 8 * hb - h), (0, 8 * wb - w)), mode="edge").astype(np.int64)
    t = p.reshape(hb, 8, wb, 8)
    s, s2 = t.sum((1, 3)), (t * t).sum((1, 3))
    var = s2 - ((s * s + 32) >> 6)
    sc = np.array([py_apply_ssim_boost(1 << 14, v, v, bd) for v in var.reshape(-1).tolist()], np.uint32)
    return var.astype(np.uint32), sc.reshape(var.shape)


@pytest.mark.parametrize("bd", BDS)
def test_activity_mask_every_remainder(bd):
    c, rng, maxv = G.ctx(), np.random.default_rng(300 + bd), (1 << bd) - 1
    seen_w, seen_h, flat, peak = set(), set(), 0, 0
    I, J = np.mgrid[0:8, 0:8]
    for r in range(8):
        W, H = 64 + r + 8 * (r % 3), 40 + (r + 3) % 8 + 8 * (r % 2)
        img = rng.integers(0, maxv + 1, (H, W)).astype(pxdt(bd))
        img[:8, :8] = rng.integers(0, maxv + 1)                          # flat
        img[8:16, 8:16] = maxv * ((I + J) % 2)                           # 0/max checkerboard: the largest variance
        img[-3:, -5:] = maxv                                             # a partial block read through the padding
        var, sc = activity_model(img, bd)
        ovar, osc, _ = oracle_mask(img, 8, bd)
        np.testing.assert_array_equal(ovar, var)
        np.testing.assert_array_equal(osc, sc)
        n = var.size
        pl = c.plane_from_host(img, 8)
        d_var, d_sc = canary(4 * n + 16), canary(4 * n + 16)
        no_scales = r == 5
        c.activity_mask_dev(pl, bd, d_var, None if no_scales else d_sc)
        c.synchronize()
        gv, gs = d_var.cpu().numpy(), d_sc.cpu().numpy()
        np.testing.assert_array_equal(gv[:4 * n].view(np.uint32).reshape(var.shape), var)
        if not no_scales:
            np.testing.assert_array_equal(gs[:4 * n].view(np.uint32).reshape(sc.shape), sc)
        assert (gv[4 * n:] == CANARY).all() and (gs[0 if no_scales else 4 * n:] == CANARY).all()
        c.plane_free(pl)
        seen_w.add(W % 8)
        seen_h.add(H % 8)
        flat += int((var == 0).sum())
        peak += int((var == 16 * maxv * maxv).sum())
    assert seen_w == seen_h == set(range(8))
    assert flat > 0 and peak > 0


def test_activity_mask_second_grid_stride_trip():
    c = G.ctx()
    W, H = 8192, 4352
    n = (W // 8) * (H // 8)
    cap = num_sms() * ACT_CTAS * ACT_THREADS
    assert cap < n < 2 * cap
    rng = np.random.default_rng(41)
    img = rng.integers(0, 256, (H, W), dtype=np.uint8)
    img[:, :64] = 17
    var, sc, _ = oracle_mask(img, 8, 8)
    pl = c.plane_from_host(img, 0)
    d_var, d_sc = canary(4 * n), canary(4 * n)
    c.activity_mask_dev(pl, 8, d_var, d_sc)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_var, np.uint32).reshape(var.shape), var)
    np.testing.assert_array_equal(G.from_dev(d_sc, np.uint32).reshape(sc.shape), sc)
    mv, ms = activity_model(img[-16:, -256:], 8)
    np.testing.assert_array_equal(var[-2:, -32:], mv)
    np.testing.assert_array_equal(sc[-2:, -32:], ms)
    c.plane_free(pl)


# ================================================================ 4. lookahead maps
def downsample_model(img, dst_pad, pad_w, pad_h):
    h, w = img.shape
    w2, h2 = (w + 1) // 2, (h + 1) // 2
    e = np.pad(img, ((0, 2 * h2 - h), (0, 2 * w2 - w)), mode="edge").astype(np.int64)
    box = (e[0::2, 0::2] + e[0::2, 1::2] + e[1::2, 0::2] + e[1::2, 1::2] + 2) >> 2
    ys = np.clip(np.arange(-dst_pad, h2 + dst_pad), 0, pad_h - 1)
    xs = np.clip(np.arange(-dst_pad, w2 + dst_pad), 0, pad_w - 1)
    return box[ys[:, None], xs[None, :]].astype(img.dtype)


@pytest.mark.parametrize("bd", BDS)
def test_downsample_pad_sizes(bd):
    c, rng = G.ctx(), np.random.default_rng(400 + bd)
    for w, h in ((1, 1), (2, 2), (3, 5), (64, 33), (127, 71)):
        img = rng.integers(0, 1 << bd, (h, w)).astype(pxdt(bd))
        img[0, 0] = (1 << bd) - 1
        src = c.plane_from_host(img, 2)
        w2, h2 = (w + 1) // 2, (h + 1) // 2
        for pad_w, pad_h in ((1, 1), (w2, h2), (1, h2), (w2, 1)):
            for dpad in (0, 5):
                dst = c.plane_alloc(w2, h2, dpad, img.itemsize)
                c.plane_downsample_dev(src, dst, pad_w, pad_h)
                c.synchronize()
                got = download_padded(c, dst, pxdt(bd))
                want = downsample_model(img, dpad, pad_w, pad_h)
                np.testing.assert_array_equal(got, want, err_msg=f"{w}x{h} pad {pad_w}x{pad_h} dst pad {dpad}")
                np.testing.assert_array_equal(oracle_downsample(img, dpad, pad_w, pad_h), want)
                c.plane_free(dst)
        c.plane_free(src)


def satd_blocks(D):
    """satd8 of (n, 8, 8) differences"""
    return ((np.abs(H8 @ D @ H8.T).sum((1, 2)) + 4) >> 3).astype(np.uint32)


def blocks8(img, wb, hb):
    return img[:8 * hb, :8 * wb].astype(np.int64).reshape(hb, 8, wb, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8)


def intra_model(img, bd):
    """estimate_intra_costs: DC of the PredictionVariant (both / left / top / none) then SATD -> (costs, variant)"""
    H, W = img.shape
    hb, wb = H // 8, W // 8
    P = img.astype(np.int64)
    left, above = np.zeros((hb, wb), np.int64), np.zeros((hb, wb), np.int64)
    if wb > 1:
        left[:, 1:] = P[:8 * hb, 8 * np.arange(1, wb) - 1].reshape(hb, 8, wb - 1).sum(1)
    if hb > 1:
        above[1:, :] = P[8 * np.arange(1, hb) - 1, :8 * wb].reshape(hb - 1, wb, 8).sum(2)
    bx, by = np.meshgrid(np.arange(wb), np.arange(hb))
    variant = (bx > 0).astype(int) + 2 * (by > 0)
    dc = np.choose(variant, [np.full((hb, wb), 128 << (bd - 8)), (left + 4) >> 3, (above + 4) >> 3,
                             (left + above + 8) >> 4])
    return satd_blocks(blocks8(img, wb, hb) - dc.reshape(-1, 1, 1)), variant.reshape(-1)


def oracle_intra(img, bd):
    H, W = img.shape
    out = np.zeros((H // 8) * (W // 8), np.uint32)
    LL().orc_estimate_intra_costs(img.ctypes.data, W, W, H, img.itemsize, bd, out.ctypes.data)
    return out


def extreme_frame(rng, W, H, bd):
    maxv = (1 << bd) - 1
    img = np.where(rng.random((H, W)) < 0.5, 0, maxv)
    I, J = np.mgrid[0:H, 0:W]
    img[: H // 2] = np.where((I[: H // 2] + J[: H // 2]) % 2, maxv, 0)
    img[:, : W // 3] = rng.integers(0, maxv + 1, (H, W // 3))
    img[-8:, -8:] = maxv
    return np.ascontiguousarray(img.astype(pxdt(bd)))


@pytest.mark.parametrize("bd", BDS)
def test_intra_costs_odd_frames_and_variants(bd):
    c, rng = G.ctx(), np.random.default_rng(500 + bd)
    variants = set()
    for W, H in ((8, 8), (9, 9), (23, 17), (77, 45), (130, 66)):
        img = extreme_frame(rng, W, H, bd)
        want, var = intra_model(img, bd)
        np.testing.assert_array_equal(oracle_intra(img, bd), want)
        pl = c.plane_from_host(img, 8)
        n = want.size
        d = canary(4 * n + 16)
        c.estimate_intra_costs_dev(pl, bd, d)
        c.synchronize()
        g = d.cpu().numpy()
        np.testing.assert_array_equal(g[:4 * n].view(np.uint32), want, err_msg=f"{W}x{H}")
        assert (g[4 * n:] == CANARY).all()
        c.plane_free(pl)
        variants |= set(var.tolist())
    assert variants == {0, 1, 2, 3}


def inter_model(org, refp, pad, mvs):
    """estimate_inter_costs' SATD per block, refp = the edge-padded reference; mvs (hb, wb, 2) (row, col)"""
    hb, wb = mvs.shape[:2]
    by, bx = np.mgrid[0:hb, 0:wb]
    rx = np.trunc((64 * bx + mvs[..., 1].astype(np.int64)) / 8).astype(np.int64).reshape(-1)
    ry = np.trunc((64 * by + mvs[..., 0].astype(np.int64)) / 8).astype(np.int64).reshape(-1)
    R = gather(refp, rx + pad, ry + pad, 8, 8).astype(np.int64)
    return satd_blocks(blocks8(org, wb, hb) - R), rx, ry


def inter_device(org_pl, ref_pl, mvs, with_costs=True):
    c = G.ctx()
    n = mvs.shape[0] * mvs.shape[1]
    d_c, d_s, d_m = canary(4 * n + 16), G.dev_empty(8), G.dev_empty(8)
    c.estimate_inter_costs_dev(org_pl, ref_pl, G.to_dev(mvs), d_c if with_costs else None, d_s, d_m)
    c.synchronize()
    g = d_c.cpu().numpy()
    assert (g[4 * n if with_costs else 0:] == CANARY).all()
    return g[:4 * n].view(np.uint32), float(G.from_dev(d_m, np.float64)[0])


@pytest.mark.parametrize("bd", BDS)
def test_inter_costs_truncation_table_and_padding_edge(bd):
    c, rng, PAD = G.ctx(), np.random.default_rng(600 + bd), 32
    W, H = 61, 45
    wb, hb = W // 8, H // 8
    org = extreme_frame(rng, W, H, bd)
    ref = rng.integers(0, 1 << bd, (H, W)).astype(pxdt(bd))
    refp = np.pad(ref, PAD, mode="edge")
    po, pr = c.plane_from_host(org, PAD), c.plane_from_host(ref, PAD)
    l, isz = LL(), org.itemsize
    orp = np.pad(org, PAD, mode="edge")
    by, bx = np.mgrid[0:hb, 0:wb]
    trunc_ne_floor, seen = 0, set()
    for k in range(35):                                             # every col / row in -17..17 at every block
        mvs = np.stack([(k + 3 * by + 11 * bx) % 35 - 17, (k + 5 * bx + 7 * by) % 35 - 17], -1).astype(np.int16)
        want, rx, ry = inter_model(org, refp, PAD, mvs)
        got, mean = inter_device(po, pr, mvs)
        np.testing.assert_array_equal(got, want, err_msg=f"table row {k}")
        assert_mean(mean, int(want.astype(np.int64).sum()), wb * hb)
        oc = np.zeros(wb * hb, np.uint32)
        om = l.orc_estimate_inter_costs(org.ctypes.data, W, refp.ctypes.data + (PAD * refp.shape[1] + PAD) * isz,
                                        refp.shape[1], W, H, isz, mvs.ctypes.data, oc.ctypes.data)
        np.testing.assert_array_equal(oc, want)
        assert om == mean
        sx = 64 * bx.reshape(-1) + mvs[..., 1].reshape(-1)
        trunc_ne_floor += int((rx != sx // 8).sum())
        for p in (0, 1, wb - 1):
            seen |= {("col", p, int(v)) for v in mvs[:, p, 1]}
        for p in (0, 1, hb - 1):
            seen |= {("row", p, int(v)) for v in mvs[p, :, 0]}
    assert trunc_ne_floor > 0
    assert len(seen) == 6 * 35
    # the far edge of the padding: reference blocks whose top-left is (-PAD | W + PAD - 8, -PAD | H + PAD - 8)
    tx = np.where((bx + by) % 2 == 0, -PAD, W + PAD - 8)
    ty = np.where(bx % 2 == 0, -PAD, H + PAD - 8)
    col = np.where(tx < 0, 8 * tx - 7, 8 * tx + 7) - 64 * bx             # sub-pel parts truncated toward zero
    row = np.where(ty < 0, 8 * ty - 7, 8 * ty + 7) - 64 * by
    mvs = np.stack([row, col], -1).astype(np.int16)
    want, rx, ry = inter_model(org, refp, PAD, mvs)
    assert set(rx.tolist()) == {-PAD, W + PAD - 8} and set(ry.tolist()) == {-PAD, H + PAD - 8}
    for with_costs in (True, False):
        got, mean = inter_device(po, pr, mvs, with_costs)
        if with_costs:
            np.testing.assert_array_equal(got, want)
        assert_mean(mean, int(want.astype(np.int64).sum()), wb * hb)
    # the importance difference at the extremes
    d_s, d_m = G.dev_empty(8), G.dev_empty(8)
    for a, b in ((org, ref), (np.full_like(org, (1 << bd) - 1), np.zeros_like(org)), (org, org)):
        pa, pb = c.plane_from_host(a, PAD), c.plane_from_host(b, PAD)
        c.importance_block_difference_dev(pa, pb, d_s, d_m)
        c.synchronize()
        total = int(np.abs((blocks8(a, wb, hb).sum((1, 2)) + 32) // 64 - (blocks8(b, wb, hb).sum((1, 2)) + 32) // 64).sum())
        assert_mean(float(G.from_dev(d_m, np.float64)[0]), total, wb * hb)
        assert l.orc_importance_block_difference(a.ctypes.data, W, b.ctypes.data, W, W, H, isz) == total / (wb * hb)
        for p in (pa, pb):
            c.plane_free(p)
    for p in (po, pr):
        c.plane_free(p)


def test_lookahead_second_grid_stride_trip():
    c, PAD = G.ctx(), 16
    W, H = 4096, 2176
    wb, hb = W // 8, H // 8
    cap = num_sms() * LA_CTAS * LA_THREADS
    assert cap < wb * hb < 2 * cap
    rng = np.random.default_rng(61)
    org = rng.integers(0, 256, (H, W), dtype=np.uint8)
    ref = rng.integers(0, 256, (H, W), dtype=np.uint8)
    po, pr = c.plane_from_host(org, PAD), c.plane_from_host(ref, PAD)
    want, _ = intra_model(org, 8)
    np.testing.assert_array_equal(oracle_intra(org, 8), want)
    d = canary(4 * wb * hb)
    c.estimate_intra_costs_dev(po, 8, d)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d, np.uint32), want)
    mvs = rng.integers(-8 * (PAD - 8), 8 * (PAD - 8) + 1, (hb, wb, 2)).astype(np.int16)
    wi, _, _ = inter_model(org, np.pad(ref, PAD, mode="edge"), PAD, mvs)
    got, mean = inter_device(po, pr, mvs)
    np.testing.assert_array_equal(got, wi)
    assert_mean(mean, int(wi.astype(np.int64).sum()), wb * hb)
    d_s, d_m = G.dev_empty(8), G.dev_empty(8)
    c.importance_block_difference_dev(po, pr, d_s, d_m)
    c.synchronize()
    total = int(np.abs((blocks8(org, wb, hb).sum((1, 2)) + 32) // 64 - (blocks8(ref, wb, hb).sum((1, 2)) + 32) // 64).sum())
    assert_mean(float(G.from_dev(d_m, np.float64)[0]), total, wb * hb)
    for p in (po, pr):
        c.plane_free(p)


# ================================================================ 5. block importances
IMP_STEPS = [(4, 3, 3, 0), (4, 2, 3, 1), (4, 1, 3, 2), (3, 2, 2, 3), (3, 1, 2, 3), (2, 1, 1, 4), (1, 0, 1, 5)]
IMP_GEOMS = [(8 * (2 + r % 3) + r, 8 * (1 + r % 2) + 8 - r) for r in range(1, 8)] + [(8, 8), (5, 3), (8, 43), (43, 8)]


def imp_window(W, H, bd, seed, PAD=40):
    """5 frames of drifting smooth content; six vector maps (mv_index 3 is shared by two steps) whose blocks mix
    random sub-pel vectors, exact multiples of 64, sources aimed wholly off the ring grid and small negative
    positions; map 5 aims every source of frame 1 at one point (one long bucket)"""
    rng = np.random.default_rng(seed)
    imgs = _frames(5, W, H, pxdt(bd), bd, rng)
    w_imp, h_imp = (W + 7) // 8, (H + 7) // 8
    n_imp, n_intra = w_imp * h_imp, (W // 8) * (H // 8)
    ys, xs = np.divmod(np.arange(n_imp), w_imp)
    mvs = np.zeros((6, n_imp, 2), np.int64)
    for m in range(5):
        kind = rng.integers(0, 4, n_imp)
        r = rng.integers(-128, 129, (n_imp, 2))
        mult = 64 * rng.integers(-1, 2, (n_imp, 2))
        off_x = np.where(rng.random(n_imp) < 0.5, -65 - rng.integers(0, 40, n_imp) - 64 * xs,
                         64 * w_imp + rng.integers(0, 40, n_imp) - 64 * xs)
        neg = -rng.integers(1, 64, (n_imp, 2)) - 64 * np.stack([ys, xs], 1)
        mvs[m] = np.choose(kind[:, None], [r, mult, np.stack([r[:, 0], off_x], 1), neg])
    px, py = rng.integers(0, 64 * w_imp), rng.integers(0, 64 * h_imp)
    mvs[5, :, 0], mvs[5, :, 1] = py - 64 * ys, px - 64 * xs
    intra = np.zeros((5, max(n_intra, 1)), np.uint32)
    intra[:, :n_intra] = rng.integers(0, 40000 << (bd - 8), (5, n_intra))
    intra[rng.random(intra.shape) < 0.1] = 0
    return Window(imgs, PAD, intra, mvs.astype(np.int16), IMP_STEPS, bd)


def imp_paths(win):
    """what the propagating sources of a window reach, from its vectors"""
    rows = min(win.h_imp, win.n_intra // win.w_imp)
    r = {"zero_weight": 0, "three_zero": 0, "none": 0, "floor_ne_trunc": 0, "longest_bucket": 0}
    for _, _, _, mi in win.steps:
        y, x = np.divmod(np.arange(rows * win.w_imp), win.w_imp)
        rx, ry = 64 * x + win.mvs[mi, :len(x), 1].astype(np.int64), 64 * y + win.mvs[mi, :len(x), 0].astype(np.int64)
        fx, fy, bx, by = rx % 64, ry % 64, rx // 64, ry // 64
        r["zero_weight"] += int(((fx == 0) | (fy == 0)).sum())
        r["three_zero"] += int(((fx == 0) & (fy == 0)).sum())
        r["none"] += int(((bx < -1) | (by < -1) | (bx >= win.w_imp) | (by >= win.h_imp)).sum())
        r["floor_ne_trunc"] += int(((rx < 0) & (fx != 0) | (ry < 0) & (fy != 0)).sum())
        if len(x):
            r["longest_bucket"] = max(r["longest_bucket"], int(np.unique(by * 4096 + bx, return_counts=True)[1].max()))
    return r


@pytest.mark.parametrize("bd", BDS)
def test_block_importances_paths(bd):
    c = G.ctx()
    tot = {}
    nonzero = 0
    for k, (W, H) in enumerate(IMP_GEOMS):
        win = imp_window(W, H, bd, 700 + 16 * bd + k)
        planes = [c.plane_from_host(im, win.pad) for im in win.imgs]
        d_imp = canary(4 * 5 * win.n_imp)
        c.block_importances_dev(planes, bd, G.to_dev(win.intra), G.to_dev(win.mvs), win.steps, d_imp)
        c.synchronize()
        got = G.from_dev(d_imp, np.float32).reshape(5, win.n_imp)
        want = oracle_importances(win)
        np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32), err_msg=f"{W}x{H}")
        np.testing.assert_array_equal(model_importances(win).view(np.uint32), want.view(np.uint32))
        for p in planes:
            c.plane_free(p)
        for key, v in imp_paths(win).items():
            tot[key] = max(tot.get(key, 0), v) if key == "longest_bucket" else tot.get(key, 0) + v
        nonzero += int((want > 0).sum())
    shapes = {((W + 7) // 8 == 1, (H + 7) // 8 == 1) for W, H in IMP_GEOMS}
    assert shapes == {(False, False), (True, True), (True, False), (False, True)}     # 1x1, 1xN, Nx1 grids
    assert {W % 8 for W, _ in IMP_GEOMS} >= set(range(1, 8)) and {H % 8 for _, H in IMP_GEOMS} >= set(range(1, 8))
    assert all(v > 0 for v in tot.values()) and tot["longest_bucket"] > 4, tot
    assert nonzero > 0
    assert {s[2] for s in IMP_STEPS} == {1, 2, 3} and len({s[3] for s in IMP_STEPS}) < len(IMP_STEPS)


# ================================================================ 6. distortion scales and scores
def ds_from_num(num):
    sh = (num << 14) & M64
    raw = (M64 if sh > M64 - 16384 else sh + 16384) // 32768
    return min(raw, DS_MAX)


def ds_model(imp, intra):
    """distortion_scale_for with the u64 arithmetic explicit -> (scale, 32768 s, paths)"""
    if intra == 0:
        return 1 << 14, None, {"intra0"}
    v = math.pow((float(intra) + float(imp)) / float(intra), 1.0 / 3.0) * 32768.0
    num = M64 if v >= 2.0 ** 64 else int(v)                              # `as u64` saturates
    paths = set()
    if num << 14 > M64:
        paths.add("wrap")
    if (num << 14) & M64 > M64 - 16384:
        paths.add("saturate")
    if num << 14 <= M64 and ((num << 14) + 16384) // 32768 > DS_MAX:
        paths.add("clamp")
    return ds_from_num(num), v, paths


def near_odd(v, ulps=8):
    if math.isinf(v):
        return False
    odd = 2 * math.floor((v - 1) / 2) + 1
    return min(abs(v - odd), abs(odd + 2 - v)) <= ulps * math.ulp(v)


def test_distortion_scales_edges():
    c = G.ctx()
    rng = np.random.default_rng(81)
    reached, near = set(), 0
    for W, H in ((8 * 40 + 3, 8 * 30 + 5), (8, 8), (5, 7), (8 * 9, 8 * 3 + 1)):
        w_imp, h_imp = (W + 7) // 8, (H + 7) // 8
        n_imp, n_intra = w_imp * h_imp, (W // 8) * (H // 8)
        intra = rng.integers(1, 1 << 20, max(n_intra, 1)).astype(np.uint32)
        imp = (rng.random(n_imp) * 10 * 40000).astype(np.float32)
        m = min(n_intra, n_imp)
        kind = rng.integers(0, 8, m)
        iv = intra[:m].astype(np.float64)
        menu = [np.zeros(m), np.full(m, 1e-45), np.full(m, 1e-40), iv * 2.0 ** 42 * rng.uniform(0.98, 1.02, m),
                iv * 2.0 ** rng.uniform(105, 107, m), np.full(m, np.inf), iv * 2.0 ** rng.uniform(-10, 40, m),
                iv * 2.0 ** rng.uniform(41.9, 42.1, m)]
        with np.errstate(over="ignore"):
            imp[:m] = np.choose(kind, menu).astype(np.float32)
        intra[:m][rng.random(m) < 0.05] = 0
        intra[:m][kind == 4] = rng.integers(1, 1 << 10, int((kind == 4).sum()))   # ratios past 2^105 stay finite
        if m:
            intra[0] = M32
        pl = c.plane_alloc(W, H, 0, 1)
        d_sc = canary(4 * n_imp + 16)
        c.distortion_scales_dev(pl, G.to_dev(imp), G.to_dev(intra) if n_intra else None, d_sc)
        c.synchronize()
        g = d_sc.cpu().numpy()
        assert (g[4 * n_imp:] == CANARY).all()
        got = g[:4 * n_imp].view(np.uint32)
        orc = np.zeros(n_imp, np.uint32)
        T().orc_distortion_scales(imp.ctypes.data, n_imp, intra.ctypes.data, n_intra, orc.ctypes.data)
        for i in range(n_imp):
            if i >= n_intra:
                assert got[i] == orc[i] == 1 << 14
                reached.add("tail")
                continue
            want, v, paths = ds_model(imp[i], int(intra[i]))
            assert orc[i] == want, (i, imp[i], intra[i])
            reached |= paths
            if v is not None and near_odd(v):
                # the device pow may differ from glibc's by 2 ULP: accept the scale of any 32768 s within 8 ULP
                near += 1
                u = 8 * math.ulp(v)
                lo, hi = max(int(v - u), 0), int(min(v + u, 2.0 ** 64))
                assert int(got[i]) in {ds_from_num(min(x, M64)) for x in range(lo, hi + 1)}, (i, imp[i], intra[i])
            else:
                assert got[i] == want, (i, imp[i], intra[i], v)
        c.plane_free(pl)
    print(f"distortion scales within 8 ULP of an odd 32768 s (checked against the neighbouring scales): {near}")
    assert {"tail", "intra0", "wrap", "saturate", "clamp"} <= reached, reached


def np_blog32(w):
    w = w.astype(np.int64)
    ip = np.frexp(w.astype(np.float64))[1].astype(np.int64)
    n = np.where(ip > 16, w >> np.maximum(ip - 16, 0), w << np.maximum(16 - ip, 0)) - 49152
    p = np.full_like(n, -1402)
    for k in (2546, -5216, 15745, -6797):
        p = ((n * p) >> 15) + k
    return np.where(w == 0, -1, (ip << 11) + (p >> 3))


def np_mul(a, b, hits):
    v = (a.astype(np.uint64) * b.astype(np.uint64) + np.uint64(8192)) >> np.uint64(14)
    hits["low"] = hits.get("low", 0) + int((v < 1).sum())
    hits["high"] = hits.get("high", 0) + int((v > DS_MAX).sum())
    return np.clip(v, 1, DS_MAX).astype(np.uint32)


def np_inv_mean(s):
    tot = int(np_blog32(s).sum())
    q = abs(tot) // len(s) * (1 if tot >= 0 else -1)
    arg = C.c_int64((((14 << 11) - q + (14 << 11)) << 46) & M64).value
    return min(max(T().orc_bexp64(arg), 1), DS_MAX)


def np_scores(d, a, hits):
    """compute_{spatio,}temporal_scores vectorised (the logexp scalars from the oracle)"""
    if a is None:
        inv = np_inv_mean(d)
        d = np_mul(d, np.uint32(inv), hits)
        st = d.copy()
    else:
        st = np_mul(d, a, hits)
        inv = np_inv_mean(st)
        st, d = np_mul(st, np.uint32(inv), hits), np_mul(d, np.uint32(inv), hits)
    return d, st, (T().orc_blog64(inv) - (14 << 57)) >> 1


def score_map(rng, n, kind):
    if kind == "high":                                   # a high mean: inv_mean < 8192, so 1 * inv clamps to 1
        s = np.exp2(rng.uniform(20, 28, n))
        s[::7] = 1
    else:                                                # a low mean: inv_mean > 2^14, so DS_MAX * inv clamps
        s = np.exp2(rng.uniform(0, 10, n))
        s[::11] = DS_MAX
    return np.clip(s, 1, DS_MAX).astype(np.uint32)


def test_temporal_scores_every_form_and_output():
    c = G.ctx()
    rng = np.random.default_rng(91)
    hits_t, hits_st = {}, {}
    cap = num_sms() * SCORES_CTAS * SCORES_THREADS
    maps = [(1, 1, "low"), (1, 7, "high"), (7, 1, "low"), (37, 23, "high"), (23, 37, "low"), (1024, 544, "low")]
    assert 1024 * 544 > cap
    for w_imp, h_imp, kind in maps:
        n = w_imp * h_imp
        d0 = score_map(rng, n, kind)
        act = np.exp2(rng.uniform(0, 28, n)).clip(1, DS_MAX).astype(np.uint32)
        act[::5], act[1::5] = 1, DS_MAX
        for form_act in (None, act):
            hits = hits_t if form_act is None else hits_st
            wd, wst, wlog = np_scores(d0, form_act, hits)
            od, ost, olog = oracle_scores(d0, form_act)
            np.testing.assert_array_equal(od, wd)
            np.testing.assert_array_equal(ost, wst)
            assert olog == wlog
            if n < 5000:
                pd, pst, plog = py_scores(d0, form_act)
                np.testing.assert_array_equal(pd, wd)
                np.testing.assert_array_equal(pst, wst)
                assert plog == wlog
            stride4 = 2 * w_imp + 5
            for null in ("none", "st", "log", "map"):
                if null == "st" and form_act is not None:
                    continue                                  # the spatiotemporal form requires it
                d_s = G.to_dev(d0)
                d_act = None if form_act is None else G.to_dev(form_act)
                d_st, d_log = canary(4 * n + 16), canary(16)
                d_map = torch.from_numpy(np.full(stride4 * 2 * h_imp + 8, 0xDEADBEEF, np.uint32).view(np.uint8)).cuda()
                c.temporal_scores_dev(w_imp, h_imp, d_s, d_act, None if null == "st" else d_st,
                                      None if null == "log" else d_log, None if null == "map" else d_map, stride4)
                c.synchronize()
                np.testing.assert_array_equal(G.from_dev(d_s, np.uint32), wd)
                gst, glog = d_st.cpu().numpy(), d_log.cpu().numpy()
                if null != "st":
                    np.testing.assert_array_equal(gst[:4 * n].view(np.uint32), wst)
                assert (gst[4 * n if null != "st" else 0:] == CANARY).all()
                if null != "log":
                    assert int(glog[:8].view(np.int64)[0]) == wlog
                assert (glog[8 if null != "log" else 0:] == CANARY).all()
                gm = G.from_dev(d_map, np.uint32)
                body = gm[:stride4 * 2 * h_imp].reshape(2 * h_imp, stride4)
                if null != "map":
                    np.testing.assert_array_equal(body[:, :2 * w_imp],
                                                  np.repeat(np.repeat(wd.reshape(h_imp, w_imp), 2, 0), 2, 1))
                    assert (body[:, 2 * w_imp:] == 0xDEADBEEF).all()           # the gap columns
                else:
                    assert (body == 0xDEADBEEF).all()
                assert (gm[stride4 * 2 * h_imp:] == 0xDEADBEEF).all()
    assert hits_t["low"] > 0 and hits_t["high"] > 0, hits_t
    assert hits_st["low"] > 0 and hits_st["high"] > 0, hits_st


# ================================================================ 7. rejected calls
def clone(p, **kw):
    q = B.Plane()
    C.memmove(C.byref(q), C.byref(p), C.sizeof(B.Plane))
    for k, v in kw.items():
        setattr(q, k, v)
    return q


def rejected(c, call, bufs, name):
    n0 = c.launches
    before = [b.clone() for b in bufs]
    with pytest.raises(B.B200Error) as e:
        call()
    assert e.value.status == B.ERR_ARG, name
    c.synchronize()
    assert c.launches == n0, name
    for b, s in zip(bufs, before):
        assert torch.equal(b, s), name


def accepted_without_launch(c, call, bufs, name):
    n0 = c.launches
    before = [b.clone() for b in bufs]
    call()
    c.synchronize()
    assert c.launches == n0, name
    for b, s in zip(bufs, before):
        assert torch.equal(b, s), name


def test_rejected_calls_launch_nothing():
    c = G.ctx()
    L, h = c.L, c.h
    rng = np.random.default_rng(99)
    p8 = c.plane_from_host(rng.integers(0, 256, (40, 48), dtype=np.uint8), 8)
    p16 = c.plane_from_host(rng.integers(0, 1024, (40, 48)).astype(np.uint16), 8)
    q16 = c.plane_from_host(rng.integers(0, 1024, (40, 48)).astype(np.uint16), 8)
    odd16 = c.plane_from_host(rng.integers(0, 1024, (37, 45)).astype(np.uint16), 0)     # no padding
    small16 = c.plane_from_host(np.zeros((7, 7), np.uint16), 8)
    blocks = G.to_dev(np.zeros(4, B.BLOCK_DTYPE))
    out, out2, scale = canary(256), canary(256), canary(4096)
    dp = C.c_void_p
    null_ctx = []

    # b200_weighted_sse_dev
    ws = lambda a, b, bl, n, w, hh, sc, o: c.weighted_sse_dev(a, b, bl, n, w, hh, sc, 16, o)
    for name, args in {"bpp differs": (p8, p16, blocks, 4, 8, 8, scale, out),
                       "bpp 3": (clone(p16, bpp=3), clone(q16, bpp=3), blocks, 4, 8, 8, scale, out),
                       "NULL data": (clone(p16, data=None), q16, blocks, 4, 8, 8, scale, out),
                       "w 3": (p16, q16, blocks, 4, 3, 8, scale, out), "h 129": (p16, q16, blocks, 4, 8, 129, scale, out),
                       "w 132": (p16, q16, blocks, 4, 132, 8, scale, out),
                       "NULL blocks": (p16, q16, None, 4, 8, 8, scale, out),
                       "NULL scale": (p16, q16, blocks, 4, 8, 8, None, out),
                       "NULL out": (p16, q16, blocks, 4, 8, 8, scale, None)}.items():
        rejected(c, lambda: ws(*args), [out, scale], "wsse " + name)
    rejected(c, lambda: c.check(L.b200_weighted_sse_dev(h, None, C.byref(q16), blocks.data_ptr(), 4, 8, 8,
                                                        scale.data_ptr(), 16, out.data_ptr())), [out], "wsse NULL plane")
    accepted_without_launch(c, lambda: ws(p16, q16, None, 0, 8, 8, None, None), [out], "wsse n 0")
    null_ctx.append(L.b200_weighted_sse_dev(None, C.byref(p16), C.byref(q16), blocks.data_ptr(), 4, 8, 8,
                                            scale.data_ptr(), 16, out.data_ptr()))

    # b200_cdef_dist_dev
    cd = lambda a, b, bl, n, w, hh, bd, o, r: c.cdef_dist_dev(a, b, bl, n, w, hh, bd, o, r)
    for name, args in {"bpp differs": (p8, p16, blocks, 4, 8, 8, 10, out, out2),
                       "w 0": (p16, q16, blocks, 4, 0, 8, 10, out, out2), "w 9": (p16, q16, blocks, 4, 9, 8, 10, out, out2),
                       "h 9": (p16, q16, blocks, 4, 8, 9, 10, out, out2), "bd 9": (p16, q16, blocks, 4, 8, 8, 9, out, out2),
                       "bd 11": (p16, q16, blocks, 4, 8, 8, 11, out, out2),
                       "bd 8 on u16": (p16, q16, blocks, 4, 8, 8, 8, out, out2),
                       "bd 10 on u8": (p8, p8, blocks, 4, 8, 8, 10, out, out2),
                       "NULL blocks": (p16, q16, None, 4, 8, 8, 10, out, out2),
                       "no output": (p16, q16, blocks, 4, 8, 8, 10, None, None)}.items():
        rejected(c, lambda: cd(*args), [out, out2], "cdef_dist " + name)
    accepted_without_launch(c, lambda: cd(p16, q16, None, 0, 8, 8, 10, None, None), [out], "cdef_dist n 0")
    null_ctx.append(L.b200_cdef_dist_dev(None, C.byref(p16), C.byref(q16), blocks.data_ptr(), 4, 8, 8, 10,
                                         out.data_ptr(), None))

    # b200_activity_mask_dev
    for name, args in {"bpp 3": (clone(p16, bpp=3), 10, out, out2), "bd 11": (p16, 11, out, out2),
                       "bd 10 on u8": (p8, 10, out, out2), "bd 8 on u16": (p16, 8, out, out2),
                       "NULL data": (clone(p16, data=None), 10, out, out2),
                       "padding below the rounding": (odd16, 10, out, out2), "NULL variances": (p16, 10, None, out2)}.items():
        rejected(c, lambda: c.activity_mask_dev(*args), [out, out2], "activity " + name)
    rejected(c, lambda: c.check(L.b200_activity_mask_dev(h, None, 10, out.data_ptr(), None)), [out], "activity NULL")
    accepted_without_launch(c, lambda: c.activity_mask_dev(clone(p16, width=0, height=0), 10, out, out2), [out, out2],
                            "activity empty plane")
    null_ctx.append(L.b200_activity_mask_dev(None, C.byref(p16), 10, out.data_ptr(), None))

    # b200_plane_downsample_dev
    d16 = c.plane_alloc(24, 20, 4, 2)
    before = download_padded(c, d16, np.uint16).copy()
    for name, args in {"bpp differs": (p8, d16, 24, 20), "bpp 3": (clone(p16, bpp=3), clone(d16, bpp=3), 24, 20),
                       "wrong size": (p16, clone(d16, width=23), 23, 20), "pad_w 0": (p16, d16, 0, 20),
                       "pad_w 25": (p16, d16, 25, 20), "pad_h 0": (p16, d16, 24, 0), "pad_h 21": (p16, d16, 24, 21),
                       "NULL dst data": (p16, clone(d16, data=None), 24, 20)}.items():
        rejected(c, lambda: c.plane_downsample_dev(*args), [], "downsample " + name)
    d_odd = c.plane_alloc(23, 19, 4, 2)
    rejected(c, lambda: c.plane_downsample_dev(odd16, d_odd, 23, 19), [], "downsample odd source without padding")
    rejected(c, lambda: c.check(L.b200_plane_downsample_dev(h, None, C.byref(d16), 24, 20)), [], "downsample NULL")
    np.testing.assert_array_equal(download_padded(c, d16, np.uint16), before)
    null_ctx.append(L.b200_plane_downsample_dev(None, C.byref(p16), C.byref(d16), 24, 20))

    # b200_estimate_intra_costs_dev
    for name, args in {"bd 9": (p16, 9, out), "bd 11": (p16, 11, out), "bd 7": (p8, 7, out), "bd 13": (p16, 13, out),
                       "bd 10 on u8": (p8, 10, out), "bd 8 on u16": (p16, 8, out),
                       "bpp 3": (clone(p16, bpp=3), 10, out), "NULL costs": (p16, 10, None),
                       "NULL data": (clone(p16, data=None), 10, out)}.items():
        rejected(c, lambda: c.estimate_intra_costs_dev(*args), [out], "intra " + name)
    rejected(c, lambda: c.check(L.b200_estimate_intra_costs_dev(h, None, 10, out.data_ptr())), [out], "intra NULL")
    accepted_without_launch(c, lambda: c.estimate_intra_costs_dev(small16, 10, out), [out], "intra 7x7 frame")
    null_ctx.append(L.b200_estimate_intra_costs_dev(None, C.byref(p16), 10, out.data_ptr()))

    # b200_estimate_inter_costs_dev and b200_importance_block_difference_dev
    mvs, sc8, mean = G.to_dev(np.zeros((5, 6, 2), np.int16)), canary(8), canary(8)
    big16 = c.plane_from_host(np.zeros((40, 56), np.uint16), 8)
    for name, (a, b) in {"bpp differs": (p8, p16), "size differs": (p16, big16), "smaller than a block": (small16, small16),
                         "bpp 3": (clone(p16, bpp=3), clone(q16, bpp=3)), "NULL data": (clone(p16, data=None), q16)}.items():
        rejected(c, lambda: c.estimate_inter_costs_dev(a, b, mvs, out, sc8, mean), [out, sc8, mean], "inter " + name)
        rejected(c, lambda: c.importance_block_difference_dev(a, b, sc8, mean), [sc8, mean], "imp diff " + name)
    for name, args in {"NULL mvs": (None, out, sc8, mean), "NULL scratch": (mvs, out, None, mean),
                       "NULL mean": (mvs, out, sc8, None)}.items():
        rejected(c, lambda: c.estimate_inter_costs_dev(p16, q16, *args), [out, sc8, mean], "inter " + name)
    for name, args in {"NULL scratch": (None, mean), "NULL mean": (sc8, None)}.items():
        rejected(c, lambda: c.importance_block_difference_dev(p16, q16, *args), [sc8, mean], "imp diff " + name)
    rejected(c, lambda: c.check(L.b200_estimate_inter_costs_dev(h, None, C.byref(q16), mvs.data_ptr(), None,
                                                                sc8.data_ptr(), mean.data_ptr())), [sc8, mean], "inter NULL")
    null_ctx.append(L.b200_estimate_inter_costs_dev(None, C.byref(p16), C.byref(q16), mvs.data_ptr(), None,
                                                    sc8.data_ptr(), mean.data_ptr()))
    null_ctx.append(L.b200_importance_block_difference_dev(None, C.byref(p16), C.byref(q16), sc8.data_ptr(),
                                                           mean.data_ptr()))

    # b200_block_importances_dev
    frames = [p16, q16, clone(q16)]
    imp = canary(4 * 3 * 30)
    intra, mv3 = G.to_dev(np.ones((3, 30), np.uint32)), G.to_dev(np.zeros((2, 30, 2), np.int16))
    good = [(2, 1, 1, 0), (1, 0, 1, 1)]
    huge = clone(p16, width=8 << 16, height=8 << 14, pad=0)
    for name, (fr, bd, it, mv, steps, dst) in {
            "bd 9": (frames, 9, intra, mv3, good, imp), "bd 11": (frames, 11, intra, mv3, good, imp),
            "bd 8 on u16": (frames, 8, intra, mv3, good, imp), "bd 13": (frames, 13, intra, mv3, good, imp),
            "bpp 3": ([clone(f, bpp=3) for f in frames], 10, intra, mv3, good, imp),
            "sizes differ": ([p16, big16, q16], 10, intra, mv3, good, imp),
            "bpp differs": ([p16, p8, q16], 10, intra, mv3, good, imp),
            "NULL frame data": ([p16, clone(q16, data=None), q16], 10, intra, mv3, good, imp),
            "empty frame": ([clone(f, width=0) for f in frames], 10, intra, mv3, good, imp),
            "padding below the ceil grid": ([odd16, odd16, odd16], 10, intra, mv3, good, imp),
            "NULL importances": (frames, 10, intra, mv3, good, None),
            "NULL intra": (frames, 10, None, mv3, good, imp), "NULL mvs": (frames, 10, intra, None, good, imp),
            "src outside": (frames, 10, intra, mv3, [(3, 1, 1, 0)], imp),
            "dst outside": (frames, 10, intra, mv3, [(1, 3, 1, 0)], imp),
            "src == dst": (frames, 10, intra, mv3, [(1, 1, 1, 0)], imp),
            "len 0": (frames, 10, intra, mv3, [(2, 1, 0, 0)], imp), "len 4": (frames, 10, intra, mv3, [(2, 1, 4, 0)], imp),
            "src not final": (frames, 10, intra, mv3, [(1, 0, 1, 0), (2, 1, 1, 1)], imp),
            "window too large": ([huge] * 3, 10, intra, mv3, good, imp)}.items():
        rejected(c, lambda: c.block_importances_dev(fr, bd, it, mv, steps, dst), [imp], "importances " + name)
    rejected(c, lambda: c.check(L.b200_block_importances_dev(h, 0, None, 10, intra.data_ptr(), mv3.data_ptr(), 0, None,
                                                             imp.data_ptr())), [imp], "importances no frames")
    n0 = c.launches
    c.block_importances_dev(frames, 10, None, None, [], imp)                  # no steps: zeroed, no kernel
    c.synchronize()
    assert c.launches == n0 and (G.from_dev(imp, np.float32)[:3 * 30] == 0).all()
    null_ctx.append(L.b200_block_importances_dev(None, 3, None, 10, None, None, 0, None, imp.data_ptr()))

    # b200_distortion_scales_dev
    fimp, fint, sc = G.to_dev(np.zeros(30, np.float32)), G.to_dev(np.ones(30, np.uint32)), canary(4 * 30)
    for name, args in {"empty frame": (clone(p16, width=0), fimp, fint, sc), "NULL importances": (p16, None, fint, sc),
                       "NULL intra with blocks": (p16, fimp, None, sc), "NULL scales": (p16, fimp, fint, None)}.items():
        rejected(c, lambda: c.distortion_scales_dev(*args), [sc], "scales " + name)
    rejected(c, lambda: c.check(L.b200_distortion_scales_dev(h, None, fimp.data_ptr(), fint.data_ptr(), sc.data_ptr())),
             [sc], "scales NULL frame")
    null_ctx.append(L.b200_distortion_scales_dev(None, C.byref(p16), fimp.data_ptr(), fint.data_ptr(), sc.data_ptr()))

    # b200_temporal_scores_dev
    s30, a30, st, lg, mp = canary(4 * 30), canary(4 * 30), canary(4 * 30), canary(8), canary(4 * 12 * 10)
    for name, args in {"w 0": (0, 5, s30, None, st, lg, None, 0), "h 0": (6, 0, s30, None, st, lg, None, 0),
                       "2^30 blocks": (1 << 15, 1 << 15, s30, None, st, lg, None, 0),
                       "product wraps": (1 << 32, 1 << 32, s30, None, st, lg, None, 0),
                       "NULL scales": (6, 5, None, None, st, lg, None, 0),
                       "activity without output": (6, 5, s30, a30, None, lg, None, 0),
                       "4x4 stride < 2 w": (6, 5, s30, None, st, lg, mp, 11)}.items():
        rejected(c, lambda: c.temporal_scores_dev(*args), [s30, st, lg, mp], "scores " + name)
    null_ctx.append(L.b200_temporal_scores_dev(None, 6, 5, s30.data_ptr(), None, None, None, None, 0))

    assert len(null_ctx) == 10 and all(s == B.ERR_ARG for s in null_ctx), null_ctx
    for p in (p8, p16, q16, odd16, small16, d16, d_odd, big16):
        c.plane_free(p)
