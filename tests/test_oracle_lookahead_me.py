"""CPU tests of the lookahead's motion vectors in the oracle (oracle/lookahead_me.c: orc_lookahead_motion, the
serial estimate_tile_motion of me.rs:153-337 / 386-534 / 633-690) against an independent pure-Python
model of the same driver, stats grid entry for entry.  The model is written from the reference text and
composes with the full_pixel_me model of tests/test_oracle_search.py.

Also shared with the GPU tests: the ctypes binding of the oracle driver and the case generator.
"""
import ctypes as C
from dataclasses import dataclass

import numpy as np
import pytest

from tests import oracle_lib as O
from tests.test_oracle_search import EMPTY, Model, full_pixel_me, i16, mv_range, tdiv8

STATS_DTYPE = np.dtype([("mv_row", "<i2"), ("mv_col", "<i2"), ("normalized_sad", "<u4")])
PAD = 64  # enough for every level (include/b200rdo.h, lookahead motion) at these sizes


def downsample(img):
    """half resolution: 2x2 means, rounded; odd edges replicated"""
    h, w = img.shape
    e = np.pad(img.astype(np.int64), ((0, h & 1), (0, w & 1)), mode="edge")
    s = e[0::2, 0::2] + e[1::2, 0::2] + e[0::2, 1::2] + e[1::2, 1::2]
    return ((s + 2) >> 2).astype(img.dtype)


def pyramid(img, pad=PAD):
    """[full, half, quarter] oracle Planes with replicated edges"""
    out, cur = [], img
    for _ in range(3):
        p = O.Plane(cur.shape[1], cur.shape[0], pad, dtype=cur.dtype)
        p.fill_from(cur)
        out.append(p)
        cur = downsample(cur)
    return out


@dataclass
class Params:
    bit_depth: int = 8
    allow_hp: int = 0
    me_lambda: float = 1.0
    full_search: int = 0
    range_scale: int = 1
    tile_w_sb: int = 64
    tile_h_sb: int = 64


def grid_dims(width, height):
    return 2 * ((width + 7) >> 3), 2 * ((height + 7) >> 3)


_BOUND = False


def _lib():
    global _BOUND
    L = O.lib()
    if not _BOUND:
        vp, pd, i32 = C.c_void_p, C.c_ssize_t, C.c_int
        L.orc_lookahead_motion.restype = None
        L.orc_lookahead_motion.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, i32, C.c_double, i32, i32, i32, i32,
                                           vp, vp]
        L.orc_lookahead_me_thresh.restype = C.c_uint32
        L.orc_lookahead_me_thresh.argtypes = [C.c_uint32, i32, i32, i32]
        _BOUND = True
    return L


def oracle_motion(cur, ref, width, height, p: Params, prev=None):
    """cur / ref: [full, half, quarter] oracle Planes -> w_in_b x h_in_b STATS_DTYPE grid"""
    wib, hib = grid_dims(width, height)
    out = np.zeros((hib, wib), STATS_DTYPE)
    cp = (C.c_void_p * 3)(*[q.origin_ptr() for q in cur])
    rp = (C.c_void_p * 3)(*[q.origin_ptr() for q in ref])
    cs = (C.c_ssize_t * 3)(*[q.stride for q in cur])
    rs = (C.c_ssize_t * 3)(*[q.stride for q in ref])
    pv = None if prev is None else np.ascontiguousarray(prev, STATS_DTYPE)
    _lib().orc_lookahead_motion(C.addressof(cp), C.addressof(cs), C.addressof(rp), C.addressof(rs), cur[0].bpp,
                                width, height, p.bit_depth, p.allow_hp, p.me_lambda, p.full_search, p.range_scale,
                                p.tile_w_sb, p.tile_h_sb, None if pv is None else pv.ctypes.data, out.ctypes.data)
    return out


# ---------------------------------------------------------------- the independent model
def model_motion(cur, ref, width, height, p: Params, prev=None):
    W8, H8 = (width + 7) & ~7, (height + 7) & ~7
    wib, hib = W8 // 4, H8 // 4
    grid = [[(0, 0, 0)] * wib for _ in range(hib)]  # (row, col, normalized_sad)
    tw, th = p.tile_w_sb * 64, p.tile_h_sb * 64
    for ty in range(0, H8, th):
        for tx in range(0, W8, tw):
            t = dict(x0=tx // 4, y0=ty // 4, w=min(tw, W8 - tx), h=min(th, H8 - ty))
            t["cols"], t["rows"] = t["w"] // 4, t["h"] // 4
            for log2 in (4, 3, 2):
                s = log2 - 2  # ssdec 2, 1, 0 (me.rs:164-168)
                lam = me.lam(p.me_lambda, s)
                for sby in range(-(-t["h"] // 64)):
                    for sbx in range(-(-t["w"] // 64)):
                        if log2 < 4:
                            me.sb(grid, t, cur, ref, p, prev, sbx, sby, log2 + 1, s, lam, True, wib, hib)
                        me.sb(grid, t, cur, ref, p, prev, sbx, sby, log2, s, lam, False, wib, hib)
    out = np.zeros((hib, wib), STATS_DTYPE)
    for y in range(hib):
        for x in range(wib):
            out[y, x] = grid[y][x]
    return out


class me:  # namespace for the model's steps
    @staticmethod
    def lam(me_lambda, s):  # me.rs:175-176
        v = me_lambda * 256.0 / float(1 << (2 * s)) * (0.5 if s == 0 else 0.125)
        return 0 if not v > 0 else min(int(v), 2**32 - 1)

    @staticmethod
    def thresh(min_sad, w, h, bd):  # me.rs:771-772
        v = np.float32(min_sad) * np.float32(1.2)
        return (min(int(v), 2**32 - 1) + ((w * h) << (bd - 8))) & 0xFFFFFFFF  # release-build wrap

    @staticmethod
    def model(cur, ref, s, t, bx, by, w, h, lam, p, wib, hib):
        fx, fy = t["x0"] + bx, t["y0"] + by
        rng = tuple(v >> s for v in mv_range(wib, hib, 4 * fx, 4 * fy, w << s, h << s))
        po = ((4 * fx) >> s, (4 * fy) >> s)
        m = Model(cur[s].data, ref[s].data, cur[s].pad, po[0], po[1], w, h, rng, lam, [(0, 0), (0, 0)],
                  bool(p.allow_hp))
        return m, rng, po

    @staticmethod
    def full_search(m, rng, po, x_lo, x_hi, y_lo, y_hi, step):  # me.rs:1464-1509
        best = (EMPTY[0], EMPTY[1], (0, 0))
        for y in range(y_lo, y_hi + 1, step):
            for x in range(x_lo, x_hi + 1, step):
                r = m.rd((i16(8 * (y - po[1])), i16(8 * (x - po[0]))))
                if r[0] < best[0]:
                    best = r
        return best

    @staticmethod
    def predictors(grid, t, prev, rng, bx, by, w, h, corner, s, wib, hib):  # me.rs:386-534
        min_sad = [2**32 - 1]

        def proc(st):
            min_sad[0] = min(min_sad[0], st[2])
            row, col = tdiv8(st[0]) * 8, tdiv8(st[1]) * 8
            return (min(max(row, rng[2]), rng[3]), min(max(col, rng[0]), rng[1]))

        def T(x, y):
            return grid[t["y0"] + y][t["x0"] + x]
        wb, hb = ((w << s) + 3) >> 2, ((h << s) + 3) >> 2
        chw, chh = min(wb >> 1, t["cols"] - 1 - bx), min(hb >> 1, t["rows"] - 1 - by)
        b, c = [], []
        if bx > 0:
            b.append(proc(T(bx - 1, by + chh)))
        if by > 0:
            b.append(proc(T(bx + chw, by - 1)))
        if corner is not None and corner[0] and bx + wb < t["cols"]:
            b.append(proc(T(bx + wb, by + chh)))
        if corner is not None and corner[1] and by + hb < t["rows"]:
            b.append(proc(T(bx + chw, by + hb)))
        if corner is not None:
            median = [proc(T(bx + chw, by + chh))]
        elif len(b) == 3:
            median = [(sorted(v[0] for v in b)[1], sorted(v[1] for v in b)[1])]
        else:
            median = []
        b.append((0, 0))
        if prev is not None:
            fx, fy = t["x0"] + bx, t["y0"] + by
            P = lambda x, y: tuple(int(v) for v in prev[y, x])  # noqa: E731
            hw, hh = min(wb >> 1, wib - 1 - fx), min(hb >> 1, hib - 1 - fy)
            if fx > 0:
                c.append(proc(P(fx - 1, fy + hh)))
            if fy > 0:
                c.append(proc(P(fx + hw, fy - 1)))
            if fx + wb < wib:
                c.append(proc(P(fx + wb, fy + hh)))
            if fy + hb < hib:
                c.append(proc(P(fx + hw, fy + hb)))
            c.append(proc(P(fx + hw, fy + hh)))
        dec = lambda v: (v[0] >> s, v[1] >> s)  # noqa: E731
        return (min_sad[0] * w * h) >> 14, [dec(v) for v in median], [dec(v) for v in b], [dec(v) for v in c]

    @staticmethod
    def sb(grid, t, cur, ref, p, prev, sbx, sby, log2, s, lam, refine, wib, hib):
        px, py = 64 * sbx, 64 * sby
        sb_w, sb_h = min(64, t["w"] - px), min(64, t["h"] - py)
        mv_size = 4 << log2
        for y in range(0, sb_h, mv_size):
            for x in range(0, sb_w, mv_size):
                bx, by = (px + x) >> 2, (py + y) >> 2
                w = min(mv_size, sb_w - x + (1 << s) - 1) >> s
                h = min(mv_size, sb_h - y + (1 << s) - 1) >> s
                m, rng, po = me.model(cur, ref, s, t, bx, by, w, h, lam, p, wib, hib)
                if refine:  # me.rs:633-690
                    st = grid[t["y0"] + by][t["x0"] + bx]
                    mr, mc = tdiv8(st[0] >> s), tdiv8(st[1] >> s)
                    r = me.full_search(m, rng, po, po[0] + max(mc - 1, tdiv8(rng[0])), po[0] + min(mc + 2, tdiv8(rng[1])),
                                       po[1] + max(mr - 1, tdiv8(rng[2])), po[1] + min(mr + 2, tdiv8(rng[3])), 1)
                else:
                    corner = None if log2 == 4 else (bool(x & mv_size), bool(y & mv_size))
                    min_sad, median, b, c = me.predictors(grid, t, prev, rng, bx, by, w, h, corner, s, wib, hib)
                    if log2 != 4:
                        r = full_pixel_me(m, [median + b + c], False, 0, 0)
                    else:
                        th = me.thresh(min_sad, w, h, p.bit_depth)
                        r = full_pixel_me(m, [median, b, c], True, th, 24)
                        if p.full_search and r[1] >= th:
                            rx, ry = (192 * p.range_scale) >> s, (64 * p.range_scale) >> s
                            f = me.full_search(m, rng, po, po[0] + max(-rx, tdiv8(rng[0])), po[0] + min(rx, tdiv8(rng[1])),
                                               po[1] + max(-ry, tdiv8(rng[2])), po[1] + min(ry, tdiv8(rng[3])), 4 >> s)
                            r = f if f[0] < r[0] else r
                st = (i16(r[2][0] << s), i16(r[2][1] << s), ((r[1] << 14) // (w * h)) & 0xFFFFFFFF)
                for yy in range(by, min(by + (1 << log2), t["rows"])):
                    for xx in range(bx, min(bx + (1 << log2), t["cols"])):
                        grid[t["y0"] + yy][t["x0"] + xx] = st


# ---------------------------------------------------------------- cases
SHIFT = (5, -3)  # (dx, dy) px: cur(x, y) = ref(x + dx, y + dy), so the vector is (8 dy, 8 dx)


def images(width, height, bd, smooth, seed):
    from tests.gpu_util import make_planes
    dtype = np.uint8 if bd == 8 else np.uint16
    return make_planes(width, height, 0, dtype, seed=seed, bit_depth=bd, smooth=smooth, shift=SHIFT)


# (width, height, tiles (w_sb, h_sb), prev, full search, range scale, bit depth, smooth, lambda)
CASES = [
    (72, 40, (64, 64), False, 0, 1, 8, True, 3.5),
    (72, 40, (1, 1), True, 1, 2, 10, False, 0.0),
    (200, 120, (64, 64), True, 0, 1, 8, True, 2.0),
    (200, 120, (2, 1), False, 1, 1, 8, False, 0.0),
    (200, 120, (2, 1), True, 1, 2, 10, True, 6.0),
    (136, 264, (1, 2), True, 0, 2, 8, False, 0.0),
    (136, 264, (64, 64), False, 1, 1, 10, True, 1.0),
    (136, 264, (2, 3), True, 1, 1, 8, True, 4.0),
]
IDS = [f"{w}x{h}-t{t[0]}x{t[1]}-prev{int(pv)}-fs{fs}-rs{rs}-bd{bd}-{'smooth' if sm else 'noise'}"
       for w, h, t, pv, fs, rs, bd, sm, _ in CASES]


def case_inputs(case, seed=11):
    """-> (cur pyramid, ref pyramid, Params, prev grid or None, cur image, ref image)"""
    w, h, tiles, with_prev, fs, rs, bd, smooth, lam = case
    cur_img, ref_img = images(w, h, bd, smooth, seed)
    p = Params(bit_depth=bd, me_lambda=lam, full_search=fs, range_scale=rs, tile_w_sb=tiles[0], tile_h_sb=tiles[1])
    prev = None
    if with_prev:  # LAST's stats: the same pair, searched against a differently shifted ref
        older, _ = images(w, h, bd, smooth, seed + 1)
        prev = oracle_motion(pyramid(older), pyramid(ref_img), w, h, p)
    return pyramid(cur_img), pyramid(ref_img), p, prev, cur_img, ref_img


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_oracle_matches_python_model(case):
    cur, ref, p, prev, _, _ = case_inputs(case)
    w, h = case[0], case[1]
    got = oracle_motion(cur, ref, w, h, p, prev)
    want = model_motion(cur, ref, w, h, p, prev)
    assert got.shape == grid_dims(w, h)[::-1]
    bad = np.argwhere(got != want)
    assert len(bad) == 0, (len(bad), bad[:4].tolist(), got[tuple(bad[0])], want[tuple(bad[0])])


def test_smooth_pattern_recovers_the_shift():
    w, h = 200, 120
    cur, ref, p, _, _, _ = case_inputs((w, h, (64, 64), False, 0, 1, 8, True, 2.0))
    got = oracle_motion(cur, ref, w, h, p)
    inner = got[4:-4, 4:-4]  # away from the replicated borders
    hit = (inner["mv_row"] == 8 * SHIFT[1]) & (inner["mv_col"] == 8 * SHIFT[0])
    assert hit.mean() > 0.9, hit.mean()


def test_prev_stats_and_tiles_change_the_result():
    """subset C and the tile grid are live inputs (a slip in either would otherwise hide)"""
    case = (136, 264, (64, 64), True, 0, 1, 8, False, 0.0)
    cur, ref, p, prev, _, _ = case_inputs(case)
    base = oracle_motion(cur, ref, 136, 264, p, prev)
    assert (base != oracle_motion(cur, ref, 136, 264, p, None)).any()
    p2 = Params(**{**p.__dict__, "tile_w_sb": 1, "tile_h_sb": 2})
    assert (base != oracle_motion(cur, ref, 136, 264, p2, prev)).any()


@pytest.mark.parametrize("min_sad,w,h,bd", [(0, 16, 16, 8), (5, 2, 2, 8), (261888, 16, 16, 10),
                                            (67108863, 16, 16, 8), (16777217, 2, 16, 10), (2**32 - 1, 1, 1, 8)])
def test_thresh_uses_the_f32_product(min_sad, w, h, bd):
    """me.rs:771-772 multiplies in f32: above 2^24 the result differs from the f64 one"""
    assert _lib().orc_lookahead_me_thresh(min_sad, w, h, bd) == me.thresh(min_sad, w, h, bd)
    if min_sad == 67108863:  # u32::MAX un-normalized for a 16x16 block: the first block of a tile
        assert me.thresh(min_sad, w, h, bd) != int(min_sad * 1.2) + (w * h << (bd - 8))
