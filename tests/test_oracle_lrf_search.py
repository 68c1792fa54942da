"""The restoration search of rdo_loop_decision (oracle/lrf_search.c) against an independent Python restatement of
rav1e src/rdo.rs:2575-2740.

The restatement shares no code with the oracle: it pads each unit by setup_integral_image's clip rule and forms
the box sums directly, solves with exact rational arithmetic (Fraction) for the fused and rounded steps and
numpy int64 for the sums, counts the subexp bits by walking the AV1 specification's
decode_signed_subexp_with_ref process, and measures with the distortion helpers of test_oracle_cdef_rdo.py.
Also holds the ctypes wrapper of orc_lrf_search and the item builder the GPU test uses."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import oracle_lib as O
from tests.test_oracle_cdef_rdo import cdef_dist, fma, mul_u64, weighted_sse
from tests.test_oracle_lrf_spec import LAYOUTS, SGR_PARAMS, XQD_MAX, XQD_MIN

WORK_FILL = 128                       # B200_LRF_WORK_FILL: v_frame Plane::new's T::cast_from(128)
FULL_SETS, REDUCED_SETS = list(range(16)), list(range(1, 16, 2))     # lrf.rs:77-86


# ---------------------------------------------------------------- inputs
def make_frame(rng, W, H, layout, bd, content="random"):
    """(lrf_in, src): planes covering the frame rounded up to 8 luma pixels."""
    planes, xdec, ydec = LAYOUTS[layout]
    mx = (1 << bd) - 1
    dt = np.uint8 if bd == 8 else np.uint16
    w8, h8 = (W + 7) & ~7, (H + 7) & ~7
    lin, src = [], []
    for p in range(planes):
        w, h = (w8 >> xdec, h8 >> ydec) if p else (w8, h8)
        yy, xx = np.mgrid[0:h, 0:w]
        if content == "flat":
            s = np.full((h, w), mx // 3)
            r = s.copy()
        elif content == "extreme":           # 0 / max checkerboards: the largest sums and xqd at its ends
            s = ((yy // 3 + xx // 5) % 2) * mx
            r = np.where(rng.random((h, w)) < 0.5, s, mx - s)
        else:
            s = (np.sin(xx / 6.0 + p) + np.cos(yy / 4.0)) * mx / 4 + mx / 2 + rng.normal(0, mx / 40, (h, w))
            r = s + rng.normal(0, mx / 25, (h, w))
        lin.append(np.ascontiguousarray(np.clip(np.rint(r), 0, mx).astype(dt)))
        src.append(np.ascontiguousarray(np.clip(np.rint(s), 0, mx).astype(dt)))
    return lin, src


def areas_and_items(rng, W, H, layout, unit_size, incoming="none", ref=None, cost=-1.0):
    """The areas rdo_loop_decision walks (the largest unit of any plane, trimmed to the frame, rdo.rs:2117-2147)
    and every item rdo.rs:2585-2611 reaches with lru_on_skip: units of each plane whose origin is inside the
    trimmed area and that is not a stretch unit (has_restoration_unit(.., false))."""
    planes, xdec, ydec = LAYOUTS[layout]
    lsw = [(unit_size[p] << (xdec if p else 0)) // 64 for p in range(planes)]
    lsh = [(unit_size[p] << (ydec if p else 0)) // 64 for p in range(planes)]
    aw, ah = max(lsw), max(lsh)
    sbw, sbh = (W + 63) // 64, (H + 63) // 64
    areas, items = [], []
    for sby in range(0, sbh, ah):
        for sbx in range(0, sbw, aw):
            a = len(areas)
            areas.append((sbx, sby, min(aw, sbw - sbx), min(ah, sbh - sby)))
            for p in range(planes):
                xd, yd = (xdec, ydec) if p else (0, 0)
                us = unit_size[p]
                cw, ch = (W + (1 << xd >> 1)) >> xd, (H + (1 << yd >> 1)) >> yd
                cols, rows = max(1, (cw + us // 2) // us), max(1, (ch + us // 2) // us)
                for ly in range(ah // lsh[p]):
                    for lx in range(aw // lsw[p]):
                        if lx * lsw[p] >= areas[a][2] or ly * lsh[p] >= areas[a][3]:
                            continue
                        ux, uy = (sbx + lx * lsw[p]) // lsw[p], (sby + ly * lsh[p]) // lsh[p]
                        if ux >= cols or uy >= rows:
                            continue
                        it = np.zeros((), B.LRF_SEARCH_ITEM_DTYPE)
                        it["area"], it["plane"], it["lru_x"], it["lru_y"] = a, p, lx, ly
                        it["none_bits"] = int(rng.integers(0, 200))
                        it["sgr_bits"] = int(rng.integers(0, 400))
                        it["incoming_cost"] = cost
                        it["sgrproj_ref"] = ref if ref is not None else [int(rng.integers(lo, hi + 1))
                                                                          for lo, hi in zip(XQD_MIN, XQD_MAX)]
                        if incoming == "sgr" or (incoming == "mixed" and rng.random() < 0.5):
                            it["incoming"]["type"] = 2
                            it["incoming"]["set"] = int(rng.integers(0, 16))
                            it["incoming"]["xqd"] = [int(rng.integers(lo, hi + 1)) for lo, hi in zip(XQD_MIN, XQD_MAX)]
                        items.append(it)
    return areas, np.array(items, B.LRF_SEARCH_ITEM_DTYPE)


# ---------------------------------------------------------------- oracle wrapper
def lrf_search(lin, src, layout, W, H, bd, unit_size, reduced, areas, items, imp=None,
               dist_scale=(16384,) * 3, lam=0.0):
    """orc_lrf_search; returns (best, cost, changed, xqd (n, 16, 2), err (n, 17), cand_cost (n, 17)) with
    sentinels (xqd 127, err 2**64-1, cost NaN) in slots the search does not reach."""
    L = O.lib()
    f = L.orc_lrf_search
    f.restype = None
    planes, xdec, ydec = LAYOUTS[layout]
    n = len(items)
    vpa, spa = C.c_void_p * 3, C.c_ssize_t * 3
    best = np.zeros(max(n, 1), B.LRF_UNIT_DTYPE)
    cost = np.full(max(n, 1), np.nan)
    changed = np.full(max(n, 1), 7, np.uint8)
    xqd = np.full((max(n, 1), 16, 2), 127, np.int8)
    err = np.full((max(n, 1), 17), np.iinfo(np.uint64).max, np.uint64)
    cc = np.full((max(n, 1), 17), np.nan)
    ar = np.ascontiguousarray(np.array(areas, np.int32).reshape(-1, 4))
    it = np.ascontiguousarray(items)
    us = (C.c_int * 3)(*unit_size, *([0] * (3 - len(unit_size))))
    ds = np.array(dist_scale, np.uint32)
    f(vpa(*[a.ctypes.data for a in lin]), spa(*[a.shape[1] for a in lin]), vpa(*[a.ctypes.data for a in src]),
      spa(*[a.shape[1] for a in src]), C.c_int(lin[0].itemsize), C.c_int(xdec), C.c_int(ydec), C.c_int(W), C.c_int(H),
      C.c_int(bd), us, C.c_int(int(reduced)), C.c_void_p(imp.ctypes.data if imp is not None else None),
      C.c_void_p(ds.ctypes.data), C.c_double(lam), C.c_void_p(ar.ctypes.data), C.c_void_p(it.ctypes.data),
      C.c_size_t(n), C.c_void_p(best.ctypes.data), C.c_void_p(cost.ctypes.data), C.c_void_p(changed.ctypes.data),
      C.c_void_p(xqd.ctypes.data), C.c_void_p(err.ctypes.data), C.c_void_p(cc.ctypes.data))
    return best[:n], cost[:n], changed[:n], xqd[:n], err[:n], cc[:n]


# ---------------------------------------------------------------- the restatement
def spec_subexp_bits(v, low, high, k, r):
    """Bits (Q3) the AV1 specification's decode_signed_subexp_with_ref_bool reads to return v: the subexp
    symbol is found by running the decoder's inverse_recenter mapping over every symbol."""
    mx, rr = high - low, r - low

    def inverse_recenter(r_, x):
        return x if x > 2 * r_ else r_ - ((x + 1) >> 1) if x & 1 else r_ + (x >> 1)

    def decode(sym):
        return inverse_recenter(rr, sym) if (rr << 1) <= mx else mx - 1 - inverse_recenter(mx - 1 - rr, sym)

    sym = [s for s in range(mx) if decode(s) == v - low]
    assert len(sym) == 1
    sym = sym[0]
    bits, i, mk = 0, 0, 0                 # decode_subexp_bool
    while True:
        b2 = k + i - 1 if i else k
        a = 1 << b2
        if mx <= mk + 3 * a:              # subexp_unif_bools: ns(mx - mk)
            n = mx - mk
            w = n.bit_length()
            m = (1 << w) - n
            return (bits + (w - 1 if sym - mk < m else w)) * 8
        bits += 1                         # subexp_more_bools
        if sym >= mk + a:
            i += 1
            mk += a
        else:
            return (bits + b2) * 8


def rate(it, typ, s, xqd):
    if typ == 0:
        return int(it["none_bits"])
    bits = int(it["sgr_bits"]) + (4 << 3)
    for i in range(2):
        if SGR_PARAMS[s][2 * i + 1 if i == 0 else 3] > 0:
            bits += spec_subexp_bits(int(xqd[i]), XQD_MIN[i], XQD_MAX[i] + 1, 4, int(it["sgrproj_ref"][i]))
    return bits


def ab(sums, sqs, n, s, bd):
    """sgrproj_sum_finish over arrays (u32 arithmetic; nothing wraps at 12 bits)"""
    one_over_n = 455 if n == 9 else 164
    sh = bd - 8
    ssq = (sqs + ((1 << 2 * sh) >> 1)) >> (2 * sh)
    sm = (sums + ((1 << sh) >> 1)) >> sh
    p = np.maximum(ssq * n - sm * sm, 0)
    z = (p * s + (1 << 19)) >> 20
    a = np.where(z >= 255, 256, np.where(z == 0, 1, ((z << 8) + z // 2) // (z + 1)))
    b = ((256 - a) * sums * one_over_n + (1 << 11)) >> 12
    return a, b


def rust_round(x):
    f = Fraction(x)
    r = math.floor(abs(f) + Fraction(1, 2))
    return r if f >= 0 else -r


def sat_i32(x):
    if x != x:
        return 0
    return int(max(-2 ** 31, min(2 ** 31 - 1, math.trunc(x) if abs(x) < 2 ** 63 else math.copysign(2 ** 31, x))))


def solve(sums, set_, n):
    h00, h11, h01, c0, c1 = (float(int(v)) for v in sums)
    h00, h01, h11 = h00 / n, h01 / n, h11 / n
    c0, c1 = c0 * (128.0 / n), c1 * (128.0 / n)
    _, s0, _, s1 = SGR_PARAMS[set_]
    if s0 <= 0:
        xq0, xq1 = 0, (0 if h11 == 0. else sat_i32(float(rust_round(c1 / h11))))
    elif s1 <= 0:
        xq0, xq1 = (0 if h00 == 0. else sat_i32(float(rust_round(c0 / h00)))), 0
    else:
        det = fma(h00, h11, -(h01 * h01))
        if det == 0.:
            xq0 = xq1 = 0
        else:
            xq0 = sat_i32(float(rust_round(fma(h11, c0, -(h01 * c1)) / det)))
            xq1 = sat_i32(float(rust_round(fma(h00, c1, -(h01 * c0)) / det)))
    x0 = min(max(xq0, -96), 31)
    x1 = ((128 - x0 - xq1 + 2 ** 31) % 2 ** 32) - 2 ** 31       # i32, wrapping
    return x0, min(max(x1, -32), 95)


def model(lin, src, layout, W, H, bd, unit_size, reduced, areas, items, imp=None, dist_scale=(16384,) * 3, lam=0.0):
    planes, xdec, ydec = LAYOUTS[layout]
    w8 = (W + 7) >> 3
    out = []
    for it in items:
        sbx, sby, sbw, sbh = areas[int(it["area"])]
        p = int(it["plane"])
        xd, yd = (xdec, ydec) if p else (0, 0)
        ax, ay = 64 * sbx, 64 * sby
        crop_w, crop_h = W - ax, H - ay
        aw, ah = (min(crop_w, 64 * sbw) + 7) & ~7, (min(crop_h, 64 * sbh) + 7) & ~7
        A = lin[p][ay >> yd:(ay + ah) >> yd, ax >> xd:(ax + aw) >> xd].astype(np.int64)
        S = src[p][ay >> yd:(ay + ah) >> yd, ax >> xd:(ax + aw) >> xd].astype(np.int64)
        us = unit_size[p]
        lsw, lsh = (us << xd) // 64, (us << yd) // 64
        px, py = int(it["lru_x"]) * lsw * 64 >> xd, int(it["lru_y"]) * lsh * 64 >> yd
        vw, vh = min(us, (crop_w >> xd) - px), min(us, (crop_h >> yd) - py)
        # the unit padded by 3 through setup_integral_image's clip rule
        rows = np.clip(py + np.arange(-3, vh + 3), max(0, py - 2), py + vh - 1)
        cols = np.clip(px + np.arange(-3, vw + 3), 0, px + vw - 1)
        P = A[np.ix_(rows, cols)]
        U = P[3:3 + vh, 3:3 + vw]
        Su = S[py:py + vh, px:px + vw]

        def box(r):                       # sums centred on rows / columns -1 .. vis
            d = 2 * r + 1
            o = 3 - 1 - r
            s = sum(P[o + i:o + i + vh + 2, o + j:o + j + vw + 2] for i in range(d) for j in range(d))
            q = sum(P[o + i:o + i + vh + 2, o + j:o + j + vw + 2] ** 2 for i in range(d) for j in range(d))
            return s, q
        b1, b2 = box(1), box(2)
        nblk_x, nblk_y = lsw * 8, lsh * 8
        bx0, by0 = int(it["lru_x"]) * nblk_x, int(it["lru_y"]) * nblk_y
        bw, bh = 8 >> xd, 8 >> yd

        def plane_error(T):
            e = 0
            for by in range(by0, min(by0 + nblk_y, ah >> 3)):
                for bx in range(bx0, min(bx0 + nblk_x, aw >> 3)):
                    bias = int(imp[(ay >> 3) + by, (ax >> 3) + bx]) if imp is not None else 1 << 14
                    s = S[by * bh:(by + 1) * bh, bx * bw:(bx + 1) * bw]
                    t = T[by * bh:(by + 1) * bh, bx * bw:(bx + 1) * bw]
                    e += mul_u64(bias, cdef_dist(s, t, bd)) if p == 0 else weighted_sse(s, t, bias)
            return mul_u64(dist_scale[p], e)

        inc = it["incoming"]
        best = (int(inc["type"]), int(inc["set"]), int(inc["xqd"][0]), int(inc["xqd"][1]))
        best_cost = float(it["incoming_cost"])
        e = plane_error(A)
        c = fma(lam, rate(it, best[0], best[1], best[2:]) / 8.0, float(e))
        cands = {0: (e, c, None)}
        if best_cost < 0 or c < best_cost:
            best, best_cost = (0, 0, 0, 0), c
        for s in (REDUCED_SETS if reduced else FULL_SETS):
            r0, s0, r1, s1 = SGR_PARAMS[s]
            yy = np.arange(vh)[:, None]
            if s0 > 0:
                a2, bb2 = ab(b2[0], b2[1], 25, s0, bd)      # rows -1 .. vh; only odd unit rows are used

                def w565(m, v):                              # row v of the unit, columns weighted 5 6 5
                    return 5 * (m[v + 1, 0:vw] + m[v + 1, 2:vw + 2]) + 6 * m[v + 1, 1:vw + 1]
                f2 = np.zeros((vh, vw), np.int64)
                for y in range(vh):
                    if y & 1:
                        f2[y] = (w565(a2, y) * U[y] + w565(bb2, y) + (1 << 7)) >> 8
                    else:
                        f2[y] = ((w565(a2, y - 1) + w565(a2, y + 1)) * U[y] + w565(bb2, y - 1) + w565(bb2, y + 1)
                                 + (1 << 8)) >> 9
            else:
                f2 = U[(yy & ~1)[:, 0]] << 4
            if s1 > 0:
                a1, bb1 = ab(b1[0], b1[1], 9, s1, bd)

                def w34(m):
                    return (3 * (m[0:vh, 0:vw] + m[2:, 0:vw] + m[0:vh, 2:] + m[2:, 2:]) +
                            4 * (m[1:vh + 1, 0:vw] + m[0:vh, 1:vw + 1] + m[1:vh + 1, 1:vw + 1] + m[2:, 1:vw + 1] +
                                 m[1:vh + 1, 2:]))
                f1 = (w34(a1) * U + w34(bb1) + (1 << 8)) >> 9
            else:
                f1 = U << 4
            u = U << 4
            sd, e2, e1 = (Su << 4) - u, f2 - u, f1 - u
            sums = [(e2 * e2).sum(), (e1 * e1).sum(), (e1 * e2).sum(), (e2 * sd).sum(), (e1 * sd).sum()]
            xq = solve(sums, s, float(vw) * float(vh))
            w0, w1 = xq
            v = w0 * f2 + w1 * u + (128 - w0 - w1) * f1
            T = np.full_like(A, WORK_FILL)
            T[py:py + vh, px:px + vw] = np.clip((v + (1 << 10)) >> 11, 0, (1 << bd) - 1)
            e = plane_error(T)
            c = fma(lam, rate(it, 2, s, xq) / 8.0, float(e))
            cands[1 + s] = (e, c, xq)
            if c < best_cost:
                best, best_cost = (2, s, w0, w1), c
        i0 = (int(inc["type"]), int(inc["set"]) if inc["type"] == 2 else 0) + \
            ((int(inc["xqd"][0]), int(inc["xqd"][1])) if inc["type"] == 2 else (0, 0))
        ch = best[0] != i0[0] or (best[0] == 2 and best != i0)
        out.append((best, best_cost, ch, cands))
    return out


def check(lin, src, layout, W, H, bd, unit_size, reduced, areas, items, imp=None, dist_scale=(16384,) * 3,
          lam=0.0):
    got = lrf_search(lin, src, layout, W, H, bd, unit_size, reduced, areas, items, imp, dist_scale, lam)
    want = model(lin, src, layout, W, H, bd, unit_size, reduced, areas, items, imp, dist_scale, lam)
    best, cost, changed, xqd, err, cc = got
    for i, (wb, wc, wch, cands) in enumerate(want):
        for c, (e, k, xq) in cands.items():
            assert err[i, c] == e, (i, c, err[i, c], e)
            assert cc[i, c] == k, (i, c)
            if xq is not None:
                assert tuple(xqd[i, c - 1]) == xq, (i, c, xqd[i, c - 1], xq)
        gb = best[i]
        assert (int(gb["type"]), int(gb["set"]), int(gb["xqd"][0]), int(gb["xqd"][1])) == wb or \
            (wb[0] == int(gb["type"]) == int(items[i]["incoming"]["type"]) and gb == items[i]["incoming"]), i
        assert cost[i] == wc and bool(changed[i]) == wch, i
    return got


CONFIGS = [("420", 64, 32), ("420", 128, 64), ("420", 128, 128), ("420", 256, 128), ("422", 64, 64),
           ("444", 64, 64), ("444", 128, 128), ("400", 64, 0), ("400", 256, 0), ("420", 64, 64)]


@pytest.mark.parametrize("layout,uy,uc", CONFIGS)
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_matches_the_restatement(layout, uy, uc, bd):
    rng = np.random.default_rng(hash((layout, uy, uc, bd)) & 0xFFFF)
    W, H = (100, 70) if uy <= 128 else (150, 90)
    lin, src = make_frame(rng, W, H, layout, bd)
    us = [uy, uc, uc][:LAYOUTS[layout][0]]
    areas, items = areas_and_items(rng, W, H, layout, us, incoming="mixed")
    assert len(items)
    imp = rng.integers(1 << 12, 1 << 16, ((H + 7) // 8, (W + 7) // 8)).astype(np.uint32) if bd != 10 else None
    check(lin, src, layout, W, H, bd, us, bd == 10, areas, items, imp, (16384, 20000, 12000), 300.0)


def test_units_with_neighbours_inside_the_area_and_odd_crops():
    """4:2:0 luma 128 / chroma 128: 4x4-superblock areas hold 2x2 luma units with real left / top neighbours;
    an odd frame size leaves vis < unit and crops that are not a multiple of 8."""
    rng = np.random.default_rng(3)
    W, H = 255, 197
    lin, src = make_frame(rng, W, H, "420", 8)
    areas, items = areas_and_items(rng, W, H, "420", [128, 128, 128])
    assert any(it["plane"] == 0 and it["lru_x"] == 1 and it["lru_y"] == 1 for it in items)
    check(lin, src, "420", W, H, 8, [128, 128, 128], False, areas, items, lam=100.0)


@pytest.mark.parametrize("content", ["flat", "extreme"])
def test_flat_and_extreme_content(content):
    rng = np.random.default_rng(4)
    W, H = 64, 64
    for bd in (8, 12):
        lin, src = make_frame(rng, W, H, "444", bd, content)
        areas, items = areas_and_items(rng, W, H, "444", [64, 64, 64])
        _, _, _, xqd, _, _ = check(lin, src, "444", W, H, bd, [64, 64, 64], False, areas, items)
        if content == "flat":
            assert (xqd[:, :, 0] == 0).all()                 # h == 0 / det == 0: (0, 0) -> xqd (0, 128 clamped)
        else:
            assert (xqd[:, :, 0] == -96).any() or (xqd[:, :, 0] == 31).any()


@pytest.mark.parametrize("ref", [(-96, -32), (31, 95), (-96, 95), (31, -32)])
def test_sgrproj_ref_at_range_ends_and_a_sgrproj_incumbent(ref):
    rng = np.random.default_rng(5)
    W, H = 64, 64
    lin, src = make_frame(rng, W, H, "420", 10)
    areas, items = areas_and_items(rng, W, H, "420", [64, 32, 32], incoming="sgr", ref=list(ref))
    check(lin, src, "420", W, H, 10, [64, 32, 32], False, areas, items, lam=500.0)


def test_subexp_counts_match_the_oracle_rates_at_every_value():
    """Every xqd against every reference at the range ends and middle, through the oracle's None rate
    (the incumbent's rate) with no distortion: cost * 8 / lambda is the rate."""
    rng = np.random.default_rng(6)
    W, H = 32, 32
    lin, src = make_frame(rng, W, H, "400", 8, "flat")
    areas, _ = areas_and_items(rng, W, H, "400", [64])
    for s in (0, 10, 14):
        for ref in ((-96, -32), (-32, 31), (31, 95)):
            its = []
            for x0 in range(-96, 32, 9):
                for x1 in range(-32, 96, 11):
                    it = np.zeros((), B.LRF_SEARCH_ITEM_DTYPE)
                    it["incoming"]["type"], it["incoming"]["set"], it["incoming"]["xqd"] = 2, s, [x0, x1]
                    it["sgrproj_ref"], it["incoming_cost"] = ref, -1.0
                    its.append(it)
            its = np.array(its, B.LRF_SEARCH_ITEM_DTYPE)
            _, _, _, _, err, cc = lrf_search(lin, src, "400", W, H, 8, [64], True, areas, its, lam=8.0)
            assert (err[:, 0] == 0).all()
            for it, c in zip(its, cc[:, 0]):
                assert c == rate(it, 2, s, it["incoming"]["xqd"])


def test_carried_cost_nothing_beats_and_exact_ties_change_nothing():
    rng = np.random.default_rng(7)
    W, H = 64, 64
    lin, src = make_frame(rng, W, H, "420", 8)
    areas, items = areas_and_items(rng, W, H, "420", [64, 32, 32], incoming="mixed", cost=0.0)
    best, cost, changed, _, _, cc = check(lin, src, "420", W, H, 8, [64, 32, 32], False, areas, items, lam=10.0)
    assert (changed == 0).all() and (cost == 0.0).all() and (best == items["incoming"]).all()
    # the None candidate's own cost carried in: a tie is not an improvement for the sets (strict <)
    items["incoming_cost"] = cc[:, 0]
    items["incoming"] = np.zeros_like(items["incoming"])
    _, cost2, changed2, _, _, cc2 = check(lin, src, "420", W, H, 8, [64, 32, 32], False, areas, items, lam=10.0)
    ties = (cc2[:, 1:] == cc2[:, :1]).all(axis=1)
    assert (cost2 <= cc[:, 0]).all() and (changed2[ties] == 0).all()


def test_the_work_fill_reaches_only_units_whose_blocks_cross_the_crop():
    """lrf_work outside the visible rect holds B200_LRF_WORK_FILL: changing it changes the set errors of exactly
    the units whose 8x8 blocks cross a crop that is not a multiple of 8 (or 4:2:0's chroma floor)."""
    global WORK_FILL
    rng = np.random.default_rng(8)
    W, H = 131, 67
    lin, src = make_frame(rng, W, H, "420", 8)
    us = [64, 32, 32]
    areas, items = areas_and_items(rng, W, H, "420", us)
    base = model(lin, src, "420", W, H, 8, us, True, areas, items)
    WORK_FILL, saved = 0, WORK_FILL
    try:
        other = model(lin, src, "420", W, H, 8, us, True, areas, items)
    finally:
        WORK_FILL = saved
    for it, a, b in zip(items, base, other):
        sbx, sby, _, _ = areas[int(it["area"])]
        p = int(it["plane"])
        d = 1 if p else 0
        px = (64 * sbx >> d) + int(it["lru_x"]) * us[p]
        py = (64 * sby >> d) + int(it["lru_y"]) * us[p]
        cw, ch = W >> d, H >> d
        bw = 8 >> d
        ex, ey = min(px + us[p], -(-W // 8) * bw), min(py + us[p], -(-H // 8) * bw)
        crosses = ex > min(px + us[p], cw) or ey > min(py + us[p], ch)
        moved = any(a[3][k][0] != b[3][k][0] for k in a[3] if k)
        assert moved == crosses, (p, px, py)
        assert a[3][0] == b[3][0]                            # None never reads lrf_work
