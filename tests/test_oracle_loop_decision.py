"""rdo_loop_decision's pass loop (oracle/loop_decision.c) against an independent Python restatement, value for
value: final indices, unit records, cost bit patterns, written flags, the last C stage's errors and costs, the
working copy and the stage count.  The restatement walks areas and superblocks in the reference's order; its C
stage uses the CDEF pieces of test_oracle_cdef_rdo.py (find_dir, filter_block, the distortions) and its L stage is
test_oracle_lrf_search.py's search model with the incumbents carried; the C stage's Sgrproj branch is restated
here with its own integral image and shares no C code.  Also: an area that stops after its first restoration
stage equals one orc_cdef_rdo pass followed by one orc_lrf_search pass, the stage rules, and traces showing that
the fixtures reach the hard paths.  Holds the ctypes wrapper and the fixture builder the GPU test uses."""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import oracle_lib as O
from tests.test_oracle_cdef_rdo import (LAYOUTS, adjust_strength, cdef_dist, cdef_rdo, filter_block, find_dir, fma,
                                        mul_u64, weighted_sse)
from tests.test_oracle_lrf_search import WORK_FILL, ab, areas_and_items, lrf_search, make_frame
from tests.test_oracle_lrf_search import model as search_model
from tests.test_oracle_lrf_search import rate as lrf_rate
from tests.test_oracle_lrf_spec import SGR_PARAMS


# ---------------------------------------------------------------- fixtures
def units_and_map(rng, W, H, layout, unit_size, skip_frac=0.0):
    """The areas rdo_loop_decision walks, every unit the reference tracks for them (lru_skip drawn with
    probability skip_frac) and the superblock -> unit map of restoration_unit_offset(.., false): -1 where the
    superblock's unit is a stretch of the last unit, which starts in another area."""
    planes, xdec, ydec = LAYOUTS[layout]
    areas, items = areas_and_items(rng, W, H, layout, unit_size)
    units = np.zeros(len(items), B.LOOP_UNIT_DTYPE)
    for f in ("area", "plane", "lru_x", "lru_y", "none_bits", "sgr_bits", "sgrproj_ref"):
        units[f] = items[f]
    units["search"] = rng.random(len(items)) >= skip_frac
    sb_unit = np.full((max(len(areas), 1), 16, 3), -1, np.int32)
    index = {(int(u["area"]), int(u["plane"]), int(u["lru_x"]), int(u["lru_y"])): k for k, u in enumerate(units)}
    for a, (_, _, sbw, sbh) in enumerate(areas):
        for p in range(planes):
            xd, yd = (xdec, ydec) if p else (0, 0)
            lsw, lsh = (unit_size[p] << xd) // 64, (unit_size[p] << yd) // 64
            for sby in range(sbh):
                for sbx in range(sbw):
                    sb_unit[a, sby * 4 + sbx, p] = index.get((a, p, sbx // lsw, sby // lsh), -1)
    return areas, units, sb_unit


# ---------------------------------------------------------------- oracle wrapper
def loop_decision(rec, src, layout, W, H, bd, enable_cdef, damping, cdef_bits, ystr, uvstr, skip8, enable_lrf,
                  unit_size, reduced, areas, units, sb_unit, imp=None, dist_scale=(16384,) * 3, lam=0.0):
    """orc_loop_decision; returns (stages, best_index (n*16 i8), unit (LRF_UNIT_DTYPE), unit_cost, written,
    err (n*16, 8), cost (n*16, 8), work) with sentinels (127, 0xEE bytes, NaN, 7, 2**64-1, NaN, 7) where
    nothing is written."""
    L = O.lib()
    f = L.orc_loop_decision
    f.restype = C.c_int
    planes, xdec, ydec = LAYOUTS[layout]
    n, nu = len(areas), len(units)
    vpa, spa = C.c_void_p * 3, C.c_ssize_t * 3
    work = [np.full_like(r, 7) for r in rec]
    best = np.full(max(n, 1) * 16, 127, np.int8)
    uo = np.frombuffer(np.full(max(nu, 1) * 12, 0xEE, np.uint8).tobytes(), B.LRF_UNIT_DTYPE).copy()
    uc = np.full(max(nu, 1), np.nan)
    wr = np.full(max(nu, 1), 7, np.uint8)
    err = np.full((max(n, 1) * 16, 8), np.iinfo(np.uint64).max, np.uint64)
    cost = np.full((max(n, 1) * 16, 8), np.nan)
    ar = np.ascontiguousarray(np.array(areas, np.int32).reshape(-1, 4))
    un = np.ascontiguousarray(units)
    mp = np.ascontiguousarray(np.asarray(sb_unit, np.int32))
    ys, us = np.array(list(ystr) + [0] * 8, np.uint8)[:8], np.array(list(uvstr) + [0] * 8, np.uint8)[:8]
    usz = (C.c_int * 3)(*unit_size, *([0] * (3 - len(unit_size))))
    ds = np.array(dist_scale, np.uint32)
    stages = f(vpa(*[a.ctypes.data for a in rec]), spa(*[a.shape[1] for a in rec]),
               vpa(*[a.ctypes.data for a in src]), spa(*[a.shape[1] for a in src]),
               vpa(*[a.ctypes.data for a in work]), spa(*[a.shape[1] for a in work]), C.c_int(rec[0].itemsize),
               C.c_int(planes), C.c_int(xdec), C.c_int(ydec), C.c_int(W), C.c_int(H), C.c_int(bd),
               C.c_int(int(enable_cdef)), C.c_int(damping), C.c_int(cdef_bits), C.c_void_p(ys.ctypes.data),
               C.c_void_p(us.ctypes.data), C.c_void_p(skip8.ctypes.data if skip8 is not None else None),
               C.c_int(int(enable_lrf)), usz, C.c_int(int(reduced)),
               C.c_void_p(imp.ctypes.data if imp is not None else None), C.c_void_p(ds.ctypes.data), C.c_double(lam),
               C.c_void_p(ar.ctypes.data), C.c_size_t(n), C.c_void_p(un.ctypes.data), C.c_size_t(nu),
               C.c_void_p(mp.ctypes.data), C.c_void_p(best.ctypes.data), C.c_void_p(uo.ctypes.data),
               C.c_void_p(uc.ctypes.data), C.c_void_p(wr.ctypes.data), C.c_void_p(err.ctypes.data),
               C.c_void_p(cost.ctypes.data))
    return stages, best, uo[:nu], uc[:nu], wr[:nu], err, cost, work


def case(seed, layout, bd, W, H, us, *, enable_cdef=True, enable_lrf=True, skip_frac=0.3, lru_skip=0.2,
         cdef_bits=2, reduced=False, lam=None, imp=True):
    """One fixture: frame, skips, areas, units, map and the call's scalar arguments."""
    rng = np.random.default_rng(seed)
    planes = LAYOUTS[layout][0]
    rec, src = make_frame(rng, W, H, layout, bd)
    w8, h8 = (W + 7) >> 3, (H + 7) >> 3
    skip8 = (rng.random((h8, w8)) < skip_frac).astype(np.uint8)
    areas, units, sb_unit = units_and_map(rng, W, H, layout, us[:planes], lru_skip)
    ystr = [int(v) for v in rng.integers(0, 64, 8)]
    uvstr = [int(v) for v in rng.integers(0, 64, 8)]
    impa = rng.integers(1 << 12, 1 << 16, (h8, w8)).astype(np.uint32) if imp else None
    return dict(rec=rec, src=src, layout=layout, W=W, H=H, bd=bd, enable_cdef=enable_cdef, damping=3 + cdef_bits,
                cdef_bits=cdef_bits, ystr=ystr, uvstr=uvstr, skip8=skip8, enable_lrf=enable_lrf,
                unit_size=us[:planes], reduced=reduced, areas=areas, units=units, sb_unit=sb_unit, imp=impa,
                dist_scale=(16384, 20000, 12000)[:3], lam=float(rng.integers(50, 400)) if lam is None else lam)


CONFIGS = [("420", (64, 32, 32)), ("420", (128, 64, 64)), ("420", (128, 128, 128)), ("420", (256, 128, 128)),
           ("422", (64, 64, 64)), ("444", (64, 64, 64)), ("444", (128, 128, 128)), ("400", (64, 0, 0)),
           ("400", (256, 0, 0))]


def matrix():
    """(id, fixture) pairs: every layout and bit depth, the search's unit configurations, areas of 1x1 .. 4x4
    superblocks with odd crops, CDEF and restoration on and off, all-skip areas and all-lru_skip units."""
    out = []
    for k, (layout, us) in enumerate(CONFIGS):
        for bd in (8, 10, 12):
            W, H = (131, 97) if max(us) <= 128 else (263, 141)
            out.append((f"{layout}-{us[0]}-{bd}", case(k * 31 + bd, layout, bd, W, H, us, reduced=bd == 10)))
    out.append(("cdef-off", case(5, "420", 8, 131, 97, (64, 32, 32), enable_cdef=False)))
    out.append(("lrf-off", case(6, "444", 10, 131, 97, (64, 64, 64), enable_lrf=False)))
    out.append(("all-skip", case(7, "420", 8, 200, 130, (128, 64, 64), skip_frac=1.0)))
    out.append(("all-lru-skip", case(8, "420", 12, 200, 130, (128, 64, 64), lru_skip=1.0)))
    out.append(("neither", case(9, "420", 8, 100, 70, (64, 32, 32), skip_frac=1.0, lru_skip=1.0)))
    out.append(("lambda-0", case(10, "422", 8, 255, 197, (128, 128, 128), lam=0.0, imp=False)))
    # a 4x4-superblock area whose Sgrproj superblocks of the second C stage read neighbours that changed
    out.append(("raster-dependency", case(40, "420", 8, 200, 200, (256, 128, 128), lam=20.0, skip_frac=0.1,
                                          lru_skip=0.0, cdef_bits=3)))
    return out


def run(fx):
    return loop_decision(fx["rec"], fx["src"], fx["layout"], fx["W"], fx["H"], fx["bd"], fx["enable_cdef"],
                         fx["damping"], fx["cdef_bits"], fx["ystr"], fx["uvstr"], fx["skip8"], fx["enable_lrf"],
                         fx["unit_size"], fx["reduced"], fx["areas"], fx["units"], fx["sb_unit"], fx["imp"],
                         fx["dist_scale"], fx["lam"])


# ---------------------------------------------------------------- tests
def test_an_area_that_stops_after_its_first_restoration_stage_is_one_cdef_pass_then_one_search():
    """With a huge lambda and free None symbols no self-guided set beats None (its rate is at least 4 << 3), so
    the first L stage changes nothing: the result is orc_cdef_rdo with each slot's rate = the none_bits of its
    mapped units, then orc_lrf_search on its output."""
    for layout, us in (("420", (128, 64, 64)), ("444", (64, 64, 64)), ("400", (256, 0, 0))):
        fx = case(21, layout, 10, 200, 130, us, lam=1e12, lru_skip=0.0, skip_frac=0.0)
        fx["units"]["none_bits"] = 0
        stages, best, uo, uc, wr, err, cost, work = run(fx)
        assert stages == 2
        planes, xdec, ydec = LAYOUTS[layout]
        n = len(fx["areas"])
        rate = np.zeros(n * 16, np.uint32)
        for s in range(n * 16):
            for p in range(planes):
                u = fx["sb_unit"][s // 16, s % 16, p]
                if u >= 0:
                    rate[s] += fx["units"][u]["none_bits"]
        out = [np.full_like(r, 7) for r in fx["rec"]]
        e2, c2, b2 = cdef_rdo(fx["rec"], fx["src"], out, xdec, ydec, fx["W"], fx["H"], fx["bd"], fx["damping"],
                              fx["cdef_bits"], fx["ystr"], fx["uvstr"], fx["skip8"], fx["imp"], fx["dist_scale"],
                              fx["lam"], [tuple(a) for a in fx["areas"]], rate)
        assert (best == b2).all()
        assert (err == e2).all() and (cost.view(np.uint64) == c2.view(np.uint64)).all()
        for p in range(planes):
            assert (work[p] == out[p]).all()
        items = np.zeros(len(fx["units"]), B.LRF_SEARCH_ITEM_DTYPE)
        for f in ("area", "plane", "lru_x", "lru_y", "none_bits", "sgr_bits", "sgrproj_ref"):
            items[f] = fx["units"][f]
        items["incoming_cost"] = -1.0
        lb, lc, lch, _, _, _ = lrf_search(out, fx["src"], layout, fx["W"], fx["H"], fx["bd"], list(us[:planes]),
                                          False, fx["areas"], items, fx["imp"], fx["dist_scale"], fx["lam"])
        assert (uo["type"] == 0).all() and (lb["type"] == 0).all() and not wr.any() and not lch.any()
        assert (uc.view(np.uint64) == lc.view(np.uint64)).all()


def test_stage_rules_without_cdef_or_restoration_work():
    # no CDEF work: C (counts as a change), L, and a C that changes nothing when L changed something
    fx = case(5, "420", 8, 131, 97, (64, 32, 32), enable_cdef=False)
    stages, best, _, _, wr, err, _, work = run(fx)
    assert stages in (2, 3) and (stages == 3) == bool(wr.any())
    vals = best[[a * 16 + s for a, (_, _, w, h) in enumerate(fx["areas"]) for s in range(16)
                 if s % 4 < w and s // 4 < h]]
    assert set(vals.tolist()) <= {-1, 127} and (vals == -1).any()  # 127: an area with no unit runs no stage
    assert (err == np.iinfo(np.uint64).max).all()
    # no restoration work: exactly one C stage, then the L stage that does nothing
    fx = case(6, "444", 10, 131, 97, (64, 64, 64), enable_lrf=False)
    assert run(fx)[0] == 2
    fx = case(8, "420", 12, 200, 130, (128, 64, 64), lru_skip=1.0)
    assert run(fx)[0] == 2
    # neither: nothing runs and nothing is written
    fx = case(9, "420", 8, 100, 70, (64, 32, 32), skip_frac=1.0, lru_skip=1.0)
    stages, best, uo, uc, wr, err, cost, work = run(fx)
    assert stages == 0 and (best == 127).all() and (wr == 7).all() and all((w == 7).all() for w in work)


# ---------------------------------------------------------------- the restatement
def sgr_superblock(P, px, py, vw, vh, set_, xqd, bd):
    """The C stage's Sgrproj branch for one plane (rdo.rs:2458-2488): setup_integral_image over the superblock's
    visible rect with crop = stripe = vis (lrf.rs:529-627: 4 real columns on the left unless px == 0, 2 real rows
    above clamped to row 0, the last column / row repeated right and below), the box sums taken from an integral
    image, then sgrproj_stripe_filter with the unit's set and xqd.  P: the area's CDEF working copy."""
    rows = np.clip(py + np.arange(-4, vh + 4), max(0, py - 2), py + vh - 1)
    cols = np.clip(px + np.arange(-4, vw + 4), 0, px + vw - 1)
    Q = P[np.ix_(rows, cols)].astype(np.int64)       # pixel (y, x) of the rect at Q[y + 4, x + 4]
    ii = np.zeros((Q.shape[0] + 1, Q.shape[1] + 1), np.int64)
    sq = np.zeros_like(ii)
    ii[1:, 1:] = Q.cumsum(0).cumsum(1)
    sq[1:, 1:] = (Q * Q).cumsum(0).cumsum(1)

    def box(im, r):                                  # (2r+1)^2 sums centred on rows / columns -1 .. vis
        y0, x0, d = 3 - r, 3 - r, 2 * r + 1
        h, w = vh + 2, vw + 2
        return (im[y0 + d:y0 + d + h, x0 + d:x0 + d + w] - im[y0:y0 + h, x0 + d:x0 + d + w]
                - im[y0 + d:y0 + d + h, x0:x0 + w] + im[y0:y0 + h, x0:x0 + w])
    U = Q[4:4 + vh, 4:4 + vw]
    _, s2, _, s1 = SGR_PARAMS[set_]
    if s2 > 0:
        a2, b2 = ab(box(ii, 2), box(sq, 2), 25, s2, bd)

        def w565(m, v):
            return 5 * (m[v + 1, 0:vw] + m[v + 1, 2:vw + 2]) + 6 * m[v + 1, 1:vw + 1]
        f2 = np.zeros((vh, vw), np.int64)
        for y in range(vh):
            if y & 1:
                f2[y] = (w565(a2, y) * U[y] + w565(b2, y) + (1 << 7)) >> 8
            else:
                f2[y] = ((w565(a2, y - 1) + w565(a2, y + 1)) * U[y] + w565(b2, y - 1) + w565(b2, y + 1)
                         + (1 << 8)) >> 9
    else:
        f2 = U[np.arange(vh) & ~1] << 4
    if s1 > 0:
        a1, b1 = ab(box(ii, 1), box(sq, 1), 9, s1, bd)

        def w34(m):
            return (3 * (m[0:vh, 0:vw] + m[2:, 0:vw] + m[0:vh, 2:] + m[2:, 2:]) +
                    4 * (m[1:vh + 1, 0:vw] + m[0:vh, 1:vw + 1] + m[1:vh + 1, 1:vw + 1] + m[2:, 1:vw + 1] +
                         m[1:vh + 1, 2:]))
        f1 = (w34(a1) * U + w34(b1) + (1 << 8)) >> 9
    else:
        f1 = U << 4
    w0, w1 = xqd
    v = w0 * f2 + w1 * (U << 4) + (128 - w0 - w1) * f1
    return np.clip((v + (1 << 10)) >> 11, 0, (1 << bd) - 1)


def model(fx, trace=None):
    """rdo_loop_decision after the deblock (rdo.rs:2104-2745), area by area.  Returns the same tuple as run(fx).
    trace (a list) receives one record per C-stage superblock evaluation: (area, stage, sbx, sby, modes, changed,
    footprint) with modes[p] the plane's branch ('sgr', 'none' or 'plain') and footprint[p] the left 4 columns
    and upper 2 rows a Sgrproj branch reads from the working copy, as they stand when the superblock is reached."""
    rec, src, layout, W, H, bd = fx["rec"], fx["src"], fx["layout"], fx["W"], fx["H"], fx["bd"]
    planes, xdec, ydec = LAYOUTS[layout]
    dec = [(0, 0)] + [(xdec, ydec)] * (planes - 1)
    cs, imp, ds, lam = bd - 8, fx["imp"], fx["dist_scale"], fx["lam"]
    ystr, uvstr, units, sb_unit = fx["ystr"], fx["uvstr"], fx["units"], fx["sb_unit"]
    n, nu = len(fx["areas"]), len(units)
    best = np.full(max(n, 1) * 16, 127, np.int8)
    uo = np.frombuffer(np.full(max(nu, 1) * 12, 0xEE, np.uint8).tobytes(), B.LRF_UNIT_DTYPE).copy()
    uc = np.full(max(nu, 1), np.nan)
    wr = np.full(max(nu, 1), 7, np.uint8)
    err = np.full((max(n, 1) * 16, 8), np.iinfo(np.uint64).max, np.uint64)
    cost = np.full((max(n, 1) * 16, 8), np.nan)
    work_out = [np.full_like(r, 7) for r in rec]
    longest = 0
    for a, (asx, asy, sb_w, sb_h) in enumerate(fx["areas"]):
        ax, ay = 64 * asx, 64 * asy
        crop_w, crop_h = W - ax, H - ay
        aw, ah = (min(crop_w, 64 * sb_w) + 7) >> 3 << 3, (min(crop_h, 64 * sb_h) + 7) >> 3 << 3
        cols, rows = aw >> 3, ah >> 3

        def skip(x, y):
            return bool(fx["skip8"][(ay >> 3) + y, (ax >> 3) + x]) if fx["skip8"] is not None else False

        def blocks(sbx, sby):
            return [(8 * sbx + bx, 8 * sby + by) for by in range(8) for bx in range(8)
                    if 8 * sbx + bx < cols and 8 * sby + by < rows]
        sb_skip = {(x, y): not fx["enable_cdef"] or all(skip(*b) for b in blocks(x, y))
                   for y in range(sb_h) for x in range(sb_w)}
        mine = [u for u in range(nu) if units[u]["area"] == a]
        cdef_work = not all(sb_skip.values())
        lrf_work = bool(fx["enable_lrf"]) and any(units[u]["search"] for u in mine)
        if not cdef_work and not lrf_work:                         # rdo.rs:2267
            continue
        rc = [rec[p][ay >> dec[p][1]:(ay + ah) >> dec[p][1], ax >> dec[p][0]:(ax + aw) >> dec[p][0]].astype(np.int64)
              for p in range(planes)]
        cw = [r.copy() for r in rc]                                # cdef_work = rec_subset.clone()
        S = [src[p][ay >> dec[p][1]:(ay + ah) >> dec[p][1], ax >> dec[p][0]:(ax + aw) >> dec[p][0]].astype(np.int64)
             for p in range(planes)]
        flt = {u: (0, 0, 0, 0) for u in mine}                      # best_lrf: (type, set, xqd0, xqd1)
        fcost = {u: -1.0 for u in mine}
        written = {u: 0 for u in mine}
        bidx = {(x, y): -1 for y in range(sb_h) for x in range(sb_w)}
        dirs = {(x, y): {(bx, by): find_dir(rc[0][8 * (8 * y + by):8 * (8 * y + by) + 8,
                                                   8 * (8 * x + bx):8 * (8 * x + bx) + 8], cs)
                         for by in range(8) for bx in range(8)
                         if 8 * x + bx < cols and 8 * y + by < rows and not skip(8 * x + bx, 8 * y + by)}
                for y in range(sb_h) for x in range(sb_w) if not sb_skip[x, y]}

        def filter_sb(sbx, sby, idx):                              # cdef_filter_superblock into cw
            ys, us = int(ystr[idx]), int(uvstr[idx])
            pri_y, sec_y, pri_uv, sec_uv = ys // 4, ys % 4, us // 4, us % 4
            sec_y += sec_y == 3
            sec_uv += sec_uv == 3
            edges = (4 if sby > 0 else 0) | 8
            for by in range(8):
                if by + 1 >= (ah - 64 * sby) >> 3:
                    edges &= ~8
                edges = (edges & ~1) | (1 if sbx > 0 else 0) | 2
                for bx in range(8):
                    if bx + 1 >= (aw - 64 * sbx) >> 3:
                        edges &= ~2
                    x, y = 8 * sbx + bx, 8 * sby + by
                    if x < cols and y < rows:
                        for p in range(planes):
                            xd, yd = dec[p]
                            bw, bh = 8 >> xd, 8 >> yd
                            px, py = x * bw, y * bh
                            if skip(x, y):
                                cw[p][py:py + bh, px:px + bw] = rc[p][py:py + bh, px:px + bw]
                                continue
                            d, var = dirs[sbx, sby][bx, by]
                            if p == 0:
                                lp, ls, ld, damp = adjust_strength(pri_y << cs, var), sec_y << cs, d if pri_y else 0, \
                                    fx["damping"] + cs
                            else:
                                lp, ls = pri_uv << cs, sec_uv << cs
                                ld = ([7, 0, 2, 4, 5, 6, 6, 6][d] if xd != yd else d) if pri_uv else 0
                                damp = fx["damping"] + cs - 1
                            cw[p][py:py + bh, px:px + bw] = filter_block(rc[p], px, py, bw, bh, lp, ls, ld, damp, cs,
                                                                         edges)
                    edges |= 1
                edges |= 4

        def sb_error(p, T, sbx, sby):                              # rdo_loop_plane_error over one superblock
            xd, yd = dec[p]
            bw, bh = 8 >> xd, 8 >> yd
            e = 0
            for x, y in blocks(sbx, sby):
                bias = int(imp[(ay >> 3) + y, (ax >> 3) + x]) if imp is not None else 1 << 14
                s_, t_ = S[p][y * bh:(y + 1) * bh, x * bw:(x + 1) * bw], T[y * bh:(y + 1) * bh, x * bw:(x + 1) * bw]
                e += mul_u64(bias, cdef_dist(s_, t_, bd)) if p == 0 else weighted_sse(s_, t_, bias)
            return mul_u64(int(ds[p]), e)

        stage = 0
        while True:
            if not stage & 1:                                      # ---- C
                changed = stage == 0
                for sby in range(sb_h):
                    for sbx in range(sb_w):
                        if sb_skip[sbx, sby]:
                            continue
                        slot = a * 16 + sby * 4 + sbx
                        modes, foot = [], []
                        for p in range(planes):
                            u = int(sb_unit[a, sby * 4 + sbx, p])
                            modes.append("plain" if u < 0 or not lrf_work else "sgr" if flt[u][0] == 2 else "none")
                            xd, yd = dec[p]
                            px, py = (64 * sbx) >> xd, (64 * sby) >> yd
                            vw, vh = min(64 >> xd, (crop_w >> xd) - px), min(64 >> yd, (crop_h >> yd) - py)
                            left = cw[p][max(0, py - 2):py + vh, max(0, px - 4):px].copy()
                            up = cw[p][max(0, py - 2):py, max(0, px - 4):px + vw].copy()
                            foot.append((left, up))
                        bc, bi = -1.0, -1
                        for idx in range(1 << fx["cdef_bits"]):
                            filter_sb(sbx, sby, idx)
                            e, r = 0, 0
                            for p in range(planes):
                                u = int(sb_unit[a, sby * 4 + sbx, p])
                                T = cw[p]
                                if modes[p] != "plain":
                                    typ, st, x0, x1 = flt[u]
                                    r += lrf_rate(units[u], typ, st, (x0, x1))
                                    if modes[p] == "sgr":
                                        xd, yd = dec[p]
                                        px, py = (64 * sbx) >> xd, (64 * sby) >> yd
                                        vw = min(64 >> xd, (crop_w >> xd) - px)
                                        vh = min(64 >> yd, (crop_h >> yd) - py)
                                        T = np.full_like(cw[p], WORK_FILL)  # lrf_work outside vis
                                        T[py:py + vh, px:px + vw] = sgr_superblock(cw[p], px, py, vw, vh, st, (x0, x1),
                                                                                   bd)
                                e += sb_error(p, T, sbx, sby)
                            c = fma(lam, r / 8.0, float(e))
                            err[slot, idx], cost[slot, idx] = e, c
                            if bc < 0 or c < bc:
                                bc, bi = c, idx
                        ch = bi != bidx[sbx, sby]
                        if ch:
                            changed = True
                            bidx[sbx, sby] = bi
                        if trace is not None:
                            trace.append((a, stage, sbx, sby, modes, ch, foot))
                        filter_sb(sbx, sby, bi)
            else:                                                  # ---- L
                changed = False
                srch = [u for u in mine if units[u]["search"]] if lrf_work else []
                if srch:
                    lin = [r.copy() for r in rec]
                    for p in range(planes):
                        xd, yd = dec[p]
                        lin[p][ay >> yd:(ay + ah) >> yd, ax >> xd:(ax + aw) >> xd] = cw[p] if cdef_work else rc[p]
                    items = np.zeros(len(srch), B.LRF_SEARCH_ITEM_DTYPE)
                    for k, u in enumerate(srch):
                        for f in ("area", "plane", "lru_x", "lru_y", "none_bits", "sgr_bits", "sgrproj_ref"):
                            items[k][f] = units[u][f]
                        items[k]["incoming"]["type"], items[k]["incoming"]["set"] = flt[u][0], flt[u][1]
                        items[k]["incoming"]["xqd"] = flt[u][2:]
                        items[k]["incoming_cost"] = fcost[u]
                    res = search_model(lin, src, layout, W, H, bd, fx["unit_size"], fx["reduced"], fx["areas"], items,
                                       imp, ds, lam)
                    for u, (b, c, ch, _) in zip(srch, res):
                        fcost[u] = c
                        if ch:
                            flt[u], written[u], changed = b if b[0] == 2 else (0, 0, 0, 0), 1, True
            stage += 1
            if not changed:
                break
        longest = max(longest, stage)
        for (x, y), b in bidx.items():
            best[a * 16 + y * 4 + x] = b
        for u in mine:
            t_, s_, x0, x1 = flt[u]
            uo[u] = np.zeros((), B.LRF_UNIT_DTYPE)
            uo[u]["type"], uo[u]["set"], uo[u]["xqd"] = t_, s_, (x0, x1)
            uc[u], wr[u] = fcost[u], written[u]
        for p in range(planes):
            xd, yd = dec[p]
            work_out[p][ay >> yd:(ay + ah) >> yd, ax >> xd:(ax + aw) >> xd] = cw[p] if cdef_work else rc[p]
    return longest, best, uo[:nu], uc[:nu], wr[:nu], err, cost, work_out


def same(got, want):
    g_st, g_b, g_uo, g_uc, g_wr, g_e, g_c, g_w = got
    w_st, w_b, w_uo, w_uc, w_wr, w_e, w_c, w_w = want
    assert g_st == w_st
    assert (g_b == w_b).all()
    assert (g_uo.view(np.uint8) == w_uo.view(np.uint8)).all()
    assert (g_uc.view(np.uint64) == w_uc.view(np.uint64)).all()
    assert (g_wr == w_wr).all()
    assert (g_e == w_e).all() and (g_c.view(np.uint64) == w_c.view(np.uint64)).all()
    for g, w in zip(g_w, w_w):
        assert (g.astype(np.int64) == w).all()


MATRIX = matrix()


@pytest.mark.parametrize("name", [m[0] for m in MATRIX])
def test_matches_the_restatement(name):
    fx = dict(MATRIX)[name]
    same(run(fx), model(fx))


def test_the_fixtures_reach_the_hard_paths():
    """Traced from the restatement over the matrix: some area runs three or more stages; some C stage after the
    first measures a superblock through the Sgrproj branch and changes its index; and in some such evaluation
    the left columns or upper rows the integral image reads from the working copy differ from what they held at
    the previous C stage, so the raster-order dependency on this pass's winners is exercised, not only present."""
    deep, sgr_change, moved = 0, False, False
    for _, fx in MATRIX:
        trace = []
        deep = max(deep, model(fx, trace)[0])
        prev = {(a, st, x, y): foot for a, st, x, y, _, _, foot in trace}
        for a, st, x, y, modes, ch, foot in trace:
            if st < 2 or "sgr" not in modes:
                continue
            sgr_change |= ch
            before = prev.get((a, st - 2, x, y))
            for p, f in enumerate(foot):
                # the same pixels when the previous C stage reached this superblock
                if modes[p] == "sgr" and before is not None and \
                        any(not np.array_equal(n_, o_) for n_, o_ in zip(f, before[p])):
                    moved = True
    assert deep >= 3
    assert sgr_change
    assert moved
