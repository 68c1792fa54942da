"""The CDEF pass of rdo_loop_decision (oracle/cdef_rdo.c) against an independent Python restatement of
rav1e src/rdo.rs:2027-2093 + 2185-2205 + 2377-2565 (RestorationFilter::None) and cdef.rs:340-570.

The restatement works on the area's scratch copy the way the reference does (no padding, edge flags
built by cdef_filter_superblock's loop) and shares no code with the oracle: the direction search,
the filter, cdef_dist_kernel, get_weighted_sse and the scale arithmetic are restated here from the
reference.  Also holds the ctypes wrapper of orc_cdef_rdo the GPU test uses."""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O

DEFAULT_STRENGTHS = [0, 4, 9, 13, 22, 31, 43, 55]    # encoder.rs:897-916
LAYOUTS = {"400": (1, 1, 1), "420": (3, 1, 1), "422": (3, 1, 0), "444": (3, 0, 0)}


# ---------------------------------------------------------------- inputs
def random_image(rng, w, h, bd, smooth=True):
    maxv = (1 << bd) - 1
    img = rng.integers(0, maxv + 1, (h + 8, w + 8)).astype(np.float64)
    if smooth:
        k = np.ones(3) / 3.0
        img = np.apply_along_axis(lambda r: np.convolve(r, k, mode="same"), 1, img)
        img = np.apply_along_axis(lambda c: np.convolve(c, k, mode="same"), 0, img)
        img += rng.normal(0, maxv / 40.0, img.shape)
    return np.clip(np.rint(img[4:4 + h, 4:4 + w]), 0, maxv).astype(np.uint8 if bd == 8 else np.uint16)


def make_frame(rng, width, height, layout, bd, flat=False):
    """(rec, src) lists of plane images covering the frame rounded up to 8 luma pixels."""
    planes, xdec, ydec = LAYOUTS[layout]
    w8, h8 = (width + 7) & ~7, (height + 7) & ~7
    rec, src = [], []
    for p in range(planes):
        w, h = (w8 >> xdec, h8 >> ydec) if p else (w8, h8)
        s = random_image(rng, w, h, bd)
        if flat:
            s[:] = 1 << (bd - 1)
            r = s.copy()
        else:
            r = np.clip(s.astype(np.int32) + rng.integers(-(4 << (bd - 8)), (4 << (bd - 8)) + 1, s.shape), 0,
                        (1 << bd) - 1).astype(s.dtype)
        rec.append(np.ascontiguousarray(r))
        src.append(np.ascontiguousarray(s))
    return rec, src


# ---------------------------------------------------------------- oracle wrapper
def cdef_rdo(rec, src, out, xdec, ydec, width, height, bd, damping, cdef_bits, ystr, uvstr, skip8=None, imp=None,
             dist_scale=(16384, 16384, 16384), lam=0.0, areas=(), rate=None):
    """orc_cdef_rdo over numpy planes (pixel (0,0) = element [0, 0]).  `out`: list of arrays written in
    place, or None.  Returns (err (n*16, 8) u64, cost (n*16, 8) f64, best (n*16,) i8); unwritten entries
    hold their sentinels (err 2**64-1, cost NaN, best 127)."""
    L = O.lib()
    f = L.orc_cdef_rdo
    f.restype = None
    planes = len(rec)
    vpa = C.c_void_p * 3
    spa = C.c_ssize_t * 3
    n = len(areas)
    err = np.full((max(n, 1) * 16, 8), np.iinfo(np.uint64).max, np.uint64)
    cost = np.full((max(n, 1) * 16, 8), np.nan)
    best = np.full(max(n, 1) * 16, 127, np.int8)
    ar = np.ascontiguousarray(np.array(areas, np.int32).reshape(-1, 4))
    ys = np.array(ystr, np.uint8)
    us = np.array(uvstr, np.uint8)
    ds = np.array(dist_scale, np.uint32)
    f(vpa(*[r.ctypes.data for r in rec]), spa(*[r.shape[1] for r in rec]),
      vpa(*[s.ctypes.data for s in src]), spa(*[s.shape[1] for s in src]),
      vpa(*[o.ctypes.data for o in out]) if out is not None else None,
      spa(*[o.shape[1] for o in out]) if out is not None else None,
      C.c_int(rec[0].itemsize), C.c_int(planes), C.c_int(xdec), C.c_int(ydec), C.c_int(width), C.c_int(height),
      C.c_int(bd), C.c_int(damping), C.c_int(cdef_bits), C.c_void_p(ys.ctypes.data), C.c_void_p(us.ctypes.data),
      C.c_void_p(skip8.ctypes.data if skip8 is not None else None),
      C.c_void_p(imp.ctypes.data if imp is not None else None), C.c_void_p(ds.ctypes.data), C.c_double(lam),
      C.c_void_p(ar.ctypes.data), C.c_size_t(n), C.c_void_p(rate.ctypes.data if rate is not None else None),
      C.c_void_p(err.ctypes.data), C.c_void_p(cost.ctypes.data), C.c_void_p(best.ctypes.data))
    return err, cost, best


# ---------------------------------------------------------------- the Python restatement
DIV = [0, 840, 420, 280, 210, 168, 140, 120, 105]                      # cdef.rs:54
CDEF_DIRS = [[(-1, 1), (-2, 2)], [(0, 1), (-1, 2)], [(0, 1), (0, 2)], [(0, 1), (1, 2)],
             [(1, 1), (2, 2)], [(1, 0), (2, 1)], [(1, 0), (2, 0)], [(1, 0), (2, -1)]]  # cdef.rs:242-251 (dy, dx)
AREA_DIV = [round(16384 / (1 + x)) for x in range(64)]                 # dist.rs:288-297


def find_dir(blk, coeff_shift):                                        # cdef.rs:84-143
    cost = [0] * 8
    partial = [[0] * 15 for _ in range(8)]
    for i in range(8):
        for j in range(8):
            x = (int(blk[i, j]) >> coeff_shift) - 128
            partial[0][i + j] += x
            partial[1][i + j // 2] += x
            partial[2][i] += x
            partial[3][3 + i - j // 2] += x
            partial[4][7 + i - j] += x
            partial[5][3 - i // 2 + j] += x
            partial[6][j] += x
            partial[7][i // 2 + j] += x
    for i in range(8):
        cost[2] += partial[2][i] ** 2
        cost[6] += partial[6][i] ** 2
    cost[2] *= DIV[8]
    cost[6] *= DIV[8]
    for i in range(7):
        cost[0] += (partial[0][i] ** 2 + partial[0][14 - i] ** 2) * DIV[i + 1]
        cost[4] += (partial[4][i] ** 2 + partial[4][14 - i] ** 2) * DIV[i + 1]
    cost[0] += partial[0][7] ** 2 * DIV[8]
    cost[4] += partial[4][7] ** 2 * DIV[8]
    for i in (1, 3, 5, 7):
        for j in range(5):
            cost[i] += partial[i][3 + j] ** 2
        cost[i] *= DIV[8]
        for j in range(3):
            cost[i] += (partial[i][j] ** 2 + partial[i][10 - j] ** 2) * DIV[2 * j + 2]
    best = max(range(8), key=lambda d: (cost[d], -d))                  # first maximum
    return best, (cost[best] - cost[(best + 4) & 7]) >> 10


def adjust_strength(strength, var):                                    # cdef.rs:315-322
    i = min((var >> 6).bit_length() - 1, 12) if (var >> 6) != 0 else 0
    return (strength * (4 + i) + 8) >> 4 if var != 0 else 0


def constrain(diff, threshold, damping):                               # cdef.rs:146-159 (vectorised)
    if threshold == 0:
        return np.zeros_like(diff)
    shift = max(0, damping - (threshold.bit_length() - 1))
    mag = np.clip(threshold - (np.abs(diff) >> shift), 0, None)
    mag = np.minimum(mag, np.abs(diff))
    return np.sign(diff) * mag


def filter_block(inp, x0, y0, bw, bh, pri, sec, direction, damping, coeff_shift, edges):
    pri, sec, damping = int(pri), int(sec), int(damping)
    """cdef_filter_block (cdef.rs:198-298) of the bw x bh block at (x0, y0) of the scratch plane `inp`."""
    big = 0x8000
    tmp = np.full((bh + 4, bw + 4), big, np.int64)
    xa = -2 if edges & 1 else 0
    xb = bw + (2 if edges & 2 else 0)
    ya = -2 if edges & 4 else 0
    yb = bh + (2 if edges & 8 else 0)
    tmp[ya + 2:yb + 2, xa + 2:xb + 2] = inp[y0 + ya:y0 + yb, x0 + xa:x0 + xb]
    x = tmp[2:2 + bh, 2:2 + bw]
    taps = (3, 3) if (pri >> coeff_shift) & 1 else (4, 2)

    def tap(dy, dx):
        return tmp[2 + dy:2 + dy + bh, 2 + dx:2 + dx + bw]
    total = np.zeros_like(x)
    mx, mn = x.copy(), x.copy()
    for k in range(2):
        for dirn, strength, weight in ((direction, pri, taps[k]), ((direction + 2) & 7, sec, (2, 1)[k]),
                                       ((direction + 6) & 7, sec, (2, 1)[k])):
            dy, dx = CDEF_DIRS[dirn][k]
            for s in (tap(dy, dx), tap(-dy, -dx)):
                total += weight * constrain(s - x, strength, damping)
                mx = np.maximum(mx, np.where(s != big, s, mx))
                mn = np.minimum(mn, s)
    v = x + ((8 + total - (total < 0)) >> 4)
    return np.clip(v, mn, mx)


def cdef_dist(s, d, bd):                                               # dist.rs:302-372, activity.rs:107-186
    s = s.astype(np.uint64)
    d = d.astype(np.uint64)
    m = 0xFFFFFFFF
    sum_s, sum_d = int(s.sum()) & m, int(d.sum()) & m
    sum_s2, sum_d2, sum_sd = int((s * s).sum()) & m, int((d * d).sum()) & m, int((s * d).sum()) & m
    sse = (sum_d2 + sum_s2 - 2 * sum_sd) & m
    div = AREA_DIV[63]
    svar = max(sum_s2 - (((sum_s * sum_s * div) + (1 << 13)) >> 14 & m), 0)
    dvar = max(sum_d2 - (((sum_d * sum_d * div) + (1 << 13)) >> 14 & m), 0)
    svar = (svar * div + (1 << 7)) >> 8 & m
    dvar = (dvar * div + (1 << 7)) >> 8 & m
    cs = bd - 8
    sv, dv = svar >> (2 * cs), dvar >> (2 * cs)
    c1, c2, c3 = 3355, 16128, 12338
    ratio = (((c1 << 15) // c3) + 1) >> 1
    x = c1 * c1 + sv * dv
    k = (x.bit_length() - 1) >> 1
    sh = 2 * k - 14
    t = (x >> sh if sh > 0 else x << -sh) & 0xFFFF
    shift = 14 + ((sh + 16) >> 1)
    n = t - 32768
    norm = (23557 + ((n * (-13490 + ((n * 6711) >> 15))) >> 15)) & 0xFFFF
    return (sse * (((ratio * (sv + dv + c2)) * norm) >> 14)) >> shift


def weighted_sse(s, d, bias):                                          # dist.rs:234-283 with one bias per 4x4
    diff = (s.astype(np.int64) - d.astype(np.int64)) ** 2
    acc = 0
    for cy in range(0, s.shape[0], 4):
        for cx in range(0, s.shape[1], 4):
            acc += (int(diff[cy:cy + 4, cx:cx + 4].sum()) * bias + 128) >> 8
    return (acc + 32) // 64


def mul_u64(scale, dist):                                              # DistortionScale::mul_u64, rdo.rs:616
    return (scale * dist + (1 << 13)) >> 14


def model(rec, src, xdec, ydec, width, height, bd, damping, cdef_bits, ystr, uvstr, skip8=None, imp=None,
          dist_scale=(16384,) * 3, lam=0.0, areas=(), rate=None, out=None):
    planes = len(rec)
    cs = bd - 8
    w8 = (width + 7) >> 3
    res = {}
    for a, (asx, asy, sb_w, sb_h) in enumerate(areas):
        ax, ay = 64 * asx, 64 * asy
        pixel_w, pixel_h = min(width - ax, sb_w * 64), min(height - ay, sb_h * 64)     # rdo.rs:2152-2157
        aw, ah = (pixel_w + 7) >> 3 << 3, (pixel_h + 7) >> 3 << 3
        dec = [(0, 0)] + [(xdec, ydec)] * (planes - 1)
        rc = [rec[p][ay >> dec[p][1]:(ay + ah) >> dec[p][1], ax >> dec[p][0]:(ax + aw) >> dec[p][0]].astype(np.int64)
              for p in range(planes)]                                  # scratch_copy
        work = [r.copy() for r in rc]                                  # cdef_work
        cols, rows = aw >> 3, ah >> 3

        def skip(x, y):
            return bool(skip8[(ay >> 3) + y, (ax >> 3) + x]) if skip8 is not None else False

        def analyze(sbx, sby):                                         # cdef_analyze_superblock
            dirs = {}
            for by in range(8):
                for bx in range(8):
                    x, y = 8 * sbx + bx, 8 * sby + by
                    if x < cols and y < rows and not skip(x, y):
                        dirs[bx, by] = find_dir(rc[0][8 * y:8 * y + 8, 8 * x:8 * x + 8], cs)
            return dirs

        def filter_sb(sbx, sby, idx, dirs):                            # cdef_filter_superblock
            ys, us = int(ystr[idx]), int(uvstr[idx])
            pri_y, sec_y, pri_uv, sec_uv = ys // 4, ys % 4, us // 4, us % 4
            sec_y += sec_y == 3
            sec_uv += sec_uv == 3
            xavail, yavail = aw - 64 * sbx, ah - 64 * sby
            edges = (4 if sby > 0 else 0) | 8
            for by in range(8):
                if by + 1 >= yavail >> 3:
                    edges &= ~8
                edges = (edges & ~1) | (1 if sbx > 0 else 0) | 2
                for bx in range(8):
                    if bx + 1 >= xavail >> 3:
                        edges &= ~2
                    x, y = 8 * sbx + bx, 8 * sby + by
                    if x < cols and y < rows:
                        for p in range(planes):
                            xd, yd = dec[p]
                            bw, bh = 8 >> xd, 8 >> yd
                            px, py = x * bw, y * bh
                            if skip(x, y):
                                work[p][py:py + bh, px:px + bw] = rc[p][py:py + bh, px:px + bw]
                                continue
                            d, var = dirs[bx, by]
                            if p == 0:
                                lp, ls, ld = adjust_strength(pri_y << cs, var), sec_y << cs, d if pri_y else 0
                                damp = damping + cs
                            else:
                                lp, ls = pri_uv << cs, sec_uv << cs
                                ld = ([7, 0, 2, 4, 5, 6, 6, 6][d] if xd != yd else d) if pri_uv else 0
                                damp = damping + cs - 1
                            work[p][py:py + bh, px:px + bw] = filter_block(rc[p], px, py, bw, bh, lp, ls, ld, damp,
                                                                           cs, edges)
                    edges |= 1
                edges |= 4

        for sby in range(sb_h):
            for sbx in range(sb_w):
                slot = a * 16 + sby * 4 + sbx
                blocks = [(8 * sbx + bx, 8 * sby + by) for by in range(8) for bx in range(8)
                          if 8 * sbx + bx < cols and 8 * sby + by < rows]
                if all(skip(x, y) for x, y in blocks):
                    res[slot] = (None, None, -1)
                    continue
                dirs = analyze(sbx, sby)
                errs, costs, best, best_cost = [], [], -1, -1.0
                for idx in range(1 << cdef_bits):
                    filter_sb(sbx, sby, idx, dirs)
                    err = 0
                    for p in range(planes):                            # rdo_loop_plane_error
                        xd, yd = dec[p]
                        bw, bh = 8 >> xd, 8 >> yd
                        pe = 0
                        for x, y in blocks:
                            bias = int(imp[(ay >> 3) + y, (ax >> 3) + x]) if imp is not None else 16384
                            s = src[p][(ay >> yd) + y * bh:(ay >> yd) + y * bh + bh,
                                       (ax >> xd) + x * bw:(ax >> xd) + x * bw + bw]
                            t = work[p][y * bh:y * bh + bh, x * bw:x * bw + bw]
                            pe += mul_u64(bias, cdef_dist(s, t, bd)) if p == 0 else weighted_sse(s, t, bias)
                        err += mul_u64(int(dist_scale[p]), pe)
                    r = int(rate[slot]) if rate is not None else 0
                    cost = fma(lam, r / 8.0, err)                # compute_rd_cost, rdo.rs:718-723
                    errs.append(err)
                    costs.append(cost)
                    if best_cost < 0 or cost < best_cost:
                        best_cost, best = cost, idx
                res[slot] = (errs, costs, best)
                filter_sb(sbx, sby, best, dirs)
        if out is not None:
            for p in range(planes):
                xd, yd = dec[p]
                out[p][ay >> yd:(ay + ah) >> yd, ax >> xd:(ax + aw) >> xd] = work[p]
    return res


def fma(a, b, c):
    """IEEE fused multiply-add in exact rational arithmetic, rounded once."""
    from fractions import Fraction
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def check(rec, src, layout, width, height, bd, damping, cdef_bits, ystr, uvstr, areas, skip8=None, imp=None,
          dist_scale=(16384,) * 3, lam=0.0, rate=None):
    planes, xdec, ydec = LAYOUTS[layout]
    out = [np.full_like(r, 7) for r in rec]
    err, cost, best = cdef_rdo(rec, src, out, xdec, ydec, width, height, bd, damping, cdef_bits, ystr, uvstr, skip8,
                               imp, dist_scale, lam, areas, rate)
    m_out = [np.full(r.shape, 7, np.int64) for r in rec]
    want = model(rec, src, xdec, ydec, width, height, bd, damping, cdef_bits, ystr, uvstr, skip8, imp, dist_scale,
                 lam, areas, rate, m_out)
    n = 1 << cdef_bits
    for slot, (errs, costs, b) in want.items():
        assert best[slot] == b, (slot, best[slot], b)
        if b >= 0:
            assert err[slot, :n].tolist() == errs, (slot, err[slot, :n], errs)
            assert [c.hex() for c in cost[slot, :n].tolist()] == [c.hex() for c in costs]
    for p in range(planes):
        assert (out[p].astype(np.int64) == m_out[p]).all(), f"plane {p}"
    return err, cost, best, out


# ---------------------------------------------------------------- tests
@pytest.mark.parametrize("layout,bd", [("420", 8), ("444", 10), ("422", 12), ("400", 8)])
@pytest.mark.parametrize("cdef_bits", [0, 1, 2, 3])
def test_areas_next_to_each_other(layout, bd, cdef_bits):
    rng = np.random.default_rng(cdef_bits * 7 + bd)
    W, H = 200, 136                                  # partial superblocks at the right and bottom
    rec, src = make_frame(rng, W, H, layout, bd)
    ystr = [int(v) for v in rng.integers(0, 64, 8)]
    uvstr = [int(v) for v in rng.integers(0, 64, 8)]
    areas = [(0, 0, 2, 1), (2, 0, 2, 2), (0, 1, 1, 2), (1, 1, 1, 1)]   # 4x3 superblocks, every one covered
    check(rec, src, layout, W, H, bd, 3 + cdef_bits, cdef_bits, ystr, uvstr, areas)


@pytest.mark.parametrize("layout", ["420", "422", "444"])
def test_skips_bias_dist_scale_and_rates(layout):
    rng = np.random.default_rng(11)
    W, H = 252, 130                                  # visible width not a multiple of 8
    bd = 10
    rec, src = make_frame(rng, W, H, layout, bd)
    w8, h8 = (W + 7) >> 3, (H + 7) >> 3
    skip8 = (rng.random((h8, w8)) < 0.4).astype(np.uint8)
    skip8[0:8, 0:8] = 1                              # superblock (0, 0): all skip
    skip8[8:16, 8:16] = 0                            # superblock (1, 1): no skip
    imp = rng.integers(4000, 60000, (h8, w8)).astype(np.uint32)
    rate = rng.integers(0, 4000, 16 * 3).astype(np.uint32)
    ystr = DEFAULT_STRENGTHS
    areas = [(0, 0, 2, 2), (2, 0, 2, 3), (0, 2, 2, 1)]
    err, cost, best, _ = check(rec, src, layout, W, H, bd, 5, 3, ystr, ystr[::-1], areas, skip8, imp,
                               (20000, 9000, 31000), 1234.5, rate)
    assert best[0] == -1 and best[5] >= 0


def test_one_4x4_area_and_flat_ties_take_the_first_index():
    rng = np.random.default_rng(5)
    W, H = 256, 256
    rec, src = make_frame(rng, W, H, "420", 8)
    check(rec, src, "420", W, H, 8, 4, 0, [37] * 8, [22] * 8, [(0, 0, 4, 4)])
    flat_rec, flat_src = make_frame(rng, 128, 64, "420", 8, flat=True)
    err, cost, best, out = check(flat_rec, flat_src, "420", 128, 64, 8, 3, 3, DEFAULT_STRENGTHS,
                                 DEFAULT_STRENGTHS, [(0, 0, 2, 1)])
    assert (best[:2] == 0).all() and (cost[0] == cost[0, 0]).all()   # every index ties: the first wins


def test_area_relative_edges_differ_from_a_frame_relative_filter():
    """At the border between two areas the reference filters each area's copy: no pixel of the
    neighbouring area is available.  A frame-relative filter (orc_cdef_filter_plane) sees them."""
    rng = np.random.default_rng(3)
    W, H = 128, 64
    rec, src = make_frame(rng, W, H, "400", 8)
    y = 4 * 9 + 3                                    # pri 9, sec 3 -> 4
    outs = []
    for areas in ([(0, 0, 1, 1), (1, 0, 1, 1)], [(0, 0, 2, 1)]):
        _, _, best, out = check(rec, src, "400", W, H, 8, 6, 0, [y] * 8, [y] * 8, areas)
        outs.append(out[0])
    dirs, var = O.cdef_analyze_frame(rec[0], 8)
    frame = O.cdef_filter_plane(rec[0], 0, 0, 0, W, H, 8, 6, None, dirs, var, np.full(2, y, np.uint8))
    assert (outs[1] == frame).all()                  # one area over the whole frame = the frame filter
    assert not (outs[0][:, 62:66] == frame[:, 62:66]).all()   # two areas differ at their shared border
    assert (outs[0][:, :60] == frame[:, :60]).all() and (outs[0][:, 68:] == frame[:, 68:]).all()
