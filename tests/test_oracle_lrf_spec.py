"""orc_lrf_filter_frame (lrf_filter_frame as rav1e runs it) against an independent model of the AV1
specification's loop restoration process, pixel for pixel over every plane's crop.

The model is written from the specification, not from lrf.rs.  It works per pixel, vectorised: the pixel's
4x4 luma block (row, col) gives the stripe (StripeNum = (row * 4 + 8) / 64, StripeStartY = (-8 + StripeNum *
64) >> subY, StripeEndY = StripeStartY + (64 >> subY) - 1) and the unit (unitRow = Min(unitRows - 1, ((row *
4 + 8) >> subY) / unitSize), unitCol = Min(unitCols - 1, ((col * 4) >> subX) / unitSize), with
count_units_in_frame for unitRows / unitCols) as loop_restore_block derives them.  get_source_sample clamps
to the plane, then above the stripe reads the pre-CDEF (deblocked) frame no higher than StripeStartY - 2,
below it the deblocked frame no lower than StripeEndY + 2, and inside it the CDEF output.  The Wiener filter
uses the rounding variables derivation with isCompound = 0 (InterRound0 = 3, or 5 at 12 bit; InterRound1 =
11, or 9 at 12 bit), its offset / limit clip of the intermediate and Clip1.  The self-guided filter runs
box_filter_process with Sgr_Params (r, s per pass): A and B from box sums of radius r around each of the
pixel's 3x3 neighbours, Round2 by 2 * (BitDepth - 8) and BitDepth - 8, p, z, a2 and oneOverN; pass 0
weighs only odd rows (6 / 5, shift 4 on odd rows), pass 1 every row (4 / 3); then the projection with
w0 / w1 / w2, where a pass with r == 0 contributes u.  Unit sizes are the ones the specification allows
(luma 64..256, chroma the luma size or, in 4:2:0 only, half of it).

Where rav1e and the specification part, the oracle follows rav1e, and each place is shown and confined:
  1. Wiener at the frame's top and bottom: rav1e reads the deblocked frame's row 0 for the 3 rows above the
     frame and row crop_h - 1 for rows below its last stripe; the specification reads the CDEF output there.
     Only pixels of Wiener units within 3 rows of the top or bottom of the crop can differ.
  2. enable_cdef == 0: rav1e leaves Sgrproj units as the CDEF output; the specification filters them.
  3. crop_h < 56 >> ydec: rav1e's Sgrproj units also write stripe 0's rows at and below crop_h; the crop
     itself still equals the specification.
  4. (Found by this model.)  A Sgrproj set whose radius-2 pass is off (sets 10-13) with xqd[0] != 0: rav1e
     uses the even row's pixel for the odd row below it in the w0 term (lrf.rs:740-749 shares f_r2_0), the
     specification the pixel itself.  Only odd rows of such units differ.  rav1e's own search never signals
     it (sgrproj_solve sets xqd[0] = 0 when s_r2 == 0, lrf.rs:1059-1066, as the bitstream infers it).
The model carries 1 and 4 as switches; with them on it must equal the oracle everywhere in the crop, and
with them off it may differ only where stated.
"""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import oracle_lib as O

LAYOUTS = {"400": (1, 1, 1), "420": (3, 1, 1), "422": (3, 1, 0), "444": (3, 0, 0)}
PAD = 8
# Sgr_Params: r0, s0, r1, s1
SGR_PARAMS = [(2, 140, 1, 3236), (2, 112, 1, 2158), (2, 93, 1, 1618), (2, 80, 1, 1438), (2, 70, 1, 1295),
              (2, 58, 1, 1177), (2, 47, 1, 1079), (2, 37, 1, 996), (2, 30, 1, 925), (2, 25, 1, 863),
              (0, -1, 1, 2589), (0, -1, 1, 1618), (0, -1, 1, 1177), (0, -1, 1, 925), (2, 56, 0, -1),
              (2, 22, 0, -1)]
TAPS_MIN, TAPS_MAX = (-5, -23, -17), (10, 8, 46)
XQD_MIN, XQD_MAX = (-96, -32), (31, 95)


def round2(x, n):
    """Round2; n may be an array of positive shifts"""
    if np.isscalar(n) and n == 0:
        return x
    return (x + (np.int64(1) << (n - 1))) >> n


def dec(p, layout):
    _, xdec, ydec = LAYOUTS[layout]
    return (xdec, ydec) if p else (0, 0)


def crop(W, H, p, layout):
    xd, yd = dec(p, layout)
    return round2(W, xd), round2(H, yd)


def count_units(us, size):
    return max((size + (us >> 1)) // us, 1)


# ---------------------------------------------------------------- frames and units
def make_frame(rng, W, H, layout, bd, content="random"):
    """(cdeffed, deblocked): padded planes, PAD pixels all round, at least stripe 0's rows tall."""
    n = LAYOUTS[layout][0]
    dt = np.uint8 if bd == 8 else np.uint16
    mx = (1 << bd) - 1
    cd, db = [], []
    for p in range(n):
        cw, ch = crop(W, H, p, layout)
        shape = (max(ch, 56 >> dec(p, layout)[1]) + 2 * PAD, cw + 2 * PAD)
        if content == "random":
            a, b = rng.integers(0, mx + 1, shape), rng.integers(0, mx + 1, shape)
        elif content == "flat":
            a, b = np.full(shape, int(rng.integers(0, mx + 1))), np.full(shape, int(rng.integers(0, mx + 1)))
        elif content == "edges":  # hard 0 / max blocks with small noise: extremes and steep edges
            yy, xx = np.mgrid[0:shape[0], 0:shape[1]]
            blk = ((yy // int(rng.integers(2, 9))) + (xx // int(rng.integers(2, 9)))) % 2
            a = np.clip(blk * mx + rng.integers(-3, 4, shape) * (1 << (bd - 8)), 0, mx)
            b = np.clip(a + rng.integers(-8, 9, shape) * (1 << (bd - 8)), 0, mx)
        else:  # smooth ramps plus noise: the filters' mid range
            yy, xx = np.mgrid[0:shape[0], 0:shape[1]]
            a = (np.sin(xx / 7.0 + p) + np.cos(yy / 5.0)) * mx / 4 + mx / 2 + rng.normal(0, mx / 64, shape)
            b = a + rng.normal(0, mx / 32, shape)
            a, b = np.clip(np.rint(a), 0, mx), np.clip(np.rint(b), 0, mx)
        cd.append(np.ascontiguousarray(a.astype(dt)))
        db.append(np.ascontiguousarray(b.astype(dt)))
    return cd, db


def unit_grid(W, H, p, layout, us):
    cw, ch = crop(W, H, p, layout)
    return count_units(us, ch), count_units(us, cw)


def random_units(rng, rows, cols, kinds=(0, 1, 2), ends=False, sets=None):
    """(rows, cols) LRF_UNIT_DTYPE records of the given kinds; `ends` draws xqd and taps from their range ends."""
    u = np.zeros((rows, cols), B.LRF_UNIT_DTYPE)
    for r in range(rows):
        for c in range(cols):
            t = int(rng.choice(kinds))
            u[r, c]["type"] = t
            if t == 2:
                u[r, c]["set"] = int(rng.integers(0, 16)) if sets is None else int(rng.choice(sets))
                u[r, c]["xqd"] = [int(rng.choice([lo, hi])) if ends else int(rng.integers(lo, hi + 1))
                                  for lo, hi in zip(XQD_MIN, XQD_MAX)]
            elif t == 1:
                u[r, c]["coeffs"] = [[int(rng.choice([lo, hi])) if ends else int(rng.integers(lo, hi + 1))
                                      for lo, hi in zip(TAPS_MIN, TAPS_MAX)] for _ in range(2)]
    return u


def legal_unit_sizes(rng, layout):
    """unit sizes the specification allows: luma 64..256, chroma the same or, in 4:2:0, half."""
    y = int(rng.choice([64, 128, 256]))
    uv = y >> int(rng.integers(0, 2)) if layout == "420" else y
    return [y, uv, uv][:LAYOUTS[layout][0]]


# ---------------------------------------------------------------- the oracle
def orc_lrf(cdeffed, deblocked, layout, bd, W, H, enable_cdef, unit_size, units):
    """orc_lrf_filter_frame on copies of the CDEF output; returns the filtered padded planes."""
    L = O.lib()
    f = L.orc_lrf_filter_frame
    f.restype = None
    n, xdec, ydec = LAYOUTS[layout]
    out = [a.copy() for a in cdeffed]
    vpa, spa = C.c_void_p * 3, C.c_ssize_t * 3

    def org(arrs):
        return vpa(*[a.ctypes.data + (PAD * a.shape[1] + PAD) * a.itemsize for a in arrs])

    recs = [np.ascontiguousarray(np.asarray(u, B.LRF_UNIT_DTYPE).reshape(-1)) for u in units]
    f(org(out), spa(*[a.shape[1] for a in out]), org(cdeffed), spa(*[a.shape[1] for a in cdeffed]), org(deblocked),
      spa(*[a.shape[1] for a in deblocked]), C.c_int(cdeffed[0].itemsize), C.c_int(n), C.c_int(xdec),
      C.c_int(ydec), C.c_int(W), C.c_int(H), C.c_int(bd), C.c_int(int(enable_cdef)),
      (C.c_int * 3)(*unit_size, *([0] * (3 - len(unit_size)))),
      vpa(*[r.ctypes.data for r in recs], *([None] * (3 - len(recs)))))
    return out


# ---------------------------------------------------------------- the specification's process
def spec_plane(cdef, deb, p, layout, bd, W, H, us, units, rav1e_wiener_edges=False, rav1e_r0_odd_rows=False):
    """LrFrame over plane p's crop (ch x cw) from padded planes."""
    subX, subY = dec(p, layout)
    PlaneEndX, PlaneEndY = round2(W, subX) - 1, round2(H, subY) - 1
    cw, ch = PlaneEndX + 1, PlaneEndY + 1
    unitRows, unitCols = count_units(us, round2(H, subY)), count_units(us, round2(W, subX))
    yy, xx = np.mgrid[0:ch, 0:cw]
    row, col = (yy << subY) >> 2, (xx << subX) >> 2
    stripeNum = (row * 4 + 8) // 64
    StripeStartY = (-8 + stripeNum * 64) >> subY
    StripeEndY = StripeStartY + (64 >> subY) - 1
    unitRow = np.minimum(unitRows - 1, ((row * 4 + 8) >> subY) // us)
    unitCol = np.minimum(unitCols - 1, ((col * 4) >> subX) // us)
    rec = np.asarray(units).reshape(unitRows, unitCols)[unitRow, unitCol]
    C_ = cdef.astype(np.int64)[PAD:, PAD:]
    D_ = deb.astype(np.int64)[PAD:, PAD:]
    last = np.where(stripeNum == 0, StripeEndY, np.minimum(StripeEndY, PlaneEndY))  # rav1e's last stripe row

    def source(dy, dx, wiener):
        x = np.clip(xx + dx, 0, PlaneEndX)
        yu = yy + dy
        y = np.clip(yu, 0, PlaneEndY)
        above, below = y < StripeStartY, y > StripeEndY
        y = np.where(above, np.maximum(StripeStartY - 2, y), np.where(below, np.minimum(StripeEndY + 2, y), y))
        v = np.where(above | below, D_[y, x], C_[y, x])
        if wiener and rav1e_wiener_edges:
            v = np.where(yu < 0, D_[0, x], v)
            v = np.where((yu > PlaneEndY) & (yu > last), D_[PlaneEndY, x], v)
        return v

    cdefpx = C_[yy, xx]
    out = cdefpx.copy()
    mx = (1 << bd) - 1
    # Wiener
    wmask = rec["type"] == 1
    if wmask.any():
        r0, r1 = (5, 9) if bd == 12 else (3, 11)
        offset = 1 << (bd + 7 - r0 - 1)
        limit = (1 << (bd + 1 + 7 - r0)) - 1
        cf = rec["coeffs"].astype(np.int64)

        def taps(pass_):
            c = cf[..., pass_, :]
            return [c[..., 0], c[..., 1], c[..., 2], 128 - 2 * (c[..., 0] + c[..., 1] + c[..., 2]), c[..., 2],
                    c[..., 1], c[..., 0]]
        vf, hf = taps(0), taps(1)
        srcw = {(dy, dx): source(dy, dx, True) for dy in range(-3, 4) for dx in range(-3, 4)}
        acc = 0
        for r in range(7):
            s = sum(hf[t] * srcw[(r - 3, t - 3)] for t in range(7))
            acc = acc + vf[r] * np.clip(round2(s, r0), -offset, limit - offset)
        out = np.where(wmask, np.clip(round2(acc, r1), 0, mx), out)
    # self-guided
    smask = rec["type"] == 2
    if smask.any():
        srcs = {(dy, dx): source(dy, dx, False) for dy in range(-3, 4) for dx in range(-3, 4)}
        sets = rec["set"].astype(np.int64)
        prm = np.array(SGR_PARAMS, np.int64)[sets]
        u = cdefpx << 4
        flt = []
        for pass_ in range(2):
            r, s = prm[..., 2 * pass_], prm[..., 2 * pass_ + 1]
            res = np.zeros_like(u)
            for rad in (1, 2):
                m = r == rad
                if not m.any():
                    continue
                n = (2 * rad + 1) ** 2
                sm = np.where(m, s, 0)
                one_over_n = ((1 << 12) + n // 2) // n
                A, Bv = {}, {}
                for i in (-1, 0, 1):
                    for j in (-1, 0, 1):
                        vals = [srcs[(i + ey, j + ex)] for ey in range(-rad, rad + 1) for ex in range(-rad, rad + 1)]
                        a = sum(v * v for v in vals)
                        b = sum(vals)
                        a = round2(a, 2 * (bd - 8))
                        d = round2(b, bd - 8)
                        pp = np.maximum(0, a * n - d * d)
                        z = round2(pp * sm, 20)
                        a2 = np.where(z >= 255, 256, np.where(z == 0, 1, ((z << 8) + z // 2) // (z + 1)))
                        A[i, j] = a2
                        Bv[i, j] = round2(((1 << 8) - a2) * b * one_over_n, 12)
                if pass_ == 0:
                    odd = (yy & 1) == 1
                    shift = np.where(odd, 4, 5)
                    wa, wb = 0, 0
                    for i in (-1, 0, 1):
                        use = ((yy + i) & 1) == 1
                        for j in (-1, 0, 1):
                            w = np.where(use, 6 if j == 0 else 5, 0)
                            wa, wb = wa + w * A[i, j], wb + w * Bv[i, j]
                else:
                    shift = 5
                    wa, wb = 0, 0
                    for i in (-1, 0, 1):
                        for j in (-1, 0, 1):
                            w = 4 if (i == 0 or j == 0) else 3
                            wa, wb = wa + w * A[i, j], wb + w * Bv[i, j]
                v = wa * cdefpx + wb
                res = np.where(m, round2(v, 8 + shift - 4), res)
            flt.append(res)
        w0 = rec["xqd"][..., 0].astype(np.int64)
        w1 = rec["xqd"][..., 1].astype(np.int64)
        w2 = (1 << 7) - w0 - w1
        u0 = u
        if rav1e_r0_odd_rows:
            u0 = np.where((yy & 1) == 1, C_[yy - 1, xx] << 4, u)
        v = w1 * u + w0 * np.where(prm[..., 0] > 0, flt[0], u0) + w2 * np.where(prm[..., 2] > 0, flt[1], u)
        out = np.where(smask, np.clip(round2(v, 11), 0, mx), out)
    return out


def spec_lr(cdeffed, deblocked, layout, bd, W, H, unit_size, units, rav1e=True):
    return [spec_plane(cdeffed[p], deblocked[p], p, layout, bd, W, H, unit_size[p], units[p], rav1e, rav1e)
            for p in range(len(cdeffed))]


def crop_of(a, W, H, p, layout):
    cw, ch = crop(W, H, p, layout)
    return a[PAD:PAD + ch, PAD:PAD + cw]


def unit_types(W, H, p, layout, us, units):
    """The unit type the specification assigns to each crop pixel, and each pixel's set."""
    subX, subY = dec(p, layout)
    cw, ch = crop(W, H, p, layout)
    yy, xx = np.mgrid[0:ch, 0:cw]
    row, col = (yy << subY) >> 2, (xx << subX) >> 2
    rows, cols = count_units(us, ch), count_units(us, cw)
    rec = np.asarray(units).reshape(rows, cols)[np.minimum(rows - 1, ((row * 4 + 8) >> subY) // us),
                                                np.minimum(cols - 1, ((col * 4) >> subX) // us)]
    return rec["type"], rec["set"], rec["xqd"][..., 0]


def check(rng_or_frame, layout, bd, W, H, unit_size, units, enable_cdef=1):
    """Oracle == model with rav1e's switches on; the pure specification differs only where stated.
    Returns (oracle planes, counts of pixels that differ from the pure specification by cause)."""
    cd, db = rng_or_frame
    got = orc_lrf(cd, db, layout, bd, W, H, enable_cdef, unit_size, units)
    shown = {"wiener_edges": 0, "r0_odd_rows": 0}
    for p in range(len(cd)):
        g = crop_of(got[p], W, H, p, layout)
        want = spec_plane(cd[p], db[p], p, layout, bd, W, H, unit_size[p], units[p], True, True)
        pure = spec_plane(cd[p], db[p], p, layout, bd, W, H, unit_size[p], units[p])
        t, sets, x0 = unit_types(W, H, p, layout, unit_size[p], units[p])
        if not enable_cdef:  # difference 2: Sgrproj units keep the CDEF output
            c = crop_of(cd[p], W, H, p, layout)
            want = np.where(t == 2, c, want)
            pure = np.where(t == 2, c, pure)
        assert (g == want).all(), f"plane {p}: {np.argwhere(g != want)[:5]}"
        ch = g.shape[0]
        yy = np.mgrid[0:ch, 0:g.shape[1]][0]
        diff = g != pure
        edge = (t == 1) & ((yy < 3) | (yy >= ch - 3))
        r0odd = (t == 2) & (sets >= 10) & (sets <= 13) & (x0 != 0) & ((yy & 1) == 1)
        assert not (diff & ~edge & ~r0odd).any(), np.argwhere(diff & ~edge & ~r0odd)[:5]
        shown["wiener_edges"] += int((diff & edge).sum())
        shown["r0_odd_rows"] += int((diff & r0odd).sum())
    return got, shown


# ---------------------------------------------------------------- tests
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_mixed_units_match_the_specification(layout, bd):
    rng = np.random.default_rng(bd * 31 + ord(layout[1]))
    W, H = 203, 139                                   # not multiples of 8 or 64
    us = legal_unit_sizes(rng, layout)
    units = [random_units(rng, *unit_grid(W, H, p, layout, us[p])) for p in range(len(us))]
    check(make_frame(rng, W, H, layout, bd), layout, bd, W, H, us, units)


@pytest.mark.parametrize("content", ["flat", "edges", "smooth"])
@pytest.mark.parametrize("layout", ["420", "444"])
def test_content(content, layout):
    rng = np.random.default_rng(len(content) * 7 + int(layout))
    for bd in (8, 12):
        W, H = 131, 97
        us = legal_unit_sizes(rng, layout)
        units = [random_units(rng, *unit_grid(W, H, p, layout, us[p]), ends=True) for p in range(len(us))]
        check(make_frame(rng, W, H, layout, bd, content), layout, bd, W, H, us, units)


@pytest.mark.parametrize("W,H", [(32, 32), (33, 35), (65, 57), (71, 121), (127, 63), (255, 129), (383, 71)])
def test_frame_sizes_and_stretched_units(W, H):
    rng = np.random.default_rng(W * 1000 + H)
    for layout in ("400", "420", "422"):
        for y in (64, 128, 256):
            us = [y, y >> (layout == "420"), y >> (layout == "420")][:LAYOUTS[layout][0]]
            units = [random_units(rng, *unit_grid(W, H, p, layout, us[p])) for p in range(len(us))]
            check(make_frame(rng, W, H, layout, 10), layout, 10, W, H, us, units)


def test_every_set_and_range_end():
    rng = np.random.default_rng(5)
    W, H = 200, 130
    for bd in (8, 10, 12):
        for s in range(16):
            for xqd in [(XQD_MIN[0], XQD_MIN[1]), (XQD_MAX[0], XQD_MAX[1]), (XQD_MIN[0], XQD_MAX[1]),
                        (XQD_MAX[0], XQD_MIN[1]), (0, 64)]:
                units = np.zeros((count_units(64, H), count_units(64, W)), B.LRF_UNIT_DTYPE)
                units["type"], units["set"], units["xqd"] = 2, s, xqd
                check(make_frame(rng, W, H, "400", bd, "edges" if s & 1 else "random"), "400", bd, W, H, [64],
                      [units])
        for taps in [TAPS_MIN, TAPS_MAX]:
            units = np.zeros((count_units(64, H), count_units(64, W)), B.LRF_UNIT_DTYPE)
            units["type"], units["coeffs"] = 1, [taps, taps]
            check(make_frame(rng, W, H, "400", bd, "edges"), "400", bd, W, H, [64], [units])


def test_difference_1_wiener_reads_the_deblocked_frame_above_and_below():
    rng = np.random.default_rng(11)
    for layout, W, H in (("420", 96, 80), ("444", 70, 121), ("420", 64, 54)):
        us = [64, 64, 64]
        units = [np.zeros(unit_grid(W, H, p, layout, 64), B.LRF_UNIT_DTYPE) for p in range(3)]
        for u in units:
            u["type"], u["coeffs"] = 1, [TAPS_MAX, TAPS_MIN]
        _, shown = check(make_frame(rng, W, H, layout, 8), layout, 8, W, H, us, units)
        assert shown["wiener_edges"] > 0, shown   # shown; check() confines it to 3 rows at the top and bottom
    # the same frames with Sgrproj units: the self-guided filter matches the specification at those rows
    for layout, W, H in (("420", 96, 80), ("444", 70, 121)):
        units = [np.zeros(unit_grid(W, H, p, layout, 64), B.LRF_UNIT_DTYPE) for p in range(3)]
        for u in units:
            u["type"], u["set"], u["xqd"] = 2, 3, (-20, 40)
        _, shown = check(make_frame(rng, W, H, layout, 8), layout, 8, W, H, [64] * 3, units)
        assert shown == {"wiener_edges": 0, "r0_odd_rows": 0}


def test_difference_2_enable_cdef_off_skips_sgrproj_units():
    rng = np.random.default_rng(12)
    W, H, layout = 150, 100, "420"
    us = [64, 32, 32]
    units = [random_units(rng, *unit_grid(W, H, p, layout, us[p]), sets=range(10)) for p in range(3)]
    frame = make_frame(rng, W, H, layout, 10)
    off, _ = check(frame, layout, 10, W, H, us, units, enable_cdef=0)   # asserts Sgrproj pixels == CDEF output
    on, _ = check(frame, layout, 10, W, H, us, units, enable_cdef=1)
    changed = 0
    for p in range(3):
        t = unit_types(W, H, p, layout, us[p], units[p])[0]
        d = crop_of(off[p], W, H, p, layout) != crop_of(on[p], W, H, p, layout)
        assert not (d & (t != 2)).any()                 # confined to Sgrproj units
        changed += int(d.sum())
    assert changed > 0


def test_difference_3_short_frames_write_below_the_crop():
    rng = np.random.default_rng(13)
    for layout, W, H in (("400", 90, 33), ("420", 64, 40), ("422", 48, 50)):
        n = LAYOUTS[layout][0]
        units = [np.zeros(unit_grid(W, H, p, layout, 64), B.LRF_UNIT_DTYPE) for p in range(n)]
        for u in units:
            u["type"], u["set"], u["xqd"] = 2, 0, (-40, 50)
        frame = make_frame(rng, W, H, layout, 8)
        got, _ = check(frame, layout, 8, W, H, [64] * n, units)    # the crop equals the specification
        below = 0
        for p in range(n):
            cw, ch = crop(W, H, p, layout)
            s0 = 56 >> dec(p, layout)[1]
            assert ch < s0
            d = got[p] != frame[0][p]
            d[PAD:PAD + ch, PAD:PAD + cw] = False
            assert not d[:PAD + ch].any() and not d[PAD + s0:].any() and not d[:, :PAD].any() \
                and not d[:, PAD + cw:].any()                  # only stripe 0's rows below the crop
            below += int(d.sum())
        assert below > 0


def test_difference_4_sets_without_radius_2_use_the_even_row_on_odd_rows():
    rng = np.random.default_rng(14)
    W, H = 100, 90
    for s in (10, 11, 12, 13):
        units = np.zeros((count_units(64, H), count_units(64, W)), B.LRF_UNIT_DTYPE)
        units["type"], units["set"], units["xqd"] = 2, s, (-50, 30)
        _, shown = check(make_frame(rng, W, H, "400", 8), "400", 8, W, H, [64], [units])
        assert shown["r0_odd_rows"] > 0
        units["xqd"] = (0, 30)                               # what sgrproj_solve and the bitstream give
        _, shown = check(make_frame(rng, W, H, "400", 8), "400", 8, W, H, [64], [units])
        assert shown["r0_odd_rows"] == 0
