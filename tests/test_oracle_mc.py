"""Cross-checks for the oracle's motion compensation (no stored vectors exist upstream; the
reference only has asm==rust random tests, asm/x86/mc.rs:624-833 — "parity unpinned")."""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O


def make_plane(dtype, bd, seed=0, w=96, h=80, pad=16):
    rng = np.random.default_rng(seed)
    p = O.Plane(w, h, pad, dtype=dtype)
    p.fill_from(rng.integers(0, 1 << bd, (h, w)).astype(dtype))
    return p


def test_filter_rows_are_av1_normative_and_sum_to_128():
    L = O.lib()
    f = (C.c_int32 * 8)()
    for mode in range(4):
        for length in (4, 8):
            for frac in range(16):
                L.orc_get_filter(mode, frac, length, f)
                assert sum(f) == 128
    L.orc_get_filter(0, 8, 8, f)
    assert list(f) == [0, 2, -14, 76, 76, -14, 2, 0]          # REGULAR half-pel (AV1 spec)
    L.orc_get_filter(2, 8, 8, f)
    assert list(f) == [-4, 12, -24, 80, 80, -24, 12, -4]      # SHARP half-pel
    L.orc_get_filter(0, 8, 4, f)
    assert list(f) == [0, 0, -12, 76, 76, -12, 0, 0]          # 4-tap variant when length <= 4
    L.orc_get_filter(3, 4, 4, f)
    assert list(f) == [0, 0, 0, 96, 32, 0, 0, 0]              # BILINEAR ignores the length rule


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10), (np.uint16, 12)])
def test_integer_position_copies_and_flat_area_is_preserved(dtype, bd):
    p = make_plane(dtype, bd)
    got = O.put_8tap(p, 8, 8, 16, 16, 0, 0, 0, 0, bd)
    np.testing.assert_array_equal(got, p.view()[8:24, 8:24])
    flat = O.Plane(64, 64, 16, dtype=dtype)
    flat.data[:] = (1 << bd) - 3
    for cf, rf in ((0, 5), (7, 0), (3, 11)):
        assert (O.put_8tap(flat, 8, 8, 8, 8, cf, rf, 0, 2, bd) == (1 << bd) - 3).all()


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10), (np.uint16, 12)])
def test_paths_against_direct_numpy_formulas(dtype, bd):
    """The four code paths (mc.rs:264-352) against their closed forms written independently."""
    p = make_plane(dtype, bd, seed=bd)
    L = O.lib()
    ib = 2 if bd == 12 else 4
    maxv = (1 << bd) - 1
    img = p.data.astype(np.int64)
    x0, y0, w, h = 10, 12, 8, 8
    fx = (C.c_int32 * 8)()
    fy = (C.c_int32 * 8)()
    rs = lambda v, b: (v + ((1 << b) >> 1)) >> b
    for mode_x, mode_y, cf, rf in ((0, 0, 0, 9), (1, 2, 5, 0), (2, 0, 13, 6), (3, 3, 8, 8)):
        L.orc_get_filter(mode_x, cf, w, fx)
        L.orc_get_filter(mode_y, rf, h, fy)
        want = np.zeros((h, w), np.int64)
        for r in range(h):
            for c in range(w):
                py, px = p.pad + y0 + r, p.pad + x0 + c
                if cf == 0:
                    s = sum(fy[k] * img[py - 3 + k, px] for k in range(8))
                    v = rs(s, 7)
                elif rf == 0:
                    s = sum(fx[k] * img[py, px - 3 + k] for k in range(8))
                    v = rs(rs(s, 7 - ib), ib)
                else:
                    inter = []
                    for k in range(8):
                        s = sum(fx[j] * img[py - 3 + k, px - 3 + j] for j in range(8))
                        t = rs(s, 7 - ib)
                        t = ((t + 32768) & 0xFFFF) - 32768          # `as i16`
                        inter.append(t)
                    v = rs(sum(fy[k] * inter[k] for k in range(8)), 7 + ib)
                want[r, c] = min(max(v, 0), maxv)
        got = O.put_8tap(p, x0, y0, w, h, cf, rf, mode_x, mode_y, bd)
        np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10), (np.uint16, 12)])
def test_avg_of_identical_preps_equals_put_at_integer_position(dtype, bd):
    """prep at an integer position is (p << ib) - bias, so avg(prep, prep) returns p exactly
    (mc.rs:377-385, :466-478)."""
    p = make_plane(dtype, bd, seed=1)
    t = O.prep_8tap(p, 4, 4, 16, 8, 0, 0, 0, 0, bd)
    np.testing.assert_array_equal(O.mc_avg(t, t, bd), p.view()[4:12, 4:20])
    # and for fractional positions avg(prep, prep) is within 1 of put (different rounding chain)
    t = O.prep_8tap(p, 4, 4, 16, 8, 5, 11, 0, 0, bd)
    d = O.mc_avg(t, t, bd).astype(np.int64) - O.put_8tap(p, 4, 4, 16, 8, 5, 11, 0, 0, bd).astype(np.int64)
    assert np.abs(d).max() <= 1


def test_get_mv_params_chroma_and_negative_vectors():
    L = O.lib()
    out = [C.c_int() for _ in range(4)]
    L.orc_get_mv_params.argtypes = [C.c_int] * 4 + [C.POINTER(C.c_int)] * 4
    L.orc_get_mv_params(-13, 27, 0, 0, *[C.byref(o) for o in out])
    # luma: offset = mv >> 3 (floor), frac = (mv << 1) & 15
    assert [o.value for o in out] == [-2, 3, (-13 * 2) & 15, (27 * 2) & 15]
    L.orc_get_mv_params(-13, 27, 1, 1, *[C.byref(o) for o in out])
    assert [o.value for o in out] == [-1, 1, -13 & 15, 27 & 15]


def test_filter_tables_have_the_normative_structure():
    """Structure every AV1 interpolation kernel has (spec section 7.11.3.4, Subpel_Filters): position 0 is the
    identity, position 16 - f is position f mirrored (the kernel sits between taps 3 and 4), every row sums to 128,
    the 4-tap variants (block dimension <= 4) have zero outer taps, BILINEAR is (128 - 8 f, 8 f)."""
    L = O.lib()
    f, g = (C.c_int32 * 8)(), (C.c_int32 * 8)()
    for mode in range(4):
        for length in (4, 8):
            L.orc_get_filter(mode, 0, length, f)
            assert list(f) == [0, 0, 0, 128, 0, 0, 0, 0]
            for frac in range(1, 16):
                L.orc_get_filter(mode, frac, length, f)
                L.orc_get_filter(mode, 16 - frac, length, g)
                assert list(f) == list(g)[::-1], (mode, length, frac)
                if length == 4 and mode != 3:
                    assert f[0] == f[1] == f[6] == f[7] == 0
    for frac in range(16):
        L.orc_get_filter(3, frac, 8, f)
        assert list(f) == [0, 0, 0, 128 - 8 * frac, 8 * frac, 0, 0, 0]


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10), (np.uint16, 12)])
def test_put_equals_the_specification_two_pass_form(dtype, bd):
    """The AV1 specification (7.11.3.4 block inter prediction, non-compound) states ONE form for every sub-pel
    position: a horizontal pass rounded by InterRound0 (3; 5 at 12 bit) into an intermediate of h + 7 rows, a vertical
    pass rounded by InterRound1 (11; 9 at 12 bit), Clip1 - with the identity kernel at position 0.  The reference's
    four special-cased paths (mc.rs:264-352) must all equal it."""
    p = make_plane(dtype, bd, seed=40 + bd)
    L = O.lib()
    r0, r1 = (5, 9) if bd == 12 else (3, 11)
    maxv = (1 << bd) - 1
    img = p.data.astype(np.int64)
    rnd = lambda v, b: (v + (1 << (b - 1))) >> b
    fx, fy = (C.c_int32 * 8)(), (C.c_int32 * 8)()
    rng = np.random.default_rng(bd)
    for w, h in ((8, 8), (4, 16), (16, 4)):
        for _ in range(6):
            cf, rf = (int(v) for v in rng.integers(0, 16, 2))
            if rng.integers(0, 3) == 0:
                cf = 0
            if rng.integers(0, 3) == 0:
                rf = 0
            mx, my = (int(v) for v in rng.integers(0, 4, 2))
            x0, y0 = (int(v) for v in rng.integers(4, 40, 2))
            L.orc_get_filter(mx, cf, w, fx)
            L.orc_get_filter(my, rf, h, fy)
            kx, ky = np.array(list(fx), np.int64), np.array(list(fy), np.int64)
            inter = np.zeros((h + 7, w), np.int64)
            for r in range(h + 7):
                for c in range(w):
                    py, px = p.pad + y0 + r - 3, p.pad + x0 + c - 3
                    inter[r, c] = rnd(int((kx * img[py, px:px + 8]).sum()), r0)
            want = np.zeros((h, w), np.int64)
            for r in range(h):
                for c in range(w):
                    want[r, c] = min(max(rnd(int((ky * inter[r:r + 8, c]).sum()), r1), 0), maxv)
            got = O.put_8tap(p, x0, y0, w, h, cf, rf, mx, my, bd)
            np.testing.assert_array_equal(got, want, err_msg=f"{w}x{h} frac ({cf},{rf}) modes ({mx},{my})")


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_intermediate_extremes_fit_i16(bd):
    """The kernels keep the horizontal pass in an i16 intermediate and run every sub-pel case through it
    (mc_dev.cuh).  That rests on the intermediate never truncating: its extremes, every positive tap on max or
    every negative tap on max, over every bank, fraction and length, lie inside i16.  The vertical pass of
    `prep` over those extremes, the value stored as i16, fits too."""
    L = O.lib()
    f = (C.c_int32 * 8)()
    r0 = 5 if bd == 12 else 3
    maxv = (1 << bd) - 1
    rnd = lambda v, b: (v + (1 << (b - 1))) >> b
    rows = []
    for mode in range(4):
        for length in (4, 8):
            for frac in range(16):
                L.orc_get_filter(mode, frac, length, f)
                rows.append(list(f))
    hi = max(rnd(sum(t for t in r if t > 0) * maxv, r0) for r in rows)
    lo = min(rnd(sum(t for t in r if t < 0) * maxv, r0) for r in rows)
    assert -32768 <= lo and hi <= 32767
    assert (hi, lo) == {8: (5865, -1785), 10: (23529, -7161), 12: (23546, -7166)}[bd]
    bias = 0 if bd == 8 else 8192
    for r in rows:
        top = sum(t * (hi if t > 0 else lo) for t in r)
        bottom = sum(t * (lo if t > 0 else hi) for t in r)
        assert -32768 <= rnd(bottom, 7) - bias and rnd(top, 7) - bias <= 32767


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10), (np.uint16, 12)])
def test_numpy_reference_of_the_gpu_sweeps_equals_the_oracle(dtype, bd):
    """tests/test_mc_paths_gpu.py compares the kernels with a vectorised restatement of the specification's
    two-pass form; on one random batch per bit depth it must equal orc_mc_blocks and orc_mc_avg."""
    from tests import test_mc_paths_gpu as T
    rng = np.random.default_rng(7 + bd)
    p = make_plane(dtype, bd, seed=bd, w=96, h=80, pad=24)
    full = p.data.astype(np.int64)
    for (w, h), (xdec, ydec), (mx, my) in (((8, 8), (0, 0), (2, 1)), ((4, 16), (1, 0), (0, 3)),
                                           ((16, 4), (1, 1), (1, 2)), ((2, 2), (1, 1), (3, 0))):
        blocks, mvs = T.random_items(rng, 40, w, h, xdec, ydec, 96, 80, 8)
        x0, y0, cf, rf = T.mv_params(blocks, mvs, xdec, ydec)
        T.assert_readable(x0, y0, w, h, 96, 80, 24)
        for kind in (0, 1):
            want = O.mc_blocks(p, blocks, mvs, w, h, mx, my, bd, xdec, ydec, kind)
            got = T.mc_ref(full, 24, x0, y0, cf, rf, w, h, mx, my, bd, kind)
            np.testing.assert_array_equal(got, want, err_msg=f"{w}x{h} kind {kind}")
        t1 = O.mc_blocks(p, blocks, mvs, w, h, mx, my, bd, xdec, ydec, 1)
        t2 = O.mc_blocks(p, blocks, mvs[::-1].copy(), w, h, my, mx, bd, xdec, ydec, 1)
        np.testing.assert_array_equal(T.avg_ref(t1, t2, bd), np.stack([O.mc_avg(a, b, bd) for a, b in zip(t1, t2)]))


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10), (np.uint16, 12)])
def test_prep_and_avg_equal_the_specification_at_extreme_tiles(dtype, bd):
    """The specification's compound form (7.11.3.4 with InterRound1 = 7, then 7.11.3.15's average rounded by
    InterPostRound) on tiles built from the tap signs, which put the intermediate at its extremes: `prep` is the
    horizontal pass rounded by InterRound0, the vertical pass rounded by 7, minus PREP_BIAS at 10 / 12 bit, and
    `avg` is (t1 + t2 + 2 PREP_BIAS) rounded by InterPostRound (5; 3 at 12 bit), then Clip1.  `put` is checked on
    the same tiles."""
    from tests.test_mc_paths_gpu import sign_tiles
    L = O.lib()
    r0, r1 = (5, 9) if bd == 12 else (3, 11)
    post = 3 if bd == 12 else 5
    bias = 0 if bd == 8 else 8192
    maxv = (1 << bd) - 1
    rnd = lambda v, b: (v + (1 << (b - 1))) >> b
    fx, fy = (C.c_int32 * 8)(), (C.c_int32 * 8)()
    w = h = 8
    for mx, my, cf, rf in ((2, 2, 8, 8), (2, 0, 8, 6), (0, 2, 4, 8), (1, 3, 9, 5), (2, 2, 7, 0), (2, 2, 0, 9)):
        L.orc_get_filter(mx, cf, w, fx)
        L.orc_get_filter(my, rf, h, fy)
        kx, ky = np.array(list(fx), np.int64), np.array(list(fy), np.int64)
        preps = []
        for tile in sign_tiles(kx, ky, maxv):
            p = O.Plane(16, 16, 8, dtype=dtype)
            p.fill_from(np.tile(tile, (2, 2)).astype(dtype))
            img = p.data.astype(np.int64)
            inter = np.zeros((h + 7, w), np.int64)
            for r in range(h + 7):
                for c in range(w):
                    inter[r, c] = rnd(int((kx * img[p.pad + r, p.pad + c:p.pad + c + 8]).sum()), r0)
            want_put = np.zeros((h, w), np.int64)
            want_prep = np.zeros((h, w), np.int64)
            for r in range(h):
                for c in range(w):
                    s = int((ky * inter[r:r + 8, c]).sum())
                    want_put[r, c] = min(max(rnd(s, r1), 0), maxv)
                    want_prep[r, c] = rnd(s, 7) - bias
            what = f"modes ({mx},{my}) frac ({cf},{rf})"
            np.testing.assert_array_equal(O.put_8tap(p, 3, 3, w, h, cf, rf, mx, my, bd), want_put, err_msg=what)
            got = O.prep_8tap(p, 3, 3, w, h, cf, rf, mx, my, bd)
            np.testing.assert_array_equal(got, want_prep, err_msg=what)
            preps.append(got.astype(np.int64))
        for a in range(len(preps)):
            for b in (a, a ^ 1):
                want = np.clip(rnd(preps[a] + preps[b] + 2 * bias, post), 0, maxv)
                got = O.mc_avg(preps[a].astype(np.int16), preps[b].astype(np.int16), bd)
                np.testing.assert_array_equal(got, want, err_msg=f"avg {what} tiles {a} {b}")
