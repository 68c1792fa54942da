"""Pins the oracle's SAD/SATD against the reference's own known-answer tests.

Golden values are rav1e's `get_sad_same_inner` / `get_satd_same_inner`
(/root/reference/src/dist.rs:418-441 and :477-500), on the pattern of `setup_planes`
(:384-413): two 640x480 planes with different strides, block at (32, 40).
"""
import numpy as np
import pytest

from tests import oracle_lib as O

SAD_KAT = [(4, 4, 1912), (4, 8, 4296), (8, 4, 3496), (8, 8, 7824), (8, 16, 16592),
           (16, 8, 14416), (16, 16, 31136), (16, 32, 60064), (32, 16, 59552),
           (32, 32, 120128), (32, 64, 186688), (64, 32, 250176), (64, 64, 438912),
           (64, 128, 654272), (128, 64, 1016768), (128, 128, 1689792), (4, 16, 8680),
           (16, 4, 6664), (8, 32, 31056), (32, 8, 27600), (16, 64, 93344), (64, 16, 116384)]
SATD_KAT = [(4, 4, 1408), (4, 8, 2016), (8, 4, 1816), (8, 8, 3984), (8, 16, 5136),
            (16, 8, 4864), (16, 16, 9984), (16, 32, 13824), (32, 16, 13760),
            (32, 32, 27952), (32, 64, 37168), (64, 32, 45104), (64, 64, 84176),
            (64, 128, 127920), (128, 64, 173680), (128, 128, 321456), (4, 16, 3136),
            (16, 4, 2632), (8, 32, 7056), (32, 8, 6624), (16, 64, 18432), (64, 16, 21312)]


def setup_planes(dtype):
    """dist.rs:384-413 restated: Plane::new(640,480,0,0,136,136) and (...,264,264); the
    pattern is written over the WHOLE allocation (padding included) from buffer indices."""
    def mk(xpad, ypad, align):
        xorigin = (xpad + align - 1) // align * align
        stride = (xorigin + 640 + xpad + align - 1) // align * align
        return xorigin, ypad, stride, 480 + 2 * ypad
    # v_frame aligns xorigin/stride to 64 bytes; the pattern is alignment-robust (xpad_off).
    align = 64 // np.dtype(dtype).itemsize
    xo_i, yo_i, st_i, rows_i = mk(136, 136, align)
    xo_r, yo_r, st_r, rows_r = mk(264, 264, align)
    xpad_off = (xo_i - 136) - 8
    j = np.arange(st_i)[None, :]
    i = np.arange(rows_i)[:, None]
    inp = (((j + i) - xpad_off) & 255).astype(dtype)
    j = np.arange(st_r)[None, :]
    i = np.arange(rows_r)[:, None]
    rec = (((j - i) - xpad_off) & 255).astype(dtype)
    return (inp, xo_i, yo_i, st_i), (rec, xo_r, yo_r, st_r)


def test_pattern_closed_form():
    (inp, xo, yo, st), (rec, xr, yr, sr) = setup_planes(np.uint8)
    x, y = 100, 77
    assert inp[yo + y, xo + x] == (x + y + 24) & 255
    assert rec[yr + y, xr + x] == (x - y + 8) & 255


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
@pytest.mark.parametrize("kind,table", [("sad", SAD_KAT), ("satd", SATD_KAT)])
def test_reference_kats(dtype, kind, table):
    L = O.lib()
    (inp, xo, yo, st), (rec, xr, yr, sr) = setup_planes(dtype)
    sfx = "u8" if dtype == np.uint8 else "u16"
    f = getattr(L, f"orc_get_{kind}_{sfx}")
    for w, h, want in table:
        got = f(O.ptr(inp, (yo + 40) * st + xo + 32), st, O.ptr(rec, (yr + 40) * sr + xr + 32), sr, w, h)
        assert got == want, (kind, sfx, w, h, got, want)


def test_satd_partial_chunks_fall_back_to_sad():
    """dist.rs:185-191: chunks that do not fit the transform are SAD'ed (frame-edge crops)."""
    rng = np.random.default_rng(3)
    a = rng.integers(0, 256, (32, 32), dtype=np.uint8)
    b = rng.integers(0, 256, (32, 32), dtype=np.uint8)
    L = O.lib()
    # 12x8: one full 8x8 + one 4x8 partial chunk
    full = L.orc_get_satd_u8(O.ptr(a), 32, O.ptr(b), 32, 8, 8)
    part = L.orc_get_sad_u8(O.ptr(a, 8), 32, O.ptr(b, 8), 32, 4, 8)
    got = L.orc_get_satd_u8(O.ptr(a), 32, O.ptr(b), 32, 12, 8)
    # un-normalised sums add, single rounding at the end (ln = 3)
    d = a[:8, :8].astype(np.int64) - b[:8, :8].astype(np.int64)
    H2 = np.array([[1, 1], [1, -1]])
    H8 = np.kron(np.kron(H2, H2), H2)
    raw = np.abs(H8 @ d @ H8.T).sum()
    assert full == (raw + 4) >> 3
    assert got == (raw + part + 4) >> 3


def test_mv_rate_and_range():
    L = O.lib()
    mv = O.Mv
    assert L.orc_get_mv_rate(mv(0, 0), mv(0, 0), 0) == 0
    # diff 8 (one pel), !hp: 8>>1 = 4 -> ilog 3 -> rate 6 per component
    assert L.orc_get_mv_rate(mv(8, 0), mv(0, 0), 0) == 6
    assert L.orc_get_mv_rate(mv(8, -8), mv(0, 0), 0) == 12
    # -1 >> 1 = -1 (arithmetic), abs 1, ilog 1 -> 2
    assert L.orc_get_mv_rate(mv(-1, 0), mv(0, 0), 0) == 2
    assert L.orc_get_mv_rate(mv(1, 0), mv(0, 0), 0) == 0
    assert L.orc_get_mv_rate(mv(1, 0), mv(0, 0), 1) == 2
    # i16 wrap: -16384 - 16384 = -32768; with hp the wrapping abs keeps i16::MIN, whose 16-bit
    # pattern has no leading zeros -> ilog 16 -> rate 32; without hp: -32768 >> 1 = -16384 -> ilog 15
    assert L.orc_get_mv_rate(mv(-16384, 0), mv(16384, 0), 1) == 32
    assert L.orc_get_mv_rate(mv(-16384, 0), mv(16384, 0), 0) == 30
    # cost = 256*sad + min(r1, r2+1)*lambda
    assert L.orc_mv_cost(10, mv(8, 0), mv(0, 0), mv(8, 0), 100, 0) == 2560 + 1 * 100
    import ctypes as C
    r = [C.c_int() for _ in range(4)]
    L.orc_get_mv_range(480, 272, 0, 0, 16, 16, *[C.byref(x) for x in r])
    assert [x.value for x in r] == [-256, (480 - 4) * 32 + 256, -256, (272 - 4) * 32 + 256]


def _i16(v):
    v &= 0xFFFF
    return v - 0x10000 if v & 0x8000 else v


def _diff_to_rate(diff, allow_hp):
    """me.rs:1516-1519 on Python integers: `diff >> 1` is i16's arithmetic shift, `d.abs()` wraps
    for i16::MIN, and v_frame's ILog::ilog of an i16 is 16 - leading_zeros of its 16-bit pattern."""
    d = diff if allow_hp else diff >> 1
    return 2 * (_i16(abs(d)) & 0xFFFF).bit_length()


def _mv_rate(a, b, allow_hp):
    """me.rs:1512-1523: the component differences are i16 subtractions (wrapping)."""
    return _diff_to_rate(_i16(a[0] - b[0]), allow_hp) + _diff_to_rate(_i16(a[1] - b[1]), allow_hp)


def _mv_cost(sad, mv, pmv0, pmv1, lam, allow_hp):
    """me.rs:1455-1460 with unbounded integers: nothing may wrap below 2^64."""
    rate = min(_mv_rate(mv, pmv0, allow_hp), _mv_rate(mv, pmv1, allow_hp) + 1)
    cost = 256 * sad + rate * lam
    assert cost < 2**64
    return cost


EXTREME_MV = [-32768, -32767, -16385, -16384, -9, -8, -1, 0, 1, 2, 8, 16383, 16384, 32766, 32767]


@pytest.mark.parametrize("allow_hp", [0, 1])
def test_mv_rate_extremes_match_bigint_restatement(allow_hp):
    """orc_get_mv_rate on every pair of extreme components, against the restatement above: i16
    wrap of `a - b`, the i16::MIN difference (ilog 16), the arithmetic shift without hp."""
    L = O.lib()
    for ar in EXTREME_MV:
        for br in EXTREME_MV:
            a, b = (ar, -br), (br, ar)
            assert L.orc_get_mv_rate(O.Mv(*a), O.Mv(*b), allow_hp) == _mv_rate(a, b, allow_hp), (a, b)
    # the wrap reaches i16::MIN from both sides
    assert _mv_rate((0, 0), (-32768, 0), 1) == 32 and _mv_rate((-1, 0), (32767, 0), 1) == 32
    assert _mv_rate((0, 0), (-32768, -32768), 0) == 60


@pytest.mark.parametrize("lam", [0, 1, 2**31, 2**32 - 1])
@pytest.mark.parametrize("allow_hp", [0, 1])
def test_mv_cost_extremes_match_bigint_restatement(lam, allow_hp):
    """orc_mv_cost at lambdas up to 2^32 - 1 and SADs up to a 128x128 12-bit block (and u32 max):
    rate * lambda needs 64 bits, and the largest cost stays below 2^39, the bound the device's
    packed argmin key relies on for every SAD a block can have."""
    L = O.lib()
    rng = np.random.default_rng(lam % 1000 + allow_hp)
    sads = [0, 1, 255 * 64 * 64, 4095 * 128 * 128, 2**32 - 1]
    for _ in range(400):
        mv, p0, p1 = [(int(rng.choice(EXTREME_MV)), int(rng.choice(EXTREME_MV))) for _ in range(3)]
        for sad in sads:
            want = _mv_cost(sad, mv, p0, p1, lam, allow_hp)
            assert L.orc_mv_cost(sad, O.Mv(*mv), O.Mv(*p0), O.Mv(*p1), lam, allow_hp) == want
            if sad <= 4095 * 128 * 128:
                assert want < 2**39
    worst = _mv_cost(4095 * 128 * 128, (0, 0), (-32768, -32768), (-32768, -32768), lam, 1)
    assert worst == 256 * 4095 * 128 * 128 + 64 * lam


def test_full_search_first_min_tiebreak():
    """me.rs:1501 strict `<`: on a flat reference every candidate ties; the first scanned
    position (y_lo, x_lo) must win when lambda = 0."""
    cur = O.Plane(64, 64, 32)
    ref = O.Plane(64, 64, 32)
    cur.data[:] = 7
    ref.data[:] = 9
    L = O.lib()
    z = O.Mv(0, 0)
    r = L.orc_full_search(cur.at(16, 16), cur.stride, ref.origin_ptr(), ref.stride, 1,
                          8, 24, 10, 22, 16, 16, 16, 16, 4, 0, z, z, 0)
    assert (r.mv.col, r.mv.row) == (8 * (8 - 16), 8 * (10 - 16))
    assert r.sad == 2 * 256 and r.cost == 256 * 512
    # with lambda > 0 the zero vector has the lowest rate and wins
    r = L.orc_full_search(cur.at(16, 16), cur.stride, ref.origin_ptr(), ref.stride, 1,
                          8, 24, 8, 24, 16, 16, 16, 16, 4, 50, z, z, 0)
    assert (r.mv.col, r.mv.row) == (0, 0)
