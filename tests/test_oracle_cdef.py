"""Pins / cross-checks for the oracle's CDEF.  `first_max_element` is pinned by the reference's
own KAT (src/cdef.rs:304-309); direction search and filter have no stored vectors upstream
("parity unpinned") and are checked on constructed inputs."""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O


def test_first_max_element_reference_kat():
    L = O.lib()

    def fme(vals):
        a = np.array(vals, np.int32)
        m = C.c_int32()
        i = L.orc_first_max_element(O.ptr(a), len(a), C.byref(m))
        return i, m.value
    assert fme([-1, -1, 1, 2, 3, 4, 6, 6]) == (6, 6)      # cdef.rs:306
    assert fme([-1, -1, 1, 2, 3, 4, 7, 6]) == (6, 7)      # cdef.rs:307
    assert fme([0, 0]) == (0, 0)                          # cdef.rs:308


def test_find_dir_on_directional_patterns():
    """Direction 2 is horizontal, 6 vertical, 0 is 45 degrees up-right (cdef.rs:78-83)."""
    i, j = np.mgrid[0:8, 0:8]
    stripes_h = ((i % 2) * 200 + 20).astype(np.uint8)     # constant along rows -> horizontal lines
    stripes_v = ((j % 2) * 200 + 20).astype(np.uint8)
    diag = (((i + j) // 2 % 2) * 200 + 20).astype(np.uint8)   # constant along i+j -> 45 deg up-right
    anti = (((i - j) // 2 % 2) * 200 + 20).astype(np.uint8)  # (a 1-px checkerboard would tie)
    assert O.cdef_find_dir(stripes_h)[0] == 2
    assert O.cdef_find_dir(stripes_v)[0] == 6
    assert O.cdef_find_dir(diag)[0] == 0
    assert O.cdef_find_dir(anti)[0] == 4
    d, v = O.cdef_find_dir(np.full((8, 8), 77, np.uint8))
    assert (d, v) == (0, 0)                               # all costs tie -> first, zero variance
    # 10-bit input is shifted down by coeff_shift before the search (cdef.rs:97)
    assert O.cdef_find_dir((stripes_h.astype(np.uint16) << 2), 10) == O.cdef_find_dir(stripes_h)


def test_adjust_strength_and_constrain_basics():
    L = O.lib()
    assert L.orc_cdef_adjust_strength(8, 0) == 0
    assert L.orc_cdef_adjust_strength(8, 63) == (8 * 4 + 8) >> 4
    assert L.orc_cdef_adjust_strength(8, 64) == (8 * (4 + 0) + 8) >> 4      # msb(1) = 0
    assert L.orc_cdef_adjust_strength(8, 1 << 20) == (8 * (4 + 12) + 8) >> 4  # capped at 12


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10)])
def test_filter_fixed_points_and_sentinel(dtype, bd):
    L = O.lib()
    rng = np.random.default_rng(0)
    # flat area is a fixed point
    img = np.full((12, 12), 100 << (bd - 8), dtype)
    dst = np.zeros((8, 8), dtype)
    L.orc_cdef_filter_block_px(O.ptr(dst), 8, O.ptr(img, 2 * 12 + 2), 12, img.itemsize, 4 << (bd - 8),
                               2 << (bd - 8), 3, 5 + bd - 8, bd, 0, 0, 15)
    assert (dst == 100 << (bd - 8)).all()
    # zero strengths copy the input
    img = rng.integers(0, 1 << bd, (12, 12)).astype(dtype)
    L.orc_cdef_filter_block_px(O.ptr(dst), 8, O.ptr(img, 2 * 12 + 2), 12, img.itemsize, 0, 0, 0,
                               5 + bd - 8, bd, 0, 0, 15)
    np.testing.assert_array_equal(dst, img[2:10, 2:10])
    # with missing edges the result never exceeds the max of the real pixels (sentinel excluded
    # from max, cdef.rs:272-275) and never drops below their min
    for edges in range(16):
        for d in range(8):
            L.orc_cdef_filter_block_px(O.ptr(dst), 8, O.ptr(img, 2 * 12 + 2), 12, img.itemsize,
                                       7 << (bd - 8), 4 << (bd - 8), d, 6 + bd - 8, bd, 0, 0, edges)
            assert dst.max() <= img.max() and dst.min() >= img.min()


def np_constrain(diff, threshold, damping):
    """constrain() of AV1 7.15.3 over an int64 array of differences (threshold > 0)."""
    shift = max(0, damping - (int(threshold).bit_length() - 1))
    mag = np.abs(diff)
    v = np.clip(threshold - (mag >> shift), 0, mag)
    return np.where(diff < 0, -v, v)


def driver_thresholds(bd):
    """Every nonzero pri / sec threshold the frame drivers can hand constrain(): luma's adjust_strength of
    pri << cs in each variance bracket (var 0, then msb(var >> 6) = 0 .. 12 and beyond), chroma's pri << cs,
    and sec << cs with sec in {1, 2, 4} (3 -> 4)."""
    L = O.lib()
    cs = bd - 8
    vars_ = [0] + [64 << i for i in range(14)]
    thr = {L.orc_cdef_adjust_strength(p << cs, v) for p in range(16) for v in vars_}
    thr |= {p << cs for p in range(16)} | {s << cs for s in (1, 2, 4)}
    return sorted(t for t in thr if t)


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_sentinel_never_contributes_at_any_legal_damping(bd):
    """cdef_dev.cuh stores CDEF_VERY_LARGE as int16 -32768 where the reference stores u16 0x8000: for every
    threshold the drivers produce and every final damping they pass (luma 3..6 + cs, chroma one less), the
    sentinel's constrain() term is 0 in both encodings, it never wins `max`, and as unsigned it never wins
    `min`.  The damping at which the term first becomes nonzero is derived, and must lie above the legal range."""
    from tests.test_oracle_cdef_spec import spec_constrain
    cs = bd - 8
    maxv = (1 << bd) - 1
    x = np.arange(maxv + 1, dtype=np.int64)
    diffs = {"u16 0x8000": 0x8000 - x, "int16 -32768": -32768 - x}
    thresholds = driver_thresholds(bd)
    assert max(thresholds) == 15 << cs                          # bracket 12 rounds pri 15 back to itself
    for t in thresholds[::7]:                                   # the vector form is the specification's
        for d in (2 + cs, 6 + cs):
            want = [spec_constrain(int(v), t, d) for v in diffs["u16 0x8000"][::97]]
            np.testing.assert_array_equal(np_constrain(diffs["u16 0x8000"][::97], t, d), want)
    legal = range(2 + cs, 6 + cs + 1)
    first_nonzero = None
    for damping in range(2 + cs, 40):
        hit = any(np_constrain(diff, t, damping).any() for diff in diffs.values() for t in thresholds)
        if damping in legal:
            assert not hit, f"sentinel contributes at legal damping {damping}"
        if hit and first_nonzero is None:
            first_nonzero = damping
    assert first_nonzero is not None and first_nonzero > max(legal)
    print(f"{bd}-bit: the sentinel term is first nonzero at final damping {first_nonzero}, legal max {max(legal)}")
    s16 = np.int64(-32768)
    assert (np.maximum(x, s16) == x).all()                       # max ignores the int16 sentinel
    assert (np.minimum(x.astype(np.uint32), np.uint32(s16 & 0xFFFFFFFF)) == x).all()   # min as unsigned


def test_frame_driver_skip_copies_and_strength_zero_is_identity():
    rng = np.random.default_rng(1)
    W, H = 128, 72
    luma = rng.integers(0, 256, (H, W)).astype(np.uint8)
    skip8 = np.zeros((H // 8, W // 8), np.uint8)
    skip8[2, 3] = 1
    dirs, var = O.cdef_analyze_frame(luma, 8, skip8)
    assert dirs[2, 3] == 0 and var[2, 3] == 0
    sb = np.full((2, 2), 4 * 5 + 2, np.uint8)
    out = O.cdef_filter_plane(luma, 0, 0, 0, W, H, 8, 5, skip8, dirs, var, sb)
    np.testing.assert_array_equal(out[16:24, 24:32], luma[16:24, 24:32])
    assert (out != luma).any()
    out0 = O.cdef_filter_plane(luma, 0, 0, 0, W, H, 8, 5, skip8, dirs, var, np.zeros((2, 2), np.uint8))
    np.testing.assert_array_equal(out0, luma)
