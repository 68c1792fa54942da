"""A second source for the oracle's CDEF: CDEF is AV1-normative (the decoder must reproduce it bit for bit), so
the AV1 specification's pseudo-code is an independent statement of what src/cdef.rs computes.  The reference holds
no stored vectors for cdef_find_dir / cdef_filter_block ("parity unpinned", SURVEY 8c); here the spec's
"CDEF direction process" (7.15.2) and "CDEF filter process" (7.15.3) are written out in plain Python - from the
specification's structure (tap tables, Div_Table, constrain, the 4-bit rounding, the clip to the neighbourhood's
min / max, availability instead of a sentinel), not from the reference's code - and compared with oracle/cdef.c on
random blocks, all 8 directions, every edge mask, the three block shapes and 8 / 10 / 12 bit."""
import numpy as np
import pytest

from tests import oracle_lib as O

# AV1 spec: Cdef_Directions[8][2][2] = (dy, dx) of tap k = 0, 1 in direction d
CDEF_DIRECTIONS = [[(-1, 1), (-2, 2)], [(0, 1), (-1, 2)], [(0, 1), (0, 2)], [(0, 1), (1, 2)],
                   [(1, 1), (2, 2)], [(1, 0), (2, 1)], [(1, 0), (2, 0)], [(1, 0), (2, -1)]]
CDEF_PRI_TAPS = [[4, 2], [3, 3]]
CDEF_SEC_TAPS = [2, 1]
DIV_TABLE = [0, 840, 420, 280, 210, 168, 140, 120, 105]


def floor_log2(x):
    return x.bit_length() - 1


def spec_constrain(diff, threshold, damping):
    if threshold == 0:
        return 0
    adj = max(0, damping - floor_log2(threshold))
    mag = abs(diff)
    v = max(0, min(mag, threshold - (mag >> adj)))
    return -v if diff < 0 else v


def spec_direction_costs(block, bit_depth):
    """7.15.2: the eight direction costs."""
    cost = [0] * 8
    partial = [[0] * 15 for _ in range(8)]
    for i in range(8):
        for j in range(8):
            x = (int(block[i][j]) >> (bit_depth - 8)) - 128
            partial[0][i + j] += x
            partial[1][i + j // 2] += x
            partial[2][i] += x
            partial[3][3 + i - j // 2] += x
            partial[4][7 + i - j] += x
            partial[5][3 - i // 2 + j] += x
            partial[6][j] += x
            partial[7][i // 2 + j] += x
    for i in range(8):
        cost[2] += partial[2][i] * partial[2][i]
        cost[6] += partial[6][i] * partial[6][i]
    cost[2] *= DIV_TABLE[8]
    cost[6] *= DIV_TABLE[8]
    for i in range(7):
        cost[0] += (partial[0][i] * partial[0][i] + partial[0][14 - i] * partial[0][14 - i]) * DIV_TABLE[i + 1]
        cost[4] += (partial[4][i] * partial[4][i] + partial[4][14 - i] * partial[4][14 - i]) * DIV_TABLE[i + 1]
    cost[0] += partial[0][7] * partial[0][7] * DIV_TABLE[8]
    cost[4] += partial[4][7] * partial[4][7] * DIV_TABLE[8]
    for i in (1, 3, 5, 7):
        for j in range(5):
            cost[i] += partial[i][3 + j] * partial[i][3 + j]
        cost[i] *= DIV_TABLE[8]
        for j in range(3):
            cost[i] += (partial[i][j] * partial[i][j] + partial[i][10 - j] * partial[i][10 - j]) * DIV_TABLE[2 * j + 2]
    return cost


def spec_direction(block, bit_depth):
    """7.15.2: returns (yDir, var)."""
    cost = spec_direction_costs(block, bit_depth)
    best, ydir = 0, 0
    for d in range(8):
        if cost[d] > best:
            best, ydir = cost[d], d
    return ydir, (best - cost[(ydir + 4) & 7]) >> 10


def spec_filter(img, w, h, pri, sec, d, damping, bit_depth, edges):
    """7.15.3 on the block at img[2:2+h, 2:2+w]; a tap is available when it lies inside the block or inside the
    2-pixel border on a side whose edge bit (L = 1, R = 2, T = 4, B = 8: that neighbour exists) is set."""
    cs = bit_depth - 8

    def avail(y, x):
        if not (-2 <= y < h + 2 and -2 <= x < w + 2):
            return False
        return (y >= 0 or edges & 4) and (y < h or edges & 8) and (x >= 0 or edges & 1) and (x < w or edges & 2)

    out = np.zeros((h, w), img.dtype)
    for i in range(h):
        for j in range(w):
            x = int(img[2 + i][2 + j])
            total, mx, mn = 0, x, x
            for k in range(2):
                for sign in (-1, 1):
                    dy, dx = CDEF_DIRECTIONS[d][k]
                    y1, x1 = i + sign * dy, j + sign * dx
                    if avail(y1, x1):
                        p = int(img[2 + y1][2 + x1])
                        total += CDEF_PRI_TAPS[(pri >> cs) & 1][k] * spec_constrain(p - x, pri, damping)
                        mx, mn = max(mx, p), min(mn, p)
                    for off in (-2, 2):
                        dy2, dx2 = CDEF_DIRECTIONS[(d + off) & 7][k]
                        y2, x2 = i + sign * dy2, j + sign * dx2
                        if avail(y2, x2):
                            s = int(img[2 + y2][2 + x2])
                            total += CDEF_SEC_TAPS[k] * spec_constrain(s - x, sec, damping)
                            mx, mn = max(mx, s), min(mn, s)
            out[i][j] = max(mn, min(mx, x + ((8 + total - (1 if total < 0 else 0)) >> 4)))
    return out


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_direction_search_equals_the_specification(bd):
    rng = np.random.default_rng(100 + bd)
    dtype = np.uint8 if bd == 8 else np.uint16
    for trial in range(300):
        kind = trial % 3
        if kind == 0:
            blk = rng.integers(0, 1 << bd, (8, 8))
        elif kind == 1:     # oriented texture + noise: real, close contests between neighbouring directions
            i, j = np.mgrid[0:8, 0:8]
            a, b = rng.integers(-3, 4, 2)
            blk = ((np.sin((a * i + b * j) * 0.7 + rng.random() * 6) * 0.4 + 0.5) * ((1 << bd) - 1)
                   + rng.normal(0, 6 << (bd - 8), (8, 8)))
        else:               # nearly flat: ties and tiny variances
            blk = (1 << (bd - 1)) + rng.integers(-2, 3, (8, 8))
        blk = np.clip(np.rint(blk), 0, (1 << bd) - 1).astype(dtype)
        assert O.cdef_find_dir(blk, bd) == spec_direction(blk, bd), trial


@pytest.mark.parametrize("bd", [8, 10, 12])
@pytest.mark.parametrize("xdec,ydec", [(0, 0), (1, 1), (1, 0)])
def test_filter_equals_the_specification(bd, xdec, ydec):
    L = O.lib()
    rng = np.random.default_rng(7 * bd + 2 * xdec + ydec)
    dtype = np.uint8 if bd == 8 else np.uint16
    w, h = 8 >> xdec, 8 >> ydec
    cs = bd - 8
    for trial in range(40):
        smooth = trial % 2 == 0     # small differences exercise the threshold - (mag >> shift) arm, noise the clip
        base = rng.integers(0, 1 << bd, (12, 12)).astype(np.float64)
        if smooth:
            base = (1 << (bd - 1)) + rng.normal(0, 5 << cs, (12, 12))
        img = np.ascontiguousarray(np.clip(np.rint(base), 0, (1 << bd) - 1).astype(dtype))
        for edges in range(16):
            d = int(rng.integers(0, 8))
            pri = int(rng.integers(0, 16)) << cs
            sec = int(rng.choice([0, 1, 2, 4])) << cs
            damping = int(rng.integers(3, 7)) + cs - (1 if xdec else 0)
            dst = np.zeros((h, w), dtype)
            L.orc_cdef_filter_block_px(O.ptr(dst), w, O.ptr(img, 2 * 12 + 2), 12, img.itemsize, pri, sec, d,
                                       damping, bd, xdec, ydec, edges)
            want = spec_filter(img, w, h, pri, sec, d, damping, bd, edges)
            np.testing.assert_array_equal(dst, want, err_msg=f"trial {trial} edges {edges} d {d} pri {pri} sec {sec}")
