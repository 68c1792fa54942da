"""orc_deblock_levels (sse_optimize, deblock.rs:1553-1617) against a brute-force level search: for every level
0..63, every edge line of a plane is filtered at that level by the specification model of
tests/test_oracle_deblock_spec.py on the UNFILTERED reconstruction, and the squared error against the source
over the pixels that edge's filter can change is summed per plane and direction.  Those sums must equal the
oracle's prefix-summed tallies exactly, and the first minimum of each (luma per direction, chroma over
vertical + horizontal) must equal its levels.

One named difference from the filter: sse_h_edge passes `vertical = true` to deblock_size (deblock.rs:1257),
so the level search sizes a HORIZONTAL edge by the transform WIDTHS of the two blocks, where the filter
(filter_h_edge, :1210) uses the heights.  The oracle follows deblock.rs, so the brute force takes the sizes
the same way; test_horizontal_sizes_follow_the_transform_width shows the difference is real on a grid with
16x4 transforms (a horizontal edge the filter treats as 4-tap is searched as 14-tap, reaching 7 rows out).
"""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O
from tests.test_oracle_deblock_spec import (LAYOUTS, PAD, edge_decision, edge_positions, gather, items_array,
                                            make_planes, origin, random_grid, sample_filter)

MAX_LEVEL = 63


def orc_levels(rec, src, layout, bd, grid, items):
    """orc_deblock_levels over padded numpy planes -> (levels (n, 4) u8, tallies (n, 3, 2, 64) i64)."""
    L = O.lib()
    f = L.orc_deblock_levels
    f.restype = None
    n, xdec, ydec = LAYOUTS[layout]
    vpa, spa = C.c_void_p * 3, C.c_ssize_t * 3
    it = items_array(items)
    levels = np.full((len(it), 4), 0xAA, np.uint8)
    tally = np.full((len(it), 3, 2, 64), -1, np.int64)
    f(vpa(*[origin(a, p, xdec, ydec) for p, a in enumerate(rec)]), spa(*[a.shape[1] for a in rec]),
      vpa(*[origin(a, p, xdec, ydec) for p, a in enumerate(src)]), spa(*[a.shape[1] for a in src]),
      C.c_int(rec[0].itemsize), C.c_int(n), C.c_int(xdec), C.c_int(ydec), C.c_int(bd),
      C.c_void_p(grid.ctypes.data), C.c_ssize_t(grid.shape[1]), C.c_void_p(it.ctypes.data), C.c_size_t(len(it)),
      C.c_void_p(levels.ctypes.data), C.c_void_p(tally.ctypes.data))
    return levels, tally


def window(fsize, plane):
    """Columns of the 14-tap line (p6 .. q6) a filter of this size can change."""
    return (1, 13) if (plane == 0 and fsize == 16) else (4, 10) if (plane == 0 and fsize == 8) else (5, 9)


def brute_tallies(rec, src, layout, bd, grid, item, h_by_width=True):
    """(3, 2, 64) tallies of one item by filtering every line at every level."""
    n, xdec, ydec = LAYOUTS[layout]
    out = np.zeros((3, 2, 64), np.int64)
    for p in range(n):
        xd, yd = (xdec, ydec) if p else (0, 0)
        ox, oy = (PAD >> xd) + ((item[0] * 4) >> xd), (PAD >> yd) + ((item[1] * 4) >> yd)
        for d, vertical in enumerate((True, False)):
            groups = {}
            for x, y in edge_positions(item, p, xdec, ydec, vertical):
                dec = edge_decision(grid, item, p, xdec, ydec, x, y, vertical,
                                    size_from_width=True if h_by_width else None)
                if dec is None:
                    continue
                px, py = (x * 4) >> xd, (y * 4) >> yd
                groups.setdefault(dec[0], []).append((gather(rec[p], ox, oy, px, py, vertical),
                                                      gather(src[p], ox, oy, px, py, vertical)))
            for fsize, lines in groups.items():
                F = np.concatenate([a for a, _ in lines])
                S = np.concatenate([b for _, b in lines])
                lo, hi = window(fsize, p)
                out[p, d, 0] += ((S[:, lo:hi] - F[:, lo:hi]) ** 2).sum()
                for lvl in range(1, MAX_LEVEL + 1):
                    G = sample_filter(F, fsize, p, np.full(len(F), lvl), bd)
                    out[p, d, lvl] += ((S[:, lo:hi] - G[:, lo:hi]) ** 2).sum()
    return out


def first_min(t):
    return int(np.flatnonzero(t == t.min())[0])


def check(rng, layout, bd, W, H, items, content="steps", grid=None, noise=6):
    n, xdec, ydec = LAYOUTS[layout]
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    if grid is None:
        grid = random_grid(rng, w4, h4, layout)
    src = make_planes(rng, W, H, layout, bd, content)
    mx = (1 << bd) - 1
    rec = [np.clip(s.astype(np.int64) + rng.integers(-noise, noise + 1, s.shape) * (1 << (bd - 8)), 0, mx)
           .astype(s.dtype) for s in src]
    levels, tally = orc_levels(rec, src, layout, bd, grid, items)
    for k, it in enumerate(items):
        want = brute_tallies(rec, src, layout, bd, grid, it)
        assert (tally[k] == want).all(), np.argwhere(tally[k] != want)[:5]
        assert levels[k, 0] == first_min(want[0, 0]) and levels[k, 1] == first_min(want[0, 1])
        for p in (1, 2):
            assert levels[k, p + 1] == (first_min(want[p, 0] + want[p, 1]) if p < n else 0)
    return levels, tally


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_frame_sizes_off_the_4_and_8_grid(layout, bd):
    rng = np.random.default_rng(bd * 10 + len(layout) + ord(layout[1]))
    W, H = 46, 30                                    # neither a multiple of 4 nor of 8
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    levels, _ = check(rng, layout, bd, W, H, [(0, 0, w4, h4, W, H)])
    assert levels[0, :2].any(), "the search never left level 0"


@pytest.mark.parametrize("layout", ["420", "422", "444"])
def test_tile_and_area_items_off_the_origin(layout):
    rng = np.random.default_rng(5)
    W, H = 150, 134
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    items = [(0, 0, 16, 16, W, H), (16, 0, w4 - 16, 16, W - 64, H), (0, 16, 32, h4 - 16, W, H - 64),
             (32, 16, w4 - 32, h4 - 16, W - 128, H - 64)]
    check(rng, layout, 10, W, H, items)


def test_ties_take_the_first_level():
    """Flat content: no filter changes a flat line, so every level ties and level 0 wins."""
    rng = np.random.default_rng(9)
    levels, tally = check(rng, "420", 8, 64, 40, [(0, 0, 16, 10, 64, 40)], content="flat", noise=0)
    assert (levels == 0).all()
    assert (tally[0, :, :, :] == tally[0, :, :, :1]).all()


def test_horizontal_sizes_follow_the_transform_width():
    rng = np.random.default_rng(21)
    W, H = 64, 64
    grid = random_grid(rng, 16, 16, "444", skip_p=0.0)
    grid["bsize"] = 17                               # BLOCK_16X4
    grid["txsize"] = 14                              # TX_16X4: 4 mi wide, 1 mi high
    item = (0, 0, 16, 16, W, H)
    src = make_planes(np.random.default_rng(1), W, H, "400", 8, "steps")
    rec = [np.clip(s.astype(np.int64) + 5, 0, 255).astype(np.uint8) for s in src]
    _, tally = orc_levels(rec, src, "400", 8, grid, [item])
    by_width = brute_tallies(rec, src, "400", 8, grid, item)
    by_height = brute_tallies(rec, src, "400", 8, grid, item, h_by_width=False)
    assert (tally[0] == by_width).all()
    assert (by_width[0, 0] == by_height[0, 0]).all()          # vertical edges agree
    assert (by_width[0, 1] != by_height[0, 1]).any()          # horizontal edges do not
