"""b200_deblock_levels_dev / b200_deblock_filter_dev against the oracle, bit for bit: levels, tallies and the
filtered planes, with every pixel outside the items' working rects untouched, the inputs unchanged, every
host rejection launching nothing, and the chain levels -> filter -> b200_cdef_rdo_dev on the device equal to
oracle deblocking -> orc_cdef_rdo."""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_oracle_cdef_rdo import DEFAULT_STRENGTHS, cdef_rdo
from tests.test_oracle_deblock import orc_levels
from tests.test_oracle_deblock_spec import (LAYOUTS, PAD, make_planes, orc_filter, random_grid, state_array,
                                            working_rect)

pytestmark = pytest.mark.gpu


class DevPlanes:
    """Padded numpy planes mirrored on the device: `views` address pixel (0, 0) with PAD readable pixels all
    round, exactly like the arrays the oracle reads."""

    def __init__(self, c, arrays, layout):
        _, xdec, ydec = LAYOUTS[layout]
        self.c, self.allocs, self.views = c, [], []
        for p, a in enumerate(arrays):
            al = c.plane_from_host(a, 0)
            xd, yd = (xdec, ydec) if p else (0, 0)
            v = B.Plane()
            C.memmove(C.byref(v), C.byref(al), C.sizeof(B.Plane))
            v.data = al.data + ((PAD >> yd) * al.stride + (PAD >> xd)) * a.itemsize
            v.width, v.height, v.pad = a.shape[1] - 2 * (PAD >> xd), a.shape[0] - 2 * (PAD >> yd), PAD >> max(xd, yd)
            self.allocs.append(al)
            self.views.append(v)
        self.like = [np.empty_like(a) for a in arrays]

    def download(self):
        out = []
        for al, like in zip(self.allocs, self.like):
            o = np.empty_like(like)
            self.c.check(self.c.L.b200_plane_download(self.c.h, C.byref(al), o.ctypes.data, o.strides[0]))
            out.append(o)
        return out

    def free(self):
        for al in self.allocs:
            self.c.plane_free(al)


def frame_setup(rng, layout, bd, W, H, content="steps", deltas=False, skip_p=0.4, noise=6):
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    grid = random_grid(rng, w4, h4, layout, skip_p=skip_p, deltas=deltas)
    src = make_planes(rng, W, H, layout, bd, content)
    mx = (1 << bd) - 1
    rec = [np.clip(s.astype(np.int64) + rng.integers(-noise, noise + 1, s.shape) * (1 << (bd - 8)), 0, mx)
           .astype(s.dtype) for s in src]
    return grid, src, rec


def run_both(rng, layout, bd, grid, src, rec, items, st, levels=None):
    """Levels (unless given) and the filter on the device and in the oracle; asserts equality and returns the
    device's filtered planes."""
    _, xdec, ydec = LAYOUTS[layout]
    c = G.ctx()
    n = len(items)
    d_rec, d_src = DevPlanes(c, rec, layout), DevPlanes(c, src, layout)
    garbage = [rng.integers(0, 1 << bd, a.shape).astype(a.dtype) for a in rec]
    d_out = DevPlanes(c, garbage, layout)
    d_mi = G.to_dev(grid.view(np.uint8).reshape(-1))
    want_lv, want_t = orc_levels(rec, src, layout, bd, grid, items)
    if levels is None:
        d_lv = G.to_dev(np.full(n * 4, 0xAA, np.uint8))
        d_t = G.to_dev(np.full(n * 3 * 2 * 64, 7, np.int64))
        c.deblock_levels_dev(d_rec.views, d_src.views, xdec, ydec, bd, d_mi, grid.shape[1], items, d_lv, d_t)
        c.synchronize()
        got_lv = G.from_dev(d_lv, np.uint8).reshape(n, 4)
        got_t = G.from_dev(d_t, np.int64).reshape(n, 3, 2, 64)
        assert (got_t == want_t).all(), np.argwhere(got_t != want_t)[:5]
        assert (got_lv == want_lv).all(), (got_lv, want_lv)
        levels = want_lv
    else:
        levels = np.asarray(levels, np.uint8).reshape(n, 4)
        d_lv = G.to_dev(levels.reshape(-1).copy())
    c.deblock_filter_dev(d_rec.views, d_out.views, xdec, ydec, bd, st, d_lv, d_mi, grid.shape[1], items)
    c.synchronize()
    got = d_out.download()
    filt = [a.copy() for a in rec]
    orc_filter(filt, layout, bd, st, levels, grid, items)
    for p in range(len(rec)):
        want = garbage[p].copy()
        for it in items:
            x0, y0, x1, y1 = working_rect(it, p, xdec, ydec)
            xo, yo = PAD >> (xdec if p else 0), PAD >> (ydec if p else 0)
            want[yo + y0:yo + y1, xo + x0:xo + x1] = filt[p][yo + y0:yo + y1, xo + x0:xo + x1]
        assert (got[p] == want).all(), f"plane {p}: {np.argwhere(got[p] != want)[:5]}"
    for dp, a in ((d_rec, rec), (d_src, src)):
        assert all((g == w).all() for g, w in zip(dp.download(), a)), "an input plane changed"
    for dp in (d_rec, d_src, d_out):
        dp.free()
    return levels, got


def mixed_items(W, H):
    """A 2x1-superblock tile, a 1x1 area and a tile-grid of the rest, all on the superblock grid."""
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    return [(0, 0, 32, 16, W, H), (32, 0, 16, 16, W - 128, H), (48, 0, w4 - 48, 16, W - 192, H),
            (0, 16, 16, h4 - 16, W, H - 64), (16, 16, w4 - 16, h4 - 16, W - 64, H - 64)]


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_matches_the_oracle(layout, bd):
    rng = np.random.default_rng(bd * 7 + ord(layout[1]))
    W, H = 301, 197                                  # odd visible sizes at the right and bottom
    grid, src, rec = frame_setup(rng, layout, bd, W, H)
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    run_both(rng, layout, bd, grid, src, rec, [(0, 0, w4, h4, W, H)], state_array())
    run_both(rng, layout, bd, grid, src, rec, mixed_items(W, H), state_array())


@pytest.mark.parametrize("layout", ["420", "422", "444"])
def test_deltas_and_level_gates(layout):
    rng = np.random.default_rng(3)
    W, H = 250, 190
    grid, src, rec = frame_setup(rng, layout, 10, W, H, deltas=True)
    items = mixed_items(W, H)
    st = state_array(1, [3, -2, 5, -7, 1, 0, -3, 2], [4, -6], block=1, shift=2, multi=1)
    # both luma levels 0 with chroma levels set: a copy; one chroma plane off; deltas raising a 0 level
    levels = [[0, 0, 40, 40], [30, 0, 0, 25], [0, 12, 33, 0], [63, 63, 63, 63], [1, 2, 3, 4]]
    run_both(rng, layout, 10, grid, src, rec, items, st, levels)
    run_both(rng, layout, 10, grid, src, rec, items, state_array(1, [1] * 8, [2, -2], block=1, shift=1, multi=0),
             levels)
    run_both(rng, layout, 10, grid, src, rec, items, st)


@pytest.mark.parametrize("bd", [8, 10])
def test_1080p_420(bd):
    rng = np.random.default_rng(1080 + bd)
    W, H = 1920, 1080
    grid, src, rec = frame_setup(rng, "420", bd, W, H, skip_p=0.5)
    lv, _ = run_both(rng, "420", bd, grid, src, rec, [(0, 0, W // 4, ((H + 7) >> 3) * 2, W, H)], state_array())
    assert lv[0, :2].any()


def test_rejections_write_nothing():
    rng = np.random.default_rng(8)
    W, H, layout, bd = 128, 64, "420", 8
    _, xdec, ydec = LAYOUTS[layout]
    grid, src, rec = frame_setup(rng, layout, bd, W, H)
    c = G.ctx()
    d_rec, d_src = DevPlanes(c, rec, layout), DevPlanes(c, src, layout)
    garbage = [rng.integers(0, 256, a.shape).astype(a.dtype) for a in rec]
    d_out = DevPlanes(c, garbage, layout)
    d_mi = G.to_dev(grid.view(np.uint8).reshape(-1))
    d_lv = G.to_dev(np.full(8, 0xAA, np.uint8))
    d_t = G.to_dev(np.full(2 * 384, 7, np.int64))
    good = [(0, 0, 16, 16, W, H), (16, 0, 16, 16, W - 64, H)]
    ms = grid.shape[1]
    st = state_array()
    launches = c.launches
    bad_levels = [
        dict(items=[(8, 0, 16, 16, W, H)]),                          # off the superblock grid
        dict(items=[(0, 0, 0, 16, W, H)]),                           # empty
        dict(items=[(0, 0, 15, 16, W, H)]),                          # odd mi_w
        dict(items=[(0, 0, 16, 16, W, H), (0, 0, 16, 16, W, H)]),    # overlapping
        dict(items=[(0, 0, 16, 16, 0, H)]),                          # vis_w <= 0
        dict(items=[(16, 0, 32, 16, W - 64, H)]),                    # past mi_stride
        dict(items=[(0, 0, 16, 16, W, H), (0, 32, 16, 16, W, 8)]),  # outside the planes
        dict(bd=10), dict(planes=2), dict(xdec=0, ydec=1), dict(ms=8),
    ]
    for kw in bad_levels:
        args = dict(items=good, bd=bd, planes=3, xdec=xdec, ydec=ydec, ms=ms)
        args.update(kw)
        views = lambda d: d.views[:args["planes"]] if args["planes"] != 2 else d.views[:2]
        with pytest.raises(B.B200Error) as e:
            c.deblock_levels_dev(views(d_rec), views(d_src), args["xdec"], args["ydec"], args["bd"], d_mi,
                                 args["ms"], args["items"], d_lv, d_t)
        assert e.value.status == B.ERR_ARG, kw
        with pytest.raises(B.B200Error) as e:
            c.deblock_filter_dev(views(d_rec), views(d_out), args["xdec"], args["ydec"], args["bd"], st, d_lv, d_mi,
                                 args["ms"], args["items"])
        assert e.value.status == B.ERR_ARG, kw
    with pytest.raises(B.B200Error) as e:                            # out aliasing in
        c.deblock_filter_dev(d_rec.views, d_rec.views, xdec, ydec, bd, st, d_lv, d_mi, ms, good)
    assert e.value.status == B.ERR_ARG
    with pytest.raises(B.B200Error) as e:                            # block_delta_shift above 3
        c.deblock_filter_dev(d_rec.views, d_out.views, xdec, ydec, bd, state_array(block=1, shift=4), d_lv, d_mi,
                             ms, good)
    assert e.value.status == B.ERR_ARG
    c.deblock_levels_dev(d_rec.views, d_src.views, xdec, ydec, bd, d_mi, ms, [], d_lv, d_t)   # nothing to do
    c.deblock_filter_dev(d_rec.views, d_out.views, xdec, ydec, bd, st, d_lv, d_mi, ms, [])
    c.synchronize()
    assert (G.from_dev(d_lv, np.uint8) == 0xAA).all()
    assert (G.from_dev(d_t, np.int64) == 7).all()
    assert all((g == w).all() for g, w in zip(d_out.download(), garbage))
    assert c.launches == launches
    for dp in (d_rec, d_src, d_out):
        dp.free()


@pytest.mark.parametrize("layout,bd", [("420", 8), ("444", 10)])
def test_chain_into_cdef_rdo(layout, bd):
    """levels -> filter -> b200_cdef_rdo_dev with no host copy in between, against oracle deblocking ->
    orc_cdef_rdo over the same loop-restoration areas."""
    rng = np.random.default_rng(44 + bd)
    W, H = 200, 136
    planes, xdec, ydec = LAYOUTS[layout]
    grid, src, rec = frame_setup(rng, layout, bd, W, H)
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    areas = [(0, 0, 2, 2), (2, 0, 2, 2), (0, 2, 4, 1)]               # cdef / restoration areas, superblocks
    items = [(sx * 16, sy * 16, min(sw * 16, w4 - sx * 16), min(sh * 16, h4 - sy * 16), W - sx * 64, H - sy * 64)
             for sx, sy, sw, sh in areas]
    c = G.ctx()
    d_rec, d_src = DevPlanes(c, rec, layout), DevPlanes(c, src, layout)
    d_deb = DevPlanes(c, [np.zeros_like(a) for a in rec], layout)
    d_mi = G.to_dev(grid.view(np.uint8).reshape(-1))
    d_lv = G.to_dev(np.zeros(len(items) * 4, np.uint8))
    c.deblock_levels_dev(d_rec.views, d_src.views, xdec, ydec, bd, d_mi, grid.shape[1], items, d_lv)
    c.deblock_filter_dev(d_rec.views, d_deb.views, xdec, ydec, bd, state_array(), d_lv, d_mi, grid.shape[1], items)
    ystr, uvstr = DEFAULT_STRENGTHS, DEFAULT_STRENGTHS[::-1]
    n = len(areas)
    d_err = G.to_dev(np.full((n * 16, 8), np.iinfo(np.uint64).max, np.uint64))
    d_cost = G.to_dev(np.zeros((n * 16, 8)))
    d_best = G.to_dev(np.full(n * 16, 127, np.int8))
    c.cdef_rdo_dev(d_deb.views, d_src.views, None, xdec, ydec, W, H, bd, 4, 3, ystr, uvstr, None, None,
                   (16384,) * 3, 300.0, areas, None, d_err, d_cost, d_best)
    c.synchronize()
    levels, _ = orc_levels(rec, src, layout, bd, grid, items)
    deb = [a.copy() for a in rec]
    orc_filter(deb, layout, bd, state_array(), levels, grid, items)
    w8, h8 = (W + 7) & ~7, (H + 7) & ~7
    crop = lambda arrs: [np.ascontiguousarray(a[PAD >> (ydec if p else 0):, PAD >> (xdec if p else 0):]
                                              [:h8 >> (ydec if p else 0), :w8 >> (xdec if p else 0)])
                         for p, a in enumerate(arrs)]
    err, cost, best = cdef_rdo(crop(deb), crop(src), None, xdec, ydec, W, H, bd, 4, 3, ystr, uvstr, lam=300.0,
                               areas=areas)
    got_best = G.from_dev(d_best, np.int8)
    got_err = G.from_dev(d_err, np.uint64).reshape(n * 16, 8)
    assert (got_best == best[:n * 16]).all()
    dec = (best[:n * 16] >= 0) & (best[:n * 16] != 127)    # decided superblocks; 127: slot outside its area
    assert dec.any()
    assert (got_err[dec] == err[:n * 16][dec]).all()
    for dp in (d_rec, d_src, d_deb):
        dp.free()
