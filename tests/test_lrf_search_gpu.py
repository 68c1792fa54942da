"""b200_lrf_search_dev (the restoration search of rdo_loop_decision) against orc_lrf_search, bit for bit: the
winner, the f64 bit patterns of every cost, changed, every candidate's xqd and error; inputs and the slots the
call does not reach are left untouched."""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_oracle_lrf_search import CONFIGS, LAYOUTS, areas_and_items, lrf_search, make_frame

pytestmark = pytest.mark.gpu
PAD = 8


def download(plane, like):
    c = G.ctx()
    out = np.empty_like(like)
    c.check(c.L.b200_plane_download(c.h, C.byref(plane), out.ctypes.data, out.strides[0]))
    return out


def run_both(lin, src, layout, W, H, bd, us, reduced, areas, items, imp=None, dist_scale=(16384,) * 3, lam=0.0):
    c = G.ctx()
    n = len(items)
    d_in = [c.plane_from_host(a, PAD) for a in lin]
    d_src = [c.plane_from_host(a, PAD) for a in src]
    d_best = G.to_dev(np.full(n, 0xEE, np.uint8).repeat(12))
    d_cost, d_changed = G.to_dev(np.full(n, np.nan)), G.to_dev(np.full(n, 7, np.uint8))
    d_xqd = G.to_dev(np.full((n, 16, 2), 127, np.int8))
    d_err = G.to_dev(np.full((n, 17), np.iinfo(np.uint64).max, np.uint64))
    d_cc = G.to_dev(np.full((n, 17), np.nan))
    _, xdec, ydec = LAYOUTS[layout]
    c.lrf_search_dev(d_in, d_src, xdec, ydec, W, H, bd, us, reduced, G.to_dev(imp) if imp is not None else None,
                     dist_scale, lam, areas, items, d_best, d_cost, d_changed, d_xqd, d_err, d_cc)
    c.synchronize()
    want = lrf_search(lin, src, layout, W, H, bd, us, reduced, areas, items, imp, dist_scale, lam)
    got = (G.from_dev(d_best, np.uint8)[:12 * n].view(B.LRF_UNIT_DTYPE), G.from_dev(d_cost, np.float64)[:n],
           G.from_dev(d_changed, np.uint8)[:n], G.from_dev(d_xqd, np.int8)[:n * 32].reshape(n, 16, 2),
           G.from_dev(d_err, np.uint64)[:n * 17].reshape(n, 17), G.from_dev(d_cc, np.float64)[:n * 17].reshape(n, 17))
    assert (got[0].view(np.uint8) == want[0].view(np.uint8)).all()
    assert (got[1].view(np.uint64) == want[1].view(np.uint64)).all()
    assert (got[2] == want[2]).all()
    assert (got[3] == want[3]).all()
    assert (got[4] == want[4]).all()
    assert (got[5].view(np.uint64) == want[5].view(np.uint64)).all()
    for d, h in zip(d_in + d_src, lin + src):                # inputs unchanged
        assert (download(d, h) == h).all()
        c.plane_free(d)
    return got


@pytest.mark.parametrize("layout,uy,uc", CONFIGS)
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_matches_the_oracle(layout, uy, uc, bd):
    rng = np.random.default_rng(hash((layout, uy, uc, bd, 1)) & 0xFFFF)
    W, H = (131, 97) if uy <= 128 else (263, 141)
    lin, src = make_frame(rng, W, H, layout, bd)
    us = [uy, uc, uc][:LAYOUTS[layout][0]]
    areas, items = areas_and_items(rng, W, H, layout, us, incoming="mixed")
    imp = rng.integers(1 << 12, 1 << 16, ((H + 7) // 8, (W + 7) // 8)).astype(np.uint32) if bd != 10 else None
    got = run_both(lin, src, layout, W, H, bd, us, bd == 10, areas, items, imp, (16384, 20000, 12000), 300.0)
    if bd == 10:                                             # reduced sets: the even sets' slots stay untouched
        assert (got[3][:, 0::2] == 127).all() and (got[4][:, 1::2] == np.iinfo(np.uint64).max).all()


@pytest.mark.parametrize("content", ["flat", "extreme"])
def test_flat_extreme_and_carried_costs(content):
    rng = np.random.default_rng(11)
    for bd in (8, 12):
        W, H = 200, 136
        lin, src = make_frame(rng, W, H, "420", bd, content)
        for cost in (-1.0, 0.0):
            areas, items = areas_and_items(rng, W, H, "420", [128, 128, 128], incoming="mixed", cost=cost)
            run_both(lin, src, "420", W, H, bd, [128, 128, 128], False, areas, items, lam=50.0)


@pytest.mark.parametrize("uy", [64, 128, 256])
def test_1080p_420(uy):
    rng = np.random.default_rng(uy)
    W, H = 1920, 1080
    lin, src = make_frame(rng, W, H, "420", 10)
    us = [uy, uy >> 1, uy >> 1]
    areas, items = areas_and_items(rng, W, H, "420", us, incoming="mixed")
    if uy == 64:
        assert len(items) == 1530
    run_both(lin, src, "420", W, H, 10, us, uy == 128, areas, items, lam=1000.0)


def test_host_rejections_launch_nothing():
    rng = np.random.default_rng(2)
    W, H = 128, 128
    lin, src = make_frame(rng, W, H, "420", 8)
    c = G.ctx()
    d_in = [c.plane_from_host(a, PAD) for a in lin]
    d_src = [c.plane_from_host(a, PAD) for a in src]
    small = [c.plane_from_host(a[:64, :64], PAD) for a in lin]
    us = [64, 32, 32]
    areas, items = areas_and_items(rng, W, H, "420", us)
    n = len(items)
    d_best, d_cost, d_ch = G.dev_empty(12 * n), G.dev_empty(8 * n), G.dev_empty(n)
    ok = dict(lrf_in=d_in, src=d_src, xdec=1, ydec=1, frame_w=W, frame_h=H, bit_depth=8, unit_size=us,
              reduced_sets=0, d_imp_scales=None, dist_scale=(16384,) * 3, lam=1.0, areas=areas, items=items,
              d_best=d_best, d_cost=d_cost, d_changed=d_ch)
    c.lrf_search_dev(**ok)
    c.synchronize()

    def item(**kw):
        it = items.copy()
        for k, v in kw.items():
            if k in ("type", "set", "xqd"):
                it[0]["incoming"][k] = v
            else:
                it[0][k] = v
        return it
    bad = [dict(bit_depth=10), dict(bit_depth=9), dict(xdec=0, ydec=1), dict(lrf_in=d_in[:2]), dict(frame_w=0),
           dict(lrf_in=small), dict(src=small), dict(unit_size=[48, 32, 32]), dict(unit_size=[64, 16, 16]),
           dict(unit_size=[512, 256, 256]), dict(unit_size=[64, 256, 256]), dict(areas=[(0, 0, 5, 1)] + areas[1:]),
           dict(areas=[(1, 1, 2, 1)] + areas[1:]), dict(areas=[]), dict(items=item(area=len(areas))),
           dict(items=item(area=-1)), dict(items=item(plane=3)), dict(items=item(lru_x=1)), dict(items=item(lru_y=-1)),
           dict(items=item(type=1)), dict(items=item(type=3)), dict(items=item(type=2, set=16)),
           dict(items=item(type=2, xqd=[-97, 0])), dict(items=item(type=2, xqd=[0, 96])),
           dict(items=item(sgrproj_ref=[32, 0])), dict(items=item(sgrproj_ref=[0, -33])), dict(d_best=None),
           dict(d_cost=None), dict(d_changed=None)]
    for b in bad:
        n0 = c.launches
        with pytest.raises(B.B200Error) as e:
            c.lrf_search_dev(**{**ok, **b})
        assert e.value.status == B.ERR_ARG, b
        assert c.launches == n0, b
    n0 = c.launches
    c.lrf_search_dev(**{**ok, "items": items[:0]})
    assert c.launches == n0
    for p in d_in + d_src + small:
        c.plane_free(p)


@pytest.mark.parametrize("layout,bd", [("420", 8), ("444", 10)])
@pytest.mark.parametrize("cdef_on", [True, False])
def test_chain_deblock_cdef_search(layout, bd, cdef_on):
    """deblock levels -> deblock filter -> (CDEF pass) -> restoration search enqueued with one final synchronise,
    against the oracle's chain: the search reads the CDEF pass's output, or the deblocked frame with CDEF off."""
    from tests.test_deblock_gpu import DevPlanes as DbDevPlanes
    from tests.test_deblock_gpu import frame_setup
    from tests.test_oracle_cdef_rdo import DEFAULT_STRENGTHS, cdef_rdo
    from tests.test_oracle_deblock import orc_levels
    from tests.test_oracle_deblock_spec import PAD as DB_PAD
    from tests.test_oracle_deblock_spec import orc_filter, state_array

    rng = np.random.default_rng(90 + bd + cdef_on)
    W, H = 200, 136
    n, xdec, ydec = LAYOUTS[layout]
    grid, src, rec = frame_setup(rng, layout, bd, W, H)
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    db_items = [(0, 0, w4, h4, W, H)]
    us = [64, 32, 32] if layout == "420" else [64, 64, 64]
    areas, items = areas_and_items(rng, W, H, layout, us, incoming="mixed")
    ni, dist_scale, lam = len(items), (16384, 18000, 18000), 400.0

    c = G.ctx()
    d_rec, d_src = DbDevPlanes(c, rec, layout), DbDevPlanes(c, src, layout)
    d_deb = DbDevPlanes(c, [np.zeros_like(a) for a in rec], layout)
    d_cdef = DbDevPlanes(c, [np.zeros_like(a) for a in rec], layout)
    d_mi = G.to_dev(grid.view(np.uint8).reshape(-1))
    d_lv = G.dev_empty(4)
    c.deblock_levels_dev(d_rec.views, d_src.views, xdec, ydec, bd, d_mi, grid.shape[1], db_items, d_lv)
    c.deblock_filter_dev(d_rec.views, d_deb.views, xdec, ydec, bd, state_array(), d_lv, d_mi, grid.shape[1], db_items)
    if cdef_on:
        na = len(areas)
        c.cdef_rdo_dev(d_deb.views, d_src.views, d_cdef.views, xdec, ydec, W, H, bd, 4, 2, DEFAULT_STRENGTHS,
                       DEFAULT_STRENGTHS, None, None, dist_scale, lam, areas, None, G.dev_empty(na * 16 * 8 * 8),
                       G.dev_empty(na * 16 * 8 * 8), G.dev_empty(na * 16))
    lrf_in = d_cdef if cdef_on else d_deb
    d_best, d_cost, d_changed = G.dev_empty(12 * ni), G.dev_empty(8 * ni), G.dev_empty(ni)
    d_err = G.dev_empty(8 * 17 * ni)
    c.lrf_search_dev(lrf_in.views, d_src.views, xdec, ydec, W, H, bd, us, False, None, dist_scale, lam, areas,
                     items, d_best, d_cost, d_changed, None, d_err, None)
    c.synchronize()

    levels, _ = orc_levels(rec, src, layout, bd, grid, db_items)
    deb = [a.copy() for a in rec]
    orc_filter(deb, layout, bd, state_array(), levels, grid, db_items)

    def frame8(a, p):                                       # pixel (0, 0) at [0, 0], the frame rounded up to 8
        xd, yd = (xdec, ydec) if p else (0, 0)
        return np.ascontiguousarray(a[DB_PAD >> yd:, DB_PAD >> xd:][:((H + 7) & ~7) >> yd, :((W + 7) & ~7) >> xd])
    deb8, src8 = [frame8(a, p) for p, a in enumerate(deb)], [frame8(a, p) for p, a in enumerate(src)]
    if cdef_on:
        lin = [np.zeros_like(a) for a in deb8]
        cdef_rdo(deb8, src8, lin, xdec, ydec, W, H, bd, 4, 2, DEFAULT_STRENGTHS, DEFAULT_STRENGTHS, None, None,
                 dist_scale, lam, areas)
    else:
        lin = deb8
    want = lrf_search(lin, src8, layout, W, H, bd, us, False, areas, items, None, dist_scale, lam)
    assert (G.from_dev(d_best, np.uint8)[:12 * ni] == want[0].view(np.uint8)).all()
    assert (G.from_dev(d_cost, np.float64)[:ni].view(np.uint64) == want[1].view(np.uint64)).all()
    assert (G.from_dev(d_changed, np.uint8)[:ni] == want[2]).all()
    assert (G.from_dev(d_err, np.uint64)[:17 * ni].reshape(ni, 17) == want[4]).all()
    for dp in (d_rec, d_src, d_deb, d_cdef):
        dp.free()
