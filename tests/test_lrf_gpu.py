"""b200_lrf_filter_dev against orc_lrf_filter_frame, bit for bit over every plane's crop, with every pixel
outside the crops untouched, the inputs unchanged, every host rejection launching nothing, and the chain
deblock filter -> CDEF -> loop restoration on the device equal to the oracle's chain."""
import ctypes as C

import numpy as np
import pytest
import torch

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_deblock_gpu import DevPlanes as DbDevPlanes
from tests.test_deblock_gpu import frame_setup
from tests.test_oracle_deblock_spec import PAD as DB_PAD
from tests.test_oracle_deblock_spec import orc_filter, state_array
from tests.test_oracle_lrf_spec import (LAYOUTS, PAD, XQD_MAX, crop, dec, make_frame, orc_lrf, random_units,
                                        unit_grid)

pytestmark = pytest.mark.gpu


class DevPlanes:
    """Padded numpy planes mirrored on the device; `views` address pixel (0, 0) with PAD readable all round."""

    def __init__(self, c, arrays):
        self.c, self.allocs, self.views = c, [], []
        for a in arrays:
            al = c.plane_from_host(a, 0)
            v = B.Plane()
            C.memmove(C.byref(v), C.byref(al), C.sizeof(B.Plane))
            v.data = al.data + (PAD * al.stride + PAD) * a.itemsize
            v.width, v.height, v.pad = a.shape[1] - 2 * PAD, a.shape[0] - 2 * PAD, PAD
            self.allocs.append(al)
            self.views.append(v)
        self.like = arrays

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


def run_both(rng, layout, bd, W, H, us, units, content="random", enable_cdef=1, same=False, frame=None):
    _, xdec, ydec = LAYOUTS[layout]
    cd, db = frame if frame is not None else make_frame(rng, W, H, layout, bd, content)
    if same:
        db = cd
    want = orc_lrf(cd, db, layout, bd, W, H, enable_cdef, us, units)
    c = G.ctx()
    d_cd = DevPlanes(c, cd)
    d_db = d_cd if same else DevPlanes(c, db)
    garbage = [rng.integers(0, 1 << bd, a.shape).astype(a.dtype) for a in cd]
    d_out = DevPlanes(c, garbage)
    n0 = c.launches
    c.lrf_filter_dev(d_cd.views, d_db.views, d_out.views, xdec, ydec, W, H, bd, enable_cdef, us, units)
    c.synchronize()
    assert c.launches == n0 + 1
    got = d_out.download()
    for p in range(len(cd)):
        cw, ch = crop(W, H, p, layout)
        exp = garbage[p].copy()
        exp[PAD:PAD + ch, PAD:PAD + cw] = want[p][PAD:PAD + ch, PAD:PAD + cw]
        assert (got[p] == exp).all(), f"plane {p}: {np.argwhere(got[p] != exp)[:5] - PAD}"
    for dp, a in ((d_cd, cd), (d_db, db)):
        assert all((g == w).all() for g, w in zip(dp.download(), a)), "an input plane changed"
    for dp in {id(d_cd): d_cd, id(d_db): d_db, id(d_out): d_out}.values():
        dp.free()


def any_unit_sizes(rng, layout):
    """what the call accepts: any power of two 32..256 per plane"""
    return [int(rng.choice([32, 64, 128, 256])) for _ in range(LAYOUTS[layout][0])]


def mixed(rng, W, H, layout, us, **kw):
    return [random_units(rng, *unit_grid(W, H, p, layout, us[p]), **kw) for p in range(len(us))]


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_matches_the_oracle(layout, bd):
    rng = np.random.default_rng(bd * 13 + ord(layout[1]))
    for W, H in ((203, 139), (32, 32), (33, 35), (383, 71)):
        for content in ("random", "edges"):
            us = any_unit_sizes(rng, layout)
            run_both(rng, layout, bd, W, H, us, mixed(rng, W, H, layout, us), content)


@pytest.mark.parametrize("layout", ["420", "422"])
def test_every_set_taps_at_their_ends_and_short_frames(layout):
    rng = np.random.default_rng(7)
    for bd in (8, 12):
        for W, H in ((150, 100), (90, 40), (64, 50)):
            us = any_unit_sizes(rng, layout)
            run_both(rng, layout, bd, W, H, us, mixed(rng, W, H, layout, us, ends=True), "edges")
        W, H = 96, 64
        for s in range(16):
            units = [np.zeros(unit_grid(W, H, p, layout, 32), B.LRF_UNIT_DTYPE) for p in range(3)]
            for u in units:
                u["type"], u["set"], u["xqd"] = 2, s, (-96, XQD_MAX[1])
            run_both(rng, layout, bd, W, H, [32] * 3, units)


@pytest.mark.parametrize("bd", [8, 10])
def test_1080p_420(bd):
    rng = np.random.default_rng(1080 + bd)
    W, H = 1920, 1080
    for us in ([64, 32, 32], [256, 256, 256]):   # RestorationState::new's small and large 1080p units
        for kinds in ((2,), (1,), (0, 1, 2)):
            run_both(rng, "420", bd, W, H, us, mixed(rng, W, H, "420", us, kinds=kinds), "smooth")


def test_enable_cdef_and_shared_inputs():
    rng = np.random.default_rng(3)
    W, H = 211, 97
    for layout in ("420", "444"):
        us = any_unit_sizes(rng, layout)
        units = mixed(rng, W, H, layout, us)
        run_both(rng, layout, 10, W, H, us, units, enable_cdef=0)
        run_both(rng, layout, 10, W, H, us, units, enable_cdef=1)
        run_both(rng, layout, 10, W, H, us, units, same=True)


def test_rejections_launch_nothing():
    rng = np.random.default_rng(9)
    W, H, layout, bd = 96, 80, "420", 8
    cd, db = make_frame(rng, W, H, layout, bd)
    c = G.ctx()
    d_cd, d_db, d_out = DevPlanes(c, cd), DevPlanes(c, db), DevPlanes(c, [np.zeros_like(a) for a in cd])
    us = [64, 32, 32]
    good = mixed(rng, W, H, layout, us)
    before = d_out.download()

    def rejected(**kw):
        a = dict(cdeffed=d_cd.views, deblocked=d_db.views, out=d_out.views, xdec=1, ydec=1, frame_w=W, frame_h=H,
                 bit_depth=bd, enable_cdef=1, unit_size=us, units=good)
        a.update(kw)
        n0 = c.launches
        with pytest.raises(B.B200Error) as e:
            c.lrf_filter_dev(**a)
        assert e.value.status == B.ERR_ARG and c.launches == n0

    def with_unit(p, **fields):
        u = [x.copy() for x in good]
        for k, v in fields.items():
            u[p].reshape(-1)[0][k] = v
        return u

    rejected(bit_depth=10)                                  # bpp does not match
    rejected(bit_depth=9)
    rejected(xdec=0, ydec=1)                                # not a layout
    rejected(frame_w=31)
    rejected(frame_h=31)
    rejected(frame_w=W + 2)                                 # planes smaller than the crop
    rejected(unit_size=[48, 32, 32])
    rejected(unit_size=[64, 16, 16])
    rejected(unit_size=[512, 32, 32])
    rejected(out=d_db.views)                                # out overlaps an input
    rejected(out=[d_out.views[0], d_cd.views[1], d_out.views[2]])
    rejected(units=with_unit(0, type=3))
    rejected(units=with_unit(1, type=2, set=16))
    rejected(units=with_unit(2, type=2, set=0, xqd=(-97, 0)))
    rejected(units=with_unit(0, type=2, set=0, xqd=(0, 96)))
    rejected(units=with_unit(1, type=1, coeffs=((11, 0, 0), (0, 0, 0))))
    rejected(units=with_unit(2, type=1, coeffs=((0, 0, 0), (0, 0, 47))))
    rejected(units=with_unit(0, type=1, coeffs=((0, -24, 0), (0, 0, 0))))
    n0 = c.launches
    cds, dbs, outs = c._plane_array(d_cd.views), c._plane_array(d_db.views), c._plane_array(d_out.views)
    good_ptrs = (C.c_void_p * 3)(*[u.ctypes.data for u in good])
    for a in ((None, dbs, outs, good_ptrs), (cds, None, outs, good_ptrs), (cds, dbs, None, good_ptrs),
              (cds, dbs, outs, None)):
        st = c.L.b200_lrf_filter_dev(c.h, *[None if x is None else C.addressof(x) for x in a[:3]], 3, 1, 1, W, H, bd,
                                     1, (C.c_int * 3)(*us), None if a[3] is None else C.addressof(a[3]))
        assert st == B.ERR_ARG
    assert c.launches == n0
    after = d_out.download()
    assert all((a == b).all() for a, b in zip(before, after)), "a rejected call wrote"
    # a None record with out-of-range Sgrproj / Wiener fields is accepted: only its own type's fields count
    c.lrf_filter_dev(d_cd.views, d_db.views, d_out.views, 1, 1, W, H, bd, 1, us,
                     with_unit(0, type=0, set=200, xqd=(-128, 127)))
    c.synchronize()
    for dp in (d_cd, d_db, d_out):
        dp.free()


@pytest.mark.parametrize("layout,bd", [("420", 8), ("444", 10)])
def test_chain_deblock_cdef_lrf(layout, bd):
    """deblock filter -> CDEF per plane -> loop restoration with no host synchronisation in between, against
    the oracle's deblock -> CDEF -> loop restoration."""
    rng = np.random.default_rng(77 + bd)
    W, H = 200, 136
    n, xdec, ydec = LAYOUTS[layout]
    grid, src, rec = frame_setup(rng, layout, bd, W, H)
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    items = [(0, 0, w4, h4, W, H)]
    levels = np.array([[20, 24, 12, 16]], np.uint8)
    sbw, sbh = (W + 63) // 64, (H + 63) // 64
    strengths = [rng.integers(0, 64, (sbh, sbw)).astype(np.uint8) for _ in range(2)]
    damping = 4
    us = [64, 32, 32] if layout == "420" else [64, 64, 64]
    units = mixed(rng, W, H, layout, us)

    c = G.ctx()
    d_rec = DbDevPlanes(c, rec, layout)
    d_deb = DbDevPlanes(c, [np.zeros_like(a) for a in rec], layout)
    d_cdef = DbDevPlanes(c, [np.zeros_like(a) for a in rec], layout)
    d_out = DbDevPlanes(c, [np.zeros_like(a) for a in rec], layout)
    d_mi = G.to_dev(grid.view(np.uint8).reshape(-1))
    d_dir = torch.empty(sbh * 8 * sbw * 8, dtype=torch.uint8, device="cuda")
    d_var = torch.empty(sbh * 8 * sbw * 8, dtype=torch.int32, device="cuda")
    c.deblock_filter_dev(d_rec.views, d_deb.views, xdec, ydec, bd, state_array(), G.to_dev(levels.reshape(-1)),
                         d_mi, grid.shape[1], items)
    c.cdef_find_dir_dev(d_deb.views[0], bd, None, d_dir, d_var)
    for p in range(n):
        xd, yd = dec(p, layout)
        c.cdef_filter_plane_dev(d_deb.views[p], d_cdef.views[p], p, xd, yd, W, H, bd, damping, None, d_dir, d_var,
                                G.to_dev(strengths[min(p, 1)]))
    c.lrf_filter_dev(d_cdef.views, d_deb.views, d_out.views, xdec, ydec, W, H, bd, 1, us, units)
    c.synchronize()
    got = d_out.download()

    deb = [a.copy() for a in rec]
    orc_filter(deb, layout, bd, state_array(), levels, grid, items)

    def crop_db(a, p):
        xd, yd = dec(p, layout)
        return np.ascontiguousarray(a[DB_PAD >> yd:, DB_PAD >> xd:][:H >> yd, :W >> xd])

    luma = crop_db(deb[0], 0)
    dirs, var = O.cdef_analyze_frame(luma, bd)
    cdefd = [O.cdef_filter_plane(crop_db(deb[p], p), p, *dec(p, layout), W, H, bd, damping, None, dirs, var,
                                 strengths[min(p, 1)]) for p in range(n)]

    def padded(a):
        return np.pad(a, PAD, mode="edge")

    want = orc_lrf([padded(a) for a in cdefd], [padded(crop_db(deb[p], p)) for p in range(n)], layout, bd, W, H, 1,
                   us, units)
    for p in range(n):
        cw, ch = crop(W, H, p, layout)
        assert (crop_db(got[p], p) == want[p][PAD:PAD + ch, PAD:PAD + cw]).all(), f"plane {p}"
    for dp in (d_rec, d_deb, d_cdef, d_out):
        dp.free()
