"""b200_loop_decision_dev (rdo_loop_decision's pass loop) against orc_loop_decision, bit for bit: the stage count,
every final index, unit record, f64 cost bit pattern and written flag, the last C stage's errors and costs and the
working copy; inputs and the slots and units the call does not reach are left untouched; rejections launch
nothing."""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_oracle_loop_decision import LAYOUTS, case, matrix, run

pytestmark = pytest.mark.gpu
PAD = 8


def download(plane, like):
    c = G.ctx()
    out = np.empty_like(like)
    c.check(c.L.b200_plane_download(c.h, C.byref(plane), out.ctypes.data, out.strides[0]))
    return out


def run_both(fx):
    c = G.ctx()
    n, nu = len(fx["areas"]), len(fx["units"])
    _, xdec, ydec = LAYOUTS[fx["layout"]]
    d_rec = [c.plane_from_host(a, PAD) for a in fx["rec"]]
    d_src = [c.plane_from_host(a, PAD) for a in fx["src"]]
    d_work = [c.plane_from_host(np.full_like(a, 7), PAD) for a in fx["rec"]]
    d_best = G.to_dev(np.full(max(n, 1) * 16, 127, np.int8))
    d_unit = G.to_dev(np.full(max(nu, 1) * 12, 0xEE, np.uint8))
    d_ucost = G.to_dev(np.full(max(nu, 1), np.nan))
    d_wr = G.to_dev(np.full(max(nu, 1), 7, np.uint8))
    d_err = G.to_dev(np.full((max(n, 1) * 16, 8), np.iinfo(np.uint64).max, np.uint64))
    d_cost = G.to_dev(np.full((max(n, 1) * 16, 8), np.nan))
    stages = c.loop_decision_dev(d_rec, d_src, d_work, xdec, ydec, fx["W"], fx["H"], fx["bd"], fx["enable_cdef"],
                                 fx["damping"], fx["cdef_bits"], fx["ystr"], fx["uvstr"], G.to_dev(fx["skip8"]),
                                 fx["enable_lrf"], fx["unit_size"], fx["reduced"],
                                 G.to_dev(fx["imp"]) if fx["imp"] is not None else None, fx["dist_scale"], fx["lam"],
                                 fx["areas"], fx["units"], fx["sb_unit"], d_best, d_unit, d_ucost, d_wr, d_err, d_cost)
    w_stages, w_best, w_uo, w_uc, w_wr, w_err, w_cost, w_work = run(fx)
    assert stages == w_stages
    assert (G.from_dev(d_best, np.int8)[:n * 16] == w_best[:n * 16]).all()
    assert (G.from_dev(d_unit, np.uint8)[:12 * nu] == w_uo.view(np.uint8)).all()
    assert (G.from_dev(d_ucost, np.float64)[:nu].view(np.uint64) == w_uc.view(np.uint64)).all()
    assert (G.from_dev(d_wr, np.uint8)[:nu] == w_wr).all()
    assert (G.from_dev(d_err, np.uint64)[:n * 128].reshape(-1, 8) == w_err[:n * 16]).all()
    assert (G.from_dev(d_cost, np.float64)[:n * 128].view(np.uint64) == w_cost[:n * 16].reshape(-1).view(np.uint64)).all()
    for d, h in zip(d_work, w_work):
        assert (download(d, h) == h).all()
    for d, h in zip(d_rec + d_src, fx["rec"] + fx["src"]):   # inputs unchanged
        assert (download(d, h) == h).all()
    for p in d_rec + d_src + d_work:
        c.plane_free(p)
    return stages


MATRIX = matrix()


@pytest.mark.parametrize("name", [m[0] for m in MATRIX])
def test_matches_the_oracle(name):
    run_both(dict(MATRIX)[name])


@pytest.mark.parametrize("uy", [64, 128, 256])
def test_1080p_420_every_area_in_one_call(uy):
    fx = case(uy, "420", 10, 1920, 1080, (uy, uy >> 1, uy >> 1), reduced=uy == 128, skip_frac=0.2)
    assert run_both(fx) >= 2


def test_host_rejections_launch_nothing():
    fx = case(3, "420", 8, 128, 128, (64, 32, 32))
    c = G.ctx()
    d_rec = [c.plane_from_host(a, PAD) for a in fx["rec"]]
    d_src = [c.plane_from_host(a, PAD) for a in fx["src"]]
    d_work = [c.plane_from_host(np.zeros_like(a), PAD) for a in fx["rec"]]
    small = [c.plane_from_host(a[:64, :64], PAD) for a in fx["rec"]]
    n, nu = len(fx["areas"]), len(fx["units"])
    outs = dict(d_best_index=G.dev_empty(16 * n), d_unit=G.dev_empty(12 * nu), d_unit_cost=G.dev_empty(8 * nu),
                d_written=G.dev_empty(nu))
    ok = dict(rec=d_rec, src=d_src, work=d_work, xdec=1, ydec=1, frame_w=128, frame_h=128, bit_depth=8,
              enable_cdef=1, damping=5, cdef_bits=2, y_strengths=fx["ystr"], uv_strengths=fx["uvstr"], d_skip8=None,
              enable_restoration=1, unit_size=[64, 32, 32], reduced_sets=0, d_imp_scales=None,
              dist_scale=(16384,) * 3, lam=10.0, areas=fx["areas"], units=fx["units"], sb_unit=fx["sb_unit"], **outs)
    c.loop_decision_dev(**ok)

    def unit(**kw):
        u = fx["units"].copy()
        for k, v in kw.items():
            u[0][k] = v
        return u

    def smap(v):
        m = fx["sb_unit"].copy()
        m[0, 0, 0] = v
        return m
    bad = [dict(bit_depth=10), dict(bit_depth=9), dict(xdec=0, ydec=1), dict(rec=d_rec[:2]), dict(frame_w=0),
           dict(rec=small), dict(src=small), dict(work=small), dict(work=d_rec), dict(work=[d_work[0], d_src[1],
                                                                                            d_work[2]]),
           dict(damping=2), dict(cdef_bits=4), dict(y_strengths=[64] * 8), dict(unit_size=[48, 32, 32]),
           dict(unit_size=[64, 16, 16]), dict(areas=[(0, 0, 5, 1)] + fx["areas"][1:]),
           dict(areas=[(1, 1, 2, 1)] + fx["areas"][1:]), dict(units=unit(area=n)), dict(units=unit(plane=3)),
           dict(units=unit(lru_x=2)), dict(units=unit(sgrproj_ref=[32, 0])), dict(sb_unit=smap(nu)),
           dict(sb_unit=smap(-2)), dict(sb_unit=smap(int(np.nonzero(fx["units"]["plane"] == 1)[0][0]))),
           dict(d_best_index=None), dict(d_unit=None), dict(d_unit_cost=None), dict(d_written=None)]
    for b in bad:
        n0 = c.launches
        with pytest.raises(B.B200Error) as e:
            c.loop_decision_dev(**{**ok, **b})
        assert e.value.status == B.ERR_ARG, b
        assert c.launches == n0, b
    n0 = c.launches
    assert c.loop_decision_dev(**{**ok, "areas": [], "units": fx["units"][:0], "sb_unit": fx["sb_unit"][:0]}) == 0
    assert c.launches == n0
    for p in d_rec + d_src + d_work + small:
        c.plane_free(p)


def _host_copies(fn):
    """Run fn under torch.profiler; returns the number of device-to-host copies it made.  A session now and then
    delivers no device activity at all (not even the marker kernel); such a record is incomplete and fn runs
    again, which only rewrites its outputs."""
    import time

    import torch
    from torch.profiler import ProfilerActivity, profile
    for attempt in range(6):
        time.sleep(0.1 * attempt)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.zeros(1, device="cuda").add_(1)
            out = fn()
            torch.cuda.synchronize()
        dev = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if dev:
            break
    assert dev, "torch.profiler recorded no CUDA activity"
    return out, sum("DtoH" in n or "Device -> Pageable" in n or "Device -> Pinned" in n for n in dev)


@pytest.mark.parametrize("layout,bd", [("420", 8), ("444", 10)])
@pytest.mark.parametrize("cdef_on", [True, False])
def test_chain_deblock_then_loop_decision(layout, bd, cdef_on):
    """deblock levels -> deblock filter -> b200_loop_decision_dev on the same areas, enqueued with no copy to the
    host but the call's one status read per stage, against the oracle chain (orc_levels, orc_filter,
    orc_loop_decision on the deblocked frame)."""
    from tests.test_deblock_gpu import DevPlanes as DbDevPlanes
    from tests.test_deblock_gpu import frame_setup
    from tests.test_oracle_deblock import orc_levels
    from tests.test_oracle_deblock_spec import PAD as DB_PAD
    from tests.test_oracle_deblock_spec import orc_filter, state_array

    rng = np.random.default_rng(70 + bd + cdef_on)
    W, H = 200, 136
    planes, xdec, ydec = LAYOUTS[layout]
    grid, src, rec = frame_setup(rng, layout, bd, W, H)
    us = (128, 64, 64) if layout == "420" else (128, 128, 128)
    fx = case(71 + bd, layout, bd, W, H, us, enable_cdef=cdef_on, skip_frac=0.2)
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    db_items = [(16 * sx, 16 * sy, min(16 * sw, w4 - 16 * sx), min(16 * sh, h4 - 16 * sy), W - 64 * sx, H - 64 * sy)
                for sx, sy, sw, sh in fx["areas"]]
    n, nu = len(fx["areas"]), len(fx["units"])

    c = G.ctx()
    d_rec, d_src = DbDevPlanes(c, rec, layout), DbDevPlanes(c, src, layout)
    d_deb = DbDevPlanes(c, [np.zeros_like(a) for a in rec], layout)
    d_work = DbDevPlanes(c, [np.zeros_like(a) for a in rec], layout)
    d_mi = G.to_dev(grid.view(np.uint8).reshape(-1))
    d_lv = G.dev_empty(4 * len(db_items))
    d_skip = G.to_dev(fx["skip8"])
    d_best = G.to_dev(np.full(n * 16, 127, np.int8))
    d_unit = G.to_dev(np.full(nu * 12, 0xEE, np.uint8))
    d_ucost, d_wr = G.to_dev(np.full(nu, np.nan)), G.to_dev(np.full(nu, 7, np.uint8))
    c.synchronize()

    def chain():
        c.deblock_levels_dev(d_rec.views, d_src.views, xdec, ydec, bd, d_mi, grid.shape[1], db_items, d_lv)
        c.deblock_filter_dev(d_rec.views, d_deb.views, xdec, ydec, bd, state_array(), d_lv, d_mi, grid.shape[1],
                             db_items)
        return c.loop_decision_dev(d_deb.views, d_src.views, d_work.views, xdec, ydec, W, H, bd, cdef_on,
                                   fx["damping"], fx["cdef_bits"], fx["ystr"], fx["uvstr"], d_skip, True,
                                   fx["unit_size"], False, None, fx["dist_scale"], fx["lam"], fx["areas"],
                                   fx["units"], fx["sb_unit"], d_best, d_unit, d_ucost, d_wr)
    stages, d2h = _host_copies(chain)
    assert stages >= 2 and d2h == stages

    levels, _ = orc_levels(rec, src, layout, bd, grid, db_items)
    deb = [a.copy() for a in rec]
    orc_filter(deb, layout, bd, state_array(), levels, grid, db_items)

    def frame8(a, p):                                       # pixel (0, 0) at [0, 0], the frame rounded up to 8
        xd, yd = (xdec, ydec) if p else (0, 0)
        return np.ascontiguousarray(a[DB_PAD >> yd:, DB_PAD >> xd:][:((H + 7) & ~7) >> yd, :((W + 7) & ~7) >> xd])
    want = run({**fx, "rec": [frame8(a, p) for p, a in enumerate(deb)],
                "src": [frame8(a, p) for p, a in enumerate(src)], "imp": None})
    assert stages == want[0]
    assert (G.from_dev(d_best, np.int8)[:n * 16] == want[1][:n * 16]).all()
    assert (G.from_dev(d_unit, np.uint8)[:12 * nu] == want[2].view(np.uint8)).all()
    assert (G.from_dev(d_ucost, np.float64)[:nu].view(np.uint64) == want[3].view(np.uint64)).all()
    assert (G.from_dev(d_wr, np.uint8)[:nu] == want[4]).all()
    for dp in (d_rec, d_src, d_deb, d_work):
        dp.free()
