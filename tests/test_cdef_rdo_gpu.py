"""b200_cdef_rdo_dev (the CDEF pass of rdo_loop_decision) against the oracle, bit for bit: err, the f64 bit
pattern of cost, best and the area's CDEF output, with every pixel outside the areas untouched."""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_oracle_cdef_rdo import DEFAULT_STRENGTHS, LAYOUTS, cdef_rdo, make_frame

pytestmark = pytest.mark.gpu
PAD = 8


def download(plane, like):
    c = G.ctx()
    out = np.empty_like(like)
    c.check(c.L.b200_plane_download(c.h, C.byref(plane), out.ctypes.data, out.strides[0]))
    return out


def run_both(rec, src, layout, W, H, bd, damping, cdef_bits, ystr, uvstr, areas, skip8=None, imp=None,
             dist_scale=(16384,) * 3, lam=0.0, rate=None, with_out=True):
    planes, xdec, ydec = LAYOUTS[layout]
    c = G.ctx()
    rng = np.random.default_rng(99)
    base = [rng.integers(0, 1 << bd, r.shape).astype(r.dtype) for r in rec]   # what `out` held before
    d_rec = [c.plane_from_host(r, PAD) for r in rec]
    d_src = [c.plane_from_host(s, PAD) for s in src]
    d_out = [c.plane_from_host(b, PAD) for b in base] if with_out else None
    n = len(areas)
    d_err = G.to_dev(np.full((n * 16, 8), np.iinfo(np.uint64).max, np.uint64))
    d_cost = G.to_dev(np.full((n * 16, 8), np.nan))
    d_best = G.to_dev(np.full(n * 16, 127, np.int8))
    c.cdef_rdo_dev(d_rec, d_src, d_out, xdec, ydec, W, H, bd, damping, cdef_bits, ystr, uvstr,
                   G.to_dev(skip8) if skip8 is not None else None, G.to_dev(imp) if imp is not None else None,
                   dist_scale, lam, areas, G.to_dev(rate) if rate is not None else None, d_err, d_cost, d_best)
    c.synchronize()
    got_err = G.from_dev(d_err, np.uint64).reshape(n * 16, 8)
    got_cost = G.from_dev(d_cost, np.float64).reshape(n * 16, 8)
    got_best = G.from_dev(d_best, np.int8)
    want_out = [b.copy() for b in base] if with_out else None
    err, cost, best = cdef_rdo(rec, src, want_out, xdec, ydec, W, H, bd, damping, cdef_bits, ystr, uvstr, skip8, imp,
                               dist_scale, lam, areas, rate)
    assert (got_best == best[:n * 16]).all()
    nidx = 1 << cdef_bits
    dec = best[:n * 16] >= 0
    assert (got_err[dec, :nidx] == err[:n * 16][dec, :nidx]).all()
    assert (got_cost[dec, :nidx].view(np.uint64) == cost[:n * 16][dec, :nidx].view(np.uint64)).all()
    if with_out:
        for p in range(planes):
            got = download(d_out[p], base[p])
            assert (got == want_out[p]).all(), f"plane {p}: {np.argwhere(got != want_out[p])[:5]}"
    for p in (d_rec + d_src + (d_out or [])):
        c.plane_free(p)
    return got_err, got_cost, got_best


@pytest.mark.parametrize("layout,bd", [("420", 8), ("420", 10), ("422", 8), ("444", 12), ("400", 10), ("444", 8)])
@pytest.mark.parametrize("cdef_bits", [0, 1, 2, 3])
def test_matches_the_oracle(layout, bd, cdef_bits):
    rng = np.random.default_rng(17 * cdef_bits + bd)
    W, H = 316, 198                                  # partial superblocks; visible width not a multiple of 8
    rec, src = make_frame(rng, W, H, layout, bd)
    w8, h8 = (W + 7) >> 3, (H + 7) >> 3
    skip8 = (rng.random((h8, w8)) < 0.3).astype(np.uint8)
    skip8[0:8, 64 // 8:128 // 8] = 1                 # an all-skip superblock
    imp = rng.integers(3000, 70000, (h8, w8)).astype(np.uint32) if cdef_bits & 1 else None
    areas = [(0, 0, 1, 1), (1, 0, 2, 2), (3, 0, 2, 1), (0, 1, 1, 3), (3, 1, 2, 2), (1, 2, 2, 2)]
    rate = rng.integers(0, 3000, len(areas) * 16).astype(np.uint32)
    ys = [int(v) for v in rng.integers(0, 64, 8)]
    us = [int(v) for v in rng.integers(0, 64, 8)]
    _, _, best = run_both(rec, src, layout, W, H, bd, 3 + cdef_bits, cdef_bits, ys, us, areas, skip8, imp,
                          (16384, 23000, 12000), 517.25, rate)
    assert best[16 * 1 + 0] == -1                   # superblock (1, 0) of area 1 is all skip


def test_flat_ties_and_no_output_planes():
    rng = np.random.default_rng(4)
    rec, src = make_frame(rng, 192, 128, "420", 8, flat=True)
    _, cost, best = run_both(rec, src, "420", 192, 128, 8, 3, 3, DEFAULT_STRENGTHS, DEFAULT_STRENGTHS,
                             [(0, 0, 3, 2)], with_out=False)
    assert (best[[0, 1, 2, 4, 5, 6]] == 0).all()


@pytest.mark.parametrize("bd", [8, 10])
def test_1080p_420_mixed_areas(bd):
    rng = np.random.default_rng(bd)
    W, H = 1920, 1080
    rec, src = make_frame(rng, W, H, "420", bd)
    skip8 = (rng.random(((H + 7) >> 3, W >> 3)) < 0.5).astype(np.uint8)
    areas, sbw, sbh = [], 30, 17
    for y in range(0, sbh, 2):
        for x in range(0, sbw, 2):
            if (x // 2 + y // 2) % 3 == 0:            # 1x1 areas here, 2x2 (trimmed at the frame) elsewhere
                areas += [(x + dx, y + dy, 1, 1) for dy in range(2) for dx in range(2) if y + dy < sbh]
            else:
                areas.append((x, y, 2, min(2, sbh - y)))
    run_both(rec, src, "420", W, H, bd, 5, 2, DEFAULT_STRENGTHS, DEFAULT_STRENGTHS[::-1], areas, skip8, None,
             (16384, 20000, 20000), 3000.0, rng.integers(0, 500, len(areas) * 16).astype(np.uint32))


def test_host_rejections_launch_nothing():
    rng = np.random.default_rng(1)
    W, H = 128, 128
    rec, src = make_frame(rng, W, H, "420", 8)
    c = G.ctx()
    d_rec = [c.plane_from_host(r, PAD) for r in rec]
    d_src = [c.plane_from_host(s, PAD) for s in src]
    d_out = [c.plane_from_host(r, PAD) for r in rec]
    small = [c.plane_from_host(r[:64, :64], PAD) for r in rec]
    d_err, d_cost, d_best = G.dev_empty(8 * 16 * 8 * 4), G.dev_empty(8 * 16 * 8 * 4), G.dev_empty(16 * 4)
    ok = dict(rec=d_rec, src=d_src, out=d_out, xdec=1, ydec=1, width=W, height=H, bit_depth=8, damping=3,
              cdef_bits=2, y_strengths=DEFAULT_STRENGTHS, uv_strengths=DEFAULT_STRENGTHS, d_skip8=None,
              d_imp_scales=None, dist_scale=(16384,) * 3, lam=0.0, areas=[(0, 0, 2, 2)], d_rate=None, d_err=d_err,
              d_cost=d_cost, d_best=d_best)
    c.cdef_rdo_dev(**ok)                             # the valid call runs
    c.synchronize()
    bad = [dict(bit_depth=10), dict(bit_depth=9), dict(cdef_bits=4), dict(cdef_bits=-1), dict(damping=2),
           dict(damping=7), dict(y_strengths=[64] + DEFAULT_STRENGTHS[1:]),
           dict(uv_strengths=DEFAULT_STRENGTHS[:3] + [70] + DEFAULT_STRENGTHS[4:]),
           dict(areas=[(1, 1, 2, 1)]), dict(areas=[(0, 0, 5, 1)]), dict(areas=[(0, 0, 0, 1)]),
           dict(areas=[(-1, 0, 1, 1)]), dict(areas=[(0, 0, 2, 1), (1, 0, 1, 2)]), dict(out=d_rec),
           dict(out=[d_out[0], d_rec[0], d_out[2]]), dict(rec=small), dict(src=small), dict(out=small),
           dict(d_err=None), dict(d_cost=None), dict(d_best=None), dict(xdec=0, ydec=1), dict(rec=d_rec[:2]),
           dict(width=0)]
    for b in bad:
        n0 = c.launches
        with pytest.raises(B.B200Error) as e:
            c.cdef_rdo_dev(**{**ok, **b})
        assert e.value.status == B.ERR_ARG, b
        assert c.launches == n0, b
    n0 = c.launches
    c.cdef_rdo_dev(**{**ok, "areas": []})             # nothing to do: nothing launched
    assert c.launches == n0
    for p in d_rec + d_src + d_out + small:
        c.plane_free(p)


def test_matches_the_public_find_dir_and_filter_calls_on_an_area_copy():
    """Copy one area into area-sized planes: there the frame-relative public calls see the area's
    edges, so find_dir + filter_plane with each superblock's winning strengths give the fused `out`."""
    rng = np.random.default_rng(8)
    W, H = 256, 192
    layout, bd = "420", 10
    rec, src = make_frame(rng, W, H, layout, bd)
    skip8 = (rng.random((H >> 3, W >> 3)) < 0.3).astype(np.uint8)
    area = (1, 1, 2, 2)                              # a 128 x 128 area inside the frame
    ys, us = DEFAULT_STRENGTHS, DEFAULT_STRENGTHS[::-1]
    c = G.ctx()
    d_rec = [c.plane_from_host(r, PAD) for r in rec]
    d_src = [c.plane_from_host(s, PAD) for s in src]
    d_out = [c.plane_from_host(r, PAD) for r in rec]
    d_err, d_cost, d_best = G.dev_empty(16 * 8 * 8), G.dev_empty(16 * 8 * 8), G.dev_empty(16)
    c.cdef_rdo_dev(d_rec, d_src, d_out, 1, 1, W, H, bd, 4, 3, ys, us, G.to_dev(skip8), None, (16384,) * 3, 0.0,
                   [area], None, d_err, d_cost, d_best)
    c.synchronize()
    best = G.from_dev(d_best, np.int8)[:16]
    fused = [download(d_out[p], rec[p]) for p in range(3)]
    x0, y0, aw, ah = 64, 64, 128, 128
    a_rec = [np.ascontiguousarray(rec[p][(y0 >> (p > 0)):(y0 + ah) >> (p > 0), (x0 >> (p > 0)):(x0 + aw) >> (p > 0)])
             for p in range(3)]
    a_skip = np.ascontiguousarray(skip8[y0 >> 3:(y0 + ah) >> 3, x0 >> 3:(x0 + aw) >> 3])
    win = [best[sby * 4 + sbx] for sby in range(2) for sbx in range(2)]
    d_a = [c.plane_from_host(r, PAD) for r in a_rec]
    d_ao = [c.plane_from_host(r, PAD) for r in a_rec]
    d_dir, d_var = G.dev_empty(256), G.dev_empty(256 * 4)
    d_skip = G.to_dev(a_skip)
    c.cdef_find_dir_dev(d_a[0], bd, d_skip, d_dir, d_var)
    for p in range(3):
        table = ys if p == 0 else us
        strength = np.array([table[max(int(w), 0)] for w in win], np.uint8)
        c.cdef_filter_plane_dev(d_a[p], d_ao[p], p, 1 if p else 0, 1 if p else 0, aw, ah, bd, 4, d_skip, d_dir, d_var,
                                G.to_dev(strength))
    c.synchronize()
    for p in range(3):
        got = download(d_ao[p], a_rec[p])
        s = p > 0
        assert (got == fused[p][y0 >> s:(y0 + ah) >> s, x0 >> s:(x0 + aw) >> s]).all(), p
    for pl in d_rec + d_src + d_out + d_a + d_ao:
        c.plane_free(pl)
