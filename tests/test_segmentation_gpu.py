"""GPU parity for segmentation (rav1e_b200/csrc/segmentation.cu) == oracle/segmentation.c through the C ABI:
every segmentation_optimize case of the CPU tests record for record (all 240 bytes), every select_segment case
item for item with the block scales, item lists longer than one grid-stride pass, the chain
temporal scores (both forms) -> optimize -> select over every block of a 1080p frame at several sizes with no
host copy in between, and host-side rejection of bad arguments before any launch."""
import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_oracle_segmentation import (AC_Q, CASES, SELECT, BW, BH, oracle_optimize, oracle_select,
                                            prev_states, scale_maps, select_inputs, to_record)
from tests.test_oracle_temporal_rdo import T as temporal_lib
from tests import oracle_lib as O

pytestmark = pytest.mark.gpu


def device_optimize(scores, w, h, base, bd, upd, prev_rec, same_buffer=False):
    c = G.ctx()
    d_sc = G.to_dev(np.ascontiguousarray(scores, np.uint32)) if scores is not None else None
    d_out = G.to_dev(np.full(1, 0x5A, np.uint8).repeat(240))
    d_prev = None
    if prev_rec is not None:
        d_prev = G.to_dev(prev_rec)
        if same_buffer:
            d_out = d_prev
    c.segmentation_optimize_dev(d_sc, w, h, base, bd, AC_Q[bd], upd, d_prev, d_out)
    c.synchronize()
    return G.from_dev(d_out, B.SEGMENTATION_DTYPE)[:1]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_optimize_matches_oracle(case):
    name, scores, w, h, base, bd, upd, pname = case
    prev = None if pname is None else prev_states()[pname]
    want = oracle_optimize(scores, w, h, base, bd, upd, prev)
    got = device_optimize(scores, w, h, base, bd, upd, None if prev is None else to_record(prev))
    assert got.tobytes() == want.tobytes(), (got, want)
    if pname is not None:  # the previous state may be the output record
        again = device_optimize(scores, w, h, base, bd, upd, to_record(prev), same_buffer=True)
        assert again.tobytes() == want.tobytes()


def device_select(items, d, a, w, h, off, level, rec, with_scale=True):
    c = G.ctx()
    n = len(items)
    d_sidx, d_scale = G.dev_empty(2 * n), (G.dev_empty(4 * n) if with_scale else None)
    c.select_segment_dev(G.to_dev(items), n, None if d is None else G.to_dev(d), None if a is None else G.to_dev(a),
                         w, h, off, level, G.to_dev(rec), d_sidx, d_scale)
    c.synchronize()
    sidx = G.from_dev(d_sidx, np.uint8)[:2 * n].reshape(n, 2)
    return sidx, (G.from_dev(d_scale, np.uint32)[:n] if with_scale else None)


@pytest.mark.parametrize("case", SELECT, ids=[c[0] for c in SELECT])
def test_select_matches_oracle(case):
    name, ci, level, off, act = case
    rec, items, d, a, w, h = select_inputs(ci, act)
    want, want_scale = oracle_select(items, d, a, w, h, off, level, rec)
    got, got_scale = device_select(items, None if off else d, a, w, h, off, level, rec)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(got_scale, want_scale)
    got2, _ = device_select(items, d, a, w, h, off, level, rec, with_scale=False)
    np.testing.assert_array_equal(got2, want)


def test_long_item_list():
    """more items than one grid-stride pass of the launch (num_sms * 4 CTAs of 256 threads)"""
    rng = np.random.default_rng(21)
    w, h = 240, 135
    rec = oracle_optimize(CASES[0][1], w, h, 100, 8, 1, None)
    d, a = scale_maps(w, h, seed=9)
    n = 300_000
    items = np.zeros(n, B.SEGMENT_ITEM_DTYPE)
    items["x"] = rng.integers(-2, 8 * w // 4 + 4, n) * 4
    items["y"] = rng.integers(-2, 8 * h // 4 + 4, n) * 4
    items["bsize"] = rng.integers(0, 23, n)
    items["skip"] = rng.random(n) < 0.2
    assert n > 132 * 4 * 256
    for level in (1, 2, 3):
        want, want_scale = oracle_select(items, d, a, w, h, 0, level, rec)
        got, got_scale = device_select(items, d, a, w, h, 0, level, rec)
        np.testing.assert_array_equal(got, want)
        np.testing.assert_array_equal(got_scale, want_scale)
        assert (want[:, 0] == 255).any() and (want[:, 0] != 255).any()


def frame_items(W, H, bs):
    bw, bh = BW[bs], BH[bs]
    ys, xs = np.meshgrid(np.arange(0, H, bh), np.arange(0, W, bw), indexing="ij")
    it = np.zeros(xs.size, B.SEGMENT_ITEM_DTYPE)
    it["x"], it["y"], it["bsize"] = xs.reshape(-1), ys.reshape(-1), bs
    it["skip"] = (np.arange(xs.size) % 7) == 3
    return it


@pytest.mark.parametrize("psy", [False, True], ids=["temporal", "spatiotemporal"])
def test_chain_1080p(psy):
    """temporal scores -> segmentation_optimize -> select_segment for every block of a 1080p frame at several
    sizes, enqueued without a host copy; checked against the oracle chain at the end"""
    c = G.ctx()
    W, H = 1920, 1080
    w, h = (W + 7) // 8, (H + 7) // 8
    d0, a0 = scale_maps(w, h, seed=13)
    n = w * h
    d_scales, d_act = G.to_dev(d0), (G.to_dev(a0) if psy else None)
    d_st = G.dev_empty(4 * n)
    c.temporal_scores_dev(w, h, d_scales, d_act, d_st)
    d_rec = G.dev_empty(240)
    c.segmentation_optimize_dev(d_st, w, h, 140, 10, AC_Q[10], 1, None, d_rec)
    sizes = (3, 6, 9, 12, 15, 16, 21)  # 8x8, 16x16, 32x32, 64x64, 128x128, 4x16, 64x16
    outs = []
    for bs in sizes:
        items = frame_items(W, H, bs)
        d_sidx, d_scale = G.dev_empty(2 * len(items)), G.dev_empty(4 * len(items))
        c.select_segment_dev(G.to_dev(items), len(items), d_scales, d_act, w, h, 0, B.SEGMENTATION_COMPLEX, d_rec,
                             d_sidx, d_scale)
        outs.append((items, d_sidx, d_scale))
    c.synchronize()

    # the oracle chain
    l = temporal_lib()
    scales, st = d0.copy(), np.zeros(n, np.uint32)
    l.orc_temporal_scores(O.ptr(scales), n, O.ptr(a0) if psy else None, O.ptr(st), None)
    rec = oracle_optimize(st, w, h, 140, 10, 1, None)
    assert G.from_dev(d_rec, B.SEGMENTATION_DTYPE)[:1].tobytes() == rec.tobytes()
    assert rec["max_segment"][0] >= 2
    for items, d_sidx, d_scale in outs:
        want, want_scale = oracle_select(items, scales, a0 if psy else None, w, h, 0, B.SEGMENTATION_COMPLEX, rec)
        np.testing.assert_array_equal(G.from_dev(d_sidx, np.uint8)[:2 * len(items)].reshape(-1, 2), want)
        np.testing.assert_array_equal(G.from_dev(d_scale, np.uint32)[:len(items)], want_scale)
        assert len(np.unique(want[:, 0])) >= 2


def test_rejections_launch_nothing():
    c = G.ctx()
    L = c.L
    w, h = 16, 9
    d_sc = G.to_dev(np.full(w * h, 16384, np.uint32))
    d_rec = G.to_dev(np.full(240, 0x5A, np.uint8))
    good = AC_Q[8].copy()
    flat = good.copy()
    flat[100] = flat[99]
    zero = good.copy()
    zero[0] = 0

    def opt(sc=d_sc, w_=w, h_=h, base=100, bd=8, q=good, upd=1, out=d_rec):
        qp = None if q is None else np.ascontiguousarray(q, np.uint16)
        return L.b200_segmentation_optimize_dev(c.h, None if sc is None else sc.data_ptr(), w_, h_, base, bd,
                                                None if qp is None else qp.ctypes.data, upd, None,
                                                None if out is None else out.data_ptr())

    items = G.to_dev(np.zeros(4, B.SEGMENT_ITEM_DTYPE))
    d_sidx = G.to_dev(np.full(8, 0x5A, np.uint8))

    def sel(it=items, n=4, sc=d_sc, w_=w, h_=h, off=0, level=2, rec=d_rec, sidx=d_sidx):
        p = lambda t: None if t is None else t.data_ptr()
        return L.b200_select_segment_dev(c.h, p(it), n, p(sc), None, w_, h_, off, level, p(rec), p(sidx), None)

    before = c.launches
    for kw in [dict(q=flat), dict(q=zero), dict(q=None), dict(bd=9), dict(bd=16), dict(base=-1), dict(base=256),
               dict(upd=2), dict(sc=None), dict(out=None), dict(w_=0), dict(h_=0), dict(w_=1 << 15, h_=1 << 15)]:
        assert opt(**kw) == B.ERR_ARG, kw
    for kw in [dict(it=None), dict(sc=None), dict(rec=None), dict(sidx=None), dict(level=0), dict(level=4),
               dict(w_=0), dict(h_=1 << 30)]:
        assert sel(**kw) == B.ERR_ARG, kw
    assert c.launches == before
    assert sel(n=0) == B.OK and sel(sc=None, off=1, n=0) == B.OK
    assert c.launches == before
    c.synchronize()
    assert (G.from_dev(d_rec, np.uint8) == 0x5A).all() and (G.from_dev(d_sidx, np.uint8) == 0x5A).all()
    assert opt(sc=None, upd=0) == B.OK  # the map is not read with update_data 0
    assert sel(sc=None, off=1) == B.OK  # nor the scale maps with the scales off
    c.synchronize()
    assert c.launches == before + 2
    rec = G.from_dev(d_rec, B.SEGMENTATION_DTYPE)[:1]
    assert rec["status"][0] == 1  # the default state has no ALT_Q segment: the reference panics
    assert (G.from_dev(d_sidx, np.uint8)[:8] == 255).all()
