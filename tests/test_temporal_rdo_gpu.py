"""GPU parity for temporal RDO (rav1e_b200/csrc/temporal_rdo.cu) == oracle/temporal_rdo.c: block
importances bit for bit (f32 compared as u32 patterns) on the CPU tests' windows at 8 and 10 bit and on
speed 6's 21-frame window at 1080p; Q14 distortion scales, both score forms and log_isqrt_mean_scale;
sse_wxh's 4x4 map feeding b200_weighted_sse_dev end to end; host-side rejection of invalid step lists."""
import math

import numpy as np
import pytest
import torch

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_activity import oracle_mask
from tests.test_oracle_rdo_dist import L as OL
from tests.test_oracle_temporal_rdo import (focus_window, oracle_importances, oracle_intra_costs, oracle_scales,
                                            oracle_scores, small_window, window_1080p)

pytestmark = pytest.mark.gpu


def upload(win):
    c = G.ctx()
    planes = [c.plane_from_host(im, win.pad) for im in win.imgs]
    return planes, G.to_dev(np.ascontiguousarray(win.intra)), G.to_dev(np.ascontiguousarray(win.mvs))


def device_importances(win, planes, d_intra, d_mvs):
    c = G.ctx()
    d_imp = G.dev_empty(4 * len(win.imgs) * win.n_imp)
    c.block_importances_dev(planes, win.bd, d_intra, d_mvs, win.steps, d_imp)
    c.synchronize()
    return G.from_dev(d_imp, np.float32)[:len(win.imgs) * win.n_imp].reshape(len(win.imgs), win.n_imp), d_imp


def free(planes):
    for p in planes:
        G.ctx().plane_free(p)


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10)])
@pytest.mark.parametrize("make", [small_window, focus_window])
def test_importances_match_oracle(make, dtype, bd):
    win = make(dtype, bd)
    planes, d_intra, d_mvs = upload(win)
    got, _ = device_importances(win, planes, d_intra, d_mvs)
    want = oracle_importances(win)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    assert (want > 0).any()
    free(planes)


def odd_boundary_ulps(imp, intra):
    """smallest distance, in ULPs of 32768 s, from 32768 s to an odd integer over the blocks that take
    the pow() path: where the Q14 value could flip between two pow() implementations"""
    best = math.inf
    for p, i in zip(imp.tolist(), intra.tolist()):
        if i == 0:
            continue
        v = 32768.0 * math.pow((i + p) / i, 1.0 / 3.0)
        odd = 2 * math.floor((v - 1) / 2) + 1
        d = min(abs(v - odd), abs(odd + 2 - v))
        best = min(best, d / math.ulp(v))
    return best


def test_1080p_window_end_to_end():
    c = G.ctx()
    win = window_1080p()
    assert len(win.steps) == 57 and win.n_imp == 240 * 135
    oracle_intra_costs(win)
    planes, d_intra, d_mvs = upload(win)
    got, d_imp = device_importances(win, planes, d_intra, d_mvs)
    again, _ = device_importances(win, planes, d_intra, d_mvs)
    want = oracle_importances(win)
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    np.testing.assert_array_equal(again.view(np.uint32), got.view(np.uint32))
    assert (want[0] > 0).mean() > 0.5

    # distortion scales of the frame being coded (frame 0)
    n, n_intra = win.n_imp, win.n_intra
    d_sc = G.dev_empty(4 * n)
    c.distortion_scales_dev(planes[0], d_imp, d_intra, d_sc)
    c.synchronize()
    want_sc = oracle_scales(win, want[0], win.intra[0])
    np.testing.assert_array_equal(G.from_dev(d_sc, np.uint32)[:n], want_sc)
    margin = odd_boundary_ulps(want[0][:n_intra], win.intra[0][:n_intra])
    print(f"smallest distance of 32768*s from an odd integer: {margin:.3g} ULP")
    assert margin > 8

    # activity scales on the device vs the oracle
    _, want_act, _ = oracle_mask(win.imgs[0], win.pad, 8)
    d_var, d_act = G.dev_empty(4 * n), G.dev_empty(4 * n)
    c.activity_mask_dev(planes[0], 8, d_var, d_act)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_act, np.uint32)[:n], want_act.reshape(-1))

    # both score forms; the spatiotemporal one also builds sse_wxh's 4x4 map
    stride4 = 2 * win.w_imp
    for act in (None, d_act):
        d_s = G.to_dev(want_sc)
        d_st, d_log = G.dev_empty(4 * n), G.dev_empty(8)
        d_map = G.dev_empty(4 * stride4 * 2 * win.h_imp)
        c.temporal_scores_dev(win.w_imp, win.h_imp, d_s, act, d_st, d_log, d_map, stride4)
        c.synchronize()
        wd, wst, wlog = oracle_scores(want_sc, None if act is None else want_act.reshape(-1))
        np.testing.assert_array_equal(G.from_dev(d_s, np.uint32)[:n], wd)
        np.testing.assert_array_equal(G.from_dev(d_st, np.uint32)[:n], wst)
        assert int(G.from_dev(d_log, np.int64)[0]) == wlog
        scale4 = np.ascontiguousarray(np.repeat(np.repeat(wd.reshape(win.h_imp, win.w_imp), 2, 0), 2, 1))
        np.testing.assert_array_equal(G.from_dev(d_map, np.uint32)[:scale4.size].reshape(scale4.shape), scale4)
    assert len(set(wd.tolist())) > 100                                  # not a constant map

    # end to end: weighted SSE of frame 0 against frame 1 with the device's map (spatiotemporal form)
    blocks = G.grid_blocks(win.W, win.H, 16, 16)
    nb = len(blocks)
    d_out = G.dev_empty(8 * nb)
    c.weighted_sse_dev(planes[0], planes[1], G.to_dev(blocks), nb, 16, 16, d_map, stride4, d_out)
    c.synchronize()
    got_sse = G.from_dev(d_out, np.uint64)[:nb]
    ol = OL()
    a, b = win.imgs[0], win.imgs[1]
    for i, blk in enumerate(blocks):
        x, y = int(blk["x"]), int(blk["y"])
        want_sse = ol.orc_weighted_sse_u8(a.ctypes.data + y * win.W + x, win.W, b.ctypes.data + y * win.W + x, win.W,
                                          scale4.ctypes.data + ((y // 4) * stride4 + x // 4) * 4, stride4, 16, 16)
        assert int(got_sse[i]) == want_sse, (i, x, y)
    free(planes)


def test_invalid_step_lists_are_rejected_before_any_launch():
    c = G.ctx()
    win = small_window()
    planes, d_intra, d_mvs = upload(win)
    d_imp = G.dev_empty(4 * len(win.imgs) * win.n_imp)
    bad = {
        "src == dst": [(2, 2, 1, 0)],
        "src outside the window": [(5, 1, 1, 0)],
        "dst outside the window": [(1, 9, 1, 0)],
        "len 0": [(2, 1, 0, 0)],
        "src not final": [(2, 1, 1, 0), (3, 2, 1, 1)],
    }
    for name, steps in bad.items():
        n0 = c.launches
        with pytest.raises(B.B200Error) as e:
            c.block_importances_dev(planes, 8, d_intra, d_mvs, steps, d_imp)
        assert e.value.status == B.ERR_ARG, name
        assert c.launches == n0, name
    # planes of different sizes or bpp
    other = c.plane_from_host(np.zeros((win.H, win.W + 8), np.uint8), win.pad)
    hbd = c.plane_from_host(np.zeros((win.H, win.W), np.uint16), win.pad)
    for odd in (other, hbd):
        with pytest.raises(B.B200Error) as e:
            c.block_importances_dev(planes[:2] + [odd], 8, d_intra, d_mvs, [(1, 0, 1, 0)], d_imp)
        assert e.value.status == B.ERR_ARG
    c.plane_free(other)
    c.plane_free(hbd)
    # the valid order of the same two steps runs
    c.block_importances_dev(planes, 8, d_intra, d_mvs, [(3, 2, 1, 1), (2, 1, 1, 0)], d_imp)
    c.synchronize()
    free(planes)
    torch.cuda.synchronize()
