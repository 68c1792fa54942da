"""GPU parity of the lookahead's motion vectors (rav1e_b200/csrc/lookahead_me.cu, b200_lookahead_motion_dev)
with the serial oracle (oracle/lookahead_me.c: orc_lookahead_motion): the stats grids bit for bit on the CPU tests'
matrix, a 1080p pair, three pairs in one call and a chained y4m sequence; identical reruns; the stated
launch count; rejection of invalid arguments before any launch."""
import numpy as np
import pytest
import torch

from rav1e_b200 import backend as B
from rav1e_b200 import y4m
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_oracle_lookahead_me import (CASES, IDS, PAD, SHIFT, STATS_DTYPE, Params, case_inputs, downsample,
                                            grid_dims, images, oracle_motion, pyramid)
from tests.test_oracle_search import tdiv8

pytestmark = pytest.mark.gpu


def levels(img):
    out = [img]
    for _ in range(2):
        out.append(downsample(out[-1]))
    return out


def dev_pyramid(img, pad=PAD):
    return [G.ctx().plane_from_host(im, pad) for im in levels(img)]


def params(p: Params):
    return B.LookaheadMeParams(p.bit_depth, p.allow_hp, p.me_lambda, p.full_search, p.range_scale, p.tile_w_sb,
                               p.tile_h_sb)


def device_motion(curs, refs, width, height, p, prev=None, has_prev=None):
    """curs / refs: lists of device pyramids -> (npairs, h_in_b, w_in_b) grids"""
    c = G.ctx()
    wib, hib = grid_dims(width, height)
    n = len(curs)
    d_stats = G.dev_empty(8 * n * wib * hib)
    d_prev = None if prev is None else G.to_dev(np.ascontiguousarray(prev, STATS_DTYPE))
    c.lookahead_motion_dev(curs, refs, params(p), d_stats, d_prev, has_prev)
    c.synchronize()
    return G.from_dev(d_stats, STATS_DTYPE)[:n * wib * hib].reshape(n, hib, wib)


def free(*pyrs):
    for pyr in pyrs:
        for q in pyr:
            G.ctx().plane_free(q)


def launches_formula(width, height, p):
    W8, H8 = (width + 7) & ~7, (height + 7) & ~7
    n = 2
    for mv in (64, 32, 16):
        n += -(-min(64 * p.tile_w_sb, W8) // mv) + -(-min(64 * p.tile_h_sb, H8) // mv) - 1
    return n


def assert_grid_equal(got, want):
    bad = np.argwhere(got != want)
    assert len(bad) == 0, (len(bad), bad[:4].tolist(), got[tuple(bad[0])], want[tuple(bad[0])])


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_device_matches_oracle(case):
    w, h = case[0], case[1]
    cur, ref, p, prev, cur_img, ref_img = case_inputs(case)
    want = oracle_motion(cur, ref, w, h, p, prev)
    dc, dr = dev_pyramid(cur_img), dev_pyramid(ref_img)
    before = G.ctx().launches
    got = device_motion([dc], [dr], w, h, p, None if prev is None else prev[None], None if prev is None else [1])
    assert G.ctx().launches - before == launches_formula(w, h, p)
    assert_grid_equal(got[0], want)
    free(dc, dr)


def test_1080p_smooth_pair_and_reruns():
    w, h = 1920, 1080
    p = Params(bit_depth=8, me_lambda=3.0, full_search=0, range_scale=1)
    cur_img, ref_img = images(w, h, 8, True, 5)
    want = oracle_motion(pyramid(cur_img), pyramid(ref_img), w, h, p)
    dc, dr = dev_pyramid(cur_img), dev_pyramid(ref_img)
    before = G.ctx().launches
    got = device_motion([dc], [dr], w, h, p)
    assert G.ctx().launches - before == launches_formula(w, h, p) == 328
    assert_grid_equal(got[0], want)
    again = device_motion([dc], [dr], w, h, p)
    assert got.tobytes() == again.tobytes()
    inner = want[8:-8, 8:-8]
    assert ((inner["mv_row"] == 8 * SHIFT[1]) & (inner["mv_col"] == 8 * SHIFT[0])).mean() > 0.9
    free(dc, dr)


def test_three_pairs_in_one_call():
    """two reference slots of one frame plus a different frame; subset C for two of them"""
    w, h = 200, 120
    p = Params(bit_depth=8, me_lambda=2.0, full_search=1, range_scale=1, tile_w_sb=2, tile_h_sb=1)
    a, r0 = images(w, h, 8, True, 21)
    _, r1 = images(w, h, 8, True, 22)
    b, _ = images(w, h, 8, False, 23)
    pairs = [(a, r0), (a, r1), (b, r0)]
    prev = np.stack([oracle_motion(pyramid(b), pyramid(r), w, h, p) for r in (r0, r1, r1)])
    flags = [1, 0, 1]
    want = [oracle_motion(pyramid(x), pyramid(r), w, h, p, prev[k] if flags[k] else None)
            for k, (x, r) in enumerate(pairs)]
    dcs = [dev_pyramid(x) for x, _ in pairs]
    drs = [dev_pyramid(r) for _, r in pairs]
    got = device_motion(dcs, drs, w, h, p, prev, flags)
    for k in range(3):
        assert_grid_equal(got[k], want[k])
    free(*dcs, *drs)


def test_invalid_arguments_rejected_without_launch():
    c = G.ctx()
    w, h = 72, 40
    cur_img, ref_img = images(w, h, 8, True, 3)
    dc, dr = dev_pyramid(cur_img), dev_pyramid(ref_img)
    p = Params()
    wib, hib = grid_dims(w, h)
    d_stats = G.dev_empty(8 * wib * hib)
    bad_half = c.plane_from_host(np.zeros((h // 2 + 1, w // 2 + 1), np.uint8), PAD)
    u16 = c.plane_from_host(np.zeros((h, w), np.uint16), PAD)
    thin = c.plane_from_host(cur_img, 40)  # the full plane needs 48
    cases = [
        ([[dc[0], bad_half, dc[2]]], [dr], p),                           # hres not (w+1)/2
        ([[u16, dc[1], dc[2]]], [dr], p),                                # mixed bpp
        ([dc], [dr], Params(tile_w_sb=0)),                               # tile size 0
        ([dc], [dr], Params(tile_h_sb=0)),
        ([[thin, dc[1], dc[2]]], [dr], p),                               # pad below the mv range's reach
        ([dc, dc], [dr, [dr[0], dr[1], bad_half]], p),                   # sizes differ across pairs
    ]
    for curs, refs, pp in cases:
        before = c.launches
        with pytest.raises(B.B200Error) as e:
            c.lookahead_motion_dev(curs, refs, params(pp), d_stats)
        assert e.value.status == 2
        assert c.launches == before
    free(dc, dr, [bad_half, u16, thin])


def inter_cost_mean(org, ref, mvs):
    """estimate_inter_costs' mean (lookahead.rs:223-267) from the stride-2 vectors, via the oracle's SATD"""
    h_imp, w_imp = org.shape[0] // 8, org.shape[1] // 8
    po, pr = O.Plane(org.shape[1], org.shape[0], PAD), O.Plane(org.shape[1], org.shape[0], PAD)
    po.fill_from(org)
    pr.fill_from(ref)
    tot = 0
    for y in range(h_imp):
        for x in range(w_imp):
            row, col = int(mvs[y, x, 0]), int(mvs[y, x, 1])
            tot += O.get_satd(po, 8 * x, 8 * y, pr, tdiv8(x * 64 + col), tdiv8(y * 64 + row), 8, 8)
    return tot / (w_imp * h_imp)


def test_y4m_chain_to_inter_costs_and_importances():
    """frames 0-4 of the golden clip, each against its predecessor (LAST): each frame's stats grid is the next
    one's subset C; the vectors, taken at stride 2 on the device, feed b200_estimate_inter_costs_dev and then
    b200_block_importances_dev over the five frames, compared with the oracle chain"""
    from tests.test_oracle_temporal_rdo import Window, oracle_importances, oracle_intra_costs
    imgs = [np.ascontiguousarray(pl[0]) for _, pl in y4m.frames("tests/golden/small_input.y4m")][:5]
    assert len(imgs) == 5
    h, w = imgs[0].shape
    p = Params(bit_depth=8, me_lambda=4.0, full_search=1, range_scale=1)
    c = G.ctx()
    dev = [dev_pyramid(im) for im in imgs]
    wib, hib = grid_dims(w, h)
    want_maps, got_maps = [], []
    prev_o, d_prev = None, None
    for k in range(1, 5):
        want = oracle_motion(pyramid(imgs[k]), pyramid(imgs[k - 1]), w, h, p, prev_o)
        d_stats = G.dev_empty(8 * wib * hib)
        c.lookahead_motion_dev([dev[k]], [dev[k - 1]], params(p), d_stats, d_prev, None if d_prev is None else [1])
        c.synchronize()
        assert_grid_equal(G.from_dev(d_stats, STATS_DTYPE).reshape(hib, wib), want)
        prev_o, d_prev = want, d_stats
        # me_stats[2y][2x].mv, gathered on the device: (row, col) i16 per importance block (ceil grid)
        d_mv = d_stats.view(torch.int16).view(hib, wib, 4)[0::2, 0::2, :2].contiguous()
        want_mv = np.stack([want["mv_row"][0::2, 0::2], want["mv_col"][0::2, 0::2]], -1)
        got_maps.append(d_mv.reshape(-1, 2))
        want_maps.append(want_mv.reshape(-1, 2))
        floor_mv = d_mv[:h // 8, :w // 8].contiguous()
        d_scratch = G.dev_empty(8)
        d_mean = torch.zeros(1, dtype=torch.float64, device="cuda")
        c.estimate_inter_costs_dev(dev[k][0], dev[k - 1][0], floor_mv, None, d_scratch, d_mean)
        c.synchronize()
        assert float(d_mean.item()) == inter_cost_mean(imgs[k], imgs[k - 1], want_mv[:h // 8, :w // 8])

    # compute_block_importances over the window, frames walked backwards, one reference each
    steps = [(k, k - 1, 1, k - 1) for k in range(4, 0, -1)]
    win = Window(imgs, PAD, np.zeros((5, (w // 8) * (h // 8)), np.uint32), np.stack(want_maps), steps, 8)
    oracle_intra_costs(win)
    want_imp = oracle_importances(win)
    d_imp = G.dev_empty(4 * 5 * win.n_imp)
    c.block_importances_dev([q[0] for q in dev], 8, G.to_dev(win.intra), torch.stack(got_maps).contiguous(), steps,
                            d_imp)
    c.synchronize()
    got_imp = G.from_dev(d_imp, np.float32)[:5 * win.n_imp].reshape(5, win.n_imp)
    np.testing.assert_array_equal(got_imp.view(np.uint32), want_imp.view(np.uint32))
    assert (want_imp[:4] > 0).any()
    free(*dev)
