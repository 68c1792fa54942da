"""GPU parity of the encode-time motion search (rav1e_b200/csrc/encode_me.cu, b200_estimate_motion_dev) with the
oracle (oracle/encode_me.c: orc_estimate_motion_items): every field of every item, all 19 sizes in one call, at 8,
10 and 12 bit, SATD and SAD, with and without high-precision vectors, every filter mode, one-tile and multi-tile
grids, pmv pairs on the range borders, several slots, invalid items; item counts past the launch grid; the stats
grids straight from b200_lookahead_motion_dev; a 1080p lookahead -> search -> inter-mode screening chain with nothing
going to the host between the calls; the existing device calls composed by hand; the pad rule and the rejections."""
import numpy as np
import pytest
import torch

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_oracle_encode_me import (ITEM_DTYPE, TX_SIZES, Enc, grid_dims, min_pad, model_predictors)
from tests.test_oracle_lookahead_me import STATS_DTYPE, Params

pytestmark = pytest.mark.gpu

EMPTY = (2**64 - 1, 2**32 - 1, 0, 0)


def params(e: Enc):
    return B.EncMeParams(e.bd, e.allow_hp, e.me_lambda, e.use_satd, e.filter_mode, e.tiles[0], e.tiles[1])


def upload(e: Enc, pad=None):
    c = G.ctx()
    pad = e.pad if pad is None else pad
    return c.plane_from_host(e.src_img, pad), [c.plane_from_host(r, pad) for r in e.ref_imgs]


def free(src, refs):
    for p in [src] + refs:
        G.ctx().plane_free(p)


def device(e: Enc, items, size_end, planes=None, d_stats=None):
    c = G.ctx()
    src, refs = planes if planes is not None else upload(e)
    d_stats = G.to_dev(np.ascontiguousarray(e.stats, STATS_DTYPE)) if d_stats is None else d_stats
    d_prev = None if e.prev is None else G.to_dev(np.ascontiguousarray(e.prev, STATS_DTYPE))
    d_out = G.dev_empty(16 * len(items))
    l0 = c.launches
    c.estimate_motion_dev(src, refs, d_stats, params(e), size_end, G.to_dev(items), len(items), d_out, d_prev,
                          e.has_prev)
    c.synchronize()
    nlaunch = c.launches - l0
    if planes is None:
        free(src, refs)
    return G.from_dev(d_out, B.ME_RESULT_DTYPE)[:len(items)], nlaunch


def assert_equal(got, want, items):
    for f in ("cost", "sad", "mv_row", "mv_col"):
        bad = np.nonzero(got[f] != want[f])[0]
        assert len(bad) == 0, (f, len(bad), items[bad[:3]], got[bad[:3]], want[bad[:3]])


# (width, height, bit depth, use_satd, allow_hp, filter mode, tiles, prev, pmv on the range border)
CASES = [(200, 120, 8, 1, 0, 0, (64, 64), True, False),
         (203, 117, 10, 0, 1, 1, (1, 1), True, True),
         (136, 88, 12, 1, 1, 2, (2, 1), True, False),
         (104, 72, 8, 0, 0, 3, (1, 2), False, True),
         (200, 120, 8, 1, 1, 1, (1, 1), True, True),
         (203, 117, 10, 1, 0, 3, (64, 64), False, False)]


@pytest.mark.parametrize("case", CASES, ids=[f"{w}x{h}-bd{bd}-satd{s}-hp{hp}-f{m}-t{t[0]}x{t[1]}-prev{int(p)}-border{int(b)}"
                                             for w, h, bd, s, hp, m, t, p, b in CASES])
def test_device_matches_oracle_every_size_in_one_call(case):
    w, h, bd, use_satd, hp, mode, tiles, prev, border = case
    e = Enc(w, h, bd=bd, nslots=3, tiles=tiles, prev=prev, seed=w + bd, allow_hp=hp, use_satd=use_satd,
            filter_mode=mode)
    items, size_end = e.items(set(range(19)), seed=bd + mode, per_size=40, pmv_near_border=border, invalid=4)
    want = e.oracle(items, size_end)
    got, nlaunch = device(e, items, size_end)
    assert nlaunch == 19
    assert_equal(got, want, items)
    wib, hib = grid_dims(w, h)
    invalid = (items["slot"] >= 3) | (items["x4"] >= wib) | (items["y4"] >= hib)
    assert invalid.sum() == 19 * 4
    assert all(tuple(got[i][f] for f in ("cost", "sad", "mv_row", "mv_col")) == EMPTY for i in np.nonzero(invalid)[0])
    assert not (got["cost"][~invalid] == EMPTY[0]).any()


def test_lookahead_grids_straight_from_the_device_and_past_the_grid_cap():
    """b200_lookahead_motion_dev's output stays on the device and feeds the call; 4x4 items at every position of
    every slot (more warps than the launch grid holds) and a few 64x64 ones"""
    w, h = 520, 264
    e = Enc(w, h, bd=8, nslots=3, tiles=(2, 2), prev=False, lookahead=True, seed=9)
    c = G.ctx()
    la = Params(bit_depth=8, me_lambda=e.me_lambda, tile_w_sb=2, tile_h_sb=2)
    from tests.test_lookahead_me_gpu import dev_pyramid, params as la_params
    dcur = dev_pyramid(e.src_img)
    drefs = [dev_pyramid(r) for r in e.ref_imgs]
    wib, hib = grid_dims(w, h)
    d_stats = G.dev_empty(8 * 3 * wib * hib)
    c.lookahead_motion_dev([dcur] * 3, drefs, la_params(la), d_stats)
    every, _ = e.items({0}, seed=2)            # 4x4 items at every position, once per slot
    every = np.concatenate([every] * 3)
    every["slot"] = np.repeat(np.arange(3), len(every) // 3)
    big, _ = e.items({4}, seed=3, per_size=30)
    items = np.ascontiguousarray(np.concatenate([every, big]))
    n44 = len(every)
    size_end = np.full(19, len(items), np.uint32)
    size_end[:4] = n44
    got, _ = device(e, items, size_end, d_stats=d_stats)
    host_stats = G.from_dev(d_stats, STATS_DTYPE)[:3 * wib * hib].reshape(3, hib, wib)
    assert host_stats.tobytes() == e.stats.tobytes()   # the device grids are the oracle's
    want = e.oracle(items, size_end)
    assert_equal(got, want, items)
    props = torch.cuda.get_device_properties(0)
    assert n44 > props.multi_processor_count * 16 * 8 // 2   # 4x4 groups run 8 warps per CTA, 16 CTAs per SM
    for pyr in [dcur] + drefs:
        for q in pyr:
            c.plane_free(q)


def test_min_pad_accepted_one_less_rejected():
    w, h = 203, 117
    sizes = {1, 11, 14}   # 8x8, 32x64, 16x4: the 64-high group sets the pad
    need = min_pad(w, h, [TX_SIZES[s] for s in sizes])
    e = Enc(w, h, bd=10, nslots=2, tiles=(1, 1), seed=4, pad=need, use_satd=1)
    items, size_end = e.items(sizes, seed=5, per_size=60, pmv_near_border=True)
    got, _ = device(e, items, size_end)
    assert_equal(got, e.oracle(items, size_end), items)
    c = G.ctx()
    for side in range(3):   # one pixel less on the source, or on one reference
        src, refs = upload(e, need)
        short = c.plane_from_host([e.src_img, e.ref_imgs[0], e.ref_imgs[1]][side], need - 1)
        if side == 0:
            src, old = short, src
        else:
            refs[side - 1], old = short, refs[side - 1]
        l0 = c.launches
        with pytest.raises(B.B200Error) as ex:
            device(e, items, size_end, planes=(src, refs))
        assert ex.value.status == B.ERR_ARG and c.launches == l0
        free(src, refs)
        c.plane_free(old)


def test_equals_composed_device_calls():
    """the host gather, then b200_me_search_dev (all_mvs), b200_me_candidates_dev (SATD at the winner) and
    b200_subpel_search_dev, for 16x16 blocks"""
    w, h = 200, 120
    e = Enc(w, h, bd=8, nslots=1, tiles=(1, 1), seed=12, use_satd=1, allow_hp=1, filter_mode=2)
    items, size_end = e.items({2}, seed=6)
    items["slot"] = 0
    got, _ = device(e, items, size_end)
    c = G.ctx()
    src, refs = upload(e)
    n = len(items)
    blocks = np.zeros(n, B.BLOCK_DTYPE)
    blocks["x"], blocks["y"] = items["x4"] * 4, items["y4"] * 4
    lists = [model_predictors(e.stats[0], e.prev[0], w, h, e.tiles, int(i["x4"]), int(i["y4"]), 16, 16) for i in items]
    offs = np.zeros(n + 1, np.uint32)
    offs[1:] = np.cumsum([len(x) for x in lists])
    preds = np.zeros(int(offs[-1]), B.CAND_DTYPE)
    flat = [v for x in lists for v in x]
    preds["mv_row"], preds["mv_col"] = [v[0] for v in flat], [v[1] for v in flat]
    pmv = np.ascontiguousarray(items["pmv"].astype(np.int16))
    d_blocks, d_pmv = G.to_dev(blocks), G.to_dev(pmv)
    p_sad = B.me_params(16, 16, w, h, e.lam(), allow_hp=True, bit_depth=8)
    d_best = G.dev_empty(16 * n)
    c.me_search_dev(src, refs[0], d_blocks, n, G.to_dev(preds), G.to_dev(offs), 1, p_sad, d_best, d_pmv)
    full = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:n].copy()
    cands = np.zeros(n, B.CAND_DTYPE)
    cands["block"] = np.arange(n)
    cands["mv_row"], cands["mv_col"] = full["mv_row"], full["mv_col"]
    p_satd = B.me_params(16, 16, w, h, e.lam(), allow_hp=True, use_satd=True, bit_depth=8)
    d_sad, d_cost = G.dev_empty(4 * n), G.dev_empty(8 * n)
    c.me_candidates_dev(src, refs[0], d_blocks, n, G.to_dev(cands), n, p_satd, None, d_pmv, d_sad, d_cost)
    full["sad"] = G.from_dev(d_sad, np.uint32)[:n]
    full["cost"] = G.from_dev(d_cost, np.uint64)[:n]
    d_out = G.dev_empty(16 * n)
    c.subpel_search_dev(src, refs[0], d_blocks, n, G.to_dev(full), p_satd, d_out, e.filter_mode, d_pmv=d_pmv)
    c.synchronize()
    assert_equal(got, G.from_dev(d_out, B.ME_RESULT_DTYPE)[:n], items)
    free(src, refs)


def test_invalid_arguments_rejected_without_launch():
    e = Enc(72, 40, bd=8, nslots=2, seed=3)
    items, size_end = e.items({1}, per_size=8)
    c = G.ctx()
    src, refs = upload(e)
    d_stats = G.to_dev(np.ascontiguousarray(e.stats, STATS_DTYPE))
    d_prev = G.to_dev(np.ascontiguousarray(e.prev, STATS_DTYPE))
    d_items, d_out = G.to_dev(items), G.dev_empty(16 * len(items))
    other = c.plane_from_host(np.zeros((40, 72), np.uint16), e.pad)
    small = c.plane_from_host(e.ref_imgs[0][:32, :64], e.pad)

    def call(refs_=refs, src_=src, p=None, ends=size_end, nitems=len(items), prev=d_prev, flags=e.has_prev):
        c.estimate_motion_dev(src_, refs_, d_stats, p or params(e), ends, d_items, nitems, d_out, prev, flags)

    call()
    bad_p = []
    for field, v in (("bit_depth", 10), ("tile_w_sb", 0), ("tile_h_sb", 0), ("filter_mode", 4)):
        q = params(e)
        setattr(q, field, v)
        bad_p.append(q)
    ends_dec = size_end.copy()
    ends_dec[0], ends_dec[1] = 5, 3
    ends_short = size_end.copy()
    ends_short[-1] -= 1
    bad = [dict(refs_=[], prev=None, flags=None), dict(refs_=refs * 4, prev=None, flags=None),
           dict(refs_=[refs[0], other]), dict(refs_=[refs[0], small]),
           dict(src_=other)] + [dict(p=q) for q in bad_p] + \
          [dict(prev=None), dict(flags=None), dict(ends=ends_dec), dict(ends=ends_short)]
    for kw in bad:
        l0 = c.launches
        with pytest.raises(B.B200Error) as ex:
            call(**kw)
        assert ex.value.status == B.ERR_ARG and c.launches == l0, kw
    free(src, refs)
    c.plane_free(other)
    c.plane_free(small)


def test_1080p_lookahead_search_screen_chain():
    """b200_lookahead_motion_dev -> b200_estimate_motion_dev -> b200_inter_mode_screen_dev for every 16x16 block of
    a 1080p frame over three slots (8x8 items of every slot too), the screening items built on the device from the
    results: each slot's mv_stack[0] vector, then NEWMV where the result is non-zero and equals neither predictor
    (rdo.rs:1219-1230); against the same chain on the oracles"""
    from tests.test_lookahead_me_gpu import dev_pyramid, params as la_params
    from tests.test_oracle_inter_screen import ITEM_DTYPE as SCREEN_ITEM, inter_mode_screen, origins
    w, h, pad = 1920, 1080, 128
    e = Enc(w, h, bd=8, nslots=3, tiles=(64, 64), prev=False, lookahead=True, seed=21, pad=pad, use_satd=1,
            me_lambda=3.0)
    c = G.ctx()
    wib, hib = grid_dims(w, h)
    dcur = dev_pyramid(e.src_img)
    drefs = [dev_pyramid(r) for r in e.ref_imgs]
    src, refs = upload(e)
    rng = np.random.default_rng(4)
    groups = []
    for s, bw in ((1, 8), (2, 16)):
        xs, ys = np.meshgrid(np.arange(0, wib, bw // 4), np.arange(0, hib, bw // 4))
        it = np.zeros(3 * xs.size, ITEM_DTYPE)
        it["x4"], it["y4"] = np.tile(xs.ravel(), 3), np.tile(ys.ravel(), 3)
        it["slot"] = np.repeat(np.arange(3), xs.size)
        it["pmv"] = rng.integers(-6, 7, (len(it), 2, 2)) * 8
        groups.append(it)
    items = np.concatenate(groups)
    size_end = np.zeros(19, np.uint32)
    size_end[1:] = len(groups[0])
    size_end[2:] = len(items)
    n16 = len(groups[1]) // 3
    d_items = G.to_dev(items)
    d_stats = G.dev_empty(8 * 3 * wib * hib)
    d_out = G.dev_empty(16 * len(items))
    d_satd, d_order = G.dev_empty(n16 * 20 * 4), G.dev_empty(n16 * 20)
    xo, yo = origins(8)
    pmv16 = torch.from_numpy(items["pmv"][len(groups[0]):].astype(np.int16)).cuda().view(3, n16, 2, 2)
    hdr = np.zeros((n16, 4), np.int16)
    hdr[:, 0], hdr[:, 1] = groups[1]["x4"][:n16] * 4, groups[1]["y4"][:n16] * 4
    d_hdr = torch.from_numpy(hdr).cuda()

    def screen_items(res16, pmv):
        """(3, n16, 2) result vectors, (3, n16, 2, 2) predictors -> (n16, 124) int16 screening items"""
        single = torch.full((3, n16), 0, dtype=torch.int16, device=res16.device)
        refw = (torch.arange(3, device=res16.device, dtype=torch.int32)[:, None] + (0xFF << 8)).to(torch.int32)
        refw = ((refw + 32768) % 65536 - 32768).to(torch.int16).expand(3, n16)
        near = torch.stack([pmv[:, :, 0, 0], pmv[:, :, 0, 1], single, single, refw, single], -1)   # (3, n16, 6)
        new = torch.stack([res16[:, :, 0], res16[:, :, 1], single, single, refw, single], -1)
        inc = ~((res16 == pmv[:, :, 0]).all(-1) | (res16 == pmv[:, :, 1]).all(-1) | (res16 == 0).all(-1))
        ents = torch.cat([near, new], 0).permute(1, 0, 2)            # (n16, 6, 6)
        keep = torch.cat([torch.ones_like(inc), inc], 0).permute(1, 0)  # (n16, 6)
        key = torch.arange(6, device=res16.device)[None] + 16 * (~keep).to(torch.int64)
        order = torch.sort(key, dim=1, stable=True).indices
        ents = torch.gather(ents, 1, order[:, :, None].expand(-1, -1, 6)) * keep.gather(1, order)[:, :, None]
        cands = torch.zeros((n16, 20, 6), dtype=torch.int16, device=res16.device)
        cands[:, :6] = ents
        nent = keep.sum(1).to(torch.int16)
        head = d_hdr.clone()
        head[:, 2] = 6 + 256 * nent     # bsize BLOCK_16X16 = 6, n
        return torch.cat([head, cands.reshape(n16, 120)], 1).contiguous()

    def chain():
        c.lookahead_motion_dev([dcur] * 3, drefs, la_params(Params(bit_depth=8, me_lambda=e.me_lambda)), d_stats)
        c.estimate_motion_dev(src, refs, d_stats, params(e), size_end, d_items, len(items), d_out)
        res = d_out.view(torch.int16).view(-1, 8)[len(groups[0]):, 6:8].reshape(3, n16, 2)
        sitems = screen_items(res, pmv16)
        c.inter_mode_screen_dev(src, (0, 0, w, h), refs, xo, yo, 0, 8, sitems, n16, d_satd, d_order)

    chain()
    c.synchronize()
    assert G.from_dev(d_stats, STATS_DTYPE)[:3 * wib * hib].tobytes() == e.stats.tobytes()
    got = G.from_dev(d_out, B.ME_RESULT_DTYPE)[:len(items)]
    want = e.oracle(items, size_end)
    assert_equal(got, want, items)
    w16 = want[len(groups[0]):]
    sitems = screen_items(torch.from_numpy(np.stack([w16["mv_row"], w16["mv_col"]], -1).astype(np.int16))
                          .reshape(3, n16, 2).cuda(), pmv16).cpu().numpy().view(SCREEN_ITEM).reshape(n16)
    satd, order = inter_mode_screen(e.src, (0, 0, w, h), e.refs, xo, yo, 0, 8, sitems)
    assert (G.from_dev(d_satd, np.uint32)[:n16 * 20].reshape(n16, 20) == satd).all()
    assert (G.from_dev(d_order, np.uint8)[:n16 * 20].reshape(n16, 20) == order).all()
    assert (sitems["n"] > 3).mean() > 0.5   # NEWMV entries are present for most blocks
    for pyr in [dcur] + drefs:
        for q in pyr:
            c.plane_free(q)
    free(src, refs)
