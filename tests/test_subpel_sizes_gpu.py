"""b200_subpel_rdo_dev (candidate lists) and b200_subpel_search_dev (subpel_diamond_search, me.rs:1311-1383)
at every AV1 block size from 4x4 to 64x64, bit exact against the oracle: per-candidate SAD / SATD and cost,
per-block winners, and the winner's coefficients against forward_transform(cur - put_8tap(winner)) in the
layout b200_fwd_txfm_pred_dev writes (the 32x32-chunked order for a side of 64)."""
import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O

pytestmark = pytest.mark.gpu

SIZES = O.TX_SIZES                      # (w, h) in TxSize order: tx_size index == position
TS = {s: i for i, s in enumerate(SIZES)}
EMPTY = np.uint64(2**64 - 1)
DTYPE = {8: np.uint8, 10: np.uint16, 12: np.uint16}
HBD12 = [(4, 4), (16, 8), (64, 64), (16, 64)]
CASES = [(w, h, bd) for (w, h) in SIZES for bd in (8, 10)] + [(w, h, 12) for (w, h) in HBD12]
IDS = [f"{w}x{h}-{bd}bit" for w, h, bd in CASES]
PAD = 160


def planes(W, H, bd, seed, shift=(2, -1)):
    cur, ref = G.make_planes(W, H, PAD, DTYPE[bd], seed=seed, bit_depth=bd, shift=shift)
    ocur, dcur = G.both_planes(cur, PAD)
    oref, dref = G.both_planes(ref, PAD)
    return cur, ocur, dcur, oref, dref


def tx_types(ts):
    return [t for t in range(17) if O.valid_txfm(ts, t)]


def coef_dtype(bd):
    import torch
    return torch.int16 if bd == 8 else torch.int32


def want_coefs(cur, oref, blocks, mv_row, mv_col, have, w, h, mode, bd, ts, tt):
    """forward_transform(cur - put_8tap(mv)) per block; rows of blocks without a winner are zero."""
    nb = len(blocks)
    resid = np.zeros((nb, h, w), np.int16)
    for b in np.nonzero(have)[0]:
        mr, mc = int(mv_row[b]), int(mv_col[b])
        x, y = int(blocks[b]["x"]), int(blocks[b]["y"])
        pred = O.put_8tap(oref, x + (mc >> 3), y + (mr >> 3), w, h, (mc << 1) & 15, (mr << 1) & 15, mode, mode, bd)
        resid[b] = cur[y:y + h, x:x + w].astype(np.int32) - pred.astype(np.int32)
    out = O.forward_transform_batch(resid, ts, tt, bd, coeff_i32=(bd > 8)).reshape(nb, w * h)
    out[~have] = 0
    return out


def list_winners(offs, want_sad, want_cost, cands):
    """first minimum per block (me.rs:1360-1365) of the oracle's per-candidate results"""
    nb = len(offs) - 1
    best = np.zeros(nb, B.ME_RESULT_DTYPE)
    best["cost"], best["sad"] = EMPTY, 2**32 - 1
    for b in range(nb):
        lo, hi = int(offs[b]), int(offs[b + 1])
        if lo == hi or want_cost[lo:hi].min() == EMPTY:
            continue
        k = lo + int(np.argmin(want_cost[lo:hi]))
        best[b] = (want_cost[k], want_sad[k], cands[k]["mv_row"], cands[k]["mv_col"])
    return best


def check_best(got, want, have):
    assert (got["cost"][~have] == EMPTY).all()
    for f in ("cost", "sad", "mv_row", "mv_col"):
        np.testing.assert_array_equal(got[f][have], want[f][have], err_msg=f)


@pytest.mark.parametrize("w,h,bd", CASES, ids=IDS)
def test_list_form_every_size(w, h, bd):
    """Candidate lists with sub-pel vectors, some far outside the frame (blocks that lose all of them get
    cost u64::MAX and zero coefficients); every valid tx_type of the size plus tx_size = -1; all four
    FilterModes on the sizes with a side of 4 (the 4-tap banks)."""
    import torch
    c = G.ctx()
    W, H = 192, 160
    ts = TS[(w, h)]
    cur, ocur, dcur, oref, dref = planes(W, H, bd, seed=w * 5 + h + bd)
    blocks = G.grid_blocks(W, H, w, h)                       # the frame's edge blocks included
    nb = len(blocks)
    cands, offs = G.random_cands(nb, 4, 6, seed=ts + bd, fullpel=False)
    cands["mv_col"][::7] = 16000                              # out of range: dropped by get_mv_range
    cands["mv_row"][cands["block"] % 11 == 3] = -16000        # every candidate of these blocks is dropped
    rng = np.random.default_rng(ts)
    pmv = (rng.integers(-16, 17, (nb, 4)) * 2).astype(np.int16)
    lam = 700
    d_blocks, d_cands, d_offs, d_pmv = G.to_dev(blocks), G.to_dev(cands), G.to_dev(offs), G.to_dev(pmv)
    modes = (0, 1, 2, 3) if min(w, h) == 4 else ((ts + bd) % 4,)
    first = True
    for mode in modes:
        for use_satd in (False, True):
            allow_hp = use_satd
            want_sad, want_cost = O.subpel_candidates(ocur, oref, blocks, cands, w, h, use_satd, lam, pmv,
                                                      allow_hp=allow_hp, filter_mode=mode, bit_depth=bd)
            want = list_winners(offs, want_sad, want_cost, cands)
            have = want["cost"] != EMPTY
            assert have.any() and not have.all()
            p = B.me_params(w, h, W, H, lam, allow_hp=allow_hp, use_satd=use_satd, bit_depth=bd)
            for tt in (tx_types(ts) + [-1] if first else [0]):
                d_sad, d_cost = G.dev_empty(4 * len(cands)), G.dev_empty(8 * len(cands))
                d_best = G.dev_empty(16 * nb)
                d_coef = torch.full((nb, w * h), 77, dtype=coef_dtype(bd), device="cuda")
                c.subpel_rdo_dev(dcur, dref, d_blocks, nb, d_cands, len(cands), d_offs, p, mode,
                                 ts if tt >= 0 else -1, max(tt, 0), d_pmv, d_sad, d_cost, d_best,
                                 d_coef if tt >= 0 else None)
                c.synchronize()
                np.testing.assert_array_equal(G.from_dev(d_sad, np.uint32)[:len(cands)], want_sad)
                np.testing.assert_array_equal(G.from_dev(d_cost, np.uint64)[:len(cands)], want_cost)
                check_best(G.from_dev(d_best, B.ME_RESULT_DTYPE)[:nb], want, have)
                if tt >= 0:
                    wc = want_coefs(cur, oref, blocks, want["mv_row"], want["mv_col"], have, w, h, mode, bd, ts, tt)
                    np.testing.assert_array_equal(d_coef.cpu().numpy(), wc, err_msg=f"tx_type {tt}")
                else:
                    assert (d_coef.cpu().numpy() == 77).all()     # no transform: the buffer is not touched
            first = False
    for pl in (dcur, dref):
        c.plane_free(pl)


def diamond_oracle(ocur, oref, blocks, start, w, h, use_satd, lam, pmv, allow_hp, mode, bd):
    import ctypes as C
    L = O.lib()
    L.orc_subpel_diamond_search_blocks.restype = None
    L.orc_subpel_diamond_search_blocks.argtypes = [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t] + [C.c_int] * 3 + \
        [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p] + [C.c_int] * 3 + [C.c_void_p, C.c_int]
    res = np.ascontiguousarray(start.copy())
    L.orc_subpel_diamond_search_blocks(ocur.origin_ptr(), ocur.stride, oref.origin_ptr(), oref.stride, ocur.bpp,
                                       2 * ((ocur.width + 7) >> 3), 2 * ((ocur.height + 7) >> 3), O.ptr(blocks),
                                       len(blocks), w, h, int(use_satd), lam, O.ptr(pmv), int(allow_hp), mode, bd,
                                       O.ptr(res), 0)
    return res


def edge_starts(blocks, W, H, w, h, rng):
    """Full-pel starts near the true shift; blocks on the right / bottom frame edge start exactly on the
    get_mv_range limit, so the diamond's points beyond it are clipped."""
    nb = len(blocks)
    st = np.zeros(nb, B.CAND_DTYPE)
    st["block"] = np.arange(nb)
    st["mv_row"] = rng.integers(-2, 2, nb) * 8
    st["mv_col"] = rng.integers(0, 4, nb) * 8
    for b in range(nb):
        x, y = int(blocks[b]["x"]), int(blocks[b]["y"])
        x_min, x_max, y_min, y_max = G.mv_range(W, H, x, y, w, h)
        if x + w >= W and b % 2 == 0:
            st["mv_col"][b] = x_max
        if y + h >= H and b % 3 == 0:
            st["mv_row"][b] = y_max
        if x == 0 and b % 2 == 1:
            st["mv_col"][b] = x_min
    return st


def start_results(ocur, oref, blocks, st, w, h, use_satd, lam, pmv, allow_hp):
    sad, cost = O.fullpel_candidates(ocur, oref, blocks, st, w, h, use_satd, lam, pmv, allow_hp)
    start = np.zeros(len(blocks), B.ME_RESULT_DTYPE)
    start["cost"], start["sad"], start["mv_row"], start["mv_col"] = cost, sad, st["mv_row"], st["mv_col"]
    return start


@pytest.mark.parametrize("w,h,bd", CASES, ids=IDS)
def test_diamond_form_every_size(w, h, bd):
    """subpel_diamond_search from full-pel starts (frame-edge blocks on their mv-range limits), SAD and SATD,
    allow_hp both ways, one FilterMode per combination (all four per size), with the transform; then the
    winners' SAD and cost against the two-launch list path (b200_me_subpel_candidates_dev)."""
    import torch
    c = G.ctx()
    W, H = 192, 160
    ts = TS[(w, h)]
    cur, ocur, dcur, oref, dref = planes(W, H, bd, seed=3 * w + h + bd)
    blocks = G.grid_blocks(W, H, w, h)
    nb = len(blocks)
    rng = np.random.default_rng(ts + 100 * bd)
    pmv = (rng.integers(-8, 9, (nb, 4)) * 2).astype(np.int16)
    lam = 500
    st = edge_starts(blocks, W, H, w, h, rng)
    d_blocks, d_pmv = G.to_dev(blocks), G.to_dev(pmv)
    types = tx_types(ts)
    moved = 0
    for k, (use_satd, allow_hp) in enumerate(((False, False), (True, False), (False, True), (True, True))):
        mode = (k + ts) % 4
        tt = types[(k * 5 + ts) % len(types)] if k < 3 else -1
        start = start_results(ocur, oref, blocks, st, w, h, use_satd, lam, pmv, allow_hp)
        want = diamond_oracle(ocur, oref, blocks, start, w, h, use_satd, lam, pmv, allow_hp, mode, bd)
        p = B.me_params(w, h, W, H, lam, allow_hp=allow_hp, use_satd=use_satd, bit_depth=bd)
        d_best = G.dev_empty(16 * nb)
        d_coef = torch.full((nb, w * h), 77, dtype=coef_dtype(bd), device="cuda")
        c.subpel_search_dev(dcur, dref, d_blocks, nb, G.to_dev(start), p, d_best, mode, ts if tt >= 0 else -1,
                            max(tt, 0), d_pmv, d_coef if tt >= 0 else None)
        c.synchronize()
        got = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:nb]
        for f in ("cost", "sad", "mv_row", "mv_col"):
            np.testing.assert_array_equal(got[f], want[f], err_msg=f"satd={use_satd} hp={allow_hp}: {f}")
        moved += int(((got["mv_row"] != start["mv_row"]) | (got["mv_col"] != start["mv_col"])).sum())
        if tt >= 0:
            wc = want_coefs(cur, oref, blocks, want["mv_row"], want["mv_col"], np.ones(nb, bool), w, h, mode, bd,
                            ts, tt)
            np.testing.assert_array_equal(d_coef.cpu().numpy(), wc, err_msg=f"tx_type {tt}")
        else:
            assert (d_coef.cpu().numpy() == 77).all()
        # the same vectors through the list path: identical SAD and cost
        lc = np.zeros(nb, B.CAND_DTYPE)
        lc["block"], lc["mv_row"], lc["mv_col"] = np.arange(nb), got["mv_row"], got["mv_col"]
        d_sad, d_cost = G.dev_empty(4 * nb), G.dev_empty(8 * nb)
        c.me_subpel_candidates_dev(dcur, dref, d_blocks, nb, G.to_dev(lc), nb, p, mode, None, d_pmv, d_sad, d_cost)
        c.synchronize()
        np.testing.assert_array_equal(G.from_dev(d_sad, np.uint32)[:nb], got["sad"])
        np.testing.assert_array_equal(G.from_dev(d_cost, np.uint64)[:nb], got["cost"])
    assert moved > 0
    for pl in (dcur, dref):
        c.plane_free(pl)


@pytest.mark.parametrize("w,h,bd", [(8, 8, 8), (64, 64, 10)])
def test_ragged_second_grid_stride_trip(w, h, bd):
    """More blocks than the capped grid holds (16 CTAs per SM, at most 8 warps each): every warp takes a
    second trip, and the last one is ragged.  The blocks repeat a small set, so the oracle runs once."""
    import torch
    c = G.ctx()
    W, H = 192, 160
    ts = TS[(w, h)]
    cur, ocur, dcur, oref, dref = planes(W, H, bd, seed=11 + w)
    base = G.grid_blocks(W, H, w, h)
    cap = torch.cuda.get_device_properties(0).multi_processor_count * 16 * 8
    reps = -(-(cap + 123) // len(base))
    n = cap + 123
    blocks = np.ascontiguousarray(np.tile(base, reps)[:n])
    nb0 = len(base)
    rng = np.random.default_rng(5)
    pmv0 = (rng.integers(-8, 9, (nb0, 4)) * 2).astype(np.int16)
    pmv = np.ascontiguousarray(np.tile(pmv0, (reps, 1))[:n])
    lam = 400
    p = B.me_params(w, h, W, H, lam, use_satd=True, bit_depth=bd)
    d_blocks, d_pmv = G.to_dev(blocks), G.to_dev(pmv)
    # list form: two candidates per block
    c0, o0 = G.random_cands(nb0, 2, 4, seed=9, fullpel=False, jitter=False)
    cands = np.zeros(2 * n, B.CAND_DTYPE)
    cands["block"] = np.repeat(np.arange(n, dtype=np.uint32), 2)
    cands["mv_row"] = np.tile(c0["mv_row"], reps)[:2 * n]
    cands["mv_col"] = np.tile(c0["mv_col"], reps)[:2 * n]
    offs = (np.arange(n + 1) * 2).astype(np.uint32)
    s0, k0 = O.subpel_candidates(ocur, oref, base, c0, w, h, True, lam, pmv0, bit_depth=bd)
    w0 = list_winners(o0, s0, k0, c0)
    have0 = w0["cost"] != EMPTY
    coef0 = want_coefs(cur, oref, base, w0["mv_row"], w0["mv_col"], have0, w, h, 0, bd, ts, 0)
    d_cost, d_best = G.dev_empty(8 * 2 * n), G.dev_empty(16 * n)
    d_coef = torch.full((n, w * h), 77, dtype=coef_dtype(bd), device="cuda")
    c.subpel_rdo_dev(dcur, dref, d_blocks, n, G.to_dev(cands), 2 * n, G.to_dev(offs), p, 0, ts, 0, d_pmv, None,
                     d_cost, d_best, d_coef)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_cost, np.uint64)[:2 * n], np.tile(k0, reps)[:2 * n])
    got = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:n]
    check_best(got, np.tile(w0, reps)[:n], np.tile(have0, reps)[:n])
    np.testing.assert_array_equal(d_coef.cpu().numpy(), np.tile(coef0, (reps, 1))[:n])
    # diamond form
    st = edge_starts(base, W, H, w, h, rng)
    start0 = start_results(ocur, oref, base, st, w, h, True, lam, pmv0, False)
    want0 = diamond_oracle(ocur, oref, base, start0, w, h, True, lam, pmv0, False, 0, bd)
    coef0 = want_coefs(cur, oref, base, want0["mv_row"], want0["mv_col"], np.ones(nb0, bool), w, h, 0, bd, ts, 0)
    d_coef.fill_(77)
    c.subpel_search_dev(dcur, dref, d_blocks, n, G.to_dev(np.tile(start0, reps)[:n]), p, d_best, 0, ts, 0, d_pmv,
                        d_coef)
    c.synchronize()
    got = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:n]
    want = np.tile(want0, reps)[:n]
    for f in ("cost", "sad", "mv_row", "mv_col"):
        np.testing.assert_array_equal(got[f], want[f], err_msg=f)
    np.testing.assert_array_equal(d_coef.cpu().numpy(), np.tile(coef0, (reps, 1))[:n])
    for pl in (dcur, dref):
        c.plane_free(pl)


@pytest.mark.parametrize("w,h", [(64, 64), (4, 16)])
def test_zero_and_one_block(w, h):
    import torch
    c = G.ctx()
    W, H, bd = 128, 96, 8
    ts = TS[(w, h)]
    cur, ocur, dcur, oref, dref = planes(W, H, bd, seed=21)
    blocks = G.grid_blocks(W, H, w, h)[1:2].copy()
    p = B.me_params(w, h, W, H, 300, use_satd=True, bit_depth=bd)
    dummy = G.dev_empty(64)
    n0 = c.launches
    c.subpel_rdo_dev(dcur, dref, dummy, 0, dummy, 0, dummy, p, 0, ts, 0, None, None, None, dummy, dummy)
    c.subpel_search_dev(dcur, dref, dummy, 0, dummy, p, dummy, 0, ts, 0, None, dummy)
    assert c.launches == n0
    st = np.zeros(1, B.CAND_DTYPE)
    st["mv_row"], st["mv_col"] = -8, 16
    pmv = np.zeros((1, 4), np.int16)
    start = start_results(ocur, oref, blocks, st, w, h, True, 300, pmv, False)
    want = diamond_oracle(ocur, oref, blocks, start, w, h, True, 300, pmv, False, 0, bd)
    d_best = G.dev_empty(16)
    d_coef = torch.zeros((1, w * h), dtype=torch.int16, device="cuda")
    c.subpel_search_dev(dcur, dref, G.to_dev(blocks), 1, G.to_dev(start), p, d_best, 0, ts, 0, None, d_coef)
    c.synchronize()
    got = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:1]
    for f in ("cost", "sad", "mv_row", "mv_col"):
        np.testing.assert_array_equal(got[f], want[f], err_msg=f)
    wc = want_coefs(cur, oref, blocks, want["mv_row"], want["mv_col"], np.ones(1, bool), w, h, 0, bd, ts, 0)
    np.testing.assert_array_equal(d_coef.cpu().numpy(), wc)
    for pl in (dcur, dref):
        c.plane_free(pl)


def test_rejections_launch_nothing():
    """Sizes that are not AV1 block sizes, and transforms that do not match the block, are B200_ERR_ARG
    before any launch."""
    c = G.ctx()
    W, H = 128, 96
    cur, ocur, dcur, oref, dref = planes(W, H, 8, seed=1)
    buf = G.dev_empty(1 << 16)
    calls = []
    for w, h in ((128, 128), (8, 64), (12, 12), (64, 128), (2, 2), (64, 8), (0, 0), (24, 16)):
        calls.append((B.me_params(w, h, W, H, 100), 0, 0))
    calls += [(B.me_params(16, 8, W, H, 100), TS[(8, 16)], 0),       # transform of another size
              (B.me_params(64, 64, W, H, 100), TS[(64, 64)], 9),     # IDTX is not a 64-point transform
              (B.me_params(32, 64, W, H, 100), TS[(32, 64)], 1),
              (B.me_params(4, 4, W, H, 100), TS[(4, 4)], 17)]
    for p, ts, tt in calls:
        n0 = c.launches
        for fn in (lambda: c.subpel_rdo_dev(dcur, dref, buf, 1, buf, 1, buf, p, 0, ts, tt, None, buf, buf, buf, buf),
                   lambda: c.subpel_search_dev(dcur, dref, buf, 1, buf, p, buf, 0, ts, tt, None, buf)):
            with pytest.raises(B.B200Error) as e:
                fn()
            assert e.value.status == B.ERR_ARG
        assert c.launches == n0
    for pl in (dcur, dref):
        c.plane_free(pl)


def halfpel_planes(W, H, bd, seed):
    """low-passed noise; cur = ref moved by (+5.5, -3) px plus noise, so the sub-pel stage has work at every
    block size: the true vector is (row -24, col +44) in eighth pels, between full-pel positions"""
    rng = np.random.default_rng(seed)
    maxv = (1 << bd) - 1
    base = rng.integers(0, maxv + 1, (H + 64, W + 64)).astype(np.float64)
    k = np.ones(5) / 5.0
    base = np.apply_along_axis(lambda r: np.convolve(r, k, mode="same"), 1, base)
    base = np.apply_along_axis(lambda r: np.convolve(r, k, mode="same"), 0, base)
    base = (base - base.min()) / (base.max() - base.min()) * maxv
    ref = base[32:32 + H, 32:32 + W]
    cur = (base[29:29 + H, 37:37 + W] + base[29:29 + H, 38:38 + W]) / 2 + rng.normal(0, 1, (H, W))
    ref = np.ascontiguousarray(np.clip(np.rint(ref), 0, maxv).astype(DTYPE[bd]))
    cur = np.ascontiguousarray(np.clip(np.rint(cur), 0, maxv).astype(DTYPE[bd]))
    ocur, dcur = G.both_planes(cur, PAD)
    oref, dref = G.both_planes(ref, PAD)
    return cur, ocur, dcur, oref, dref


def chain_predictors(nb, seed, shift):
    """one subset of predictors per block, scattered around the true motion in full pels"""
    rng = np.random.default_rng(seed)
    counts = rng.integers(1, 6, nb)
    offs = np.zeros(nb + 1, np.uint32)
    offs[1:] = np.cumsum(counts)
    preds = np.zeros(int(offs[-1]), B.CAND_DTYPE)
    mv = (np.array([shift[1], shift[0]]) + rng.integers(-4, 5, (len(preds), 2))) * 8
    preds["mv_row"], preds["mv_col"] = mv[:, 0], mv[:, 1]
    return preds, offs


@pytest.mark.parametrize("w,h", [(64, 64), (32, 16)])
@pytest.mark.parametrize("bd", [8, 10])
def test_estimate_motion_chain_1080p(w, h, bd):
    """estimate_motion (me.rs:536-631) on a 1080p pair: full_pixel_me on the device, the SATD rescore of each
    winner (me.rs:596-616, one candidate per block), then the diamond search with the transform - equal to
    the oracle's full_pixel_me_blocks -> fullpel_candidates(use_satd) -> subpel_diamond_search."""
    import torch
    c = G.ctx()
    W, H = 1920, 1080
    ts = TS[(w, h)]
    shift = (5, -3)
    cur, ocur, dcur, oref, dref = halfpel_planes(W, H, bd, seed=w + h + bd)
    blocks = G.grid_blocks(W, H, w, h)
    nb = len(blocks)
    rng = np.random.default_rng(bd)
    pmv = (rng.integers(-6, 7, (nb, 4)) * 8).astype(np.int16)
    lam = 1200 << (bd - 8)
    preds, offs = chain_predictors(nb, bd + w, shift)
    d_blocks, d_pmv = G.to_dev(blocks), G.to_dev(pmv)
    # 1. full-pel search
    full = O.full_pixel_me_blocks(ocur, oref, blocks, preds, offs, 1, w, h, lam, pmv)
    p_sad = B.me_params(w, h, W, H, lam, bit_depth=bd)
    d_full = G.dev_empty(16 * nb)
    c.me_search_dev(dcur, dref, d_blocks, nb, G.to_dev(preds), G.to_dev(offs), 1, p_sad, d_full, d_pmv)
    c.synchronize()
    got_full = G.from_dev(d_full, B.ME_RESULT_DTYPE)[:nb]
    for f in ("cost", "sad", "mv_row", "mv_col"):
        np.testing.assert_array_equal(got_full[f], full[f], err_msg=f"full-pel {f}")
    # 2. SATD rescore of the winner
    rc = np.zeros(nb, B.CAND_DTYPE)
    rc["block"], rc["mv_row"], rc["mv_col"] = np.arange(nb), full["mv_row"], full["mv_col"]
    sad, cost = O.fullpel_candidates(ocur, oref, blocks, rc, w, h, True, lam, pmv)
    p_satd = B.me_params(w, h, W, H, lam, use_satd=True, bit_depth=bd)
    d_sad, d_cost = G.dev_empty(4 * nb), G.dev_empty(8 * nb)
    c.me_candidates_dev(dcur, dref, d_blocks, nb, G.to_dev(rc), nb, p_satd, None, d_pmv, d_sad, d_cost)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_sad, np.uint32)[:nb], sad)
    np.testing.assert_array_equal(G.from_dev(d_cost, np.uint64)[:nb], cost)
    start = np.zeros(nb, B.ME_RESULT_DTYPE)
    start["cost"], start["sad"], start["mv_row"], start["mv_col"] = cost, sad, full["mv_row"], full["mv_col"]
    # 3. sub-pel diamond search + the winner's transform
    want = diamond_oracle(ocur, oref, blocks, start, w, h, True, lam, pmv, False, 0, bd)
    d_start = G.dev_empty(16 * nb)
    d_start.copy_(G.to_dev(start))
    d_coef = torch.zeros((nb, w * h), dtype=coef_dtype(bd), device="cuda")
    c.subpel_search_dev(dcur, dref, d_blocks, nb, d_start, p_satd, d_start, 0, ts, 0, d_pmv, d_coef)  # in place
    c.synchronize()
    got = G.from_dev(d_start, B.ME_RESULT_DTYPE)[:nb]
    for f in ("cost", "sad", "mv_row", "mv_col"):
        np.testing.assert_array_equal(got[f], want[f], err_msg=f"sub-pel {f}")
    assert ((got["mv_row"] != start["mv_row"]) | (got["mv_col"] != start["mv_col"])).any()   # the sub-pel stage moved
    wc = want_coefs(cur, oref, blocks, want["mv_row"], want["mv_col"], np.ones(nb, bool), w, h, 0, bd, ts, 0)
    np.testing.assert_array_equal(d_coef.cpu().numpy(), wc)
    for pl in (dcur, dref):
        c.plane_free(pl)
