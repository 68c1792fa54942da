"""b200_intra_tx_size_type_dev against the oracle (oracle/tx_size_type.c), bit for bit: the best (size, type),
the rd's f64 bits and every candidate record."""
import numpy as np
import pytest
import torch

import ctypes as C

from rav1e_b200.backend import COEFF_CHAIN_DTYPE, ERR_ARG, TX_BEST_DTYPE, TX_CAND_DTYPE, B200Error
from tests import coeff_rate_cases as K
from tests import gpu_util as G
from tests import oracle_lib as O
from tests import tx_size_type_cases as T
from tests.test_oracle_tx_size_type import CASES, PAD, _pieces, run_case

pytestmark = pytest.mark.gpu


def device(src, rec, rect, w, h, bd, dm, red, lam, ds, sc, cdfs, it):
    c = G.ctx()
    dsrc, drec = c.plane_from_host(src, PAD), c.plane_from_host(rec, PAD)
    d_best = G.dev_empty(16 * max(1, len(it)))
    d_cands = G.dev_empty(24 * 21 * max(1, len(it)))
    d_sc = G.to_dev(sc) if sc is not None else None
    d_cdfs = G.to_dev(cdfs)
    c.intra_tx_size_type_dev(drec, dsrc, rect, w, h, bd, dm, red, lam, ds, d_sc, 0 if sc is None else sc.shape[1],
                             d_cdfs, len(cdfs), G.to_dev(it), len(it), d_best, d_cands)
    c.synchronize()
    return (G.from_dev(d_best, TX_BEST_DTYPE)[:len(it)],
            G.from_dev(d_cands, TX_CAND_DTYPE)[:21 * len(it)].reshape(len(it), 21), c, drec, dsrc, d_cdfs)


def assert_same(got, want):
    gb, gc = got
    wb, wc = want
    np.testing.assert_array_equal(gb["tx_size"], wb["tx_size"])
    np.testing.assert_array_equal(gb["tx_type"], wb["tx_type"])
    np.testing.assert_array_equal(gb["rd"].view(np.uint64), wb["rd"].view(np.uint64))
    for f in ("state", "rate", "dist"):
        np.testing.assert_array_equal(gc[f], wc[f], err_msg=f)
    np.testing.assert_array_equal(gc["rd"].view(np.uint64), wc["rd"].view(np.uint64))


@pytest.mark.parametrize("case", range(len(CASES)))
def test_device_equals_oracle(case):
    w, h, bd, dm, red, rect, scale = CASES[case]
    src, rec, rect, it, cdfs, sc, lam, ds, best, cands = run_case(w, h, bd, dm, red, rect, scale, seed=40 + case)
    gb, gc, *_ = device(src, rec, rect, w, h, bd, dm, red, lam, ds, sc, cdfs, it)
    assert_same((gb, gc), (best, cands))


@pytest.mark.parametrize("dm", [2, 0])
def test_1080p_batch_past_the_grid(dm):
    """Every 16x16 block of a 1080p frame with three modes: more candidates than the launch grid."""
    w, h = 1920, 1080
    src, rec = T.make_case(w, h, 8, 7)
    it = T.grid_items(w, h, 16, 16, [0, 1, 12])
    cdfs = K.default_cdfs()
    lam = 0.0013 * 140 * 140
    best, cands = T.oracle(src, rec, PAD, (0, 0, w, h), w, h, 8, dm, 0, lam, 16384, None, cdfs, it)
    assert_same(device(src, rec, (0, 0, w, h), w, h, 8, dm, 0, lam, 16384, None, cdfs, it)[:2], (best, cands))


def test_invalid_items_next_to_valid_and_inputs_unchanged():
    src, rec = T.make_case(64, 64, 10, 3)
    rng = np.random.default_rng(3)
    it = T.items(rng, 64, 64, 10)
    cdfs = K.default_cdfs()
    it[0]["bsize"] = 14
    it[2]["mode"] = 13
    it[4]["x"] = 6
    it[6]["y"] = 64
    it[8]["snapshot"] = 9
    want = T.oracle(src, rec, PAD, (0, 0, 64, 64), 64, 64, 10, 1, 0, 300.0, 16384, None, cdfs, it)
    gb, gc, c, drec, dsrc, d_cdfs = device(src, rec, (0, 0, 64, 64), 64, 64, 10, 1, 0, 300.0, 16384, None, cdfs, it)
    assert_same((gb, gc), want)
    np.testing.assert_array_equal(G.from_dev(d_cdfs, np.uint8)[:cdfs.nbytes], cdfs.view(np.uint8))
    assert (gb["tx_size"][[0, 2, 4, 6, 8]] == 0xFF).all() and (gb["tx_size"][[1, 3, 5, 7, 9]] != 0xFF).all()
    for plane, img in ((drec, rec), (dsrc, src)):
        out = np.zeros_like(img)
        c.check(c.L.b200_plane_download(c.h, __import__("ctypes").byref(plane), out.ctypes.data, out.strides[0]))
        np.testing.assert_array_equal(out, img)


def test_host_rejections_leave_outputs_untouched():
    c = G.ctx()
    src, rec = T.make_case(64, 64, 8, 5)
    dsrc, drec = c.plane_from_host(src, PAD), c.plane_from_host(rec, PAD)
    small = c.plane_from_host(src, 32)
    it = T.items(np.random.default_rng(5), 64, 64, 4)
    it["snapshot"] = 0
    d_it, d_cdfs = G.to_dev(it), G.to_dev(K.default_cdfs())
    d_best = torch.full((64,), 0x5A, dtype=torch.uint8, device="cuda")
    good = dict(rec=drec, src=dsrc, rect=(0, 0, 64, 64), width=64, height=64, bit_depth=8, dist_mode=2,
                reduced_tx_set=0, lam=100.0, dist_scale=16384, d_scale4x4=None, scale_stride=0, d_cdfs=d_cdfs,
                ncdfs=1, d_items=d_it, n=4, d_best=d_best)
    bad = [dict(bit_depth=10), dict(rect=(0, 0, 65, 64)), dict(rec=small), dict(src=small), dict(dist_mode=3),
           dict(reduced_tx_set=2), dict(lam=-1.0), dict(lam=float("inf")), dict(d_cdfs=None), dict(ncdfs=0),
           dict(d_items=None), dict(d_best=None), dict(width=65), dict(d_scale4x4=d_best, scale_stride=8)]
    other = c.plane_from_host(src[:48], PAD)
    bad += [dict(rec=other), dict(width=40), dict(n=1 << 30)]  # sizes differ; region past 4 * w_in_b = 40
    n0 = c.launches
    args = [good[k] for k in ("rec", "src")]
    assert c.L.b200_intra_tx_size_type_dev(None, C.byref(args[0]), C.byref(args[1]), 0, 0, 64, 64, 64, 64, 8, 2, 0,
                                           100.0, 16384, None, 0, d_cdfs.data_ptr(), 1, d_it.data_ptr(), 4,
                                           d_best.data_ptr(), None) == ERR_ARG  # NULL ctx
    for b in bad:
        with pytest.raises(B200Error):
            c.intra_tx_size_type_dev(**{**good, **b})
    c.synchronize()
    assert c.launches == n0
    assert (d_best.cpu().numpy() == 0x5A).all()


def test_flat_frame_ties_keep_the_larger_size():
    """lambda 0 on a flat frame: every rd away from the top / left edges is 0 and the first size wins."""
    w = h = 64
    flat = np.full((h, w), 97, np.uint8)
    it = np.concatenate([T.grid_items(w, h, 16, 16, [0, 1, 2, 9]), T.grid_items(w, h, 32, 32, [0, 12])])
    cdfs = K.default_cdfs()
    for dm in (0, 1, 2):
        want = T.oracle(flat, flat, PAD, (0, 0, w, h), w, h, 8, dm, 0, 0.0, 16384, None, cdfs, it)
        got = device(flat, flat, (0, 0, w, h), w, h, 8, dm, 0, 0.0, 16384, None, cdfs, it)[:2]
        assert_same(got, want)
        inner = (it["x"] > 0) & (it["y"] > 0)
        assert (got[0]["rd"][inner] == 0.0).all()
        assert (got[0]["tx_size"][inner] == np.array([T.MAX_TX[b] for b in it["bsize"][inner]])).all()


def test_full_size_candidates_equal_the_three_call_chain():
    """tx_size == bsize: the level-0 records equal intra prediction (the oracle's pinned pieces) ->
    b200_encode_tx_blocks_dev -> b200_coeff_rate_dev -> b200_compute_rd_cost_dev, tx-domain distortion at
    default scales, the same chain test_tx_type_decision_end_to_end runs with an inter prediction."""
    import torch
    c = G.ctx()
    w, h, bd = 192, 128, 8
    src, rec = T.make_case(w, h, bd, 21)
    rng = np.random.default_rng(21)
    blocks = G.grid_blocks(w, h, 16, 16)
    n = len(blocks)
    it = T.grid_items(w, h, 16, 16, [0])
    it["mode"] = rng.integers(0, 13, n)
    it["ief"] = rng.integers(-1, 2, n)
    it["above"] = rng.choice([0, 1, 3, 64 + 2, 128 + 5], (n, 16))
    it["left"] = rng.choice([0, 2, 5, 64 + 1, 128 + 7], (n, 16))
    cdfs = K.default_cdfs()[:1]
    lam = 0.0013 * 140 * 140
    # the predictions, one per block, from rec's edges through the oracle's pinned pieces
    L = _pieces()
    orec = O.Plane(w, h, PAD, rec.dtype)
    orec.fill_from(rec)
    pred = rec.copy()
    for b in range(n):
        x, y, m = int(it[b]["x"]), int(it[b]["y"]), int(it[b]["mode"])
        edge = np.zeros(O.EDGE_LEN, rec.dtype)
        il, ia = C.c_int(), C.c_int()
        L.orc_get_intra_edges(edge.ctypes.data, orec.origin_ptr(), orec.stride, 1, w, h, 0, 0, w, h, 0, 0, x >> 2,
                              y >> 2, 0, 0, 6, x, y, 16, 16, bd, m, int(it[b]["ief"] >= 0), 0, C.byref(il),
                              C.byref(ia))
        variant = 0 if (x, y) == (0, 0) else 1 if y == 0 else 2 if x == 0 else 3
        pm = m if m != 12 else [0, 2, 1, 12][variant]
        pred[y:y + 16, x:x + 16] = O.predict_intra(pm, variant, edge, 16, 16, bd, O.MODE_ANGLE.get(O.MODES[pm], 0),
                                                   int(it[b]["ief"]) if 1 <= m <= 8 else -1, left_len=il.value,
                                                   above_len=ia.value, plane_w=w, plane_h=h, dst_x=x, dst_y=y)
    dsrc, dpred = c.plane_from_host(src, PAD), c.plane_from_host(pred, PAD)
    gb, gc, *_ = device(src, rec, (0, 0, w, h), w, h, bd, 0, 0, lam, 16384, None, cdfs, it)
    d_blocks = G.to_dev(blocks)
    for k, ty in enumerate(T.type_list(2, 0, 0)):
        d_q = torch.zeros(n * 256, dtype=torch.int16, device="cuda")
        d_eob = torch.zeros(n, dtype=torch.int16, device="cuda")
        d_dist = torch.zeros(n, dtype=torch.int64, device="cuda")
        c.encode_tx_blocks_dev(dsrc, dpred, None, d_blocks, n, None, 2, ty, bd, 120, 140, 1, 0, None, d_q, None,
                               d_eob, d_dist)
        eob = d_eob.cpu().numpy().view(np.uint16)
        items = np.array([K.item(b, int(eob[b]), 2, ty, 0, 6, int(it[b]["mode"])) for b in range(n)])
        chains = np.zeros(n, COEFF_CHAIN_DTYPE)
        chains["init_rng"], chains["item_begin"], chains["item_count"] = 32768, np.arange(n), 1
        chains["above"][:, 0], chains["left"][:, 0] = it["above"], it["left"]
        d_rate = torch.zeros(n, dtype=torch.int32, device="cuda")
        c.coeff_rate_dev(G.to_dev(cdfs), 1, G.to_dev(chains), n, G.to_dev(items), n, d_q, n * 256, 0, d_rate)
        d_cost = torch.zeros(n, dtype=torch.float64, device="cuda")
        c.compute_rd_cost_dev(lam, d_rate, d_dist, n, d_cost)
        c.synchronize()
        col = gc[:, T.TX_TYPES.index(ty)]
        np.testing.assert_array_equal(col["state"], 0)
        np.testing.assert_array_equal(col["rate"], d_rate.cpu().numpy().view(np.uint32))
        np.testing.assert_array_equal(col["dist"], d_dist.cpu().numpy().view(np.uint64))
        np.testing.assert_array_equal(col["rd"].view(np.uint64), d_cost.cpu().numpy().view(np.uint64))
