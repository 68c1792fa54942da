"""b200_coeff_rate_dev against oracle/coeff_rate.c, bit for bit: the oracle cases (every tx size and type set,
planes 0 / 1 / 2, chains of up to 16 blocks, clipped windows, random CDFs, init_rng spread) at i16 and i32, 1080p
tx-type-decision batches past the launch's grid, invalid chains beside valid ones, every host-side rejection,
unchanged inputs, and rdo_tx_type_decision as three device calls."""
import numpy as np
import pytest
import torch

from rav1e_b200 import backend as B
from tests import coeff_rate_cases as K
from tests import gpu_util as G
from tests import oracle_lib as O

pytestmark = pytest.mark.gpu


def run(c, cdfs, chains, items, q, cul=True):
    ins = [G.to_dev(a) for a in (cdfs, chains, items, q)]
    before = [t.clone() for t in ins]
    d_rate = torch.full((max(1, len(chains)),), -1, dtype=torch.int32, device="cuda")
    d_cul = torch.full((max(1, len(items)),), 0xEE, dtype=torch.uint8, device="cuda") if cul else None
    c.coeff_rate_dev(ins[0], len(cdfs), ins[1], len(chains), ins[2], len(items), ins[3], len(q),
                     int(q.dtype == np.int32), d_rate, d_cul)
    c.synchronize()
    for a, b in zip(ins, before):
        assert torch.equal(a, b), "an input changed"
    rate = d_rate.cpu().numpy().view(np.uint32)[:len(chains)]
    return rate, (d_cul.cpu().numpy()[:len(items)] if cul else None)


@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_oracle_cases_bit_exact(is32):
    c = G.ctx()
    cdfs, chains, items, q = K.oracle_cases(seed=21 + is32, is32=is32)
    want, want_cul = K.oracle_rate(cdfs, chains, items, q)
    got, got_cul = run(c, cdfs, chains, items, q)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(got_cul, want_cul)
    assert (want != 0xFFFFFFFF).all()


def test_levels_read_the_whole_coded_block():
    """Nonzero coefficients past eob change the levels the contexts read (txb_init_levels takes the whole block)."""
    rng = np.random.default_rng(4)
    b = K.Batch(np.concatenate([K.default_cdfs(), K.random_cdfs(rng, 1)]), 0)
    for t in range(19):
        for tt in (0, 10, 11):
            eob = int(rng.choice(K.eob_choices(rng, t)[1:3]))
            blk = K.make_block(rng, t, tt, eob, 0, tail=True)
            b.add_chain([K.item(b.add_block(blk), eob, t, tt, plane=1, bsize=K.bsize_of(64, 64) if t < 4 else None)],
                        snapshot=int(rng.integers(0, 5)))
    cdfs, chains, items, q = b.arrays()
    want, want_cul = K.oracle_rate(cdfs, chains, items, q)
    got, got_cul = run(G.ctx(), cdfs, chains, items, q)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(got_cul, want_cul)


@pytest.mark.parametrize("bd", [8, 10])
def test_1080p_tx_type_batch_past_the_grid(bd):
    c = G.ctx()
    T = K.tx_decision_batch(c, 1920, 1080, bd, seed=bd)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert len(T["chains"]) > sms * 16 * 4  # more chains than the launch has warps (16 CTAs of 4 per SM)
    q = T["q"]
    want, want_cul = K.oracle_rate(T["cdfs"], T["chains"], T["items"], q)
    got, got_cul = run(c, T["cdfs"], T["chains"], T["items"], q)
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(got_cul, want_cul)
    assert (T["eob"] > 0).mean() > 0.5


def test_invalid_chains_next_to_valid_ones():
    rng = np.random.default_rng(8)
    b = K.Batch(K.default_cdfs(), 0)
    good = K.make_block(rng, 1, 0, 10, 0)
    gi = b.add_block(good)
    zt = good.copy()
    zt[K.scan_order(1, 0)[9]] = 0
    zi = b.add_block(zt)
    mn = good.copy()
    mn[3] = -32768
    mi = b.add_block(mn)
    ok = K.item(gi, 10, 1, 0)
    bad = [K.item(gi, 10, 19, 0), K.item(gi, 10, 1, 16), K.item(gi, 65, 1, 0), K.item(zi, 10, 1, 0),
           K.item(gi, 10, 1, 0, plane=3), K.item(gi, 10, 1, 0, x4=15), K.item(gi, 10, 1, 0, y4=14, clip_h4=3),
           K.item(gi, 10, 1, 0, clip_h4=0), K.item(gi, 10, 1, 4), K.item(gi, 10, 1, 0, mode=13),
           K.item(gi, 10, 1, 0, mode=34), K.item(mi, 10, 1, 0), K.item(1000, 10, 1, 0),
           K.item(gi, 10, 1, 0, bsize=22)]
    for it in bad:
        b.add_chain([ok])
        b.add_chain([ok, it, ok])
    b.add_chain([ok], snapshot=4)
    b.add_chain([ok], init_rng=32767)
    b.add_chain([ok], init_rng=65536)
    cdfs, chains, items, q = b.arrays()
    bogus = chains[-1].copy()
    bogus["item_begin"], bogus["item_count"] = len(items) - 1, 2
    chains = np.concatenate([chains, bogus[None]])
    want, want_cul = K.oracle_rate(cdfs, chains, items, q)
    got, got_cul = run(G.ctx(), cdfs, chains, items, q)
    np.testing.assert_array_equal(got, want)
    assert (got[0:2 * len(bad):2] != 0xFFFFFFFF).all() and (got[1:2 * len(bad):2] == 0xFFFFFFFF).all()
    assert (got[2 * len(bad):] == 0xFFFFFFFF).all()
    # items of invalid chains keep what d_cul_level held
    valid_items = np.zeros(len(items), bool)
    for ch, r in zip(chains, got):
        if r != 0xFFFFFFFF:
            valid_items[int(ch["item_begin"]):int(ch["item_begin"]) + int(ch["item_count"])] = True
    assert (got_cul[~valid_items] == 0xEE).all()
    np.testing.assert_array_equal(got_cul[valid_items], want_cul[valid_items])


def test_host_rejections_launch_nothing():
    c = G.ctx()
    rng = np.random.default_rng(2)
    b = K.Batch(K.default_cdfs(), 0)
    b.add_chain([K.item(b.add_block(K.make_block(rng, 0, 0, 5, 0)), 5, 0, 0)])
    cdfs, chains, items, q = b.arrays()
    dc, dch, dit, dq = (G.to_dev(a) for a in (cdfs, chains, items, q))
    d_rate = torch.full((4,), 7, dtype=torch.int32, device="cuda")
    d_cul = torch.full((4,), 9, dtype=torch.uint8, device="cuda")
    L = c.L
    cases = [
        (None, dc, 4, dch, 1, dit, 1, dq, len(q), 0, d_rate, d_cul),       # NULL ctx
        (c.h, None, 4, dch, 1, dit, 1, dq, len(q), 0, d_rate, d_cul),      # NULL cdfs
        (c.h, dc, 4, None, 1, dit, 1, dq, len(q), 0, d_rate, d_cul),       # NULL chains
        (c.h, dc, 4, dch, 1, dit, 1, dq, len(q), 0, None, d_cul),          # NULL rate
        (c.h, dc, 4, dch, 1, None, 1, dq, len(q), 0, d_rate, d_cul),       # NULL items
        (c.h, dc, 4, dch, 1, dit, 1, None, len(q), 0, d_rate, d_cul),      # NULL coefficients
        (c.h, dc, 0, dch, 1, dit, 1, dq, len(q), 0, d_rate, d_cul),        # no snapshot
        (c.h, dc, 4, dch, 1, dit, 1, dq, len(q), 2, d_rate, d_cul),        # coeff_is_i32 2
        (c.h, dc, 4, dch, 1 << 31, dit, 1, dq, len(q), 0, d_rate, d_cul),  # nchains 2^31
        (c.h, dc, 4, dch, 1, dit, 1 << 31, dq, len(q), 0, d_rate, d_cul),  # nitems 2^31
    ]
    p = B._dev_ptr
    for args in cases:
        c.synchronize()
        n0 = c.launches
        st = L.b200_coeff_rate_dev(*[p(a) if isinstance(a, torch.Tensor) else a for a in args])
        assert st == B.ERR_ARG, args
        c.synchronize()
        assert c.launches == n0
        assert (d_rate.cpu().numpy() == 7).all() and (d_cul.cpu().numpy() == 9).all()
    # zero chains: nothing to do, nothing launched
    n0 = c.launches
    assert L.b200_coeff_rate_dev(c.h, None, 0, None, 0, None, 0, None, 0, 0, None, None) == 0
    assert c.launches == n0


def test_tx_type_decision_end_to_end():
    """rdo_tx_type_decision without its early exit, at unit distortion scale: encode_tx_blocks x types ->
    coeff_rate -> compute_rd_cost with one group per block; d_best is the oracle's first minimum."""
    c = G.ctx()
    T = K.tx_decision_batch(c, 640, 368, 8, seed=31)
    n, types = T["n"], T["types"]
    nt = len(types)
    d_cdfs, d_chains, d_items = (G.to_dev(a) for a in (T["cdfs"], T["chains"], T["items"]))
    d_rate = torch.zeros(n * nt, dtype=torch.int32, device="cuda")
    c.coeff_rate_dev(d_cdfs, len(T["cdfs"]), d_chains, n * nt, d_items, len(T["items"]), T["d_q"],
                     T["d_q"].numel(), 0, d_rate)
    dist = np.stack([T["dist"][tt] for tt in types], axis=1).reshape(-1).astype(np.uint64)  # block-major
    d_dist = G.to_dev(dist)
    offs = (np.arange(n + 1) * nt).astype(np.uint32)
    d_best = torch.zeros(n, dtype=torch.int32, device="cuda")
    lam = 0.0013 * 140 * 140
    c.compute_rd_cost_dev(lam, d_rate, d_dist, n * nt, None, G.to_dev(offs), n, d_best)
    c.synchronize()
    rate, _ = K.oracle_rate(T["cdfs"], T["chains"], T["items"], T["q"])
    np.testing.assert_array_equal(d_rate.cpu().numpy().view(np.uint32), rate)
    L = O.lib()
    L.orc_compute_rd_cost.restype = __import__("ctypes").c_double
    L.orc_compute_rd_cost.argtypes = [__import__("ctypes").c_double, __import__("ctypes").c_uint32,
                                      __import__("ctypes").c_uint64]
    cost = np.array([L.orc_compute_rd_cost(lam, int(r), int(d)) for r, d in zip(rate, dist)]).reshape(n, nt)
    want = np.argmin(cost, axis=1)  # first minimum, as the strict `<` of the RDO loop
    got = d_best.cpu().numpy().view(np.uint32)
    np.testing.assert_array_equal(got, want)
    assert len(set(want.tolist())) > 1  # the decision is not constant
