"""GPU parity tests for the SAD/SATD/ME path: CUDA (through the C ABI) == oracle, bit exact.

Mirrors the reference's own test layout: the KATs of src/dist.rs:416-533 run against the
per-call `rav1e_*_cuda` symbols (the table entries a Rust wrapper would call), and the
asm==rust random-input equivalence tests of src/asm/x86/dist/mod.rs:738-969 become
CUDA==oracle tests over candidate batches.
"""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_oracle_dist import SAD_KAT, SATD_KAT, setup_planes

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
def test_percall_kats(dtype):
    """dist.rs:418-441 / :477-500 through rav1e_sad{W}x{H}_cuda etc. (byte strides)."""
    L = B.lib()
    (inp, xo, yo, st), (rec, xr, yr, sr) = setup_planes(dtype)
    isz = inp.itemsize
    hbd = dtype == np.uint16
    for kind, table in (("sad", SAD_KAT), ("satd", SATD_KAT)):
        for w, h, want in table:
            if kind == "sad":
                name = f"rav1e_sad_{w}x{h}_hbd_cuda" if hbd else f"rav1e_sad{w}x{h}_cuda"
            else:
                name = f"rav1e_satd_{w}x{h}_hbd_cuda" if hbd else f"rav1e_satd_{w}x{h}_cuda"
            f = getattr(L, name)
            args = [O.ptr(inp, (yo + 40) * st + xo + 32), st * isz,
                    O.ptr(rec, (yr + 40) * sr + xr + 32), sr * isz]
            if kind == "satd" and hbd:
                args.append(255)
            assert f(*args) == want, (name, want)


def test_percall_noncanonical_size():
    """Frame-edge crops (e.g. 16x12) go to the generic path (asm/x86/dist/mod.rs:299)."""
    L = B.lib()
    rng = np.random.default_rng(5)
    a = rng.integers(0, 256, (40, 48), dtype=np.uint8)
    b = rng.integers(0, 256, (40, 64), dtype=np.uint8)
    for w, h in ((16, 12), (12, 8), (20, 20), (8, 12)):
        want = O.lib().orc_get_sad_u8(O.ptr(a), 48, O.ptr(b), 64, w, h)
        assert L.b200_get_sad(O.ptr(a), 48, O.ptr(b), 64, w, h, 1) == want
        want = O.lib().orc_get_satd_u8(O.ptr(a), 48, O.ptr(b), 64, w, h)
        assert L.b200_get_satd(O.ptr(a), 48, O.ptr(b), 64, w, h, 1) == want


CAND_ROWS = [
    # (w, h, dtype, bit_depth, use_satd, per_block, max_px, kernel the dispatcher picks)
    # dense lists: the grouped kernel stages one window per group of blocks
    (16, 16, np.uint8, 8, False, 40, 40, "me_cand_group_u8<16, 16, false>"),  # some candidates fall outside get_mv_range
    (16, 16, np.uint8, 8, True, 12, 24, "me_cand_group_u8<16, 16, true>"),
    (8, 8, np.uint8, 8, False, 30, 16, "me_cand_group_u8<8, 8, false>"),
    (32, 32, np.uint8, 8, False, 20, 40, "me_cand_group_u8<32, 32, false>"),
    (4, 4, np.uint8, 8, False, 9, 12, "me_cand_warp_u8<4, 4, false>"),   # 9 x 16 px: a sparse list
    (4, 8, np.uint8, 8, True, 9, 12, "me_cand_group_u8<4, 8, true>"),
    (64, 64, np.uint8, 8, False, 6, 70, "me_cand_group_u8<64, 64, false>"),
    (128, 128, np.uint8, 8, True, 2, 8, "me_cand_generic<unsigned char>+me_best_from_cost"),  # beyond 64x64
    (16, 8, np.uint8, 8, False, 17, 30, "me_cand_group_u8<16, 8, false>"),
    # non-canonical crop: partial chunks -> SAD, generic kernel
    (16, 12, np.uint8, 8, True, 5, 10, "me_cand_generic<unsigned char>+me_best_from_cost"),
    (16, 16, np.uint16, 10, False, 25, 24, "me_chunk_lists<unsigned short, 16, 16, false>"),
    (16, 16, np.uint16, 10, True, 10, 24, "me_chunk_lists<unsigned short, 16, 16, true>"),
    (32, 16, np.uint16, 12, True, 7, 24, "me_chunk_lists<unsigned short, 32, 16, true>"),
    (64, 64, np.uint16, 12, False, 3, 24, "me_cand_generic<unsigned short>+me_best_from_cost"),
    # sparse lists (few candidates per block), no window staging: SATD goes to the staged 8x8-chunk
    # kernel, SAD and the SATD sizes it does not serve (4xN, more than 32 chunks) to the warp-per-block kernel
    (16, 16, np.uint8, 8, True, 4, 40, "me_chunk_lists<unsigned char, 16, 16, true>"),
    (16, 16, np.uint8, 8, False, 3, 40, "me_cand_warp_u8<16, 16, false>"),
    (8, 8, np.uint8, 8, True, 2, 30, "me_chunk_lists<unsigned char, 8, 8, true>"),
    (32, 32, np.uint8, 8, True, 3, 64, "me_chunk_lists<unsigned char, 32, 32, true>"),
    (4, 8, np.uint8, 8, True, 3, 20, "me_cand_warp_u8<4, 8, true>"),
    (64, 64, np.uint8, 8, True, 2, 72, "me_cand_warp_u8<64, 64, true>"),
    # the same list with a +-60 px reach sits just above the sparse threshold: grouped kernel
    (64, 64, np.uint8, 8, True, 2, 60, "me_cand_group_u8<64, 64, true>"),
    (32, 16, np.uint8, 8, False, 1, 50, "me_cand_warp_u8<32, 16, false>"),
    # sparse SATD lists through the staged 8x8-chunk kernel: every block size it serves, more
    # candidates per block than one batch holds, blocks without candidates (jitter)
    (16, 16, np.uint8, 8, True, 8, 64, "me_chunk_lists<unsigned char, 16, 16, true>"),
    (16, 16, np.uint8, 8, True, 13, 90, "me_chunk_lists<unsigned char, 16, 16, true>"),
    (8, 16, np.uint8, 8, True, 5, 40, "me_chunk_lists<unsigned char, 8, 16, true>"),
    (16, 8, np.uint8, 8, True, 9, 60, "me_chunk_lists<unsigned char, 16, 8, true>"),
    (16, 32, np.uint8, 8, True, 5, 60, "me_chunk_lists<unsigned char, 16, 32, true>"),
    (32, 16, np.uint8, 8, True, 6, 60, "me_chunk_lists<unsigned char, 32, 16, true>"),
    (32, 64, np.uint8, 8, True, 2, 60, "me_chunk_lists<unsigned char, 32, 64, true>"),
    (64, 32, np.uint8, 8, True, 3, 70, "me_chunk_lists<unsigned char, 64, 32, true>"),
    (8, 8, np.uint8, 8, True, 1, 70, "me_chunk_lists<unsigned char, 8, 8, true>"),
    # high bit depth through the staged chunk kernel (16-bit lanes), dense and sparse, SAD and SATD
    (8, 8, np.uint16, 10, False, 40, 30, "me_chunk_lists<unsigned short, 8, 8, false>"),
    (8, 8, np.uint16, 12, True, 3, 30, "me_chunk_lists<unsigned short, 8, 8, true>"),
    (16, 16, np.uint16, 12, False, 70, 50, "me_chunk_lists<unsigned short, 16, 16, false>"),
    (16, 32, np.uint16, 10, True, 6, 40, "me_chunk_lists<unsigned short, 16, 32, true>"),
    (32, 32, np.uint16, 10, False, 9, 60, "me_chunk_lists<unsigned short, 32, 32, false>"),
    (32, 32, np.uint16, 12, True, 2, 60, "me_chunk_lists<unsigned short, 32, 32, true>"),
    (8, 16, np.uint16, 10, False, 12, 30, "me_chunk_lists<unsigned short, 8, 16, false>"),
]


CAND_CASES = [r[:7] for r in CAND_ROWS]
CAND_KERNEL = {r[:7]: r[7] for r in CAND_ROWS}
assert len(CAND_KERNEL) == len(CAND_ROWS)


@pytest.mark.parametrize("w,h,dtype,bd,use_satd,per_block,max_px", CAND_CASES)
def test_candidate_list_matches_oracle(w, h, dtype, bd, use_satd, per_block, max_px):
    kernel = CAND_KERNEL[(w, h, dtype, bd, use_satd, per_block, max_px)]
    W, H, PAD = 352, 288, 160
    cur, ref = G.make_planes(W, H, PAD, dtype, seed=w * 131 + h, bit_depth=bd)
    ocur, dcur = G.both_planes(cur, PAD)
    oref, dref = G.both_planes(ref, PAD)
    blocks = G.grid_blocks(W, H, w, h)
    cands, offs = G.random_cands(len(blocks), per_block, max_px, seed=7, fullpel=(w != 8))
    rng = np.random.default_rng(11)
    pmv = (rng.integers(-64, 65, (len(blocks), 4)) * 4).astype(np.int16)
    lam = 1234
    want_sad, want_cost = O.fullpel_candidates(ocur, oref, blocks, cands, w, h, use_satd, lam, pmv)

    c = G.ctx()
    p = B.me_params(w, h, W, H, lam, use_satd=use_satd, bit_depth=bd, window_hint_px=max_px)
    d_blocks, d_cands, d_offs, d_pmv = map(G.to_dev, (blocks, cands, offs, pmv))
    d_sad, d_cost = G.dev_empty(4 * len(cands)), G.dev_empty(8 * len(cands))
    d_best = G.dev_empty(16 * len(blocks))
    launched = G.profiled_kernels(lambda: c.me_candidates_dev(dcur, dref, d_blocks, len(blocks), d_cands, len(cands),
                                                              p, d_offs, d_pmv, d_sad, d_cost, d_best))
    assert launched == kernel.split("+"), launched
    got_sad = G.from_dev(d_sad, np.uint32)[:len(cands)]
    got_cost = G.from_dev(d_cost, np.uint64)[:len(cands)]
    np.testing.assert_array_equal(got_sad, want_sad)
    np.testing.assert_array_equal(got_cost, want_cost)
    best = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:len(blocks)]
    for b in range(len(blocks)):
        lo, hi = int(offs[b]), int(offs[b + 1])
        if lo == hi or want_cost[lo:hi].min() == np.uint64(2**64 - 1):
            assert best[b]["cost"] == np.uint64(2**64 - 1) and best[b]["sad"] == 0xFFFFFFFF
            continue
        k = lo + int(np.argmin(want_cost[lo:hi]))      # numpy argmin = first minimum
        assert best[b]["cost"] == want_cost[k]
        assert best[b]["sad"] == want_sad[k]
        assert (best[b]["mv_row"], best[b]["mv_col"]) == (cands[k]["mv_row"], cands[k]["mv_col"])
    # ungrouped call (no CSR): per-candidate outputs only, same values
    d_sad2 = G.dev_empty(4 * len(cands))
    perm = np.random.default_rng(1).permutation(len(cands))
    c.me_candidates_dev(dcur, dref, d_blocks, len(blocks), G.to_dev(cands[perm]), len(cands), p,
                        None, d_pmv, d_sad2, None, None)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_sad2, np.uint32)[:len(cands)], want_sad[perm])
    for pl in (dcur, dref):
        c.plane_free(pl)


@pytest.mark.parametrize("hint", [4, 12, 1000])
def test_candidate_list_wrong_window_hint(hint):
    """window_hint_px is advisory: a hint smaller (or absurdly larger) than the candidates'
    reach must not change any result (the grouped kernel re-derives the window)."""
    W, H, PAD, w, h = 352, 288, 160, 16, 16
    cur, ref = G.make_planes(W, H, PAD, np.uint8, seed=91)
    ocur, dcur = G.both_planes(cur, PAD)
    oref, dref = G.both_planes(ref, PAD)
    blocks = G.grid_blocks(W, H, w, h)
    cands, offs = G.random_cands(len(blocks), 64, 40, seed=17)
    want_sad, want_cost = O.fullpel_candidates(ocur, oref, blocks, cands, w, h, False, 321)
    c = G.ctx()
    p = B.me_params(w, h, W, H, 321, window_hint_px=hint)
    d_blocks, d_cands, d_offs = map(G.to_dev, (blocks, cands, offs))
    d_sad, d_cost = G.dev_empty(4 * len(cands)), G.dev_empty(8 * len(cands))
    d_best = G.dev_empty(16 * len(blocks))
    c.me_candidates_dev(dcur, dref, d_blocks, len(blocks), d_cands, len(cands), p, d_offs, None,
                        d_sad, d_cost, d_best)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_sad, np.uint32)[:len(cands)], want_sad)
    np.testing.assert_array_equal(G.from_dev(d_cost, np.uint64)[:len(cands)], want_cost)
    best = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:len(blocks)]
    for b in range(len(blocks)):
        lo, hi = int(offs[b]), int(offs[b + 1])
        assert best[b]["cost"] == want_cost[lo:hi].min()
    for pl in (dcur, dref):
        c.plane_free(pl)


MULTI_ROWS = [
    # (w, h, dtype, bit_depth, use_satd, per_block, max_px, kernels launched)
    (16, 16, np.uint8, 8, False, 64, 40, "me_cand_group_u8<16, 16, false>"),   # grouped cooperative kernel
    (16, 16, np.uint8, 8, False, 4, 30, "me_cand_warp_u8<16, 16, false>"),     # warp-per-block kernel (sparse lists)
    (16, 16, np.uint8, 8, True, 4, 30, "me_chunk_lists<unsigned char, 16, 16, true>"),  # sparse SATD lists
    # 6 SATD candidates per block over +-30 px are just dense enough for the grouped kernel
    (16, 16, np.uint8, 8, True, 6, 30, "me_cand_group_u8<16, 16, true>"),
    (8, 8, np.uint8, 8, False, 40, 16, "me_cand_group_u8<8, 8, false>"),       # grouped, thread per candidate
    (32, 32, np.uint8, 8, True, 20, 30, "me_cand_group_u8<32, 32, true>"),
    # non-canonical size: generic kernel, pair by pair, then the segmented argmin
    (16, 12, np.uint8, 8, False, 9, 12, "me_cand_generic<unsigned char>+me_best_from_cost"),
    (16, 16, np.uint16, 10, False, 12, 20, "me_chunk_lists<unsigned short, 16, 16, false>"),  # high bit depth
    (64, 64, np.uint16, 12, True, 3, 20, "me_cand_generic<unsigned short>+me_best_from_cost"),  # HBD beyond 32x32
]


MULTI_CASES = [r[:7] for r in MULTI_ROWS]
MULTI_KERNEL = {r[:7]: r[7] for r in MULTI_ROWS}
assert len(MULTI_KERNEL) == len(MULTI_ROWS)


@pytest.mark.parametrize("w,h,dtype,bd,use_satd,per_block,max_px", MULTI_CASES)
def test_multi_pair_launch_matches_oracle(w, h, dtype, bd, use_satd, per_block, max_px):
    """b200_me_candidates_multi_dev: several (cur, ref) pairs with different images, different
    block subsets (one of them empty) in one call == the oracle pair by pair."""
    kernel = MULTI_KERNEL[(w, h, dtype, bd, use_satd, per_block, max_px)]
    W, H, PAD = 320, 192, 96
    grid = G.grid_blocks(W, H, w, h)
    subsets = [grid, grid[5:37], grid[:0], grid[::3].copy(), grid[-9:]]
    lam = 555
    curs, refs, blocks, cands, offs, want_sad, want_cost, want_best = [], [], [], [], [np.zeros(1, np.uint32)], [], [], []
    nb_tot = nc_tot = 0
    block_end, cand_end = [], []
    rng = np.random.default_rng(77)
    pmvs = []
    for k, sub in enumerate(subsets):
        cur, ref = G.make_planes(W, H, PAD, dtype, seed=300 + k, bit_depth=bd, shift=(k - 2, 2 - k))
        ocur, dcur = G.both_planes(cur, PAD)
        oref, dref = G.both_planes(ref, PAD)
        curs.append(dcur)
        refs.append(dref)
        sub = np.ascontiguousarray(sub)
        c, o = G.random_cands(len(sub), per_block, max_px, seed=40 + k, fullpel=True)
        pmv = (rng.integers(-32, 33, (len(sub), 4)) * 4).astype(np.int16)
        if len(sub):
            ws, wc = O.fullpel_candidates(ocur, oref, sub, c, w, h, use_satd, lam, pmv)
        else:
            ws, wc = np.zeros(0, np.uint32), np.zeros(0, np.uint64)
        want_sad.append(ws)
        want_cost.append(wc)
        cg = c.copy()
        cg["block"] += nb_tot
        blocks.append(sub)
        cands.append(cg)
        offs.append((o[1:].astype(np.uint64) + nc_tot).astype(np.uint32))
        pmvs.append(pmv)
        nb_tot += len(sub)
        nc_tot += len(c)
        block_end.append(nb_tot)
        cand_end.append(nc_tot)
    blocks, cands, offs = np.concatenate(blocks), np.concatenate(cands), np.concatenate(offs)
    pmv = np.concatenate(pmvs)
    want_sad, want_cost = np.concatenate(want_sad), np.concatenate(want_cost)
    c = G.ctx()
    p = B.me_params(w, h, W, H, lam, use_satd=use_satd, bit_depth=bd, window_hint_px=max_px)
    d_blocks, d_cands, d_offs, d_pmv = map(G.to_dev, (blocks, cands, offs, pmv))
    d_sad, d_cost, d_best = G.dev_empty(4 * nc_tot), G.dev_empty(8 * nc_tot), G.dev_empty(16 * nb_tot)
    pairs = B.PlanePairs(curs, refs, block_end, cand_end)
    launched = G.profiled_kernels(lambda: c.me_candidates_multi_dev(pairs, d_blocks, nb_tot, d_cands, nc_tot, p,
                                                                    d_offs, d_pmv, d_sad, d_cost, d_best))
    assert set(launched) == set(kernel.split("+")), launched
    np.testing.assert_array_equal(G.from_dev(d_sad, np.uint32)[:nc_tot], want_sad)
    np.testing.assert_array_equal(G.from_dev(d_cost, np.uint64)[:nc_tot], want_cost)
    best = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:nb_tot]
    for b in range(nb_tot):
        lo, hi = int(offs[b]), int(offs[b + 1])
        if lo == hi or want_cost[lo:hi].min() == np.uint64(2**64 - 1):
            assert best[b]["cost"] == np.uint64(2**64 - 1)
            continue
        k = lo + int(np.argmin(want_cost[lo:hi]))
        assert best[b]["cost"] == want_cost[k] and best[b]["sad"] == want_sad[k]
        assert (best[b]["mv_row"], best[b]["mv_col"]) == (cands[k]["mv_row"], cands[k]["mv_col"])
    for pl in curs + refs:
        c.plane_free(pl)


def test_multi_pair_more_pairs_than_one_launch_holds():
    """40 pairs > the 32-entry table of one launch: split internally, same results as 40 calls."""
    W, H, PAD, w, h = 128, 96, 64, 16, 16
    grid = G.grid_blocks(W, H, w, h)
    nb = len(grid)
    c = G.ctx()
    NP = 40
    imgs = [G.make_planes(W, H, PAD, np.uint8, seed=500 + k) for k in range(3)]
    dplanes = [(c.plane_from_host(cu, PAD), c.plane_from_host(re, PAD)) for cu, re in imgs]
    curs = [dplanes[k % 3][0] for k in range(NP)]
    refs = [dplanes[(k + 1) % 3][1] for k in range(NP)]
    cl, ol = [], [np.zeros(1, np.uint32)]
    for k in range(NP):
        cc, oo = G.random_cands(nb, 48, 24, seed=600 + k, jitter=False)
        cc["block"] += k * nb
        cl.append(cc)
        ol.append(oo[1:] + np.uint32(k * nb * 48))
    cands, offs = np.concatenate(cl), np.concatenate(ol)
    blocks = np.tile(grid, NP)
    p = B.me_params(w, h, W, H, 900, window_hint_px=24)
    d_blocks, d_cands, d_offs = map(G.to_dev, (blocks, cands, offs))
    d_best = G.dev_empty(16 * nb * NP)
    pairs = B.PlanePairs(curs, refs, [(k + 1) * nb for k in range(NP)],
                         [(k + 1) * nb * 48 for k in range(NP)])
    c.me_candidates_multi_dev(pairs, d_blocks, nb * NP, d_cands, len(cands), p, d_offs, None, None,
                              None, d_best)
    c.synchronize()
    got = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:nb * NP].copy()
    d_one = G.dev_empty(16 * nb)
    d_grid = G.to_dev(grid)
    for k in range(NP):
        ck = cl[k].copy()
        ck["block"] -= k * nb
        c.me_candidates_dev(curs[k], refs[k], d_grid, nb, G.to_dev(ck), len(ck), p,
                            G.to_dev(np.arange(nb + 1, dtype=np.uint32) * 48), None, None, None, d_one)
        c.synchronize()
        one = G.from_dev(d_one, B.ME_RESULT_DTYPE)[:nb]
        np.testing.assert_array_equal(got[k * nb:(k + 1) * nb], one)
    for a, b in dplanes:
        c.plane_free(a)
        c.plane_free(b)


@pytest.mark.parametrize("hint,dx", [(32, 4), (32, 0), (48, 12), (24, 8)])
def test_candidate_list_unaligned_block_columns(hint, dx):
    """Blocks that do not start on 16-pixel columns (4x4-unit offsets inside a superblock) and
    hints that are / are not multiples of 16: the TMA-staged window, its 16-byte column rule and
    the hand-staged fall back must all give the oracle's numbers."""
    W, H, PAD, w, h = 352, 288, 160, 16, 16
    cur, ref = G.make_planes(W, H, PAD, np.uint8, seed=123)
    ocur, dcur = G.both_planes(cur, PAD)
    oref, dref = G.both_planes(ref, PAD)
    blocks = G.grid_blocks(W - 16, H - 16, w, h)
    blocks["x"] += dx
    blocks["y"] += 4
    cands, offs = G.random_cands(len(blocks), 64, hint, seed=29)
    want_sad, want_cost = O.fullpel_candidates(ocur, oref, blocks, cands, w, h, False, 700)
    c = G.ctx()
    p = B.me_params(w, h, W, H, 700, window_hint_px=hint)
    d_blocks, d_cands, d_offs = map(G.to_dev, (blocks, cands, offs))
    d_sad, d_cost = G.dev_empty(4 * len(cands)), G.dev_empty(8 * len(cands))
    c.me_candidates_dev(dcur, dref, d_blocks, len(blocks), d_cands, len(cands), p, d_offs, None,
                        d_sad, d_cost, None)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_sad, np.uint32)[:len(cands)], want_sad)
    np.testing.assert_array_equal(G.from_dev(d_cost, np.uint64)[:len(cands)], want_cost)
    for pl in (dcur, dref):
        c.plane_free(pl)


def test_mv_list_resident_equals_candidate_records():
    """b200_me_mvs_resident (4-byte MotionVector lists, block from the CSR) == the same lists
    as b200_cand records through b200_me_candidates_resident."""
    W, H, PAD, w, h = 320, 192, 96, 16, 16
    cur, ref = G.make_planes(W, H, PAD, np.uint8, seed=21)
    c = G.ctx()
    dcur, dref = c.plane_from_host(cur, PAD), c.plane_from_host(ref, PAD)
    blocks = G.grid_blocks(W, H, w, h)
    cands, offs = G.random_cands(len(blocks), 40, 30, seed=4)
    mvs = np.stack([cands["mv_row"], cands["mv_col"]], axis=1).astype(np.int16).copy()
    p = B.me_params(w, h, W, H, 450, window_hint_px=30)
    n, nb = len(cands), len(blocks)
    out_a = (np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(nb, B.ME_RESULT_DTYPE))
    out_b = (np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(nb, B.ME_RESULT_DTYPE))
    c.me_candidates_resident(dcur, dref, blocks, cands, p, offs, out_a)
    c.me_mvs_resident(dcur, dref, blocks, mvs, p, offs, out_b)
    c.synchronize()
    for x, y in zip(out_a, out_b):
        np.testing.assert_array_equal(x, y)
    assert (out_a[2]["cost"] != np.uint64(2**64 - 1)).all()
    for pl in (dcur, dref):
        c.plane_free(pl)


def test_candidate_list_host_buffers():
    """The `_batch` form (host pointers, copies inside) gives the same numbers."""
    W, H, PAD, w, h = 320, 192, 96, 16, 16
    cur, ref = G.make_planes(W, H, PAD, np.uint8, seed=3)
    ocur = O.Plane(W, H, PAD)
    ocur.fill_from(cur)
    oref = O.Plane(W, H, PAD)
    oref.fill_from(ref)
    blocks = G.grid_blocks(W, H, w, h)
    cands, offs = G.random_cands(len(blocks), 33, 20, seed=9)
    want_sad, want_cost = O.fullpel_candidates(ocur, oref, blocks, cands, w, h, False, 77)
    c = G.ctx()
    p = B.me_params(w, h, W, H, 77, window_hint_px=20)
    sad, cost, best = c.me_candidates_batch(B.host_plane(ocur.data, PAD), B.host_plane(oref.data, PAD),
                                            blocks, cands, p, offs, None, True, True, True)
    np.testing.assert_array_equal(sad, want_sad)
    np.testing.assert_array_equal(cost, want_cost)
    for b in range(len(blocks)):
        lo, hi = int(offs[b]), int(offs[b + 1])
        if lo < hi:
            assert best[b]["cost"] == want_cost[lo:hi].min()


FS_CASES = [
    # (w, h, dtype, bd, range_x, range_y, step, lambda)
    (16, 16, np.uint8, 8, 48, 16, 4, 0),
    (16, 16, np.uint8, 8, 48, 16, 4, 3200),
    (16, 16, np.uint8, 8, 24, 8, 2, 500),      # hres level: step 2
    (16, 16, np.uint8, 8, 12, 4, 1, 500),      # qres level: step 1
    (8, 8, np.uint8, 8, 20, 12, 4, 100),
    (32, 32, np.uint8, 8, 32, 16, 4, 100),
    (64, 64, np.uint8, 8, 16, 8, 4, 100),
    (16, 8, np.uint8, 8, 16, 8, 4, 100),       # generic path
    (16, 16, np.uint16, 10, 16, 8, 4, 900),
    (16, 16, np.uint8, 8, 192, 64, 4, 6400),   # full-resolution lookahead window
]


@pytest.mark.parametrize("w,h,dtype,bd,rx,ry,step,lam", FS_CASES)
def test_full_search_matches_oracle(w, h, dtype, bd, rx, ry, step, lam):
    big = rx > 100
    W, H, PAD = (256, 128, 96) if big else (192, 128, 96)
    cur, ref = G.make_planes(W, H, PAD, dtype, seed=rx + ry + step, bit_depth=bd, shift=(5, -3))
    ocur, dcur = G.both_planes(cur, PAD)
    oref, dref = G.both_planes(ref, PAD)
    blocks = G.grid_blocks(W, H, w, h)
    if big:
        blocks = np.ascontiguousarray(blocks[::5])
    want = O.full_search_blocks(ocur, oref, blocks, w, h, rx, ry, step, lam)
    c = G.ctx()
    p = B.me_params(w, h, W, H, lam, bit_depth=bd)
    d_best = G.dev_empty(16 * len(blocks))
    c.me_full_search_dev(dcur, dref, G.to_dev(blocks), len(blocks), p, rx, ry, step, d_best)
    c.synchronize()
    got = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:len(blocks)]
    for f in ("cost", "sad", "mv_row", "mv_col"):
        np.testing.assert_array_equal(got[f], want[f], err_msg=f)
    for pl in (dcur, dref):
        c.plane_free(pl)


def test_full_search_flat_ties_pick_first_position():
    """me.rs:1501: strict `<` => first scanned position wins on a flat reference."""
    W, H, PAD = 128, 96, 96
    cur = np.full((H, W), 7, np.uint8)
    ref = np.full((H, W), 9, np.uint8)
    ocur, dcur = G.both_planes(cur, PAD)
    oref, dref = G.both_planes(ref, PAD)
    blocks = G.grid_blocks(W, H, 16, 16)
    want = O.full_search_blocks(ocur, oref, blocks, 16, 16, 48, 16, 4, 0)
    c = G.ctx()
    d_best = G.dev_empty(16 * len(blocks))
    c.me_full_search_dev(dcur, dref, G.to_dev(blocks), len(blocks), B.me_params(16, 16, W, H, 0),
                         48, 16, 4, d_best)
    c.synchronize()
    got = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:len(blocks)]
    for f in ("cost", "sad", "mv_row", "mv_col"):
        np.testing.assert_array_equal(got[f], want[f], err_msg=f)
    assert (got["sad"] == 512).all()


def test_1080p_properties():
    """Full BASELINE size: size-independent properties instead of a full oracle pass.
    (1) cur == ref shifted by a known vector => full search finds it with sad 0;
    (2) zero-mv candidates on identical planes => sad 0;
    (3) a 1/64 sample of candidates equals the oracle."""
    W, H, PAD = 1920, 1080, 96
    rng = np.random.default_rng(0)
    base = rng.integers(0, 256, (H + 2 * PAD, W + 2 * PAD), dtype=np.uint8)
    dx, dy = 8, -4
    ref_full = base
    cur_full = np.roll(base, (-dy, -dx), axis=(0, 1))   # cur(x,y) = ref(x+dx, y+dy)
    c = G.ctx()
    L = c.L
    # device planes carrying their own (non-replicated) border: upload the padded arrays whole
    def dev_plane(full):
        p = B.Plane()
        c.check(L.b200_plane_alloc(c.h, W + 2 * PAD, H + 2 * PAD, 0, 1, C.byref(p)))
        c.check(L.b200_plane_upload(c.h, C.byref(p), full.ctypes.data, full.strides[0]))
        q = B.Plane()
        q.data = p.data + PAD * p.stride + PAD
        q.stride, q.width, q.height, q.pad, q.bpp, q.alloc = p.stride, W, H, PAD, 1, None
        return p, q
    pc, dcur = dev_plane(cur_full)
    pr, dref = dev_plane(ref_full)
    blocks = G.grid_blocks(W, H, 16, 16)
    # keep blocks whose displaced window stays clear of the wrap-around of np.roll
    inner = (blocks["x"] >= 64) & (blocks["x"] < W - 80) & (blocks["y"] >= 64) & (blocks["y"] < H - 80)
    d_best = G.dev_empty(16 * len(blocks))
    p = B.me_params(16, 16, W, H, 0)
    c.me_full_search_dev(dcur, dref, G.to_dev(blocks), len(blocks), p, 48, 16, 4, d_best)
    c.synchronize()
    got = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:len(blocks)]
    assert (got["sad"][inner] == 0).all()
    assert (got["mv_col"][inner] == 8 * dx).all() and (got["mv_row"][inner] == 8 * dy).all()
    # (2)
    cands = np.zeros(len(blocks), B.CAND_DTYPE)
    cands["block"] = np.arange(len(blocks))
    d_sad = G.dev_empty(4 * len(cands))
    c.me_candidates_dev(dref, dref, G.to_dev(blocks), len(blocks), G.to_dev(cands), len(cands), p,
                        None, None, d_sad, None, None)
    c.synchronize()
    assert (G.from_dev(d_sad, np.uint32)[:len(cands)] == 0).all()
    # (3)
    cands, offs = G.random_cands(len(blocks), 64, 48, seed=2, jitter=False)
    d_sad = G.dev_empty(4 * len(cands))
    p = B.me_params(16, 16, W, H, 0, window_hint_px=48)
    c.me_candidates_dev(dcur, dref, G.to_dev(blocks), len(blocks), G.to_dev(cands), len(cands), p,
                        G.to_dev(offs), None, d_sad, None, None)
    c.synchronize()
    got_sad = G.from_dev(d_sad, np.uint32)[:len(cands)]
    ocur = O.Plane(W, H, PAD)
    ocur.data[:] = cur_full
    oref = O.Plane(W, H, PAD)
    oref.data[:] = ref_full
    sel = np.arange(0, len(cands), 64)
    want, _ = O.fullpel_candidates(ocur, oref, blocks, cands[sel], 16, 16, False, 0, want_cost=False)
    np.testing.assert_array_equal(got_sad[sel], want)
    # checksum-of-everything against a full (threaded) oracle pass: 522k candidates, ~1 s of CPU
    want_all, _ = O.fullpel_candidates(ocur, oref, blocks, cands, 16, 16, False, 0, want_cost=False)
    np.testing.assert_array_equal(got_sad, want_all)
    c.check(L.b200_plane_free(c.h, C.byref(pc)))
    c.check(L.b200_plane_free(c.h, C.byref(pr)))


def test_resident_planes_async_pipeline():
    """b200_me_candidates_resident + b200_fwd_txfm_residual_resident in asynchronous mode over two
    contexts: results are valid after b200_ctx_synchronize and equal the oracle."""
    import torch
    W, H, PAD, w, h = 320, 192, 96, 16, 16
    cur, ref = G.make_planes(W, H, PAD, np.uint8, seed=8)
    ocur = O.Plane(W, H, PAD)
    ocur.fill_from(cur)
    oref = O.Plane(W, H, PAD)
    oref.fill_from(ref)
    blocks = G.grid_blocks(W, H, w, h)
    pin = lambda a: torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).pin_memory().numpy().view(a.dtype)
    ctxs = [B.Context(0), B.Context(0)]
    outs = []
    for k, c in enumerate(ctxs):
        c.set_async(True)
        dcur, dref = c.plane_from_host(cur, PAD), c.plane_from_host(ref, PAD)
        cands, offs = G.random_cands(len(blocks), 20, 24, seed=30 + k)
        hb, hc, ho = pin(blocks), pin(cands), pin(offs)
        best = pin(np.zeros(len(blocks), B.ME_RESULT_DTYPE))
        coef = pin(np.zeros((len(blocks), 256), np.int16)).reshape(len(blocks), 256)
        p = B.me_params(w, h, W, H, 99, window_hint_px=24)
        c.me_candidates_resident(dcur, dref, hb, hc, p, ho, (None, None, best))
        c.fwd_txfm_residual_resident(dcur, dref, hb, best, coef, 2, 0, 8)
        outs.append((c, cands, offs, best, coef, dcur, dref))
    for c, cands, offs, best, coef, dcur, dref in outs:
        c.synchronize()
        _, want_cost = O.fullpel_candidates(ocur, oref, blocks, cands, w, h, False, 99)
        resid = np.zeros((len(blocks), 16, 16), np.int16)
        for b in range(len(blocks)):
            lo, hi = int(offs[b]), int(offs[b + 1])
            assert best[b]["cost"] == want_cost[lo:hi].min()
            dx, dy = int(np.trunc(best[b]["mv_col"] / 8)), int(np.trunc(best[b]["mv_row"] / 8))
            x, y = int(blocks[b]["x"]) + PAD, int(blocks[b]["y"]) + PAD
            resid[b] = (ocur.data[y:y + 16, x:x + 16].astype(np.int32) -
                        oref.data[y + dy:y + dy + 16, x + dx:x + dx + 16].astype(np.int32))
        np.testing.assert_array_equal(coef, O.forward_transform_batch(resid, 2, 0, 8))
        c.plane_free(dcur)
        c.plane_free(dref)
        c.close()


@pytest.mark.parametrize("dtype,bd,w,h,use_satd", [(np.uint8, 8, 16, 16, True), (np.uint8, 8, 8, 8, False),
                                                  (np.uint16, 10, 16, 16, True), (np.uint16, 10, 32, 16, True),
                                                  (np.uint16, 12, 8, 16, False), (np.uint8, 8, 64, 64, True)])
def test_subpel_candidates_match_oracle(dtype, bd, w, h, use_satd):
    """get_subpel_mv_rd (me.rs:1411-1442): 8-tap MC + SATD/SAD + cost + first-min winner, for the
    diamond pattern of subpel_diamond_search around random full-pel vectors (BASELINE config 4)."""
    W, H, PAD = 320, 192, 160
    cur, ref = G.make_planes(W, H, PAD, dtype, seed=bd + w, bit_depth=bd)
    ocur, dcur = G.both_planes(cur, PAD)
    oref, dref = G.both_planes(ref, PAD)
    blocks = G.grid_blocks(W, H, w, h)
    nb = len(blocks)
    rng = np.random.default_rng(4)
    centre = rng.integers(-20, 21, (nb, 2)) * 8
    pattern = np.array([(0, 0)] + [(r * s, c * s) for s in (4, 2, 1) for r, c in ((1, 0), (0, 1), (-1, 0), (0, -1))])
    cands = np.zeros(nb * len(pattern), B.CAND_DTYPE)
    cands["block"] = np.repeat(np.arange(nb, dtype=np.uint32), len(pattern))
    mv = centre[:, None, :] + pattern[None, :, :]
    cands["mv_row"], cands["mv_col"] = mv[:, :, 0].reshape(-1), mv[:, :, 1].reshape(-1)
    offs = (np.arange(nb + 1) * len(pattern)).astype(np.uint32)
    pmv = (rng.integers(-64, 65, (nb, 4)) * 2).astype(np.int16)
    lam = 777
    want_sad, want_cost = O.subpel_candidates(ocur, oref, blocks, cands, w, h, use_satd, lam, pmv,
                                              allow_hp=True, filter_mode=0, bit_depth=bd)
    c = G.ctx()
    p = B.me_params(w, h, W, H, lam, allow_hp=True, use_satd=use_satd, bit_depth=bd)
    d_sad, d_cost = G.dev_empty(4 * len(cands)), G.dev_empty(8 * len(cands))
    d_best = G.dev_empty(16 * nb)
    c.me_subpel_candidates_dev(dcur, dref, G.to_dev(blocks), nb, G.to_dev(cands), len(cands), p, 0,
                               G.to_dev(offs), G.to_dev(pmv), d_sad, d_cost, d_best)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_sad, np.uint32)[:len(cands)], want_sad)
    np.testing.assert_array_equal(G.from_dev(d_cost, np.uint64)[:len(cands)], want_cost)
    best = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:nb]
    for b in range(nb):
        lo, hi = int(offs[b]), int(offs[b + 1])
        k = lo + int(np.argmin(want_cost[lo:hi]))
        assert best[b]["cost"] == want_cost[k] and best[b]["sad"] == want_sad[k]
        assert (best[b]["mv_row"], best[b]["mv_col"]) == (cands[k]["mv_row"], cands[k]["mv_col"])
    for pl in (dcur, dref):
        c.plane_free(pl)
