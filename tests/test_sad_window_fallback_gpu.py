"""The cooperative SAD path of me_cand_group_u8<16, 16, false> with a search-range hint: candidates
the hinted window does not cover take their SAD from the reference plane in their own lane, and the
first minimum is a 32-bit warp key when every cost fits (the 64-bit key otherwise).

The current frame is the reference displaced by more than the hint, so the best vector of every
block lies outside the window: a version that drops the per-candidate fallback, or reads the wrong
pixels for it, gets sads, costs and winners that differ from the oracle.  Lists cover one lane, one
warp and scattered candidates outside the window, costs on both sides of the 32-bit key bound, a
predictor table with p0 != p1, and equal costs in different warps and rounds of one block.
"""
import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O

pytestmark = pytest.mark.gpu

W, H, PAD, BW, BH = 352, 288, 160, 16, 16
HINT = 16
SHIFT = (30, -28)             # true motion (x, y) in pixels: beyond the hint
KERNEL = "me_cand_group_u8<16, 16, false>"


def _planes():
    cur, ref = G.make_planes(W, H, PAD, np.uint8, seed=23, shift=SHIFT)
    ocur, dcur = G.both_planes(cur, PAD)
    oref, dref = G.both_planes(ref, PAD)
    return ocur, dcur, oref, dref


def _in_window(nb, per_block, seed, jitter=False):
    return G.random_cands(nb, per_block, HINT, seed=seed, jitter=jitter)


def _set_true(c, idx):
    c["mv_col"][idx] = SHIFT[0] * 8
    c["mv_row"][idx] = SHIFT[1] * 8


def _run(cands, offs, blocks, lam, pmv=None):
    ocur, dcur, oref, dref = _planes()
    c = G.ctx()
    p = B.me_params(BW, BH, W, H, lam, window_hint_px=HINT)
    want_sad, want_cost = O.fullpel_candidates(ocur, oref, blocks, cands, BW, BH, False, lam, pmv=pmv)
    d_blocks, d_cands, d_offs = map(G.to_dev, (blocks, cands, offs))
    d_pmv = G.to_dev(pmv) if pmv is not None else None
    d_sad, d_cost = G.dev_empty(4 * len(cands)), G.dev_empty(8 * len(cands))
    d_best = G.dev_empty(16 * len(blocks))

    def call():
        c.me_candidates_dev(dcur, dref, d_blocks, len(blocks), d_cands, len(cands), p, d_offs, d_pmv,
                            d_sad, d_cost, d_best)
        c.synchronize()
    assert G.profiled_kernels(call) == [KERNEL]
    sad = G.from_dev(d_sad, np.uint32)[:len(cands)]
    cost = G.from_dev(d_cost, np.uint64)[:len(cands)]
    best = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:len(blocks)]
    for pl in (dcur, dref):
        c.plane_free(pl)
    np.testing.assert_array_equal(sad, want_sad)
    np.testing.assert_array_equal(cost, want_cost)
    for b in range(len(blocks)):
        lo, hi = int(offs[b]), int(offs[b + 1])
        k = lo + int(np.argmin(want_cost[lo:hi]))        # numpy: the first minimum
        assert (best[b]["cost"], best[b]["sad"]) == (want_cost[k], want_sad[k]), b
        assert (best[b]["mv_row"], best[b]["mv_col"]) == (cands[k]["mv_row"], cands[k]["mv_col"]), b
    return want_sad, want_cost


def _outside_sets(nb, per_block):
    """candidate indices moved to the true vector: one lane, one whole warp, scattered lanes"""
    return {
        "one_lane": [(nb // 2) * per_block + 17],                     # blocks well inside the frame
        "one_warp": list(range((nb // 2 + 1) * per_block + 32, (nb // 2 + 1) * per_block + 64)),
        "scattered": list(range(3, nb * per_block, 97)),
    }


@pytest.mark.parametrize("which", ["one_lane", "one_warp", "scattered"])
@pytest.mark.parametrize("lam", [6400, 1 << 22])     # 32-bit warp keys / beyond their bound: 64-bit keys
def test_out_of_window_candidates(which, lam):
    blocks = G.grid_blocks(W, H, BW, BH)
    per_block = 64
    cands, offs = _in_window(len(blocks), per_block, seed=31)
    idx = _outside_sets(len(blocks), per_block)[which]
    _set_true(cands, idx)
    sad, _ = _run(cands, offs, blocks, lam)
    assert (sad[idx[:1]] != 0xFFFFFFFF).all()             # in range: the fallback ran


def test_out_of_window_with_predictors():
    """p0 != p1 in some blocks of a group: both rates, and the fallback's cost uses them"""
    blocks = G.grid_blocks(W, H, BW, BH)
    cands, offs = _in_window(len(blocks), 48, seed=37, jitter=True)
    _set_true(cands, list(range(0, len(cands), 13)))
    rng = np.random.default_rng(5)
    pmv = (rng.integers(-40, 41, (len(blocks), 4)) * 8).astype(np.int16)
    pmv[::3, 2:] = pmv[::3, :2]                         # p0 == p1 in every third block
    _run(cands, offs, blocks, 777, pmv=pmv)


@pytest.mark.parametrize("lam", [6400, 1 << 22])
def test_ties_across_warps_and_rounds(lam):
    """equal minimum costs in different warps (and rounds) of one block: the lowest index wins"""
    blocks = G.grid_blocks(W, H, BW, BH)
    per_block = 300                                     # a block spans several warps and two rounds
    cands, offs = _in_window(len(blocks), per_block, seed=41)
    for b in range(len(blocks)):
        lo = b * per_block
        # the same (outside) vector in the second warp of the block, then in earlier-indexed slots of later warps
        _set_true(cands, [lo + 40, lo + 70, lo + 260, lo + 299])
        # an in-window duplicate pair straddling a warp boundary: equal costs, the first one is not the minimum
        cands[lo + 31] = cands[lo + 33]
    _, cost = _run(cands, offs, blocks, lam)
    lo = (len(blocks) // 2) * per_block                 # a block well inside the frame: the vector is in range
    assert cost[lo + 40] != 2**64 - 1 and cost[lo + 40] == cost[lo + 70] == cost[lo + 260]
