"""The oracle's subpel_diamond_search (orc_subpel_diamond_search_blocks) at every AV1 block size, 4x4 to
64x64, against an independent restatement of me.rs:1311-1383 in Python: the four diamond points
(row+1, col+1, row-1, col-1 scaled by the radius) are scored with the oracle's get_subpel_mv_rd
(O.subpel_candidates), the first strict minimum is taken, the centre moves while that point is strictly
cheaper, and the radius halves from 1/2 pel down to 1/4 pel (1/8 pel with allow_hp).  This pins the
oracle at the sizes the device's diamond search is compared against."""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O

SIZES = O.TX_SIZES
EMPTY = np.uint64(2**64 - 1)


def frame(kind, W, H, bd, seed):
    """'smooth': low-passed noise, cur = ref shifted by half a pixel to the right (true mv col +4);
    'noise': independent noise in both frames."""
    rng = np.random.default_rng(seed)
    maxv = (1 << bd) - 1
    dtype = np.uint8 if bd == 8 else np.uint16
    if kind == "noise":
        ref = rng.integers(0, maxv + 1, (H, W))
        cur = rng.integers(0, maxv + 1, (H, W))
    else:
        base = rng.integers(0, 256, (H + 8, W + 8)).astype(np.float64)
        k = np.ones(5) / 5
        base = np.apply_along_axis(lambda r: np.convolve(r, k, "same"), 1, base)
        base = np.apply_along_axis(lambda r: np.convolve(r, k, "same"), 0, base) * (maxv / 255.0)
        ref = np.rint(base[4:4 + H, 4:4 + W])
        cur = np.rint((base[4:4 + H, 4:4 + W] + base[4:4 + H, 5:5 + W]) / 2)
    planes = []
    for img in (cur, ref):
        p = O.Plane(W, H, 96, dtype=dtype)
        p.fill_from(np.clip(img, 0, maxv).astype(dtype))
        planes.append(p)
    return planes


def blocks_for(W, H, w, h, cap=96):
    """A w x h grid over the frame (its edges included), thinned to at most `cap` blocks."""
    xs, ys = np.arange(0, W - w + 1, w), np.arange(0, H - h + 1, h)
    b = np.zeros(len(xs) * len(ys), O.BLOCK_DTYPE)
    b["x"], b["y"] = np.tile(xs, len(ys)), np.repeat(ys, len(xs))
    step = max(1, len(b) // cap)
    return np.ascontiguousarray(b[::step])


def oracle_search(ocur, oref, blocks, start, w, h, use_satd, lam, pmv, allow_hp, bd):
    L = O.lib()
    L.orc_subpel_diamond_search_blocks.restype = None
    L.orc_subpel_diamond_search_blocks.argtypes = [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t] + [C.c_int] * 3 + \
        [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p] + [C.c_int] * 3 + [C.c_void_p, C.c_int]
    res = start.copy()
    L.orc_subpel_diamond_search_blocks(ocur.origin_ptr(), ocur.stride, oref.origin_ptr(), oref.stride, ocur.bpp,
                                       2 * ((ocur.width + 7) >> 3), 2 * ((ocur.height + 7) >> 3), O.ptr(blocks),
                                       len(blocks), w, h, int(use_satd), lam, O.ptr(pmv), int(allow_hp), 0, bd,
                                       O.ptr(res), 0)
    return res


def wrap16(v):
    return ((np.asarray(v, np.int64) + 32768) % 65536 - 32768).astype(np.int16)


def python_search(ocur, oref, blocks, start, w, h, use_satd, lam, pmv, allow_hp, bd):
    """me.rs:1311-1383, every block's loop advanced in lockstep; one oracle call scores the four diamond
    points of all blocks still searching."""
    res = start.copy()
    nb = len(blocks)
    radius = np.full(nb, 2)
    end = 0 if allow_hp else 1
    active = np.ones(nb, bool)
    pattern = ((1, 0), (0, 1), (-1, 0), (0, -1))          # DIAMOND_R1_PATTERN_SUBPEL, {row, col}
    while active.any():
        idx = np.nonzero(active)[0]
        cands = np.zeros(4 * len(idx), O.CAND_DTYPE)
        cands["block"] = np.repeat(idx, 4)
        for k, (dr, dc) in enumerate(pattern):
            cands["mv_row"][k::4] = wrap16(res["mv_row"][idx].astype(np.int64) + (dr << radius[idx]))
            cands["mv_col"][k::4] = wrap16(res["mv_col"][idx].astype(np.int64) + (dc << radius[idx]))
        sad, cost = O.subpel_candidates(ocur, oref, blocks, cands, w, h, use_satd, lam, pmv, allow_hp, 0, bd)
        for j, b in enumerate(idx):
            best = None
            best_cost = EMPTY
            for k in range(4):
                if cost[4 * j + k] < best_cost:              # strict: the first minimum wins
                    best, best_cost = 4 * j + k, cost[4 * j + k]
            if res["cost"][b] <= best_cost:
                if radius[b] == end:
                    active[b] = False
                else:
                    radius[b] -= 1
            else:
                res[b]["cost"], res[b]["sad"] = best_cost, sad[best]
                res[b]["mv_row"], res[b]["mv_col"] = cands["mv_row"][best], cands["mv_col"][best]
    return res


@pytest.mark.parametrize("bd", [8, 10])
@pytest.mark.parametrize("w,h", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_oracle_diamond_search_equals_the_move_to_best_loop(w, h, bd):
    W, H = 192, 160
    moved = 0
    for kind, lam in (("smooth", 300), ("noise", 0)):
        ocur, oref = frame(kind, W, H, bd, seed=w * 7 + h + bd)
        blocks = blocks_for(W, H, w, h)
        nb = len(blocks)
        rng = np.random.default_rng(w + 3 * h)
        pmv = (rng.integers(-8, 9, (nb, 4)) * 2).astype(np.int16)
        for use_satd in (False, True):
            # full-pel starting points around the true vector, scored like the full-pel stage's winner
            st = np.zeros(nb, O.CAND_DTYPE)
            st["block"] = np.arange(nb)
            st["mv_row"] = rng.integers(-1, 2, nb) * 8
            st["mv_col"] = rng.integers(-1, 2, nb) * 8
            for allow_hp in (False, True):
                sad, cost = O.fullpel_candidates(ocur, oref, blocks, st, w, h, use_satd, lam, pmv, allow_hp)
                start = np.zeros(nb, O.ME_RESULT_DTYPE)
                start["cost"], start["sad"], start["mv_row"], start["mv_col"] = cost, sad, st["mv_row"], st["mv_col"]
                want = python_search(ocur, oref, blocks, start, w, h, use_satd, lam, pmv, allow_hp, bd)
                got = oracle_search(ocur, oref, blocks, start, w, h, use_satd, lam, pmv, allow_hp, bd)
                for f in ("cost", "sad", "mv_row", "mv_col"):
                    np.testing.assert_array_equal(got[f], want[f], err_msg=f"{kind} satd={use_satd} hp={allow_hp}: {f}")
                assert (got["cost"] <= start["cost"]).all()
                moved += int(((got["mv_row"] != start["mv_row"]) | (got["mv_col"] != start["mv_col"])).sum())
    assert moved > 0
