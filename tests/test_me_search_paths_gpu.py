"""The full-pel motion search on every kernel path, bit exact against the oracle: b200_me_search_dev /
b200_me_search_multi_dev (me_search.cu + the state machine of me_search_dev.cuh), b200_me_full_search_dev
(me_full_search.cu) and b200_lookahead_motion_dev (lookahead_me.cu).

The launch geometry mirrored here:
- me_search.cu      `min(ceil(n / 4), 64 * num_sms)` CTAs of 4 warps, one warp per block, grid-stride loop;
                    plane pairs cut into launches of kMaxPairs = 32, a chunk with no block skipped;
- me_search_dev.cuh a lane keeps its org words in registers iff the block has at most 8 * kOrgRegs = 128
                    words (w * bpp / 4 words per row), and rows of fewer than 8 words share a step;
- me_full_search.cu `me_full_search_u8<W, H, NP>` for bpp 1, ref stride % 4 == 0, 8/16/32/64 squares and at
                    most 200 KiB of staged window, grid min(n, 32 * num_sms); else `me_full_search_generic<T>`,
                    grid min(n, 16 * num_sms);
- lookahead_me.cu   grid_for: min(ceil(items / 4), 32 * num_sms) CTAs of 4 warps.
The sections:
1. every AV1 block size through the search at 8 and 10 bit (12 bit on a subset), both predictor-subset forms,
   each case on the org-cache side and row-segment rule the formula gives;
2. the search ladder's edges: umh_range values, thresholds 0 and UINT32_MAX, an empty median, no predictor at
   all or none in range (the diamond still starts from the zero vector), lambda 0 and UINT32_MAX, 12-bit 0 / 4095 at 128x128, predictors on
   and one eighth-pel past every get_mv_range limit at exactly min_pad;
3. a second grid-stride trip, and a multi-pair call of 100 pairs (four chunks, one of them 32 empty pairs);
4. caller-built plane views at byte offsets 0..3 and strides that are a multiple of 4 bytes but not of 16;
5. the exhaustive grid on every route, with the kernel each case reached, second grid trips and flat ties;
6. the lookahead at frame sizes that are not multiples of 8, odd tiles, 12 bit, range scale 16, extreme
   lambdas and a multi-pair call past the grid cap, with the launch count of each call;
7. read footprints: every byte outside the contracted pad replaced between two runs;
8. host rejections (no launch, outputs untouched), empty calls, unchanged inputs and sentinels past the outputs.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_lookahead_me_gpu import assert_grid_equal, device_motion, free, launches_formula, levels, params
from tests.test_me_cand_edges_gpu import oracle_plane, padded
from tests.test_me_search_gpu import predictor_subsets
from tests.test_oracle_lookahead_me import STATS_DTYPE, Params, case_inputs, grid_dims, images, oracle_motion, pyramid

pytestmark = pytest.mark.gpu

U8, U16 = np.uint8, np.uint16
EMPTY_COST = np.uint64(2**64 - 1)
EMPTY_SAD = np.uint32(0xFFFFFFFF)
K_ORG_REGS = 16            # me_search_dev.cuh kOrgRegs
SEARCH_WARPS_PER_SM = 64 * 4   # me_search.cu: 64 CTAs per SM of 4 warps
FS_U8_CTAS_PER_SM = 32     # me_full_search.cu launch_fs_u8
FS_GENERIC_CTAS_PER_SM = 16
LA_WARPS_PER_SM = 32 * 4   # lookahead_me.cu grid_for
SENTINEL = 0xA5


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def bits(dtype):
    return 8 if dtype == U8 else 10


def org_cache(w, h, bpp):
    """me_search.cu: (cached, narrow) - the lanes keep the org block in registers iff it has at most
    8 * kOrgRegs words; rows of fewer than 8 words share one step of a candidate's 8 lanes."""
    nw = w * bpp // 4
    return nw * h <= 8 * K_ORG_REGS, nw < 8


def stride4(cols, bpp=1):
    """An element stride >= cols whose byte pitch is a multiple of 4 but not of 16."""
    s = cols
    while (s * bpp) % 4 or (s * bpp) % 16 == 0:
        s += 1
    return s


def default_view(full, pad):
    return G.ViewPlane(full, pad, stride4(full.shape[1] + 40, full.itemsize), 0)


def sentinel_out(nbytes, extra=64):
    t = torch.full((nbytes + extra,), SENTINEL, dtype=torch.uint8, device="cuda")
    return t


def assert_sentinel(t, nbytes):
    tail = t[nbytes:].cpu().numpy()
    assert (tail == SENTINEL).all(), "bytes past the output were written"


def assert_best_equal(got, want, what=""):
    for f in ("cost", "sad", "mv_row", "mv_col"):
        np.testing.assert_array_equal(got[f], want[f], err_msg=f"{what} {f}")


class Snapshot:
    """Byte copies of device tensors, to check that a call left its inputs alone."""

    def __init__(self, *ts):
        self.ts = [t for t in ts if t is not None]
        self.copies = [t.clone() for t in self.ts]

    def check(self):
        torch.cuda.synchronize()
        for t, c in zip(self.ts, self.copies):
            assert torch.equal(t, c), "an input changed"


# ---------------------------------------------------------------- the search: one call, all checks
def run_search(cur_full, ref_full, pad, blocks, preds, offs, nsubsets, w, h, lam, pmv=None, thresh=None, umh=0,
               bd=8, views=None, allow_hp=False, want=None):
    """b200_me_search_dev on planes built by `views(full, pad)` (default: a 16-byte-misaligned-pitch view
    at offset 0) against the oracle; inputs unchanged, nothing written past the output."""
    width, height = cur_full.shape[1] - 2 * pad, cur_full.shape[0] - 2 * pad
    n = len(blocks)
    blocks, preds = np.ascontiguousarray(blocks), np.ascontiguousarray(preds)
    offs = np.ascontiguousarray(offs, np.uint32)
    if want is None:
        want = O.full_pixel_me_blocks(oracle_plane(cur_full, pad), oracle_plane(ref_full, pad), blocks, preds, offs,
                                      nsubsets, w, h, lam, pmv, thresh, umh, allow_hp)
    make = views or default_view
    vc, vr = make(cur_full, pad), make(ref_full, pad)
    c = G.ctx()
    p = B.me_params(w, h, width, height, lam, allow_hp=allow_hp, bit_depth=bd)
    d_blocks, d_offs = G.to_dev(blocks), G.to_dev(offs)
    d_preds = G.to_dev(preds) if len(preds) else None
    d_pmv = None if pmv is None else G.to_dev(np.ascontiguousarray(pmv, np.int16))
    d_thresh = None if thresh is None else G.to_dev(np.ascontiguousarray(thresh, np.uint32))
    snap = Snapshot(d_blocks, d_offs, d_preds, d_pmv, d_thresh, vc.buf, vr.buf)
    d_best = sentinel_out(16 * n)
    before = c.launches
    c.me_search_dev(vc.plane, vr.plane, d_blocks, n, d_preds, d_offs, nsubsets, p, d_best, d_pmv, d_thresh, umh)
    c.synchronize()
    assert c.launches - before == (1 if n else 0)
    got = G.from_dev(d_best[:16 * n], B.ME_RESULT_DTYPE)
    assert_best_equal(got, want)
    assert_sentinel(d_best, 16 * n)
    snap.check()
    return got


def search_planes(W, H, pad, dtype, seed, bd=None, smooth=True):
    cur, ref = G.make_planes(W, H, pad, dtype, seed=seed, bit_depth=bd or bits(dtype), smooth=smooth, shift=(5, -3))
    return padded(cur, pad), padded(ref, pad)


def spread_blocks(W, H, w, h, extra, seed):
    """The raster grid plus `extra` blocks at random 4-aligned positions (overlapping the grid)."""
    g = G.grid_blocks(W, H, w, h)
    rng = np.random.default_rng(seed)
    e = np.zeros(extra, B.BLOCK_DTYPE)
    e["x"] = rng.integers(0, (W - w) // 4 + 1, extra) * 4
    e["y"] = rng.integers(0, (H - h) // 4 + 1, extra) * 4
    return np.concatenate([g, e])


# ---------------------------------------------------------------- 1. every block size
SUBSET12 = [(4, 4), (8, 32), (16, 16), (16, 32), (32, 8), (64, 16), (128, 128)]
SIZE_CASES = ([(w, h, U8, 8) for w, h in B.BLOCK_SIZES] + [(w, h, U16, 10) for w, h in B.BLOCK_SIZES]
              + [(w, h, U16, 12) for w, h in SUBSET12])


def size_id(w, h, dt, bd):
    cached, narrow = org_cache(w, h, np.dtype(dt).itemsize)
    return f"{w}x{h}-bd{bd}-{'cached' if cached else 'uncached'}{'-narrow' if narrow else ''}"


def test_every_depth_reaches_both_sides_of_the_cache_boundary():
    for bd in (8, 10, 12):
        kinds = {org_cache(w, h, np.dtype(dt).itemsize) for w, h, dt, b in SIZE_CASES if b == bd}
        assert {k[0] for k in kinds} == {True, False}, bd
        assert {k[1] for k in kinds} == {True, False}, bd


@pytest.mark.parametrize("w,h,dt,bd", SIZE_CASES, ids=[size_id(*c) for c in SIZE_CASES])
def test_every_block_size(w, h, dt, bd):
    """Every BlockSize at 8 / 10 (and a subset at 12) bit, all_mvs and median | b | c with UMH; thresholds
    spread so that some blocks stop at a subset and some run the whole ladder."""
    bpp = np.dtype(dt).itemsize
    cached, narrow = org_cache(w, h, bpp)
    # the formula in me_search.cu, restated: the id names the side, and the side is what the formula gives
    assert (w * bpp // 4) * h <= 128 if cached else (w * bpp // 4) * h > 128
    assert narrow == (w * bpp < 32)
    W, H = 256, 256
    pad = max(160, G.min_pad(W, H, w, h))
    cur_full, ref_full = search_planes(W, H, pad, dt, seed=w * 13 + h + bd, bd=bd)
    blocks = spread_blocks(W, H, w, h, 24, seed=w + h)
    if len(blocks) > 1200:
        blocks = blocks[::3].copy()
    n = len(blocks)
    rng = np.random.default_rng(w * h + bd)
    pmv = (rng.integers(-40, 41, (n, 4)) * rng.choice([1, 4, 8], (n, 4))).astype(np.int16)
    lam = int(rng.integers(0, 3000)) << (bd - 8)
    for nsubsets in (1, 3):
        preds, offs = predictor_subsets(n, nsubsets, seed=w + 3 * h + nsubsets, max_px=20)
        thresh = None
        if nsubsets == 3:
            thresh = rng.integers(0, (w * h) << (bd - 8 + 3), n).astype(np.uint32)
        got = run_search(cur_full, ref_full, pad, blocks, preds, offs, nsubsets, w, h, lam, pmv, thresh,
                         24 if nsubsets == 3 else 0, bd)
        assert (got["cost"] != EMPTY_COST).mean() > 0.9
        if nsubsets == 3:     # both kinds of exit: below a threshold, and the whole ladder
            assert (got["sad"] < thresh).any() and (got["sad"] >= thresh).any()


# ---------------------------------------------------------------- 2. the ladder's edges
def ladder_case(seed, w=16, h=16, dtype=U8, W=192, H=128, pad=96, nsubsets=3, drop_median_every=5):
    cur_full, ref_full = search_planes(W, H, pad, dtype, seed=seed)
    blocks = G.grid_blocks(W, H, w, h)
    n = len(blocks)
    preds, offs = predictor_subsets(n, nsubsets, seed=seed + 1, max_px=24, drop_median_every=drop_median_every)
    pmv = (np.random.default_rng(seed).integers(-30, 31, (n, 4)) * 8).astype(np.int16)
    return cur_full, ref_full, pad, blocks, preds, offs, pmv


@pytest.mark.parametrize("umh", [0, 1, 2, 3, 5, 23, 64])
def test_umh_ranges(umh):
    """Cross lines of (umh + 1) / 2 and (umh / 2 + 1) / 2 points, umh / 4 hexagon scales; thresholds 0 so that
    every block runs the ladder to its end."""
    cur_full, ref_full, pad, blocks, preds, offs, pmv = ladder_case(100 + umh)
    thresh = np.zeros(len(blocks), np.uint32)
    run_search(cur_full, ref_full, pad, blocks, preds, offs, 3, 16, 16, 700, pmv, thresh, umh)


@pytest.mark.parametrize("t", [0, 2**32 - 1], ids=["zero", "max"])
def test_thresholds_at_their_limits(t):
    cur_full, ref_full, pad, blocks, preds, offs, pmv = ladder_case(7)
    thresh = np.full(len(blocks), t, np.uint32)
    got = run_search(cur_full, ref_full, pad, blocks, preds, offs, 3, 16, 16, 400, pmv, thresh, 24)
    if t:
        assert (got["sad"] < thresh).all()


def test_every_median_subset_empty():
    cur_full, ref_full, pad, blocks, preds, offs, pmv = ladder_case(8, drop_median_every=1)
    assert (offs[0:-1:3] == offs[1::3]).all()
    thresh = np.random.default_rng(8).integers(0, 4000, len(blocks)).astype(np.uint32)
    run_search(cur_full, ref_full, pad, blocks, preds, offs, 3, 16, 16, 400, pmv, thresh, 24)


@pytest.mark.parametrize("nsubsets", [1, 3])
def test_no_usable_predictor(nsubsets):
    """Every subset empty, or every predictor outside get_mv_range: get_best_predictor leaves
    MotionSearchResult::empty() (cost 2^64 - 1, sad 0xFFFFFFFF, mv 0) and fullpel_diamond_search starts from
    its zero vector, whose diamond neighbours are always in range.  So the search never returns the empty
    record: both lists give the same in-range winners (rejected predictors leave no trace)."""
    W, H, pad, w, h = 128, 96, 96, 16, 16
    cur_full, ref_full = search_planes(W, H, pad, U8, seed=9)
    blocks = G.grid_blocks(W, H, w, h)
    n = len(blocks)
    thresh = np.zeros(n, np.uint32) if nsubsets == 3 else None
    umh = 24 if nsubsets == 3 else 0
    none = run_search(cur_full, ref_full, pad, blocks, np.zeros(0, B.CAND_DTYPE), np.zeros(n * nsubsets + 1, np.uint32),
                      nsubsets, w, h, 500, None, thresh, umh)
    rows = []
    for b in blocks:
        x_min, x_max, y_min, y_max = G.mv_range(W, H, int(b["x"]), int(b["y"]), w, h)
        rows += [(x_max + 1, 0), (x_min - 1, 8), (0, y_max + 8), (16, y_min - 1), (x_max + 8, y_max + 8)]
    preds = np.zeros(len(rows), B.CAND_DTYPE)
    preds["mv_col"], preds["mv_row"] = [r[0] for r in rows], [r[1] for r in rows]
    counts = np.zeros((n, nsubsets), np.int64)
    counts[:] = (5,) if nsubsets == 1 else (1, 2, 2)
    offs = np.zeros(n * nsubsets + 1, np.uint32)
    offs[1:] = np.cumsum(counts.reshape(-1))
    out = run_search(cur_full, ref_full, pad, blocks, preds, offs, nsubsets, w, h, 500, None, thresh, umh)
    np.testing.assert_array_equal(out, none)
    assert (none["cost"] != EMPTY_COST).all() and (none["sad"] != EMPTY_SAD).all()


@pytest.mark.parametrize("allow_hp", [False, True])
@pytest.mark.parametrize("lam", [0, 2**32 - 1])
def test_lambda_at_its_limits(lam, allow_hp):
    cur_full, ref_full, pad, blocks, preds, offs, pmv = ladder_case(10 + allow_hp)
    pmv[::3] = (-32768, 32767, 32767, -32768)
    thresh = np.random.default_rng(3).integers(0, 6000, len(blocks)).astype(np.uint32)
    for nsubsets, ps in ((3, (preds, offs)), (1, predictor_subsets(len(blocks), 1, seed=4, max_px=20))):
        run_search(cur_full, ref_full, pad, blocks, ps[0], ps[1], nsubsets, 16, 16, lam, pmv,
                   thresh if nsubsets == 3 else None, 24 if nsubsets == 3 else 0, allow_hp=allow_hp)


@pytest.mark.parametrize("pattern", ["max_vs_zero", "random_extremes"])
def test_12bit_extremes_at_128x128(pattern):
    """cur at 4095 against ref at 0 (SAD 4095 * 16384 in the u32 sums), and random 0 / 4095 pixels."""
    W, H, w, h = 384, 256, 128, 128
    pad = G.min_pad(W, H, w, h)
    shape = (H + 2 * pad, W + 2 * pad)
    if pattern == "max_vs_zero":
        cur_full, ref_full = np.full(shape, 4095, U16), np.zeros(shape, U16)
    else:
        rng = np.random.default_rng(12)
        cur_full = (rng.integers(0, 2, shape) * 4095).astype(U16)
        ref_full = (rng.integers(0, 2, shape) * 4095).astype(U16)
    blocks = spread_blocks(W, H, w, h, 8, seed=5)
    n = len(blocks)
    for nsubsets in (1, 3):
        preds, offs = predictor_subsets(n, nsubsets, seed=20 + nsubsets, max_px=40)
        thresh = np.zeros(n, np.uint32) if nsubsets == 3 else None
        got = run_search(cur_full, ref_full, pad, blocks, preds, offs, nsubsets, w, h, 2**32 - 1, None, thresh,
                         24 if nsubsets == 3 else 0, bd=12)
        if pattern == "max_vs_zero":
            assert (got["sad"][got["cost"] != EMPTY_COST] == 4095 * w * h).all()


BORDER_W, BORDER_H = 348, 284     # w_in_b / h_in_b round up to 352 x 288


def edge_blocks(bw, bh):
    w8, h8 = 8 * ((BORDER_W + 7) >> 3), 8 * ((BORDER_H + 7) >> 3)
    xs = sorted(set(range(0, w8 - bw + 1, bw)) | {w8 - bw})
    ys = sorted(set(range(0, h8 - bh + 1, bh)) | {h8 - bh})
    pos = [(x, y) for y in ys for x in xs if x in (xs[0], xs[-1]) or y in (ys[0], ys[-1])]
    b = np.zeros(len(pos), B.BLOCK_DTYPE)
    b["x"], b["y"] = [q[0] for q in pos], [q[1] for q in pos]
    return b


def border_lists(blocks, w, h, nsubsets, seed):
    """Per block: border_cands' vectors on and past every limit (1/8 and 1 px), split over the subsets."""
    edge = G.border_cands(blocks, BORDER_W, BORDER_H, w, h)
    n = len(blocks)
    counts = np.bincount(edge["block"], minlength=n)
    if nsubsets == 1:
        offs = np.zeros(n + 1, np.uint32)
        offs[1:] = np.cumsum(counts)
        return edge, offs
    rng = np.random.default_rng(seed)
    cnt = np.zeros((n, 3), np.int64)
    for b in range(n):
        k = int(counts[b])
        cut = np.sort(rng.integers(0, k + 1, 2))
        cnt[b] = (min(cut[0], 1), cut[1] - min(cut[0], 1), k - cut[1])
    offs = np.zeros(3 * n + 1, np.uint32)
    offs[1:] = np.cumsum(cnt.reshape(-1))
    return edge, offs


@pytest.mark.parametrize("nsubsets", [1, 3])
@pytest.mark.parametrize("w,h,dt", [(4, 4, U8), (16, 16, U8), (64, 32, U8), (8, 8, U16), (32, 32, U16)])
def test_predictors_on_the_mv_range_limits(w, h, dt, nsubsets):
    """Predictors exactly on x_min / x_max / y_min / y_max and the corners, then one eighth-pel and one pixel
    beyond, on the edge blocks of a 348 x 284 frame whose planes carry exactly min_pad: the limits are
    accepted, the rest rejected in every stage, and the right-most footprint ends on the last readable byte."""
    pad = G.min_pad(BORDER_W, BORDER_H, w, h)
    cur_full, ref_full = search_planes(BORDER_W, BORDER_H, pad, dt, seed=w + h)
    blocks = edge_blocks(w, h)
    preds, offs = border_lists(blocks, w, h, nsubsets, seed=w)
    thresh = np.zeros(len(blocks), np.uint32) if nsubsets == 3 else None
    run_search(cur_full, ref_full, pad, blocks, preds, offs, nsubsets, w, h, 300, None, thresh,
               24 if nsubsets == 3 else 0, bd=bits(dt))


# ---------------------------------------------------------------- 3. grid and chunking
def test_second_grid_trip():
    sms = num_sms()
    W, H, w, h, pad = 512, 256, 4, 4, 64
    cur_full, ref_full = search_planes(W, H, pad, U8, seed=31)
    grid = G.grid_blocks(W, H, w, h)
    reps = (SEARCH_WARPS_PER_SM * sms) // len(grid) + 1
    blocks = np.tile(grid, reps)
    n = len(blocks)
    ctas = min(-(-n // 4), 64 * sms)
    assert n > 4 * ctas, "every warp has one block: no second trip"
    rng = np.random.default_rng(31)
    pmv = (rng.integers(-20, 21, (n, 4)) * 8).astype(np.int16)
    preds, offs = predictor_subsets(n, 3, seed=32, max_px=12)
    thresh = rng.integers(0, 200, n).astype(np.uint32)
    run_search(cur_full, ref_full, pad, blocks, preds, offs, 3, w, h, 200, pmv, thresh, 16)


def test_multi_pair_chunks():
    """100 pairs = four launches' worth of kMaxPairs = 32: pairs 32..63 are all empty (a whole chunk skipped),
    empty pairs inside the other chunks, pmv and thresholds present.  Equal to the oracle pair by pair, to
    per-pair calls, and one launch per non-empty chunk."""
    W, H, PAD, w, h = 96, 64, 64, 16, 16
    c = G.ctx()
    imgs = [search_planes(W, H, PAD, U8, seed=50 + k) for k in range(3)]
    views = [(default_view(a, PAD), default_view(b, PAD)) for a, b in imgs]
    NP = 100
    empty = {3, 17, 64, 99} | set(range(32, 64))
    grid = G.grid_blocks(W, H, w, h)
    rng = np.random.default_rng(60)
    per_pair = []
    for k in range(NP):
        cnt = 0 if k in empty else int(rng.integers(1, len(grid) + 1))
        per_pair.append(np.ascontiguousarray(grid[rng.permutation(len(grid))[:cnt]]))
    counts = [len(b) for b in per_pair]
    ends = np.cumsum(counts).astype(np.uint32)
    nb = int(ends[-1])
    blocks = np.concatenate(per_pair)
    preds, offs = predictor_subsets(nb, 3, seed=61, max_px=16)
    pmv = (rng.integers(-24, 25, (nb, 4)) * 8).astype(np.int16)
    thresh = rng.integers(0, 3000, nb).astype(np.uint32)
    chunks = [range(k0, min(k0 + 32, NP)) for k0 in range(0, NP, 32)]
    assert len(chunks) == 4 and all(counts[k] == 0 for k in chunks[1])
    nonempty = sum(any(counts[k] for k in ch) for ch in chunks)
    assert nonempty == 3
    curs = [views[k % 3][0].plane for k in range(NP)]
    refs = [views[(k + 1) % 3][1].plane for k in range(NP)]
    p = B.me_params(w, h, W, H, 450)
    d_blocks, d_preds, d_offs, d_pmv, d_thresh = map(G.to_dev, (blocks, preds, offs, pmv, thresh))
    snap = Snapshot(d_blocks, d_preds, d_offs, d_pmv, d_thresh)
    d_best = sentinel_out(16 * nb)
    before = c.launches
    c.me_search_multi_dev(B.PlanePairs(curs, refs, ends, ends), d_blocks, nb, d_preds, d_offs, 3, p, d_best,
                          d_pmv, d_thresh, 24)
    c.synchronize()
    assert c.launches - before == nonempty
    got = G.from_dev(d_best[:16 * nb], B.ME_RESULT_DTYPE).copy()
    assert_sentinel(d_best, 16 * nb)
    snap.check()
    ocur = [oracle_plane(a, PAD) for a, _ in imgs]
    oref = [oracle_plane(b, PAD) for _, b in imgs]
    d_one = G.dev_empty(16 * len(grid))
    b0 = 0
    for k in range(NP):
        b1 = int(ends[k])
        if b1 == b0:
            continue
        o = offs[3 * b0:3 * b1 + 1]
        sub_preds, sub_offs = preds[o[0]:o[-1]], (o - o[0]).astype(np.uint32)
        want = O.full_pixel_me_blocks(ocur[k % 3], oref[(k + 1) % 3], per_pair[k], sub_preds, sub_offs, 3, w, h, 450,
                                      pmv[b0:b1], thresh[b0:b1], 24)
        assert_best_equal(got[b0:b1], want, f"pair {k} vs oracle")
        c.me_search_dev(curs[k], refs[k], G.to_dev(per_pair[k]), b1 - b0, G.to_dev(sub_preds), G.to_dev(sub_offs), 3,
                        p, d_one, G.to_dev(pmv[b0:b1]), G.to_dev(thresh[b0:b1]), 24)
        c.synchronize()
        np.testing.assert_array_equal(got[b0:b1], G.from_dev(d_one, B.ME_RESULT_DTYPE)[:b1 - b0])
        b0 = b1


# ---------------------------------------------------------------- 4. caller-built plane views
def offset_views(cur_off, ref_off, cur_extra=40, ref_extra=76):
    state = {"n": 0}

    def make(full, pad):
        first = state["n"] % 2 == 0
        state["n"] += 1
        stride = stride4(full.shape[1] + (cur_extra if first else ref_extra), full.itemsize)
        return G.ViewPlane(full, pad, stride, cur_off if first else ref_off)
    return make


VIEW_SEARCH = [(16, 16, U8, o) for o in [(0, 1), (1, 2), (2, 3), (3, 0), (3, 3)]]
VIEW_SEARCH += [(32, 32, U8, o) for o in [(1, 3), (2, 1)]]
VIEW_SEARCH += [(8, 8, U16, o) for o in [(0, 2), (2, 0), (2, 2)]] + [(32, 16, U16, (2, 2))]


@pytest.mark.parametrize("w,h,dt,offs_", VIEW_SEARCH,
                         ids=[f"{w}x{h}-{'u8' if d == U8 else 'u16'}-off{o[0]}{o[1]}" for w, h, d, o in VIEW_SEARCH])
def test_search_on_plane_views(w, h, dt, offs_):
    """Org and ref with pixel (0,0) at byte offsets 0..3 past a 128-byte boundary (0 / 2 at 16 bit), pitches a
    multiple of 4 bytes but not of 16: load_word's and partial_sad's realignment at every shift."""
    W, H, pad = 160, 128, 96
    cur_full, ref_full = search_planes(W, H, pad, dt, seed=w + sum(offs_))
    views = offset_views(*offs_)
    vc = views(cur_full, pad)
    assert (vc.plane.data % 4, (vc.plane.stride * vc.plane.bpp) % 16 != 0) == (offs_[0], True)
    blocks = spread_blocks(W, H, w, h, 16, seed=w)
    n = len(blocks)
    rng = np.random.default_rng(w + h)
    pmv = (rng.integers(-20, 21, (n, 4)) * 8).astype(np.int16)
    for nsubsets in (1, 3):
        preds, offs = predictor_subsets(n, nsubsets, seed=70 + nsubsets, max_px=24)
        thresh = rng.integers(0, 6000, n).astype(np.uint32) if nsubsets == 3 else None
        run_search(cur_full, ref_full, pad, blocks, preds, offs, nsubsets, w, h, 500, pmv, thresh,
                   24 if nsubsets == 3 else 0, bd=bits(dt), views=offset_views(*offs_))


# ---------------------------------------------------------------- 5. the exhaustive grid
def fs_kernel(route, w, h, dtype):
    if route == "u8":
        return f"me_full_search_u8<{w}, {h}, {4 if w >= 8 else 2}>"
    return f"me_full_search_generic<{'unsigned char' if dtype == U8 else 'unsigned short'}>"


def fs_staging_bytes(w, h, rx, ry):
    """b200_me_full_search_dev's u8 staging size (the kernel's row_words for the unclamped window)."""
    np_ = 4 if w >= 8 else 2
    row_words = ((2 * rx + w + 3) // 4 + np_ + 4 + 3) & ~3
    return row_words * 4 * (2 * ry + h)


def fs_route(w, h, dtype, ref_stride, rx, ry):
    u8 = (dtype == U8 and ref_stride % 4 == 0 and fs_staging_bytes(w, h, rx, ry) <= 200 * 1024
          and w == h and w in (8, 16, 32, 64))
    return "u8" if u8 else "generic"


def run_full(cur_full, ref_full, pad, blocks, w, h, rx, ry, step, lam, route, bd=8, views=None, want=None):
    width, height = cur_full.shape[1] - 2 * pad, cur_full.shape[0] - 2 * pad
    dtype = cur_full.dtype.type
    blocks = np.ascontiguousarray(blocks)
    n = len(blocks)
    if want is None:
        want = O.full_search_blocks(oracle_plane(cur_full, pad), oracle_plane(ref_full, pad), blocks, w, h, rx, ry,
                                    step, lam)
    make = views or default_view
    vc, vr = make(cur_full, pad), make(ref_full, pad)
    assert fs_route(w, h, dtype, vr.plane.stride, rx, ry) == route
    c = G.ctx()
    p = B.me_params(w, h, width, height, lam, bit_depth=bd)
    d_blocks = G.to_dev(blocks)
    snap = Snapshot(d_blocks, vc.buf, vr.buf)
    d_best = sentinel_out(16 * n)
    k = G.profiled_kernels(lambda: c.me_full_search_dev(vc.plane, vr.plane, d_blocks, n, p, rx, ry, step, d_best))
    assert k == [fs_kernel(route, w, h, dtype)], k
    got = G.from_dev(d_best[:16 * n], B.ME_RESULT_DTYPE)
    assert_best_equal(got, want)
    assert_sentinel(d_best, 16 * n)
    snap.check()
    return got, vc, vr


@pytest.mark.parametrize("step", [1, 2, 3, 4, 5])
@pytest.mark.parametrize("w", [8, 16, 32, 64])
def test_full_search_u8_every_square_and_step(w, step):
    """me_full_search_u8<W, W, 4> at steps 1..5 (4: the aligned LDS.128 form; others: the funnel shift) with
    ref.data 1..3 bytes off a word: the staging's realignment (mis != 0)."""
    W, H, pad = 192, 128, 96
    cur_full, ref_full = search_planes(W, H, pad, U8, seed=w + step)
    blocks = spread_blocks(W, H, w, w, 6, seed=step)
    rx, ry = (24, 12) if w < 64 else (16, 10)
    mis = 1 + (w // 8 + step) % 3
    run_full(cur_full, ref_full, pad, blocks, w, w, rx, ry, step, 300 * step, "u8",
             views=offset_views(step % 4, mis))


GENERIC_TRIGGERS = [
    # (label, w, h, dtype, bd, rx, ry, step, ref_extra)
    ("non_square", 16, 8, U8, 8, 20, 12, 4, 76),
    ("non_square_step3", 32, 16, U8, 8, 16, 8, 3, 76),
    ("bd10", 16, 16, U16, 10, 20, 12, 4, 76),
    ("bd12", 32, 32, U16, 12, 16, 8, 2, 76),
    ("bd12_small", 4, 8, U16, 12, 12, 8, 1, 76),
    ("ref_stride_odd", 16, 16, U8, 8, 20, 12, 4, 77),
    ("staging_over_200k", 64, 64, U8, 8, 192, 200, 4, 76),
]


@pytest.mark.parametrize("label,w,h,dt,bd,rx,ry,step,ref_extra", GENERIC_TRIGGERS, ids=[g[0] for g in GENERIC_TRIGGERS])
def test_full_search_generic_triggers(label, w, h, dt, bd, rx, ry, step, ref_extra):
    W, H, pad = (256, 192, 96) if label == "staging_over_200k" else (160, 128, 96)
    if label == "staging_over_200k":
        assert fs_staging_bytes(w, h, rx, ry) > 200 * 1024
    cur_full, ref_full = search_planes(W, H, pad, dt, seed=w + h + bd, bd=bd)
    blocks = G.grid_blocks(W, H, w, h) if label == "staging_over_200k" else spread_blocks(W, H, w, h, 6, seed=w)

    def views(full, p, state={"n": 0}):
        first = state["n"] % 2 == 0
        state["n"] += 1
        cols = full.shape[1] + (40 if first else ref_extra)
        stride = cols if label == "ref_stride_odd" and not first else stride4(cols, full.itemsize)
        return G.ViewPlane(full, p, stride, 0 if first else (2 if dt == U16 else 1))
    run_full(cur_full, ref_full, pad, blocks, w, h, rx, ry, step, 900, "generic", bd=bd, views=views)


@pytest.mark.parametrize("route,w,h,dt", [("u8", 8, 8, U8), ("generic", 16, 8, U8), ("generic", 16, 16, U16)])
def test_full_search_second_grid_trip(route, w, h, dt):
    sms = num_sms()
    cap = (FS_U8_CTAS_PER_SM if route == "u8" else FS_GENERIC_CTAS_PER_SM) * sms
    W, H, pad = 256, 128, 64
    cur_full, ref_full = search_planes(W, H, pad, dt, seed=w * h)
    grid = G.grid_blocks(W, H, w, h)
    blocks = np.tile(grid, cap // len(grid) + 1)
    assert len(blocks) > cap, "one block per CTA: no second trip"
    run_full(cur_full, ref_full, pad, blocks, w, h, 4, 4, 4, 200, route, bd=bits(dt))


@pytest.mark.parametrize("route,w,h,dt,step", [("u8", 16, 16, U8, 3), ("u8", 8, 8, U8, 4), ("u8", 64, 64, U8, 1),
                                               ("generic", 16, 8, U8, 4), ("generic", 16, 16, U16, 2)])
def test_full_search_flat_ties(route, w, h, dt, step):
    """Flat planes, lambda 0: every position ties and the first one scanned (y_lo, x_lo) wins."""
    W, H, pad = 128, 96, 96
    shape = (H + 2 * pad, W + 2 * pad)
    cur_full, ref_full = np.full(shape, 7, dt), np.full(shape, 9 if dt == U8 else 900, dt)
    blocks = G.grid_blocks(W, H, w, h)
    rx, ry = 24, 12
    want = np.zeros(len(blocks), B.ME_RESULT_DTYPE)
    d = w * h * abs(int(cur_full[0, 0]) - int(ref_full[0, 0]))
    for k, b in enumerate(blocks):
        x_min, x_max, y_min, y_max = G.mv_range(W, H, int(b["x"]), int(b["y"]), w, h)
        dx, dy = max(-rx, int(np.fix(x_min / 8))), max(-ry, int(np.fix(y_min / 8)))
        want[k] = (256 * d, d, 8 * dy, 8 * dx)
    got, _, _ = run_full(cur_full, ref_full, pad, blocks, w, h, rx, ry, step, 0, route, bd=bits(dt))
    assert_best_equal(got, want, "closed form")


# ---------------------------------------------------------------- 6. lookahead geometry
LA_CASES = [
    # (width, height, tiles (w_sb, h_sb), prev, full search, range scale, bit depth, smooth, lambda)
    (1, 1, (64, 64), False, 1, 1, 8, False, 1.0),
    (7, 5, (1, 1), True, 1, 2, 10, True, 2.0),
    (9, 17, (3, 2), False, 0, 1, 12, False, 0.0),
    (65, 33, (1, 1), True, 1, 16, 8, True, 3.0),
    (65, 33, (64, 64), False, 1, 4, 10, False, 1e12),
    (203, 139, (3, 2), True, 1, 16, 12, True, 1e12),
    (203, 139, (1, 1), False, 0, 1, 8, False, 0.0),
    (203, 139, (4, 3), False, 1, 16, 12, False, 0.0),
    (1918, 1078, (64, 64), False, 0, 1, 8, True, 3.0),
]
LA_IDS = [f"{w}x{h}-t{t[0]}x{t[1]}-prev{int(pv)}-fs{fs}-rs{rs}-bd{bd}-lam{lam:g}"
          for w, h, t, pv, fs, rs, bd, sm, lam in LA_CASES]


def la_need(width, height, s):
    """b200_lookahead_motion_dev's pad requirement for both level-s planes (include/b200rdo.h)."""
    W8, H8 = (width + 7) & ~7, (height + 7) & ~7
    mv_full = 32 if s == 0 else 64
    wm, hm = min(mv_full, W8 + (1 << s) - 1) >> s, min(mv_full, H8 + (1 << s) - 1) >> s
    pw, ph = (width + (1 << s) - 1) >> s, (height + (1 << s) - 1) >> s
    return max((16 >> s) + wm, (16 >> s) + hm, ((W8 + 16) >> s) + wm - pw, ((H8 + 16) >> s) + hm - ph)


def la_views(img, pads, offset=0):
    out = []
    for s, im in enumerate(levels(img)):
        full = padded(im, pads[s])
        out.append(G.ViewPlane(full, pads[s], stride4(full.shape[1] + 20, full.itemsize), offset))
    return out


@pytest.mark.parametrize("case", LA_CASES, ids=LA_IDS)
def test_lookahead_geometry(case):
    """Frames whose sides are not multiples of 8 (W8 > width, odd half and quarter planes, crop() rounding of
    the edge blocks), tiles of 1x1, 3x2, 4x3 and frame size, 12 bit, range scale 16 with the exhaustive grid
    at quarter resolution, lambda 0 and one that saturates to UINT32_MAX; planes at exactly the pad the
    launcher requires."""
    w, h = case[0], case[1]
    cur, ref, p, prev, cur_img, ref_img = case_inputs(case)
    if p.me_lambda >= 1e12:
        assert p.me_lambda * 256.0 * 0.5 >= 2**32 - 1
    want = oracle_motion(cur, ref, w, h, p, prev)
    pads = [la_need(w, h, s) for s in range(3)]
    vc, vr = la_views(cur_img, pads, 1 if p.bit_depth == 8 else 2), la_views(ref_img, pads, 3 if p.bit_depth == 8 else 0)
    wib, hib = grid_dims(w, h)
    c = G.ctx()
    d_prev = None if prev is None else G.to_dev(np.ascontiguousarray(prev[None], STATS_DTYPE))
    snap = Snapshot(d_prev, *[v.buf for v in vc + vr])
    d_stats = sentinel_out(8 * wib * hib)
    before = c.launches
    c.lookahead_motion_dev([[v.plane for v in vc]], [[v.plane for v in vr]], params(p), d_stats, d_prev,
                           None if prev is None else [1])
    c.synchronize()
    assert c.launches - before == launches_formula(w, h, p)
    got = G.from_dev(d_stats[:8 * wib * hib], STATS_DTYPE).reshape(hib, wib)
    assert_grid_equal(got, want)
    assert_sentinel(d_stats, 8 * wib * hib)
    snap.check()


def test_lookahead_multi_pair_past_the_grid_cap():
    """Enough pairs of 636 x 356 frames in 1x1-superblock tiles that the 16 px level's diagonal and refinement
    launches both have more items than 4 warps x 32 CTAs per SM: a second grid-stride trip.  Pairs share three
    pyramids, so the oracle runs once per distinct (cur, ref)."""
    sms = num_sms()
    w, h = 636, 356
    W8, H8 = (w + 7) & ~7, (h + 7) & ~7
    p = Params(bit_depth=8, me_lambda=2.0, full_search=1, range_scale=2, tile_w_sb=1, tile_h_sb=1)
    diag_items = -(-W8 // 16) * -(-H8 // 64)         # nbx x tile rows at the 16 px level
    refine_items = -(-W8 // 32) * -(-H8 // 32)       # the 32 px blocks re-searched before it
    npairs = LA_WARPS_PER_SM * sms // min(diag_items, refine_items) + 2
    assert npairs * diag_items > LA_WARPS_PER_SM * sms and npairs * refine_items > LA_WARPS_PER_SM * sms
    imgs = [images(w, h, 8, sm, 90 + k)[k % 2] for k, sm in enumerate((True, False, True))]
    combos = [(k % 3, (k + 1 + k // 3) % 3) for k in range(npairs)]
    combos = [(a, b if b != a else (b + 1) % 3) for a, b in combos]
    opyr = [pyramid(im) for im in imgs]
    want = {cb: oracle_motion(opyr[cb[0]], opyr[cb[1]], w, h, p) for cb in set(combos)}
    dpyr = [[G.ctx().plane_from_host(im, 64) for im in levels(img)] for img in imgs]
    c = G.ctx()
    before = c.launches
    got = device_motion([dpyr[a] for a, _ in combos], [dpyr[b] for _, b in combos], w, h, p)
    assert c.launches - before == launches_formula(w, h, p)
    for k, cb in enumerate(combos):
        assert_grid_equal(got[k], want[cb])
    free(*dpyr)


# ---------------------------------------------------------------- 7. read footprints
def scramble_outside(view, rng):
    """Overwrite every byte of the view's buffer outside the padded image (pixel (-pad, -pad) to
    (width + pad, height + pad)) with random bytes."""
    pl = view.plane
    host = view.buf.cpu().numpy().copy()
    start = pl.data - view.buf.data_ptr() - pl.pad * (pl.stride + 1) * pl.bpp
    pitch, row = pl.stride * pl.bpp, (pl.width + 2 * pl.pad) * pl.bpp
    keep = np.zeros(host.size, bool)
    r = np.arange(pl.height + 2 * pl.pad)[:, None] * pitch + start + np.arange(row)[None, :]
    keep[r.reshape(-1)] = True
    assert keep.sum() < host.size
    host[~keep] = rng.integers(0, 256, int((~keep).sum()), dtype=np.uint8)
    view.buf.copy_(torch.from_numpy(host))


SEARCH_FOOTPRINT = [(16, 16, U8, (1, 3)), (64, 64, U8, (3, 1)), (4, 4, U8, (2, 2)), (32, 32, U16, (2, 0)),
                    (8, 16, U16, (0, 2))]


@pytest.mark.parametrize("w,h,dt,offs_", SEARCH_FOOTPRINT,
                         ids=[f"{w}x{h}-{'u8' if d == U8 else 'u16'}" for w, h, d, _ in SEARCH_FOOTPRINT])
def test_search_reads_stay_inside_min_pad(w, h, dt, offs_):
    """Planes with exactly min_pad at unaligned origins; predictors on every get_mv_range limit, the ladder
    run to its end.  Every byte outside the padded planes replaced: the results do not change."""
    pad = G.min_pad(BORDER_W, BORDER_H, w, h)
    cur_full, ref_full = search_planes(BORDER_W, BORDER_H, pad, dt, seed=w * 3 + h)
    blocks = edge_blocks(w, h)
    preds, offs = border_lists(blocks, w, h, 3, seed=h)
    thresh = np.zeros(len(blocks), np.uint32)
    made, make = [], offset_views(*offs_)

    def views(full, p):
        made.append(make(full, p))
        return made[-1]
    got = run_search(cur_full, ref_full, pad, blocks, preds, offs, 3, w, h, 300, None, thresh, 24, bd=bits(dt),
                     views=views)
    vc, vr = made
    rng = np.random.default_rng(w + h)
    for v in (vc, vr):
        scramble_outside(v, rng)
    c = G.ctx()
    p = B.me_params(w, h, BORDER_W, BORDER_H, 300, bit_depth=bits(dt))
    d_best = G.dev_empty(16 * len(blocks))
    c.me_search_dev(vc.plane, vr.plane, G.to_dev(blocks), len(blocks), G.to_dev(preds), G.to_dev(offs), 3, p, d_best,
                    None, G.to_dev(thresh), 24)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_best, B.ME_RESULT_DTYPE)[:len(blocks)], got)


FULL_FOOTPRINT = [
    # (label, frame w, h, block w, h, dtype, rx, ry, step, ref offset, route)
    ("u8_16x16_right_edge", 128, 96, 16, 16, U8, 48, 16, 4, 0, "u8"),
    ("u8_16x16_mis3", 124, 92, 16, 16, U8, 48, 16, 4, 3, "u8"),
    ("u8_64x64_step3", 200, 136, 64, 64, U8, 40, 24, 3, 1, "u8"),
    ("u8_8x8_step5", 100, 60, 8, 8, U8, 30, 20, 5, 2, "u8"),
    ("generic_16x8", 124, 92, 16, 8, U8, 48, 16, 4, 1, "generic"),
    ("generic_u16", 124, 92, 16, 16, U16, 40, 16, 2, 2, "generic"),
]


@pytest.mark.parametrize("label,W,H,w,h,dt,rx,ry,step,roff,route", FULL_FOOTPRINT, ids=[f[0] for f in FULL_FOOTPRINT])
def test_full_search_reads_stay_inside_min_pad(label, W, H, w, h, dt, rx, ry, step, roff, route):
    """Windows clamped to get_mv_range on planes with exactly min_pad, every block of the frame (the right-most
    column included: the staging of me_full_search_u8 ends on the window's last byte)."""
    pad = G.min_pad(W, H, w, h)
    cur_full, ref_full = search_planes(W, H, pad, dt, seed=W + w + step)
    blocks = G.grid_blocks(W, H, w, h)
    got, vc, vr = run_full(cur_full, ref_full, pad, blocks, w, h, rx, ry, step, 250, route, bd=bits(dt),
                           views=offset_views(0, roff))
    rng = np.random.default_rng(W + h)
    for v in (vc, vr):
        scramble_outside(v, rng)
    c = G.ctx()
    d_best = G.dev_empty(16 * len(blocks))
    c.me_full_search_dev(vc.plane, vr.plane, G.to_dev(blocks), len(blocks), B.me_params(w, h, W, H, 250,
                         bit_depth=bits(dt)), rx, ry, step, d_best)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_best, B.ME_RESULT_DTYPE)[:len(blocks)], got)


@pytest.mark.parametrize("case", [LA_CASES[1], LA_CASES[3], LA_CASES[5], LA_CASES[7]], ids=lambda c: f"{c[0]}x{c[1]}")
def test_lookahead_reads_stay_inside_the_required_pad(case):
    w, h = case[0], case[1]
    cur, ref, p, prev, cur_img, ref_img = case_inputs(case, seed=23)
    want = oracle_motion(cur, ref, w, h, p, prev)
    pads = [la_need(w, h, s) for s in range(3)]
    vc, vr = la_views(cur_img, pads, 2), la_views(ref_img, pads, 0)
    d_prev = None if prev is None else G.to_dev(np.ascontiguousarray(prev[None], STATS_DTYPE))
    flags = None if prev is None else [1]
    wib, hib = grid_dims(w, h)
    c = G.ctx()

    def run():
        d = G.dev_empty(8 * wib * hib)
        c.lookahead_motion_dev([[v.plane for v in vc]], [[v.plane for v in vr]], params(p), d, d_prev, flags)
        c.synchronize()
        return G.from_dev(d, STATS_DTYPE)[:wib * hib].reshape(hib, wib)
    first = run()
    assert_grid_equal(first, want)
    rng = np.random.default_rng(w * h)
    for v in vc + vr:
        scramble_outside(v, rng)
    assert first.tobytes() == run().tobytes()


# ---------------------------------------------------------------- 8. rejections and hygiene
def plane_copy(pl, **kw):
    q = B.Plane()
    C.memmove(C.byref(q), C.byref(pl), C.sizeof(B.Plane))
    for k, v in kw.items():
        setattr(q, k, v)
    return q


def arr_of(planes):
    a = (B.Plane * max(len(planes), 1))()
    for k, pl in enumerate(planes):
        C.memmove(C.byref(a[k]), C.byref(pl), C.sizeof(B.Plane))
    return a


def expect_rejected(call, outs):
    c = G.ctx()
    snaps = [o.clone() for o in outs]
    before = c.launches
    st = call()
    assert st == B.ERR_ARG, st
    assert c.launches == before
    torch.cuda.synchronize()
    for o, s in zip(outs, snaps):
        assert torch.equal(o, s), "a rejected call wrote its output"


def test_search_rejections():
    c = G.ctx()
    L = c.L
    W, H, pad, w, h = 64, 64, 96, 16, 16
    cur_full, ref_full = search_planes(W, H, pad, U8, seed=1)
    vc, vr = default_view(cur_full, pad), default_view(ref_full, pad)
    cur, ref = vc.plane, vr.plane
    blocks = G.grid_blocks(W, H, w, h)
    n = len(blocks)
    preds, offs = predictor_subsets(n, 3, seed=1, max_px=8)
    d_blocks, d_preds, d_offs = map(G.to_dev, (blocks, preds, offs))
    d_thresh = G.to_dev(np.zeros(n, np.uint32))
    d_best = sentinel_out(16 * n)
    P = lambda **kw: B.me_params(kw.get("w", w), kw.get("h", h), W, H, 100)  # noqa: E731
    vp = lambda t: None if t is None else t.data_ptr()  # noqa: E731

    def single(ctx=True, cur_=cur, ref_=ref, blocks_=d_blocks, nb=n, offs_=d_offs, nsub=3, thresh_=d_thresh,
               params_=None, umh=24, best=d_best, use_params=True):
        pp = params_ or P()
        return L.b200_me_search_dev(c.h if ctx else None, C.byref(cur_) if cur_ is not None else None,
                                    C.byref(ref_) if ref_ is not None else None, vp(blocks_), nb, vp(d_preds),
                                    vp(offs_), nsub, None, vp(thresh_), C.byref(pp) if use_params else None, umh,
                                    vp(best))
    bad = [
        lambda: single(ctx=False),
        lambda: single(cur_=None),
        lambda: single(ref_=None),
        lambda: single(nb=2**32),
        lambda: single(use_params=False),
        lambda: single(nsub=2),
        lambda: single(nsub=0),
        lambda: single(thresh_=None),
        lambda: single(params_=P(w=2)),
        lambda: single(params_=P(w=12)),
        lambda: single(params_=P(w=256)),
        lambda: single(params_=P(h=0)),
        lambda: single(params_=P(h=129)),
        lambda: single(umh=-1),
        lambda: single(umh=65),
        lambda: single(cur_=plane_copy(cur, data=None)),
        lambda: single(ref_=plane_copy(ref, data=None)),
        lambda: single(ref_=plane_copy(ref, bpp=2)),
        lambda: single(cur_=plane_copy(cur, bpp=3), ref_=plane_copy(ref, bpp=3)),
        lambda: single(cur_=plane_copy(cur, stride=cur.stride + 1)),
        lambda: single(ref_=plane_copy(ref, stride=ref.stride + 2)),
        lambda: single(blocks_=None),
        lambda: single(offs_=None),
        lambda: single(best=None),
    ]
    for k, call in enumerate(bad):
        expect_rejected(call, [d_best])

    def multi(npairs=2, curs=None, refs=None, ends=(n, 2 * n), nb=2 * n, blocks_=None, best=None):
        cs, rs = arr_of(curs or [cur] * npairs), arr_of(refs or [ref] * npairs)
        e = np.ascontiguousarray(ends, np.uint32)
        return L.b200_me_search_multi_dev(c.h, npairs, C.addressof(cs), C.addressof(rs),
                                          e.ctypes.data, vp(blocks_), nb, vp(d_preds), vp(d_offs), 1, None, None,
                                          C.byref(P()), 0, vp(best))
    d_b2, d_best2 = G.to_dev(np.tile(blocks, 2)), sentinel_out(32 * n)
    bad_multi = [
        lambda: multi(npairs=0, ends=(0,), nb=0, blocks_=d_b2, best=d_best2),
        lambda: multi(ends=(n + 1, n), blocks_=d_b2, best=d_best2),          # decreasing
        lambda: multi(ends=(n, 2 * n - 1), blocks_=d_b2, best=d_best2),      # does not end at nblocks
        lambda: multi(nb=2**32, ends=(n, 2 * n), blocks_=d_b2, best=d_best2),
        lambda: multi(refs=[ref, plane_copy(ref, data=None)], blocks_=d_b2, best=d_best2),
        lambda: multi(curs=[cur, plane_copy(cur, stride=cur.stride + 1)], blocks_=d_b2, best=d_best2),
        lambda: multi(curs=[cur, plane_copy(cur, bpp=2)], refs=[ref, plane_copy(ref, bpp=2)], blocks_=d_b2,
                      best=d_best2),
        lambda: multi(blocks_=None, best=d_best2),
    ]
    for call in bad_multi:
        expect_rejected(call, [d_best2])

    # nblocks == 0 with NULL device pointers: OK, nothing launched
    before = c.launches
    assert single(nb=0, blocks_=None, offs_=None, best=None, thresh_=None, nsub=1) == B.OK
    assert multi(ends=(0, 0), nb=0) == B.OK
    assert c.launches == before
    assert_sentinel(d_best, 0)


def test_full_search_rejections():
    c = G.ctx()
    L = c.L
    W, H, pad, w, h = 64, 64, 96, 16, 16
    cur_full, ref_full = search_planes(W, H, pad, U8, seed=2)
    vc, vr = default_view(cur_full, pad), default_view(ref_full, pad)
    cur, ref = vc.plane, vr.plane
    blocks = G.grid_blocks(W, H, w, h)
    n = len(blocks)
    d_blocks, d_best = G.to_dev(blocks), sentinel_out(16 * n)
    vp = lambda t: None if t is None else t.data_ptr()  # noqa: E731

    def call(ctx=True, cur_=cur, ref_=ref, blocks_=d_blocks, nb=n, pw=w, ph=h, satd=False, rx=16, ry=8, step=4,
             best=d_best, use_params=True):
        p = B.me_params(pw, ph, W, H, 100, use_satd=satd)
        return L.b200_me_full_search_dev(c.h if ctx else None, C.byref(cur_) if cur_ is not None else None,
                                         C.byref(ref_) if ref_ is not None else None, vp(blocks_), nb,
                                         C.byref(p) if use_params else None, rx, ry, step, vp(best))
    bad = [
        lambda: call(ctx=False), lambda: call(cur_=None), lambda: call(ref_=None), lambda: call(use_params=False),
        lambda: call(cur_=plane_copy(cur, data=None)), lambda: call(ref_=plane_copy(ref, bpp=2)),
        lambda: call(cur_=plane_copy(cur, bpp=4), ref_=plane_copy(ref, bpp=4)),
        lambda: call(pw=0), lambda: call(ph=129), lambda: call(pw=256),
        lambda: call(rx=-1), lambda: call(ry=-1), lambda: call(step=0), lambda: call(satd=True),
        lambda: call(blocks_=None), lambda: call(best=None),
    ]
    for f in bad:
        expect_rejected(f, [d_best])
    before = c.launches
    assert call(nb=0, blocks_=None, best=None) == B.OK
    assert c.launches == before
    assert_sentinel(d_best, 0)


def test_lookahead_rejections():
    c = G.ctx()
    L = c.L
    w, h = 72, 40
    cur_img, ref_img = images(w, h, 8, True, 3)
    pads = [la_need(w, h, s) for s in range(3)]
    vc, vr = la_views(cur_img, pads), la_views(ref_img, pads)
    cur, ref = [v.plane for v in vc], [v.plane for v in vr]
    wib, hib = grid_dims(w, h)
    d_stats = sentinel_out(8 * wib * hib)
    d_prev = G.to_dev(np.zeros(wib * hib, STATS_DTYPE))

    def call(curs=None, refs=None, p=None, ctx=True, npairs=1, prev=None, flags=None, stats=d_stats, use_p=True):
        cs, rs = arr_of(curs or cur), arr_of(refs or ref)
        pp = params(p or Params())
        fl = None if flags is None else np.ascontiguousarray(flags, np.uint8)
        return L.b200_lookahead_motion_dev(c.h if ctx else None, npairs, C.addressof(cs), C.addressof(rs),
                                           C.byref(pp) if use_p else None, None if prev is None else prev.data_ptr(),
                                           None if fl is None else fl.ctypes.data,
                                           None if stats is None else stats.data_ptr())
    thin = [[plane_copy(q, pad=q.pad - (s == k)) for s, q in enumerate(cur)] for k in range(3)]
    thin_ref = [[plane_copy(q, pad=q.pad - (s == k)) for s, q in enumerate(ref)] for k in range(3)]
    bad = [
        lambda: call(ctx=False), lambda: call(use_p=False), lambda: call(stats=None), lambda: call(npairs=0),
        lambda: call(prev=d_prev),                                        # d_prev without has_prev
        lambda: call(p=Params(range_scale=0)), lambda: call(p=Params(range_scale=17)),
        lambda: call(p=Params(bit_depth=10)),                             # bpp 1 at 10 bit
        lambda: call(curs=[plane_copy(q, bpp=3) for q in cur], refs=[plane_copy(q, bpp=3) for q in ref]),
        lambda: call(curs=[plane_copy(cur[0], width=8193)] + cur[1:]),
        lambda: call(curs=[plane_copy(cur[0], data=None)] + cur[1:]),
        lambda: call(refs=ref[:2] + [plane_copy(ref[2], data=None)]),
        lambda: call(refs=[plane_copy(ref[0], bpp=2)] + ref[1:]),
    ] + [lambda k=k: call(curs=thin[k]) for k in range(3)] + [lambda k=k: call(refs=thin_ref[k]) for k in range(3)]
    for f in bad:
        expect_rejected(f, [d_stats])
    # 16-bit planes: the bit depth must be 9..12
    u16 = [G.ViewPlane(padded(im.astype(U16), pads[s]), pads[s], stride4(im.shape[1] + 2 * pads[s] + 8, 2), 0)
           for s, im in enumerate(levels(cur_img))]
    for bd in (8, 13):
        expect_rejected(lambda: call(curs=[v.plane for v in u16], refs=[v.plane for v in u16],
                                     p=Params(bit_depth=bd)), [d_stats])
    # exactly the required pads are accepted (the footprint test runs on them)
    assert call() == B.OK
    c.synchronize()
    assert_sentinel(d_stats, 8 * wib * hib)
