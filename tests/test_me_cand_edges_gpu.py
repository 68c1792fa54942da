"""Candidate-list ME (b200_me_candidates_dev / _multi_dev) at the edges where its kernels can go
wrong: which kernel the dispatcher picks, first-minimum ties, get_mv_range borders at the smallest
legal padding, block orders other than raster, caller-built plane descriptors, extreme lambdas,
predictors and pixel values, and the paths selected by environment variables.

Every case runs through the single-pair entry point and through the multi-pair one (the same
pair twice around an empty pair), and compares sad, cost and the per-block winner with the oracle
(oracle_lib.fullpel_candidates, pinned by the reference's SAD/SATD known answers): the winner is
numpy's first argmin of the oracle costs, or the empty record when a block has no candidate in
range.  Each case also asserts the kernel its single-pair call reached (torch.profiler; the
multi-pair routing is pinned by MULTI_CASES in test_me_gpu.py), so that a changed threshold cannot
move a case off the path it was written for without a failing test.
"""
import os

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_oracle_dist import _mv_rate

pytestmark = pytest.mark.gpu

EMPTY_COST = np.uint64(2**64 - 1)
EMPTY_SAD = np.uint32(0xFFFFFFFF)
U8, U16 = np.uint8, np.uint16

# kernel (name<template args>) each route launches; "generic" is per pair, then the segmented argmin
def kernels_for(route, w, h, dtype, satd, env=None):
    t = "unsigned char" if dtype == U8 else "unsigned short"
    s = "true" if satd else "false"
    if route == "chunk" and env == "B200_OLD_SATD" and dtype == U8:
        route = "warp"
    if route == "chunk" and env == "B200_HBD_GENERIC" and dtype == U16:
        route = "generic"
    return {"group": [f"me_cand_group_u8<{w}, {h}, {s}>"],
            "warp": [f"me_cand_warp_u8<{w}, {h}, {s}>"],
            "chunk": [f"me_chunk_lists<{t}, {w}, {h}, {s}>"],
            "generic": [f"me_cand_generic<{t}>", "me_best_from_cost"]}[route]


def expected_best(cands, offs, want_sad, want_cost):
    nb = len(offs) - 1
    best = np.zeros(nb, B.ME_RESULT_DTYPE)
    best["cost"], best["sad"] = EMPTY_COST, EMPTY_SAD     # MotionSearchResult::empty(): mv 0
    for b in range(nb):
        lo, hi = int(offs[b]), int(offs[b + 1])
        if lo == hi:
            continue
        k = lo + int(np.argmin(want_cost[lo:hi]))
        if want_cost[k] != EMPTY_COST:
            best[b] = (want_cost[k], want_sad[k], cands[k]["mv_row"], cands[k]["mv_col"])
    return best


def assert_best_equal(got, want, what):
    for f in ("cost", "sad", "mv_row", "mv_col"):
        np.testing.assert_array_equal(got[f], want[f], err_msg=f"{what}: best.{f}")


def padded(img, pad):
    return np.pad(img, pad, mode="edge")


def oracle_plane(full, pad):
    p = O.Plane(full.shape[1] - 2 * pad, full.shape[0] - 2 * pad, pad, dtype=full.dtype)
    p.data[:] = full
    return p


ROUTE_LOG = []


def run_case(cur_full, ref_full, pad, blocks, cands, offs, w, h, route, *, satd=False, bd=8, lam=0, hint=0,
             pmv=None, allow_hp=False, views=None, env=None, want_best=None):
    """Evaluate one candidate list on the device twice (single pair; pairs (A, empty, A)) and compare
    every output with the oracle; the kernel the single-pair call launched must be `route`'s.  cur_full / ref_full are the padded images (pixel (0,0) at
    [pad, pad]); `views(full, pad)` builds the device descriptors (default: a 128-byte aligned
    plane that holds the padding as given).  `want_best`: an independent statement of the winners,
    checked against the oracle's before the device is."""
    dtype = cur_full.dtype
    width, height = cur_full.shape[1] - 2 * pad, cur_full.shape[0] - 2 * pad
    blocks, cands = np.ascontiguousarray(blocks), np.ascontiguousarray(cands)
    offs = np.ascontiguousarray(offs, np.uint32)
    nb, nc = len(blocks), len(cands)
    assert nc == int(offs[-1]) and (np.diff(cands["block"].astype(np.int64)) >= 0).all()
    ocur, oref = oracle_plane(cur_full, pad), oracle_plane(ref_full, pad)
    opmv = None if pmv is None else np.ascontiguousarray(pmv, np.int16)
    want_sad, want_cost = O.fullpel_candidates(ocur, oref, blocks, cands, w, h, satd, lam, opmv, allow_hp)
    best = expected_best(cands, offs, want_sad, want_cost)
    if want_best is not None:
        assert_best_equal(best, want_best, "oracle vs closed form")
    make = views or (lambda full, p: G.ViewPlane(full, p, G_stride(full), 0))
    vc, vr = make(cur_full, pad), make(ref_full, pad)
    dcur, dref = vc.plane, vr.plane
    c = G.ctx()
    p = B.me_params(w, h, width, height, lam, allow_hp=allow_hp, use_satd=satd, bit_depth=bd, window_hint_px=hint)
    want_k = kernels_for(route, w, h, dtype, satd, env)

    d_blocks, d_cands, d_offs = map(G.to_dev, (blocks, cands, offs))
    d_pmv = None if pmv is None else G.to_dev(opmv)
    d_sad, d_cost, d_best = G.dev_empty(4 * nc), G.dev_empty(8 * nc), G.dev_empty(16 * nb)
    k1 = G.profiled_kernels(lambda: c.me_candidates_dev(dcur, dref, d_blocks, nb, d_cands, nc, p, d_offs, d_pmv,
                                                        d_sad, d_cost, d_best))
    np.testing.assert_array_equal(G.from_dev(d_sad, np.uint32)[:nc], want_sad, err_msg="sad")
    np.testing.assert_array_equal(G.from_dev(d_cost, np.uint64)[:nc], want_cost, err_msg="cost")
    assert_best_equal(G.from_dev(d_best, B.ME_RESULT_DTYPE)[:nb], best, "single pair")

    # pairs (A, empty, A): block / candidate indices of the second copy are global
    c2 = np.concatenate([cands, cands])
    c2["block"][nc:] += nb
    o2 = np.concatenate([offs, offs[1:] + np.uint32(nc)])
    b2 = np.concatenate([blocks, blocks])
    d2_pmv = None if pmv is None else G.to_dev(np.concatenate([opmv, opmv]))
    pairs = B.PlanePairs([dcur] * 3, [dref] * 3, [nb, nb, 2 * nb], [nc, nc, 2 * nc])
    d_sad2, d_cost2, d_best2 = G.dev_empty(8 * nc), G.dev_empty(16 * nc), G.dev_empty(32 * nb)
    c.me_candidates_multi_dev(pairs, G.to_dev(b2), 2 * nb, G.to_dev(c2), 2 * nc, p, G.to_dev(o2), d2_pmv,
                              d_sad2, d_cost2, d_best2)
    c.synchronize()
    np.testing.assert_array_equal(G.from_dev(d_sad2, np.uint32)[:2 * nc], np.tile(want_sad, 2), err_msg="multi sad")
    np.testing.assert_array_equal(G.from_dev(d_cost2, np.uint64)[:2 * nc], np.tile(want_cost, 2),
                                  err_msg="multi cost")
    assert_best_equal(G.from_dev(d_best2, B.ME_RESULT_DTYPE)[:2 * nb], np.tile(best, 2), "multi pair")

    ROUTE_LOG.append((os.environ.get("PYTEST_CURRENT_TEST", "?").split(" ")[0], k1))
    assert k1 == want_k, f"single-pair call reached {k1}, expected {want_k}"
    return want_sad, want_cost, best


def G_stride(full):
    """Row pitch of the default device planes: 128-byte multiple with room for a TMA map's lead."""
    return (full.shape[1] + 224 + 127) // 128 * 128


@pytest.fixture(scope="module", autouse=True)
def _print_routing_table():
    yield
    if ROUTE_LOG:
        print("\nkernel reached by each case (single-pair call):")
        for name, k in ROUTE_LOG:
            print(f"  {name}: {' + '.join(k)}")


def env_params(cases, relevant):
    """Each case with no variable set, and again under every variable that can change its path."""
    out = []
    for case in cases:
        out.append(pytest.param(None, *case, id=f"{case[0]}-default"))
        for e in relevant(*case[1:]):
            out.append(pytest.param(e, *case, id=f"{case[0]}-{e}"))
    return out


def relevant_envs(w, h, dtype, satd, route):
    e = []
    if route == "group" and not satd and dtype == U8 and 16 <= w <= 64:
        e.append("B200_NO_TMA")
    if route == "chunk" and dtype == U8:
        e.append("B200_OLD_SATD")
    if dtype == U16:
        e.append("B200_HBD_GENERIC")
    return e


# ------------------------------------------------------------------ 2. first-minimum ties

# (label, w, h, dtype, satd, route); "hint" on the cooperative paths: the window hint is set, else 0
TIE_PATHS = [
    ("coop16", 16, 16, U8, False, "group"),
    ("coop16_nohint", 16, 16, U8, False, "group"),
    ("coop32", 32, 32, U8, False, "group"),
    ("coop64", 64, 64, U8, False, "group"),
    ("satd_group", 16, 16, U8, True, "group"),
    ("warp", 16, 16, U8, False, "warp"),
    ("chunk_u8", 16, 16, U8, True, "chunk"),
    ("chunk_u16", 16, 16, U16, True, "chunk"),
    ("generic", 16, 12, U8, False, "generic"),
]
TIE_LENGTHS = [1, 31, 33, 257, 600]


def tie_hint(label, n, w, h, reach):
    """A window hint that keeps the case on its path for a list of n candidates per block: the
    dispatcher takes the sparse kernels when n * w * h * 4 < (2 hint + w) * (2 hint + h)."""
    if label.endswith("nohint"):
        return 0
    if label in ("warp", "chunk_u8"):
        return 400
    return reach


def first_in_range_positions(nb, n):
    """Per block, the index of its first in-range candidate: lane, warp and CTA-round borders."""
    cand = [0, 1, 30, 31, 32, 33, 63, 64, 127, 128, 255, 256, 257, 511, 599]
    pos = [p for p in cand if p < n] or [0]
    return np.array([pos[b % len(pos)] for b in range(nb)])


def tie_case(label, w, h, dtype, satd, route, n, periodic):
    """Blocks of 16 x 16 .. 64 x 64 on a small frame; per block n candidates, those before f_b out
    of get_mv_range (empty), the rest tie on cost (lambda 0).  Flat planes: every in-range
    candidate ties.  Periodic planes (period 8, cur = ref shifted by (3, 5) px): only candidates
    on the period tie, at SAD 0; they sit at f_b, a few later places and again (the same vector)
    at the end of the list."""
    W, H, pad = 192, 128, 96
    maxv = 255 if dtype == U8 else 1023
    if periodic:
        rng = np.random.default_rng(w + 7 * n)
        T = rng.integers(0, maxv + 1, (8, 8))
        ys, xs = np.mgrid[-pad:H + pad, -pad:W + pad]
        dy, dx = 5, 3
        ref_full = T[ys % 8, xs % 8].astype(dtype)
        cur_full = T[(ys + dy) % 8, (xs + dx) % 8].astype(dtype)
    else:
        cur_full = np.full((H + 2 * pad, W + 2 * pad), 7, dtype)
        ref_full = np.full((H + 2 * pad, W + 2 * pad), 9 if dtype == U8 else 900, dtype)
    blocks = G.grid_blocks(W, H, max(w, 32), max(h, 32))[:12]
    nb = len(blocks)
    reach = 2 if n == 1 else 8
    rng = np.random.default_rng(1000 + n + w)
    f = first_in_range_positions(nb, n)
    cands = np.zeros(nb * n, B.CAND_DTYPE)
    cands["block"] = np.repeat(np.arange(nb, dtype=np.uint32), n)
    mv = rng.integers(-reach, reach + 1, (nb, n, 2)) * 8
    if periodic:      # off the period: columns a multiple of 8 px, the matching shift is 3 px mod 8
        mv[:, :, 1] = rng.integers(-1, 2, (nb, n)) * 64
    for b in range(nb):
        x_min, x_max, y_min, y_max = G.mv_range(W, H, int(blocks[b]["x"]), int(blocks[b]["y"]), w, h)
        mv[b, :f[b], 1] = x_max + 8 * (1 + np.arange(f[b]) % 3)        # out of range: empty
        if periodic:
            on = [f[b]] + [q for q in (f[b] + 1, f[b] + 32, f[b] + 255) if q < n - 1]
            for j, q in enumerate(on):
                mv[b, q] = (8 * (5 + 8 * (j % 2)), 8 * (3 - 8 * (j // 2 % 2)))
            if n - 1 > f[b]:
                mv[b, n - 1] = mv[b, f[b]]                               # duplicate of the winner
    cands["mv_row"], cands["mv_col"] = mv[:, :, 0].reshape(-1), mv[:, :, 1].reshape(-1)
    offs = (np.arange(nb + 1) * n).astype(np.uint32)
    # closed form: the first in-range candidate wins, with the SAD / SATD of a flat or matching block
    want = np.zeros(nb, B.ME_RESULT_DTYPE)
    k = np.arange(nb) * n + f
    if periodic:
        d = 0
    elif satd:
        d = (w // 8) * (h // 8) * 8 * abs(int(cur_full[0, 0]) - int(ref_full[0, 0]))
    else:
        d = w * h * abs(int(cur_full[0, 0]) - int(ref_full[0, 0]))
    want["cost"], want["sad"] = 256 * d, d
    want["mv_row"], want["mv_col"] = cands["mv_row"][k], cands["mv_col"][k]
    hint = tie_hint(label, n, w, h, (8 if n == 1 else 13) if periodic else reach)
    return cur_full, ref_full, pad, blocks, cands, offs, hint, want


@pytest.mark.parametrize("periodic", [False, True], ids=["flat", "periodic"])
@pytest.mark.parametrize("n", TIE_LENGTHS)
@pytest.mark.parametrize("env,label,w,h,dtype,satd,route",
                         env_params(TIE_PATHS, relevant_envs))
def test_ties_pick_first_minimum(monkeypatch, env, label, w, h, dtype, satd, route, n, periodic):
    if label == "coop16_nohint" and n == 1:
        route = "warp"      # one candidate per block and no hint: a sparse list
    if env:
        monkeypatch.setenv(env, "1")
    cur_full, ref_full, pad, blocks, cands, offs, hint, want = tie_case(label, w, h, dtype, satd, route, n, periodic)
    run_case(cur_full, ref_full, pad, blocks, cands, offs, w, h, route, satd=satd,
             bd=8 if dtype == U8 else 10, lam=0, hint=hint, env=env, want_best=want)


@pytest.mark.parametrize("env,label,w,h,dtype,satd,route",
                         env_params([p for p in TIE_PATHS if p[0] != "coop16_nohint"],
                                    relevant_envs))
def test_rate_ties_pick_first_minimum(monkeypatch, env, label, w, h, dtype, satd, route):
    """Equal SAD everywhere (flat planes), lambda > 0, two predictors: the cost is decided by
    min(r1, r2 + 1) alone, which takes few distinct values, so most blocks have tied minima."""
    if env:
        monkeypatch.setenv(env, "1")
    n = 64
    cur_full, ref_full, pad, blocks, _, _, _, _ = tie_case(label, w, h, dtype, satd, route, 1, False)
    nb = len(blocks)
    rng = np.random.default_rng(w * 3 + satd)
    cands = np.zeros(nb * n, B.CAND_DTYPE)
    cands["block"] = np.repeat(np.arange(nb, dtype=np.uint32), n)
    cands["mv_row"] = rng.integers(-2, 3, nb * n) * 8
    cands["mv_col"] = rng.integers(-2, 3, nb * n) * 8
    pmv = (rng.integers(-3, 4, (nb, 4)) * 8).astype(np.int16)
    offs = (np.arange(nb + 1) * n).astype(np.uint32)
    lam = 100
    d = w * h * abs(int(cur_full[0, 0]) - int(ref_full[0, 0]))
    if satd:
        d = (w // 8) * (h // 8) * 8 * abs(int(cur_full[0, 0]) - int(ref_full[0, 0]))
    want = np.zeros(nb, B.ME_RESULT_DTYPE)
    ties = 0
    for b in range(nb):
        p0, p1 = tuple(int(v) for v in pmv[b, :2]), tuple(int(v) for v in pmv[b, 2:])
        rates = [min(_mv_rate((int(q["mv_row"]), int(q["mv_col"])), p0, 0),
                     _mv_rate((int(q["mv_row"]), int(q["mv_col"])), p1, 0) + 1)
                 for q in cands[b * n:(b + 1) * n]]
        k = b * n + int(np.argmin(rates))
        ties += rates.count(min(rates)) > 1
        want[b] = (256 * d + min(rates) * lam, d, cands[k]["mv_row"], cands[k]["mv_col"])
    assert ties >= nb // 2
    hint = 400 if label in ("warp", "chunk_u8") else 48
    run_case(cur_full, ref_full, pad, blocks, cands, offs, w, h, route, satd=satd, bd=8 if dtype == U8 else 10,
             lam=lam, hint=hint, pmv=pmv, env=env, want_best=want)


# ------------------------------------------------------------------ 3. get_mv_range borders

BORDER_W, BORDER_H = 348, 284     # not multiples of 8: w_in_b / h_in_b round up to 352 x 288
BORDER_SIZES = [(4, 4, U8), (8, 8, U8), (16, 16, U8), (32, 32, U8), (64, 64, U8), (16, 16, U16), (32, 32, U16)]


def edge_blocks(bw, bh):
    """Every block of the 8-aligned grid that touches a frame edge (corners included), raster order."""
    w8, h8 = 8 * ((BORDER_W + 7) >> 3), 8 * ((BORDER_H + 7) >> 3)
    # the last column / row sits flush with the 8-aligned edge, where the far limit is nearest
    xs = sorted(set(range(0, w8 - bw + 1, bw)) | {w8 - bw})
    ys = sorted(set(range(0, h8 - bh + 1, bh)) | {h8 - bh})
    pos = [(x, y) for y in ys for x in xs if x in (xs[0], xs[-1]) or y in (ys[0], ys[-1])]
    b = np.zeros(len(pos), B.BLOCK_DTYPE)
    b["x"], b["y"] = [p[0] for p in pos], [p[1] for p in pos]
    return b


def border_planes(dtype, pad, seed):
    maxv = 255 if dtype == U8 else 1023
    cur, ref = G.make_planes(BORDER_W, BORDER_H, pad, dtype, seed=seed, bit_depth=8 if dtype == U8 else 10)
    for img in (cur, ref):     # outermost visible rows / columns unlike their neighbours
        for sl_edge, sl_in in (((slice(None), -1), (slice(None), -2)), ((-1, slice(None)), (-2, slice(None))),
                               ((slice(None), 0), (slice(None), 1)), ((0, slice(None)), (1, slice(None)))):
            img[sl_edge] = ((img[sl_in].astype(np.int64) + maxv // 2) % (maxv + 1)).astype(dtype)
    return padded(cur, pad), padded(ref, pad)


BORDER_KINDS = [("dense_sad", False), ("sparse_sad", False), ("sparse_satd", True)]


def border_route(kind, w, h, dtype, satd):
    if dtype == U16:
        return "chunk"
    if kind.startswith("dense"):
        return "group"
    return "chunk" if satd and w >= 8 and h >= 8 and (w // 8) * (h // 8) <= 32 else "warp"


BORDER_CASES = [(f"{w}x{h}{'' if dt == U8 else '_u16'}-{kind}", w, h, dt, satd, border_route(kind, w, h, dt, satd))
                for w, h, dt in BORDER_SIZES for kind, satd in BORDER_KINDS
                if not (dt == U16 and kind == "sparse_sad")]


@pytest.mark.parametrize("pad_kind", ["pad88", "minpad"])
@pytest.mark.parametrize("env,label,w,h,dtype,satd,route", env_params(BORDER_CASES, relevant_envs))
def test_mv_range_borders(monkeypatch, env, label, w, h, dtype, satd, route, pad_kind):
    """Candidates exactly on x_min / x_max / y_min / y_max and the corners, plus one eighth-pel and
    one full-pel beyond, for blocks on all four edges of a 348 x 284 frame.  With the smallest pad
    the reach allows (4 w_in_b - width + 16 + w), the right-most accepted footprint ends on the last
    readable column: a window, TMA box or over-read that stops short or shifts changes a SAD."""
    if env:
        monkeypatch.setenv(env, "1")
    pad = 88 if pad_kind == "pad88" else G.min_pad(BORDER_W, BORDER_H, w, h)
    assert pad >= 16 + max(w, h)
    cur_full, ref_full = border_planes(dtype, pad, seed=w + h + pad)
    blocks = edge_blocks(w, h)
    dense = label.endswith("dense_sad")
    hint = 16 + max(w, h) + 1 if dense else 400
    edge = G.border_cands(blocks, BORDER_W, BORDER_H, w, h, reach=hint if dense else None)
    rng = np.random.default_rng(w * h)
    per = 64 if dense else 3
    fill = np.zeros(len(blocks) * per, B.CAND_DTYPE)
    fill["block"] = np.repeat(np.arange(len(blocks), dtype=np.uint32), per)
    r = min(hint, 24) if dense else 12
    fill["mv_row"], fill["mv_col"] = rng.integers(-r, r + 1, (2, len(fill))) * 8
    cands, offs = G.merge_lists(len(blocks), edge, fill)
    _, want_cost, _ = run_case(cur_full, ref_full, pad, blocks, cands, offs, w, h, route, satd=satd,
                               bd=8 if dtype == U8 else 10, lam=300, hint=hint, env=env)
    # the limits themselves are accepted, everything beyond them is not
    rng_ok = np.array([G.mv_range(BORDER_W, BORDER_H, int(b["x"]), int(b["y"]), w, h) for b in blocks])[cands["block"]]
    inside = ((cands["mv_col"] >= rng_ok[:, 0]) & (cands["mv_col"] <= rng_ok[:, 1]) &
              (cands["mv_row"] >= rng_ok[:, 2]) & (cands["mv_row"] <= rng_ok[:, 3]))
    np.testing.assert_array_equal(want_cost != EMPTY_COST, inside)
    assert (cands["mv_col"] == rng_ok[:, 1]).any() and (cands["mv_row"] == rng_ok[:, 3]).any()


# ------------------------------------------------------------------ 4. block orders

NR_W, NR_H = 336, 208     # 21 x 13 blocks of 16 x 16: raster rows end inside a group


def nonraster_blocks(order):
    grid = G.grid_blocks(NR_W, NR_H, 16, 16)
    rng = np.random.default_rng(42)
    if order == "raster":
        return grid
    if order in ("zorder", "hint_small"):
        return G.zorder_blocks(NR_W, NR_H, 16, 16)
    if order == "permuted":
        return grid[rng.permutation(len(grid))]
    if order == "repeated":
        return grid[np.sort(rng.integers(0, len(grid), len(grid)))][::-1].copy()
    if order == "far_apart":        # consecutive blocks in opposite corners: groups halve down to one block
        corners = [(0, 0), (NR_W - 16, NR_H - 16), (0, NR_H - 16), (NR_W - 16, 0)]
        b = np.zeros(48, B.BLOCK_DTYPE)
        for k in range(len(b)):
            x, y = corners[k % 4]
            b[k] = (x + (16 if x == 0 else -16) * (k // 4 % 3), y + (16 if y == 0 else -16) * (k // 12))
        return b
    raise ValueError(order)


NR_ORDERS = ["raster", "zorder", "permuted", "repeated", "far_apart", "hint_small"]
NR_KINDS = [("sad_dense", False, "group"), ("satd_dense", True, "group"), ("satd_sparse", True, "chunk")]
NR_CASES = [(f"{o}-{k}", 16, 16, U8, s, r) for o in NR_ORDERS for k, s, r in NR_KINDS]


@pytest.mark.parametrize("env,label,w,h,dtype,satd,route", env_params(NR_CASES, relevant_envs))
def test_nonraster_block_lists(monkeypatch, env, label, w, h, dtype, satd, route):
    """Z order inside 64 x 64 superblocks, a seeded permutation, repeated blocks, and lists that
    force the grouped kernel's fallbacks: blocks far apart (halving down to single blocks, then
    direct loads when even one block's candidates outgrow the window) and a hint smaller than the
    candidates' reach (exact bounding box).  Raster rows of 21 blocks end inside a group (split at
    the row break).  The CSR stays in ascending block index order; only positions move."""
    if env:
        monkeypatch.setenv(env, "1")
    order, kind = label.split("-")
    blocks = nonraster_blocks(order)
    pad = 160
    cur, ref = G.make_planes(NR_W, NR_H, pad, U8, seed=len(blocks) + satd)
    per = {"sad_dense": 64, "satd_dense": 16, "satd_sparse": 4}[kind]
    reach = 60 if order == "far_apart" else 24
    cands, offs = G.random_cands(len(blocks), per, reach, seed=5 + len(order))
    hint = {"hint_small": 4, "far_apart": 8}.get(order, reach)
    if kind == "satd_sparse":
        hint = 400
    pmv = (np.random.default_rng(3).integers(-16, 17, (len(blocks), 4)) * 8).astype(np.int16)
    run_case(padded(cur, pad), padded(ref, pad), pad, blocks, cands, offs, 16, 16, route, satd=satd, lam=900,
             hint=hint, pmv=pmv, env=env)


# ------------------------------------------------------------------ 5. caller-built plane views

VW, VH, VPAD = 320, 192, 48


def view_maker(offset=0, with_alloc=True, cur_stride=None, ref_stride=None):
    """Device descriptors over buffers built here: pixel (0,0) `offset` bytes past a 16-byte
    boundary, `alloc` set or NULL, the cur / ref element strides chosen freely."""
    state = {"n": 0}

    def make(full, pad):
        is_cur = state["n"] == 0
        state["n"] += 1
        stride = (cur_stride if is_cur else ref_stride) or G_stride(full)
        return G.ViewPlane(full, pad, stride, offset, with_alloc)
    return make


def _stride4(cols):     # a multiple of 4, not of 16
    s = (cols + 3) // 4 * 4
    return s + 4 if s % 16 == 0 else s


def _odd(cols):         # not a multiple of 4
    return cols + 1 if (cols + 1) % 4 else cols + 3


VIEW_CASES = []
for _off in (1, 4, 12):
    for _alloc in (True, False):
        VIEW_CASES.append((f"off{_off}_{'alloc' if _alloc else 'noalloc'}",
                           dict(offset=_off, with_alloc=_alloc), "group", "warp"))
VIEW_CASES += [
    ("cur_stride_mult4", dict(cur_stride=_stride4(VW + 2 * VPAD)), "group", "chunk"),
    ("cur_stride_odd", dict(cur_stride=_odd(VW + 2 * VPAD)), "group", "group"),
    ("both_strides_odd", dict(cur_stride=_odd(VW + 2 * VPAD), ref_stride=_odd(VW + 2 * VPAD) + 4), "generic",
     "generic"),
]


@pytest.mark.parametrize("kind", ["dense_sad", "sparse_satd"])
@pytest.mark.parametrize("label,view,dense_route,sparse_route", VIEW_CASES, ids=[c[0] for c in VIEW_CASES])
def test_caller_built_plane_views(label, view, dense_route, sparse_route, kind):
    """Descriptors not made by b200_plane_alloc: origins 1, 4 and 12 bytes off a 16-byte boundary
    with and without `alloc` (the TMA lead derivation and the hand-staged window origin), a cur
    stride that is a multiple of 4 but not of 16, strides that are not multiples of 4.  The
    8x8-chunk kernel needs 16-byte aligned reference rows and the word-pitch kernels a cur stride
    that is a multiple of 4; the rest fall back to the kernels that take any layout."""
    satd = kind == "sparse_satd"
    cur, ref = G.make_planes(VW, VH, VPAD, U8, seed=len(label))
    blocks = G.grid_blocks(VW, VH, 16, 16)
    cands, offs = G.random_cands(len(blocks), 4 if satd else 64, 24, seed=len(label) + 1)
    route = sparse_route if satd else dense_route
    run_case(padded(cur, VPAD), padded(ref, VPAD), VPAD, blocks, cands, offs, 16, 16, route, satd=satd, lam=500,
             hint=400 if satd else 24, views=view_maker(**view))


# ------------------------------------------------------------------ 6. extreme parameters

EXT_PATHS = [
    ("group_sad", 16, 16, U8, False, "group"),
    ("group_satd", 16, 16, U8, True, "group"),
    ("warp_sad", 16, 16, U8, False, "warp"),
    ("chunk_u8", 16, 16, U8, True, "chunk"),
    ("chunk_u16", 16, 16, U16, True, "chunk"),
    ("generic", 16, 12, U8, True, "generic"),
]
EXT_PMV = [32767, -32767, -32768, 0, 8, -1]


@pytest.mark.parametrize("allow_hp", [False, True])
@pytest.mark.parametrize("lam", [0, 1, 2**31, 2**32 - 1])
@pytest.mark.parametrize("label,w,h,dtype,satd,route", EXT_PATHS, ids=[p[0] for p in EXT_PATHS])
def test_extreme_lambda_and_predictors(label, w, h, dtype, satd, route, lam, allow_hp):
    """lambda up to 2^32 - 1 (rate * lambda needs 64 bits; cost reaches 2^38) with predictors at
    +-32767 and -32768, so that mv - pmv wraps in i16 and reaches i16::MIN (rate 16 per component
    with allow_hp).  Eighth-pel candidates -1 / +1 hit the wrap from both sides."""
    W, H, pad = 128, 96, 96
    cur, ref = G.make_planes(W, H, pad, dtype, seed=lam % 97 + w, bit_depth=8 if dtype == U8 else 12)
    blocks = G.grid_blocks(W, H, 16, 16)
    nb = len(blocks)
    rng = np.random.default_rng(lam % 1009 + allow_hp)
    per = 64 if route == "group" else 6
    cands, offs = G.random_cands(nb, per, 12, seed=lam % 13, jitter=False, fullpel=False)
    special = np.array([-1, 1, 0, -8, 8, -7], np.int16)
    cands["mv_row"][::per] = special[np.arange(nb) % len(special)]
    cands["mv_col"][1::per] = special[(np.arange(nb) + 3) % len(special)]
    pmv = rng.choice(EXT_PMV, (nb, 4)).astype(np.int16)
    pmv[0] = (-32768, -32768, 32767, 32767)
    pmv[1] = (32767, -32768, -32768, 32767)
    cands[2]["mv_row"], cands[2]["mv_col"] = 0, 0                    # 0 - (-32768) wraps to i16::MIN
    cands[per + 2]["mv_row"], cands[per + 2]["mv_col"] = -1, -1      # -1 - 32767 = i16::MIN
    run_case(padded(cur, pad), padded(ref, pad), pad, blocks, cands, offs, w, h, route, satd=satd,
             bd=8 if dtype == U8 else 12, lam=lam, hint=400 if route != "group" else 12, pmv=pmv, allow_hp=allow_hp)


def hadamard_sign(ys, xs):
    """(-1)^popcount(x & y) on 8 x 8 tiles: its 2-D Hadamard transform has all 64 coefficients at
    +-8 times the amplitude, the largest sum |coeff| any +-max block can give."""
    v = (ys % 8) & (xs % 8)
    par = (v ^ (v >> 1) ^ (v >> 2)) & 1
    return 1 - 2 * par


@pytest.mark.parametrize("satd", [False, True], ids=["sad", "satd"])
@pytest.mark.parametrize("pattern", ["max_vs_zero", "hadamard"])
@pytest.mark.parametrize("w,h,route", [(32, 32, "chunk"), (64, 64, "generic"), (128, 128, "generic")])
def test_full_scale_12bit(w, h, route, pattern, satd):
    """12-bit pixels at full scale on the largest blocks: org all 4095 against ref all 0, and a
    +-4095 difference on the Hadamard pattern with the largest SATD.  The SAD / SATD sums must not
    wrap in their u32 (or packed u16) accumulators."""
    W = H = 256
    pad = 160
    ys, xs = np.mgrid[-pad:H + pad, -pad:W + pad]
    if pattern == "max_vs_zero":
        cur_full = np.full(ys.shape, 4095, U16)
        ref_full = np.zeros(ys.shape, U16)
    else:
        s = hadamard_sign(ys, xs)
        cur_full = np.where(s > 0, 4095, 0).astype(U16)
        ref_full = (4095 - cur_full).astype(U16)
    blocks = G.grid_blocks(W, H, w, h)
    cands, offs = G.random_cands(len(blocks), 8, 2, seed=w, jitter=False)
    cands["mv_row"] *= 8        # multiples of 8 px: the pattern stays aligned
    cands["mv_col"] *= 8
    want_sad, _, _ = run_case(cur_full, ref_full, pad, blocks, cands, offs, w, h, route, satd=satd, bd=12, lam=2**32 - 1,
                              hint=16)
    nch = (w // 8) * (h // 8)
    if not satd:
        want = 4095 * w * h
    elif pattern == "max_vs_zero":
        want = nch * 8 * 4095            # DC only: (64 * 4095 per chunk + 4) >> 3
    else:
        want = nch * 64 * 4095           # 64 coefficients of 8 * 4095 per chunk, >> 3
    assert (want_sad == want).all()


# ------------------------------------------------------------------ routing coverage

def test_routes_cover_every_candidate_kernel():
    """The cases above, taken together, reach every kernel the dispatcher can launch for candidate
    lists (each case asserts its own kernel on the device)."""
    seen = set()
    for cases in (TIE_PATHS, BORDER_CASES, NR_CASES):
        for label, w, h, dt, s, r in cases:
            for e in [None] + relevant_envs(w, h, dt, s, r):
                seen.update(kernels_for(r, w, h, dt, s, e))
    for _, view, dr, sr in VIEW_CASES:
        seen.update(kernels_for(dr, 16, 16, U8, False) + kernels_for(sr, 16, 16, U8, True))
    for label, w, h, dt, s, r in EXT_PATHS:
        seen.update(kernels_for(r, w, h, dt, s))
    families = {
        "me_cand_group_u8 SAD": lambda k: k.startswith("me_cand_group_u8<") and k.endswith("false>"),
        "me_cand_group_u8 SATD": lambda k: k.startswith("me_cand_group_u8<") and k.endswith("true>"),
        "me_cand_warp_u8 SAD": lambda k: k.startswith("me_cand_warp_u8<") and k.endswith("false>"),
        "me_cand_warp_u8 SATD": lambda k: k.startswith("me_cand_warp_u8<") and k.endswith("true>"),
        "me_chunk_lists u8": lambda k: k.startswith("me_chunk_lists<unsigned char"),
        "me_chunk_lists u16": lambda k: k.startswith("me_chunk_lists<unsigned short"),
        "me_cand_generic u8": lambda k: k == "me_cand_generic<unsigned char>",
        "me_cand_generic u16": lambda k: k == "me_cand_generic<unsigned short>",
        "me_best_from_cost": lambda k: k == "me_best_from_cost",
    }
    missing = [f for f, hit in families.items() if not any(hit(k) for k in seen)]
    assert not missing, missing
