"""CPU tests of the encode-time motion search in the oracle (oracle/encode_me.c).

- orc_enc_subset_predictors (get_subset_predictors, me.rs:386-534, in CORNER mode with tile-local subset B) against
  an independent Python model written from the reference text, predictor list for predictor list, over every block
  size at every 4x4 position of frames whose sizes are and are not multiples of 8, several tile grids, with and
  without LAST's stats.
- orc_estimate_motion_items against me.c's stages composed by hand: orc_full_pixel_me_blocks with one subset, the
  SATD get_fullpel_mv_rd re-measure through orc_fullpel_candidates, then orc_subpel_diamond_search_blocks.

Also shared with the GPU tests: the ctypes bindings and the case generator.
"""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O
from tests.test_oracle_lookahead_me import STATS_DTYPE, Params, oracle_motion, pyramid
from tests.test_oracle_search import mv_range, tdiv8

ITEM_DTYPE = np.dtype([("x4", "<u2"), ("y4", "<u2"), ("slot", "u1"), ("pad_", "u1"), ("pmv", "<i2", (2, 2))])
MV_DTYPE = np.dtype([("row", "<i2"), ("col", "<i2")])
TX_SIZES = [(4, 4), (8, 8), (16, 16), (32, 32), (64, 64), (4, 8), (8, 4), (8, 16), (16, 8), (16, 32), (32, 16),
            (32, 64), (64, 32), (4, 16), (16, 4), (8, 32), (32, 8), (16, 64), (64, 16)]
PAD = 96  # >= the pad b200_estimate_motion_dev needs for 64-sided blocks of any frame size


def grid_dims(width, height):
    return 2 * ((width + 7) >> 3), 2 * ((height + 7) >> 3)


def min_pad(width, height, sizes):
    """the pad include/b200rdo.h states for b200_estimate_motion_dev over the given (w, h) sizes"""
    W8, H8 = (width + 7) & ~7, (height + 7) & ~7
    return max(max(w + 19, W8 - width + w + 20, h + 19, H8 - height + h + 20) for w, h in sizes)


_BOUND = False


def _lib():
    global _BOUND
    L = O.lib()
    if not _BOUND:
        vp, pd, i32, sz = C.c_void_p, C.c_ssize_t, C.c_int, C.c_size_t
        L.orc_enc_subset_predictors.restype = i32
        L.orc_enc_subset_predictors.argtypes = [vp, vp] + [i32] * 8 + [vp, vp]
        L.orc_estimate_motion_items.restype = None
        L.orc_estimate_motion_items.argtypes = [vp, pd, vp, vp] + [i32] * 4 + [vp, vp, vp, i32, i32, C.c_double] + \
            [i32] * 4 + [vp, vp, sz, vp, i32]
        L.orc_subpel_diamond_search_blocks.restype = None
        L.orc_subpel_diamond_search_blocks.argtypes = [vp, pd, vp, pd] + [i32] * 3 + [vp, sz] + [i32] * 3 + \
            [C.c_uint32, vp] + [i32] * 3 + [vp, i32]
        _BOUND = True
    return L


def oracle_predictors(stats, prev, width, height, tiles, x4, y4, w, h):
    wib, hib = grid_dims(width, height)
    out = np.zeros(11, MV_DTYPE)
    st = np.ascontiguousarray(stats, STATS_DTYPE)
    pv = None if prev is None else np.ascontiguousarray(prev, STATS_DTYPE)
    n = _lib().orc_enc_subset_predictors(st.ctypes.data, None if pv is None else pv.ctypes.data, wib, hib, tiles[0],
                                         tiles[1], x4, y4, w, h, out.ctypes.data, None)
    return [(int(v["row"]), int(v["col"])) for v in out[:n]]


class Enc:
    """one frame's inputs: source, nslots references, the stats grids, the settings"""

    def __init__(self, width, height, bd=8, nslots=2, tiles=(64, 64), prev=True, lookahead=False, seed=1, pad=PAD,
                 allow_hp=0, use_satd=1, filter_mode=0, me_lambda=2.5):
        from tests.gpu_util import make_planes
        self.width, self.height, self.bd, self.nslots, self.tiles, self.pad = width, height, bd, nslots, tiles, pad
        self.allow_hp, self.use_satd, self.filter_mode, self.me_lambda = allow_hp, use_satd, filter_mode, me_lambda
        dtype = np.uint8 if bd == 8 else np.uint16
        rng = np.random.default_rng(seed)
        self.src_img = None
        self.ref_imgs = []
        shifts = [(5, -3), (-2, 4), (3, 3), (-6, -1), (1, -5), (4, 2), (-3, -4)]
        for k in range(nslots):
            cur, ref = make_planes(width, height, 0, dtype, seed=seed, bit_depth=bd, smooth=True, shift=shifts[k])
            if k == 0:
                self.src_img = cur
            self.ref_imgs.append(ref if k == 0 else np.clip(ref.astype(np.int64) + rng.integers(-3, 4, ref.shape), 0,
                                                            (1 << bd) - 1).astype(dtype))
        wib, hib = grid_dims(width, height)
        if lookahead:  # the lookahead's own grids (the encode pass reads them unchanged)
            p = Params(bit_depth=bd, me_lambda=me_lambda, tile_w_sb=tiles[0], tile_h_sb=tiles[1])
            sp = pyramid(self.src_img)
            self.stats = np.stack([oracle_motion(sp, pyramid(r), width, height, p) for r in self.ref_imgs])
            older = make_planes(width, height, 0, dtype, seed=seed + 7, bit_depth=bd, smooth=True)[0]
            op = pyramid(older)
            self.prev = np.stack([oracle_motion(op, pyramid(r), width, height, p) for r in self.ref_imgs]) \
                if prev else None
        else:  # scattered grids: vectors near and far (process_cand clamps the far ones)
            def grids(s):
                g = np.zeros((nslots, hib, wib), STATS_DTYPE)
                r = np.random.default_rng(s)
                g["mv_row"] = np.where(r.random(g.shape) < 0.1, r.integers(-4000, 4001, g.shape),
                                       r.integers(-60, 61, g.shape))
                g["mv_col"] = np.where(r.random(g.shape) < 0.1, r.integers(-4000, 4001, g.shape),
                                       r.integers(-60, 61, g.shape))
                g["normalized_sad"] = r.integers(0, 1 << 20, g.shape)
                return g
            self.stats = grids(seed + 100)
            self.prev = grids(seed + 200) if prev else None
        self.has_prev = None if self.prev is None else [1 if k % 3 != 2 else 0 for k in range(nslots)]
        self.src = O.Plane(width, height, pad, dtype)
        self.src.fill_from(self.src_img)
        self.refs = []
        for r in self.ref_imgs:
            q = O.Plane(width, height, pad, dtype)
            q.fill_from(r)
            self.refs.append(q)

    def items(self, sizes, seed=3, per_size=None, pmv_near_border=False, invalid=0):
        """items of the given TxSize indices, grouped by size -> (items, size_end).  Positions: every 4x4 offset of
        the frame (or `per_size` random ones), slots cycling; pmv scattered, or on the range borders."""
        rng = np.random.default_rng(seed)
        wib, hib = grid_dims(self.width, self.height)
        groups = []
        for s in range(19):
            if s not in sizes:
                groups.append(np.zeros(0, ITEM_DTYPE))
                continue
            w, h = TX_SIZES[s]
            if per_size is None:
                pos = [(x, y) for y in range(hib) for x in range(wib)]
            else:
                pos = list(zip(rng.integers(0, wib, per_size), rng.integers(0, hib, per_size)))
            it = np.zeros(len(pos) + invalid, ITEM_DTYPE)
            it["x4"][:len(pos)] = [p[0] for p in pos]
            it["y4"][:len(pos)] = [p[1] for p in pos]
            it["slot"] = rng.integers(0, self.nslots, len(it))
            it["pmv"] = rng.integers(-200, 201, (len(it), 2, 2))
            if pmv_near_border:
                for k in range(len(pos)):
                    x_min, x_max, y_min, y_max = mv_range(wib, hib, 4 * pos[k][0], 4 * pos[k][1], w, h)
                    it["pmv"][k] = [[y_min + int(rng.integers(-9, 10)), x_max + int(rng.integers(-9, 10))],
                                    [y_max + int(rng.integers(-9, 10)), x_min + int(rng.integers(-9, 10))]]
            for k in range(len(pos), len(it)):  # invalid: slot out of range, or outside the 4x4 grid
                kind = k % 3
                it["slot"][k] = 7 if kind == 0 else 0
                it["x4"][k] = wib + (k % 5) if kind == 1 else 0
                it["y4"][k] = hib if kind == 2 else 0
            groups.append(it)
        size_end = np.cumsum([len(g) for g in groups]).astype(np.uint32)
        return np.ascontiguousarray(np.concatenate(groups)), size_end

    def oracle(self, items, size_end, threads=0):
        out = np.zeros(len(items), O.ME_RESULT_DTYPE)
        refs = (C.c_void_p * self.nslots)(*[r.origin_ptr() for r in self.refs])
        strides = (C.c_ssize_t * self.nslots)(*[r.stride for r in self.refs])
        st = np.ascontiguousarray(self.stats, STATS_DTYPE)
        pv = None if self.prev is None else np.ascontiguousarray(self.prev, STATS_DTYPE)
        hp = None if self.has_prev is None else np.ascontiguousarray(self.has_prev, np.uint8)
        ends = np.ascontiguousarray(size_end, np.uint32)
        _lib().orc_estimate_motion_items(
            self.src.origin_ptr(), self.src.stride, C.addressof(refs), C.addressof(strides), self.nslots,
            self.src.bpp, self.width, self.height, st.ctypes.data, None if pv is None else pv.ctypes.data,
            None if hp is None else hp.ctypes.data, self.bd, self.allow_hp, self.me_lambda, self.use_satd,
            self.filter_mode, self.tiles[0], self.tiles[1], ends.ctypes.data, items.ctypes.data, len(items),
            out.ctypes.data, threads)
        return out

    def lam(self):
        v = self.me_lambda * 256.0 * 0.5
        return 0 if not v > 0 else min(int(v), 2**32 - 1)


# ---------------------------------------------------------------- the independent model of the gathering
def model_predictors(stats, prev, width, height, tiles, x4, y4, w, h):
    """get_subset_predictors, me.rs:386-534, CORNER { right: true, bottom: true }, ssdec 0, as all_mvs()"""
    wib, hib = grid_dims(width, height)
    x_min, x_max, y_min, y_max = mv_range(wib, hib, 4 * x4, 4 * y4, w, h)
    tw, th = 16 * tiles[0], 16 * tiles[1]
    tx, ty = (x4 // tw) * tw, (y4 // th) * th
    cols, rows = min(tw, wib - tx), min(th, hib - ty)   # TileMEStats cropped at the frame
    bx, by = x4 - tx, y4 - ty                           # tile_bo

    def proc(st):
        return (min(max(tdiv8(int(st["mv_row"])) * 8, y_min), y_max), min(max(tdiv8(int(st["mv_col"])) * 8, x_min), x_max))

    def T(x, y):
        return stats[ty + y, tx + x]
    wb, hb = (w + 3) >> 2, (h + 3) >> 2
    chw, chh = min(wb >> 1, cols - 1 - bx), min(hb >> 1, rows - 1 - by)
    b = []
    if bx > 0:
        b.append(proc(T(bx - 1, by + chh)))
    if by > 0:
        b.append(proc(T(bx + chw, by - 1)))
    if bx + wb < cols:
        b.append(proc(T(bx + wb, by + chh)))
    if by + hb < rows:
        b.append(proc(T(bx + chw, by + hb)))
    median = proc(T(bx + chw, by + chh))
    b.append((0, 0))
    c = []
    if prev is not None:
        hw, hh = min(wb >> 1, wib - 1 - x4), min(hb >> 1, hib - 1 - y4)
        if x4 > 0:
            c.append(proc(prev[y4 + hh, x4 - 1]))
        if y4 > 0:
            c.append(proc(prev[y4 - 1, x4 + hw]))
        if x4 + wb < wib:
            c.append(proc(prev[y4 + hh, x4 + wb]))
        if y4 + hb < hib:
            c.append(proc(prev[y4 + hb, x4 + hw]))
        c.append(proc(prev[y4 + hh, x4 + hw]))
    return [median] + b + c


def reach(width, height, tiles, x4, y4, w, h):
    """which edge cases a block exercises (for the coverage assertions)"""
    wib, hib = grid_dims(width, height)
    tw, th = 16 * tiles[0], 16 * tiles[1]
    tx, ty = (x4 // tw) * tw, (y4 // th) * th
    cols, rows = min(tw, wib - tx), min(th, hib - ty)
    bx, by = x4 - tx, y4 - ty
    wb, hb = w >> 2, h >> 2
    out = set()
    if (wb >> 1) > cols - 1 - bx or (hb >> 1) > rows - 1 - by:
        out.add("clipped_half")
    if bx + wb == cols - 1 or by + hb == rows - 1:
        out.add("neighbour_just_inside")
    if bx + wb == cols or by + hb == rows:
        out.add("neighbour_just_outside")
    if cols < tw or rows < th:
        out.add("cropped_tile")
    if bx == 0 or by == 0:
        out.add("tile_edge")
    if bx > 0 and by > 0 and bx + wb < cols and by + hb < rows:
        out.add("interior")
    return out


GATHER_CASES = [(200, 120, (1, 1), True), (203, 117, (2, 1), True), (203, 117, (64, 64), False),
                (72, 40, (1, 1), False), (136, 264, (1, 2), True)]


@pytest.mark.parametrize("case", GATHER_CASES, ids=[f"{w}x{h}-t{t[0]}x{t[1]}-prev{int(p)}" for w, h, t, p in GATHER_CASES])
def test_predictors_match_python_model(case):
    width, height, tiles, with_prev = case
    e = Enc(width, height, nslots=1, tiles=tiles, prev=with_prev, seed=width + height)
    wib, hib = grid_dims(width, height)
    seen = set()
    for s, (w, h) in enumerate(TX_SIZES):
        for y4 in range(hib):
            for x4 in range(wib):
                got = oracle_predictors(e.stats[0], None if e.prev is None else e.prev[0], width, height, tiles, x4,
                                        y4, w, h)
                want = model_predictors(e.stats[0], None if e.prev is None else e.prev[0], width, height, tiles, x4,
                                        y4, w, h)
                assert got == want, (s, x4, y4, got, want)
                seen |= reach(width, height, tiles, x4, y4, w, h)
    want_seen = {"clipped_half", "neighbour_just_inside", "neighbour_just_outside", "tile_edge", "interior"}
    if tiles != (64, 64) or width % 64 or height % 64:
        want_seen.add("cropped_tile")
    assert want_seen <= seen, want_seen - seen


def test_subset_c_and_tiles_change_the_lists():
    """LAST's stats and the tile grid are live inputs of the gathering"""
    e = Enc(200, 120, nslots=1, tiles=(1, 1), seed=5)
    a = oracle_predictors(e.stats[0], e.prev[0], 200, 120, (1, 1), 17, 15, 16, 16)
    assert a != oracle_predictors(e.stats[0], None, 200, 120, (1, 1), 17, 15, 16, 16)
    assert oracle_predictors(e.stats[0], e.prev[0], 200, 120, (1, 1), 16, 16, 16, 16) != \
        oracle_predictors(e.stats[0], e.prev[0], 200, 120, (64, 64), 16, 16, 16, 16)


def composed_chain(e: Enc, items, size_end):
    """me.c's stages by hand, per (size, slot): all_mvs through orc_full_pixel_me_blocks (one subset), the SATD
    re-measure through orc_fullpel_candidates, orc_subpel_diamond_search_blocks"""
    wib, hib = grid_dims(e.width, e.height)
    out = np.zeros(len(items), O.ME_RESULT_DTYPE)
    out["cost"], out["sad"] = 2**64 - 1, 2**32 - 1
    lo = 0
    for s in range(19):
        hi = int(size_end[s])
        w, h = TX_SIZES[s]
        for slot in range(e.nslots):
            idx = [i for i in range(lo, hi) if items[i]["slot"] == slot and items[i]["x4"] < wib and items[i]["y4"] < hib]
            if not idx:
                continue
            blocks = np.zeros(len(idx), O.BLOCK_DTYPE)
            blocks["x"], blocks["y"] = items["x4"][idx] * 4, items["y4"][idx] * 4
            pmv = np.ascontiguousarray(items["pmv"][idx].astype(np.int16))
            prev = None if e.prev is None or not e.has_prev[slot] else e.prev[slot]
            lists = [model_predictors(e.stats[slot], prev, e.width, e.height, e.tiles, int(items["x4"][i]),
                                      int(items["y4"][i]), w, h) for i in idx]
            offs = np.zeros(len(idx) + 1, np.uint32)
            offs[1:] = np.cumsum([len(x) for x in lists])
            preds = np.zeros(int(offs[-1]), O.CAND_DTYPE)
            flat = [v for x in lists for v in x]
            preds["mv_row"], preds["mv_col"] = [v[0] for v in flat], [v[1] for v in flat]
            preds["block"] = np.repeat(np.arange(len(idx)), [len(x) for x in lists])
            res = O.full_pixel_me_blocks(e.src, e.refs[slot], blocks, preds, offs, 1, w, h, e.lam(), pmv=pmv,
                                         allow_hp=e.allow_hp)
            if e.use_satd:
                c = np.zeros(len(idx), O.CAND_DTYPE)
                c["block"] = np.arange(len(idx))
                c["mv_row"], c["mv_col"] = res["mv_row"], res["mv_col"]
                sad, cost = O.fullpel_candidates(e.src, e.refs[slot], blocks, c, w, h, True, e.lam(), pmv, e.allow_hp)
                res["sad"], res["cost"] = sad, cost
            _lib().orc_subpel_diamond_search_blocks(
                e.src.origin_ptr(), e.src.stride, e.refs[slot].origin_ptr(), e.refs[slot].stride, e.src.bpp, wib, hib,
                blocks.ctypes.data, len(idx), w, h, e.use_satd, e.lam(), pmv.ctypes.data, e.allow_hp, e.filter_mode,
                e.bd, res.ctypes.data, 0)
            out[idx] = res
        lo = hi
    return out


@pytest.mark.parametrize("bd,use_satd,allow_hp,mode,tiles", [(8, 1, 0, 0, (64, 64)), (10, 0, 1, 2, (1, 1)),
                                                             (12, 1, 1, 3, (2, 1))])
def test_driver_equals_composed_stages(bd, use_satd, allow_hp, mode, tiles):
    e = Enc(104, 72, bd=bd, nslots=3, tiles=tiles, use_satd=use_satd, allow_hp=allow_hp, filter_mode=mode,
            seed=bd + mode)
    items, size_end = e.items(set(range(19)), per_size=12, pmv_near_border=bd == 10, invalid=3)
    got = e.oracle(items, size_end)
    want = composed_chain(e, items, size_end)
    assert got.tobytes() == want.tobytes()
    valid = (items["slot"] < e.nslots) & (items["x4"] < grid_dims(104, 72)[0]) & (items["y4"] < grid_dims(104, 72)[1])
    assert (got["cost"][~valid] == 2**64 - 1).all() and (got["cost"][valid] != 2**64 - 1).all()
    assert ((got["mv_row"] | got["mv_col"]) & 7)[valid].any()   # the sub-pel stage moved some vectors
