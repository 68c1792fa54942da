"""orc_deblock_filter (deblock_filter_frame in rav1e's lagged edge order) against an independent model of the
AV1 specification's loop filter process (section 7.14), pixel for pixel.

The model is written from the specification, not from deblock.rs: the filter size process (base size from the
two transform sizes in the edge's direction, 16 / 8 / 4 for luma and 8 / 4 for chroma, where chroma 8 is the
6-tap class), the adaptive filter strength with sharpness 0 (limit = max(1, lvl), blimit = 2 * (lvl + 2) +
limit, thresh = lvl >> 4, each shifted up by BitDepth - 8), the filter mask, hev, flat and flat2 processes with
those thresholds (rav1e inverts them into levels), the narrow filter in the signed domain with filter4_clamp,
and the generic wide filter (n taps each side, n2 double-weighted centre taps, Round2 by log2Size).  Chroma
transform sizes come from the chroma block's dimensions, capped at 32 (get_tx_size).  Where a decision depends
on which 4x4 block is read, the model reads the blocks rav1e reads (deblock.rs:72-93: the current block at the
edge position, the previous one on the odd mi row / column in subsampled planes), which is where rav1e keeps
its mode info.

Order.  The model runs every vertical edge of a plane first and then every horizontal edge (the
specification's two passes), and inside a pass it computes every edge from the picture as it was when the
pass began and asserts that no pixel is written by two edges.  rav1e filters vertical edges one mi row ahead
of horizontal ones (deblock.rs:1334-1458).  Equality with that order is the correctness argument for the
device's form, which runs all edges of one direction in parallel.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import oracle_lib as O

LAYOUTS = {"400": (1, 1, 1), "420": (3, 1, 1), "422": (3, 1, 0), "444": (3, 0, 0)}
# BlockSize (partition.rs:130-153) in pixels
BSIZE_DIMS = [(4, 4), (4, 8), (8, 4), (8, 8), (8, 16), (16, 8), (16, 16), (16, 32), (32, 16), (32, 32), (32, 64),
              (64, 32), (64, 64), (64, 128), (128, 64), (128, 128), (4, 16), (16, 4), (8, 32), (32, 8), (16, 64),
              (64, 16)]
# TxSize (transform/mod.rs:101-123) in pixels
TX_DIMS = [(4, 4), (8, 8), (16, 16), (32, 32), (64, 64), (4, 8), (8, 4), (8, 16), (16, 8), (16, 32), (32, 16),
           (32, 64), (64, 32), (4, 16), (16, 4), (8, 32), (32, 8), (16, 64), (64, 16)]
INVALID_422 = {(4, 8), (8, 16), (16, 32), (32, 64), (64, 128), (4, 16), (8, 32), (16, 64)}  # no subsampled_size
PAD = 16


# ---------------------------------------------------------------- block grids
def random_grid(rng, w4, h4, layout, skip_p=0.4, intra_p=0.3, deltas=False):
    """A consistent FrameBlocks image (DEBLOCK_MI_DTYPE, h4 x w4): 64x64 superblocks partitioned recursively
    into every block size the layout allows, one transform size per block that tiles it, and per block a
    skip flag, a reference (0 = intra) with a mode of its kind and, with `deltas`, block deltas."""
    g = np.zeros((((h4 + 15) // 16) * 16, ((w4 + 15) // 16) * 16), B.DEBLOCK_MI_DTYPE)
    bad = INVALID_422 if layout == "422" else set()

    def place(x, y, bw, bh):
        bs = BSIZE_DIMS.index((bw, bh))
        txs = [t for t, (tw, th) in enumerate(TX_DIMS) if bw % tw == 0 and bh % th == 0]
        tx = int(rng.choice(txs))
        intra = rng.random() < intra_p
        rec = (bs, tx, int(rng.integers(0, 13)) if intra else int(rng.integers(14, 34)), int(rng.random() < skip_p),
               0 if intra else int(rng.integers(1, 8)),
               tuple(int(v) for v in rng.integers(-8, 8, 4)) if deltas else (0, 0, 0, 0), (0, 0, 0))
        x4, y4 = x // 4, y // 4
        g[y4:y4 + bh // 4, x4:x4 + bw // 4] = rec

    def split(x, y, s):
        opts = ["none", "horz", "split"] + ([] if layout == "422" else ["vert"])
        if s >= 16:
            opts += ["horz4"] + ([] if layout == "422" else ["vert4"])
        if s == 4:
            return place(x, y, 4, 4)
        o = opts[int(rng.integers(0, len(opts)))]
        if o == "none":
            place(x, y, s, s)
        elif o == "horz":
            place(x, y, s, s // 2), place(x, y + s // 2, s, s // 2)
        elif o == "vert":
            place(x, y, s // 2, s), place(x + s // 2, y, s // 2, s)
        elif o == "horz4":
            for k in range(4):
                place(x, y + k * s // 4, s, s // 4)
        elif o == "vert4":
            for k in range(4):
                place(x + k * s // 4, y, s // 4, s)
        else:
            for k in range(4):
                split(x + (k & 1) * s // 2, y + (k >> 1) * s // 2, s // 2)

    for sy in range(0, g.shape[0] * 4, 64):
        for sx in range(0, g.shape[1] * 4, 64):
            split(sx, sy, 64)
    assert all(BSIZE_DIMS[b] not in bad for b in g["bsize"].ravel())
    return np.ascontiguousarray(g[:h4, :w4])


def make_planes(rng, w, h, layout, bd, content="random"):
    """Frame planes with PAD pixels of border (the arrays include the border)."""
    planes, xdec, ydec = LAYOUTS[layout]
    dt = np.uint8 if bd == 8 else np.uint16
    out = []
    for p in range(planes):
        pw, ph = (w + 2 * PAD) >> (xdec if p else 0), (h + 2 * PAD) >> (ydec if p else 0)
        mx = (1 << bd) - 1
        if content == "random":
            a = rng.integers(0, 1 << bd, (ph, pw))
        elif content == "flat":
            a = np.full((ph, pw), int(rng.integers(0, 1 << bd)))
        else:  # oriented steps on a smooth ramp: every filter class and threshold gets reached
            yy, xx = np.mgrid[0:ph, 0:pw]
            ang = rng.random() * np.pi
            base = (np.cos(ang) * xx + np.sin(ang) * yy) * rng.uniform(0.2, 3)
            steps = (((xx // int(rng.integers(3, 9))) + (yy // int(rng.integers(3, 9)))) % 3) * rng.uniform(1, 9)
            a = base + steps + rng.normal(0, rng.uniform(0, 2), (ph, pw))
            a = a * (1 << (bd - 8))
        out.append(np.ascontiguousarray(np.clip(np.rint(a), 0, mx).astype(dt)))
    return out


def origin(arr, p, xdec, ydec):
    """Pointer to pixel (0, 0) of a padded plane array."""
    return arr.ctypes.data + ((PAD >> (ydec if p else 0)) * arr.shape[1] + (PAD >> (xdec if p else 0))) * arr.itemsize


def state_array(deltas_enabled=0, ref_deltas=(0,) * 8, mode_deltas=(0, 0), block=0, shift=0, multi=0):
    s = np.zeros(1, B.DEBLOCK_STATE_DTYPE)
    s["deltas_enabled"], s["ref_deltas"], s["mode_deltas"] = deltas_enabled, ref_deltas, mode_deltas
    s["block_deltas_enabled"], s["block_delta_shift"], s["block_delta_multi"] = block, shift, multi
    return s


def items_array(items):
    return np.ascontiguousarray(np.asarray(items, np.int32).reshape(-1, 6))


def orc_filter(planes_arr, layout, bd, state, levels, grid, items):
    """orc_deblock_filter in place over padded numpy planes."""
    L = O.lib()
    f = L.orc_deblock_filter
    f.restype = None
    n, xdec, ydec = LAYOUTS[layout]
    vpa, spa = C.c_void_p * 3, C.c_ssize_t * 3
    it = items_array(items)
    lv = np.ascontiguousarray(np.asarray(levels, np.uint8).reshape(-1, 4))
    f(vpa(*[origin(a, p, xdec, ydec) for p, a in enumerate(planes_arr)]), spa(*[a.shape[1] for a in planes_arr]),
      C.c_int(planes_arr[0].itemsize), C.c_int(n), C.c_int(xdec), C.c_int(ydec), C.c_int(bd),
      C.c_void_p(state.ctypes.data), C.c_void_p(lv.ctypes.data), C.c_void_p(grid.ctypes.data),
      C.c_ssize_t(grid.shape[1]), C.c_void_p(it.ctypes.data), C.c_size_t(len(it)))


def working_rect(item, p, xdec, ydec):
    """The plane-p rect (x0, y0, x1, y1), in plane pixels of the frame, that the filter owns for an item."""
    mx, my, mw, mh, vw, vh = item
    xd, yd = (xdec, ydec) if p else (0, 0)
    w, h = min(mw * 4, (vw + 7) & ~7), min(mh * 4, (vh + 7) & ~7)
    return (mx * 4) >> xd, (my * 4) >> yd, ((mx * 4) >> xd) + (w >> xd), ((my * 4) >> yd) + (h >> yd)


# ---------------------------------------------------------------- the specification's processes
def thresholds(lvl, bd):
    """7.14.4 with loop_filter_sharpness 0: (limitBd, blimitBd, threshBd)."""
    shift = 0
    limit = np.maximum(1, lvl >> shift)
    blimit = 2 * (lvl + 2) + limit
    thresh = lvl >> 4
    return limit << (bd - 8), blimit << (bd - 8), thresh << (bd - 8)


def filter4_clamp(x, bd):
    return np.clip(x, -(1 << (bd - 1)), (1 << (bd - 1)) - 1)


def sample_filter(F, fsize, plane, lvl, bd):
    """7.14.6: F is (N, 14) with columns p6 .. p0 q0 .. q6; fsize the filter size process's output (4, 8, 16
    luma; 4, 8 chroma).  Returns the filtered lines (N, 14)."""
    F = F.astype(np.int64)
    lvl = np.asarray(lvl, np.int64)
    p = [F[:, 6 - k] for k in range(7)]
    q = [F[:, 7 + k] for k in range(7)]
    limitBd, blimitBd, threshBd = thresholds(lvl, bd)
    one = 1 << (bd - 8)
    flen = 4 if fsize == 4 else 6 if plane else fsize if fsize == 8 else 16
    hev = (abs(p[1] - p[0]) > threshBd) | (abs(q[1] - q[0]) > threshBd)
    mask = (abs(p[1] - p[0]) <= limitBd) & (abs(q[1] - q[0]) <= limitBd) & \
           (abs(p[0] - q[0]) * 2 + abs(p[1] - q[1]) // 2 <= blimitBd)
    if flen >= 6:
        mask &= (abs(p[2] - p[1]) <= limitBd) & (abs(q[2] - q[1]) <= limitBd)
    if flen >= 8:
        mask &= (abs(p[3] - p[2]) <= limitBd) & (abs(q[3] - q[2]) <= limitBd)
    flat = np.zeros_like(mask)
    if flen >= 6:
        flat = (abs(p[1] - p[0]) <= one) & (abs(q[1] - q[0]) <= one) & (abs(p[2] - p[0]) <= one) & \
               (abs(q[2] - q[0]) <= one)
    if flen >= 8:
        flat &= (abs(p[3] - p[0]) <= one) & (abs(q[3] - q[0]) <= one)
    flat2 = np.zeros_like(mask)
    if flen == 16:
        flat2 = np.ones_like(mask)
        for k in (4, 5, 6):
            flat2 &= (abs(p[k] - p[0]) <= one) & (abs(q[k] - q[0]) <= one)
    out = F.copy()
    # narrow filter process (7.14.6.3)
    nar = mask & ((fsize == 4) | ~flat)
    off = 0x80 << (bd - 8)
    ps1, ps0, qs0, qs1 = p[1] - off, p[0] - off, q[0] - off, q[1] - off
    f = np.where(hev, filter4_clamp(ps1 - qs1, bd), 0)
    f = filter4_clamp(f + 3 * (qs0 - ps0), bd)
    f1 = filter4_clamp(f + 4, bd) >> 3
    f2 = filter4_clamp(f + 3, bd) >> 3
    oq0 = filter4_clamp(qs0 - f1, bd) + off
    op0 = filter4_clamp(ps0 + f2, bd) + off
    fr = (f1 + 1) >> 1
    oq1 = np.where(hev, q[1], filter4_clamp(qs1 - fr, bd) + off)
    op1 = np.where(hev, p[1], filter4_clamp(ps1 + fr, bd) + off)
    for col, v in ((5, op1), (6, op0), (7, oq0), (8, oq1)):
        out[:, col] = np.where(nar, v, out[:, col])
    # wide filter process (7.14.6.4)
    for log2, sel in ((3, mask & flat & ((flen != 16) | ~flat2)), (4, mask & flat & flat2 & (flen == 16))):
        if fsize == 4 or not sel.any():
            continue
        n = 6 if log2 == 4 else 3 if plane == 0 else 2
        n2 = 0 if (log2 == 3 and plane == 0) else 1
        Fk = lambda k: q[k] if k >= 0 else p[-k - 1]
        for i in range(-n, n):
            t = 0
            for j in range(-n, n + 1):
                pk = min(max(i + j, -(n + 1)), n)
                t = t + Fk(pk) * (2 if abs(j) <= n2 else 1)
            out[:, 7 + i] = np.where(sel, (t + (1 << (log2 - 1))) >> log2, out[:, 7 + i])
    return out


def chroma_tx_dims(bs, xdec, ydec):
    """get_tx_size for a chroma plane: the chroma block, at least 4x4, each side capped at 32."""
    bw, bh = BSIZE_DIMS[bs]
    return min(max(bw >> xdec, 4), 32), min(max(bh >> ydec, 4), 32)


def filter_level(st, lv, blk, plane, vertical):
    """7.14.4's level for one block: the delta_lf'd base level, then the ref / mode deltas."""
    i = (0 if vertical else 1) if plane == 0 else plane + 1
    base = int(lv[i])
    if st["block_deltas_enabled"]:
        d = int(blk["deltas"][i if st["block_delta_multi"] else 0]) << int(st["block_delta_shift"])
        base = min(max(d + base, 0), 63)
    if not st["deltas_enabled"]:
        return base
    ref, mode = int(blk["ref0"]), int(blk["mode"])
    shift = base >> 5
    if ref == 0:
        return min(max(base + (int(st["ref_deltas"][0]) << shift), 0), 63)
    mode_type = 1 if (mode >= 14 and mode not in (18, 32)) else 0     # NEARESTMV .. except GLOBALMV, GLOBAL_GLOBALMV
    return min(max(base + (int(st["ref_deltas"][ref]) << shift) + (int(st["mode_deltas"][mode_type]) << shift),
                   0), 63)


def edge_decision(grid, item, plane, xdec, ydec, x, y, vertical, size_from_width=None):
    """(filter size per the filter size process, current block, previous block) for the 4x4 edge at
    item-relative luma mi (x, y), or None.  size_from_width overrides the direction the size is read in."""
    mx, my = item[0], item[1]
    xd, yd = (xdec, ydec) if plane else (0, 0)
    blk = grid[my + y, mx + x]
    prev = grid[my + (y | yd), mx + (x | xd) - (1 << xd)] if vertical else grid[my + (y | yd) - (1 << yd), mx + (x | xd)]

    def txd(b):
        return TX_DIMS[int(b["txsize"])] if plane == 0 else chroma_tx_dims(int(b["bsize"]), xd, yd)
    tw, th = txd(blk)
    pos = ((x * 4) >> xd) if vertical else ((y * 4) >> yd)
    if pos % (tw if vertical else th):
        return None
    bw, bh = BSIZE_DIMS[int(blk["bsize"])]
    block_edge = (x * 4) % bw == 0 if vertical else (y * 4) % bh == 0
    skip_inter = lambda b: bool(b["skip"]) and int(b["ref0"]) != 0
    if not (block_edge or not skip_inter(blk) or not skip_inter(prev)):
        return None
    ptw, pth = txd(prev)
    by_w = vertical if size_from_width is None else size_from_width
    base = min(tw, ptw) if by_w else min(th, pth)
    fsize = min(16, base) if plane == 0 else min(8, base)
    return fsize, blk, prev


def extent(mi_n, vis, dec):
    return (min(mi_n, (vis + 3) >> 2) + (1 << dec >> 1)) >> dec << dec


def edge_positions(item, plane, xdec, ydec, vertical):
    xd, yd = (xdec, ydec) if plane else (0, 0)
    cols, rows = extent(item[2], item[4], xd), extent(item[3], item[5], yd)
    return [(x, y) for y in range(0, rows, 1 << yd) for x in range(0, cols, 1 << xd)
            if (x > 0 if vertical else y > 0)]


def gather(img, ox, oy, px, py, vertical, lines=4):
    """(lines, 14) taps p6 .. q6 of the edge at plane pixel (px, py) of the item, from `img` (plane array with
    the item origin at (ox, oy) in array coordinates)."""
    if vertical:
        return np.stack([img[oy + py + i, ox + px - 7: ox + px + 7] for i in range(lines)]).astype(np.int64)
    return np.stack([img[oy + py - 7: oy + py + 7, ox + px + i] for i in range(lines)]).astype(np.int64)


def spec_filter(planes_arr, layout, bd, st, levels, grid, items):
    """The specification's two passes per plane per item, each pass computed from the picture as it was when
    the pass began; returns filtered copies."""
    n, xdec, ydec = LAYOUTS[layout]
    out = [a.copy() for a in planes_arr]
    for k, it in enumerate(items):
        lv = levels[k]
        if lv[0] == 0 and lv[1] == 0:
            continue
        for p in range(n):
            if p and lv[p + 1] == 0:
                continue
            xd, yd = (xdec, ydec) if p else (0, 0)
            ox, oy = (PAD >> xd) + ((it[0] * 4) >> xd), (PAD >> yd) + ((it[1] * 4) >> yd)
            for vertical in (True, False):
                snap = out[p].copy()
                written = np.zeros(snap.shape, np.int32)
                for x, y in edge_positions(it, p, xdec, ydec, vertical):
                    d = edge_decision(grid, it, p, xdec, ydec, x, y, vertical)
                    if d is None:
                        continue
                    fsize, blk, prev = d
                    lvl = filter_level(st, lv, blk, p, vertical) or filter_level(st, lv, prev, p, vertical)
                    if lvl == 0:
                        continue
                    px, py = (x * 4) >> xd, (y * 4) >> yd
                    F = gather(snap, ox, oy, px, py, vertical)
                    G = sample_filter(F, fsize, p, np.full(4, lvl), bd)
                    reach = 6 if (p == 0 and fsize == 16) else 3 if (p == 0 and fsize == 8) else 2
                    for i in range(4):
                        for t in range(7 - reach, 7 + reach):
                            yy, xx = (oy + py + i, ox + px - 7 + t) if vertical else (oy + py - 7 + t, ox + px + i)
                            written[yy, xx] += 1
                            out[p][yy, xx] = G[i, t]
                assert written.max() <= 1, "two edges of one pass touch the same pixel"
    return out


# ---------------------------------------------------------------- tests
def run_case(rng, layout, bd, W, H, items, levels, st, content="random", deltas=False, skip_p=0.4):
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    grid = random_grid(rng, w4, h4, layout, skip_p=skip_p, deltas=deltas)
    planes = make_planes(rng, W, H, layout, bd, content)
    want = spec_filter(planes, layout, bd, st[0], levels, grid, items)
    got = [a.copy() for a in planes]
    orc_filter(got, layout, bd, st, levels, grid, items)
    for p in range(len(planes)):
        assert (got[p] == want[p]).all(), f"plane {p}: {np.argwhere(got[p] != want[p])[:5]}"
    return planes, got


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("bd", [8, 10, 12])
@pytest.mark.parametrize("content", ["random", "steps", "flat"])
def test_frame_matches_the_specification(layout, bd, content):
    rng = np.random.default_rng(zlib.crc32(f"{layout}{bd}{content}".encode()))
    W, H = 76, 58                                    # not multiples of 8: partial blocks at the right and bottom
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    levels = [[int(v) for v in rng.integers(1, 64, 4)]]
    planes, got = run_case(rng, layout, bd, W, H, [(0, 0, w4, h4, W, H)], levels, state_array(), content)
    if content == "steps":
        assert any((g != p).any() for g, p in zip(got, planes)), "nothing was filtered"


@pytest.mark.parametrize("layout", ["420", "422", "444"])
def test_every_level_with_deltas(layout):
    """Every level 0..63 on each of the four slots, with ref / mode deltas and block deltas (multi and single)."""
    rng = np.random.default_rng(7)
    W, H = 48, 32
    w4, h4 = 24, 16
    for lvl in range(64):
        st = state_array(1, [int(v) for v in rng.integers(-16, 16, 8)], [int(v) for v in rng.integers(-16, 16, 2)],
                         block=int(lvl % 3 != 0), shift=lvl % 4, multi=lvl & 1)
        levels = [[lvl, (lvl * 7) % 64, (lvl * 13) % 64, 63 - lvl]]
        run_case(rng, layout, [8, 10, 12][lvl % 3], W, H, [(0, 0, w4, h4, W, H)], levels, st, "steps", deltas=True)


@pytest.mark.parametrize("layout", ["420", "444"])
def test_tile_and_area_items_off_the_origin(layout):
    """Items off the origin: nothing is filtered across their left or top border, and each keeps its own
    visible size; the chroma-only gate and the both-luma-zero gate."""
    rng = np.random.default_rng(11)
    W, H = 200, 140
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    items = [(0, 0, 32, 16, W, H), (32, 0, w4 - 32, 16, W - 128, H), (0, 16, 16, h4 - 16, W, H - 64),
             (16, 16, w4 - 16, h4 - 16, W - 64, H - 64)]
    levels = [[20, 30, 10, 40], [0, 0, 30, 30], [5, 0, 0, 63], [63, 63, 63, 0]]
    run_case(rng, layout, 10, W, H, items, levels, state_array(), "steps")


def test_skip_inter_switches_interior_edges_off():
    """All blocks skip and inter: only block edges are filtered; the same grid with intra blocks filters the
    transform edges inside blocks as well."""
    rng = np.random.default_rng(3)
    W, H = 64, 64
    item = [(0, 0, 16, 16, W, H)]
    grid = random_grid(rng, 16, 16, "444", skip_p=1.0, intra_p=0.0)
    planes = make_planes(rng, W, H, "444", 8, "steps")
    inter = [a.copy() for a in planes]
    orc_filter(inter, "444", 8, state_array(), [[40, 40, 40, 40]], grid, item)
    want = spec_filter(planes, "444", 8, state_array()[0], [[40, 40, 40, 40]], grid, item)
    assert all((a == b).all() for a, b in zip(inter, want))
    grid["ref0"] = 0
    intra = [a.copy() for a in planes]
    orc_filter(intra, "444", 8, state_array(), [[40, 40, 40, 40]], grid, item)
    want = spec_filter(planes, "444", 8, state_array()[0], [[40, 40, 40, 40]], grid, item)
    assert all((a == b).all() for a, b in zip(intra, want))
    assert any((a != b).any() for a, b in zip(inter, intra))
