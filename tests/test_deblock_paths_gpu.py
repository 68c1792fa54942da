"""Deblocking on every kernel path, bit exact against the oracle (orc_deblock_levels / orc_deblock_filter), with
the coverage of each section counted by the specification model of tests/test_oracle_deblock_spec.py.

The kernels (deblock.cu):
- `deblock_sse_kernel<T>`: the level search, one 256-thread CTA per (64x64 luma tile of an item, plane); each
  edge segment adds its SSE deltas to i64 tallies in shared memory, flushed with 64-bit atomics into a
  per-item scratch row at `item0 + k`;
- `deblock_levels_finish_kernel`: one thread per item, prefix sums and the first minimum;
- `deblock_filter_kernel<T>`: the filter, one CTA per (64x64 luma tile, plane), the tile plus a 7-pixel halo
  staged in shared memory, all vertical edges, a barrier, all horizontal edges.
The launch geometry mirrored here:
- deblock.cu:25   kDbMaxItems = 160: an item list is cut every 160 items, each launch with its own `item0`;
- deblock.cu:664  the level search may read 4 rows (4 >> ydec in chroma) above and below each working rect;
- deblock.cu:703  the filter reads and writes the working rect only;
- deblock.cu:691  the level search adds one finish launch after its item launches.
The sections:
1. every filter class (none, narrow2, narrow4, wide6, wide8, wide14) of every edge size (luma 4 / 8 / 14,
   chroma 4 / 6) on lines built at the mask, hev, flat and flat2 thresholds, with lines pinned at 0 and at the
   maximum so the narrow filter's pixel and range clamps fire: the level search, the filter at the searched
   levels and at levels 1, 20, 32 and 63, every layout at 8 / 10 / 12 bit;
2. item lists past 160: one item per superblock of a 1080p frame, a mixed list whose launch boundary falls
   inside a superblock row, exactly 160 and 161 items; launch counts;
3. read footprints: everything outside what each call may read replaced between two runs, visible sizes at
   every remainder mod 8, and the three rows above an item that the by-width 14-tap search reads;
4. caller-built planes: a different stride, pad and base alignment for every plane of rec / src / in / out,
   garbage in the padding, an mi grid wider than the frame with random padding bytes;
5. ref / mode / block deltas at their limits: the i8 wrap of the block delta and the previous-block fallback;
6. tallies past 2^32 at 12-bit 4:4:4 1080p, as one item and as 200.
Every section asserts that it reached what it claims from the oracle's and the model's own numbers."""
import collections
import math
import zlib

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_deblock_gpu import DevPlanes, frame_setup, run_both
from tests.test_oracle_deblock import orc_levels
from tests.test_oracle_deblock_spec import (BSIZE_DIMS, LAYOUTS, PAD, edge_decision, edge_positions, filter4_clamp,
                                            make_planes, orc_filter, random_grid, sample_filter, state_array,
                                            thresholds, working_rect)

pytestmark = pytest.mark.gpu

BDS = [8, 10, 12]
ITEMS_PER_LAUNCH = 160      # deblock.cu:25   kDbMaxItems
SEARCH_MARGIN = 4           # deblock.cu:664  rows above / below a working rect the level search may read
FIXED_LEVELS = [1, 20, 32, 63]
MIN_LINES = 32
NONE, NARROW2, NARROW4, WIDE6, WIDE8, WIDE14 = range(6)
CLASS_NAMES = ["none", "narrow2", "narrow4", "wide6", "wide8", "wide14"]
# the classes an edge of each (plane kind, taps) can take
REACHABLE = {("luma", 4): (NONE, NARROW2, NARROW4), ("luma", 8): (NONE, NARROW2, NARROW4, WIDE8),
             ("luma", 14): (NONE, NARROW2, NARROW4, WIDE8, WIDE14),
             ("chroma", 4): (NONE, NARROW2, NARROW4), ("chroma", 6): (NONE, NARROW2, NARROW4, WIDE6)}


def seed(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def taps_of(fsize, plane):
    """The specification's filter size (4 / 8 / 16 luma, 4 / 8 chroma) as the device's tap count."""
    return {4: 4, 8: 6 if plane else 8, 16: 14}[fsize]


def plane_kind(p):
    return "chroma" if p else "luma"


# ---------------------------------------------------------------- the specification's decisions per line
def line_class(F, fsize, plane, lvl, bd):
    """The filter class of each (N, 14) line p6 .. q6 at levels lvl (N,) by the mask, hev, flat and flat2
    processes (7.14.6.2), and for narrow lines whether filter4_clamp's signed range or the pixel range cut a
    value: (class, range clamp, pixel clamp)."""
    F = F.astype(np.int64)
    lvl = np.broadcast_to(np.asarray(lvl, np.int64), (len(F),))
    p = [F[:, 6 - k] for k in range(7)]
    q = [F[:, 7 + k] for k in range(7)]
    limitBd, blimitBd, threshBd = thresholds(lvl, bd)
    one = 1 << (bd - 8)
    flen = 4 if fsize == 4 else 6 if plane else fsize if fsize == 8 else 16
    hev = (abs(p[1] - p[0]) > threshBd) | (abs(q[1] - q[0]) > threshBd)
    mask = (abs(p[1] - p[0]) <= limitBd) & (abs(q[1] - q[0]) <= limitBd) & \
           (abs(p[0] - q[0]) * 2 + abs(p[1] - q[1]) // 2 <= blimitBd) & (lvl > 0)
    for k in range(2, {4: 1, 6: 2, 8: 3, 16: 3}[flen] + 1):
        mask &= (abs(p[k] - p[k - 1]) <= limitBd) & (abs(q[k] - q[k - 1]) <= limitBd)
    flat = np.zeros_like(mask)
    if flen >= 6:
        flat = np.ones_like(mask)
        for k in range(1, 3 if flen == 6 else 4):
            flat &= (abs(p[k] - p[0]) <= one) & (abs(q[k] - q[0]) <= one)
    flat2 = np.zeros_like(mask)
    if flen == 16:
        flat2 = np.ones_like(mask)
        for k in (4, 5, 6):
            flat2 &= (abs(p[k] - p[0]) <= one) & (abs(q[k] - q[0]) <= one)
    wide = WIDE6 if flen == 6 else WIDE8
    cls = np.where(flat, np.where(flat2, WIDE14, wide), np.where(hev, NARROW2, NARROW4))
    cls = np.where(mask, cls, NONE)
    # the narrow filter (7.14.6.3) with every clamp checked
    off, lo, hi = 0x80 << (bd - 8), -(1 << (bd - 1)), (1 << (bd - 1)) - 1
    out = lambda v: (v < lo) | (v > hi)
    ps1, ps0, qs0, qs1 = p[1] - off, p[0] - off, q[0] - off, q[1] - off
    f0 = np.where(hev, ps1 - qs1, 0)
    f = filter4_clamp(f0, bd) + 3 * (qs0 - ps0)
    fc = filter4_clamp(f, bd)
    rng_clamp = out(f0) | out(f) | out(fc + 4) | out(fc + 3)
    f1, f2 = filter4_clamp(fc + 4, bd) >> 3, filter4_clamp(fc + 3, bd) >> 3
    fr = (f1 + 1) >> 1
    px_clamp = out(qs0 - f1) | out(ps0 + f2) | (~hev & (out(ps1 + fr) | out(qs1 - fr)))
    nar = (cls == NARROW2) | (cls == NARROW4)
    return cls, nar & rng_clamp, nar & px_clamp


def mask_level(F, fsize, plane, bd):
    """The smallest level 1..63 at which each line is filtered, 64 when none is."""
    out = np.full(len(F), 64)
    for L in range(63, 0, -1):
        cls, _, _ = line_class(F, fsize, plane, L, bd)
        out[cls != NONE] = L
    return out


def edge_table(grid, item, p, xdec, ydec, vertical, by_width=None):
    """Every filtered edge of one direction of an item's plane: (plane-pixel positions (n, 2), specification
    sizes (n,), [(block, previous block)])."""
    xd, yd = (xdec, ydec) if p else (0, 0)
    pos, fs, blocks = [], [], []
    for x, y in edge_positions(item, p, xdec, ydec, vertical):
        d = edge_decision(grid, item, p, xdec, ydec, x, y, vertical, size_from_width=by_width)
        if d is not None:
            pos.append(((x * 4) >> xd, (y * 4) >> yd))
            fs.append(d[0])
            blocks.append((d[1], d[2]))
    return np.asarray(pos, np.int64).reshape(-1, 2), np.asarray(fs, np.int64), blocks


def line_index(pos, ox, oy, vertical):
    """Array indices (4n, 14) of the taps p6 .. q6 of every line of the edges at `pos`, item origin (ox, oy)."""
    i, t = np.arange(4)[None, :, None], np.arange(-7, 7)[None, None, :]
    x, y = pos[:, 0, None, None] + ox, pos[:, 1, None, None] + oy
    if vertical:
        rows, cols = y + i + 0 * t, x + t + 0 * i
    else:
        rows, cols = y + t + 0 * i, x + i + 0 * t
    return rows.reshape(-1, 14), cols.reshape(-1, 14)


def vertical_pass(img, ox, oy, pos, fs, lvls, p, bd):
    """The specification's vertical pass over one plane (every edge from the unfiltered picture; no pixel is
    written twice, tests/test_oracle_deblock_spec.py)."""
    out = img.copy()
    for f in np.unique(fs):
        sel = (fs == f) & (lvls > 0)
        if not sel.any():
            continue
        rows, cols = line_index(pos[sel], ox, oy, True)
        G_ = sample_filter(img[rows, cols], int(f), p, np.repeat(lvls[sel], 4), bd)
        out[rows, cols] = G_
    return out


# ---------------------------------------------------------------- 1. every filter class at its thresholds
GRIDS = {16: 2, 8: 1, 4: 0}      # uniform grids: block side (px) -> the square TxSize of that side


def uniform_grid(w4, h4, side):
    g = np.zeros((h4, w4), B.DEBLOCK_MI_DTYPE)
    g["bsize"], g["txsize"] = BSIZE_DIMS.index((side, side)), GRIDS[side]
    return g                      # intra, not skipped: every transform edge is filtered


def spacing(side, p, dec):
    """(edge spacing, taps) of one direction of plane p on a uniform grid of side x side blocks."""
    if p == 0:
        return side, {16: 14, 8: 8, 4: 4}[side]
    P = max(4, side >> dec)
    return P, 6 if P >= 8 else 4


def line_pool(N, h, bd, plane):
    """Lines of 2h pixels (p_{h-1} .. p0 q0 .. q_{h-1}) whose N-tap edge lands on a threshold: flat and flat2 at
    one step and one past (1 << shift, +1), hev at and past each 16-level boundary, limit-driven masks, and
    steps that put the mask on 0..2, 19..21, 31..33 and 62..64; plus lines pinned at 0 or the maximum and
    spikes that drive the narrow filter's clamps."""
    fl, mx, mid = 1 << (bd - 8), (1 << bd) - 1, 1 << (bd - 1)
    fsize = {4: 4, 6: 8, 8: 8, 14: 16}[N]
    z = [0] * 8
    fams = [(z, z), ([0, 0, fl, 0, fl, fl, 0, fl], [0, fl, 0, fl, 0, 0, fl, 0]),
            ([0, 0, 0, 0, fl + 1, 0, 0, 0], z), (z, [0, 0, 0, 0, 0, 0, fl + 1, fl + 1]),
            ([0, fl, fl, fl, fl, fl, fl, fl], z), ([0, 0, 0, fl + 1] + [fl + 1] * 4, z),
            ([0, 0, fl + 1] + [fl + 1] * 5, z), ([0, fl + 1] + [fl + 1] * 6, z)]
    for j in (fl, 2 * fl, 2 * fl + 1, 3 * fl, 3 * fl + 1, 4 * fl, 5 * fl):
        fams.append(([0] + [j] * 7, [0] + [-j] * 7))
    inner = {4: 1, 6: 2, 8: 3, 14: 3}[N]          # the tap whose step alone sets the limit part of the mask
    for t in (1, 2, 19, 20, 21, 31, 32, 33, 62, 63, 64):
        for m in (t * fl, t * fl - fl + 1):
            fams.append(([0] * inner + [m] * (8 - inner), z))
    targets = (0, 1, 2, 3, 19, 20, 21, 31, 32, 33, 47, 48, 49, 62, 63, 64)
    lines = []

    def line(po, qo, d, base=mid):
        return np.array([base + po[i] for i in range(h - 1, -1, -1)] + [base + d + qo[i] for i in range(h)])

    def as14(L):
        return np.concatenate([np.full(7 - h, L[0]), L, np.full(7 - h, L[-1])]) if h < 7 else L[h - 7:h + 7]

    ds = np.arange(0, 100 * fl)
    for po, qo in fams:
        cand = np.stack([as14(line(po, qo, int(d))) for d in ds])
        ml = mask_level(cand, fsize, plane, bd)
        for t in targets:
            hit = np.flatnonzero(ml >= t)
            if len(hit):
                d = int(ds[hit[0]])
                lines += [line(po, qo, d), line(po, qo, -d), line([-v for v in po], [-v for v in qo], -d)]
    for S in (8 * fl, 32 * fl, 63 * fl):
        for D in (fl, 4 * fl, 12 * fl):              # q side pinned at 0, a hev spike at p1: q0 - f1 clamps
            lo = np.array([D + S] * (h - 1) + [D] + [0] * h)
            lines += [lo, mx - lo, lo[::-1], mx - lo[::-1]]
    for S in (40 * fl, 63 * fl):
        for D in (2 * fl, 20 * fl, 40 * fl):         # |p1 - q1| past 128 << shift: filter4_clamp's range
            r = np.array([mid + S] * (h - 1) + [mid, mid - D] + [mid - D - S] * (h - 1))
            lines += [r, r[::-1]]
    for D in (2 * fl, 3 * fl):                       # narrow4 at the maximum: p1 + f3 clamps
        r = np.array([mx] * (h - 1) + [mx - D, mx, mx - fl] + [mx - fl] * (h - 2))
        lines += [r, mx - r]
    return np.clip(np.stack(lines), 0, mx)


def designed_plane(rng, pw, ph, v, hz, mx):
    """Rows of the top half built of pool lines around each vertical edge, columns of the bottom half around
    each horizontal edge; v / hz = (edge spacing, pool)."""
    img = np.zeros((ph, pw), np.int64)
    top = ph // 2
    (Pv, pool_v), (Ph, pool_h) = v, hz
    pick = pool_v[rng.integers(0, len(pool_v), (top, pw // Pv + 1))].reshape(top, -1)
    img[:top] = pick[:, Pv // 2:Pv // 2 + pw]
    pick = pool_h[rng.integers(0, len(pool_h), (pw, (ph - top) // Ph + 1))].reshape(pw, -1)
    img[top:] = pick[:, Ph // 2:Ph // 2 + ph - top].T
    return np.clip(img, 0, mx)


def count_lines(counts, stage, planes, layout, bd, grid, item, lv, by_width):
    """Adds every filtered line of the item to counts[(stage, plane kind, taps, class)]; lv = the four levels
    (the level search is counted at level 63).  The horizontal lines of the filter are read after the
    specification's vertical pass."""
    n, xdec, ydec = LAYOUTS[layout]
    for p in range(n):
        xd, yd = (xdec, ydec) if p else (0, 0)
        ox, oy = PAD >> xd, PAD >> yd
        img = planes[p].astype(np.int64)
        for vertical in (True, False):
            pos, fs, _ = edge_table(grid, item, p, xdec, ydec, vertical, by_width)
            level = lv[(0 if vertical else 1) if p == 0 else p + 1]
            if level == 0 or not len(pos):
                continue
            for f in np.unique(fs):
                rows, cols = line_index(pos[fs == f], ox, oy, vertical)
                cls, rc, pc = line_class(img[rows, cols], int(f), p, level, bd)
                key = (stage, plane_kind(p), taps_of(int(f), p))
                for c in np.unique(cls):
                    counts[key + (int(c),)] += int((cls == c).sum())
                counts[(stage, "range clamp")] += int(rc.sum())
                counts[(stage, "pixel clamp")] += int(pc.sum())
            if vertical and stage == "filter":
                img = vertical_pass(img, ox, oy, pos, fs, np.full(len(pos), level), p, bd)


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("bd", BDS)
def test_every_filter_class_at_its_thresholds(layout, bd):
    n, xdec, ydec = LAYOUTS[layout]
    W, H = 256, 128
    w4, h4 = W // 4, H // 4
    item = (0, 0, w4, h4, W, H)
    mx, fl = (1 << bd) - 1, 1 << (bd - 8)
    rng = seed("classes", layout, bd)
    counts = collections.Counter()
    for side in GRIDS:
        grid = uniform_grid(w4, h4, side)
        rec, src = [], []
        for p in range(n):
            xd, yd = (xdec, ydec) if p else (0, 0)
            (Pv, Nv), (Ph, Nh) = spacing(side, p, xd), spacing(side, p, yd)
            pools = {(P, N): line_pool(N, P // 2, bd, p) for P, N in {(Pv, Nv), (Ph, Nh)}}
            img = designed_plane(rng, W >> xd, H >> yd, (Pv, pools[(Pv, Nv)]), (Ph, pools[(Ph, Nh)]), mx)
            pad = ((PAD >> yd,) * 2, (PAD >> xd,) * 2)
            dt = np.uint8 if bd == 8 else np.uint16
            rec.append(np.pad(img, pad, mode="edge").astype(dt))
            s = img + rng.integers(-3, 4, img.shape) * fl
            src.append(np.pad(np.clip(s, 0, mx), pad, mode="edge").astype(dt))
        lv, _ = run_both(rng, layout, bd, grid, src, rec, [item], state_array())
        count_lines(counts, "search", rec, layout, bd, grid, item, [63] * 4, True)
        count_lines(counts, "filter", rec, layout, bd, grid, item, lv[0], None)
        for L in FIXED_LEVELS:
            run_both(rng, layout, bd, grid, src, rec, [item], state_array(), [[L] * 4])
            count_lines(counts, "filter", rec, layout, bd, grid, item, [L] * 4, None)
    print(f"\n{layout} {bd}-bit:", {f"{k[0]} {k[1]}{k[2]} {CLASS_NAMES[k[3]]}" if len(k) == 4 else " ".join(k): v
                                    for k, v in sorted(counts.items(), key=str)})
    for stage in ("search", "filter"):
        for (kind, taps), classes in REACHABLE.items():
            if kind == "chroma" and n == 1:
                continue
            for c in classes:
                got = counts[(stage, kind, taps, c)]
                assert got >= MIN_LINES, f"{stage}: {kind} {taps}-tap {CLASS_NAMES[c]} on {got} lines"
    for what in ("range clamp", "pixel clamp"):
        assert counts[("filter", what)] >= MIN_LINES, (what, counts[("filter", what)])


# ---------------------------------------------------------------- device runs with the launch counts
def dev_levels(c, rec_v, src_v, xdec, ydec, bd, d_mi, ms, items):
    n = len(items)
    d_lv = G.to_dev(np.full(n * 4, 0xAA, np.uint8))
    d_t = G.to_dev(np.full(n * 3 * 2 * 64, 7, np.int64))
    before = c.launches
    c.deblock_levels_dev(rec_v, src_v, xdec, ydec, bd, d_mi, ms, items, d_lv, d_t)
    c.synchronize()
    return (G.from_dev(d_lv, np.uint8).reshape(n, 4), G.from_dev(d_t, np.int64).reshape(n, 3, 2, 64),
            c.launches - before)


def dev_filter(c, in_v, out_v, xdec, ydec, bd, st, levels, d_mi, ms, items):
    d_lv = G.to_dev(np.ascontiguousarray(levels, np.uint8).reshape(-1))
    before = c.launches
    c.deblock_filter_dev(in_v, out_v, xdec, ydec, bd, st, d_lv, d_mi, ms, items)
    c.synchronize()
    return c.launches - before


def filtered_expectation(rec, garbage, layout, bd, st, levels, grid, items):
    """The oracle's filtered planes inside each working rect, `garbage` everywhere else."""
    _, xdec, ydec = LAYOUTS[layout]
    filt = [a.copy() for a in rec]
    orc_filter(filt, layout, bd, st, levels, grid, items)
    want = [g.copy() for g in garbage]
    for p in range(len(rec)):
        xo, yo = PAD >> (xdec if p else 0), PAD >> (ydec if p else 0)
        for it in items:
            x0, y0, x1, y1 = working_rect(it, p, xdec, ydec)
            want[p][yo + y0:yo + y1, xo + x0:xo + x1] = filt[p][yo + y0:yo + y1, xo + x0:xo + x1]
    return want


def run_counted(rng, layout, bd, grid, src, rec, items, st=None):
    """Levels and filter on the device against the oracle; returns (levels, tallies, filter output,
    level-search launches, filter launches)."""
    st = state_array() if st is None else st
    _, xdec, ydec = LAYOUTS[layout]
    c = G.ctx()
    d_rec, d_src = DevPlanes(c, rec, layout), DevPlanes(c, src, layout)
    garbage = [rng.integers(0, 1 << bd, a.shape).astype(a.dtype) for a in rec]
    d_out = DevPlanes(c, garbage, layout)
    d_mi = G.to_dev(grid.view(np.uint8).reshape(-1))
    ms = grid.shape[1]
    lv, t, n_lv = dev_levels(c, d_rec.views, d_src.views, xdec, ydec, bd, d_mi, ms, items)
    want_lv, want_t = orc_levels(rec, src, layout, bd, grid, items)
    assert (t == want_t).all(), np.argwhere(t != want_t)[:5]
    assert (lv == want_lv).all(), np.argwhere(lv != want_lv)[:5]
    n_f = dev_filter(c, d_rec.views, d_out.views, xdec, ydec, bd, st, lv, d_mi, ms, items)
    got = d_out.download()
    want = filtered_expectation(rec, garbage, layout, bd, st, lv, grid, items)
    for p in range(len(rec)):
        assert (got[p] == want[p]).all(), f"plane {p}: {np.argwhere(got[p] != want[p])[:5]}"
    for dp in (d_rec, d_src, d_out):
        dp.free()
    return lv, t, got, n_lv, n_f


# ---------------------------------------------------------------- 2. item lists past 160
def sb_item(sx, sy, sw, sh, W, H):
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    return (sx * 16, sy * 16, min(sw * 16, w4 - sx * 16), min(sh * 16, h4 - sy * 16), W - sx * 64, H - sy * 64)


def check_launches(n, n_lv, n_f):
    groups = math.ceil(n / ITEMS_PER_LAUNCH)
    assert (n_lv, n_f) == (groups + 1, groups), (n, n_lv, n_f)


def test_one_item_per_superblock_of_a_1080p_frame_shuffled():
    rng = seed("sb items")
    W, H = 1920, 1080
    grid, src, rec = frame_setup(rng, "420", 8, W, H, skip_p=0.5)
    items = [sb_item(sx, sy, 1, 1, W, H) for sy in range(17) for sx in range(30)]
    items = [items[k] for k in rng.permutation(len(items))]
    assert len(items) == 510
    lv, t, _, n_lv, n_f = run_counted(rng, "420", 8, grid, src, rec, items)
    check_launches(len(items), n_lv, n_f)
    assert len({tuple(r) for r in lv}) > 10, "the items' levels hardly differ"


def test_mixed_item_sizes_with_a_launch_boundary_inside_a_superblock_row():
    rng = seed("mixed items")
    W, H = 1920, 1080
    grid, src, rec = frame_setup(rng, "420", 10, W, H)
    items = [sb_item(sx, 0, 3, 3, W, H) for sx in range(0, 30, 3)]
    for sy in range(3, 17):
        sx, k = 0, sy
        while sx < 30:
            sw = min(1 + (k & 1), 30 - sx)
            items.append(sb_item(sx, sy, sw, 1, W, H))
            sx, k = sx + sw, k + 1
    b = ITEMS_PER_LAUNCH
    assert len(items) > b and items[b - 1][1] == items[b][1], "the launch boundary is not inside a superblock row"
    assert {(it[2], it[3]) for it in items[10:]} >= {(16, 16), (32, 16)}
    _, _, _, n_lv, n_f = run_counted(rng, "420", 10, grid, src, rec, items)
    check_launches(len(items), n_lv, n_f)


@pytest.mark.parametrize("n", [ITEMS_PER_LAUNCH, ITEMS_PER_LAUNCH + 1])
def test_item_counts_at_the_launch_limit(n):
    rng = seed("limit", n)
    W, H = 1920, 1080
    grid, src, rec = frame_setup(rng, "422", 8, W, H)
    all_items = [sb_item(sx, sy, 1, 1, W, H) for sy in range(17) for sx in range(30)]
    items = [all_items[k] for k in sorted(rng.permutation(len(all_items))[:n], reverse=True)]
    _, _, _, n_lv, n_f = run_counted(rng, "422", 8, grid, src, rec, items)
    check_launches(n, n_lv, n_f)


# ---------------------------------------------------------------- 3. read footprints
def strip_grid(rng, w4, h4, layout):
    """16x16 regions of 16x4 blocks with 16x4 transforms, 4x16 with 4x16 (not in 4:2:2) or one 16x16 block; the
    regions in mi rows 16..19 are all 16x4, so the by-width search of the item at mi row 16 reads 3 rows above."""
    g = np.zeros((h4, w4), B.DEBLOCK_MI_DTYPE)
    kinds = [(16, 4, 14), (16, 16, 2)] + ([] if layout == "422" else [(4, 16, 13)])
    for ry in range(0, h4, 4):
        for rx in range(0, w4, 4):
            bw, bh, tx = kinds[0] if ry == 16 else kinds[int(rng.integers(0, len(kinds)))]
            g[ry:ry + 4, rx:rx + 4]["bsize"] = BSIZE_DIMS.index((bw, bh))
            g[ry:ry + 4, rx:rx + 4]["txsize"] = tx
    g["skip"] = rng.random((h4, w4)) < 0.3
    g["ref0"] = rng.integers(0, 8, (h4, w4)) * (rng.random((h4, w4)) < 0.6)
    g["mode"] = np.where(g["ref0"] == 0, 0, 20)
    return g


def outside(shape, rects):
    """Boolean mask of the array positions outside the union of rects (array coordinates)."""
    m = np.ones(shape, bool)
    for x0, y0, x1, y1 in rects:
        m[max(y0, 0):y1, max(x0, 0):x1] = False
    return m


def footprint(items, p, xdec, ydec, margin):
    xd, yd = (xdec, ydec) if p else (0, 0)
    xo, yo = PAD >> xd, PAD >> yd
    return [(xo + x0, yo + y0 - (margin >> yd), xo + x1, yo + y1 + (margin >> yd))
            for x0, y0, x1, y1 in (working_rect(it, p, xdec, ydec) for it in items)]


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_reads_stay_inside_the_promised_footprint(layout):
    n, xdec, ydec = LAYOUTS[layout]
    c = G.ctx()
    reached = 0
    for r in range(1, 8):
        rng = seed("footprint", layout, r)
        bd = BDS[r % 3]
        # visible sizes r and 8 - r past a multiple of 8; a 4:2:2 chroma plane has 8 rows of pad here, which
        # the search margin and the rounding of vis_h up to 8 must fit in: vis_h % 8 in 4..7 there
        W, H = 168 + r, 112 - (r if layout != "422" else 4 - r % 4)
        w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
        grid = strip_grid(rng, w4, h4, layout)
        src = make_planes(rng, W, H, layout, bd, "steps")
        rec = [np.clip(s.astype(np.int64) + rng.integers(-5, 6, s.shape) * (1 << (bd - 8)), 0, (1 << bd) - 1)
               .astype(s.dtype) for s in src]
        items = [(16, 0, w4 - 16, 16, W - 64, H), (0, 16, 16, h4 - 16, W, H - 64),
                 (16, 16, w4 - 16, h4 - 16, W - 64, H - 64), (0, 0, 16, 16, W, H)]
        st = state_array()
        lv, t, _, _, _ = run_counted(rng, layout, bd, grid, src, rec, items, st)
        d_mi = G.to_dev(grid.view(np.uint8).reshape(-1))
        ms = grid.shape[1]

        def scramble(arrs, margin):
            out = []
            for p, a in enumerate(arrs):
                m = outside(a.shape, footprint(items, p, xdec, ydec, margin))
                b = a.copy()
                b[m] = (b[m].astype(np.int64) + rng.integers(1, 1 << bd, int(m.sum()))) % (1 << bd)
                out.append(b)
            return out
        # the level search: working rects plus 4 >> ydec rows above and below
        rec2, src2 = scramble(rec, SEARCH_MARGIN), scramble(src, SEARCH_MARGIN)
        d_rec, d_src = DevPlanes(c, rec2, layout), DevPlanes(c, src2, layout)
        lv2, t2, _ = dev_levels(c, d_rec.views, d_src.views, xdec, ydec, bd, d_mi, ms, items)
        assert (t2 == t).all() and (lv2 == lv).all(), f"r={r}: the level search read outside its footprint"
        # the filter: the working rects only
        in3 = scramble(rec, 0)
        d_in = DevPlanes(c, in3, layout)
        garbage = [rng.integers(0, 1 << bd, a.shape).astype(a.dtype) for a in rec]
        d_out = DevPlanes(c, garbage, layout)
        dev_filter(c, d_in.views, d_out.views, xdec, ydec, bd, st, lv, d_mi, ms, items)
        want = filtered_expectation(rec, garbage, layout, bd, st, lv, grid, items)
        got = d_out.download()
        for p in range(n):
            assert (got[p] == want[p]).all(), f"r={r} plane {p}: the filter read outside the working rects"
        # the converse: only the 3 luma rows above the item at mi row 16 change
        rec4 = [a.copy() for a in rec]
        x0, y0, x1, _ = working_rect(items[1], 0, xdec, ydec)
        rows = slice(PAD + y0 - 3, PAD + y0)
        rec4[0][rows, PAD + x0:PAD + x1] = rng.integers(0, 1 << bd, (3, x1 - x0))
        d_rec4 = DevPlanes(c, rec4, layout)
        d_src4 = DevPlanes(c, src, layout)
        lv4, t4, _ = dev_levels(c, d_rec4.views, d_src4.views, xdec, ydec, bd, d_mi, ms, items)
        want_lv, want_t = orc_levels(rec4, src, layout, bd, grid, items)
        assert (t4 == want_t).all() and (lv4 == want_lv).all()
        assert (t4[1, 0, 1] != t[1, 0, 1]).any(), "the rows above the item did not reach the level search"
        assert (t4[[0, 2]] == t[[0, 2]]).all()         # item 3 owns those rows; items 0 and 2 lie to the right
        reached += 1
        for dp in (d_rec, d_src, d_in, d_out, d_rec4, d_src4):
            dp.free()
    assert reached == 7


# ---------------------------------------------------------------- 4. caller-built planes and mi
def px_view(host, org, stride, w, h, dt):
    """The w x h pixels at byte offset `org` of a byte array, `stride` pixels per row."""
    it = np.dtype(dt).itemsize
    return np.ndarray((h, w), dt, buffer=host, offset=org, strides=(stride * it, it))


@pytest.mark.parametrize("layout,bd", [("420", 8), ("422", 10), ("444", 12), ("400", 10)])
def test_caller_built_planes_and_a_wide_mi_grid(layout, bd):
    rng = seed("views", layout, bd)
    n, xdec, ydec = LAYOUTS[layout]
    W, H = 160, 100
    w4, h4 = ((W + 7) >> 3) * 2, ((H + 7) >> 3) * 2
    ms = 48                                          # mi_stride past the frame's 40 columns
    grid = random_grid(rng, ms, h4, layout, deltas=True)
    grid["pad_"] = rng.integers(0, 256, grid["pad_"].shape)
    items = [(0, 0, 32, 16, W, H), (32, 0, 16, 16, W - 128, H), (0, 16, 32, h4 - 16, W, H - 64),
             (32, 16, 16, h4 - 16, W - 128, H - 64)]
    assert w4 < ms and any(it[0] + it[2] == ms for it in items)
    rec = [np.clip(s.astype(np.int64) + rng.integers(-9, 10, s.shape) * (1 << (bd - 8)), 0, (1 << bd) - 1)
           .astype(s.dtype) for s in make_planes(rng, W, H, layout, bd, "steps")]
    src = [np.clip(r.astype(np.int64) + rng.integers(-4, 5, r.shape), 0, (1 << bd) - 1).astype(r.dtype)
           for r in rec]
    for p, a in enumerate(rec + src):                # garbage, not replicated edges, in every border
        xd, yd = (xdec, ydec) if p % n else (0, 0)
        border = np.ones(a.shape, bool)
        border[PAD >> yd:a.shape[0] - (PAD >> yd), PAD >> xd:a.shape[1] - (PAD >> xd)] = False
        a[border] = rng.integers(0, 1 << bd, int(border.sum()))

    def views(arrs, lo):
        """Each plane at its own pad (at least lo >> ydec), stride and base alignment, cut from the PAD arrays."""
        vs = []
        for p, a in enumerate(arrs):
            xd, yd = (xdec, ydec) if p else (0, 0)
            pmax = PAD >> max(xd, yd)
            pad = int(rng.integers(max(lo >> yd, 1), pmax + 1))
            h, w = a.shape[0] - 2 * (PAD >> yd), a.shape[1] - 2 * (PAD >> xd)
            full = a[(PAD >> yd) - pad:(PAD >> yd) + h + pad, (PAD >> xd) - pad:(PAD >> xd) + w + pad]
            stride = full.shape[1] + int(rng.integers(0, 40))
            vs.append(G.ViewPlane(full, pad, stride, a.itemsize * int(rng.integers(0, 64))))
        return vs
    c = G.ctx()
    d_mi = G.to_dev(grid.view(np.uint8).reshape(-1))
    # pads cover the working rects' rounding past the visible 100 rows (4) plus, for rec and src, the margin
    rv, sv = views(rec, 4 + SEARCH_MARGIN), views(src, 4 + SEARCH_MARGIN)
    assert len({v.plane.stride for v in rv + sv}) > 1
    lv, t, _ = dev_levels(c, [v.plane for v in rv], [v.plane for v in sv], xdec, ydec, bd, d_mi, ms, items)
    want_lv, want_t = orc_levels(rec, src, layout, bd, grid, items)
    assert (t == want_t).all() and (lv == want_lv).all()
    st = state_array(1, [5, -3, 2, 0, -1, 4, 1, -6], [3, -2], block=1, shift=1, multi=1)
    iv = views(rec, 4)
    garbage = [rng.integers(0, 1 << bd, a.shape).astype(a.dtype) for a in rec]
    ov = views(garbage, 4)
    before = [v.buf.cpu().numpy().copy() for v in ov]
    levels = np.array([[40, 30, 20, 50], [63, 1, 9, 33], [12, 50, 63, 0], [25, 25, 30, 30]], np.uint8)
    dev_filter(c, [v.plane for v in iv], [v.plane for v in ov], xdec, ydec, bd, st, levels, d_mi, ms, items)
    filt = [a.copy() for a in rec]
    orc_filter(filt, layout, bd, st, levels, grid, items)
    assert any((f != r).any() for f, r in zip(filt, rec)), "nothing was filtered"
    for p, v in enumerate(ov):
        xd, yd = (xdec, ydec) if p else (0, 0)
        want = before[p].copy()
        org = v.plane.data - v.buf.data_ptr()
        dt = rec[p].dtype
        wv = px_view(want, org, v.plane.stride, v.plane.width + v.plane.pad, v.plane.height + v.plane.pad, dt)
        for it in items:
            x0, y0, x1, y1 = working_rect(it, p, xdec, ydec)
            wv[y0:y1, x0:x1] = filt[p][(PAD >> yd) + y0:(PAD >> yd) + y1, (PAD >> xd) + x0:(PAD >> xd) + x1]
        got = v.buf.cpu().numpy()
        assert (got == want).all(), f"plane {p}: bytes {np.flatnonzero(got != want)[:5]}"


# ---------------------------------------------------------------- 5. deltas at their limits
BOUNDARY_MODES = [0, 12, 13, 14, 17, 18, 19, 31, 32, 33]   # mode_type flips at 14 and for 18 / 32


def rav1e_level(st, lv, blk, p, vertical):
    """deblock_adjusted_level with rav1e's i8 arithmetic; returns (level, whether the i8 sum wrapped)."""
    idx = (0 if vertical else 1) if p == 0 else p + 1
    level, wrapped = int(lv[idx]), False
    if st["block_deltas_enabled"]:
        d = int(blk["deltas"][idx if st["block_delta_multi"] else 0])
        exact = (d << int(st["block_delta_shift"])) + level
        i8 = lambda v: (v + 128) % 256 - 128
        s = i8(i8(d << int(st["block_delta_shift"])) + level)
        wrapped = s != exact
        level = min(max(s, 0), 63)
    if st["deltas_enabled"]:
        ref, mode = int(blk["ref0"]), int(blk["mode"])
        mt = 1 if (mode >= 14 and mode not in (18, 32)) else 0
        l5 = level >> 5
        level = min(max(level + (int(st["ref_deltas"][ref & 7]) << l5)
                        + (0 if ref == 0 else int(st["mode_deltas"][mt]) << l5), 0), 63)
    return level, wrapped


@pytest.mark.parametrize("layout", ["420", "444"])
def test_deltas_at_their_limits(layout):
    rng = seed("deltas", layout)
    n, xdec, ydec = LAYOUTS[layout]
    W, H, bd = 128, 96, 10
    w4, h4 = W // 4, H // 4
    grid, src, rec = frame_setup(rng, layout, bd, W, H)
    grid["ref0"] = rng.integers(0, 8, grid.shape)
    grid["mode"] = rng.choice(BOUNDARY_MODES, grid.shape)
    grid["deltas"] = rng.integers(-63, 64, grid["deltas"].shape)
    items = [(0, 0, 16, 16, W, H), (16, 0, w4 - 16, 16, W - 64, H), (0, 16, w4, h4 - 16, W, H - 64)]
    tables = {(p, v): edge_table(grid, it, p, xdec, ydec, v) for it in items[:1] for p in range(n)
              for v in (True, False)}
    delta_sets = [([63] * 8, [63, 63]), ([-63] * 8, [-63, -63]), ([63, -63, 63, -63, -63, 63, 0, 63], [-63, 63])]
    level_sets = [[1, 2, 63, 0], [63, 62, 0, 1], [2, 0, 63, 63]]
    wraps = fallbacks = 0
    for shift in range(4):
        for multi in (0, 1):
            for k, (rd, md) in enumerate(delta_sets):
                st = state_array(int(k != 1 or shift != 0), rd, md, block=1, shift=shift, multi=multi)
                lv = level_sets[(shift + multi + k) % 3]
                levels = [lv] + [level_sets[(shift + k + j) % 3] for j in (1, 2)]
                run_both(rng, layout, bd, grid, src, rec, items, st, levels)
                for (p, v), (_, _, blocks) in tables.items():
                    if lv[0] == 0 and lv[1] == 0:
                        continue
                    for blk, prev in blocks:
                        lb, wb = rav1e_level(st[0], lv, blk, p, v)
                        wraps += wb
                        fallbacks += lb == 0 and rav1e_level(st[0], lv, prev, p, v)[0] > 0
    print(f"\n{layout}: {wraps} edges with a wrapped block delta, {fallbacks} on the previous block's level")
    assert wraps >= 100 and fallbacks >= 100, (wraps, fallbacks)


# ---------------------------------------------------------------- 6. tallies past 2^32
def test_tallies_past_2_to_the_32():
    rng = seed("tallies")
    W, H, bd, layout = 1920, 1080, 12, "444"
    w4, h4 = W // 4, ((H + 7) >> 3) * 2
    grid = random_grid(rng, w4, h4, layout)
    src = make_planes(rng, W, H, layout, bd, "steps")
    rec = [np.clip(s.astype(np.int64) + rng.integers(-4095, 4096, s.shape), 0, 4095).astype(s.dtype) for s in src]
    items = [(0, 0, w4, h4, W, H)]
    split = []
    for sy in range(17):
        widths = [3] * 6 + [2] * 6 if sy >= 4 else [3] * 8 + [2] * 3
        sx = 0
        for sw in widths:
            split.append(sb_item(sx, sy, sw, 1, W, H))
            sx += sw
        assert sx == 30
    assert len(split) == 200
    c = G.ctx()
    _, xdec, ydec = LAYOUTS[layout]
    d_rec, d_src = DevPlanes(c, rec, layout), DevPlanes(c, src, layout)
    d_mi = G.to_dev(grid.view(np.uint8).reshape(-1))
    for its in (items, split):
        lv, t, _ = dev_levels(c, d_rec.views, d_src.views, xdec, ydec, bd, d_mi, w4, its)
        want_lv, want_t = orc_levels(rec, src, layout, bd, grid, its)
        assert (t == want_t).all(), np.argwhere(t != want_t)[:5]
        assert (lv == want_lv).all()
        big = int(np.abs(want_t).max())
        print(f"\n{len(its)} items: largest |tally| {big} ({big / 2 ** 32:.1f} x 2^32)")
        assert big > 2 ** 32
    for dp in (d_rec, d_src):
        dp.free()
