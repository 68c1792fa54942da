"""Motion compensation on every kernel path, bit exact against a numpy restatement of the AV1 specification's
single two-pass form (7.11.3.4) rather than against the oracle's four special-cased paths.

mc.cu has three kernels:
- `mc_put_fast_kernel<T, N, N>`: `put` at the squares 8 / 16 / 32 / 64 through b200_mc_blocks_dev (packed
  words, mc_dev.cuh);
- `mc_kernel<T>`: `prep`, every other shape, the per-call forms, and every `put` while B200_MC_GENERIC is set;
- `mc_avg_kernel<T>`: b200_mc_avg_dev and b200_mc_avg.
The sweeps, each at 8 / 10 / 12 bit:
1. every (mode_x, mode_y) pair on the fast kernel at all four sizes and in all three layouts, every
   (col_frac, row_frac) pair of the layout with both vector signs, and the same items on the generic kernel;
2. the generic kernel, `put` and `prep`, at every shape the 22 block sizes give at 4:4:4, 4:2:2 and 4:2:0;
3. extreme pixels: tiles built from the tap signs of every bank and fraction, which drive the i16
   intermediate to its computed extremes and the final clamp to its largest overshoot, also through `mc_avg`;
4. blocks at odd positions, overhanging the plane, and footprints that touch the first and the last readable
   pixel of the padded plane;
5. launch geometry: one grid pass plus a ragged second trip of each kernel's grid-stride loop, n = 1, and
   n = 0 with a sentinel-filled output;
6. the per-call forms at every shape, into a destination wider than the block;
7. PlaneSlice::clamp of the footprint origin, which changes no pixel while the footprint stays inside the
   edge-replicated padding.
Before each launch the test asserts that every footprint lies inside the padded plane."""
import ctypes as C

import numpy as np
import pytest
from numpy.lib.stride_tricks import sliding_window_view

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O

pytestmark = pytest.mark.gpu

BDS = [8, 10, 12]
LAYOUTS = [(0, 0), (1, 0), (1, 1)]                         # (xdec, ydec): 4:4:4, 4:2:2, 4:2:0
PAIRS = [(mx, my) for mx in range(4) for my in range(4)]   # FilterMode: REGULAR, SMOOTH, SHARP, BILINEAR
FAST_SIZES = [8, 16, 32, 64]
LUMA_SIZES = [(4, 4), (4, 8), (8, 4), (8, 8), (8, 16), (16, 8), (16, 16), (16, 32), (32, 16), (32, 32),
              (32, 64), (64, 32), (64, 64), (64, 128), (128, 64), (128, 128), (4, 16), (16, 4), (8, 32),
              (32, 8), (16, 64), (64, 16)]                 # the 22 BlockSizes as (w, h)
SHAPES = [(w >> xd, h >> yd, xd, yd) for xd, yd in LAYOUTS for w, h in LUMA_SIZES]
PREP_BIAS = 8192                                           # mc.rs:357, 10 and 12 bit
SENTINEL = 0xA5                                            # every output byte before a launch

# Launch geometry mirrored from mc.cu: warps (= blocks) per CTA = min(8, shared-memory budget / bytes per
# warp), grids capped at num_sms * CTAS_PER_SM CTAs, then a grid-stride loop over the rest.
MC_MAX_WARPS = 8          # mc.cu:187, :222
FAST_SMEM = 128 * 1024    # mc.cu:187  launch_mc_fast
GENERIC_SMEM = 96 * 1024  # mc.cu:222  launch_mc
MC_CTAS_PER_SM = 16       # mc.cu:194, :233  min(ctas, num_sms * 16)
AVG_THREADS = 256         # mc.cu:304  one element per thread
AVG_CTAS_PER_SM = 32      # mc.cu:304  min(ctas, num_sms * 32)


def align16(v):
    return (v + 15) // 16 * 16


def fast_wpc(n, bpp):
    """McLayout<T, N, N>: a (N + 7) x (N + 8) pixel tile and the transposed N x (N + 8) i16 intermediate."""
    return min(MC_MAX_WARPS, max(1, FAST_SMEM // align16((n + 7) * (n + 8) * bpp + n * (n + 8) * 2)))


def generic_wpc(w, h, bpp):
    te = (w + 7) * (h + 7)
    return min(MC_MAX_WARPS, max(1, GENERIC_SMEM // align16((te + (te & 1)) * bpp + (h + 7) * w * 2)))


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------- reference
def pxdt(bd):
    return np.uint8 if bd == 8 else np.uint16


def rnd(v, b):
    return (v + (1 << (b - 1))) >> b


def round0(bd):        # InterRound0
    return 5 if bd == 12 else 3


def round1(bd):        # InterRound1 of a single prediction; 7 for compound (prep)
    return 9 if bd == 12 else 11


def bias(bd):
    return 0 if bd == 8 else PREP_BIAS


_TAPS = {}


def taps(mode, length):
    """(16, 8) int64: get_filter(mode, frac, length) for every fraction, read through the oracle.  The 4-tap
    banks apply when the dimension is <= 4; BILINEAR ignores the length."""
    key = (mode, length <= 4)
    if key not in _TAPS:
        f = (C.c_int32 * 8)()
        t = np.zeros((16, 8), np.int64)
        for frac in range(16):
            O.lib().orc_get_filter(mode, frac, 4 if length <= 4 else 8, f)
            t[frac] = list(f)
        _TAPS[key] = t
    return _TAPS[key]


def fracs(dec):
    """The fractions get_mv_params yields in a dimension with decimation `dec`: even ones only at full size."""
    return list(range(0, 16, 2 - dec))


def mv_from(off, frac, dec):
    """The MotionVector component whose get_mv_params gives full-pel offset `off` and fraction `frac`."""
    return (off << (3 + dec)) + (frac >> (1 - dec))


def mv_params(blocks, mvs, xdec, ydec):
    """get_mv_params (predict.rs:284-297) per item: (x0, y0, col_frac, row_frac); `>>` floors."""
    mvs = np.asarray(mvs, np.int64).reshape(-1, 2)
    r, c = mvs[:, 0], mvs[:, 1]
    x0 = blocks["x"].astype(np.int64) + (c >> (3 + xdec))
    y0 = blocks["y"].astype(np.int64) + (r >> (3 + ydec))
    return x0, y0, (c << (1 - xdec)) & 15, (r << (1 - ydec)) & 15


def assert_readable(x0, y0, w, h, width, height, pad):
    """Every (w + 7) x (h + 7) footprint, columns x0 - 3 .. x0 + w + 3, inside [-pad, width + pad) and
    likewise for the rows: nothing may read past the padding."""
    assert (x0 - 3 >= -pad).all() and (x0 + w + 3 < width + pad).all(), "footprint leaves the padded plane"
    assert (y0 - 3 >= -pad).all() and (y0 + h + 3 < height + pad).all(), "footprint leaves the padded plane"


def hpass(full, pad, x0, y0, cf, w, h, mode_x, bd):
    """The horizontal pass over the h + 7 footprint rows of every item, rounded by InterRound0 and kept wide:
    (n, h + 7, w) int64.  `full` is the padded plane, pixel (0, 0) at (pad, pad)."""
    rows = pad + np.asarray(y0)[:, None] - 3 + np.arange(h + 7)
    cols = pad + np.asarray(x0)[:, None] - 3 + np.arange(w + 7)
    assert rows.min() >= 0 and cols.min() >= 0 and rows.max() < full.shape[0] and cols.max() < full.shape[1]
    tile = full[rows[:, :, None], cols[:, None, :]]                          # one gather for all items
    return rnd(np.einsum("nrck,nk->nrc", sliding_window_view(tile, 8, axis=2), taps(mode_x, w)[cf]), round0(bd))


def vpass(inter, rf, h, mode_y, bd, kind, clip=True):
    """The vertical pass: `put` (kind 0) rounded by InterRound1 then Clip1 (skipped with clip=False), `prep`
    (kind 1) rounded by 7 minus PREP_BIAS."""
    s = np.einsum("nrck,nk->nrc", sliding_window_view(inter, 8, axis=1), taps(mode_y, h)[rf])
    if kind == 1:
        return rnd(s, 7) - bias(bd)
    v = rnd(s, round1(bd))
    return np.clip(v, 0, (1 << bd) - 1) if clip else v


def mc_ref(full, pad, x0, y0, cf, rf, w, h, mode_x, mode_y, bd, kind):
    return vpass(hpass(full, pad, x0, y0, cf, w, h, mode_x, bd), rf, h, mode_y, bd, kind)


def avg_ref(t1, t2, bd):
    """mc_avg: (t1 + t2 + 2 * PREP_BIAS) rounded by InterPostRound (ib + 1), then Clip1."""
    ib = 2 if bd == 12 else 4
    return np.clip(rnd(t1.astype(np.int64) + t2 + 2 * bias(bd), ib + 1), 0, (1 << bd) - 1)


def inter_extremes(bd):
    """The intermediate's extremes over every bank and fraction: all positive taps on max, or all negative."""
    hi = lo = 0
    for mode in range(4):
        for length in (4, 8):
            t = taps(mode, length)
            hi = max(hi, int(rnd(np.where(t > 0, t, 0).sum(1) * ((1 << bd) - 1), round0(bd)).max()))
            lo = min(lo, int(rnd(np.where(t < 0, t, 0).sum(1) * ((1 << bd) - 1), round0(bd)).min()))
    return hi, lo


def sign_tiles(tx, ty, maxv):
    """8 x 8 tiles for the taps tx (columns) and ty (rows): max where the two taps' signs agree (0 counts as
    positive) and 0 elsewhere - the outer product that puts the horizontal pass at its maximum in rows with
    ty >= 0 and at its minimum in rows with ty < 0 - then its complement, both +-max checkerboards and flat
    0 / max."""
    sx, sy = np.where(tx < 0, -1, 1), np.where(ty < 0, -1, 1)
    p = np.where(sy[:, None] == sx[None, :], maxv, 0).astype(np.int64)
    i, j = np.mgrid[0:8, 0:8]
    chk = ((i + j) & 1) * maxv
    z = np.zeros((8, 8), np.int64)
    return [p, maxv - p, chk, maxv - chk, z, z + maxv]


# ---------------------------------------------------------------- device side
@pytest.fixture
def planes():
    """make(img, pad) -> (the padded plane as int64, device plane); device planes are freed afterwards."""
    made = []

    def make(img, pad):
        op, dp = G.both_planes(img, pad)
        made.append(dp)
        return op.data.astype(np.int64), dp
    yield make
    for dp in made:
        G.ctx().plane_free(dp)


def dev_out(nelems, elem_bytes, slack=64):
    import torch
    return torch.full(((nelems + slack) * elem_bytes,), SENTINEL, dtype=torch.uint8, device="cuda")


def host_out(d, n, w, h, dtype):
    """The n packed w x h outputs as int64; every byte after them must still hold the sentinel."""
    raw = d.cpu().numpy()
    size = n * w * h * np.dtype(dtype).itemsize
    assert (raw[size:] == SENTINEL).all(), "bytes written past the last block"
    return raw[:size].view(dtype).reshape(n, h, w).astype(np.int64)


def run_blocks(dp, blocks, mvs, w, h, mx, my, bd, xdec, ydec, kind):
    n = len(blocks)
    dt = np.int16 if kind == 1 else pxdt(bd)
    d = dev_out(n * w * h, np.dtype(dt).itemsize)
    G.ctx().mc_blocks_dev(dp, G.to_dev(blocks), G.to_dev(np.ascontiguousarray(mvs, np.int16)), n, w, h, mx, my,
                          bd, xdec, ydec, kind, d)
    G.ctx().synchronize()
    return host_out(d, n, w, h, dt)


def run_avg(t1, t2, w, h, bd):
    import torch
    n = len(t1)
    d = dev_out(n * w * h, np.dtype(pxdt(bd)).itemsize)
    G.ctx().mc_avg_dev(torch.from_numpy(np.ascontiguousarray(t1, np.int16)).cuda(),
                       torch.from_numpy(np.ascontiguousarray(t2, np.int16)).cuda(), d, n, w, h, bd)
    G.ctx().synchronize()
    return host_out(d, n, w, h, pxdt(bd))


def make_blocks(xs, ys):
    b = np.zeros(len(xs), B.BLOCK_DTYPE)
    b["x"], b["y"] = xs, ys
    return b


def noise(rng, bd, width, height):
    return rng.integers(0, 1 << bd, (height, width)).astype(pxdt(bd))


def mc_kernels(fn):
    return G.profiled_kernels(fn, prefix="mc_")


def check(got, want, what):
    np.testing.assert_array_equal(got, want, err_msg=what)


# ---------------------------------------------------------------- 1. fast kernel, every filter pair
def frac_sweep(rng, w, h, xdec, ydec, width, height, reach):
    """Two items per (col_frac, row_frac) pair of the layout: vector signs (+, +) and (-, -) at even pairs,
    (+, -) and (-, +) at odd ones, full-pel offsets up to `reach`.  So each of the integer / H-only / V-only /
    HV classes meets both signs in both components."""
    rows = []
    for k, (cf, rf) in enumerate((a, b) for a in fracs(xdec) for b in fracs(ydec)):
        for sr, sc in (((1, 1), (-1, -1)) if k % 2 == 0 else ((1, -1), (-1, 1))):
            offs = [int(rng.integers(0, reach + 1)) if s > 0 else -int(rng.integers(1, reach + 1)) for s in (sr, sc)]
            rows.append((int(rng.integers(0, width - w + 1)), int(rng.integers(0, height - h + 1)),
                         mv_from(offs[0], rf, ydec), mv_from(offs[1], cf, xdec)))
    a = np.array(rows, np.int64)
    return make_blocks(a[:, 0], a[:, 1]), a[:, 2:].astype(np.int16)


@pytest.mark.parametrize("n", FAST_SIZES)
@pytest.mark.parametrize("bd", BDS)
def test_fast_kernel_every_filter_pair(bd, n, planes, monkeypatch):
    """All 16 (mode_x, mode_y) pairs of `put` at n x n, in every layout, on mc_put_fast_kernel and on mc_kernel
    (B200_MC_GENERIC, read by launch_mc on every call), with every fraction pair of the layout."""
    monkeypatch.delenv("B200_MC_GENERIC", raising=False)
    width, height, pad, reach = 256, 192, 32, 12
    rng = np.random.default_rng(1000 * bd + n)
    full, dp = planes(noise(rng, bd, width, height), pad)
    ran = set()
    for xdec, ydec in LAYOUTS:
        blocks, mvs = frac_sweep(rng, n, n, xdec, ydec, width, height, reach)
        x0, y0, cf, rf = mv_params(blocks, mvs, xdec, ydec)
        assert_readable(x0, y0, n, n, width, height, pad)
        assert set(zip(cf.tolist(), rf.tolist())) == {(a, b) for a in fracs(xdec) for b in fracs(ydec)}
        for cls in ((cf == 0) & (rf == 0), (cf != 0) & (rf == 0), (cf == 0) & (rf != 0), (cf != 0) & (rf != 0)):
            m = mvs[cls].astype(np.int64)
            assert (m < 0).any(0).all() and (m >= 0).any(0).all()
        for mx in range(4):
            inter = hpass(full, pad, x0, y0, cf, n, n, mx, bd)
            for my in range(4):
                want = vpass(inter, rf, n, my, bd, 0)
                for generic in (False, True):
                    if generic:
                        monkeypatch.setenv("B200_MC_GENERIC", "1")
                    got = run_blocks(dp, blocks, mvs, n, n, mx, my, bd, xdec, ydec, 0)
                    monkeypatch.delenv("B200_MC_GENERIC", raising=False)
                    check(got, want, f"{n}x{n} {bd}-bit dec ({xdec},{ydec}) modes ({mx},{my}) generic={generic}")
                    ran.add((xdec, ydec, mx, my, generic))
    assert len(ran) == len(LAYOUTS) * len(PAIRS) * 2
    # the routing: the same call runs the fast kernel, and the generic one under B200_MC_GENERIC
    tname = "unsigned char" if bd == 8 else "unsigned short"
    call = lambda: run_blocks(dp, blocks[:3], mvs[:3], n, n, 2, 2, bd, xdec, ydec, 0)
    assert mc_kernels(call) == [f"mc_put_fast_kernel<{tname}, {n}, {n}>"]
    monkeypatch.setenv("B200_MC_GENERIC", "1")
    assert mc_kernels(call) == [f"mc_kernel<{tname}>"]


# ---------------------------------------------------------------- 2. generic kernel, every shape
def random_items(rng, count, w, h, xdec, ydec, width, height, reach):
    """Blocks anywhere in the plane; the first four vectors are integer, H only, V only and HV."""
    xs = rng.integers(0, width - w + 1, count)
    ys = rng.integers(0, height - h + 1, count)
    fx, fy = fracs(xdec), fracs(ydec)
    mvs = np.array([(mv_from(int(rng.integers(-reach, reach + 1)), int(rng.choice(fy)), ydec),
                     mv_from(int(rng.integers(-reach, reach + 1)), int(rng.choice(fx)), xdec)) for _ in range(count)])
    mvs[:4] = [(mv_from(-2, 0, ydec), mv_from(3, 0, xdec)), (mv_from(1, 0, ydec), mv_from(-1, fx[-1], xdec)),
               (mv_from(-1, fy[1], ydec), mv_from(0, 0, xdec)), (mv_from(-3, fy[-1], ydec), mv_from(-1, fx[1], xdec))]
    return make_blocks(xs, ys), mvs.astype(np.int16)


@pytest.mark.parametrize("bd", BDS)
def test_generic_kernel_every_shape(bd, planes, monkeypatch):
    """`put` and `prep` on mc_kernel at all 66 (shape, layout) items.  Shape s runs the pairs (j, (j + s) % 4)
    for j = 0..3: every shape meets every mode in each direction (so a 4-tap bank wherever a dimension is <= 4,
    and BILINEAR), and every pair occurs at many shapes."""
    monkeypatch.setenv("B200_MC_GENERIC", "1")
    width, height, pad, reach = 256, 192, 32, 12
    rng = np.random.default_rng(bd)
    full, dp = planes(noise(rng, bd, width, height), pad)
    shapes_of = {p: set() for p in PAIRS}
    for s, (w, h, xdec, ydec) in enumerate(SHAPES):
        blocks, mvs = random_items(rng, 24, w, h, xdec, ydec, width, height, reach)
        x0, y0, cf, rf = mv_params(blocks, mvs, xdec, ydec)
        assert_readable(x0, y0, w, h, width, height, pad)
        for j in range(4):
            mx, my = j, (j + s) % 4
            inter = hpass(full, pad, x0, y0, cf, w, h, mx, bd)
            for kind in (0, 1):
                got = run_blocks(dp, blocks, mvs, w, h, mx, my, bd, xdec, ydec, kind)
                check(got, vpass(inter, rf, h, my, bd, kind), f"{w}x{h} dec ({xdec},{ydec}) ({mx},{my}) kind {kind}")
            shapes_of[(mx, my)].add((w, h, xdec, ydec))
    assert min(len(v) for v in shapes_of.values()) >= 16
    tname = "unsigned char" if bd == 8 else "unsigned short"
    assert mc_kernels(lambda: run_blocks(dp, blocks[:2], mvs[:2], 8, 8, 0, 0, bd, 0, 0, 0)) == [f"mc_kernel<{tname}>"]


# ---------------------------------------------------------------- 3. extreme pixels
CELL = 16      # each extreme item owns a 16 x 16 cell; its footprint starts at the cell's corner
EXT_GROUPS = [(0, 8), (1, 8), (2, 8), (3, 8), (0, 4), (1, 4)]     # (mode, block side): banks 0 .. 5


def extreme_items(bd):
    """The image, and per bank group the blocks / 4:2:0 vectors of every (f, f), (f, 0), (0, f) fraction pair
    (at 4:2:0 every fraction 0 .. 15 is reachable) times the six sign tiles, each tile repeated over the cell."""
    maxv = (1 << bd) - 1
    combos = [(f, f) for f in range(16)] + [(f, 0) for f in range(1, 16)] + [(0, f) for f in range(1, 16)]
    per_group = len(combos) * 6
    cols = 32
    nrows = -(-per_group * len(EXT_GROUPS) // cols)
    img = np.zeros((nrows * CELL, cols * CELL), np.int64)
    groups = []
    k = 0
    for mode, side in EXT_GROUPS:
        xs, ys, mvs = [], [], []
        for cf, rf in combos:
            for tile in sign_tiles(taps(mode, side)[cf], taps(mode, side)[rf], maxv):
                cx, cy = (k % cols) * CELL, (k // cols) * CELL
                img[cy:cy + CELL, cx:cx + CELL] = np.tile(tile, (CELL // 8, CELL // 8))
                xs.append(cx + 3)
                ys.append(cy + 3)
                mvs.append((rf, cf))       # 4:2:0: full-pel offset 0, fraction = the vector itself
                k += 1
        groups.append((mode, side, make_blocks(xs, ys), np.array(mvs, np.int16)))
    return img.astype(pxdt(bd)), groups


@pytest.mark.parametrize("bd", BDS)
def test_extreme_pixels_reach_the_intermediate_bounds(bd, planes, monkeypatch):
    """The sign tiles of every bank and fraction through both `put` kernels, `prep`, and `mc_avg` of two extreme
    preps.  The reference itself must reach the intermediate's computed extremes (23 546 / -7 166 at 12 bit) and
    overshoot both ends of the final clamp, so the input is known to drive them."""
    maxv = (1 << bd) - 1
    img, groups = extreme_items(bd)
    height, width = img.shape
    pad = 16
    full, dp = planes(img, pad)
    hi = lo = 0
    over = under = False
    for mode, side, blocks, mvs in groups:
        x0, y0, cf, rf = mv_params(blocks, mvs, 1, 1)
        assert_readable(x0, y0, side, side, width, height, pad)
        inter = hpass(full, pad, x0, y0, cf, side, side, mode, bd)
        hi, lo = max(hi, int(inter.max())), min(lo, int(inter.min()))
        raw = vpass(inter, rf, side, mode, bd, 0, clip=False)
        over, under = over or bool((raw > maxv).any()), under or bool((raw < 0).any())
        want = np.clip(raw, 0, maxv)
        for generic in ((False, True) if side == 8 else (True,)):
            if generic:
                monkeypatch.setenv("B200_MC_GENERIC", "1")
            got = run_blocks(dp, blocks, mvs, side, side, mode, mode, bd, 1, 1, 0)
            monkeypatch.delenv("B200_MC_GENERIC", raising=False)
            check(got, want, f"put mode {mode} {side}x{side} generic={generic}")
        t = vpass(inter, rf, side, mode, bd, 1)
        assert t.min() >= -32768 and t.max() <= 32767
        check(run_blocks(dp, blocks, mvs, side, side, mode, mode, bd, 1, 1, 1), t, f"prep mode {mode} {side}x{side}")
        # each pred with itself, and with its complement tile (pattern 2k <-> 2k + 1 of the same fractions)
        partner = np.arange(len(t)) ^ 1
        for t2 in (t, t[partner]):
            check(run_avg(t, t2, side, side, bd), avg_ref(t, t2, bd), f"avg mode {mode} {side}x{side}")
    assert (hi, lo) == inter_extremes(bd)
    assert (hi, lo) == {8: (5865, -1785), 10: (23529, -7161), 12: (23546, -7166)}[bd]
    assert over and under


# ---------------------------------------------------------------- 4. positions
@pytest.mark.parametrize("bd", BDS)
def test_odd_overhanging_and_edge_touching_positions(bd, planes, monkeypatch):
    """Odd block positions, blocks hanging over every side of the plane, and vectors whose footprints start on
    the first readable pixel (-pad, -pad) or end on the last (width + pad - 1, height + pad - 1)."""
    width, height, pad, reach = 200, 120, 48, 8
    rng = np.random.default_rng(40 + bd)
    full, dp = planes(noise(rng, bd, width, height), pad)
    touched = set()
    for (w, h), (xdec, ydec), (mx, my) in (((8, 8), (0, 0), (2, 2)), ((16, 16), (1, 0), (0, 2)),
                                           ((32, 32), (1, 1), (2, 1)), ((4, 16), (1, 1), (2, 0)),
                                           ((32, 8), (1, 0), (3, 2)), ((2, 4), (0, 0), (1, 2))):
        fx, fy = fracs(xdec), fracs(ydec)
        xs, ys, mvs = [], [], []
        for _ in range(12):                                    # odd positions
            xs.append(2 * int(rng.integers(0, (width - w) // 2)) + 1)
            ys.append(2 * int(rng.integers(0, (height - h) // 2)) + 1)
            mvs.append((mv_from(int(rng.integers(-reach, reach + 1)), int(rng.choice(fy)), ydec),
                        mv_from(int(rng.integers(-reach, reach + 1)), int(rng.choice(fx)), xdec)))
        for bx in (-w + 1, -w // 2, width - w // 2, width - 1):  # hanging over each side
            for by in (-h + 1, height // 2, height - 1):
                xs.append(bx)
                ys.append(by)
                mvs.append((mv_from(int(rng.integers(-2, 3)), int(rng.choice(fy)), ydec),
                            mv_from(int(rng.integers(-2, 3)), int(rng.choice(fx)), xdec)))
        # footprints on the padded plane's first / last readable column and row, at fraction 0 and at the half
        for tx in (3 - pad, width + pad - 4 - w):
            for ty in (3 - pad, height // 3, height + pad - 4 - h):
                for f in (0, 8):
                    bx, by = int(rng.integers(0, width - w + 1)), int(rng.integers(0, height - h + 1))
                    xs.append(bx)
                    ys.append(by)
                    mvs.append((mv_from(ty - by, f, ydec), mv_from(tx - bx, f, xdec)))
        blocks, mvs = make_blocks(xs, ys), np.array(mvs, np.int16)
        x0, y0, cf, rf = mv_params(blocks, mvs, xdec, ydec)
        assert_readable(x0, y0, w, h, width, height, pad)
        assert (x0 - 3).min() == -pad and (x0 + w + 3).max() == width + pad - 1
        assert (y0 - 3).min() == -pad and (y0 + h + 3).max() == height + pad - 1
        touched.add((w, h))
        inter = hpass(full, pad, x0, y0, cf, w, h, mx, bd)
        for kind in (0, 1):
            want = vpass(inter, rf, h, my, bd, kind)
            for generic in ((False, True) if kind == 0 and w == h and w in FAST_SIZES else (True,)):
                if generic:
                    monkeypatch.setenv("B200_MC_GENERIC", "1")
                got = run_blocks(dp, blocks, mvs, w, h, mx, my, bd, xdec, ydec, kind)
                monkeypatch.delenv("B200_MC_GENERIC", raising=False)
                check(got, want, f"{w}x{h} dec ({xdec},{ydec}) kind {kind} generic={generic}")
    assert len(touched) == 6


# ---------------------------------------------------------------- 5. launch geometry
def repeated(rng, unique_blocks, unique_mvs, n):
    idx = rng.integers(0, len(unique_blocks), n)
    return idx, np.ascontiguousarray(unique_blocks[idx]), np.ascontiguousarray(unique_mvs[idx])


@pytest.mark.parametrize("bd", BDS)
def test_grid_stride_second_trip_and_tiny_counts(bd, planes, monkeypatch):
    """Each kernel gets one full capped grid pass plus a ragged second trip, then n = 1 and n = 0 (the
    sentinel-filled output stays untouched).  Large counts repeat 101 distinct items in random order; the
    reference is computed once per distinct item."""
    monkeypatch.delenv("B200_MC_GENERIC", raising=False)
    width, height, pad, reach = 192, 128, 32, 12
    bpp = 1 if bd == 8 else 2
    sms = num_sms()
    rng = np.random.default_rng(70 + bd)
    full, dp = planes(noise(rng, bd, width, height), pad)
    tname = "unsigned char" if bd == 8 else "unsigned short"
    trips = {}
    # (kernel, w, h, kind, layout, blocks per CTA)
    for name, w, h, kind, (xdec, ydec), wpc in (
            (f"mc_put_fast_kernel<{tname}, 8, 8>", 8, 8, 0, (1, 0), fast_wpc(8, bpp)),
            (f"mc_kernel<{tname}>", 4, 4, 0, (1, 1), generic_wpc(4, 4, bpp)),
            (f"mc_kernel<{tname}>", 8, 4, 1, (0, 0), generic_wpc(8, 4, bpp))):
        ub, um = random_items(rng, 101, w, h, xdec, ydec, width, height, reach)
        x0, y0, cf, rf = mv_params(ub, um, xdec, ydec)
        assert_readable(x0, y0, w, h, width, height, pad)
        uwant = mc_ref(full, pad, x0, y0, cf, rf, w, h, 2, 1, bd, kind)
        one_pass = sms * MC_CTAS_PER_SM * wpc                 # blocks the capped grid covers per trip
        n = one_pass + one_pass // 2 + 3
        assert n % wpc != 0 and (n + wpc - 1) // wpc > sms * MC_CTAS_PER_SM
        for count in (n, 1, 0):
            idx, blocks, mvs = repeated(rng, ub, um, count)
            call = lambda: trips.__setitem__((name, kind, count),
                                             run_blocks(dp, blocks, mvs, w, h, 2, 1, bd, xdec, ydec, kind))
            if count == n:
                assert mc_kernels(call) == [name]
            else:
                call()
            check(trips[(name, kind, count)], uwant[idx], f"{name} kind {kind} n={count}")
    # mc_avg_kernel: elements, not blocks, stride the grid
    w, h = 8, 8
    per_pass = sms * AVG_CTAS_PER_SM * AVG_THREADS
    n = (per_pass + per_pass // 2) // (w * h) + 3
    assert n * w * h > per_pass and (n * w * h) % AVG_THREADS != 0
    lim = 1 << 14
    ut1 = rng.integers(-lim, lim, (97, h, w))
    ut2 = rng.integers(-lim, lim, (97, h, w))
    ut1[0], ut2[0] = 32767, 32767
    ut1[1], ut2[1] = -32768, -32768
    for count in (n, 1, 0):
        idx = rng.integers(0, 97, count)
        got = {}
        call = lambda: got.setdefault("v", run_avg(ut1[idx], ut2[idx], w, h, bd))
        if count == n:
            assert mc_kernels(call) == [f"mc_avg_kernel<{tname}>"]
        else:
            call()
        check(got["v"], avg_ref(ut1[idx], ut2[idx], bd), f"mc_avg n={count}")


# ---------------------------------------------------------------- 6. per-call forms
@pytest.mark.parametrize("bd", BDS)
def test_percall_forms_every_shape(bd):
    """b200_put_8tap / b200_prep_8tap / b200_mc_avg (host pointers, byte strides, explicit fractions) at every
    shape of sweep 2, into a destination wider than the block: nothing outside the w x h window changes."""
    L = B.lib()
    width, height, pad = 160, 160, 16
    rng = np.random.default_rng(90 + bd)
    img = noise(rng, bd, width, height)
    op = O.Plane(width, height, pad, dtype=img.dtype)
    op.fill_from(img)
    full = op.data.astype(np.int64)
    isz = op.bpp
    px = pxdt(bd)
    sent_px = np.frombuffer(bytes([SENTINEL] * isz), px)[0]
    sent_i16 = np.frombuffer(bytes([SENTINEL] * 2), np.int16)[0]
    shapes = sorted({(w, h) for w, h, _, _ in SHAPES})
    for s, (w, h) in enumerate(shapes):
        preps = []
        for j, (cf, rf) in enumerate(((int(rng.integers(1, 16)), int(rng.integers(1, 16))), (0, 2 * s % 16 + 1),
                                      (2 * s % 16 + 1, 0))):
            mx, my = (s + j) % 4, (s + 2 * j + 1) % 4
            x, y = int(rng.integers(0, width - w + 1)), int(rng.integers(0, height - h + 1))
            xa, ya = np.array([x]), np.array([y])
            assert_readable(xa, ya, w, h, width, height, pad)
            inter = hpass(full, pad, xa, ya, np.array([cf]), w, h, mx, bd)
            dst = np.full((h, w + 5), sent_px, px)
            L.b200_put_8tap(dst.ctypes.data, dst.strides[0], op.at(x, y), op.stride * isz, w, h, cf, rf, mx, my, bd)
            check(dst[:, :w], vpass(inter, np.array([rf]), h, my, bd, 0)[0], f"put {w}x{h} ({cf},{rf}) ({mx},{my})")
            assert (dst[:, w:] == sent_px).all()
            tmp = np.full(w * h + 16, sent_i16, np.int16)
            L.b200_prep_8tap(tmp.ctypes.data, op.at(x, y), op.stride * isz, w, h, cf, rf, mx, my, bd)
            want = vpass(inter, np.array([rf]), h, my, bd, 1)[0]
            check(tmp[:w * h].reshape(h, w), want, f"prep {w}x{h} ({cf},{rf}) ({mx},{my})")
            assert (tmp[w * h:] == sent_i16).all()
            preps.append(np.ascontiguousarray(want.astype(np.int16)))
        for t1, t2 in ((preps[0], preps[1]), (preps[2], preps[2])):
            dst = np.full((h, w + 3), sent_px, px)
            L.b200_mc_avg(dst.ctypes.data, dst.strides[0], t1.ctypes.data, t2.ctypes.data, w, h, bd)
            check(dst[:, :w], avg_ref(t1, t2, bd), f"avg {w}x{h}")
            assert (dst[:, w:] == sent_px).all()


# ---------------------------------------------------------------- 7. PlaneSlice::clamp inside the padding
@pytest.mark.parametrize("bd", BDS)
def test_origin_clamp_inside_the_padding_changes_nothing(bd, planes, monkeypatch):
    """rav1e clamps the footprint origin (position + (mv >> 3) - 3) to [-pad, width] x [-pad, height]
    (predict.rs:296, PlaneSlice::clamp); the kernels do not.  Past width - 1 every column of the edge-replicated
    padding repeats that column (likewise for rows), so while the unclamped footprint stays inside the padding
    both read the same pixels.  Vectors here cross the clamp threshold on each side."""
    monkeypatch.delenv("B200_MC_GENERIC", raising=False)
    width, height, pad = 96, 64, 80
    rng = np.random.default_rng(110 + bd)
    full, dp = planes(noise(rng, bd, width, height), pad)
    active_x = active_y = 0
    for (w, h), (xdec, ydec), (mx, my) in (((8, 8), (0, 0), (2, 2)), ((16, 16), (1, 1), (0, 0)),
                                           ((4, 8), (1, 0), (1, 2)), ((32, 16), (0, 0), (2, 3)),
                                           ((64, 64), (1, 0), (2, 1))):
        fx, fy = fracs(xdec), fracs(ydec)
        xs, ys, mvs = [], [], []
        qxs = [width - 2, width - 1, width, width + 1, width + 5, width + pad - w - 7, -pad, -pad + 3]
        qys = [height - 1, height, height + 1, height + 9, height + pad - h - 7, -pad, 0]
        for qx in qxs:
            for qy in qys:
                bx, by = int(rng.integers(0, width - w + 1)), int(rng.integers(0, height - h + 1))
                xs.append(bx)
                ys.append(by)
                mvs.append((mv_from(qy + 3 - by, int(rng.choice(fy)), ydec), mv_from(qx + 3 - bx, int(rng.choice(fx)), xdec)))
        blocks, mvs = make_blocks(xs, ys), np.array(mvs, np.int16)
        x0, y0, cf, rf = mv_params(blocks, mvs, xdec, ydec)
        assert_readable(x0, y0, w, h, width, height, pad)
        cx = np.clip(x0 - 3, -pad, width) + 3
        cy = np.clip(y0 - 3, -pad, height) + 3
        active_x += int((cx != x0).sum())
        active_y += int((cy != y0).sum())
        for kind in (0, 1):
            want = mc_ref(full, pad, cx, cy, cf, rf, w, h, mx, my, bd, kind)
            check(mc_ref(full, pad, x0, y0, cf, rf, w, h, mx, my, bd, kind), want, "clamp moved a pixel")
            got = run_blocks(dp, blocks, mvs, w, h, mx, my, bd, xdec, ydec, kind)
            check(got, want, f"{w}x{h} dec ({xdec},{ydec}) kind {kind}")
    assert active_x > 0 and active_y > 0
