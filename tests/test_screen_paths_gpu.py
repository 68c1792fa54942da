"""Mode screening on every kernel path, bit exact against the oracle (orc_intra_mode_screen, orc_inter_mode_screen,
orc_cfl_alpha) in every output array.

The kernels:
- `intra_screen_kernel<T>` (intra_screen.cu): b200_intra_mode_screen_dev; one 128-thread CTA per item gathers the
  edges, stages the tx-sized source block and sums every screened mode's SATD in shared memory;
- `inter_screen_bucket_kernel` and `inter_screen_kernel<T, CLS>` (inter_screen.cu): b200_inter_mode_screen_dev; the
  first validates every item and appends the valid ones to one bucket per size class in ctx->dwork, then one launch
  per class walks its bucket, one warp per item;
- `cfl_alpha_kernel<T>` (cfl_alpha.cu): b200_cfl_alpha_dev; one 128-thread CTA per item, luma AC, both chroma
  planes' DC and the SSE of all 33 alphas.
The launch geometry mirrored here:
- intra_screen.cu:236  grid min(nitems, num_sms * 8), one item per CTA per trip;
- cfl_alpha.cu:290     grid min(nitems, num_sms * 16), one item per CTA per trip;
- inter_screen.cu:257  bucket grid min(ceil(n / 256), num_sms * 8) CTAs of 256 threads (inter_screen.cu:32), one
  item per thread per trip;
- inter_screen.cu:249  class grid min(ceil(n / wpc), num_sms * 8) CTAs of wpc <= 8 warps (inter_screen.cu:33,
  :245), one item per warp per trip;
- inter_screen.cu:77   size classes by the longest side: <= 16, <= 32, <= 64; inter_screen.cu:260-262 launch all
  three whatever their counts;
- inter_screen.cu:296  16 + 3 * 4 * nitems bytes of ctx->dwork, which capi.cu:130 grows to 1.25x rounded up to
  1 MiB after a stream synchronise.
The padding each host check requires, and no more, is what the planes here declare:
- intra_screen.cu:216  rec and src pad >= 64;
- inter_screen.cu:277, :291  refs pad >= max(xorigin, yorigin, 71), src pad >= 64;
- cfl_alpha.cu:254     luma width + pad >= frame_width + 31 (likewise in height); the chroma planes need none.
The sweeps:
1. read footprints: every plane is built from one padded image whose padding holds random values (not the edge
   replicated), seen identically by the oracle and the device, and the device buffer carries a poison ring past
   the declared padding, so a read of the wrong padded pixel or past the padding is a mismatch, never a fault.
   Intra: blocks of every size overhanging the plane's right and bottom edges, in the whole plane and in a tile
   off the origin.  Inter: vectors on every side of PlaneSlice::clamp, up to +-4000 pel and +-32767, at two
   origins.  CfL: every cfl_allowed size on the last visible column and row of frames whose size is not a
   multiple of 8, at 4:2:0, 4:2:2 and 4:4:4;
2. grid-stride trips: intra and CfL at one full grid pass plus a ragged second one; inter with more items than
   the bucket kernel's threads and, in every size class, more valid items than the class kernel's warps (most
   of them empty or invalid, a few thousand real ones spread through the list);
3. inter size classes: calls with every item in one class at 8 and 16 bit, a call with classes 0 and 2 only,
   four launches in each; garbage in the unused entries cands[n..19] changes nothing;
4. caller-built views: odd element strides, pixel (0, 0) 1, 3 and 17 bytes past a 128-byte boundary (twice that
   at 16 bit), alloc NULL, every plane at its own stride; the input buffers are unchanged afterwards;
5. extreme content at 12 bit (and 8 bit for CfL): all-maximum, all-zero and alternating 0 / max images, and a
   source that is the bitwise complement of the reconstruction, at each kernel's largest blocks (intra 64x64 and
   the 128-sided sizes with TX_64X64, inter 64x64 compound, CfL 32x32 at 4:4:4);
6. ordering: inter calls of growing size, so ctx->dwork grows between them, interleaved with intra and CfL
   calls on one context with no host synchronise, then one synchronise and every result checked.
Every output buffer is filled with a sentinel before each launch."""
import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_oracle_cfl_alpha import BLOCK_32X32, NALPHA, Frame, cfl_alpha, grid_items, odd_items
from tests.test_oracle_inter_screen import (ENTRIES, ITEM_DTYPE, SCREEN_SIZES, inter_mode_screen, make_item, origins,
                                            random_items)
from tests.test_oracle_intra_edges import BSIZES
from tests.test_oracle_intra_screen import intra_mode_screen, make_items

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5                 # every output byte before a launch
RING = 16                       # poison pixels past each device plane's declared padding
MODES = 13                      # intra_screen.cu:33  kModes

# Launch geometry mirrored from the sources
INTRA_CTAS_PER_SM = 8           # intra_screen.cu:236  min(nitems, num_sms * 8)
CFL_CTAS_PER_SM = 16            # cfl_alpha.cu:290     min(nitems, num_sms * 16)
BUCKET_THREADS = 256            # inter_screen.cu:32   kBucketThreads
BUCKET_CTAS_PER_SM = 8          # inter_screen.cu:257  min(ceil(n / 256), num_sms * 8)
CLASS_MAX_WARPS = 8             # inter_screen.cu:33   kMaxWarps: wpc <= 8 (inter_screen.cu:245)
CLASS_CTAS_PER_SM = 8           # inter_screen.cu:249  min(ceil(n / wpc), num_sms * 8)
INTER_LAUNCHES = 4              # inter_screen.cu:258-262  the bucket kernel and one launch per size class
# The padding each host check accepts at least
INTRA_PAD = 64                  # intra_screen.cu:216  kMaxTx
INTER_SRC_PAD = 64              # inter_screen.cu:291
INTER_REF_PAD = 71              # inter_screen.cu:277  max(xorigin, yorigin, 64 + 7)
CFL_LUMA_REACH = 31             # cfl_alpha.cu:254     luma width + pad >= frame_width + 31

BLOCK_64X64 = 12
LAYOUTS = [(1, 1), (1, 0), (0, 0)]                      # 4:2:0, 4:2:2, 4:4:4


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def second_trip(cap):
    """An item count with one full grid pass and a ragged second one."""
    return cap + cap // 2 + 3


def profiled_launches(fn):
    """Run `fn` under torch.profiler: (its result, [(kernel name, CTAs, threads per CTA)] in launch order), from
    the trace's kernel records, so a test can show that its grids are the capped ones it claims to pass."""
    import json
    import os
    import tempfile
    import time
    import torch
    from torch.profiler import ProfilerActivity, profile
    # a session now and then records no device activity at all (tests/gpu_util.py): run it again
    for attempt in range(6):
        time.sleep(0.1 * attempt)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                events = json.load(f)["traceEvents"]
        kernels = [(e["name"], e["args"]["grid"][0], e["args"]["block"][0]) for e in events
                   if e.get("cat") == "kernel"]
        if kernels:
            return out, kernels
    raise AssertionError("torch.profiler recorded no CUDA kernels: the launch grids cannot be checked")


def launched(kernels, name):
    return [(g, b) for k, g, b in kernels if name in k]


def pxdt(bd):
    return np.uint8 if bd == 8 else np.uint16


def size_class(bs):
    """inter_screen.cu:76-77: the longest side <= 16, 32, 64."""
    side = max(BSIZES[bs])
    return 0 if side <= 16 else 1 if side <= 32 else 2


CLASS_SIZES = [[bs for bs in SCREEN_SIZES if size_class(bs) == c] for c in range(3)]


def dwork_reserved(nbytes):
    """What b200_reserve_dwork allocates for `nbytes` (capi.cu:130): 1.25x, rounded up to 1 MiB."""
    mib = 1 << 20
    return (nbytes + nbytes // 4 + mib - 1) // mib * mib


def inter_dwork(n):
    return 16 + 3 * n * 4                               # inter_screen.cu:296


# ---------------------------------------------------------------- planes seen by both sides
class Padded:
    """One padded image seen by both sides.  `host` is the oracle's O.Plane: the visible image and `pad` pixels of
    random, non-replicated padding, written to `.data` directly.  `dev` is a caller-built b200_plane (a
    G.ViewPlane) over the same pixels, declaring the same `pad`, whose buffer carries RING further pixels of
    poison all around: a read past the declared padding is a mismatch, and still inside the allocation."""

    def __init__(self, rng, img, pad, bd, stride_extra=0, offset=0, with_alloc=True):
        h, w = img.shape
        maxv = (1 << bd) - 1
        self.pad = pad
        inner = rng.integers(0, maxv + 1, (h + 2 * pad, w + 2 * pad)).astype(img.dtype)
        inner[pad:pad + h, pad:pad + w] = img
        self.host = O.Plane(w, h, pad, dtype=img.dtype)
        self.host.data[:] = inner
        P = pad + RING
        full = rng.integers(0, maxv + 1, (h + 2 * P, w + 2 * P)).astype(img.dtype)
        full[RING:RING + h + 2 * pad, RING:RING + w + 2 * pad] = inner
        self.view = G.ViewPlane(full, P, full.shape[1] + stride_extra, offset, with_alloc)
        self.view.plane.pad = pad
        self.before = self.view.buf.cpu().numpy().copy()

    @property
    def dev(self):
        return self.view.plane

    def unchanged(self):
        return (self.view.buf.cpu().numpy() == self.before).all()


def extreme(kind, h, w, bd, rng):
    maxv = (1 << bd) - 1
    if kind == "max":
        img = np.full((h, w), maxv)
    elif kind == "zero":
        img = np.zeros((h, w))
    elif kind == "checker":                              # alternating 0 / max
        img = (np.add.outer(np.arange(h), np.arange(w)) % 2) * maxv
    else:
        img = rng.integers(0, maxv + 1, (h, w))
    return img.astype(pxdt(bd))


def complement(img, bd):
    return ((1 << bd) - 1 - img.astype(np.int64)).astype(img.dtype)


def sentinel(nbytes):
    t = G.dev_empty(nbytes)
    t.fill_(SENTINEL)
    return t


def assert_same(got, want, items, what):
    """Every output array equal; the first differing items in the message."""
    for g, w, name in zip(got, want, ("first output", "second output")):
        assert g.shape == w.shape, (what, name, g.shape, w.shape)
        bad = np.nonzero((g != w).reshape(len(g), -1).any(1))[0]
        assert len(bad) == 0, (what, name, len(bad), bad[:4], items[bad[:2]], g[bad[:2]], w[bad[:2]])


# ---------------------------------------------------------------- one call of each kernel
def intra_outs(n):
    return sentinel(n * MODES * 4), sentinel(n * MODES)


def intra_launch(c, rec, src, rect, bd, nmr, d_items, n, outs):
    c.intra_mode_screen_dev(rec.dev, src.dev, rect, bd, nmr, d_items, n, *outs)
    return outs


def intra_read(outs, n):
    return (G.from_dev(outs[0], np.uint32)[:n * MODES].reshape(n, MODES),
            G.from_dev(outs[1], np.uint8)[:n * MODES].reshape(n, MODES))


def intra_check(rec, src, rect, bd, nmr, items, what=""):
    c = G.ctx()
    n = len(items)
    outs = intra_launch(c, rec, src, rect, bd, nmr, G.to_dev(items), n, intra_outs(n))
    c.synchronize()
    got = intra_read(outs, n)
    assert_same(got, intra_mode_screen(rec.host, src.host, rect, bd, nmr, items), items, what)
    return got


def inter_outs(n):
    return sentinel(n * ENTRIES * 4), sentinel(n * ENTRIES)


def inter_launch(c, src, refs, rect, xo, yo, mode, bd, d_items, n, outs):
    c.inter_mode_screen_dev(src.dev, rect, [r.dev for r in refs], xo, yo, mode, bd, d_items, n, *outs)
    return outs


def inter_read(outs, n):
    return (G.from_dev(outs[0], np.uint32)[:n * ENTRIES].reshape(n, ENTRIES),
            G.from_dev(outs[1], np.uint8)[:n * ENTRIES].reshape(n, ENTRIES))


def inter_check(src, refs, rect, xo, yo, mode, bd, items, what=""):
    c = G.ctx()
    n = len(items)
    d_items, outs = G.to_dev(items), inter_outs(n)
    before = c.launches
    inter_launch(c, src, refs, rect, xo, yo, mode, bd, d_items, n, outs)
    c.synchronize()
    assert c.launches == before + INTER_LAUNCHES, what
    got = inter_read(outs, n)
    want = inter_mode_screen(src.host, rect, [r.host for r in refs], xo, yo, mode, bd, items)
    assert_same(got, want, items, what)
    return got


class CflFrame:
    """The three rec planes and the two chroma src planes of a frame, each a Padded (src luma is rec luma: the
    call does not read it)."""

    def __init__(self, rng, W, H, xdec, ydec, bd, luma=None, chroma=None, luma_pad=CFL_LUMA_REACH, chroma_pad=0,
                 views=None):
        self.W, self.H, self.xdec, self.ydec, self.bd = W, H, xdec, ydec, bd
        cw, ch = (W + xdec) >> xdec, (H + ydec) >> ydec
        dt, maxv = pxdt(bd), (1 << bd) - 1
        luma = luma if luma is not None else rng.integers(0, maxv + 1, (H, W)).astype(dt)
        chroma = chroma if chroma is not None else [rng.integers(0, maxv + 1, (ch, cw)).astype(dt) for _ in range(4)]
        views = views or [{}] * 5
        self.rec = [Padded(rng, luma, luma_pad, bd, **views[0])] + \
                   [Padded(rng, chroma[k], chroma_pad, bd, **views[1 + k]) for k in range(2)]
        self.src = [self.rec[0]] + [Padded(rng, chroma[2 + k], chroma_pad, bd, **views[3 + k]) for k in range(2)]
        F = Frame.__new__(Frame)                         # the oracle's frame over the same host planes
        F.xdec, F.ydec, F.width, F.height, F.bd = xdec, ydec, W, H, bd
        F.rec, F.src = [p.host for p in self.rec], [p.host for p in self.src]
        self.oracle = F

    def planes(self):
        return self.rec + self.src[1:]


def cfl_outs(n):
    return sentinel(n * 2), sentinel(n * 2 * NALPHA * 8)


def cfl_launch(c, fr, rect, d_items, n, outs):
    c.cfl_alpha_dev([p.dev for p in fr.rec], [p.dev for p in fr.src], fr.xdec, fr.ydec, rect, fr.W, fr.H, fr.bd,
                    d_items, n, *outs)
    return outs


def cfl_read(outs, n):
    return (G.from_dev(outs[0], np.int8)[:n * 2].reshape(n, 2),
            G.from_dev(outs[1], np.uint64)[:n * 2 * NALPHA].reshape(n, 2, NALPHA))


def cfl_check(fr, rect, items, what=""):
    c = G.ctx()
    n = len(items)
    outs = cfl_launch(c, fr, rect, G.to_dev(items), n, cfl_outs(n))
    c.synchronize()
    got = cfl_read(outs, n)
    assert_same(got, cfl_alpha(fr.oracle, rect, items), items, what)
    return got


# ---------------------------------------------------------------- item lists
def intra_overhanging(rng, rect, bsizes=range(22)):
    """Blocks of every size on the region's last block column / row (aligned to the size) and on its last
    4x4 column / row, plus each on the top row and left column."""
    rw, rh = rect[2], rect[3]
    lx, ly = (rw - 1) // 4 * 4, (rh - 1) // 4 * 4
    out = []
    for bs in bsizes:
        bw, bh = BSIZES[bs]
        ax, ay = (rw - 1) // bw * bw, (rh - 1) // bh * bh
        for x, y in ((ax, ay), (lx, ly), (lx, 0), (0, ly), (ax, ly), (lx, ay)):
            it = make_items(rng, rw, rh, 1, bsizes=[bs], iefs=(int(rng.integers(-1, 2)),))
            it["x"], it["y"] = x, y
            out.append(it)
    return np.concatenate(out)


def clamp_entries(W, H, x, y):
    """Vectors that start the footprint past each side of the plane (tests/test_inter_screen_gpu.py), single
    and compound."""
    ents = []
    for row, col in ((0, -8 * 4000), (0, 8 * 4000), (-8 * 4000, 0), (8 * 4000, 0),
                     (8 * (H - y + 16) + 3, 8 * (W - x + 16) + 5), (-8 * (y + 200) - 1, -8 * (x + 150) + 2),
                     (-32767, 32767), (32767, -32768), (8 * (H - y) - 4, 8 * (W - x) - 9),
                     (-8 * (y + 3) + 6, 8 * (W - x + 2) - 3), (8 * (H - y + 1) + 1, -8 * (x + 4) - 7)):
        ents.append(((len(ents) & 1), None, (row, col), None))
    ents.append((0, 1, (8 * (H + 40), 0), (0, -8 * (W + 200) + 6)))
    ents.append((1, 0, (-8 * 300, 8 * 500 + 4), (8 * 3 + 1, 8 * 2)))
    ents.append((1, 1, (32767, 32767), (-32768, -32768)))
    return ents[:ENTRIES]


def inter_clamp_items(W, H, rect):
    items = []
    rw, rh = rect[2], rect[3]
    for bs in SCREEN_SIZES:
        bw, bh = BSIZES[bs]
        ax, ay = (rw - 1) // bw * bw, (rh - 1) // bh * bh
        for x, y in ((0, 0), (ax, ay), (ax, 0), (0, ay), ((rw - 1) // 4 * 4, (rh - 1) // 4 * 4)):
            items.append(make_item(x, y, bs, clamp_entries(W, H, rect[0] + x, rect[1] + y)))
    return np.array(items)


def inter_list(rng, rect_w, rect_h, nrefs, total, valid_per_class, real_per_class, reach=24):
    """`total` items: in each size class `valid_per_class` valid ones, `real_per_class` of them with entries and
    the rest with n = 0 and random bytes in every cands row; all others invalid, each for one of seven reasons.
    Every kind is spread through the whole list.  Returns (items, number of real items)."""
    items = rng.integers(0, 256, (total, ITEM_DTYPE.itemsize), dtype=np.uint8).view(ITEM_DTYPE).reshape(total)
    order = rng.permutation(total)
    nvalid = 3 * valid_per_class
    assert nvalid <= total
    # the valid ones: empty lists at aligned positions inside the region
    for c in range(3):
        idx = order[c * valid_per_class:(c + 1) * valid_per_class]
        items["bsize"][idx] = rng.choice(CLASS_SIZES[c], len(idx))
        items["x"][idx] = 4 * rng.integers(0, (rect_w + 3) // 4, len(idx))
        items["y"][idx] = 4 * rng.integers(0, (rect_h + 3) // 4, len(idx))
        items["n"][idx] = 0
        real = idx[:real_per_class]
        items[real] = random_items(rng, rect_w, rect_h, len(real), nrefs, bsizes=CLASS_SIZES[c], reach=reach)
    # the invalid ones: a valid-looking item with one fault
    inv = order[nvalid:]
    m = len(inv)
    items["bsize"][inv] = rng.choice(SCREEN_SIZES, m)
    items["x"][inv] = 4 * rng.integers(0, (rect_w + 3) // 4, m)
    items["y"][inv] = 4 * rng.integers(0, (rect_h + 3) // 4, m)
    items["n"][inv] = rng.integers(0, ENTRIES + 1, m)
    why = np.arange(m) % 7
    sel = lambda r: inv[why == r]
    items["bsize"][sel(0)] = rng.integers(22, 256, len(sel(0)))          # no such BlockSize
    items["bsize"][sel(1)] = rng.choice([13, 14, 15], len(sel(1)))        # 128-sided
    items["n"][sel(2)] = rng.integers(ENTRIES + 1, 256, len(sel(2)))      # more than 20 entries
    items["x"][sel(3)] = rect_w + 4 * rng.integers(0, 64, len(sel(3)))    # outside the region
    items["y"][sel(4)] = -4 * rng.integers(1, 64, len(sel(4)))
    items["x"][sel(5)] += rng.integers(1, 4, len(sel(5)))                 # not a multiple of 4
    s6 = sel(6)                                                           # an entry's reference >= nrefs
    items["n"][s6] = rng.integers(1, ENTRIES + 1, len(s6))
    k6 = rng.integers(0, items["n"][s6].astype(np.int64))
    ref = items["cands"]["ref"]
    side = rng.integers(0, 2, len(s6))
    ref[s6, k6, 0] = np.where(side == 0, rng.integers(nrefs, 256, len(s6)), ref[s6, k6, 0] % nrefs)
    ref[s6, k6, 1] = np.where(side == 1, rng.integers(nrefs, 255, len(s6)), 0xFF)
    return items, 3 * min(real_per_class, valid_per_class)


# ================================================================ 1. read footprints
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_intra_reads_stay_inside_the_declared_padding(bd):
    """Blocks overhanging the plane stage their tx-sized source from src's padding (rav1e reads it there, not
    a clamped row); the edges are gathered at the plane's and the tile's borders."""
    rng = np.random.default_rng(100 + bd)
    W, H = 150, 110
    dt = pxdt(bd)
    rec = Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), INTRA_PAD, bd)
    src = Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), INTRA_PAD, bd)
    for rect in ((0, 0, W, H), (40, 24, W - 40, H - 24)):
        items = intra_overhanging(rng, rect)
        for nmr in (3, 7):
            intra_check(rec, src, rect, bd, nmr, items, (rect, nmr))
    assert rec.unchanged() and src.unchanged()


@pytest.mark.parametrize("bd", [8, 10, 12])
@pytest.mark.parametrize("origin", ["frame", "small"])
def test_inter_reads_stay_inside_the_clamped_footprint(bd, origin):
    """PlaneSlice::clamp to [-xorigin, width] x [-yorigin, height] (inter_screen.cu:122-123): the footprint of a
    vector past any side starts exactly on the clamp, in random padding; the references declare only the
    padding the host check asks for."""
    rng = np.random.default_rng(200 + bd + len(origin))
    W, H = 150, 110
    dt = pxdt(bd)
    xo, yo = origins(bd) if origin == "frame" else (24, 8)
    src = Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), INTER_SRC_PAD, bd)
    refs = [Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), max(xo, yo, INTER_REF_PAD), bd)
            for _ in range(2)]
    for k, rect in enumerate(((0, 0, W, H), (32, 16, W - 32, H - 16))):
        inter_check(src, refs, rect, xo, yo, (bd + k) & 3, bd, inter_clamp_items(W, H, rect), (rect, xo, yo))
    assert src.unchanged() and all(r.unchanged() for r in refs)


@pytest.mark.parametrize("xdec,ydec", LAYOUTS)
def test_cfl_luma_reads_stay_inside_the_declared_padding(xdec, ydec):
    """luma_ac reads past the visible luma up to the luma tx width (max_luma_w / max_luma_h, cfl_alpha.cu:109-117):
    planes exactly the frame's size, luma with the 31 pixels of padding the host check asks for, chroma with
    none.  Every cfl_allowed size on the last visible column and row."""
    for (W, H), bd in (((101, 75), 8), ((86, 58), 10), ((57, 99), 12)):
        rng = np.random.default_rng(300 + 10 * xdec + ydec + bd)
        fr = CflFrame(rng, W, H, xdec, ydec, bd)
        aw, ah = (W + 7) // 8 * 8, (H + 7) // 8 * 8
        for rect in ((0, 0, aw, ah), (16, 8, aw - 16, ah - 8)):
            items = grid_items(rng, rect, range(BLOCK_32X32 + 1))
            bw = np.array([BSIZES[b][0] for b in items["bsize"]])
            bh = np.array([BSIZES[b][1] for b in items["bsize"]])
            edge = (items["x"] + bw >= rect[2]) | (items["y"] + bh >= rect[3])
            last = odd_items(rect)
            last = last[(last["x"] >= rect[2] - 8) | (last["y"] >= rect[3] - 8)]
            items = np.concatenate([items[edge], last])
            alpha, sse = cfl_check(fr, rect, items, (W, H, bd, rect))
            assert (sse != np.uint64(0xFFFFFFFFFFFFFFFF)).any()
        assert all(p.unchanged() for p in fr.planes())


# ================================================================ 2. grid-stride trips
@pytest.mark.parametrize("bd", [8, 12])
def test_intra_second_grid_trip(bd):
    cap = num_sms() * INTRA_CTAS_PER_SM
    n = second_trip(cap)
    rng = np.random.default_rng(400 + bd)
    W, H = 256, 192
    dt = pxdt(bd)
    rec = Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), INTRA_PAD, bd)
    src = Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), INTRA_PAD, bd)
    items = make_items(rng, W, H, n)
    bad = rng.choice(np.arange(cap, n), 8, replace=False)               # invalid items in the second trip
    items["bsize"][bad[:4]] = 22
    items["x"][bad[4:]] = W
    (satd, _), kernels = profiled_launches(lambda: intra_check(rec, src, (0, 0, W, H), bd, 3 if bd == 8 else 7, items))
    assert launched(kernels, "intra_screen_kernel<") == [(cap, 128)]
    assert (satd[bad] == np.uint32(0xFFFFFFFF)).all() and (satd[cap:] != np.uint32(0xFFFFFFFF)).any()


@pytest.mark.parametrize("bd", [8, 10])
def test_cfl_second_grid_trip(bd):
    cap = num_sms() * CFL_CTAS_PER_SM
    n = second_trip(cap)
    rng = np.random.default_rng(500 + bd)
    W, H = 250, 190
    fr = CflFrame(rng, W, H, 1, 1, bd)
    rect = (0, 0, 256, 192)
    items = np.concatenate([grid_items(rng, rect, range(BLOCK_32X32 + 1)), odd_items((64, 64, 64, 64))])
    items = items[rng.choice(len(items), n, replace=len(items) < n)]
    (alpha, sse), kernels = profiled_launches(lambda: cfl_check(fr, rect, items))
    assert launched(kernels, "cfl_alpha_kernel<") == [(cap, 128)]
    assert (sse[cap:] != np.uint64(0xFFFFFFFFFFFFFFFF)).any()


@pytest.mark.parametrize("bd", [8, 12])
def test_inter_bucket_and_class_grid_trips(bd):
    """More items than the bucket kernel's num_sms * 8 CTAs of 256 threads, and in every class more valid items
    than num_sms * 8 CTAs of kMaxWarps warps: both grid-stride loops run a second, ragged trip.  Most items are
    invalid or empty (they still need their output rows); 1800 real ones carry the SATDs."""
    sms = num_sms()
    total = second_trip(sms * BUCKET_CTAS_PER_SM * BUCKET_THREADS)
    per_class = second_trip(sms * CLASS_CTAS_PER_SM * CLASS_MAX_WARPS)
    rng = np.random.default_rng(600 + bd)
    W, H = 256, 192
    dt = pxdt(bd)
    xo, yo = origins(bd)
    src = Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), INTER_SRC_PAD, bd)
    refs = [Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), max(xo, yo, INTER_REF_PAD), bd)
            for _ in range(2)]
    items, real = inter_list(rng, W, H, 2, total, per_class, 600)
    (satd, order), kernels = profiled_launches(lambda: inter_check(src, refs, (0, 0, W, H), xo, yo, 0, bd, items))
    # every launch at its cap, and one pass of each grid covers fewer items than it is given
    assert launched(kernels, "inter_screen_bucket_kernel") == [(sms * BUCKET_CTAS_PER_SM, BUCKET_THREADS)]
    classes = launched(kernels, "inter_screen_kernel<")
    assert len(classes) == 3
    for ctas, threads in classes:
        assert ctas == sms * CLASS_CTAS_PER_SM and threads <= 32 * CLASS_MAX_WARPS and ctas * threads // 32 < per_class
    live = (satd != np.uint32(0xFFFFFFFF)).any(1)
    assert live.sum() == real                          # every real item produced SATDs, nothing else did
    assert live[sms * BUCKET_CTAS_PER_SM * BUCKET_THREADS:].any()


# ================================================================ 3. inter size classes
@pytest.mark.parametrize("bd", [8, 12])
@pytest.mark.parametrize("classes", [(0,), (1,), (2,), (0, 2)])
def test_inter_calls_with_empty_classes(bd, classes):
    """Every item in one class (the others' launches find an empty bucket), and classes 0 and 2 only.  At 16
    bit class 2 needs about 44 KB of shared memory per warp, the fewest warps per CTA."""
    rng = np.random.default_rng(700 + bd + 10 * sum(classes) + len(classes))
    W, H = 200, 136
    dt = pxdt(bd)
    xo, yo = origins(bd)
    src = Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), INTER_SRC_PAD, bd)
    refs = [Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), max(xo, yo, INTER_REF_PAD), bd)
            for _ in range(3)]
    sizes = [bs for c in classes for bs in CLASS_SIZES[c]]
    items = random_items(rng, W, H, 120, 3, bsizes=sizes, reach=40)
    rng.shuffle(items)
    inter_check(src, refs, (0, 0, W, H), xo, yo, int(rng.integers(0, 4)), bd, items, classes)


@pytest.mark.parametrize("bd", [8, 10])
def test_inter_unused_entries_are_ignored(bd):
    """cands[n..19] of every item hold random bytes (references >= nrefs, 0xFE, wild vectors): the results equal
    those of the same items with the unused entries zeroed, and the oracle's."""
    rng = np.random.default_rng(800 + bd)
    W, H = 160, 128
    dt = pxdt(bd)
    xo, yo = origins(bd)
    src = Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), INTER_SRC_PAD, bd)
    refs = [Padded(rng, rng.integers(0, 1 << bd, (H, W)).astype(dt), max(xo, yo, INTER_REF_PAD), bd)
            for _ in range(2)]
    clean = random_items(rng, W, H, 190, 2)
    clean["n"][::19] = 0
    garbage = clean.copy()
    raw = rng.integers(0, 256, (len(clean), ENTRIES, garbage.dtype["cands"].base.itemsize), dtype=np.uint8)
    noise = raw.view(garbage.dtype["cands"].base).reshape(len(clean), ENTRIES)
    unused = np.arange(ENTRIES)[None, :] >= clean["n"][:, None]
    cands = garbage["cands"]
    cands[unused] = noise[unused]
    assert (garbage["cands"]["ref"][unused] >= 2).any()
    want = inter_check(src, refs, (0, 0, W, H), xo, yo, 1, bd, clean, "zeroed")
    got = inter_check(src, refs, (0, 0, W, H), xo, yo, 1, bd, garbage, "garbage")
    assert_same(got, want, garbage, "garbage vs zeroed")


# ================================================================ 4. caller-built views
def view_args(k, cols, bpp, offset, with_alloc):
    """Plane k's view: an odd element stride of its own past the `cols` of its padded image, pixel (0, 0) `offset`
    elements past a 128-byte boundary."""
    extra = 2 * k + 1 + cols % 2
    return dict(stride_extra=extra, offset=offset * bpp, with_alloc=with_alloc)


@pytest.mark.parametrize("bd", [8, 12])
@pytest.mark.parametrize("offset", [1, 3, 17])
def test_caller_built_views(bd, offset):
    """Each kernel on planes at odd element strides, every plane's different, pixel (0, 0) `offset` bytes (twice
    that at 16 bit) past a 128-byte boundary; alloc NULL at offset 3.  The inputs are not written."""
    rng = np.random.default_rng(900 + 10 * bd + offset)
    bpp = 1 if bd == 8 else 2
    dt = pxdt(bd)
    with_alloc = offset != 3
    va = lambda k, cols: view_args(k, cols, bpp, offset, with_alloc)
    W, H = 148, 108
    img = lambda h, w: rng.integers(0, 1 << bd, (h, w)).astype(dt)
    # intra
    rec = Padded(rng, img(H, W), INTRA_PAD, bd, **va(0, W + 2 * INTRA_PAD + 2 * RING))
    src = Padded(rng, img(H, W), INTRA_PAD, bd, **va(1, W + 2 * INTRA_PAD + 2 * RING))
    assert rec.dev.stride != src.dev.stride and rec.dev.stride % 2 and src.dev.stride % 2
    for rect in ((0, 0, W, H), (36, 20, W - 36, H - 20)):
        items = np.concatenate([make_items(rng, rect[2], rect[3], 88), intra_overhanging(rng, rect, [3, 9, 12, 15])])
        intra_check(rec, src, rect, bd, 7, items, ("intra", rect))
    # inter
    xo, yo = origins(bd)
    rp = max(xo, yo, INTER_REF_PAD)
    isrc = Padded(rng, img(H, W), INTER_SRC_PAD, bd, **va(2, W + 2 * INTER_SRC_PAD + 2 * RING))
    refs = [Padded(rng, img(H, W), rp, bd, **va(3 + k, W + 2 * rp + 2 * RING)) for k in range(3)]
    assert len({p.dev.stride for p in [isrc] + refs}) == 4
    items = np.concatenate([random_items(rng, W, H, 150, 3, reach=40), inter_clamp_items(W, H, (0, 0, W, H))[::3]])
    inter_check(isrc, refs, (0, 0, W, H), xo, yo, 3, bd, items, "inter")
    # CfL, 4:2:0 and 4:2:2
    for xdec, ydec in ((1, 1), (1, 0)):
        cw, ch = (W + xdec) >> xdec, (H + ydec) >> ydec
        views = [va(0, W + 2 * CFL_LUMA_REACH + 2 * RING)] + [va(1 + k, cw + 2 * RING) for k in range(4)]
        fr = CflFrame(rng, W, H, xdec, ydec, bd, views=views)
        rect = (0, 0, 152, 112)
        items = np.concatenate([grid_items(rng, rect, range(BLOCK_32X32 + 1), per_size=12), odd_items((96, 64, 56, 48))])
        cfl_check(fr, rect, items, ("cfl", xdec, ydec))
        assert all(p.unchanged() for p in fr.planes())
    assert all(p.unchanged() for p in [rec, src, isrc] + refs)
    assert all((p.dev.alloc is not None) == with_alloc for p in [rec, src, isrc] + refs)


# ================================================================ 5. extreme content
KINDS = [("max", "complement"), ("zero", "complement"), ("checker", "complement"), ("checker", "same"),
         ("random", "complement")]


def pair(kind, how, h, w, bd, rng):
    a = extreme(kind, h, w, bd, rng)
    return a, complement(a, bd) if how == "complement" else a.copy()


def test_intra_extreme_content_at_the_largest_blocks():
    """12 bit, the 64x64 and 128-sided blocks (all TX_64X64): the largest per-mode shared sums."""
    bd = 12
    rng = np.random.default_rng(1000)
    W, H = 320, 256
    rect = (64, 64, W - 64, H - 64)
    items = []
    for bs in (BLOCK_64X64, 13, 14, 15):
        bw, bh = BSIZES[bs]
        for x, y in ((0, 0), (64, 0), (0, 64), (64, 64), ((rect[2] - 1) // 4 * 4, (rect[3] - 1) // 4 * 4)):
            it = make_items(rng, rect[2], rect[3], 3, bsizes=[bs])
            it["x"], it["y"] = x, y
            items.append(it)
    items = np.concatenate(items)
    peak = 0
    for kind, how in KINDS:
        r_img, s_img = pair(kind, how, H, W, bd, rng)
        rec, src = Padded(rng, r_img, INTRA_PAD, bd), Padded(rng, s_img, INTRA_PAD, bd)
        for nmr in (3, 7):
            satd, _ = intra_check(rec, src, rect, bd, nmr, items, (kind, how, nmr))
            peak = max(peak, int(satd.max()))
    assert peak >= 64 * 64 * ((1 << bd) - 1) // 8           # a full-range difference over a whole 64x64


def test_inter_extreme_content_at_64x64_compound():
    bd = 12
    rng = np.random.default_rng(1100)
    W, H = 256, 192
    xo, yo = origins(bd)
    rp = max(xo, yo, INTER_REF_PAD)
    items = random_items(rng, W, H, 60, 3, bsizes=[BLOCK_64X64], reach=80)
    for it in items:                                           # every entry compound
        n = int(it["n"])
        it["cands"]["ref"][:n, 1] = rng.integers(0, 3, n)
        it["cands"]["mv"][:n, 1] = rng.integers(-8 * 80, 8 * 80 + 1, (n, 2))
    clamp = inter_clamp_items(W, H, (0, 0, W, H))
    items = np.concatenate([items, clamp[clamp["bsize"] == BLOCK_64X64]])
    for kind, how in KINDS:
        s_img, r_img = pair(kind, how, H, W, bd, rng)
        src = Padded(rng, s_img, INTER_SRC_PAD, bd)
        refs = [Padded(rng, r_img if k != 1 else s_img, rp, bd) for k in range(3)]
        inter_check(src, refs, (0, 0, W, H), xo, yo, int(rng.integers(0, 4)), bd, items, (kind, how))


@pytest.mark.parametrize("bd", [8, 12])
def test_cfl_extreme_content_at_32x32_444(bd):
    """4:4:4 32x32 with TX_32X32: AC samples up to +-(max << 3) / 2, 16 squared full-range differences per
    chunk, the largest per-alpha sums."""
    rng = np.random.default_rng(1200 + bd)
    W, H = 160, 128
    rect = (0, 0, W, H)
    items = grid_items(rng, rect, [BLOCK_32X32], tx_random=False)
    for kind, how in KINDS:
        luma = extreme("checker" if kind != "random" else "random", H, W, bd, rng)
        c_rec, c_src = pair(kind, how, H, W, bd, rng)
        fr = CflFrame(rng, W, H, 0, 0, bd, luma=luma, chroma=[c_rec, c_rec.copy(), c_src, complement(c_src, bd)])
        alpha, sse = cfl_check(fr, rect, items, (kind, how))
        assert (sse != np.uint64(0xFFFFFFFFFFFFFFFF)).any()


# ================================================================ 6. ordering
def test_back_to_back_calls_without_a_host_sync():
    """On a fresh context, inter calls whose scratch needs grow past each reservation (b200_reserve_dwork
    synchronises and reallocates), with intra and CfL calls between them, all enqueued with no host
    synchronise; one synchronise at the end, then every result is checked."""
    import torch
    rng = np.random.default_rng(1300)
    bd = 8
    W, H = 256, 192
    xo, yo = origins(bd)
    img = lambda: rng.integers(0, 1 << bd, (H, W)).astype(np.uint8)
    rec, src = Padded(rng, img(), INTRA_PAD, bd), Padded(rng, img(), INTRA_PAD, bd)
    isrc = Padded(rng, img(), INTER_SRC_PAD, bd)
    refs = [Padded(rng, img(), max(xo, yo, INTER_REF_PAD), bd) for _ in range(2)]
    fr = CflFrame(rng, W, H, 1, 1, bd)
    sizes = [500, 100_000, 200_000]
    reserved = 0
    for n in sizes:                                            # each call's scratch outgrows the last reservation
        assert inter_dwork(n) > reserved
        reserved = dwork_reserved(inter_dwork(n))
    calls = []
    for k, n in enumerate(sizes):
        items, _ = inter_list(rng, W, H, 2, n, min(n // 4, 4000), 150)
        calls.append(("inter", items, k & 3))
        calls.append(("intra", make_items(rng, W, H, 300), 3 + 4 * (k & 1)))
        calls.append(("cfl", grid_items(rng, (0, 0, W, H), range(BLOCK_32X32 + 1), per_size=40), None))
    # every input uploaded and every output filled before the first call: nothing but the calls in between
    d_items = [G.to_dev(items) for _, items, _ in calls]
    outs = [{"inter": inter_outs, "intra": intra_outs, "cfl": cfl_outs}[kind](len(items)) for kind, items, _ in calls]
    c = B.Context(0, use_torch_stream=True)
    try:
        torch.cuda.synchronize()
        for (kind, items, arg), d, o in zip(calls, d_items, outs):
            n = len(items)
            if kind == "inter":
                inter_launch(c, isrc, refs, (0, 0, W, H), xo, yo, arg, bd, d, n, o)
            elif kind == "intra":
                intra_launch(c, rec, src, (0, 0, W, H), bd, arg, d, n, o)
            else:
                cfl_launch(c, fr, (0, 0, W, H), d, n, o)
        c.synchronize()
    finally:
        c.close()
    for (kind, items, arg), o in zip(calls, outs):
        n = len(items)
        if kind == "inter":
            got = inter_read(o, n)
            want = inter_mode_screen(isrc.host, (0, 0, W, H), [r.host for r in refs], xo, yo, arg, bd, items)
        elif kind == "intra":
            got = intra_read(o, n)
            want = intra_mode_screen(rec.host, src.host, (0, 0, W, H), bd, arg, items)
        else:
            got = cfl_read(o, n)
            want = cfl_alpha(fr.oracle, (0, 0, W, H), items)
        assert_same(got, want, items, (kind, n))
