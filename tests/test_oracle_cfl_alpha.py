"""orc_cfl_alpha (rdo_cfl_alpha, rdo.rs:1593-1689, with luma_ac, predict.rs:644-698, and clip_visible_bsize,
rdo.rs:228-253) against an independent Python restatement that calls only the oracle's pieces: pred_cfl_ac,
get_intra_edges, the intra predictors and get_weighted_sse.  The restatement does the orchestration itself:
validity, uv_tx_size, the visible area at the frame block offset (2 mod 4 for a sub-8x8 block at an odd
position in 4:2:0), the sub-8x8 luma offset, frame_clipped_bw / bh against the frame rounded up to 8, the per
block w_pad / h_pad, the variant from the 4-aligned chroma origin, alpha 0 as DC_PRED and the early exit.
Both outputs are compared entry for entry."""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O
from tests.test_oracle_intra_edges import BSIZES, L as OL

LAYOUTS = [(1, 1), (1, 0), (0, 0)]                        # 4:2:0, 4:2:2, 4:4:4
DEPTHS = [(np.uint8, 8), (np.uint16, 10), (np.uint16, 12)]
# b200_cfl_item / orc_cfl_item (oracle/cfl_alpha.h)
CFL_ITEM_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2"), ("bsize", "u1"), ("tx_size", "u1"), ("pad_", "u1", (2,))])
NALPHA = 33
SSE_MAX = np.uint64(0xFFFFFFFFFFFFFFFF)
BLOCK_32X32 = 9
PAD = 48


def tx_index(w, h):
    return O.TX_SIZES.index((w, h))


def largest_luma_tx(bsize):
    bw, bh = BSIZES[bsize]
    return tx_index(min(bw, 64), min(bh, 64))


class Frame:
    """The three planes of rec and src with the frame size fi.width x fi.height they belong to.  The planes
    may be larger than the frame (rav1e's are 8-aligned): what lies past the frame is data, not replication."""

    def __init__(self, rec_imgs, src_imgs, xdec, ydec, width, height, bd):
        self.xdec, self.ydec, self.width, self.height, self.bd = xdec, ydec, width, height, bd
        self.rec = [self._plane(i) for i in rec_imgs]
        self.src = [self._plane(i) for i in src_imgs]

    @staticmethod
    def _plane(img):
        p = O.Plane(img.shape[1], img.shape[0], PAD, dtype=img.dtype)
        p.fill_from(img)
        return p

    @property
    def chroma(self):
        return (self.width + self.xdec) >> self.xdec, (self.height + self.ydec) >> self.ydec


def random_image(rng, w, h, bd, dtype, smooth=True, amp=None):
    maxv = (1 << bd) - 1
    img = rng.integers(0, maxv + 1, (h, w)).astype(np.float64)
    if smooth:
        k = np.ones(5) / 5.0
        img = np.apply_along_axis(lambda r: np.convolve(r, k, mode="same"), 1, img)
        img = np.apply_along_axis(lambda c: np.convolve(c, k, mode="same"), 0, img)
    if amp is not None:
        img = maxv / 2 + (img - img.mean()) * amp
    return np.clip(np.rint(img), 0, maxv).astype(dtype)


def make_frame(rng, W, H, xdec, ydec, bd, dtype, extra=32, chroma_extra=0):
    """Random planes.  The luma plane is `extra` pixels wider and taller than the frame, filled with fresh data
    there, so the columns / rows in [W, align8(W)) that luma_ac reads are not a replication of the last one."""
    cw, ch = (W + xdec) >> xdec, (H + ydec) >> ydec
    rec = [random_image(rng, W + extra, H + extra, bd, dtype)] + \
          [random_image(rng, cw + chroma_extra, ch + chroma_extra, bd, dtype) for _ in range(2)]
    src = [rec[0]] + [random_image(rng, cw + chroma_extra, ch + chroma_extra, bd, dtype) for _ in range(2)]
    return Frame(rec, src, xdec, ydec, W, H, bd)


def cfl_alpha(F: Frame, rect, items, threads=0):
    """orc_cfl_alpha -> (alpha n x 2 int8, sse n x 2 x 33 uint64)."""
    items = np.ascontiguousarray(items, CFL_ITEM_DTYPE)
    n = len(items)
    alpha = np.full((n, 2), 99, np.int8)
    sse = np.zeros((n, 2, NALPHA), np.uint64)
    f = O.lib().orc_cfl_alpha
    f.restype = None
    f.argtypes = [C.c_void_p] * 4 + [C.c_int] * 12 + [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int]
    recp = (C.c_void_p * 3)(*[p.origin_ptr() for p in F.rec])
    srcp = (C.c_void_p * 3)(*[p.origin_ptr() for p in F.src])
    recs = (C.c_ssize_t * 3)(*[p.stride for p in F.rec])
    srcs = (C.c_ssize_t * 3)(*[p.stride for p in F.src])
    f(recp, recs, srcp, srcs, F.rec[0].bpp, F.rec[1].width, F.rec[1].height, F.xdec, F.ydec, *rect, F.width,
      F.height, F.bd, O.ptr(items) if n else None, n, O.ptr(alpha), O.ptr(sse), threads)
    return alpha, sse


# ------------------------------------------------------------------ the restatement
def _wsse():
    l = O.lib()
    for n in ("orc_weighted_sse_u8", "orc_weighted_sse_u16"):
        f = getattr(l, n)
        f.restype = C.c_uint64
        f.argtypes = [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_size_t, C.c_int, C.c_int]
    return l


UNIT = np.full(64, 1 << 14, np.uint32)                    # |_, _| DistortionScale::default(), 8 per row


def valid(F, rect, x, y, bs, tx):
    if bs > BLOCK_32X32 or tx >= 19:                       # cfl_allowed
        return False
    if (F.xdec, F.ydec) == (1, 0) and BSIZES[bs] in ((4, 8), (8, 16), (16, 32)):   # no subsampled_size
        return False
    bw, bh = BSIZES[bs]
    tw, th = O.TX_SIZES[tx]
    if tw > bw or th > bh or not (0 <= x < rect[2] and 0 <= y < rect[3]) or x % 4 or y % 4:
        return False
    bx, by = x >> 2, y >> 2                                # has_chroma, width_mi / height_mi
    return (bx % 2 == 1 or (bw >> 2) % 2 == 0 or F.xdec == 0) and (by % 2 == 1 or (bh >> 2) % 2 == 0 or F.ydec == 0)


def model_block(F, rect, x, y, bs, tx):
    """The block's luma AC, its uv tx size, visible area and per-plane (edge, lens, variant, origin) — or None
    when the reference evaluates nothing."""
    rx, ry, rw, rh = rect
    xdec, ydec = F.xdec, F.ydec
    bw, bh = BSIZES[bs]
    tw, th = max(bw >> xdec, 4), max(bh >> ydec, 4)        # subsampled_size == uv_tx_size.block_size()
    fw, fh = F.chroma

    def clip(frame, blk, pos):                             # clip_visible_bsize
        return blk if pos + blk <= frame else 0 if pos >= frame else frame - pos
    vis_w, vis_h = clip(fw, tw, (rx + x) >> xdec), clip(fh, th, (ry + y) >> ydec)
    if vis_w == 0 or vis_h == 0:
        return None
    # luma_ac
    lbx = (x >> 2) - (1 if xdec and bw == 4 else 0)
    lby = (y >> 2) - (1 if ydec and bh == 4 else 0)
    fbx, fby = (rx >> 2) + lbx, (ry >> 2) + lby
    w_in_b, h_in_b = 2 * ((F.width + 7) >> 3), 2 * ((F.height + 7) >> 3)
    txw, txh = O.TX_SIZES[tx]
    mlw = -(-min((w_in_b - fbx) * 4, bw) // txw) * txw if bw > 8 else bw
    mlh = -(-min((h_in_b - fby) * 4, bh) // txh) * txh if bh > 8 else bh
    w_pad, h_pad = (bw - mlw) >> (2 + xdec), (bh - mlh) >> (2 + ydec)
    lp = F.rec[0]
    y0, x0 = lp.pad + ry + 4 * lby, lp.pad + rx + 4 * lbx
    ac = O.pred_cfl_ac(lp.data[y0:y0 + 64, x0:x0 + 64], tw, th, w_pad, h_pad, xdec, ydec)
    planes = []
    crx, cry, crw, crh = rx >> xdec, ry >> ydec, rw >> xdec, rh >> ydec     # TileRect::decimated
    po_x, po_y = ((x >> 2) >> xdec) << 2, ((y >> 2) >> ydec) << 2            # tile_bo.plane_offset
    variant = 0 if (po_x, po_y) == (0, 0) else 1 if po_y == 0 else 2 if po_x == 0 else 3
    for p in (1, 2):
        rec = F.rec[p]
        edge = np.zeros(O.EDGE_LEN, rec.data.dtype)
        il, ia = C.c_int(), C.c_int()
        OL().orc_get_intra_edges(edge.ctypes.data, rec.at(crx, cry), rec.stride, rec.bpp, rec.width, rec.height, crx,
                                 cry, crw, crh, xdec, ydec, x >> 2, y >> 2, 0, 0, bs, po_x, po_y, tw, th, F.bd, 13, 0,
                                 0, C.byref(il), C.byref(ia))
        planes.append((edge, il.value, ia.value, crx + po_x, cry + po_y))
    return dict(ac=ac, tw=tw, th=th, vis=(vis_w, vis_h), variant=variant, planes=planes)


def predict(F, blk, p, alpha):
    """predict_intra with UV_CFL_PRED at `alpha` (alpha 0 is DC_PRED, predict.rs:236)."""
    edge, il, ia, dx, dy = blk["planes"][p - 1]
    rec = F.rec[p]
    return O.predict_intra(0 if alpha == 0 else 13, blk["variant"], edge, blk["tw"], blk["th"], F.bd, angle=alpha,
                           ac=blk["ac"] if alpha else None, left_len=il, above_len=ia, plane_w=rec.width,
                           plane_h=rec.height, dst_x=dx, dst_y=dy)


def model_item(F, rect, it):
    """(alphas, sse rows, trace): trace[p] lists (alpha, improvements in that iteration) per iteration run."""
    x, y, bs, tx = int(it["x"]), int(it["y"]), int(it["bsize"]), int(it["tx_size"])
    alphas, sse, trace = [0, 0], np.full((2, NALPHA), SSE_MAX, np.uint64), [[], []]
    if not valid(F, rect, x, y, bs, tx):
        return alphas, sse, trace
    blk = model_block(F, rect, x, y, bs, tx)
    if blk is None:
        return alphas, sse, trace
    l = _wsse()
    fn = l.orc_weighted_sse_u8 if F.rec[0].bpp == 1 else l.orc_weighted_sse_u16
    for p in (1, 2):
        _, _, _, dx, dy = blk["planes"][p - 1]

        def cost(al):
            pred = predict(F, blk, p, al)
            v = fn(F.src[p].at(dx, dy), F.src[p].stride, pred.ctypes.data, blk["tw"], UNIT.ctypes.data, 8,
                   *blk["vis"])
            sse[p - 1][al + 16] = v
            return v
        best = (cost(0), 0)                                 # rdo.rs:1664-1680
        count = 2
        for al in range(1, 17):
            c = (cost(al), cost(-al))
            imp = 0
            if c[0] < best[0]:
                best, count, imp = (c[0], al), count + 2, imp + 1
            if c[1] < best[0]:
                best, count, imp = (c[1], -al), count + 2, imp + 1
            trace[p - 1].append((al, imp))
            if count < al:
                break
        alphas[p - 1] = best[1]
    return alphas, sse, trace


def check(F, rect, items):
    alpha, sse = cfl_alpha(F, rect, items)
    traces = []
    for k, it in enumerate(items):
        ma, ms, tr = model_item(F, rect, it)
        assert list(alpha[k]) == ma, (k, it, list(alpha[k]), ma)
        assert (sse[k] == ms).all(), (k, it)
        traces.append(tr)
    return alpha, sse, traces


def grid_items(rng, rect, bsizes, per_size=None, tx_random=True):
    """Blocks of each size at positions aligned to the size inside the region (every one, or a sample of
    `per_size`), tx_size the size's largest luma tx, or for a third of them a random smaller one."""
    out = []
    for bs in bsizes:
        bw, bh = BSIZES[bs]
        pos = [(x, y) for y in range(0, rect[3], bh) for x in range(0, rect[2], bw)]
        if per_size is not None and len(pos) > per_size:
            pos = [pos[i] for i in rng.choice(len(pos), per_size, replace=False)]
        for x, y in pos:
            tx = largest_luma_tx(bs)
            if tx_random and rng.random() < 0.33:
                cands = [t for t, (w, h) in enumerate(O.TX_SIZES) if w <= bw and h <= bh]
                tx = int(rng.choice(cands))
            out.append((x, y, bs, tx))
    items = np.zeros(len(out), CFL_ITEM_DTYPE)
    for k, (x, y, bs, tx) in enumerate(out):
        items[k]["x"], items[k]["y"], items[k]["bsize"], items[k]["tx_size"] = x, y, bs, tx
    return items


def odd_items(rect, bsizes=(0, 1, 2)):
    """Sub-8x8 blocks at every 4x4 position of the region: odd and even, on the tile's top row and left
    column (all four prediction variants)."""
    out = [(x, y, bs) for bs in bsizes for y in range(0, rect[3], 4) for x in range(0, rect[2], 4)]
    items = np.zeros(len(out), CFL_ITEM_DTYPE)
    for k, (x, y, bs) in enumerate(out):
        items[k]["x"], items[k]["y"], items[k]["bsize"], items[k]["tx_size"] = x, y, bs, largest_luma_tx(bs)
    return items


# ------------------------------------------------------------------ coverage
@pytest.mark.parametrize("xdec,ydec", LAYOUTS)
@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_every_allowed_size_in_tiles(xdec, ydec, dtype, bd):
    """Every cfl_allowed size (and the sizes past BLOCK_32X32, which are invalid), tiles at and off the plane
    origin, a frame whose size is odd and not a multiple of 8."""
    rng = np.random.default_rng(100 * xdec + 10 * ydec + bd)
    W, H = 101, 75
    F = make_frame(rng, W, H, xdec, ydec, bd, dtype)
    for rect in ((0, 0, 104, 80), (32, 16, 72, 64), (64, 48, 40, 32)):
        items = grid_items(rng, rect, range(22), per_size=24)
        alpha, sse, _ = check(F, rect, items)
        # something was evaluated, and every invalid size got the sentinels
        assert (sse != SSE_MAX).any()
        bad = items["bsize"] > BLOCK_32X32
        assert (sse[bad] == SSE_MAX).all() and (alpha[bad] == 0).all()


@pytest.mark.parametrize("xdec,ydec", LAYOUTS)
def test_sub8x8_blocks_at_odd_positions_and_tile_edges(xdec, ydec):
    rng = np.random.default_rng(7 + xdec + ydec)
    W, H = 70, 46
    for dtype, bd in DEPTHS:
        F = make_frame(rng, W, H, xdec, ydec, bd, dtype)
        for rect in ((0, 0, 72, 48), (24, 16, 48, 32)):
            items = odd_items(rect)
            alpha, sse, _ = check(F, rect, items)
            if (xdec, ydec) == (1, 1):
                odd = (items["x"] % 8 == 4) & (items["y"] % 8 == 4) & (items["bsize"] == 0)
                assert odd.any() and (sse[odd] != SSE_MAX).any()     # only the odd 4x4 carry chroma


def test_422_shapes_without_a_subsampled_size_are_invalid():
    rng = np.random.default_rng(5)
    F = make_frame(rng, 64, 64, 1, 0, 8, np.uint8)
    items = grid_items(rng, (0, 0, 64, 64), [1, 4, 7, 3, 6, 9], tx_random=False)
    alpha, sse, _ = check(F, (0, 0, 64, 64), items)
    bad = np.isin(items["bsize"], [1, 4, 7])
    assert (sse[bad] == SSE_MAX).all() and (sse[~bad] != SSE_MAX).any()


def test_invalid_items_get_the_sentinels():
    rng = np.random.default_rng(13)
    F = make_frame(rng, 96, 96, 1, 1, 8, np.uint8)
    rect = (16, 16, 64, 64)
    rows = [(8, 8, 11, 3), (8, 8, 10, 3), (8, 8, 16, 0), (8, 8, 19, 0),  # 64x32, 32x64, 4x16, 32x8
            (8, 8, 3, 19), (8, 8, 3, 2), (8, 8, 5, 7),                   # tx 19, 16x16 in 8x8, 8x16 in 16x8
            (64, 8, 3, 1), (8, -4, 3, 1), (6, 8, 3, 1), (8, 10, 3, 1),   # outside, not a multiple of 4
            (0, 0, 0, 0),                                                 # 4x4 at an even position: no chroma
            (8, 8, 3, 1), (12, 12, 0, 0), (0, 0, 9, 2), (8, 8, 9, 3)]     # valid (alignment is not checked)
    items = np.zeros(len(rows), CFL_ITEM_DTYPE)
    for k, (x, y, bs, tx) in enumerate(rows):
        items[k]["x"], items[k]["y"], items[k]["bsize"], items[k]["tx_size"] = x, y, bs, tx
    alpha, sse, _ = check(F, rect, items)
    assert (sse[:12] == SSE_MAX).all() and (alpha[:12] == 0).all()
    assert (sse[12:] != SSE_MAX).any(axis=(1, 2)).all()


def test_visible_area_partial_chunks_and_zero():
    """Frames whose chroma is 1..3 pixels wide past the last whole chunk (those pixels are dropped), a 4:2:0
    sub-8x8 block whose visible x is 2 (mod 4), and blocks with no visible chroma at all."""
    rng = np.random.default_rng(17)
    for (xdec, ydec), (W, H) in (((1, 1), (37, 29)), ((0, 0), (35, 30)), ((1, 0), (42, 27)), ((1, 1), (43, 45))):
        F = make_frame(rng, W, H, xdec, ydec, 10, np.uint16)
        rect = (0, 0, (W + 7) // 8 * 8, (H + 7) // 8 * 8)
        items = np.concatenate([grid_items(rng, rect, range(10), tx_random=False), odd_items(rect)])
        alpha, sse, _ = check(F, rect, items)
        nothing = (sse == SSE_MAX).all(axis=(1, 2))
        assert nothing.any() and (~nothing).any()
    # 4:2:0, W = 38: the chroma frame is 19 wide.  A 4x4 block at luma x = 36 (odd 4x4 column) has its chroma
    # origin at 16 but its visible x at 18: visible width 1, no whole chunk, SSE 0 for every alpha evaluated
    F = make_frame(rng, 38, 40, 1, 1, 8, np.uint8)
    items = np.zeros(1, CFL_ITEM_DTYPE)
    items[0]["x"], items[0]["y"] = 36, 4
    alpha, sse, tr = check(F, (0, 0, 40, 40), items)
    assert (sse[0][:, 13:20] == 0).all() and (sse[0][:, :13] == SSE_MAX).all() and (alpha[0] == 0).all()


def test_luma_past_the_visible_width_is_read():
    """luma_ac reads the reconstructed luma in [width, align8(width)) (and up to the tx width past it): changing
    only those columns and rows changes the result, and both runs equal the restatement."""
    rng = np.random.default_rng(19)
    W, H = 83, 59
    F = make_frame(rng, W, H, 1, 1, 8, np.uint8)
    rect = (0, 0, 88, 64)
    items = grid_items(rng, rect, range(10), tx_random=False)
    a0, s0, _ = check(F, rect, items)
    lp = F.rec[0]
    lp.data[:, lp.pad + W:] = rng.integers(0, 256, lp.data[:, lp.pad + W:].shape)
    lp.data[lp.pad + H:, :] = rng.integers(0, 256, lp.data[lp.pad + H:, :].shape)
    a1, s1, _ = check(F, rect, items)
    assert (s0 != s1).any()


def test_luma_tx_smaller_than_the_block():
    """32x32 with TX_16X16 (and the other smaller tx sizes) at the frame's right / bottom edge, where max_luma_w
    rounds frame_clipped_bw up to the tx size rather than the block."""
    rng = np.random.default_rng(23)
    W, H = 72, 72
    F = make_frame(rng, W, H, 1, 1, 8, np.uint8)
    rows = []
    for tx in range(19):
        tw, th = O.TX_SIZES[tx]
        if tw <= 32 and th <= 32:
            rows += [(64, 0, 9, tx), (0, 64, 9, tx), (64, 64, 9, tx), (64, 32, 9, tx)]
    items = np.zeros(len(rows), CFL_ITEM_DTYPE)
    for k, (x, y, bs, tx) in enumerate(rows):
        items[k]["x"], items[k]["y"], items[k]["bsize"], items[k]["tx_size"] = x, y, bs, tx
    alpha, sse, _ = check(F, (0, 0, 72, 72), items)
    big = sse[items["tx_size"] == 3]
    small = sse[items["tx_size"] == 2]
    assert (big != small).any()                            # TX_32X32 vs TX_16X16: different w_pad


# ------------------------------------------------------------------ the early exit
def flat_frame(W, H, xdec, ydec, bd, dtype, v):
    cw, ch = (W + xdec) >> xdec, (H + ydec) >> ydec
    imgs = [np.full((H + 32, W + 32), v, dtype)] + [np.full((ch, cw), v, dtype) for _ in range(2)]
    return Frame(imgs, [imgs[0]] + [i.copy() for i in imgs[1:]], xdec, ydec, W, H, bd)


def test_flat_content_stops_after_seven_alphas():
    for dtype, bd in DEPTHS:
        F = flat_frame(64, 64, 1, 1, bd, dtype, (1 << bd) // 3)
        rect = (0, 0, 64, 64)
        items = grid_items(np.random.default_rng(0), rect, range(10), tx_random=False)
        keep = [(x >= 8 and y >= 8 and valid(F, rect, x, y, b, t)) for x, y, b, t in
                zip(items["x"], items["y"], items["bsize"], items["tx_size"])]
        items = items[np.array(keep)]                             # away from the tile's DC constants
        alpha, sse, _ = check(F, rect, items)
        live = (sse != SSE_MAX).any(axis=(1, 2))
        assert live.all() and (alpha == 0).all()
        assert ((sse != SSE_MAX).sum(axis=2) == 7).all()          # 0, +-1, +-2, +-3
        assert (sse[:, :, 13:20] == 0).all()


def plant(F, rect, it, targets):
    """Write dc + scaled(alpha*, ac) (the prediction at alpha*) of each plane into src at the block, so the
    search's minimum is alpha*.  targets = (alpha* of plane 1, of plane 2); None leaves the plane flat at DC."""
    blk = model_block(F, rect, int(it["x"]), int(it["y"]), int(it["bsize"]), int(it["tx_size"]))
    assert blk is not None
    for p in (1, 2):
        _, _, _, dx, dy = blk["planes"][p - 1]
        pred = predict(F, blk, p, targets[p - 1] or 0)
        s = F.src[p]
        s.data[s.pad + dy:s.pad + dy + blk["th"], s.pad + dx:s.pad + dx + blk["tw"]] = pred


def test_planted_alphas_are_found():
    """Chroma = dc + scaled(alpha*, ac) for alpha* over -16..16: the search finds alpha*; ±16 and the other
    large values are reachable only through one improvement per iteration."""
    for (xdec, ydec), (dtype, bd) in zip(LAYOUTS, DEPTHS):
        rng = np.random.default_rng(29 + bd)
        W, H = 128, 96
        F = make_frame(rng, W, H, xdec, ydec, bd, dtype)
        F.rec[0] = Frame._plane(random_image(rng, W + 32, H + 32, bd, dtype, amp=0.6))
        rect = (0, 0, W, H)
        items = grid_items(rng, rect, [6, 9], tx_random=False)      # 16x16, 32x32: disjoint chroma blocks
        items = items[(items["x"] > 0) & (items["y"] > 0)][:33]
        wanted = []
        for k, it in enumerate(items):
            a_u = [-16, 16, -9, 9, 12, -12, 5, -5, 1, -1, 2, -2, 3, -3, 4, -4, 0][k % 17]
            a_v = -a_u if k % 3 else 16 - (k % 7)
            plant(F, rect, it, (a_u, a_v))
            wanted.append((a_u, a_v))
        alpha, sse, traces = check(F, rect, items)
        assert [tuple(a) for a in alpha] == wanted
        for (au, av), s in zip(wanted, sse):
            assert s[0][au + 16] == 0 and s[1][av + 16] == 0


def dc_zero_444(bd, dtype, targets_p, targets_n):
    """A 4:4:4 4x4 block at (8, 8) of a black chroma reconstruction (DC 0) whose luma is 100 +- 8 in a checker
    board: AC +-64, so scaled(alpha, ac) = +-alpha.  Pixels with AC +64 want their target `targets_p`, pixels
    with AC -64 `targets_n`.  The prediction clamps at 0, so the cost falls on both sides of alpha 0."""
    W, H = 32, 32
    luma = np.full((H + 32, W + 32), 100 << (bd - 8), dtype)
    chk = (np.add.outer(np.arange(4), np.arange(4)) % 2 == 0)
    luma[8:12, 8:12] = np.where(chk, (100 << (bd - 8)) + 8, (100 << (bd - 8)) - 8)
    black = np.zeros((H, W), dtype)
    src = np.zeros((H, W), dtype)
    src[8:12, 8:12] = np.where(chk, targets_p, targets_n)
    F = Frame([luma, black, black.copy()], [luma, src, src.copy()], 0, 0, W, H, bd)
    items = np.zeros(1, CFL_ITEM_DTYPE)
    items[0]["x"], items[0]["y"], items[0]["bsize"], items[0]["tx_size"] = 8, 8, 0, 0
    return F, items


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_both_signs_improve_in_one_iteration(dtype, bd):
    """AC +64 pixels want alpha 3, AC -64 pixels want alpha -5 (equal counts): at alpha 1 both +1 and -1 beat
    the best, so count grows by 4; -5 wins."""
    F, items = dc_zero_444(bd, dtype, 3, 5)
    alpha, sse, traces = check(F, (0, 0, 32, 32), items)
    assert tuple(alpha[0]) == (-5, -5)
    assert traces[0][0][0] == (1, 2)


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_exact_ties_keep_the_earlier_alpha(dtype, bd):
    """Both halves want alpha 4 in their own sign: cost(+a) == cost(-a) at every a, and +a (evaluated first)
    wins; and a block whose AC is too small to move the prediction at alpha 1 ties cost(+-1) with cost(0),
    where 0 stays."""
    F, items = dc_zero_444(bd, dtype, 4, 4)
    alpha, sse, traces = check(F, (0, 0, 32, 32), items)
    assert tuple(alpha[0]) == (4, 4)
    assert (sse[0][:, 16 + 4] == sse[0][:, 16 - 4]).all()
    # AC +-8: scaled(1, 8) = (8 + 32) >> 6 = 0
    W, H = 32, 32
    luma = np.full((H + 32, W + 32), 100, dtype)
    chk = (np.add.outer(np.arange(4), np.arange(4)) % 2 == 0)
    luma[8:12, 8:12] = np.where(chk, 101, 99)
    black = np.zeros((H, W), dtype)
    src = np.zeros((H, W), dtype)
    src[8:12, 8:12] = np.where(chk, 1, 0)
    F = Frame([luma, black, black.copy()], [luma, src, src.copy()], 0, 0, W, H, bd)
    alpha, sse, traces = check(F, (0, 0, 32, 32), items)
    assert tuple(alpha[0]) == (0, 0) and sse[0][0][15] == sse[0][0][16] == sse[0][0][17]


def test_one_plane_zero_and_both_zero():
    rng = np.random.default_rng(31)
    W, H = 64, 64
    F = make_frame(rng, W, H, 1, 1, 8, np.uint8)
    F.rec[0] = Frame._plane(random_image(rng, W + 32, H + 32, 8, np.uint8, amp=0.6))
    rect = (0, 0, W, H)
    items = grid_items(rng, rect, [6], tx_random=False)[5:8]
    plant(F, rect, items[0], (7, None))
    plant(F, rect, items[1], (None, -6))
    plant(F, rect, items[2], (None, None))
    alpha, sse, _ = check(F, rect, items)
    assert [tuple(a) for a in alpha] == [(7, 0), (0, -6), (0, 0)]
