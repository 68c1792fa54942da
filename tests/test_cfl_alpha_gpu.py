"""GPU parity for b200_cfl_alpha_dev == orc_cfl_alpha (rdo_cfl_alpha, rdo.rs:1593-1689, with luma_ac and
clip_visible_bsize), bit for bit in d_alpha and d_sse: every cfl_allowed size in 4:2:0 / 4:2:2 / 4:4:4 at
8 / 10 / 12 bit, sub-8x8 blocks at odd positions, tiles off the origin, odd frame sizes, partial chunks and
empty visible areas, small luma tx sizes, the early exit's constructions, a 1080p 4:2:0 call with every size
mixed; then invalid items next to valid ones, each output alone, every host-side rejection, rec and src left
untouched, and a cross-check against the existing AC, edge and prediction calls composed by hand."""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_oracle_cfl_alpha import (CFL_ITEM_DTYPE, DEPTHS, LAYOUTS, NALPHA, SSE_MAX, Frame,
                                         cfl_alpha, dc_zero_444, flat_frame, grid_items, make_frame, odd_items,
                                         plant, random_image, valid)
from tests.test_oracle_intra_edges import BSIZES

pytestmark = pytest.mark.gpu

PAD = 64


def upload(F):
    c = G.ctx()
    return [c.plane_from_host(p.view(), PAD) for p in F.rec], [c.plane_from_host(p.view(), PAD) for p in F.src]


def free(*plane_lists):
    c = G.ctx()
    for pl in plane_lists:
        for p in pl:
            c.plane_free(p)


def run_device(F, rect, items, want_alpha=True, want_sse=True, planes=None):
    c = G.ctx()
    rec, src = planes if planes is not None else upload(F)
    n = len(items)
    d_alpha = G.dev_empty(n * 2) if want_alpha else None
    d_sse = G.dev_empty(n * 2 * NALPHA * 8) if want_sse else None
    c.cfl_alpha_dev(rec, src, F.xdec, F.ydec, rect, F.width, F.height, F.bd, G.to_dev(items), n, d_alpha, d_sse)
    c.synchronize()
    if planes is None:
        free(rec, src)
    alpha = G.from_dev(d_alpha, np.int8)[:n * 2].reshape(n, 2) if want_alpha else None
    sse = G.from_dev(d_sse, np.uint64)[:n * 2 * NALPHA].reshape(n, 2, NALPHA) if want_sse else None
    return alpha, sse


def check(F, rect, items):
    want_alpha, want_sse = cfl_alpha(F, rect, items)
    alpha, sse = run_device(F, rect, items)
    bad = np.nonzero((alpha != want_alpha).any(1) | (sse != want_sse).any((1, 2)))[0]
    assert len(bad) == 0, (len(bad), items[bad[:4]], alpha[bad[:4]], want_alpha[bad[:4]])
    return alpha, sse


@pytest.mark.parametrize("xdec,ydec", LAYOUTS)
@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_every_allowed_size_in_tiles(xdec, ydec, dtype, bd):
    rng = np.random.default_rng(200 + 100 * xdec + 10 * ydec + bd)
    W, H = 101, 75
    F = make_frame(rng, W, H, xdec, ydec, bd, dtype)
    for rect in ((0, 0, 104, 80), (32, 16, 72, 64), (64, 48, 40, 32)):
        items = grid_items(rng, rect, range(22))
        rng.shuffle(items)
        check(F, rect, items)


@pytest.mark.parametrize("xdec,ydec", LAYOUTS)
def test_sub8x8_blocks_at_odd_positions_and_tile_edges(xdec, ydec):
    rng = np.random.default_rng(27 + xdec + ydec)
    for dtype, bd in DEPTHS:
        F = make_frame(rng, 70, 46, xdec, ydec, bd, dtype)
        for rect in ((0, 0, 72, 48), (24, 16, 48, 32)):
            check(F, rect, odd_items(rect))


def test_visible_area_partial_chunks_and_zero():
    rng = np.random.default_rng(37)
    for (xdec, ydec), (W, H) in (((1, 1), (37, 29)), ((0, 0), (35, 30)), ((1, 0), (42, 27)), ((1, 1), (43, 45)),
                                 ((1, 1), (38, 40))):
        for dtype, bd in DEPTHS:
            F = make_frame(rng, W, H, xdec, ydec, bd, dtype)
            rect = (0, 0, (W + 7) // 8 * 8, (H + 7) // 8 * 8)
            check(F, rect, np.concatenate([grid_items(rng, rect, range(10)), odd_items(rect)]))


def test_luma_tx_smaller_than_the_block():
    rng = np.random.default_rng(43)
    for (xdec, ydec), (dtype, bd) in zip(LAYOUTS, DEPTHS):
        F = make_frame(rng, 72, 72, xdec, ydec, bd, dtype)
        rows = [(x, y, bs, tx) for bs in (5, 6, 7, 8, 9) for tx in range(19)
                for x, y in ((64, 0), (0, 64), (64, 64), (64, 32), (48, 48))
                if O.TX_SIZES[tx][0] <= BSIZES[bs][0] and O.TX_SIZES[tx][1] <= BSIZES[bs][1]]
        items = np.zeros(len(rows), CFL_ITEM_DTYPE)
        for k, (x, y, bs, tx) in enumerate(rows):
            items[k]["x"], items[k]["y"], items[k]["bsize"], items[k]["tx_size"] = x, y, bs, tx
        check(F, (0, 0, 72, 72), items)


def test_early_exit_constructions():
    """Flat content (7 alphas), planted alphas over -16..16, both signs improving in one iteration, exact ties,
    one plane at 0 with the other not."""
    for dtype, bd in DEPTHS:
        F = flat_frame(64, 64, 1, 1, bd, dtype, (1 << bd) // 3)
        items = grid_items(np.random.default_rng(0), (0, 0, 64, 64), range(10), tx_random=False)
        alpha, sse = check(F, (0, 0, 64, 64), items)
        live = (sse != SSE_MAX).any(axis=(1, 2))
        assert live.any() and ((sse[live] != SSE_MAX).sum(axis=2) == 7).all()
        for tp, tn, want in ((3, 5, -5), (4, 4, 4)):
            F, items = dc_zero_444(bd, dtype, tp, tn)
            alpha, _ = check(F, (0, 0, 32, 32), items)
            assert tuple(alpha[0]) == (want, want)
    for (xdec, ydec), (dtype, bd) in zip(LAYOUTS, DEPTHS):
        rng = np.random.default_rng(59 + bd)
        W, H = 128, 96
        F = make_frame(rng, W, H, xdec, ydec, bd, dtype)
        F.rec[0] = Frame._plane(random_image(rng, W + 32, H + 32, bd, dtype, amp=0.6))
        rect = (0, 0, W, H)
        items = grid_items(rng, rect, [6, 9], tx_random=False)
        items = items[(items["x"] > 0) & (items["y"] > 0)][:34]
        wanted = []
        for k, it in enumerate(items):
            a_u = [-16, 16, -9, 9, 12, -12, 5, -5, 1, -1, 2, -2, 3, -3, 4, -4, 0][k % 17]
            a_v = None if k == 33 else -a_u if k % 3 else 16 - (k % 7)
            plant(F, rect, it, (a_u, a_v))
            wanted.append((a_u, a_v or 0))
        alpha, _ = check(F, rect, items)
        assert [tuple(a) for a in alpha] == wanted


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10)])
def test_1080p_every_size_mixed_in_one_call(dtype, bd):
    """Every chroma-carrying block of every cfl_allowed size of a 1080p 4:2:0 frame (a sample of 40000, in
    random order) in one call, over the whole frame and over a tile inside it."""
    rng = np.random.default_rng(1080 + bd)
    W, H = 1920, 1080
    F = make_frame(rng, W, H, 1, 1, bd, dtype)
    for rect in ((0, 0, W, 1080), (640, 384, 640, 384)):
        items = grid_items(rng, rect, range(10))
        keep = np.array([valid(F, rect, int(i["x"]), int(i["y"]), int(i["bsize"]), int(i["tx_size"])) for i in items])
        items = items[keep]
        items = items[rng.permutation(len(items))[:40000]]
        check(F, rect, items)


@pytest.mark.parametrize("xdec,ydec", [(1, 0), (0, 0)])
def test_422_and_444_frames_every_size_mixed(xdec, ydec):
    rng = np.random.default_rng(422 + xdec + ydec)
    for dtype, bd in DEPTHS:
        F = make_frame(rng, 333, 197, xdec, ydec, bd, dtype)
        items = np.concatenate([grid_items(rng, (0, 0, 336, 200), range(22)), odd_items((64, 64, 64, 64))])
        rng.shuffle(items)
        check(F, (0, 0, 336, 200), items)


def test_invalid_items_beside_valid_ones():
    rng = np.random.default_rng(61)
    F = make_frame(rng, 96, 96, 1, 1, 8, np.uint8)
    rect = (16, 16, 64, 64)
    rows = [(8, 8, 11, 3), (8, 8, 3, 1), (8, 8, 16, 0), (12, 12, 0, 0), (8, 8, 3, 19), (0, 0, 9, 2),
            (64, 8, 3, 1), (8, 8, 9, 3), (6, 8, 3, 1), (16, 16, 6, 2), (0, 0, 0, 0), (4, 4, 0, 0), (8, 8, 5, 7)]
    items = np.zeros(len(rows), CFL_ITEM_DTYPE)
    for k, (x, y, bs, tx) in enumerate(rows):
        items[k]["x"], items[k]["y"], items[k]["bsize"], items[k]["tx_size"] = x, y, bs, tx
    alpha, sse = check(F, rect, items)
    for k in (0, 2, 4, 6, 8, 10, 12):
        assert (sse[k] == SSE_MAX).all() and (alpha[k] == 0).all()
    for k in (1, 3, 5, 7, 9, 11):
        assert (sse[k] != SSE_MAX).any()


def test_each_output_alone():
    rng = np.random.default_rng(67)
    F = make_frame(rng, 128, 96, 1, 1, 10, np.uint16)
    items = grid_items(rng, (0, 0, 128, 96), range(10))
    want_alpha, want_sse = cfl_alpha(F, (0, 0, 128, 96), items)
    alpha, sse = run_device(F, (0, 0, 128, 96), items, want_sse=False)
    assert sse is None and (alpha == want_alpha).all()
    alpha, sse = run_device(F, (0, 0, 128, 96), items, want_alpha=False)
    assert alpha is None and (sse == want_sse).all()


def download(p):
    c = G.ctx()
    out = np.zeros((p.height, p.width), np.uint8 if p.bpp == 1 else np.uint16)
    c.check(c.L.b200_plane_download(c.h, C.byref(p), out.ctypes.data, out.strides[0]))
    return out


def test_rec_and_src_are_not_written():
    rng = np.random.default_rng(71)
    F = make_frame(rng, 96, 64, 1, 1, 8, np.uint8)
    rec, src = upload(F)
    before = [download(p) for p in rec + src]
    items = grid_items(rng, (0, 0, 96, 64), range(10))
    alpha, sse = run_device(F, (0, 0, 96, 64), items, planes=(rec, src))
    want_alpha, want_sse = cfl_alpha(F, (0, 0, 96, 64), items)
    assert (alpha == want_alpha).all() and (sse == want_sse).all()
    after = [download(p) for p in rec + src]
    assert all((a == b).all() for a, b in zip(before, after))
    free(rec, src)


def test_host_side_rejections_launch_nothing():
    c = G.ctx()
    rng = np.random.default_rng(73)
    F = make_frame(rng, 64, 64, 1, 1, 8, np.uint8)
    rec, src = upload(F)
    F16 = make_frame(rng, 64, 64, 1, 1, 10, np.uint16)
    rec16, src16 = upload(F16)
    small_c = c.plane_from_host(np.zeros((31, 32), np.uint8), PAD)
    big_c = c.plane_from_host(np.zeros((40, 40), np.uint8), PAD)
    lum64 = c.plane_from_host(np.zeros((64, 64), np.uint8), 30)       # the frame's size, pad 30: one short
    lum64_ok = c.plane_from_host(np.zeros((64, 64), np.uint8), 31)
    items = grid_items(rng, (0, 0, 64, 64), range(10))
    n = len(items)
    d_items = G.to_dev(items)
    d_alpha, d_sse = G.dev_empty(n * 2), G.dev_empty(n * 2 * NALPHA * 8)
    d_alpha.fill_(0x5A)
    d_sse.fill_(0x5A)
    ok = dict(rec=rec, src=src, xdec=1, ydec=1, rect=(0, 0, 64, 64), width=64, height=64, bit_depth=8,
              d_items=d_items, n=n, d_alpha=d_alpha, d_sse=d_sse)

    def call(**kw):
        a = dict(ok, **kw)
        c.cfl_alpha_dev(a["rec"], a["src"], a["xdec"], a["ydec"], a["rect"], a["width"], a["height"],
                        a["bit_depth"], a["d_items"], a["n"], a["d_alpha"], a["d_sse"])
    bad = [
        dict(d_alpha=None, d_sse=None),                                   # both outputs NULL
        dict(d_items=None),                                               # NULL items
        dict(bit_depth=9), dict(bit_depth=10),                            # bit depth, bpp vs bit depth
        dict(rec=rec16, src=src16),                                       # 16-bit planes at 8 bit
        dict(rec=[rec[0], rec16[1], rec[2]]),                             # one plane's bpp differs
        dict(xdec=0, ydec=1), dict(xdec=2, ydec=1),                       # layouts
        dict(rec=[rec[0], small_c, rec[2]], src=[src[0], small_c, src[2]]),   # chroma smaller than the frame
        dict(src=[src[0], big_c, src[2]]),                                # src / rec chroma sizes differ
        dict(width=72), dict(height=80),                                  # luma smaller than the frame
        dict(rect=(4, 0, 56, 64)), dict(rect=(0, 12, 64, 48)),            # origin not 8-aligned
        dict(rect=(0, 0, 72, 64)), dict(rect=(0, 0, 64, 72)),             # outside the frame's 8x8 blocks
        dict(rect=(-8, 0, 64, 64)), dict(rect=(0, 0, 0, 64)),
        dict(rec=[lum64, rec[1], rec[2]]),                                # luma pad 30 < 31
        dict(width=0),
    ]
    before = c.launches
    for kw in bad:
        with pytest.raises(B.B200Error) as e:
            call(**kw)
        assert e.value.status == B.ERR_ARG, kw
    assert c.launches == before
    call(n=0)                                                             # no items: nothing to launch
    assert c.launches == before
    c.synchronize()
    assert (G.from_dev(d_alpha, np.uint8) == 0x5A).all() and (G.from_dev(d_sse, np.uint8) == 0x5A).all()
    call(rec=[lum64_ok, rec[1], rec[2]])                                  # pad 31 is enough
    c.synchronize()
    assert c.launches == before + 1
    call()
    c.synchronize()
    want_alpha, want_sse = cfl_alpha(F, (0, 0, 64, 64), items)
    assert (G.from_dev(d_alpha, np.int8)[:n * 2].reshape(n, 2) == want_alpha).all()
    assert (G.from_dev(d_sse, np.uint64)[:n * 2 * NALPHA].reshape(n, 2, NALPHA) == want_sse).all()
    free(rec, src, rec16, src16, [small_c, big_c, lum64, lum64_ok])


def test_matches_the_existing_calls_composed_by_hand():
    """Interior 16x16 and 32x32 blocks of a 4:2:0 frame (w_pad = h_pad = 0): b200_pred_cfl_ac_dev, then
    b200_get_intra_edges_dev per chroma plane, then b200_predict_intra_dev with 33 items per (block, plane); the
    SSE over whole chunks and the selection on the host.  Both must equal the fused call."""
    c = G.ctx()
    rng = np.random.default_rng(79)
    for dtype, bd in ((np.uint8, 8), (np.uint16, 10)):
        W, H = 256, 192
        F = make_frame(rng, W, H, 1, 1, bd, dtype)
        rect = (64, 64, 128, 128)
        rec, src = upload(F)
        for bs in (6, 9):
            bw, bh = BSIZES[bs]
            tw, th = bw // 2, bh // 2
            items = grid_items(rng, rect, [bs], tx_random=False)
            n = len(items)
            alpha, sse = run_device(F, rect, items, planes=(rec, src))
            # AC: luma positions in the plane
            blocks = np.zeros(n, B.BLOCK_DTYPE)
            blocks["x"], blocks["y"] = items["x"] + rect[0], items["y"] + rect[1]
            d_ac = G.dev_empty(n * tw * th * 2)
            c.pred_cfl_ac_dev(rec[0], G.to_dev(blocks), n, tw, th, 0, 0, 1, 1, d_ac)
            crect = (rect[0] // 2, rect[1] // 2, rect[2] // 2, rect[3] // 2)
            eitems = np.zeros(n, B.EDGE_ITEM_DTYPE)
            eitems["po_x"], eitems["po_y"] = items["x"] // 2, items["y"] // 2
            eitems["part_x"], eitems["part_y"] = items["x"] // 4, items["y"] // 4
            eitems["bsize"], eitems["tx_size"], eitems["mode"] = bs, O.TX_SIZES.index((tw, th)), 13
            got_sse = np.zeros((n, 2, NALPHA), np.uint64)
            for p in (1, 2):
                d_edges = G.dev_empty(n * O.EDGE_LEN * F.rec[0].bpp)
                d_lens = G.dev_empty(n * 2)
                c.get_intra_edges_dev(rec[p], crect, 1, 1, bd, G.to_dev(eitems), n, d_edges, d_lens)
                c.synchronize()
                lens = G.from_dev(d_lens, np.uint8)[:n * 2].reshape(n, 2)
                pitems = np.zeros(n * NALPHA, B.INTRA_ITEM_DTYPE)
                for k in range(n):
                    px, py = int(eitems[k]["po_x"]), int(eitems[k]["po_y"])
                    for ai in range(NALPHA):
                        r = pitems[k * NALPHA + ai]
                        r["edge"], r["ac"], r["x"], r["y"] = k, k, crect[0] + px, crect[1] + py
                        r["angle"], r["mode"] = ai - 16, 0 if ai == 16 else 13
                        r["variant"] = 0 if (px, py) == (0, 0) else 1 if py == 0 else 2 if px == 0 else 3
                        r["ief"], r["left_len"], r["above_len"] = -1, lens[k][0], lens[k][1]
                d_out = G.dev_empty(n * NALPHA * tw * th * F.rec[0].bpp)
                c.predict_intra_dev(d_edges, G.to_dev(pitems), len(pitems), d_ac, tw, th, bd, rec[p].width,
                                    rec[p].height, d_out)
                c.synchronize()
                preds = G.from_dev(d_out, dtype)[:n * NALPHA * tw * th].reshape(n, NALPHA, th, tw).astype(np.int64)
                sv = F.src[p].view()
                for k in range(n):
                    x0, y0 = crect[0] + int(eitems[k]["po_x"]), crect[1] + int(eitems[k]["po_y"])
                    org = sv[y0:y0 + th, x0:x0 + tw].astype(np.int64)
                    got_sse[k, p - 1] = ((preds[k] - org[None]) ** 2).sum(axis=(1, 2))
            for k in range(n):
                for p in range(2):
                    cost = got_sse[k, p]
                    best, bc, count, seen = 0, cost[16], 2, {0}
                    for al in range(1, 17):
                        seen |= {al, -al}
                        if cost[16 + al] < bc:
                            best, bc, count = al, cost[16 + al], count + 2
                        if cost[16 - al] < bc:
                            best, bc, count = -al, cost[16 - al], count + 2
                        if count < al:
                            break
                    assert alpha[k, p] == best, (k, p)
                    for al in range(-16, 17):
                        assert sse[k, p, al + 16] == (cost[al + 16] if al in seen else SSE_MAX), (k, p, al)
        free(rec, src)
