"""GPU parity for b200_inter_mode_screen_dev == orc_inter_mode_screen (rdo.rs:1281-1363 with predict_inter,
predict.rs:284-421), bit for bit in both outputs: every block size in tiles, blocks overhanging the frame,
vectors that hit PlaneSlice::clamp on every side, 8 / 10 / 12 bit, single-only, compound-only and mixed lists
over up to 7 references, flat content, a 1080p region with every size mixed in one call; then invalid items
beside valid ones, each output alone, and the host-side rejections."""
import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_oracle_intra_edges import BSIZES
from tests.test_oracle_inter_screen import (DEPTHS, ENTRIES, SCREEN_SIZES, SINGLE, host_plane, inter_mode_screen,
                                            list_item, make_item, origins, random_block_list, random_image,
                                            random_items)

pytestmark = pytest.mark.gpu

SRC_PAD = 64


def ref_pad(bd):
    return max(*origins(bd), 71)


def run_device(src_img, ref_imgs, rect, filter_mode, bd, items, want_satd=True, want_order=True):
    c = G.ctx()
    xo, yo = origins(bd)
    src = c.plane_from_host(src_img, SRC_PAD)
    refs = [c.plane_from_host(r, ref_pad(bd)) for r in ref_imgs]
    n = len(items)
    d_satd = G.dev_empty(n * ENTRIES * 4) if want_satd else None
    d_order = G.dev_empty(n * ENTRIES) if want_order else None
    c.inter_mode_screen_dev(src, rect, refs, xo, yo, filter_mode, bd, G.to_dev(items), n, d_satd, d_order)
    c.synchronize()
    satd = G.from_dev(d_satd, np.uint32)[:n * ENTRIES].reshape(n, ENTRIES) if want_satd else None
    order = G.from_dev(d_order, np.uint8)[:n * ENTRIES].reshape(n, ENTRIES) if want_order else None
    for p in [src] + refs:
        c.plane_free(p)
    return satd, order


def check(src_img, ref_imgs, rect, filter_mode, bd, items):
    xo, yo = origins(bd)
    src = host_plane(src_img, SRC_PAD)
    refs = [host_plane(r, ref_pad(bd)) for r in ref_imgs]
    want_satd, want_order = inter_mode_screen(src, rect, refs, xo, yo, filter_mode, bd, items)
    satd, order = run_device(src_img, ref_imgs, rect, filter_mode, bd, items)
    bad = np.nonzero((satd != want_satd).any(1) | (order != want_order).any(1))[0]
    assert len(bad) == 0, (len(bad), items[bad[:2]], satd[bad[:2]], want_satd[bad[:2]])
    return satd, order


def images(rng, w, h, bd, dtype, nrefs, smooth=True):
    return (random_image(rng, w, h, bd, dtype, smooth=smooth),
            [random_image(rng, w, h, bd, dtype, smooth=smooth) for _ in range(nrefs)])


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_every_block_size_in_tiles(dtype, bd):
    rng = np.random.default_rng(100 + bd)
    W, H = 300, 236
    src_img, ref_imgs = images(rng, W, H, bd, dtype, 3)
    for k, rect in enumerate(((0, 0, W, H), (64, 48, W - 64, H - 48), (128, 64, 128, 128))):
        items = random_items(rng, rect[2], rect[3], 380, 3)
        check(src_img, ref_imgs, rect, k, bd, items)


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_blocks_overhanging_the_frame_and_the_clamp_on_every_side(dtype, bd):
    rng = np.random.default_rng(7 + bd)
    W, H = 150, 110
    src_img, ref_imgs = images(rng, W, H, bd, dtype, 2, smooth=False)
    items = []
    for bs in SCREEN_SIZES:
        bw, bh = BSIZES[bs]
        for x, y in ((0, 0), (((W - 1) // bw) * bw, ((H - 1) // bh) * bh), (((W - 1) // bw) * bw, 0)):
            ents = []
            for row, col in ((0, -8 * 4000), (0, 8 * 4000), (-8 * 4000, 0), (8 * 4000, 0),
                             (8 * (H - y + 16) + 3, 8 * (W - x + 16) + 5), (-8 * (y + 200) - 1, -8 * (x + 150) + 2),
                             (-32767, 32767), (32767, -32768), (8 * (H - y) - 4, 8 * (W - x) - 9)):
                ents.append((int(rng.integers(0, 2)), None, (row, col), None))
            ents.append((0, 1, (8 * (H + 40), 0), (0, -8 * (W + 200) + 6)))
            ents.append((1, 0, (-8 * 300, 8 * 500 + 4), (8 * 3 + 1, 8 * 2)))
            items.append(make_item(x, y, bs, ents))
    check(src_img, ref_imgs, (0, 0, W, H), 2, bd, np.array(items))


@pytest.mark.parametrize("kind", ["single", "compound", "mixed"])
def test_lists_up_to_20_entries_over_7_references(kind):
    rng = np.random.default_rng(len(kind))
    for dtype, bd in DEPTHS:
        W, H = 192, 160
        src_img, ref_imgs = images(rng, W, H, bd, dtype, 7)
        items = random_items(rng, W, H, 190, 7, compound=kind != "single")
        for it in items:
            it["n"] = ENTRIES if rng.integers(0, 2) else it["n"]
            for k in range(ENTRIES):
                c = it["cands"][k]
                if kind == "single":
                    c["ref"][1] = SINGLE
                elif kind == "compound" or (kind == "mixed" and k % 3 == 0):
                    c["ref"][1] = int(rng.integers(0, 7))
                    c["mv"][1] = rng.integers(-200, 201, 2)
        check(src_img, ref_imgs, (0, 0, W, H), int(rng.integers(0, 4)), bd, items)


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_realistic_lists(dtype, bd):
    """Items from the mode-list model (rdo.rs:1158-1318): two references, with and without near modes."""
    rng = np.random.default_rng(30 + bd)
    W, H = 256, 192
    src_img, ref_imgs = images(rng, W, H, bd, dtype, 2)
    items = []
    for k in range(400):
        bs = SCREEN_SIZES[k % len(SCREEN_SIZES)]
        bw, bh = BSIZES[bs]
        lst = random_block_list(rng, bw, bh, include_near_mvs=bool(k & 1))
        items.append(list_item(int(rng.integers(0, W // bw)) * bw, int(rng.integers(0, H // bh)) * bh, bs, lst))
    check(src_img, ref_imgs, (0, 0, W, H), 0, bd, np.array(items))


def test_flat_content_keeps_the_list_order():
    rng = np.random.default_rng(9)
    for dtype, bd in DEPTHS:
        img = np.full((128, 192), (1 << bd) // 3, dtype)
        items = random_items(rng, 160, 112, 190, 2, reach=300)
        satd, order = check(img, [img.copy(), img.copy()], (32, 16, 160, 112), 0, bd, items)
        assert (order == np.arange(ENTRIES)).all()
        for k, it in enumerate(items):
            assert (satd[k][:it["n"]] == 0).all()


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_1080p_every_size_mixed_in_one_call(dtype, bd):
    rng = np.random.default_rng(1080 + bd)
    W, H = 1920, 1080
    src_img, ref_imgs = images(rng, W, H, bd, dtype, 2)
    for rect in ((0, 0, W, H), (640, 384, 640, 384)):
        items = random_items(rng, rect[2], rect[3], 3000, 2, reach=40)
        rng.shuffle(items)
        check(src_img, ref_imgs, rect, 0, bd, items)


def test_invalid_items_beside_valid_ones():
    rng = np.random.default_rng(13)
    src_img, ref_imgs = images(rng, 96, 96, 8, np.uint8, 2)
    items = random_items(rng, 64, 64, 20, 2, bsizes=[3, 12, 21])
    items[0]["bsize"] = 22
    items[2]["bsize"] = 14
    items[4]["n"] = 21
    items[6]["cands"][0]["ref"][0] = 2
    items[8]["cands"][items[8]["n"] - 1]["ref"][1] = 9
    items[10]["x"] = 64
    items[12]["y"] = -4
    items[14]["x"] = 6
    items[16]["n"] = 0
    satd, order = check(src_img, ref_imgs, (16, 16, 64, 64), 0, 8, items)
    for k in (0, 2, 4, 6, 8, 10, 12, 14, 16):
        assert (satd[k] == np.uint32(0xFFFFFFFF)).all() and (order[k] == np.arange(ENTRIES)).all()
    for k in (1, 3, 5, 7, 9, 11, 13, 15, 17, 19):
        assert (satd[k][:items[k]["n"]] < 0xFFFFFFFF).all()


def test_each_output_alone():
    rng = np.random.default_rng(17)
    src_img, ref_imgs = images(rng, 128, 96, 10, np.uint16, 2)
    items = random_items(rng, 128, 96, 200, 2)
    xo, yo = origins(10)
    want_satd, want_order = inter_mode_screen(host_plane(src_img, SRC_PAD), (0, 0, 128, 96),
                                              [host_plane(r, ref_pad(10)) for r in ref_imgs], xo, yo, 1, 10, items)
    satd, order = run_device(src_img, ref_imgs, (0, 0, 128, 96), 1, 10, items, want_order=False)
    assert order is None and (satd == want_satd).all()
    satd, order = run_device(src_img, ref_imgs, (0, 0, 128, 96), 1, 10, items, want_satd=False)
    assert satd is None and (order == want_order).all()


def test_host_side_rejections_launch_nothing():
    c = G.ctx()
    img8, img16 = np.zeros((64, 64), np.uint8), np.zeros((64, 64), np.uint16)
    src = c.plane_from_host(img8, 64)
    ref = c.plane_from_host(img8, 128)
    ref16 = c.plane_from_host(img16, 128)
    small = c.plane_from_host(np.zeros((32, 64), np.uint8), 128)
    thin_src = c.plane_from_host(img8, 32)
    thin_ref = c.plane_from_host(img8, 100)           # below xorigin 128
    items = G.to_dev(random_items(np.random.default_rng(0), 64, 64, 4, 1))
    d_satd, d_order = G.dev_empty(4 * ENTRIES * 4), G.dev_empty(4 * ENTRIES)
    r = (0, 0, 64, 64)
    ok = (src, r, [ref], 128, 88, 0, 8, items, 4, d_satd, d_order)
    bad = [
        (src, r, [ref], 128, 88, 0, 9, items, 4, d_satd, d_order),            # bit depth
        (src, r, [ref], 128, 88, 0, 10, items, 4, d_satd, d_order),           # bpp vs bit depth
        (src, r, [ref16], 128, 88, 0, 8, items, 4, d_satd, d_order),          # ref bpp differs
        (src, r, [], 128, 88, 0, 8, items, 4, d_satd, d_order),               # nrefs 0
        (src, r, [ref] * 9, 128, 88, 0, 8, items, 4, d_satd, d_order),        # nrefs 9
        (src, r, [ref, small], 128, 88, 0, 8, items, 4, d_satd, d_order),     # ref size differs
        (src, (8, 0, 64, 64), [ref], 128, 88, 0, 8, items, 4, d_satd, d_order),   # region outside the plane
        (src, (0, -4, 64, 32), [ref], 128, 88, 0, 8, items, 4, d_satd, d_order),
        (src, (0, 0, 0, 64), [ref], 128, 88, 0, 8, items, 4, d_satd, d_order),
        (src, r, [ref], 128, 88, 4, 8, items, 4, d_satd, d_order),            # filter mode
        (src, r, [ref], 128, 88, -1, 8, items, 4, d_satd, d_order),
        (thin_src, r, [ref], 128, 88, 0, 8, items, 4, d_satd, d_order),      # src padding below 64
        (src, r, [thin_ref], 128, 88, 0, 8, items, 4, d_satd, d_order),      # ref padding below xorigin
        (src, r, [ref], 136, 88, 0, 8, items, 4, d_satd, d_order),
        (src, r, [ref], 0, 130, 0, 8, items, 4, d_satd, d_order),             # ... below yorigin
        (src, r, [ref], -1, 88, 0, 8, items, 4, d_satd, d_order),             # negative origin
        (src, r, [ref], 128, -8, 0, 8, items, 4, d_satd, d_order),
        (src, r, [ref], 128, 88, 0, 8, items, 4, None, None),                 # both outputs NULL
        (src, r, [ref], 128, 88, 0, 8, None, 4, d_satd, d_order),            # NULL items
    ]
    before = c.L.b200_ctx_launch_count(c.h)
    for args in bad:
        with pytest.raises(B.B200Error) as e:
            c.inter_mode_screen_dev(*args)
        assert e.value.status == B.ERR_ARG, args[1:7]
    assert c.L.b200_ctx_launch_count(c.h) == before
    c.inter_mode_screen_dev(*ok[:8], 0, d_satd, d_order)                      # no items: nothing to launch
    assert c.L.b200_ctx_launch_count(c.h) == before
    c.inter_mode_screen_dev(*ok)
    c.synchronize()
    assert c.L.b200_ctx_launch_count(c.h) == before + 4                      # bucketing + three size classes
    for p in (src, ref, ref16, small, thin_src, thin_ref):
        c.plane_free(p)
