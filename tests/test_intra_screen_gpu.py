"""GPU parity for b200_intra_mode_screen_dev == orc_intra_mode_screen (rdo.rs:1433-1511 with predict_intra,
predict.rs:205-249), bit for bit in both outputs: every block size, tiles off the plane origin, blocks
overhanging the frame, 8 / 10 / 12 bit, ief -1 / 0 / 1, num_modes_rdo 3 and 7, flat content, a 1080p
region with every block size mixed in one call; then the host-side rejections, invalid items next to
valid ones, and each output alone."""
import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_oracle_intra_edges import BSIZES
from tests.test_oracle_intra_screen import DEPTHS, intra_mode_screen, make_items, planes, random_image

pytestmark = pytest.mark.gpu

PAD = 80


def run_device(rec_img, src_img, rect, bd, num_modes_rdo, items, want_satd=True, want_modes=True):
    c = G.ctx()
    rec = c.plane_from_host(rec_img, PAD)
    src = c.plane_from_host(src_img, PAD)
    n = len(items)
    d_satd = G.dev_empty(n * 13 * 4) if want_satd else None
    d_modes = G.dev_empty(n * 13) if want_modes else None
    c.intra_mode_screen_dev(rec, src, rect, bd, num_modes_rdo, G.to_dev(items), n, d_satd, d_modes)
    c.synchronize()
    satd = G.from_dev(d_satd, np.uint32)[:n * 13].reshape(n, 13) if want_satd else None
    modes = G.from_dev(d_modes, np.uint8)[:n * 13].reshape(n, 13) if want_modes else None
    return satd, modes


def check(rec_img, src_img, rect, bd, num_modes_rdo, items):
    rec, src = planes(rec_img, src_img, PAD)
    want_satd, want_modes = intra_mode_screen(rec, src, rect, bd, num_modes_rdo, items)
    satd, modes = run_device(rec_img, src_img, rect, bd, num_modes_rdo, items)
    bad = np.nonzero((satd != want_satd).any(1) | (modes != want_modes).any(1))[0]
    assert len(bad) == 0, (len(bad), items[bad[:4]], satd[bad[:4]], want_satd[bad[:4]])
    return satd, modes


@pytest.mark.parametrize("dtype,bd", DEPTHS)
@pytest.mark.parametrize("num_modes_rdo", [3, 7])
def test_every_block_size_in_tiles(dtype, bd, num_modes_rdo):
    rng = np.random.default_rng(100 + bd * 10 + num_modes_rdo)
    W, H = 300, 236
    rec_img = random_image(rng, W, H, bd, dtype, smooth=True)
    src_img = random_image(rng, W, H, bd, dtype, smooth=bool(num_modes_rdo & 4))
    for rect in ((0, 0, W, H), (64, 48, W - 64, H - 48), (128, 64, 128, 128)):
        items = make_items(rng, rect[2], rect[3], 660)
        items[:22]["x"] = 0
        items[22:44]["y"] = 0
        items[44:66]["x"] = 0
        items[44:66]["y"] = 0
        check(rec_img, src_img, rect, bd, num_modes_rdo, items)


def test_blocks_overhanging_the_frame():
    rng = np.random.default_rng(7)
    W, H = 150, 110
    for dtype, bd in DEPTHS:
        items = np.concatenate([make_items(rng, W, H, 3, bsizes=[bs]) for bs in range(22)])
        for k, it in enumerate(items):      # the last block column / row, partly outside the frame
            bw, bh = BSIZES[it["bsize"]]
            items[k]["x"] = ((W - 1) // bw) * bw
            items[k]["y"] = ((H - 1) // bh) * bh if k % 3 != 1 else 0
        check(random_image(rng, W, H, bd, dtype), random_image(rng, W, H, bd, dtype), (0, 0, W, H), bd, 3, items)


def test_flat_content_keeps_the_cdf_order():
    rng = np.random.default_rng(9)
    for dtype, bd in DEPTHS:
        img = np.full((128, 192), (1 << bd) // 3, dtype)
        rect = (32, 16, 160, 112)
        items = make_items(rng, rect[2], rect[3], 66)
        items["y"][(items["x"] == 0) & (items["y"] == 0)] = 64
        for num_modes_rdo in (3, 7):
            satd, modes = check(img, img.copy(), rect, bd, num_modes_rdo, items)
            assert (satd == 0).all() and (modes == items["modes"]).all()


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_1080p_every_size_mixed_in_one_call(dtype, bd):
    """A whole frame's worth of blocks of every size in one call, on random and on smooth content, and the
    same over a tile region inside the larger plane."""
    rng = np.random.default_rng(1080 + bd)
    W, H = 1920, 1080
    for smooth in (False, True):
        rec_img = random_image(rng, W, H, bd, dtype, smooth=smooth)
        src_img = random_image(rng, W, H, bd, dtype, smooth=smooth)
        for rect in ((0, 0, W, H), (640, 384, 640, 384)):
            items = make_items(rng, rect[2], rect[3], 6000)
            rng.shuffle(items)
            check(rec_img, src_img, rect, bd, 3 if smooth else 7, items)


def test_invalid_items_beside_valid_ones():
    rng = np.random.default_rng(13)
    img_r, img_s = random_image(rng, 96, 96, 8, np.uint8), random_image(rng, 96, 96, 8, np.uint8)
    items = make_items(rng, 64, 64, 12, bsizes=[3, 12])
    items[0]["bsize"] = 22
    items[2]["modes"][4] = 13
    items[4]["modes"][5] = items[4]["modes"][6]
    items[6]["x"] = 64
    items[8]["y"] = -4
    items[10]["x"] = 6
    items[11]["modes"][0] = 255
    satd, modes = check(img_r, img_s, (16, 16, 64, 64), 8, 3, items)
    for k in (0, 2, 4, 6, 8, 10, 11):
        assert (satd[k] == np.uint32(0xFFFFFFFF)).all() and (modes[k] == items[k]["modes"]).all()
    for k in (1, 3, 5, 7, 9):
        assert sorted(modes[k]) == list(range(13))


def test_each_output_alone():
    rng = np.random.default_rng(17)
    img_r, img_s = random_image(rng, 128, 96, 10, np.uint16), random_image(rng, 128, 96, 10, np.uint16)
    items = make_items(rng, 128, 96, 200)
    rec, src = planes(img_r, img_s, PAD)
    want_satd, want_modes = intra_mode_screen(rec, src, (0, 0, 128, 96), 10, 7, items)
    satd, modes = run_device(img_r, img_s, (0, 0, 128, 96), 10, 7, items, want_modes=False)
    assert modes is None and (satd == want_satd).all()
    satd, modes = run_device(img_r, img_s, (0, 0, 128, 96), 10, 7, items, want_satd=False)
    assert satd is None and (modes == want_modes).all()


def test_host_side_rejections_launch_nothing():
    c = G.ctx()
    img8 = np.zeros((64, 64), np.uint8)
    img16 = np.zeros((64, 64), np.uint16)
    rec = c.plane_from_host(img8, PAD)
    src = c.plane_from_host(img8, PAD)
    rec16 = c.plane_from_host(img16, PAD)
    small = c.plane_from_host(np.zeros((32, 64), np.uint8), PAD)
    thin = c.plane_from_host(img8, 32)
    items = G.to_dev(make_items(np.random.default_rng(0), 64, 64, 4))
    d_satd, d_modes = G.dev_empty(4 * 13 * 4), G.dev_empty(4 * 13)
    ok = (rec, src, (0, 0, 64, 64), 8, 3, items, 4, d_satd, d_modes)
    bad = [
        (rec, src, (0, 0, 64, 64), 8, 5, items, 4, d_satd, d_modes),      # num_modes_rdo
        (rec, src, (0, 0, 64, 64), 8, 1, items, 4, d_satd, d_modes),
        (rec, src, (0, 0, 64, 64), 10, 3, items, 4, d_satd, d_modes),     # bpp vs bit depth
        (rec16, src, (0, 0, 64, 64), 10, 3, items, 4, d_satd, d_modes),   # rec / src bpp differ
        (rec, src, (0, 0, 64, 64), 9, 3, items, 4, d_satd, d_modes),
        (rec, small, (0, 0, 64, 32), 8, 3, items, 4, d_satd, d_modes),    # size mismatch
        (rec, src, (8, 0, 64, 64), 8, 3, items, 4, d_satd, d_modes),      # region outside the plane
        (rec, src, (0, -4, 64, 32), 8, 3, items, 4, d_satd, d_modes),
        (rec, src, (0, 0, 0, 64), 8, 3, items, 4, d_satd, d_modes),
        (thin, src, (0, 0, 64, 64), 8, 3, items, 4, d_satd, d_modes),     # padding below 64
        (rec, thin, (0, 0, 64, 64), 8, 3, items, 4, d_satd, d_modes),
        (rec, src, (0, 0, 64, 64), 8, 3, items, 4, None, None),           # both outputs NULL
        (rec, src, (0, 0, 64, 64), 8, 3, None, 4, d_satd, d_modes),       # NULL items
    ]
    before = c.L.b200_ctx_launch_count(c.h)
    for args in bad:
        with pytest.raises(B.B200Error) as e:
            c.intra_mode_screen_dev(*args)
        assert e.value.status == B.ERR_ARG, args
    assert c.L.b200_ctx_launch_count(c.h) == before
    c.intra_mode_screen_dev(*ok[:6], 0, d_satd, d_modes)                  # no items: nothing to launch
    assert c.L.b200_ctx_launch_count(c.h) == before
    c.intra_mode_screen_dev(*ok)
    c.synchronize()
    assert c.L.b200_ctx_launch_count(c.h) == before + 1
