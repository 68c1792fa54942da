"""orc_intra_mode_screen (rdo.rs:1433-1511 with predict_intra, predict.rs:205-249) against an independent
Python restatement of the screening that calls only the oracle's pinned pieces: get_intra_edges, the
intra predictors and get_satd.  The restatement does the orchestration itself: PredictionVariant from
the tile-relative position, PAETH at the tile's edges, intra_mode_to_angle, the edge filter for
directional modes only, bsize.tx_size(), the skipped first num_modes_rdo / 2 modes, the stable sort and
the zeros of unscreened modes."""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O
from tests.test_oracle_intra_edges import BSIZES, L as OL

# RAV1E_INTRA_MODES (predict.rs:42-56), the order the CDF sort starts from
RAV1E_INTRA_MODES = [0, 2, 1, 9, 11, 10, 12, 3, 4, 5, 6, 7, 8]
MODE_ANGLE = {1: 90, 2: 180, 3: 45, 4: 135, 5: 113, 6: 157, 7: 203, 8: 67}
DEPTHS = [(np.uint8, 8), (np.uint16, 10), (np.uint16, 12)]
# b200_intra_screen_item / orc_intra_screen_item (oracle/intra_screen.h)
INTRA_SCREEN_ITEM_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2"), ("bsize", "u1"), ("ief", "i1"),
                                    ("modes", "u1", (13,)), ("pad_", "u1")])


def intra_mode_screen(rec: O.Plane, src: O.Plane, rect, bit_depth, num_modes_rdo, items, threads=0):
    """orc_intra_mode_screen: (satd n x 13 by discriminant, modes n x 13 after the tail sort)."""
    items = np.ascontiguousarray(items, INTRA_SCREEN_ITEM_DTYPE)
    n = len(items)
    satd = np.zeros((n, 13), np.uint32)
    modes = np.zeros((n, 13), np.uint8)
    f = O.lib().orc_intra_mode_screen
    f.restype = None
    f.argtypes = [C.c_void_p, C.c_ssize_t, C.c_void_p, C.c_ssize_t] + [C.c_int] * 9 + [C.c_void_p, C.c_size_t,
                                                                                        C.c_void_p, C.c_void_p, C.c_int]
    f(rec.origin_ptr(), rec.stride, src.origin_ptr(), src.stride, rec.bpp, rec.width, rec.height, *rect, bit_depth,
      num_modes_rdo, O.ptr(items) if n else None, n, O.ptr(satd), O.ptr(modes), threads)
    return satd, modes


def random_image(rng, w, h, bd, dtype, smooth=False):
    img = rng.integers(0, 1 << bd, (h, w)).astype(np.float64)
    if smooth:
        k = np.ones(9) / 9.0
        img = np.apply_along_axis(lambda r: np.convolve(r, k, mode="same"), 1, img)
        img = np.apply_along_axis(lambda c: np.convolve(c, k, mode="same"), 0, img)
    return np.clip(np.rint(img), 0, (1 << bd) - 1).astype(dtype)


def planes(rec_img, src_img, pad=80):
    rec = O.Plane(rec_img.shape[1], rec_img.shape[0], pad, dtype=rec_img.dtype)
    rec.fill_from(rec_img)
    src = O.Plane(src_img.shape[1], src_img.shape[0], pad, dtype=src_img.dtype)
    src.fill_from(src_img)
    return rec, src


def make_items(rng, rect_w, rect_h, n, bsizes=range(22), iefs=(-1, 0, 1), mode_order=None):
    """Blocks at positions aligned to their size inside the region, each with its own mode order."""
    items = np.zeros(n, INTRA_SCREEN_ITEM_DTYPE)
    bsizes = list(bsizes)
    for k in range(n):
        bs = bsizes[k % len(bsizes)]
        bw, bh = BSIZES[bs]
        x = int(rng.integers(0, (rect_w + bw - 1) // bw)) * bw
        y = int(rng.integers(0, (rect_h + bh - 1) // bh)) * bh
        items[k]["x"], items[k]["y"], items[k]["bsize"] = x, y, bs
        items[k]["ief"] = iefs[k % len(iefs)]
        items[k]["modes"] = mode_order if mode_order is not None else rng.permutation(RAV1E_INTRA_MODES)
    return items


def model_screen(rec, src, rect, bd, num_modes_rdo, it):
    """The screening of one item, orchestrated here from the oracle's edge, predictor and SATD."""
    rx, ry, rw, rh = rect
    x, y, bs, ief = int(it["x"]), int(it["y"]), int(it["bsize"]), int(it["ief"])
    modes = [int(m) for m in it["modes"]]
    bw, bh = BSIZES[bs]
    tw, th = min(bw, 64), min(bh, 64)                       # bsize.tx_size()
    edge = np.zeros(O.EDGE_LEN, rec.data.dtype)
    il, ia = C.c_int(), C.c_int()
    OL().orc_get_intra_edges(edge.ctypes.data, rec.at(rx, ry), rec.stride, rec.bpp, rec.width, rec.height, rx, ry,
                             rw, rh, 0, 0, x >> 2, y >> 2, 0, 0, bs, x, y, tw, th, bd, -1, int(ief >= 0), 0,
                             C.byref(il), C.byref(ia))
    variant = 0 if (x, y) == (0, 0) else 1 if y == 0 else 2 if x == 0 else 3      # PredictionVariant::new
    satds = [0] * 13
    satd_fn = O.lib().orc_get_satd_u8 if rec.bpp == 1 else O.lib().orc_get_satd_u16
    for lm in modes[num_modes_rdo // 2:]:
        mode = {0: 0, 2: 1, 1: 2, 3: 12}[variant] if lm == 12 else lm      # PAETH -> DC / V / H
        pred = O.predict_intra(mode, variant, edge, tw, th, bd, angle=MODE_ANGLE.get(mode, 0),
                               ief=ief if 1 <= lm <= 8 else -1, left_len=il.value, above_len=ia.value,
                               plane_w=rec.width, plane_h=rec.height, dst_x=rx + x, dst_y=ry + y)
        satds[lm] = satd_fn(src.at(rx + x, ry + y), src.stride, pred.ctypes.data, tw, tw, th)
    skip = num_modes_rdo // 2
    return satds, modes[:skip] + sorted(modes[skip:], key=lambda m: satds[m])


def check_against_model(rec, src, rect, bd, num_modes_rdo, items):
    satd, modes = intra_mode_screen(rec, src, rect, bd, num_modes_rdo, items)
    for k, it in enumerate(items):
        ms, mm = model_screen(rec, src, rect, bd, num_modes_rdo, it)
        assert list(satd[k]) == ms, (k, it)
        assert list(modes[k]) == mm, (k, it)
    return satd, modes


@pytest.mark.parametrize("dtype,bd", DEPTHS)
@pytest.mark.parametrize("num_modes_rdo", [3, 7])
def test_every_block_size_in_a_tile_off_the_origin(dtype, bd, num_modes_rdo):
    rng = np.random.default_rng(bd * 10 + num_modes_rdo)
    W, H = 300, 236                                   # not a multiple of 8: blocks overhang the frame
    rec_img = random_image(rng, W, H, bd, dtype, smooth=True)
    src_img = random_image(rng, W, H, bd, dtype, smooth=bool(bd & 2))
    rec, src = planes(rec_img, src_img)
    for rect in ((0, 0, W, H), (64, 48, W - 64, H - 48), (128, 64, 128, 128)):
        items = make_items(rng, rect[2], rect[3], 132)
        # blocks on the tile's top row and left column, whatever make_items drew
        items[:22]["x"] = 0
        items[22:44]["y"] = 0
        items[44:66]["x"] = 0
        items[44:66]["y"] = 0
        check_against_model(rec, src, rect, bd, num_modes_rdo, items)


def test_blocks_overhanging_the_frame():
    rng = np.random.default_rng(5)
    W, H = 150, 110
    for dtype, bd in DEPTHS:
        rec, src = planes(random_image(rng, W, H, bd, dtype), random_image(rng, W, H, bd, dtype))
        items = np.zeros(0, INTRA_SCREEN_ITEM_DTYPE)
        for bs, (bw, bh) in enumerate(BSIZES):
            it = make_items(rng, W, H, 3, bsizes=[bs])
            it["x"] = ((W - 1) // bw) * bw                 # the last block column / row, partly outside
            it["y"] = [((H - 1) // bh) * bh, 0, ((H - 1) // bh) * bh]
            items = np.concatenate([items, it])
        check_against_model(rec, src, (0, 0, W, H), bd, 3, items)


def test_flat_content_keeps_the_cdf_order():
    """Every screened mode predicts the flat value away from the tile's top-left corner (where the edges
    are the documented constants): all SATDs are 0 and the stable sort must leave the CDF order as it was."""
    rng = np.random.default_rng(9)
    for dtype, bd in DEPTHS:
        v = (1 << bd) // 3
        img = np.full((128, 192), v, dtype)
        rec, src = planes(img, img.copy())
        rect = (32, 16, 160, 112)
        items = make_items(rng, rect[2], rect[3], 66)
        corner = (items["x"] == 0) & (items["y"] == 0)
        items["y"][corner] = 64
        for num_modes_rdo in (3, 7):
            satd, modes = check_against_model(rec, src, rect, bd, num_modes_rdo, items)
            assert (satd == 0).all()
            assert (modes == items["modes"]).all()


def test_unscreened_modes_are_zero_and_lead_the_list():
    rng = np.random.default_rng(11)
    rec, src = planes(random_image(rng, 128, 128, 8, np.uint8), random_image(rng, 128, 128, 8, np.uint8))
    items = make_items(rng, 128, 128, 44)
    for num_modes_rdo in (3, 7):
        satd, modes = intra_mode_screen(rec, src, (0, 0, 128, 128), 8, num_modes_rdo, items)
        skip = num_modes_rdo // 2
        for k, it in enumerate(items):
            assert list(modes[k][:skip]) == list(it["modes"][:skip])
            assert sorted(modes[k]) == list(range(13))
            assert all(satd[k][m] == 0 for m in it["modes"][:skip])
            assert all(satd[k][m] > 0 for m in it["modes"][skip:])


def test_invalid_items_get_the_max_row_and_their_list():
    rng = np.random.default_rng(13)
    rec, src = planes(random_image(rng, 96, 96, 8, np.uint8), random_image(rng, 96, 96, 8, np.uint8))
    items = make_items(rng, 64, 64, 8, bsizes=[3])
    items[0]["bsize"] = 22
    items[1]["modes"][4] = 13
    items[2]["modes"][5] = items[2]["modes"][6]
    items[3]["x"] = 64                                # outside the 64x64 region
    items[4]["y"] = -4
    items[5]["x"] = 6                                 # not a multiple of 4
    satd, modes = intra_mode_screen(rec, src, (16, 16, 64, 64), 8, 3, items)
    for k in range(6):
        assert (satd[k] == np.uint32(0xFFFFFFFF)).all()
        assert (modes[k] == items[k]["modes"]).all()
    for k in (6, 7):
        ms, mm = model_screen(rec, src, (16, 16, 64, 64), 8, 3, items[k])
        assert list(satd[k]) == ms and list(modes[k]) == mm
