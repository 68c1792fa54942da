"""orc_inter_mode_screen (rdo.rs:1281-1363 with predict_inter, predict.rs:284-421) against an independent
Python restatement of the screening that calls only the oracle's pinned pieces: put_8tap, prep_8tap, mc_avg
and get_satd.  The restatement does the orchestration itself: get_mv_params with PlaneSlice::clamp, single
vs compound by the second reference, the stable sort.  Also: prep_8tap against the AV1 specification's
two-pass compound form, compound of one reference twice == single, the clamp-free case against
orc_mc_blocks + SATD, and a model of the mode list construction (rdo.rs:1158-1318) that the GPU tests and
the benchmark use to generate realistic items."""
import ctypes as C

import numpy as np
import pytest

from tests import oracle_lib as O
from tests.test_oracle_intra_edges import BSIZES

ENTRIES = 20
SINGLE = 0xFF
DEPTHS = [(np.uint8, 8), (np.uint16, 10), (np.uint16, 12)]
SCREEN_SIZES = [bs for bs, (w, h) in enumerate(BSIZES) if max(w, h) <= 64]      # the 19 sizes 4x4 .. 64x64
# b200_inter_screen_item / orc_inter_screen_item (oracle/inter_screen.h)
CAND_DTYPE = np.dtype([("mv", "<i2", (2, 2)), ("ref", "u1", (2,)), ("pad_", "u1", (2,))])
ITEM_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2"), ("bsize", "u1"), ("n", "u1"), ("pad_", "u1", (2,)),
                       ("cands", CAND_DTYPE, (ENTRIES,))])
assert ITEM_DTYPE.itemsize == 248


def origins(bd):
    """v_frame's luma origins: xorigin aligned to 64 bytes (tests/test_oracle_dist.py), yorigin 88."""
    return (128 if bd == 8 else 96), 88


def inter_mode_screen(src: O.Plane, rect, refs, xorigin, yorigin, filter_mode, bd, items, threads=0):
    """orc_inter_mode_screen: (satd n x 20, order n x 20)."""
    items = np.ascontiguousarray(items, ITEM_DTYPE)
    n = len(items)
    satd = np.zeros((n, ENTRIES), np.uint32)
    order = np.zeros((n, ENTRIES), np.uint8)
    ptrs = (C.c_void_p * len(refs))(*[r.origin_ptr() for r in refs])
    strides = (C.c_ssize_t * len(refs))(*[r.stride for r in refs])
    f = O.lib().orc_inter_mode_screen
    f.restype = None
    f.argtypes = ([C.c_void_p, C.c_ssize_t] + [C.c_int] * 4 + [C.c_void_p, C.c_void_p] + [C.c_int] * 8 +
                  [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_int])
    f(src.origin_ptr(), src.stride, *rect, ptrs, strides, len(refs), src.bpp, src.width, src.height, xorigin, yorigin,
      filter_mode, bd, O.ptr(items) if n else None, n, O.ptr(satd), O.ptr(order), threads)
    return satd, order


def random_image(rng, w, h, bd, dtype, smooth=False):
    img = rng.integers(0, 1 << bd, (h, w)).astype(np.float64)
    if smooth:
        k = np.ones(9) / 9.0
        img = np.apply_along_axis(lambda r: np.convolve(r, k, mode="same"), 1, img)
        img = np.apply_along_axis(lambda c: np.convolve(c, k, mode="same"), 0, img)
    return np.clip(np.rint(img), 0, (1 << bd) - 1).astype(dtype)


def host_plane(img, pad):
    p = O.Plane(img.shape[1], img.shape[0], pad, dtype=img.dtype)
    p.fill_from(img)
    return p


def make_item(x, y, bs, entries):
    """entries: [(ref0, ref1 or None, (row, col), (row, col) or None), ...]"""
    it = np.zeros(1, ITEM_DTYPE)[0]
    it["x"], it["y"], it["bsize"], it["n"] = x, y, bs, len(entries)
    for k, (r0, r1, m0, m1) in enumerate(entries):
        it["cands"][k]["ref"] = (r0, SINGLE if r1 is None else r1)
        it["cands"][k]["mv"][0] = m0
        it["cands"][k]["mv"][1] = m1 if m1 is not None else (0, 0)
    return it


def random_items(rng, rect_w, rect_h, count, nrefs, bsizes=SCREEN_SIZES, reach=24, compound=True):
    """Blocks aligned to their size inside the region, with lists of 1..20 random entries."""
    items = np.zeros(count, ITEM_DTYPE)
    bsizes = list(bsizes)
    for k in range(count):
        bs = bsizes[k % len(bsizes)]
        bw, bh = BSIZES[bs]
        x = int(rng.integers(0, (rect_w + bw - 1) // bw)) * bw
        y = int(rng.integers(0, (rect_h + bh - 1) // bh)) * bh
        ents = []
        for _ in range(int(rng.integers(1, ENTRIES + 1))):
            mv = lambda: tuple(int(v) for v in rng.integers(-8 * reach, 8 * reach + 1, 2))
            r0 = int(rng.integers(0, nrefs))
            if compound and nrefs > 1 and rng.integers(0, 2):
                ents.append((r0, int(rng.integers(0, nrefs)), mv(), mv()))
            else:
                ents.append((r0, None, mv(), None))
        items[k] = make_item(x, y, bs, ents)
    return items


# ---------------------------------------------------------------- the independent restatement
def model_screen(src, rect, refs, xorigin, yorigin, filter_mode, bd, it):
    """The screening of one item, orchestrated here from put_8tap / prep_8tap / mc_avg / get_satd."""
    rx, ry = rect[0], rect[1]
    bw, bh = BSIZES[int(it["bsize"])]
    po_x, po_y = rx + int(it["x"]), ry + int(it["y"])

    def source(ref, mv):
        row, col = int(mv[0]), int(mv[1])
        # get_mv_params: offsets are arithmetic shifts, fractions ((mv << 1) & 15)
        qx = min(max(po_x + (col >> 3) - 3, -xorigin), ref.width)        # PlaneSlice::clamp
        qy = min(max(po_y + (row >> 3) - 3, -yorigin), ref.height)
        return qx + 3, qy + 3, (col * 2) & 15, (row * 2) & 15

    satds = []
    for k in range(int(it["n"])):
        c = it["cands"][k]
        if int(c["ref"][1]) == SINGLE:
            x, y, cf, rf = source(refs[int(c["ref"][0])], c["mv"][0])
            pred = O.put_8tap(refs[int(c["ref"][0])], x, y, bw, bh, cf, rf, filter_mode, filter_mode, bd)
        else:
            tmps = []
            for i in range(2):
                ref = refs[int(c["ref"][i])]
                x, y, cf, rf = source(ref, c["mv"][i])
                tmps.append(O.prep_8tap(ref, x, y, bw, bh, cf, rf, filter_mode, filter_mode, bd))
            pred = O.mc_avg(tmps[0], tmps[1], bd)
        satd_fn = O.lib().orc_get_satd_u8 if src.bpp == 1 else O.lib().orc_get_satd_u16
        pred = np.ascontiguousarray(pred)
        satds.append(satd_fn(src.at(po_x, po_y), src.stride, pred.ctypes.data, bw, bw, bh))
    order = sorted(range(len(satds)), key=lambda k: satds[k]) + list(range(len(satds), ENTRIES))
    return satds + [0xFFFFFFFF] * (ENTRIES - len(satds)), order


def check_against_model(src, rect, refs, xorigin, yorigin, filter_mode, bd, items):
    satd, order = inter_mode_screen(src, rect, refs, xorigin, yorigin, filter_mode, bd, items)
    for k, it in enumerate(items):
        ms, mo = model_screen(src, rect, refs, xorigin, yorigin, filter_mode, bd, it)
        assert list(satd[k]) == ms, (k, it)
        assert list(order[k]) == mo, (k, it)
    return satd, order


def setup(rng, w, h, dtype, bd, nrefs, smooth=True):
    xo, yo = origins(bd)
    pad = max(xo, yo, 71)
    src = host_plane(random_image(rng, w, h, bd, dtype, smooth=smooth), 64)
    refs = [host_plane(random_image(rng, w, h, bd, dtype, smooth=smooth), pad) for _ in range(nrefs)]
    return src, refs, xo, yo


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_every_block_size_and_filter_in_a_tile_off_the_origin(dtype, bd):
    rng = np.random.default_rng(bd)
    W, H = 212, 156                                   # not a multiple of 8: blocks overhang the frame
    src, refs, xo, yo = setup(rng, W, H, dtype, bd, 3)
    for mode in range(4):
        for rect in ((0, 0, W, H), (64, 32, W - 64, H - 32)):
            items = random_items(rng, rect[2], rect[3], 19, 3)
            check_against_model(src, rect, refs, xo, yo, mode, bd, items)


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_integer_and_each_fraction_kind(dtype, bd):
    """Integer, H-only, V-only and HV vectors, single and compound, at every size."""
    rng = np.random.default_rng(20 + bd)
    src, refs, xo, yo = setup(rng, 96, 96, dtype, bd, 2)
    items = []
    for bs in SCREEN_SIZES:
        ents = []
        for fr, fc in ((0, 0), (0, 3), (5, 0), (7, 1), (-3, -5)):
            m = (16 + fr, -24 + fc)
            ents += [(0, None, m, None), (0, 1, m, (-m[0], m[1] + 1))]
        items.append(make_item(0, 0, bs, ents))
    check_against_model(src, (0, 0, 96, 96), refs, xo, yo, 0, bd, np.array(items))


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_vectors_that_hit_the_clamp_on_every_side(dtype, bd):
    """Vectors that start the footprint past each edge of the plane, up to +-4000 px, and the block on
    the right / bottom edge with the 16 px get_mv_range allows."""
    rng = np.random.default_rng(40 + bd)
    W, H = 120, 88
    src, refs, xo, yo = setup(rng, W, H, dtype, bd, 2, smooth=False)
    items = []
    for bs in SCREEN_SIZES:
        bw, bh = BSIZES[bs]
        for x, y in ((0, 0), (((W - 1) // bw) * bw, ((H - 1) // bh) * bh)):
            ents = []
            for row, col in ((0, -8 * 4000), (0, 8 * 4000), (-8 * 4000, 0), (8 * 4000 // 8 * 8, 0),
                             (8 * (H - y + 16) + 3, 8 * (W - x + 16) + 5), (-8 * (y + 200) - 1, -8 * (x + 150) + 2),
                             (-32767, 32767), (32767, -32768)):
                ents.append((int(rng.integers(0, 2)), None, (row, col), None))
            ents.append((0, 1, (8 * (H + 40), 0), (0, -8 * (W + 200) + 6)))
            ents.append((1, 0, (-8 * 300, 8 * 500 + 4), (8 * 3 + 1, 8 * 2)))
            items.append(make_item(x, y, bs, ents))
    check_against_model(src, (0, 0, W, H), refs, xo, yo, 2, bd, np.array(items))


def test_flat_content_keeps_the_list_order():
    rng = np.random.default_rng(9)
    for dtype, bd in DEPTHS:
        xo, yo = origins(bd)
        img = np.full((96, 128), (1 << bd) // 3, dtype)
        src = host_plane(img, 64)
        refs = [host_plane(img.copy(), max(xo, yo, 71)) for _ in range(2)]
        items = random_items(rng, 96, 64, 38, 2, reach=200)
        satd, order = check_against_model(src, (16, 16, 96, 64), refs, xo, yo, 0, bd, items)
        for k, it in enumerate(items):
            assert (satd[k][:it["n"]] == 0).all()
            assert list(order[k]) == list(range(ENTRIES))


def test_compound_of_one_reference_twice_equals_single_at_integer_vectors():
    """At an integer position prep is (p << ib) - bias, so the average of two identical preps reproduces put
    exactly (mc.rs:377-385, :466-478): same ref, same vector, same SATD.  (At a fraction the two rounding
    chains differ by up to 1 per pixel, as tests/test_oracle_mc.py states.)"""
    rng = np.random.default_rng(11)
    for dtype, bd in DEPTHS:
        src, refs, xo, yo = setup(rng, 128, 96, dtype, bd, 2, smooth=False)
        items = []
        for k, bs in enumerate(SCREEN_SIZES * 2):
            bw, bh = BSIZES[bs]
            singles = [(int(rng.integers(0, 2)), tuple(8 * int(v) for v in rng.integers(-90, 91, 2))) for _ in range(10)]
            ents = [(r, None, m, None) for r, m in singles] + [(r, r, m, m) for r, m in singles]
            items.append(make_item((k * 16) % 128 // bw * bw, (k * 8) % 96 // bh * bh, bs, ents))
        satd, _ = inter_mode_screen(src, (0, 0, 128, 96), refs, xo, yo, k & 3, bd, np.array(items))
        assert (satd[:, :10] == satd[:, 10:]).all()


@pytest.mark.parametrize("dtype,bd", DEPTHS)
def test_prep_equals_the_specification_two_pass_form(dtype, bd):
    """AV1 7.11.3.4 with isCompound: a horizontal pass rounded by InterRound0 (3; 5 at 12 bit), a vertical pass
    rounded by InterRound1 = 7, no clip; rav1e stores that minus PREP_BIAS (8192 at 10 / 12 bit) in i16.  The
    reference's four special-cased paths (mc.rs:360-451) must all equal it."""
    rng = np.random.default_rng(60 + bd)
    p = host_plane(random_image(rng, 64, 64, bd, dtype), 16)
    L = O.lib()
    r0 = 5 if bd == 12 else 3
    bias = 0 if bd == 8 else 8192
    img = p.data.astype(np.int64)
    rnd = lambda v, b: (v + (1 << (b - 1))) >> b
    fx, fy = (C.c_int32 * 8)(), (C.c_int32 * 8)()
    for w, h in ((8, 8), (4, 16), (16, 4), (4, 4)):
        for _ in range(6):
            cf, rf = (int(v) for v in rng.integers(0, 16, 2))
            if rng.integers(0, 3) == 0:
                cf = 0
            if rng.integers(0, 3) == 0:
                rf = 0
            mx, my = (int(v) for v in rng.integers(0, 4, 2))
            x0, y0 = (int(v) for v in rng.integers(4, 40, 2))
            L.orc_get_filter(mx, cf, w, fx)
            L.orc_get_filter(my, rf, h, fy)
            kx, ky = np.array(list(fx), np.int64), np.array(list(fy), np.int64)
            inter = np.zeros((h + 7, w), np.int64)
            for r in range(h + 7):
                for c in range(w):
                    py, px = p.pad + y0 + r - 3, p.pad + x0 + c - 3
                    inter[r, c] = rnd(int((kx * img[py, px:px + 8]).sum()), r0)
            want = np.zeros((h, w), np.int64)
            for r in range(h):
                for c in range(w):
                    want[r, c] = rnd(int((ky * inter[r:r + 8, c]).sum()), 7) - bias
            got = O.prep_8tap(p, x0, y0, w, h, cf, rf, mx, my, bd)
            np.testing.assert_array_equal(got, want, err_msg=f"{w}x{h} frac ({cf},{rf}) modes ({mx},{my})")


def test_without_the_clamp_equals_mc_blocks_and_satd():
    """Vectors that keep the footprint inside [-origin, size]: the screen is orc_mc_blocks' put + get_satd."""
    rng = np.random.default_rng(70)
    for dtype, bd in DEPTHS:
        src, refs, xo, yo = setup(rng, 160, 128, dtype, bd, 1)
        items = random_items(rng, 160, 128, 38, 1, reach=20)
        satd, _ = inter_mode_screen(src, (0, 0, 160, 128), refs, xo, yo, 0, bd, items)
        for k, it in enumerate(items):
            bw, bh = BSIZES[int(it["bsize"])]
            n = int(it["n"])
            blocks = np.zeros(n, O.BLOCK_DTYPE)
            blocks["x"], blocks["y"] = int(it["x"]), int(it["y"])
            mvs = np.ascontiguousarray(it["cands"]["mv"][:n, 0, :]).astype(np.int16)
            preds = O.mc_blocks(refs[0], blocks, mvs, bw, bh, 0, 0, bd)
            for j in range(n):
                pr = np.ascontiguousarray(preds[j])
                f = O.lib().orc_get_satd_u8 if src.bpp == 1 else O.lib().orc_get_satd_u16
                assert satd[k][j] == f(src.at(int(it["x"]), int(it["y"])), src.stride, pr.ctypes.data, bw, bw, bh)


def test_invalid_items_get_the_max_row_and_the_identity_order():
    rng = np.random.default_rng(13)
    src, refs, xo, yo = setup(rng, 96, 96, np.uint8, 8, 2)
    items = random_items(rng, 64, 64, 9, 2, bsizes=[3])
    items[0]["bsize"] = 22
    items[1]["bsize"] = 13                            # 64x128
    items[2]["n"] = 21
    items[3]["cands"][0]["ref"][0] = 2                # ref index >= nrefs
    items[4]["cands"][items[4]["n"] - 1]["ref"][1] = 7
    items[5]["x"] = 64                                # outside the 64x64 region
    items[6]["y"] = -4
    items[7]["x"] = 6                                 # not a multiple of 4
    items[8]["n"] = 0                                 # valid and empty
    satd, order = inter_mode_screen(src, (16, 16, 64, 64), refs, xo, yo, 0, 8, items)
    for k in range(9):
        assert (satd[k] == np.uint32(0xFFFFFFFF)).all()
        assert list(order[k]) == list(range(ENTRIES))


# ---------------------------------------------------------------- the mode list (rdo.rs:1158-1318)
NEARESTMV, NEAR0MV, NEAR1MV, NEAR2MV, GLOBALMV, NEWMV = "NEARESTMV", "NEAR0MV", "NEAR1MV", "NEAR2MV", "GLOBALMV", "NEWMV"
COMPOUND_MODES = ["GLOBAL_GLOBALMV", "NEAREST_NEARESTMV", "NEW_NEWMV", "NEAREST_NEWMV", "NEW_NEARESTMV",
                  "NEAR_NEAR0MV", "NEAR_NEAR1MV", "NEAR_NEAR2MV"]          # RAV1E_INTER_COMPOUND_MODES
NEAR_IDX = {NEAR0MV: 1, NEAR1MV: 2, NEAR2MV: 3, "NEAR_NEAR0MV": 1, "NEAR_NEAR1MV": 2, "NEAR_NEAR2MV": 3}


def build_mode_list(bw, bh, stacks, me_mvs, include_near_mvs, compound_ok, fwd=None, bwd=None, comp_stack=()):
    """inter_mode_set / mvs_set / ref_frames_set of rdo.rs:1158-1318 for one block.

    stacks[i]: find_mvrefs' stack of single reference i, a list of (this_mv, comp_mv); me_mvs[i]: its
    estimate_motion vector; compound_ok: reference_mode != SINGLE; fwd / bwd: indices of the first forward /
    backward reference; comp_stack: the compound stack.  Returns [(mode, (ref0, ref1 or None), (mv0, mv1))]."""
    zero = (0, 0)
    ref_sets = [(i, None) for i in range(len(stacks))]
    mvs_from_me = [(m, zero) for m in me_mvs]
    mv_stacks = [list(s) for s in stacks]
    modes = []
    for i, st in enumerate(stacks):
        modes.append((NEARESTMV, i))
        if len(st) >= 1:
            modes.append((NEAR0MV, i))
        if len(st) >= 2:
            modes.append((GLOBALMV, i))
        if include_near_mvs:
            if len(st) >= 3:
                modes.append((NEAR1MV, i))
            if len(st) >= 4:
                modes.append((NEAR2MV, i))
        same = any(s[0] == me_mvs[i] for s in st[:4 if include_near_mvs else 2])
        if not same and me_mvs[i] != zero:
            modes.append((NEWMV, i))
    if compound_ok and min(bw, bh) >= 8 and fwd is not None and bwd is not None:
        ref_sets.append((fwd, bwd))
        mvs_from_me.append((me_mvs[fwd], me_mvs[bwd]))
        mv_stacks.append(list(comp_stack))
        ci = len(ref_sets) - 1
        for m in COMPOUND_MODES:
            near = m in NEAR_IDX
            if include_near_mvs or not near:
                if not (near and NEAR_IDX[m] >= len(comp_stack)):
                    modes.append((m, ci))
    out = []
    for m, i in modes:
        st = mv_stacks[i]
        if m in (NEWMV, "NEW_NEWMV"):
            mvs = mvs_from_me[i]
        elif m in (NEARESTMV, "NEAREST_NEARESTMV"):
            mvs = (st[0][0], st[0][1]) if st else (zero, zero)
        elif m in (NEAR0MV, "NEAR_NEAR0MV"):
            mvs = (st[1][0], st[1][1]) if len(st) > 1 else (zero, zero)
        elif m in (NEAR1MV, NEAR2MV, "NEAR_NEAR1MV", "NEAR_NEAR2MV"):
            mvs = (st[NEAR_IDX[m]][0], st[NEAR_IDX[m]][1])
        elif m == "NEAREST_NEWMV":
            mvs = (st[0][0], mvs_from_me[i][1])
        elif m == "NEW_NEARESTMV":
            mvs = (mvs_from_me[i][0], st[0][1])
        else:                                         # GLOBALMV, GLOBAL_GLOBALMV
            mvs = (zero, zero)
        out.append((m, ref_sets[i], mvs))
    assert len(out) <= ENTRIES
    return out


def list_item(x, y, bs, mode_list):
    """The device item of a built list: ref indices into the call's refs[] = the single-reference indices."""
    return make_item(x, y, bs, [(r[0], r[1], mvs[0], mvs[1] if r[1] is not None else None)
                                for _, r, mvs in mode_list])


def random_block_list(rng, bw, bh, nrefs=2, include_near_mvs=False, reach=12, compound_ok=True):
    """A realistic list: stacks around a common motion, ME vectors near the stack's head."""
    base = [tuple(int(v) for v in rng.integers(-8 * reach, 8 * reach + 1, 2)) for _ in range(nrefs)]
    jit = lambda m: (m[0] + int(rng.integers(-6, 7)), m[1] + int(rng.integers(-6, 7)))
    stacks = []
    for i in range(nrefs):
        st = [(jit(base[i]), (0, 0)) for _ in range(int(rng.integers(0, 5)))]
        stacks.append(st)
    me = [stacks[i][0][0] if stacks[i] and rng.integers(0, 4) == 0 else jit(base[i]) for i in range(nrefs)]
    comp = [(jit(base[0]), jit(base[-1])) for _ in range(int(rng.integers(1, 5)))]
    return build_mode_list(bw, bh, stacks, me, include_near_mvs, compound_ok, 0 if nrefs > 1 else None,
                           nrefs - 1 if nrefs > 1 else None, comp)


def test_mode_list_quirks():
    z = (0, 0)
    a, b, c = (8, -16), (3, 5), (40, 40)
    # NEAR0MV with a one-entry stack: zero vectors; NEWMV dropped when it equals a stack entry
    lst = build_mode_list(16, 16, [[(a, z)]], [a], False, False)
    assert [m for m, _, _ in lst] == [NEARESTMV, NEAR0MV]
    assert lst[1][2] == (z, z)
    # NEWMV dropped when zero, kept otherwise; GLOBALMV from two entries, with zero vectors
    assert [m for m, _, _ in build_mode_list(16, 16, [[(a, z), (b, z)]], [z], False, False)] == \
        [NEARESTMV, NEAR0MV, GLOBALMV]
    lst = build_mode_list(16, 16, [[(a, z), (b, z), (c, z)]], [c], False, False)
    assert [m for m, _, _ in lst] == [NEARESTMV, NEAR0MV, GLOBALMV, NEWMV] and lst[2][2] == (z, z)
    # the third entry counts for NEWMV only with include_near_mvs
    assert NEWMV not in [m for m, _, _ in build_mode_list(16, 16, [[(a, z), (b, z), (c, z)]], [c], True, False)]
    # compound entries need both directions and min(w, h) >= 8
    stacks, me, comp = [[(a, z)], [(b, z)]], [c, b], [(a, b), (b, c)]
    full = build_mode_list(16, 8, stacks, me, False, True, 0, 1, comp)
    assert [m for m, _, _ in full if "_" in m] == ["GLOBAL_GLOBALMV", "NEAREST_NEARESTMV", "NEW_NEWMV",
                                                   "NEAREST_NEWMV", "NEW_NEARESTMV"]
    assert not [m for m, _, _ in build_mode_list(8, 4, stacks, me, False, True, 0, 1, comp) if "_" in m]
    assert not [m for m, _, _ in build_mode_list(16, 16, stacks, me, False, True, 0, None, comp) if "_" in m]
    assert not [m for m, _, _ in build_mode_list(16, 16, stacks, me, False, False, 0, 1, comp) if "_" in m]
    # NEAREST_NEWMV / NEW_NEARESTMV mix the compound stack and the ME vectors
    d = {m: mvs for m, _, mvs in full}
    assert d["NEAREST_NEWMV"] == (a, b) and d["NEW_NEARESTMV"] == (c, b) and d["NEW_NEWMV"] == (c, b)
    # with include_near_mvs, the NEAR_NEAR modes the compound stack is long enough for
    near = build_mode_list(16, 16, stacks, me, True, True, 0, 1, comp)
    assert [m for m, _, _ in near if m.startswith("NEAR_NEAR")] == ["NEAR_NEAR0MV"]
    assert {m: mvs for m, _, mvs in near}["NEAR_NEAR0MV"] == (b, c)


def test_realistic_lists_against_the_model():
    rng = np.random.default_rng(80)
    for dtype, bd in DEPTHS:
        src, refs, xo, yo = setup(rng, 160, 128, dtype, bd, 2)
        items = []
        for k, bs in enumerate(SCREEN_SIZES * 2):
            bw, bh = BSIZES[bs]
            lst = random_block_list(rng, bw, bh, include_near_mvs=bool(k & 1))
            items.append(list_item(((k * 8) % 160) // bw * bw, ((k * 24) % 128) // bh * bh, bs, lst))
        check_against_model(src, (0, 0, 160, 128), refs, xo, yo, 0, bd, np.array(items))
