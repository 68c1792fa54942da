"""CDEF on every kernel path, bit exact against the oracle and, for a fixed-seed sample of every section, against
the AV1 specification restated in tests/test_oracle_cdef_spec.py.

The kernels (cdef.cu, on the device primitives of cdef_dev.cuh):
- `cdef_find_dir_kernel<T>`: b200_cdef_find_dir_dev / b200_cdef_tiles_dev with find_dir and the per-call
  b200_cdef_dir; one thread per 8x8 luma block, a grid-stride loop over each item's rect;
- `cdef_filter_kernel<T>`: the frame-level filter, one CTA per 64 x 16 pixel tile of an item, up to 32 items per
  launch, the grid sized from the largest item of the launch;
- `cdef_filter_tmp16_kernel<T>`: the per-call b200_cdef_filter_block on a caller-built padded u16 tile.
The sections:
1. a 584 x 520 frame (partial superblocks at the right and bottom) whose strength maps hold all 64 strengths, with
   blocks built to reach every direction and every adjust_strength variance bracket: luma at damping 3..6 and
   4:2:0 / 4:2:2 / 4:4:4 chroma at damping 3 and 6, at 8 / 10 / 12 bit;
2. 40-item lists over three frames: find_dir + filter on luma, filter only on 4:2:0 and 4:2:2 chroma, find_dir
   only without an output plane; out planes hold a canary outside the items' rects;
3. find_dir's grid-stride loop sent round a second time, with 32 items and with one 8K item;
4. caller-built planes: garbage in the input's padding, an output whose 4-pixel groups are partly misaligned;
5. the per-call forms: every shape x direction x edge mask of b200_cdef_filter_block, and b200_cdef_dir on
   directional, maximum-contrast, low-bit-noise and tied blocks;
6. rejected arguments launch nothing and write nothing.
Each section asserts that it reached what it claims, from the oracle's own dir / var and the strengths."""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_oracle_cdef_spec import floor_log2, spec_direction, spec_direction_costs, spec_filter

pytestmark = pytest.mark.gpu

BDS = [8, 10, 12]
CHROMA = [(1, 1), (1, 0), (0, 0)]          # (xdec, ydec): 4:2:0, 4:2:2, 4:4:4
SENT_DIR, SENT_VAR = 0xEE, -0x5A5A5A5       # dir / var before a launch

# Launch geometry mirrored from the sources.
ITEMS_PER_LAUNCH = 32      # cdef.cu:20   kCdefMaxItems: an item list is cut every 32 items
DIR_THREADS = 128          # cdef.cu:191  one 8x8 block per thread, 128-thread CTAs
DIR_CTAS_PER_SM = 16       # cdef.cu:189  grid.x = min(ceil(blocks / 128), num_sms * 16 / n), then a grid-stride loop
TILE_W, TILE_H = 64, 16    # cdef.cu:64   kCdefTW x kCdefTH pixels per filter CTA

# AV1 spec Cdef_Uv_Dir[subsampling_x][subsampling_y][yDir]
CDEF_UV_DIR = [[[0, 1, 2, 3, 4, 5, 6, 7], [1, 2, 2, 2, 3, 4, 6, 0]],
               [[7, 0, 2, 4, 5, 6, 6, 6], [0, 1, 2, 3, 4, 5, 6, 7]]]

_I, _J = np.mgrid[0:8, 0:8]
# the 15 partial-sum lines of each direction (7.15.2): a block constant along them is oriented in that direction
LINES = [_I + _J, _I + _J // 2, _I, 3 + _I - _J // 2, 7 + _I - _J, 3 - _I // 2 + _J, _J, _I // 2 + _J]


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def pxdt(bd):
    return np.uint8 if bd == 8 else np.uint16


# ---------------------------------------------------------------- content
def stripes(rng, d, amp):
    """An 8x8 block in 8-bit units, constant along direction d's lines, line values mid +- amp."""
    mid = rng.uniform(min(amp, 127.5), max(255 - amp, 127.5))
    return mid + amp * rng.uniform(-1, 1, 15)[LINES[d]]


def block_of_kind(rng, k):
    """Kind k of the 64-entry menu -> (8x8 block in 8-bit units, exact): `exact` blocks hold only 0 and the maximum.
    k < 40: stripes in direction k % 8 (k < 24 strong, the rest log-uniform amplitudes, so var spans every
    adjust_strength bracket); then random, flat, 0/max checkerboard, 0/max step edge, 0/max alternating rows or
    columns (var past the bracket clamp) and weaker stripes in a random direction."""
    if k < 24:
        return stripes(rng, k % 8, rng.uniform(24, 127)), False
    if k < 40:
        return stripes(rng, k % 8, 2.0 ** rng.uniform(-1, 7)), False
    if k < 44:
        return rng.uniform(0, 255, (8, 8)), False
    if k < 47:
        return np.full((8, 8), rng.uniform(0, 255)), False
    if k < 50:
        return 255.0 * ((_I + _J) % 2), True
    if k < 54:
        a, b = rng.integers(-2, 3, 2)
        return 255.0 * (a * _I + b * _J > rng.integers(-4, 5)), True
    if k < 58:
        return 255.0 * ((_I if k < 56 else _J) % 2), True
    return stripes(rng, int(rng.integers(0, 8)), 2.0 ** rng.uniform(-1, 5)), False


def textured(rng, W, H, bd):
    """A W x H frame of menu blocks, each superblock holding every kind once in a random order.  Non-exact blocks
    get random low bits at 10 / 12 bit (the direction search shifts them away, the filter does not)."""
    cs, maxv = bd - 8, (1 << bd) - 1
    out = np.zeros((H, W), np.int64)
    perms = {}
    for by in range(H // 8):
        for bx in range(W // 8):
            perm = perms.setdefault((by >> 3, bx >> 3), rng.permutation(64))
            blk, exact = block_of_kind(rng, int(perm[(by & 7) * 8 + (bx & 7)]))
            if exact:
                v = np.where(blk > 0, maxv, 0)
            else:
                v = (np.clip(np.rint(blk), 0, 255).astype(np.int64) << cs) | rng.integers(0, 1 << cs, (8, 8))
            out[8 * by:8 * by + 8, 8 * bx:8 * bx + 8] = v
    return out.astype(pxdt(bd))


def edge_mask(gy, gx, h8, w8):
    return int(gx > 0) | int(gx + 1 < w8) << 1 | int(gy > 0) << 2 | int(gy + 1 < h8) << 3


def var_class(v):
    """adjust_strength's bracket: -1 for var == 0, then min(msb(var >> 6), 13) with 13 standing for the clamp."""
    return -1 if v == 0 else (min(floor_log2(v >> 6), 13) if v >> 6 else 0)


def adjust_np(strength, var):
    vs = var >> 6
    i = np.where(vs > 0, np.minimum(np.floor(np.log2(np.maximum(vs, 1))).astype(np.int64), 12), 0)
    return np.where(var != 0, (strength * (4 + i) + 8) >> 4, 0)


def spec_block_params(strength, plane, xdec, ydec, ydir, var, damping, bd):
    """7.15.1 for one 8x8 block: (priStr, secStr, dir, damping); the coded secondary strength 3 means 4."""
    cs = bd - 8
    pri, sec = strength >> 2, strength & 3
    sec = 4 if sec == 3 else sec
    pri_str, sec_str = pri << cs, sec << cs
    if plane == 0:
        d = 0 if pri_str == 0 else ydir
        var_str = min(floor_log2(var >> 6), 12) if var >> 6 else 0
        pri_str = (pri_str * (4 + var_str) + 8) >> 4 if var else 0
    else:
        d = 0 if pri_str == 0 else CDEF_UV_DIR[xdec][ydec][ydir]
    return pri_str, sec_str, d, damping + cs - (1 if plane else 0)


def spec_check_blocks(img, got, plane, xdec, ydec, bd, damping, skip8, dirs, var, strength, picks):
    """The specification's filter of the picked 8x8 blocks (availability from the block's place in the frame)."""
    h8, w8 = dirs.shape
    bw, bh = 8 >> xdec, 8 >> ydec
    padded = np.pad(img, 2, mode="edge")          # never read where a neighbour is missing
    for gy, gx in picks:
        src = padded[gy * bh:gy * bh + bh + 4, gx * bw:gx * bw + bw + 4]
        if skip8 is not None and skip8[gy, gx]:
            want = src[2:2 + bh, 2:2 + bw]
        else:
            p, s, d, dmp = spec_block_params(int(strength[gy >> 3, gx >> 3]), plane, xdec, ydec, int(dirs[gy, gx]),
                                             int(var[gy, gx]), damping, bd)
            want = spec_filter(src, bw, bh, p, s, d, dmp, bd, edge_mask(gy, gx, h8, w8))
        np.testing.assert_array_equal(got[gy * bh:(gy + 1) * bh, gx * bw:(gx + 1) * bw], want,
                                      err_msg=f"spec, plane {plane} block ({gy}, {gx})")


def sample_blocks(rng, h8, w8, n):
    corners = [(0, 0), (0, w8 - 1), (h8 - 1, 0), (h8 - 1, w8 - 1)]
    return corners + [divmod(int(b), w8) for b in rng.choice(h8 * w8, n, replace=False)]


def dev_dir_var(n):
    import torch
    return (torch.full((n,), SENT_DIR, dtype=torch.uint8, device="cuda"),
            torch.full((n,), SENT_VAR, dtype=torch.int32, device="cuda"))


def download(c, p, shape, dtype):
    got = np.zeros(shape, dtype)
    c.check(c.L.b200_plane_download(c.h, C.byref(p), got.ctypes.data, got.strides[0]))
    return got


# ---------------------------------------------------------------- 1. strength x direction x variance
SW, SH = 584, 520        # 73 x 65 blocks, 10 x 9 superblocks: the last column and row are 8 pixels
# edge masks (L 1, R 2, T 4, B 8) of the interior, the four sides and the four corners of a frame
FRAME_PLACES = {15, 14, 13, 11, 7, 10, 9, 6, 5}


def sweep_inputs(rng, bd):
    """Frame, skip mask and the luma / chroma strength maps of section 1.  64 of the 72 whole superblocks take
    the 64 strengths once each; the 65th is skipped entirely; the rest and the partial ones get pri != 0."""
    luma = textured(rng, SW, SH, bd)
    w8, h8, sbw, sbh = SW // 8, SH // 8, (SW + 63) // 64, (SH + 63) // 64
    skip8 = (rng.random((h8, w8)) < 0.1).astype(np.uint8)
    for gy, gx in ((0, 3), (h8 - 1, 5), (4, 0), (6, w8 - 1), (0, w8 - 2)):   # skipped blocks on the border
        skip8[gy, gx] = 1
    for gy, gx in ((0, 0), (0, w8 - 1), (h8 - 1, 0), (h8 - 1, w8 - 1)):
        skip8[gy, gx] = 0
    whole = [(y, x) for y in range(sbh) for x in range(sbw) if 64 * (x + 1) <= SW and 64 * (y + 1) <= SH]
    y, x = whole.pop(int(rng.integers(len(whole))))
    skip8[8 * y:8 * y + 8, 8 * x:8 * x + 8] = 1
    maps = []
    for _ in range(2):
        order = [whole[i] for i in rng.permutation(len(whole))]
        m = rng.integers(4, 64, (sbh, sbw))
        for s, (y, x) in enumerate(order[:64]):
            m[y, x] = s
        maps.append(m.astype(np.uint8))
    return luma, skip8, maps[0], maps[1]


def assert_sweep_coverage(bd, skip8, ystr, uvstr, dirs, var):
    """What the frame reaches, from the oracle's dir / var and the strengths."""
    cs = bd - 8
    h8, w8 = skip8.shape
    live = skip8 == 0
    gy, gx = np.nonzero(live)
    ys, us = ystr[gy >> 3, gx >> 3].astype(np.int64), uvstr[gy >> 3, gx >> 3].astype(np.int64)
    dv, vv = dirs[gy, gx].astype(np.int64), var[gy, gx].astype(np.int64)
    assert set(ys.tolist()) == set(range(64)) and set(us.tolist()) == set(range(64))
    pairs = {(s, d) for s, d in zip(ys.tolist(), dv.tolist()) if s >> 2}
    assert pairs == {(s, d) for s in range(4, 64) for d in range(8)}, sorted(
        {(s, d) for s in range(4, 64) for d in range(8)} - pairs)[:10]
    assert {var_class(v) for v in vv[ys >> 2 != 0].tolist()} == set(range(-1, 14))
    lp = adjust_np((ys >> 2) << cs, vv)
    assert set(((lp[lp != 0] >> cs) & 1).tolist()) == {0, 1}          # both primary tap sets on luma
    assert set((us[us >> 2 != 0] >> 2 & 1).tolist()) == {0, 1}        # and on chroma
    assert set(dv[us >> 2 != 0].tolist()) == set(range(8))            # every source direction of the 4:2:2 remap
    for strn, s in ((ystr, ys), (uvstr, us)):
        masks = {edge_mask(a, b, h8, w8) for a, b, t in zip(gy.tolist(), gx.tolist(), s.tolist()) if t}
        assert masks == FRAME_PLACES, masks


@pytest.mark.parametrize("bd", BDS)
def test_strength_direction_variance_sweep(bd):
    c = G.ctx()
    rng = np.random.default_rng(1000 + bd)
    luma, skip8, ystr, uvstr = sweep_inputs(rng, bd)
    h8, w8 = skip8.shape
    dirs, var = O.cdef_analyze_frame(luma, bd, skip8)
    assert_sweep_coverage(bd, skip8, ystr, uvstr, dirs, var)

    # the device's directions
    d_skip = G.to_dev(skip8)
    d_dir, d_var = dev_dir_var(dirs.size)
    pl = c.plane_from_host(luma, 0)
    c.cdef_find_dir_dev(pl, bd, d_skip, d_dir, d_var)
    c.synchronize()
    np.testing.assert_array_equal(d_dir.cpu().numpy().reshape(dirs.shape), dirs)
    np.testing.assert_array_equal(d_var.cpu().numpy().reshape(var.shape), var)
    for b in sample_blocks(rng, h8, w8, 40):
        if not skip8[b]:
            blk = luma[8 * b[0]:8 * b[0] + 8, 8 * b[1]:8 * b[1] + 8]
            assert spec_direction(blk, bd) == (dirs[b], var[b]), b

    runs = [(0, 0, 0, dmp) for dmp in (3, 4, 5, 6)] + [(1, xd, yd, dmp) for xd, yd in CHROMA for dmp in (3, 6)]
    d_y, d_uv = G.to_dev(ystr), G.to_dev(uvstr)
    for plane, xd, yd, dmp in runs:
        img = np.ascontiguousarray(luma[::1 << yd, ::1 << xd]) if plane else luma
        strn = uvstr if plane else ystr
        want = O.cdef_filter_plane(img, plane, xd, yd, SW, SH, bd, dmp, skip8, dirs, var, strn)
        pin = c.plane_from_host(img, 0)
        pout = c.plane_from_host(np.zeros_like(img), 0)
        c.cdef_filter_plane_dev(pin, pout, plane, xd, yd, SW, SH, bd, dmp, d_skip, d_dir, d_var,
                                d_uv if plane else d_y)
        got = download(c, pout, img.shape, img.dtype)
        np.testing.assert_array_equal(got, want, err_msg=f"plane {plane} ({xd}, {yd}) damping {dmp}")
        spec_check_blocks(img, got, plane, xd, yd, bd, dmp, skip8, dirs, var, strn, sample_blocks(rng, h8, w8, 10))
        c.plane_free(pin)
        c.plane_free(pout)
    c.plane_free(pl)


# ---------------------------------------------------------------- 2. item lists
IW, IH = 320, 192        # 40 x 24 blocks per frame
STRIPS = [2, 3, 1, 4, 5, 2, 3, 4]


def frame_rects(rng, first_full):
    """Disjoint rects covering a 40 x 24 block grid: strips of STRIPS heights cut into pieces; the second strip
    starts with a 3-block piece (the next begins at rx8 = 3, off the superblock grid)."""
    w8 = IW // 8
    rects, y = [], 0
    for s, h in enumerate(STRIPS):
        x = 0
        while x < w8:
            if s == 0 and first_full:
                w = w8
            elif x == 0 and s in (1, 2):
                w = 3 if s == 1 else 1                   # strip 1 starts with 3 blocks, strip 2 (1 high) with one
            else:
                w = int(rng.choice([1, 2, 5, 9, 13]))
            w = min(w, w8 - x)
            rects.append((x, y, w, h))
            x += w
        y += h
    return rects


def pick_items(rng):
    """40 (frame, rect) items over 3 frames: the smallest first, a full-width strip, a 1x1 rect and rx8 = 3 rects;
    in each 32-item launch some item needs more filter tiles than the launch's first."""
    cand = [(f, r) for f in range(3) for r in frame_rects(rng, f == 0)]
    one = next(q for q in cand if q[1][2] * q[1][3] == 1)
    full = next(q for q in cand if q[1][2] == IW // 8)
    off = next(q for q in cand if q[1][0] == 3 and q != one)
    rest = [q for q in cand if q not in (one, full, off)]
    rest = [rest[i] for i in rng.choice(len(rest), 37, replace=False)]
    body = [off] + rest
    body = [body[i] for i in rng.permutation(len(body))]
    items = [one] + body
    items.insert(ITEMS_PER_LAUNCH + 4, full)        # the widest item, inside the second launch
    return items


def tiles_of(r, xdec, ydec):
    return -(-(r[2] * 8 >> xdec) // TILE_W) * -(-(r[3] * 8 >> ydec) // TILE_H)


def rect_mask(rects, h8, w8):
    m = np.zeros((h8, w8), bool)
    for x, y, w, h in rects:
        m[y:y + h, x:x + w] = True
    return m


@pytest.mark.parametrize("plane,xdec,ydec,bd", [(0, 0, 0, 10), (1, 1, 1, 8), (1, 1, 0, 12)])
def test_item_lists_across_the_32_item_split(plane, xdec, ydec, bd):
    import torch
    c = G.ctx()
    rng = np.random.default_rng(200 + 10 * plane + 2 * xdec + ydec)
    w8, h8 = IW // 8, IH // 8
    items_fr = pick_items(rng)
    assert len(set(items_fr)) == 40 and items_fr[0][1][2:] == (1, 1)
    assert min(r[2] * r[3] for _, r in items_fr) == 1 and any(r[2] == w8 for _, r in items_fr)
    assert any(r[0] == 3 for _, r in items_fr)
    for k0 in (0, ITEMS_PER_LAUNCH):               # a grid sized from a launch's first item would fall short
        chunk = items_fr[k0:k0 + ITEMS_PER_LAUNCH]
        assert max(tiles_of(r, xdec, ydec) for _, r in chunk) > tiles_of(chunk[0][1], xdec, ydec)
    for f in range(3):
        m = np.zeros((h8, w8), int)
        for x, y, w, h in (r for g, r in items_fr if g == f):
            m[y:y + h, x:x + w] += 1
        assert m.max() <= 1                         # disjoint rects inside one frame

    lumas = [textured(rng, IW, IH, bd) for _ in range(3)]
    skips = [(rng.random((h8, w8)) < 0.15).astype(np.uint8) for _ in range(3)]
    strn = rng.integers(0, 64, ((IH + 63) // 64, (IW + 63) // 64)).astype(np.uint8)
    damping = int(rng.integers(3, 7))
    ana = [O.cdef_analyze_frame(lumas[f], bd, skips[f]) for f in range(3)]
    imgs = lumas if plane == 0 else [np.ascontiguousarray(lu[::1 << ydec, ::1 << xdec]) for lu in lumas]
    wants = [O.cdef_filter_plane(imgs[f], plane, xdec, ydec, IW, IH, bd, damping, skips[f], *ana[f], strn)
             for f in range(3)]
    canaries = [rng.integers(0, 1 << bd, im.shape).astype(im.dtype) for im in imgs]
    pin = [c.plane_from_host(im, 0) for im in imgs]
    pout = [c.plane_from_host(cn, 0) for cn in canaries]
    d_skip = [G.to_dev(s) for s in skips]
    if plane == 0:
        dv = [dev_dir_var(w8 * h8) for _ in range(3)]
    else:                                          # chroma: the luma analysis comes in
        dv = [(torch.from_numpy(a[0].reshape(-1)).cuda(), torch.from_numpy(a[1].reshape(-1)).cuda()) for a in ana]
    items = (B.CdefItem * 40)()
    for k, (f, r) in enumerate(items_fr):
        it = items[k]
        it.inp, it.out = C.pointer(pin[f]), C.pointer(pout[f])
        it.d_skip8, it.d_dir, it.d_var = d_skip[f].data_ptr(), dv[f][0].data_ptr(), dv[f][1].data_ptr()
        it.rx8, it.ry8, it.rw8, it.rh8 = r
    n0 = c.launches
    c.cdef_tiles_dev(items, plane, xdec, ydec, IW, IH, bd, damping, G.to_dev(strn), find_dir=plane == 0, filter=True)
    c.synchronize()
    assert c.launches - n0 == (4 if plane == 0 else 2)     # 40 items = 2 launches per phase
    for f in range(3):
        m = rect_mask([r for g, r in items_fr if g == f], h8, w8)
        pm = np.repeat(np.repeat(m, 8 >> ydec, 0), 8 >> xdec, 1)
        got = download(c, pout[f], imgs[f].shape, imgs[f].dtype)
        np.testing.assert_array_equal(got[pm], wants[f][pm], err_msg=f"frame {f} inside the rects")
        np.testing.assert_array_equal(got[~pm], canaries[f][~pm], err_msg=f"frame {f} outside the rects")
        if plane == 0:
            gd, gv = dv[f][0].cpu().numpy().reshape(h8, w8), dv[f][1].cpu().numpy().reshape(h8, w8)
            np.testing.assert_array_equal(gd[m], ana[f][0][m])
            np.testing.assert_array_equal(gv[m], ana[f][1][m])
            assert (gd[~m] == SENT_DIR).all() and (gv[~m] == SENT_VAR).all()
        picks = [(gy, gx) for gy, gx in sample_blocks(rng, h8, w8, 30) if m[gy, gx]][:8]
        spec_check_blocks(imgs[f], got, plane, xdec, ydec, bd, damping, skips[f], *ana[f], strn, picks)

    if plane == 0:                                 # find_dir only, no output plane
        dv2 = [dev_dir_var(w8 * h8) for _ in range(3)]
        for k, (f, r) in enumerate(items_fr):
            items[k].out = None
            items[k].d_dir, items[k].d_var = dv2[f][0].data_ptr(), dv2[f][1].data_ptr()
        n0 = c.launches
        c.cdef_tiles_dev(items, 0, 0, 0, IW, IH, bd, 0, None, find_dir=True, filter=False)
        c.synchronize()
        assert c.launches - n0 == 2
        for f in range(3):
            m = rect_mask([r for g, r in items_fr if g == f], h8, w8)
            gd, gv = dv2[f][0].cpu().numpy().reshape(h8, w8), dv2[f][1].cpu().numpy().reshape(h8, w8)
            np.testing.assert_array_equal(gd[m], ana[f][0][m])
            np.testing.assert_array_equal(gv[m], ana[f][1][m])
            assert (gd[~m] == SENT_DIR).all() and (gv[~m] == SENT_VAR).all()
    for p in pin + pout:
        c.plane_free(p)


# ---------------------------------------------------------------- 3. find_dir's second grid-stride trip
def test_find_dir_grid_stride_second_trip():
    c = G.ctx()
    rng = np.random.default_rng(300)
    sms = num_sms()
    W, H = 1024, 576
    n8 = (W // 8) * (H // 8)
    per_trip = (sms * DIR_CTAS_PER_SM // ITEMS_PER_LAUNCH) * DIR_THREADS
    assert n8 > per_trip, (n8, per_trip)           # each item's loop goes round a second time
    luma = textured(rng, W, H, 8)
    masks = [None] + [(rng.random((H // 8, W // 8)) < p).astype(np.uint8) for p in (0.05, 0.3, 0.7)]
    wants = [O.cdef_analyze_frame(luma, 8, m) for m in masks]
    pl = c.plane_from_host(luma, 0)
    d_masks = [None] + [G.to_dev(m) for m in masks[1:]]
    outs = [dev_dir_var(n8) for _ in range(ITEMS_PER_LAUNCH)]
    items = (B.CdefItem * ITEMS_PER_LAUNCH)()
    for k in range(ITEMS_PER_LAUNCH):
        it = items[k]
        it.inp, it.out = C.pointer(pl), None
        it.d_skip8 = None if d_masks[k % 4] is None else d_masks[k % 4].data_ptr()
        it.d_dir, it.d_var = outs[k][0].data_ptr(), outs[k][1].data_ptr()
        it.rx8, it.ry8, it.rw8, it.rh8 = 0, 0, W // 8, H // 8
    n0 = c.launches
    c.cdef_tiles_dev(items, 0, 0, 0, W, H, 8, 0, None, find_dir=True, filter=False)
    c.synchronize()
    assert c.launches - n0 == 1
    for k in range(ITEMS_PER_LAUNCH):
        np.testing.assert_array_equal(outs[k][0].cpu().numpy().reshape(H // 8, W // 8), wants[k % 4][0], err_msg=k)
        np.testing.assert_array_equal(outs[k][1].cpu().numpy().reshape(H // 8, W // 8), wants[k % 4][1], err_msg=k)
    c.plane_free(pl)

    W, H = 7680, 4320                               # one item: the whole 8K luma plane
    n8 = (W // 8) * (H // 8)
    assert n8 > sms * DIR_CTAS_PER_SM * DIR_THREADS, n8
    luma = rng.integers(0, 1024, (H, W)).astype(np.uint16)
    dirs, var = O.cdef_analyze_frame(luma, 10)
    pl = c.plane_from_host(luma, 0)
    d_dir, d_var = dev_dir_var(n8)
    c.cdef_find_dir_dev(pl, 10, None, d_dir, d_var)
    c.synchronize()
    np.testing.assert_array_equal(d_dir.cpu().numpy().reshape(dirs.shape), dirs)
    np.testing.assert_array_equal(d_var.cpu().numpy().reshape(var.shape), var)
    c.plane_free(pl)


# ---------------------------------------------------------------- 4. planes built by the caller
def test_input_padding_is_never_read():
    """The filter must take the sentinel outside the plane, whatever the input's padding holds."""
    c = G.ctx()
    rng = np.random.default_rng(400)
    W, H, pad = 200, 136, 8
    for plane, xd, yd, bd in ((0, 0, 0, 10), (1, 1, 1, 8), (1, 1, 0, 12)):
        luma = textured(rng, W, H, bd)
        skip8 = (rng.random((H // 8, W // 8)) < 0.1).astype(np.uint8)
        dirs, var = O.cdef_analyze_frame(luma, bd, skip8)
        img = np.ascontiguousarray(luma[::1 << yd, ::1 << xd])
        strn = rng.integers(4, 64, ((H + 63) // 64, (W + 63) // 64)).astype(np.uint8)
        want = O.cdef_filter_plane(img, plane, xd, yd, W, H, bd, 6, skip8, dirs, var, strn)
        garbage = rng.integers(0, 1 << bd, (img.shape[0] + 2 * pad, img.shape[1] + 2 * pad)).astype(img.dtype)
        garbage[pad:-pad, pad:-pad] = img
        views = [G.ViewPlane(np.pad(img, pad, mode="edge"), pad, img.shape[1] + 2 * pad, 0),
                 G.ViewPlane(garbage, pad, img.shape[1] + 2 * pad + 3, 2 * img.itemsize)]
        d_skip, d_dir, d_var, d_str = G.to_dev(skip8), G.to_dev(dirs), G.to_dev(var), G.to_dev(strn)
        outs = []
        for v in views:
            pout = c.plane_from_host(np.zeros_like(img), 0)
            c.cdef_filter_plane_dev(v.plane, pout, plane, xd, yd, W, H, bd, 6, d_skip, d_dir, d_var, d_str)
            outs.append(download(c, pout, img.shape, img.dtype))
            c.plane_free(pout)
        np.testing.assert_array_equal(outs[0], want)
        np.testing.assert_array_equal(outs[1], outs[0], err_msg=f"plane {plane} ({xd}, {yd}) read its padding")


def test_misaligned_output_takes_the_scalar_stores():
    """An output plane whose element offset and odd stride leave part of the 4-pixel groups unaligned: those go
    through the scalar stores, the rest through the vector store.  Nothing outside the plane's pixels changes."""
    c = G.ctx()
    rng = np.random.default_rng(500)
    W, H = 264, 136
    for plane, xd, yd, bd in ((0, 0, 0, 8), (1, 1, 0, 12), (1, 1, 1, 10)):
        luma = textured(rng, W, H, bd)
        skip8 = (rng.random((H // 8, W // 8)) < 0.1).astype(np.uint8)
        dirs, var = O.cdef_analyze_frame(luma, bd, skip8)
        img = np.ascontiguousarray(luma[::1 << yd, ::1 << xd])
        h, w = img.shape
        strn = rng.integers(0, 64, ((H + 63) // 64, (W + 63) // 64)).astype(np.uint8)
        want = O.cdef_filter_plane(img, plane, xd, yd, W, H, bd, 4, skip8, dirs, var, strn)
        pad, bpp = 4, img.itemsize
        stride = w + 2 * pad + 1                        # odd: the alignment of a row's groups changes row by row
        canvas = rng.integers(0, 1 << bd, (h + 2 * pad, w + 2 * pad)).astype(img.dtype)
        vp = G.ViewPlane(canvas, pad, stride, 3 * bpp)
        base, data = vp.buf.data_ptr(), vp.plane.data
        # the kernel's 4-pixel groups start at multiples of 4 (whole-plane tiles are 64 pixels wide)
        gx = np.arange(0, w, 4)
        addr = data + (np.arange(h)[:, None] * stride + gx[None, :]) * bpp
        vec = (addr % (4 * bpp) == 0) & (gx[None, :] + 4 <= w)
        share = 1 - vec.mean()
        assert 0.5 < share < 0.9, share                 # both store paths, measured from the addresses
        before = vp.buf.cpu().numpy().copy()
        pin = c.plane_from_host(img, 0)
        c.cdef_filter_plane_dev(pin, vp.plane, plane, xd, yd, W, H, bd, 4, G.to_dev(skip8), G.to_dev(dirs),
                                G.to_dev(var), G.to_dev(strn))
        c.synchronize()
        after = vp.buf.cpu().numpy()
        expect = before.copy()
        off = data - base
        for y in range(h):
            o = off + y * stride * bpp
            expect[o:o + w * bpp] = want[y].view(np.uint8)
        np.testing.assert_array_equal(after, expect, err_msg=f"plane {plane} ({xd}, {yd}) {bd}-bit")
        c.plane_free(pin)


# ---------------------------------------------------------------- 5. per-call forms
@pytest.mark.parametrize("bd", BDS)
def test_percall_filter_block_every_shape_direction_edge(bd):
    L, OL = B.lib(), O.lib()
    rng = np.random.default_rng(600 + bd)
    cs, maxv = bd - 8, (1 << bd) - 1
    dtype = pxdt(bd)
    isz = np.dtype(dtype).itemsize
    sel_seen, ends_seen = set(), set()
    n = 0
    for xdec, ydec in ((0, 0), (1, 1), (1, 0)):
        xs, ys = 8 >> xdec, 8 >> ydec
        lo, hi = 3 + cs - xdec, 6 + cs - xdec           # final damping: luma 3..6 + cs, chroma one less
        for d in range(8):
            for edges in range(16):
                kind = rng.choice(3, (ys + 4, xs + 4), p=[0.2, 0.45, 0.35])
                tmp = np.where(kind == 0, 0, np.where(kind == 1, maxv, rng.integers(0, maxv + 1, kind.shape)))
                tmp = tmp.astype(np.uint16)
                if not edges & 1:
                    tmp[:, :2] = 0x8000
                if not edges & 2:
                    tmp[:, -2:] = 0x8000
                if not edges & 4:
                    tmp[:2, :] = 0x8000
                if not edges & 8:
                    tmp[-2:, :] = 0x8000
                pri = (15 if n % 3 == 0 else int(rng.integers(0, 16))) << cs
                sec = (0, 1, 2, 4)[(n // 3) % 4] << cs
                damping = hi if n % 2 else lo
                n += 1
                want = np.zeros((ys, xs), dtype)
                OL.orc_cdef_filter_block(O.ptr(want), xs, isz, O.ptr(tmp, 2 * (xs + 4) + 2), xs + 4, pri, sec,
                                         d, damping, bd, xdec, ydec, edges)
                got = np.full((ys, xs + 3), 0x5A, dtype)    # a destination wider than the block
                L.b200_cdef_filter_block(got.ctypes.data, (xs + 3) * isz, O.ptr(tmp, 2 * (xs + 4) + 2),
                                         (xs + 4) * 2, pri, sec, d, damping, bd, xdec, ydec)
                msg = f"{xs}x{ys} dir {d} edges {edges} pri {pri} sec {sec} damping {damping}"
                np.testing.assert_array_equal(got[:, :xs], want, err_msg=msg)
                assert (got[:, xs:] == 0x5A).all(), msg
                np.testing.assert_array_equal(spec_filter(tmp, xs, ys, pri, sec, d, damping, bd, edges), want,
                                              err_msg="spec " + msg)
                sel_seen.add((pri >> cs) & 1 if pri else None)
                ends_seen.add((xdec, damping))
    assert {0, 1} <= sel_seen
    assert ends_seen == {(x, e + cs - x) for x in (0, 1) for e in (3, 6)}


@pytest.mark.parametrize("bd", BDS)
def test_percall_dir_patterns_contrast_low_bits_and_ties(bd):
    L = B.lib()
    rng = np.random.default_rng(700 + bd)
    cs, maxv = bd - 8, (1 << bd) - 1
    dtype = pxdt(bd)
    isz = np.dtype(dtype).itemsize

    def dev_dir(blk):
        img = np.zeros((8, 24), dtype)                   # the block inside a wider image
        img[:, 8:16] = blk
        v = C.c_uint32()
        d = L.b200_cdef_dir(img.ctypes.data + 8 * isz, 24 * isz, C.byref(v), bd)
        return d, v.value

    def check(blk):
        blk = blk.astype(dtype)
        got = dev_dir(blk)
        assert got == O.cdef_find_dir(blk, bd) == spec_direction(blk, bd), got
        return got

    # one oriented block per direction
    for d in range(8):
        for _ in range(4):
            blk = (np.clip(np.rint(stripes(rng, d, rng.uniform(40, 120))), 0, 255).astype(np.int64) << cs)
            assert check(blk)[0] == d
    # maximum contrast: the largest variances, past adjust_strength's clamp
    big = []
    for blk in (_I % 2, _J % 2, (_I + _J) // 2 % 2, (_I - _J) // 2 % 2, 1 - _I % 2, (_I + _J) % 2, _I // 4 % 2):
        big.append(check(np.where(blk > 0, maxv, 0))[1])
    assert max(big) >> 6 >= 1 << 13, big
    # random low bits at 10 / 12 bit are shifted away before the search
    for t in range(24):
        b8 = np.clip(np.rint(stripes(rng, t % 8, 2.0 ** rng.uniform(0, 7))), 0, 255).astype(np.int64)
        blk = (b8 << cs) | rng.integers(0, 1 << cs, (8, 8))
        assert check(blk) == O.cdef_find_dir(b8.astype(np.uint8), 8)
    # ties: a block symmetric under transpose has cost[1] == cost[7], cost[2] == cost[6], cost[3] == cost[5]
    ties, tied = 0, set()
    for t in range(240):
        if t % 2:
            s = rng.integers(0, 256, (8, 8))
        else:
            s = stripes(rng, 1 + t % 3, rng.uniform(8, 120))
        sym = np.rint((s + s.T) / 2).astype(np.int64) << cs | (rng.integers(0, 1 << cs, (8, 8)) if cs else 0)
        sym = np.minimum(sym, maxv)
        cost = spec_direction_costs(sym, bd)
        best = max(cost)
        first = cost.index(best)
        got = check(sym)
        assert got[0] == first
        if cost.count(best) > 1:
            ties += 1
            tied.add(first)
    assert ties >= 60 and tied == {1, 2, 3}, (ties, tied)   # shared maxima 1 / 7, 2 / 6 and 3 / 5, first wins


# ---------------------------------------------------------------- 6. rejections
RW, RH = 64, 320         # 8 x 40 blocks: 40 one-row items, items[k] = row k
# (id, call arguments that differ from the valid luma call, (in, out) planes, {item index: field overrides});
# plane names resolve in the fixture below
REJECTIONS = [
    ("item35_null_dir", {}, ("luma", "out"), {35: dict(d_dir=None)}),
    ("item35_rect_outside", {}, ("luma", "out"), {35: dict(rx8=RW // 8 - 1, rw8=2)}),
    ("out_is_in_with_find_dir", {}, ("luma", "out"), {7: dict(out="luma")}),
    ("null_strengths", dict(d_strength_sb=None), ("luma", "out"), {}),
    ("damping_2", dict(damping=2), ("luma", "out"), {}),
    ("damping_7", dict(damping=7), ("luma", "out"), {}),
    ("layout_440", dict(plane=1, xdec=0, ydec=1, find_dir=False), ("luma", "out"), {}),
    ("luma_with_xdec", dict(xdec=1), ("luma", "out"), {}),
    ("in_smaller_than_luma", {}, ("luma", "out"), {3: dict(inp="small")}),
    ("out_smaller_than_luma", {}, ("luma", "out"), {3: dict(out="small")}),
    ("in_stride_below_width", {}, ("luma", "out"), {3: dict(inp="short_stride")}),
    ("chroma_in_smaller", dict(plane=1, xdec=1, ydec=1, find_dir=False), ("csmall", "cout"), {}),
    ("chroma_out_smaller", dict(plane=1, xdec=1, ydec=1, find_dir=False), ("chroma", "csmall"), {}),
    ("out_bpp_differs", {}, ("luma", "out"), {3: dict(out="wide")}),
    ("rect_outside_grid", {}, ("luma", "out"), {0: dict(ry8=RH // 8)}),
    ("bit_depth_9", dict(bit_depth=9), ("luma", "out"), {}),
    ("luma_width_not_multiple_of_8", dict(luma_w=RW - 4), ("luma", "out"), {}),
]


@pytest.fixture(scope="module")
def rejection_setup():
    c = G.ctx()
    rng = np.random.default_rng(800)
    luma = textured(rng, RW, RH, 8)
    canary = rng.integers(0, 256, (RH, RW)).astype(np.uint8)
    ccanary = np.ascontiguousarray(canary[::2, ::2])
    pl = {"luma": c.plane_from_host(luma, 0), "out": c.plane_from_host(canary, 0),
          "small": c.plane_from_host(luma[:RH - 8], 0), "wide": c.plane_from_host(luma.astype(np.uint16), 0),
          "chroma": c.plane_from_host(luma[::2, ::2], 0), "cout": c.plane_from_host(ccanary, 0),
          "csmall": c.plane_from_host(canary[:RH // 2 - 1, ::2], 0)}
    owned = list(pl.values())
    pl["short_stride"] = B.Plane.from_buffer_copy(pl["luma"])
    pl["short_stride"].stride = RW - 1
    d_dir, d_var = dev_dir_var((RW // 8) * (RH // 8))
    d_str = G.to_dev(rng.integers(0, 64, ((RH + 63) // 64, 1)).astype(np.uint8))

    def items_for(inp, out, over=None):
        items = (B.CdefItem * 40)()
        for k in range(40):
            it = items[k]
            it.inp, it.out = C.pointer(pl[inp]), C.pointer(pl[out])
            it.d_dir, it.d_var = d_dir.data_ptr(), d_var.data_ptr()
            it.rx8, it.ry8, it.rw8, it.rh8 = 0, k, RW // 8, 1
            for a, v in (over or {}).get(k, {}).items():
                setattr(it, a, C.pointer(pl[v]) if isinstance(v, str) else v)
        return items

    ok = dict(plane=0, xdec=0, ydec=0, luma_w=RW, luma_h=RH, bit_depth=8, damping=5, d_strength_sb=d_str,
              find_dir=True, filter=True)
    # the valid forms of the calls run: luma find_dir + filter, 4:2:0 chroma filter
    c.cdef_tiles_dev(items_for("luma", "out"), **ok)
    c.cdef_tiles_dev(items_for("chroma", "cout"), **{**ok, "plane": 1, "xdec": 1, "ydec": 1, "find_dir": False})
    c.synchronize()
    yield c, pl, items_for, ok, d_dir, d_var, canary, ccanary
    for p in owned:
        c.plane_free(p)


@pytest.mark.parametrize("case", REJECTIONS, ids=[r[0] for r in REJECTIONS])
def test_rejection_launches_nothing_and_writes_nothing(rejection_setup, case):
    c, pl, items_for, ok, d_dir, d_var, canary, ccanary = rejection_setup
    name, kw, (inp, out), over = case
    d_dir.fill_(SENT_DIR)
    d_var.fill_(SENT_VAR)
    c.check(c.L.b200_plane_upload(c.h, C.byref(pl["out"]), canary.ctypes.data, canary.strides[0]))
    c.check(c.L.b200_plane_upload(c.h, C.byref(pl["cout"]), ccanary.ctypes.data, ccanary.strides[0]))
    c.synchronize()
    items = items_for(inp, out, over)
    n0 = c.launches
    with pytest.raises(B.B200Error) as e:
        c.cdef_tiles_dev(items, **{**ok, **kw})
    assert e.value.status == B.ERR_ARG
    assert c.launches == n0
    c.synchronize()
    assert (d_dir.cpu().numpy() == SENT_DIR).all() and (d_var.cpu().numpy() == SENT_VAR).all()
    np.testing.assert_array_equal(download(c, pl["out"], canary.shape, canary.dtype), canary)
    np.testing.assert_array_equal(download(c, pl["cout"], ccanary.shape, ccanary.dtype), ccanary)


def test_no_items_launch_nothing(rejection_setup):
    c, pl, items_for, ok, *_ = rejection_setup
    n0 = c.launches
    c.cdef_tiles_dev((B.CdefItem * 0)(), **ok)
    assert c.launches == n0
