"""Intra prediction on every kernel path, bit exact against the oracle and, for a fixed-seed sample of every
sweep, against the AV1 specification restated in tests/test_oracle_predict_spec.py.

The kernels:
- `ipred_kernel<T>` (ipred.cu): b200_predict_intra_dev and the per-call b200_predict_intra; one CTA per
  (block, mode) item running the preparation and per-pixel predictors of ipred_dev.cuh on a CtaGroup;
- `cfl_ac_kernel<T>` (ipred.cu): b200_pred_cfl_ac_dev, the CfL "ac" input;
- `intra_edges_kernel<T>` (intra_edges.cu): b200_get_intra_edges_dev, one warp per IntraEdge buffer
  (intra_edges_dev.cuh).
The sweeps:
1. all 19 TxSizes x the 8 directional modes x angle deltas -3..3 x ief -1 / 0 / 1 at 8 / 10 / 12 bit, with
   the non-directional modes mixed in, on random, ramp and all-maximum edges at the lengths the encoder
   gives; one shuffled launch per (size, bit depth), larger than the grid cap;
2. edge buffers built on the device for luma, 4:2:0 and 4:2:2 chroma, in the whole frame and in two tiles,
   including blocks on the frame's last column and row, predicted at the device lengths; the prediction is
   repeated with every entry outside the initialised slices randomised; the edge launch is larger than its
   grid cap;
3. the edge filter's num_above / num_left clip at the plane's right and bottom border;
4. CfL: ac for every block size the kernel accepts, every legal padding, 4:2:0 / 4:2:2 / 4:4:4 and four
   kinds of luma at 8 / 10 / 12 bit, then the prediction at alphas -16 .. 16 with every DC variant;
5. the per-call form at 10 and 12 bit into a destination wider than the block;
6. the host-side checks: n = 0 and rejected arguments launch nothing.
Every output buffer is filled with a sentinel before each launch."""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_intra_edges_gpu import TX, make_items, oracle_edges
from tests.test_oracle_intra_edges import BSIZES
from tests.test_oracle_predict_spec import (spec_directional, spec_nondirectional, strength_selection,
                                            upsample_selection)

pytestmark = pytest.mark.gpu

BDS = [8, 10, 12]
LAYOUTS = [(0, 0), (1, 1), (1, 0)]                     # (xdec, ydec): luma / 4:4:4, 4:2:0, 4:2:2
M = {n: i for i, n in enumerate(O.MODES)}
DIRECTIONAL = list(O.MODE_ANGLE)                        # V, H, D45, D135, D113, D157, D203, D67
ANGLE_OF = {M[n]: a for n, a in O.MODE_ANGLE.items()}
DELTAS = range(-3, 4)
NONDIR = [("DC_PRED", v) for v in range(4)] + [(m, 3) for m in ("SMOOTH_PRED", "SMOOTH_V_PRED", "SMOOTH_H_PRED",
                                                                  "PAETH_PRED", "V_PRED", "H_PRED")]
SENTINEL = 0xA5                                         # every output byte before a launch

# Launch geometry mirrored from the sources: each kernel's grid is capped, then a grid-stride loop runs the rest.
IPRED_CTAS_PER_SM = 32    # ipred.cu:141  min(nitems, num_sms * 32), one item per CTA per trip
CFL_CTAS_PER_SM = 32      # ipred.cu:162  min(nblocks, num_sms * 32), one block per CTA per trip
EDGE_WARPS_PER_CTA = 8    # intra_edges.cu:73  one item per warp
EDGE_CTAS_PER_SM = 16     # intra_edges.cu:74  min(ceil(nitems / 8), num_sms * 16)


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def second_trip(cap):
    """An item count with one full grid pass and a ragged second one."""
    return cap + cap // 2 + 3


def pxdt(bd):
    return np.uint8 if bd == 8 else np.uint16


# ---------------------------------------------------------------- items and references
def is_directional(mode, angle):
    return 1 <= mode <= 8 and not (mode == M["V_PRED"] and angle == 90) and not (mode == M["H_PRED"] and angle == 180)


def encoder_lens(w, h, mode, angle):
    """(init_left, init_above) that get_intra_edges gives a block with a left neighbour (partition.rs:704-707):
    the left column grows by the bottom-left part only above 180 degrees, the row by the top-right below 90."""
    d = is_directional(mode, angle)
    return h + (w if d and angle > 180 else 0), w + (h if d and angle < 90 else 0)


def corner_filters(w, h, angle, ief):
    """get_intra_edges filters the top-left entry for these predictions (partition.rs:886-892)."""
    return ief >= 0 and 90 < angle < 180 and w + h >= 24


def corner_filtered(e):
    f = e.copy()
    f[128] = (int(e[127]) * 5 + int(e[128]) * 6 + int(e[129]) * 5 + 8) >> 4
    return f


def make_intra_items(rows):
    """rows of (edge, ac, x, y, angle, mode, variant, ief, left_len, above_len)."""
    return np.array([tuple(int(v) for v in r) + (0,) for r in rows], B.INTRA_ITEM_DTYPE)


def oracle_batch(edges, items, w, h, bd, ac=None, plane_wh=(4096, 4096)):
    """orc_predict_intra_batch: the oracle's predict_intra for every item (OpenMP)."""
    f = O.lib().orc_predict_intra_batch
    f.restype = None
    f.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p] + [C.c_int] * 5 + [C.c_void_p]
    edges, items = np.ascontiguousarray(edges), np.ascontiguousarray(items)
    out = np.zeros((len(items), h, w), edges.dtype)
    acp = None if ac is None else np.ascontiguousarray(ac, np.int16)
    f(edges.ctypes.data, edges.itemsize, items.ctypes.data, len(items), None if acp is None else acp.ctypes.data,
      w, h, bd, plane_wh[0], plane_wh[1], out.ctypes.data)
    return out


def extend(vals, n):
    """The first n entries of an edge whose initialised part is `vals`, the last value repeated beyond it (the
    specification's edge preparation replicates it; the reference leaves the rest uninitialised)."""
    vals = [int(v) for v in vals]
    return (vals + [vals[-1]] * n)[:n]


def spec_predict(e_raw, it, w, h, bd, plane_wh=(4096, 4096)):
    """The specification's prediction of item `it` from the edge buffer `e_raw`, whose top-left entry has not been
    through get_intra_edges' corner filter (spec_directional applies it).  Only the entries inside the item's
    lengths are read.  At the lengths the encoder gives (init_left = h without the bottom-left part, init_above
    = w without the top-right part) the reference never reads past them, so the replicated tail never reaches
    a predicted pixel: no sampled item disagrees with the specification."""
    mode, angle, variant, ief = int(it["mode"]), int(it["angle"]), int(it["variant"]), int(it["ief"])
    tl = int(e_raw[128])
    if is_directional(mode, angle):
        n = w + h + 1
        above = extend(e_raw[129:129 + int(it["above_len"])], n)
        left = extend(e_raw[127::-1][:int(it["left_len"])], n)
        return spec_directional([tl] + above, [tl] + left, w, h, angle, bd, ief >= 0, max(ief, 0), int(it["x"]),
                                int(it["y"]), plane_wh[0] - 1, plane_wh[1] - 1)
    name = "DC_PRED" if mode == M["UV_CFL_PRED"] else O.MODES[mode]
    return spec_nondirectional(name, variant, e_raw[129:129 + w], e_raw[127::-1][:h], tl, w, h, bd)


def describe(it, w, h):
    return (f"{w}x{h} {O.MODES[int(it['mode'])]} angle {int(it['angle'])} ief {int(it['ief'])} variant "
            f"{int(it['variant'])} lens ({int(it['left_len'])}, {int(it['above_len'])}) at ({int(it['x'])}, "
            f"{int(it['y'])}) edge {int(it['edge'])}")


def check(got, want, items, w, h, what, name=None):
    bad = np.flatnonzero((got.reshape(len(got), -1) != want.reshape(len(want), -1)).any(1))
    if len(bad):
        first = name(bad[0]) if name else describe(items[bad[0]], w, h)
        raise AssertionError(f"{what}: {len(bad)} of {len(got)} items differ, first: {first}")


def spec_sample(rng, raw, items, got, w, h, bd, count, plane_wh=(4096, 4096), raw_of=None):
    """Compares a fixed-seed sample of `count` directional and count // 3 other items with the specification;
    raw_of(k) gives item k's unfiltered edge (default: raw[item.edge % len(raw)])."""
    d = np.array([is_directional(int(it["mode"]), int(it["angle"])) for it in items], bool)
    picks = []
    for pool, c in ((np.flatnonzero(d), count), (np.flatnonzero(~d), count // 3)):
        if len(pool):
            picks += rng.choice(pool, min(c, len(pool)), replace=False).tolist()
    for k in picks:
        e = raw_of(k) if raw_of else raw[int(items[k]["edge"]) % len(raw)]
        want = spec_predict(e, items[k], w, h, bd, plane_wh)
        np.testing.assert_array_equal(got[k], want, err_msg="specification: " + describe(items[k], w, h))


# ---------------------------------------------------------------- device side
def dev_out(nbytes, slack=256):
    import torch
    return torch.full((nbytes + slack,), SENTINEL, dtype=torch.uint8, device="cuda")


def host_out(d, nbytes, dtype, shape):
    raw = d.cpu().numpy()
    assert (raw[nbytes:] == SENTINEL).all(), "bytes written past the last output"
    return raw[:nbytes].view(dtype).reshape(shape)


def predict(d_edges, items, w, h, bd, d_ac=None, plane_wh=(4096, 4096)):
    n = len(items)
    nbytes = n * w * h * np.dtype(pxdt(bd)).itemsize
    d = dev_out(nbytes)
    G.ctx().predict_intra_dev(d_edges, G.to_dev(items), n, d_ac, w, h, bd, plane_wh[0], plane_wh[1], d)
    G.ctx().synchronize()
    return host_out(d, nbytes, pxdt(bd), (n, h, w))


def ipred_kernels(fn):
    return G.profiled_kernels(fn, prefix="ipred_")


def tname(bd):
    return "unsigned char" if bd == 8 else "unsigned short"


# ---------------------------------------------------------------- 1. every angle, size and filter setting
def synthetic_edges(rng, bd, per_kind):
    """Raw edge buffers of three kinds - uniform random, a smooth ramp (rising or falling through the corner)
    and all-maximum - followed by the same buffers with the top-left entry corner-filtered."""
    maxv = (1 << bd) - 1
    raw = []
    for k in range(per_kind):
        ramp = np.sort(rng.integers(0, maxv + 1, O.EDGE_LEN))
        raw += [rng.integers(0, maxv + 1, O.EDGE_LEN), ramp if k % 2 else ramp[::-1], np.full(O.EDGE_LEN, maxv)]
    raw = np.array(raw).astype(pxdt(bd))
    return raw, np.concatenate([raw, np.array([corner_filtered(e) for e in raw])])


def sweep_row(w, h, r, nraw, mode, angle, variant, ief, x=64, y=64):
    """An item on raw edge r, or on its corner-filtered copy where get_intra_edges would have filtered it."""
    edge = r + nraw if is_directional(mode, angle) and corner_filters(w, h, angle, ief) else r
    return (edge, 0, x, y, angle, mode, variant, ief) + encoder_lens(w, h, mode, angle)


@pytest.mark.parametrize("bd", BDS)
def test_every_angle_size_and_filter_setting(bd):
    """All 56 angles x ief -1 / 0 / 1 plus the non-directional modes at every TxSize, on every edge kind, in one
    shuffled launch per size: consecutive items of a CTA differ in kind, and the launch is half as large again
    as the capped grid, so the grid-stride loop makes a ragged second trip."""
    rng = np.random.default_rng(10 + bd)
    raw, edges = synthetic_edges(rng, bd, 4)
    d_edges = G.to_dev(edges)
    nraw = len(raw)
    cap = num_sms() * IPRED_CTAS_PER_SM
    n = second_trip(cap)
    combos = [(M[m], ANGLE_OF[M[m]] + 3 * d, 3, ief) for m in DIRECTIONAL for d in DELTAS for ief in (-1, 0, 1)]
    combos += [(M[m], ANGLE_OF.get(M[m], 0), v, -1) for m, v in NONDIR]
    assert len({c[1] for c in combos if 1 <= c[0] <= 8}) == 56             # 90 and 180 included
    strengths, ups = set(), set()
    for w, h in O.TX_SIZES:
        rows = [sweep_row(w, h, r, nraw, *c) for r in range(nraw) for c in combos]
        for _ in range(n - len(rows)):
            rows.append(sweep_row(w, h, int(rng.integers(nraw)), nraw, *combos[int(rng.integers(len(combos)))]))
        rows = [rows[i] for i in rng.permutation(len(rows))]
        items = make_intra_items(rows)
        assert len(items) == n and cap < n < 2 * cap
        if (w, h) == (8, 8):
            got = {}
            assert ipred_kernels(lambda: got.setdefault("v", predict(d_edges, items, w, h, bd))) == \
                [f"ipred_kernel<{tname(bd)}>"]
            got = got["v"]
        else:
            got = predict(d_edges, items, w, h, bd)
        check(got, oracle_batch(edges, items, w, h, bd), items, w, h, f"{w}x{h} {bd}-bit")
        spec_sample(rng, raw, items, got, w, h, bd, 12)
        for mode, angle, _, ief in combos:
            if is_directional(mode, angle) and ief >= 0:
                for delta in (angle - 90, angle - 180):
                    strengths.add(strength_selection(w, h, ief, delta))
                ups.add(("above", upsample_selection(w, h, ief, angle - 90)))
                ups.add(("left", upsample_selection(w, h, ief, angle - 180)))
    assert {1, 2, 3} <= strengths
    assert {("above", 1), ("left", 1)} <= ups


# ---------------------------------------------------------------- 2. real edge buffers end to end
def border_items(rng, rw, rh, dec):
    """Transform blocks on the region's last column, last row and bottom-right corner, each its own partition,
    for every TxSize whose luma partition exists (and is at most 64 x 64)."""
    rows = []
    for ts, (tw, th) in enumerate(TX):
        luma = (tw << dec[0], th << dec[1])
        if luma not in BSIZES or max(luma) > 64:
            continue
        lastx, lasty = (rw - 1) // tw * tw, (rh - 1) // th * th
        for x, y in ((lastx, int(rng.integers(0, lasty // th + 1)) * th),
                     (int(rng.integers(0, lastx // tw + 1)) * tw, lasty), (lastx, lasty)):
            mode = int(rng.choice(list(range(14)) + [255]))
            rows.append((x, y, (x << dec[0]) >> 2, (y << dec[1]) >> 2, 0, 0, BSIZES.index(luma), ts, mode,
                         int(rng.integers(-3, 4)) if 1 <= mode <= 8 else 0, int(rng.integers(0, 2)), 0))
    return np.array(rows, B.EDGE_ITEM_DTYPE)


def prediction_for(rng, it, k, lens, rect):
    """The b200_intra_item the encoder would predict from edge buffer k: the variant from the region-relative
    position (PredictionVariant::new, predict.rs:126-135), PAETH remapped as predict_intra does
    (predict.rs:228-234), the filter type drawn where the edge filter is on.  Edges gathered for no mode (255)
    drive a non-directional mode, CfL edges a CfL prediction with alpha 0."""
    x, y = int(it["po_x"]), int(it["po_y"])
    variant = (1 if x else 0) + (2 if y else 0)
    m, delta = int(it["mode"]), int(it["angle_delta"])
    if m == 255:
        m, delta = int(rng.choice([0, 9, 10, 11, 12])), 0
    if m == M["PAETH_PRED"]:
        m = {0: 0, 2: 1, 1: 2, 3: m}[variant]
    angle = ANGLE_OF.get(m, 0) + 3 * delta
    ief = int(rng.integers(0, 2)) if is_directional(m, angle) and it["enable_ief"] else -1
    return (k, 0, rect[0] + x, rect[1] + y, angle, m, variant, ief, lens[k, 0], lens[k, 1])


def initialised(lens):
    """(n, 257): the entries [128 - init_left, 129 + init_above) of each buffer."""
    idx = np.arange(O.EDGE_LEN)
    return (idx >= 128 - lens[:, :1].astype(int)) & (idx < 129 + lens[:, 1:].astype(int))


def randomise_outside(rng, edges, lens, maxv):
    """Every entry outside the initialised slices replaced by a random value."""
    out = rng.integers(0, maxv + 1, edges.shape).astype(edges.dtype)
    inside = initialised(lens)
    out[inside] = edges[inside]
    return out


@pytest.mark.parametrize("bd", BDS)
def test_real_edge_buffers_end_to_end(bd):
    """b200_get_intra_edges_dev -> b200_predict_intra_dev at the device lengths == oracle edges -> oracle
    prediction, for luma and 4:2:0 / 4:2:2 chroma in the frame, in a tile inside it and in a tile at its
    bottom-right.  The frame launch of the luma plane runs more items than intra_edges_kernel's capped grid
    holds.  The prediction must not change when the entries outside the initialised slices hold random values
    (uninitialised memory upstream)."""
    c = G.ctx()
    rng = np.random.default_rng(200 + bd)
    maxv = (1 << bd) - 1
    edge_cap = num_sms() * EDGE_CTAS_PER_SM * EDGE_WARPS_PER_CTA
    big = second_trip(edge_cap)
    short_zones, angles, overhang, origin = set(), set(), {"x": False, "y": False}, 0
    for dec in LAYOUTS:
        PW, PH = 208 >> dec[0], 152 >> dec[1]
        img = rng.integers(0, maxv + 1, (PH, PW)).astype(pxdt(bd))
        pl = c.plane_from_host(img, 8)
        for rect in ((0, 0, PW, PH), (64 >> dec[0], 64 >> dec[1], 96 >> dec[0], 64 >> dec[1]),
                     (128 >> dec[0], 64 >> dec[1], 128 >> dec[0], 128 >> dec[1])):
            rw, rh = min(rect[2], PW - rect[0]), min(rect[3], PH - rect[1])
            border = border_items(rng, rw, rh, dec)
            n = big if (dec, rect[0]) == ((0, 0), 0) else 1500
            items = np.concatenate([make_items(rng, rw, rh, dec, n - len(border)), border])
            d_edges = dev_out(n * 257 * img.itemsize)
            d_lens = dev_out(2 * n)
            call = lambda: c.get_intra_edges_dev(pl, rect, dec[0], dec[1], bd, G.to_dev(items), n, d_edges, d_lens)
            if n == big:
                assert (n + EDGE_WARPS_PER_CTA - 1) // EDGE_WARPS_PER_CTA > num_sms() * EDGE_CTAS_PER_SM
                assert G.profiled_kernels(call, prefix="intra_edges_") == [f"intra_edges_kernel<{tname(bd)}>"]
            else:
                call()
            c.synchronize()
            got_e = host_out(d_edges, n * 257 * img.itemsize, img.dtype, (n, 257))
            lens = host_out(d_lens, 2 * n, np.uint8, (n, 2))
            want_e = np.zeros_like(got_e)
            for k in range(n):
                want_e[k], il, ia = oracle_edges(img, rect, dec, bd, items[k])
                assert (int(lens[k, 0]), int(lens[k, 1])) == (il, ia), items[k]
            # Only the initialised slices are compared: where tx_w > tx_h the reference writes up to tx_w top-right
            # pixels (likewise bottom-left), past init_above; the device writes zeros there.
            inside = initialised(lens)
            check(np.where(inside, got_e, 0), np.where(inside, want_e, 0), None, 0, 0,
                  f"edges {bd}-bit dec {dec} rect {rect}", lambda k: str(items[k]))
            assert (got_e[~inside] == 0).all(), "entries outside the initialised slices are not zero"
            origin += int(((items["po_x"] == 0) & (items["po_y"] == 0)).sum())
            tws, ths = np.array(TX)[items["tx_size"]].T
            overhang["x"] |= bool((items["po_x"] + tws > rw).any())
            overhang["y"] |= bool((items["po_y"] + ths > rh).any())
            pit = make_intra_items([prediction_for(rng, it, k, lens, rect) for k, it in enumerate(items)])
            rand_e = randomise_outside(rng, got_e, lens, maxv)
            d_rand = G.to_dev(rand_e)
            for ts, (tw, th) in enumerate(TX):
                sel = np.flatnonzero(items["tx_size"] == ts)
                if len(sel) == 0:
                    continue
                p = pit[sel]
                what = f"{bd}-bit dec {dec} rect {rect}"
                got = predict(d_edges, p, tw, th, bd, plane_wh=(PW, PH))
                check(got, oracle_batch(want_e, p, tw, th, bd, plane_wh=(PW, PH)), p, tw, th, what)
                check(predict(d_rand, p, tw, th, bd, plane_wh=(PW, PH)), got, p, tw, th,
                      what + " with random entries outside the lengths")

                def unfiltered(j):                      # the buffer before get_intra_edges' corner filter
                    it = items[sel[j]].copy()
                    it["enable_ief"] = 0
                    return oracle_edges(img, rect, dec, bd, it)[0]
                spec_sample(rng, None, p, got, tw, th, bd, 3, plane_wh=(PW, PH), raw_of=unfiltered)
                for it in p:
                    mode, angle = int(it["mode"]), int(it["angle"])
                    if 1 <= mode <= 8:
                        angles.add(angle)
                    if is_directional(mode, angle):
                        if min(int(it["left_len"]), int(it["above_len"])) < tw + th:
                            short_zones.add(1 if angle < 90 else 2 if angle < 180 else 3)
        c.plane_free(pl)
    assert short_zones == {1, 2, 3}
    assert len(angles) == 56
    assert overhang == {"x": True, "y": True} and origin > 0


# ---------------------------------------------------------------- 3. plane-border clipping of the filter length
@pytest.mark.parametrize("bd", BDS)
def test_filter_length_clipped_at_the_plane_border(bd):
    """num_above = min(w, plane_w - x) + ... and num_left likewise (predict.rs:1335-1400): dst_x at plane_w - k
    for k = 1, 2, w/2, w - 1, w, w + 4 - clipped, exactly full and not clipped - and the same for y, for every
    directional angle with either filter type."""
    rng = np.random.default_rng(300 + bd)
    raw, edges = synthetic_edges(rng, bd, 2)
    d_edges = G.to_dev(edges)
    nraw = len(raw)
    PW, PH = 1000, 600
    for w, h in O.TX_SIZES:
        rows, seen = [], {"above": set(), "left": set()}
        for m in DIRECTIONAL:
            for d in DELTAS:
                angle = ANGLE_OF[M[m]] + 3 * d
                if not is_directional(M[m], angle):
                    continue
                for ief in (0, 1):
                    pos = [(PW - k, 64) for k in sorted({1, 2, w // 2, w - 1, w, w + 4})]
                    pos += [(64, PH - k) for k in sorted({1, 2, h // 2, h - 1, h, h + 4})]
                    for x, y in pos:
                        rows.append(sweep_row(w, h, int(rng.integers(nraw)), nraw, M[m], angle, 3, ief, x, y))
                        if strength_selection(w, h, ief, angle - 90):
                            seen["above"].add(int(np.sign(PW - x - w)))   # clipped / full / not
                        if strength_selection(w, h, ief, angle - 180):
                            seen["left"].add(int(np.sign(PH - y - h)))
        assert seen == {"above": {-1, 0, 1}, "left": {-1, 0, 1}}, (w, h, seen)
        items = make_intra_items(rows)
        got = predict(d_edges, items, w, h, bd, plane_wh=(PW, PH))
        check(got, oracle_batch(edges, items, w, h, bd, plane_wh=(PW, PH)), items, w, h, f"{w}x{h} {bd}-bit border")
        spec_sample(rng, raw, items, got, w, h, bd, 6, plane_wh=(PW, PH))


# ---------------------------------------------------------------- 4. CfL
CFL_SIDES = (4, 8, 16, 32)
CFL_ALPHAS = (-16, -1, 0, 1, 16)
BAND = 128                # the luma plane: four 128-wide bands of random, zero, maximum and checkerboard luma


def cfl_luma(rng, bd, xdec, ydec):
    maxv = (1 << bd) - 1
    img = np.zeros((BAND, 4 * BAND), np.int64)
    img[:, :BAND] = rng.integers(0, maxv + 1, (BAND, BAND))
    img[:, 2 * BAND:3 * BAND] = maxv
    yy, xx = np.mgrid[0:BAND, 0:BAND]
    img[:, 3 * BAND:] = maxv * (((yy >> ydec) + (xx >> xdec)) & 1)    # 0 / max per chroma position
    return img.astype(pxdt(bd))


def cfl_blocks(rng, per_kind):
    """Luma block positions, per_kind in each band, 8-aligned so the checkerboard follows the chroma grid."""
    xs, ys = [], []
    for kind in range(4):
        for _ in range(per_kind):
            xs.append(kind * BAND + 8 * int(rng.integers(0, (BAND - 64) // 8 + 1)))
            ys.append(8 * int(rng.integers(0, (BAND - 64) // 8 + 1)))
    b = np.zeros(len(xs), B.BLOCK_DTYPE)
    b["x"], b["y"] = xs, ys
    return b


def spec_cfl_ac(luma, bw, bh, w_pad, h_pad, xdec, ydec):
    """7.11.5: L = (sum of the co-located luma samples) << (3 - subX - subY), the position clamped to the last
    one inside MaxLumaW x MaxLumaH; ac = L - Round2(sum of L, log2 w + log2 h).  Returns (ac, L)."""
    max_w = max((bw - 4 * w_pad) << xdec, 8)
    max_h = max((bh - 4 * h_pad) << ydec, 8)
    ly = np.minimum(np.arange(bh) << ydec, max_h - (1 << ydec))
    lx = np.minimum(np.arange(bw) << xdec, max_w - (1 << xdec))
    lum = luma.astype(np.int64)
    L = sum(lum[ly[:, None] + dy, lx[None, :] + dx] for dy in range(1 << ydec) for dx in range(1 << xdec))
    L = L << (3 - xdec - ydec)
    shift = (bw.bit_length() - 1) + (bh.bit_length() - 1)
    return L - ((int(L.sum()) + (1 << (shift - 1))) >> shift), L


def run_cfl_ac(pl, blocks, bw, bh, w_pad, h_pad, xdec, ydec):
    n = len(blocks)
    d = dev_out(n * bw * bh * 2)
    G.ctx().pred_cfl_ac_dev(pl, G.to_dev(blocks), n, bw, bh, w_pad, h_pad, xdec, ydec, d)
    G.ctx().synchronize()
    return host_out(d, n * bw * bh * 2, np.int16, (n, bh * bw))


def cfl_edges(rng, bd):
    """Random, all-zero and all-maximum edges: the last two push the prediction past 0 and the maximum."""
    maxv = (1 << bd) - 1
    return np.array([rng.integers(0, maxv + 1, O.EDGE_LEN), np.zeros(O.EDGE_LEN), np.full(O.EDGE_LEN, maxv)]
                    ).astype(pxdt(bd))


def spec_cfl_pred(edges, items, ac, w, h, bd):
    """DC (spec_nondirectional) + Round2Signed(alpha * ac, 6), clipped; also returns the unclipped values."""
    dc = {}
    for e in range(len(edges)):
        for v in range(4):
            dc[e, v] = int(spec_nondirectional("DC_PRED", v, edges[e][129:129 + w], edges[e][127::-1][:h],
                                               int(edges[e][128]), w, h, bd)[0, 0])
    base = np.array([dc[int(it["edge"]), int(it["variant"])] for it in items], np.int64)
    q6 = items["angle"].astype(np.int64)[:, None] * ac[items["ac"].astype(np.int64)].astype(np.int64)
    raw = base[:, None] + np.sign(q6) * ((np.abs(q6) + 32) >> 6)
    return np.clip(raw, 0, (1 << bd) - 1).reshape(len(items), h, w), raw


def cfl_items(rng, nac, nedges, bw, bh, count):
    """Every (variant, alpha) on every edge, then random ones; one random ac block each."""
    rows = [(e, int(rng.integers(nac)), v, a) for e in range(nedges) for v in range(4) for a in CFL_ALPHAS]
    rows += [(int(rng.integers(nedges)), int(rng.integers(nac)), int(rng.integers(4)), int(rng.choice(CFL_ALPHAS)))
             for _ in range(max(0, count - len(rows)))]
    return make_intra_items([(e, a, 64, 64, alpha, M["UV_CFL_PRED"], v, -1, bh, bw) for e, a, v, alpha in rows])


@pytest.mark.parametrize("bd", BDS)
def test_cfl_every_bit_depth(bd):
    """cfl_ac_kernel at every block size 4..32 x 4..32, every legal (w_pad, h_pad) and every layout, on random,
    zero, maximum and checkerboard luma, against the oracle and the specification; then CfL predictions at
    alphas -16, -1, 0, 1, 16 with all four DC variants.  One ac launch and two prediction launches (one of them
    with every alpha 0 and no ac buffer) exceed their grid caps."""
    c = G.ctx()
    rng = np.random.default_rng(400 + bd)
    maxv = (1 << bd) - 1
    edges = cfl_edges(rng, bd)
    d_edges = G.to_dev(edges)
    max_l = max_ac = 0
    under = over = False
    for xdec, ydec in LAYOUTS:
        luma = cfl_luma(rng, bd, xdec, ydec)
        pl = c.plane_from_host(luma, 0)
        blocks = cfl_blocks(rng, 2)
        for bw in CFL_SIDES:
            for bh in CFL_SIDES:
                lw, lh = bw << xdec, bh << ydec
                acs = []
                for w_pad in range(bw // 4):
                    for h_pad in range(bh // 4):
                        got = run_cfl_ac(pl, blocks, bw, bh, w_pad, h_pad, xdec, ydec)
                        for i, b in enumerate(blocks):
                            sub = np.ascontiguousarray(luma[b["y"]:b["y"] + lh, b["x"]:b["x"] + lw])
                            want = O.pred_cfl_ac(sub, bw, bh, w_pad, h_pad, xdec, ydec)
                            spec, L = spec_cfl_ac(sub, bw, bh, w_pad, h_pad, xdec, ydec)
                            what = f"ac {bw}x{bh} pad ({w_pad},{h_pad}) dec ({xdec},{ydec}) block {i}"
                            np.testing.assert_array_equal(got[i], want, err_msg=what)
                            np.testing.assert_array_equal(got[i], spec.reshape(-1), err_msg=what + " (spec)")
                            max_l = max(max_l, int(L.max()))
                        max_ac = max(max_ac, int(np.abs(got).max()))
                        acs.append(got)
                ac = np.concatenate(acs)
                items = cfl_items(rng, len(ac), len(edges), bw, bh, 2 * len(ac))
                got = predict(d_edges, items, bw, bh, bd, G.to_dev(ac))
                check(got, oracle_batch(edges, items, bw, bh, bd, ac), items, bw, bh, f"CfL {bw}x{bh}")
                spec, raw = spec_cfl_pred(edges, items, ac, bw, bh, bd)
                check(got, spec, items, bw, bh, f"CfL {bw}x{bh} (spec)")
                under, over = under or bool((raw < 0).any()), over or bool((raw > maxv).any())
        c.plane_free(pl)
    assert max_l == maxv << 3 and max_ac >= maxv << 2
    assert under and over
    # the grid-stride loops: one capped pass plus a ragged second trip of each kernel
    xdec, ydec, bw, bh, w_pad, h_pad = 1, 0, 16, 8, 1, 0
    luma = cfl_luma(rng, bd, xdec, ydec)
    pl = c.plane_from_host(luma, 0)
    ublocks = cfl_blocks(rng, 16)
    uwant = np.array([O.pred_cfl_ac(np.ascontiguousarray(luma[b["y"]:b["y"] + bh, b["x"]:b["x"] + 2 * bw]),
                                    bw, bh, w_pad, h_pad, xdec, ydec) for b in ublocks])
    n = second_trip(num_sms() * CFL_CTAS_PER_SM)
    idx = rng.integers(0, len(ublocks), n)
    got = {}
    assert G.profiled_kernels(lambda: got.setdefault("v", run_cfl_ac(pl, ublocks[idx], bw, bh, w_pad, h_pad, xdec,
                                                                      ydec)), prefix="cfl_") == \
        [f"cfl_ac_kernel<{tname(bd)}>"]
    np.testing.assert_array_equal(got["v"], uwant[idx], err_msg="ac, second trip")
    c.plane_free(pl)
    ac = got["v"]
    n = second_trip(num_sms() * IPRED_CTAS_PER_SM)
    items = cfl_items(rng, len(ac), len(edges), bw, bh, n)
    items = items[rng.permutation(len(items))]
    check(predict(d_edges, items, bw, bh, bd, G.to_dev(ac)), oracle_batch(edges, items, bw, bh, bd, ac), items,
          bw, bh, "CfL, second trip")
    items["angle"] = 0                                     # pred_cfl_inner returns before reading ac
    check(predict(d_edges, items, bw, bh, bd, None), oracle_batch(edges, items, bw, bh, bd, None), items, bw, bh,
          "CfL, alpha 0 without an ac buffer")


# ---------------------------------------------------------------- 5. per-call form
@pytest.mark.parametrize("bd", [10, 12])
def test_percall_form(bd):
    """b200_predict_intra (host pointers, byte stride) for every non-directional mode, a filtered and an
    unfiltered sample of the directional angles (some at the plane border) and CfL at alphas -16 / 5 / 16, into
    a destination wider than the block: the bytes between rows stay untouched."""
    L = B.lib()
    rng = np.random.default_rng(500 + bd)
    maxv = (1 << bd) - 1
    sent = np.frombuffer(bytes([SENTINEL] * 2), np.uint16)[0]
    PW, PH = 512, 384
    ran = set()
    for w, h in ((4, 4), (8, 16), (16, 4), (32, 32), (64, 16), (4, 16), (64, 64)):
        e = rng.integers(0, maxv + 1, O.EDGE_LEN).astype(np.uint16)
        cases = [(M[m], v, ANGLE_OF.get(M[m], 0), -1, None) for m, v in NONDIR]
        for m in DIRECTIONAL:
            for ief in (-1, 0, 1):
                cases.append((M[m], 3, ANGLE_OF[M[m]] + 3 * int(rng.choice([-3, -2, -1, 1, 2, 3])), ief, None))
        ac = rng.integers(-(maxv << 3), (maxv << 3) + 1, w * h).astype(np.int16)
        cases += [(M["UV_CFL_PRED"], v, alpha, -1, ac) for v, alpha in ((3, -16), (1, 5), (2, 16), (0, 16))]
        for k, (mode, variant, angle, ief, a) in enumerate(cases):
            x, y = (PW - w // 2, PH - h // 2) if k % 2 else (64, 32)
            ll, al = encoder_lens(w, h, mode, angle)
            dst = np.full((h, w + 5), sent, np.uint16)
            L.b200_predict_intra(mode, variant, dst.ctypes.data, dst.strides[0], w, h, bd,
                                 None if a is None else a.ctypes.data, angle, ief, e.ctypes.data, ll, al, PW, PH, x, y)
            want = O.predict_intra(mode, variant, e, w, h, bd, angle=angle, ief=ief, ac=a, left_len=ll, above_len=al,
                                   plane_w=PW, plane_h=PH, dst_x=x, dst_y=y)
            what = f"{w}x{h} {O.MODES[mode]} variant {variant} angle {angle} ief {ief} at ({x}, {y})"
            np.testing.assert_array_equal(dst[:, :w], want, err_msg=what)
            assert (dst[:, w:] == sent).all(), what + ": wrote between rows"
            ran.add("cfl" if a is not None else "filtered" if ief >= 0 and is_directional(mode, angle) else mode)
    assert {"cfl", "filtered"} <= ran and len(ran) >= 10


# ---------------------------------------------------------------- 6. host side
def test_empty_and_rejected_launches_do_nothing():
    """n = 0 launches nothing and writes nothing; a w or h that is not a TxSize side, a bad bit depth, a CfL
    block outside 4..32 or not a power of two, and ydec without xdec are rejected with ERR_ARG before any
    launch."""
    c = G.ctx()
    edges = G.to_dev(np.zeros((1, O.EDGE_LEN), np.uint16))
    items = G.to_dev(make_intra_items([(0, 0, 64, 64, 0, M["DC_PRED"], 3, -1, 8, 8)]))
    out = dev_out(64 * 64 * 2)

    def unchanged(fn):
        n0 = c.launches
        fn()
        c.synchronize()
        assert c.launches == n0
        assert (out.cpu().numpy() == SENTINEL).all()

    def rejected(fn):
        n0 = c.launches
        with pytest.raises(B.B200Error) as e:
            fn()
        assert e.value.status == B.ERR_ARG
        c.synchronize()
        assert c.launches == n0
        assert (out.cpu().numpy() == SENTINEL).all()

    unchanged(lambda: c.predict_intra_dev(edges, items, 0, None, 8, 8, 10, 4096, 4096, out))
    for w, h, bd in ((0, 8, 10), (2, 8, 10), (8, 12, 10), (128, 8, 10), (8, 128, 10), (8, 6, 10), (8, 8, 9),
                     (8, 8, 7), (8, 8, 16), (8, 8, 0)):
        rejected(lambda: c.predict_intra_dev(edges, items, 1, None, w, h, bd, 4096, 4096, out))
    luma = c.plane_from_host(np.zeros((64, 64), np.uint16), 0)
    blocks = G.to_dev(np.zeros(1, B.BLOCK_DTYPE))
    unchanged(lambda: c.pred_cfl_ac_dev(luma, blocks, 0, 8, 8, 0, 0, 1, 1, out))
    for bw, bh, xdec, ydec in ((2, 8, 1, 1), (8, 2, 1, 1), (64, 8, 0, 0), (8, 64, 0, 0), (12, 8, 1, 1),
                               (8, 24, 1, 1), (0, 8, 1, 1), (8, 8, 0, 1), (8, 8, 2, 0), (8, 8, 1, 2)):
        rejected(lambda: c.pred_cfl_ac_dev(luma, blocks, 1, bw, bh, 0, 0, xdec, ydec, out))
    eitems = G.to_dev(np.zeros(1, B.EDGE_ITEM_DTYPE))
    unchanged(lambda: c.get_intra_edges_dev(luma, (0, 0, 64, 64), 0, 0, 10, eitems, 0, out, out))
    c.plane_free(luma)
