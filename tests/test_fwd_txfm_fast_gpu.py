"""The DCT_DCT fast path of the fused residual + forward transform (fwd_dct_fast_kernel, fwd_txfm.cu).

b200_fwd_txfm_residual_dev, _residual_multi_dev and _pred_dev send 8-bit DCT_DCT at every size with both sides
in 8..32 to a kernel of its own when every plane row and the output start on 16-byte boundaries: compile-time
shifts, rows read as aligned 16-byte segments, whole-block coefficient stores, block bookkeeping shared
through shuffles.  Every call is checked against the oracle's diff + forward_transform chain: each accepted
(size, bit depth) at the extreme residuals, NULL and empty winners, vectors to the last readable pixel of
the padding on all four sides, plane pairs whose block ranges cut across a warp's blocks, and the planes,
predictions and outputs off the 16-byte grid and the 10 / 12-bit planes that take fwd_txfm_kernel instead.
Which kernel each case ran is checked under torch.profiler when test_zz_fwd_txfm_routes_gpu.py runs this file
again in a process of its own.
"""
import ctypes
import os

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_tx_paths_gpu import (EMPTY, PAD, W, H, Planes, extreme_tiles, gather, images, motion,
                                     num_sms, positions, pxt, read_blocks, residual, sentinel, tcft)

pytestmark = pytest.mark.gpu

BDS = [8, 10, 12]
FAST_SIZES = [ts for ts, (w, h) in enumerate(O.TX_SIZES) if 8 <= w <= 32 and 8 <= h <= 32]
FAST, GENERIC = "fwd_dct_fast_kernel", "fwd_txfm_kernel"


def expected(bd):
    """The kernel an aligned DCT_DCT call runs at bit depth bd."""
    return FAST if bd == 8 else GENERIC


def fwd(res, ts, bd, tt=0):
    return O.forward_transform_batch(res, ts, tt, bd, coeff_i32=bd > 8)


def routed(fn, want):
    """Run fn, the calls of one case.  With FWD_TXFM_PROFILE_ROUTES=1 (test_zz_fwd_txfm_routes_gpu.py runs this
    file again that way, in a process of its own) also assert under torch.profiler that they ran `want`."""
    if os.environ.get("FWD_TXFM_PROFILE_ROUTES") != "1":
        fn()
        return
    names = G.profiled_kernels(fn, prefix="fwd_")
    assert {k for k in (FAST, GENERIC) if any(n.startswith(k) for n in names)} == {want}, names


def check(got, want, msg):
    np.testing.assert_array_equal(got.cpu().numpy(), want, err_msg=msg)


def view(plane, dx):
    """The same pixels seen from `dx` pixels further right (an unaligned base for odd dx)."""
    v = B.Plane()
    ctypes.memmove(ctypes.byref(v), ctypes.byref(plane), ctypes.sizeof(B.Plane))
    v.data = plane.data + dx * plane.bpp
    v.width = plane.width - dx
    return v


def shifted(blocks, dx):
    b = blocks.copy()
    b["x"] += dx
    return b


@pytest.mark.parametrize("bd", BDS)
@pytest.mark.parametrize("ts", FAST_SIZES)
def test_fast_path_every_size_at_the_extremes(ts, bd):
    """Each size the fast kernel accepts, at 8 bit on the fast kernel and at 10 / 12 bit on the generic one:
    +-max residual tiles, uniform noise elsewhere, sub-pel winners truncated toward zero, every fifth winner
    empty, and a NULL mv_src; single-pair and multi-pair forms and packed predictions."""
    c = G.ctx()
    rng = np.random.default_rng(100 * ts + bd)
    w, h = O.TX_SIZES[ts]
    n = 3 * 32 + 5
    blocks = read_blocks(n, w, h, rng)
    P = Planes(*images(bd, rng, positions(blocks), w, h))
    mv = motion(n, rng)
    d_blocks, d_mv = G.to_dev(blocks), G.to_dev(mv)
    res_mv = residual(P.ocur, P.oref, blocks, mv, w, h)
    assert np.abs(res_mv).max() == (1 << bd) - 1 and res_mv.min() == -((1 << bd) - 1)
    pred = rng.integers(0, 1 << bd, (n, h, w)).astype(pxt(bd))
    for k, (_, p) in enumerate(extreme_tiles(w, h, bd)):
        pred[k] = p
    res_pred = (gather(P.ocur, blocks["x"], blocks["y"], w, h) - pred).astype(np.int16)
    ends = np.array([0, 17, 17, 40, n], np.uint32)
    swapped = (np.searchsorted(ends, np.arange(n), side="right") % 2 == 1)[:, None]
    pairs = B.PlanePairs([P.dref if k % 2 else P.dcur for k in range(len(ends))],
                         [P.dcur if k % 2 else P.dref for k in range(len(ends))], ends, ends)
    want = {"residual": fwd(res_mv, ts, bd), "NULL mv": fwd(residual(P.ocur, P.oref, blocks, None, w, h), ts, bd),
            "pred": fwd(res_pred, ts, bd)}
    want["multi"] = np.where(swapped, fwd(residual(P.oref, P.ocur, blocks, mv, w, h), ts, bd), want["residual"])
    got = {k: sentinel((n, w * h), tcft(bd)) for k in want}
    d_pred = G.to_dev(pred)

    def calls():
        c.fwd_txfm_residual_dev(P.dcur, P.dref, d_blocks, n, d_mv, got["residual"], ts, 0, bd)
        c.fwd_txfm_residual_dev(P.dcur, P.dref, d_blocks, n, None, got["NULL mv"], ts, 0, bd)
        c.fwd_txfm_residual_multi_dev(pairs, d_blocks, n, d_mv, got["multi"], ts, 0, bd)
        c.fwd_txfm_pred_dev(P.dcur, d_pred, d_blocks, n, got["pred"], ts, 0, bd)

    routed(calls, expected(bd))
    for k in want:
        check(got[k], want[k], f"{k} ts={ts} bd={bd}")
    P.free()


@pytest.mark.parametrize("bd", [8, 10])
def test_fast_path_reaches_every_padding_edge(bd):
    """Vectors that put a block's rows and columns on the first and last readable pixel of the padding on
    all four sides, at every byte offset within a 16-byte segment, and one past an empty winner."""
    c = G.ctx()
    rng = np.random.default_rng(7 + bd)
    P = Planes(*images(bd, rng))
    for ts in (1, 2, 3, 15, 16):
        w, h = O.TX_SIZES[ts]
        xs, ys, mvr, mvc, cost = [], [], [], [], []
        for x, dxs in ((0, range(-PAD, -PAD + 17)), (W - w, range(PAD - 16, PAD + 1))):
            for y, dy in ((0, -PAD), (H - h, PAD)):
                for dx in dxs:
                    xs.append(x), ys.append(y), mvr.append(8 * dy), mvc.append(8 * dx), cost.append(1)
        # fractions truncate toward zero: -8 * PAD - 7 still reaches -PAD
        xs += [0, W - w]
        ys += [0, H - h]
        mvr += [-8 * PAD - 7, 8 * PAD + 7]
        mvc += [-8 * PAD - 7, 8 * PAD + 7]
        cost += [3, 3]
        # an empty winner with a vector far outside the padding means zero motion
        xs.append(0), ys.append(0), mvr.append(-8 * (PAD + 64)), mvc.append(-8 * (PAD + 64)), cost.append(EMPTY)
        n = len(xs)
        blocks = np.zeros(n, B.BLOCK_DTYPE)
        blocks["x"], blocks["y"] = xs, ys
        mv = np.zeros(n, B.ME_RESULT_DTYPE)
        mv["mv_row"], mv["mv_col"], mv["cost"] = mvr, mvc, np.array(cost, np.uint64)
        want = fwd(residual(P.ocur, P.oref, blocks, mv, w, h), ts, bd)
        got = sentinel((n, w * h), tcft(bd))
        routed(lambda: c.fwd_txfm_residual_dev(P.dcur, P.dref, G.to_dev(blocks), n, G.to_dev(mv),
                                               got, ts, 0, bd), expected(bd))
        check(got, want, f"ts={ts} bd={bd}")
    P.free()


@pytest.mark.parametrize("ts", [1, 2, 3])
def test_fast_path_pair_ranges_across_warp_groups(ts):
    """Enough blocks that warps make more than one pass of 32 blocks, with pair ranges that end inside a warp's
    blocks and inside one round of a warp, empty pairs, and a total that is not a multiple of any grouping;
    plus the small counts where some warps get one round or none."""
    c = G.ctx()
    bd = 8
    rng = np.random.default_rng(ts)
    w, h = O.TX_SIZES[ts]
    P = Planes(*images(bd, rng))
    # more than 32 blocks per resident warp (at most 32 warps per SM): a second pass
    big = (num_sms() * 32 * 32 + 37,) if w * h <= 256 else ()
    for n in (1, 3, 33, 1000 + 3) + big:
        blocks = read_blocks(max(n, 4), w, h, rng)[:n]
        mv = motion(n, rng)
        cuts = np.sort(rng.integers(1, n, 5)) if n > 1 else np.zeros(0, np.int64)
        ends = np.concatenate([[0], cuts, [n, n]]).astype(np.uint32)
        swapped = (np.searchsorted(ends, np.arange(n), side="right") % 2 == 1)[:, None]
        pairs = B.PlanePairs([P.dref if k % 2 else P.dcur for k in range(len(ends))],
                             [P.dcur if k % 2 else P.dref for k in range(len(ends))], ends, ends)
        want = np.where(swapped, fwd(residual(P.oref, P.ocur, blocks, mv, w, h), ts, bd),
                        fwd(residual(P.ocur, P.oref, blocks, mv, w, h), ts, bd))
        got = sentinel((n + 1, w * h), tcft(bd))
        routed(lambda: c.fwd_txfm_residual_multi_dev(pairs, G.to_dev(blocks), n, G.to_dev(mv), got,
                                                     ts, 0, bd), FAST)
        check(got[:n], want, f"ts={ts} n={n}")
        assert (got[n].cpu().numpy() == -12345).all(), "wrote past the last block"
    P.free()


@pytest.mark.parametrize("bd", [8, 10])
def test_unaligned_planes_and_outputs_take_the_generic_kernel(bd):
    """A plane whose pixel (0,0) is off the 16-byte grid, a plane with an odd pitch, a prediction buffer and
    an output off the grid: each call runs fwd_txfm_kernel and gives the oracle's coefficients, the same
    ones the fast kernel gives on the aligned planes."""
    import torch
    c = G.ctx()
    rng = np.random.default_rng(30 + bd)
    ts = 2
    w, h = O.TX_SIZES[ts]
    cur, ref = images(bd, rng)
    P = Planes(cur, ref)
    n = 2 * 32 + 9
    blocks = read_blocks(n, w, h, rng)
    blocks["x"] = np.minimum(blocks["x"], W - w - 1)
    mv = motion(n, rng)
    d_mv = G.to_dev(mv)
    # 1. the planes seen one pixel to the right: the oracle reads the blocks one pixel to the right
    want1 = fwd(residual(P.ocur, P.oref, shifted(blocks, 1), mv, w, h), ts, bd)
    got1, fast1 = sentinel((n, w * h), tcft(bd)), sentinel((n, w * h), tcft(bd))
    vc, vr = view(P.dcur, 1), view(P.dref, 1)
    routed(lambda: c.fwd_txfm_residual_dev(vc, vr, G.to_dev(blocks), n, d_mv, got1, ts, 0,
                                           bd), GENERIC)
    routed(lambda: c.fwd_txfm_residual_dev(P.dcur, P.dref, G.to_dev(shifted(blocks, 1)), n, d_mv,
                                           fast1, ts, 0, bd), expected(bd))
    check(got1, want1, "unaligned base")
    check(fast1, want1, "aligned base")
    # 2. an odd pitch: a torch buffer holding the padded image rows at pitch width + 2 * PAD + 1
    px = pxt(bd)
    pitch = W + 2 * PAD + 1
    rows = P.oref.data.astype(px)
    host = np.zeros((rows.shape[0], pitch), px)
    host[:, :rows.shape[1]] = rows
    buf = torch.from_numpy(host.view(np.uint8).reshape(-1)).cuda()
    odd = B.Plane()
    ctypes.memmove(ctypes.byref(odd), ctypes.byref(P.dref), ctypes.sizeof(B.Plane))
    bpp = np.dtype(px).itemsize
    odd.data, odd.stride, odd.alloc = buf.data_ptr() + (PAD * pitch + PAD) * bpp, pitch, None
    want2 = fwd(residual(P.ocur, P.oref, blocks, mv, w, h), ts, bd)
    got2 = sentinel((n, w * h), tcft(bd))
    routed(lambda: c.fwd_txfm_residual_dev(P.dcur, odd, G.to_dev(blocks), n, d_mv, got2, ts, 0,
                                           bd), GENERIC)
    check(got2, want2, "odd pitch")
    # 3. an output one coefficient off the grid
    out = sentinel((n * w * h + 1,), tcft(bd))
    routed(lambda: c.fwd_txfm_residual_dev(P.dcur, P.dref, G.to_dev(blocks), n, d_mv, out[1:], ts, 0,
                                           bd), GENERIC)
    np.testing.assert_array_equal(out[1:].cpu().numpy().reshape(n, w * h), want2, err_msg="unaligned output")
    # 4. packed predictions one block-row off the grid
    pred = rng.integers(0, 1 << bd, (n, h, w)).astype(px)
    res_pred = (gather(P.ocur, blocks["x"], blocks["y"], w, h) - pred).astype(np.int16)
    raw = np.zeros(pred.nbytes + 16, np.uint8)
    raw[2:2 + pred.nbytes] = pred.view(np.uint8).reshape(-1)
    d_raw = G.to_dev(raw)
    got4 = sentinel((n, w * h), tcft(bd))
    routed(lambda: c.fwd_txfm_pred_dev(P.dcur, d_raw[2:], G.to_dev(blocks), n, got4, ts, 0,
                                       bd), GENERIC)
    check(got4, fwd(res_pred, ts, bd), "unaligned prediction")
    # 5. the other transform types at the same size stay on the generic kernel
    got5 = sentinel((n, w * h), tcft(bd))
    routed(lambda: c.fwd_txfm_residual_dev(P.dcur, P.dref, G.to_dev(blocks), n, d_mv, got5, ts, 1,
                                           bd), GENERIC)
    check(got5, fwd(residual(P.ocur, P.oref, blocks, mv, w, h), ts, bd, tt=1), "ADST_DCT")
    P.free()
