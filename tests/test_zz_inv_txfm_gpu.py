"""GPU parity for the inverse transform + reconstruction: CUDA (through the C ABI) ==
oracle/inv_txfm.c, bit exact, over every valid (TxSize, TxType) pair at 8 and 10 bit with realistic
(quantized) coefficients, plus the device-resident encode_tx_block chain (residual -> forward transform
-> quantize -> dequantize -> inverse transform add) against the same chain of oracle functions, and the
fused encode kernel against the three separate steps at 11 (size, type, bit depth) points.

12 bit, coefficients at the clamps and type limits, every pair of the fused encode kernel against the
oracle and the grid-stride loops are covered by tests/test_tx_paths_gpu.py.
"""
import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_oracle_inv_txfm import inverse_add
from tests.test_oracle_quantize import chain as oracle_chain

pytestmark = pytest.mark.gpu


def download(c, plane, like):
    import ctypes
    out = np.zeros(like.shape, like.dtype)
    c.check(c.L.b200_plane_download(c.h, ctypes.byref(plane), out.ctypes.data, out.strides[0]))
    return out


def coded_dims(ts):
    w, h = O.TX_SIZES[ts]
    return min(w, 32), min(h, 32)


@pytest.mark.parametrize("bd", [8, 10])
def test_every_valid_pair_matches_oracle(bd):
    import torch
    c = G.ctx()
    rng = np.random.default_rng(bd)
    px = np.uint8 if bd == 8 else np.uint16
    ct = np.int16 if bd == 8 else np.int32
    W, H = 256, 192
    for ts, tt in O.valid_txfm_combos():
        w, h = O.TX_SIZES[ts]
        cw, ch = coded_dims(ts)
        blocks = G.grid_blocks(W, H, w, h)[:24]
        n = len(blocks)
        base = rng.integers(0, 1 << bd, (H, W)).astype(px)
        # realistic dequantized coefficients: forward transform of a residual, coarsely quantized
        res = rng.integers(-60, 61, (n, h, w)).astype(np.int16) << (bd - 8)
        coef = O.forward_transform_batch(res, ts, tt, bd, coeff_i32=(bd > 8))
        coef = coef.reshape(n, -1)[:, :cw * ch]
        coef = ((coef // 8) * 8).astype(ct)
        want = base.copy()
        for i, b in enumerate(blocks):
            x, y = int(b["x"]), int(b["y"])
            tile = np.ascontiguousarray(want[y:y + h, x:x + w])
            want[y:y + h, x:x + w] = inverse_add(coef[i], tile, ts, tt, bd)
        dpl = c.plane_from_host(base, 0)
        c.inverse_transform_add_dev(torch.from_numpy(np.ascontiguousarray(coef)).cuda(), dpl, G.to_dev(blocks), n,
                                    ts, tt, bd)
        c.synchronize()
        got = download(c, dpl, base)
        np.testing.assert_array_equal(got, want, err_msg=f"ts={ts} tt={tt} bd={bd}")
        c.plane_free(dpl)


def test_encode_tx_block_chain_on_device():
    """diff + forward transform -> quantize -> dequantize -> inverse transform add into the
    prediction: the reconstructed block must equal the oracle's."""
    import torch
    c = G.ctx()
    W, H, PAD = 256, 128, 96
    cur, ref = G.make_planes(W, H, PAD, np.uint8, seed=31)
    ocur, dcur = G.both_planes(cur, PAD)
    oref, dref = G.both_planes(ref, PAD)
    blocks = G.grid_blocks(W, H, 16, 16)
    n = len(blocks)
    resid = np.zeros((n, 16, 16), np.int16)
    for i, b in enumerate(blocks):
        x, y = int(b["x"]) + PAD, int(b["y"]) + PAD
        resid[i] = ocur.data[y:y + 16, x:x + 16].astype(np.int32) - oref.data[y:y + 16, x:x + 16].astype(np.int32)
    coef = O.forward_transform_batch(resid, 2, 0, 8).reshape(n, 256)
    _, rco, _, _ = oracle_chain(coef, 2, 0, 90, 72, False)
    want = ref.copy()                                   # reconstruction = prediction (zero-mv ref) + inverse
    for i, b in enumerate(blocks):
        x, y = int(b["x"]), int(b["y"])
        want[y:y + 16, x:x + 16] = inverse_add(rco[i], np.ascontiguousarray(want[y:y + 16, x:x + 16]), 2, 0, 8)
    d_blocks = G.to_dev(blocks)
    d_coef = torch.empty((n, 256), dtype=torch.int16, device="cuda")
    d_q = torch.empty((n, 256), dtype=torch.int16, device="cuda")
    d_r = torch.empty((n, 256), dtype=torch.int16, device="cuda")
    c.fwd_txfm_residual_dev(dcur, dref, d_blocks, n, None, d_coef, 2, 0, 8)
    c.quantize_dev(d_coef, n, 2, 0, 90, 72, False, False, d_q, d_r, None, None)
    drec = c.plane_from_host(ref, 0)
    c.inverse_transform_add_dev(d_r, drec, d_blocks, n, 2, 0, 8)
    c.synchronize()
    got = download(c, drec, ref)
    np.testing.assert_array_equal(got, want)
    # the loop is closed: reconstruction error is bounded by the quantizer step
    assert np.abs(got.astype(np.int32) - cur.astype(np.int32)).mean() < 12
    for pl in (dcur, dref, drec):
        c.plane_free(pl)


@pytest.mark.parametrize("ts,tt,bd", [(2, 0, 8), (1, 3, 8), (0, 1, 8), (3, 0, 10), (4, 0, 8), (9, 0, 8), (13, 1, 10),
                                      (5, 9, 8), (16, 9, 12), (11, 0, 10), (8, 10, 8)])
def test_encode_tx_blocks_one_call_equals_the_three_steps(ts, tt, bd):
    """the fused kernel (b200_encode_tx_blocks_dev: coefficients stay on the SM) == b200_fwd_txfm_residual_dev +
    b200_quantize_dev + b200_inverse_transform_add_dev called one after the other, every output, with
    motion-displaced predictions."""
    import torch
    c = G.ctx()
    W, H, PAD = 256, 192, 64
    dtype = np.uint8 if bd == 8 else np.uint16
    cur, ref = G.make_planes(W, H, PAD, dtype, seed=44 + ts, bit_depth=bd)
    _, dcur = G.both_planes(cur, PAD)
    _, dref = G.both_planes(ref, PAD)
    w, h = O.TX_SIZES[ts]
    blocks = G.grid_blocks(W, H, w, h)
    n = len(blocks)
    d_blocks = G.to_dev(blocks)
    rng = np.random.default_rng(ts)
    mv = np.zeros(n, B.ME_RESULT_DTYPE)
    mv["cost"] = 1
    mv["cost"][::7] = np.uint64(2**64 - 1)                  # empty results: zero motion
    mv["mv_row"], mv["mv_col"] = rng.integers(-5, 6, n) * 8, rng.integers(-5, 6, n) * 8
    d_mv = G.to_dev(mv)
    ct = torch.int16 if bd == 8 else torch.int32
    coded = c.L.b200_coded_tx_area(ts)
    mk = lambda k: torch.empty((n, k), dtype=ct, device="cuda")
    co1, q1, r1, co2, q2, r2 = mk(w * h), mk(coded), mk(coded), mk(w * h), mk(coded), mk(coded)
    e1, e2 = (torch.zeros(n, dtype=torch.int16, device="cuda") for _ in range(2))
    d1, d2 = (torch.zeros(n, dtype=torch.int64, device="cuda") for _ in range(2))
    rec1, rec2 = c.plane_from_host(ref, 0), c.plane_from_host(ref, 0)
    dcq, acq = 70 << (bd - 8), 60 << (bd - 8)
    c.fwd_txfm_residual_dev(dcur, dref, d_blocks, n, d_mv, co1, ts, tt, bd)
    c.quantize_dev(co1, n, ts, tt, dcq, acq, False, bd > 8, q1, r1, e1, d1)
    c.inverse_transform_add_dev(r1, rec1, d_blocks, n, ts, tt, bd)
    c.encode_tx_blocks_dev(dcur, dref, rec2, d_blocks, n, d_mv, ts, tt, bd, dcq, acq, False, True, co2, q2, r2, e2, d2)
    c.synchronize()
    for a, b in ((co1, co2), (q1, q2), (r1, r2), (e1, e2), (d1, d2)):
        assert torch.equal(a, b)
    np.testing.assert_array_equal(download(c, rec1, ref), download(c, rec2, ref))
    # optional outputs left out: nothing else changes
    q3 = mk(coded)
    rec3 = c.plane_from_host(ref, 0)
    c.encode_tx_blocks_dev(dcur, dref, rec3, d_blocks, n, d_mv, ts, tt, bd, dcq, acq, False, True, None, q3, None, None, None)
    c.synchronize()
    assert torch.equal(q3, q1)
    np.testing.assert_array_equal(download(c, rec3, ref), download(c, rec1, ref))
    for pl in (dcur, dref, rec1, rec2, rec3):
        c.plane_free(pl)
