"""The fused transform kernels on every (size, type, bit depth) they accept, against the CPU oracle composed
step by step: O.forward_transform_batch of cur - prediction, the quantize chain (test_oracle_quantize.chain),
inverse_add (test_oracle_inv_txfm) and put_8tap / subpel_candidates for the sub-pel leg.  Every comparison
is bit exact.

The plain forward kernel is pinned elsewhere (test_txfm_gpu.py).  Each fused kernel carries its own copy of
the residual load, the FLIPADST row / column flips and the coefficient store, so each is swept here:
- inputs mix uniform full-range pixels with extreme blocks (cur = max over a prediction of 0 and the
  reverse, a +-max checkerboard, an asymmetric ramp that a missing flip cannot cancel);
- motion vectors carry negative sub-pel fractions (the full-pel part is mv / 8, truncated toward zero),
  empty ME results (cost == u64::MAX: zero motion) and a NULL d_mv_src;
- block counts are not multiples of the blocks a CTA carries, plus n = 1 and n = 0 (nothing written);
- the last section gives every kernel more blocks than its capped grid covers in one pass, so the
  grid-stride loop makes a second, ragged trip."""
import ctypes

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests import oracle_lib as O
from tests.test_oracle_inv_txfm import inverse_add
from tests.test_oracle_quantize import chain

pytestmark = pytest.mark.gpu

EMPTY = np.uint64(2**64 - 1)
BDS = [8, 10, 12]
W, H, PAD = 256, 192, 32     # planes of the per-pair sweeps
R = 12                       # full-pel motion stays below R px, inside PAD with the 8-tap footprint

# Launch geometry mirrored from the sources: blocks per CTA = TX_THREADS / max(w, h), grids capped at
# num_sms * CTAS_PER_SM CTAs, then a grid-stride loop over the rest.
TX_THREADS = 128          # kTxThreads (fwd_txfm.cu:44), kInvThreads (inv_txfm_dev.cuh:109), kEncThreads (encode_tx.cu:45)
FWD_CTAS_PER_SM = 32      # fwd_txfm.cu:136   min(ctas, num_sms * 32)
INV_CTAS_PER_SM = 32      # inv_txfm.cu:50    min(ctas, num_sms * 32)
ENC_CTAS_PER_SM = 16      # encode_tx.cu:155  min(ctas, num_sms * 16)
SRDO_CTAS_PER_SM = 16     # subpel_rdo.cu:257 min(ctas, num_sms * 16)
SRDO_WARPS_8X8_U8 = 8     # subpel_rdo.cu:247 wpc = min(8, 160 KiB / bytes per warp): 8 for 8x8 u8 blocks


def pxt(bd):
    return np.uint8 if bd == 8 else np.uint16


def cft(bd):
    return np.int16 if bd == 8 else np.int32


def tcft(bd):
    import torch
    return torch.int16 if bd == 8 else torch.int32


def per_cta(w, h):
    return TX_THREADS // max(w, h)


def ragged(w, h):
    """Two and a half CTAs' worth of blocks plus one: never a multiple of the blocks per CTA."""
    p = per_cta(w, h)
    return 2 * p + p // 2 + 1


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def past_one_stride(ctas_per_sm, blocks_per_cta):
    """A block count whose grid-stride loop makes a second trip that ends ragged."""
    stride = num_sms() * ctas_per_sm * blocks_per_cta
    return stride + stride // 2 + 7


def combos_by_size(max_type=16):
    out = {}
    for ts, tt in O.valid_txfm_combos():
        if tt <= max_type:
            out.setdefault(ts, []).append(tt)
    return out


def extreme_tiles(w, h, bd):
    """(cur, prediction) tiles: max over 0, 0 over max, a +-max checkerboard, an asymmetric ramp over 0."""
    m = (1 << bd) - 1
    i, j = np.mgrid[0:h, 0:w]
    chk = ((i + j) & 1) * m
    ramp = (i * w + j) * m // (w * h - 1)
    z = np.zeros((h, w), np.int64)
    return [(z + m, z), (z, z + m), (chk, m - chk), (ramp, z)]


def images(bd, rng, paint=(), w=0, h=0, width=W, height=H):
    """Uniform full-range cur and ref; the extreme tiles painted at `paint` (cur and ref at the same place)."""
    cur = rng.integers(0, 1 << bd, (height, width)).astype(pxt(bd))
    ref = rng.integers(0, 1 << bd, (height, width)).astype(pxt(bd))
    for (x, y), (c, r) in zip(paint, extreme_tiles(w, h, bd)):
        cur[y:y + h, x:x + w] = c
        ref[y:y + h, x:x + w] = r
    return cur, ref


class Planes:
    """cur / ref as padded oracle planes and as device planes."""

    def __init__(self, cur, ref, pad=PAD):
        self.ocur, self.dcur = G.both_planes(cur, pad)
        self.oref, self.dref = G.both_planes(ref, pad)

    def free(self):
        G.ctx().plane_free(self.dcur)
        G.ctx().plane_free(self.dref)


def download(plane, like):
    c = G.ctx()
    out = np.zeros(like.shape, like.dtype)
    c.check(c.L.b200_plane_download(c.h, ctypes.byref(plane), out.ctypes.data, out.strides[0]))
    return out


def trunc8(v):
    v = np.asarray(v, np.int64)
    return np.where(v < 0, -((-v) // 8), v // 8)


def gather(op, x, y, w, h):
    rows = (np.asarray(y, np.int64) + op.pad)[:, None, None] + np.arange(h)[None, :, None]
    cols = (np.asarray(x, np.int64) + op.pad)[:, None, None] + np.arange(w)[None, None, :]
    return op.data[rows, cols].astype(np.int32)


def residual(ocur, oref, blocks, mv, w, h):
    """cur - ref displaced by the full-pel part of each result (None or an empty result: zero motion)."""
    x, y = blocks["x"].astype(np.int64), blocks["y"].astype(np.int64)
    dx = dy = 0
    if mv is not None:
        live = mv["cost"] != EMPTY
        dx, dy = np.where(live, trunc8(mv["mv_col"]), 0), np.where(live, trunc8(mv["mv_row"]), 0)
    return (gather(ocur, x, y, w, h) - gather(oref, x + dx, y + dy, w, h)).astype(np.int16)


def motion(n, rng):
    """ME results with sub-pel vectors (fractions -9, -7, -1, 1, 7, 9), every fifth one empty.  The first
    four belong to the extreme blocks and all mean zero motion: empty with a far vector, or a vector whose
    full-pel part truncates to 0 (-7, -1) where a floor would give -1."""
    mv = np.zeros(n, B.ME_RESULT_DTYPE)
    frac = np.array([-9, -7, -1, 0, 1, 7, 9])
    mv["mv_row"] = rng.integers(-(R - 2), R - 1, n) * 8 + rng.choice(frac, n)
    mv["mv_col"] = rng.integers(-(R - 2), R - 1, n) * 8 + rng.choice(frac, n)
    mv["cost"] = rng.integers(0, 1 << 40, n)
    mv["cost"][::5] = EMPTY
    head = [(EMPTY, 8 * (R - 2), -8 * (R - 2)), (5, -7, -1), (EMPTY, -9, 9), (5, -1, -7)]
    for k, (cost, r, c) in enumerate(head[:n]):
        mv["cost"][k], mv["mv_row"][k], mv["mv_col"][k] = cost, r, c
    return mv


def write_blocks(w, h, width=W, height=H):
    """Non-overlapping blocks, 4-px aligned but not size-aligned: a grid of pitch (w + 4, h + 4) from (4, 4)."""
    xs, ys = np.arange(4, width - w + 1, w + 4), np.arange(4, height - h + 1, h + 4)
    b = np.zeros(len(xs) * len(ys), B.BLOCK_DTYPE)
    b["x"], b["y"] = np.tile(xs, len(ys)), np.repeat(ys, len(xs))
    return b


def read_blocks(n, w, h, rng):
    """Random 4-px aligned positions that may overlap; the first four are disjoint (the extreme blocks)."""
    b = np.zeros(n, B.BLOCK_DTYPE)
    b["x"] = 4 * rng.integers(0, (W - w) // 4 + 1, n)
    b["y"] = 4 * rng.integers(0, (H - h) // 4 + 1, n)
    b[:4] = write_blocks(w, h)[:4]
    return b


def positions(blocks, k=4):
    return [(int(b["x"]), int(b["y"])) for b in blocks[:k]]


def reconstruct(img, blocks, rco, ts, tt, bd):
    w, h = O.TX_SIZES[ts]
    out = img.copy()
    for i, b in enumerate(blocks):
        x, y = int(b["x"]), int(b["y"])
        out[y:y + h, x:x + w] = inverse_add(rco[i], np.ascontiguousarray(out[y:y + h, x:x + w]), ts, tt, bd)
    return out


def sentinel(shape, dtype, value=-12345):
    import torch
    return torch.full(shape, value, dtype=dtype, device="cuda")


# ------------------------------------------------------------------------------------------ 1. fused residual
@pytest.mark.parametrize("bd", BDS)
def test_fused_residual_transforms_every_pair(bd):
    """b200_fwd_txfm_residual_dev, _residual_multi_dev and _pred_dev (fwd_txfm_kernel<..., PLANES=true>,
    fwd_txfm.cu:59-126, and the pair split at :275-294) on all 160 valid pairs.  Until now they ran only
    at 16x16 DCT_DCT / ADST_DCT, at 8 and 10 bit, and never with a FLIPADST type: a lost ud / lr flip, a
    wrong pair lookup or a floored mv / 8 in this copy of the residual load passed the suite."""
    c = G.ctx()
    rng = np.random.default_rng(10 + bd)
    i32 = bd > 8
    npairs = 35                                           # two launches: the host splits every 32 pairs
    for ts, types in combos_by_size().items():
        w, h = O.TX_SIZES[ts]
        n = ragged(w, h)
        blocks = read_blocks(n, w, h, rng)
        P = Planes(*images(bd, rng, positions(blocks), w, h))
        mv = motion(n, rng)
        d_blocks, d_mv = G.to_dev(blocks), G.to_dev(mv)
        res_mv = residual(P.ocur, P.oref, blocks, mv, w, h)
        res_0 = residual(P.ocur, P.oref, blocks, None, w, h)
        res_sw = residual(P.oref, P.ocur, blocks, mv, w, h)
        # _multi: pair k is (cur, ref) for even k and (ref, cur) for odd k; the first pair and any
        # repeated end are empty, the last three pairs (second launch) hold blocks
        ends = np.concatenate([[0], np.sort(rng.integers(1, n, npairs - 2)), [n]]).astype(np.uint32)
        swapped = (np.searchsorted(ends, np.arange(n), side="right") % 2 == 1)[:, None]
        pairs = B.PlanePairs([P.dref if k % 2 else P.dcur for k in range(npairs)],
                             [P.dcur if k % 2 else P.dref for k in range(npairs)], ends, ends)
        # _pred: packed predictions from the MC kernel at the same sub-pel vectors; the extreme blocks
        # get their extreme predictions instead
        mvs = np.ascontiguousarray(np.stack([mv["mv_row"], mv["mv_col"]], 1).astype(np.int16))
        d_pred = G.dev_empty(n * w * h * (1 if bd == 8 else 2))
        c.mc_blocks_dev(P.dref, d_blocks, G.to_dev(mvs), n, w, h, 0, 0, bd, 0, 0, 0, d_pred)
        c.synchronize()
        pred = G.from_dev(d_pred, pxt(bd))[:n * w * h].reshape(n, h, w).copy()
        for k, (_, p) in enumerate(extreme_tiles(w, h, bd)):
            pred[k] = p
        d_pred = G.to_dev(pred)
        res_pred = (gather(P.ocur, blocks["x"], blocks["y"], w, h) - pred).astype(np.int16)
        for tt in types:
            fwd = lambda r: O.forward_transform_batch(r, ts, tt, bd, coeff_i32=i32)
            want_mv = fwd(res_mv)
            want = {"residual": want_mv, "residual NULL mv": fwd(res_0),
                    "multi": np.where(swapped, fwd(res_sw), want_mv), "pred": fwd(res_pred)}
            got = {k: sentinel((n, w * h), tcft(bd)) for k in want}
            c.fwd_txfm_residual_dev(P.dcur, P.dref, d_blocks, n, d_mv, got["residual"], ts, tt, bd)
            c.fwd_txfm_residual_dev(P.dcur, P.dref, d_blocks, n, None, got["residual NULL mv"], ts, tt, bd)
            c.fwd_txfm_residual_multi_dev(pairs, d_blocks, n, d_mv, got["multi"], ts, tt, bd)
            c.fwd_txfm_pred_dev(P.dcur, d_pred, d_blocks, n, got["pred"], ts, tt, bd)
            c.synchronize()
            for k in want:
                np.testing.assert_array_equal(got[k].cpu().numpy(), want[k], err_msg=f"{k} ts={ts} tt={tt} bd={bd}")
        # n = 1 writes block 0 only; n = 0 writes nothing
        tt = types[-1]
        want0 = O.forward_transform_batch(res_mv[:1], ts, tt, bd, coeff_i32=i32)[0]
        for nb in (1, 0):
            outs = [sentinel((n, w * h), tcft(bd)) for _ in range(3)]
            c.fwd_txfm_residual_dev(P.dcur, P.dref, d_blocks, nb, d_mv, outs[0], ts, tt, bd)
            e = np.full(npairs, nb, np.uint32)
            c.fwd_txfm_residual_multi_dev(B.PlanePairs([P.dcur] * npairs, [P.dref] * npairs, e, e), d_blocks, nb,
                                          d_mv, outs[1], ts, tt, bd)
            c.fwd_txfm_pred_dev(P.dcur, d_pred, d_blocks, nb, outs[2], ts, tt, bd)
            c.synchronize()
            for k, o in enumerate(outs):
                o = o.cpu().numpy()
                assert (o[nb:] == -12345).all(), (nb, k, ts)
                if nb:
                    want_first = want0 if k < 2 else O.forward_transform_batch(res_pred[:1], ts, tt, bd, coeff_i32=i32)[0]
                    np.testing.assert_array_equal(o[0], want_first, err_msg=f"n=1 call {k} ts={ts}")
        P.free()


# ------------------------------------------------------------------------------------------ 2. encode_tx
def quantizers(bd):
    s = bd - 8
    return [(1, 1), (52 << s, 44 << s), (1336 << s, 1000 << s), (65535, 65535)]


@pytest.mark.parametrize("bd", BDS)
def test_encode_tx_blocks_every_pair(bd):
    """b200_encode_tx_blocks_dev (encode_tx.cu:73-140) == forward transform -> quantize chain ->
    inverse_add, on all 159 pairs with tx_type < 16, inter and intra, over quantizers from (1, 1) to
    (65535, 65535), into a reconstruction plane unlike `ref`.  It used to be compared with the oracle
    only at 16x16 DCT_DCT, and never ran a FLIPADST type, is_intra = 1, need_recon_pixel = 0, a
    sub-pel vector, TX_64X32, TX_16X64 or TX_64X16.  Alternate pairs also run with need_recon_pixel = 0
    (rec must stay byte-identical) or with zero motion (NULL d_mv_src) and every optional output NULL."""
    import torch
    c = G.ctx()
    rng = np.random.default_rng(20 + bd)
    i32 = bd > 8
    qs = quantizers(bd)
    k = 0
    seen_eob0 = 0
    for ts, types in combos_by_size(15).items():
        w, h = O.TX_SIZES[ts]
        blocks = write_blocks(w, h)[:ragged(w, h)]
        n = len(blocks)
        P = Planes(*images(bd, rng, positions(blocks), w, h))
        rec0 = rng.integers(0, 1 << bd, (H, W)).astype(pxt(bd))
        drec = c.plane_from_host(rec0, 0)
        mv = motion(n, rng)
        d_blocks, d_mv = G.to_dev(blocks), G.to_dev(mv)
        res_mv = residual(P.ocur, P.oref, blocks, mv, w, h)
        res_0 = residual(P.ocur, P.oref, blocks, None, w, h)
        coded = c.L.b200_coded_tx_area(ts)
        for tt in types:
            coef_mv = O.forward_transform_batch(res_mv, ts, tt, bd, coeff_i32=i32)
            for intra in (0, 1):
                dcq, acq = qs[k % len(qs)]
                variant = k % 2
                k += 1
                tag = f"ts={ts} tt={tt} bd={bd} intra={intra} q=({dcq},{acq})"
                q, r, eob, dist = chain(coef_mv, ts, tt, dcq, acq, intra)
                outs = [sentinel((n, w * h), tcft(bd)), sentinel((n, coded), tcft(bd)),
                        sentinel((n, coded), tcft(bd)), sentinel((n,), torch.int16), sentinel((n,), torch.int64)]
                c.plane_upload(drec, rec0)
                c.encode_tx_blocks_dev(P.dcur, P.dref, drec, d_blocks, n, d_mv, ts, tt, bd, dcq, acq, intra, True,
                                       *outs)
                c.synchronize()
                got_rec = download(drec, rec0)

                def check(outs, msg):
                    co, qo, ro, eo, do = (o.cpu().numpy() for o in outs)
                    np.testing.assert_array_equal(co, coef_mv, err_msg="coeffs " + msg)
                    np.testing.assert_array_equal(qo, q, err_msg="qcoeffs " + msg)
                    np.testing.assert_array_equal(ro, r, err_msg="rcoeffs " + msg)
                    np.testing.assert_array_equal(eo.view(np.uint16), eob, err_msg="eob " + msg)
                    np.testing.assert_array_equal(do.view(np.uint64), dist, err_msg="dist " + msg)

                check(outs, tag)
                np.testing.assert_array_equal(got_rec, reconstruct(rec0, blocks, r, ts, tt, bd), err_msg="rec " + tag)
                for i in np.nonzero(eob == 0)[0]:               # eob 0: the reconstruction is what rec held
                    x, y = int(blocks[i]["x"]), int(blocks[i]["y"])
                    assert (got_rec[y:y + h, x:x + w] == rec0[y:y + h, x:x + w]).all(), tag
                    seen_eob0 += 1
                if variant == 0:                                # need_recon_pixel = 0: rec untouched
                    outs = [sentinel(tuple(o.shape), o.dtype) for o in outs]
                    c.plane_upload(drec, rec0)
                    c.encode_tx_blocks_dev(P.dcur, P.dref, drec, d_blocks, n, d_mv, ts, tt, bd, dcq, acq, intra,
                                           False, *outs)
                    c.synchronize()
                    check(outs, "no recon " + tag)
                    assert (download(drec, rec0) == rec0).all(), "no recon " + tag
                else:                                           # NULL d_mv_src and every optional output NULL
                    q0, r0, _, _ = chain(O.forward_transform_batch(res_0, ts, tt, bd, coeff_i32=i32), ts, tt, dcq,
                                         acq, intra)
                    qo = sentinel((n, coded), tcft(bd))
                    c.plane_upload(drec, rec0)
                    c.encode_tx_blocks_dev(P.dcur, P.dref, drec, d_blocks, n, None, ts, tt, bd, dcq, acq, intra,
                                           True, None, qo, None, None, None)
                    c.synchronize()
                    np.testing.assert_array_equal(qo.cpu().numpy(), q0, err_msg="NULL mv " + tag)
                    np.testing.assert_array_equal(download(drec, rec0), reconstruct(rec0, blocks, r0, ts, tt, bd),
                                                  err_msg="NULL mv rec " + tag)
        # n = 1 writes block 0 only; n = 0 writes nothing
        tt = types[-1]
        q, r, _, _ = chain(O.forward_transform_batch(res_mv[:1], ts, tt, bd, coeff_i32=i32), ts, tt, 52, 44, 0)
        for nb in (1, 0):
            qo = sentinel((n, coded), tcft(bd))
            c.plane_upload(drec, rec0)
            c.encode_tx_blocks_dev(P.dcur, P.dref, drec, d_blocks, nb, d_mv, ts, tt, bd, 52, 44, 0, True, None, qo,
                                   None, None, None)
            c.synchronize()
            qo = qo.cpu().numpy()
            assert (qo[nb:] == -12345).all(), (nb, ts)
            np.testing.assert_array_equal(qo[:nb], q[:nb])
            np.testing.assert_array_equal(download(drec, rec0), reconstruct(rec0, blocks[:nb], r, ts, tt, bd))
        c.plane_free(drec)
        P.free()
    assert seen_eob0 > 0


# ------------------------------------------------------------------------------------------ 3. inverse
def extreme_coeffs(n, m, bd, rng):
    """Per block, cycling: uniform over the whole type (i16) or far past the row clamp (i32), the type's
    top everywhere, its bottom everywhere, values at the row clamp's edges and at 2^(bd+8), a lone DC at
    the type's top, and small realistic values."""
    if bd == 8:
        lo, hi, wide = -32768, 32767, 32768
        edge = [-32768, -32767, 32766, 32767]
    else:
        lo, hi, wide = -(1 << 30), 1 << 30, 1 << (bd + 10)
        r = 1 << (bd + 7)
        edge = [-r - 1, -r, r - 1, r, -(1 << (bd + 8)), 1 << (bd + 8)]
    c = np.zeros((n, m), np.int64)
    for i in range(n):
        kind = i % 6
        if kind == 0:
            c[i] = rng.integers(-wide, wide, m)
        elif kind == 1:
            c[i] = hi
        elif kind == 2:
            c[i] = lo
        elif kind == 3:
            c[i] = rng.choice(edge, m)
        elif kind == 4:
            c[i, 0] = hi
        else:
            c[i] = rng.integers(-64, 65, m) << (bd - 8)
    return np.ascontiguousarray(c.astype(cft(bd)))


def dst_tiles(img, blocks, w, h, bd, rng):
    """Destination areas at 0, at max, at mid-grey and random, so the pixel clamp engages both ways."""
    m = (1 << bd) - 1
    for i, b in enumerate(blocks):
        x, y = int(b["x"]), int(b["y"])
        img[y:y + h, x:x + w] = [0, m, (m + 1) // 2][i % 4] if i % 4 < 3 else rng.integers(0, m + 1, (h, w))


@pytest.mark.parametrize("bd", BDS)
def test_inverse_transform_add_at_the_clamps(bd):
    """b200_inverse_transform_add_dev (inv_txfm.cu:26-43, inv_txfm_dev.cuh:114-166) on all 160 pairs
    (WHT_WHT 4x4 included) at 8, 10 and 12 bit, with coefficients over the whole coefficient type, into
    destinations at 0 and at max.  The device inverse had never run at 12 bit, and its row clamp
    (bd + 8) and column clamp (max(bd + 6, 16)) never engaged on the device: the old coefficients were
    quantized transforms of +-60 residuals."""
    import torch
    c = G.ctx()
    rng = np.random.default_rng(30 + bd)
    WI, HI = 320, 256
    img = rng.integers(0, 1 << bd, (HI, WI)).astype(pxt(bd))
    dpl = c.plane_from_host(img, 0)
    for ts, tt in O.valid_txfm_combos():
        w, h = O.TX_SIZES[ts]
        blocks = write_blocks(w, h, WI, HI)[:ragged(w, h)]
        n = len(blocks)
        coef = extreme_coeffs(n, min(w, 32) * min(h, 32), bd, rng)
        dst = img.copy()
        dst_tiles(dst, blocks, w, h, bd, rng)
        want = reconstruct(dst, blocks, coef, ts, tt, bd)
        c.plane_upload(dpl, dst)
        c.inverse_transform_add_dev(torch.from_numpy(coef).cuda(), dpl, G.to_dev(blocks), n, ts, tt, bd)
        c.synchronize()
        np.testing.assert_array_equal(download(dpl, dst), want, err_msg=f"ts={ts} tt={tt} bd={bd}")
        if tt == 0:                                        # n = 0 writes nothing
            c.inverse_transform_add_dev(torch.from_numpy(coef).cuda(), dpl, G.to_dev(blocks), 0, ts, tt, bd)
            c.synchronize()
            np.testing.assert_array_equal(download(dpl, dst), want)
    c.plane_free(dpl)


# ------------------------------------------------------------------------------------------ 4. sub-pel RDO
def diamond_oracle(ocur, oref, blocks, start, pmv, n, width, height, use_satd, lam, bd):
    L = O.lib()
    L.orc_subpel_diamond_search_blocks.restype = None
    L.orc_subpel_diamond_search_blocks.argtypes = [ctypes.c_void_p, ctypes.c_ssize_t, ctypes.c_void_p,
                                                   ctypes.c_ssize_t] + [ctypes.c_int] * 3 + \
        [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_uint32,
         ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p, ctypes.c_int]
    out = start.copy()
    L.orc_subpel_diamond_search_blocks(ocur.origin_ptr(), ocur.stride, oref.origin_ptr(), oref.stride, ocur.bpp,
                                       2 * ((width + 7) >> 3), 2 * ((height + 7) >> 3), O.ptr(blocks), len(blocks),
                                       n, n, int(use_satd), lam, O.ptr(pmv), 0, 0, bd, O.ptr(out), 0)
    return out


def winners(cands, offs, sad, cost):
    """First minimum per block (me.rs:1360-1365): (results, has-a-winner mask)."""
    nb = len(offs) - 1
    best = np.zeros(nb, B.ME_RESULT_DTYPE)
    best["cost"] = EMPTY
    have = np.zeros(nb, bool)
    for b in range(nb):
        lo, hi = int(offs[b]), int(offs[b + 1])
        if lo == hi or cost[lo:hi].min() == EMPTY:
            continue
        k = lo + int(np.argmin(cost[lo:hi]))
        best[b] = (cost[k], sad[k], cands[k]["mv_row"], cands[k]["mv_col"])
        have[b] = True
    return best, have


def winner_residual(ocur, oref, blocks, best, have, n, bd):
    mvs = np.ascontiguousarray(np.stack([best["mv_row"], best["mv_col"]], 1).astype(np.int16))
    pred = O.mc_blocks(oref, blocks, mvs, n, n, 0, 0, bd)
    res = gather(ocur, blocks["x"], blocks["y"], n, n) - pred.astype(np.int32)
    res[~have] = 0
    return res.astype(np.int16)


@pytest.mark.parametrize("n,bd", [(n, bd) for n in (8, 16, 32) for bd in BDS])
def test_subpel_transform_leg_every_type(n, bd):
    """b200_subpel_rdo_dev and b200_subpel_search_dev with the transform on (subpel_rdo.cu:204-235) for
    every valid tx_type of the block size (16 at 8x8 and 16x16, {DCT_DCT, IDTX} at 32x32), SAD and SATD:
    the winners and the winners' coefficients.  Only tx types {0, 1, 3, 9} and {0} ran before, at 8 and
    10 bit, so the leg's own flips were never exercised."""
    import torch
    c = G.ctx()
    ts = {8: 1, 16: 2, 32: 3}[n]
    types = [t for t in range(16) if O.valid_txfm(ts, t)]
    assert len(types) == (2 if n == 32 else 16)
    WS, HS, PS = 256, 160, 96
    m = (1 << bd) - 1
    rng = np.random.default_rng(40 + n + bd)
    cur, ref = images(bd, rng, width=WS, height=HS)
    blocks = G.grid_blocks(WS, HS, n, n)
    nb = len(blocks)
    gx, gy = blocks["x"] // n, blocks["y"] // n
    ext = np.nonzero((gx % 3 == 1) & (gy % 3 == 1))[0][:4]
    # extreme blocks: cur = max / 0 / checkerboard / ramp over a flat reference (0 / max / 0 / 0) that
    # covers every 8-tap footprint of their candidates (vectors within 3 px)
    for k, (cc, _), rv in zip(ext, extreme_tiles(n, n, bd), (0, m, 0, 0)):
        x, y = int(blocks[k]["x"]), int(blocks[k]["y"])
        cur[y:y + n, x:x + n] = cc
        ref[max(y - 8, 0):y + n + 8, max(x - 8, 0):x + n + 8] = rv
    ocur, dcur = G.both_planes(cur, PS)
    oref, dref = G.both_planes(ref, PS)
    cands, offs = G.random_cands(nb, 6, 6, seed=50 + n, fullpel=False)
    cands["mv_col"][::17] = 16000                        # outside the mv range: empty
    for k in ext:
        s = slice(int(offs[k]), int(offs[k + 1]))
        cands["mv_row"][s] = cands["mv_row"][s] % 48 - 24
        cands["mv_col"][s] = cands["mv_col"][s] % 48 - 24
    cands["mv_col"][int(offs[-2]):] = 16000              # the last block has no candidate in range: zeros
    pmv = (rng.integers(-16, 17, (nb, 4)) * 2).astype(np.int16)
    lam = 700
    # full-pel starting points for the diamond search (zero motion for the extreme blocks)
    start_c = np.zeros(nb, B.CAND_DTYPE)
    start_c["block"] = np.arange(nb)
    start_c["mv_row"], start_c["mv_col"] = rng.integers(-3, 2, nb) * 8, rng.integers(0, 5, nb) * 8
    start_c["mv_row"][ext] = start_c["mv_col"][ext] = 0
    d_blocks, d_cands, d_offs, d_pmv = G.to_dev(blocks), G.to_dev(cands), G.to_dev(offs), G.to_dev(pmv)
    for use_satd in (False, True):
        p = B.me_params(n, n, WS, HS, lam, use_satd=use_satd, bit_depth=bd)
        want_sad, want_cost = O.subpel_candidates(ocur, oref, blocks, cands, n, n, use_satd, lam, pmv,
                                                  filter_mode=0, bit_depth=bd)
        best, have = winners(cands, offs, want_sad, want_cost)
        assert have[ext].all() and not have[-1]
        res = winner_residual(ocur, oref, blocks, best, have, n, bd)
        ssad, scost = O.fullpel_candidates(ocur, oref, blocks, start_c, n, n, False, lam, pmv)
        start = np.zeros(nb, B.ME_RESULT_DTYPE)
        start["cost"], start["sad"], start["mv_row"], start["mv_col"] = scost, ssad, start_c["mv_row"], start_c["mv_col"]
        want_ds = diamond_oracle(ocur, oref, blocks, start, pmv, n, WS, HS, use_satd, lam, bd)
        res_ds = winner_residual(ocur, oref, blocks, want_ds, np.ones(nb, bool), n, bd)
        d_start = G.to_dev(start)
        for tt in types:
            tag = f"n={n} bd={bd} satd={use_satd} tt={tt}"
            d_sad, d_cost, d_best = G.dev_empty(4 * len(cands)), G.dev_empty(8 * len(cands)), G.dev_empty(16 * nb)
            d_coef = sentinel((nb, n * n), tcft(bd), 77)
            c.subpel_rdo_dev(dcur, dref, d_blocks, nb, d_cands, len(cands), d_offs, p, 0, ts, tt, d_pmv, d_sad,
                             d_cost, d_best, d_coef)
            d_best2 = G.dev_empty(16 * nb)
            d_coef2 = sentinel((nb, n * n), tcft(bd), 77)
            c.subpel_search_dev(dcur, dref, d_blocks, nb, d_start, p, d_best2, 0, ts, tt, d_pmv, d_coef2)
            c.synchronize()
            np.testing.assert_array_equal(G.from_dev(d_sad, np.uint32)[:len(cands)], want_sad, err_msg=tag)
            np.testing.assert_array_equal(G.from_dev(d_cost, np.uint64)[:len(cands)], want_cost, err_msg=tag)
            got = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:nb]
            for f in ("cost", "sad", "mv_row", "mv_col"):
                np.testing.assert_array_equal(got[f][have], best[f][have], err_msg=f"{f} {tag}")
            assert (got["cost"][~have] == EMPTY).all(), tag
            coef = d_coef.cpu().numpy()
            want = O.forward_transform_batch(res, ts, tt, bd, coeff_i32=bd > 8)
            np.testing.assert_array_equal(coef[have], want[have], err_msg="rdo coeffs " + tag)
            assert (coef[~have] == 0).all(), tag
            got2 = G.from_dev(d_best2, B.ME_RESULT_DTYPE)[:nb]
            for f in ("cost", "sad", "mv_row", "mv_col"):
                np.testing.assert_array_equal(got2[f], want_ds[f], err_msg=f"search {f} {tag}")
            np.testing.assert_array_equal(d_coef2.cpu().numpy(), O.forward_transform_batch(res_ds, ts, tt, bd,
                                                                                           coeff_i32=bd > 8),
                                          err_msg="search coeffs " + tag)
        # n = 1 writes block 0 only; n = 0 writes nothing
        tt = types[-1]
        want0 = O.forward_transform_batch(res[:1], ts, tt, bd, coeff_i32=bd > 8)[0]
        for k in (1, 0):
            d_coef = sentinel((nb, n * n), tcft(bd), 77)
            d_coef2 = sentinel((nb, n * n), tcft(bd), 77)
            c.subpel_rdo_dev(dcur, dref, d_blocks, k, d_cands, len(cands), d_offs, p, 0, ts, tt, d_pmv, None, None,
                             None, d_coef)
            c.subpel_search_dev(dcur, dref, d_blocks, k, d_start, p, G.dev_empty(16), 0, ts, tt, d_pmv, d_coef2)
            c.synchronize()
            for o in (d_coef.cpu().numpy(), d_coef2.cpu().numpy()):
                assert (o[k:] == 77).all(), (k, use_satd)
            if k:
                np.testing.assert_array_equal(d_coef.cpu().numpy()[0], want0)
    for pl in (dcur, dref):
        c.plane_free(pl)


# ------------------------------------------------------------------------------------------ 5. grid-stride
def tiled(tiles, idx, rows, per_row):
    """Raster image whose block i (per_row blocks to a row) is tiles[idx[i]]."""
    _, h, w = tiles.shape
    return np.ascontiguousarray(tiles[idx].reshape(rows, per_row, h, w).transpose(0, 2, 1, 3).reshape(rows * h,
                                                                                                      per_row * w))


def raster_blocks(n, per_row, w, h):
    b = np.zeros(n, B.BLOCK_DTYPE)
    i = np.arange(n)
    b["x"], b["y"] = w * (i % per_row), h * (i // per_row)
    return b


def test_grid_stride_forward_transforms():
    """fwd_txfm_kernel's grid-stride loop (fwd_txfm.cu:56, grid capped at :136) on a second, ragged trip,
    in both instantiations: plain (b200_fwd_txfm_dev) and fused (residual with motion, and packed
    predictions).  4x4 FLIPADST_FLIPADST, 8 bit; positions repeat (the kernel only reads).  No test had
    reached a second trip: the largest launch was 1,005 CTAs."""
    import torch
    c = G.ctx()
    rng = np.random.default_rng(50)
    n = past_one_stride(FWD_CTAS_PER_SM, per_cta(4, 4))
    tt = 6
    blocks = np.zeros(n, B.BLOCK_DTYPE)
    blocks["x"], blocks["y"] = 4 * rng.integers(0, 16, n), 4 * rng.integers(0, 12, n)
    blocks[:4] = write_blocks(4, 4, 64, 48)[:4]
    P = Planes(*images(8, rng, positions(blocks), 4, 4, 64, 48))
    mv = motion(n, rng)
    d_blocks = G.to_dev(blocks)
    res = residual(P.ocur, P.oref, blocks, mv, 4, 4)
    want = O.forward_transform_batch(res, 0, tt, 8, coeff_i32=False)
    outs = [sentinel((n, 16), torch.int16) for _ in range(3)]
    c.fwd_txfm_residual_dev(P.dcur, P.dref, d_blocks, n, G.to_dev(mv), outs[0], 0, tt, 8)
    c.fwd_txfm_dev(torch.from_numpy(res).cuda(), 16, 4, outs[1], n, 0, tt, 8, False)
    mvs = np.ascontiguousarray(np.stack([mv["mv_row"], mv["mv_col"]], 1).astype(np.int16))
    d_pred = G.dev_empty(n * 16)
    c.mc_blocks_dev(P.dref, d_blocks, G.to_dev(mvs), n, 4, 4, 0, 0, 8, 0, 0, 0, d_pred)
    c.fwd_txfm_pred_dev(P.dcur, d_pred, d_blocks, n, outs[2], 0, tt, 8)
    c.synchronize()
    pred = G.from_dev(d_pred, np.uint8)[:n * 16].reshape(n, 4, 4)
    want_pred = O.forward_transform_batch((gather(P.ocur, blocks["x"], blocks["y"], 4, 4) - pred).astype(np.int16),
                                          0, tt, 8, coeff_i32=False)
    for name, o, wnt in zip(("residual", "plain", "pred"), outs, (want, want, want_pred)):
        np.testing.assert_array_equal(o.cpu().numpy(), wnt, err_msg=name)
    P.free()


def test_grid_stride_inverse_transform():
    """inv_txfm_add_kernel's grid-stride loop (inv_txfm.cu:35, grid capped at :50) on a second, ragged
    trip: 4x4 FLIPADST_ADST over distinct blocks of a raster plane.  Block i carries coefficient set
    i % 251 over destination tile i % 251, so every block is checked against 251 oracle results."""
    import torch
    c = G.ctx()
    rng = np.random.default_rng(51)
    tt, K, per_row = 8, 251, 384
    n = past_one_stride(INV_CTAS_PER_SM, per_cta(4, 4))
    rows = -(-n // per_row)
    idx = np.arange(rows * per_row) % K
    pool = extreme_coeffs(K, 16, 8, rng)
    dpool = rng.integers(0, 256, (K, 4, 4)).astype(np.uint8)
    dpool[0::4], dpool[1::4] = 0, 255
    done = np.stack([inverse_add(pool[k], dpool[k].copy(), 0, tt, 8) for k in range(K)])
    dst = tiled(dpool, idx, rows, per_row)
    want = tiled(np.concatenate([done, dpool]), np.where(np.arange(rows * per_row) < n, idx, idx + K), rows, per_row)
    dpl = c.plane_from_host(dst, 0)
    c.inverse_transform_add_dev(torch.from_numpy(np.ascontiguousarray(pool[idx[:n]])).cuda(), dpl,
                                G.to_dev(raster_blocks(n, per_row, 4, 4)), n, 0, tt, 8)
    c.synchronize()
    np.testing.assert_array_equal(download(dpl, dst), want)
    c.plane_free(dpl)


def test_grid_stride_encode_tx():
    """encode_tx_kernel's grid-stride loop (encode_tx.cu:73, grid capped at :155) on a second, ragged
    trip: 4x4 FLIPADST_DCT, zero motion, every output.  Block i of the raster plane has cur / ref / rec
    tiles i % 251, so every block is checked against 251 oracle chains."""
    import torch
    c = G.ctx()
    rng = np.random.default_rng(52)
    tt, K, per_row, dcq, acq = 4, 251, 320, 24, 20
    n = past_one_stride(ENC_CTAS_PER_SM, per_cta(4, 4))
    rows = -(-n // per_row)
    idx = np.arange(rows * per_row) % K
    cpool, rpool, recpool = (rng.integers(0, 256, (K, 4, 4)).astype(np.uint8) for _ in range(3))
    for k, (cc, rr) in enumerate(extreme_tiles(4, 4, 8)):
        cpool[k], rpool[k] = cc, rr
    coef = O.forward_transform_batch(cpool.astype(np.int16) - rpool.astype(np.int16), 0, tt, 8, coeff_i32=False)
    q, r, eob, dist = chain(coef, 0, tt, dcq, acq, 0)
    done = np.stack([inverse_add(r[k], recpool[k].copy(), 0, tt, 8) for k in range(K)])
    P = Planes(tiled(cpool, idx, rows, per_row), tiled(rpool, idx, rows, per_row), 8)
    rec = tiled(recpool, idx, rows, per_row)
    drec = c.plane_from_host(rec, 0)
    outs = [sentinel((n, 16), torch.int16), sentinel((n, 16), torch.int16), sentinel((n, 16), torch.int16),
            sentinel((n,), torch.int16), sentinel((n,), torch.int64)]
    c.encode_tx_blocks_dev(P.dcur, P.dref, drec, G.to_dev(raster_blocks(n, per_row, 4, 4)), n, None, 0, tt, 8, dcq,
                           acq, 0, True, *outs)
    c.synchronize()
    co, qo, ro, eo, do = (o.cpu().numpy() for o in outs)
    i = idx[:n]
    np.testing.assert_array_equal(co, coef[i])
    np.testing.assert_array_equal(qo, q[i])
    np.testing.assert_array_equal(ro, r[i])
    np.testing.assert_array_equal(eo.view(np.uint16), eob[i])
    np.testing.assert_array_equal(do.view(np.uint64), dist[i])
    want = tiled(np.concatenate([done, recpool]), np.where(np.arange(rows * per_row) < n, idx, idx + K), rows,
                 per_row)
    np.testing.assert_array_equal(download(drec, rec), want)
    c.plane_free(drec)
    P.free()


def test_grid_stride_subpel_rdo():
    """subpel_rdo_kernel's grid-stride loop (subpel_rdo.cu:117, grid capped at :257) on a second,
    ragged trip: 8x8 blocks at 8 bit (8 warps per CTA), SATD, ADST_FLIPADST, winners and coefficients
    of every block."""
    import torch
    c = G.ctx()
    rng = np.random.default_rng(53)
    tt, per_row, PS, lam = 7, 240, 32, 400
    n = past_one_stride(SRDO_CTAS_PER_SM, SRDO_WARPS_8X8_U8)
    WS, HS = 8 * per_row, 8 * -(-n // per_row)
    cur, ref = images(8, rng, width=WS, height=HS)
    ocur, dcur = G.both_planes(cur, PS)
    oref, dref = G.both_planes(ref, PS)
    blocks = raster_blocks(n, per_row, 8, 8)
    cands, offs = G.random_cands(n, 3, 4, seed=54, fullpel=False)
    pmv = (rng.integers(-16, 17, (n, 4)) * 2).astype(np.int16)
    sad, cost = O.subpel_candidates(ocur, oref, blocks, cands, 8, 8, True, lam, pmv, bit_depth=8)
    best, have = winners(cands, offs, sad, cost)
    res = winner_residual(ocur, oref, blocks, best, have, 8, 8)
    p = B.me_params(8, 8, WS, HS, lam, use_satd=True, bit_depth=8)
    d_best = G.dev_empty(16 * n)
    d_coef = sentinel((n, 64), torch.int16, 77)
    c.subpel_rdo_dev(dcur, dref, G.to_dev(blocks), n, G.to_dev(cands), len(cands), G.to_dev(offs), p, 0, 1, tt,
                     G.to_dev(pmv), None, None, d_best, d_coef)
    c.synchronize()
    got = G.from_dev(d_best, B.ME_RESULT_DTYPE)[:n]
    for f in ("cost", "sad", "mv_row", "mv_col"):
        np.testing.assert_array_equal(got[f], best[f], err_msg=f)
    want = O.forward_transform_batch(res, 1, tt, 8, coeff_i32=False)
    want[~have] = 0
    np.testing.assert_array_equal(d_coef.cpu().numpy(), want)
    for pl in (dcur, dref):
        c.plane_free(pl)
