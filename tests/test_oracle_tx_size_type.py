"""The oracle's intra transform size / type decision (oracle/tx_size_type.c) against an independent Python
restatement: every evaluated candidate re-encoded one transform block at a time through the pinned oracle pieces
(get_intra_edges, predict_intra, forward transform, quantize chain, inverse transform, coefficient chain,
weighted SSE / cdef_dist kernel, rd cost) on a copy of the whole reconstruction plane, as the reference writes
into `rec`; and rdo_tx_size_type's ladder and rules (rdo.rs:725-802, :1701-1823) over those candidates."""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200.backend import COEFF_CHAIN_DTYPE, TX_CUT, TX_EVALUATED, TX_INVALID, TX_NOT_IN_LADDER, TX_NOT_IN_SET
from tests import coeff_rate_cases as K
from tests import oracle_lib as O
from tests import tx_size_type_cases as T

PAD = 64


def _pieces():
    L = T._lib()
    vp, pd, i32, u32, sz = C.c_void_p, C.c_ssize_t, C.c_int, C.c_uint32, C.c_size_t
    L.orc_get_intra_edges.restype = None
    L.orc_get_intra_edges.argtypes = [vp, vp, pd] + [i32] * 22 + [C.POINTER(i32)] * 2
    L.orc_quantize_chain_batch.restype = None
    L.orc_quantize_chain_batch.argtypes = [vp, sz, i32, i32, u32, u32, i32, i32, vp, vp, vp, vp, i32]
    L.orc_inverse_transform_add.restype = None
    L.orc_inverse_transform_add.argtypes = [vp, i32, vp, pd, i32, i32, i32, i32]
    for n in ("orc_weighted_sse_u8", "orc_weighted_sse_u16"):
        getattr(L, n).restype = C.c_uint64
        getattr(L, n).argtypes = [vp, pd, vp, pd, vp, sz, i32, i32]
    for n in ("orc_cdef_dist_kernel_u8", "orc_cdef_dist_kernel_u16"):
        getattr(L, n).restype = u32
        getattr(L, n).argtypes = [vp, pd, vp, pd, i32, i32, i32, vp]
    L.orc_compute_rd_cost.restype = C.c_double
    L.orc_compute_rd_cost.argtypes = [C.c_double, u32, C.c_uint64]
    return L


def scale_mul(scale, d):  # DistortionScale::mul_u64, rdo.rs:613-615
    return (int(scale) * int(d) + (1 << 13)) >> 14


def encode_candidate(P, it, tx, ty):
    """rdo_tx_type_decision's body for one (tx_size, tx_type): write_tx_blocks' luma loop (encoder.rs:2243-2311 ->
    encode_tx_block :1404-1658) into a copy of the padded rec plane, the counter's rate, the distortion, the rd."""
    L = _pieces()
    src, rec, pad, (rx, ry, rw, rh) = P["src"], P["rec"], PAD, P["rect"]
    W, H, bd, dm = P["w"], P["h"], P["bd"], P["dm"]
    work = rec.data.copy()  # the reference writes predictions and reconstructions into rec
    bpp, stride = work.itemsize, work.shape[1]
    is32 = int(bpp == 2)

    def addr(a, x, y):  # region coordinates
        return a.ctypes.data + ((pad + ry + y) * stride + pad + rx + x) * bpp
    bs, x0, y0, mode = int(it["bsize"]), int(it["x"]), int(it["y"]), int(it["mode"])
    bw, bh, tw, th = T.BS_W[bs], T.BS_H[bs], T.TX_W[tx], T.TX_H[tx]
    w_in_b, h_in_b = 2 * ((W + 7) >> 3), 2 * ((H + 7) >> 3)
    coded = min(tw, 32) * min(th, 32)
    qdt = np.int32 if is32 else np.int16
    qs, items, txd = [], [], 0
    for by in range(bh // th):
        for bx in range(bw // tw):
            px, py = x0 + bx * tw, y0 + by * th
            if px >> 2 >= (rw + 3) >> 2 or py >> 2 >= (rh + 3) >> 2:  # tx_bo past the tile's mi extent
                continue
            edge = np.zeros(O.EDGE_LEN, work.dtype)
            il, ia = C.c_int(), C.c_int()
            L.orc_get_intra_edges(edge.ctypes.data, addr(work, 0, 0), stride, bpp, W, H, rx, ry, rw, rh, 0, 0,
                                  x0 >> 2, y0 >> 2, bx, by, bs, px, py, tw, th, bd, mode, int(it["ief"] >= 0), 0,
                                  C.byref(il), C.byref(ia))
            variant = 0 if (px, py) == (0, 0) else 1 if py == 0 else 2 if px == 0 else 3  # PredictionVariant::new
            m = mode if mode != 12 else [0, 2, 1, 12][variant]  # PAETH at the tile's edges (predict.rs:231-239)
            angle = O.MODE_ANGLE.get(O.MODES[m], 0)
            ief = int(it["ief"]) if 1 <= mode <= 8 else -1
            pred = O.predict_intra(m, variant, edge, tw, th, bd, angle, ief, left_len=il.value, above_len=ia.value,
                                   plane_w=W, plane_h=H, dst_x=rx + px, dst_y=ry + py)
            r0, c0 = pad + ry + py, pad + rx + px
            work[r0:r0 + th, c0:c0 + tw] = pred
            fx, fy = rx + px, ry + py
            visible = fx < W and fy < H  # clip_visible_bsize of the tx block
            s_blk = src.data[r0:r0 + th, c0:c0 + tw].astype(np.int32)
            resid = np.ascontiguousarray((s_blk - pred.astype(np.int32)) if visible else np.zeros((th, tw)),
                                         np.int16)
            coeffs = np.zeros(tw * th, qdt)
            O.lib().orc_forward_transform(resid.ctypes.data, coeffs.ctypes.data, tw, tx, ty, bd, is32)
            q, r = np.zeros(coded, qdt), np.zeros(coded, qdt)
            eob, raw = np.zeros(1, np.uint16), np.zeros(1, np.uint64)
            L.orc_quantize_chain_batch(coeffs.ctypes.data, 1, tx, ty, int(it["dc_quant"]), int(it["ac_quant"]), 1,
                                       is32, q.ctypes.data, r.ctypes.data, eob.ctypes.data, raw.ctypes.data, 1)
            cw, ch = min((w_in_b - (fx >> 2)) << 2, tw), min((h_in_b - (fy >> 2)) << 2, th)  # frame_clipped_tx
            items.append(K.item(len(qs), int(eob[0]), tx, ty, 0, bs, mode, P["red"], bx * tw // 4, by * th // 4,
                                cw >> 2, ch >> 2))
            qs.append(q)
            if eob[0] > 0 and ((tw, th) != (bw, bh) or dm != 0):
                L.orc_inverse_transform_add(r.ctypes.data, is32, work.ctypes.data + (r0 * stride + c0) * bpp, stride,
                                            bpp, tx, ty, bd)
            if dm == 0 and visible:
                txd += scale_mul(P["ds"], scale_mul(P["bias"](fx >> 2, fy >> 2), raw[0]))
    chain = np.zeros(1, COEFF_CHAIN_DTYPE)
    chain["snapshot"], chain["init_rng"], chain["item_count"] = it["snapshot"], 32768, len(items)
    chain["above"][0, 0], chain["left"][0, 0] = it["above"], it["left"]
    rate = int(K.oracle_rate(P["cdfs"], chain, np.array(items), np.concatenate(qs))[0][0])
    if dm == 0:
        dist = txd
    else:  # compute_distortion's luma term over the visible block (rdo.rs:254-293)
        fx0, fy0 = rx + x0, ry + y0
        vw, vh = max(0, min(bw, W - fx0)), max(0, min(bh, H - fy0))
        sp = addr(src.data, x0, y0)
        dp = addr(work, x0, y0)
        dist = 0
        if vw and vh and dm == 1:  # sse_wxh: one bias per 4x4 chunk
            nw, nh = -(-vw // 4), -(-vh // 4)
            sc = np.array([[P["bias"]((fx0 >> 2) + cx, (fy0 >> 2) + cy) for cx in range(nw)] for cy in range(nh)],
                          np.uint32)
            f = L.orc_weighted_sse_u8 if bpp == 1 else L.orc_weighted_sse_u16
            dist = f(sp, stride, dp, stride, sc.ctypes.data, nw, vw, vh)
        elif vw and vh:  # cdef_dist_wxh: 8x8 steps
            f = L.orc_cdef_dist_kernel_u8 if bpp == 1 else L.orc_cdef_dist_kernel_u16
            for yy in range(0, vh, 8):
                for xx in range(0, vw, 8):
                    v = f(sp + (yy * stride + xx) * bpp, stride, dp + (yy * stride + xx) * bpp, stride,
                          min(8, vw - xx), min(8, vh - yy), bd, None)
                    dist += scale_mul(P["bias"]((fx0 + xx) >> 2, (fy0 + yy) >> 2), v)
        dist = scale_mul(P["ds"], dist)
    return rate, dist, L.orc_compute_rd_cost(P["lam"], rate, dist)


def restate(it, cands, reduced):
    """rdo_tx_size_type over the recorded (rate, dist, rd): expected states and (size, type, rd)."""
    best_rd, best_size, best_type = np.finfo(np.float64).max, T.MAX_TX[it["bsize"]], 0
    states = np.full(21, TX_NOT_IN_LADDER)
    lad = T.ladder(int(it["bsize"]))
    for l, t in enumerate(lad):
        lst = T.type_list(t, int(it["skip"]), reduced)
        first, cut, size_rd, size_type = True, False, np.finfo(np.float64).max, 0
        for k, ty in enumerate(T.TX_TYPES):
            if ty not in lst:
                states[l * 7 + k] = TX_NOT_IN_SET
                continue
            if cut:
                states[l * 7 + k] = TX_CUT
                continue
            states[l * 7 + k] = TX_EVALUATED
            rd = cands[l * 7 + k]["rd"]
            if first:
                first = False
                if rd > best_rd:
                    cut = True
                    continue
            if rd < size_rd:
                size_rd, size_type = rd, ty
        if size_rd < best_rd:
            best_rd, best_size, best_type = size_rd, t, size_type
    return states, (best_size, best_type, best_rd)


CASES = [  # (w, h, bd, dist_mode, reduced, rect, scale)
    (96, 80, 8, 2, 0, None, False),
    (96, 80, 10, 1, 1, None, False),
    (100, 76, 12, 0, 0, None, True),
    (120, 90, 8, 0, 1, (32, 16, 88, 74), False),
    (70, 66, 8, 1, 0, None, True),
    (128, 96, 10, 2, 0, (16, 8, 112, 88), True),
]


def run_case(w, h, bd, dist_mode, reduced, rect, scale, seed, n=60):
    src, rec = T.make_case(w, h, bd, seed)
    rect = rect or (0, 0, w, h)
    rng = np.random.default_rng(seed)
    it = T.items(rng, rect[2], rect[3], n)
    cdfs = np.concatenate([K.default_cdfs(), K.random_cdfs(rng, 2)])
    it["snapshot"] %= len(cdfs)
    w_in_b = 2 * ((w + 7) >> 3)
    sc = rng.integers(1 << 12, 1 << 16, (2 * ((h + 7) >> 3), w_in_b)).astype(np.uint32) if scale else None
    lam = 0.0013 * 140 * 140 * (1 << (2 * (bd - 8)))
    ds = int(rng.integers(12000, 20000))
    best, cands = T.oracle(src, rec, PAD, rect, w, h, bd, dist_mode, reduced, lam, ds, sc, cdfs, it)
    return src, rec, rect, it, cdfs, sc, lam, ds, best, cands


@pytest.mark.parametrize("case", range(len(CASES)))
def test_candidates_equal_the_restatement(case):
    """Every EVALUATED record's rate, distortion and rd equal the candidate re-encoded from the pieces."""
    w, h, bd, dm, red, rect, scale = CASES[case]
    src, rec, rect, it, cdfs, sc, lam, ds, best, cands = run_case(w, h, bd, dm, red, rect, scale, seed=40 + case,
                                                                  n=24)
    osrc, orec = O.Plane(w, h, PAD, src.dtype), O.Plane(w, h, PAD, rec.dtype)
    osrc.fill_from(src)
    orec.fill_from(rec)
    P = dict(src=osrc, rec=orec, rect=rect, w=w, h=h, bd=bd, dm=dm, red=red, lam=lam, ds=ds, cdfs=cdfs,
             bias=(lambda x4, y4: 1 << 14) if sc is None else (lambda x4, y4: int(sc[y4, x4])))
    checked = 0
    for i in range(len(it)):
        for l, t in enumerate(T.ladder(int(it[i]["bsize"]))):
            for k, ty in enumerate(T.TX_TYPES):
                c = cands[i][l * 7 + k]
                if c["state"] != TX_EVALUATED:
                    continue
                rate, dist, rd = encode_candidate(P, it[i], t, ty)
                assert (int(c["rate"]), int(c["dist"])) == (rate, dist), (i, l, k)
                assert c["rd"] == rd
                checked += 1
    assert checked > 0


@pytest.mark.parametrize("case", range(len(CASES)))
def test_decision_rules(case):
    w, h, bd, dm, red, rect, scale = CASES[case]
    _, _, _, it, _, _, _, _, best, cands = run_case(w, h, bd, dm, red, rect, scale, seed=40 + case)
    for i in range(len(it)):
        states, (sz, ty, rd) = restate(it[i], cands[i], red)
        np.testing.assert_array_equal(cands[i]["state"], states)
        off = cands[i]["state"] != TX_EVALUATED
        assert (cands[i]["rate"][off] == 0).all() and (cands[i]["dist"][off] == 0).all()
        assert (best[i]["tx_size"], best[i]["tx_type"]) == (sz, ty) and best[i]["rd"] == rd
        assert T.TX_W[sz] <= T.BS_W[it[i]["bsize"]] and T.TX_H[sz] <= T.BS_H[it[i]["bsize"]]


def test_fixtures_show_every_rule():
    """Across the cases: the early exit fires at a later size, the ladder continues past it and wins there,
    winners spread over sizes and types, every size and mode occurs."""
    exits = wins_after_exit = clipped = paeth_edge = upsampled = 0
    winners, seen_sizes, seen_modes = set(), set(), set()
    for case, (w, h, bd, dm, red, rect, scale) in enumerate(CASES):
        _, _, rect, it, _, _, _, _, best, cands = run_case(w, h, bd, dm, red, rect, scale, seed=40 + case)
        for i in range(len(it)):
            bs, x, y, m = int(it[i]["bsize"]), int(it[i]["x"]), int(it[i]["y"]), int(it[i]["mode"])
            clipped += rect[0] + x + T.BS_W[bs] > w or rect[1] + y + T.BS_H[bs] > h
            paeth_edge += m == 12 and (x == 0 or y == 0)
            # D113 / D157 / D203 / D67 are 23 degrees off an axis: the edge filter upsamples at w + h <= 16
            upsampled += m in (5, 6, 7, 8) and it[i]["ief"] == 0 and any(
                T.TX_W[t] + T.TX_H[t] <= 16 for t in T.ladder(bs))
            st = cands[i]["state"].reshape(3, 7)
            seen_sizes.add(int(it[i]["bsize"]))
            seen_modes.add(int(it[i]["mode"]))
            lad = T.ladder(int(it[i]["bsize"]))
            for l in range(1, len(lad)):
                if (st[l] == TX_CUT).any():
                    exits += 1
                    if any(best[i]["tx_size"] == lad[m] for m in range(l + 1, len(lad))):
                        wins_after_exit += 1
            winners.add((int(best[i]["tx_size"]), int(best[i]["tx_type"])))
    assert exits > 0 and wins_after_exit > 0
    assert clipped > 0 and paeth_edge > 0 and upsampled > 0
    assert len({s for s, _ in winners}) >= 8 and len({t for _, t in winners}) >= 5
    assert seen_sizes == set(T.SIZES) and seen_modes == set(range(13))


def test_size_tie_keeps_the_larger_size():
    """At lambda 0 on a flat frame every candidate away from the frame's top / left edges predicts exactly: all rds are 0, the first size's first type
    wins, and no later size is cut (0 > 0 is false) while none replaces it (0 < 0 is false)."""
    w = h = 64
    flat = np.full((h, w), 97, np.uint8)
    it = T.grid_items(w, h, 16, 16, [0, 1, 2, 9])
    it = np.concatenate([it, T.grid_items(w, h, 32, 32, [0, 12])])
    it = it[(it["x"] > 0) & (it["y"] > 0)]  # at the frame's top / left the edges are the 128 +- 1 constants
    cdfs = K.default_cdfs()
    for dm in (0, 1, 2):
        best, cands = T.oracle(flat, flat, PAD, (0, 0, w, h), w, h, 8, dm, 0, 0.0, 16384, None, cdfs, it)
        for i in range(len(it)):
            lad = T.ladder(int(it[i]["bsize"]))
            rds = [cands[i][l * 7]["rd"] for l in range(len(lad))]
            assert len(lad) > 1 and rds == [0.0] * len(lad)
            assert (cands[i]["state"] != TX_CUT).all()
            assert (best[i]["tx_size"], best[i]["tx_type"], best[i]["rd"]) == (lad[0], 0, 0.0)
            states, want = restate(it[i], cands[i], 0)
            np.testing.assert_array_equal(cands[i]["state"], states)


def test_invalid_items():
    src, rec = T.make_case(64, 64, 8, 3)
    rng = np.random.default_rng(3)
    it = T.items(rng, 64, 64, 8)
    it["snapshot"] = 0
    it[0]["bsize"] = 13
    it[1]["mode"] = 13
    it[2]["x"] = 6
    it[3]["y"] = 64
    it[4]["dc_quant"] = 0
    it[5]["ac_quant"] = 65536
    it[6]["snapshot"] = 4
    best, cands = T.oracle(src, rec, PAD, (0, 0, 64, 64), 64, 64, 8, 2, 0, 100.0, 16384, None, K.default_cdfs(), it)
    assert (best["tx_size"][:7] == 0xFF).all() and (best["rd"][:7] == -1.0).all()
    assert (cands["state"][:7] == TX_INVALID).all()
    assert best[7]["tx_size"] != 0xFF
