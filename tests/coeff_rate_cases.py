"""Coefficient-rate cases shared by the oracle test, the GPU test and bench_kernels.py --coeff-rate: the CDF
snapshots (golden defaults and random valid ones), chains of transform blocks built from seeded coefficients,
and the ctypes binding of oracle/coeff_rate.c."""
import ctypes as C
import json
import os

import numpy as np

from rav1e_b200.backend import COEFF_CDFS_DTYPE, COEFF_CHAIN_DTYPE, COEFF_ITEM_DTYPE
from tests import oracle_lib as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "coeff_cdf_kats.json")
# TxSize 0..18 log2 width / height (transform/mod.rs), BlockSize 0..21 (partition.rs:130-153)
TX_WL = [2, 3, 4, 5, 6, 2, 3, 3, 4, 4, 5, 5, 6, 2, 4, 3, 5, 4, 6]
TX_HL = [2, 3, 4, 5, 6, 3, 2, 4, 3, 5, 4, 6, 5, 4, 2, 5, 3, 6, 4]
BS_WL = [2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5, 6, 6, 6, 7, 7, 2, 4, 3, 5, 4, 6]
BS_HL = [2, 3, 2, 3, 4, 3, 4, 5, 4, 5, 6, 5, 6, 7, 6, 7, 4, 2, 5, 3, 6, 4]
# the AV1 specification's inverse tx-type lists per TxSet (DCTONLY, INTER_3, INTRA_2, INTRA_1, INTER_2, INTER_1)
INV_SET = [[0], [9, 0], [9, 0, 3, 1, 2], [9, 0, 10, 11, 3, 1, 2], [9, 10, 11, 0, 1, 2, 4, 5, 3, 6, 7, 8],
           [9, 10, 11, 12, 13, 14, 15, 0, 1, 2, 4, 5, 3, 6, 7, 8]]
NEARESTMV = 14


def coded(t):
    return min(1 << TX_WL[t], 32), min(1 << TX_HL[t], 32)


def bsize_of(w, h):
    return next(b for b in range(22) if (1 << BS_WL[b], 1 << BS_HL[b]) == (w, h))


def tx_set(t, is_inter, reduced):
    """get_tx_set (transform_unit.rs:123-148), from the specification's rule."""
    up, sq = max(TX_WL[t], TX_HL[t]) - 2, min(TX_WL[t], TX_HL[t]) - 2
    if up > 3:
        return 0
    if is_inter:
        return 1 if (reduced or up == 3) else 4 if sq == 2 else 5
    if up == 3:
        return 0
    return 2 if (reduced or sq == 2) else 3


def default_cdfs():
    """The four golden default snapshots (q contexts 0..3) as COEFF_CDFS_DTYPE."""
    d = json.load(open(GOLDEN))
    return np.frombuffer(np.array(d["default_cdfs"], dtype="<u2").tobytes(), dtype=COEFF_CDFS_DTYPE).copy()


def random_cdfs(rng, n):
    """n random valid snapshots: strictly ordered inverse CDFs of every row, counts 0..32."""
    out = np.zeros(n, COEFF_CDFS_DTYPE)
    for name in COEFF_CDFS_DTYPE.names:
        a = out[name]
        nsym = a.shape[-1]
        rows = a.reshape(-1, nsym)
        for r in rows:
            cuts = np.sort(rng.choice(np.arange(1, 32768 // 64), nsym - 1, replace=False))[::-1] * 64
            cuts -= rng.integers(0, 64, nsym - 1)
            r[:nsym - 1] = np.sort(cuts)[::-1]
            r[nsym - 1] = rng.integers(0, 33)
    return out


def _level(rng, is32):
    """Magnitudes reaching every coding path: base 1 / 2, br 3..14 (1 / 2 / 3 / 14), golomb 15.., the 127 cap and
    long golomb codes (i32 magnitudes for high bit depth)."""
    k = rng.random()
    if k < 0.45:
        return int(rng.integers(1, 3))
    if k < 0.75:
        return int(rng.choice([3, 4, 5, 6, 13, 14]))
    if k < 0.9:
        return int(rng.choice([15, 16, 30, 126, 127, 128, 200]))
    hi = (1 << 31) - 1 if is32 else 32767
    return int(rng.integers(129, hi + 1)) if rng.random() < 0.7 else hi


def make_block(rng, t, tx_type, eob, is32, zero_frac=0.5, tail=False):
    """One coded block in the quantizer's layout (column-major, index = col * H + row): nonzero at scan[eob - 1],
    random below it (zero_frac of them 0), zero past it unless tail."""
    cw, ch = coded(t)
    area = cw * ch
    scan = scan_order(t, tx_type)
    blk = np.zeros(area, np.int64)
    for c in range(eob):
        if c == eob - 1 or rng.random() >= zero_frac:
            v = _level(rng, is32)
            blk[scan[c]] = -v if rng.random() < 0.5 else v
    if tail:
        for c in range(eob, area):
            if rng.random() < 0.3:
                blk[scan[c]] = int(rng.integers(-200, 201))
    return blk


_SCANS = {}


def scan_order(t, tx_type):
    key = (t, 0 if tx_type < 10 else 2 if tx_type & 1 else 1)
    if key not in _SCANS:
        area = coded(t)[0] * coded(t)[1]
        s = np.zeros(area, np.uint16)
        O.lib().orc_scan_order(t, tx_type, s.ctypes.data, None)
        _SCANS[key] = s
    return _SCANS[key]


class Batch:
    """Chains under construction: items, blocks (one coefficient buffer per call) and CDF snapshots."""

    def __init__(self, cdfs, is32):
        self.cdfs, self.is32 = cdfs, is32
        self.chains, self.items, self.coeffs = [], [], []
        self.ncoef = 0

    def add_block(self, blk):
        """Appends a coded block; returns its `block` index for its own size (the buffer is kept aligned)."""
        area = len(blk)
        pad = (-self.ncoef) % area
        if pad:
            self.coeffs.append(np.zeros(pad, np.int64))
            self.ncoef += pad
        idx = self.ncoef // area
        self.coeffs.append(blk)
        self.ncoef += area
        return idx

    def add_chain(self, items, snapshot=0, init_rng=32768, above=None, left=None):
        ch = np.zeros((), COEFF_CHAIN_DTYPE)
        ch["snapshot"], ch["init_rng"] = snapshot, init_rng
        ch["item_begin"], ch["item_count"] = len(self.items), len(items)
        if above is not None:
            ch["above"] = above
        if left is not None:
            ch["left"] = left
        self.chains.append(ch)
        self.items += items
        return len(self.chains) - 1

    def arrays(self):
        dt = np.int32 if self.is32 else np.int16
        q = np.concatenate(self.coeffs).astype(dt) if self.coeffs else np.zeros(1, dt)
        chains = np.array(self.chains, COEFF_CHAIN_DTYPE) if self.chains else np.zeros(0, COEFF_CHAIN_DTYPE)
        items = np.array(self.items, COEFF_ITEM_DTYPE) if self.items else np.zeros(0, COEFF_ITEM_DTYPE)
        return self.cdfs, chains, items, q


def item(block, eob, t, tx_type, plane=0, bsize=None, mode=0, reduced=0, x4=0, y4=0, clip_w4=None, clip_h4=None):
    it = np.zeros((), COEFF_ITEM_DTYPE)
    ts = t if t < 19 else 0  # out-of-range sizes (invalid-item tests) take 4x4 geometry
    w4, h4 = 1 << (TX_WL[ts] - 2), 1 << (TX_HL[ts] - 2)
    it["block"], it["eob"], it["tx_size"], it["tx_type"], it["plane"] = block, eob, t, tx_type, plane
    it["plane_bsize"] = bsize_of(1 << TX_WL[ts], 1 << TX_HL[ts]) if bsize is None else bsize
    it["mode"], it["reduced_tx_set"], it["x4"], it["y4"] = mode, reduced, x4, y4
    it["clip_w4"] = w4 if clip_w4 is None else clip_w4
    it["clip_h4"] = h4 if clip_h4 is None else clip_h4
    return it


def eob_choices(rng, t):
    area = coded(t)[0] * coded(t)[1]
    return [0, 1, int(rng.integers(2, max(3, area // 2))), area]


def oracle_cases(seed, is32, full=True):
    """The oracle cases: every tx size x every valid type of each set (intra, inter, reduced) at planes 0 / 1 / 2,
    eob 0 / 1 / mid / full, chains of up to 16 blocks sharing a context window, frame-clipped blocks, random
    windows, golden and random CDF snapshots, init_rng across 32768..65535."""
    rng = np.random.default_rng(seed)
    cdfs = np.concatenate([default_cdfs(), random_cdfs(rng, 3)])
    b = Batch(cdfs, is32)

    def one(t, tx_type, plane, mode, reduced, eob, **kw):
        blk = make_block(rng, t, tx_type, eob, is32)
        return item(b.add_block(blk), eob, t, tx_type, plane=plane, mode=mode, reduced=reduced, **kw)

    def rnd_window():
        v = rng.integers(0, 64, (3, 16)) | (rng.integers(0, 3, (3, 16)) << 6)
        return v.astype(np.uint8)

    for t in range(19):
        for is_inter in (0, 1):
            for reduced in (0, 1):
                types = INV_SET[tx_set(t, is_inter, reduced)]
                for k, tt in enumerate(types):
                    eobs = eob_choices(rng, t)
                    eob = eobs[k % 4] if full or t < 2 or k % 4 != 3 else eobs[2]
                    mode = int(rng.integers(NEARESTMV, 34)) if is_inter else int(rng.integers(0, 13))
                    b.add_chain([one(t, tt, 0, mode, reduced, eob)], snapshot=int(rng.integers(0, len(cdfs))),
                                init_rng=int(rng.integers(32768, 65536)) if rng.random() < 0.5 else 32768,
                                above=rnd_window(), left=rnd_window())
        for plane in (1, 2):
            for eob in eob_choices(rng, t)[:3 if not full and t >= 2 else 4]:
                bs = rng.choice([bsize_of(1 << TX_WL[t], 1 << TX_HL[t]), min(21, bsize_of(1 << TX_WL[t], 1 << TX_HL[t]) + 3)])
                b.add_chain([one(t, int(rng.integers(0, 16)), plane, int(rng.integers(0, 14)), 0, eob, bsize=int(bs))],
                            snapshot=int(rng.integers(0, len(cdfs))), above=rnd_window(), left=rnd_window())
    # chains of up to 16 blocks whose later txb_skip / dc_sign contexts come from earlier blocks
    for n in (2, 4, 16):
        for _ in range(3):
            items = []
            t = int(rng.choice([0, 1, 5, 6, 13, 14]))
            w4, h4 = 1 << (TX_WL[t] - 2), 1 << (TX_HL[t] - 2)
            plane = int(rng.integers(0, 3))
            for k in range(n):
                x4, y4 = (k * w4) % (16 - w4 + 1), (k * h4 // 2) % (16 - h4 + 1)
                tt = int(rng.choice(INV_SET[tx_set(t, 0, 0)])) if plane == 0 else int(rng.integers(0, 16))
                items.append(one(t, tt, plane, int(rng.integers(0, 13)), 0, int(rng.choice(eob_choices(rng, t))),
                                 bsize=bsize_of(16, 16), x4=x4, y4=y4))
            b.add_chain(items, snapshot=int(rng.integers(0, len(cdfs))), init_rng=int(rng.integers(32768, 65536)))
    # frame-clipped blocks: fewer window entries read than the tx block writes
    for t in (1, 2, 3, 4, 9, 12):
        w4, h4 = 1 << (TX_WL[t] - 2), 1 << (TX_HL[t] - 2)
        for plane in (0, 1):
            tt = 0
            b.add_chain([one(t, tt, plane, 0, 0, int(rng.choice(eob_choices(rng, t)[1:])), bsize=bsize_of(64, 64),
                             clip_w4=max(1, w4 // 2), clip_h4=max(1, h4 - 1))],
                        snapshot=int(rng.integers(0, len(cdfs))), above=rnd_window(), left=rnd_window())
    return b.arrays()


# ---------------------------------------------------------------- oracle binding
def _lib():
    L = O.lib()
    if not getattr(L, "_coeff_rate_bound", False):
        vp, sz, i32 = C.c_void_p, C.c_size_t, C.c_int
        L.orc_coeff_rate.restype = None
        L.orc_coeff_rate.argtypes = [vp, sz, vp, sz, vp, sz, vp, sz, i32, vp, vp]
        L.orc_coeff_encode_chain.restype = C.c_long
        L.orc_coeff_encode_chain.argtypes = [vp, sz, vp, vp, sz, vp, sz, i32, vp, sz, vp, vp]
        L.orc_ec_encode_script.restype = C.c_long
        L.orc_ec_encode_script.argtypes = [vp, sz, vp, i32, vp, sz, vp]
        L.orc_coeff_table.restype = i32
        L.orc_coeff_table.argtypes = [C.c_char_p, vp]
        L.orc_scan_order.restype = None
        L.orc_scan_order.argtypes = [i32, i32, vp, vp]
        L._coeff_rate_bound = True
    return L


def oracle_rate(cdfs, chains, items, q):
    rate = np.zeros(len(chains), np.uint32)
    cul = np.full(max(1, len(items)), 0xEE, np.uint8)
    _lib().orc_coeff_rate(cdfs.ctypes.data, len(cdfs), chains.ctypes.data, len(chains), items.ctypes.data,
                          len(items), q.ctypes.data, len(q), int(q.dtype == np.int32), rate.ctypes.data,
                          cul.ctypes.data)
    return rate, cul[:len(items)]


def oracle_encode(cdfs, chain, items, q):
    """(bytes, [encoder tell_frac, counter tell_frac], symbol count) of one chain, None if invalid."""
    cap = 1 << 22
    out = np.zeros(cap, np.uint8)
    tf = np.zeros(2, np.uint32)
    nsym = C.c_long(0)
    ch = np.array(chain, COEFF_CHAIN_DTYPE)
    n = _lib().orc_coeff_encode_chain(cdfs.ctypes.data, len(cdfs), ch.ctypes.data, items.ctypes.data, len(items),
                                      q.ctypes.data, len(q), int(q.dtype == np.int32), out.ctypes.data, cap,
                                      tf.ctypes.data, C.byref(nsym))
    if n == -1:
        return None
    assert n >= 0, n
    return out[:n].tobytes(), tf, nsym.value


def oracle_script(ops, cdf):
    ops = np.ascontiguousarray(np.array(ops, np.int32).reshape(-1))
    cdf = np.ascontiguousarray(np.array(cdf if cdf is not None else [0], np.uint16))
    out = np.zeros(1 << 12, np.uint8)
    tf = np.zeros(2, np.uint32)
    n = _lib().orc_ec_encode_script(ops.ctypes.data, len(ops) // 3, cdf.ctypes.data, len(cdf), out.ctypes.data,
                                    len(out), tf.ctypes.data)
    assert n >= 0
    return out[:n].tobytes(), tf


# ---------------------------------------------------------------- rdo_tx_type_decision batches on the device
def tx_decision_batch(c, width, height, bd, seed, tx_size=2, dc_q=140, ac_q=160, pad=32):
    """Every tx_size block of a seeded frame through b200_encode_tx_blocks_dev for all 16 intra types (zero
    motion against a second frame as the prediction), then one chain per (block, type of its set), block-major
    as rdo_tx_type_decision walks them (types outside the set skipped, rdo.rs:1734).
    Returns a dict of device buffers and host copies."""
    import torch

    from tests import gpu_util as G
    dt = np.uint8 if bd == 8 else np.uint16
    cur, ref = G.make_planes(width, height, pad, dt, seed=seed, bit_depth=bd)
    dcur, dref = c.plane_from_host(cur, pad), c.plane_from_host(ref, pad)
    tw, th = 1 << TX_WL[tx_size], 1 << TX_HL[tx_size]
    blocks = G.grid_blocks(width, height, tw, th)
    n = len(blocks)
    cw, ch = coded(tx_size)
    area = cw * ch
    is32 = bd > 8
    ctype = torch.int32 if is32 else torch.int16
    d_blocks = G.to_dev(blocks)
    d_q = torch.zeros(16 * n * area, dtype=ctype, device="cuda")
    d_eob = torch.zeros(16 * n, dtype=torch.int16, device="cuda")
    d_dist = torch.zeros(16 * n, dtype=torch.int64, device="cuda")
    for tt in range(16):
        c.encode_tx_blocks_dev(dcur, dref, dref, d_blocks, n, None, tx_size, tt, bd, dc_q, ac_q, True, False, None,
                               d_q[tt * n * area:], None, d_eob[tt * n:], d_dist[tt * n:])
    c.synchronize()
    eob = d_eob.cpu().numpy().view(np.uint16).reshape(16, n)
    types = INV_SET[tx_set(tx_size, 0, 0)]
    b = Batch(default_cdfs(), is32)
    bs = bsize_of(tw, th)
    for i in range(n):
        for tt in types:
            b.add_chain([item(tt * n + i, int(eob[tt, i]), tx_size, tt, bsize=bs, mode=0)])
    cdfs, chains, items, _ = b.arrays()
    return {"n": n, "types": types, "area": area, "is32": is32, "d_q": d_q, "d_eob": d_eob, "d_dist": d_dist,
            "q": d_q.cpu().numpy(), "eob": eob, "dist": d_dist.cpu().numpy().view(np.uint64).reshape(16, n),
            "cdfs": cdfs, "chains": chains, "items": items, "planes": (dcur, dref)}
