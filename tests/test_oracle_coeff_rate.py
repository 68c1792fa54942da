"""Pins oracle/coeff_rate.c (the coefficient rate, rav1e's write_coeffs_lv_map through its WriterCounter) from
three sides, none of which reads the oracle's own symbol stream:

1. Tables: the spec-restated context and tx-set tables equal the reference's by sha256, and the golden default
   CDFs are the reference's (tests/golden/coeff_cdf_kats.json).
2. The AV1 specification: the decoder below, written from the symbol decoder and CDF adaptation (8.2), the
   coeffs() syntax (5.11.39) and its context derivations (8.3.2) in the specification's row-major orientation,
   decodes the oracle encoder's bytes and reproduces every item's tx_type, eob and coefficients, from the CDFs
   the chain carried.  ec.rs's own round-trip tests (booleans, cdf, mixed) are restated against it too.
3. The counter: an independent WriterCounter / frac_compute, fed with the symbols the decoder read, equals the
   oracle's rate for the chain's init_rng; the encoder backend's tell_frac equals the counter's.
"""
import hashlib
import json
import struct

import numpy as np
import pytest

from tests import coeff_rate_cases as K

WL, HL = K.TX_WL, K.TX_HL


# ---------------------------------------------------------------- independent WriterCounter (ec.rs:193-201, 334-379)
class Counter:
    def __init__(self, rng):
        self.rng, self.bits = rng, 0

    def store(self, fl, fh, nms):
        r = self.rng
        u = r if fl >= 32768 else (((r >> 8) * (fl >> 6)) >> 1) + 4 * nms
        v = (((r >> 8) * (fh >> 6)) >> 1) + 4 * (nms - 1)
        rr = (u - v) & 0xFFFF
        d = 16 - rr.bit_length()
        self.bits += d
        self.rng = (rr << d) & 0xFFFF

    def tell_frac(self):
        rng, lq = self.rng, 0
        for _ in range(3):
            rng = (rng * rng) >> 15
            b = rng >> 16
            lq = (lq << 1) | b
            rng >>= b
        return ((self.bits + 1) << 3) - lq


# ---------------------------------------------------------------- decoder from the AV1 specification (8.2)
class SpecDecoder:
    def __init__(self, data):
        self.data, self.bitpos = data, 0
        sz = len(data)
        nb = min(sz * 8, 15)
        buf = self.f(nb)
        self.value = ((1 << 15) - 1) ^ (buf << (15 - nb))
        self.range = 1 << 15
        self.maxbits = 8 * sz - 15
        self.log = []  # (fl, fh, nms) of each symbol in the encoder's inverse-CDF terms, for the counter

    def f(self, n):
        x = 0
        for _ in range(n):
            byte = self.data[self.bitpos >> 3] if (self.bitpos >> 3) < len(self.data) else 0
            x = (x << 1) | ((byte >> (7 - (self.bitpos & 7))) & 1)
            self.bitpos += 1
        return x

    def symbol(self, cdf, adapt=True):
        """read_symbol (8.2.6) over a specification CDF: N + 1 entries, cdf[N - 1] = 32768, cdf[N] the count."""
        n = len(cdf) - 1
        cur, s = self.range, -1
        while True:
            s += 1
            prev = cur
            fq = (1 << 15) - cdf[s]
            cur = (((self.range >> 8) * (fq >> 6)) >> 1) + 4 * (n - s - 1)
            if not self.value < cur:
                break
        fl = 32768 if s == 0 else 32768 - cdf[s - 1]
        fh = cdf[n] if s == n - 1 else 32768 - cdf[s]
        self.log.append((fl, fh, n - s))
        self.range = prev - cur
        self.value -= cur
        bits = 15 - (self.range.bit_length() - 1)
        self.range <<= bits
        nb = min(bits, max(0, self.maxbits))
        new = self.f(nb)
        self.value = (new << (bits - nb)) ^ (((self.value + 1) << bits) - 1)
        self.maxbits -= bits
        if adapt:  # 8.2.6's CDF update
            rate = 3 + (cdf[n] > 15) + (cdf[n] > 31) + min(n.bit_length() - 1, 2)
            tmp = 0
            for i in range(n - 1):
                if i == s:
                    tmp = 1 << 15
                if tmp < cdf[i]:
                    cdf[i] -= (cdf[i] - tmp) >> rate
                else:
                    cdf[i] += (tmp - cdf[i]) >> rate
            cdf[n] += cdf[n] < 32
        return s

    def boolean(self, f=16384):
        """read_bool with P(1) = f / 32768 (f = 16384: read_literal's bits)"""
        return self.symbol([32768 - f, 32768, 0], adapt=False)

    def literal(self, n):
        x = 0
        for _ in range(n):
            x = (x << 1) | self.boolean()
        return x


def spec_cdfs(snapshot):
    """The chain's snapshot in the specification's form: cdf[i] = 32768 - icdf[i], then 32768, then the count."""
    out = {}
    for name in snapshot.dtype.names:
        a = snapshot[name].astype(np.int64)
        rows = a.reshape(-1, a.shape[-1])
        out[name] = [[32768 - int(v) for v in r[:-1]] + [32768, int(r[-1])] for r in rows]
        out[name + "_shape"] = a.shape[:-1]
    return out


def row(cdfs, name, *idx):
    shape = cdfs[name + "_shape"]
    flat = 0
    for i, d in zip(idx, shape):
        flat = flat * d + i
    return cdfs[name][flat]


SIG_REF = {0: [(0, 1), (1, 0), (1, 1), (0, 2), (2, 0)], 1: [(0, 1), (1, 0), (0, 2), (0, 3), (0, 4)],
           2: [(0, 1), (1, 0), (2, 0), (3, 0), (4, 0)]}
MAG_REF = {0: [(0, 1), (1, 0), (1, 1)], 1: [(0, 1), (1, 0), (0, 2)], 2: [(0, 1), (1, 0), (2, 0)]}


def tx_class(tx_type):  # get_tx_class: V_* vertical (2), H_* horizontal (1)
    return 0 if tx_type < 10 else (1 if tx_type & 1 else 2)


def coeff_base_offset(t, row_, col):  # Coeff_Base_Ctx_Offset[txSz][min(row, 4)][min(col, 4)] by its rule
    w, h = 1 << WL[t], 1 << HL[t]
    if row_ == 0 and col == 0:
        return 0
    if w < h and row_ < 2:
        return 11
    if w > h and col < 2:
        return 16
    return 1 if row_ + col < 2 else 6 if row_ + col < 4 else 21


def spec_scan(t, tx_type):
    """The scan as row-major positions: the context's table (coefficient index col * H + row) transposed."""
    cw, ch = K.coded(t)
    s = K.scan_order(t, tx_type).astype(np.int64)
    return [(p % ch) * cw + p // ch for p in s]


def decode_item(dec, cdfs, it, win, eob_cdf_from_area=False):
    """coeffs() (5.11.39) for one transform block; win: per plane {"above": [(level, dc)] * 16, "left": ...}.
    Returns (tx_type or None, eob, coefficients in the quantizer's column-major layout)."""
    t, plane = int(it["tx_size"]), int(it["plane"])
    ptype = int(plane > 0)
    w, h = 1 << WL[t], 1 << HL[t]
    cw, ch = K.coded(t)
    bwl = cw.bit_length() - 1
    sq, up = min(WL[t], HL[t]) - 2, max(WL[t], HL[t]) - 2
    ctx_sz = (sq + up + 1) >> 1
    x4, y4, w4c, h4c = int(it["x4"]), int(it["y4"]), int(it["clip_w4"]), int(it["clip_h4"])
    above = win[plane]["above"][x4:x4 + w4c]
    left = win[plane]["left"][y4:y4 + h4c]
    bw, bh = 1 << K.BS_WL[int(it["plane_bsize"])], 1 << K.BS_HL[int(it["plane_bsize"])]
    if plane == 0:  # 8.3.2, all_zero
        top = min(max([lv for lv, _ in above] + [0]), 255)
        lft = min(max([lv for lv, _ in left] + [0]), 255)
        if bw == w and bh == h:
            ctx = 0
        elif top == 0 and lft == 0:
            ctx = 1
        elif top == 0 or lft == 0:
            ctx = 2 + (max(top, lft) > 3)
        elif max(top, lft) <= 3:
            ctx = 4
        elif min(top, lft) <= 3:
            ctx = 5
        else:
            ctx = 6
    else:
        a = any(lv | dc for lv, dc in above)
        lf = any(lv | dc for lv, dc in left)
        ctx = int(a) + int(lf) + 7 + (3 if bw * bh > w * h else 0)
    dc_sign = sum(-1 if dc == 1 else 1 if dc == 2 else 0 for _, dc in above + left)
    dc_ctx = 1 if dc_sign < 0 else 2 if dc_sign > 0 else 0
    all_zero = dec.symbol(row(cdfs, "txb_skip", ctx_sz, ctx))
    quant = [0] * (cw * ch)
    cul, dc_cat, eob, tx_type = 0, 0, 0, None
    if not all_zero:
        if plane == 0:  # transform_type (5.11.47)
            is_inter = int(it["mode"]) >= K.NEARESTMV
            st = K.tx_set(t, is_inter, int(it["reduced_tx_set"]))
            if st > 0:
                if is_inter:
                    name = {5: "inter_tx_1", 4: "inter_tx_2", 1: "inter_tx_3"}[st]
                    sym = dec.symbol(row(cdfs, name, sq))
                else:
                    name = {3: "intra_tx_1", 2: "intra_tx_2"}[st]
                    sym = dec.symbol(row(cdfs, name, sq, int(it["mode"])))
                tx_type = K.INV_SET[st][sym]
            else:
                tx_type = 0
            ptx = tx_type
        else:
            ptx = int(it["tx_type"])  # compute_tx_type's result for chroma is side information here
        cls = tx_class(ptx)
        scan = spec_scan(t, ptx)
        multi = (WL[t] + HL[t] - 4) if eob_cdf_from_area else (min(WL[t], 5) + min(HL[t], 5) - 4)
        eob_pt = dec.symbol(row(cdfs, "eob_flag%d" % (16 << min(multi, 6)), ptype, int(cls != 0))) + 1
        eob = eob_pt if eob_pt < 2 else (1 << (eob_pt - 2)) + 1
        shift = eob_pt - 3
        if shift >= 0:
            if dec.symbol(row(cdfs, "eob_extra", ctx_sz, ptype, eob_pt - 3)):
                eob += 1 << shift
            for i in range(1, max(0, eob_pt - 2)):
                shift = max(0, eob_pt - 2) - 1 - i
                if dec.literal(1):
                    eob += 1 << shift
        for c in range(eob - 1, -1, -1):
            pos = scan[c]
            r0, c0 = pos >> bwl, pos & (cw - 1)
            if c == eob - 1:
                ectx = 0 if c == 0 else 1 if c <= cw * ch // 8 else 2 if c <= cw * ch // 4 else 3
                level = dec.symbol(row(cdfs, "coeff_base_eob", ctx_sz, ptype, ectx)) + 1
            else:
                mag = 0
                for dr, dcl in SIG_REF[cls]:
                    rr, cc = r0 + dr, c0 + dcl
                    if rr < ch and cc < cw:
                        mag += min(abs(quant[(rr << bwl) + cc]), 3)
                bctx = min((mag + 1) >> 1, 4)
                if cls == 0:
                    bctx = 0 if pos == 0 else bctx + coeff_base_offset(t, min(r0, 4), min(c0, 4))
                else:
                    bctx += 26 + 5 * min(r0 if cls == 2 else c0, 2)
                level = dec.symbol(row(cdfs, "coeff_base", ctx_sz, ptype, bctx))
            if level > 2:
                mag = 0
                for dr, dcl in MAG_REF[cls]:
                    rr, cc = r0 + dr, c0 + dcl
                    if rr < ch and cc < cw:
                        mag += min(quant[rr * cw + cc], 15)
                mag = min((mag + 1) >> 1, 6)
                if pos == 0:
                    brc = mag
                elif (cls == 0 and r0 < 2 and c0 < 2) or (cls == 1 and c0 == 0) or (cls == 2 and r0 == 0):
                    brc = mag + 7
                else:
                    brc = mag + 14
                for _ in range(4):
                    br = dec.symbol(row(cdfs, "coeff_br", min(ctx_sz, 3), ptype, brc))
                    level += br
                    if br < 3:
                        break
            quant[pos] = level
        for c in range(eob):
            pos = scan[c]
            sign = 0
            if quant[pos]:
                sign = dec.symbol(row(cdfs, "dc_sign", ptype, dc_ctx)) if c == 0 else dec.literal(1)
            if quant[pos] > 14:
                length = 0
                while True:
                    length += 1
                    if dec.literal(1):
                        break
                    assert length < 40
                x = 1
                for _ in range(length - 1):
                    x = (x << 1) | dec.literal(1)
                quant[pos] = x + 14
            if pos == 0 and quant[pos] > 0:
                dc_cat = 1 if sign else 2
            cul = (cul + quant[pos]) & 0xFFFFFFFF
            if sign:
                quant[pos] = -quant[pos]
        cul = min(63, cul)
    for i in range(w >> 2):
        win[plane]["above"][x4 + i] = (cul, dc_cat)
    for i in range(h >> 2):
        win[plane]["left"][y4 + i] = (cul, dc_cat)
    col_major = np.zeros(cw * ch, np.int64)
    for pos, v in enumerate(quant):
        col_major[(pos & (cw - 1)) * ch + (pos >> bwl)] = v
    return tx_type, eob, col_major


def decode_chain(data, cdfs_snapshot, chain, items, eob_cdf_from_area=()):
    dec = SpecDecoder(data)
    cdfs = spec_cdfs(cdfs_snapshot)
    win = [{"above": [(int(v) & 63, int(v) >> 6) for v in chain["above"][p]],
            "left": [(int(v) & 63, int(v) >> 6) for v in chain["left"][p]]} for p in range(3)]
    out = []
    for k in range(int(chain["item_count"])):
        it = items[int(chain["item_begin"]) + k]
        out.append(decode_item(dec, cdfs, it, win, int(it["tx_size"]) in eob_cdf_from_area))
    return out, dec.log


# ---------------------------------------------------------------- 1. tables
def test_restated_tables_match_the_reference_digests():
    d = json.load(open(K.GOLDEN))
    buf = np.zeros(1024, np.int32)
    for name, info in d["table_digests"].items():
        n = K._lib().orc_coeff_table(name.encode(), buf.ctypes.data)
        assert n == info["n"], name
        assert hashlib.sha256(struct.pack("<%di" % n, *buf[:n].tolist())).hexdigest() == info["sha256"], name


def test_golden_defaults_are_valid_inverse_cdfs():
    cdfs = K.default_cdfs()
    assert len(cdfs) == 4
    for name in cdfs.dtype.names:
        a = cdfs[name].reshape(4, -1, cdfs[name].shape[-1]).astype(np.int64)
        assert (a[..., -1] == 0).all(), name  # adaptation counts start at 0
        assert (np.diff(a[..., :-1], axis=-1) <= 0).all() and (a[..., :-1] < 32768).all(), name
    # cdf_context.rs:124-128: the tx-type CDFs do not depend on the q context
    for name in ("intra_tx_1", "intra_tx_2", "inter_tx_1", "inter_tx_2", "inter_tx_3"):
        assert (cdfs[name] == cdfs[name][0]).all()


# ---------------------------------------------------------------- 2. ec.rs's round trips against the spec decoder
EC_CDF = [7296, 3819, 1716, 0]


def _spec(icdf):
    return [32768 - v for v in icdf[:-1]] + [32768, 0]


def test_ec_booleans_round_trip():
    vals = [(0, 1), (1, 2), (0, 3), (1, 1), (1, 2), (0, 3)]
    data, tf = K.oracle_script([(0, v, f) for v, f in vals], None)
    dec = SpecDecoder(data)
    assert [dec.boolean(f) for _, f in vals] == [v for v, _ in vals]
    assert tf[0] == tf[1]


@pytest.mark.parametrize("ops", [
    [(1, s, 0) for s in (0, 0, 0, 1, 1, 1, 2, 2, 2)],
    [(1, 0, 0), (0, 1, 2), (1, 0, 0), (0, 1, 2), (1, 0, 0), (0, 1, 2), (1, 1, 0), (0, 1, 1), (1, 1, 0),
     (0, 0, 2), (1, 1, 0), (1, 2, 0), (1, 2, 0), (1, 2, 0)]], ids=["cdf", "mixed"])
def test_ec_symbols_round_trip(ops):
    data, tf = K.oracle_script(ops, EC_CDF)
    dec = SpecDecoder(data)
    got = [dec.symbol(_spec(EC_CDF), adapt=False) if k == 1 else dec.boolean(f) for k, _, f in ops]
    assert got == [s for _, s, _ in ops]
    assert tf[0] == tf[1]


# ---------------------------------------------------------------- 2 + 3. every oracle case
# TX_16X64 / TX_64X16: encode_eob picks the eob CDF by tx_size.area_log2() - 4 (block_unit.rs:1866), i.e.
# eob_flag_cdf1024, where 5.11.39's eobMultisize (64-point dimensions counted as 32) picks eob_pt_512.
AREA_EOB_SIZES = (17, 18)


def _check_cases(cdfs, chains, items, q):
    rate, cul = K.oracle_rate(cdfs, chains, items, q)
    nsyms = 0
    for c, ch in enumerate(chains):
        ch32 = ch.copy()
        ch32["init_rng"] = 32768
        enc = K.oracle_encode(cdfs, ch32, items, q)
        assert enc is not None, c
        data, tf, nsym = enc
        decoded, log = decode_chain(data, cdfs[int(ch["snapshot"])], ch, items, AREA_EOB_SIZES)
        assert len(log) == nsym, c
        for k, (tx_type, eob, coeffs) in enumerate(decoded):
            it = items[int(ch["item_begin"]) + k]
            cw, chh = K.coded(int(it["tx_size"]))
            area = cw * chh
            blk = q[int(it["block"]) * area:(int(it["block"]) + 1) * area].astype(np.int64)
            assert eob == int(it["eob"]), (c, k)
            assert (coeffs == blk).all(), (c, k)
            if int(it["plane"]) == 0 and eob > 0:
                st = K.tx_set(int(it["tx_size"]), int(it["mode"]) >= K.NEARESTMV, int(it["reduced_tx_set"]))
                assert tx_type == (int(it["tx_type"]) if st > 0 else 0), (c, k)
        cnt = Counter(32768)
        for s in log:
            cnt.store(*s)
        assert tf[0] == tf[1] == cnt.tell_frac(), c  # encoder and counter share lr_compute
        cnt = Counter(int(ch["init_rng"]))
        start = cnt.tell_frac()
        for s in log:
            cnt.store(*s)
        assert rate[c] == cnt.tell_frac() - start, c
        nsyms += nsym
    return rate, cul, nsyms


@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_oracle_cases_decode_and_count(is32):
    cdfs, chains, items, q = K.oracle_cases(seed=11 + is32, is32=is32, full=bool(is32))
    rate, cul, nsyms = _check_cases(cdfs, chains, items, q)
    assert (rate != 0xFFFFFFFF).all()
    assert nsyms > 50000
    # reach: every size, eob 0 / 1 / full, golomb-long magnitudes, chains of 16, clipped windows, init_rng spread
    assert set(items["tx_size"].tolist()) == set(range(19))
    area = np.array([K.coded(int(t))[0] * K.coded(int(t))[1] for t in items["tx_size"]])
    assert (items["eob"] == 0).any() and (items["eob"] == 1).any() and (items["eob"] == area).any()
    assert np.abs(q.astype(np.int64)).max() >= (30000 if not is32 else 1 << 30)
    assert chains["item_count"].max() == 16 and (chains["init_rng"] != 32768).any()


def test_eob_cdf_of_16x64_and_64x16_follows_the_reference_not_5_11_39():
    """The one place rav1e's symbol stream and the specification's coeffs() part: 4:1 blocks with a 64-point
    side.  Decoding those with eob_pt_512 (the specification's choice) does not reproduce the block."""
    rng = np.random.default_rng(5)
    b = K.Batch(K.default_cdfs(), 0)
    for t in AREA_EOB_SIZES:
        blk = K.make_block(rng, t, 0, 300, 0)
        b.add_chain([K.item(b.add_block(blk), 300, t, 0)])
    cdfs, chains, items, q = b.arrays()
    for ch in chains:
        data, _, _ = K.oracle_encode(cdfs, ch, items, q)
        it = items[int(ch["item_begin"])]
        area = 512
        blk = q[int(it["block"]) * area:(int(it["block"]) + 1) * area]
        try:
            (_, eob, coeffs), = decode_chain(data, cdfs[0], ch, items)[0]
            assert eob != 300 or (coeffs != blk).any()
        except (AssertionError, IndexError):
            pass
        (_, eob, coeffs), = decode_chain(data, cdfs[0], ch, items, AREA_EOB_SIZES)[0]
        assert eob == 300 and (coeffs == blk).all()


def test_chain_contexts_carry_from_block_to_block():
    """A later block's txb_skip / dc_sign contexts come from earlier blocks: the same second block costs
    differently after a zero and after a large negative-DC first block."""
    rng = np.random.default_rng(3)
    b = K.Batch(K.default_cdfs(), 0)
    second = K.make_block(rng, 1, 0, 20, 0)
    for first_dc in (0, -500):
        blk = np.zeros(64, np.int64)
        blk[0] = first_dc
        i0 = K.item(b.add_block(blk), 1 if first_dc else 0, 1, 0, bsize=K.bsize_of(16, 16))
        i1 = K.item(b.add_block(second), 20, 1, 0, bsize=K.bsize_of(16, 16))
        b.add_chain([i0, i1])
    cdfs, chains, items, q = b.arrays()
    rate, cul = K.oracle_rate(cdfs, chains, items, q)
    assert cul[0] == 0 and cul[2] == 63 | 64
    assert rate[0] != rate[1]
    _check_cases(cdfs, chains, items, q)


def test_invalid_chains():
    rng = np.random.default_rng(9)
    b = K.Batch(K.default_cdfs(), 0)
    good = K.make_block(rng, 1, 0, 10, 0)
    gi = b.add_block(good)
    zero_tail = good.copy()
    zero_tail[K.scan_order(1, 0)[9]] = 0
    zi = b.add_block(zero_tail)
    mn = good.copy()
    mn[5] = -32768
    mi = b.add_block(mn)
    ok = K.item(gi, 10, 1, 0)
    bad = [K.item(gi, 10, 19, 0), K.item(gi, 10, 1, 16), K.item(gi, 65, 1, 0), K.item(zi, 10, 1, 0),
           K.item(gi, 10, 1, 0, plane=3), K.item(gi, 10, 1, 0, x4=15), K.item(gi, 10, 1, 0, clip_w4=0),
           K.item(gi, 10, 1, 4), K.item(gi, 10, 1, 0, mode=13), K.item(gi, 10, 1, 0, mode=34),
           K.item(mi, 10, 1, 0), K.item(1000, 10, 1, 0), K.item(gi, 10, 1, 0, bsize=22)]
    b.add_chain([ok])
    for it in bad:
        b.add_chain([ok, it])
    b.add_chain([ok], snapshot=4)
    b.add_chain([ok], init_rng=32767)
    b.add_chain([ok], init_rng=65536)
    cdfs, chains, items, q = b.arrays()
    rate, _ = K.oracle_rate(cdfs, chains, items, q)
    assert rate[0] != 0xFFFFFFFF and (rate[1:] == 0xFFFFFFFF).all()
    # a luma type outside its set is valid where write_tx_type does not assert: eob 0, or a DCT-only set
    b = K.Batch(K.default_cdfs(), 0)
    blk = K.make_block(rng, 3, 4, 10, 0)
    i32x32 = b.add_block(blk)
    b.add_chain([K.item(i32x32, 10, 3, 4)])  # 32x32 intra: DCT-only, no tx_type symbol
    b.add_chain([K.item(b.add_block(np.zeros(16, np.int64)), 0, 0, 12)])
    cdfs, chains, items, q = b.arrays()
    rate, _ = K.oracle_rate(cdfs, chains, items, q)
    assert (rate != 0xFFFFFFFF).all()
