"""The coefficient rate on every kernel path, bit exact against the oracle: b200_coeff_rate_dev (coeff_rate.cu and
coeff_rate_dev.cuh's count_item, the per-block counter the transform size / type kernel shares) against
oracle/coeff_rate.c, rates and cul_level bytes.

The launch geometry mirrored here (coeff_rate.cu):
- `min(ceil(n / 4), 16 * num_sms)` CTAs of 4 warps, grid-stride loop;
- one warp per chain, so chain `ci` runs on warp `ci mod (4 * grid)`, after every earlier chain of that warp,
  in the same shared-memory CDF copy;
- lane 0 runs the serial coder; the other lanes build levels, contexts and cul_level's partial sums.
The sections:
1. every context of get_txb_ctx: luma txb_skip 0-6 and chroma 7-12 at every txs_ctx, dc_sign 0-2, window
   bytes with sign fields 1-3, frame-clipped reads with entries past the clip, windows at 16 - width_mi and
   the 64x128 / 128x64 / 128x128 plane sizes around 64-point transforms;
2. every eob group at its first and last eob for all 19 sizes and the three scan classes, the top eob_extra
   bit, the last-position thresholds of the coded area, DCT-only luma sets with other types;
3. magnitudes: the base / br / golomb borders, 127-capped neighbours, every golomb length in i16 and i32,
   the same values as i16 and i32, and the u32 wrap of cul_level's sum read by the next block;
4. CDF regions within a chain: every sharing pair across sizes, planes, intra / inter and reduced sets, one
   chain coding every region twice, a ~2000-item chain, snapshot counts 0 / 15 / 16 / 31 / 32 and saturated
   rows at init_rng 32768 and 65535;
5. warp reuse: every section-4 chain on a warp that just ran a chain adapting every region from another
   snapshot, then an invalid and an empty chain; empty, overlapping and out-of-order item ranges; an
   init_rng sweep;
6. read footprints restated from the contract's context rules, every other byte replaced between runs,
   misaligned base pointers, ncoeffs at and below the last block, sentinels past the outputs, NULL cul_level.
The reach assertions and the footprint restatement (pinned on the oracle) need no device.
"""
from collections import Counter

import numpy as np
import pytest

from rav1e_b200.backend import COEFF_CDFS_DTYPE, COEFF_CHAIN_DTYPE
from tests import coeff_rate_cases as K
from tests.test_oracle_coeff_rate import coeff_base_offset

WL, HL, BWL, BHL = K.TX_WL, K.TX_HL, K.BS_WL, K.BS_HL
INV = 0xFFFFFFFF
WARPS_PER_SM = 16 * 4  # coeff_rate.cu: 16 CTAs per SM of kWarps = 4
SIZES_BY_TXS = {0: [0], 1: [1, 5, 6, 13, 14], 2: [2, 7, 8, 15, 16], 3: [3, 9, 10, 17, 18], 4: [4, 11, 12]}
MAG_ZERO = (0, 64, 128, 192)  # luma: no magnitude after & 63, sign fields 0..3
EOB_GROUPS = [(1, 1), (2, 2)] + [((1 << (g - 2)) + 1, 1 << (g - 1)) for g in range(3, 12)]
_OFF = {n: COEFF_CDFS_DTYPE.fields[n][1] // 2 for n in COEFF_CDFS_DTYPE.names}


gpu = pytest.mark.gpu


def txs_of(t):
    return (min(WL[t], HL[t]) + max(WL[t], HL[t]) - 4 + 1) >> 1


def tx_cls(tt):
    return 0 if tt < 10 else (1 if tt & 1 else 2)


def area_of(t):
    cw, ch = K.coded(t)
    return cw * ch


def row_span(name, idx):
    """(first u16, length) of one CDF row of a snapshot."""
    shape = COEFF_CDFS_DTYPE[name].shape
    flat = int(np.ravel_multi_index(idx, shape[:-1])) if len(shape) > 1 else 0
    return _OFF[name] + flat * shape[-1], shape[-1]


def region(name, idx):
    """The CDF region a row belongs to: the unit coeff_rate_dev.cuh copies on first use."""
    if name.startswith("eob_flag") or name == "dc_sign":
        return (name,) + tuple(idx)
    keep = {"txb_skip": 1, "eob_extra": 2, "coeff_base_eob": 2, "coeff_base": 2, "coeff_br": 2, "intra_tx_1": 2,
            "intra_tx_2": 2, "inter_tx_1": 1, "inter_tx_2": 1, "inter_tx_3": 1}[name]
    return (name,) + tuple(idx[:keep])


def luma_setup(t, tt):
    """(mode, reduced) under which luma (t, tt) with eob > 0 is valid: tt in its set, or a DCT-only set."""
    for is_inter in (0, 1):
        for reduced in (0, 1):
            types = K.INV_SET[K.tx_set(t, is_inter, reduced)]
            if len(types) == 1 or tt in types:
                mode = (K.NEARESTMV + (t + tt) % 20) if is_inter else (t * 5 + tt) % 13
                return mode, reduced
    raise AssertionError((t, tt))


# ---------------------------------------------------------------- restatement of the contract's context rules
def skip_dc_ctx(above, left, it):
    """get_txb_ctx (b200rdo.h): the txb_skip and dc_sign contexts from the window entries the item reads."""
    t, plane, bs = int(it["tx_size"]), int(it["plane"]), int(it["plane_bsize"])
    a = [int(v) for v in above[plane][int(it["x4"]):int(it["x4"]) + int(it["clip_w4"])]]
    lf = [int(v) for v in left[plane][int(it["y4"]):int(it["y4"]) + int(it["clip_h4"])]]
    dc = sum({1: -1, 2: 1}.get(v >> 6, 0) for v in a + lf)
    top = lft = 0
    for v in a:
        top |= v
    for v in lf:
        lft |= v
    if plane == 0:
        if (BWL[bs], BHL[bs]) == (WL[t], HL[t]):
            skip = 0
        else:
            top, lft = top & 63, lft & 63
            mx, mn = min(top | lft, 4), min(top, lft, 4)
            skip = 1 if not mx else (2 + (mx > 3)) if not mn else 4 if mx <= 3 else 5 if mn <= 3 else 6
    else:
        skip = (top != 0) + (lft != 0) + (10 if BWL[bs] + BHL[bs] > WL[t] + HL[t] else 7)
    return skip, (1 if dc < 0 else 2 if dc > 0 else 0)


def eob_pt_of(eob):
    return eob if eob < 3 else (eob - 1).bit_length() + 1


def trace_chain(ch, items, q, contexts=True):
    """What one valid chain codes, restated item by item: per item a dict of its contexts, eob group, golomb
    lengths and cul_level byte; the chain's symbols as a Counter of (CDF field, row index); the window entries
    read before the chain writes them.  contexts=False skips the per-coefficient base / br rows (their
    regions are still recorded)."""
    above, left = ch["above"].astype(np.int64).copy(), ch["left"].astype(np.int64).copy()
    written = np.zeros((2, 3, 16), bool)
    syms, regions, win_reads, out = Counter(), set(), set(), []
    b0, n = int(ch["item_begin"]), int(ch["item_count"])
    for it in items[b0:b0 + n]:
        t, plane, eob, tt = int(it["tx_size"]), int(it["plane"]), int(it["eob"]), int(it["tx_type"])
        ptype, txs, cls = int(plane > 0), txs_of(t), tx_cls(tt)
        x4, y4 = int(it["x4"]), int(it["y4"])
        for side, s0, cnt in ((0, x4, int(it["clip_w4"])), (1, y4, int(it["clip_h4"]))):
            for i in range(s0, s0 + cnt):
                if not written[side, plane, i]:
                    win_reads.add((side, plane, i))
        skip, dc_ctx = skip_dc_ctx(above, left, it)
        rec = {"t": t, "plane": plane, "ptype": ptype, "txs": txs, "skip": skip, "dc_ctx": None, "eob": eob,
               "cls": cls, "eob_pt": 0, "top_bit": None, "last_ctx": None, "golomb": [], "br": False}

        def use(name, *idx):
            syms[(name, tuple(int(i) for i in idx))] += 1
            regions.add(region(name, idx))

        use("txb_skip", txs, skip)
        cl = 0
        if eob:
            area = area_of(t)
            cw, chh = K.coded(t)
            blk = np.asarray(q[int(it["block"]) * area:(int(it["block"]) + 1) * area], np.int64)
            scan = K.scan_order(t, tt).astype(np.int64)
            if plane == 0:
                is_inter, sq = int(it["mode"]) >= K.NEARESTMV, min(WL[t], HL[t]) - 2
                st = K.tx_set(t, is_inter, int(it["reduced_tx_set"]))
                if len(K.INV_SET[st]) > 1:
                    if is_inter:
                        use({5: "inter_tx_1", 4: "inter_tx_2", 1: "inter_tx_3"}[st], sq)
                    else:
                        use({3: "intra_tx_1", 2: "intra_tx_2"}[st], sq, int(it["mode"]))
            pt = eob_pt_of(eob)
            rec["eob_pt"] = pt
            use("eob_flag%d" % (16 << min(WL[t] + HL[t] - 4, 6)), ptype, int(cls != 0))
            if pt >= 3:
                use("eob_extra", txs, ptype, pt - 3)
                rec["top_bit"] = ((eob - ((1 << (pt - 2)) + 1)) >> (pt - 3)) & 1
            c = eob - 1
            rec["last_ctx"] = 0 if c == 0 else 1 if c <= area // 8 else 2 if c <= area // 4 else 3
            use("coeff_base_eob", txs, ptype, rec["last_ctx"])
            mags = np.abs(blk)
            lv = np.zeros((cw + 4, chh + 4), np.int64)
            lv[:cw, :chh] = np.minimum(mags, 127).reshape(cw, chh)
            bhl = chh.bit_length() - 1
            brt = min(txs, 3)
            for c in range(eob - 1, -1, -1):
                pos = int(scan[c])
                level = int(mags[pos])
                if c < eob - 1:
                    regions.add(("coeff_base", txs, ptype))
                if level > 2:
                    rec["br"] = True
                    regions.add(("coeff_br", brt, ptype))
                if not contexts:
                    continue
                col, row = pos >> bhl, pos & (chh - 1)
                if c < eob - 1:
                    g = lambda dc_, dr: min(3, int(lv[col + dc_, row + dr]))  # noqa: E731
                    mag = g(0, 1) + g(1, 0)
                    mag += (g(1, 1) + g(0, 2) + g(2, 0)) if cls == 0 else (g(0, 2) + g(0, 3) + g(0, 4)) if cls == 2 \
                        else (g(2, 0) + g(3, 0) + g(4, 0))
                    if cls == 0 and pos == 0:
                        ctx = 0
                    else:
                        ctx = min((mag + 1) >> 1, 4)
                        ctx += coeff_base_offset(t, min(row, 4), min(col, 4)) if cls == 0 else \
                            26 + 5 * min(col if cls == 1 else row, 2)
                    use("coeff_base", txs, ptype, ctx)
                if level > 2:
                    m = int(lv[col, row + 1] + lv[col + 1, row])
                    m += int(lv[col + 1, row + 1] if cls == 0 else lv[col + 2, row] if cls == 1 else lv[col, row + 2])
                    m = min((m + 1) >> 1, 6)
                    near = (row < 2 and col < 2) if cls == 0 else col == 0 if cls == 1 else row == 0
                    br = m if pos == 0 else m + 7 if near else m + 14
                    for _ in range(min((level - 3) // 3 + 1, 4)):
                        use("coeff_br", brt, ptype, br)
            dc = int(blk[scan[0]])
            if dc:
                use("dc_sign", ptype, dc_ctx)
                rec["dc_ctx"] = dc_ctx
            for c in range(eob):
                if mags[scan[c]] > 14:
                    rec["golomb"].append(int(mags[scan[c]] - 14).bit_length())
            cul = int(mags[scan[:eob]].sum()) & 0xFFFFFFFF
            rec["cul_sum"] = cul
            cl = min(cul, 63)
            if dc:
                cl = cl | 64 if dc < 0 else cl + 128
        rec["cul"] = cl
        w4, h4 = 1 << (WL[t] - 2), 1 << (HL[t] - 2)
        above[plane][x4:x4 + w4] = cl
        left[plane][y4:y4 + h4] = cl
        written[0, plane, x4:x4 + w4] = True
        written[1, plane, y4:y4 + h4] = True
        out.append(rec)
    return out, syms, regions, win_reads


def trace_all(chains, items, q, contexts=True):
    return [trace_chain(ch, items, q, contexts) for ch in chains]


# ---------------------------------------------------------------- fixtures
def snapshots(rng):
    return np.concatenate([K.default_cdfs(), K.random_cdfs(rng, 3)])


def bigger_bsizes(t):
    """Plane block sizes that hold the transform and are larger than it."""
    return [b for b in range(22) if BWL[b] >= WL[t] and BHL[b] >= HL[t] and (BWL[b], BHL[b]) != (WL[t], HL[t])]


def entries(v, n, zero_pool, rng):
    """n window entries whose OR is v (3 as 1 | 2 when n > 1), padded with entries from zero_pool."""
    out = [int(rng.choice(zero_pool)) for _ in range(n)]
    if v == 3 and n > 1:
        out[0] = (out[0] & 0xC0) | 1
        out[-1] = (out[-1] & 0xC0) | 2
    elif v:
        out[int(rng.integers(0, n))] = (int(rng.choice(zero_pool)) & 0xC0) | v
    return out


def noise_window(rng):
    return rng.integers(0, 256, (3, 16)).astype(np.uint8)


def ctx_block(rng, t, tt, is32):
    """A block with a nonzero DC (so dc_sign is coded) and a small random eob."""
    area = area_of(t)
    eob = int(rng.integers(1, min(area, 40) + 1))
    blk = K.make_block(rng, t, tt, eob, is32)
    if blk[0] == 0:
        blk[0] = int(rng.choice([-3, -1, 1, 2, 20]))
    return blk, eob


def context_cases(is32, seed=31):
    """Section 1: single-block chains with constructed windows.  Returns (arrays, notes) where notes[i] is the
    skip context chain i was built for, or None when the case is about something else."""
    rng = np.random.default_rng(seed)
    b = K.Batch(snapshots(rng), is32)
    notes = []

    def add(t, tt, plane, bs, a_vals, l_vals, x4=0, y4=0, clip_w4=None, clip_h4=None, mode=None, reduced=0,
            want=None, past=None):
        blk, eob = ctx_block(rng, t, tt, is32)
        if mode is None:
            mode = int(rng.integers(0, 13)) if plane == 0 else int(rng.integers(0, 14))
        above, left = noise_window(rng), noise_window(rng)
        above[plane, x4:x4 + len(a_vals)] = a_vals
        left[plane, y4:y4 + len(l_vals)] = l_vals
        if past is not None:  # entries just past the clip, which would change the contexts if read
            above[plane, x4 + len(a_vals):x4 + (1 << (WL[t] - 2))] = past
            left[plane, y4 + len(l_vals):y4 + (1 << (HL[t] - 2))] = past
        b.add_chain([K.item(b.add_block(blk), eob, t, tt, plane=plane, bsize=bs, mode=mode, reduced=reduced, x4=x4,
                            y4=y4, clip_w4=clip_w4, clip_h4=clip_h4)],
                    snapshot=int(rng.integers(0, len(b.cdfs))), above=above, left=left)
        notes.append(want)

    def luma_type(t):
        return int(rng.choice(K.INV_SET[K.tx_set(t, 0, 0)]))

    sign_pools = [(0,), (0, 64), (0, 128), (0, 64, 128), (0, 192), (64, 128, 192)]
    k = 0
    for txs, sizes in SIZES_BY_TXS.items():
        for t in sizes:  # context 0: the transform is the plane block
            w4, h4 = 1 << (WL[t] - 2), 1 << (HL[t] - 2)
            add(t, luma_type(t), 0, K.bsize_of(1 << WL[t], 1 << HL[t]), entries(4, w4, MAG_ZERO, rng),
                entries(63, h4, MAG_ZERO, rng), x4=16 - w4, y4=16 - h4, want=0)
        for top in (0, 1, 3, 4, 63):
            for lft in (0, 1, 3, 4, 63):
                t = sizes[k % len(sizes)]
                bigs = bigger_bsizes(t)
                bs = bigs[k % len(bigs)]
                w4, h4 = 1 << (WL[t] - 2), 1 << (HL[t] - 2)
                pool = sign_pools[k % len(sign_pools)]
                x4, y4 = (0, 0) if k % 2 else (16 - w4, 16 - h4)
                mx, mn = min(top | lft, 4), min(top, lft, 4)
                want = 1 if not mx else (2 + (mx > 3)) if not mn else 4 if mx <= 3 else 5 if mn <= 3 else 6
                add(t, luma_type(t), 0, bs, entries(top, w4, pool, rng), entries(lft, h4, pool, rng), x4=x4, y4=y4,
                    want=want)
                k += 1
        for bigger in (0, 1):  # chroma: 7 + (top != 0) + (left != 0), + 3 when the plane block is larger
            for a_nz in (0, 1):
                for l_nz in (0, 1):
                    for rep in range(2):
                        t = sizes[k % len(sizes)]
                        bigs = bigger_bsizes(t)
                        bs = bigs[k % len(bigs)] if bigger else K.bsize_of(1 << WL[t], 1 << HL[t])
                        w4, h4 = 1 << (WL[t] - 2), 1 << (HL[t] - 2)
                        nz = [1, 64, 128, 192, 255, 63 | 128][k % 6]
                        av = [0] * w4
                        lv = [0] * h4
                        if a_nz:
                            av[k % w4] = nz
                        if l_nz:
                            lv[(k + 1) % h4] = [64, 192, 3, 128 | 7][k % 4]
                        x4, y4 = (0, 0) if rep else (16 - w4, 16 - h4)
                        add(t, int(rng.integers(0, 16)), 1 + (k % 2), bs, av, lv, x4=x4, y4=y4,
                            want=7 + 3 * bigger + a_nz + l_nz)
                        k += 1
    # frame-clipped reads: zeros inside the clip, entries past it that would change both contexts
    for t in (1, 2, 3, 4, 7, 8, 9, 10, 11, 12, 17, 18):
        w4, h4 = 1 << (WL[t] - 2), 1 << (HL[t] - 2)
        for plane in (0, 1):
            cw4, ch4 = max(1, w4 // 2), max(1, h4 - 1)
            bs = bigger_bsizes(t)[0]
            add(t, luma_type(t) if plane == 0 else int(rng.integers(0, 16)), plane, bs, [0] * cw4, [0] * ch4,
                x4=16 - w4, y4=0, clip_w4=cw4, clip_h4=ch4, past=128 | 9, want=1 if plane == 0 else 10)
    # plane sizes 13..15 around the 64-point transforms
    for t in (4, 11, 12, 17, 18):
        w4, h4 = 1 << (WL[t] - 2), 1 << (HL[t] - 2)
        for bs in (13, 14, 15):
            for plane in (0, 2):
                add(t, 0 if plane == 0 else int(rng.integers(0, 16)), plane, bs, entries(3, w4, (0, 64), rng),
                    entries(0, h4, (0,), rng), want=2 if plane == 0 else 11)
    return b.arrays(), notes


def eob_cases(is32, seed=32):
    """Section 2: every eob group at its first and last eob, for every size and scan class, plus the
    last-position thresholds and DCT-only luma sets with other types."""
    rng = np.random.default_rng(seed)
    b = K.Batch(snapshots(rng), is32)

    def add(t, tt, plane, eob):
        blk = K.make_block(rng, t, tt, eob, is32)
        if plane == 0:
            mode, reduced = luma_setup(t, tt)
        else:
            mode, reduced = int(rng.integers(0, 14)), 0
        b.add_chain([K.item(b.add_block(blk), eob, t, tt, plane=plane, mode=mode, reduced=reduced)],
                    snapshot=int(rng.integers(0, len(b.cdfs))), above=noise_window(rng), left=noise_window(rng))

    for t in range(19):
        area = area_of(t)
        for ci, tt in enumerate((0, 10, 11)):
            for g, (lo, hi) in enumerate(EOB_GROUPS):
                if lo > area:
                    break
                for j, eob in enumerate(sorted({lo, min(hi, area)})):
                    add(t, tt, (0, 1, 2)[(g + ci + j) % 3], eob)
            for eob in (area // 8 + 1, area // 8 + 2, area // 4 + 1, area // 4 + 2):
                add(t, tt, (0, 1)[(t + ci) % 2], eob)
                add(t, tt, (1, 0)[(t + ci) % 2], eob)
    for t in (4, 11, 12, 17, 18, 3, 9, 10, 15, 16):  # DCT-only luma sets (intra, and inter for 64-point) with tt != 0
        for tt in (1, 5, 8, 14):
            add(t, tt, 0, int(rng.integers(1, area_of(t) + 1)))
    return b.arrays()


LEVELS = (1, 2, 3, 14, 15, 16, 127, 128)


def golomb_levels(is32):
    top = 30 if is32 else 14
    lv = sorted({14 + (1 << k) - 1 for k in range(1, top + 1)} | {14 + (1 << k) for k in range(top + 1)})
    return lv + [(1 << 31) - 1 if is32 else 32767]


def magnitude_cases(is32, seed=33, i16_values=False):
    """Section 3: base / br / golomb borders, 127-capped neighbourhoods and every golomb length, each value
    with both signs and with a zero, negative and positive DC.  i16_values: only values an i16 holds."""
    rng = np.random.default_rng(seed)
    b = K.Batch(snapshots(rng), is32)
    big = is32 and not i16_values

    def add(t, tt, vals, plane=0, tail=()):
        area = area_of(t)
        scan = K.scan_order(t, tt)
        blk = np.zeros(area, np.int64)
        blk[scan[:len(vals)]] = vals
        for c, v in tail:
            blk[scan[c]] = v
        eob = len(vals)
        while blk[scan[eob - 1]] == 0:
            eob -= 1
        mode, reduced = luma_setup(t, tt) if plane == 0 else (0, 0)
        b.add_chain([K.item(b.add_block(blk), eob, t, tt, plane=plane, mode=mode, reduced=reduced)],
                    snapshot=int(rng.integers(0, len(b.cdfs))), above=noise_window(rng), left=noise_window(rng))

    k = 0
    for lv in LEVELS + tuple(golomb_levels(big)):
        for dc in (0, -1, 1):
            t, tt = [(1, 0), (0, 10), (2, 11), (7, 0), (5, 10)][k % 5]
            plane = k % 2
            vals = [dc * lv, lv, -lv, int(rng.integers(0, 4)), -lv if k % 3 else lv]
            vals += [int(rng.choice([0, 1, -2, 3, lv, -lv])) for _ in range(k % 7)] + [lv * (1 - 2 * (k & 1))]
            add(t, tt, vals, plane=plane)
            k += 1
    for t, tt in ((0, 0), (1, 10), (2, 0), (3, 0), (7, 11)):  # 127-capped neighbourhoods (levels read as 127)
        area = area_of(t)
        hi = (1 << 31) - 1 if big else 32767
        vals = rng.integers(127, 300, area)
        far = rng.random(area) < 0.1
        vals[far] = rng.integers(128, hi, int(far.sum()), endpoint=True)
        add(t, tt, list(vals * rng.choice([-1, 1], area)), plane=t % 2)
    return b.arrays()


def wrap_cases(seed=34):
    """i32 blocks whose scan-order magnitudes up to eob sum to 2^32 + k: cul_level keeps the u32 sum's k (plus
    the DC's sign bits), and the next block of the chain reads that byte in its txb_skip and dc_sign contexts."""
    rng = np.random.default_rng(seed)
    b = K.Batch(snapshots(rng), 1)
    m = (1 << 31) - 1
    for k in range(4):
        for plane, t, bs in ((0, 0, K.bsize_of(16, 16)), (1, 1, K.bsize_of(32, 32)), (0, 2, K.bsize_of(32, 32))):
            scan = K.scan_order(t, 0)
            blk = np.zeros(area_of(t), np.int64)
            dc = [m, -m, 0, 2 + k][k]
            rest = {0: [-m, 2 + k], 1: [m, 2 + k], 2: [m, -m, -(2 + k)], 3: [m, -m]}[k]
            vals = [dc] + rest
            blk[scan[:len(vals)]] = vals
            blk[scan[len(vals) + 3]] = 77  # past eob: not in the sum
            nxt = K.make_block(rng, t, 0, 6, 1)
            items = [K.item(b.add_block(blk), len(vals), t, 0, plane=plane, bsize=bs),
                     K.item(b.add_block(nxt), 6, t, 0, plane=plane, bsize=bs)]
            b.add_chain(items, snapshot=int(rng.integers(0, len(b.cdfs))))
    return b.arrays()


# ---------------------------------------------------------------- section 4: CDF regions
def region_items(b, rng, is32):
    """Groups of items that share CDF rows across sizes, planes, intra / inter and reduced sets."""
    def it(t, tt, plane=0, mode=0, reduced=0, eob=None, x4=0, y4=0, bs=None):
        area = area_of(t)
        eob = eob or int(rng.integers(max(2, area // 8), area + 1))
        blk = K.make_block(rng, t, tt, eob, is32, zero_frac=0.2)
        return K.item(b.add_block(blk), eob, t, tt, plane=plane, bsize=bs, mode=mode, reduced=reduced, x4=x4, y4=y4)

    g = {}
    g["br_txs3_4"] = [it(3, 0), it(4, 0), it(11, 0, eob=500), it(3, 0), it(3, 0, plane=1), it(4, 0, plane=2)]
    g["br_txs4_3"] = [it(4, 0, plane=1), it(3, 5, plane=2), it(12, 0), it(9, 0)]
    g["eob1024"] = [it(t, 0, plane=p) for p in (0, 1) for t in (3, 11, 12, 4, 17, 18)] + [it(3, 10, plane=1),
                                                                                          it(4, 11, plane=2)]
    g["eob_area"] = [it(1, 0), it(13, 0), it(14, 0), it(7, 0), it(8, 0), it(1, 10, plane=1), it(13, 11, plane=2),
                     it(5, 0, plane=1), it(6, 0, plane=2)]
    intra = []
    for m in (0, 5, 12):
        intra += [it(t, tt, mode=m) for t, tt in ((0, 10), (5, 3), (6, 11), (13, 1), (14, 0))]  # intra_tx_1[0][m]
        intra += [it(t, tt, mode=m) for t, tt in ((1, 2), (7, 11), (8, 9))]                       # intra_tx_1[1][m]
        intra += [it(t, tt, mode=m, reduced=1) for t, tt in ((0, 3), (6, 9), (1, 1), (8, 0))]     # intra_tx_2[0/1]
        intra += [it(2, 3, mode=m), it(2, 9, mode=m, reduced=1)]                                  # intra_tx_2[2][m]
    g["intra_rows"] = intra
    N = K.NEARESTMV
    g["inter_rows"] = ([it(t, tt, mode=N + 3) for t, tt in ((0, 15), (5, 12), (6, 0), (13, 7), (14, 10))] +
                       [it(t, tt, mode=N + 9) for t, tt in ((1, 13), (7, 4), (8, 11))] +
                       [it(2, 8, mode=N), it(2, 10, mode=N + 1)] +
                       [it(t, tt, mode=N + 2, reduced=1) for t, tt in ((0, 9), (5, 0), (1, 9), (2, 0))] +
                       [it(15, 9, mode=N), it(16, 0, mode=N + 5), it(9, 9, mode=N), it(10, 0, mode=N + 4),
                        it(3, 9, mode=N + 6), it(3, 0, mode=N + 7)])
    g["planes_1_2"] = [it(1, 4, plane=1), it(1, 12, plane=2), it(2, 0, plane=2), it(2, 7, plane=1),
                       it(0, 0, plane=2, x4=1), it(0, 5, plane=1, x4=1)]
    g["intra_inter_reduced"] = [it(1, 0, mode=3), it(1, 0, mode=N + 1), it(1, 9, mode=4, reduced=1),
                                it(1, 10, mode=N + 2), it(1, 9, mode=N, reduced=1), it(1, 11, mode=3),
                                it(1, 0, plane=1)]
    for name in list(g):  # each row adapted by one member is read by another: the group again, reversed
        g[name] = g[name] + g[name][::-1]
    return g


def all_region_items(b, rng, is32):
    """Items that code every region a valid item can select."""
    def it(t, tt, plane=0, mode=0, reduced=0):
        area = area_of(t)
        eob = int(rng.integers(max(2, area // 16), max(3, area // 3)))
        blk = K.make_block(rng, t, tt, eob, is32, zero_frac=0.2)
        scan = K.scan_order(t, tt)
        blk[scan[0]] = int(rng.choice([-5, 4, 9]))  # a br symbol and a dc_sign in every item
        return K.item(b.add_block(blk), eob, t, tt, plane=plane, mode=mode, reduced=reduced)

    N = K.NEARESTMV
    items = []
    for m in range(13):
        items += [it(0, 10, mode=m), it(1, 11, mode=m)]                              # intra_tx_1, sq 0 / 1
        items += [it(0, 3, mode=m, reduced=1), it(1, 1, mode=m, reduced=1), it(2, 2, mode=m)]  # intra_tx_2 sq 0-2
    items += [it(0, 12, mode=N), it(1, 14, mode=N + 1), it(2, 4, mode=N + 2)]         # inter_tx_1 sq 0-1, inter_tx_2
    items += [it(0, 9, mode=N, reduced=1), it(1, 0, mode=N, reduced=1), it(2, 9, mode=N, reduced=1),
              it(3, 9, mode=N + 3)]                                                   # inter_tx_3 sq 0-3
    for t in (0, 1, 2, 3, 4):                                                         # every (txs_ctx, ptype)
        items += [it(t, 0, mode=m % 13) for m in range(1)] + [it(t, 6, plane=1), it(t, 0, plane=2)]
    for t in (0, 5, 1, 7, 2, 9, 3):                                                   # every eob_flag row
        for plane in (0, 1):
            for tt in (0, 10):
                if plane == 0 and tt == 10:
                    mode, reduced = luma_setup(t, tt)
                    items.append(it(t, tt, mode=mode, reduced=reduced))
                else:
                    items.append(it(t, tt, plane=plane))
    return items


def every_region():
    """The regions of the contract's CDF layout a valid item can select."""
    r = {("txb_skip", s) for s in range(5)} | {("dc_sign", p, d) for p in range(2) for d in range(3)}
    for s in range(5):
        for p in range(2):
            r |= {("eob_extra", s, p), ("coeff_base_eob", s, p), ("coeff_base", s, p)}
    r |= {("coeff_br", s, p) for s in range(4) for p in range(2)}
    r |= {("intra_tx_1", sq, m) for sq in range(2) for m in range(13)}
    r |= {("intra_tx_2", sq, m) for sq in range(3) for m in range(13)}
    r |= {("inter_tx_1", 0), ("inter_tx_1", 1), ("inter_tx_2", 2)} | {("inter_tx_3", sq) for sq in range(4)}
    r |= {("eob_flag%d" % (16 << m), p, c) for m in range(7) for p in range(2) for c in range(2)}
    return r


def count_snapshot(base, cnt):
    s = base.copy()
    for name in COEFF_CDFS_DTYPE.names:
        s[name][..., -1] = cnt
    return s


def saturated_snapshot(base, rng):
    """Rows adaptation can produce at its limits: equal adjacent values, entries at 0 and near 32767."""
    s = base.copy()
    for name in COEFF_CDFS_DTYPE.names:
        a = s[name]
        rows = a.reshape(-1, a.shape[-1])
        n = rows.shape[1] - 1
        for i, r in enumerate(rows):
            kind = i % 4
            if kind == 0:
                r[:n] = 0
            elif kind == 1:
                r[:n] = 32767
            elif kind == 2 and n > 1:
                r[:n] = np.sort(np.repeat(rng.integers(1, 32767, (n + 1) // 2), 2)[:n])[::-1]
            else:
                r[:n] = [32767 - j if j < n // 2 else 0 for j in range(n)]
            r[n] = int(rng.choice([0, 31, 32]))
        s[name] = rows.reshape(a.shape)
    return s


def region_cases(is32, seed=35, poison=False):
    """Section 4: chains named by what they share.  Returns (arrays, names).  poison: one more chain, last,
    that codes every region three times from a snapshot no other chain uses."""
    rng = np.random.default_rng(seed)
    cdfs = snapshots(rng)
    cdfs = np.concatenate([cdfs] + [count_snapshot(cdfs[0:1], c) for c in (0, 15, 16, 31, 32)] +
                          [saturated_snapshot(cdfs[1:2], rng)] + ([K.random_cdfs(rng, 1)] if poison else []))
    b = K.Batch(cdfs, is32)
    names = []
    for name, items in region_items(b, rng, is32).items():
        for snap in (0, int(rng.integers(1, 4))):
            b.add_chain(items, snapshot=snap, init_rng=int(rng.integers(32768, 65536)))
            names.append(name)
    every = all_region_items(b, rng, is32)
    sat = len(cdfs) - 1 - poison
    for snap in range(sat + 1):
        b.add_chain(every + every, snapshot=snap)
        names.append("every_region_twice")
    for rng0 in (32768, 65535):
        b.add_chain(every, snapshot=sat, init_rng=rng0)
        names.append("saturated")
    long_items = []
    for i in range(2000):
        t = int(rng.choice([0, 0, 1, 5, 6]))
        plane = int(rng.integers(0, 3))
        tt = int(rng.choice(K.INV_SET[K.tx_set(t, 0, 0)])) if plane == 0 else int(rng.integers(0, 16))
        eob = int(rng.choice([0, 1, 2, 3, 5, 9, area_of(t)]))
        blk = K.make_block(rng, t, tt, eob, is32)
        w4, h4 = 1 << (WL[t] - 2), 1 << (HL[t] - 2)
        long_items.append(K.item(b.add_block(blk), eob, t, tt, plane=plane, mode=int(rng.integers(0, 13)),
                                 bsize=K.bsize_of(16, 16), x4=(i * w4) % (16 - w4 + 1),
                                 y4=(i * 3 * h4) % (16 - h4 + 1)))
    for snap, rng0 in ((5, 32768), (sat, 65535)):
        b.add_chain(long_items, snapshot=snap, init_rng=rng0)
        names.append("long")
    if poison:
        b.add_chain(all_region_items(b, rng, is32) * 3, snapshot=len(cdfs) - 1, init_rng=33333)
        names.append("poison")
    return b.arrays(), names


# ---------------------------------------------------------------- CPU: reach of every section
def all_records(tr):
    return [r for recs, _, _, _ in tr for r in recs]


def valid(rate):
    return (np.asarray(rate) != INV).all()


def test_contexts_reach_every_txb_skip_and_dc_sign_context():
    (cdfs, chains, items, q), notes = context_cases(0)
    tr = trace_all(chains, items, q, contexts=False)
    reached = set()
    for (recs, _, _, _), want in zip(tr, notes):
        r = recs[0]
        if want is not None:
            assert r["skip"] == want, (r, want)
        reached.add((r["ptype"], r["txs"], r["skip"]))
    assert {(0, s, c) for s in range(5) for c in range(7)} <= reached
    assert {(1, s, c) for s in range(5) for c in range(7, 13)} <= reached
    dcs = {(r["ptype"], r["dc_ctx"]) for r in all_records(tr)}
    assert {(p, d) for p in range(2) for d in range(3)} <= dcs
    # luma: the exact-3 OR against 0 (2) and >= 4 against 0 (3), as the issue's weakest border
    assert {(0, s, 2) for s in range(5)} <= reached and {(0, s, 3) for s in range(5)} <= reached
    # window bytes with sign fields 1, 2 and 3 and zero magnitude are read
    bytes_read = set()
    for ch, it in zip(chains, items):
        p = int(it["plane"])
        bytes_read |= set(ch["above"][p][int(it["x4"]):int(it["x4"]) + int(it["clip_w4"])].tolist())
    assert {64, 128, 192} <= bytes_read and any(v > 192 for v in bytes_read)
    # clipped reads: reading the whole tx width would change a context; windows at 16 - width_mi
    clipped = [(ch, it) for ch, it in zip(chains, items) if it["clip_w4"] < 1 << (WL[int(it["tx_size"])] - 2)]
    assert len(clipped) >= 20
    for ch, it in clipped:
        full = it.copy()
        full["clip_w4"], full["clip_h4"] = 1 << (WL[int(it["tx_size"])] - 2), 1 << (HL[int(it["tx_size"])] - 2)
        assert skip_dc_ctx(ch["above"], ch["left"], full) != skip_dc_ctx(ch["above"], ch["left"], it)
    assert all(any(int(it["x4"]) == 16 - (1 << (WL[t] - 2)) for it in items if int(it["tx_size"]) == t)
               for t in range(19))
    assert {13, 14, 15} <= {int(it["plane_bsize"]) for it in items if int(it["tx_size"]) in (4, 11, 12, 17, 18)}
    rate, cul = K.oracle_rate(cdfs, chains, items, q)
    assert valid(rate)
    np.testing.assert_array_equal(cul, [r["cul"] for r in all_records(tr)])


def test_sign_field_3_adds_nothing_to_dc_ctx():
    """A window byte of 192..255 counts as no sign; luma reads its magnitude bits, chroma counts it non-zero."""
    rng = np.random.default_rng(5)
    blk = K.make_block(rng, 1, 0, 7, 0)
    blk[0] = 9
    out = {}
    for plane in (0, 1):
        for a0 in (0, 192, 192 | 5, 5):
            b = K.Batch(K.default_cdfs(), 0)
            ab, lf = np.zeros((3, 16), np.uint8), np.zeros((3, 16), np.uint8)
            ab[plane, 0], lf[plane, 0] = a0, 64
            b.add_chain([K.item(b.add_block(blk), 7, 1, 0, plane=plane, bsize=K.bsize_of(16, 16))], above=ab, left=lf)
            out[plane, a0] = K.oracle_rate(*b.arrays())[0][0]
    assert out[0, 0] == out[0, 192] and out[0, 5] == out[0, 192 | 5] and out[0, 0] != out[0, 5]
    assert out[1, 192] == out[1, 5] == out[1, 192 | 5]


def test_eob_cases_reach_every_group_and_threshold():
    cdfs, chains, items, q = eob_cases(0)
    recs = all_records(trace_all(chains, items, q, contexts=False))
    for t in range(19):
        area = area_of(t)
        for cls in range(3):
            mine = [r for r in recs if r["t"] == t and r["cls"] == cls]
            groups = {g + 1 for g, (lo, _) in enumerate(EOB_GROUPS) if lo <= area}
            assert {r["eob_pt"] for r in mine} == groups, (t, cls)
            firsts = {r["eob"] for r in mine}
            assert {lo for lo, _ in EOB_GROUPS if lo <= area} <= firsts
            assert {min(hi, area) for lo, hi in EOB_GROUPS if lo <= area} <= firsts
            assert {0, 1} <= {r["top_bit"] for r in mine if r["eob_pt"] >= 3} or area < 3
            assert {area // 8 + 1, area // 8 + 2, area // 4 + 1, area // 4 + 2} <= firsts
            assert {r["last_ctx"] for r in mine} == {0, 1, 2, 3}
    # 64-point sizes code their 32x32 / 16x32 area with eob_flag1024 / eob_flag512
    for t in (4, 11, 12, 17, 18):
        assert max(r["eob"] for r in recs if r["t"] == t) == area_of(t)
    dct_only_other = [r for r, it in zip(recs, items) if r["plane"] == 0 and int(it["tx_type"]) not in (0, 10, 11)]
    assert {4, 11, 12, 17, 18, 3, 9, 10, 15, 16} <= {r["t"] for r in dct_only_other}
    rate, cul = K.oracle_rate(cdfs, chains, items, q)
    assert valid(rate)
    np.testing.assert_array_equal(cul, [r["cul"] for r in recs])


@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_magnitude_cases_reach_every_golomb_length(is32):
    cdfs, chains, items, q = magnitude_cases(is32)
    recs = all_records(trace_all(chains, items, q, contexts=False))
    lens = {g for r in recs for g in r["golomb"]}
    assert lens == set(range(1, (31 if is32 else 15) + 1))
    mags = {abs(int(v)) for v in q}
    assert set(LEVELS) <= mags and set(golomb_levels(is32)) <= mags
    assert {r["dc_ctx"] is None for r in recs} == {True, False}
    assert {None, 0, 1, 2} >= {r["dc_ctx"] for r in recs}
    rate, cul = K.oracle_rate(cdfs, chains, items, q)
    assert valid(rate)
    np.testing.assert_array_equal(cul, [r["cul"] for r in recs])


def test_i16_values_as_i32_give_the_same_rates():
    cdfs, chains, items, q = magnitude_cases(0)
    a = K.oracle_rate(cdfs, chains, items, q)
    b = K.oracle_rate(cdfs, chains, items, q.astype(np.int32))
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])


def test_wrap_cases_sum_to_2_32_plus_k():
    cdfs, chains, items, q = wrap_cases()
    tr = trace_all(chains, items, q)
    firsts = [recs[0] for recs, _, _, _ in tr]
    assert sorted({r["cul_sum"] for r in firsts}) == [0, 1, 2, 3]
    for r in firsts:
        assert r["cul"] & 63 == r["cul_sum"]
    rate, cul = K.oracle_rate(cdfs, chains, items, q)
    assert valid(rate)
    np.testing.assert_array_equal(cul, [r["cul"] for r in all_records(tr)])
    # the byte the next block reads is k, not 63: a saturated sum would give the luma blocks other contexts
    for ch, (recs, _, _, _) in zip(chains, tr):
        if recs[1]["plane"]:
            continue
        nxt = items[int(ch["item_begin"]) + 1]
        win = np.zeros((3, 16), np.uint8)
        win[0, :] = (recs[0]["cul"] & 0xC0) | 63
        assert skip_dc_ctx(win, win, nxt)[0] != recs[1]["skip"]


@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_region_cases_reach_every_region_and_share_rows(is32):
    (cdfs, chains, items, q), names = region_cases(is32)
    tr = trace_all(chains, items, q, contexts=False)
    every = every_region()
    for (recs, syms, regions, _), name in zip(tr, names):
        if name == "every_region_twice":
            assert every <= regions, sorted(every - regions)
    # each sharing pair: one row coded by items that differ in size, plane or type
    users = {}
    for (recs, syms, regions, _), ch in zip(tr, chains):
        b0 = int(ch["item_begin"])
        for k, r in enumerate(recs):
            it = items[b0 + k]
            key = (r["t"], r["plane"], int(it["mode"]) >= K.NEARESTMV, int(it["reduced_tx_set"]), int(it["tx_type"]))
            for reg in trace_chain_item_regions(r, it):
                users.setdefault(reg, set()).add(key)
    assert len({u[0] for u in users[("coeff_br", 3, 0)]} & {3, 4, 11, 12, 17, 18}) >= 4
    assert {0, 1} <= {u[1] > 0 for u in users[("coeff_br", 3, 1)]} | {0, 1}
    assert {3, 11, 12, 4, 17, 18} <= {u[0] for u in users[("eob_flag1024", 0, 0)]}
    assert {0, 5, 6, 13, 14} <= {u[0] for u in users[("intra_tx_1", 0, 0)]}
    assert {1, 7, 8} <= {u[0] for u in users[("intra_tx_1", 1, 5)]}
    assert len(users[("intra_tx_2", 2, 12)]) >= 2 and len(users[("intra_tx_2", 0, 0)]) >= 2
    assert {1, 2} <= {u[1] for u in users[("dc_sign", 1, 0)] | users[("dc_sign", 1, 1)] | users[("dc_sign", 1, 2)]}
    assert {False, True} <= {u[2] for u in users[("coeff_base", 1, 0)]}
    assert {0, 1} <= {u[3] for u in users[("coeff_base", 1, 0)]}
    assert {0, 1, 2} <= {u[1] for u in users[("coeff_br", 3, 0)] | users[("coeff_br", 3, 1)]}
    assert len({u[0] for u in users[("inter_tx_3", 2)]}) >= 3 and len({u[0] for u in users[("inter_tx_1", 0)]}) >= 5
    # the long chain: ~2000 items whose rows adapt past count 32
    li = names.index("long")
    assert int(chains[li]["item_count"]) >= 2000
    long = trace_chain(chains[li], items, q)[1]
    assert sum(1 for v in long.values() if v >= 32) >= 40
    assert {0, 15, 16, 31, 32} <= {int(cdfs[s]["txb_skip"][0, 0, 1]) for s in chains["snapshot"]}
    rate, cul = K.oracle_rate(cdfs, chains, items, q)
    assert valid(rate)


def trace_chain_item_regions(rec, it):
    """The regions one traced item selected (for the sharing assertions)."""
    t, txs, ptype = rec["t"], rec["txs"], rec["ptype"]
    r = {("txb_skip", txs)}
    if rec["eob"]:
        r |= {("eob_flag%d" % (16 << min(WL[t] + HL[t] - 4, 6)), ptype, int(rec["cls"] != 0)),
              ("coeff_base", txs, ptype)}
        if rec["br"]:
            r.add(("coeff_br", min(txs, 3), ptype))
        if rec["dc_ctx"] is not None:
            r.add(("dc_sign", ptype, rec["dc_ctx"]))
        if rec["plane"] == 0:
            is_inter, sq = int(it["mode"]) >= K.NEARESTMV, min(WL[t], HL[t]) - 2
            st = K.tx_set(t, is_inter, int(it["reduced_tx_set"]))
            if len(K.INV_SET[st]) > 1:
                r.add(({5: "inter_tx_1", 4: "inter_tx_2", 1: "inter_tx_3"}[st], sq) if is_inter else
                      ({3: "intra_tx_1", 2: "intra_tx_2"}[st], sq, int(it["mode"])))
    return r


# ---------------------------------------------------------------- CPU: the footprint restatement on the oracle
def footprint(chains, items, q):
    """What a call may read, per the contract: the coded blocks and items of valid chains, the snapshot rows
    their symbols select, and the window entries read before the chain writes them."""
    tr = trace_all(chains, items, q)
    ncdf = COEFF_CDFS_DTYPE.itemsize // 2
    cdf_keep = np.zeros((int(chains["snapshot"].max()) + 1 if len(chains) else 1, ncdf), bool)
    item_keep = np.zeros(len(items), bool)
    q_keep = np.zeros(len(q), bool)
    win_keep = np.zeros((len(chains), 2, 3, 16), bool)
    for ci, (ch, (recs, syms, _, wr)) in enumerate(zip(chains, tr)):
        b0, n = int(ch["item_begin"]), int(ch["item_count"])
        item_keep[b0:b0 + n] = True
        for it in items[b0:b0 + n]:
            a = area_of(int(it["tx_size"]))
            q_keep[int(it["block"]) * a:(int(it["block"]) + 1) * a] = True
        for name, idx in syms:
            s, ln = row_span(name, idx)
            cdf_keep[int(ch["snapshot"]), s:s + ln] = True
        for side, p, i in wr:
            win_keep[ci, side, p, i] = True
    return tr, cdf_keep, item_keep, q_keep, win_keep


def scrambled(cdfs, chains, items, q, fp, seed):
    """Copies with every byte outside the footprint replaced."""
    _, cdf_keep, item_keep, q_keep, win_keep = fp
    rng = np.random.default_rng(seed)
    c2 = cdfs.copy().view(np.uint16).reshape(len(cdfs), -1)
    keep = np.zeros(c2.shape, bool)
    keep[:cdf_keep.shape[0]] = cdf_keep
    c2[~keep] = rng.integers(0, 1 << 16, int((~keep).sum()))
    ch2 = chains.copy()
    for ci in range(len(ch2)):
        for side, f in ((0, "above"), (1, "left")):
            w = ch2[ci][f]
            w[~win_keep[ci, side]] = rng.integers(0, 256, int((~win_keep[ci, side]).sum()))
            ch2[ci][f] = w
    it2 = items.copy()
    raw = it2.view(np.uint8).reshape(len(it2), -1)
    raw[~item_keep] = rng.integers(0, 256, raw[~item_keep].shape)
    q2 = q.copy()
    info = np.iinfo(q.dtype)
    q2[~q_keep] = rng.integers(info.min, info.max, int((~q_keep).sum()), endpoint=True)
    return c2.view(COEFF_CDFS_DTYPE).reshape(-1), ch2, it2, q2


def footprint_fixture(is32):
    """Valid chains of sections 1, 3 and 4 in one call, over one coefficient buffer, plus unused items and
    snapshots."""
    (cdfs, chains, items, q), _ = region_cases(is32, seed=40)
    keep = np.zeros(len(chains), bool)
    keep[::3] = True
    keep[-1] = True  # the long chain
    rng = np.random.default_rng(41)
    extra = K.random_cdfs(rng, 2)
    return np.concatenate([cdfs, extra]), chains[keep], items, q


@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_footprint_restatement_pinned_on_the_oracle(is32):
    cdfs, chains, items, q = footprint_fixture(is32)
    fp = footprint(chains, items, q)
    want = K.oracle_rate(cdfs, chains, items, q)
    assert valid(want[0])
    assert not fp[2].all() and not fp[3].all()  # unused items and coefficients are part of the scramble
    for seed in (1, 2):
        got = K.oracle_rate(*scrambled(cdfs, chains, items, q, fp, seed))
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1][fp[2]], want[1][fp[2]])
    # the check has teeth: replacing one coded row changes that chain's rate
    rng = np.random.default_rng(3)
    for ci in rng.choice(len(chains), 6, replace=False):
        syms = fp[0][ci][1]
        name, idx = sorted(syms)[int(rng.integers(0, len(syms)))]
        c2 = cdfs.copy()
        s, ln = row_span(name, idx)
        flat = c2.view(np.uint16).reshape(len(c2), -1)
        snap = int(chains[ci]["snapshot"])
        n = ln - 1
        flat[snap, s:s + n] = np.sort(rng.choice(np.arange(1, 512), n, replace=False))[::-1] * 64 if n > 0 else []
        flat[snap, s + n] = 31 - int(flat[snap, s + n]) % 32
        got = K.oracle_rate(c2, chains, items, q)[0]
        assert got[ci] != want[0][ci], (name, idx)


# ---------------------------------------------------------------- device
def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev_run(cdfs, chains, items, q, cul=True, offset=False, ncoeffs=None, check_inputs=True):
    """One b200_coeff_rate_dev call.  offset: every buffer at one element past an aligned address (d_cdfs at 2
    bytes).  Sentinels past d_rate[nchains] and d_cul_level[nitems] are checked untouched."""
    import torch

    from tests import gpu_util as G
    c = G.ctx()
    is32 = int(q.dtype == np.int32)

    def place(a, off):
        raw = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        t = torch.zeros(raw.size + off + 16, dtype=torch.uint8, device="cuda")
        t[off:off + raw.size] = torch.from_numpy(raw).cuda()
        return t, t[off:]

    qoff = q.dtype.itemsize if offset else 0
    bufs = [place(a, o) for a, o in ((cdfs, 2 if offset else 0), (chains, 0), (items, 0), (q, qoff))]
    before = [t.clone() for t, _ in bufs]
    n, m = len(chains), len(items)
    d_rate = torch.full((n + 4,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    d_cul = torch.full((m + 8,), 0xEE, dtype=torch.uint8, device="cuda") if cul else None
    c.coeff_rate_dev(bufs[0][1], len(cdfs), bufs[1][1], n, bufs[2][1], m, bufs[3][1],
                     len(q) if ncoeffs is None else ncoeffs, is32, d_rate, d_cul)
    c.synchronize()
    if check_inputs:
        for (t, _), b in zip(bufs, before):
            assert torch.equal(t, b), "an input changed"
    rate = d_rate.cpu().numpy().view(np.uint32)
    assert (rate[n:] == 0x5A5A5A5A).all(), "d_rate written past nchains"
    if not cul:
        return rate[:n], None
    cb = d_cul.cpu().numpy()
    assert (cb[m:] == 0xEE).all(), "d_cul_level written past nitems"
    return rate[:n], cb[:m]


def assert_oracle(cdfs, chains, items, q, **kw):
    want, want_cul = K.oracle_rate(cdfs, chains, items, q)
    got, got_cul = dev_run(cdfs, chains, items, q, **kw)
    np.testing.assert_array_equal(got, want)
    if got_cul is not None:
        np.testing.assert_array_equal(got_cul, want_cul)
    return want, want_cul


@gpu
@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_contexts_on_device(is32):
    arrays, _ = context_cases(is32)
    assert valid(assert_oracle(*arrays)[0])


@gpu
@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_eob_groups_on_device(is32):
    assert valid(assert_oracle(*eob_cases(is32))[0])


@gpu
@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_magnitudes_on_device(is32):
    assert valid(assert_oracle(*magnitude_cases(is32))[0])


@gpu
def test_i16_values_carried_as_i32_on_device():
    cdfs, chains, items, q = magnitude_cases(0)
    a = dev_run(cdfs, chains, items, q)
    b = dev_run(cdfs, chains, items, q.astype(np.int32))
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])
    np.testing.assert_array_equal(a[0], K.oracle_rate(cdfs, chains, items, q)[0])


@gpu
def test_cul_level_sum_wraps_in_u32_on_device():
    cdfs, chains, items, q = wrap_cases()
    _, cul = assert_oracle(cdfs, chains, items, q)
    assert sorted({int(v) & 63 for v in cul[0::2]}) == [0, 1, 2, 3]


def warp_reuse_layout(chains, items, nwarps, poison):
    """Targets run on warps that first ran `poison` (a chain adapting every region from another snapshot),
    then an invalid chain, then an empty one (which copies only the regions every chain starts with, from the
    poison's snapshot): chain i of the targets is chain 3 * nwarps + i, sharing warp i.  Returns the chains and
    the targets' first index."""
    assert len(chains) <= nwarps
    empty = np.zeros((), COEFF_CHAIN_DTYPE)
    empty["snapshot"], empty["init_rng"] = poison["snapshot"], 40000
    empty["item_begin"] = len(items)  # an empty chain may start at nitems
    bad = poison.copy()
    bad["init_rng"] = 32767
    out = np.zeros(4 * nwarps, COEFF_CHAIN_DTYPE)
    out[:] = empty
    out[:len(chains)] = poison
    out[nwarps:nwarps + len(chains)] = bad
    out[3 * nwarps:3 * nwarps + len(chains)] = chains
    return out, 3 * nwarps


@gpu
@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_regions_on_reused_warps(is32):
    """Every section-4 chain on a warp whose shared CDF copy holds another snapshot's adapted rows: a region
    the chain fails to copy reads stale values."""
    (cdfs, chains, items, q), names = region_cases(is32, poison=True)
    assert names[-1] == "poison"
    poison, chains = chains[-1], chains[:-1]
    nwarps = WARPS_PER_SM * num_sms()
    layout, first = warp_reuse_layout(chains, items, nwarps, poison)
    want, _ = assert_oracle(cdfs, layout, items, q)
    assert valid(want[first:first + len(chains)]) and valid(want[:len(chains)])
    assert (want[nwarps:nwarps + len(chains)] == INV).all()
    assert (want[len(chains):nwarps] == 0).all() and (want[2 * nwarps:3 * nwarps] == 0).all()


@gpu
def test_empty_overlapping_and_out_of_order_ranges():
    rng = np.random.default_rng(60)
    b = K.Batch(snapshots(rng), 0)
    items = []
    for k in range(12):
        t = int(rng.choice([0, 1, 6]))
        eob = int(rng.integers(0, area_of(t) + 1))
        blk = K.make_block(rng, t, 0, eob, 0)
        items.append(K.item(b.add_block(blk), eob, t, 0, bsize=K.bsize_of(16, 16), x4=k % 8, y4=(3 * k) % 8,
                            plane=k % 3))
    b.add_chain(items)
    cdfs, chains, its, q = b.arrays()
    ch = []
    for begin, count in ((0, 12), (3, 5), (5, 7), (0, 4), (11, 1), (4, 0), (12, 0), (8, 4), (2, 9), (7, 3), (0, 12)):
        c = chains[0].copy()
        c["item_begin"], c["item_count"] = begin, count
        c["snapshot"], c["init_rng"] = int(rng.integers(0, 4)), int(rng.integers(32768, 65536))
        c["above"], c["left"] = noise_window(rng), noise_window(rng)
        ch.append(c)
    ch = np.array(ch, COEFF_CHAIN_DTYPE)
    want, _ = assert_oracle(cdfs, ch, its, q, cul=False)  # chains sharing an item write it different bytes
    assert valid(want) and want[5] == 0 and want[6] == 0


@gpu
def test_init_rng_sweep():
    rng = np.random.default_rng(61)
    b = K.Batch(snapshots(rng), 0)
    blk = K.make_block(rng, 1, 0, 20, 0)
    bi = b.add_block(blk)
    for r in np.linspace(32768, 65535, 257).astype(int).tolist() + [32769, 65534]:
        b.add_chain([K.item(bi, 20, 1, 0, bsize=K.bsize_of(16, 16))], snapshot=r % 4, init_rng=r,
                    above=noise_window(rng), left=noise_window(rng))
        b.add_chain([], init_rng=r)
        b.add_chain([K.item(bi, 0, 1, 0)], init_rng=r)
    cdfs, chains, items, q = b.arrays()
    want, _ = assert_oracle(cdfs, chains, items, q)
    assert valid(want) and (want[1::3] == 0).all() and len(set(want[0::3].tolist())) > 3


@gpu
@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_read_footprint_on_device(is32):
    cdfs, chains, items, q = footprint_fixture(is32)
    fp = footprint(chains, items, q)
    want, want_cul = assert_oracle(cdfs, chains, items, q)
    for seed in (1, 2):
        got, got_cul = dev_run(*scrambled(cdfs, chains, items, q, fp, seed))
        np.testing.assert_array_equal(got, want)
        np.testing.assert_array_equal(got_cul[fp[2]], want_cul[fp[2]])
        assert (got_cul[~fp[2]] == 0xEE).all()  # items in no chain keep their bytes


@gpu
@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_misaligned_base_pointers(is32):
    (cdfs, chains, items, q), _ = context_cases(is32, seed=70)
    want = K.oracle_rate(cdfs, chains, items, q)
    got = dev_run(cdfs, chains, items, q, offset=True)
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])


@gpu
@pytest.mark.parametrize("is32", [0, 1], ids=["i16", "i32"])
def test_ncoeffs_at_the_last_block(is32):
    rng = np.random.default_rng(71)
    b = K.Batch(snapshots(rng), is32)
    for t in (0, 1, 2, 3, 4, 9):
        for _ in range(2):
            eob = int(rng.integers(1, area_of(t) + 1))
            b.add_chain([K.item(b.add_block(K.make_block(rng, t, 0, eob, is32)), eob, t, 0)])
    cdfs, chains, items, q = b.arrays()
    last = max(range(len(items)), key=lambda i: (int(items[i]["block"]) + 1) * area_of(int(items[i]["tx_size"])))
    end = (int(items[last]["block"]) + 1) * area_of(int(items[last]["tx_size"]))
    assert end == len(q)
    full, _ = assert_oracle(cdfs, chains, items, q, ncoeffs=end)
    assert valid(full)
    for n in (end - 1, end - 7, end - area_of(3) // 2):  # one short, and not a multiple of any area
        want = K.oracle_rate(cdfs, chains, items, q[:n])
        got = dev_run(cdfs, chains, items, q, ncoeffs=n)
        np.testing.assert_array_equal(got[0], want[0])
        assert got[0][chains["item_begin"].tolist().index(last)] == INV
        ok = want[0] != INV
        assert ok.sum() >= len(chains) - 3
        np.testing.assert_array_equal(got[1][ok], want[1][ok])  # one item per chain


@gpu
def test_null_cul_level_gives_the_same_rates():
    (cdfs, chains, items, q), _ = region_cases(0)
    a, _ = dev_run(cdfs, chains, items, q, cul=False)
    np.testing.assert_array_equal(a, K.oracle_rate(cdfs, chains, items, q)[0])
