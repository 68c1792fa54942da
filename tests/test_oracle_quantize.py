"""CPU tests of the oracle's quantize -> dequantize -> tx-distortion chain (oracle/quantize.c).

Pinned by the reference's own tests where it has them (golden fixtures extracted by
tests/golden/make_golden.py): get_log_tx_scale (quantize/mod.rs:186-215), divu_pair == integer
division (:173-181), and the scan tables (sha256 of all 42 tables + the (TxSize, TxType) map of
scan_order.rs).  The quantizer loop itself has no stored vectors upstream: it is cross-checked
against an independent numpy/Python model and the reference's own debug assertion (eob == last
non-zero coefficient in scan order, quantize/mod.rs:349-357)."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest

from tests import oracle_lib as O

KATS = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_kats.json")))
TX_NAMES = ["TX_4X4", "TX_8X8", "TX_16X16", "TX_32X32", "TX_64X64", "TX_4X8", "TX_8X4", "TX_8X16", "TX_16X8",
            "TX_16X32", "TX_32X16", "TX_32X64", "TX_64X32", "TX_4X16", "TX_16X4", "TX_8X32", "TX_32X8",
            "TX_16X64", "TX_64X16"]               # transform/mod.rs:101-123 order


def L():
    l = O.lib()
    l.orc_get_log_tx_scale.restype = C.c_int
    l.orc_divu_pair.restype = C.c_uint32
    l.orc_divu_pair.argtypes = [C.c_uint32, C.c_void_p]
    l.orc_divu_gen.argtypes = [C.c_uint32, C.c_void_p]
    l.orc_scan_order.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    l.orc_quantize_chain_batch.restype = None
    l.orc_quantize_chain_batch.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_uint32, C.c_uint32,
                                           C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_int]
    return l


def chain(coeffs, tx_size, tx_type, dcq, acq, is_intra, threads=0):
    """coeffs: (n, area) int16 or int32 -> qcoeffs, rcoeffs, eob, tx_dist"""
    l = L()
    n = len(coeffs)
    coded = l.orc_coded_tx_area(tx_size)
    coeffs = np.ascontiguousarray(coeffs)
    q = np.full((n, coded), 77, coeffs.dtype)       # garbage: the chain zero-fills itself
    r = np.zeros((n, coded), coeffs.dtype)
    eob = np.zeros(n, np.uint16)
    dist = np.zeros(n, np.uint64)
    l.orc_quantize_chain_batch(coeffs.ctypes.data, n, tx_size, tx_type, dcq, acq, int(is_intra),
                               int(coeffs.dtype == np.int32), q.ctypes.data, r.ctypes.data, eob.ctypes.data,
                               dist.ctypes.data, threads)
    return q, r, eob, dist


def test_log_tx_scale_kat():
    l = L()
    for name, want in KATS["log_tx_scale"]:
        assert l.orc_get_log_tx_scale(TX_NAMES.index(name)) == want, name


def test_divu_pair_kat():
    """quantize/mod.rs:173-181: x / d == divu_pair(x, divu_gen(d)) for d in 1..1024, x in 0..1000
    (extended here to the 16-bit step sizes and 21-bit magnitudes the encoder can reach)."""
    l = L()
    d3 = (C.c_uint32 * 3)()
    for d in range(1, 1024):
        l.orc_divu_gen(d, d3)
        for x in range(0, 1000, 7):
            assert l.orc_divu_pair(x, d3) == x // d
    rng = np.random.default_rng(0)
    for d in rng.integers(1, 1 << 15, 300):
        l.orc_divu_gen(int(d), d3)
        for x in rng.integers(0, 1 << 22, 50):
            assert l.orc_divu_pair(int(x), d3) == int(x) // int(d)


def test_scan_orders_match_every_reference_table():
    l = L()
    for ts, name in enumerate(TX_NAMES):
        coded = l.orc_coded_tx_area(ts)
        for tt in range(16):
            scan, iscan = np.zeros(coded, np.uint16), np.zeros(coded, np.uint16)
            l.orc_scan_order(ts, tt, scan.ctypes.data, iscan.ctypes.data)
            ref = KATS["scan_tables"][KATS["scan_map"][name][tt]]
            assert ref["n"] == coded
            assert list(scan[:8]) == ref["first8"]
            assert hashlib.sha256(scan.astype("<u2").tobytes()).hexdigest() == ref["sha256"], (name, tt)
            assert (iscan[scan] == np.arange(coded)).all()         # invert(), scan_order.rs:895-903


def py_quantize(c, scan, iscan, lts, dcq, acq, intra):
    """Independent model of quantize/mod.rs:269-361 on Python ints."""
    coded = len(scan)
    q = [0] * coded
    dc_off = dcq * (109 if intra else 108) // 256
    off0 = acq * (98 if intra else 97) // 256
    off1 = acq * (109 if intra else 108) // 256
    off_eob = acq * (88 if intra else 44) // 256
    sgn = lambda v, s: -v if s < 0 else v
    c0 = int(c[0]) << lts
    q[0] = sgn((abs(c0) + dc_off) // dcq, c0)
    deadzone = -(-(acq - off_eob) // (1 << lts))        # ceil
    em1 = max([int(iscan[i]) if abs(int(c[i])) >= deadzone else 0 for i in range(coded)] + [0])
    eob = em1 + 1 if em1 > 0 else int(q[0] != 0)
    lm = 1
    for j in range(1, eob):
        pos = int(scan[j])
        cf = int(c[pos]) << lts
        a = abs(cf)
        l0 = a // acq
        off = off1 if l0 > 1 - lm else off0
        aq = l0 + (1 if a + off >= (l0 + 1) * acq else 0)
        if lm != 0 and aq == 0:
            lm = 0
        elif aq > 1:
            lm = 1
        q[pos] = sgn(aq, cf)
    return q, eob


CASES = [(0, 0, 48, 40, True), (1, 3, 120, 96, False), (2, 0, 300, 260, False), (2, 10, 1336, 1828, True),
         (3, 9, 33, 28, False), (4, 0, 90, 80, True), (9, 0, 500, 480, False), (18, 0, 64, 57, False),
         (13, 11, 21, 19, True), (11, 0, 1200, 999, False), (0, 15, 4, 4, True)]


@pytest.mark.parametrize("ts,tt,dcq,acq,intra", CASES)
def test_chain_matches_python_model(ts, tt, dcq, acq, intra):
    l = L()
    w, h = O.TX_SIZES[ts]
    area, coded = w * h, l.orc_coded_tx_area(ts)
    lts = l.orc_get_log_tx_scale(ts)
    scan, iscan = np.zeros(coded, np.uint16), np.zeros(coded, np.uint16)
    l.orc_scan_order(ts, tt, scan.ctypes.data, iscan.ctypes.data)
    rng = np.random.default_rng(ts * 31 + tt)
    n = 24
    # energy compacted towards low frequencies in scan order, like real transform output
    env = np.zeros(area)
    env[:coded][scan] = 2500.0 / (1.0 + np.arange(coded)) ** 0.9
    env[coded:] = 3.0
    for dtype in (np.int16, np.int32):
        c = np.rint(rng.normal(0, 1, (n, area)) * env).astype(dtype)
        c[3] = 0                                             # an all-zero block
        c[4, 1:] = 0                                         # DC only
        q, r, eob, dist = chain(c, ts, tt, dcq, acq, intra)
        for i in range(n):
            wq, weob = py_quantize(c[i], scan, iscan, lts, dcq, acq, intra)
            assert list(q[i]) == wq, (i, dtype)
            assert int(eob[i]) == weob
            # the reference's own debug assertion (quantize/mod.rs:349-357)
            nz = np.nonzero(np.array(wq)[scan])[0]
            assert weob == (int(nz[-1]) + 1 if len(nz) else 0)
            # dequantize (:368-392) and the raw transform-domain distortion (encoder.rs:1611-1640)
            off = (1 << lts) - 1
            wr = [((v * (dcq if k == 0 else acq)) + (off if v < 0 else 0)) >> lts for k, v in enumerate(wq)]
            assert list(r[i]) == wr
            raw = sum((int(a) - b) ** 2 for a, b in zip(c[i][:coded], wr)) + sum(int(a) ** 2 for a in c[i][coded:])
            bits = 2 * (3 - lts)
            assert int(dist[i]) == (raw + (1 << (bits - 1))) >> bits


def test_deadzone_is_the_documented_threshold():
    """quantize/mod.rs:284-291: abs(coeff) < deadzone  <=>  ((abs(coeff) << s) + ac_offset_eob) / ac_quant == 0,
    which fixes the meaning of v_frame's align_power_of_two_and_shift (off disk) as a ceiling shift."""
    for acq in (4, 9, 57, 260, 1828, 21387):
        for intra in (True, False):
            off = acq * (88 if intra else 44) // 256
            for s in (0, 1, 2):
                dz = (acq - off + (1 << s) - 1) >> s
                for a in range(max(dz - 3, 0), dz + 3):
                    assert (a < dz) == ((((a << s) + off) // acq) == 0)
