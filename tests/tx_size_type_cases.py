"""Fixtures for the intra transform size / type decision: planes, item batches and the oracle
(oracle/tx_size_type.c).  Shared by tests/test_oracle_tx_size_type.py, tests/test_intra_tx_size_type_gpu.py
and bench_kernels.py --tx-size-type."""
import ctypes as C

import numpy as np

from rav1e_b200.backend import TX_BEST_DTYPE, TX_CAND_DTYPE, TX_ITEM_DTYPE
from tests import coeff_rate_cases as K
from tests import gpu_util as G
from tests import oracle_lib as O

BS_W = [4, 4, 8, 8, 8, 16, 16, 16, 32, 32, 32, 64, 64, 64, 128, 128, 4, 16, 8, 32, 16, 64]
BS_H = [4, 8, 4, 8, 16, 8, 16, 32, 16, 32, 64, 32, 64, 128, 64, 128, 16, 4, 32, 8, 64, 16]
SIZES = [b for b in range(22) if b not in (13, 14, 15)]  # the 19 sizes 4x4 .. 64x64
MAX_TX = [0, 5, 6, 1, 7, 8, 2, 9, 10, 3, 11, 12, 4, 4, 4, 4, 13, 14, 15, 16, 17, 18]
SUB_TX = [0, 0, 1, 2, 3, 0, 0, 1, 1, 2, 2, 3, 3, 5, 6, 7, 8, 9, 10]
TX_TYPES = [0, 1, 2, 3, 9, 10, 11]  # RAV1E_TX_TYPES
TX_W = [4, 8, 16, 32, 64, 4, 8, 8, 16, 16, 32, 32, 64, 4, 16, 8, 32, 16, 64]
TX_H = [4, 8, 16, 32, 64, 8, 4, 16, 8, 32, 16, 64, 32, 16, 4, 32, 8, 64, 16]


def _lib():
    L = K._lib()
    if not getattr(L, "_tx_size_type_bound", False):
        vp, pd, sz, i32 = C.c_void_p, C.c_ssize_t, C.c_size_t, C.c_int
        L.orc_intra_tx_size_type.restype = None
        L.orc_intra_tx_size_type.argtypes = [vp, pd, vp, pd] + [i32] * 12 + [C.c_double, C.c_uint32, vp, sz, vp, sz,
                                                                                 vp, sz, vp, vp, i32]
        L._tx_size_type_bound = True
    return L


def make_case(width, height, bd, seed, pad=64):
    """(src, rec) numpy images: rec is src plus coding noise, so predictions from rec see real edges."""
    dtype = np.uint8 if bd == 8 else np.uint16
    rng = np.random.default_rng(seed)
    src, _ = G.make_planes(width, height, pad, dtype, seed=seed, bit_depth=bd)
    noise = rng.integers(-3 << (bd - 8), (3 << (bd - 8)) + 1, src.shape)
    rec = np.clip(src.astype(np.int64) + noise, 0, (1 << bd) - 1).astype(dtype)
    return src, rec


def items(rng, rect_w, rect_h, n, sizes=SIZES, modes=range(13), ncdfs=4, qmax=400, skip_frac=0.15):
    it = np.zeros(n, TX_ITEM_DTYPE)
    for k in range(n):
        b = int(rng.choice(list(sizes)))
        it[k]["bsize"] = b
        it[k]["x"] = int(rng.integers(0, max(1, (rect_w + 3) // 4))) * 4
        it[k]["y"] = int(rng.integers(0, max(1, (rect_h + 3) // 4))) * 4
        it[k]["mode"] = int(rng.choice(list(modes)))
        it[k]["ief"] = int(rng.integers(-1, 2))
        it[k]["skip"] = int(rng.random() < skip_frac)
        it[k]["dc_quant"] = int(rng.integers(4, qmax))
        it[k]["ac_quant"] = int(rng.integers(4, qmax))
        it[k]["snapshot"] = int(rng.integers(0, ncdfs))
        it[k]["above"] = rng.choice([0, 1, 3, 64 + 2, 128 + 5, 63], 16)
        it[k]["left"] = rng.choice([0, 2, 5, 64 + 1, 128 + 7, 63], 16)
    return it


def grid_items(width, height, bw, bh, modes, q=(120, 140), ief=0):
    """Every bw x bh block of the frame with each of `modes`."""
    bs = [b for b in SIZES if BS_W[b] == bw and BS_H[b] == bh][0]
    pos = [(x, y) for y in range(0, height, bh) for x in range(0, width, bw)]
    it = np.zeros(len(pos) * len(modes), TX_ITEM_DTYPE)
    for k, ((x, y), m) in enumerate((p, m) for p in pos for m in modes):
        it[k]["x"], it[k]["y"], it[k]["bsize"], it[k]["mode"], it[k]["ief"] = x, y, bs, m, ief
        it[k]["dc_quant"], it[k]["ac_quant"] = q
    return it


def oracle(src, rec, pad, rect, width, height, bd, dist_mode, reduced, lam, dist_scale, scale, cdfs, it,
           threads=0):
    """orc_intra_tx_size_type over padded copies of src / rec: (best, cands)."""
    osrc, orec = O.Plane(src.shape[1], src.shape[0], pad, src.dtype), O.Plane(rec.shape[1], rec.shape[0], pad, rec.dtype)
    osrc.fill_from(src)
    orec.fill_from(rec)
    best = np.zeros(len(it), TX_BEST_DTYPE)
    cands = np.zeros((len(it), 21), TX_CAND_DTYPE)
    sc = None if scale is None else np.ascontiguousarray(scale, np.uint32)
    _lib().orc_intra_tx_size_type(orec.origin_ptr(), orec.stride, osrc.origin_ptr(), osrc.stride, orec.bpp,
                                  src.shape[1], src.shape[0], rect[0], rect[1], rect[2], rect[3], width, height, bd,
                                  dist_mode, reduced, lam, dist_scale, None if sc is None else sc.ctypes.data,
                                  0 if sc is None else sc.shape[1], cdfs.ctypes.data, len(cdfs),
                                  it.ctypes.data if len(it) else None, len(it), best.ctypes.data, cands.ctypes.data,
                                  threads)
    return best, cands


def ladder(bsize):
    t, out = MAX_TX[bsize], []
    for _ in range(3):
        out.append(t)
        if SUB_TX[t] == t:
            break
        t = SUB_TX[t]
    return out


def type_list(t, skip, reduced):
    set_ = K.tx_set(t, False, reduced)
    if set_ == 0 or skip:
        return [0]
    return [0, 1, 2, 3, 9] if set_ == 2 else list(TX_TYPES)
