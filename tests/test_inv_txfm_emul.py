"""CPU check of the CUDA inverse-transform SOURCE: tests/cpp/inv_txfm_emul.cu includes
rav1e_b200/csrc/inv_txfm.cu and replays the kernel's per-thread row / column passes on the host
(they are __host__ __device__ functions), and the result must equal oracle/inv_txfm.c bit for bit
for every valid (TxSize, TxType) pair at 8, 10 and 12 bit, on realistic coefficients and on coefficients
at the limits of their type (i16 at 8 bit, +-2^30 for i32), where the row and column clamps and the
wrapping i32 arithmetic decide the result.  What is left for the hardware runs
(tests/test_zz_inv_txfm_gpu.py, tests/test_tx_paths_gpu.py) is the launch geometry and the
shared-memory hand-off."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import oracle_lib as O
from tests.test_oracle_inv_txfm import inverse_add

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("inv_emul") / "libinvemul.so")
    nvcc = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17",
                           "-ccbin", "/usr/bin/g++", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
                           "-shared", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "inv_txfm_emul.cu"), "-o", out,
                           "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    lib = C.CDLL(out)
    lib.emul_inverse_transform_add.restype = C.c_int
    lib.emul_inverse_transform_add.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                               C.c_int, C.c_int, C.c_int]
    return lib


def blocks_of(ts, W, H, n):
    w, h = O.TX_SIZES[ts]
    xs, ys = np.arange(0, W - w + 1, w), np.arange(0, H - h + 1, h)
    blocks = np.zeros(min(n, len(xs) * len(ys)), B.BLOCK_DTYPE)
    blocks["x"] = np.tile(xs, len(ys))[:len(blocks)]
    blocks["y"] = np.repeat(ys, len(xs))[:len(blocks)]
    return blocks


def emulate_and_compare(emul, coef, base, blocks, ts, tt, bd):
    w, h = O.TX_SIZES[ts]
    want = base.copy()
    for i, b in enumerate(blocks):
        x, y = int(b["x"]), int(b["y"])
        want[y:y + h, x:x + w] = inverse_add(coef[i], np.ascontiguousarray(want[y:y + h, x:x + w]), ts, tt, bd)
    got = base.copy()
    rc = emul.emul_inverse_transform_add(coef.ctypes.data, got.ctypes.data, base.shape[1], got.itemsize,
                                         blocks.ctypes.data, len(blocks), ts, tt, bd)
    assert rc == 0
    np.testing.assert_array_equal(got, want, err_msg=f"ts={ts} tt={tt} bd={bd}")


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_cuda_source_passes_equal_oracle(emul, bd):
    rng = np.random.default_rng(100 + bd)
    px = np.uint8 if bd == 8 else np.uint16
    ct = np.int16 if bd == 8 else np.int32
    W, H = 192, 128
    for ts, tt in O.valid_txfm_combos():
        w, h = O.TX_SIZES[ts]
        cw, ch = min(w, 32), min(h, 32)
        blocks = blocks_of(ts, W, H, 6)
        n = len(blocks)
        base = rng.integers(0, 1 << bd, (H, W)).astype(px)
        res = rng.integers(-255, 256, (n, h, w)).astype(np.int16) << (bd - 8)
        coef = O.forward_transform_batch(res, ts, tt, bd, coeff_i32=(bd > 8)).reshape(n, -1)[:, :cw * ch]
        coef = np.ascontiguousarray(((coef // 4) * 4).astype(ct))
        if ts % 3 == 0:
            coef[0] = rng.integers(-30000, 30001, cw * ch).astype(ct)       # drive the clamps
        emulate_and_compare(emul, coef, base, blocks, ts, tt, bd)


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_cuda_source_passes_equal_oracle_at_type_limits(emul, bd):
    """Coefficients at the limits of the coefficient type: i16 at 8 bit, +-2^30 for i32 (the rectangular
    scaling then wraps in i32, as the reference's release build does), over destinations at 0 and at max."""
    rng = np.random.default_rng(200 + bd)
    px = np.uint8 if bd == 8 else np.uint16
    ct = np.int16 if bd == 8 else np.int32
    lo, hi = (-32768, 32767) if bd == 8 else (-(1 << 30), 1 << 30)
    W, H = 192, 128
    for ts, tt in O.valid_txfm_combos():
        w, h = O.TX_SIZES[ts]
        m = min(w, 32) * min(h, 32)
        blocks = blocks_of(ts, W, H, 5)
        coef = np.zeros((len(blocks), m), np.int64)
        for i in range(len(blocks)):
            coef[i] = [hi, lo, rng.choice([lo, hi, lo + 1, hi - 1, 0], m), rng.integers(lo, hi + 1, m), 0][i]
        coef[-1, 0] = hi                                                # a lone DC at the top
        base = rng.integers(0, 1 << bd, (H, W)).astype(px)
        for i, b in enumerate(blocks):
            x, y = int(b["x"]), int(b["y"])
            base[y:y + h, x:x + w] = ((1 << bd) - 1) * (i % 2)
        emulate_and_compare(emul, np.ascontiguousarray(coef.astype(ct)), base, blocks, ts, tt, bd)


def test_unimplemented_pairs_are_rejected(emul):
    """INV_TXFM_FNS holes (inverse.rs:1593-1623): ADST beyond 16, identity at 64, WHT beyond 4."""
    z = np.zeros(4096, np.int16)
    d = np.zeros((64, 64), np.uint8)
    b = np.zeros(1, B.BLOCK_DTYPE)
    for ts, tt in ((3, 1), (4, 9), (1, 16), (9, 1)):
        assert emul.emul_inverse_transform_add(z.ctypes.data, d.ctypes.data, 64, 1, b.ctypes.data, 1, ts, tt, 8) == -1
