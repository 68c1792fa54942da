"""ActivityMask (activity.rs:21-100): the oracle against numpy, and the CUDA source's per-thread
variance function replayed on the CPU (tests/cpp/activity_emul.cu) against the oracle.  The launch
itself is covered by tests/test_zz_activity_gpu.py on hardware."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import oracle_lib as O
from tests.test_oracle_rdo_dist import L as OL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def oracle_mask(img, pad, bd):
    """img: visible area; returns (variances, scales) as (hb, wb) arrays"""
    l = OL()
    l.orc_activity_mask.restype = None
    l.orc_activity_mask.argtypes = [C.c_void_p, C.c_ssize_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    h, w = img.shape
    p = np.pad(img, pad, mode="edge")
    wb, hb = (w + 7) // 8, (h + 7) // 8
    var, sc = np.zeros((hb, wb), np.uint32), np.zeros((hb, wb), np.uint32)
    l.orc_activity_mask(p.ctypes.data + (pad * p.shape[1] + pad) * p.itemsize, p.shape[1], p.itemsize, w, h, bd,
                        var.ctypes.data, sc.ctypes.data)
    return var, sc, p


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 10), (np.uint16, 12)])
def test_oracle_variance_matches_numpy(dtype, bd):
    rng = np.random.default_rng(bd)
    img = rng.integers(0, 1 << bd, (70, 93)).astype(dtype)       # not multiples of 8: reads the padding
    img[:16, :16] = 37                                           # flat blocks: variance exactly 0
    var, sc, p = oracle_mask(img, 8, bd)
    l = OL()
    for by in range(var.shape[0]):
        for bx in range(var.shape[1]):
            blk = p[8 + 8 * by:16 + 8 * by, 8 + 8 * bx:16 + 8 * bx].astype(np.int64)
            s, s2 = int(blk.sum()), int((blk * blk).sum())
            assert int(var[by, bx]) == s2 - ((s * s + 32) >> 6)
            assert int(sc[by, bx]) == l.orc_apply_ssim_boost(1 << 14, int(var[by, bx]), int(var[by, bx]), bd)
    assert var[0, 0] == 0 and var[1, 1] == 0
    # flat blocks get the largest boost, busy blocks are damped (activity.rs:168-172)
    assert sc[0, 0] > sc[-1, -1]


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("act_emul") / "libactemul.so")
    nvcc = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17",
                           "-ccbin", "/usr/bin/g++", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
                           "-shared", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "activity_emul.cu"), "-o", out,
                           "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    lib = C.CDLL(out)
    lib.emul_variances.restype = None
    lib.emul_variances.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_void_p]
    return lib


@pytest.mark.parametrize("dtype,bd", [(np.uint8, 8), (np.uint16, 12)])
def test_cuda_source_variance_equals_oracle(emul, dtype, bd):
    rng = np.random.default_rng(7 + bd)
    img = rng.integers(0, 1 << bd, (64, 120)).astype(dtype)
    img[8:16] = (1 << bd) - 1                                    # saturated rows
    var, _, p = oracle_mask(img, 8, bd)
    got = np.zeros_like(var)
    emul.emul_variances(p.ctypes.data + (8 * p.shape[1] + 8) * p.itemsize, p.shape[1], p.itemsize, var.shape[1],
                        var.shape[0], got.ctypes.data)
    np.testing.assert_array_equal(got, var)
