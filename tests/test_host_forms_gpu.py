"""Host-buffer forms (`*_batch` / `*_resident`) against their `_dev` twins on the same seeded data, a call
rejected after its buffers are staged, and contexts on two devices in one process."""
import ctypes as C

import numpy as np
import pytest

from rav1e_b200 import backend as B
from tests import gpu_util as G
from tests.test_oracle_cdef_rdo import DEFAULT_STRENGTHS, make_frame

pytestmark = pytest.mark.gpu

W, H, PAD = 320, 192, 96
CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7


def _ctx(device=0):
    return B.Context(device, use_torch_stream=True)


def _padded(img, pad):
    return np.ascontiguousarray(np.pad(img, pad, mode="edge"))


def _dev(a, device=0):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8).reshape(-1).copy()).to(f"cuda:{device}")


def _empty(nbytes, device=0):
    import torch
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=f"cuda:{device}")


def _host(t, dtype):
    return t.cpu().numpy().view(dtype)


def _planes(c, seed):
    cur, ref = G.make_planes(W, H, PAD, np.uint8, seed=seed)
    return cur, ref, c.plane_from_host(cur, PAD), c.plane_from_host(ref, PAD)


@pytest.mark.parametrize("async_mode", [False, True])
def test_me_host_forms_equal_dev(async_mode):
    c = _ctx()
    try:
        cur, ref, dcur, dref = _planes(c, 40)
        blocks = G.grid_blocks(W, H, 16, 16)
        cands, offs = G.random_cands(len(blocks), 30, 24, seed=41)
        pmv = np.random.default_rng(42).integers(-64, 65, (len(blocks), 4)).astype(np.int16)
        p = B.me_params(16, 16, W, H, 120, window_hint_px=24)
        n, nb = len(cands), len(blocks)
        d_sad, d_cost, d_best = _empty(4 * n), _empty(8 * n), _empty(16 * nb)
        c.me_candidates_dev(dcur, dref, _dev(blocks), nb, _dev(cands), n, p, _dev(offs), _dev(pmv), d_sad, d_cost,
                            d_best)
        c.synchronize()
        want = (_host(d_sad, np.uint32), _host(d_cost, np.uint64), _host(d_best, B.ME_RESULT_DTYPE))
        assert (want[2]["cost"] != np.uint64(2**64 - 1)).any()
        c.set_async(async_mode)
        outs = [tuple(np.zeros(k, d) for k, d in ((n, np.uint32), (n, np.uint64), (nb, B.ME_RESULT_DTYPE)))
                for _ in range(3)]
        got = c.me_candidates_batch(B.host_plane(_padded(cur, PAD), PAD), B.host_plane(_padded(ref, PAD), PAD),
                                    blocks, cands, p, offs, pmv, out=outs[0])
        c.me_candidates_resident(dcur, dref, blocks, cands, p, offs, outs[1], pmv=pmv)
        mvs = np.ascontiguousarray(np.stack([cands["mv_row"], cands["mv_col"]], axis=1).astype(np.int16))
        c.me_mvs_resident(dcur, dref, blocks, mvs, p, offs, outs[2], pmv=pmv)
        c.synchronize()
        for out in (got,) + tuple(outs[1:]):
            for x, y in zip(out, want):
                np.testing.assert_array_equal(x, y)
        c.plane_free(dcur)
        c.plane_free(dref)
    finally:
        c.close()


@pytest.mark.parametrize("async_mode", [False, True])
def test_fwd_txfm_host_forms_equal_dev(async_mode):
    import torch
    c = _ctx()
    try:
        rng = np.random.default_rng(43)
        n, w, h, stride = 37, 16, 16, 24
        scratch = rng.integers(-255, 256, (n, h, stride)).astype(np.int16)
        d_out = torch.empty((n, w * h), dtype=torch.int16, device="cuda")
        c.fwd_txfm_dev(torch.from_numpy(scratch).cuda(), h * stride, stride, d_out, n, 2, 1, 8, False)
        cur, ref, dcur, dref = _planes(c, 44)
        blocks = G.grid_blocks(W, H, 16, 16)
        mv = np.zeros(len(blocks), B.ME_RESULT_DTYPE)
        mv["mv_row"] = rng.integers(-40, 41, len(blocks)) * 8
        mv["mv_col"] = rng.integers(-40, 41, len(blocks)) * 8
        d_res = torch.empty((len(blocks), 256), dtype=torch.int16, device="cuda")
        c.fwd_txfm_residual_dev(dcur, dref, _dev(blocks), len(blocks), _dev(mv), d_res, 2, 0, 8)
        c.synchronize()
        want_tx, want_res = d_out.cpu().numpy(), d_res.cpu().numpy()
        c.set_async(async_mode)
        got_tx = np.zeros((n, w * h), np.int16)
        c.check(c.L.b200_fwd_txfm_batch(c.h, scratch.ctypes.data, h * stride, stride, got_tx.ctypes.data, n, 2, 1, 8,
                                        0))
        got_res = np.zeros((len(blocks), 256), np.int16)
        c.fwd_txfm_residual_resident(dcur, dref, blocks, mv, got_res, 2, 0, 8)
        c.synchronize()
        np.testing.assert_array_equal(got_tx, want_tx)
        np.testing.assert_array_equal(got_res, want_res)
        c.plane_free(dcur)
        c.plane_free(dref)
    finally:
        c.close()


def test_full_search_batch_equals_dev():
    c = _ctx()
    try:
        cur, ref, dcur, dref = _planes(c, 45)
        blocks = G.grid_blocks(W, H, 16, 16)
        p = B.me_params(16, 16, W, H, 300)
        d_best = _empty(16 * len(blocks))
        c.me_full_search_dev(dcur, dref, _dev(blocks), len(blocks), p, 48, 16, 4, d_best)
        c.synchronize()
        want = _host(d_best, B.ME_RESULT_DTYPE)
        got = c.me_full_search_batch(B.host_plane(_padded(cur, PAD), PAD), B.host_plane(_padded(ref, PAD), PAD),
                                     blocks, p, 48, 16, 4)
        np.testing.assert_array_equal(got, want)
        c.plane_free(dcur)
        c.plane_free(dref)
    finally:
        c.close()


def _pool_used(device):
    cu = C.CDLL("libcuda.so.1")
    dev, pool, used = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuDeviceGet(C.byref(dev), device) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT, C.byref(used)) == 0
    return used.value


def test_rejected_call_after_staging_frees_its_arena():
    """w = 256 passes the host-side checks, so both 1080p planes are staged before the `_dev` call
    rejects the block size: the call returns ERR_ARG and hands its arena back every time."""
    c = _ctx()
    try:
        FW, FH, FP = 1920, 1080, 64
        cur, ref = G.make_planes(FW, FH, FP, np.uint8, seed=46)
        hcur, href = B.host_plane(_padded(cur, FP), FP), B.host_plane(_padded(ref, FP), FP)
        blocks = G.grid_blocks(FW, FH, 256, 256)
        cands, offs = G.random_cands(len(blocks), 4, 8, seed=47)
        bad = B.me_params(256, 256, FW, FH, 0)
        c.synchronize()
        before = _pool_used(0)
        for _ in range(50):
            with pytest.raises(B.B200Error) as e:
                c.me_candidates_batch(hcur, href, blocks, cands, bad, offs)
            assert e.value.status == B.ERR_ARG
        c.synchronize()
        assert _pool_used(0) == before
        # the context still works: a valid call equals the resident form
        blocks = G.grid_blocks(FW, FH, 16, 16)
        cands, offs = G.random_cands(len(blocks), 6, 8, seed=48)
        p = B.me_params(16, 16, FW, FH, 50, window_hint_px=8)
        sad, _, _ = c.me_candidates_batch(hcur, href, blocks, cands, p, offs)
        dcur, dref = c.plane_from_host(cur, FP), c.plane_from_host(ref, FP)
        want = (np.zeros(len(cands), np.uint32), None, None)
        c.me_candidates_resident(dcur, dref, blocks, cands, p, offs, want)
        c.synchronize()
        np.testing.assert_array_equal(sad, want[0])
        c.plane_free(dcur)
        c.plane_free(dref)
    finally:
        c.close()


def _large_smem_kernels(device):
    """Every kernel family that opts in to more than 48 KB of dynamic shared memory, on one device."""
    import torch
    c = _ctx(device)
    out = {}
    try:
        cur, ref, dcur, dref = _planes(c, 50)
        blocks = G.grid_blocks(W, H, 16, 16)
        nb = len(blocks)
        d_blocks = _dev(blocks, device)
        # grouped candidate-list kernel (dense lists inside the window hint)
        cands, offs = G.random_cands(nb, 40, 20, seed=51)
        p = B.me_params(16, 16, W, H, 90, window_hint_px=20)
        d_sad, d_best = _empty(4 * len(cands), device), _empty(16 * nb, device)
        c.me_candidates_dev(dcur, dref, d_blocks, nb, _dev(cands, device), len(cands), p, _dev(offs, device),
                            None, d_sad, None, d_best)
        # square fast `put`
        mvs = np.random.default_rng(52).integers(-60, 61, (nb, 2)).astype(np.int16)
        d_mc = _empty(nb * 256, device)
        c.mc_blocks_dev(dref, d_blocks, _dev(mvs, device), nb, 16, 16, 0, 0, 8, 0, 0, 0, d_mc)
        # fused encode chain
        coded = c.L.b200_coded_tx_area(2)
        d_co = torch.empty((nb, 256), dtype=torch.int16, device=f"cuda:{device}")
        d_q = torch.empty((nb, coded), dtype=torch.int16, device=f"cuda:{device}")
        d_r = torch.empty((nb, coded), dtype=torch.int16, device=f"cuda:{device}")
        rec = c.plane_from_host(ref, 0)
        c.encode_tx_blocks_dev(dcur, dref, rec, d_blocks, nb, None, 2, 0, 8, 70, 60, False, True, d_co, d_q, d_r)
        # sub-pel RDO with the transform
        sc, so = G.random_cands(nb, 3, 4, seed=53, fullpel=False)
        d_cost, d_sbest = _empty(8 * len(sc), device), _empty(16 * nb, device)
        d_coef = torch.zeros((nb, 256), dtype=torch.int16, device=f"cuda:{device}")
        c.subpel_rdo_dev(dcur, dref, d_blocks, nb, _dev(sc, device), len(sc), _dev(so, device),
                         B.me_params(16, 16, W, H, 200, use_satd=True), 0, 2, 0, None, None, d_cost, d_sbest, d_coef)
        # CDEF RDO
        rng = np.random.default_rng(54)
        frec, fsrc = make_frame(rng, 128, 128, "420", 8)
        d_rec = [c.plane_from_host(r, 8) for r in frec]
        d_src = [c.plane_from_host(s, 8) for s in fsrc]
        d_err, d_ccost, d_cbest = _empty(8 * 16 * 8, device), _empty(8 * 16 * 8, device), _empty(16, device)
        c.cdef_rdo_dev(d_rec, d_src, None, 1, 1, 128, 128, 8, 3, 3, DEFAULT_STRENGTHS, DEFAULT_STRENGTHS, None, None,
                       (16384,) * 3, 0.0, [(0, 0, 2, 2)], None, d_err, d_ccost, d_cbest)
        c.synchronize()
        out = {"me": (_host(d_sad, np.uint32), _host(d_best, np.uint8)), "mc": (_host(d_mc, np.uint8),),
               "encode": (d_q.cpu().numpy(), d_r.cpu().numpy()),
               "subpel": (_host(d_cost, np.uint64), _host(d_sbest, np.uint8), d_coef.cpu().numpy()),
               "cdef": (_host(d_err, np.uint64), _host(d_cbest, np.int8))}
        for pl in [dcur, dref, rec] + d_rec + d_src:
            c.plane_free(pl)
    finally:
        c.close()
    return out


def test_two_devices_in_one_process():
    """The shared-memory opt-in belongs to the device: contexts on device 0 and then device 1 must both
    launch the kernels above 48 KB, and compute the same results."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible CUDA devices")
    a, b = _large_smem_kernels(0), _large_smem_kernels(1)
    for k in a:
        for x, y in zip(a[k], b[k]):
            np.testing.assert_array_equal(x, y, err_msg=k)
