"""ctypes binding of libb200rdo.so (include/b200rdo.h) + torch device-memory helpers.

Fails loudly: `lib()` raises if the shared library is missing; `Context()` raises if no
CUDA device is usable.  Nothing here computes on the CPU.
"""
import ctypes as C
import os

import numpy as np

PKG = os.path.dirname(os.path.abspath(__file__))
# B200RDO_LIB: load another build of the same ABI (kernel experiments, packaging)
LIB_PATH = os.environ.get("B200RDO_LIB") or os.path.join(PKG, "libb200rdo.so")
_LIB = None

OK, ERR_CUDA, ERR_ARG, ERR_NODEV, ERR_OOM = range(5)


class B200Error(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"b200rdo status {status}: {msg}")
        self.status = status


class Plane(C.Structure):
    _fields_ = [("data", C.c_void_p), ("stride", C.c_int32), ("width", C.c_int32),
                ("height", C.c_int32), ("pad", C.c_int32), ("bpp", C.c_int32),
                ("alloc", C.c_void_p)]


class HostPlane(C.Structure):
    _fields_ = [("data", C.c_void_p), ("stride", C.c_ssize_t), ("width", C.c_int32),
                ("height", C.c_int32), ("pad", C.c_int32), ("bpp", C.c_int32)]


class MeParams(C.Structure):
    _fields_ = [("w", C.c_int32), ("h", C.c_int32), ("frame_w_in_b", C.c_int32),
                ("frame_h_in_b", C.c_int32), ("lambda_", C.c_uint32),
                ("allow_high_precision_mv", C.c_int32), ("use_satd", C.c_int32),
                ("bit_depth", C.c_int32), ("window_hint_px", C.c_int32)]


class CdefItem(C.Structure):
    _fields_ = [("inp", C.POINTER(Plane)), ("out", C.POINTER(Plane)), ("d_skip8", C.c_void_p),
                ("d_dir", C.c_void_p), ("d_var", C.c_void_p), ("rx8", C.c_int32), ("ry8", C.c_int32),
                ("rw8", C.c_int32), ("rh8", C.c_int32)]


class CdefRdoArea(C.Structure):
    """b200_cdef_rdo_area: a loop-restoration area in frame-absolute superblocks."""
    _fields_ = [("sbx", C.c_int32), ("sby", C.c_int32), ("sb_w", C.c_int32), ("sb_h", C.c_int32)]


class FramePipeCfg(C.Structure):
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("pad", C.c_int32), ("bpp", C.c_int32),
                ("bit_depth", C.c_int32), ("block_w", C.c_int32), ("block_h", C.c_int32), ("lambda_", C.c_uint32),
                ("sad_per_block", C.c_int32), ("satd_per_block", C.c_int32), ("window_hint_px", C.c_int32),
                ("tx_size", C.c_int32), ("tx_type", C.c_int32), ("dc_quant", C.c_uint32), ("ac_quant", C.c_uint32)]


class ImpStep(C.Structure):
    """b200_imp_step: one update_block_importances step of the lookahead window."""
    _fields_ = [("src", C.c_uint32), ("dst", C.c_uint32), ("len", C.c_uint32), ("mv_index", C.c_uint32)]


class LookaheadMeParams(C.Structure):
    """b200_lookahead_me_params: the frame's ME settings for b200_lookahead_motion_dev."""
    _fields_ = [("bit_depth", C.c_int32), ("allow_high_precision_mv", C.c_int32), ("me_lambda", C.c_double),
                ("me_allow_full_search", C.c_int32), ("me_range_scale", C.c_int32),
                ("tile_w_sb", C.c_int32), ("tile_h_sb", C.c_int32)]


ME_STATS_DTYPE = np.dtype([("mv_row", "<i2"), ("mv_col", "<i2"), ("normalized_sad", "<u4")])


class EncMeParams(C.Structure):
    """b200_enc_me_params: the frame's settings for b200_estimate_motion_dev."""
    _fields_ = [("bit_depth", C.c_int32), ("allow_high_precision_mv", C.c_int32), ("me_lambda", C.c_double),
                ("use_satd_subpel", C.c_int32), ("filter_mode", C.c_int32), ("tile_w_sb", C.c_int32),
                ("tile_h_sb", C.c_int32)]


# b200_enc_me_item: frame 4x4 offset, reference slot, the two mv-stack predictors (row, col)
ENC_ME_ITEM_DTYPE = np.dtype([("x4", "<u2"), ("y4", "<u2"), ("slot", "u1"), ("pad_", "u1"), ("pmv", "<i2", (2, 2))])
assert ENC_ME_ITEM_DTYPE.itemsize == 14


def imp_steps(steps):
    """[(src, dst, len, mv_index), ...] -> a ctypes array of ImpStep (execution order)."""
    arr = (ImpStep * max(len(steps), 1))()
    for k, s in enumerate(steps):
        arr[k] = ImpStep(*[int(v) for v in s])
    return arr


BLOCK_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2")])
CAND_DTYPE = np.dtype([("block", "<u4"), ("mv_row", "<i2"), ("mv_col", "<i2")])
INTRA_ITEM_DTYPE = np.dtype([("edge", "<u4"), ("ac", "<u4"), ("x", "<i2"), ("y", "<i2"),
                             ("angle", "<i2"), ("mode", "u1"), ("variant", "u1"), ("ief", "i1"),
                             ("left_len", "u1"), ("above_len", "u1"), ("pad_", "u1")])
EDGE_ITEM_DTYPE = np.dtype([("po_x", "<i2"), ("po_y", "<i2"), ("part_x", "<i2"), ("part_y", "<i2"), ("bx", "u1"),
                            ("by", "u1"), ("bsize", "u1"), ("tx_size", "u1"), ("mode", "u1"), ("angle_delta", "i1"),
                            ("enable_ief", "u1"), ("pad_", "u1")])
INTRA_SCREEN_ITEM_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2"), ("bsize", "u1"), ("ief", "i1"),
                                    ("modes", "u1", (13,)), ("pad_", "u1")])
INTER_SCREEN_CAND_DTYPE = np.dtype([("mv", "<i2", (2, 2)), ("ref", "u1", (2,)), ("pad_", "u1", (2,))])
INTER_SCREEN_ITEM_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2"), ("bsize", "u1"), ("n", "u1"), ("pad_", "u1", (2,)),
                                    ("cands", INTER_SCREEN_CAND_DTYPE, (20,))])
assert INTER_SCREEN_CAND_DTYPE.itemsize == 12 and INTER_SCREEN_ITEM_DTYPE.itemsize == 248
CFL_ITEM_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2"), ("bsize", "u1"), ("tx_size", "u1"), ("pad_", "u1", (2,))])
assert CFL_ITEM_DTYPE.itemsize == 8
CFL_ALPHAS = 33              # b200_cfl_alpha_dev's d_sse entries per (item, chroma plane): alpha -16 ..= 16
INTER_SCREEN_SINGLE = 0xFF   # b200_inter_screen_cand.ref[1] of a single-reference entry (NONE_FRAME)
# b200_deblock_mi / b200_deblock_item / b200_deblock_state (include/b200rdo.h)
DEBLOCK_MI_DTYPE = np.dtype([("bsize", "u1"), ("txsize", "u1"), ("mode", "u1"), ("skip", "u1"), ("ref0", "i1"),
                             ("deltas", "i1", (4,)), ("pad_", "u1", (3,))])
DEBLOCK_ITEM_DTYPE = np.dtype([("mi_x", "<i4"), ("mi_y", "<i4"), ("mi_w", "<i4"), ("mi_h", "<i4"), ("vis_w", "<i4"),
                               ("vis_h", "<i4")])
DEBLOCK_STATE_DTYPE = np.dtype([("deltas_enabled", "u1"), ("ref_deltas", "i1", (8,)), ("mode_deltas", "i1", (2,)),
                                ("block_deltas_enabled", "u1"), ("block_delta_shift", "u1"),
                                ("block_delta_multi", "u1"), ("pad_", "u1", (2,))])
assert DEBLOCK_MI_DTYPE.itemsize == 12 and DEBLOCK_ITEM_DTYPE.itemsize == 24 and DEBLOCK_STATE_DTYPE.itemsize == 16
# b200_lrf_unit (include/b200rdo.h): type 0 None, 1 Wiener, 2 Sgrproj
LRF_UNIT_DTYPE = np.dtype([("type", "u1"), ("set", "u1"), ("xqd", "i1", (2,)), ("coeffs", "i1", (2, 3)),
                           ("pad_", "u1", (2,))])
assert LRF_UNIT_DTYPE.itemsize == 12
# b200_lrf_search_item (include/b200rdo.h)
LRF_SEARCH_ITEM_DTYPE = np.dtype(
    {"names": ["area", "plane", "lru_x", "lru_y", "incoming", "none_bits", "incoming_cost", "sgr_bits", "sgrproj_ref"],
     "formats": ["<i4", "<i4", "<i4", "<i4", LRF_UNIT_DTYPE, "<u4", "<f8", "<u4", ("i1", (2,))],
     "offsets": [0, 4, 8, 12, 16, 28, 32, 40, 44], "itemsize": 48})
# b200_loop_unit (include/b200rdo.h)
LOOP_UNIT_DTYPE = np.dtype([("area", "<i4"), ("plane", "<i4"), ("lru_x", "<i4"), ("lru_y", "<i4"),
                            ("none_bits", "<u4"), ("sgr_bits", "<u4"), ("sgrproj_ref", "i1", (2,)), ("search", "u1"),
                            ("pad_", "u1")])
assert LOOP_UNIT_DTYPE.itemsize == 28
ME_RESULT_DTYPE = np.dtype(
    {"names": ["cost", "sad", "mv_row", "mv_col"],
     "formats": ["<u8", "<u4", "<i2", "<i2"], "offsets": [0, 8, 12, 14], "itemsize": 16})
# b200_segmentation / b200_segment_item (include/b200rdo.h)
SEGMENTATION_DTYPE = np.dtype([("enabled", "u1"), ("update_data", "u1"), ("update_map", "u1"), ("preskip", "u1"),
                               ("last_active_segid", "u1"), ("min_segment", "u1"), ("max_segment", "u1"),
                               ("pad_", "u1"), ("features", "u1", (8, 8)), ("data", "<i2", (8, 8)),
                               ("threshold", "<u4", (7,)), ("qidx", "u1", (8,)), ("status", "<i4")])
SEGMENT_ITEM_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2"), ("bsize", "u1"), ("skip", "u1"), ("pad_", "u1", (2,))])
assert SEGMENTATION_DTYPE.itemsize == 240 and SEGMENT_ITEM_DTYPE.itemsize == 8
SEGMENTATION_SIMPLE, SEGMENTATION_COMPLEX, SEGMENTATION_FULL = 1, 2, 3  # SegmentationLevel discriminants
# b200_coeff_cdfs / b200_coeff_chain / b200_coeff_item (include/b200rdo.h)
COEFF_CDFS_DTYPE = np.dtype([("txb_skip", "<u2", (5, 13, 2)), ("dc_sign", "<u2", (2, 3, 2)),
                             ("eob_extra", "<u2", (5, 2, 9, 2))]
                            + [(f"eob_flag{16 << i}", "<u2", (2, 2, 5 + i)) for i in range(7)]
                            + [("coeff_base_eob", "<u2", (5, 2, 4, 3)), ("coeff_base", "<u2", (5, 2, 42, 4)),
                               ("coeff_br", "<u2", (5, 2, 21, 4)), ("intra_tx_1", "<u2", (4, 13, 7)),
                               ("intra_tx_2", "<u2", (4, 13, 5)), ("inter_tx_1", "<u2", (4, 16)),
                               ("inter_tx_2", "<u2", (4, 12)), ("inter_tx_3", "<u2", (4, 2))])
COEFF_CHAIN_DTYPE = np.dtype([("snapshot", "<u4"), ("init_rng", "<u4"), ("item_begin", "<u4"), ("item_count", "<u4"),
                              ("above", "u1", (3, 16)), ("left", "u1", (3, 16))])
COEFF_ITEM_DTYPE = np.dtype([("block", "<u4"), ("eob", "<u2"), ("tx_size", "u1"), ("tx_type", "u1"), ("plane", "u1"),
                             ("plane_bsize", "u1"), ("mode", "u1"), ("reduced_tx_set", "u1"), ("x4", "u1"),
                             ("y4", "u1"), ("clip_w4", "u1"), ("clip_h4", "u1")])
assert COEFF_CDFS_DTYPE.itemsize == 7860 and COEFF_CHAIN_DTYPE.itemsize == 112 and COEFF_ITEM_DTYPE.itemsize == 16
# intra transform size / type decision records (include/b200rdo.h b200_tx_item / b200_tx_best / b200_tx_cand)
TX_ITEM_DTYPE = np.dtype([("x", "<i2"), ("y", "<i2"), ("bsize", "u1"), ("mode", "u1"), ("ief", "i1"), ("skip", "u1"),
                          ("dc_quant", "<u4"), ("ac_quant", "<u4"), ("snapshot", "<u4"), ("above", "u1", (16,)),
                          ("left", "u1", (16,))])
TX_BEST_DTYPE = np.dtype([("rd", "<f8"), ("tx_size", "u1"), ("tx_type", "u1"), ("pad_", "u1", (6,))])
TX_CAND_DTYPE = np.dtype([("rd", "<f8"), ("dist", "<u8"), ("rate", "<u4"), ("state", "<u4")])
TX_EVALUATED, TX_NOT_IN_SET, TX_CUT, TX_NOT_IN_LADDER, TX_INVALID = 0, 1, 2, 3, 255
assert TX_ITEM_DTYPE.itemsize == 52 and TX_BEST_DTYPE.itemsize == 16 and TX_CAND_DTYPE.itemsize == 24

BLOCK_SIZES = [(4, 4), (4, 8), (4, 16), (8, 4), (8, 8), (8, 16), (8, 32), (16, 4), (16, 8),
               (16, 16), (16, 32), (16, 64), (32, 8), (32, 16), (32, 32), (32, 64), (64, 16),
               (64, 32), (64, 64), (64, 128), (128, 64), (128, 128)]


class PlanePairs:
    """Host-side table for b200_me_candidates_multi_dev: plane descriptors of each (cur, ref) pair
    and the running ends of each pair's blocks / candidates in the concatenated arrays."""

    def __init__(self, curs, refs, block_end, cand_end):
        self.n = len(curs)
        assert len(refs) == self.n and len(block_end) == self.n and len(cand_end) == self.n
        self.curs = (Plane * self.n)()
        self.refs = (Plane * self.n)()
        for k in range(self.n):
            C.memmove(C.byref(self.curs[k]), C.byref(curs[k]), C.sizeof(Plane))
            C.memmove(C.byref(self.refs[k]), C.byref(refs[k]), C.sizeof(Plane))
        self.block_end = np.ascontiguousarray(block_end, np.uint32)
        self.cand_end = np.ascontiguousarray(cand_end, np.uint32)


def lib():
    """Load the CUDA backend.  Raises if it has not been built (no fallback)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m rav1e_b200.build` "
            "(or __graft_entry__.build()); rav1e_b200 has no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, sz, i32, u32 = C.c_void_p, C.c_size_t, C.c_int, C.c_uint32
    pp = C.POINTER(Plane)
    php = C.POINTER(HostPlane)
    pmp = C.POINTER(MeParams)
    L.b200_abi_version.restype = i32
    L.b200_device_count.restype = i32
    L.b200_ctx_create.argtypes = [i32, C.POINTER(vp)]
    L.b200_ctx_destroy.argtypes = [vp]
    L.b200_ctx_destroy.restype = None
    L.b200_last_error.argtypes = [vp]
    L.b200_last_error.restype = C.c_char_p
    L.b200_ctx_set_stream.argtypes = [vp, vp]
    L.b200_ctx_reset_stream.argtypes = [vp]
    L.b200_ctx_set_async.argtypes = [vp, i32]
    L.b200_ctx_get_stream.argtypes = [vp]
    L.b200_ctx_get_stream.restype = vp
    L.b200_ctx_synchronize.argtypes = [vp]
    L.b200_ctx_launch_count.argtypes = [vp]
    L.b200_ctx_launch_count.restype = C.c_uint64
    L.b200_malloc.argtypes = [vp, sz, C.POINTER(vp)]
    L.b200_free.argtypes = [vp, vp]
    L.b200_memcpy_h2d.argtypes = [vp, vp, vp, sz]
    L.b200_memcpy_d2h.argtypes = [vp, vp, vp, sz]
    L.b200_plane_alloc.argtypes = [vp, i32, i32, i32, i32, pp]
    L.b200_plane_free.argtypes = [vp, pp]
    L.b200_plane_upload.argtypes = [vp, pp, vp, C.c_ssize_t]
    L.b200_plane_download.argtypes = [vp, pp, vp, C.c_ssize_t]
    L.b200_get_sad.argtypes = [vp, C.c_ssize_t, vp, C.c_ssize_t, i32, i32, i32]
    L.b200_get_sad.restype = u32
    L.b200_get_satd.argtypes = [vp, C.c_ssize_t, vp, C.c_ssize_t, i32, i32, i32]
    L.b200_get_satd.restype = u32
    for w, h in BLOCK_SIZES:
        for name, extra in ((f"rav1e_sad{w}x{h}_cuda", []), (f"rav1e_sad_{w}x{h}_hbd_cuda", []),
                            (f"rav1e_satd_{w}x{h}_cuda", []),
                            (f"rav1e_satd_{w}x{h}_hbd_cuda", [u32])):
            f = getattr(L, name)
            f.argtypes = [vp, C.c_ssize_t, vp, C.c_ssize_t] + extra
            f.restype = u32
    L.b200_me_candidates_dev.argtypes = [vp, pp, pp, vp, sz, vp, sz, vp, vp, pmp, vp, vp, vp]
    L.b200_encode_tx_blocks_dev.argtypes = [vp, pp, pp, pp, vp, sz, vp, i32, i32, i32, u32, u32, i32, i32, vp, vp, vp, vp, vp]
    L.b200_inverse_transform_add_dev.argtypes = [vp, vp, pp, vp, sz, i32, i32, i32]
    L.b200_quantize_dev.argtypes = [vp, vp, sz, i32, i32, u32, u32, i32, i32, vp, vp, vp, vp]
    L.b200_weighted_sse.restype = C.c_uint64
    L.b200_weighted_sse.argtypes = [vp, C.c_ssize_t, vp, C.c_ssize_t, vp, C.c_ssize_t, i32, i32, i32]
    L.b200_cdef_dist_kernel.restype = u32
    L.b200_cdef_dist_kernel.argtypes = [vp, C.c_ssize_t, vp, C.c_ssize_t, i32, i32, i32, vp]
    L.b200_compute_rd_cost_dev.argtypes = [vp, C.c_double, vp, vp, sz, vp, sz, vp, vp]
    L.b200_compute_rd_cost.argtypes = [C.c_double, u32, C.c_uint64]
    L.b200_compute_rd_cost.restype = C.c_double
    L.b200_activity_mask_dev.argtypes = [vp, pp, i32, vp, vp]
    L.b200_weighted_sse_dev.argtypes = [vp, pp, pp, vp, sz, i32, i32, vp, sz, vp]
    L.b200_cdef_dist_dev.argtypes = [vp, pp, pp, vp, sz, i32, i32, i32, vp, vp]
    L.b200_me_search_dev.argtypes = [vp, pp, pp, vp, sz, vp, vp, i32, vp, vp, pmp, i32, vp]
    L.b200_me_search_multi_dev.argtypes = [vp, sz, vp, vp, vp, vp, sz, vp, vp, i32, vp, vp, pmp, i32, vp]
    L.b200_me_candidates_multi_dev.argtypes = [vp, sz, vp, vp, vp, vp, vp, sz, vp, sz, vp, vp, pmp, vp, vp, vp]
    L.b200_me_subpel_candidates_dev.argtypes = [vp, pp, pp, vp, sz, vp, sz, vp, vp, pmp, i32, vp, vp, vp]
    L.b200_subpel_rdo_dev.argtypes = [vp, pp, pp, vp, sz, vp, sz, vp, vp, pmp, i32, i32, i32, vp, vp, vp, vp]
    L.b200_subpel_search_dev.argtypes = [vp, pp, pp, vp, sz, vp, vp, pmp, i32, i32, i32, vp, vp]
    L.b200_me_full_search_dev.argtypes = [vp, pp, pp, vp, sz, pmp, i32, i32, i32, vp]
    L.b200_block_residual_dev.argtypes = [vp, pp, pp, vp, sz, vp, i32, i32, vp]
    L.b200_me_candidates_batch.argtypes = [vp, php, php, vp, sz, vp, sz, vp, vp, pmp, vp, vp, vp]
    L.b200_me_candidates_resident.argtypes = [vp, pp, pp, vp, sz, vp, sz, vp, vp, pmp, vp, vp, vp]
    L.b200_me_mvs_resident.argtypes = [vp, pp, pp, vp, sz, vp, sz, vp, vp, pmp, vp, vp, vp]
    L.b200_fwd_txfm_residual_resident.argtypes = [vp, pp, pp, vp, sz, vp, vp, i32, i32, i32]
    L.b200_me_full_search_batch.argtypes = [vp, php, php, vp, sz, pmp, i32, i32, i32, vp]
    L.b200_valid_av1_transform.argtypes = [i32, i32]
    L.b200_tx_width.argtypes = [i32]
    L.b200_tx_height.argtypes = [i32]
    L.b200_forward_transform.argtypes = [vp, vp, sz, i32, i32, i32, i32]
    L.b200_forward_transform.restype = None
    L.b200_fwd_txfm_dev.argtypes = [vp, vp, sz, sz, vp, sz, i32, i32, i32, i32]
    L.b200_fwd_txfm_residual_dev.argtypes = [vp, pp, pp, vp, sz, vp, vp, i32, i32, i32]
    L.b200_fwd_txfm_residual_multi_dev.argtypes = [vp, sz, vp, vp, vp, vp, sz, vp, vp, i32, i32, i32]
    L.b200_fwd_txfm_pred_dev.argtypes = [vp, pp, vp, vp, sz, vp, i32, i32, i32]
    L.b200_fwd_txfm_batch.argtypes = [vp, vp, sz, sz, vp, sz, i32, i32, i32, i32]
    L.b200_put_8tap.argtypes = [vp, C.c_ssize_t, vp, C.c_ssize_t] + [i32] * 7
    L.b200_put_8tap.restype = None
    L.b200_prep_8tap.argtypes = [vp, vp, C.c_ssize_t] + [i32] * 7
    L.b200_prep_8tap.restype = None
    L.b200_mc_avg.argtypes = [vp, C.c_ssize_t, vp, vp, i32, i32, i32]
    L.b200_mc_avg.restype = None
    L.b200_mc_blocks_dev.argtypes = [vp, pp, vp, vp, sz] + [i32] * 8 + [vp]
    L.b200_mc_avg_dev.argtypes = [vp, vp, vp, vp, sz, i32, i32, i32]
    L.b200_cdef_dir.argtypes = [vp, C.c_ssize_t, C.POINTER(u32), i32]
    L.b200_cdef_dir.restype = i32
    L.b200_cdef_filter_block.argtypes = [vp, C.c_ssize_t, vp, C.c_ssize_t] + [i32] * 7
    L.b200_cdef_filter_block.restype = None
    L.b200_cdef_find_dir_dev.argtypes = [vp, pp, i32, vp, vp, vp]
    L.b200_cdef_filter_plane_dev.argtypes = [vp, pp, pp] + [i32] * 7 + [vp, vp, vp, vp]
    L.b200_cdef_find_dir_rect_dev.argtypes = [vp, pp, i32, vp, vp, vp] + [i32] * 4
    L.b200_cdef_filter_rect_dev.argtypes = [vp, pp, pp] + [i32] * 7 + [vp, vp, vp, vp] + [i32] * 4
    L.b200_cdef_tiles_dev.argtypes = [vp, vp, sz] + [i32] * 7 + [vp, i32, i32]
    L.b200_predict_intra.argtypes = [i32, i32, vp, C.c_ssize_t, i32, i32, i32, vp, i32, i32, vp] + [i32] * 6
    L.b200_predict_intra.restype = None
    L.b200_predict_intra_dev.argtypes = [vp, vp, vp, sz, vp, i32, i32, i32, i32, i32, vp]
    L.b200_frame_pipe_create.argtypes = [vp, C.POINTER(FramePipeCfg), C.POINTER(vp)]
    L.b200_frame_pipe_destroy.argtypes = [vp]
    L.b200_frame_pipe_destroy.restype = None
    L.b200_frame_pipe_nblocks.argtypes = [vp]
    L.b200_frame_pipe_nblocks.restype = sz
    L.b200_frame_pipe_push.argtypes = [vp, vp, C.c_ssize_t] + [vp] * 8
    L.b200_frame_pipe_set_lists.argtypes = [vp, vp, vp, vp]
    L.b200_frame_pipe_push_packed.argtypes = [vp, vp, C.c_ssize_t] + [vp] * 5 + [sz, C.POINTER(sz)]
    L.b200_plane_downsample_dev.argtypes = [vp, pp, pp, i32, i32]
    L.b200_estimate_intra_costs_dev.argtypes = [vp, pp, i32, vp]
    L.b200_estimate_inter_costs_dev.argtypes = [vp, pp, pp, vp, vp, vp, vp]
    L.b200_importance_block_difference_dev.argtypes = [vp, pp, pp, vp, vp]
    L.b200_block_importances_dev.argtypes = [vp, sz, vp, i32, vp, vp, sz, vp, vp]
    L.b200_distortion_scales_dev.argtypes = [vp, pp, vp, vp, vp]
    L.b200_temporal_scores_dev.argtypes = [vp, sz, sz, vp, vp, vp, vp, vp, sz]
    L.b200_segmentation_optimize_dev.argtypes = [vp, vp, sz, sz, i32, i32, vp, i32, vp, vp]
    L.b200_select_segment_dev.argtypes = [vp, vp, sz, vp, vp, sz, sz, i32, i32, vp, vp, vp]
    L.b200_coeff_rate_dev.argtypes = [vp, vp, sz, vp, sz, vp, sz, vp, sz, i32, vp, vp]
    L.b200_intra_tx_size_type_dev.argtypes = [vp, pp, pp] + [i32] * 9 + [C.c_double, C.c_uint32, vp, sz, vp, sz,
                                                                          vp, sz, vp, vp]
    L.b200_lookahead_motion_dev.argtypes = [vp, sz, vp, vp, C.POINTER(LookaheadMeParams), vp, vp, vp]
    L.b200_estimate_motion_dev.argtypes = [vp, pp, sz, vp, vp, vp, vp, C.POINTER(EncMeParams), vp, vp, sz, vp]
    L.b200_get_intra_edges_dev.argtypes = [vp, pp] + [i32] * 7 + [vp, sz, vp, vp]
    L.b200_pred_cfl_ac_dev.argtypes = [vp, pp, vp, sz] + [i32] * 6 + [vp]
    L.b200_intra_mode_screen_dev.argtypes = [vp, pp, pp] + [i32] * 6 + [vp, sz, vp, vp]
    L.b200_inter_mode_screen_dev.argtypes = [vp, pp] + [i32] * 4 + [vp] + [i32] * 5 + [vp, sz, vp, vp]
    L.b200_cdef_rdo_dev.argtypes = [vp, vp, vp, vp] + [i32] * 8 + [vp] * 5 + [C.c_double, vp, sz, vp, vp, vp, vp]
    L.b200_cfl_alpha_dev.argtypes = [vp, vp, vp] + [i32] * 9 + [vp, sz, vp, vp]
    L.b200_deblock_levels_dev.argtypes = [vp, vp, vp] + [i32] * 4 + [vp, i32, vp, sz, vp, vp]
    L.b200_deblock_filter_dev.argtypes = [vp, vp, vp] + [i32] * 4 + [vp, vp, vp, i32, vp, sz]
    L.b200_lrf_filter_dev.argtypes = [vp, vp, vp, vp] + [i32] * 7 + [vp, vp]
    L.b200_loop_decision_dev.argtypes = [vp, vp, vp, vp] + [i32] * 9 + [vp, vp, vp, i32, vp, i32, vp, vp,
                                                                        C.c_double, vp, sz, vp, sz] + [vp] * 8
    L.b200_lrf_search_dev.argtypes = [vp, vp, vp] + [i32] * 6 + [vp, i32, vp, vp, C.c_double, vp, sz, vp, sz] + [vp] * 6
    _LIB = L
    return L


def _np_ptr(a):
    return None if a is None else a.ctypes.data


def _dev_ptr(t):
    """torch CUDA tensor -> raw device pointer (None passes through)."""
    return None if t is None else t.data_ptr()


class Context:
    """One b200_ctx (one per process/GPU; the Rust side would hold one per rayon worker)."""

    def __init__(self, device=0, use_torch_stream=False):
        self.L = lib()
        h = C.c_void_p()
        st = self.L.b200_ctx_create(device, C.byref(h))
        if st != OK:
            raise B200Error(st, self.L.b200_last_error(None).decode())
        self.h = h
        self.device = device
        if use_torch_stream:
            import torch
            self.check(self.L.b200_ctx_set_stream(h, torch.cuda.current_stream(device).cuda_stream))

    def check(self, st):
        if st != OK:
            raise B200Error(st, self.L.b200_last_error(self.h).decode())

    def close(self):
        if self.h:
            self.L.b200_ctx_destroy(self.h)
            self.h = None

    def synchronize(self):
        self.check(self.L.b200_ctx_synchronize(self.h))

    @property
    def launches(self):
        return int(self.L.b200_ctx_launch_count(self.h))

    # ---- planes
    def plane_from_host(self, img, pad):
        """Upload a 2-D numpy array (u8/u16) as a padded device plane (edges replicated)."""
        img = np.ascontiguousarray(img)
        assert img.ndim == 2 and img.dtype in (np.uint8, np.uint16)
        p = Plane()
        self.check(self.L.b200_plane_alloc(self.h, img.shape[1], img.shape[0], pad, img.itemsize,
                                           C.byref(p)))
        self.check(self.L.b200_plane_upload(self.h, C.byref(p), img.ctypes.data, img.strides[0]))
        return p

    def plane_free(self, p):
        self.check(self.L.b200_plane_free(self.h, C.byref(p)))

    # ---- ME, device resident (torch tensors hold descriptors/results)
    def me_candidates_dev(self, cur, ref, d_blocks, nblocks, d_cands, ncands, params, d_offsets=None,
                          d_pmv=None, d_sad=None, d_cost=None, d_best=None):
        self.check(self.L.b200_me_candidates_dev(
            self.h, C.byref(cur), C.byref(ref), _dev_ptr(d_blocks), nblocks, _dev_ptr(d_cands),
            ncands, _dev_ptr(d_offsets), _dev_ptr(d_pmv), C.byref(params), _dev_ptr(d_sad),
            _dev_ptr(d_cost), _dev_ptr(d_best)))

    def me_candidates_multi_dev(self, pairs, d_blocks, nblocks, d_cands, ncands, params,
                                d_offsets=None, d_pmv=None, d_sad=None, d_cost=None, d_best=None):
        """One launch over several (cur, ref) plane pairs (`pairs`: a PlanePairs)."""
        self.check(self.L.b200_me_candidates_multi_dev(
            self.h, pairs.n, C.addressof(pairs.curs), C.addressof(pairs.refs),
            pairs.block_end.ctypes.data, pairs.cand_end.ctypes.data,
            _dev_ptr(d_blocks), nblocks, _dev_ptr(d_cands), ncands, _dev_ptr(d_offsets),
            _dev_ptr(d_pmv), C.byref(params), _dev_ptr(d_sad), _dev_ptr(d_cost), _dev_ptr(d_best)))

    def me_search_dev(self, cur, ref, d_blocks, nblocks, d_preds, d_subset_offsets, nsubsets, params,
                      d_best, d_pmv=None, d_thresh=None, umh_range=0):
        """full_pixel_me's search stages for every block (include/b200rdo.h)."""
        self.check(self.L.b200_me_search_dev(
            self.h, C.byref(cur), C.byref(ref), _dev_ptr(d_blocks), nblocks, _dev_ptr(d_preds),
            _dev_ptr(d_subset_offsets), nsubsets, _dev_ptr(d_pmv), _dev_ptr(d_thresh), C.byref(params),
            umh_range, _dev_ptr(d_best)))

    def me_search_multi_dev(self, pairs, d_blocks, nblocks, d_preds, d_subset_offsets, nsubsets, params,
                            d_best, d_pmv=None, d_thresh=None, umh_range=0):
        self.check(self.L.b200_me_search_multi_dev(
            self.h, pairs.n, C.addressof(pairs.curs), C.addressof(pairs.refs), pairs.block_end.ctypes.data,
            _dev_ptr(d_blocks), nblocks, _dev_ptr(d_preds), _dev_ptr(d_subset_offsets), nsubsets,
            _dev_ptr(d_pmv), _dev_ptr(d_thresh), C.byref(params), umh_range, _dev_ptr(d_best)))

    def me_subpel_candidates_dev(self, cur, ref, d_blocks, nblocks, d_cands, ncands, params, filter_mode=0,
                                 d_offsets=None, d_pmv=None, d_sad=None, d_cost=None, d_best=None):
        self.check(self.L.b200_me_subpel_candidates_dev(
            self.h, C.byref(cur), C.byref(ref), _dev_ptr(d_blocks), nblocks, _dev_ptr(d_cands), ncands,
            _dev_ptr(d_offsets), _dev_ptr(d_pmv), C.byref(params), filter_mode, _dev_ptr(d_sad),
            _dev_ptr(d_cost), _dev_ptr(d_best)))

    def subpel_rdo_dev(self, cur, ref, d_blocks, nblocks, d_cands, ncands, d_offsets, params, filter_mode=0,
                       tx_size=-1, tx_type=0, d_pmv=None, d_sad=None, d_cost=None, d_best=None, d_coeffs=None):
        self.check(self.L.b200_subpel_rdo_dev(
            self.h, C.byref(cur), C.byref(ref), _dev_ptr(d_blocks), nblocks, _dev_ptr(d_cands), ncands,
            _dev_ptr(d_offsets), _dev_ptr(d_pmv), C.byref(params), filter_mode, tx_size, tx_type, _dev_ptr(d_sad),
            _dev_ptr(d_cost), _dev_ptr(d_best), _dev_ptr(d_coeffs)))

    def subpel_search_dev(self, cur, ref, d_blocks, nblocks, d_start, params, d_best, filter_mode=0, tx_size=-1,
                          tx_type=0, d_pmv=None, d_coeffs=None):
        self.check(self.L.b200_subpel_search_dev(
            self.h, C.byref(cur), C.byref(ref), _dev_ptr(d_blocks), nblocks, _dev_ptr(d_start), _dev_ptr(d_pmv),
            C.byref(params), filter_mode, tx_size, tx_type, _dev_ptr(d_best), _dev_ptr(d_coeffs)))

    def me_full_search_dev(self, cur, ref, d_blocks, nblocks, params, range_x, range_y, step, d_best):
        self.check(self.L.b200_me_full_search_dev(
            self.h, C.byref(cur), C.byref(ref), _dev_ptr(d_blocks), nblocks, C.byref(params),
            range_x, range_y, step, _dev_ptr(d_best)))

    def block_residual_dev(self, cur, ref, d_blocks, nblocks, d_mv_src, w, h, d_out):
        self.check(self.L.b200_block_residual_dev(self.h, C.byref(cur), C.byref(ref),
                                                  _dev_ptr(d_blocks), nblocks, _dev_ptr(d_mv_src),
                                                  w, h, _dev_ptr(d_out)))

    # ---- quantize -> dequantize -> tx-domain distortion
    def quantize_dev(self, d_coeffs, n, tx_size, tx_type, dc_quant, ac_quant, is_intra, coeff_i32, d_q,
                     d_r=None, d_eob=None, d_dist=None):
        self.check(self.L.b200_quantize_dev(self.h, _dev_ptr(d_coeffs), n, tx_size, tx_type, dc_quant, ac_quant,
                                            int(is_intra), int(coeff_i32), _dev_ptr(d_q), _dev_ptr(d_r),
                                            _dev_ptr(d_eob), _dev_ptr(d_dist)))

    def encode_tx_blocks_dev(self, cur, ref, rec, d_blocks, n, d_mv_src, tx_size, tx_type, bd, dc_quant, ac_quant,
                             is_intra, need_recon, d_coeffs, d_q, d_r, d_eob=None, d_dist=None):
        self.check(self.L.b200_encode_tx_blocks_dev(
            self.h, C.byref(cur), C.byref(ref), C.byref(rec) if rec is not None else None, _dev_ptr(d_blocks), n,
            _dev_ptr(d_mv_src), tx_size, tx_type, bd, dc_quant, ac_quant, int(is_intra), int(need_recon),
            _dev_ptr(d_coeffs), _dev_ptr(d_q), _dev_ptr(d_r), _dev_ptr(d_eob), _dev_ptr(d_dist)))

    def inverse_transform_add_dev(self, d_coeffs, dst, d_blocks, n, tx_size, tx_type, bd):
        self.check(self.L.b200_inverse_transform_add_dev(self.h, _dev_ptr(d_coeffs), C.byref(dst), _dev_ptr(d_blocks),
                                                         n, tx_size, tx_type, bd))

    # ---- lookahead
    def plane_alloc(self, width, height, pad, bpp):
        p = Plane()
        self.check(self.L.b200_plane_alloc(self.h, width, height, pad, bpp, C.byref(p)))
        return p

    def plane_downsample_dev(self, src, dst, pad_w, pad_h):
        self.check(self.L.b200_plane_downsample_dev(self.h, C.byref(src), C.byref(dst), pad_w, pad_h))

    def estimate_intra_costs_dev(self, luma, bit_depth, d_costs):
        self.check(self.L.b200_estimate_intra_costs_dev(self.h, C.byref(luma), bit_depth, _dev_ptr(d_costs)))

    def estimate_inter_costs_dev(self, org, ref, d_mvs, d_costs, d_scratch, d_mean):
        self.check(self.L.b200_estimate_inter_costs_dev(self.h, C.byref(org), C.byref(ref), _dev_ptr(d_mvs),
                                                        _dev_ptr(d_costs), _dev_ptr(d_scratch), _dev_ptr(d_mean)))

    def importance_block_difference_dev(self, org, ref, d_scratch, d_mean):
        self.check(self.L.b200_importance_block_difference_dev(self.h, C.byref(org), C.byref(ref),
                                                               _dev_ptr(d_scratch), _dev_ptr(d_mean)))

    def lookahead_motion_dev(self, curs, refs, params, d_stats, d_prev=None, has_prev=None):
        """compute_motion_vectors for len(curs) (frame, reference slot) pairs: curs / refs are lists of
        (full, half, quarter) Plane triples; d_stats receives len(curs) grids of w_in_b x h_in_b
        ME_STATS_DTYPE; d_prev (optional) holds LAST's final grids, used where has_prev[k] is true."""
        n = len(curs)
        assert len(refs) == n
        arrs = []
        for side in (curs, refs):
            arr = (Plane * (3 * n))()
            for k, trip in enumerate(side):
                assert len(trip) == 3
                for s, p in enumerate(trip):
                    C.memmove(C.byref(arr[3 * k + s]), C.byref(p), C.sizeof(Plane))
            arrs.append(arr)
        flags = None
        if has_prev is not None:
            flags = np.ascontiguousarray(np.asarray(has_prev, np.uint8).reshape(n))
        self.check(self.L.b200_lookahead_motion_dev(self.h, n, C.addressof(arrs[0]), C.addressof(arrs[1]),
                                                    C.byref(params), _dev_ptr(d_prev), _np_ptr(flags),
                                                    _dev_ptr(d_stats)))

    def estimate_motion_dev(self, src, refs, d_stats, params, size_end, d_items, nitems, d_out, d_prev=None,
                            has_prev=None):
        """estimate_motion for a batch of (block, reference slot) items (include/b200rdo.h): src a Plane, refs a
        list of Plane (one per slot); d_stats / d_prev len(refs) ME_STATS_DTYPE grids on the device; size_end the
        19 cumulative item counts in TxSize order; d_items ENC_ME_ITEM_DTYPE, d_out ME_RESULT_DTYPE."""
        n = len(refs)
        arr = (Plane * max(n, 1))()
        for k, p in enumerate(refs):
            C.memmove(C.byref(arr[k]), C.byref(p), C.sizeof(Plane))
        ends = np.ascontiguousarray(np.asarray(size_end, np.uint32).reshape(19))
        flags = None
        if has_prev is not None:
            flags = np.ascontiguousarray(np.asarray(has_prev, np.uint8).reshape(n))
        self.check(self.L.b200_estimate_motion_dev(self.h, C.byref(src), n, C.addressof(arr), _dev_ptr(d_stats),
                                                   _dev_ptr(d_prev), _np_ptr(flags), C.byref(params),
                                                   ends.ctypes.data, _dev_ptr(d_items), nitems, _dev_ptr(d_out)))

    # ---- temporal RDO
    def block_importances_dev(self, frames, bit_depth, d_intra_costs, d_mvs, steps, d_importances):
        """frames: list of Plane (the window's source luma); steps: [(src, dst, len, mv_index), ...] in
        execution order; d_importances: len(frames) x ceil(W/8)*ceil(H/8) f32, zeroed then propagated."""
        arr = (Plane * len(frames))()
        for k, p in enumerate(frames):
            C.memmove(C.byref(arr[k]), C.byref(p), C.sizeof(Plane))
        st = imp_steps(steps)
        self.check(self.L.b200_block_importances_dev(self.h, len(frames), C.addressof(arr), bit_depth,
                                                     _dev_ptr(d_intra_costs), _dev_ptr(d_mvs), len(steps),
                                                     C.addressof(st), _dev_ptr(d_importances)))

    def distortion_scales_dev(self, frame, d_importances, d_intra_costs, d_scales):
        self.check(self.L.b200_distortion_scales_dev(self.h, C.byref(frame), _dev_ptr(d_importances),
                                                     _dev_ptr(d_intra_costs), _dev_ptr(d_scales)))

    def temporal_scores_dev(self, w_imp, h_imp, d_scales, d_activity=None, d_spatiotemporal=None,
                            d_log_isqrt_mean_scale=None, d_scale4x4=None, scale4x4_stride=0):
        """d_activity None: compute_temporal_scores, else compute_spatiotemporal_scores (include/b200rdo.h)."""
        self.check(self.L.b200_temporal_scores_dev(self.h, w_imp, h_imp, _dev_ptr(d_scales), _dev_ptr(d_activity),
                                                   _dev_ptr(d_spatiotemporal), _dev_ptr(d_log_isqrt_mean_scale),
                                                   _dev_ptr(d_scale4x4), scale4x4_stride))

    def segmentation_optimize_dev(self, d_spatiotemporal, w_imp, h_imp, base_q_idx, bit_depth, ac_q, update_data,
                                  d_prev, d_out):
        """segmentation_optimize (include/b200rdo.h).  ac_q: the 256-entry ac_qlookup table for bit_depth (host
        array); d_prev may be None (SegmentationState::default()); d_out receives one SEGMENTATION_DTYPE record."""
        q = np.ascontiguousarray(ac_q, dtype=np.uint16)
        assert q.shape == (256,)
        self.check(self.L.b200_segmentation_optimize_dev(self.h, _dev_ptr(d_spatiotemporal), w_imp, h_imp,
                                                         int(base_q_idx), int(bit_depth), q.ctypes.data,
                                                         int(update_data), _dev_ptr(d_prev), _dev_ptr(d_out)))

    def select_segment_dev(self, d_items, n, d_scales, d_activity, w_imp, h_imp, scales_off, level, d_seg, d_sidx,
                           d_scale=None):
        """select_segment for n SEGMENT_ITEM_DTYPE items: d_sidx (n x 2 u8) and d_scale (n u32, may be None)."""
        self.check(self.L.b200_select_segment_dev(self.h, _dev_ptr(d_items), n, _dev_ptr(d_scales),
                                                  _dev_ptr(d_activity), w_imp, h_imp, int(scales_off), int(level),
                                                  _dev_ptr(d_seg), _dev_ptr(d_sidx), _dev_ptr(d_scale)))

    def coeff_rate_dev(self, d_cdfs, ncdfs, d_chains, nchains, d_items, nitems, d_qcoeffs, ncoeffs, coeff_is_i32,
                       d_rate, d_cul_level=None):
        """write_coeffs_lv_map's rate for nchains COEFF_CHAIN_DTYPE chains (include/b200rdo.h): d_rate (nchains
        u32, 1/8 bit, UINT32_MAX for an invalid chain) and d_cul_level (nitems u8, may be None)."""
        self.check(self.L.b200_coeff_rate_dev(self.h, _dev_ptr(d_cdfs), ncdfs, _dev_ptr(d_chains), nchains,
                                              _dev_ptr(d_items), nitems, _dev_ptr(d_qcoeffs), ncoeffs,
                                              int(coeff_is_i32), _dev_ptr(d_rate), _dev_ptr(d_cul_level)))

    def intra_tx_size_type_dev(self, rec, src, rect, width, height, bit_depth, dist_mode, reduced_tx_set, lam,
                               dist_scale, d_scale4x4, scale_stride, d_cdfs, ncdfs, d_items, n, d_best, d_cands=None):
        """rdo_tx_size_type for n TX_ITEM_DTYPE items (include/b200rdo.h): rect = (x, y, w, h) of the tile region;
        width / height = fi.width / fi.height; dist_mode 0 tx-domain, 1 sse, 2 cdef_dist; d_scale4x4 (per frame
        4x4, scale_stride entries per row) may be None; d_best (n TX_BEST_DTYPE) and d_cands (n x 21
        TX_CAND_DTYPE, may be None)."""
        self.check(self.L.b200_intra_tx_size_type_dev(self.h, C.byref(rec), C.byref(src), rect[0], rect[1], rect[2],
                                                      rect[3], width, height, bit_depth, dist_mode, reduced_tx_set,
                                                      float(lam), int(dist_scale), _dev_ptr(d_scale4x4), scale_stride,
                                                      _dev_ptr(d_cdfs), ncdfs, _dev_ptr(d_items), n, _dev_ptr(d_best),
                                                      _dev_ptr(d_cands)))

    # ---- RDO cost
    def compute_rd_cost_dev(self, lam, d_rate, d_dist, n, d_cost=None, d_offsets=None, ngroups=0, d_best=None):
        self.check(self.L.b200_compute_rd_cost_dev(self.h, float(lam), _dev_ptr(d_rate), _dev_ptr(d_dist), n,
                                                   _dev_ptr(d_offsets), ngroups, _dev_ptr(d_cost), _dev_ptr(d_best)))

    # ---- RDO distortion
    def weighted_sse_dev(self, src1, src2, d_blocks, n, w, h, d_scale, scale_stride, d_out):
        self.check(self.L.b200_weighted_sse_dev(self.h, C.byref(src1), C.byref(src2), _dev_ptr(d_blocks), n,
                                                w, h, _dev_ptr(d_scale), scale_stride, _dev_ptr(d_out)))

    def activity_mask_dev(self, luma, bit_depth, d_variances, d_scales=None):
        self.check(self.L.b200_activity_mask_dev(self.h, C.byref(luma), bit_depth, _dev_ptr(d_variances),
                                                 _dev_ptr(d_scales)))

    def cdef_dist_dev(self, src, dst, d_blocks, n, w, h, bit_depth, d_out=None, d_raw=None):
        self.check(self.L.b200_cdef_dist_dev(self.h, C.byref(src), C.byref(dst), _dev_ptr(d_blocks), n, w, h,
                                             bit_depth, _dev_ptr(d_out), _dev_ptr(d_raw)))

    # ---- motion compensation
    def mc_blocks_dev(self, ref, d_blocks, d_mvs, n, w, h, mode_x, mode_y, bit_depth, xdec, ydec,
                      kind, d_out):
        self.check(self.L.b200_mc_blocks_dev(self.h, C.byref(ref), _dev_ptr(d_blocks), _dev_ptr(d_mvs),
                                             n, w, h, mode_x, mode_y, bit_depth, xdec, ydec, kind,
                                             _dev_ptr(d_out)))

    def mc_avg_dev(self, d_t1, d_t2, d_dst, n, w, h, bit_depth):
        self.check(self.L.b200_mc_avg_dev(self.h, _dev_ptr(d_t1), _dev_ptr(d_t2), _dev_ptr(d_dst),
                                          n, w, h, bit_depth))

    # ---- CDEF
    def cdef_find_dir_dev(self, luma, bit_depth, d_skip8, d_dir, d_var):
        self.check(self.L.b200_cdef_find_dir_dev(self.h, C.byref(luma), bit_depth, _dev_ptr(d_skip8),
                                                 _dev_ptr(d_dir), _dev_ptr(d_var)))

    def cdef_filter_plane_dev(self, inp, out, plane, xdec, ydec, luma_w, luma_h, bit_depth, damping,
                              d_skip8, d_dir, d_var, d_strength_sb):
        self.check(self.L.b200_cdef_filter_plane_dev(
            self.h, C.byref(inp), C.byref(out), plane, xdec, ydec, luma_w, luma_h, bit_depth,
            damping, _dev_ptr(d_skip8), _dev_ptr(d_dir), _dev_ptr(d_var), _dev_ptr(d_strength_sb)))

    def cdef_find_dir_rect_dev(self, luma, bit_depth, d_skip8, d_dir, d_var, rect8):
        self.check(self.L.b200_cdef_find_dir_rect_dev(self.h, C.byref(luma), bit_depth, _dev_ptr(d_skip8),
                                                      _dev_ptr(d_dir), _dev_ptr(d_var), *rect8))

    def cdef_filter_rect_dev(self, inp, out, plane, xdec, ydec, luma_w, luma_h, bit_depth, damping, d_skip8, d_dir,
                             d_var, d_strength_sb, rect8):
        self.check(self.L.b200_cdef_filter_rect_dev(
            self.h, C.byref(inp), C.byref(out), plane, xdec, ydec, luma_w, luma_h, bit_depth, damping,
            _dev_ptr(d_skip8), _dev_ptr(d_dir), _dev_ptr(d_var), _dev_ptr(d_strength_sb), *rect8))

    def cdef_tiles_dev(self, items, plane, xdec, ydec, luma_w, luma_h, bit_depth, damping, d_strength_sb,
                       find_dir=True, filter=True):
        """items: a ctypes array of CdefItem (keep the Plane objects it points to alive)."""
        self.check(self.L.b200_cdef_tiles_dev(self.h, C.addressof(items), len(items), plane, xdec, ydec, luma_w,
                                              luma_h, bit_depth, damping, _dev_ptr(d_strength_sb), int(find_dir),
                                              int(filter)))

    def cdef_rdo_dev(self, rec, src, out, xdec, ydec, width, height, bit_depth, damping, cdef_bits, y_strengths,
                     uv_strengths, d_skip8, d_imp_scales, dist_scale, lam, areas, d_rate, d_err, d_cost, d_best):
        """rec / src / out: lists of 1 or 3 Plane (out may be None); areas: [(sbx, sby, sb_w, sb_h), ...];
        d_err (n_areas * 16 * 8 u64), d_cost (same, f64), d_best (n_areas * 16 i8) (include/b200rdo.h)."""
        def arr(planes):
            if planes is None:
                return None
            a = (Plane * len(planes))()
            for k, p in enumerate(planes):
                C.memmove(C.byref(a[k]), C.byref(p), C.sizeof(Plane))
            return a
        r, s_, o = arr(rec), arr(src), arr(out)
        ar = np.ascontiguousarray(np.asarray(areas, np.int32).reshape(-1, 4))   # b200_cdef_rdo_area rows
        ys = (C.c_uint8 * 8)(*[int(v) for v in y_strengths])
        us = (C.c_uint8 * 8)(*[int(v) for v in uv_strengths])
        ds = (C.c_uint32 * 3)(*[int(v) for v in dist_scale])
        self.check(self.L.b200_cdef_rdo_dev(
            self.h, C.addressof(r), C.addressof(s_), C.addressof(o) if o is not None else None, len(rec), xdec, ydec,
            width, height, bit_depth, damping, cdef_bits, C.addressof(ys), C.addressof(us), _dev_ptr(d_skip8),
            _dev_ptr(d_imp_scales), C.addressof(ds), float(lam), ar.ctypes.data, len(areas), _dev_ptr(d_rate),
            _dev_ptr(d_err), _dev_ptr(d_cost), _dev_ptr(d_best)))

    # ---- deblocking
    @staticmethod
    def _plane_array(planes):
        a = (Plane * len(planes))()
        for k, p in enumerate(planes):
            C.memmove(C.byref(a[k]), C.byref(p), C.sizeof(Plane))
        return a

    @staticmethod
    def _deblock_items(items):
        """DEBLOCK_ITEM_DTYPE records or rows of six ints -> a contiguous (n, 6) int32 array."""
        a = np.ascontiguousarray(items)
        if a.dtype.names:
            a = a.view(np.int32)
        return np.ascontiguousarray(np.asarray(a, np.int32).reshape(-1, 6))

    def deblock_levels_dev(self, rec, src, xdec, ydec, bit_depth, d_mi, mi_stride, items, d_levels, d_tally=None):
        """rec / src: lists of 1 or 3 Plane; d_mi: DEBLOCK_MI_DTYPE records on the device, mi_stride per row;
        items: a host DEBLOCK_ITEM_DTYPE array (or rows of (mi_x, mi_y, mi_w, mi_h, vis_w, vis_h)); d_levels
        (4 u8 per item) and d_tally (items x 3 x 2 x 64 i64, may be None) on the device (include/b200rdo.h)."""
        r, s_ = self._plane_array(rec), self._plane_array(src)
        it = self._deblock_items(items)
        self.check(self.L.b200_deblock_levels_dev(self.h, C.addressof(r), C.addressof(s_), len(rec), xdec, ydec,
                                                  bit_depth, _dev_ptr(d_mi), mi_stride, it.ctypes.data, len(it),
                                                  _dev_ptr(d_levels), _dev_ptr(d_tally)))

    def deblock_filter_dev(self, inp, out, xdec, ydec, bit_depth, state, d_levels, d_mi, mi_stride, items):
        """inp / out: lists of 1 or 3 Plane; state: a DEBLOCK_STATE_DTYPE scalar array; d_levels: 4 u8 per item
        on the device; the rest as deblock_levels_dev."""
        i_, o = self._plane_array(inp), self._plane_array(out)
        it = self._deblock_items(items)
        st = np.ascontiguousarray(np.asarray(state, DEBLOCK_STATE_DTYPE).reshape(1))
        self.check(self.L.b200_deblock_filter_dev(self.h, C.addressof(i_), C.addressof(o), len(inp), xdec, ydec,
                                                  bit_depth, st.ctypes.data, _dev_ptr(d_levels), _dev_ptr(d_mi),
                                                  mi_stride, it.ctypes.data, len(it)))

    # ---- loop restoration
    def lrf_filter_dev(self, cdeffed, deblocked, out, xdec, ydec, frame_w, frame_h, bit_depth, enable_cdef,
                       unit_size, units):
        """cdeffed / deblocked / out: lists of 1 or 3 Plane; unit_size: one per plane; units: one host
        LRF_UNIT_DTYPE array per plane, (rows, cols) or flat in row-major order (include/b200rdo.h)."""
        c_, d_, o = self._plane_array(cdeffed), self._plane_array(deblocked), self._plane_array(out)
        n = len(cdeffed)
        recs = [np.ascontiguousarray(np.asarray(u, LRF_UNIT_DTYPE).reshape(-1)) for u in units]
        us = (C.c_int * 3)(*[int(v) for v in unit_size], *([0] * (3 - len(unit_size))))
        ptrs = (C.c_void_p * 3)(*[r.ctypes.data for r in recs], *([None] * (3 - len(recs))))
        self.check(self.L.b200_lrf_filter_dev(self.h, C.addressof(c_), C.addressof(d_), C.addressof(o), n, xdec, ydec,
                                              frame_w, frame_h, bit_depth, int(enable_cdef), C.addressof(us),
                                              C.addressof(ptrs)))

    def lrf_search_dev(self, lrf_in, src, xdec, ydec, frame_w, frame_h, bit_depth, unit_size, reduced_sets,
                       d_imp_scales, dist_scale, lam, areas, items, d_best, d_cost, d_changed, d_xqd=None, d_err=None,
                       d_cand_cost=None):
        """lrf_in / src: lists of 1 or 3 Plane; areas: [(sbx, sby, sb_w, sb_h), ...]; items: a host
        LRF_SEARCH_ITEM_DTYPE array; outputs on the device: d_best (LRF_UNIT_DTYPE per item), d_cost (f64),
        d_changed (u8), optional d_xqd (items x 16 x 2 i8), d_err (items x 17 u64), d_cand_cost (items x 17
        f64) (include/b200rdo.h)."""
        i_, s_ = self._plane_array(lrf_in), self._plane_array(src)
        ar = np.ascontiguousarray(np.asarray(areas, np.int32).reshape(-1, 4))
        it = np.ascontiguousarray(np.asarray(items, LRF_SEARCH_ITEM_DTYPE).reshape(-1))
        us = (C.c_int * 3)(*[int(v) for v in unit_size], *([0] * (3 - len(unit_size))))
        ds = (C.c_uint32 * 3)(*[int(v) for v in dist_scale])
        self.check(self.L.b200_lrf_search_dev(
            self.h, C.addressof(i_), C.addressof(s_), len(lrf_in), xdec, ydec, frame_w, frame_h, bit_depth,
            C.addressof(us), int(reduced_sets), _dev_ptr(d_imp_scales), C.addressof(ds), float(lam), ar.ctypes.data,
            len(ar), it.ctypes.data, len(it), _dev_ptr(d_best), _dev_ptr(d_cost), _dev_ptr(d_changed),
            _dev_ptr(d_xqd), _dev_ptr(d_err), _dev_ptr(d_cand_cost)))

    def loop_decision_dev(self, rec, src, work, xdec, ydec, frame_w, frame_h, bit_depth, enable_cdef, damping,
                          cdef_bits, y_strengths, uv_strengths, d_skip8, enable_restoration, unit_size, reduced_sets,
                          d_imp_scales, dist_scale, lam, areas, units, sb_unit, d_best_index, d_unit, d_unit_cost,
                          d_written, d_err=None, d_cost=None):
        """rdo_loop_decision's pass loop (include/b200rdo.h).  rec / src / work: lists of 1 or 3 Plane; areas:
        [(sbx, sby, sb_w, sb_h), ...]; units: a host LOOP_UNIT_DTYPE array; sb_unit: n_areas x 16 x 3 int32 unit
        indices or -1; outputs on the device: d_best_index (n_areas * 16 i8), d_unit (LRF_UNIT_DTYPE per unit),
        d_unit_cost (f64), d_written (u8), optional d_err / d_cost (n_areas * 16 * 8).  Synchronises the
        stream; returns the stage count (-1: still changing after B200_LOOP_MAX_STAGES)."""
        r, s_, w = self._plane_array(rec), self._plane_array(src), self._plane_array(work)
        ar = np.ascontiguousarray(np.asarray(areas, np.int32).reshape(-1, 4))
        un = np.ascontiguousarray(np.asarray(units, LOOP_UNIT_DTYPE).reshape(-1))
        mp = np.ascontiguousarray(np.asarray(sb_unit, np.int32).reshape(-1))
        ys = (C.c_uint8 * 8)(*[int(v) for v in y_strengths])
        us_ = (C.c_uint8 * 8)(*[int(v) for v in uv_strengths])
        usz = (C.c_int * 3)(*[int(v) for v in unit_size], *([0] * (3 - len(unit_size))))
        ds = (C.c_uint32 * 3)(*[int(v) for v in dist_scale])
        stages = C.c_int(0)
        self.check(self.L.b200_loop_decision_dev(
            self.h, C.addressof(r), C.addressof(s_), C.addressof(w), len(rec), xdec, ydec, frame_w, frame_h,
            bit_depth, int(enable_cdef), damping, cdef_bits, C.addressof(ys), C.addressof(us_), _dev_ptr(d_skip8),
            int(enable_restoration), C.addressof(usz), int(reduced_sets), _dev_ptr(d_imp_scales), C.addressof(ds),
            float(lam), ar.ctypes.data, len(ar), un.ctypes.data if len(un) else None, len(un), mp.ctypes.data,
            _dev_ptr(d_best_index), _dev_ptr(d_unit), _dev_ptr(d_unit_cost), _dev_ptr(d_written), _dev_ptr(d_err),
            _dev_ptr(d_cost), C.byref(stages)))
        return stages.value

    # ---- intra prediction
    def predict_intra_dev(self, d_edges, d_items, n, d_ac, w, h, bit_depth, plane_w, plane_h, d_out):
        self.check(self.L.b200_predict_intra_dev(self.h, _dev_ptr(d_edges), _dev_ptr(d_items), n,
                                                 _dev_ptr(d_ac), w, h, bit_depth, plane_w, plane_h,
                                                 _dev_ptr(d_out)))

    def get_intra_edges_dev(self, plane, rect, xdec, ydec, bit_depth, d_items, n, d_edges, d_lens=None):
        self.check(self.L.b200_get_intra_edges_dev(self.h, C.byref(plane), rect[0], rect[1], rect[2], rect[3], xdec,
                                                   ydec, bit_depth, _dev_ptr(d_items), n, _dev_ptr(d_edges),
                                                   _dev_ptr(d_lens)))

    def intra_mode_screen_dev(self, rec, src, rect, bit_depth, num_modes_rdo, d_items, n, d_satd, d_modes):
        """rect = (x, y, w, h) of the tile region; d_items: INTRA_SCREEN_ITEM_DTYPE on the device;
        d_satd (n x 13 u32) and d_modes (n x 13 u8) may each be None."""
        self.check(self.L.b200_intra_mode_screen_dev(self.h, C.byref(rec), C.byref(src), rect[0], rect[1], rect[2],
                                                     rect[3], bit_depth, num_modes_rdo, _dev_ptr(d_items), n,
                                                     _dev_ptr(d_satd), _dev_ptr(d_modes)))

    def inter_mode_screen_dev(self, src, rect, refs, xorigin, yorigin, filter_mode, bit_depth, d_items, n, d_satd,
                              d_order):
        """rect = (x, y, w, h) of the tile region; refs: a list of Plane (the entries' `ref` indices address
        it); d_items: INTER_SCREEN_ITEM_DTYPE on the device; d_satd (n x 20 u32) and d_order (n x 20 u8) may
        each be None."""
        arr = (Plane * max(len(refs), 1))()
        for k, p in enumerate(refs):
            C.memmove(C.byref(arr[k]), C.byref(p), C.sizeof(Plane))
        self.check(self.L.b200_inter_mode_screen_dev(self.h, C.byref(src), rect[0], rect[1], rect[2], rect[3],
                                                     C.addressof(arr), len(refs), xorigin, yorigin, filter_mode,
                                                     bit_depth, _dev_ptr(d_items), n, _dev_ptr(d_satd),
                                                     _dev_ptr(d_order)))

    def cfl_alpha_dev(self, rec, src, xdec, ydec, rect, width, height, bit_depth, d_items, n, d_alpha, d_sse):
        """rec / src: lists of the 3 frame Planes (src[0] is not read); rect = (x, y, w, h) of the tile in luma
        pixels; width / height = fi.width / fi.height; d_items: CFL_ITEM_DTYPE on the device; d_alpha (n x 2 i8)
        and d_sse (n x 2 x 33 u64) may each be None (include/b200rdo.h)."""
        def arr(planes):
            a = (Plane * 3)()
            for k, p in enumerate(planes):
                C.memmove(C.byref(a[k]), C.byref(p), C.sizeof(Plane))
            return a
        r, s_ = arr(rec), arr(src)
        self.check(self.L.b200_cfl_alpha_dev(self.h, C.addressof(r), C.addressof(s_), xdec, ydec, rect[0], rect[1],
                                             rect[2], rect[3], width, height, bit_depth, _dev_ptr(d_items), n,
                                             _dev_ptr(d_alpha), _dev_ptr(d_sse)))

    def pred_cfl_ac_dev(self, luma, d_blocks, n, bw, bh, w_pad, h_pad, xdec, ydec, d_ac):
        self.check(self.L.b200_pred_cfl_ac_dev(self.h, C.byref(luma), _dev_ptr(d_blocks), n, bw, bh,
                                               w_pad, h_pad, xdec, ydec, _dev_ptr(d_ac)))

    # ---- forward transform
    def fwd_txfm_dev(self, d_in, in_block_stride, in_row_stride, d_out, n, tx_size, tx_type, bd,
                     coeff_i32):
        self.check(self.L.b200_fwd_txfm_dev(self.h, _dev_ptr(d_in), in_block_stride, in_row_stride,
                                            _dev_ptr(d_out), n, tx_size, tx_type, bd, int(coeff_i32)))

    def fwd_txfm_residual_dev(self, cur, ref, d_blocks, nblocks, d_mv_src, d_out, tx_size, tx_type, bd):
        self.check(self.L.b200_fwd_txfm_residual_dev(self.h, C.byref(cur), C.byref(ref),
                                                     _dev_ptr(d_blocks), nblocks, _dev_ptr(d_mv_src),
                                                     _dev_ptr(d_out), tx_size, tx_type, bd))

    def fwd_txfm_residual_multi_dev(self, pairs, d_blocks, nblocks, d_mv_src, d_out, tx_size, tx_type, bd):
        self.check(self.L.b200_fwd_txfm_residual_multi_dev(
            self.h, pairs.n, C.addressof(pairs.curs), C.addressof(pairs.refs),
            pairs.block_end.ctypes.data, _dev_ptr(d_blocks), nblocks, _dev_ptr(d_mv_src),
            _dev_ptr(d_out), tx_size, tx_type, bd))

    def fwd_txfm_pred_dev(self, cur, d_pred, d_blocks, nblocks, d_out, tx_size, tx_type, bd):
        self.check(self.L.b200_fwd_txfm_pred_dev(self.h, C.byref(cur), _dev_ptr(d_pred), _dev_ptr(d_blocks),
                                                 nblocks, _dev_ptr(d_out), tx_size, tx_type, bd))

    def fwd_txfm_batch(self, residual, tx_size, tx_type, bd=8, coeff_i32=None, out=None):
        """residual: int16 (n, h, w) numpy -> (n, w*h) coefficients (host buffers, copies inside)."""
        residual = np.ascontiguousarray(residual, dtype=np.int16)
        n, h, w = residual.shape
        if coeff_i32 is None:
            coeff_i32 = bd > 8
        if out is None:
            out = np.empty((n, w * h), np.int32 if coeff_i32 else np.int16)
        self.check(self.L.b200_fwd_txfm_batch(self.h, residual.ctypes.data, h * w, w,
                                              out.ctypes.data, n, tx_size, tx_type, bd,
                                              int(coeff_i32)))
        return out

    # ---- ME, host buffers (numpy in / numpy out; copies inside)
    def me_candidates_batch(self, cur_hp, ref_hp, blocks, cands, params, offsets=None, pmv=None,
                            want_sad=True, want_cost=False, want_best=False, out=None):
        """`out` = optional (sad, cost, best) preallocated (e.g. pinned) numpy arrays."""
        n, nb = len(cands), len(blocks)
        if out is not None:
            sad, cost, best = out
        else:
            sad = np.empty(n, np.uint32) if want_sad else None
            cost = np.empty(n, np.uint64) if want_cost else None
            best = np.empty(nb, ME_RESULT_DTYPE) if want_best else None
        self.check(self.L.b200_me_candidates_batch(
            self.h, C.byref(cur_hp), C.byref(ref_hp), _np_ptr(blocks), nb, _np_ptr(cands), n,
            _np_ptr(offsets), _np_ptr(pmv), C.byref(params), _np_ptr(sad), _np_ptr(cost),
            _np_ptr(best)))
        return sad, cost, best

    def set_async(self, enable=True):
        self.check(self.L.b200_ctx_set_async(self.h, int(enable)))

    def plane_upload(self, plane, img):
        self.check(self.L.b200_plane_upload(self.h, C.byref(plane), img.ctypes.data, img.strides[0]))

    def me_candidates_resident(self, cur, ref, blocks, cands, params, offsets, out, pmv=None):
        """Resident planes, host descriptors; `out` = (sad|None, cost|None, best|None) host arrays."""
        sad, cost, best = out
        self.check(self.L.b200_me_candidates_resident(
            self.h, C.byref(cur), C.byref(ref), _np_ptr(blocks), len(blocks), _np_ptr(cands),
            len(cands), _np_ptr(offsets), _np_ptr(pmv), C.byref(params), _np_ptr(sad), _np_ptr(cost),
            _np_ptr(best)))

    def me_mvs_resident(self, cur, ref, blocks, mvs, params, offsets, out, pmv=None):
        """Like me_candidates_resident with the candidates as an (n, 2) int16 array of
        (row, col) MotionVectors; the CSR `offsets` names each candidate's block."""
        sad, cost, best = out
        self.check(self.L.b200_me_mvs_resident(
            self.h, C.byref(cur), C.byref(ref), _np_ptr(blocks), len(blocks), _np_ptr(mvs), len(mvs),
            _np_ptr(offsets), _np_ptr(pmv), C.byref(params), _np_ptr(sad), _np_ptr(cost), _np_ptr(best)))

    def fwd_txfm_residual_resident(self, cur, ref, blocks, mv_src, out, tx_size, tx_type, bd):
        self.check(self.L.b200_fwd_txfm_residual_resident(
            self.h, C.byref(cur), C.byref(ref), _np_ptr(blocks), len(blocks), _np_ptr(mv_src),
            out.ctypes.data, tx_size, tx_type, bd))

    def me_full_search_batch(self, cur_hp, ref_hp, blocks, params, range_x, range_y, step):
        best = np.empty(len(blocks), ME_RESULT_DTYPE)
        self.check(self.L.b200_me_full_search_batch(
            self.h, C.byref(cur_hp), C.byref(ref_hp), _np_ptr(blocks), len(blocks),
            C.byref(params), range_x, range_y, step, _np_ptr(best)))
        return best


class FramePipe:
    """b200_frame_pipe: one per context; push() one frame per call (include/b200rdo.h)."""

    def __init__(self, ctx, width, height, pad, block=(16, 16), lambda_=0, sad_per_block=0, satd_per_block=0,
                 window_hint_px=0, tx_size=-1, tx_type=0, dc_quant=0, ac_quant=0, bit_depth=8):
        self.ctx = ctx
        cfg = FramePipeCfg(width, height, pad, 1 if bit_depth == 8 else 2, bit_depth, block[0], block[1], lambda_,
                           sad_per_block, satd_per_block, window_hint_px, tx_size, tx_type, dc_quant, ac_quant)
        h = C.c_void_p()
        ctx.check(ctx.L.b200_frame_pipe_create(ctx.h, C.byref(cfg), C.byref(h)))
        self.h = h
        self.cfg = cfg
        self.nblocks = int(ctx.L.b200_frame_pipe_nblocks(h))

    def push(self, frame, sad_offsets=None, satd_offsets=None, centers=None, best_sad=None, best_satd=None,
             coeffs=None, eob=None, tx_dist=None):
        """frame: 2-D numpy array (visible area); lists / outputs: numpy arrays (pinned for speed)."""
        self.ctx.check(self.ctx.L.b200_frame_pipe_push(
            self.h, frame.ctypes.data, frame.strides[0], _np_ptr(sad_offsets), _np_ptr(satd_offsets), _np_ptr(centers),
            _np_ptr(best_sad), _np_ptr(best_satd), _np_ptr(coeffs), _np_ptr(eob), _np_ptr(tx_dist)))

    def set_lists(self, sad_offsets, satd_offsets, centers=None):
        """upload the candidate lists once: later pushes may leave them out (only the frame crosses PCIe)"""
        self.ctx.check(self.ctx.L.b200_frame_pipe_set_lists(self.h, _np_ptr(sad_offsets), _np_ptr(satd_offsets),
                                                            _np_ptr(centers)))

    def push_packed(self, frame, best_sad=None, best_satd=None, eob=None, tx_dist=None, packed=None):
        """quantizing pipe with resident lists: per block eob + tx-domain distortion, and in `packed` only the eob
        quantized coefficients of each block in scan order, block after block.  Returns their total count (which may
        exceed len(packed): then only len(packed) were copied)."""
        n = C.c_size_t(0)
        cap = 0 if packed is None else packed.size
        self.ctx.check(self.ctx.L.b200_frame_pipe_push_packed(
            self.h, frame.ctypes.data, frame.strides[0], _np_ptr(best_sad), _np_ptr(best_satd), _np_ptr(eob),
            _np_ptr(tx_dist), _np_ptr(packed), cap, C.byref(n)))
        return int(n.value)

    def close(self):
        if self.h:
            self.ctx.L.b200_frame_pipe_destroy(self.h)
            self.h = None


def host_plane(arr2d_full, pad):
    """HostPlane over a numpy array that already contains `pad` border pixels on each side."""
    a = arr2d_full
    assert a.ndim == 2 and a.flags.c_contiguous
    h, w = a.shape[0] - 2 * pad, a.shape[1] - 2 * pad
    hp = HostPlane()
    hp.data = a.ctypes.data + pad * a.strides[0] + pad * a.itemsize
    hp.stride = a.strides[0]
    hp.width, hp.height, hp.pad, hp.bpp = w, h, pad, a.itemsize
    hp._keep = a
    return hp


def me_params(w, h, frame_w, frame_h, lambda_=0, allow_hp=False, use_satd=False, bit_depth=8,
              window_hint_px=0):
    p = MeParams()
    p.w, p.h = w, h
    p.frame_w_in_b = 2 * ((frame_w + 7) >> 3)   # encoder.rs:852
    p.frame_h_in_b = 2 * ((frame_h + 7) >> 3)
    p.lambda_ = lambda_
    p.allow_high_precision_mv = int(allow_hp)
    p.use_satd = int(use_satd)
    p.bit_depth = bit_depth
    p.window_hint_px = window_hint_px
    return p
