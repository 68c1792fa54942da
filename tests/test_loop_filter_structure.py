"""The loop-filter RDO keeps one copy of each shared piece: the restoration search's kernels are defined and
launched only in csrc/lrf_search.cu (b200_lrf_search_dev and the pass loop of b200_loop_decision_dev both go
through lrf_search_launch), and the CDEF tile filter is called only from the superblock evaluation that
b200_cdef_rdo_dev and the pass loop share (csrc/cdef_sb_dev.cuh) and from the frame filter (csrc/cdef.cu)."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rav1e_b200", "csrc")


def _code():
    out = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".h")):
            with open(os.path.join(CSRC, f)) as fh:
                out[f] = re.sub(r"//[^\n]*|/\*.*?\*/", "", fh.read(), flags=re.S)
    return out


def _files_matching(pattern):
    return sorted(f for f, s in _code().items() if re.search(pattern, s))


def test_restoration_search_kernels_live_in_lrf_search_cu():
    for k in ("lrf_search_tiles", "lrf_search_solve", "lrf_search_decide"):
        assert _files_matching(r"__global__[^;{]*\b" + k + r"\s*\(") == ["lrf_search.cu"], k
        assert _files_matching(r"\b" + k + r"\b[^;]*<<<") == ["lrf_search.cu"], k
    assert _files_matching(r"\blrf_search_tiles<") == ["lrf_search.cu"]


def test_cdef_tile_filter_called_from_superblock_header_and_frame_filter():
    calls = r"(?<!int )\bcdef_filter_tile_px\s*\("  # a call, not the definition in cdef_dev.cuh
    assert _files_matching(calls) == ["cdef.cu", "cdef_sb_dev.cuh"]
