"""The host-buffer and per-call entry points stage through one helper (csrc/host_stage.cuh), opt kernels
in to dynamic shared memory through one per-context function (b200_smem_opt_in, csrc/common.cuh) and
abort through one fatal path (b200_percall_check): no entry point carries its own copy of that plumbing."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rav1e_b200", "csrc")


def _sources():
    out = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".h")):
            with open(os.path.join(CSRC, f)) as fh:
                out[f] = fh.read()
    return out


def _files_calling(name):
    return sorted(f for f, s in _sources().items() if re.search(r"\b" + name + r"\s*\(", s))


def test_stream_ordered_allocation_only_in_host_stage():
    assert _files_calling("cudaMallocAsync") == ["host_stage.cuh"]
    assert _files_calling("cudaFreeAsync") == ["host_stage.cuh"]


def test_smem_opt_in_only_in_common():
    assert _files_calling("cudaFuncSetAttribute") == ["common.cuh"]


def test_one_fatal_path():
    hits = [(f, m) for f, s in _sources().items() for m in re.findall(r'"b200rdo: FATAL[^"]*"', s)]
    assert len(hits) == 1, hits
