"""examples/stream_frames.cpp is the C-ABI-only walk through the frame pipe (create, resident lists, one packed push
per frame).  Here: it compiles and links against the shared library with nothing but the public header, and on a
machine without a GPU it fails loudly instead of computing anything on the CPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "rav1e_b200")


def build(tmp_path):
    exe = str(tmp_path / "stream_frames")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "examples/stream_frames.cpp"),
                           "-o", exe, "-L" + PKG, "-lb200rdo", "-Wl,-rpath," + PKG])
    return exe


def test_example_builds_and_refuses_to_run_without_a_gpu(tmp_path):
    import torch
    exe = build(tmp_path)
    if torch.cuda.is_available():
        pytest.skip("GPU present: the run on the device is "
                    "tests/test_frame_pipe_paths_gpu.py::test_stream_frames_example_matches_the_oracle")
    r = subprocess.run([exe, "2"], capture_output=True, text=True)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr

