"""Which kernel each case of test_fwd_txfm_fast_gpu.py runs: the file again, in a process of its own with
FWD_TXFM_PROFILE_ROUTES=1, so every case also asserts under torch.profiler that aligned 8-bit DCT_DCT calls
ran fwd_dct_fast_kernel and everything else fwd_txfm_kernel.  The profiler sessions stay out of the suite's
own process.  (Named to run last: the child process profiles the same device.)"""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fwd_txfm_kernel_routes():
    env = dict(os.environ, FWD_TXFM_PROFILE_ROUTES="1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_fwd_txfm_fast_gpu.py")],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "failed" not in r.stdout, r.stdout[-2000:]
