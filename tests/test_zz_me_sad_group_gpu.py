"""B200_SAD_GROUP, the cooperative SAD kernel's group width, is read once per process: the
block-order cases of test_me_cand_edges_gpu.py run again in a fresh process with it set.  (Named to
run last: the child process profiles the same device.)"""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("group", [1, 16])
def test_sad_group_override(group):
    """B200_SAD_GROUP (the cooperative SAD kernel's group width, read once per process) at 1 and at
    16 = kMaxGroup, the size of the kernel's per-block key array: the block-order cases again, in a
    fresh process with the variable set."""
    env = dict(os.environ, B200_SAD_GROUP=str(group))
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        os.path.join(ROOT, "tests", "test_me_cand_edges_gpu.py"),
                        "-k", "test_nonraster_block_lists and sad_dense and default"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "6 passed" in r.stdout, r.stdout[-2000:]
