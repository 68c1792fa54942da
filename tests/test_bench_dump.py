"""bench.py --dump-outputs without a GPU: step_outputs on CPU tensors laid out like the timed step's buffers.  The
files are float32 / float64, hold exactly the values of the rows they name, come out the same from two calls, and
stay under the 64 MB limit at any frame count (whole outputs at one frame, seeded samples at many)."""
import numpy as np
import pytest
import torch

import bench
from rav1e_b200 import backend as B

NB = bench.BW * bench.BH  # coefficients per 16x16 block


def buffers(F, nb, fill):
    n_sad, n_satd = nb * bench.CAND_SAD, nb * bench.CAND_SATD
    g = torch.Generator().manual_seed(F)
    make = (lambda n, hi, dt: torch.randint(0, hi, (n,), generator=g, dtype=dt)) if fill else \
        (lambda n, hi, dt: torch.empty(n, dtype=dt))
    d_sad = make(F * n_sad, 65281, torch.int32).view(torch.uint8)
    d_satd = make(F * n_satd, 65281, torch.int32).view(torch.uint8)
    d_best = make(F * nb * 16, 256, torch.uint8)
    d_best2 = make(F * nb * 16, 256, torch.uint8)
    d_coef = make(F * nb * NB, 4096, torch.int16)
    return (F, nb, n_sad, n_satd, d_sad, d_satd, d_best, d_best2, d_coef)


def test_one_frame_is_dumped_whole_and_exactly(tmp_path):
    args = buffers(1, 8160, fill=True)
    F, nb, n_sad, n_satd, d_sad, d_satd, d_best, d_best2, d_coef = args
    out = bench.step_outputs(*args)
    assert all(a.dtype in (np.float32, np.float64) for a in out.values())
    np.testing.assert_array_equal(out["block_index"], np.arange(F * nb))
    np.testing.assert_array_equal(out["sad_candidates"], d_sad.view(torch.int32).numpy())
    np.testing.assert_array_equal(out["satd_candidates"], d_satd.view(torch.int32).numpy())
    np.testing.assert_array_equal(out["coef"], d_coef.view(-1, NB).numpy())
    best = d_best2.numpy().view(B.ME_RESULT_DTYPE)
    np.testing.assert_array_equal(out["satd_winner_cost"], best["cost"].astype(np.float64))
    np.testing.assert_array_equal(out["satd_winner_mv_col"], best["mv_col"])
    again = bench.step_outputs(*args)
    assert all(np.array_equal(out[k], again[k]) for k in out)
    bench.dump_outputs(str(tmp_path), out)
    assert sorted(p.name for p in tmp_path.iterdir()) == sorted(k + ".npy" for k in out)
    np.testing.assert_array_equal(np.load(tmp_path / "coef.npy"), out["coef"])


@pytest.mark.parametrize("F", [32, 80])
def test_many_frames_are_sampled_within_the_limit(F):
    args = buffers(F, 8160, fill=False)
    out = bench.step_outputs(*args)
    assert sum(a.nbytes for a in out.values()) <= bench.DUMP_LIMIT
    assert len(out["sad_candidates"]) == bench.DUMP_CANDIDATES == len(out["satd_candidates"])
    assert len(out["coef"]) == bench.DUMP_COEF_BLOCKS
    assert len(out["sad_winner_sad"]) == min(F * 8160, bench.DUMP_BLOCKS)
    idx = out["sad_candidates_index"].astype(np.int64)
    np.testing.assert_array_equal(out["sad_candidates"], args[4].view(torch.int32).numpy()[idx].view(np.uint32).astype(np.float32))
    np.testing.assert_array_equal(idx, bench.step_outputs(*args)["sad_candidates_index"])
