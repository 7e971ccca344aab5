"""GPU, two processes: persia_core at replica_size = 2 with PERSIA_B200_SHARED_TIER=1 and PERSIA_B200_HBM_ROWS far
below each rank's entries, so nearly every entry lives in a shared host tier.

  * Infer (on one GPU, devices = [0, 0], or two): the job of test_gpu_persia_core_remote_infer.py run as it is, with
    the switch and 8 HBM rows per rank set in the ranks' environment.  Each rank loads its part of the checkpoint into a
    shard with a shared tier (checkpoint inserts through pb_image_insert), exports it frozen with its tier, opens its
    peer's (the tier's rows through /proc/<pid>/fd), applies an `.inc` packet and serves its requests alone.  About 375
    entries per rank and 8 HBM rows: the outputs, which must equal the oracle with 2 servers bit for bit, are nearly all
    read from tiers, half of them from the other process's host rows.
  * Train (two GPUs; skipped with fewer): the job of test_gpu_live_remote_dist.py with the switch, so each rank's shard
    is created with a shared tier and exported live with it when the optimizer is registered, and rank 0 alone
    evaluates mid-training through the tiered read.  Rank 0's eval outputs and every final entry equal, bit for bit,
    the same job untiered.  The HBM rows hold the run's entries: persia_core's eviction policy frees an eighth of the
    rows every fourth request, which cannot keep up with a batch's new signs at fewer rows, and a refused admission
    (zeros, no gradient) would change the results; entries moving through a live tier beside reads are covered on
    virtual ranks (test_gpu_shared_tier_remote.py).

The switch reaches the ranks through the environment: torch.multiprocessing.spawn starts them with this process's."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_gpu_live_remote_dist import _spawn as _train_job  # noqa: E402
from test_gpu_persia_core_remote_infer import test_infer_job_two_replicas_serve_alone as _infer_job  # noqa: E402

pytestmark = pytest.mark.gpu


def _shared_tiers(monkeypatch, hbm_rows, capacity):
    monkeypatch.setenv("PERSIA_B200_SHARED_TIER", "1")
    monkeypatch.setenv("PERSIA_B200_HBM_ROWS", str(hbm_rows))
    monkeypatch.setenv("PERSIA_B200_CAPACITY", str(capacity))


def test_infer_job_with_shared_tiers(oracle, tmp_path, monkeypatch):
    _shared_tiers(monkeypatch, 8, 1 << 14)
    _infer_job(oracle, tmp_path)


def test_train_job_with_shared_tiers_rank_zero_evaluates(oracle, tmp_path, monkeypatch):
    import torch

    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    monkeypatch.setenv("PERSIA_B200_CAPACITY", str(1 << 16))
    base = _train_job(str(tmp_path / "plain"), True)
    _shared_tiers(monkeypatch, 4096, 1 << 16)  # (each rank's table holds about 2,300 signs at the end)
    tiered = _train_job(str(tmp_path / "tiered"), True)
    for r in range(2):
        assert len(tiered[r][1]) == len(base[r][1])
        for (_, a), (_, b) in zip(tiered[r][1], base[r][1]):  # rank 0's evals
            assert a.tobytes() == b.tobytes(), r
        np.testing.assert_array_equal(tiered[r][2], base[r][2])
        assert tiered[r][3].tobytes() == base[r][3].tobytes(), r
