"""GPU, two processes: persia_core at replica_size = 2 with PERSIA_B200_GROW=shared, so that every rank's table is
growable and exportable (growth mode 2), read in place by its peer while it grows.

  * Infer (on one GPU, devices = [0, 0], or two): the job of test_gpu_persia_core_remote_infer.py with the switch set
    in the ranks' environment and a checkpoint of about 150,000 signs, so that each rank's table grows as it loads its
    part (pb_image_insert) before its export, and again, rows and an index doubling, as it applies its `.inc` packet
    after the export (frozen): its peer maps those chunks from the socket it registered in _start_remote.  Outputs
    must equal the oracle with 2 parameter servers bit for bit, for summation and raw slots.
  * Train (two GPUs; skipped with fewer): the job of test_gpu_live_remote_dist.py with the switch, so that each
    rank's shard grows while it trains and is exported live when the optimizer is registered, and rank 0 alone
    evaluates mid-training through eval_ctx, reading its peer's growing table.  Rank 0's eval outputs and every final
    entry equal, bit for bit, the same job with eager tables.

The switch reaches the ranks through the environment: torch.multiprocessing.spawn starts them with this process's."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_gpu_persia_core_remote_infer as infer_job  # noqa: E402
from test_gpu_live_remote_dist import _spawn as _train_job  # noqa: E402

pytestmark = pytest.mark.gpu


def _fd_handles():
    import persia_b200.shard as SH
    from persia_b200 import native as N

    s = SH.EmbeddingShard(8, 1024, 0)
    try:
        return N.load().pb_table_set_growth(s.h, 2) == 0
    finally:
        s.close()


def test_infer_job_grows_under_readers(oracle, tmp_path, monkeypatch):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if not _fd_handles():
        pytest.skip("the device cannot export memory as POSIX file descriptors")
    monkeypatch.setenv("PERSIA_B200_GROW", "shared")
    monkeypatch.setenv("PERSIA_B200_CAPACITY", str(1 << 22))
    monkeypatch.delenv("PERSIA_B200_HBM_ROWS", raising=False)
    # (the job's checkpoint, packet and batches are written by this process from CARD; its ranks read the files)
    monkeypatch.setattr(infer_job, "CARD", {"a": 50, "b": 150_000, "r": 20_000})
    infer_job.test_infer_job_two_replicas_serve_alone(oracle, tmp_path)


def test_train_job_grows_under_rank_zero_evals(oracle, tmp_path, monkeypatch):
    import torch

    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    monkeypatch.setenv("PERSIA_B200_CAPACITY", str(1 << 22))
    monkeypatch.delenv("PERSIA_B200_HBM_ROWS", raising=False)
    monkeypatch.delenv("PERSIA_B200_GROW", raising=False)
    base = _train_job(str(tmp_path / "eager"), True)
    monkeypatch.setenv("PERSIA_B200_GROW", "shared")
    grown = _train_job(str(tmp_path / "grown"), True)
    for r in range(2):
        assert len(grown[r][1]) == len(base[r][1])
        for (_, a), (_, b) in zip(grown[r][1], base[r][1]):  # rank 0's evals
            assert a.tobytes() == b.tobytes(), r
        np.testing.assert_array_equal(grown[r][2], base[r][2])
        assert grown[r][3].tobytes() == base[r][3].tobytes(), r
