"""CPU, world_size 2 and 3, gloo: persia_core's per-step agreement on the sharded workers' sizes (_agree_and_resize).
Every rank brings its own local needs (stub workers: no device); all ranks must reach the same agreed needs and the same
resize decisions, and call the workers in the order they were given (the step's collective order).  A new worker starts
at cap 8, so its first step is sized by the same agreement."""
import os
import socket
import sys
import threading

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from persia_b200.worker import ShardedEmbeddingWorker as W  # noqa: E402

STEPS = [  # per step, per worker: (need of rank r, f32 of rank r) as functions of r
    [(lambda r: 4 + r, lambda r: False), (lambda r: 3, lambda r: False)],
    [(lambda r: 100 * (r + 1), lambda r: r == 1), (lambda r: 7, lambda r: False)],
    [(lambda r: 50, lambda r: False), (lambda r: 5000 if r == 0 else 1, lambda r: False)],
    [(lambda r: 10, lambda r: False), (lambda r: 2, lambda r: r == 0)],
]


class _Stub:
    """A worker's sizing state without a device: resize decides with ShardedEmbeddingWorker's own rule."""

    grown_cap = staticmethod(W.grown_cap)

    def __init__(self, name, log, cap=8):
        self.name, self.log, self.cap, self.rows_f32 = name, log, cap, False

    def resize(self, need, rows_f32):
        to = W._resize_to(self, need, rows_f32)
        self.log.append((self.name, need, rows_f32, to))
        if to is not None:
            self.cap, self.rows_f32 = to
        return to is not None


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _run(rank, port, q, R):
    from persia_b200 import persia_core as pc

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=R)
    try:
        log = []
        workers = [_Stub("raw:a", log), _Stub("dim32:0", log)]
        groups = [{"lock": threading.Lock()} for _ in workers]
        agreed = []
        for step in STEPS:
            plan = [(g, wk, (need(rank), f32(rank))) for g, wk, (need, f32) in zip(groups, workers, step)]
            agreed.append(pc._agree_and_resize(plan, "cpu"))
        q.put((rank, agreed, log, [(w.cap, w.rows_f32) for w in workers]))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("R", [2, 3])
def test_ranks_agree_on_sizes_and_resizes(R):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_run, args=(r, port, q, R)) for r in range(R)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(R))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = [[(max(n(r) for r in range(R)), any(f(r) for r in range(R))) for n, f in step] for step in STEPS]
    for rank, agreed, log, final in res:
        assert agreed == want, rank
        assert log == res[0][2], rank  # same decisions, same order
        assert [name for name, *_ in log] == ["raw:a", "dim32:0"] * len(STEPS)
        assert final == res[0][3]
    log = res[0][2]
    assert log[0][3] is None and log[2][3] is not None  # grows only when the agreed need exceeds the cap
    assert log[3][3] is None and log[5][3] is not None  # the max of the ranks' needs resizes everyone
    assert res[0][3][0][1] and res[0][3][1][1]  # f32 rows, once needed by any rank, kept


def test_grown_cap_from_a_new_workers_cap():
    """From the cap of 8 a worker starts with, an agreed need n > 8 grows the exchange to 1.5 x n + 1024, rounded up to
    a multiple of 8, up to needs past 2^31; a need of 8 or less keeps cap 8."""
    for n in [*range(9, 10**6 + 1), *range(2**31 - 64, 2**31 + 64), 2**32 - 1]:
        assert W.grown_cap(n, 8) == (int(n * 1.5) + 1024 + 7) // 8 * 8, n
    assert [W.grown_cap(n, 8) for n in range(9)] == [8] * 9


def _ragged_slots(rank):
    rng = np.random.default_rng(5 + rank)
    return [rng.integers(0, c, size=n, dtype=np.uint64) for n, c in zip([300 * (rank + 1), 0, 40], [2**64 - 1, 9, 25])]


def _run_first_step(rank, port, q, R, pf, prefix_bit):
    from persia_b200 import persia_core as pc
    from persia_b200.worker import distinct_per_owner

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=R)
    try:
        wk = _Stub("new", [])
        need = int(distinct_per_owner(_ragged_slots(rank), pf, R, prefix_bit).max())  # (what prepare counts on the GPU)
        pc._agree_and_resize([({"lock": threading.Lock()}, wk, (need, True))], "cpu")
        q.put((rank, wk.cap, wk.rows_f32))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("R", [2, 3])
def test_first_step_sizes_a_new_worker_from_ragged_slots_at_the_prefix_width(oracle, R):
    """A new worker's first step over ragged slots, with and without an index prefix, at a 12-bit prefix width: every
    rank's exchange gets 1.5 x the most distinct signs one rank's batch asks of one owner + 1024, rounded up to a
    multiple of 8, and f32 rows."""
    prefix_bit = 12
    pf = [oracle.index_prefix(0, prefix_bit), 0, oracle.index_prefix(3, prefix_bit)]
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_run_first_step, args=(r, port, q, R, pf, prefix_bit)) for r in range(R)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in range(R))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    worst = 0
    for r in range(R):
        counts = np.zeros(R, np.int64)
        for x, prefix in zip(_ragged_slots(r), pf):
            for owner in oracle.shard_of(np.unique(oracle.add_prefix(x, prefix_bit, prefix)), R):
                counts[owner] += 1
        worst = max(worst, int(counts.max()))
    assert worst > 8
    assert res == [(r, (int(worst * 1.5) + 1024 + 7) // 8 * 8, True) for r in range(R)]
