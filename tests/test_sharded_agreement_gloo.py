"""CPU, world_size 2 and 3, gloo: persia_core's per-step agreement on the sharded workers' sizes (_agree_and_resize).
Every rank brings its own local needs (stub workers: no device); all ranks must reach the same agreed needs and the same
resize decisions, and call the workers in the order they were given (the step's collective order)."""
import os
import socket
import sys
import threading

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
