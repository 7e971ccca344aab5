"""CPU, world_size 2 and 3, gloo: the sharded protocol (tests/exchange_model.py) with two slots sharing a feature group,
against the oracle's embedding worker with R parameter servers.  A sign that both slots hold is two entries of one
rank's request, stepped in slot order; the owner applies the requests in rank order: (r0, a), (r0, b), (r1, a), (r1, b)."""
import os
import socket
import sys

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

S, B, DIM = 3, 64, 8
CARD = [5, 200, 100000]  # slots 0 and 1 share a key space: ids 0..4 of slot 0 are also ids of slot 1
GROUPS = (0, 0, 1)
STEPS = 3


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _batches(R):
    rng = np.random.default_rng(78)
    out = []
    for step in range(STEPS):
        ids = np.stack([np.concatenate([rng.integers(0, CARD[s], size=B, dtype=np.uint64) for s in range(S)]) for _ in range(R)])
        g = (rng.standard_normal((R, S, B, DIM)) * 1e-2).astype(np.float16)
        if step == 1:
            g[0, 1, 3, 2] = np.nan  # rank 0 drops slot 1 of its request; its slot 0 entries of the same signs still apply
        out.append((ids, g))
    return out


def _skip(rank, R, step):
    return [1, 0, 0] if (rank == R - 1 and step == 2) else None  # add_skipped_gradient on slot 0 of the last rank


def _run(rank, port, q, R):
    import oracle
    from exchange_model import ExchangeModel
    from persia_b200.worker import ShardedEmbeddingWorker

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=R)
    try:
        pf = [oracle.index_prefix(g) for g in GROUPS]
        cap = ShardedEmbeddingWorker.calibrate_cap([ids[rank] for ids, _ in _batches(R)], B, pf, R, margin=1.0, extra=0)
        m = ExchangeModel(oracle, pf, DIM, oracle.Optim(oracle.SGD, lr=0.1, wd=0.0), rank, R, cap)
        outs, sts = [], []
        for step, (ids, g) in enumerate(_batches(R)):
            outs.append(m.forward(ids[rank], B).copy())
            sts.append(m.backward(g[rank], skip=_skip(rank, R, step)))
        assert not m.overflow
        probe = oracle.add_prefix(np.arange(400, dtype=np.uint64), 8, pf[0])
        own = probe[oracle.shard_of(probe, R) == rank]
        ent = {int(s): m.ps.get_entry(int(s)) for s in own}
        q.put((rank, outs, sts, {k: v for k, v in ent.items() if v is not None}))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("R", [2, 3])
def test_sharded_protocol_shared_group_equals_oracle(R):
    import oracle

    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_run, args=(r, port, q, R)) for r in range(R)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(R):
        rank, outs, sts, ent = q.get(timeout=180)
        res[rank] = (outs, sts, ent)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0

    pf = [oracle.index_prefix(g) for g in GROUPS]
    w = oracle.Worker([oracle.SlotCfg(DIM, prefix=p) for p in pf], n_ps=R)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1, wd=0.0))
    row_off = np.arange(S * B + 1, dtype=np.uint32)
    for step, (ids, g) in enumerate(_batches(R)):
        octx = [w.forward(ids[r], row_off, B, training=True) for r in range(R)]
        for r in range(R):
            for s in range(S):
                np.testing.assert_array_equal(res[r][0][step][s].view(np.uint16), octx[r][0][s].view(np.uint16))
        for r in range(R):
            assert w.backward(octx[r][1], [g[r, s] for s in range(S)], skip=_skip(r, R, step)) == res[r][1][step]
    n = 0
    for r in range(R):
        for sign, e in res[r][2].items():
            ref = w.get_entry(sign)
            assert ref is not None and e.tobytes() == ref.tobytes()
            n += 1
    assert n > 100
