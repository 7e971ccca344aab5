"""CPU, world_size 2 and 3, gloo: the sharded protocol (tests/exchange_model.py — what csrc/pb_shard.cu implements on the
GPU) against the oracle's embedding worker with R parameter servers, plus the host-side pieces of
persia_b200.worker that need no device: the collective cap calibration and the exchange-area geometry."""
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

S, B, DIM = 3, 64, 8
CARD = [5, 200, 100000]
STEPS = 3


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _batches(R):
    rng = np.random.default_rng(77)
    out = []
    for step in range(STEPS):
        ids = np.stack([np.concatenate([rng.integers(0, CARD[s], size=B, dtype=np.uint64) for s in range(S)]) for _ in range(R)])
        g = (rng.standard_normal((R, S, B, DIM)) * 1e-2).astype(np.float16)
        if step == 1:
            g[0, 1, 3, 2] = np.nan  # rank 0 drops slot 1 of its request
        out.append((ids, g))
    return out


def _run(rank, port, q, R):
    import oracle
    from exchange_model import ExchangeModel
    from persia_b200.worker import ShardedEmbeddingWorker, distinct_per_owner

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=R)
    try:
        pf = [oracle.index_prefix(i) for i in range(S)]
        mine = [ids[rank] for ids, _ in _batches(R)]
        cap = ShardedEmbeddingWorker.calibrate_cap(mine, B, pf, R, margin=1.0, extra=0)  # collective MAX over the ranks
        worst = max(int(distinct_per_owner(ids[r].reshape(S, B), pf, R).max()) for ids, _ in _batches(R) for r in range(R))
        assert cap == (worst + 7) // 8 * 8 and cap < S * B
        m = ExchangeModel(oracle, pf, DIM, oracle.Optim(oracle.SGD, lr=0.1, wd=0.0), rank, R, cap)
        outs, sts = [], []
        for ids, g in _batches(R):
            outs.append(m.forward(ids[rank], B).copy())
            sts.append(m.backward(g[rank], skip=[0, 0, 1] if (rank == R - 1 and len(outs) == 3) else None))
        assert not m.overflow
        probe = np.concatenate([oracle.add_prefix(np.arange(min(c, 400), dtype=np.uint64), 8, pf[i]) for i, c in enumerate(CARD)])
        own = probe[oracle.shard_of(probe, R) == rank]
        ent = {int(s): m.ps.get_entry(int(s)) for s in own}
        q.put((rank, outs, sts, {k: v for k, v in ent.items() if v is not None}))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("R", [2, 3, 4, 5])
def test_sharded_protocol_equals_oracle_requests_in_rank_order(R):
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

    # the reference: R NN workers' batches = R requests; lookups of a step first, then the updates in rank order
    pf = [oracle.index_prefix(i) for i in range(S)]
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
            skip = [0, 0, 1] if (r == R - 1 and step == 2) else None
            assert w.backward(octx[r][1], [g[r, s] for s in range(S)], skip=skip) == res[r][1][step]
    n = 0
    for r in range(R):
        for sign, e in res[r][2].items():
            ref = w.get_entry(sign)
            assert ref is not None and e.tobytes() == ref.tobytes()
            n += 1
    assert n > 100


def _owner_counts(slot_ids, R, prefix_bit):
    """The per-owner count written out in numpy: each slot's distinct prefixed signs, bucketed by farmhash64 % R."""
    from persia_b200.persia_core import farmhash64_np

    counts = np.zeros(R, np.int64)
    spacing = np.uint64((1 << (64 - prefix_bit)) - 1)
    for x, prefix in slot_ids:
        u = np.unique(x % spacing + np.uint64(prefix) if prefix else x)
        counts += np.bincount((farmhash64_np(u) % np.uint64(R)).astype(np.int64), minlength=R)
    return counts


@pytest.mark.parametrize("prefix_bit", [8, 12])
@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_distinct_per_owner_ragged_slots(oracle, R, prefix_bit):
    """Ragged slots with repeats, an empty one, and slots with and without an index prefix (two share one): per owner,
    the distinct signs of each slot, summed over the slots."""
    from persia_b200.worker import distinct_per_owner

    rng = np.random.default_rng(1000 * R + prefix_bit)
    sizes, cards = [300, 0, 1, 257, 64, 500], [50, 10, 3, 1 << 40, 2**64 - 1, 200]
    slot_ids = [rng.integers(0, c, size=n, dtype=np.uint64) for n, c in zip(sizes, cards)]
    slot_ids[4][:3] = [2**64 - 1, 0, 2**64 - 1]  # ids the prefix wraps and leaves
    pf = [oracle.index_prefix(0, prefix_bit), 0, oracle.index_prefix(1, prefix_bit), 0, oracle.index_prefix(0, prefix_bit),
          oracle.index_prefix(2, prefix_bit)]
    got = distinct_per_owner(slot_ids, pf, R, prefix_bit)
    want = np.zeros(R, np.int64)
    for x, p in zip(slot_ids, pf):
        for owner in oracle.shard_of(np.unique(oracle.add_prefix(x, prefix_bit, p)), R):
            want[owner] += 1
    assert got.tolist() == want.tolist() and want.sum() > 500
    assert got.tolist() == _owner_counts(list(zip(slot_ids, pf)), R, prefix_bit).tolist()


def test_exchange_area_geometry():
    """pb_xchg_bytes is plain host arithmetic (no GPU): areas grow with R, cap, dim and the row format, in 256-byte steps."""
    from persia_b200.worker import ShardedEmbeddingWorker as W

    a = W.area_bytes(2, 1024, 128)
    assert a % 256 == 0 and a >= 2 * 1024 * (8 + 128 * 2 + 128 * 4 + 4)
    assert W.area_bytes(8, 1024, 128) > 3 * a
    assert W.area_bytes(2, 1024, 128, rows_f32=True) - a == 2 * 1024 * 128 * 2
