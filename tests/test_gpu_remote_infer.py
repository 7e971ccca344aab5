"""GPU: inference on R GPUs one rank at a time (pb_forward_remote / pb_forward_raw_remote through RemoteReader).

R virtual ranks share cuda:0, as in test_gpu_worker.py: each has its own table, context and stream.  The ranks train a
few collective steps (group_forward / group_backward), and the collective path's inference outputs are taken
(group_forward(training=False)).  Then every table is exported and each rank sends its inference batch ALONE, one rank
after another, with no call on any other rank in between: a remote read needs no peer to take part.  Outputs must be
the collective path's bit for bit (and the oracle's with R parameter servers: bit for bit where the oracle pools in the
same order, one id per sample), and the owners' lookup_miss counters must grow as the collective path made them grow.
"""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from util import full_row_off, make_batch, same_bits, to_dev_i32, to_dev_ids  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _misses(ws):
    return [int(w.shard.counters()["lookup_miss"]) for w in ws]


def _train_group(torch, oracle, R, S, dim, B, pf, sqrt, ragged, rng, card, steps=2):
    """R virtual ranks and the oracle, trained `steps` collective steps on the same batches."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    max_ids = 4 if ragged else 1
    ws = W.local_group(R, S, dim, pf, 1 << 16, cap=S * B * max_ids, optimizer=dict(kind=N.OPT_SGD, lr=0.05, wd=0.001),
                       max_batch=B, sqrt_scaling=sqrt, rows_f32=ragged, max_ids_per_sample=max_ids)
    w = oracle.Worker([oracle.SlotCfg(dim, sqrt_scaling=bool(sqrt[i]), prefix=pf[i]) for i in range(S)], n_ps=R)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.05, wd=0.001))
    for x in ws:  # (table storage is allocated with a device-wide sync: not while a peer spins on a flag)
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    for _ in range(steps):
        bs = [make_batch(rng, S, B, card, max_ids=max_ids, allow_empty=ragged) for _ in range(R)]
        W.group_forward(ws, [to_dev_ids(b[0], DEV) for b in bs], B, training=True,
                        row_offs=[to_dev_i32(b[1], DEV) for b in bs] if ragged else None,
                        slot_occ_offs=[b[2] for b in bs])
        torch.cuda.synchronize()
        octx = [w.forward(b[0], b[1] if ragged else full_row_off(S, B), B, training=True)[1] for b in bs]
        g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16)
        W.group_backward(ws, [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)])
        torch.cuda.synchronize()
        for r in range(R):
            w.backward(octx[r], [g[r, i] for i in range(S)])
    return ws, w


@pytest.mark.parametrize("R,dim,layout", [(2, 64, "one"), (3, 12, "ragged"), (4, 128, "groups"), (8, 128, "one"),
                                          (2, 128, "ragged")])
def test_remote_matches_collective_one_rank_at_a_time(torch_cuda, oracle, R, dim, layout):
    from persia_b200.worker import RemoteReader
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    rng = np.random.default_rng(1000 * R + dim)
    S, B, card = 4, 256, [5, 300, 40000, 17]
    ragged = layout == "ragged"
    groups = layout == "groups"
    pf = [oracle.index_prefix(i // 2 if groups else i) for i in range(S)]  # "groups": slots 0, 1 and 2, 3 share a group
    sqrt = [True, False, True, False] if ragged else [False] * S
    ws, w = _train_group(torch, oracle, R, S, dim, B, pf, sqrt, ragged, rng, card)
    # the collective path's inference outputs and misses (batches hold signs never trained: misses on their owners)
    bs = [make_batch(rng, S, B, [c * 2 for c in card], max_ids=4 if ragged else 1, allow_empty=ragged) for _ in range(R)]
    d_ids = [to_dev_ids(b[0], DEV) for b in bs]
    d_off = [to_dev_i32(b[1], DEV) for b in bs] if ragged else None
    m0 = _misses(ws)
    want = W.group_forward(ws, d_ids, B, training=False, row_offs=d_off, slot_occ_offs=[b[2] for b in bs])
    torch.cuda.synchronize()
    want = [x.cpu().numpy() for x in want]
    m1 = _misses(ws)
    assert sum(m1) > sum(m0)
    readers = RemoteReader.local_group([x.shard for x in ws])
    try:
        for r in range(R):  # one rank at a time: nothing runs on the others
            got = readers[r].forward(d_ids[r], B, pf, sqrt, row_off=d_off[r] if ragged else None, slot_occ_off=bs[r][2])
            readers[r].stream.synchronize()
            got = got.cpu().numpy()
            assert same_bits(got, want[r]), (r, layout)
            ref, _ = w.forward(bs[r][0], bs[r][1] if ragged else full_row_off(S, B), B, training=False, keep_ctx=False)
            for i in range(S):
                if ragged:  # the oracle sums a sample's ids in shard order, here in sample order: one f16 step
                    np.testing.assert_allclose(got[i].astype(np.float32), ref[i].astype(np.float32), rtol=2e-3, atol=8e-3)
                else:
                    assert same_bits(got[i], ref[i]), (r, i)
        m2 = _misses(ws)
        assert [b - a for a, b in zip(m1, m2)] == [b - a for a, b in zip(m0, m1)]  # counted on the owners, as there
        for x in ws:
            assert x.shard.counters()["wait_errors"] == 0
    finally:
        for rd in readers:
            rd.close()


@pytest.mark.parametrize("R,dim", [(2, 12), (4, 64)])
def test_remote_raw_matches_collective(torch_cuda, oracle, R, dim):
    from persia_b200 import native as N
    from persia_b200.worker import RemoteReader, ShardedRawWorker

    torch = torch_cuda
    rng = np.random.default_rng(R * dim)
    B, fixed, card = 300, 5, 3000
    prefix = oracle.index_prefix(3)
    ws = ShardedRawWorker.local_group(R, 1, dim, [prefix], 1 << 16, cap=B * 6,
                                      optimizer=dict(kind=N.OPT_SGD, lr=0.05, wd=0.0), max_batch=B, max_ids_per_sample=6)
    for x in ws:
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()

    def batches():
        bs = [make_batch(rng, 1, B, card, max_ids=6, allow_empty=True) for _ in range(R)]
        return [to_dev_ids(b[0], DEV) for b in bs], [to_dev_i32(b[1], DEV) for b in bs]

    for _ in range(2):  # a few collective training steps
        ids, offs = batches()
        res = ShardedRawWorker.group_forward_raw(ws, ids, B, fixed, training=True, row_offs=offs)
        torch.cuda.synchronize()
        grads = [torch.from_numpy((rng.standard_normal((int(x[4][0]), dim)) * 1e-2).astype(np.float32)).to(DEV)
                 for x in res]
        ShardedRawWorker.group_backward_raw(ws, grads)
        torch.cuda.synchronize()
    ids, offs = batches()
    ids = [torch.cat([i, torch.tensor([10 ** 9 + r], dtype=torch.int64, device=DEV)]) for r, i in enumerate(ids)]  # a miss
    offs = [torch.cat([o[:-1], o[-1:] + 1]) for o in offs]
    m0 = _misses(ws)
    want = ShardedRawWorker.group_forward_raw(ws, ids, B, fixed, training=False, row_offs=offs)
    torch.cuda.synchronize()
    want = [[t.cpu().numpy() for t in x] for x in want]
    m1 = _misses(ws)
    readers = RemoteReader.local_group([x.shard for x in ws])
    try:
        for r in range(R):
            got = readers[r].forward_raw(ids[r], B, fixed, prefix, row_off=offs[r])
            readers[r].stream.synchronize()
            table, index, non_empty, num, counts = [t.cpu().numpy() for t in got]
            U, ne = counts.tolist()
            assert counts.tolist() == want[r][4].tolist()
            assert same_bits(table[:U + 1], want[r][0][:U + 1])  # row u + 1 = f16(row), rounded once
            assert (index == want[r][1]).all() and (non_empty[:ne] == want[r][2][:ne]).all()
            assert (num == want[r][3]).all()
        m2 = _misses(ws)
        assert [b - a for a, b in zip(m1, m2)] == [b - a for a, b in zip(m0, m1)]
        assert all(x.shard.counters()["wait_errors"] == 0 for x in ws)
    finally:
        for rd in readers:
            rd.close()


def test_remote_forward_graph_replay(torch_cuda, oracle):
    """One remote forward captured in a CUDA graph (after an eager call of the same size) and replayed on new ids gives
    the bytes of an eager call."""
    from persia_b200.worker import RemoteReader

    torch = torch_cuda
    rng = np.random.default_rng(5)
    R, S, B, dim, card = 2, 4, 512, 128, [5, 300, 40000, 17]
    pf = [oracle.index_prefix(i) for i in range(S)]
    ws, _ = _train_group(torch, oracle, R, S, dim, B, pf, [False] * S, False, rng, card, steps=1)
    readers = RemoteReader.local_group([x.shard for x in ws])
    try:
        rd = readers[1]
        ids_dev = torch.zeros(S * B, dtype=torch.int64, device=DEV)
        out = torch.empty((S, B, dim), dtype=torch.float16, device=DEV)
        with torch.cuda.stream(rd.stream):
            rd.forward(ids_dev, B, pf, out=out)  # eager warm-up: the context and its staging exist from here on
        rd.stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=rd.stream, capture_error_mode="thread_local"):
            rd.forward(ids_dev, B, pf, out=out)
        for _ in range(2):
            ids = make_batch(rng, S, B, [c * 2 for c in card])[0]
            ids_dev.copy_(to_dev_ids(ids, DEV))
            torch.cuda.synchronize()
            with torch.cuda.stream(rd.stream):
                graph.replay()
            rd.stream.synchronize()
            got = out.cpu().numpy()
            eager = rd.forward(to_dev_ids(ids, DEV), B, pf)
            rd.stream.synchronize()
            assert same_bits(got, eager.cpu().numpy())
    finally:
        for r in readers:
            r.close()


def test_reads_beside_inserts(torch_cuda):
    """An owner rewrites the same signs with pb_set_rows on its stream while a reader on another stream reads them
    remotely: every returned row is one version's whole row (each version writes one value in every column), and the
    reader's wait_errors stays 0.  Run once, with a fixed number of iterations."""
    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200.worker import RemoteReader

    torch = torch_cuda
    R, dim, n, iters = 2, 128, 4096, 64
    shards = []
    for _ in range(R):
        s = SH.EmbeddingShard(dim, 1 << 16, 0)
        s.set_optimizer(N.OPT_SGD, lr=0.1)
        s.configure()
        shards.append(s)
    cand = torch.arange(1, 8 * n, dtype=torch.int64, device=DEV)
    owned = cand[SH.shard_of(cand, R) == 0][:n].contiguous()  # signs owner 0 holds
    assert owned.numel() == n

    def version(v):
        return torch.full((n, dim), float(v), dtype=torch.float32, device=DEV)  # exact in f16

    shards[0].set_entries(owned, version(0))
    torch.cuda.synchronize()
    readers = RemoteReader.local_group(shards)
    try:
        owner_stream = torch.cuda.Stream(device=DEV)
        vers = [version(v) for v in range(1, iters + 1)]
        outs = []
        torch.cuda.synchronize()
        for v in range(iters):  # the two streams run side by side on the device
            with torch.cuda.stream(owner_stream):
                shards[0].set_entries(owned, vers[v])
            with torch.cuda.stream(readers[1].stream):
                outs.append(readers[1].forward(owned, n, [0]))
        torch.cuda.synchronize()
        seen = set()
        for o in outs:
            o = o[0].float()
            lo, hi = o.min(dim=1).values, o.max(dim=1).values
            assert torch.equal(lo, hi), "a row mixed two versions"
            assert float(lo.min()) >= 0 and float(hi.max()) <= iters
            seen.update(torch.unique(lo).tolist())
        assert len(seen) > 1  # (the reads did run beside the writes)
        assert shards[1].counters()["wait_errors"] == 0
        assert shards[0].counters()["lookup_miss"] == 0
    finally:
        for rd in readers:
            rd.close()
        for s in shards:
            s.close()


def test_exported_table_refuses_what_moves_cells(torch_cuda):
    """From the export on, a table refuses with PB_ERR_STATE, before enqueuing anything, every call that moves cells or
    steps rows; set_entries and inference forwards stay allowed.  A table with a host tier (and the tier) cannot be
    exported."""
    from persia_b200 import native as N
    from persia_b200 import shard as SH

    torch = torch_cuda
    lib = N.load()
    dim, B = 16, 64
    s = SH.EmbeddingShard(dim, 4096, 0)
    s.set_optimizer(N.OPT_SGD, lr=0.1)
    s.configure()
    s.set_eviction(check_every=1)
    ctx = SH.BatchContext(4 * B, 4 * B, [0], None, 8, 0)
    ids = torch.arange(B, dtype=torch.int64, device=DEV)
    ctx.forward(s, ids, [0, B], B, training=True)  # a pending batch: its backward comes after the export
    torch.cuda.synchronize()
    blob = s.export_view()
    assert len(blob) == int(lib.pb_table_view_bytes())
    g = torch.zeros((1, B, dim), dtype=torch.float16, device=DEV)

    def refused(fn):
        torch.cuda.synchronize()
        n0 = int(lib.pb_launch_count())
        with pytest.raises(N.PersiaB200Error) as e:
            fn()
        assert e.value.code == N.PB_ERR_STATE, str(e.value)
        assert int(lib.pb_launch_count()) == n0

    refused(lambda: ctx.backward(s, g))
    refused(lambda: ctx.forward(s, ids, [0, B], B, training=True))
    refused(lambda: s.update(ids[:4], torch.zeros((4, dim), dtype=torch.float32, device=DEV)))
    refused(lambda: s.clear())
    refused(lambda: s.stage(ids, [0, B], [0]))  # the eviction check a training request would run
    refused(lambda: s.lookup(ids, training=True))
    raw = SH.BatchContext(4 * B, 4 * B, [0], None, 8, 0)
    refused(lambda: raw.forward_raw(s, ids, B, 1, training=True))
    # still allowed: inserts, reads and inference
    s.set_entries(ids[:2], torch.ones((2, dim), dtype=torch.float32, device=DEV))
    out = ctx.forward(s, ids, [0, B], B, training=False)
    torch.cuda.synchronize()
    assert (out[0, :2].float() == 1).all()
    assert len(s) == B
    # a host tier, and a table with one, are never exported
    t = SH.EmbeddingShard(dim, 1024, 0, tier_rows=1024)
    t.set_optimizer(N.OPT_SGD, lr=0.1)
    for h in (t.h, t.host_tier.h):
        b = ctypes.create_string_buffer(int(lib.pb_table_view_bytes()))
        assert lib.pb_table_export_view(h, b) == N.PB_ERR_STATE
    for x in (ctx, raw, s, t):
        x.close()


def test_view_blob_round_trip_same_process(torch_cuda):
    """The blob opens in the exporting process through its own pointers: a one-rank remote read and a two-rank one
    (rank 1 reading rank 0's view) return the rows set on the owner."""
    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200.worker import RemoteReader

    torch = torch_cuda
    dim = 12
    shards = []
    for _ in range(2):
        s = SH.EmbeddingShard(dim, 1024, 0)
        s.set_optimizer(N.OPT_SGD, lr=0.1)
        shards.append(s)
    signs = torch.arange(1, 200, dtype=torch.int64, device=DEV)
    owner = SH.shard_of(signs, 2)
    ent = torch.randn((signs.numel(), dim), device=DEV).half().float()
    for r in range(2):
        shards[r].set_entries(signs[owner == r], ent[owner == r])
    readers = RemoteReader.local_group(shards)
    try:
        for rd in readers:
            out = rd.forward(signs, signs.numel(), [0])
            rd.stream.synchronize()
            assert torch.equal(out[0].float(), ent)
    finally:
        for rd in readers:
            rd.close()
        for s in shards:
            s.close()
