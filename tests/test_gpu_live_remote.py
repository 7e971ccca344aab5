"""GPU: reads of live-exported tables on R GPUs one rank at a time (pb_table_export_live_view + RemoteReader).

R virtual ranks share cuda:0, as in test_gpu_remote_infer.py, but the tables are exported live before any training: the
ranks keep training through the collective path (group_forward / group_backward) while each rank reads its peers'
tables in place.  Between steps a read equals the collective inference bit for bit; beside a step it sees each element
before or after the step; across capacity sweeps and index rebuilds it never returns another sign's row.
"""
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


def _misses(shards):
    return [int(s.counters()["lookup_miss"]) for s in shards]


def _live_readers(torch, shards):
    """Every shard exported live and viewed by the others, one reader per rank on a stream of its own."""
    from persia_b200.shard import TableView
    from persia_b200.worker import RemoteReader

    blobs = [s.export_live_view() for s in shards]
    return [RemoteReader(s, [TableView(b, s.device) if q != r else None for q, b in enumerate(blobs)], r,
                         stream=torch.cuda.Stream(device=s.device)) for r, s in enumerate(shards)]


def _allocate(torch, ws):
    for x in ws:  # (table storage is allocated with a device-wide sync: not while a peer spins on a flag)
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()


def _close(readers):
    for rd in readers:
        rd.close()


# ---- 1. between steps: the collective inference's outputs, bit for bit --------------------------------------------------
@pytest.mark.parametrize("R,dim,layout", [(2, 8, "one"), (4, 64, "ragged"), (2, 128, "ragged"), (4, 128, "one")])
def test_live_read_between_steps_matches_collective(torch_cuda, oracle, R, dim, layout):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    rng = np.random.default_rng(31 * R + dim)
    S, B, card = 3, 256, [7, 500, 30000]
    ragged = layout == "ragged"
    max_ids = 4 if ragged else 1
    pf = [oracle.index_prefix(i) for i in range(S)]
    sqrt = [True, False, True] if ragged else [False] * S
    ws = W.local_group(R, S, dim, pf, 1 << 16, cap=S * B * max_ids, optimizer=dict(kind=N.OPT_SGD, lr=0.05, wd=0.001),
                       max_batch=B, sqrt_scaling=sqrt, rows_f32=ragged, max_ids_per_sample=max_ids)
    w = oracle.Worker([oracle.SlotCfg(dim, sqrt_scaling=bool(sqrt[i]), prefix=pf[i]) for i in range(S)], n_ps=R)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.05, wd=0.001))
    _allocate(torch, ws)
    readers = _live_readers(torch, [x.shard for x in ws])
    try:
        for step in range(3):
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
            # inference batches hold signs never trained too: misses on their owners
            qs = [make_batch(rng, S, B, [c * 2 for c in card], max_ids=max_ids, allow_empty=ragged) for _ in range(R)]
            d_ids = [to_dev_ids(b[0], DEV) for b in qs]
            d_off = [to_dev_i32(b[1], DEV) for b in qs] if ragged else [None] * R
            m0 = _misses([x.shard for x in ws])
            want = W.group_forward(ws, d_ids, B, training=False, row_offs=d_off if ragged else None,
                                   slot_occ_offs=[b[2] for b in qs])
            torch.cuda.synchronize()
            want = [x.cpu().numpy() for x in want]
            m1 = _misses([x.shard for x in ws])
            assert sum(m1) > sum(m0)
            for r in range(R):  # one rank at a time
                got = readers[r].forward(d_ids[r], B, pf, sqrt, row_off=d_off[r], slot_occ_off=qs[r][2])
                readers[r].stream.synchronize()
                got = got.cpu().numpy()
                assert same_bits(got, want[r]), (step, r)
                ref, _ = w.forward(qs[r][0], qs[r][1] if ragged else full_row_off(S, B), B, training=False, keep_ctx=False)
                for i in range(S):
                    if ragged:  # the oracle sums a sample's ids in shard order, here in sample order: one f16 step
                        np.testing.assert_allclose(got[i].astype(np.float32), ref[i].astype(np.float32), rtol=2e-3,
                                                   atol=8e-3)
                    else:
                        assert same_bits(got[i], ref[i]), (step, r, i)
            m2 = _misses([x.shard for x in ws])
            assert [b - a for a, b in zip(m1, m2)] == [b - a for a, b in zip(m0, m1)]
        for x in ws:
            assert x.shard.counters()["wait_errors"] == 0
    finally:
        _close(readers)


def test_live_raw_read_between_steps_matches_collective(torch_cuda, oracle):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedRawWorker

    torch = torch_cuda
    R, dim, B, fixed, card = 2, 64, 300, 5, 3000
    rng = np.random.default_rng(77)
    prefix = oracle.index_prefix(3)
    ws = ShardedRawWorker.local_group(R, 1, dim, [prefix], 1 << 16, cap=B * 6,
                                      optimizer=dict(kind=N.OPT_SGD, lr=0.05, wd=0.0), max_batch=B, max_ids_per_sample=6)
    _allocate(torch, ws)
    readers = _live_readers(torch, [x.shard for x in ws])

    def batches():
        bs = [make_batch(rng, 1, B, card, max_ids=6, allow_empty=True) for _ in range(R)]
        return [to_dev_ids(b[0], DEV) for b in bs], [to_dev_i32(b[1], DEV) for b in bs]

    try:
        for step in range(3):
            ids, offs = batches()
            res = ShardedRawWorker.group_forward_raw(ws, ids, B, fixed, training=True, row_offs=offs)
            torch.cuda.synchronize()
            grads = [torch.from_numpy((rng.standard_normal((int(x[4][0]), dim)) * 1e-2).astype(np.float32)).to(DEV)
                     for x in res]
            ShardedRawWorker.group_backward_raw(ws, grads)
            torch.cuda.synchronize()
            ids, offs = batches()
            ids = [torch.cat([i, torch.tensor([10 ** 9 + r], dtype=torch.int64, device=DEV)]) for r, i in enumerate(ids)]
            offs = [torch.cat([o[:-1], o[-1:] + 1]) for o in offs]
            m0 = _misses([x.shard for x in ws])
            want = ShardedRawWorker.group_forward_raw(ws, ids, B, fixed, training=False, row_offs=offs)
            torch.cuda.synchronize()
            want = [[t.cpu().numpy() for t in x] for x in want]
            m1 = _misses([x.shard for x in ws])
            for r in range(R):
                got = readers[r].forward_raw(ids[r], B, fixed, prefix, row_off=offs[r])
                readers[r].stream.synchronize()
                got = [t.cpu().numpy() for t in got]
                U, ne = int(want[r][4][0]), int(want[r][4][1])
                assert same_bits(got[0][:U + 1], want[r][0][:U + 1]), (step, r)
                np.testing.assert_array_equal(got[1], want[r][1])
                np.testing.assert_array_equal(got[2][:ne], want[r][2][:ne])
                np.testing.assert_array_equal(got[3], want[r][3])
                np.testing.assert_array_equal(got[4], want[r][4])
            m2 = _misses([x.shard for x in ws])
            assert [b - a for a, b in zip(m1, m2)] == [b - a for a, b in zip(m0, m1)]
    finally:
        _close(readers)


# ---- 2. beside a step: every element before or after it ----------------------------------------------------------------
def test_live_read_beside_a_step_sees_before_or_after(torch_cuda):
    """SGD at lr 1 with gradients k / 1024 (|k| <= 4): every sign's summed gradient is exact in any order, so the step
    has one serial answer per element.  The read batch holds signs resident before the step only (no admission)."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, S, B, dim = 2, 2, 1024, 64
    card = [2000, 2000]
    rng = np.random.default_rng(5)
    pf = [0, 0]  # (ids taken as they are)
    ws = W.local_group(R, S, dim, pf, 1 << 16, cap=S * B, optimizer=dict(kind=N.OPT_SGD, lr=1.0, wd=0.0), max_batch=B)
    _allocate(torch, ws)
    readers = _live_readers(torch, [x.shard for x in ws])

    def grads():
        g = (rng.integers(-4, 5, size=(R, S, B, dim)) / 1024.0).astype(np.float16)
        out = [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)]
        torch.cuda.synchronize()
        return out

    def train(ids):
        d, g = [to_dev_ids(b, DEV) for b in ids], grads()
        out = W.group_forward(ws, d, B, training=True, slot_occ_offs=[[0, B, 2 * B]] * R)
        W.group_backward(ws, g)
        torch.cuda.synchronize()
        del out

    try:
        warm = [make_batch(rng, S, B, card)[0] for _ in range(R)]
        for _ in range(2):
            train(warm)
        torch.cuda.synchronize()
        q = to_dev_ids(warm[0], DEV)  # resident signs only
        slot_off = [0, B, 2 * B]
        reads = 0
        for step in range(6):
            before = W.group_forward(ws, [q] + [to_dev_ids(w_, DEV) for w_ in warm[1:]], B, training=False,
                                     slot_occ_offs=[slot_off] * R)[0]
            torch.cuda.synchronize()
            before = before.cpu().numpy()
            nxt = [to_dev_ids(warm[r] if step % 2 else make_batch(rng, S, B, card)[0], DEV) for r in range(R)]
            g = grads()  # (these tensors, and the step's outputs, stay alive until the device is idle)
            outs = [readers[0].forward(q, B, pf, slot_occ_off=slot_off)]
            step_out = W.group_forward(ws, nxt, B, training=True, slot_occ_offs=[slot_off] * R)
            outs.append(readers[0].forward(q, B, pf, slot_occ_off=slot_off))
            W.group_backward(ws, g)
            outs.append(readers[0].forward(q, B, pf, slot_occ_off=slot_off))
            torch.cuda.synchronize()
            del step_out, g, nxt
            outs = [o.cpu().numpy() for o in outs]
            after = W.group_forward(ws, [q] + [to_dev_ids(w_, DEV) for w_ in warm[1:]], B, training=False,
                                    slot_occ_offs=[slot_off] * R)[0]
            torch.cuda.synchronize()
            after = after.cpu().numpy()
            assert not same_bits(before, after)  # the step moved the rows read
            bv, av = before.view(np.uint16), after.view(np.uint16)
            for o in outs:
                ov = o.view(np.uint16)
                assert np.all((ov == bv) | (ov == av)), step
                reads += 1
        assert reads == 18
        for x in ws:
            assert x.shard.counters()["wait_errors"] == 0
    finally:
        _close(readers)


# ---- 3. across sweeps and rebuilds: never another sign's row -----------------------------------------------------------
def test_live_read_across_sweeps_and_rebuilds(torch_cuda):
    """SGD at lr 0: every resident row stays its sign's initial row (a function of the sign alone), so a returned row is
    zeros (evicted before the probe, or never admitted) or exactly that sign's initial row; another sign's row, or a
    torn one, fails.  A small capacity with an eviction check on every step churns the index into rebuilds."""
    from persia_b200 import native as N
    from persia_b200.shard import EmbeddingShard
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, B, dim, cap = 2, 2048, 64, 6000
    rng = np.random.default_rng(9)
    ws = W.local_group(R, 1, dim, [0], cap, cap=B, optimizer=dict(kind=N.OPT_SGD, lr=0.0, wd=0.0), max_batch=B)
    for x in ws:
        x.shard.set_eviction(check_every=1, low_water=cap // 3, target_free=cap // 2, keep_batches=1)
    _allocate(torch, ws)
    ref = EmbeddingShard(dim, 1 << 20, 0)
    ref.set_optimizer(kind=N.OPT_SGD, lr=0.0, wd=0.0)
    ref.configure()  # (the workers' initialisation bounds)
    readers = _live_readers(torch, [x.shard for x in ws])
    try:
        hist, empty, rows_seen, zeros_seen = [], [], 0, 0
        for step in range(80):
            ids = [rng.integers(0, 1 << 40, size=B, dtype=np.uint64) for _ in range(R)]
            # reads of the last steps' signs (some evicted since) and of this step's, issued beside the step
            pool = np.concatenate(hist[-3:] + [ids[0]]) if hist else ids[0]
            q = rng.choice(pool, size=B).astype(np.uint64)
            d_q = to_dev_ids(q, DEV)
            torch.cuda.synchronize()  # (the readers' streams do not wait for the copy)
            # (every tensor of the step stays alive until the device is idle: the workers' streams still use them)
            d_ids = [to_dev_ids(b, DEV) for b in ids]
            zeros = [[torch.zeros((B, dim), dtype=torch.float16, device=DEV)] for _ in range(R)]
            torch.cuda.synchronize()
            outs = [readers[r].forward(d_q, B, [0]) for r in range(R)]
            step_out = W.group_forward(ws, d_ids, B, training=True, slot_occ_offs=[[0, B]] * R)
            outs += [readers[r].forward(d_q, B, [0]) for r in range(R)]
            W.group_backward(ws, zeros)
            outs += [readers[r].forward(d_q, B, [0]) for r in range(R)]
            torch.cuda.synchronize()
            del step_out, zeros, d_ids
            hist.append(np.concatenate(ids))
            want = ref.lookup(d_q, training=True).half().cpu().numpy().view(np.uint16)  # each sign's initial row
            for o in outs:
                ov = o[0].cpu().numpy().view(np.uint16)
                zero = np.all(ov == 0, axis=1)
                mine = np.all(ov == want, axis=1)
                assert np.all(zero | mine), step
                rows_seen += int(mine.sum())
                zeros_seen += int((zero & ~mine).sum())
            empty.append(ws[0].shard.index_stats()["empty"])
        assert rows_seen > 0 and zeros_seen > 0
        # EMPTY cells only get fewer between rebuilds: more of them after a step means that step rebuilt the index
        assert any(b > a for a, b in zip(empty, empty[1:])), empty
        for x in ws:
            assert x.shard.counters()["wait_errors"] == 0
    finally:
        _close(readers)
        ref.close()


# ---- 4. tables without the export, and a captured step -----------------------------------------------------------------
def test_live_export_adds_no_launch_to_a_training_step(torch_cuda):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    lib = N.load()
    R, B, dim, cap = 2, 1024, 64, 3000
    rng = np.random.default_rng(2)

    def group():
        ws = W.local_group(R, 1, dim, [0], cap, cap=B, optimizer=dict(kind=N.OPT_SGD, lr=0.1, wd=0.0), max_batch=B)
        for x in ws:
            x.shard.set_eviction(check_every=1, low_water=cap // 3, target_free=cap // 2, keep_batches=1)
        _allocate(torch, ws)
        return ws

    plain, live = group(), group()
    readers = _live_readers(torch, [x.shard for x in live])
    try:
        for step in range(4):
            ids = [to_dev_ids(rng.integers(0, 1 << 40, size=B, dtype=np.uint64), DEV) for _ in range(R)]
            g = [[torch.full((B, dim), 1.0 / 64, dtype=torch.float16, device=DEV)] for _ in range(R)]
            counts = []
            for ws in (plain, live):
                torch.cuda.synchronize()
                n0 = lib.pb_launch_count()
                W.group_forward(ws, ids, B, training=True, slot_occ_offs=[[0, B]] * R)
                W.group_backward(ws, g)
                torch.cuda.synchronize()
                counts.append(lib.pb_launch_count() - n0)
            assert counts[0] == counts[1], (step, counts)
    finally:
        _close(readers)


def test_live_table_captured_step_equals_eager(torch_cuda):
    """One GPU's training step (pb_forward / pb_backward with an eviction check on every step) captured once in a CUDA
    graph on a live-exported table and replayed on new batches, against the same steps eager on a table that is not
    exported: the sweeps raise and lower the live table's word inside the graph, and every output and row stays the
    eager table's."""
    from persia_b200 import native as N
    from persia_b200.shard import BatchContext, EmbeddingShard

    torch = torch_cuda
    S, B, dim, cap = 2, 512, 32, 20000
    pf = [1 << 56, 2 << 56]
    shards = []
    for _ in range(2):
        s = EmbeddingShard(dim, cap, 0)
        s.set_optimizer(kind=N.OPT_ADAGRAD, lr=0.05, initialization=0.01)
        s.configure()
        # every check sweeps (free rows stay below the low water mark), yet the 12000 signs the batches draw always fit:
        # no admission is refused, so no outcome depends on which lane pops a free row first
        s.set_eviction(check_every=1, low_water=cap, target_free=cap, keep_batches=1)
        shards.append(s)
    plain, live = shards
    live.export_live_view()
    ctxs = [BatchContext(S * B, S * B, pf) for _ in range(2)]
    rng = np.random.default_rng(4)
    slot_off = [0, B, 2 * B]
    ids_dev = torch.empty(S * B, dtype=torch.int64, device=DEV)
    g_dev = torch.zeros((S, B, dim), dtype=torch.float16, device=DEV)
    outs = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(2)]
    seen = set()

    def draw():
        ids = rng.integers(0, 6000, size=S * B, dtype=np.uint64)
        seen.update(ids.tolist())
        ids_dev.copy_(to_dev_ids(ids, DEV))
        g_dev.copy_(torch.from_numpy((rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)).to(DEV))
        torch.cuda.synchronize()  # (the steps run on another stream)

    stream = torch.cuda.Stream()
    draw()
    with torch.cuda.stream(stream):
        for k in range(2):
            ctxs[k].forward(shards[k], ids_dev, slot_off, B, training=True, out=outs[k])  # warm-up: a real step
            ctxs[k].backward(shards[k], [g_dev[i] for i in range(S)])
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            ctxs[1].forward(live, ids_dev, slot_off, B, training=True, out=outs[1])
            ctxs[1].backward(live, [g_dev[i] for i in range(S)])
    for it in range(12):
        draw()
        with torch.cuda.stream(stream):
            ctxs[0].forward(plain, ids_dev, slot_off, B, training=True, out=outs[0])  # eager
            ctxs[0].backward(plain, [g_dev[i] for i in range(S)])
            graph.replay()
            stream.synchronize()
        assert same_bits(outs[1].cpu().numpy(), outs[0].cpu().numpy()), it
    assert live.index_stats()["tomb"] > 0  # the replays swept rows
    assert plain.counters()["capacity_refused"] == 0 and live.counters()["capacity_refused"] == 0
    signs = to_dev_ids(np.array(sorted(seen), np.uint64), DEV)
    (pa, pf_), (la, lf) = plain.get_entries(signs), live.get_entries(signs)
    assert torch.equal(pf_, lf)
    assert same_bits(pa[pf_].cpu().numpy(), la[lf].cpu().numpy())
    for c in ctxs:
        c.close()
    for s in shards:
        s.close()


# ---- 5. writes: pb_set_rows and pb_table_clear ---------------------------------------------------------------------------
def test_live_set_rows_and_clear_are_seen_by_reads(torch_cuda):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, B, dim = 2, 256, 64
    ws = W.local_group(R, 1, dim, [0], 1 << 14, cap=B, optimizer=dict(kind=N.OPT_SGD, lr=0.1, wd=0.0), max_batch=B)
    _allocate(torch, ws)
    readers = _live_readers(torch, [x.shard for x in ws])
    try:
        from persia_b200.shard import shard_of

        signs = np.arange(1, B + 1, dtype=np.uint64) * 7919
        d = to_dev_ids(signs, DEV)
        own = shard_of(d, R).cpu().numpy()  # every sign is set on its owner
        vals = (np.arange(B * dim, dtype=np.float32).reshape(B, dim) % 97 - 48) / 64.0
        for r in range(R):
            m = own == r
            ent = np.zeros((int(m.sum()), ws[r].shard.entry_len), np.float32)
            ent[:, :dim] = vals[m]
            ws[r].shard.set_entries(d[torch.from_numpy(m).to(DEV)], torch.from_numpy(ent).to(DEV))
        torch.cuda.synchronize()  # (the reader's stream does not wait for the calls on this one)
        got = readers[0].forward(d, B, [0])
        readers[0].stream.synchronize()
        assert same_bits(got[0].cpu().numpy(), vals.astype(np.float16))
        m0 = _misses([x.shard for x in ws])
        ws[1].shard.clear()
        torch.cuda.synchronize()
        got = readers[0].forward(d, B, [0])
        readers[0].stream.synchronize()
        got = got[0].cpu().numpy().view(np.uint16)
        cleared = own == 1
        assert cleared.any() and not cleared.all()
        assert np.all(got[cleared] == 0)
        assert same_bits(got[~cleared].view(np.float16), vals[~cleared].astype(np.float16))
        m1 = _misses([x.shard for x in ws])
        assert m1[1] == int(cleared.sum()) and m1[0] == m0[0]  # (the clear zeroed rank 1's counters)
    finally:
        _close(readers)


# ---- 6. refusals --------------------------------------------------------------------------------------------------------
def test_live_export_refusals(torch_cuda):
    from persia_b200 import native as N
    from persia_b200.shard import EmbeddingShard

    a = EmbeddingShard(16, 1024, 0)
    a.set_optimizer(kind=N.OPT_SGD, lr=0.1)
    a.export_view()
    with pytest.raises(N.PersiaB200Error, match="one export mode"):
        a.export_live_view()
    b = EmbeddingShard(16, 1024, 0)
    b.set_optimizer(kind=N.OPT_SGD, lr=0.1)
    b.export_live_view()
    b.export_live_view()  # (the same mode again: another blob)
    with pytest.raises(N.PersiaB200Error, match="one export mode"):
        b.export_view()
    t = EmbeddingShard(16, 1024, 0, tier_rows=1024)
    t.set_optimizer(kind=N.OPT_SGD, lr=0.1)
    with pytest.raises(N.PersiaB200Error, match="host tier"):
        t.export_live_view()
    with pytest.raises(N.PersiaB200Error, match="host tier"):
        t.host_tier.export_live_view()
    for s in (a, b, t):
        s.close()
