"""GPU: raw (embedding_summation: false) slots on the sharded path (pb_forward_raw_sharded / pb_backward_raw_sharded
through ShardedRawWorker) against the oracle's embedding worker with R parameter servers.

R virtual ranks share cuda:0, as in test_gpu_worker.py.  The oracle runs R raw forward requests, then R raw backward
requests in rank order: an owner applies the step's R gradient requests in rank order, so a sign that several ranks
hold takes one optimizer step per rank.  Everything compares bit for bit (Adagrad against the oracle's exact-rsqrt
mode): the distinct-sign table, index, non_empty_index, sample_id_num, U, statuses and every touched entry read from
its owner."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from util import to_dev_i32, to_dev_ids  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
M = 2**64


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def _optim(N, oracle, kind):
    if kind == oracle.SGD:
        return dict(kind=N.OPT_SGD, lr=0.05, wd=0.001), oracle.Optim(oracle.SGD, lr=0.05, wd=0.001)
    if kind == oracle.ADAGRAD:
        return (dict(kind=N.OPT_ADAGRAD, lr=0.02, initialization=0.01, eps=1e-10),
                oracle.Optim(oracle.ADAGRAD, lr=0.02, init_acc=0.01, eps=1e-10))
    if kind == oracle.ADAM:
        return (dict(kind=N.OPT_ADAM, lr=0.01, beta1=0.9, beta2=0.999, eps=1e-8),
                oracle.Optim(oracle.ADAM, lr=0.01, b1=0.9, b2=0.999, eps=1e-8))
    return (dict(kind=N.OPT_ADAGRAD_VW, lr=0.02, initialization=0.01, eps=1e-10),
            oracle.Optim(oracle.ADAGRAD_VW, lr=0.02, init_acc=0.01, eps=1e-10))


def _warm(torch, ws):
    for x in ws:  # table storage is allocated on first use, with a device-wide sync: not while a peer spins on a flag
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()


def _raw_group(torch, oracle, R, dim, kind, B, fixed, prefix, cap, max_ids=1, shards=None):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedRawWorker

    gpu_opt, cpu_opt = _optim(N, oracle, kind)
    ws = ShardedRawWorker.local_group(R, 1, dim, [prefix], 1 << 16, cap=cap, optimizer=gpu_opt, max_batch=B,
                                      max_ids_per_sample=max_ids, shards=shards)
    w = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=prefix)], n_ps=R)
    w.configure()
    w.set_optimizer(cpu_opt)
    _warm(torch, ws)
    return ws, w


def _ragged(rng, B, card, max_ids, allow_empty=True):
    counts = rng.integers(0 if allow_empty else 1, max_ids + 1, size=B)
    row_off = np.zeros(B + 1, np.uint32)
    row_off[1:] = np.cumsum(counts)
    return rng.integers(0, card, size=int(row_off[-1]), dtype=np.uint64), row_off


def _single(rng, B, card):
    return rng.integers(0, card, size=B, dtype=np.uint64), np.arange(B + 1, dtype=np.uint32)


def _forward(torch, ws, w, batches, B, fixed, training=True, single=False, slot=0):
    """Both sides' forward of one step; compares everything and returns [(U, oracle ctx)] per rank."""
    from persia_b200.worker import ShardedRawWorker as W

    torch.cuda.synchronize()
    ids = [to_dev_ids(b[0], DEV) for b in batches]
    offs = None if single else [to_dev_i32(b[1], DEV) for b in batches]
    torch.cuda.synchronize()
    res = W.group_forward_raw(ws, ids, B, fixed, training=training, row_offs=offs)
    torch.cuda.synchronize()
    out = []
    for r, (table, index, non_empty, num, counts) in enumerate(res):
        U, ne = counts.cpu().numpy().tolist()
        wt, wi, wne, wnum, octx = w.forward_raw(slot, batches[r][0], batches[r][1], B, training=training)
        assert U == wt.shape[0] - 1, r
        assert table[:U + 1].cpu().numpy().tobytes() == wt.tobytes(), r
        np.testing.assert_array_equal(index.cpu().numpy(), wi)
        assert ne == wne.size
        np.testing.assert_array_equal(non_empty[:ne].cpu().numpy(), wne)
        np.testing.assert_array_equal(num.cpu().numpy().view(np.uint32), wnum)
        out.append((U, octx))
    return out


def _backward(torch, ws, w, octx, grads, scales=None, slot=0):
    """grads: per rank a numpy [U, dim] array or None (add_skipped_gradient); the oracle applies rank 0, 1, ..."""
    from persia_b200.worker import ShardedRawWorker as W

    dg = [torch.from_numpy(g).to(DEV) if g is not None else None for g in grads]
    torch.cuda.synchronize()
    sts = W.group_backward_raw(ws, dg, scales=scales, want_status=True)
    torch.cuda.synchronize()
    for r, g in enumerate(grads):
        sc = scales[r] if scales is not None else 1.0
        want = w.backward_raw(slot, octx[r][1], g, scale=sc, skip=g is None)
        assert sts[r].item() == want, (r, sts[r].item(), want)


def _check_rows(torch, oracle, shards, w, signs, R, statuses=()):
    signs = np.array(sorted(signs), np.uint64)
    owner = oracle.shard_of(signs, R)
    for r in range(R):
        mine = signs[owner == r]
        if mine.size:
            ent, found = shards[r].get_entries(to_dev_ids(mine, DEV))
            ent = ent.cpu().numpy()
            assert found.all()
            for k, sign in enumerate(mine):
                ref = w.get_entry(int(sign))
                assert ref is not None and ent[k].tobytes() == ref.tobytes(), (r, k, sign)
        assert len(shards[r]) == w.ps_len(r)
        assert shards[r].counters()["wait_errors"] == 0
    for x in statuses:
        assert x.status() == (False, False)


def _signs(oracle, ids, prefix):
    return oracle.add_prefix(ids, 8, prefix).tolist() if prefix else ids.tolist()


@pytest.mark.parametrize("R,dim,kind,fixed", [(1, 64, 1, 5), (2, 12, 0, 1), (2, 130, 1, 10), (3, 64, 3, 5),
                                              (4, 128, 2, 10), (8, 128, 1, 5), (4, 130, 0, 5), (8, 12, 3, 1),
                                              (3, 128, 0, 10), (2, 64, 2, 5)])
def test_virtual_ranks_raw_match_oracle(torch_cuda, oracle, R, dim, kind, fixed):
    """Ragged batches with empty samples and rows longer than sample_fixed_size, the single-id layout, f16 (with
    +-inf) and f32 gradients, a loss scale, a NaN on rank 0 and add_skipped_gradient on the last rank.  The
    cardinality is low, so most signs are held by several ranks in a step."""
    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(1000 * R + dim + fixed)
        B, card, max_ids = 300, 400, 12
        pf = oracle.index_prefix(0)
        ws, w = _raw_group(torch, oracle, R, dim, kind, B, fixed, pf, cap=B * max_ids, max_ids=max_ids)
        seen = set()
        for step in range(5):
            single = step == 1
            batches = [_single(rng, B, card) if single else _ragged(rng, B, card, max_ids) for _ in range(R)]
            for b in batches:
                seen.update(_signs(oracle, b[0], pf))
            octx = _forward(torch, ws, w, batches, B, fixed, single=single)
            f16 = step % 2 == 1
            grads = []
            for r in range(R):
                g = (rng.standard_normal((octx[r][0], dim)) * 1e-2).astype(np.float16 if f16 else np.float32)
                if f16 and g.size:
                    g[0, 0], g[-1, -1] = np.inf, -np.inf  # clamp to +-65504 (persia-common lib.rs:163-180)
                grads.append(g)
            if step == 2 and grads[0].size:
                grads[0][grads[0].shape[0] // 2, dim - 1] = np.nan  # rank 0's whole request is dropped; the others stand
            if step == 3 and R > 1:
                grads[R - 1] = None  # add_skipped_gradient on the last rank
            scales = [128.0 if step >= 2 else 1.0] * R
            _backward(torch, ws, w, octx, grads, scales)
        _check_rows(torch, oracle, [x.shard for x in ws], w, seen, R, ws)
    finally:
        oracle.set_rsqrt_exact(False)


@pytest.mark.parametrize("kind", [0, 3])
def test_raw_empty_batches(torch_cuda, oracle, kind):
    """A rank without ids (U = 0) while the others have some, then a step in which every rank is empty: the calls are
    collective all the same, and an empty request advances no Adam beta power."""
    torch = torch_cuda
    rng = np.random.default_rng(21 + kind)
    R, B, dim, fixed = 3, 64, 16, 4
    pf = oracle.index_prefix(0)
    ws, w = _raw_group(torch, oracle, R, dim, kind, B, fixed, pf, cap=B * 4, max_ids=4)
    seen = set()
    empty = (np.zeros(0, np.uint64), np.zeros(B + 1, np.uint32))
    for step in range(4):
        batches = [_ragged(rng, B, 90, 4) for _ in range(R)]
        if step == 1:
            batches[1] = empty
        if step == 2:
            batches = [empty] * R
        for b in batches:
            seen.update(_signs(oracle, b[0], pf))
        octx = _forward(torch, ws, w, batches, B, fixed)
        if step == 2:
            assert all(u == 0 for u, _ in octx)
        grads = [(rng.standard_normal((u, dim)) * 1e-2).astype(np.float32) for u, _ in octx]
        _backward(torch, ws, w, octx, grads)
    _check_rows(torch, oracle, [x.shard for x in ws], w, seen, R, ws)


def test_raw_inference_does_not_admit(torch_cuda, oracle):
    """training = 0: unseen signs still get a number and read as zeros; no shard grows."""
    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(5)
        R, B, dim, fixed = 4, 128, 64, 5
        pf = oracle.index_prefix(0)
        ws, w = _raw_group(torch, oracle, R, dim, oracle.ADAGRAD, B, fixed, pf, cap=B * 6, max_ids=6)
        seen = set()
        batches = [_ragged(rng, B, 200, 6) for _ in range(R)]
        for b in batches:
            seen.update(_signs(oracle, b[0], pf))
        octx = _forward(torch, ws, w, batches, B, fixed)
        _backward(torch, ws, w, octx, [(rng.standard_normal((u, dim)) * 1e-2).astype(np.float32) for u, _ in octx])
        sizes = [len(x.shard) for x in ws]
        batches = [_ragged(rng, B, 400, 6) for _ in range(R)]  # half of these were never seen
        _forward(torch, ws, w, batches, B, fixed, training=False)
        assert [len(x.shard) for x in ws] == sizes
        _check_rows(torch, oracle, [x.shard for x in ws], w, seen, R, ws)
    finally:
        oracle.set_rsqrt_exact(False)


def test_raw_negative_zero_survives(torch_cuda, oracle):
    """A -0 element of a row reaches the f16 table as 0x8000: the requester rounds the f32 row itself."""
    torch = torch_cuda
    R, B, dim, fixed = 2, 8, 16, 2
    pf = oracle.index_prefix(0)
    ws, w = _raw_group(torch, oracle, R, dim, oracle.SGD, B, fixed, pf, cap=64)
    signs = oracle.add_prefix(np.arange(B, dtype=np.uint64), 8, pf)
    owner = oracle.shard_of(signs, R)
    L = ws[0].shard.entry_len
    ent = np.full((B, L), 0.25, np.float32)
    ent[:, 1::2] = -0.0
    for r in range(R):
        mine = owner == r
        if mine.any():
            ws[r].shard.set_entries(to_dev_ids(signs[mine], DEV), torch.from_numpy(ent[mine].copy()).to(DEV))
    w.set_embedding(signs, ent, dim)
    torch.cuda.synchronize()
    ids = np.arange(B, dtype=np.uint64)
    batches = [(ids, np.arange(B + 1, dtype=np.uint32))] * R
    for training in (False, True):  # (the oracle's table holds f16(row): its -0 elements are 0x8000 too)
        _forward(torch, ws, w, batches, B, fixed, training=training, single=True)


def test_raw_negative_zero_bits(torch_cuda, oracle):
    """The same, read as bits (R = 1: a whole call per rank needs no peer)."""
    torch = torch_cuda
    B, dim, fixed = 4, 8, 1
    pf = oracle.index_prefix(0)
    ws, w = _raw_group(torch, oracle, 1, dim, oracle.SGD, B, fixed, pf, cap=16)
    signs = oracle.add_prefix(np.arange(B, dtype=np.uint64), 8, pf)
    ent = np.full((B, ws[0].shard.entry_len), -0.0, np.float32)
    ws[0].shard.set_entries(to_dev_ids(signs, DEV), torch.from_numpy(ent).to(DEV))
    torch.cuda.synchronize()
    table, _, _, _, counts = ws[0].forward_raw(to_dev_ids(np.arange(B, dtype=np.uint64), DEV), B, fixed, training=False)
    U = int(counts[0])
    bits = table[1:U + 1].cpu().numpy().view(np.uint16)
    assert U == B and (bits == 0x8000).all()
    assert (table[0].cpu().numpy().view(np.uint16) == 0).all()


@pytest.mark.parametrize("kind", [0, 2, 3])  # SGD, vectorwise Adagrad (per-request owner kernel), Adam (shared beta powers)
def test_raw_mixed_step_shares_the_table(torch_cuda, oracle, kind):
    """Per rank: a summation worker with 3 slots and two raw slots of the same dim on the same table.  The step's calls
    run in one order on every rank — raw slots in batch order, then the summation slots — and the oracle, one worker
    holding all five slots, applies the requests in that order."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker, ShardedRawWorker as RW

    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(33 + kind)
        R, B, dim, fixed, max_ids = 3, 200, 32, 4, 6
        pf = [oracle.index_prefix(i) for i in range(5)]
        gpu_opt, cpu_opt = _optim(N, oracle, kind)
        sw = ShardedEmbeddingWorker.local_group(R, 3, dim, pf[:3], 1 << 16, cap=3 * B, optimizer=gpu_opt, max_batch=B)
        shards = [x.shard for x in sw]
        rws = [RW.local_group(R, 1, dim, [pf[3 + i]], 1 << 16, cap=B * max_ids, optimizer=gpu_opt, max_batch=B,
                              max_ids_per_sample=max_ids, shards=shards) for i in range(2)]
        assert all(rws[i][r].shard is shards[r] for i in range(2) for r in range(R))
        w = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pf[:3]] +
                          [oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=p) for p in pf[3:]], n_ps=R)
        w.configure()
        w.set_optimizer(cpu_opt)
        _warm(torch, sw)
        # the summation slots hold one id per sample; the raw slots take no part in the oracle's summation requests
        sum_off = np.concatenate([np.arange(3 * B + 1, dtype=np.uint32), np.full(2 * B, 3 * B, np.uint32)])
        seen = set()
        for step in range(3):
            raw_b = [[_ragged(rng, B, 150, max_ids) for _ in range(R)] for _ in range(2)]
            sum_ids = [np.concatenate([rng.integers(0, c, size=B, dtype=np.uint64) for c in (20, 300, 5000)])
                       for _ in range(R)]
            for i in range(2):
                for b in raw_b[i]:
                    seen.update(_signs(oracle, b[0], pf[3 + i]))
            for r in range(R):
                for s in range(3):
                    seen.update(_signs(oracle, sum_ids[r][s * B:(s + 1) * B], pf[s]))
            octx = [_forward(torch, rws[i], w, raw_b[i], B, fixed, slot=3 + i) for i in range(2)]
            torch.cuda.synchronize()
            outs = ShardedEmbeddingWorker.group_forward(sw, [to_dev_ids(x, DEV) for x in sum_ids], B, training=True)
            torch.cuda.synchronize()
            sctx = []
            for r in range(R):
                want, c = w.forward(sum_ids[r], sum_off, B, training=True)
                sctx.append(c)
                got = outs[r].cpu().numpy()
                for s in range(3):
                    np.testing.assert_array_equal(got[s].view(np.uint16), want[s].view(np.uint16))
            for i in range(2):
                grads = [(rng.standard_normal((u, dim)) * 1e-2).astype(np.float32) for u, _ in octx[i]]
                _backward(torch, rws[i], w, octx[i], grads, slot=3 + i)
            g = (rng.standard_normal((R, 3, B, dim)) * 1e-2).astype(np.float16)
            torch.cuda.synchronize()
            ShardedEmbeddingWorker.group_backward(sw, [[torch.from_numpy(g[r, s]).to(DEV) for s in range(3)] for r in range(R)])
            torch.cuda.synchronize()
            for r in range(R):
                zero = np.zeros((B, dim), np.float16)
                w.backward(sctx[r], [g[r, s] for s in range(3)] + [zero, zero], skip=[0, 0, 0, 1, 1])
        _check_rows(torch, oracle, shards, w, seen, R, sw + rws[0] + rws[1])
    finally:
        oracle.set_rsqrt_exact(False)


def test_raw_pending_rows_survive_eviction(torch_cuda, oracle):
    """Four raw slots of one dim on each rank's table; before every training forward the capacity sweep releases every
    row older than keep_batches = 1 request.  The first slot's rows are two requests old when the fourth forward
    sweeps: they are spared only because pending raw forwards count as pending batches, so every gradient still lands
    on its own sign's row and nothing is evicted before the backward."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedRawWorker as RW

    torch = torch_cuda
    rng = np.random.default_rng(77)
    R, B, dim, fixed, max_ids, n_raw = 2, 64, 16, 3, 4, 4
    pf = [oracle.index_prefix(i) for i in range(n_raw)]
    gpu_opt, cpu_opt = _optim(N, oracle, oracle.SGD)
    first = RW.local_group(R, 1, dim, [pf[0]], 1 << 12, cap=B * max_ids, optimizer=gpu_opt, max_batch=B,
                           max_ids_per_sample=max_ids)
    shards = [x.shard for x in first]
    groups = [first] + [RW.local_group(R, 1, dim, [p], 1 << 12, cap=B * max_ids, optimizer=gpu_opt, max_batch=B,
                                       max_ids_per_sample=max_ids, shards=shards) for p in pf[1:]]
    for s in shards:
        s.set_eviction(check_every=1, low_water=s.capacity, target_free=s.capacity, keep_batches=1)
    w = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=p) for p in pf], n_ps=R)
    w.configure()
    w.set_optimizer(cpu_opt)
    _warm(torch, first)
    batches = [[_ragged(rng, B, 100, max_ids, allow_empty=False) for _ in range(R)] for _ in range(n_raw)]
    seen = {s for i in range(n_raw) for b in batches[i] for s in _signs(oracle, b[0], pf[i])}
    octx = [_forward(torch, groups[i], w, batches[i], B, fixed, slot=i) for i in range(n_raw)]
    for i in range(n_raw):
        grads = [(rng.standard_normal((u, dim)) * 1e-2).astype(np.float32) for u, _ in octx[i]]
        _backward(torch, groups[i], w, octx[i], grads, slot=i)
    _check_rows(torch, oracle, shards, w, seen, R, [x for g in groups for x in g])


def test_raw_no_prefix_marker_signs(torch_cuda, oracle):
    """index_prefix 0: ids reach the owners unchanged, including 2^64-1 (the scratch set's extra cell) and the values
    that collide with the index's cell markers, which every owner keeps in cells of their own."""
    torch = torch_cuda
    R, B, dim, fixed = 3, 4, 8, 3
    ws, w = _raw_group(torch, oracle, R, dim, oracle.SGD, B, fixed, 0, cap=64, max_ids=4)
    base = np.array([M - 1, 7, M - 2, M - 1, M - 3, 7, M - 3, 0], np.uint64)
    row_off = np.array([0, 3, 3, 7, 8], np.uint32)
    for it in range(2):
        batches = [(np.roll(base, r + it), row_off) for r in range(R)]
        octx = _forward(torch, ws, w, batches, B, fixed)
        assert all(u == 5 for u, _ in octx)
        _backward(torch, ws, w, octx, [np.full((5, dim), 0.25 * (it + r + 1), np.float32) for r in range(R)])
    _check_rows(torch, oracle, [x.shard for x in ws], w, np.unique(base), R, ws)


def test_raw_overflow_is_flagged(torch_cuda, oracle):
    """A pair that needs more than cap slots raises the status flag, never the wait flag."""
    torch = torch_cuda
    from persia_b200.worker import ShardedRawWorker as W

    R, B, dim = 2, 256, 16
    ws, _ = _raw_group(torch, oracle, R, dim, oracle.SGD, B, 2, oracle.index_prefix(0), cap=16)
    ids = [to_dev_ids(np.arange(B, dtype=np.uint64) + 1000 * r, DEV) for r in range(R)]
    torch.cuda.synchronize()
    W.group_forward_raw(ws, ids, B, 2, training=False)
    torch.cuda.synchronize()
    assert all(x.status()[0] for x in ws) and not any(x.status()[1] for x in ws)


def test_raw_graph_replay(torch_cuda, oracle):
    """The raw forward and backward phases of every rank captured in CUDA graphs (single-id layout: n_occ is fixed) and
    replayed for three steps with new ids and gradients; U stays on the device."""
    from persia_b200 import native as N

    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(17)
        R, B, dim, fixed = 4, 256, 64, 3
        pf = oracle.index_prefix(0)
        ws, w = _raw_group(torch, oracle, R, dim, oracle.ADAGRAD, B, fixed, pf, cap=B)
        ids_dev = [torch.zeros(B, dtype=torch.int64, device=DEV) for _ in range(R)]
        g_dev = [torch.zeros((B, dim), dtype=torch.float32, device=DEV) for _ in range(R)]
        bufs = [None] * R
        fwd = (N.PHASE_SEND, N.PHASE_SERVE, N.PHASE_FINISH)
        bwd = (N.PHASE_SEND, N.PHASE_SERVE)

        def enqueue(r, kind, ph):
            if kind == "f":
                bufs[r] = ws[r].forward_raw(ids_dev[r], B, fixed, training=True, out=bufs[r], phases=ph)
            else:
                ws[r].backward_raw(g_dev[r], phases=ph)

        torch.cuda.synchronize()
        for kind, phs in (("f", fwd), ("b", bwd)):  # eager warm-up step: id 0 everywhere, zero gradients
            for ph in phs:
                for r in range(R):
                    enqueue(r, kind, ph)
        torch.cuda.synchronize()
        zero = np.zeros(B, np.uint64)
        octx = [w.forward_raw(0, zero, np.arange(B + 1, dtype=np.uint32), B)[4] for _ in range(R)]
        for r in range(R):
            w.backward_raw(0, octx[r], np.zeros((1, dim), np.float32))
        graphs = {}
        for r in range(R):
            for kind, phs in (("f", fwd), ("b", bwd)):
                for ph in phs:
                    gph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(gph, stream=ws[r].stream, capture_error_mode="thread_local"):
                        enqueue(r, kind, ph)
                    graphs[(r, kind, ph)] = gph
        seen = {int(oracle.add_prefix(zero[:1], 8, pf)[0])}
        for it in range(3):
            ids = [rng.integers(0, 700, size=B, dtype=np.uint64) for _ in range(R)]
            for r in range(R):
                ids_dev[r].copy_(to_dev_ids(ids[r], DEV))
                seen.update(_signs(oracle, ids[r], pf))
            torch.cuda.synchronize()
            for ph in fwd:
                for r in range(R):
                    with torch.cuda.stream(ws[r].stream):
                        graphs[(r, "f", ph)].replay()
            torch.cuda.synchronize()
            octx, grads = [], []
            for r in range(R):
                table, index, non_empty, num, counts = bufs[r]
                U, ne = counts.cpu().numpy().tolist()
                wt, wi, wne, wnum, c = w.forward_raw(0, ids[r], np.arange(B + 1, dtype=np.uint32), B)
                assert table[:U + 1].cpu().numpy().tobytes() == wt.tobytes()
                np.testing.assert_array_equal(index.cpu().numpy(), wi)
                np.testing.assert_array_equal(non_empty[:ne].cpu().numpy(), wne)
                np.testing.assert_array_equal(num[:B].cpu().numpy().view(np.uint32), wnum)
                octx.append(c)
                g = (rng.standard_normal((U, dim)) * 1e-2).astype(np.float32)
                g_dev[r][:U].copy_(torch.from_numpy(g).to(DEV))
                grads.append(g)
            torch.cuda.synchronize()
            for ph in bwd:
                for r in range(R):
                    with torch.cuda.stream(ws[r].stream):
                        graphs[(r, "b", ph)].replay()
            torch.cuda.synchronize()
            for r in range(R):
                assert w.backward_raw(0, octx[r], grads[r]) == 0
        _check_rows(torch, oracle, [x.shard for x in ws], w, seen, R, ws)
    finally:
        oracle.set_rsqrt_exact(False)


def test_raw_sharded_abi_refusals(torch_cuda, oracle):
    """Bad arguments are refused before anything is enqueued: no launch, no change to the table."""
    import ctypes as C

    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200.worker import ShardedEmbeddingWorker, ShardedRawWorker

    torch = torch_cuda
    lib = N.load()
    B, dim, fixed = 16, 16, 2
    pf = oracle.index_prefix(0)
    ws, w = _raw_group(torch, oracle, 1, dim, oracle.SGD, B, fixed, pf, cap=64)
    x = ws[0]
    ids = to_dev_ids(np.arange(B, dtype=np.uint64), DEV)
    octx = _forward(torch, ws, w, [(np.arange(B, dtype=np.uint64), np.arange(B + 1, dtype=np.uint32))], B, fixed,
                    single=True)
    signs = to_dev_ids(oracle.add_prefix(np.arange(B, dtype=np.uint64), 8, pf), DEV)
    before = x.shard.get_entries(signs)[0].cpu().numpy()
    n_before = len(x.shard)
    table = torch.empty((B + 2, dim), dtype=torch.float16, device=DEV)
    index = torch.empty(B * fixed, dtype=torch.int64, device=DEV)
    ne = torch.empty(B * fixed, dtype=torch.int64, device=DEV)
    num = torch.empty(B, dtype=torch.int32, device=DEV)
    counts = torch.empty(2, dtype=torch.int32, device=DEV)
    ctx2 = SH.BatchContext(64, 64, [pf, oracle.index_prefix(1)], device=torch.device(DEV))
    other = ShardedRawWorker.local_group(1, 1, 32, [pf], 1 << 10, cap=64, optimizer=dict(kind=N.OPT_SGD, lr=0.1),
                                         max_batch=B)[0]
    f16x = ShardedEmbeddingWorker.local_group(1, 1, dim, [pf], 1 << 10, cap=64, optimizer=dict(kind=N.OPT_SGD, lr=0.1),
                                              max_batch=B)[0]
    st = C.c_void_p(x.stream.cuda_stream)

    def fwd(shard=x.shard.h, ctx=x.ctx.h, xchg=x.h, tab=table.data_ptr(), fx=fixed):
        return lib.pb_forward_raw_sharded(shard, ctx, xchg, ids.data_ptr(), B, None, B, fx, 1, tab, index.data_ptr(),
                                          ne.data_ptr(), num.data_ptr(), counts.data_ptr(), st, 0)

    g = torch.zeros((B + 1, dim), dtype=torch.float32, device=DEV)
    torch.cuda.synchronize()
    launches = lib.pb_launch_count()
    assert fwd(tab=table.data_ptr() + 2) == N.PB_ERR_INVALID      # misaligned table
    assert fwd(xchg=other.h) == N.PB_ERR_INVALID                   # exchange of another dim
    assert fwd(ctx=ctx2.h) == N.PB_ERR_STATE                       # a 2-slot context
    assert fwd(fx=0) == N.PB_ERR_INVALID                           # sample_fixed_size 0
    assert fwd(xchg=f16x.h, ctx=f16x.ctx.h, shard=f16x.shard.h) == N.PB_ERR_INVALID  # f16 rows
    assert lib.pb_backward_raw_sharded(x.shard.h, x.ctx.h, x.h, g.data_ptr() + 4, 0, 1.0, None, st, 0) == N.PB_ERR_INVALID
    assert lib.pb_backward_raw_sharded(x.shard.h, x.ctx.h, other.h, g.data_ptr(), 0, 1.0, None, st, 0) == N.PB_ERR_INVALID
    assert lib.pb_backward_raw_sharded(x.shard.h, ctx2.h, x.h, g.data_ptr(), 0, 1.0, None, st, 0) == N.PB_ERR_STATE
    assert lib.pb_backward_raw_sharded(other.shard.h, other.ctx.h, other.h, g.data_ptr(), 0, 1.0, None, st, 0) == N.PB_ERR_STATE
    torch.cuda.synchronize()
    assert lib.pb_launch_count() == launches
    assert len(x.shard) == n_before
    assert x.shard.get_entries(signs)[0].cpu().numpy().tobytes() == before.tobytes()
    # the pending forward still takes its gradient; a second backward is "backward_ref_id not found"
    x.backward_raw(g[:octx[0][0]])
    from persia_b200.native import PersiaB200Error
    with pytest.raises(PersiaB200Error):
        x.backward_raw(g[:octx[0][0]])


@pytest.mark.parametrize("dim", [12, 130])
def test_summation_adam_per_request_owner_update(torch_cuda, oracle, dim):
    """Rows the single-launch owner update cannot cover with one chunk per lane (dim 12: three 4-wide chunks; 130: odd)
    are stepped by the per-request kernel, which the raw path shares with the summation path.  With Adam it must use
    each request's beta powers, like the single-launch kernel."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    rng = np.random.default_rng(dim)
    R, S, B = 3, 2, 200
    pf = [oracle.index_prefix(i) for i in range(S)]
    gpu_opt, cpu_opt = _optim(N, oracle, oracle.ADAM)
    ws = W.local_group(R, S, dim, pf, 1 << 16, cap=S * B, optimizer=gpu_opt, max_batch=B)
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pf], n_ps=R)
    w.configure()
    w.set_optimizer(cpu_opt)
    _warm(torch, ws)
    row_off = np.arange(S * B + 1, dtype=np.uint32)
    seen = set()
    for step in range(3):
        ids = [np.concatenate([rng.integers(0, c, size=B, dtype=np.uint64) for c in (40, 900)]) for _ in range(R)]
        torch.cuda.synchronize()
        outs = W.group_forward(ws, [to_dev_ids(x, DEV) for x in ids], B, training=True)
        torch.cuda.synchronize()
        octx = []
        for r in range(R):
            want, c = w.forward(ids[r], row_off, B, training=True)
            octx.append(c)
            for s in range(S):
                np.testing.assert_array_equal(outs[r][s].cpu().numpy().view(np.uint16), want[s].view(np.uint16))
                seen.update(_signs(oracle, ids[r][s * B:(s + 1) * B], pf[s]))
        g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float32)
        torch.cuda.synchronize()
        W.group_backward(ws, [[torch.from_numpy(g[r, s]).to(DEV) for s in range(S)] for r in range(R)])
        torch.cuda.synchronize()
        for r in range(R):
            w.backward(octx[r], [g[r, s] for s in range(S)])
    _check_rows(torch, oracle, [x.shard for x in ws], w, seen, R, ws)


# ---- one process per GPU over symmetric memory (needs >= 2 GPUs) --------------------------------------------------------
def _rank_main(rank, world, port, result_dir):
    import torch
    import torch.distributed as dist

    import oracle
    from persia_b200 import native as N
    from persia_b200.worker import ShardedRawWorker

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    B, dim, fixed, max_ids = 300, 64, 5, 8
    pf = oracle.index_prefix(0)
    wk = ShardedRawWorker.distributed(1, dim, [pf], 1 << 16, B * max_ids, dict(kind=N.OPT_ADAGRAD, lr=0.02,
                                      initialization=0.01, eps=1e-10), dev, max_batch=B, max_ids_per_sample=max_ids)
    rng = np.random.default_rng(42)
    res, seen = {}, set()
    for step in range(3):
        batches = [_ragged(rng, B, 400, max_ids) for _ in range(world)]  # every rank draws all, keeps its own
        ids, row_off = batches[rank]
        table, index, ne, num, counts = wk.forward_raw(torch.from_numpy(ids.view(np.int64)).to(dev), B, fixed,
                                                       row_off=torch.from_numpy(row_off.view(np.int32)).to(dev))
        U = int(counts[0])
        gs = [(rng.standard_normal((int(np.unique(b[0]).size), dim)) * 1e-2).astype(np.float32) for b in batches]
        wk.backward_raw(torch.from_numpy(gs[rank]).to(dev))
        torch.cuda.synchronize()
        dist.barrier()
        res[f"table{step}"] = table[:U + 1].cpu().numpy()
        res[f"index{step}"] = index.cpu().numpy()
        for b in batches:
            seen.update(oracle.add_prefix(b[0], 8, pf).tolist())
    signs = np.array(sorted(seen), np.uint64)
    mine = signs[oracle.shard_of(signs, world) == rank]
    ent, found = wk.shard.get_entries(torch.from_numpy(mine.view(np.int64)).to(dev))
    assert found.all() and wk.status() == (False, False)
    np.savez(os.path.join(result_dir, f"rank{rank}.npz"), signs=mine, ent=ent.cpu().numpy(), **res)
    dist.barrier()
    dist.destroy_process_group()


def test_raw_two_processes_symmetric_memory(torch_cuda, oracle, tmp_path):
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs; the virtual-rank tests above cover R > 1 on one GPU")
    import torch.multiprocessing as mp

    world = 2
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_rank_main, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    oracle.set_rsqrt_exact(True)
    try:
        B, dim, fixed, max_ids = 300, 64, 5, 8
        pf = oracle.index_prefix(0)
        w = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=pf)], n_ps=world)
        w.configure()
        w.set_optimizer(oracle.Optim(oracle.ADAGRAD, lr=0.02, init_acc=0.01, eps=1e-10))
        rng = np.random.default_rng(42)
        res = [np.load(os.path.join(str(tmp_path), f"rank{r}.npz")) for r in range(world)]
        for step in range(3):
            batches = [_ragged(rng, B, 400, max_ids) for _ in range(world)]
            gs = [(rng.standard_normal((int(np.unique(b[0]).size), dim)) * 1e-2).astype(np.float32) for b in batches]
            octx = []
            for r in range(world):
                wt, wi, _, _, c = w.forward_raw(0, batches[r][0], batches[r][1], B)
                assert res[r][f"table{step}"].tobytes() == wt.tobytes()
                np.testing.assert_array_equal(res[r][f"index{step}"], wi)
                octx.append(c)
            for r in range(world):
                w.backward_raw(0, octx[r], gs[r])
        for r in range(world):
            for k, sign in enumerate(res[r]["signs"]):
                assert res[r]["ent"][k].tobytes() == w.get_entry(int(sign)).tobytes()
    finally:
        oracle.set_rsqrt_exact(False)


# ---- two processes, two GPUs: TrainCtx with a raw slot beside summation slots of its dim ----------------------------------
_TC_B, _TC_DIM, _TC_FIXED, _TC_STEPS, _TC_DENSE = 128, 32, 4, 4, 6
_TC_CONFIG = {"slots_config": {"seq": {"dim": _TC_DIM, "embedding_summation": False, "sample_fixed_size": _TC_FIXED},
                               "s0": {"dim": _TC_DIM}, "s1": {"dim": _TC_DIM}, "s2": {"dim": _TC_DIM}}}


def _tc_batch(rng):
    """One rank's batch: a sequence feature (0..6 ids per sample, some rows longer than sample_fixed_size) and three
    one-id features of the same dim."""
    seq = [rng.integers(0, 60, size=int(rng.integers(0, 7)), dtype=np.uint64) for _ in range(_TC_B)]
    sums = [rng.integers(0, c, size=_TC_B, dtype=np.uint64) for c in (5, 300, 5000)]
    dense = rng.standard_normal((_TC_B, _TC_DENSE)).astype(np.float32)
    label = (dense[:, 0] > 0).astype(np.float32).reshape(_TC_B, 1)
    return seq, sums, dense, label


def _trainctx_raw_rank(rank, world, port, result_dir):
    import torch

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    import oracle
    from persia_b200 import api
    from persia_b200 import persia_core as PC

    class Tower(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(4 * _TC_DIM + _TC_DENSE, 1)

        def forward(self, non_id, emb):
            parts = [non_id[0]]
            for e in emb:
                if e.dim() == 3:  # raw slot: [B, fixed, dim + 1], the last channel is the padding mask
                    e = e[:, :, :-1].sum(dim=1)
                parts.append(e.float())
            return self.lin(torch.cat(parts, dim=1)).squeeze(1)

    PC.reset()
    PC.set_embedding_config(_TC_CONFIG)
    torch.manual_seed(0)
    model = Tower().cuda()
    dense_opt = torch.optim.SGD(model.parameters(), lr=0.1)
    loss_fn = torch.nn.BCEWithLogitsLoss()
    rng = np.random.default_rng(5)
    _, slots = PC.parse_embedding_config(_TC_CONFIG)
    pf = {s.name: s.index_prefix for s in slots}
    res, seen = {}, set()
    with api.TrainCtx(model=model, embedding_optimizer=api.Adagrad(lr=0.05), dense_optimizer=dense_opt, device_id=rank,
                      mixed_precision=False, embedding_config=api.EmbeddingConfig()) as ctx:
        for step in range(_TC_STEPS):
            batches = [_tc_batch(rng) for _ in range(world)]  # every rank draws all, keeps its own
            for seq, sums, _, _ in batches:
                for x in seq:
                    seen.update(oracle.add_prefix(x, 8, pf["seq"]).tolist())
                for i in range(3):
                    seen.update(oracle.add_prefix(sums[i], 8, pf[f"s{i}"]).tolist())
            seq, sums, dense, label = batches[rank]
            pb = api.PersiaBatch([api.IDTypeFeature("seq", seq)] +
                                 [api.IDTypeFeatureWithSingleID(f"s{i}", sums[i]) for i in range(3)],
                                 non_id_type_features=[api.NonIDTypeFeature(dense, name="dense")],
                                 labels=[api.Label(label, name="click")], requires_grad=True)
            out, labels = ctx.forward(ctx.get_embedding_from_data(pb, 0))
            cache = ctx.current_batch.id_type_feature_embedding_cache_torch_tensors
            _, distinct, index, nz, sel = cache[0]
            res[f"table{step}"] = distinct.detach().cpu().numpy()
            res[f"index{step}"] = index.cpu().numpy()
            res[f"embs{step}"] = np.stack([c[-1].detach().cpu().numpy() for c in cache[1:]])
            ctx.backward(loss_fn(out, labels[0].squeeze(1)))
            # the [U, dim] f32 gradient TrainCtx hands over for the raw slot (persia/ctx.py:970-980)
            g = torch.zeros_like(distinct, dtype=torch.float32)
            g.index_add_(0, index.view(-1)[nz.view(-1)], sel.grad.index_select(0, nz.view(-1)).float())
            res[f"rawgrad{step}"] = g[1:].cpu().numpy()
            res[f"grads{step}"] = np.stack([c[-1].grad.detach().cpu().numpy() for c in cache[1:]])
        ctx.backward_engine.flush()
        torch.cuda.synchronize()
        import torch.distributed as dist

        dist.barrier()
        signs = np.array(sorted(seen), np.uint64)
        ent = ctx.common_context.get_entries(signs, _TC_DIM, missing_ok=True)
        keep = [k for k, e in enumerate(ent) if e is not None]
        np.savez(os.path.join(result_dir, f"rank{rank}.npz"), signs=signs[keep], ent=np.stack([ent[k] for k in keep]),
                 **res)
        dist.barrier()
    PC.reset()


def test_two_process_trainctx_raw_slot_matches_oracle(torch_cuda, oracle, tmp_path):
    """TrainCtx on two ranks with replica_size 2: a raw slot consumed as persia/ctx.py consumes it (index_select of the
    distinct-sign table, the [U, dim] gradient built by index_add) beside three summation slots of the same dim, all on
    each rank's one table.  The oracle with 2 parameter servers replays the step in the ranks' call order: raw slot,
    then the summation slots; each forward and each backward in rank order."""
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    from persia_b200 import persia_core as PC

    world = 2
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    saved = {k: os.environ.pop(k, None) for k in ("RANK", "WORLD_SIZE")}
    try:
        mp.spawn(_trainctx_raw_rank, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    finally:
        os.environ.update({k: v for k, v in saved.items() if v is not None})
    res = [np.load(os.path.join(str(tmp_path), f"rank{r}.npz")) for r in range(world)]
    _, slots = PC.parse_embedding_config(_TC_CONFIG)
    pf = {s.name: s.index_prefix for s in slots}
    B, dim = _TC_B, _TC_DIM
    w = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=_TC_FIXED, prefix=pf["seq"])] +
                      [oracle.SlotCfg(dim, prefix=pf[f"s{i}"]) for i in range(3)], n_ps=world)
    w.configure(wb=10.0)
    w.set_optimizer(oracle.Optim(oracle.ADAGRAD, lr=0.05, init_acc=0.01, eps=1e-10))
    # the summation requests carry no ids of the raw slot (slot 0)
    sum_off = np.concatenate([np.zeros(B, np.uint32), np.arange(3 * B + 1, dtype=np.uint32)])
    rng = np.random.default_rng(5)
    oracle.set_rsqrt_exact(True)
    try:
        for step in range(_TC_STEPS):
            batches = [_tc_batch(rng) for _ in range(world)]
            rctx, sctx = [], []
            for r in range(world):
                seq_ids, seq_off = oracle.lil_to_csr([x.tolist() for x in batches[r][0]])
                wt, wi, _, _, c = w.forward_raw(0, seq_ids, seq_off, B)
                assert res[r][f"table{step}"].tobytes() == wt.tobytes(), (step, r)
                np.testing.assert_array_equal(res[r][f"index{step}"], wi)
                rctx.append(c)
            for r in range(world):
                want, c = w.forward(np.concatenate(batches[r][1]), sum_off, B, training=True)
                for i in range(3):
                    assert res[r][f"embs{step}"][i].tobytes() == want[1 + i].tobytes(), (step, r, i)
                sctx.append(c)
            for r in range(world):
                g = res[r][f"rawgrad{step}"]
                assert w.backward_raw(0, rctx[r], g if g.shape[0] else None, skip=not g.shape[0]) in (0, 1)
            for r in range(world):
                zero = np.zeros((B, dim), np.float16)
                w.backward(sctx[r], [zero] + [res[r][f"grads{step}"][i] for i in range(3)], skip=[1, 0, 0, 0])
        n = 0
        for r in range(world):
            for k, sign in enumerate(res[r]["signs"]):
                assert res[r]["ent"][k].tobytes() == w.get_entry(int(sign)).tobytes(), (r, k)
                n += 1
        assert n > 0
    finally:
        oracle.set_rsqrt_exact(False)
