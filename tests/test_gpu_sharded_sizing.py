"""GPU: every sharded step sized from its own batch (PB_PHASE_PREPARE, pb_xchg_need, the workers' prepare / resize), on
R virtual ranks of one GPU.

A worker starts from a small first batch (cap 8, B = 16) and later batches — larger, ragged, skewed, a raw slot that
grows — are prepared, agreed (the max over the ranks, as persia_core's all-reduce) and resized before they are sent.
Every step must equal the oracle's embedding worker with R parameter servers, as test_gpu_worker.py checks it, and
PREPARE alone must leave every table, counter and exchange as it was."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_gpu_worker import _optim  # noqa: E402
from util import held_rows, make_batch, pool_model, same_bits, slot_signs, to_dev_i32, to_dev_ids  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MARKERS = np.array([2 ** 64 - 1, 2 ** 64 - 2, 2 ** 64 - 3], np.uint64)  # the index's reserved keys, as signs


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _warm(torch, ws):
    for x in ws:  # table storage is allocated on first use, with a device-wide sync: not while a peer spins on a flag
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()


def _ragged_raw(rng, B, card, max_ids):
    counts = rng.integers(0, max_ids + 1, size=B)
    row_off = np.zeros(B + 1, np.uint32)
    row_off[1:] = np.cumsum(counts)
    return rng.integers(0, card, size=int(row_off[-1]), dtype=np.uint64), row_off


# ---- PREPARE's count ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prefix_bit", [8, 12])
@pytest.mark.parametrize("R", [1, 2, 3, 4, 5])
def test_prepare_counts_match_host(torch_cuda, oracle, R, prefix_bit):
    """Each rank's need is the most distinct (slot, sign) items it sends one owner, as distinct_per_owner counts them:
    single-id and ragged (with empty samples) layouts, slots sharing a feature group, the marker-valued signs (no
    prefix), and a raw slot."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW, distinct_per_owner

    torch = torch_cuda
    rng = np.random.default_rng(10 * R + prefix_bit)
    S, B, dim = 4, 300, 16
    gpu_opt, _ = _optim(N, oracle, oracle.SGD)
    p = [(i + 1) << (64 - prefix_bit) for i in range(S)]
    layouts = {"distinct": p, "shared": [p[0], p[0], p[1], p[1]], "marker": [0] * S}
    for name, pf in layouts.items():
        ws = W.local_group(R, S, dim, pf, 1 << 14, cap=8, optimizer=gpu_opt, max_batch=16, prefix_bit=prefix_bit)
        for ragged in (False, True):
            for r, w in enumerate(ws):
                ids, row_off, slot_off = make_batch(rng, S, B, [5, 200, 5000, 1 << 40], max_ids=4 if ragged else 1,
                                                    allow_empty=ragged)
                if name == "marker":
                    ids[:3] = MARKERS
                need, f32 = w.prepare(to_dev_ids(ids, DEV), B, to_dev_i32(row_off, DEV) if ragged else None, slot_off)
                want = distinct_per_owner([ids[slot_off[s]:slot_off[s + 1]] for s in range(S)], pf, R, prefix_bit)
                assert (need, f32) == (int(want.max()), ragged), (name, ragged, r)
        for w in ws:
            w.close()
        for pr in (p[0], 0):
            rws = RW.local_group(R, 1, dim, [pr], 1 << 14, cap=8, optimizer=gpu_opt, max_batch=16, prefix_bit=prefix_bit)
            for r, w in enumerate(rws):
                ids, row_off = _ragged_raw(rng, B, 3000, 6)
                if not pr:
                    ids[:3] = MARKERS
                need, f32 = w.prepare_raw(to_dev_ids(ids, DEV), B, 4, to_dev_i32(row_off, DEV))
                assert (need, f32) == (int(distinct_per_owner([ids], [pr], R, prefix_bit).max()), True), (pr, r)
            for w in rws:
                w.close()
    torch.cuda.synchronize()


# ---- PREPARE alone changes nothing -------------------------------------------------------------------------------------
def _snapshot(ws):
    """Every rank's counters, index stats, incremental stats, exchange status, resident signs with their recency, and
    their entries (read last, and only of resident signs: a read-back of an absent sign counts as a lookup miss)."""
    out = []
    for w in ws:
        s = w.shard
        head = (s.counters(), s.index_stats(), s.incremental_stats(), w.status())
        es, er = s.export_signs()
        ent, found = s.get_entries(es)
        assert found.all()
        out.append(head + (es.cpu().numpy().tobytes(), er.cpu().numpy().tobytes(), ent.cpu().numpy().tobytes()))
    return out


def test_prepare_has_no_side_effects(torch_cuda, oracle):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW

    torch = torch_cuda
    rng = np.random.default_rng(5)
    R, S, B, dim = 3, 3, 200, 32
    pf = [oracle.index_prefix(i) for i in range(S + 1)]
    gpu_opt, _ = _optim(N, oracle, oracle.ADAGRAD)
    ws = W.local_group(R, S, dim, pf[:S], 1 << 12, cap=S * B, optimizer=gpu_opt, max_batch=B)
    rws = RW.local_group(R, 1, dim, [pf[S]], 1 << 12, cap=4 * B, optimizer=gpu_opt, max_batch=B, max_ids_per_sample=4,
                         shards=[w.shard for w in ws])
    for w in ws:
        w.shard.set_eviction(check_every=1, low_water=1 << 11, target_free=1 << 11, keep_batches=1)
        w.shard.enable_incremental(1 << 14)
    _warm(torch, ws)
    card = [50, 3000, 1 << 30]
    first = [make_batch(rng, S, B, card)[0] for _ in range(R)]
    W.group_forward(ws, [to_dev_ids(x, DEV) for x in first], B)
    W.group_backward(ws, [torch.full((S, B, dim), 0.01, dtype=torch.float16, device=DEV) for _ in range(R)])
    torch.cuda.synchronize()
    later = [make_batch(rng, S, 2 * B, card, max_ids=3, allow_empty=True) for _ in range(R)]
    raw = [_ragged_raw(rng, B, 2000, 4) for _ in range(R)]
    for b in later:
        b[0][:3] = MARKERS
    before = _snapshot(ws)
    W.group_prepare(ws, [to_dev_ids(b[0], DEV) for b in later], 2 * B, row_offs=[to_dev_i32(b[1], DEV) for b in later],
                    slot_occ_offs=[b[2] for b in later])
    RW.group_prepare_raw(rws, [to_dev_ids(b[0], DEV) for b in raw], B, 4, row_offs=[to_dev_i32(b[1], DEV) for b in raw])
    torch.cuda.synchronize()
    after = _snapshot(ws)
    for r in range(R):
        for k, (x, y) in enumerate(zip(after[r], before[r])):
            assert x == y, (r, k)
    assert [w.status() for w in rws] == [(False, False)] * R


# ---- PREPARE then SEND equals SEND -------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 2, 3])
def test_prepare_then_send_equals_plain(torch_cuda, oracle, R):
    """Two identical groups get the same batches; one prepares every batch first.  Outputs and tables agree bit for bit
    (R = 1: against phases = 0 itself)."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW

    torch = torch_cuda
    rng = np.random.default_rng(40 + R)
    S, B, dim, fixed = 3, 256, 64, 3
    pf = [oracle.index_prefix(i) for i in range(S + 1)]
    gpu_opt, _ = _optim(N, oracle, oracle.ADAM)
    groups = []
    for _ in range(2):
        ws = W.local_group(R, S, dim, pf[:S], 1 << 15, cap=4 * S * B, optimizer=gpu_opt, max_batch=B, rows_f32=True,
                           max_ids_per_sample=4)
        rws = RW.local_group(R, 1, dim, [pf[S]], 1 << 15, cap=4 * B, optimizer=gpu_opt, max_batch=B, max_ids_per_sample=4,
                             shards=[w.shard for w in ws])
        _warm(torch, ws)
        groups.append((ws, rws))
    for step in range(3):
        ragged = step == 1
        sb = [make_batch(rng, S, B, [30, 2000, 1 << 30], max_ids=4 if ragged else 1, allow_empty=ragged) for _ in range(R)]
        rb = [_ragged_raw(rng, B, 500, 4) for _ in range(R)]
        res = []
        g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16)
        for k, (ws, rws) in enumerate(groups):
            ids = [to_dev_ids(b[0], DEV) for b in sb]
            offs = [to_dev_i32(b[1], DEV) for b in sb] if ragged else None
            rids, roffs = [to_dev_ids(b[0], DEV) for b in rb], [to_dev_i32(b[1], DEV) for b in rb]
            torch.cuda.synchronize()
            if k == 1:
                RW.group_prepare_raw(rws, rids, B, fixed, row_offs=roffs)
                W.group_prepare(ws, ids, B, row_offs=offs, slot_occ_offs=[b[2] for b in sb])
            if R == 1:
                raw = [rws[0].forward_raw(rids[0], B, fixed, row_off=roffs[0])]
                outs = [ws[0].forward(ids[0], B, row_off=offs[0] if offs else None, slot_occ_off=sb[0][2])]
            else:
                raw = RW.group_forward_raw(rws, rids, B, fixed, row_offs=roffs)
                outs = W.group_forward(ws, ids, B, row_offs=offs, slot_occ_offs=[b[2] for b in sb])
            torch.cuda.synchronize()
            res.append(([o.cpu().numpy().tobytes() for o in outs],
                        [(t[:int(c[0]) + 1].cpu().numpy().tobytes(), i.cpu().numpy().tobytes()) for t, i, _, _, c in raw]))
            RW.group_backward_raw(rws, [torch.full((int(x[4][0]), dim), 0.02, device=DEV) for x in raw])
            W.group_backward(ws, [torch.from_numpy(g[r]).to(DEV) for r in range(R)])
            torch.cuda.synchronize()
        assert res[0] == res[1], step
    snaps = [_snapshot(ws) for ws, _ in groups]
    for r in range(R):
        for k, (x, y) in enumerate(zip(snaps[0][r], snaps[1][r])):
            assert k == 1 or x == y, (r, k)  # (index stats: the cells admissions take depend on their timing)


# ---- a run that grows ------------------------------------------------------------------------------------------------
def _grow_step(torch, oracle, ws, rws, w, pf, rng, B, layout, seen, fixed=4, sized=True):
    """One training step of the summation worker (3 slots) and the raw worker (slot 3) on R virtual ranks, sized from
    its own batch when `sized`; compares outputs with the oracle `w` unless it is None (bit for bit; ragged outputs bit
    for bit with the sample-order model, as test_gpu_worker.py) and returns the outputs and the raw tables."""
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW

    R, S, dim = len(ws), 3, ws[0].dim
    card = {"single": [40, 3000, 1 << 30], "ragged": [40, 3000, 1 << 30], "skewed": [1 << 40] * 3}[layout]
    sb = [make_batch(rng, S, B, card, max_ids=8 if layout == "ragged" else 1, allow_empty=layout == "ragged")
          for _ in range(R)]
    rb = [_ragged_raw(rng, B, 40 * B, 8) for _ in range(R)]
    ids, rids = [to_dev_ids(b[0], DEV) for b in sb], [to_dev_ids(b[0], DEV) for b in rb]
    offs = [to_dev_i32(b[1], DEV) for b in sb] if sb[0][1] is not None else None
    roffs = [to_dev_i32(b[1], DEV) for b in rb]
    torch.cuda.synchronize()
    if sized:  # persia_core's step: prepare every worker, agree, resize, then send
        raw_need = RW.group_prepare_raw(rws, rids, B, fixed, row_offs=roffs)
        sum_need = W.group_prepare(ws, ids, B, row_offs=offs, slot_occ_offs=[b[2] for b in sb])
        RW.group_resize(rws, *raw_need)
        W.group_resize(ws, *sum_need)
    raw = RW.group_forward_raw(rws, rids, B, fixed, row_offs=roffs)
    outs = W.group_forward(ws, ids, B, row_offs=offs, slot_occ_offs=[b[2] for b in sb])
    torch.cuda.synchronize()
    grads = [(rng.standard_normal((int(x[4][0]), dim)) * 1e-2).astype(np.float32) for x in raw]
    g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16)
    result = ([o.cpu().numpy().tobytes() for o in outs],
              [t[:int(c[0]) + 1].cpu().numpy().tobytes() for t, _, _, _, c in raw])
    signs = [slot_signs(oracle, b[0], b[2], pf[:S]) for b in sb]
    for r in range(R):
        seen.update(signs[r].tolist())
        seen.update(oracle.add_prefix(rb[r][0], 8, pf[S]).tolist())
    if w is None:
        RW.group_backward_raw(rws, [torch.from_numpy(x).to(DEV) for x in grads])
        W.group_backward(ws, [torch.from_numpy(g[r]).to(DEV) for r in range(R)])
        torch.cuda.synchronize()
        return result
    rows = held_rows(torch, oracle, [x.shard for x in ws], np.concatenate(signs)) if offs else None
    rctx, sctx = [], []
    for r in range(R):
        table, index, _, _, counts = raw[r]
        U = int(counts[0])
        wt, wi, _, _, c = w.forward_raw(S, rb[r][0], rb[r][1], B, training=True)
        assert table[:U + 1].cpu().numpy().tobytes() == wt.tobytes(), (layout, r)
        np.testing.assert_array_equal(index.cpu().numpy(), wi)
        rctx.append((U, c))
        row_off = sb[r][1] if offs else np.arange(S * B + 1, dtype=np.uint32)
        full = np.concatenate([row_off, np.full(B, row_off[-1], np.uint32)])
        want, c = w.forward(sb[r][0], full, B, training=True)
        sctx.append(c)
        got = outs[r].cpu().numpy()
        if offs:
            model = pool_model(rows, signs[r], sb[r][1], B, None, dim=dim)
            for s in range(S):
                assert same_bits(got[s], model[s]), (layout, r, s)
                np.testing.assert_allclose(got[s].astype(np.float32), want[s].astype(np.float32), rtol=2e-3, atol=8e-3)
        else:
            for s in range(S):
                np.testing.assert_array_equal(got[s].view(np.uint16), want[s].view(np.uint16))
    RW.group_backward_raw(rws, [torch.from_numpy(x).to(DEV) for x in grads])
    W.group_backward(ws, [torch.from_numpy(g[r]).to(DEV) for r in range(R)])
    torch.cuda.synchronize()
    zero = np.zeros((B, dim), np.float16)
    for r in range(R):
        w.backward_raw(S, rctx[r][1], grads[r])
        w.backward(sctx[r], [g[r, s] for s in range(S)] + [zero], skip=[0, 0, 0, 1])
    return result


def _grow_groups(torch, oracle, R, kind, capacity, cap, max_batch, rows_f32=False, max_ids=1):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW

    pf = [oracle.index_prefix(i) for i in range(4)]
    gpu_opt, cpu_opt = _optim(N, oracle, kind)
    ws = W.local_group(R, 3, 32, pf[:3], capacity, cap=cap, optimizer=gpu_opt, max_batch=max_batch, rows_f32=rows_f32,
                       max_ids_per_sample=max_ids)
    rws = RW.local_group(R, 1, 32, [pf[3]], capacity, cap=cap, optimizer=gpu_opt, max_batch=max_batch,
                         max_ids_per_sample=max_ids, shards=[x.shard for x in ws])
    w = oracle.Worker([oracle.SlotCfg(32, prefix=p) for p in pf[:3]] +
                      [oracle.SlotCfg(32, summation=False, sample_fixed_size=4, prefix=pf[3])], n_ps=R)
    w.configure()
    w.set_optimizer(cpu_opt)
    _warm(torch, ws)
    return ws, rws, w, pf


def _check_rows(torch, oracle, ws, rws, w, seen):
    R = len(ws)
    signs = np.array(sorted(seen), np.uint64)
    owner = oracle.shard_of(signs, R)
    for r in range(R):
        mine = signs[owner == r]
        ent, found = ws[r].shard.get_entries(to_dev_ids(mine, DEV))
        ent, found = ent.cpu().numpy(), found.cpu().numpy()
        for k, sign in enumerate(mine):
            ref = w.get_entry(int(sign))
            assert (ref is not None) == bool(found[k]), (r, sign)
            assert ref is None or ent[k].tobytes() == ref.tobytes(), (r, k, sign)
        assert len(ws[r].shard) == w.ps_len(r)
        assert ws[r].shard.counters()["wait_errors"] == 0
    for x in ws + rws:
        assert x.status() == (False, False)


GROWTH = [("single", 16), ("single", 512), ("ragged", 256), ("skewed", 2048), ("single", 64)]


@pytest.mark.parametrize("kind", [0, 1, 2, 3])  # SGD, Adagrad, vectorwise Adagrad, Adam
@pytest.mark.parametrize("R", [2, 3, 4])
def test_growth_run_matches_oracle(torch_cuda, oracle, R, kind):
    """First batch B = 16, cap 8; then B = 512, ragged up to 8 ids per sample, a skewed batch (every id distinct: each
    owner gets far more than 10 x the first cap), and a raw slot whose batches grow with them."""
    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(100 * R + kind)
        ws, rws, w, pf = _grow_groups(torch, oracle, R, kind, 1 << 16, cap=8, max_batch=16)
        seen = set()
        for layout, B in GROWTH:
            _grow_step(torch, oracle, ws, rws, w, pf, rng, B, layout, seen)
            _check_rows(torch, oracle, ws, rws, w, seen)
        assert ws[0].cap > 80 and ws[0].rows_f32 and rws[0].cap > 8
        assert len({(x.cap, x.rows_f32) for x in ws}) == 1
    finally:
        oracle.set_rsqrt_exact(False)


def test_growth_run_with_eviction_equals_a_large_run(torch_cuda, oracle):
    """With eviction on, a run that grows ends with the tables, counters and checkpoint contents (list order and
    entries) of a run sized large from its first step."""
    torch = torch_cuda
    runs = []
    for grow in (True, False):
        rng = np.random.default_rng(77)
        ws, rws, w, pf = _grow_groups(torch, oracle, 2, oracle.SGD, 1 << 15, cap=8 if grow else 1 << 14,
                                      max_batch=16 if grow else 2048, rows_f32=not grow, max_ids=1 if grow else 8)
        for x in ws:
            # every check frees a whole step's rows: no admission is refused (which of two racing admissions gets the
            # last free row depends on timing), while the run still evicts
            x.shard.set_eviction(check_every=1, low_water=1 << 14, target_free=1 << 14, keep_batches=1)
        seen, outs = set(), []
        for layout, B in GROWTH:
            outs.append(_grow_step(torch, oracle, ws, rws, None, pf, rng, B, layout, seen, sized=grow))
        runs.append((outs, _snapshot(ws)))
        assert all(x.shard.counters()["capacity_refused"] == 0 for x in ws)
        assert sum(x.shard.counters()["admitted"] for x in ws) < len(seen)  # rows were evicted
        assert all(x.status() == (False, False) for x in ws + rws)
    for step, (x, y) in enumerate(zip(runs[0][0], runs[1][0])):
        assert x == y, step
    for r in range(2):  # the checkpoint's contents: list order (signs by recency) and entries; and the counters
        for k, (x, y) in enumerate(zip(runs[0][1][r], runs[1][1][r])):
            assert k == 1 or x == y, (r, k)  # (index stats: the cells admissions take depend on their timing)


def test_exchange_replaced_keeps_adam_powers_and_incremental_set(torch_cuda, oracle):
    torch = torch_cuda
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW

    rng = np.random.default_rng(9)
    ws, rws, w, pf = _grow_groups(torch, oracle, 2, oracle.ADAM, 1 << 16, cap=4096, max_batch=512, rows_f32=True,
                                  max_ids=8)
    for x in ws:
        x.shard.enable_incremental(1 << 16)
    seen = set()
    _grow_step(torch, oracle, ws, rws, w, pf, rng, 512, "single", seen, sized=False)
    held = [x.shard.incremental_stats() for x in ws]
    assert W.group_resize(ws, 2 * 4096 + 1, True) and RW.group_resize(rws, 2 * 4096 + 1, True)
    assert ws[0].cap > 8192 and [x.shard.incremental_stats() for x in ws] == held
    _grow_step(torch, oracle, ws, rws, w, pf, rng, 512, "single", seen, sized=False)  # Adam's powers: from the table
    _check_rows(torch, oracle, ws, rws, w, seen)
    assert sum(x.shard.incremental_stats()["held"] for x in ws) >= sum(h["held"] for h in held) > 0
