"""GPU: slots that share a feature group on the sharded path (pb_forward_sharded / pb_backward_sharded) against the
oracle's embedding worker with R parameter servers.

Two slots of one group share a key space: a sign in both is one row, and a rank's request holds it once per slot, in
slot order.  The owner applies the R requests in rank order, so the row is stepped (r0, a), (r0, b), (r1, a), (r1, b):
rank-major, then slot order.  R virtual ranks share cuda:0, as in test_gpu_worker.py; the oracle runs R forward
requests, then R backward requests in rank order, and everything is compared bit for bit (Adagrad in the oracle's
exact-rsqrt mode): outputs, slot statuses, every touched entry, shard sizes and the miss counters."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from util import (full_row_off, held_rows, make_batch, pool_model, same_bits, slot_signs, to_dev_i32,  # noqa: E402
                  to_dev_ids)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GROUPS = [0, 1, 0, 0, 2, 0]  # group 0: slots 0, 2, 3, 5 (a chain of four, not adjacent)
CARD = [3, 50, 2, 40, 2000, 5]  # low cardinality: most signs of group 0 sit in several slots and on every rank


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
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


def _group(torch, oracle, R, groups, dim, kind, B, sqrt=None, rows_f32=False, max_ids=1, capacity=1 << 16, cap=None):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker

    S = len(groups)
    pf = [oracle.index_prefix(g) for g in groups]
    gpu_opt, cpu_opt = _optim(N, oracle, kind)
    ws = ShardedEmbeddingWorker.local_group(R, S, dim, pf, capacity, cap=cap or S * B * max_ids, optimizer=gpu_opt,
                                            max_batch=B, sqrt_scaling=sqrt, rows_f32=rows_f32, max_ids_per_sample=max_ids)
    w = oracle.Worker([oracle.SlotCfg(dim, sqrt_scaling=bool(sqrt[i]) if sqrt else False, prefix=pf[i]) for i in range(S)],
                      n_ps=R)
    w.configure()
    w.set_optimizer(cpu_opt)
    for x in ws:  # table storage is allocated on first use, with a device-wide sync: not while a peer spins on a flag
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    return ws, w, pf


def _check_rows(torch, oracle, ws, w, signs, R, sizes=True):
    signs = np.array(sorted(signs), np.uint64)
    owner = oracle.shard_of(signs, R)
    for r in range(R):
        mine = signs[owner == r]
        if mine.size:
            ent, found = ws[r].shard.get_entries(to_dev_ids(mine, DEV))
            ent = ent.cpu().numpy()
            assert found.all()
            for k, sign in enumerate(mine):
                ref = w.get_entry(int(sign))
                assert ref is not None and ent[k].tobytes() == ref.tobytes(), (r, k, sign)
        if sizes:
            assert len(ws[r].shard) == w.ps_len(r)
    for x in ws:
        assert x.status() == (False, False)
        assert x.shard.counters()["wait_errors"] == 0
    assert sum(x.shard.counters()["gradient_id_miss"] for x in ws) == w.grad_miss()


def _train(torch, oracle, ws, w, pf, rng, R, B, dim, card, steps, f32=False, nan_step=None, skip_step=None):
    """`steps` training steps of every rank, checked against the oracle; returns the signs touched.  nan_step: a NaN
    in slot 2 (group 0) of rank 0's gradient; skip_step: add_skipped_gradient on slot 3 (group 0) of the last rank."""
    from persia_b200.worker import ShardedEmbeddingWorker as W

    S = len(pf)
    outs = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
    seen = set()
    for step in range(steps):
        ids = [make_batch(rng, S, B, card)[0] for _ in range(R)]
        torch.cuda.synchronize()
        W.group_forward(ws, [to_dev_ids(i, DEV) for i in ids], B, training=True, outs=outs)
        torch.cuda.synchronize()
        octx = []
        for r in range(R):
            want, c = w.forward(ids[r], full_row_off(S, B), B, training=True)
            octx.append(c)
            got = outs[r].cpu().numpy()
            for i in range(S):
                np.testing.assert_array_equal(got[i].view(np.uint16), want[i].view(np.uint16), err_msg=f"{step} {r} {i}")
                seen.update(w.ctx_signs(c, i).tolist())
        g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float32 if f32 else np.float16)
        skip = [None] * R
        if step == nan_step:
            g[0, 2, B // 3, dim - 1] = np.nan  # rank 0 drops slot 2; its slots 0, 3, 5 of the same group still apply
        dg = [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)]
        if step == skip_step:
            dg[R - 1][3] = None
            skip[R - 1] = [0, 0, 0, 1, 0, 0]
        torch.cuda.synchronize()
        sts = W.group_backward(ws, dg, want_status=True)
        torch.cuda.synchronize()
        for r in range(R):
            ost = w.backward(octx[r], [g[r, i] for i in range(S)], skip=skip[r])
            assert sts[r].cpu().numpy().tolist() == ost, (step, r)
    return seen


@pytest.mark.parametrize("R,dim,kind,f32", [
    (1, 64, 1, False), (2, 64, 0, False), (2, 128, 1, False), (3, 128, 2, False), (4, 64, 3, False),
    (8, 128, 1, False), (2, 12, 2, False), (3, 130, 1, True), (2, 256, 0, False), (4, 256, 2, False),
    (2, 128, 3, False), (8, 64, 2, False), (3, 64, 2, True), (2, 64, 3, True)])
def test_groups_match_oracle(torch_cuda, oracle, R, dim, kind, f32):
    """Groups [0, 1, 0, 0, 2, 0] (a chain of up to four entries, non-adjacent slots), every optimizer, the one-launch
    owner kernel (dims 64, 128) and the per-request one (12, 130, 256, vectorwise Adagrad); a NaN in one slot of the
    group on rank 0 and add_skipped_gradient on another of its slots on the last rank (Adam: beta powers per request)."""
    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(1000 * R + dim + kind)
        B = 600
        ws, w, pf = _group(torch, oracle, R, GROUPS, dim, kind, B)
        seen = _train(torch, oracle, ws, w, pf, rng, R, B, dim, CARD, 4, f32=f32, nan_step=1,
                      skip_step=2 if R > 1 else None)
        _check_rows(torch, oracle, ws, w, seen, R)
    finally:
        oracle.set_rsqrt_exact(False)


@pytest.mark.parametrize("dim,kind", [(128, 1), (256, 2), (64, 3)])
def test_groups_hot_signs_across_ranks(torch_cuda, oracle, dim, kind):
    """Signs repeated more than 32 and 256 times in each slot of a group (the requester's warm and hot reduce) on four
    ranks: every rank holds them in all four slots of the group."""
    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(dim + kind)
        R, B = 4, 2000
        ws, w, pf = _group(torch, oracle, R, GROUPS, dim, kind, B)
        seen = _train(torch, oracle, ws, w, pf, rng, R, B, dim, [4, 30, 2, 60, 5000, 6], 2)
        _check_rows(torch, oracle, ws, w, seen, R)
    finally:
        oracle.set_rsqrt_exact(False)


def test_groups_ragged_sqrt_scale(torch_cuda, oracle):
    """Ragged layout (several ids per sample, empty samples), sqrt scaling and a loss scale, f32 rows."""
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(5)
        R, B, dim = 3, 300, 32
        groups, card = [0, 0, 1, 0], [5, 7, 4000, 300]
        S = len(groups)
        sqrt = [True, False, True, False]
        ws, w, pf = _group(torch, oracle, R, groups, dim, oracle.ADAGRAD, B, sqrt=sqrt, rows_f32=True, max_ids=5)
        seen = set()
        for step in range(3):
            batches = [make_batch(rng, S, B, card, max_ids=5, allow_empty=True) for _ in range(R)]
            dev_in = [(to_dev_ids(b[0], DEV), to_dev_i32(b[1], DEV)) for b in batches]
            pre = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
            torch.cuda.synchronize()
            outs = W.group_forward(ws, [d[0] for d in dev_in], B, training=True, row_offs=[d[1] for d in dev_in],
                                   slot_occ_offs=[b[2] for b in batches], outs=pre)
            torch.cuda.synchronize()
            # every rank's rows after the forward (it admits, it steps nothing), each from its owner
            signs = [slot_signs(oracle, b[0], b[2], pf) for b in batches]
            rows = held_rows(torch, oracle, [x.shard for x in ws], np.concatenate(signs))
            octx = []
            for r in range(R):
                want, c = w.forward(batches[r][0], batches[r][1], B, training=True)
                model = pool_model(rows, signs[r], batches[r][1], B, sqrt, dim=dim)
                octx.append(c)
                got = outs[r].cpu().numpy()
                for i in range(S):
                    assert same_bits(got[i], model[i]), (step, r, i)  # sample order, bit for bit
                    # (a sample's ids are summed in sample order here, in shard order there: one f16 step apart at most)
                    np.testing.assert_allclose(got[i].astype(np.float32), want[i].astype(np.float32), rtol=2e-3, atol=8e-3)
                    seen.update(w.ctx_signs(c, i).tolist())
            g = (rng.integers(-64, 65, size=(R, S, B, dim)) / 4.0).astype(np.float16)  # x 1/128 stays exact in f32
            scale = [128.0, 1.0, 128.0, 1.0]
            dg = [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)]
            torch.cuda.synchronize()
            W.group_backward(ws, dg, scales=scale)
            torch.cuda.synchronize()
            for r in range(R):
                w.backward(octx[r], [g[r, i] for i in range(S)], scale=scale)
        _check_rows(torch, oracle, ws, w, seen, R)
    finally:
        oracle.set_rsqrt_exact(False)


def test_groups_inference(torch_cuda, oracle):
    """Inference between training steps: nothing is admitted, absent signs read as zeros."""
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(9)
        R, B, dim = 3, 400, 64
        S = len(GROUPS)
        ws, w, pf = _group(torch, oracle, R, GROUPS, dim, oracle.ADAGRAD, B)
        seen = _train(torch, oracle, ws, w, pf, rng, R, B, dim, CARD, 1)
        ids = [make_batch(rng, S, B, [6, 80, 4, 60, 4000, 9])[0] for _ in range(R)]
        outs = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
        torch.cuda.synchronize()
        W.group_forward(ws, [to_dev_ids(i, DEV) for i in ids], B, training=False, outs=outs)
        torch.cuda.synchronize()
        for r in range(R):
            want, _ = w.forward(ids[r], full_row_off(S, B), B, training=False, keep_ctx=False)
            got = outs[r].cpu().numpy()
            for i in range(S):
                np.testing.assert_array_equal(got[i].view(np.uint16), want[i].view(np.uint16))
        seen |= _train(torch, oracle, ws, w, pf, rng, R, B, dim, CARD, 1)
        _check_rows(torch, oracle, ws, w, seen, R)
    finally:
        oracle.set_rsqrt_exact(False)


@pytest.mark.parametrize("dim", [64, 130])
def test_groups_capacity_bounded_counts_misses(torch_cuda, oracle, dim):
    """A table too small for the batch: signs it could not admit take no step, and every applied entry of such a sign
    counts as a gradient miss — a sign in three slots of a group counts three times.  Admitted signs match the oracle."""
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(dim)
        R, B = 2, 500
        groups, card = [0, 0, 1, 0], [1500, 1500, 30, 1500]  # ~1200 signs of group 0 per rank, many in two slots
        S = len(groups)
        ws, w, pf = _group(torch, oracle, R, groups, dim, oracle.ADAGRAD, B, capacity=512)
        for x in ws:
            x.shard.set_eviction(check_every=0)
        ids = [make_batch(rng, S, B, card)[0] for _ in range(R)]
        outs = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
        torch.cuda.synchronize()
        W.group_forward(ws, [to_dev_ids(i, DEV) for i in ids], B, training=True, outs=outs)
        g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16)
        torch.cuda.synchronize()
        W.group_backward(ws, [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)])
        torch.cuda.synchronize()
        octx = [w.forward(ids[r], full_row_off(S, B), B, training=True)[1] for r in range(R)]
        for r in range(R):
            w.backward(octx[r], [g[r, i] for i in range(S)])
        entries = [np.unique(oracle.add_prefix(ids[r][i * B:(i + 1) * B], 8, pf[i])) for r in range(R) for i in range(S)]
        signs = np.unique(np.concatenate(entries))
        owner = oracle.shard_of(signs, R)
        present = set()
        for r in range(R):
            mine = signs[owner == r]
            ent, found = ws[r].shard.get_entries(to_dev_ids(mine, DEV))
            ent, found = ent.cpu().numpy(), found.cpu().numpy().astype(bool)
            for k in np.flatnonzero(found):
                assert ent[k].tobytes() == w.get_entry(int(mine[k])).tobytes()
                present.add(int(mine[k]))
        missing = sum(int(s) not in present for e in entries for s in e.tolist())
        assert len(present) < signs.size and missing > 0
        assert sum(x.shard.counters()["gradient_id_miss"] for x in ws) == missing
        for x in ws:
            assert x.status() == (False, False) and x.shard.counters()["wait_errors"] == 0
    finally:
        oracle.set_rsqrt_exact(False)


def test_groups_graph_replay(torch_cuda, oracle):
    """A whole step of every rank captured in CUDA graphs (one per rank and phase) and replayed: the link kernel, the
    chain marks and the owners' walks need no host sync and no allocation."""
    from persia_b200 import native as N

    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(13)
        R, B, dim = 3, 512, 128
        S = len(GROUPS)
        ws, w, pf = _group(torch, oracle, R, GROUPS, dim, oracle.ADAM, B)
        ids_dev = [torch.zeros(S * B, dtype=torch.int64, device=DEV) for _ in range(R)]
        g_dev = [torch.zeros((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
        outs = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
        plan = [("f", N.PHASE_SEND), ("f", N.PHASE_SERVE), ("f", N.PHASE_FINISH), ("b", N.PHASE_SEND), ("b", N.PHASE_SERVE)]

        def enqueue(r, kind, ph):
            if kind == "f":
                ws[r].forward(ids_dev[r], B, training=True, out=outs[r], phases=ph)
            else:
                ws[r].backward(g_dev[r], phases=ph)

        def oracle_step(ids, g):
            octx = [w.forward(ids[r], full_row_off(S, B), B, training=True) for r in range(R)]
            for r in range(R):
                w.backward(octx[r][1], [g[r, i] for i in range(S)])
            return [o[0] for o in octx]

        torch.cuda.synchronize()
        for kind, ph in plan:  # eager warm-up step (id 0 in every slot, zero gradients)
            for r in range(R):
                enqueue(r, kind, ph)
        torch.cuda.synchronize()
        oracle_step([np.zeros(S * B, np.uint64)] * R, np.zeros((R, S, B, dim), np.float16))
        graphs = {}
        for r in range(R):
            for kind, ph in plan:
                gph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gph, stream=ws[r].stream, capture_error_mode="thread_local"):
                    enqueue(r, kind, ph)
                graphs[(r, kind, ph)] = gph
        seen = {int(oracle.add_prefix(np.zeros(1, np.uint64), 8, p)[0]) for p in pf}
        for it in range(3):
            ids = [make_batch(rng, S, B, CARD)[0] for _ in range(R)]
            g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16)
            for r in range(R):
                ids_dev[r].copy_(to_dev_ids(ids[r], DEV))
                g_dev[r].copy_(torch.from_numpy(g[r]).to(DEV))
            torch.cuda.synchronize()
            for kind, ph in plan:
                for r in range(R):
                    with torch.cuda.stream(ws[r].stream):
                        graphs[(r, kind, ph)].replay()
            torch.cuda.synchronize()
            want = oracle_step(ids, g)
            for r in range(R):
                got = outs[r].cpu().numpy()
                for i in range(S):
                    np.testing.assert_array_equal(got[i].view(np.uint16), want[r][i].view(np.uint16))
                    seen.update(oracle.add_prefix(ids[r][i * B:(i + 1) * B], 8, pf[i]).tolist())
        _check_rows(torch, oracle, ws, w, seen, R)
    finally:
        oracle.set_rsqrt_exact(False)


def test_groups_overflow_is_flagged(torch_cuda, oracle):
    """A pair that needs more than cap slots raises the status flag, with chains too; nothing faults."""
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, B, dim = 2, 256, 16
    S = len(GROUPS)
    ws, w, pf = _group(torch, oracle, R, GROUPS, dim, oracle.SGD, B, cap=16)
    rng = np.random.default_rng(3)
    ids = [make_batch(rng, S, B, [300, 300, 300, 300, 300, 300])[0] for _ in range(R)]
    outs = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
    torch.cuda.synchronize()
    W.group_forward(ws, [to_dev_ids(i, DEV) for i in ids], B, training=True, outs=outs)
    torch.cuda.synchronize()
    W.group_backward(ws, [torch.zeros((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)])
    torch.cuda.synchronize()
    assert all(x.status()[0] for x in ws) and not any(x.status()[1] for x in ws)
    assert all(x.shard.counters()["wait_errors"] == 0 for x in ws)


def test_groups_then_distinct_groups_on_same_workers(torch_cuda, oracle):
    """Steps with a shared group, then steps whose slots are all in groups of their own on the same exchanges and
    tables (the request carries no chain words; the marks of the earlier requests must not count)."""
    from persia_b200 import shard as SH

    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(21)
        R, B, dim = 2, 600, 64
        S = len(GROUPS)
        ws, w, pf = _group(torch, oracle, R, GROUPS, dim, oracle.ADAGRAD, B)
        seen = _train(torch, oracle, ws, w, pf, rng, R, B, dim, CARD, 2)
        _check_rows(torch, oracle, ws, w, seen, R)
        # new feature groups (fresh key spaces, fresh rows on both sides) on the same exchanges and tables
        pf2 = [oracle.index_prefix(10 + i) for i in range(S)]
        for x in ws:
            x.ctx.close()
            x.ctx = SH.BatchContext(S * B, S * B, pf2, None, 8, x.device)
        w2 = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pf2], n_ps=R)
        w2.configure()
        w2.set_optimizer(oracle.Optim(oracle.ADAGRAD, lr=0.02, init_acc=0.01, eps=1e-10))
        seen2 = _train(torch, oracle, ws, w2, pf2, rng, R, B, dim, CARD, 2, nan_step=1)
        _check_rows(torch, oracle, ws, w2, seen2, R, sizes=False)
    finally:
        oracle.set_rsqrt_exact(False)
