"""GPU: tables larger than HBM on R GPUs — every rank's shard has a host-memory tier (pb_table_attach_tier) and serves the
sharded calls (pb_forward_sharded / pb_forward_raw_sharded and their backwards, through ShardedEmbeddingWorker /
ShardedRawWorker).  An owner moves the tier-held signs of a training request back into HBM rows before it probes them
(k_tier_restore_recv) and reads them in place for an inference request (k_owner_lookup_tier).

R virtual ranks share cuda:0, driven phase by phase as in test_gpu_worker.py.  Values compare bit for bit against the
oracle's embedding worker with R parameter servers, which never evicts: the union of HBM and tier behaves like one
unbounded table (Adagrad-type optimizers against the oracle's exact-rsqrt mode)."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from util import (f16_ulp_diff, full_row_off, held_rows, make_batch, pool_model, same_bits, slot_signs,  # noqa: E402
                  to_dev_i32, to_dev_ids)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


OPTIMS = {  # GPU keywords, oracle keywords
    "SGD": (dict(lr=0.05, wd=0.001), dict(lr=0.05, wd=0.001)),
    "ADAGRAD": (dict(lr=0.02, initialization=0.01, eps=1e-10), dict(lr=0.02, init_acc=0.01, eps=1e-10)),
    "ADAGRAD_VW": (dict(lr=0.02, initialization=0.01, eps=1e-10), dict(lr=0.02, init_acc=0.01, eps=1e-10)),
    "ADAM": (dict(lr=0.01, beta1=0.9, beta2=0.999, eps=1e-8), dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8)),
}


def _optim(N, oracle, name):
    g, o = OPTIMS[name]
    return dict(kind=getattr(N, "OPT_" + name), **g), oracle.Optim(getattr(oracle, name), **o)


def _oracle(oracle, slots, R, cpu_opt):
    w = oracle.Worker(slots, n_ps=R)
    w.configure()
    w.set_optimizer(cpu_opt)
    return w


def _warm(torch, ws):
    for x in ws:  # table storage is allocated on first use, with a device-wide sync: not while a peer spins on a flag
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()


def _tier_sum(ws, field):
    return sum(int(x.shard.tier_stats()[field]) for x in ws)


def _counter_sum(ws, field):
    return sum(int(x.shard.counters()[field]) for x in ws)


def _check_entries(torch, oracle, ws, oracles, signs, R):
    """Every sign seen has its oracle entry, read from its owner (HBM or tier), and every shard holds as many entries as
    its oracle parameter server."""
    torch.cuda.synchronize()
    signs = np.array(sorted(signs), np.uint64)
    owner = oracle.shard_of(signs, R)
    for r in range(R):
        mine = signs[owner == r]
        if mine.size:
            ent, found = ws[r].shard.get_entries(to_dev_ids(mine, DEV))
            ent, found = ent.cpu().numpy(), found.cpu().numpy()
            assert found.all(), (r, int((~found.astype(bool)).sum()))
            for k, sign in enumerate(mine):
                ref = next(e for e in (o.get_entry(int(sign)) for o in oracles) if e is not None)
                assert same_bits(ent[k], ref), (r, k, int(sign))
        assert len(ws[r].shard) == sum(o.ps_len(r) for o in oracles), r


def _final_checks(ws, statuses=()):
    for x in list(ws) + list(statuses):
        assert x.status() == (False, False)
    ts = {f: _tier_sum(ws, f) for f in ("moved_out", "restored", "dropped", "refused")}
    assert ts["moved_out"] > 0 and ts["restored"] > 0 and ts["dropped"] == 0 and ts["refused"] == 0, ts
    for f in ("wait_errors", "capacity_refused", "gradient_id_miss"):
        assert _counter_sum(ws, f) == 0, f


def _ragged(rng, B, card, max_ids):
    row_off = np.zeros(B + 1, np.uint32)
    row_off[1:] = np.cumsum(rng.integers(0, max_ids + 1, size=B))
    return rng.integers(0, card, size=int(row_off[-1]), dtype=np.uint64), row_off


# ---------------------------------------------------------------------------------------------- 1. parity over churn
@pytest.mark.parametrize("R", [2, 4])
@pytest.mark.parametrize("name,dim", [("SGD", 16), ("ADAGRAD", 32), ("ADAGRAD_VW", 20), ("ADAM", 24)])
def test_sharded_tier_parity_over_churn(torch_cuda, oracle, R, name, dim):
    """C = 1024 HBM rows per rank over about 4 C keys per owner: two summation slots (one-id and ragged steps, f16 and
    f32 gradients, loss scales) and a raw slot share every rank's tiered table, one eviction check per training request.
    After every step the outputs, the raw tables and the statuses equal the oracle's, every sign seen has its oracle
    entry in HBM or in the tier, and every shard holds as many entries as its oracle server."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW

    torch = torch_cuda
    C, T, S, B, RB, fixed = 1024, 1 << 14, 2, 64, 48, 3
    card, raw_card = [1600 * R, 1600 * R], 900 * R
    pf = [oracle.index_prefix(g) for g in (0, 1)]
    rpf = oracle.index_prefix(2)
    gpu_opt, cpu_opt = _optim(N, oracle, name)
    oracle.set_rsqrt_exact(True)
    try:
        ws = W.local_group(R, S, dim, pf, C, cap=S * B * 3, optimizer=gpu_opt, max_batch=B, rows_f32=True,
                           max_ids_per_sample=3, tier_rows=T)
        rws = RW.local_group(R, 1, dim, [rpf], C, cap=RB * 4, optimizer=gpu_opt, max_batch=RB, max_ids_per_sample=4,
                             shards=[x.shard for x in ws])
        for x in ws:  # protected: the last two requests; the sweep frees down to C / 2
            x.shard.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=2)
        w = _oracle(oracle, [oracle.SlotCfg(dim, prefix=p) for p in pf], R, cpu_opt)
        wr = _oracle(oracle, [oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=rpf)], R, cpu_opt)
        _warm(torch, ws)
        rng = np.random.default_rng(R * 100 + dim)
        seen = set()
        for step in range(24):
            # ---- summation slots
            batches = [make_batch(rng, S, B, card, max_ids=3 if step % 2 else 1) for _ in range(R)]
            ragged = batches[0][1] is not None
            d_ids = [to_dev_ids(b[0], DEV) for b in batches]
            d_ro = [to_dev_i32(b[1], DEV) for b in batches] if ragged else None
            torch.cuda.synchronize()
            outs = W.group_forward(ws, d_ids, B, training=True, row_offs=d_ro, slot_occ_offs=[b[2] for b in batches])
            torch.cuda.synchronize()
            signs = [slot_signs(oracle, b[0], b[2], pf) for b in batches]  # the forward restores and admits, steps nothing
            rows = held_rows(torch, oracle, [x.shard for x in ws], np.concatenate(signs))
            octx = []
            for r in range(R):
                ro = batches[r][1] if ragged else full_row_off(S, B)
                want, c = w.forward(batches[r][0], ro, B, training=True)
                octx.append(c)
                got = outs[r].cpu().numpy()
                model = pool_model(rows, signs[r], batches[r][1], B, None, dim=dim)
                counts = np.diff(ro).reshape(S, B)
                for i in range(S):
                    assert same_bits(got[i], model[i]), (step, r, i)
                    one = counts[i] <= 1  # a sample of several ids may differ by 1 f16 ulp: f32 sum order
                    np.testing.assert_array_equal(got[i][one].view(np.uint16), want[i][one].view(np.uint16),
                                                  err_msg=str((step, r, i)))
                    assert f16_ulp_diff(got[i][~one], want[i][~one]) <= 1, (step, r, i)
                    seen.update(w.ctx_signs(c, i).tolist())
            f32 = step % 4 >= 2
            scale = [128.0, 1.0] if f32 else [1.0, 64.0]
            g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float32 if f32 else np.float16)
            dg = [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)]
            torch.cuda.synchronize()
            sts = W.group_backward(ws, dg, scales=scale, want_status=True)
            torch.cuda.synchronize()
            for r in range(R):
                assert sts[r].cpu().numpy().tolist() == w.backward(octx[r], [g[r, i] for i in range(S)], scale=scale), \
                    (step, r)
            # ---- the raw slot: requests of their own on the same tables
            rb = [_ragged(rng, RB, raw_card, 4) for _ in range(R)]
            torch.cuda.synchronize()
            res = RW.group_forward_raw(rws, [to_dev_ids(b[0], DEV) for b in rb], RB, fixed,
                                       row_offs=[to_dev_i32(b[1], DEV) for b in rb])
            torch.cuda.synchronize()
            rctx, rg = [], []
            for r, (table, index, _, _, cnt) in enumerate(res):
                U = int(cnt[0])
                wt, wi, _, _, oc = wr.forward_raw(0, rb[r][0], rb[r][1], RB, training=True)
                assert table[:U + 1].cpu().numpy().tobytes() == wt.tobytes(), (step, r)
                np.testing.assert_array_equal(index.cpu().numpy(), wi)
                rctx.append(oc)
                rg.append((rng.standard_normal((U, dim)) * 1e-2).astype(np.float32) if U else None)
                seen.update(oracle.add_prefix(rb[r][0], 8, rpf).tolist())
            torch.cuda.synchronize()
            rsts = RW.group_backward_raw(rws, [torch.from_numpy(x).to(DEV) if x is not None else None for x in rg],
                                         scales=[32.0] * R, want_status=True)
            torch.cuda.synchronize()
            for r in range(R):
                want = wr.backward_raw(0, rctx[r], rg[r], scale=32.0, skip=rg[r] is None)
                assert rsts[r].item() == want, (step, r)
            _check_entries(torch, oracle, ws, (w, wr), seen, R)
        _final_checks(ws, rws)
    finally:
        oracle.set_rsqrt_exact(False)


# ---------------------------------------------------------------------------------------------- 2. collective inference
@pytest.mark.parametrize("rows_f32", [False, True])
def test_sharded_tier_inference_reads_in_place(torch_cuda, oracle, rows_f32):
    """Training pushes many signs into the tiers; a training=False step over seen and never-seen signs then returns the
    oracle's outputs bit for bit (f16(0 + row) on f16 exchanges, the pooled f32 rows on f32 ones), moves nothing (the
    tier statistics stay as they were) and counts as lookup misses exactly the signs no table holds."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, S, B, dim, C = 2, 2, 64, 32, 512  # a step brings an owner about S * B signs: a quarter of the HBM rows
    card = [2400, 2400]
    pf = [oracle.index_prefix(i) for i in range(S)]
    gpu_opt, cpu_opt = _optim(N, oracle, "ADAGRAD")
    oracle.set_rsqrt_exact(True)
    try:
        ws = W.local_group(R, S, dim, pf, C, cap=S * B, optimizer=gpu_opt, max_batch=B, rows_f32=rows_f32,
                           tier_rows=1 << 13)
        for x in ws:
            x.shard.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=1)
        w = _oracle(oracle, [oracle.SlotCfg(dim, prefix=p) for p in pf], R, cpu_opt)
        _warm(torch, ws)
        rng = np.random.default_rng(5 + rows_f32)
        seen = set()
        for step in range(12):
            ids = [make_batch(rng, S, B, card)[0] for _ in range(R)]
            torch.cuda.synchronize()
            W.group_forward(ws, [to_dev_ids(x, DEV) for x in ids], B, training=True)
            torch.cuda.synchronize()
            octx = [w.forward(ids[r], full_row_off(S, B), B, training=True)[1] for r in range(R)]
            g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16)
            W.group_backward(ws, [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)])
            torch.cuda.synchronize()
            for r in range(R):
                w.backward(octx[r], [g[r, i] for i in range(S)])
            for r in range(R):
                seen.update(slot_signs(oracle, ids[r], [s * B for s in range(S + 1)], pf).tolist())
        assert _counter_sum(ws, "capacity_refused") == 0
        ts0 = [x.shard.tier_stats() for x in ws]
        assert sum(t["host_rows"] for t in ts0) > len(seen) // 3, ts0  # a good part of them lives in the tiers
        miss0 = _counter_sum(ws, "lookup_miss")
        # inference: seen signs (mostly tier-held) and fresh ones (ids >= card: no table holds them)
        ids = [np.concatenate([rng.integers(0, card[i] + 100, size=B, dtype=np.uint64) for i in range(S)])
               for _ in range(R)]
        torch.cuda.synchronize()
        outs = W.group_forward(ws, [to_dev_ids(x, DEV) for x in ids], B, training=False)
        torch.cuda.synchronize()
        absent = 0
        for r in range(R):
            want, _ = w.forward(ids[r], full_row_off(S, B), B, training=False)
            got = outs[r].cpu().numpy()
            for i in range(S):
                np.testing.assert_array_equal(got[i].view(np.uint16), want[i].view(np.uint16), err_msg=str((r, i)))
            sg = slot_signs(oracle, ids[r], [s * B for s in range(S + 1)], pf)
            absent += sum(1 for x in np.unique(sg).tolist() if x not in seen)  # one entry per distinct sign and request
        assert absent > 0
        assert [x.shard.tier_stats() for x in ws] == ts0  # nothing moved
        assert _counter_sum(ws, "lookup_miss") - miss0 == absent
        _check_entries(torch, oracle, ws, (w,), seen, R)
        for x in ws:
            assert x.status() == (False, False)
    finally:
        oracle.set_rsqrt_exact(False)


# ---------------------------------------------------------------------------------------------- 3. refused restore
def test_sharded_tier_restore_refused_when_pending_batches_hold_every_row(torch_cuda, oracle):
    """On R = 2 owners: every HBM row protected by two pending training forwards (keep = max(keep, pending + 1)), a
    third training forward of tier-held signs finds no free row.  They read zeros, their gradients are gradient misses,
    their tier entries stay as they were and the refusals are counted; once no batch is pending, the next request
    restores them with their values."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, C, dim = 2, 64, 16
    pf = oracle.index_prefix(0)
    gpu_opt, cpu_opt = _optim(N, oracle, "SGD")
    groups = [W.local_group(R, 1, dim, [pf], C, cap=256, optimizer=gpu_opt, max_batch=256, tier_rows=1024)]
    shards = [x.shard for x in groups[0]]
    groups += [W.local_group(R, 1, dim, [pf], C, cap=256, optimizer=gpu_opt, max_batch=256, shards=shards)
               for _ in range(2)]
    for s in shards:
        s.set_eviction(check_every=1, low_water=C, target_free=C, keep_batches=1)
    w = _oracle(oracle, [oracle.SlotCfg(dim, prefix=pf)], R, cpu_opt)
    _warm(torch, groups[0])
    rng = np.random.default_rng(9)
    sgn = lambda ids: oracle.add_prefix(np.asarray(ids, np.uint64), 8, pf)  # noqa: E731

    def fwd(ws, ids):
        """One training step's forward of group `ws`, rank r sending ids[r] (batches of their own sizes)."""
        d_ids = [to_dev_ids(x, DEV) for x in ids]
        outs = [None] * R
        torch.cuda.synchronize()
        for ph in (N.PHASE_SEND, N.PHASE_SERVE, N.PHASE_FINISH):
            for r, x in enumerate(ws):
                outs[r] = x.forward(d_ids[r], ids[r].size, True, out=outs[r], phases=ph)
        torch.cuda.synchronize()
        octx = [w.forward(ids[r], full_row_off(1, ids[r].size), ids[r].size, training=True) for r in range(R)]
        return [o.cpu().numpy()[0] for o in outs], [o[0][0] for o in octx], [o[1] for o in octx]

    def bwd(ws, ids, octx, train):
        """train: per rank whether its gradient goes (else add_skipped_gradient); the oracle steps what goes."""
        gs = [(rng.standard_normal((ids[r].size, dim)) * 1e-2).astype(np.float16) for r in range(R)]
        torch.cuda.synchronize()
        W.group_backward(ws, [[torch.from_numpy(gs[r]).to(DEV) if train[r] else None] for r in range(R)])
        torch.cuda.synchronize()
        return gs

    def oracle_bwd(octx, gs, train):
        for r in range(R):
            if train[r]:
                w.backward(octx[r], [gs[r]])
            else:
                w.backward(octx[r], [np.zeros_like(gs[r])], skip=[1])

    X = np.arange(40, dtype=np.uint64)
    other = lambda k: np.arange(100 + 10 * k, 110 + 10 * k, dtype=np.uint64)  # noqa: E731
    _, _, o = fwd(groups[0], [X, other(9)])
    oracle_bwd(o, bwd(groups[0], [X, other(9)], o, [True, True]), [True, True])
    for k in range(3):  # X ages out into the tiers
        ids = [other(2 * k), other(2 * k + 1)]
        _, _, o = fwd(groups[0], ids)
        oracle_bwd(o, bwd(groups[0], ids, o, [True, True]), [True, True])
    xs = sgn(X)
    owner = oracle.shard_of(xs, R)
    for r in range(R):
        held = set(shards[r]._export_table(shards[r].host_tier.h)[0].cpu().numpy().view(np.uint64).tolist())
        assert set(xs[owner == r].tolist()) <= held, r
    torch.cuda.synchronize()
    before = [s.get_entries(to_dev_ids(xs, DEV))[0].cpu().numpy() for s in shards]
    before = np.where((owner == 0)[:, None], before[0], before[1])
    # two pending forwards fill both owners' HBM; the pending rule protects every row from the checks of later calls
    A = [np.arange(1000, 1030, dtype=np.uint64), np.arange(1500, 1530, dtype=np.uint64)]
    _, _, oa = fwd(groups[1], A)
    need = [C - int(s.counters()["admitted"]) for s in shards]
    assert min(need) > 0
    cand = np.arange(2000, 4000, dtype=np.uint64)
    cown = oracle.shard_of(sgn(cand), R)
    fill = np.concatenate([cand[cown == q][:need[q]] for q in range(R)])
    Bb = [fill, A[1][:1]]  # rank 1 only refreshes a row of the pending batch
    _, _, ob = fwd(groups[2], Bb)
    assert all(int(s.counters()["admitted"]) == C for s in shards)
    refused0, gmiss0 = _tier_sum(groups[0], "refused"), _counter_sum(groups[0], "gradient_id_miss")
    Xc = [X, A[1][:1]]
    got, _, oc = fwd(groups[0], Xc)
    assert not got[0].view(np.uint16).any()  # every restore refused: zeros
    assert _tier_sum(groups[0], "refused") - refused0 == X.size
    # X's gradients go and are misses; every other request is skipped (the oracle steps nothing)
    bwd(groups[0], Xc, oc, [True, False])
    assert _counter_sum(groups[0], "gradient_id_miss") - gmiss0 == X.size
    oracle_bwd(oc, [np.zeros((x.size, dim), np.float16) for x in Xc], [False, False])
    for ws, ids, o in ((groups[1], A, oa), (groups[2], Bb, ob)):
        oracle_bwd(o, bwd(ws, ids, o, [False, False]), [False, False])
    torch.cuda.synchronize()
    after = [s.get_entries(to_dev_ids(xs, DEV)) for s in shards]
    for r in range(R):
        assert after[r][1].cpu().numpy()[owner == r].all()
    after = np.where((owner == 0)[:, None], after[0][0].cpu().numpy(), after[1][0].cpu().numpy())
    assert after.tobytes() == before.tobytes()
    got, want, o = fwd(groups[0], Xc)  # no batch pending: the checks free rows, X comes back with its values
    np.testing.assert_array_equal(got[0].view(np.uint16), want[0].view(np.uint16))
    oracle_bwd(o, bwd(groups[0], Xc, o, [True, True]), [True, True])
    torch.cuda.synchronize()
    for r in range(R):
        mine = xs[owner == r]
        ent, found = shards[r].get_entries(to_dev_ids(mine, DEV))
        assert found.cpu().numpy().all()
        ent = ent.cpu().numpy()
        for k, sign in enumerate(mine):
            assert same_bits(ent[k], w.get_entry(int(sign))), (r, int(sign))
    for ws in groups:
        for x in ws:
            assert x.status() == (False, False)
    assert _counter_sum(groups[0], "wait_errors") == 0


# ---------------------------------------------------------------------------------------------- 4. CUDA graph
def test_sharded_tier_graph_replay(torch_cuda, oracle):
    """A tiered virtual-rank step — eviction check with moves out, restores, lookups, backward — captured in CUDA graphs
    phase by phase (as test_virtual_ranks_graph_replay) and replayed over churn: outputs and entries equal the oracle's,
    which the eager steps also equal."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, S, B, dim, C = 2, 2, 128, 64, 1024  # a step brings an owner about S * B signs: a quarter of the HBM rows
    card = [3000, 3000]
    pf = [oracle.index_prefix(i) for i in range(S)]
    gpu_opt, cpu_opt = _optim(N, oracle, "ADAGRAD")
    oracle.set_rsqrt_exact(True)
    try:
        ws = W.local_group(R, S, dim, pf, C, cap=S * B, optimizer=gpu_opt, max_batch=B, tier_rows=1 << 13)
        for x in ws:
            x.shard.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=1)
        w = _oracle(oracle, [oracle.SlotCfg(dim, prefix=p) for p in pf], R, cpu_opt)
        _warm(torch, ws)
        rng = np.random.default_rng(21)
        ids_dev = [torch.zeros(S * B, dtype=torch.int64, device=DEV) for _ in range(R)]
        g_dev = [torch.zeros((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
        outs = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
        plan = [("f", N.PHASE_SEND), ("f", N.PHASE_SERVE), ("f", N.PHASE_FINISH), ("b", N.PHASE_SEND), ("b", N.PHASE_SERVE)]

        def enqueue(r, kind, ph):
            if kind == "f":
                ws[r].forward(ids_dev[r], B, training=True, out=outs[r], phases=ph)
            else:
                ws[r].backward(g_dev[r], phases=ph)

        def step(ids, g, graphs=None):
            for r in range(R):
                ids_dev[r].copy_(to_dev_ids(ids[r], DEV))
                g_dev[r].copy_(torch.from_numpy(g[r]).to(DEV))
            torch.cuda.synchronize()
            for kind, ph in plan:
                for r in range(R):
                    if graphs is None:
                        enqueue(r, kind, ph)
                    else:
                        with torch.cuda.stream(ws[r].stream):
                            graphs[(r, kind, ph)].replay()
            torch.cuda.synchronize()
            octx = [w.forward(ids[r], full_row_off(S, B), B, training=True) for r in range(R)]
            for r in range(R):
                w.backward(octx[r][1], [g[r, i] for i in range(S)])
            for r in range(R):
                got = outs[r].cpu().numpy()
                for i in range(S):
                    np.testing.assert_array_equal(got[i].view(np.uint16), octx[r][0][i].view(np.uint16))
                    seen.update(oracle.add_prefix(ids[r][i * B:(i + 1) * B], 8, pf[i]).tolist())

        def draw():
            return ([make_batch(rng, S, B, card)[0] for _ in range(R)],
                    (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16))

        seen = set()
        for _ in range(3):  # eager steps (they also warm up every allocation)
            step(*draw())
        graphs = {}
        for r in range(R):
            for kind, ph in plan:
                gph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gph, stream=ws[r].stream, capture_error_mode="thread_local"):
                    enqueue(r, kind, ph)
                graphs[(r, kind, ph)] = gph
        moved0 = _tier_sum(ws, "moved_out"), _tier_sum(ws, "restored")
        for _ in range(6):
            step(*draw(), graphs=graphs)
        assert _tier_sum(ws, "moved_out") > moved0[0] and _tier_sum(ws, "restored") > moved0[1]
        _check_entries(torch, oracle, ws, (w,), seen, R)
        _final_checks(ws)
    finally:
        oracle.set_rsqrt_exact(False)


# ---------------------------------------------------------------------------------------------- 5. incremental set
def test_sharded_tier_incremental_marks(torch_cuda, oracle):
    """With enable_incremental on every owner, tiered steps mark exactly the signs their gradients stepped on that
    owner (a host model: the signs of every request whose slot was not skipped), whether the sign sits in HBM or in the
    tier when the set is taken; the taken entries equal the oracle's."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, S, B, dim, C = 2, 2, 64, 16, 512  # a step brings an owner about S * B signs: a quarter of the HBM rows
    card = [1500, 1500]
    pf = [oracle.index_prefix(i) for i in range(S)]
    gpu_opt, cpu_opt = _optim(N, oracle, "SGD")
    ws = W.local_group(R, S, dim, pf, C, cap=S * B, optimizer=gpu_opt, max_batch=B, tier_rows=1 << 13)
    for x in ws:
        x.shard.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=1)
        x.enable_incremental(1 << 14)
    w = _oracle(oracle, [oracle.SlotCfg(dim, prefix=p) for p in pf], R, cpu_opt)
    _warm(torch, ws)
    rng = np.random.default_rng(33)
    marked = set()
    for step in range(14):
        ids = [make_batch(rng, S, B, card)[0] for _ in range(R)]
        torch.cuda.synchronize()
        W.group_forward(ws, [to_dev_ids(x, DEV) for x in ids], B, training=True)
        torch.cuda.synchronize()
        octx = [w.forward(ids[r], full_row_off(S, B), B, training=True)[1] for r in range(R)]
        g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16)
        skip = [[0] * S for _ in range(R)]
        if step % 3 == 1:
            skip[step % R][1] = 1  # one rank skips slot 1: its signs of that slot are not stepped by its request
        dg = [[None if skip[r][i] else torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)]
        W.group_backward(ws, dg)
        torch.cuda.synchronize()
        for r in range(R):
            w.backward(octx[r], [g[r, i] for i in range(S)], skip=skip[r])
            for i in range(S):
                if not skip[r][i]:
                    marked.update(oracle.add_prefix(ids[r][i * B:(i + 1) * B], 8, pf[i]).tolist())
    assert _tier_sum(ws, "moved_out") > 0 and _tier_sum(ws, "restored") > 0
    assert _counter_sum(ws, "capacity_refused") == 0 and _counter_sum(ws, "gradient_id_miss") == 0
    signs = np.array(sorted(marked), np.uint64)
    owner = oracle.shard_of(signs, R)
    for r in range(R):
        got, ent, skipped = ws[r].take_incremental()
        got = np.asarray(got).view(np.uint64)
        assert skipped == 0, r
        assert got.tolist() == signs[owner == r].tolist(), r
        for k, sign in enumerate(got):
            assert same_bits(np.asarray(ent)[k], w.get_entry(int(sign))), (r, int(sign))
    for x in ws:
        assert x.status() == (False, False)


# ---------------------------------------------------------------------------------------------- 6. two processes
def _rank_main(rank, world, port, result_dir):
    import torch
    import torch.distributed as dist

    import oracle
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    S, B, dim, C, card = 2, 256, 64, 512, [3000, 3000]
    pf = [oracle.index_prefix(i) for i in range(S)]
    wk = ShardedEmbeddingWorker.distributed(S, dim, pf, C, cap=S * B, device=dev, max_batch=B, tier_rows=1 << 14,
                                            optimizer=dict(kind=N.OPT_ADAGRAD, lr=0.02, initialization=0.01, eps=1e-10))
    wk.shard.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=1)
    rng = np.random.default_rng(43)
    outs, seen = [], set()
    for step in range(8):
        ids = [make_batch(rng, S, B, card)[0] for _ in range(world)]  # every rank draws all, keeps its own
        g = (rng.standard_normal((world, S, B, dim)) * 1e-2).astype(np.float16)
        out = wk.forward(torch.from_numpy(ids[rank].view(np.int64)).to(dev), B, training=True)
        wk.backward(torch.from_numpy(g[rank]).to(dev))
        torch.cuda.synchronize()
        dist.barrier()
        outs.append(out.cpu().numpy())
        for r in range(world):
            for i in range(S):
                seen.update(oracle.add_prefix(ids[r][i * B:(i + 1) * B], 8, pf[i]).tolist())
    signs = np.array(sorted(seen), np.uint64)
    mine = signs[oracle.shard_of(signs, world) == rank]
    ent, found = wk.shard.get_entries(torch.from_numpy(mine.view(np.int64)).to(dev))
    ts = wk.shard.tier_stats()
    assert found.all() and wk.status() == (False, False)
    assert ts["moved_out"] > 0 and ts["restored"] > 0 and ts["refused"] == 0 and ts["dropped"] == 0, ts
    np.savez(os.path.join(result_dir, f"rank{rank}.npz"), outs=np.stack(outs), signs=mine, ent=ent.cpu().numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_tier_two_processes_symmetric_memory(torch_cuda, oracle, tmp_path):
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
        S, B, dim, card = 2, 256, 64, [3000, 3000]
        pf = [oracle.index_prefix(i) for i in range(S)]
        w = _oracle(oracle, [oracle.SlotCfg(dim, prefix=p) for p in pf], world,
                    oracle.Optim(oracle.ADAGRAD, lr=0.02, init_acc=0.01, eps=1e-10))
        rng = np.random.default_rng(43)
        res = [np.load(os.path.join(str(tmp_path), f"rank{r}.npz")) for r in range(world)]
        for step in range(8):
            ids = [make_batch(rng, S, B, card)[0] for _ in range(world)]
            g = (rng.standard_normal((world, S, B, dim)) * 1e-2).astype(np.float16)
            octx = [w.forward(ids[r], full_row_off(S, B), B, training=True) for r in range(world)]
            for r in range(world):
                for i in range(S):
                    np.testing.assert_array_equal(res[r]["outs"][step][i].view(np.uint16), octx[r][0][i].view(np.uint16))
            for r in range(world):
                w.backward(octx[r][1], [g[r, i] for i in range(S)])
        for r in range(world):
            for k, sign in enumerate(res[r]["signs"]):
                assert res[r]["ent"][k].tobytes() == w.get_entry(int(sign)).tobytes()
    finally:
        oracle.set_rsqrt_exact(False)
