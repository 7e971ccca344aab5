"""GPU: staging on R GPUs (pb_tier_stage_sharded through worker.TierStager).  Every rank sends its next training batch's
signs to their owners one step early; each owner runs the eviction check that batch would run and moves the tier-held
signs it received back into HBM, on the stager's stream, beside the current backward.  Moves never change a value, and
a sign the stage does not move is restored by the forward as before, so a staged run equals the unstaged run bit for
bit, and both equal the oracle's embedding worker with R parameter servers.

R virtual ranks share cuda:0, driven phase by phase as in test_gpu_sharded_tier.py."""
import ctypes as C
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
FIELDS = ("lookup_miss", "gradient_id_miss", "capacity_refused", "wait_errors")


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


def _sum(ws, fn, field):
    return sum(int(fn(x)[field]) for x in ws)


def _forward_restores(ws):
    """Restores done by the forwards: all restores less the staged ones."""
    return _sum(ws, lambda x: x.shard.tier_stats(), "restored") - _sum(ws, lambda x: x.shard.stage_stats(), "staged")


# ---------------------------------------------------------------------------------------------- the churn workload
class Churn:
    """Two summation slots (one-id and ragged steps, f16 and f32 gradients, loss scales) and a raw slot on every rank's
    tiered table, one eviction check per training request; C HBM rows per rank over about 4 C keys per owner.  All
    batches are drawn up front, so a stage can bring batch i + 1 while batch i trains."""

    S, B, RB, fixed = 2, 64, 48, 3

    def __init__(self, oracle, R, dim, steps, seed):
        rng = np.random.default_rng(seed)
        self.R, self.dim, self.steps = R, dim, steps
        self.pf = [oracle.index_prefix(g) for g in (0, 1)]
        self.rpf = oracle.index_prefix(2)
        card, raw_card = [1600 * R, 1600 * R], 900 * R
        self.sum = [[make_batch(rng, self.S, self.B, card, max_ids=3 if i % 2 else 1) for _ in range(R)]
                    for i in range(steps)]
        self.raw = []
        for _ in range(steps):
            per = []
            for _ in range(R):
                ro = np.zeros(self.RB + 1, np.uint32)
                ro[1:] = np.cumsum(rng.integers(0, 5, size=self.RB))
                per.append((rng.integers(0, raw_card, size=int(ro[-1]), dtype=np.uint64), ro))
            self.raw.append(per)
        self.f32 = [i % 4 >= 2 for i in range(steps)]
        self.g = [(rng.standard_normal((R, self.S, self.B, dim)) * 1e-2).astype(np.float32 if f else np.float16)
                  for f in self.f32]
        self.rseed = seed + 1

    def stage_batch(self, i, r):
        """(ids, slot offsets) of step i's training requests of rank r, as one stage: the summation slots, then the raw
        slot (prefixes self.pf + [self.rpf])."""
        ids, _, so = self.sum[i][r]
        rids = self.raw[i][r][0]
        return np.concatenate([ids, rids]), list(so) + [len(ids) + len(rids)]


def _build(torch, oracle, N, R, name, dim, C=1024, T=1 << 14, stage_cap=None, staged=True):
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW, TierStager

    gpu_opt, _ = _optim(N, oracle, name)
    S, B, RB = Churn.S, Churn.B, Churn.RB
    pf = [oracle.index_prefix(g) for g in (0, 1)]
    ws = W.local_group(R, S, dim, pf, C, cap=S * B * 3, optimizer=gpu_opt, max_batch=B, rows_f32=True,
                       max_ids_per_sample=3, tier_rows=T)
    rws = RW.local_group(R, 1, dim, [oracle.index_prefix(2)], C, cap=RB * 4, optimizer=gpu_opt, max_batch=RB,
                         max_ids_per_sample=4, shards=[x.shard for x in ws])
    for x in ws:  # protected: the last two requests; the sweep frees down to C / 2
        x.shard.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=2)
    stagers = TierStager.local_group([x.shard for x in ws], stage_cap or (S * B * 3 + RB * 4)) if staged else None
    _warm(torch, ws)
    return ws, rws, stagers


def _run(torch, oracle, N, wl, ws, rws, stagers, sync, check=None):
    """Runs the workload; returns what a run computes: per step the outputs, raw tables and statuses; then every seen
    sign's entry (HBM or tier) and the table counters.  stagers: stage batch i + 1 after forward i, before backward i.
    sync: synchronise after every call (else the stage runs on its stream beside the backward).  check(i, what, a, b):
    called after step i's forwards ("forward", their outputs) and backwards ("backward", the step's results)."""
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW, TierStager

    R, S, B, RB = wl.R, wl.S, wl.B, wl.RB
    rng = np.random.default_rng(wl.rseed)
    sy = torch.cuda.synchronize if sync else (lambda: None)
    prefixes = wl.pf + [wl.rpf]
    got, seen = [], set()
    fwd_miss = [0] * R  # lookup misses of the forwards (pb_get_rows counts a tier-held sign it reads as one too)

    def lookup_misses():
        torch.cuda.synchronize()
        return [int(x.shard.counters()["lookup_miss"]) for x in ws]

    def stage_ids(i):
        nxt = [wl.stage_batch(i, r) for r in range(R)]
        return [to_dev_ids(x[0], DEV) for x in nxt], [x[1] for x in nxt]

    if stagers:
        d_stage = stage_ids(0)
        torch.cuda.synchronize()
        TierStager.group_stage(stagers, *d_stage, prefixes)
    for i in range(wl.steps):
        # every input on the device first (the calls run on the workers' and stagers' streams, and the tensors live
        # until the step has synchronised)
        batches, rb = wl.sum[i], wl.raw[i]
        ragged = batches[0][1] is not None
        d_ids = [to_dev_ids(b[0], DEV) for b in batches]
        d_ro = [to_dev_i32(b[1], DEV) for b in batches] if ragged else None
        d_rids = [to_dev_ids(b[0], DEV) for b in rb]
        d_rro = [to_dev_i32(b[1], DEV) for b in rb]
        d_stage = stage_ids(i + 1) if stagers and i + 1 < wl.steps else None
        dg = [[torch.from_numpy(wl.g[i][r, s]).to(DEV) for s in range(S)] for r in range(R)]
        m0 = lookup_misses()
        outs = W.group_forward(ws, d_ids, B, training=True, row_offs=d_ro, slot_occ_offs=[b[2] for b in batches])
        sy()
        res = RW.group_forward_raw(rws, d_rids, RB, wl.fixed, row_offs=d_rro)
        sy()
        fwd_miss = [a + c - b for a, b, c in zip(fwd_miss, m0, lookup_misses())]
        if check is not None:
            torch.cuda.synchronize()
            check(i, "forward", outs, res)
        if d_stage is not None:
            TierStager.group_stage(stagers, *d_stage, prefixes)
            sy()
        scale = [128.0, 1.0] if wl.f32[i] else [1.0, 64.0]
        sts = W.group_backward(ws, dg, scales=scale, want_status=True)
        sy()
        torch.cuda.synchronize()  # (U of the raw forward)
        rg = []
        for r in range(R):
            U = int(res[r][4][0])
            rg.append(torch.from_numpy((rng.standard_normal((U, wl.dim)) * 1e-2).astype(np.float32)).to(DEV) if U else None)
        torch.cuda.synchronize()
        rsts = RW.group_backward_raw(rws, rg, scales=[32.0] * R, want_status=True)
        torch.cuda.synchronize()
        step = dict(outs=[o.cpu().numpy().tobytes() for o in outs],
                    raw=[(t[:int(c[0]) + 1].cpu().numpy().tobytes(), ix.cpu().numpy().tobytes())
                         for t, ix, _, _, c in res],
                    sts=[s.cpu().numpy().tolist() for s in sts], rsts=[s.item() for s in rsts],
                    rg=[x.cpu().numpy() if x is not None else None for x in rg])
        if check is not None:
            check(i, "backward", step, None)
        got.append(step)
        for r in range(R):
            seen.update(slot_signs(oracle, batches[r][0], batches[r][2], wl.pf).tolist())
            seen.update(oracle.add_prefix(rb[r][0], 8, wl.rpf).tolist())
    counters = [[fwd_miss[r]] + [int(x.shard.counters()[f]) for f in FIELDS[1:]] for r, x in enumerate(ws)]
    signs = np.array(sorted(seen), np.uint64)
    owner = oracle.shard_of(signs, R)
    ents = []
    for r in range(R):
        ent, found = ws[r].shard.get_entries(to_dev_ids(signs[owner == r], DEV))
        assert found.cpu().numpy().all(), r
        ents.append(ent.cpu().numpy())
    for x in list(ws) + list(rws):
        assert x.status() == (False, False)
    return dict(steps=got, signs=signs, ents=ents, counters=counters, lens=[len(x.shard) for x in ws],
                stage_status=[s.status() for s in stagers or []])


def _oracle_check(torch, oracle, N, wl, ws, name):
    """check() of _run comparing each step with the oracle (as test_gpu_sharded_tier.py does); returns it and the two
    oracle workers."""
    _, cpu_opt = _optim(N, oracle, name)
    R, S, B, RB, dim = wl.R, wl.S, wl.B, wl.RB, wl.dim
    w = _oracle(oracle, [oracle.SlotCfg(dim, prefix=p) for p in wl.pf], R, cpu_opt)
    wr = _oracle(oracle, [oracle.SlotCfg(dim, summation=False, sample_fixed_size=wl.fixed, prefix=wl.rpf)], R, cpu_opt)
    st = {}

    def check(i, what, a, b):
        batches = wl.sum[i]
        ragged = batches[0][1] is not None
        if what == "forward":
            outs, res = a, b
            signs = [slot_signs(oracle, x[0], x[2], wl.pf) for x in batches]
            rows = held_rows(torch, oracle, [x.shard for x in ws], np.concatenate(signs))
            st["octx"], st["rctx"] = [], []
            for r in range(R):
                ro = batches[r][1] if ragged else full_row_off(S, B)
                want, c = w.forward(batches[r][0], ro, B, training=True)
                st["octx"].append(c)
                got = outs[r].cpu().numpy()
                model = pool_model(rows, signs[r], batches[r][1], B, None, dim=dim)
                counts = np.diff(ro).reshape(S, B)
                for s in range(S):
                    assert same_bits(got[s], model[s]), (i, r, s)
                    one = counts[s] <= 1  # a sample of several ids may differ by 1 f16 ulp: f32 sum order
                    np.testing.assert_array_equal(got[s][one].view(np.uint16), want[s][one].view(np.uint16))
                    assert f16_ulp_diff(got[s][~one], want[s][~one]) <= 1, (i, r, s)
                table, index, _, _, cnt = res[r]
                rb = wl.raw[i][r]
                wt, wi, _, _, oc = wr.forward_raw(0, rb[0], rb[1], RB, training=True)
                assert table[:int(cnt[0]) + 1].cpu().numpy().tobytes() == wt.tobytes(), (i, r)
                np.testing.assert_array_equal(index.cpu().numpy(), wi)
                st["rctx"].append(oc)
        else:
            step = a
            scale = [128.0, 1.0] if wl.f32[i] else [1.0, 64.0]
            for r in range(R):
                assert step["sts"][r] == w.backward(st["octx"][r], [wl.g[i][r, s] for s in range(S)], scale=scale), (i, r)
                g = step["rg"][r]
                assert step["rsts"][r] == wr.backward_raw(0, st["rctx"][r], g, scale=32.0, skip=g is None), (i, r)

    return check, (w, wr)


def _check_entries(oracle, result, oracles, R):
    owner = oracle.shard_of(result["signs"], R)
    for r in range(R):
        for k, sign in enumerate(result["signs"][owner == r]):
            ref = next(e for e in (o.get_entry(int(sign)) for o in oracles) if e is not None)
            assert same_bits(result["ents"][r][k], ref), (r, k, int(sign))
        assert result["lens"][r] == sum(o.ps_len(r) for o in oracles), r


def _same_results(a, b):
    assert len(a["steps"]) == len(b["steps"])
    for i, (x, y) in enumerate(zip(a["steps"], b["steps"])):
        for k in ("outs", "raw", "sts", "rsts"):
            assert x[k] == y[k], (i, k)
    assert a["signs"].tobytes() == b["signs"].tobytes()
    for r, (x, y) in enumerate(zip(a["ents"], b["ents"])):
        assert x.tobytes() == y.tobytes(), r
    assert a["counters"] == b["counters"] and a["lens"] == b["lens"]


def _close(*groups):
    for g in groups:
        for x in g or []:
            x.close()


# ---------------------------------------------------------------------------------------------- 1. parity, 2. beside
@pytest.mark.parametrize("R", [2, 4])
@pytest.mark.parametrize("name,dim", [("SGD", 16), ("ADAGRAD", 32), ("ADAGRAD_VW", 20), ("ADAM", 24)])
def test_staged_equals_unstaged_and_oracle(torch_cuda, oracle, R, name, dim):
    """The unstaged run equals the oracle step by step; the staged run (every call synchronised) equals the unstaged one
    bit for bit: outputs, statuses, raw tables, every entry afterwards and the counters.  The stage moves signs, and the
    forwards restore strictly fewer."""
    from persia_b200 import native as N

    torch = torch_cuda
    wl = Churn(oracle, R, dim, 16, R * 100 + dim)
    oracle.set_rsqrt_exact(True)
    try:
        ws, rws, _ = _build(torch, oracle, N, R, name, dim, staged=False)
        check, oracles = _oracle_check(torch, oracle, N, wl, ws, name)
        plain = _run(torch, oracle, N, wl, ws, rws, None, sync=True, check=check)
        _check_entries(oracle, plain, oracles, R)
        assert all(c[1:] == [0, 0, 0] for c in plain["counters"]), plain["counters"]
        restores_plain = _forward_restores(ws)
        assert restores_plain > 0 and _sum(ws, lambda x: x.shard.tier_stats(), "moved_out") > 0
        _close(rws, ws)
        ws, rws, stagers = _build(torch, oracle, N, R, name, dim)
        staged = _run(torch, oracle, N, wl, ws, rws, stagers, sync=True)
        _same_results(plain, staged)
        assert staged["stage_status"] == [(False, False)] * R
        assert _sum(ws, lambda x: x.shard.stage_stats(), "staged") > 0
        assert _forward_restores(ws) < restores_plain
        assert _sum(ws, lambda x: x.shard.tier_stats(), "dropped") == 0
        _close(stagers, rws, ws)
    finally:
        oracle.set_rsqrt_exact(False)


@pytest.mark.parametrize("R", [2, 4])
def test_stage_beside_the_backward(torch_cuda, oracle, R):
    """No synchronisation inside a step: each rank's stage runs on its stager's stream while its backwards run on the
    workers' streams.  Results equal the serial unstaged run's."""
    from persia_b200 import native as N

    torch = torch_cuda
    name, dim = "ADAGRAD", 32
    wl = Churn(oracle, R, dim, 12, 7 + R)
    oracle.set_rsqrt_exact(True)
    try:
        ws, rws, _ = _build(torch, oracle, N, R, name, dim, staged=False)
        plain = _run(torch, oracle, N, wl, ws, rws, None, sync=True)
        _close(rws, ws)
        ws, rws, stagers = _build(torch, oracle, N, R, name, dim)
        beside = _run(torch, oracle, N, wl, ws, rws, stagers, sync=False)
        _same_results(plain, beside)
        assert beside["stage_status"] == [(False, False)] * R
        assert _sum(ws, lambda x: x.shard.stage_stats(), "staged") > 0
        _close(stagers, rws, ws)
    finally:
        oracle.set_rsqrt_exact(False)


# ---------------------------------------------------------------------------------------------- 4. cap overflow
def test_stage_cap_overflow(torch_cuda, oracle):
    """A stage exchange whose cap is smaller than what a stage sends one owner: status()[0] is raised, the signs that
    fit are staged, the rest restored by the forward, and the results equal the unstaged run's."""
    from persia_b200 import native as N

    torch = torch_cuda
    R, name, dim = 2, "SGD", 16
    wl = Churn(oracle, R, dim, 10, 77)
    ws, rws, _ = _build(torch, oracle, N, R, name, dim, staged=False)
    plain = _run(torch, oracle, N, wl, ws, rws, None, sync=True)
    _close(rws, ws)
    ws, rws, stagers = _build(torch, oracle, N, R, name, dim, stage_cap=24)
    small = _run(torch, oracle, N, wl, ws, rws, stagers, sync=True)
    _same_results(plain, small)
    assert small["stage_status"] == [(True, False)] * R
    staged = _sum(ws, lambda x: x.shard.stage_stats(), "staged")
    assert 0 < staged
    assert _forward_restores(ws) > 0
    _close(stagers, rws, ws)


# ---------------------------------------------------------------------------------------------- 3. no free rows
def test_stage_skips_when_pending_batches_hold_every_row(torch_cuda, oracle):
    """Two pending forwards hold every HBM row of both owners (keep = max(keep, pending + 1)); a stage of tier-held signs
    finds no free row: every one is counted as skipped and nothing moves.  Once no batch is pending the forward restores
    them, with their values, as the oracle computes."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W, TierStager

    torch = torch_cuda
    R, C, dim = 2, 64, 16
    pf = oracle.index_prefix(0)
    gpu_opt, cpu_opt = _optim(N, oracle, "SGD")
    groups = [W.local_group(R, 1, dim, [pf], C, cap=256, optimizer=gpu_opt, max_batch=256, tier_rows=1024)]
    shards = [x.shard for x in groups[0]]
    groups += [W.local_group(R, 1, dim, [pf], C, cap=256, optimizer=gpu_opt, max_batch=256, shards=shards)
               for _ in range(2)]
    stagers = TierStager.local_group(shards, 256)
    for s in shards:
        s.set_eviction(check_every=1, low_water=C, target_free=C, keep_batches=1)
    w = _oracle(oracle, [oracle.SlotCfg(dim, prefix=pf)], R, cpu_opt)
    _warm(torch, groups[0])
    rng = np.random.default_rng(9)
    sgn = lambda ids: oracle.add_prefix(np.asarray(ids, np.uint64), 8, pf)  # noqa: E731

    def fwd(ws, ids):
        torch.cuda.synchronize()
        d_ids = [to_dev_ids(x, DEV) for x in ids]
        outs = [None] * R
        for ph in (N.PHASE_SEND, N.PHASE_SERVE, N.PHASE_FINISH):
            for r, x in enumerate(ws):
                outs[r] = x.forward(d_ids[r], ids[r].size, True, out=outs[r], phases=ph)
        torch.cuda.synchronize()
        octx = [w.forward(ids[r], full_row_off(1, ids[r].size), ids[r].size, training=True) for r in range(R)]
        return [o.cpu().numpy()[0] for o in outs], [o[0][0] for o in octx], [o[1] for o in octx]

    def bwd(ws, ids, octx, train):
        gs = [(rng.standard_normal((ids[r].size, dim)) * 1e-2).astype(np.float16) for r in range(R)]
        torch.cuda.synchronize()
        W.group_backward(ws, [[torch.from_numpy(gs[r]).to(DEV) if train[r] else None] for r in range(R)])
        torch.cuda.synchronize()
        for r in range(R):
            if train[r]:
                w.backward(octx[r], [gs[r]])
            else:
                w.backward(octx[r], [np.zeros_like(gs[r])], skip=[1])

    X = np.arange(40, dtype=np.uint64)
    other = lambda k: np.arange(100 + 10 * k, 110 + 10 * k, dtype=np.uint64)  # noqa: E731
    _, _, o = fwd(groups[0], [X, other(9)])
    bwd(groups[0], [X, other(9)], o, [True, True])
    for k in range(3):  # X ages out into the tiers
        ids = [other(2 * k), other(2 * k + 1)]
        _, _, o = fwd(groups[0], ids)
        bwd(groups[0], ids, o, [True, True])
    xs = sgn(X)
    owner = oracle.shard_of(xs, R)
    torch.cuda.synchronize()
    # two pending forwards fill both owners' HBM
    A = [np.arange(1000, 1030, dtype=np.uint64), np.arange(1500, 1530, dtype=np.uint64)]
    _, _, oa = fwd(groups[1], A)
    need = [C - int(s.counters()["admitted"]) for s in shards]
    assert min(need) > 0
    cand = np.arange(2000, 4000, dtype=np.uint64)
    cown = oracle.shard_of(sgn(cand), R)
    Bb = [np.concatenate([cand[cown == q][:need[q]] for q in range(R)]), A[1][:1]]
    _, _, ob = fwd(groups[2], Bb)
    assert all(int(s.counters()["admitted"]) == C for s in shards)
    ts0 = [s.tier_stats() for s in shards]
    Xc = [X, A[1][:1]]
    TierStager.group_stage(stagers, [to_dev_ids(x, DEV) for x in Xc], [[0, x.size] for x in Xc], [pf])
    torch.cuda.synchronize()
    st = [s.stage_stats() for s in shards]
    assert sum(x["staged"] for x in st) == 0 and sum(x["skipped"] for x in st) == X.size, st
    assert [s.tier_stats() for s in shards] == ts0  # nothing moved
    for ws, ids, o in ((groups[1], A, oa), (groups[2], Bb, ob)):  # the pending batches go, skipped
        bwd(ws, ids, o, [False, False])
    ids = [other(7), other(8)]  # one more request, so that the next check may free the rows of both
    _, _, o = fwd(groups[0], ids)
    bwd(groups[0], ids, o, [True, True])
    got, want, o = fwd(groups[0], Xc)  # the forward's check frees rows, its restore brings X back
    np.testing.assert_array_equal(got[0].view(np.uint16), want[0].view(np.uint16))
    assert sum(s.tier_stats()["refused"] for s in shards) == 0
    bwd(groups[0], Xc, o, [True, True])
    torch.cuda.synchronize()
    for r in range(R):
        mine = xs[owner == r]
        ent, found = shards[r].get_entries(to_dev_ids(mine, DEV))
        assert found.cpu().numpy().all()
        for k, sign in enumerate(mine):
            assert same_bits(ent.cpu().numpy()[k], w.get_entry(int(sign))), (r, int(sign))
    for x in [y for g in groups for y in g] + stagers:
        assert x.status() == (False, False)
    _close(stagers, groups[2], groups[1], groups[0])


# ---------------------------------------------------------------------------------------------- 5. untrained, 6. no tier
def test_staged_batch_that_never_trains_changes_nothing(torch_cuda, oracle):
    """After tiered training, a stage of seen (mostly tier-held) and never-seen signs moves entries but changes no
    value and admits nothing: every entry reads as before and each shard holds as many entries."""
    from persia_b200 import native as N
    from persia_b200.worker import TierStager

    torch = torch_cuda
    R, name, dim = 2, "ADAM", 24
    wl = Churn(oracle, R, dim, 8, 5)
    ws, rws, _ = _build(torch, oracle, N, R, name, dim, staged=False)
    res = _run(torch, oracle, N, wl, ws, rws, None, sync=True)
    stagers = TierStager.local_group([x.shard for x in ws], 4096)
    rng = np.random.default_rng(1)
    signs, owner = res["signs"], oracle.shard_of(res["signs"], R)
    ids = [np.concatenate([signs[rng.permutation(signs.size)[:700]], np.arange(1 << 40, (1 << 40) + 300, dtype=np.uint64)])
           for _ in range(R)]
    TierStager.group_stage(stagers, [to_dev_ids(x, DEV) for x in ids], [[0, x.size] for x in ids], [0])
    torch.cuda.synchronize()
    assert _sum(ws, lambda x: x.shard.stage_stats(), "staged") > 0
    for r in range(R):
        ent, found = ws[r].shard.get_entries(to_dev_ids(signs[owner == r], DEV))
        assert found.cpu().numpy().all()
        assert ent.cpu().numpy().tobytes() == res["ents"][r].tobytes(), r
        assert len(ws[r].shard) == res["lens"][r]
        assert [int(ws[r].shard.counters()[f]) for f in FIELDS[1:]] == res["counters"][r][1:]
    _close(stagers, rws, ws)


def test_stage_without_a_tier_is_a_collective_no_op(torch_cuda, oracle):
    """Untiered shards: the stage is still collective (every owner waits for and consumes the flags), and tables and
    counters stay as they were; the next steps still equal the oracle."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W, TierStager

    torch = torch_cuda
    R, S, B, dim, C = 2, 2, 64, 16, 4096
    pf = [oracle.index_prefix(i) for i in range(S)]
    gpu_opt, cpu_opt = _optim(N, oracle, "ADAGRAD")
    oracle.set_rsqrt_exact(True)
    try:
        ws = W.local_group(R, S, dim, pf, C, cap=S * B, optimizer=gpu_opt, max_batch=B)
        stagers = TierStager.local_group([x.shard for x in ws], S * B)
        w = _oracle(oracle, [oracle.SlotCfg(dim, prefix=p) for p in pf], R, cpu_opt)
        _warm(torch, ws)
        rng = np.random.default_rng(3)
        seen = set()
        for step in range(4):
            ids = [make_batch(rng, S, B, [500, 500])[0] for _ in range(R)]
            torch.cuda.synchronize()
            snap = [(x.shard.counters(), len(x.shard)) for x in ws]
            TierStager.group_stage(stagers, [to_dev_ids(x, DEV) for x in ids], [[s * B for s in range(S + 1)]] * R, pf)
            torch.cuda.synchronize()
            assert [(x.shard.counters(), len(x.shard)) for x in ws] == snap
            assert all(x.shard.stage_stats() == {"staged": 0, "skipped": 0} for x in ws)
            outs = W.group_forward(ws, [to_dev_ids(x, DEV) for x in ids], B, training=True)
            torch.cuda.synchronize()
            octx = [w.forward(ids[r], full_row_off(S, B), B, training=True) for r in range(R)]
            for r in range(R):
                np.testing.assert_array_equal(outs[r].cpu().numpy().view(np.uint16), np.asarray(octx[r][0]).view(np.uint16))
                for i in range(S):
                    seen.update(oracle.add_prefix(ids[r][i * B:(i + 1) * B], 8, pf[i]).tolist())
            g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16)
            W.group_backward(ws, [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)])
            torch.cuda.synchronize()
            for r in range(R):
                w.backward(octx[r][1], [g[r, i] for i in range(S)])
        signs = np.array(sorted(seen), np.uint64)
        owner = oracle.shard_of(signs, R)
        for r in range(R):
            ent = ws[r].shard.get_entries(to_dev_ids(signs[owner == r], DEV))[0].cpu().numpy()
            for k, sign in enumerate(signs[owner == r]):
                assert same_bits(ent[k], w.get_entry(int(sign)))
        for x in ws + stagers:
            assert x.status() == (False, False)
        _close(stagers, ws)
    finally:
        oracle.set_rsqrt_exact(False)


# ---------------------------------------------------------------------------------------------- 7. CUDA graph
def test_staged_step_graph_replay_equals_eager(torch_cuda, oracle):
    """A whole virtual-rank step — forwards, the next batch's stage forked onto the stagers' streams, backwards — is
    captured in one CUDA graph and replayed over churn.  Outputs and entries equal the same staged steps run eagerly on
    a second set of tables, and the oracle's."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W, TierStager

    torch = torch_cuda
    R, S, B, dim, C = 2, 2, 128, 64, 1024
    card = [3000, 3000]
    pf = [oracle.index_prefix(i) for i in range(S)]
    gpu_opt, cpu_opt = _optim(N, oracle, "ADAGRAD")
    rng = np.random.default_rng(21)
    steps = 9
    ids = [[make_batch(rng, S, B, card)[0] for _ in range(R)] for _ in range(steps + 1)]
    gs = [(rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16) for _ in range(steps)]
    so = [s * B for s in range(S + 1)]
    oracle.set_rsqrt_exact(True)
    try:
        def group():
            ws = W.local_group(R, S, dim, pf, C, cap=S * B, optimizer=gpu_opt, max_batch=B, tier_rows=1 << 13)
            for x in ws:
                x.shard.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=1)
            _warm(torch, ws)
            return ws, TierStager.local_group([x.shard for x in ws], S * B)

        ids_dev = [torch.zeros(S * B, dtype=torch.int64, device=DEV) for _ in range(R)]
        nxt_dev = [torch.zeros(S * B, dtype=torch.int64, device=DEV) for _ in range(R)]
        g_dev = [torch.zeros((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
        outs = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]

        def enqueue(ws, stagers):
            W.group_forward(ws, ids_dev, B, training=True, outs=outs)
            TierStager.group_stage(stagers, nxt_dev, [so] * R, pf)
            W.group_backward(ws, g_dev)

        def load(i):
            for r in range(R):
                ids_dev[r].copy_(to_dev_ids(ids[i][r], DEV))
                nxt_dev[r].copy_(to_dev_ids(ids[i + 1][r], DEV))
                g_dev[r].copy_(torch.from_numpy(gs[i][r]).to(DEV))
            torch.cuda.synchronize()

        w = _oracle(oracle, [oracle.SlotCfg(dim, prefix=p) for p in pf], R, cpu_opt)
        eager_ws, eager_st = group()
        graph_ws, graph_st = group()
        eager, replayed = [], []
        for grp, out in (((eager_ws, eager_st), eager), ((graph_ws, graph_st), replayed)):
            TierStager.group_stage(grp[1], [to_dev_ids(x, DEV) for x in ids[0]], [so] * R, pf)
            for i in range(3):  # eager steps for both (they also warm up every allocation)
                load(i)
                enqueue(*grp)
                torch.cuda.synchronize()
                out.append([o.cpu().numpy().tobytes() for o in outs])
        for i in range(3, steps):
            load(i)
            enqueue(eager_ws, eager_st)
            torch.cuda.synchronize()
            eager.append([o.cpu().numpy().tobytes() for o in outs])
        cap = torch.cuda.Stream(device=DEV)
        side = [x.stream for x in graph_ws] + [s.stream for s in graph_st]
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=cap, capture_error_mode="thread_local"):
            for s in side:  # fork: every rank's worker and stager streams join the capture
                s.wait_stream(cap)
            enqueue(graph_ws, graph_st)
            for s in side:  # join
                cap.wait_stream(s)
        for i in range(3, steps):
            load(i)
            with torch.cuda.stream(cap):
                graph.replay()
            torch.cuda.synchronize()
            replayed.append([o.cpu().numpy().tobytes() for o in outs])
        assert replayed == eager
        for i in range(steps):  # and both equal the oracle
            octx = [w.forward(ids[i][r], full_row_off(S, B), B, training=True) for r in range(R)]
            for r in range(R):
                assert eager[i][r] == np.asarray(octx[r][0]).tobytes(), (i, r)
                w.backward(octx[r][1], [gs[i][r, s] for s in range(S)])
        seen = np.array(sorted({int(x) for i in range(steps) for r in range(R) for s in range(S)
                                for x in oracle.add_prefix(ids[i][r][s * B:(s + 1) * B], 8, pf[s])}), np.uint64)
        owner = oracle.shard_of(seen, R)
        for r in range(R):
            mine = to_dev_ids(seen[owner == r], DEV)
            a = eager_ws[r].shard.get_entries(mine)[0].cpu().numpy()
            b = graph_ws[r].shard.get_entries(mine)[0].cpu().numpy()
            assert a.tobytes() == b.tobytes(), r
            for k, sign in enumerate(seen[owner == r]):
                assert same_bits(a[k], w.get_entry(int(sign)))
        assert _sum(graph_ws, lambda x: x.shard.stage_stats(), "staged") > 0
        for x in eager_ws + graph_ws + eager_st + graph_st:
            assert x.status() == (False, False)
        _close(eager_st, graph_st, eager_ws, graph_ws)
    finally:
        oracle.set_rsqrt_exact(False)


# ---------------------------------------------------------------------------------------------- 8. refusals
def test_stage_refusals(torch_cuda, oracle):
    """Each exchange is refused in the other's calls; PHASE_FINISH and PHASE_PREPARE are refused; so are a host tier and
    a table exported for remote reads."""
    from persia_b200 import native as N, shard as SH
    from persia_b200.worker import ShardedEmbeddingWorker as W, TierStager

    torch = torch_cuda
    R, dim = 2, 16
    pf = oracle.index_prefix(0)
    gpu_opt, _ = _optim(N, oracle, "SGD")
    ws = W.local_group(R, 1, dim, [pf], 256, cap=64, optimizer=gpu_opt, max_batch=64, tier_rows=1024)
    stagers = TierStager.local_group([x.shard for x in ws], 64)
    _warm(torch, ws)
    lib = N.load()
    ids = to_dev_ids(np.arange(8, dtype=np.uint64), DEV)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def stage(table, xchg, phases=0):
        return lib.pb_tier_stage_sharded(table, xchg, SH._ptr(ids), 8, SH._slot_offsets([0, 8], 1), SH._prefixes([pf]), 1,
                                         8, st, phases)

    assert stage(ws[0].shard.h, ws[0].h) == N.PB_ERR_INVALID  # a batch exchange
    assert b"stage" in lib.pb_last_error()
    for ph in (N.PHASE_FINISH, N.PHASE_PREPARE, N.PHASE_SEND | N.PHASE_FINISH):
        assert stage(ws[0].shard.h, stagers[0].h, ph) == N.PB_ERR_INVALID
    assert stage(ws[0].shard.host_tier.h, stagers[0].h) == N.PB_ERR_STATE  # a host tier
    out = torch.empty((1, 8, dim), dtype=torch.float16, device=DEV)
    assert lib.pb_forward_sharded(ws[0].shard.h, ws[0].ctx.h, stagers[0].h, SH._ptr(ids), 8, None,
                                  SH._slot_offsets([0, 8], 1), 8, 1, SH._ptr(out), st, 0) == N.PB_ERR_INVALID
    # a frozen export: untiered tables (a tiered one cannot be exported)
    plain = [SH.EmbeddingShard(dim, 256, 0) for _ in range(R)]
    for s in plain:
        s.set_optimizer(**gpu_opt)
        s.configure()
        s.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    pst = TierStager.local_group(plain, 64)
    plain[0].export_view()
    assert stage(plain[0].h, pst[0].h) == N.PB_ERR_STATE
    for x in ws + stagers + pst:
        assert x.status() == (False, False)
    _close(pst, stagers, ws)
    for s in plain:
        s.close()


# ---------------------------------------------------------------------------------------------- 9. two processes
def _rank_main(rank, world, port, result_dir):
    import torch
    import torch.distributed as dist

    import oracle
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker, TierStager

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    S, B, dim, C, card = 2, 256, 64, 512, [3000, 3000]
    pf = [oracle.index_prefix(i) for i in range(S)]
    wk = ShardedEmbeddingWorker.distributed(S, dim, pf, C, cap=S * B, device=dev, max_batch=B, tier_rows=1 << 14,
                                            optimizer=dict(kind=N.OPT_ADAGRAD, lr=0.02, initialization=0.01, eps=1e-10))
    wk.shard.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=1)
    stager = TierStager.distributed(wk.shard, S * B)
    rng = np.random.default_rng(43)
    batches = [[make_batch(rng, S, B, card)[0] for _ in range(world)] for _ in range(9)]  # every rank draws all
    so = [s * B for s in range(S + 1)]
    outs, seen = [], set()
    stager.stage(torch.from_numpy(batches[0][rank].view(np.int64)).to(dev), so, pf)
    for step in range(8):
        ids = batches[step]
        g = (rng.standard_normal((world, S, B, dim)) * 1e-2).astype(np.float16)
        out = wk.forward(torch.from_numpy(ids[rank].view(np.int64)).to(dev), B, training=True)
        stager.stage(torch.from_numpy(batches[step + 1][rank].view(np.int64)).to(dev), so, pf)
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
    assert found.all() and wk.status() == (False, False) and stager.status() == (False, False)
    assert wk.shard.stage_stats()["staged"] > 0
    np.savez(os.path.join(result_dir, f"rank{rank}.npz"), outs=np.stack(outs), signs=mine, ent=ent.cpu().numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_stage_two_processes_symmetric_memory(torch_cuda, oracle, tmp_path):
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
        batches = [[make_batch(rng, S, B, card)[0] for _ in range(world)] for _ in range(9)]
        res = [np.load(os.path.join(str(tmp_path), f"rank{r}.npz")) for r in range(world)]
        for step in range(8):
            ids = batches[step]
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
