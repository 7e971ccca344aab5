"""GPU: a table larger than HBM on one GPU — an HBM table with a host-memory tier behind it (pb_table_attach_tier,
pb_tier.cu).  Eviction checks move their victims into the tier, training requests move tier-held signs back first,
inference and direct updates use them where they are, and the union of the two tables behaves like one table of both capacities: values against an unbounded oracle bit for bit,
the resident set and the move counters against a host model of the batch-granular policy."""
import os

import numpy as np
import pytest

from util import (f16_ulp_diff, full_row_off, held_rows, make_batch, pool_model, same_bits, slot_signs, to_dev_i32,
                  to_dev_ids)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EV_BINS = 1024


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


@pytest.fixture(scope="module")
def pb(torch_cuda):
    from persia_b200 import shard

    return shard


def _optim_kw(kw):
    return {{"mom": "g_square_momentum", "init_acc": "initialization", "b1": "beta1", "b2": "beta2"}.get(k, k): v
            for k, v in kw.items()}


def _entries_match(s, ws, signs, what):
    """Every sign's whole entry, wherever it lives, equals the oracle's (NaN matches NaN)."""
    ent, found = s.get_entries(to_dev_ids(signs, DEV))
    ent, found = ent.cpu().numpy(), found.cpu().numpy()
    assert found.all(), (what, int((~found.astype(bool)).sum()))
    for k, sign in enumerate(signs):
        ref = next(r for r in (w.get_entry(int(sign)) for w in ws) if r is not None)
        assert same_bits(ent[k], ref), (what, k, int(sign))


def _raw_batch(rng, B, card, max_ids):
    row_off = np.zeros(B + 1, np.uint32)
    row_off[1:] = np.cumsum(rng.integers(0, max_ids + 1, size=B))
    return rng.integers(0, card, size=int(row_off[-1]), dtype=np.uint64), row_off


# ---------------------------------------------------------------------------------------------- 1. parity over churn
@pytest.mark.parametrize("kind_name,dim,kw", [("SGD", 16, {"lr": 0.1, "wd": 0.01}),
                                               ("ADAGRAD", 32, {"lr": 0.02, "init_acc": 0.01}),
                                               ("ADAGRAD_VW", 20, {"lr": 0.02}),
                                               ("ADAM", 24, {"lr": 0.001})])
def test_tier_parity_over_churn(torch_cuda, pb, oracle, kind_name, dim, kw):
    """HBM rows C = 2048 over a key space of ~4.4 C: two summation slots (their own feature groups; single-id and
    multi-id steps) and a raw slot (a third group) share the table, one eviction check per training request.  After every
    step the outputs and every entry seen equal the unbounded oracle's, and HBM + tier hold exactly the signs seen."""
    torch = torch_cuda
    kind = getattr(oracle, kind_name)
    C, T, fixed = 2048, 1 << 14, 3
    card = [3000, 3000]
    raw_card = 3000
    pf = [oracle.index_prefix(g) for g in (0, 1)]
    rpf = oracle.index_prefix(2)
    oracle.set_rsqrt_exact(True)
    try:
        s = pb.EmbeddingShard(dim, C, 0, tier_rows=T)
        s.set_optimizer(kind, **_optim_kw(kw))
        s.configure()
        # protected: the last three requests (<= 3 x 256 rows); the sweep frees down to C / 2
        s.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=2)
        ctx = pb.BatchContext(1 << 12, 1 << 12, pf)
        rctx = pb.BatchContext(1 << 12, 1 << 12, [rpf])
        w = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pf], n_ps=1)
        wr = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=rpf)], n_ps=1)
        for o in (w, wr):
            o.configure()
            o.set_optimizer(oracle.Optim(kind, **kw))
        rng = np.random.default_rng(dim)
        seen = set()
        for step in range(44):
            S, B = 2, 64
            ids, row_off, slot_off = make_batch(rng, S, B, card, max_ids=3 if step % 2 else 1)
            ro_dev = to_dev_i32(row_off, DEV) if row_off is not None else None
            got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=ro_dev, training=True).cpu().numpy()
            ro = row_off if row_off is not None else full_row_off(S, B)
            want, octx = w.forward(ids, ro, B, training=True)
            signs = slot_signs(oracle, ids, slot_off, pf)  # the forward admits and restores, it steps nothing
            model = pool_model(held_rows(torch, oracle, [s], signs), signs, row_off, B, None, dim=dim)
            counts = np.diff(ro).reshape(S, B)
            for i in range(S):
                assert same_bits(got[i], model[i]), step
                one = counts[i] <= 1  # a sample of several ids may differ by 1 f16 ulp: f32 sum order (test_gpu_parity)
                np.testing.assert_array_equal(got[i][one].view(np.uint16), want[i][one].view(np.uint16), err_msg=str(step))
                assert f16_ulp_diff(got[i][~one], want[i][~one]) <= 1, step
                seen.update(w.ctx_signs(octx, i).tolist())
            f32 = step % 4 >= 2
            scale = [128.0, 1.0] if f32 else [1.0, 64.0]
            g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float32 if f32 else np.float16)
            st = ctx.backward(s, [torch.from_numpy(g[i]).to(DEV) for i in range(S)], scales=scale, want_status=True)
            assert st.cpu().numpy().tolist() == w.backward(octx, [g[i] for i in range(S)], scale=scale), step
            # the raw slot: a request of its own on the same table
            rids, rro = _raw_batch(rng, 48, raw_card, 4)
            table, index, _, _, cnt = rctx.forward_raw(s, to_dev_ids(rids, DEV), 48, fixed, row_off=to_dev_i32(rro, DEV))
            U = int(cnt[0])
            wt, wi, _, _, rctx_o = wr.forward_raw(0, rids, rro, 48, training=True)
            assert table[:U + 1].cpu().numpy().tobytes() == wt.tobytes(), step
            np.testing.assert_array_equal(index.cpu().numpy(), wi)
            seen.update(oracle.add_prefix(rids, 8, rpf).tolist())
            rg = (rng.standard_normal((U, dim)) * 1e-2).astype(np.float32)
            rctx.backward_raw(s, torch.from_numpy(rg).to(DEV) if U else None, scale=32.0)
            if U:
                assert wr.backward_raw(0, rctx_o, rg, scale=32.0) == 0
            signs = np.array(sorted(seen), np.uint64)
            _entries_match(s, (w, wr), signs, step)
            assert len(s) == len(seen), (step, len(s), len(seen))
        ts = s.tier_stats()
        assert ts["moved_out"] > C and ts["restored"] > 0 and ts["dropped"] == 0 and ts["refused"] == 0, ts
        c = s.counters()
        assert c["capacity_refused"] == 0 and c["gradient_id_miss"] == 0 and c["wait_errors"] == 0, c
    finally:
        oracle.set_rsqrt_exact(False)


@pytest.mark.parametrize("kind_name,dim,kw", [("ADAGRAD", 16, {"lr": 0.02, "init_acc": 0.01, "eps": 1e-10}),
                                               ("SGD", 32, {"lr": 0.05, "wd": 0.001})])
def test_tier_parity_with_warm_signs(torch_cuda, pb, oracle, kind_name, dim, kw):
    """Three slots of cardinality 40, 3000 and 40000 at batch 200 over C = 2500 HBM rows and ~10^4 signs: slot 0's
    signs recur about 5 times per batch, so warm items go through restores too.  Every training forward starts with at
    least S x B free HBM rows.  Outputs and every entry seen equal the unbounded oracle's bit for bit."""
    torch = torch_cuda
    kind = getattr(oracle, kind_name)
    rng = np.random.default_rng(17 + dim)
    S, B, card, steps, C = 3, 200, [40, 3000, 40000], 40, 2500
    pf = [oracle.index_prefix(i) for i in range(S)]
    s = pb.EmbeddingShard(dim, C, 0, tier_rows=1 << 14)
    s.set_optimizer(kind, **_optim_kw(kw))
    s.configure()
    s.set_eviction(check_every=1, low_water=S * B, target_free=S * B, keep_batches=1)
    ctx = pb.BatchContext(4 * S * B, 4 * S * B, pf)
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf[i]) for i in range(S)], n_ps=1)  # never evicts
    w.configure()
    w.set_optimizer(oracle.Optim(kind, **kw))
    oracle.set_rsqrt_exact(True)
    try:
        seen = set()
        for step in range(steps):
            ids, _, slot_off = make_batch(rng, S, B, card)
            got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, training=True).cpu().numpy()
            want, octx = w.forward(ids, full_row_off(S, B), B, training=True)
            for i in range(S):
                assert got[i].tobytes() == want[i].tobytes(), (step, i)
                seen.update(w.ctx_signs(octx, i).tolist())
            g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
            ctx.backward(s, [torch.from_numpy(g[i]).to(DEV) for i in range(S)])
            w.backward(octx, [g[i] for i in range(S)])
        torch.cuda.synchronize()
        ts = s.tier_stats()
        assert len(seen) > 2 * C and ts["moved_out"] > 0 and ts["restored"] > 0, (len(seen), ts)
        assert ts["dropped"] == 0 and ts["refused"] == 0, ts
        assert len(s) == len(seen)  # every sign lives in exactly one of the two tables
        assert s.counters()["capacity_refused"] == 0
        signs = np.array(sorted(seen), np.uint64)
        ent, found = s.get_entries(to_dev_ids(signs, DEV))
        ent, found = ent.cpu().numpy(), found.cpu().numpy()
        assert found.all()
        for k, sign in enumerate(signs):
            assert ent[k].tobytes() == w.get_entry(int(sign)).tobytes(), int(sign)
    finally:
        oracle.set_rsqrt_exact(False)
        ctx.close()
        s.close()


# ---------------------------------------------------------------------------------------------- 2. union LRU
class UnionModel:
    """The resident sets of an HBM table of C rows and its tier of T rows under pb_table_set_eviction's policy with a
    tier (pb_index.cu launch_evict_tier): the HBM sweep picks its victims as without a tier; the tier drops its oldest
    entries (1024-bin age histogram, last bin clamped, ages >= 1) until it can hold them; they move over, keeping their
    recency.  A training request then restores its tier-held signs and admits its new ones."""

    def __init__(self, C, T, low, target, keep):
        self.C, self.T, self.low, self.target, self.keep = C, T, low, target, keep
        self.hbm, self.tier = {}, {}
        self.tick = self.moved = self.restored = self.dropped = 0

    def _threshold(self, table, want, keep):
        hist = np.zeros(EV_BINS, np.int64)
        for r in table.values():
            hist[min(self.tick - r, EV_BINS - 1)] += 1
        got, thr = 0, None
        for a in range(EV_BINS - 1, keep, -1):
            got += int(hist[a])
            thr = a
            if got >= want:
                break
        return thr if got else None

    def check(self, pending=0):
        free = self.C - len(self.hbm)
        if free >= self.low:
            return
        thr = self._threshold(self.hbm, self.target - free, max(self.keep, pending + 1))
        if thr is None:
            return
        victims = [s for s, r in self.hbm.items() if self.tick - r >= thr]
        tfree = self.T - len(self.tier)
        if len(victims) > tfree:
            tthr = self._threshold(self.tier, len(victims) - tfree, 0)
            if tthr is not None:
                gone = [s for s, r in self.tier.items() if self.tick - r >= tthr]
                for x in gone:
                    del self.tier[x]
                self.dropped += len(gone)
        assert len(victims) <= self.T - len(self.tier), "the test's policy would lose victims"
        for x in victims:
            self.tier[x] = self.hbm.pop(x)
        self.moved += len(victims)

    def train(self, signs, pending=0):
        self.check(pending)
        self.tick += 1
        need = [x for x in signs if x not in self.hbm]
        assert len(need) <= self.C - len(self.hbm), "the test's batch would be refused in part (race-dependent)"
        for x in signs:
            if x in self.tier:
                del self.tier[x]
                self.restored += 1
            self.hbm[x] = self.tick

    def union(self):
        u = dict(self.hbm)
        u.update(self.tier)
        return u


def test_tier_union_lru_matches_host_model(torch_cuda, pb, oracle):
    """C + T smaller than the key space: the union holds exactly the signs (and recencies) the model keeps, and the
    moved / restored / dropped counters equal the model's."""
    torch = torch_cuda
    C, T, dim = 1024, 1536, 16
    s = pb.EmbeddingShard(dim, C, 0, tier_rows=T)
    s.set_optimizer(oracle.SGD, lr=0.05)
    s.configure()
    s.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=2)
    pf = oracle.index_prefix(0)
    ctx = pb.BatchContext(1 << 12, 1 << 12, [pf])
    model = UnionModel(C, T, C // 2, C // 2, 2)
    rng = np.random.default_rng(7)
    for step in range(150):
        B = 160
        # a hot range that comes back often (restores) and a long tail (moves, tier drops)
        ids = np.where(rng.random(B) < 0.5, rng.integers(0, 1500, size=B), rng.integers(0, 20000, size=B)).astype(np.uint64)
        ctx.forward(s, to_dev_ids(ids, DEV), [0, B], B, training=True)
        ctx.backward(s, [torch.zeros((B, dim), dtype=torch.float16, device=DEV)])
        signs = oracle.add_prefix(ids, 8, pf)
        _, first = np.unique(signs, return_index=True)
        model.train([int(x) for x in signs[np.sort(first)]])
        if step % 10 == 9 or step == 149:
            got_s, got_r = s.export_signs()
            got = dict(zip(got_s.cpu().numpy().view(np.uint64).tolist(),
                           (got_r.cpu().numpy().astype(np.int64) & 0xFFFFFFFF).tolist()))
            assert got == model.union(), step
            ts = s.tier_stats()
            assert (ts["moved_out"], ts["restored"], ts["dropped"]) == (model.moved, model.restored, model.dropped), \
                (step, ts, model.moved, model.restored, model.dropped)
            assert ts["host_rows"] == len(model.tier) and s.counters()["admitted"] == len(model.hbm), step
    assert model.dropped > T and model.restored > 0


# ---------------------------------------------------------------------------------------------- 3. refused restore
def test_tier_refused_restore_keeps_the_entry(torch_cuda, pb, oracle):
    """A batch whose tier-held signs outnumber the free HBM rows: the refused ones read as zeros and are counted, their
    tier entries stay as they were, and a later step (with rows free again) brings them back with their values."""
    torch = torch_cuda
    C, dim = 128, 16
    s = pb.EmbeddingShard(dim, C, 0, tier_rows=1024)
    s.set_optimizer(oracle.SGD, lr=0.1)
    s.configure()
    s.set_eviction(check_every=1, low_water=C, target_free=C, keep_batches=1)
    pf = oracle.index_prefix(0)
    ctx = pb.BatchContext(1 << 10, 1 << 10, [pf])
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1))
    rng = np.random.default_rng(3)

    def step(ids, train_grad=True):
        B = ids.size
        got = ctx.forward(s, to_dev_ids(ids, DEV), [0, B], B, training=True).cpu().numpy()[0]
        want, octx = w.forward(ids, full_row_off(1, B), B, training=True)
        if train_grad:
            g = (rng.standard_normal((1, B, dim)) * 1e-2).astype(np.float16)
            ctx.backward(s, [torch.from_numpy(g[0]).to(DEV)])
            w.backward(octx, [g[0]])
        else:  # add_skipped_gradient: the rows stay as they are on both sides
            ctx.backward(s, [None])
            w.backward(octx, [np.zeros((B, dim), np.float16)], skip=[1])
        return got, want[0]

    X = np.arange(40, dtype=np.uint64)
    got, want = step(X)
    np.testing.assert_array_equal(got.view(np.uint16), want.view(np.uint16))
    for k in range(3):  # X ages out of HBM into the tier
        step(np.arange(1000 + 30 * k, 1030 + 30 * k, dtype=np.uint64))
    xs = oracle.add_prefix(X, 8, pf)
    tier_signs = set(s._export_table(s.host_tier.h)[0].cpu().numpy().view(np.uint64).tolist())
    assert set(xs.tolist()) <= tier_signs
    before, _ = s.get_entries(to_dev_ids(xs, DEV))
    before = before.cpu().numpy()
    # no more sweeps; fill HBM until 5 rows are free
    s.set_eviction(check_every=0)
    fill = C - 5 - int(s.counters()["admitted"])
    assert fill > 0
    step(np.arange(5000, 5000 + fill, dtype=np.uint64), train_grad=False)
    assert s.counters()["admitted"] == C - 5
    refused0 = s.tier_stats()["refused"]
    got, want = step(X, train_grad=False)
    zero = ~got.view(np.uint16).any(axis=1)
    assert int(zero.sum()) == 35 and s.tier_stats()["refused"] - refused0 == 35
    np.testing.assert_array_equal(got[~zero].view(np.uint16), want[~zero].view(np.uint16))
    assert s.counters()["admitted"] == C
    after, found = s.get_entries(to_dev_ids(xs, DEV))
    assert found.all() and after.cpu().numpy().tobytes() == before.tobytes()  # every entry, restored or not, unchanged
    assert len(s) == w.ps_len(0)
    # sweeps again: the fillers age out and X comes back with its values
    s.set_eviction(check_every=1, low_water=C, target_free=C, keep_batches=1)
    step(np.arange(9000, 9010, dtype=np.uint64))
    got, want = step(X)
    np.testing.assert_array_equal(got.view(np.uint16), want.view(np.uint16))
    _entries_match(s, (w,), xs, "after")


def test_tier_restore_refused_when_pending_batches_hold_every_row(torch_cuda, pb, oracle):
    """Every HBM row protected by the keep = max(keep, pending + 1) rule of two pending training forwards: a third
    training forward of tier-held signs finds no free row, reads them as zeros and counts them; once the gradients came
    back, the next request restores them with their values."""
    torch = torch_cuda
    C, dim = 64, 16
    s = pb.EmbeddingShard(dim, C, 0, tier_rows=1024)
    s.set_optimizer(oracle.SGD, lr=0.1)
    s.configure()
    s.set_eviction(check_every=1, low_water=C, target_free=C, keep_batches=1)
    pf = oracle.index_prefix(0)
    ctxs = [pb.BatchContext(1 << 9, 1 << 9, [pf]) for _ in range(3)]
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1))
    rng = np.random.default_rng(9)

    def fwd(ctx, ids):
        got = ctx.forward(s, to_dev_ids(ids, DEV), [0, ids.size], ids.size, training=True).cpu().numpy()[0]
        want, octx = w.forward(ids, full_row_off(1, ids.size), ids.size, training=True)
        return got, want[0], octx

    def bwd(ctx, octx, B, train):
        if train:
            g = (rng.standard_normal((B, dim)) * 1e-2).astype(np.float16)
            ctx.backward(s, [torch.from_numpy(g).to(DEV)])
            w.backward(octx, [g])
        else:
            ctx.backward(s, [None])
            w.backward(octx, [np.zeros((B, dim), np.float16)], skip=[1])

    X = np.arange(20, dtype=np.uint64)
    _, _, o = fwd(ctxs[0], X)
    bwd(ctxs[0], o, 20, True)
    for k in range(3):  # X ages out into the tier
        f = np.arange(100 + 10 * k, 110 + 10 * k, dtype=np.uint64)
        _, _, o = fwd(ctxs[0], f)
        bwd(ctxs[0], o, 10, True)
    xs = oracle.add_prefix(X, 8, pf)
    assert set(xs.tolist()) <= set(s._export_table(s.host_tier.h)[0].cpu().numpy().view(np.uint64).tolist())
    before = s.get_entries(to_dev_ids(xs, DEV))[0].cpu().numpy()
    # two pending forwards fill HBM; the pending rule protects every row from the checks of the next calls
    _, _, oa = fwd(ctxs[0], np.arange(1000, 1030, dtype=np.uint64))
    nb = C - int(s.counters()["admitted"])
    assert nb > 0
    _, _, ob = fwd(ctxs[1], np.arange(2000, 2000 + nb, dtype=np.uint64))
    assert s.counters()["admitted"] == C
    refused0 = s.tier_stats()["refused"]
    got, want, oc = fwd(ctxs[2], X)
    assert not got.view(np.uint16).any()  # every restore refused: zeros
    assert s.tier_stats()["refused"] - refused0 == X.size
    for ctx, o, B in ((ctxs[0], oa, 30), (ctxs[1], ob, nb), (ctxs[2], oc, 20)):
        bwd(ctx, o, B, False)
    after, found = s.get_entries(to_dev_ids(xs, DEV))
    assert found.all() and after.cpu().numpy().tobytes() == before.tobytes()
    got, want, o = fwd(ctxs[0], X)  # no batch pending: the check frees rows, X comes back with its values
    np.testing.assert_array_equal(got.view(np.uint16), want.view(np.uint16))
    bwd(ctxs[0], o, 20, True)
    _entries_match(s, (w,), xs, "after")


def test_tier_inference_and_direct_update_read_in_place(torch_cuda, pb, oracle):
    """One inference pass over far more tier-held signs than HBM has free rows — pb_forward (single- and multi-id),
    pb_lookup and a raw slot — returns the oracle's values and moves nothing; pb_update steps tier-held rows where they
    are, as the oracle's update_gradient_mixed does."""
    torch = torch_cuda
    C, dim, fixed = 256, 16, 3
    s = pb.EmbeddingShard(dim, C, 0, tier_rows=1 << 13)
    s.set_optimizer(oracle.SGD, lr=0.1, wd=0.01)
    s.configure()
    s.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=1)
    pf, rpf = oracle.index_prefix(0), oracle.index_prefix(1)
    ctx = pb.BatchContext(1 << 13, 1 << 13, [pf])
    rctx = pb.BatchContext(1 << 13, 1 << 13, [rpf])
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf)], n_ps=1)
    wr = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=rpf)], n_ps=1)
    for o in (w, wr):
        o.configure()
        o.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1, wd=0.01))
    rng = np.random.default_rng(13)
    card = 2000
    for step in range(40):  # train over 2000 keys per group: most end up in the tier
        ids = rng.integers(0, card, size=64, dtype=np.uint64)
        ctx.forward(s, to_dev_ids(ids, DEV), [0, 64], 64, training=True)
        _, octx = w.forward(ids, full_row_off(1, 64), 64, training=True)
        g = (rng.standard_normal((64, dim)) * 1e-2).astype(np.float16)
        ctx.backward(s, [torch.from_numpy(g).to(DEV)])
        w.backward(octx, [g])
        rids, rro = _raw_batch(rng, 32, card, 3)
        _, _, _, _, cnt = rctx.forward_raw(s, to_dev_ids(rids, DEV), 32, fixed, row_off=to_dev_i32(rro, DEV))
        _, _, _, _, ro = wr.forward_raw(0, rids, rro, 32, training=True)
        U = int(cnt[0])
        rg = (rng.standard_normal((U, dim)) * 1e-2).astype(np.float32)
        rctx.backward_raw(s, torch.from_numpy(rg).to(DEV) if U else None)
        if U:
            wr.backward_raw(0, ro, rg)
    tier_signs = set(s._export_table(s.host_tier.h)[0].cpu().numpy().view(np.uint64).tolist())
    free = C - int(s.counters()["admitted"])
    st0 = s.tier_stats()
    # summation slot, single-id then multi-id: every id of the batch a tier-held sign
    held = np.array(sorted(x - pf for x in tier_signs if (x >> 56) == (pf >> 56)), np.uint64)
    assert held.size > 4 * free, (held.size, free)
    B = held.size
    got = ctx.forward(s, to_dev_ids(held, DEV), [0, B], B, training=False).cpu().numpy()[0]
    want, _ = w.forward(held, full_row_off(1, B), B, training=False)
    np.testing.assert_array_equal(got.view(np.uint16), want[0].view(np.uint16))
    ids, row_off, slot_off = make_batch(rng, 1, 300, card, max_ids=4)
    got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, 300, row_off=to_dev_i32(row_off, DEV), training=False)
    want, _ = w.forward(ids, row_off, 300, training=False)
    signs = oracle.add_prefix(ids, 8, pf)  # tier-held signs read in place: the model reads them from the tier too
    model = pool_model(held_rows(torch, oracle, [s], signs), signs, row_off, 300, None, dim=dim)
    assert same_bits(got.cpu().numpy()[0], model[0])
    assert f16_ulp_diff(got.cpu().numpy()[0], want[0]) <= 1
    # pb_lookup
    signs = oracle.add_prefix(held, 8, pf)
    got = s.lookup(to_dev_ids(signs, DEV), training=False).cpu().numpy().reshape(-1)
    assert got.tobytes() == w.ps_lookup(0, signs, np.full(signs.size, dim, np.uint32), False).tobytes()
    # raw slot
    rids, rro = _raw_batch(rng, 400, card, 3)
    table, index, _, _, cnt = rctx.forward_raw(s, to_dev_ids(rids, DEV), 400, fixed, row_off=to_dev_i32(rro, DEV),
                                               training=False)
    wt, wi, _, _, _ = wr.forward_raw(0, rids, rro, 400, training=False)
    assert table[:int(cnt[0]) + 1].cpu().numpy().tobytes() == wt.tobytes()
    np.testing.assert_array_equal(index.cpu().numpy(), wi)
    st1 = s.tier_stats()
    assert (st1["restored"], st1["moved_out"], st1["refused"]) == (st0["restored"], st0["moved_out"], st0["refused"])
    # pb_update: tier-held rows stepped in place, an HBM-held one and an absent one alongside
    upd = np.concatenate([signs[:500], np.array([int(oracle.add_prefix(np.array([10**9], np.uint64), 8, pf)[0])],
                                                 np.uint64)])
    grads = (rng.standard_normal((upd.size, dim)) * 1e-2).astype(np.float32)
    gm0 = s.counters()["gradient_id_miss"]
    s.update(to_dev_ids(upd, DEV), torch.from_numpy(grads).to(DEV))
    w.ps_update(0, upd, np.full(upd.size, dim, np.uint32), grads.reshape(-1))
    assert s.counters()["gradient_id_miss"] - gm0 == 1  # only the absent sign
    _entries_match(s, (w,), upd[:500], "update")
    assert s.tier_stats()["restored"] == st0["restored"]


# ---------------------------------------------------------------------------------------------- 4. tier index churn
def test_tier_index_churn_keeps_empty_cells(torch_cuda, pb, oracle):
    """60+ turnovers of the tier: every eviction check rebuilds the tier's index too, so its EMPTY cells never run out
    (tests/test_gpu_index_churn.py does the same for an HBM table)."""
    torch = torch_cuda
    C, T, dim, B = 1024, 512, 8, 300
    s = pb.EmbeddingShard(dim, C, 0, tier_rows=T)
    s.set_optimizer(oracle.SGD, lr=0.05)
    s.configure()
    s.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=1)
    nc = 1024  # index cells of a 512-row table: next_pow2(max(1024, 1.5 x 512))
    nxt = 1 << 32
    for step in range(130):
        signs = np.arange(nxt, nxt + B, dtype=np.uint64)  # fresh signs only
        nxt += B
        s.lookup(to_dev_ids(signs, DEV), training=True)
        st = s.host_tier.index_stats()
        ts = s.tier_stats()
        assert st["live"] == ts["host_rows"] and st["live"] + st["tomb"] + st["empty"] == nc, (step, st, ts)
        assert st["empty"] >= nc // 8, (step, st)  # the check's moves come before its rebuild decision
        assert len(s) == B * (step + 1) - ts["dropped"], step
    ts = s.tier_stats()
    assert ts["dropped"] >= 60 * T and ts["refused"] == 0, ts
    # tier entries still hold their initial rows (nothing trains them)
    keep_s, _ = s._export_table(s.host_tier.h)
    keep_s = keep_s.cpu().numpy().view(np.uint64)[:64]
    ent, found = s.get_entries(to_dev_ids(keep_s, DEV))
    assert found.all()
    for k, sign in enumerate(keep_s):
        assert ent[k, :dim].cpu().numpy().tobytes() == oracle.init_row(int(sign), dim, -0.01, 0.01).tobytes()


# ---------------------------------------------------------------------------------------------- 5. graph capture
def test_tier_step_in_a_cuda_graph(torch_cuda, pb, oracle):
    """A training step with a tier attached — eviction check with moves, restores, forward, backward — captured once and
    replayed 10 times from a seeded state equals the oracle: nothing in it waits on the host."""
    torch = torch_cuda
    S, B, dim, C = 2, 256, 32, 2048
    card = [2000, 2000]
    pf = [oracle.index_prefix(g) for g in (0, 1)]
    oracle.set_rsqrt_exact(True)
    try:
        s = pb.EmbeddingShard(dim, C, 0, tier_rows=1 << 14)
        s.set_optimizer(oracle.ADAGRAD, lr=0.02, initialization=0.01)
        s.configure()
        # protected: the last two requests (<= 2 x 512 rows); the sweep frees down to C / 2
        s.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=1)
        ctx = pb.BatchContext(S * B, S * B, pf)
        w = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pf], n_ps=1)
        w.configure()
        w.set_optimizer(oracle.Optim(oracle.ADAGRAD, lr=0.02, init_acc=0.01))
        rng = np.random.default_rng(11)
        seen = set()

        def oracle_step(ids_np, g):
            want, octx = w.forward(ids_np, full_row_off(S, B), B, training=True)
            for i in range(S):
                seen.update(w.ctx_signs(octx, i).tolist())
            w.backward(octx, [g[i] for i in range(S)])
            return want

        for _ in range(6):  # seeded state: rows already in the tier
            ids_np, _, slot_off = make_batch(rng, S, B, card)
            g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
            ctx.forward(s, to_dev_ids(ids_np, DEV), slot_off, B, training=True)
            ctx.backward(s, [torch.from_numpy(g[i]).to(DEV) for i in range(S)])
            oracle_step(ids_np, g)
        assert s.tier_stats()["moved_out"] > 0
        ids_np, _, slot_off = make_batch(rng, S, B, card)
        ids_dev = to_dev_ids(ids_np, DEV)
        g_dev = torch.zeros((S, B, dim), dtype=torch.float16, device=DEV)
        out = torch.empty((S, B, dim), dtype=torch.float16, device=DEV)
        grads = [g_dev[i] for i in range(S)]
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            ctx.forward(s, ids_dev, slot_off, B, training=True, out=out)  # warm-up: a real step, zero gradients
            ctx.backward(s, grads)
            stream.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=stream):
                ctx.forward(s, ids_dev, slot_off, B, training=True, out=out)
                ctx.backward(s, grads)
        oracle_step(ids_np, np.zeros((S, B, dim), np.float16))
        restored0 = s.tier_stats()["restored"]
        for it in range(10):
            ids_np, _, _ = make_batch(rng, S, B, card)
            g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
            ids_dev.copy_(to_dev_ids(ids_np, DEV))
            g_dev.copy_(torch.from_numpy(g).to(DEV))
            graph.replay()
            torch.cuda.synchronize()
            want = oracle_step(ids_np, g)
            got = out.cpu().numpy()
            for i in range(S):
                np.testing.assert_array_equal(got[i].view(np.uint16), want[i].view(np.uint16), err_msg=str(it))
        _entries_match(s, (w,), np.array(sorted(seen), np.uint64), "replays")
        assert len(s) == len(seen)
        assert s.tier_stats()["restored"] > restored0  # the replays moved rows both ways
    finally:
        oracle.set_rsqrt_exact(False)


# ---------------------------------------------------------------------------------------------- 6. persia_core surface
CFG = {"feature_index_prefix_bit": 8,
       "slots_config": {"user": {"dim": 16}, "tags": {"dim": 16, "sqrt_scaling": True}}}


def test_tier_through_persia_core(torch_cuda, oracle, tmp_path, monkeypatch):
    """PERSIA_B200_HBM_ROWS below the capacity: the surface trains against the oracle with most rows in host memory;
    get_embedding_size counts both tables; an inference lookup of a tier-held sign returns its value; a dump ->
    clear_embeddings -> load round trip returns every entry; set_embedding places more rows than HBM holds."""
    import torch
    import torch.utils.dlpack as dl

    from persia_b200 import checkpoint as CK
    from persia_b200 import persia_core as impl
    from persia_b200.persia_core import parse_embedding_config

    hbm = 1024
    monkeypatch.setenv("PERSIA_B200_CAPACITY", str(1 << 16))
    monkeypatch.setenv("PERSIA_B200_HBM_ROWS", str(hbm))
    impl.reset()
    pc = impl.install()
    try:
        pc.set_embedding_config(CFG)
        ctx = pc.PersiaCommonContext(10, 0, 1, 0)
        opt = pc.optim.OptimizerBase()
        opt.init_sgd(0.05, 0.0)
        opt.apply()
        ctx.configure_embedding_parameter_servers(-0.01, 0.01, 1.0, True, 10.0)
        bwd = pc.backward.Backward(8)  # not launched: updates apply in this thread, in step order
        _, slots = parse_embedding_config(CFG)
        by = {x.name: x for x in slots}
        w = oracle.Worker([oracle.SlotCfg(16, sqrt_scaling=x.sqrt_scaling, prefix=x.index_prefix) for x in slots], n_ps=1)
        w.configure(-0.01, 0.01, 1.0, True, 10.0)
        w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.05, wd=0.0))
        rng = np.random.default_rng(5)
        B, seen = 8, set()

        def batch(user, tags, training=True):
            b = pc.data.PersiaBatch()
            b.add_id_type_feature_with_single_id(user, "user")
            b.add_id_type_feature(tags, "tags")
            b.add_label(np.zeros((B, 1), np.float32), np.dtype(np.float32), "y")
            b.converted_id_type_features2embedding_tensor(training)
            return b

        def csr(user, tags):
            rows = [np.array([x], np.uint64) for x in user] + tags
            off = np.zeros(len(rows) + 1, np.uint32)
            off[1:] = np.cumsum([len(r) for r in rows])
            return np.concatenate(rows), off

        def compare(tb, user, tags, training):
            embs = {t.name: t for t in (e.get_sum_embedding() for e in tb.consume_all_id_type_feature_embedding_tensors())}
            ids, off = csr(user, tags)
            want, octx = w.forward(ids, off, B, training=training)
            # rows after the forward (it admits and restores, it steps nothing), wherever they live
            signs = np.concatenate([oracle.add_prefix(np.array(user, np.uint64), 8, by["user"].index_prefix),
                                    oracle.add_prefix(ids[B:], 8, by["tags"].index_prefix)])
            torch.cuda.synchronize()
            ent = ctx.get_entries(signs, 16, missing_ok=True)
            rows = {int(x): e[:16] for x, e in zip(signs, ent) if e is not None}
            model = pool_model(rows, signs, off, B, [by["user"].sqrt_scaling, by["tags"].sqrt_scaling], dim=16)
            xs = {}
            for k, n in enumerate(("user", "tags")):
                t = embs[n]
                x = dl.from_dlpack(t.dlpack)
                got = x.cpu().numpy()
                if n == "user":
                    np.testing.assert_array_equal(got.view(np.uint16), want[k].view(np.uint16))
                else:  # several ids per sample: 1 f16 ulp of f32 sum order (test_gpu_parity)
                    assert f16_ulp_diff(got, want[k]) <= 1
                assert same_bits(got, model[k]), n
                xs[n] = (t, x)
            return xs, octx

        for step in range(90):
            user = rng.integers(0, 1500, size=B, dtype=np.uint64)
            tags = [rng.integers(0, 1500, size=rng.integers(1, 4), dtype=np.uint64) for _ in range(B)]
            tb = ctx.get_embedding_from_data(batch(user, tags), 0)
            xs, octx = compare(tb, user, tags, True)
            for k in range(2):
                seen.update(w.ctx_signs(octx, k).tolist())
            gs = {n: (rng.standard_normal((B, 16)) * 1e-2).astype(np.float16) for n in xs}
            gb = tb.create_gradient_batch()
            keep = []
            for n in xs:
                gt = torch.from_numpy(gs[n]).to(DEV)
                keep.append(gt)
                gb.add_gradient(n, gt.data_ptr(), list(gt.shape), True, 1.0)
            torch.cuda.synchronize()
            bwd.update_id_type_feature_gradient_batched(gb)
            torch.cuda.synchronize()
            w.backward(octx, [gs["user"], gs["tags"]])
        from persia_b200.persia_core import _S

        sh = _S.groups[16]["shard"]
        assert sh.capacity == hbm and sh.host_tier is not None and sh.host_tier.capacity == (1 << 16) - hbm
        assert ctx.get_embedding_size() == [len(seen)] == [w.ps_len(0)]
        assert sh.tier_stats()["host_rows"] > 0 and sh.tier_stats()["restored"] > 0
        signs = np.array(sorted(seen), np.uint64)
        got = ctx.get_entries(signs, 16)
        for k, x in enumerate(signs):
            assert got[k].tobytes() == w.get_entry(int(x)).tobytes()
        # an eval-style (training = false) lookup of tier-held signs returns their values
        tier_signs = sh._export_table(sh.host_tier.h)[0].cpu().numpy().view(np.uint64)
        pu = np.uint64(by["user"].index_prefix)
        user = (tier_signs[(tier_signs >> np.uint64(56)) == (pu >> np.uint64(56))] - pu)[:B]
        assert user.size == B
        tags = [np.array([1], np.uint64)] * B
        tb = ctx.get_embedding_from_data(batch(user, tags, training=False), 0)
        compare(tb, user, tags, False)
        # dump -> clear -> load: every entry comes back; the file lists both tables oldest first
        order, _ = sh.export_signs()
        order = order.cpu().numpy().view(np.uint64)
        ctx.dump(str(tmp_path))
        with open(os.path.join(tmp_path, "s0", "replica_0_shard_0.emb"), "rb") as f:
            fsigns, _, fent = CK.decode_list(f.read())
        np.testing.assert_array_equal(fsigns, order)
        ctx.clear_embeddings()
        assert ctx.get_embedding_size() == [0] and sh.tier_stats()["host_rows"] == 0
        ctx.load(str(tmp_path))
        assert ctx.get_embedding_size() == [len(seen)]
        again = ctx.get_entries(fsigns, 16)
        for k in range(fsigns.size):
            assert again[k].tobytes() == fent[k].tobytes()
        # set_embedding of more rows than HBM holds: the overflow goes to the tier
        ctx.clear_embeddings()
        n = 3 * hbm
        new = oracle.add_prefix(np.arange(n, dtype=np.uint64), 8, by["user"].index_prefix)
        vals = rng.standard_normal((n, 16)).astype(np.float32)
        ctx.set_embedding([(int(new[k]), vals[k], np.zeros(0, np.float32)) for k in range(n)])
        assert ctx.get_embedding_size() == [n] and sh.tier_stats()["host_rows"] == n - hbm
        assert sh.counters()["capacity_refused"] == 0 and sh.tier_stats()["dropped"] == 0  # stored, not refused
        back = ctx.get_entries(new, 16)
        assert np.asarray(back).tobytes() == vals.tobytes()
    finally:
        impl.reset()
