"""GPU: staging a training request's host-tier moves one batch ahead (pb_tier_stage, pb_tier.cu k_tier_stage).  A stage
issued on a second stream right after forward(i), beside backward(i), runs the eviction check and the tier restores of
batch i+1; results equal the unstaged run's bit for bit, counters follow a host model of check -> stamped restores ->
train, and the library's ordering holds inside CUDA graphs."""
import os

import numpy as np
import pytest

from util import f16_ulp_diff, full_row_off, make_batch, same_bits, to_dev_i32, to_dev_ids

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


def _raw_batch(rng, B, card, max_ids):
    row_off = np.zeros(B + 1, np.uint32)
    row_off[1:] = np.cumsum(rng.integers(0, max_ids + 1, size=B))
    return rng.integers(0, card, size=int(row_off[-1]), dtype=np.uint64), row_off


def _tier_signs(s):
    return set(s._export_table(s.host_tier.h)[0].cpu().numpy().view(np.uint64).tolist())


def _hbm_signs(s):
    return set(s._export_table(s.h)[0].cpu().numpy().view(np.uint64).tolist())


def _stage(torch, s, side, ids, slot_off, prefixes):
    """pb_tier_stage on `side`, forked from the current stream (it runs beside what the current stream does next)."""
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        s.stage(to_dev_ids(ids, DEV), slot_off, prefixes)


# ---------------------------------------------------------------------------------------------- 1. parity over churn
PARITY = [("SGD", 16, {"lr": 0.1, "wd": 0.01}), ("ADAGRAD", 33, {"lr": 0.02, "init_acc": 0.01}),
          ("ADAGRAD_VW", 128, {"lr": 0.02}), ("ADAM", 33, {"lr": 0.001}), ("SGD", 128, {"lr": 0.05}),
          ("ADAM", 16, {"lr": 0.002})]


@pytest.mark.parametrize("kind_name,dim,kw", PARITY)
def test_stage_parity_over_churn(torch_cuda, pb, oracle, tmp_path, kind_name, dim, kw):
    """One seeded workload on fresh tables, unstaged and staged: HBM rows C = 2048 over ~4 C keys; three summation
    slots (slots 0 and 1 share a feature group; ragged multi-id steps) and a raw slot (a group of its own) share the
    table, one eviction check per request.  Staged: pb_tier_stage(i + 1) of the summation and raw ids on a second stream
    right after forward(i), beside backward(i).  Every step's outputs are bit-identical between the runs and equal the
    oracle's; every seen sign's entry and len() are equal; nothing dropped, export order and checkpoint bytes equal."""
    torch = torch_cuda
    from persia_b200 import checkpoint as CK

    kind = getattr(oracle, kind_name)
    C, T, fixed, S, B, RB, steps = 2048, 1 << 14, 3, 3, 64, 48, 30
    card, raw_card = [3000, 3000, 2500], 3000
    pf = [oracle.index_prefix(g) for g in (0, 0, 1)]
    rpf = oracle.index_prefix(2)
    rng = np.random.default_rng(100 + dim)
    plan = []  # the workload, drawn once
    for step in range(steps + 1):
        ids, row_off, slot_off = make_batch(rng, S, B, card, max_ids=3 if step % 2 else 1)
        f32 = step % 4 >= 2
        g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float32 if f32 else np.float16)
        rids, rro = _raw_batch(rng, RB, raw_card, 4)
        rg = (rng.standard_normal((len(rids), dim)) * 1e-2).astype(np.float32)
        plan.append((ids, row_off, slot_off, g, [128.0, 1.0, 2.0] if f32 else [1.0, 64.0, 1.0], rids, rro, rg))

    def stage_ids(k):
        ids, _, slot_off, _, _, rids, _, _ = plan[k]
        return np.concatenate([ids, rids]), list(slot_off) + [int(slot_off[-1]) + len(rids)], pf + [rpf]

    def run(staged, w=None, wr=None):
        s = pb.EmbeddingShard(dim, C, 0, tier_rows=T)
        s.set_optimizer(kind, **_optim_kw(kw))
        s.configure()
        s.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=2)
        ctx = pb.BatchContext(1 << 12, 1 << 12, pf)
        rctx = pb.BatchContext(1 << 12, 1 << 12, [rpf])
        side = torch.cuda.Stream()
        outs, seen = [], set()
        for step in range(steps):
            ids, row_off, slot_off, g, scale, rids, rro, rg = plan[step]
            ro_dev = to_dev_i32(row_off, DEV) if row_off is not None else None
            got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=ro_dev, training=True)
            if staged and step + 1 < steps:  # (a stage stamps the rows it moves: only batches that train are staged)
                _stage(torch, s, side, *stage_ids(step + 1))
            st = ctx.backward(s, [torch.from_numpy(g[i]).to(DEV) for i in range(S)], scales=scale, want_status=True)
            got = got.cpu().numpy()
            outs.append(got.tobytes())
            if w is not None:
                ro = row_off if row_off is not None else full_row_off(S, B)
                want, octx = w.forward(ids, ro, B, training=True)
                counts = np.diff(ro).reshape(S, B)
                for i in range(S):
                    one = counts[i] <= 1
                    np.testing.assert_array_equal(got[i][one].view(np.uint16), want[i][one].view(np.uint16),
                                                  err_msg=str(step))
                    assert f16_ulp_diff(got[i][~one], want[i][~one]) <= 1, step
                    seen.update(w.ctx_signs(octx, i).tolist())
                assert st.cpu().numpy().tolist() == w.backward(octx, [g[i] for i in range(S)], scale=scale), step
            table, index, _, _, cnt = rctx.forward_raw(s, to_dev_ids(rids, DEV), RB, fixed, row_off=to_dev_i32(rro, DEV))
            U = int(cnt[0])
            outs.append(table[:U + 1].cpu().numpy().tobytes() + index.cpu().numpy().tobytes())
            if wr is not None:
                wt, wi, _, _, rctx_o = wr.forward_raw(0, rids, rro, RB, training=True)
                assert table[:U + 1].cpu().numpy().tobytes() == wt.tobytes(), step
                np.testing.assert_array_equal(index.cpu().numpy(), wi)
                seen.update(oracle.add_prefix(rids, 8, rpf).tolist())
            rgu = rg[:U]
            rctx.backward_raw(s, torch.from_numpy(np.ascontiguousarray(rgu)).to(DEV) if U else None, scale=32.0)
            if wr is not None and U:
                assert wr.backward_raw(0, rctx_o, rgu, scale=32.0) == 0
        torch.cuda.synchronize()
        return s, outs, seen

    oracle.set_rsqrt_exact(True)
    try:
        w = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pf], n_ps=1)
        wr = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=rpf)], n_ps=1)
        for o in (w, wr):
            o.configure()
            o.set_optimizer(oracle.Optim(kind, **kw))
        s1, outs1, seen = run(True, w, wr)
        s0, outs0, _ = run(False)
    finally:
        oracle.set_rsqrt_exact(False)
    for k, (a, b) in enumerate(zip(outs0, outs1)):
        assert a == b, k
    sg = s1.stage_stats()
    assert sg["staged"] > 0, sg
    ts0, ts1 = s0.tier_stats(), s1.tier_stats()
    assert ts1["moved_out"] > C and ts1["restored"] > 0 and ts0["restored"] > 0, (ts0, ts1)
    assert ts0["refused"] == ts1["refused"] == 0 and s1.counters()["capacity_refused"] == 0
    signs = np.array(sorted(seen), np.uint64)
    e0, f0 = s0.get_entries(to_dev_ids(signs, DEV))
    e1, f1 = s1.get_entries(to_dev_ids(signs, DEV))
    assert bool(f0.all()) and bool(f1.all())
    assert e0.cpu().numpy().tobytes() == e1.cpu().numpy().tobytes()
    for k, sign in enumerate(signs):  # and the oracle's
        ref = next(r for r in (w.get_entry(int(sign)), wr.get_entry(int(sign))) if r is not None)
        assert same_bits(e1[k].cpu().numpy(), ref), int(sign)
    assert len(s0) == len(s1) == len(seen)
    if ts0["dropped"] == 0 and ts1["dropped"] == 0:
        a, ra = s0.export_signs()
        b, rb = s1.export_signs()
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
        assert ra.cpu().numpy().tobytes() == rb.cpu().numpy().tobytes()
        CK.dump_shards(str(tmp_path / "u"), [s0])
        CK.dump_shards(str(tmp_path / "s"), [s1])
        name = os.path.join("s0", "replica_0_shard_0.emb")
        assert open(tmp_path / "u" / name, "rb").read() == open(tmp_path / "s" / name, "rb").read()
    for s in (s0, s1):
        s.close()


# ---------------------------------------------------------------------------------------------- 2. what a stage moves
def _aged_out(torch, pb, oracle, C, keep):
    """X (40 signs) trained once, then aged out into the tier by three filler steps."""
    dim = 16
    s = pb.EmbeddingShard(dim, C, 0, tier_rows=1024)
    s.set_optimizer(oracle.SGD, lr=0.1)
    s.configure()
    s.set_eviction(check_every=1, low_water=C, target_free=C, keep_batches=keep)
    pf = oracle.index_prefix(0)
    ctx = pb.BatchContext(1 << 10, 1 << 10, [pf])

    def step(ids):
        ctx.forward(s, to_dev_ids(ids, DEV), [0, ids.size], ids.size, training=True)
        ctx.backward(s, [torch.full((ids.size, dim), 1e-3, dtype=torch.float16, device=DEV)])

    X = np.arange(40, dtype=np.uint64)
    step(X)
    for k in range(3):
        step(np.arange(1000 + 30 * k, 1030 + 30 * k, dtype=np.uint64))
    return s, ctx, pf, X, step


def test_stage_moves_what_it_should(torch_cuda, pb, oracle):
    """A stage of a batch holding X twice over and some HBM-held and unseen signs moves exactly X's distinct tier-held
    signs (host-computed) into HBM, counted in stage stats [0] and tier stats [2]; the forward that follows restores
    nothing, and its own check (keep_batches = 1, sweeping down to empty) leaves every staged row in HBM."""
    torch = torch_cuda
    C = 128
    s, ctx, pf, X, step = _aged_out(torch, pb, oracle, C, keep=1)
    xs = oracle.add_prefix(X, 8, pf)
    held = _tier_signs(s)
    assert set(xs.tolist()) <= held
    ids = np.concatenate([X, X[::-1], np.arange(1060, 1070, dtype=np.uint64), np.arange(7000, 7005, dtype=np.uint64)])
    want = len(set(oracle.add_prefix(ids, 8, pf).tolist()) & held)
    before = s.get_entries(to_dev_ids(xs, DEV))[0].cpu().numpy()
    r0 = s.tier_stats()["restored"]
    s.stage(to_dev_ids(ids, DEV), [0, ids.size], [pf])
    sg = s.stage_stats()
    assert sg == {"staged": want, "skipped": 0}, (sg, want)
    assert s.tier_stats()["restored"] - r0 == want
    assert set(xs.tolist()) <= _hbm_signs(s) and not (set(xs.tolist()) & _tier_signs(s))
    assert s.get_entries(to_dev_ids(xs, DEV))[0].cpu().numpy().tobytes() == before.tobytes()  # moved, not changed
    r1, m1 = s.tier_stats()["restored"], s.tier_stats()["moved_out"]
    ctx.forward(s, to_dev_ids(ids, DEV), [0, ids.size], ids.size, training=True)
    ts = s.tier_stats()
    assert ts["restored"] == r1, ts  # the forward restored nothing
    assert set(xs.tolist()) <= _hbm_signs(s)  # its own check (it ran: check_every = 1) kept the staged rows
    assert ts["moved_out"] >= m1
    assert s.counters()["capacity_refused"] == 0


# ---------------------------------------------------------------------------------------------- 3. no free rows
def test_stage_skips_when_pending_batches_hold_every_row(torch_cuda, pb, oracle):
    """Every HBM row protected by two pending training forwards: a stage of tier-held X finds no free row, counts every
    sign in stage stats [1] only, and leaves refused restores [4] and the tier entries as they were; the forward of X
    then behaves exactly as without the stage (zeros, X.size refused), and once the gradients came back the next
    request restores X with its values."""
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
    for k in range(3):
        f = np.arange(100 + 10 * k, 110 + 10 * k, dtype=np.uint64)
        _, _, o = fwd(ctxs[0], f)
        bwd(ctxs[0], o, 10, True)
    xs = oracle.add_prefix(X, 8, pf)
    assert set(xs.tolist()) <= _tier_signs(s)
    before = s.get_entries(to_dev_ids(xs, DEV))[0].cpu().numpy()
    _, _, oa = fwd(ctxs[0], np.arange(1000, 1030, dtype=np.uint64))
    nb = C - int(s.counters()["admitted"])
    _, _, ob = fwd(ctxs[1], np.arange(2000, 2000 + nb, dtype=np.uint64))
    assert s.counters()["admitted"] == C
    ts0, sg0 = s.tier_stats(), s.stage_stats()
    s.stage(to_dev_ids(X, DEV), [0, X.size], [pf])
    ts1, sg1 = s.tier_stats(), s.stage_stats()
    assert sg1["skipped"] - sg0["skipped"] == X.size and sg1["staged"] == sg0["staged"], (sg0, sg1)
    assert ts1 == ts0, (ts0, ts1)  # refused [4] included: nothing moved, nothing counted
    assert s.get_entries(to_dev_ids(xs, DEV))[0].cpu().numpy().tobytes() == before.tobytes()
    assert set(xs.tolist()) <= _tier_signs(s)
    got, want, oc = fwd(ctxs[2], X)
    assert not got.view(np.uint16).any()
    assert s.tier_stats()["refused"] - ts0["refused"] == X.size
    for ctx, o, B in ((ctxs[0], oa, 30), (ctxs[1], ob, nb), (ctxs[2], oc, 20)):
        bwd(ctx, o, B, False)
    after, found = s.get_entries(to_dev_ids(xs, DEV))
    assert found.all() and after.cpu().numpy().tobytes() == before.tobytes()
    got, want, o = fwd(ctxs[0], X)
    np.testing.assert_array_equal(got.view(np.uint16), want.view(np.uint16))
    bwd(ctxs[0], o, 20, True)


# ---------------------------------------------------------------------------------------------- 4. one clock
class StagedUnionModel:
    """The resident sets of an HBM table of C rows and its tier of T rows under pb_table_set_eviction's policy with a
    tier, with stages: check (keep = max(keep, pending + 1)) -> the stage's restores, each moved row stamped with the
    current batch number, a restore that finds no free row skipped -> the request's own check, batch number + 1, its
    restores and admissions."""

    def __init__(self, C, T, low, target, keep):
        self.C, self.T, self.low, self.target, self.keep = C, T, low, target, keep
        self.hbm, self.tier = {}, {}
        self.tick = self.moved = self.restored = self.dropped = self.staged = self.skipped = 0

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

    def stage(self, signs, pending):
        self.check(pending)
        want = [x for x in signs if x in self.tier]
        assert len(want) <= self.C - len(self.hbm), "the test's stage would skip in part (race-dependent)"
        for x in want:
            del self.tier[x]
            self.hbm[x] = self.tick
        self.staged += len(want)
        self.restored += len(want)

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


def test_stage_union_lru_matches_host_model(torch_cuda, pb, oracle):
    """C + T smaller than the key space, a stage of batch i + 1 beside every backward(i): the union holds exactly the
    signs and recencies the model keeps, and moved / restored / dropped and the stage counters equal the model's."""
    torch = torch_cuda
    C, T, dim, B, steps = 1024, 1536, 16, 160, 150
    s = pb.EmbeddingShard(dim, C, 0, tier_rows=T)
    s.set_optimizer(oracle.SGD, lr=0.05)
    s.configure()
    s.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=2)
    pf = oracle.index_prefix(0)
    ctx = pb.BatchContext(1 << 12, 1 << 12, [pf])
    side = torch.cuda.Stream()
    model = StagedUnionModel(C, T, C // 2, C // 2, 2)
    rng = np.random.default_rng(7)
    batches = [np.where(rng.random(B) < 0.5, rng.integers(0, 1500, size=B), rng.integers(0, 20000, size=B))
               .astype(np.uint64) for _ in range(steps + 1)]

    def distinct(ids):
        signs = oracle.add_prefix(ids, 8, pf)
        _, first = np.unique(signs, return_index=True)
        return [int(x) for x in signs[np.sort(first)]]

    for step in range(steps):
        ctx.forward(s, to_dev_ids(batches[step], DEV), [0, B], B, training=True)
        model.train(distinct(batches[step]))  # its own check: no batch pending
        _stage(torch, s, side, batches[step + 1], [0, B], [pf])
        model.stage(distinct(batches[step + 1]), pending=1)  # beside backward(step): one batch pending
        ctx.backward(s, [torch.zeros((B, dim), dtype=torch.float16, device=DEV)])
        if step % 10 == 9 or step == steps - 1:
            got_s, got_r = s.export_signs()
            got = dict(zip(got_s.cpu().numpy().view(np.uint64).tolist(),
                           (got_r.cpu().numpy().astype(np.int64) & 0xFFFFFFFF).tolist()))
            assert got == model.union(), step
            ts, sg = s.tier_stats(), s.stage_stats()
            assert (ts["moved_out"], ts["restored"], ts["dropped"]) == (model.moved, model.restored, model.dropped), \
                (step, ts, model.moved, model.restored, model.dropped)
            assert (sg["staged"], sg["skipped"]) == (model.staged, model.skipped), (step, sg, model.staged)
            assert ts["host_rows"] == len(model.tier) and s.counters()["admitted"] == len(model.hbm), step
    assert model.dropped > 0 and model.staged > 0


# ---------------------------------------------------------------------------------------------- 5. raw slots, pb_lookup
def test_stage_raw_slot_and_lookup_match_unstaged(torch_cuda, pb, oracle):
    """Two tables with one history of training lookups (most signs end up in the tier).  Staged ids of a raw slot, then
    pb_forward_raw, give the same table, index and rows as without the stage; so do staged signs (prefix 0) and a
    training pb_lookup."""
    torch = torch_cuda
    C, dim, fixed = 256, 16, 3
    rpf = oracle.index_prefix(1)
    shards = []
    for _ in range(2):
        s = pb.EmbeddingShard(dim, C, 0, tier_rows=4096)
        s.set_optimizer(oracle.ADAGRAD, lr=0.02, initialization=0.01)
        s.configure()
        s.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=1)
        shards.append(s)
    rng = np.random.default_rng(21)
    for _ in range(40):  # (requests small enough that no admission is ever refused: both histories are the same)
        signs = oracle.add_prefix(rng.integers(0, 1500, size=50, dtype=np.uint64), 8, rpf)
        for s in shards:
            s.lookup(to_dev_ids(signs, DEV), training=True)
    rids, rro = _raw_batch(rng, 30, 1500, 3)
    st0 = shards[1].stage_stats()["staged"]
    shards[1].stage(to_dev_ids(rids, DEV), [0, rids.size], [rpf])
    assert shards[1].stage_stats()["staged"] > st0
    res = []
    for s in shards:
        rctx = pb.BatchContext(1 << 10, 1 << 10, [rpf])
        table, index, non_empty, num, cnt = rctx.forward_raw(s, to_dev_ids(rids, DEV), 30, fixed,
                                                             row_off=to_dev_i32(rro, DEV))
        U = int(cnt[0])
        res.append((table[:U + 1].cpu().numpy().tobytes(), index.cpu().numpy().tobytes(),
                    non_empty[:int(cnt[1])].cpu().numpy().tobytes(), num.cpu().numpy().tobytes()))
        rctx.backward_raw(s, None)
        rctx.close()
    assert res[0] == res[1]
    signs = np.unique(oracle.add_prefix(rng.integers(0, 1500, size=60, dtype=np.uint64), 8, rpf))  # fits the free rows
    st1 = shards[1].stage_stats()["staged"]
    shards[1].stage(to_dev_ids(signs, DEV), [0, signs.size], [0])
    assert shards[1].stage_stats()["staged"] > st1
    outs = [s.lookup(to_dev_ids(signs, DEV), training=True).cpu().numpy().tobytes() for s in shards]
    assert outs[0] == outs[1]
    allk = np.array(sorted(set(shards[0].export_signs()[0].cpu().numpy().view(np.uint64).tolist())), np.uint64)
    e = [s.get_entries(to_dev_ids(allk, DEV))[0].cpu().numpy().tobytes() for s in shards]
    assert e[0] == e[1] and len(shards[0]) == len(shards[1])
    for s in shards:
        assert s.tier_stats()["refused"] == 0 and s.counters()["capacity_refused"] == 0


# ---------------------------------------------------------------------------------------------- 6. CUDA graph
def test_stage_in_a_cuda_graph(torch_cuda, pb, oracle):
    """forward(cur) -> fork pb_tier_stage(next) on a side stream || backward(cur) -> join, captured once and replayed 10
    times from a seeded state, equals the oracle.  A stage issued outside a capture that has not completed makes the
    first captured call fail with PB_ERR_STATE."""
    torch = torch_cuda
    from persia_b200 import native as N

    S, B, dim, C = 2, 256, 32, 2048
    card = [2000, 2000]
    pf = [oracle.index_prefix(g) for g in (0, 1)]
    oracle.set_rsqrt_exact(True)
    try:
        s = pb.EmbeddingShard(dim, C, 0, tier_rows=1 << 14)
        s.set_optimizer(oracle.ADAGRAD, lr=0.02, initialization=0.01)
        s.configure()
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
        seq = [make_batch(rng, S, B, card)[0] for _ in range(12)]
        cur, nxt = to_dev_ids(seq[0], DEV), to_dev_ids(seq[1], DEV)
        g_dev = torch.zeros((S, B, dim), dtype=torch.float16, device=DEV)
        out = torch.empty((S, B, dim), dtype=torch.float16, device=DEV)
        grads = [g_dev[i] for i in range(S)]
        stream, side = torch.cuda.Stream(), torch.cuda.Stream()

        def step():
            ctx.forward(s, cur, slot_off, B, training=True, out=out)
            side.wait_stream(stream)
            with torch.cuda.stream(side):
                s.stage(nxt, slot_off, pf)
            ctx.backward(s, grads)
            stream.wait_stream(side)

        with torch.cuda.stream(stream):
            step()  # warm-up: a real step, zero gradients
            stream.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=stream):
                step()
        oracle_step(seq[0], np.zeros((S, B, dim), np.float16))
        sg0, r0 = s.stage_stats()["staged"], s.tier_stats()["restored"]
        for it in range(10):
            g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
            cur.copy_(to_dev_ids(seq[it + 1], DEV))
            nxt.copy_(to_dev_ids(seq[it + 2], DEV))
            g_dev.copy_(torch.from_numpy(g).to(DEV))
            graph.replay()
            torch.cuda.synchronize()
            want = oracle_step(seq[it + 1], g)
            got = out.cpu().numpy()
            for i in range(S):
                np.testing.assert_array_equal(got[i].view(np.uint16), want[i].view(np.uint16), err_msg=str(it))
        signs = np.array(sorted(seen), np.uint64)
        ent, found = s.get_entries(to_dev_ids(signs, DEV))
        ent = ent.cpu().numpy()
        assert bool(found.all())
        for k, sign in enumerate(signs):
            assert same_bits(ent[k], w.get_entry(int(sign))), int(sign)
        assert len(s) == len(seen)
        assert s.stage_stats()["staged"] > sg0 and s.tier_stats()["restored"] > r0
        # a stage outside the capture, still running when the capture begins (a sleep ahead of it on its stream)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(200_000_000)
            s.stage(nxt, slot_off, pf)
        g2 = torch.cuda.CUDAGraph()
        with torch.cuda.stream(stream):
            g2.capture_begin()
            try:
                with pytest.raises(N.PersiaB200Error) as ei:
                    ctx.forward(s, cur, slot_off, B, training=True, out=out)
            finally:
                g2.capture_end()
        assert ei.value.code == N.PB_ERR_STATE, ei.value
        torch.cuda.synchronize()
        ctx.forward(s, cur, slot_off, B, training=True, out=out)  # outside a capture the same call waits and runs
        ctx.backward(s, grads)
        torch.cuda.synchronize()
    finally:
        oracle.set_rsqrt_exact(False)


# ---------------------------------------------------------------------------------------------- 7. no tier
def test_stage_without_a_tier_does_nothing(torch_cuda, pb, oracle):
    torch = torch_cuda
    from persia_b200 import native as N

    s = pb.EmbeddingShard(16, 256, 0)
    s.set_optimizer(oracle.SGD, lr=0.1)
    s.configure()
    s.set_eviction(check_every=1, low_water=128, target_free=128, keep_batches=1)
    signs = oracle.add_prefix(np.arange(300, dtype=np.uint64), 8, oracle.index_prefix(0))
    s.lookup(to_dev_ids(signs[:200], DEV), training=True)
    torch.cuda.synchronize()
    c0, n0 = s.counters(), N.load().pb_launch_count()
    s.stage(to_dev_ids(signs, DEV), [0, signs.size], [0])
    torch.cuda.synchronize()
    assert N.load().pb_launch_count() == n0 and s.counters() == c0
    assert s.stage_stats() == {"staged": 0, "skipped": 0} and s.tier_stats()["restored"] == 0


# ---------------------------------------------------------------------------------------------- 9. persia_core
CFG = {"feature_index_prefix_bit": 8,
       "slots_config": {"user": {"dim": 16}, "tags": {"dim": 16, "sqrt_scaling": True},
                        "hs": {"dim": 16, "hash_stack_config": {"hash_stack_rounds": 2, "embedding_size": 400}}}}


def _core_loop(tmp, monkeypatch, bypass):
    """A Forward-engine training loop (dataflow path, staleness 1) over a table of 2048 HBM rows and a tier; returns the
    outputs of every step, the entries of every sign, the checkpoint bytes and the stage counters."""
    import torch
    import torch.utils.dlpack as dl

    from persia_b200 import persia_core as impl

    monkeypatch.setenv("PERSIA_B200_CAPACITY", str(1 << 14))
    monkeypatch.setenv("PERSIA_B200_HBM_ROWS", "2048")  # (check every 4 requests, down to 256 free rows)
    if bypass:
        monkeypatch.setattr(impl, "_stage", lambda batch: None)
    impl.reset()
    pc = impl.install()
    fwd = None
    try:
        pc.set_embedding_config(CFG)
        ctx = pc.PersiaCommonContext(10, 0, 1, 0)
        opt = pc.optim.OptimizerBase()
        opt.init_adagrad(0.02, 0.0, 1.0, 0.01, 1e-10, False)
        opt.apply()
        ctx.configure_embedding_parameter_servers(-0.01, 0.01, 1.0, True, 10.0)
        bwd = pc.backward.Backward(8)  # not launched: updates apply in this thread, in step order
        B, steps, outs = 4, 150, []
        ch = pc.utils.PersiaBatchDataChannel(steps + 8)  # holds every batch: all are sent before training starts
        pc.nats.initialize_dataflow(1, ch.get_sender())
        fwd = pc.forward.Forward(8, True, 1)
        fwd.set_input_channel(ch.get_receiver())
        fwd.launch(1)
        rng = np.random.default_rng(31)
        for _ in range(steps):  # every batch sent ahead: batch i + 1 is staged while batch i trains
            b = pc.data.PersiaBatch()
            user = rng.integers(0, 3000, size=B, dtype=np.uint64)
            tags = [rng.integers(0, 3000, size=rng.integers(1, 4), dtype=np.uint64) for _ in range(B)]
            hs = rng.integers(0, 5000, size=B, dtype=np.uint64)
            b.add_id_type_feature_with_single_id(user, "user")
            b.add_id_type_feature(tags, "tags")
            b.add_id_type_feature_with_single_id(hs, "hs")
            b.add_non_id_type_feature(np.zeros((B, 1), np.float32), np.dtype(np.float32), "dense")
            b.add_label(np.zeros((B, 1), np.float32), np.dtype(np.float32), "y")
            b.converted_id_type_features2embedding_tensor(True)
            ctx.send_id_type_features_to_embedding_worker(b)
            ctx.send_non_id_type_features_to_nn_worker(b)
        for _ in range(steps):
            tb = fwd.get_batch(10000)
            embs = [e.get_sum_embedding() for e in tb.consume_all_id_type_feature_embedding_tensors()]
            gb = tb.create_gradient_batch()
            keep = []
            for t in embs:
                x = dl.from_dlpack(t.dlpack)
                outs.append(x.cpu().numpy().tobytes())
                gt = (x.float() * 0.5 + 1e-3).half().contiguous()
                keep.append(gt)
                gb.add_gradient(t.name, gt.data_ptr(), list(gt.shape), True, 1.0)
            torch.cuda.synchronize()
            bwd.update_id_type_feature_gradient_batched(gb)
            torch.cuda.synchronize()
        from persia_b200.persia_core import _S

        sh = _S.groups[16]["shard"]
        assert sh.host_tier is not None
        order = sh.export_signs()[0].cpu().numpy().view(np.uint64)
        ent = ctx.get_entries(order, 16)
        ctx.dump(str(tmp))
        with open(os.path.join(tmp, "s0", "replica_0_shard_0.emb"), "rb") as f:
            ck = f.read()
        assert sh.counters()["capacity_refused"] == 0 and sh.tier_stats()["refused"] == 0
        return outs, order.tobytes(), [e.tobytes() for e in ent], ck, sh.stage_stats(), sh.tier_stats()
    finally:
        if fwd is not None:
            fwd.shutdown()
        impl.reset()


def test_stage_through_persia_core(torch_cuda, tmp_path, monkeypatch):
    """The Forward engine stages every training batch of a group with a tier: trained with staging and with it
    bypassed, the outputs, entries and checkpoint are the same, and the staged loop staged rows."""
    a = _core_loop(tmp_path / "a", monkeypatch, bypass=False)
    b = _core_loop(tmp_path / "b", monkeypatch, bypass=True)
    assert a[4]["staged"] > 0 and b[4]["staged"] == 0, (a[4], b[4])
    assert a[5]["restored"] > 0 and b[5]["restored"] > 0
    assert a[0] == b[0]
    assert a[2] == b[2] and len(a[2]) == len(b[2])
    if a[5]["dropped"] == 0 and b[5]["dropped"] == 0:
        assert a[1] == b[1] and a[3] == b[3]
