"""GPU: the shard's hash index under long eviction churn, against a host model of the batch-granular capacity policy.

The index (pb_probe.cuh, pb_index.cu) decides which row a sign gets: probing, admission into EMPTY cells and tombstones,
the capacity sweep, the free-row stack and the rebuild that drops tombstones.  The model below restates what of it is
deterministic: the resident set, each sign's recency (the training-request number export_signs returns) and the
counters.  It does not model the cell layout, which depends on races.  Its sweep is maybe_evict + k_evict_*: every
check_every-th training call, before the call's batch number is bumped, if fewer than low_water rows are free, the
oldest rows are released until target_free are, walking a 1024-bin age histogram (last bin clamped) oldest first and
never releasing ages <= max(keep, pending batches + 1).

Which signs of a batch are refused when its new signs exceed the free rows is race-dependent, so the churn tests use
batches and policies that never refuse.  Values are compared with an unbounded oracle bit for bit; a sign the model
evicted and the GPU re-admits starts again from its initial entry, which is seeded by the sign, so the oracle's entry
is reset to init_row(sign) ++ initial state at that point.  Tables stay at capacity <= 8192 (<= 2048 buckets)."""
import numpy as np
import pytest

from hash_set_keys import mix64
from util import full_row_off, to_dev_i32, to_dev_ids

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
M64 = (1 << 64) - 1
EV_BINS = 1024
LO, HI = -0.01, 0.01


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def n_cells(cap):
    want = max(1024, cap + cap // 2)
    return 1 << (want - 1).bit_length()


class IndexModel:
    """Resident set, recency and counters of one table under pb_table_set_eviction's policy."""

    def __init__(self, capacity, check_every=0, low=0, target=0, keep=2):
        self.cap, self.every, self.low, self.target, self.keep = capacity, check_every, low, target, keep
        self.res = {}      # sign -> batch number of its last training use
        self.gone = set()  # signs evicted at least once
        self.tick = self.calls = self.evicted = 0

    def sweep(self, pending=0):
        free = self.cap - len(self.res)
        if free >= self.low:
            return []
        want = self.target - free
        hist = np.zeros(EV_BINS, np.int64)
        for r in self.res.values():
            hist[min(self.tick - r, EV_BINS - 1)] += 1
        keep = max(self.keep, pending + 1)
        got, thr = 0, None
        for a in range(EV_BINS - 1, keep, -1):
            got += int(hist[a])
            thr = a
            if got >= want:
                break
        if not got:
            return []
        out = [s for s, r in self.res.items() if self.tick - r >= thr]
        for s in out:
            del self.res[s]
        self.gone.update(out)
        self.evicted += len(out)
        return out

    def train(self, signs, pending=0):
        """One training request over its distinct signs.  Returns (newly admitted signs, signs re-admitted after an
        eviction, whether an eviction check ran)."""
        checked = False
        if self.every:
            self.calls += 1
            if self.calls % self.every == 0:
                self.sweep(pending)
                checked = True
        self.tick += 1
        new = [s for s in signs if s not in self.res]
        assert len(new) <= self.cap - len(self.res), "the test's batch would be refused in part (race-dependent)"
        for s in signs:
            self.res[s] = self.tick
        back = [s for s in new if s in self.gone]
        return new, back, checked

    def export(self):
        return np.array(list(self.res), np.uint64), np.array(list(self.res.values()), np.int64)


def by_recency(s, r):
    o = np.lexsort((s, r))
    return s[o], r[o]


def check_export(shard, model, what):
    s, r = shard.export_signs()
    s, r = by_recency(s.cpu().numpy().view(np.uint64), r.cpu().numpy().astype(np.int64) & 0xFFFFFFFF)
    ms, mr = by_recency(*model.export())
    assert np.unique(s).size == s.size, (what, "a sign sits in two cells")
    assert s.size == ms.size, (what, s.size, ms.size)
    np.testing.assert_array_equal(s, ms, err_msg=str(what))
    np.testing.assert_array_equal(r, mr, err_msg=str(what))


def check_stats(shard, model, fresh, what):
    """Live cells equal the model's resident signs, and at least n_cells / 8 cells were EMPTY after the last eviction
    check: `fresh` = signs admitted since (each used up at most one EMPTY cell)."""
    st = shard.index_stats()
    nc = n_cells(shard.capacity)
    assert st["live"] == len(model.res), (what, st)
    assert st["live"] + st["tomb"] + st["empty"] == nc, (what, st)
    assert st["empty"] + fresh >= nc // 8, (what, st, fresh)
    return st


def check_counters(shard, model, what, misses=0):
    """misses: lookups of absent signs the test made on purpose (inference lookups, get_entries)."""
    c = shard.counters()
    assert c["capacity_refused"] == 0 and c["lookup_miss"] == misses and c["gradient_id_miss"] == 0, (what, c)
    assert c["admitted"] == len(model.res), (what, c, len(model.res))


def check_entries(shard, w, model, what):
    signs = np.array(sorted(model.res), np.uint64)
    ent, found = shard.get_entries(to_dev_ids(signs, DEV))
    ent, found = ent.cpu().numpy(), found.cpu().numpy()
    assert found.all(), what
    for k, sign in enumerate(signs):
        ref = w.get_entry(int(sign))
        assert ref is not None and ent[k].tobytes() == ref.tobytes(), (what, k, int(sign))


def reset_oracle(oracle, w, opt, signs, dim):
    """A re-admitted sign starts from its initial entry (seeded by the sign)."""
    if signs:
        ent = np.stack([opt.new_entry(oracle.init_row(int(s), dim, LO, HI)) for s in signs])
        w.set_embedding(np.array(signs, np.uint64), ent, dim)


def optim_pair(oracle, kind):
    if kind == oracle.SGD:
        return dict(lr=0.05, wd=0.001), oracle.Optim(oracle.SGD, lr=0.05, wd=0.001)
    return dict(lr=0.02, initialization=0.01, eps=1e-10), oracle.Optim(oracle.ADAGRAD, lr=0.02, init_acc=0.01, eps=1e-10)


def new_shard(pb, oracle, dim, cap, kind, tier_rows=0):
    gpu, cpu = optim_pair(oracle, kind)
    s = pb.EmbeddingShard(dim, cap, 0, tier_rows=tier_rows)
    s.set_optimizer(kind, **gpu)
    s.configure(init_lower=LO, init_upper=HI)
    return s, cpu


class Churn:
    """Request k: `fresh` never-seen signs, the whole hot set, and `warm` draws from a re-used pool (evicted and
    re-admitted as the table turns over).  Distinct signs per request <= fresh + hot + warm."""

    def __init__(self, rng, base, fresh, n_hot, n_warm_pool, warm):
        self.rng, self.next, self.fresh, self.warm = rng, base, fresh, warm
        self.hot = np.arange(n_hot, dtype=np.uint64) + np.uint64(base + (1 << 40))
        self.pool = np.arange(n_warm_pool, dtype=np.uint64) + np.uint64(base + (1 << 41))

    def ids(self):
        f = np.arange(self.fresh, dtype=np.uint64) + np.uint64(self.next)
        self.next += self.fresh
        w = self.rng.choice(self.pool, size=self.warm, replace=True)
        q = np.concatenate([f, self.hot, w, self.hot[: len(self.hot) // 2]])  # hot signs repeat inside a request
        self.rng.shuffle(q)
        return q


def distinct_in_order(a):
    _, i = np.unique(a, return_index=True)
    return [int(x) for x in a[np.sort(i)]]


# ---- long churn through the three probing kernels ------------------------------------------------------------------
CHURN = [  # (path, capacity, optimizer, dim): load 1/2 and 2/3 of the index, SGD and Adagrad, dims 8 and 64
    ("lookup", 4096, 0, 8), ("lookup", 5461, 1, 64),
    ("batch", 4096, 1, 64), ("batch", 5461, 0, 8),
    ("owner", 4096, 0, 64), ("owner", 5461, 1, 8),
]


@pytest.mark.parametrize("path,cap,kind,dim", CHURN)
def test_long_churn_matches_model(torch_cuda, oracle, path, cap, kind, dim):
    """60-80 turnovers of the table's rows: after every call the resident set and recency equal the model's, the
    counters match, the index keeps n_cells / 8 EMPTY cells after every eviction check (the rebuild), and every 10
    calls every resident entry equals the unbounded oracle's."""
    torch = torch_cuda
    from persia_b200 import shard as pb

    rng = np.random.default_rng(cap + dim + kind)
    fresh, hot, pool, warm = 400, 40, 1500, 100
    low, target = 600, 1200  # a request adds <= fresh + warm = 500 < low new signs: nothing is ever refused
    turnovers = 64 if cap == 4096 else 70
    calls = turnovers * cap // fresh
    oracle.set_rsqrt_exact(True)
    try:
        if path == "owner":
            # each owner gets about half of the fresh signs of a step: twice the steps for the same turnovers
            _churn_owner(torch, oracle, rng, cap, kind, dim, 2 * calls, fresh, hot, pool, warm, low, target)
            return
        s, opt = new_shard(pb, oracle, dim, cap, kind)
        s.set_eviction(check_every=1, low_water=low, target_free=target, keep_batches=2)
        m = IndexModel(cap, 1, low, target, 2)
        pf = oracle.index_prefix(0)
        w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf)], n_ps=1)
        w.configure(lo=LO, hi=HI)
        w.set_optimizer(opt)
        ctx = pb.BatchContext(4096, 4096, [pf]) if path == "batch" else None
        gen = Churn(rng, 1 << 20, fresh, hot, pool, warm)
        for k in range(calls):
            ids = gen.ids()
            if path == "lookup":
                signs = distinct_in_order(ids)
                new, back, _ = m.train(signs)
                reset_oracle(oracle, w, opt, back, dim)
                got = s.lookup(to_dev_ids(ids, DEV), training=True).cpu().numpy()
                want = w.ps_lookup(0, ids, np.full(ids.size, dim, np.uint32), True).reshape(ids.size, dim)
                assert got.tobytes() == want.tobytes(), k
                u = np.array(signs, np.uint64)
                g = (rng.standard_normal((u.size, dim)) * 1e-2).astype(np.float32)
                s.update(to_dev_ids(u, DEV), torch.from_numpy(g).to(DEV))
                w.ps_update(0, u, np.full(u.size, dim, np.uint32), g)
            else:
                B = ids.size
                signs = distinct_in_order(oracle.add_prefix(ids, 8, pf))
                new, back, _ = m.train(signs)
                reset_oracle(oracle, w, opt, back, dim)
                got = ctx.forward(s, to_dev_ids(ids, DEV), [0, B], B, training=True).cpu().numpy()
                want, octx = w.forward(ids, full_row_off(1, B), B, training=True)
                assert got[0].tobytes() == want[0].tobytes(), k
                g = (rng.standard_normal((B, dim)) * 1e-2).astype(np.float16)
                ctx.backward(s, [torch.from_numpy(g).to(DEV)])
                w.backward(octx, [g])
            check_export(s, m, k)
            check_counters(s, m, k)
            check_stats(s, m, len(new), k)
            if k % 10 == 9 or k == calls - 1:
                check_entries(s, w, m, k)
        assert m.evicted > (turnovers - 2) * cap and m.gone, (m.evicted, turnovers * cap)
    finally:
        oracle.set_rsqrt_exact(False)


def _churn_owner(torch, oracle, rng, cap, kind, dim, calls, fresh, hot, pool, warm, low, target):
    """The sharded owner lookup (k_owner_lookup) at R = 2 virtual ranks on one GPU: each rank's table is the owner of the
    signs farmhash64 sends it; one model per owner sees the distinct signs of both ranks' requests."""
    from persia_b200.worker import ShardedEmbeddingWorker as W

    R, per = 2, fresh // 2
    pf = [oracle.index_prefix(0)]
    gpu, opt = optim_pair(oracle, kind)
    B = per + hot + warm // 2 + hot // 2
    ws = W.local_group(R, 1, dim, pf, cap, cap=B, optimizer=dict(kind=kind, **gpu), max_batch=B)
    for x in ws:
        x.shard.configure(init_lower=LO, init_upper=HI)
        x.shard.set_eviction(check_every=1, low_water=low, target_free=target, keep_batches=2)
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))  # (allocates; the absent sign 0 is a miss)
    torch.cuda.synchronize()
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf[0])], n_ps=R)
    w.configure(lo=LO, hi=HI)
    w.set_optimizer(opt)
    models = [IndexModel(cap, 1, low, target, 2) for _ in range(R)]
    gens = [Churn(rng, (1 << 20) + (r << 36), per, hot, pool, warm // 2) for r in range(R)]
    gens[1].hot, gens[1].pool = gens[0].hot, gens[0].pool  # both ranks share the hot set and the warm pool
    outs = [torch.empty((1, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
    for k in range(calls):
        ids = [gens[r].ids() for r in range(R)]
        signs = np.concatenate([oracle.add_prefix(i, 8, pf[0]) for i in ids])
        owner = oracle.shard_of(signs, R)
        fresh_n = []
        for q in range(R):
            new, back, _ = models[q].train(distinct_in_order(signs[owner == q]))
            reset_oracle(oracle, w, opt, back, dim)
            fresh_n.append(len(new))
        torch.cuda.synchronize()
        W.group_forward(ws, [to_dev_ids(i, DEV) for i in ids], B, training=True, outs=outs)
        torch.cuda.synchronize()
        octx = []
        for r in range(R):
            want, c = w.forward(ids[r], full_row_off(1, B), B, training=True)
            octx.append(c)
            assert outs[r].cpu().numpy()[0].tobytes() == want[0].tobytes(), (k, r)
        g = (rng.standard_normal((R, B, dim)) * 1e-2).astype(np.float16)
        W.group_backward(ws, [[torch.from_numpy(g[r]).to(DEV)] for r in range(R)])
        torch.cuda.synchronize()
        for r in range(R):
            w.backward(octx[r], [g[r]])
        for q in range(R):
            sh = ws[q].shard
            check_export(sh, models[q], (k, q))
            check_counters(sh, models[q], (k, q), misses=1)
            check_stats(sh, models[q], fresh_n[q], (k, q))
            if k % 10 == 9 or k == calls - 1:
                check_entries(sh, w, models[q], (k, q))
    for x in ws:
        assert x.status() == (False, False)
    assert all(m.evicted > 55 * cap for m in models), [m.evicted for m in models]


def test_default_policy_churn(torch_cuda, oracle):
    """persia_core's policy (check_every 4, low_water cap/16, target cap/8, keep 2) through the same churn, with
    requests small enough that four of them never take more than low_water rows."""
    from persia_b200 import shard as pb

    rng = np.random.default_rng(4)
    cap, dim = 4096, 8
    s, opt = new_shard(pb, oracle, dim, cap, oracle.SGD)
    s.set_eviction()  # the defaults
    m = IndexModel(cap, 4, cap // 16, cap // 8, 2)
    w = oracle.Worker([oracle.SlotCfg(dim)], n_ps=1)
    w.configure(lo=LO, hi=HI)
    w.set_optimizer(opt)
    gen = Churn(rng, 1 << 30, 48, 16, 400, 16)  # <= 64 new signs per request, 4 x 64 = cap / 16
    calls, since = 60 * cap // 48, 0
    for k in range(calls):
        ids = gen.ids()
        signs = distinct_in_order(ids)
        new, back, checked = m.train(signs)
        since = len(new) if checked else since + len(new)
        reset_oracle(oracle, w, opt, back, dim)
        got = s.lookup(to_dev_ids(ids, DEV), training=True).cpu().numpy()
        want = w.ps_lookup(0, ids, np.full(ids.size, dim, np.uint32), True).reshape(ids.size, dim)
        assert got.tobytes() == want.tobytes(), k
        if k % 8 == 7 or k == calls - 1:
            check_export(s, m, k)
            check_counters(s, m, k)
            check_stats(s, m, since, k)
    check_entries(s, w, m, "end")
    assert m.evicted > 55 * cap, m.evicted


# ---- probe sequences that wrap, duplicates, refusal, marker signs ---------------------------------------------------
def _homed_in(bucket, mask, count, start):
    out, base = [], start
    while len(out) < count:
        c = np.arange(base, base + (1 << 20), dtype=np.uint64)
        out.extend(c[(mix64(c) & np.uint64(mask)) == np.uint64(bucket)].tolist())
        base += 1 << 20
    return np.array(out[:count], np.uint64)


def test_probe_wraps_past_the_last_bucket(torch_cuda, oracle):
    """More than 8 signs homed in the last bucket overflow into bucket 0.  Some are evicted and re-admitted, and signs
    homed there that were never admitted are looked up: the resident set follows the model, values are the initial
    ones, absent signs read zeros."""
    from persia_b200 import shard as pb

    cap, dim = 4096, 8
    mask = n_cells(cap) // 8 - 1
    last = _homed_in(mask, mask, 16, 1 << 24)
    zero = _homed_in(0, mask, 4, 1 << 26)
    first, absent = np.concatenate([last[:12], zero]), last[12:]
    s, opt = new_shard(pb, oracle, dim, cap, oracle.SGD)
    s.set_eviction(check_every=1, low_water=cap, target_free=cap, keep_batches=1)  # every check releases ages >= 2
    m = IndexModel(cap, 1, cap, cap, 1)

    def call(q, what):
        m.train(distinct_in_order(q))
        got = s.lookup(to_dev_ids(q, DEV), training=True).cpu().numpy()
        np.testing.assert_array_equal(got, np.stack([oracle.init_row(int(x), dim, LO, HI) for x in q]), err_msg=what)
        check_export(s, m, what)
        check_counters(s, m, what)
        check_stats(s, m, len(q), what)

    call(first, "admit 12 + 4")
    call(np.concatenate([last[:6], zero[:2]]), "refresh half")
    call(np.array([7], np.uint64), "age 2")
    call(np.array([8], np.uint64), "evict the other half")
    assert not any(int(x) in m.res for x in last[6:12])
    call(last[6:12][::-1].copy(), "re-admit")
    got = s.lookup(to_dev_ids(absent, DEV), training=False).cpu().numpy()
    np.testing.assert_array_equal(got, 0)
    _, found = s.get_entries(to_dev_ids(np.concatenate([absent, last[:12]]), DEV))
    assert found.cpu().numpy().tolist() == [False] * 4 + [int(x) in m.res for x in last[:12]]


def test_duplicate_admissions_into_tombstones(torch_cuda, oracle):
    """A table full of tombstones, then one training lookup in which each of 100 new signs appears 32 times in shuffled
    order: every sign ends in exactly one cell, and all its occurrences read its initial row."""
    from persia_b200 import shard as pb

    rng = np.random.default_rng(32)
    cap, dim = 4096, 16
    s, opt = new_shard(pb, oracle, dim, cap, oracle.SGD)
    s.set_eviction(check_every=1, low_water=cap, target_free=cap, keep_batches=1)
    m = IndexModel(cap, 1, cap, cap, 1)
    for k, q in enumerate([np.arange(1, 4001, dtype=np.uint64)] + [np.array([5000 + j], np.uint64) for j in range(3)]):
        m.train(distinct_in_order(q))
        s.lookup(to_dev_ids(q, DEV), training=True)
        check_export(s, m, k)
    st = s.index_stats()
    assert st["tomb"] >= 3990, st
    new = np.arange(10_000, 10_100, dtype=np.uint64)
    q = np.repeat(new, 32)
    rng.shuffle(q)
    m.train(distinct_in_order(q))
    got = s.lookup(to_dev_ids(q, DEV), training=True).cpu().numpy()
    np.testing.assert_array_equal(got, np.stack([oracle.init_row(int(x), dim, LO, HI) for x in q]))
    check_export(s, m, "dups")
    check_counters(s, m, "dups")
    assert len(s) == len(m.res)


def test_refusal_then_sweep_admits(torch_cuda, oracle):
    """check_every = 0: a request with more new signs than free rows admits as many as there are rows and refuses the
    rest, which read zeros.  Once a sweep has released rows, the refused signs come in with their initial values."""
    from persia_b200 import shard as pb

    cap, dim = 1000, 8
    s, opt = new_shard(pb, oracle, dim, cap, oracle.ADAGRAD)
    old = np.arange(1, 901, dtype=np.uint64)
    s.lookup(to_dev_ids(old, DEV), training=True)
    more = np.arange(5000, 5300, dtype=np.uint64)
    got = s.lookup(to_dev_ids(more, DEV), training=True).cpu().numpy()
    c = s.counters()
    assert c["admitted"] == cap and c["capacity_refused"] == 200 and c["lookup_miss"] == 200, c
    _, found = s.get_entries(to_dev_ids(more, DEV))
    found = found.cpu().numpy()
    assert found.sum() == 100
    np.testing.assert_array_equal(got[~found], 0)
    assert (np.abs(got[found]).sum(axis=1) > 0).all()
    st = s.index_stats()
    # the refused signs' cells were rolled back to tombstones (which later refused signs may have reused and rolled back)
    assert st["live"] == cap and 1 <= st["tomb"] <= 200, st
    s.set_eviction(check_every=1, low_water=cap, target_free=cap, keep_batches=1)
    keep = more[found][:1]
    s.lookup(to_dev_ids(keep, DEV), training=True)  # the sweep before it spares ages <= 1: nothing goes yet
    assert len(s) == cap
    refused = more[~found]
    got = s.lookup(to_dev_ids(refused, DEV), training=True).cpu().numpy()  # the old 900 are two requests old now
    np.testing.assert_array_equal(got, np.stack([oracle.init_row(int(x), dim, LO, HI) for x in refused]))
    ent, f2 = s.get_entries(to_dev_ids(refused, DEV))
    assert f2.all()
    opt = optim_pair(oracle, oracle.ADAGRAD)[1]
    np.testing.assert_array_equal(ent.cpu().numpy(), np.stack([opt.new_entry(oracle.init_row(int(x), dim, LO, HI))
                                                                for x in refused]))
    c = s.counters()
    assert c["capacity_refused"] == 200 and c["admitted"] == 100 + 200, c


def test_marker_signs_through_eviction_and_the_tier(torch_cuda, oracle):
    """2^64-1, 2^64-2 and 2^64-3 equal the index's cell markers and live in reserved cells: they are evicted, re-admitted
    and exported.  On a table with a host tier, an eviction check moves them into the tier's reserved cells under their
    own values, reads use them there, and a training lookup brings them back bit for bit."""
    torch = torch_cuda
    from persia_b200 import shard as pb

    cap, dim = 64, 8
    markers = np.array([M64, M64 - 1, M64 - 2], np.uint64)
    other = np.arange(1, 11, dtype=np.uint64)
    s, opt = new_shard(pb, oracle, dim, cap, oracle.SGD)
    s.set_eviction(check_every=1, low_water=cap, target_free=cap, keep_batches=1)
    m = IndexModel(cap, 1, cap, cap, 1)
    init = np.stack([oracle.init_row(int(x), dim, LO, HI) for x in markers])
    misses = [0]

    def call(q, what):
        m.train(distinct_in_order(q))
        out = s.lookup(to_dev_ids(q, DEV), training=True).cpu().numpy()
        check_export(s, m, what)
        check_counters(s, m, what, misses[0])
        return out

    np.testing.assert_array_equal(call(np.concatenate([markers, other]), "admit")[:3], init)
    g = np.full((3, dim), 0.5, np.float32)
    s.update(to_dev_ids(markers, DEV), torch.from_numpy(g).to(DEV))
    call(other[:1], "age 1")
    call(other[1:2], "age 2")
    call(other[2:3], "age 3")  # its sweep releases the rows two requests old: the markers among them
    assert not any(int(x) in m.res for x in markers)
    np.testing.assert_array_equal(s.lookup(to_dev_ids(markers, DEV), training=False).cpu().numpy(), 0)
    misses[0] += 3
    np.testing.assert_array_equal(call(markers[::-1].copy(), "re-admit")[::-1], init)  # from the initial value again
    s.update(to_dev_ids(markers, DEV), torch.from_numpy(g).to(DEV))
    before = s.get_entries(to_dev_ids(markers, DEV))[0].cpu().numpy()
    call(other[5:6], "age 1")
    call(other[6:7], "age 2")
    assert set(m.res) == {int(x) for x in markers} | {int(other[5]), int(other[6])}
    got, _ = s.export_signs()
    assert set(int(x) for x in got.cpu().numpy().view(np.uint64)) == set(m.res)

    # the same signs on a table with a host tier (IndexModel counts HBM rows only: the tier is checked directly)
    t, _ = new_shard(pb, oracle, dim, cap, oracle.SGD, tier_rows=256)
    t.set_eviction(check_every=1, low_water=cap, target_free=cap, keep_batches=1)

    def signs_of(h):
        return set(t._export_table(h)[0].cpu().numpy().view(np.uint64).tolist())

    try:
        t.lookup(to_dev_ids(markers, DEV), training=True)
        t.update(to_dev_ids(markers, DEV), torch.from_numpy(g).to(DEV))  # the entries `before` holds: init + one step
        np.testing.assert_array_equal(t.get_entries(to_dev_ids(markers, DEV))[0].cpu().numpy(), before)
        for _ in range(3):  # the check before the third releases the rows two requests old: the markers move out
            t.lookup(to_dev_ids(other[:1], DEV), training=True)
        ts = t.tier_stats()
        assert ts["moved_out"] == 3 and ts["host_rows"] == 3 and ts["restored"] == 0, ts
        assert t.index_stats()["live"] == 1 and signs_of(t.h) == {int(other[0])}
        # in the tier's reserved cells, not its normal ones
        assert t.host_tier.index_stats()["live"] == 0 and signs_of(t.host_tier.h) == {int(x) for x in markers}
        got, _ = t.export_signs()
        assert set(got.cpu().numpy().view(np.uint64).tolist()) == {int(x) for x in markers} | {int(other[0])}
        e2, found = t.get_entries(to_dev_ids(markers, DEV))
        assert found.all()
        np.testing.assert_array_equal(e2.cpu().numpy(), before)
        np.testing.assert_array_equal(t.lookup(to_dev_ids(markers, DEV), training=False).cpu().numpy(), before[:, :dim])
        assert t.tier_stats()["restored"] == 0  # read in place
        t.lookup(to_dev_ids(markers, DEV), training=True)  # restored under their own signs
        ts = t.tier_stats()
        assert ts["restored"] == 3 and ts["moved_out"] == 3 and ts["host_rows"] == 0, ts
        assert t.host_tier.index_stats()["live"] == 0 and not signs_of(t.host_tier.h)
        assert signs_of(t.h) == {int(x) for x in markers} | {int(other[0])}
        e2, found = t.get_entries(to_dev_ids(markers, DEV))
        assert found.all()
        np.testing.assert_array_equal(e2.cpu().numpy(), before)
        assert t.counters()["capacity_refused"] == 0
    finally:
        t.close()


# ---- a pending local raw forward keeps its rows ---------------------------------------------------------------------
def test_local_raw_pending_rows_survive_the_sweep(torch_cuda, oracle):
    """Four raw slots and one summation slot of one dim share one table; before every training forward the sweep
    releases every row older than keep_batches = 1 request.  The first raw slot's rows are older than that when the
    later forwards sweep: they stay only because a pending raw forward counts as a pending batch, so every gradient
    lands on its own sign's row (bit for bit with the oracle) and no gradient id goes missing."""
    torch = torch_cuda
    from persia_b200 import shard as pb

    rng = np.random.default_rng(91)
    B, dim, fixed, n_raw = 64, 16, 3, 4
    pf = [oracle.index_prefix(i) for i in range(n_raw + 1)]
    s, opt = new_shard(pb, oracle, dim, 4096, oracle.SGD)
    s.set_eviction(check_every=1, low_water=4096, target_free=4096, keep_batches=1)
    slots = [oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=p) for p in pf[:n_raw]]
    w = oracle.Worker(slots + [oracle.SlotCfg(dim, prefix=pf[n_raw])], n_ps=1)
    w.configure(lo=LO, hi=HI)
    w.set_optimizer(opt)
    ctxs = [pb.BatchContext(4 * B, 4 * B, [p]) for p in pf[:n_raw]]
    sctx = pb.BatchContext(B, B, [pf[n_raw]])
    oracle.set_rsqrt_exact(True)
    try:
        pend, raw_signs = [], set()
        for i in range(n_raw):
            cnt = rng.integers(1, 5, size=B)
            ro = np.zeros(B + 1, np.uint32)
            ro[1:] = np.cumsum(cnt)
            ids = rng.integers(0, 150, size=int(ro[-1]), dtype=np.uint64)
            table, _, _, _, counts = ctxs[i].forward_raw(s, to_dev_ids(ids, DEV), B, fixed, row_off=to_dev_i32(ro, DEV))
            otab, _, _, _, octx = w.forward_raw(i, ids, ro, B)
            U = int(counts[0].item())
            assert U == otab.shape[0] - 1
            assert table[: U + 1].cpu().numpy().tobytes() == otab.tobytes(), i
            pend.append((U, octx))
            raw_signs.update(int(x) for x in oracle.add_prefix(ids, 8, pf[i]))
        sid = rng.integers(0, 150, size=B, dtype=np.uint64)  # a summation batch on the same table sweeps too
        sctx.forward(s, to_dev_ids(sid, DEV), [0, B], B, training=True)
        for i in range(n_raw):
            U, octx = pend[i]
            g = (rng.standard_normal((U, dim)) * 1e-1).astype(np.float32)
            ctxs[i].backward_raw(s, torch.from_numpy(g).to(DEV))
            w.backward_raw(i, octx, g)
        sctx.backward(s, [None])  # skipped: its rows keep their initial values
        torch.cuda.synchronize()
        assert s.counters()["gradient_id_miss"] == 0
        sum_signs = {int(x) for x in oracle.add_prefix(sid, 8, pf[n_raw])}
        signs, _ = s.export_signs()
        signs = signs.cpu().numpy().view(np.uint64)
        assert set(int(x) for x in signs) == raw_signs | sum_signs  # nothing was evicted
        ent, _ = s.get_entries(to_dev_ids(signs, DEV))
        ent = ent.cpu().numpy()
        for k, sign in enumerate(signs):
            if int(sign) in sum_signs:
                ref = opt.new_entry(oracle.init_row(int(sign), dim, LO, HI))
            else:
                ref = w.get_entry(int(sign))
            assert ref is not None and ent[k].tobytes() == ref.tobytes(), (k, int(sign))
    finally:
        oracle.set_rsqrt_exact(False)
