"""GPU: the set of updated signs behind incremental updates (pb_inc.cu, EmbeddingShard.take_incremental).

A host model decides every assertion: the distinct signs that took an optimizer step since the last take, fed by each
test's own knowledge of slot status and of which signs had rows.  After every take the taken signs equal the model's
(minus the ones no table holds any more, which are skipped and counted), and every taken entry equals get_entries and
the oracle's entry bit for bit (the oracle in exact-rsqrt mode)."""
import numpy as np
import pytest

from util import (DEV, full_row_off, held_rows, make_batch, pair, ragged_with_multiplicities, slot_signs, to_dev_i32,
                  to_dev_ids)

pytestmark = pytest.mark.gpu
U64 = np.uint64


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


@pytest.fixture(autouse=True)
def exact_rsqrt(oracle):
    oracle.set_rsqrt_exact(True)
    yield
    oracle.set_rsqrt_exact(False)


OPT = {0: dict(lr=0.05, wd=0.001), 1: dict(lr=0.02, init_acc=0.01, eps=1e-10),
       2: dict(lr=0.02, init_acc=0.01, eps=1e-10), 3: dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8)}


def _grads(rng, S, B, dim, f32=False):
    return (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float32 if f32 else np.float16)


def train_step(torch, s, ctx, w, ids, row_off, slot_off, B, g, model, skip=(), nan=(), rows_of=None):
    """One batched step on the GPU and in the oracle; the model takes the signs of every applied slot that had a row
    (rows_of: the signs that had one; None = all)."""
    S = ctx.n_slots
    ro = row_off if row_off is not None else full_row_off(S, B)
    ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=to_dev_i32(row_off, DEV) if row_off is not None else None)
    _, octx = w.forward(ids, ro, B, training=True)
    per_slot = [w.ctx_signs(octx, i) for i in range(S)]
    g = g.copy()
    for i in nan:
        g[i, B // 2, 0] = np.nan
    grads = [None if i in skip else torch.from_numpy(np.ascontiguousarray(g[i])).to(DEV) for i in range(S)]
    st = ctx.backward(s, grads, want_status=True).cpu().numpy().tolist()
    ost = w.backward(octx, [g[i] for i in range(S)], skip=[int(i in skip) for i in range(S)])
    assert st == ost
    for i in range(S):
        if st[i] == 0:
            sg = per_slot[i] if rows_of is None else np.intersect1d(per_slot[i], rows_of)
            model.update(int(x) for x in sg)
    return st


def check_take(torch, s, w, model, skipped=0, pending_held=None):
    """Takes the set and checks it against the model; empties the model."""
    st0 = s.incremental_stats()
    assert st0["held"] == len(model) + skipped
    assert s.incremental_held() == len(model) + skipped  # (synchronised by the stats call)
    signs, ent, n_skip = s.take_incremental()
    got = signs.view(U64)
    assert n_skip == skipped
    assert np.all(got[:-1] < got[1:])
    assert got.tolist() == sorted(model)
    if got.size:
        again, found = s.get_entries(to_dev_ids(got, DEV))
        assert bool(found.all())
        assert again.cpu().numpy().tobytes() == ent.tobytes()
        for k, x in enumerate(got):
            ref = w.get_entry(int(x))
            assert ref is not None and ref.tobytes() == ent[k].tobytes(), (k, int(x))
    st1 = s.incremental_stats()
    assert st1["held"] == 0 and st1["taken"] == st0["taken"] + len(model) + skipped
    assert s.incremental_held() == 0
    model.clear()


@pytest.mark.parametrize("kind,dim,layout", [(0, 33, "single"), (1, 128, "ragged"), (2, 1, "sqrt"), (3, 33, "ragged"),
                                             (0, 128, "hash"), (3, 1, "single"), (1, 33, "sqrt"), (2, 128, "hash")])
def test_batched_marks(torch_cuda, pb, oracle, kind, dim, layout):
    torch = torch_cuda
    rng = np.random.default_rng(kind * 100 + dim)
    S, B = 3, 300
    sqrt = [False, True, True] if layout == "sqrt" else None
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, sqrt=sqrt, optim_kw=OPT[kind])
    s.enable_incremental(1 << 14)
    model = set()
    for step in range(6):
        if layout == "hash":  # hash-stacked slots: the ids the table sees are the stacked keys
            raw, _, _ = make_batch(rng, S, B, [50, 4000, 1 << 40])
            ids = pb.hash_stack(to_dev_ids(raw, DEV), 2, 1000).cpu().numpy().view(U64)
            row_off = np.arange(0, S * B * 2 + 1, 2, dtype=np.uint32)
            slot_off = [i * B * 2 for i in range(S + 1)]
        else:
            ids, row_off, slot_off = make_batch(rng, S, B, [7, 500, 100000], max_ids=1 if layout == "single" else 4,
                                                allow_empty=layout != "single")
        train_step(torch, s, ctx, w, ids, row_off, slot_off, B, _grads(rng, S, B, dim, f32=kind == 2), model)
        if step % 3 == 2:
            check_take(torch, s, w, model)
    assert s.incremental_stats()["dropped"] == 0


def test_nan_skip_and_shared_groups(torch_cuda, pb, oracle):
    """A NaN-dropped slot and a skipped slot mark nothing of their own, but a sign that an applied slot of the same
    group holds is marked (once); slots sharing a group step the sign once per slot and it is held once."""
    torch = torch_cuda
    rng = np.random.default_rng(5)
    S, B, dim = 4, 256, 16
    s, ctx, w, pf = pair(pb, oracle, S, dim, 3, groups=[0, 0, 1, 1], optim_kw=OPT[3])
    s.enable_incremental(1 << 14)
    model = set()
    for step, (skip, nan) in enumerate([((), ()), ((1,), (2,)), ((0,), ()), ((), (3,)), ((0, 1), (2, 3))]):
        ids, row_off, slot_off = make_batch(rng, S, B, [30, 30, 400, 400], max_ids=2)
        st = train_step(torch, s, ctx, w, ids, row_off, slot_off, B, _grads(rng, S, B, dim), model, skip=skip, nan=nan)
        assert [i for i in range(S) if st[i] == 1] == list(skip) and [i for i in range(S) if st[i] == 2] == list(nan)
        check_take(torch, s, w, model)


def test_raw_slot(torch_cuda, pb, oracle):
    torch = torch_cuda
    rng = np.random.default_rng(9)
    dim, B, fixed = 24, 200, 4
    pf = oracle.index_prefix(0)
    s = pb.EmbeddingShard(dim, 1 << 14, 0)
    s.set_optimizer(1, lr=0.02, initialization=0.01, eps=1e-10)
    s.configure()
    ctx = pb.BatchContext(4 * B, 4 * B, [pf])
    w = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=pf)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(1, **OPT[1]))
    s.enable_incremental(1 << 12)
    model = set()
    for step, mode in enumerate(["apply", "nan", "skip", "apply", "f16"]):
        ids, ro = ragged_with_multiplicities(rng, B, [6, 3], 3)
        ctx.forward_raw(s, to_dev_ids(ids, DEV), B, fixed, row_off=to_dev_i32(ro, DEV))
        _, _, _, _, octx = w.forward_raw(0, ids, ro, B)
        uniq = ids[np.sort(np.unique(ids, return_index=True)[1])]
        g = (rng.standard_normal((uniq.size, dim)) * 1e-2).astype(np.float16 if mode == "f16" else np.float32)
        if mode == "nan":
            g[1, 2] = np.nan
        gd = None if mode == "skip" else torch.from_numpy(g).to(DEV)
        st = ctx.backward_raw(s, gd, want_status=True).item()
        assert st == w.backward_raw(0, octx, None if mode == "skip" else g, skip=mode == "skip")
        if st == 0:
            model.update(int(x) for x in oracle.add_prefix(uniq, 8, pf))
        check_take(torch, s, w, model)


def test_update_direct_and_marker_signs(torch_cuda, pb, oracle):
    """pb_update marks the signs it found (absent ones are skipped); signs equal to the set's markers use its reserved
    cells."""
    torch = torch_cuda
    rng = np.random.default_rng(11)
    dim = 8
    s, _, w, _ = pair(pb, oracle, 1, dim, 0, optim_kw=OPT[0])
    s.enable_incremental(64)
    special = np.array([0xFFFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFE, 0xFFFFFFFFFFFFFFFD, 0, 1, 12345], U64)
    ent = rng.uniform(-0.1, 0.1, (special.size, dim)).astype(np.float32)
    s.set_entries(to_dev_ids(special, DEV), torch.from_numpy(ent).to(DEV))
    w.set_embedding(special, ent, dim)
    assert s.incremental_stats()["held"] == 0  # set_entries marks nothing
    model = set()
    for sel in ([0, 1, 2], [3, 4, 5], [0, 5]):
        signs = np.concatenate([special[sel], np.array([777, 0xFFFFFFFFFFFF0000], U64)])  # two absent
        g = (rng.standard_normal((signs.size, dim)) * 0.1).astype(np.float32)
        s.update(to_dev_ids(signs, DEV), torch.from_numpy(g).to(DEV))
        w.ps_update(0, signs, np.full(signs.size, dim, np.uint32), g)
        model.update(int(x) for x in special[sel])
    check_take(torch, s, w, model)


def test_refused_admissions_and_eviction_churn(torch_cuda, pb, oracle):
    """A sign refused at admission has no row: its gradient is a miss and it is not marked.  Then eviction churn between
    mark and take: signs evicted since they were marked are skipped and counted."""
    torch = torch_cuda
    rng = np.random.default_rng(13)
    S, B, dim = 2, 256, 16
    s, ctx, w, pf = pair(pb, oracle, S, dim, 0, cap=300, optim_kw=OPT[0])
    s.enable_incremental(1 << 12)
    model = set()
    ids, row_off, slot_off = make_batch(rng, S, B, [100000, 100000])
    signs = slot_signs(oracle, ids, slot_off, pf)
    # the oracle has no capacity bound: read which signs got a row from the table
    ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B)
    had = np.array(sorted(held_rows(torch, oracle, [s], signs)), U64)
    assert 0 < had.size < np.unique(signs).size
    ctx.backward(s, [torch.from_numpy(g).to(DEV) for g in _grads(rng, S, B, dim)])
    assert s.counters()["gradient_id_miss"] > 0
    signs_taken, _, n_skip = s.take_incremental()
    assert n_skip == 0 and signs_taken.view(U64).tolist() == had.tolist()
    # churn: a table of 512 rows, eviction every request, the marked rows of step 0 pushed out by later steps
    s2, ctx2, w2, pf2 = pair(pb, oracle, 1, dim, 0, cap=512, optim_kw=OPT[0])
    s2.set_eviction(check_every=1, low_water=200, target_free=300, keep_batches=1)
    s2.enable_incremental(1 << 12)
    marked = set()
    for step in range(6):
        ids = (np.arange(200, dtype=U64) + U64(200 * step))
        ctx2.forward(s2, to_dev_ids(ids, DEV), [0, 200], 200)
        had = held_rows(torch, oracle, [s2], oracle.add_prefix(ids, 8, pf2[0]))  # (a sweep may free too few rows)
        ctx2.backward(s2, [torch.from_numpy(_grads(rng, 1, 200, dim)[0]).to(DEV)])
        marked.update(had)
    alive = set(held_rows(torch, oracle, [s2], np.array(sorted(marked), U64)))
    assert 0 < len(alive) < len(marked)
    got, ent, n_skip = s2.take_incremental()
    assert got.view(U64).tolist() == sorted(alive) and n_skip == len(marked) - len(alive)
    ref, found = s2.get_entries(torch.from_numpy(got).to(DEV))
    assert bool(found.all()) and ref.cpu().numpy().tobytes() == ent.tobytes()


def test_full_set_drops_exactly(torch_cuda, pb, oracle):
    torch = torch_cuda
    rng = np.random.default_rng(17)
    S, B, dim = 1, 1000, 8
    s, ctx, w, pf = pair(pb, oracle, S, dim, 1, optim_kw=OPT[1])
    s_ref, ctx_ref, _, _ = pair(pb, oracle, S, dim, 1, optim_kw=OPT[1])
    cap = 1500
    s.enable_incremental(cap)
    seen = set()
    for step in range(4):
        ids = rng.integers(0, 1 << 40, size=B, dtype=U64)  # distinct in practice
        g = _grads(rng, S, B, dim)
        for sh, cx in ((s, ctx), (s_ref, ctx_ref)):
            cx.forward(sh, to_dev_ids(ids, DEV), [0, B], B)
            cx.backward(sh, [torch.from_numpy(g[0]).to(DEV)])
        seen.update(int(x) for x in oracle.add_prefix(ids, 8, pf[0]))
        st = s.incremental_stats()
        assert st["held"] == min(len(seen), cap) and st["dropped"] == max(0, len(seen) - cap)
        assert st["inserted"] == st["held"]
    # training is unchanged by a full set
    every = np.array(sorted(seen), U64)
    a = s.get_entries(to_dev_ids(every, DEV))[0].cpu().numpy()
    b = s_ref.get_entries(to_dev_ids(every, DEV))[0].cpu().numpy()
    assert a.tobytes() == b.tobytes()
    got, _, _ = s.take_incremental()
    assert got.size == cap and set(got.view(U64).tolist()) <= seen


def test_take_too_small_leaves_set(torch_cuda, pb, oracle):
    torch = torch_cuda
    s, ctx, w, pf = pair(pb, oracle, 1, 4, 0, optim_kw=OPT[0])
    s.enable_incremental(1000)
    ids = np.arange(100, dtype=U64)
    ctx.forward(s, to_dev_ids(ids, DEV), [0, 100], 100)
    ctx.backward(s, [torch.zeros(100, 4, dtype=torch.float16, device=DEV) + 0.01])
    lib = s.lib
    count = torch.zeros(1, dtype=torch.int32, device=DEV)
    buf = torch.full((99,), -7, dtype=torch.int64, device=DEV)
    from persia_b200 import native as N
    import ctypes as C

    N.check(lib.pb_inc_take(s.h, C.c_void_p(buf.data_ptr()), 99, C.c_void_p(count.data_ptr()),
                            C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert int(count) == 100 and bool((buf == -7).all())
    assert s.incremental_stats()["held"] == 100
    got, _, _ = s.take_incremental()
    assert got.view(U64).tolist() == sorted(int(x) for x in oracle.add_prefix(ids, 8, pf[0]))


def test_graph_captured_step(torch_cuda, pb, oracle):
    """A captured forward + backward, replayed: every replay marks that replay's signs."""
    torch = torch_cuda
    rng = np.random.default_rng(23)
    S, B, dim = 2, 256, 16
    s, ctx, w, pf = pair(pb, oracle, S, dim, 1, optim_kw=OPT[1])
    s.enable_incremental(1 << 12)
    d_ids = torch.zeros(S * B, dtype=torch.int64, device=DEV)
    g = torch.zeros(S, B, dim, dtype=torch.float16, device=DEV)
    first, _, _ = make_batch(rng, S, B, [1000, 1000])
    d_ids.copy_(to_dev_ids(first, DEV))
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):  # warm-up (allocations happen outside the capture)
        ctx.forward(s, d_ids, [0, B, 2 * B], B)
        ctx.backward(s, [g[0], g[1]])
    torch.cuda.synchronize()
    s.take_incremental()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        ctx.forward(s, d_ids, [0, B, 2 * B], B)
        ctx.backward(s, [g[0], g[1]])
    torch.cuda.synchronize()
    s.take_incremental()  # (capture ran nothing)
    model = set()
    for rep in range(3):
        ids, _, slot_off = make_batch(rng, S, B, [1000, 1000])
        d_ids.copy_(to_dev_ids(ids, DEV))
        gh = _grads(rng, S, B, dim)
        g.copy_(torch.from_numpy(gh))
        torch.cuda.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        model.update(int(x) for x in slot_signs(oracle, ids, slot_off, pf))
        got, _, n_skip = s.take_incremental()
        assert n_skip == 0 and got.view(U64).tolist() == sorted(model)
        model.clear()


def _run(torch, pb, oracle, enable, rng_seed=29):
    rng = np.random.default_rng(rng_seed)
    S, B, dim = 3, 256, 32
    s, ctx, w, pf = pair(pb, oracle, S, dim, 3, groups=[0, 0, 1], optim_kw=OPT[3])
    if enable == "disabled":
        s.enable_incremental(100)
        s.enable_incremental(0)
    elif enable == "on":
        s.enable_incremental(1 << 12)
    outs, counts = [], []
    lib = s.lib
    for step in range(4):
        ids, row_off, slot_off = make_batch(rng, S, B, [50, 50, 3000], max_ids=3)
        torch.cuda.synchronize()
        n0 = lib.pb_launch_count()
        out = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=to_dev_i32(row_off, DEV))
        ctx.backward(s, [torch.from_numpy(x).to(DEV) for x in _grads(rng, S, B, dim)])
        torch.cuda.synchronize()
        counts.append(lib.pb_launch_count() - n0)
        outs.append(out.cpu().numpy().tobytes())
    signs, _ = s.export_signs()
    ent, _ = s.get_entries(signs)
    return outs, counts, signs.cpu().numpy().tobytes() + ent.cpu().numpy().tobytes()


def test_disabled_and_never_enabled_are_unchanged(torch_cuda, pb, oracle):
    torch = torch_cuda
    never = _run(torch, pb, oracle, "never")
    off = _run(torch, pb, oracle, "disabled")
    on = _run(torch, pb, oracle, "on")
    assert off[1] == never[1]  # the same kernels, launch for launch
    assert on[1] == never[1]  # the mark replaces the scratch-set clear: one launch each way
    assert off[0] == never[0] and on[0] == never[0]
    assert off[2] == never[2] and on[2] == never[2]


def test_host_tier(torch_cuda, pb, oracle):
    """With a host tier: staging and tier moves mark nothing; pb_update steps a tier-held sign in place and marks it;
    its entry is read from the tier; set_entries and checkpoint loads mark nothing."""
    torch = torch_cuda
    rng = np.random.default_rng(31)
    dim, B = 16, 150  # at most 150 restores a step: the check before each request leaves >= 200 rows free
    pf = oracle.index_prefix(0)
    s = pb.EmbeddingShard(dim, 512, 0, tier_rows=4096)
    s.set_optimizer(0, lr=0.05, wd=0.001)
    s.configure()
    s.set_eviction(check_every=1, low_water=200, target_free=300, keep_batches=1)
    s.enable_incremental(1 << 12)
    ctx = pb.BatchContext(B, B, [pf])
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(0, **OPT[0]))
    # seed entries straight into both tables: set_entries marks nothing
    every = oracle.add_prefix(np.arange(2000, dtype=U64), 8, pf)
    ent = rng.uniform(-0.05, 0.05, (every.size, dim)).astype(np.float32)
    s.set_entries(to_dev_ids(every, DEV), torch.from_numpy(ent).to(DEV))
    w.set_embedding(every, ent, dim)
    assert s.tier_stats()["host_rows"] > 0
    assert s.incremental_stats() == {"held": 0, "inserted": 0, "dropped": 0, "taken": 0}
    # the seeded rows carry the current batch number: age them (training lookups of one other sign), so that the sweeps
    # before the steps below free rows for every restore they need
    for _ in range(3):
        s.lookup(to_dev_ids(np.array([1 << 62], U64), DEV), training=True)
    # stages and the moves of inference lookups mark nothing
    for step in range(3):
        ids = rng.integers(0, 2000, size=B, dtype=U64)
        s.stage(to_dev_ids(ids, DEV), [0, B], [pf])
        ctx.forward(s, to_dev_ids(ids, DEV), [0, B], B, training=False)
    assert s.incremental_stats()["inserted"] == 0
    # training: forward moves tier-held signs in, evictions push others out; every applied sign is marked
    model, trained = set(), set()
    for step in range(4):
        ids = rng.integers(0, 2000, size=B, dtype=U64)
        ctx.forward(s, to_dev_ids(ids, DEV), [0, B], B)
        # the signs that had a row: the batch's signs now in HBM (a restore that found no free row left its sign in
        # the tier: a gradient miss, not marked)
        hbm = set(s._export_table(s.h)[0].cpu().numpy().view(U64).tolist())
        sg = {int(x) for x in oracle.add_prefix(ids, 8, pf)}
        ctx.backward(s, [torch.from_numpy(_grads(rng, 1, B, dim)[0]).to(DEV)])
        model.update(sg & hbm)
        trained.update(sg)
    assert s.tier_stats()["moved_out"] > 0
    alive = set(held_rows(torch, oracle, [s], np.array(sorted(model), U64)))
    assert alive == model  # the tier keeps everything here
    assert s.incremental_stats()["held"] == len(model)
    got, ent, n_skip = s.take_incremental()
    assert n_skip == 0 and got.view(U64).tolist() == sorted(model)
    again, _ = s.get_entries(torch.from_numpy(got).to(DEV))
    assert again.cpu().numpy().tobytes() == ent.tobytes()
    model.clear()
    # pb_update of tier-held signs (and an absent one): stepped in place, marked, read from the tier
    tsigns, _ = s._export_table(s.host_tier.h)
    tier_held = np.array([x for x in np.sort(tsigns.cpu().numpy().view(U64)) if int(x) not in trained][:50], U64)
    assert tier_held.size == 50  # seeded, never trained: the oracle holds the same entries
    upd = np.concatenate([tier_held, np.array([0xABCDEF], U64)])
    g = (rng.standard_normal((upd.size, dim)) * 0.1).astype(np.float32)
    before = s.tier_stats()
    s.update(to_dev_ids(upd, DEV), torch.from_numpy(g).to(DEV))
    w.ps_update(0, upd, np.full(upd.size, dim, np.uint32), g)
    assert s.tier_stats()["restored"] == before["restored"]  # stepped in place
    model.update(int(x) for x in tier_held)
    check_take(torch, s, w, model)
    # a checkpoint load goes through set_entries: nothing marked
    import tempfile
    from persia_b200 import checkpoint as ck

    with tempfile.TemporaryDirectory() as d:
        ck.dump_shards(d, [s])
        ck.load_shards(d, {dim: s})
    assert s.incremental_stats()["held"] == 0


def _sharded(torch, oracle, R, groups, raw):
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW

    rng = np.random.default_rng(R * 10 + len(groups) + raw)
    dim, B, cap = 16, 128, 1 << 12
    pfs = [oracle.index_prefix(gi) for gi in groups]
    gopt = dict(kind=1, lr=0.02, initialization=0.01, eps=1e-10)
    S = len(groups)
    ws = W.local_group(R, S, dim, pfs, cap, cap=S * B, optimizer=gopt, max_batch=B, rows_f32=True,
                       max_ids_per_sample=3)
    rws = RW.local_group(R, 1, dim, [oracle.index_prefix(7)], cap, cap=3 * B, optimizer=gopt, max_batch=B,
                         max_ids_per_sample=3, shards=[x.shard for x in ws]) if raw else None
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pfs], n_ps=R)
    w.configure()
    w.set_optimizer(oracle.Optim(1, **OPT[1]))
    wr = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=4, prefix=oracle.index_prefix(7))],
                       n_ps=R) if raw else None
    if raw:
        wr.configure()
        wr.set_optimizer(oracle.Optim(1, **OPT[1]))
    for x in ws:
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
        x.enable_incremental(1 << 13)
    applied = set()
    for step in range(3):
        batches = [make_batch(rng, S, B, [40, 40, 900][:S], max_ids=3) for _ in range(R)]
        torch.cuda.synchronize()
        W.group_forward(ws, [to_dev_ids(b[0], DEV) for b in batches], B,
                        row_offs=[to_dev_i32(b[1], DEV) for b in batches], slot_occ_offs=[b[2] for b in batches])
        torch.cuda.synchronize()
        grads, octxs = [], []
        for r, (ids, ro, so) in enumerate(batches):  # the oracle as the owners run it: every lookup, then rank order
            g = _grads(rng, S, B, dim)
            if step == 1 and r == 0:
                g[0, 3, 1] = np.nan  # rank 0's slot 0 is dropped; other ranks' entries of its signs still apply
            grads.append(g)
            octxs.append(w.forward(ids, ro, B, training=True)[1])
        for r in range(R):
            per = [w.ctx_signs(octxs[r], i) for i in range(S)]
            st = w.backward(octxs[r], [grads[r][i] for i in range(S)])
            for i in range(S):
                if st[i] == 0:
                    applied.update(int(x) for x in per[i])
        W.group_backward(ws, [[torch.from_numpy(np.ascontiguousarray(g[i])).to(DEV) for i in range(S)] for g in grads])
        torch.cuda.synchronize()
        if raw:
            rb = [ragged_with_multiplicities(rng, B, [5, 3], 3) for _ in range(R)]
            res = RW.group_forward_raw(rws, [to_dev_ids(b[0], DEV) for b in rb], B, 4,
                                       row_offs=[to_dev_i32(b[1], DEV) for b in rb])
            torch.cuda.synchronize()
            rgrads, rctx = [], []
            for r, (ids, ro) in enumerate(rb):
                rctx.append(wr.forward_raw(0, ids, ro, B)[4])
                uniq = ids[np.sort(np.unique(ids, return_index=True)[1])]
                gr = (rng.standard_normal((uniq.size, dim)) * 1e-2).astype(np.float32)
                if step == 2 and r == R - 1:
                    gr[0, 0] = np.nan  # the whole request is dropped
                rgrads.append((uniq, gr))
            for r in range(R):
                uniq, gr = rgrads[r]
                if wr.backward_raw(0, rctx[r], gr) == 0:
                    applied.update(int(x) for x in oracle.add_prefix(uniq, 8, oracle.index_prefix(7)))
            rgrads = [g for _, g in rgrads]
            RW.group_backward_raw(rws, [torch.from_numpy(g).to(DEV) for g in rgrads])
            torch.cuda.synchronize()
    every = np.array(sorted(applied), U64)
    owner = oracle.shard_of(every, R)
    for r, x in enumerate(ws):
        assert x.status() == (False, False)
        got, ent, n_skip = x.take_incremental()
        assert n_skip == 0
        assert got.view(U64).tolist() == every[owner == r].tolist()
        for k, sg in enumerate(got.view(U64)):  # the summation slots' oracle, or the raw slot's
            ref = w.get_entry(int(sg))
            if ref is None:
                ref = wr.get_entry(int(sg))
            assert ref is not None and ref.tobytes() == ent[k].tobytes(), (r, int(sg))
        assert x.incremental_stats()["held"] == 0


@pytest.mark.parametrize("R,groups,raw", [(2, [0, 1], False), (3, [0, 0, 1], False), (2, [0, 0], True),
                                          (3, [0], True)])
def test_sharded_owner_marks(torch_cuda, oracle, R, groups, raw):
    """Each owner's taken set is the union over ranks of the applied entries whose sign it owns; requesters mark
    nothing of other owners' signs."""
    _sharded(torch_cuda, oracle, R, groups, raw)
