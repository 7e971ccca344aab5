"""GPU: contexts of up to PB_MAX_SLOTS = 128 slots, and feature groups of many slots, against the oracle bit for bit.

A context's per-slot state is held in slot-indexed tables and four-word slot masks (slot >> 5): the dead-slot mask of
every reduce kernel, the round masks of shared feature groups, the applied mask of the incremental marks, the owner's
Adam group bits; k_nan_scan runs with grid.y = n_slots, k_slot_status and k_adam_advance as one block of 128 threads;
the warm and hot work cursors are kept per round.  So the settings that live in those tables (NaN gradients, skipped
slots, sqrt scaling, loss scales, hot items) are put at the slots on either side of each word boundary:
31, 32, 63, 64, 95, 96 and 127.  Outputs are compared with a sample-order model of the pooled forward (and with the
oracle's, exactly where a sample holds one id), statuses and every touched entry with the oracle (Adagrad in its
exact-rsqrt mode).  The last part drives the persia_core surface with more than 128 summation slots of one dim, which
it splits into contexts of at most 128 slots without splitting a feature group."""
import os
import zlib

import numpy as np
import pytest

from util import (DEV, _seed_rows, batch_with_multiplicities, entries_equal, full_row_off, held_rows, make_batch, pair,
                  pool_model, same_bits, slot_signs, to_dev_i32, to_dev_ids)

pytestmark = pytest.mark.gpu
SGD, ADAGRAD, ADAGRAD_VW, ADAM = 0, 1, 2, 3
KINDS = (SGD, ADAGRAD, ADAGRAD_VW, ADAM)
OPT = {SGD: dict(lr=0.05, wd=0.001), ADAGRAD: dict(lr=0.02, init_acc=0.01, eps=1e-10),
       ADAGRAD_VW: dict(lr=0.02, init_acc=0.01, eps=1e-10), ADAM: dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8)}
EDGE = (31, 32, 63, 64, 95, 96, 127)  # the slots on either side of every word of a slot mask
WARM_MAX = 32  # items of more occurrences are hot


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


def _edges(S):
    return [s for s in EDGE if s < S]


def _csr(counts, rng, card):
    """counts [S, B] ids per sample -> ids (card: per-slot cardinality), row_off, slot_off."""
    S, B = counts.shape
    row_off = np.zeros(S * B + 1, np.uint32)
    row_off[1:] = np.cumsum(counts.reshape(-1))
    ids = np.concatenate([rng.integers(0, card, size=int(counts[s].sum()), dtype=np.uint64) for s in range(S)])
    return ids, row_off, [int(row_off[s * B]) for s in range(S + 1)]


def _layout(rng, S, B, layout, card=40):
    """One batch of S slots.  Layouts:
      uniform         one id per sample: no row_off, SlotsDev.uniform set (slot_of_occ's shortcut)
      ragged          0..3 ids per sample; slots 0, S-1 and the run 30..34 across the first word boundary are empty
                      (slot_of_occ's binary search over occ_off with repeated offsets, empty dedup regions)
      single          every slot holds exactly one occurrence (regions of 2 * 1 + 2 cells)
      ragged_uniform  ragged, but every slot holds the same number of occurrences: uniform is set while row_off is given"""
    if layout == "uniform":
        return make_batch(rng, S, B, card)
    counts = np.zeros((S, B), np.int64)
    if layout == "ragged":
        counts = rng.integers(0, 4, size=(S, B))
        for s in [0, S - 1] + list(range(30, 35)):
            if s < S:
                counts[s] = 0
    elif layout == "single":
        counts[np.arange(S), rng.integers(0, B, size=S)] = 1
    else:
        assert layout == "ragged_uniform"
        base = rng.integers(0, 4, size=B)
        base[:2] = [0, 3]  # (ragged for sure)
        for s in range(S):
            counts[s] = rng.permutation(base)
    return _csr(counts, rng, card)


def _step(torch, oracle, s, ctx, w, pf, batch, B, dim, rng, seen, sqrt=None, scales=None, nan=(), skip=(), stats=False,
          f32=False):
    """One training step of the GPU context and the oracle.  The forward is compared bit for bit with the sample-order
    model over the rows the table holds after it (and with the oracle where a sample holds at most one id: the oracle
    sums a sample's ids in another order); statuses must equal the oracle's and name exactly the NaN and skipped slots."""
    ids, row_off, slot_off = batch
    S = ctx.n_slots
    got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=to_dev_i32(row_off, DEV) if row_off is not None else None,
                      training=True).cpu().numpy()
    signs = slot_signs(oracle, ids, slot_off, pf)
    if stats:
        want = dict(items=0, cold=0, warm=0, hot=0)
        for i in range(S):
            c = np.unique(signs[slot_off[i]:slot_off[i + 1]], return_counts=True)[1]
            want["items"] += c.size
            want["cold"] += int((c == 1).sum())
            want["warm"] += int(((c >= 2) & (c <= WARM_MAX)).sum())
            want["hot"] += int((c > WARM_MAX).sum())
        st = ctx.batch_stats()
        assert {k: st[k] for k in want} == want, (st, want)
        assert st["occurrences"] == ids.size
    model = pool_model(held_rows(torch, oracle, [s], signs), signs, row_off, B, sqrt, dim=dim) if ids.size else None
    ro = row_off if row_off is not None else full_row_off(S, B)
    want, octx = w.forward(ids, ro, B, training=True)
    one = np.diff(ro).reshape(S, B) <= 1
    for i in range(S):
        if model is not None:
            assert same_bits(got[i], model[i]), i
        assert same_bits(got[i][one[i]], want[i][one[i]]), i
        seen.update(w.ctx_signs(octx, i).tolist())
    g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float32 if f32 else np.float16)
    for i in nan:
        g[i, B // 2, dim - 1] = np.nan
    grads = [None if i in skip else torch.from_numpy(g[i]).to(DEV) for i in range(S)]
    st = ctx.backward(s, grads, scales=scales, want_status=True).cpu().numpy().tolist()
    ost = w.backward(octx, [g[i] for i in range(S)], scale=scales, skip=[int(i in skip) for i in range(S)])
    assert st == ost
    assert [i for i in range(S) if st[i] == 2] == sorted(nan) and [i for i in range(S) if st[i] == 1] == sorted(skip)


def _check_rows(torch, s, w, seen):
    entries_equal(torch, s, w, np.array(sorted(seen), np.uint64))
    assert len(s) == w.ps_len(0)


# ---------------------------------------------------------------------------------------------- 1. slot counts
@pytest.mark.parametrize("S", [31, 32, 33, 64, 65, 127, 128])
@pytest.mark.parametrize("kind", KINDS)
def test_slot_counts(torch_cuda, pb, oracle, S, kind):
    """S slots of one id per sample (the uniform shortcut), three steps.  NaN gradients, skipped slots and loss scales
    of 4 sit only at the word-edge slots below S (at S - 1 when S < 32), and their roles turn at every step: a third of
    the edge slots carries a NaN, a third is skipped, the rest applies its scaled gradient, so every edge slot is dead
    in some step and live and scaled in another.  k_nan_scan's grid.y rows, the dead-slot mask words of the cold, warm
    and hot reduces, the per-slot 1/scale and k_slot_status's thread per slot; Adam's k_adam_advance over S groups."""
    torch = torch_cuda
    rng = np.random.default_rng(1000 * kind + S)
    B, dim = 64, (16 if kind % 2 else 33)
    edges = _edges(S) or [S - 1]
    scales = [4.0 if i in edges else 1.0 for i in range(S)]
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, optim_kw=OPT[kind])
    seen = set()
    for step in range(3):
        nan, skip = edges[step % 3::3], edges[(step + 1) % 3::3]
        _step(torch, oracle, s, ctx, w, pf, _layout(rng, S, B, "uniform"), B, dim, rng, seen, scales=scales, nan=nan,
              skip=skip, f32=kind == ADAGRAD_VW)
    _check_rows(torch, s, w, seen)


# ---------------------------------------------------------------------------------------------- 2. layouts
@pytest.mark.parametrize("layout,S,kind", [
    ("ragged", 128, SGD), ("ragged", 65, ADAGRAD), ("ragged", 128, ADAM), ("ragged", 33, ADAGRAD_VW),
    ("single", 128, ADAGRAD), ("single", 33, ADAM), ("ragged_uniform", 128, ADAGRAD_VW), ("ragged_uniform", 64, SGD),
    ("uniform", 128, ADAM)])
def test_layouts(torch_cuda, pb, oracle, layout, S, kind):
    """Ragged layouts at many slots (see _layout): slot_of_occ's binary search over occ_off with runs of equal offsets
    across a word boundary, the dedup regions 2 * occ_off[s] + 2 * s of empty and one-occurrence slots, and uniform set
    beside a row_off.  Sqrt scaling at the word-edge slots only (k_expand_pool's per-slot factor), NaN and skipped
    slots there too, over two steps."""
    torch = torch_cuda
    rng = np.random.default_rng([zlib.crc32(layout.encode()), S, kind])
    B, dim = 64, 32
    edges = _edges(S)
    sqrt = [i in edges for i in range(S)]
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, sqrt=sqrt, optim_kw=OPT[kind])
    seen = set()
    for step in range(2):
        nan, skip = (edges[0::2], edges[1::2]) if step == 0 else (edges[1::2], [])
        _step(torch, oracle, s, ctx, w, pf, _layout(rng, S, B, layout), B, dim, rng, seen, sqrt=sqrt, nan=nan, skip=skip,
              stats=True)
    _check_rows(torch, s, w, seen)


# ---------------------------------------------------------------------------------------------- 3. hot items
def _hot_batch(rng, S, B, per_slot):
    ids = np.concatenate([batch_with_multiplicities(rng, B, per_slot(s)) if per_slot(s) else
                          rng.integers(0, 1000, size=B, dtype=np.uint64) for s in range(S)])
    return ids, None, [s * B for s in range(S + 1)]


@pytest.mark.parametrize("mode", ["bitmap", "list"])
@pytest.mark.parametrize("kind", [SGD, ADAGRAD, ADAM])
def test_hot_items_at_word_edges(torch_cuda, pb, oracle, mode, kind):
    """Hot items (> 32 occurrences, k_reduce_hot) and warm items at the word-edge slots of a 128-slot context, with a
    NaN slot and a skipped slot among them and loss scales.
      bitmap  hot items only at the edge slots (B = 300): each finds room in the bitmap pool.
      list    36 hot items in every slot at B = 1200: they need more bitmap words (36 * 128 * 38) than the pool holds,
              so the ones handed out last come with occurrence lists.  No counter shows which mode an item got: this
              rests on pb_ctx_create sizing the pool at max(4096, max_occurrences) words (one per occurrence the
              context holds; the assertion below restates it), with the context sized to the batch.  (The pool holds
              them all below B ~ 1056, whatever the slot count: hence the larger batch.)"""
    torch = torch_cuda
    S = 128
    rng = np.random.default_rng(7 + kind + (mode == "list"))
    if mode == "bitmap":
        B, dim = 300, 64
        per_slot = lambda s: [40, 33, 5, 2] if s in EDGE else None  # noqa: E731
    else:
        B, dim = 1200, 16
        per_slot = lambda s: [33] * 36  # noqa: E731
        assert 36 * S * ((B + 31) // 32) > max(4096, S * B)  # bitmap words wanted > the pool's words
    scales = [8.0 if i in EDGE else 1.0 for i in range(S)]
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, optim_kw=OPT[kind], max_occ=S * B)
    seen = set()
    for step in range(2):
        _step(torch, oracle, s, ctx, w, pf, _hot_batch(rng, S, B, per_slot), B, dim, rng, seen, scales=scales,
              nan=[63 if step == 0 else 96], skip=[64 if step == 0 else 127], stats=True)
    _check_rows(torch, s, w, seen)


# ---------------------------------------------------------------------------------------------- 4. feature groups
def _group_layout(name, S):
    if name == "all128":
        return [0] * S
    if name == "span30_34":  # one group across the first word boundary, every other slot a group of its own
        return [0 if 30 <= i <= 34 else i + 1 for i in range(S)]
    return [i % 3 if i % 4 else 3 + i for i in range(S)]  # three interleaved groups, and singles


@pytest.mark.parametrize("groups", ["all128", "span30_34", "interleaved"])
@pytest.mark.parametrize("kind", KINDS)
def test_feature_groups_of_many_slots(torch_cuda, pb, oracle, groups, kind):
    """Slots of one feature group share rows and are stepped in slot order, one round per slot of the group.
      all128       one group of all 128 slots: 128 rounds.  Ids 0, 1, 2 sit in every slot, id 0 cold, warm or hot in
                   turn (1, 5, 40 occurrences), so its row is stepped 128 times in slot order through the cold, warm
                   and hot reduces; a NaN slot and a skipped slot in the middle of the group (and at word edges) drop
                   their rounds only.
      span30_34    one group of slots 30..34 (round masks across words 0 and 1).
      interleaved  three groups of interleaved slots beside single-slot groups.
    Two batches: a round mask, a bitmap or a cursor left dirty by the first would show in the second."""
    torch = torch_cuda
    S, B, dim = 128, 96, 16 if kind != ADAGRAD_VW else 33
    gl = _group_layout(groups, S)
    rng = np.random.default_rng(31 * kind + len(groups))
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, groups=gl, optim_kw=OPT[kind])
    seen = set()
    plan = [([40, 63], [77, 64]), ([31, 96], [50, 127])]
    for step, (nan, skip) in enumerate(plan):
        ids = np.concatenate([batch_with_multiplicities(rng, B, [[1, 5, 40][i % 3], 3, 2]) if gl.count(gl[i]) > 1 else
                              rng.integers(0, 60, size=B, dtype=np.uint64) for i in range(S)])
        _step(torch, oracle, s, ctx, w, pf, (ids, None, [i * B for i in range(S + 1)]), B, dim, rng, seen,
              scales=[2.0 if i in EDGE else 1.0 for i in range(S)], nan=nan, skip=skip, stats=True)
    _check_rows(torch, s, w, seen)


# ---------------------------------------------------------------------------------------------- 5. Adam's pair table
def test_adam_pair_limit(torch_cuda, pb, oracle):
    """A table holds 255 feature-group pairs of beta powers plus pb_update's own.  A 128-slot and a 127-slot context
    train on one table, every slot its own group (255 groups at prefix_bit 8), with a different set of skipped slots at
    every step so that the groups advance different numbers of times.  Then a context at prefix_bit 9 whose one slot
    would be a 256th group: its backward is refused (PB_ERR_CAPACITY) before any kernel is launched, its rows keep what
    its forward admitted, and the next steps of the first two contexts still match the oracle (no pair moved).
    pb_update steps signs of no group in between: it keeps its own pair throughout."""
    from persia_b200 import native as N

    torch = torch_cuda
    rng = np.random.default_rng(255)
    dim, B = 16, 64
    o = OPT[ADAM]
    s = pb.EmbeddingShard(dim, 1 << 16, 0)
    s.set_optimizer(ADAM, lr=o["lr"], beta1=o["b1"], beta2=o["b2"], eps=o["eps"])
    s.configure()
    sides = []
    for groups in (range(0, 128), range(128, 255)):
        pf = [oracle.index_prefix(g) for g in groups]
        w = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pf], n_ps=1)
        w.configure()
        w.set_optimizer(oracle.Optim(ADAM, **o))
        sides.append((pb.BatchContext(len(pf) * B, len(pf) * B, pf), w, pf, set()))
    wu = oracle.Worker([oracle.SlotCfg(dim)], n_ps=1)  # pb_update's signs: no prefix (key 0 in the oracle)
    wu.configure()
    wu.set_optimizer(oracle.Optim(ADAM, **o))
    direct = _seed_rows(torch, oracle, [s], wu, np.arange(1000, 1064, dtype=np.uint64), dim, ADAM, o,
                        lambda x, d: rng.uniform(-0.01, 0.01, size=(x.size, d)), 1)

    def update():
        g = (rng.standard_normal((direct.size, dim)) * 1e-2).astype(np.float32)
        s.update(to_dev_ids(direct, DEV), torch.from_numpy(g).to(DEV))
        wu.ps_update(0, direct, np.full(direct.size, dim, np.uint32), g)

    def train(step):
        for ctx, w, pf, seen in sides:
            S = ctx.n_slots
            skip = [i for i in range(S) if (i * 7 + step) % 5 == 0]
            _step(torch, oracle, s, ctx, w, pf, _layout(rng, S, B, "uniform", card=30), B, dim, rng, seen, skip=skip)

    for step in range(3):
        update()
        train(step)
    pf9 = oracle.index_prefix(0, 9)
    assert pf9 not in [p for side in sides for p in side[2]]
    ctx9 = pb.BatchContext(B, B, [pf9], None, 9)
    w9 = oracle.Worker([oracle.SlotCfg(dim, prefix=pf9)], n_ps=1, prefix_bit=9)
    w9.configure()
    w9.set_optimizer(oracle.Optim(ADAM, **o))
    ids9 = rng.integers(0, 50, size=B, dtype=np.uint64)
    got = ctx9.forward(s, to_dev_ids(ids9, DEV), [0, B], B, training=True).cpu().numpy()
    want, octx9 = w9.forward(ids9, full_row_off(1, B), B, training=True)
    assert same_bits(got[0], want[0])
    signs9 = w9.ctx_signs(octx9, 0)
    torch.cuda.synchronize()
    launches = N.load().pb_launch_count()
    g9 = torch.from_numpy((rng.standard_normal((B, dim)) * 1e-2).astype(np.float16)).to(DEV)
    with pytest.raises(N.PersiaB200Error) as e:
        ctx9.backward(s, [g9])
    assert e.value.code == N.PB_ERR_CAPACITY
    assert N.load().pb_launch_count() == launches
    entries_equal(torch, s, w9, signs9)  # as the forward admitted them
    for step in range(3, 5):
        update()
        train(step)
    for _, w, _, seen in sides:
        entries_equal(torch, s, w, np.array(sorted(seen), np.uint64))
    entries_equal(torch, s, wu, direct)


# ---------------------------------------------------------------------------------------------- 6. incremental marks
def test_incremental_marks_at_128_slots(torch_cuda, pb, oracle):
    """The incremental set after steps with NaN and skipped slots above 32 (the applied mask's words 1..3), two groups
    spanning words: the marked signs equal the host model's, their entries the oracle's."""
    from test_gpu_incremental import check_take, train_step

    torch = torch_cuda
    rng = np.random.default_rng(128)
    S, B, dim = 128, 64, 16
    groups = [0 if i in (31, 32, 95) else 1 if i in (63, 64, 127) else 2 + i for i in range(S)]
    s, ctx, w, pf = pair(pb, oracle, S, dim, ADAGRAD, groups=groups, optim_kw=OPT[ADAGRAD])
    s.enable_incremental(1 << 16)
    model = set()
    for step, (skip, nan) in enumerate([((), ()), ((32, 64, 127), (31, 96)), ((95,), (63, 64, 100)),
                                        ((33, 65, 97), (34, 66, 98))]):
        ids, row_off, slot_off = _layout(rng, S, B, "ragged" if step % 2 else "uniform", card=30)
        g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
        st = train_step(torch, s, ctx, w, ids, row_off, slot_off, B, g, model, skip=skip, nan=nan)
        assert [i for i in range(S) if st[i] == 1] == sorted(skip) and [i for i in range(S) if st[i] == 2] == sorted(nan)
        check_take(torch, s, w, model)


# ---------------------------------------------------------------------------------------------- 7. tier stage
def test_tier_stage_at_128_slots(torch_cuda, pb, oracle):
    """pb_tier_stage of the next batch's 128 slots with a host tier behind a small HBM table: outputs and every entry
    equal the unstaged run's bit for bit, and the stage moved rows."""
    torch = torch_cuda
    S, B, dim, C = 128, 16, 16, 8192
    rng = np.random.default_rng(3)
    pf = [oracle.index_prefix(g) for g in range(S)]
    plan = [make_batch(rng, S, B, 150) for _ in range(12)]
    grads = [(rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16) for _ in plan]

    def run(staged):
        s = pb.EmbeddingShard(dim, C, 0, tier_rows=1 << 16)
        s.set_optimizer(ADAGRAD, lr=0.02, initialization=0.01)
        s.configure()
        s.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=2)
        ctx = pb.BatchContext(S * B, S * B, pf)
        outs = []
        for k, (ids, _, slot_off) in enumerate(plan):
            if staged:
                s.stage(to_dev_ids(ids, DEV), slot_off, pf)
            outs.append(ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B).cpu().numpy().tobytes())
            ctx.backward(s, [torch.from_numpy(grads[k][i]).to(DEV) for i in range(S)])
        torch.cuda.synchronize()
        return s, outs

    s0, o0 = run(False)
    s1, o1 = run(True)
    assert o0 == o1
    assert s1.stage_stats()["staged"] > 0 and s0.stage_stats()["staged"] == 0
    assert s1.tier_stats()["refused"] == 0 and s1.counters()["capacity_refused"] == 0
    signs = np.unique(np.concatenate([slot_signs(oracle, ids, so, pf) for ids, _, so in plan]))
    e0, f0 = s0.get_entries(to_dev_ids(signs, DEV))
    e1, f1 = s1.get_entries(to_dev_ids(signs, DEV))
    assert bool(f0.all()) and bool(f1.all())
    assert e0.cpu().numpy().tobytes() == e1.cpu().numpy().tobytes() and len(s0) == len(s1)


# ---------------------------------------------------------------------------------------------- 8. R virtual ranks
def _sharded(torch, oracle, R, S, dim, kind, B, groups, shards=None, pf=None):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    pf = pf if pf is not None else [oracle.index_prefix(g) for g in groups]
    o = OPT[kind]
    gopt = dict(kind=kind, lr=o["lr"], wd=o.get("wd", 0.0), initialization=o.get("init_acc", 0.01),
                eps=o.get("eps", 1e-10), beta1=o.get("b1", 0.9), beta2=o.get("b2", 0.999))
    ws = W.local_group(R, S, dim, pf, 1 << 16, cap=S * B, optimizer=gopt, max_batch=B, shards=shards,
                       rows_f32=kind == ADAGRAD_VW)
    assert N.OPT_ADAM == ADAM
    for x in ws:  # table storage is allocated on first use, with a device-wide sync: not while a peer spins on a flag
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    return ws, pf


def _oracle_worker(oracle, pf, dim, kind, R):
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pf], n_ps=R)
    w.configure()
    w.set_optimizer(oracle.Optim(kind, **OPT[kind]))
    return w


def _sharded_rows(torch, oracle, ws, w, seen, R):
    signs = np.array(sorted(seen), np.uint64)
    owner = oracle.shard_of(signs, R)
    for r in range(R):
        mine = signs[owner == r]
        ent, found = ws[r].shard.get_entries(to_dev_ids(mine, DEV))
        assert bool(found.all())
        ent = ent.cpu().numpy()
        for k, x in enumerate(mine):
            assert ent[k].tobytes() == w.get_entry(int(x)).tobytes(), (r, k, int(x))
    for x in ws:
        assert x.status() == (False, False) and x.shard.counters()["wait_errors"] == 0


@pytest.mark.parametrize("R,groups,kind,dim", [
    (2, "singles", ADAM, 64), (3, "singles", ADAGRAD_VW, 16), (3, "singles", SGD, 64), (2, "chain", ADAGRAD, 64),
    (3, "chain", ADAM, 64), (2, "chain", ADAGRAD_VW, 16)])
def test_sharded_128_slots(torch_cuda, oracle, R, groups, kind, dim):
    """S = 128 on R virtual ranks (pb_forward_sharded / pb_backward_sharded).
      singles  128 groups of one slot: with Adam the owner's apresent bits of a request fill all four words of a group
               row (k_owner_adam_pows); vectorwise Adagrad takes the per-request owner path.
      chain    all 128 slots one feature group, ids 0..3 in every slot on every rank: every sign's chain holds exactly
               PB_MAX_SLOTS entries, the bound of the owner's chain walks; a NaN slot (rank 0) and a skipped slot (last
               rank) sit inside the chain and the walk passes over them.
    NaN at word-edge slots on rank 0, skips at others on the last rank, loss scales at the edges."""
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    S, B = 128, 64
    rng = np.random.default_rng(R * 10 + kind + len(groups))
    ws, pf = _sharded(torch, oracle, R, S, dim, kind, B, list(range(S)) if groups == "singles" else [0] * S)
    w = _oracle_worker(oracle, pf, dim, kind, R)
    card = 1000 if groups == "singles" else 4
    scales = [4.0 if i in EDGE else 1.0 for i in range(S)]
    seen = set()
    for step, (nan, skip) in enumerate([([31, 64, 77], [32, 95]), ([63, 127], [96, 50])]):
        ids = [make_batch(rng, S, B, card)[0] for _ in range(R)]
        torch.cuda.synchronize()
        outs = W.group_forward(ws, [to_dev_ids(i, DEV) for i in ids], B, training=True)
        torch.cuda.synchronize()
        octx = []
        for r in range(R):
            want, c = w.forward(ids[r], full_row_off(S, B), B, training=True)
            octx.append(c)
            got = outs[r].cpu().numpy()
            for i in range(S):
                assert same_bits(got[i], want[i]), (step, r, i)
                seen.update(w.ctx_signs(c, i).tolist())
        g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16)
        for i in nan:
            g[0, i, B // 3, dim - 1] = np.nan
        dg = [[None if (r == R - 1 and i in skip) else torch.from_numpy(g[r, i]).to(DEV) for i in range(S)]
              for r in range(R)]
        torch.cuda.synchronize()
        sts = W.group_backward(ws, dg, scales=scales, want_status=True)
        torch.cuda.synchronize()
        for r in range(R):
            sk = [int(r == R - 1 and i in skip) for i in range(S)]
            ost = w.backward(octx[r], [g[r, i] for i in range(S)], scale=scales, skip=sk)
            assert sts[r].cpu().numpy().tolist() == ost, (step, r)
    _sharded_rows(torch, oracle, ws, w, seen, R)


def test_sharded_chunk_workers_share_tables(torch_cuda, oracle):
    """What persia_core does on R GPUs with more than 128 summation slots of one dim: one sharded worker per chunk of
    slot_chunks, all on the rank's one table, driven in chunk order (forwards, then backwards).  180 slots: 140 groups
    of one slot and one of 40 (slots 100..139, moved whole into the second chunk), Adam, R = 2, against one oracle
    worker holding all 180 slots."""
    from persia_b200.persia_core import slot_chunks
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, S, B, dim, kind = 2, 180, 64, 16, ADAM
    groups = [200 if 100 <= i < 140 else i for i in range(S)]
    pf = [oracle.index_prefix(g) for g in groups]
    chunks = slot_chunks(pf)
    assert chunks == [list(range(100)), list(range(100, S))]
    workers = []
    for c in chunks:
        ws, _ = _sharded(torch, oracle, R, len(c), dim, kind, B, None, shards=[x.shard for x in workers[0]]
                         if workers else None, pf=[pf[i] for i in c])
        workers.append(ws)
    w = _oracle_worker(oracle, pf, dim, kind, R)
    rng = np.random.default_rng(180)
    seen = set()
    for step in range(3):
        ids = [make_batch(rng, S, B, 50)[0] for _ in range(R)]
        torch.cuda.synchronize()
        outs = [W.group_forward(ws, [to_dev_ids(ids[r][c[0] * B:(c[-1] + 1) * B], DEV) for r in range(R)], B)
                for c, ws in zip(chunks, workers)]
        torch.cuda.synchronize()
        g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float16)
        for c, ws in zip(chunks, workers):
            W.group_backward(ws, [[torch.from_numpy(g[r, i]).to(DEV) for i in c] for r in range(R)])
        torch.cuda.synchronize()
        octx = []
        for r in range(R):  # every rank's request is looked up before any is applied, ranks in rank order
            want, c = w.forward(ids[r], full_row_off(S, B), B, training=True)
            octx.append(c)
            for k, ch in enumerate(chunks):
                got = outs[k][r].cpu().numpy()
                for j, i in enumerate(ch):
                    assert same_bits(got[j], want[i]), (step, r, i)
                    seen.update(w.ctx_signs(c, i).tolist())
        for r in range(R):
            w.backward(octx[r], [g[r, i] for i in range(S)])
    _sharded_rows(torch, oracle, workers[0], w, seen, R)


# ---------------------------------------------------------------------------------------------- 9. persia_core surface
def surface_config(n_raw=0):
    """300 summation slots of dim 16: 220 groups of one slot, feature groups of 50 and of 30 (222 groups, under the 255
    prefix_bit 8 allows), and n_raw raw slots of the same dim."""
    slots = {f"s{i}": {"dim": 16} for i in range(300)}
    slots.update({f"r{i}": {"dim": 16, "embedding_summation": False, "sample_fixed_size": 3} for i in range(n_raw)})
    return {"feature_index_prefix_bit": 8, "slots_config": slots,
            "feature_groups": {"ga": [f"s{i}" for i in range(40, 90)], "gb": [f"s{i}" for i in range(150, 300, 5)]}}


def surface_batch(pc, rng, B, card=40, n_raw=0):
    b = pc.data.PersiaBatch()
    ids = {}
    for i in range(300):
        ids[f"s{i}"] = rng.integers(0, card, size=B, dtype=np.uint64)
        b.add_id_type_feature_with_single_id(ids[f"s{i}"], f"s{i}")
    for i in range(n_raw):
        ids[f"r{i}"] = [rng.integers(0, card, size=rng.integers(0, 4), dtype=np.uint64) for _ in range(B)]
        b.add_id_type_feature(ids[f"r{i}"], f"r{i}")
    b.add_label(np.zeros((B, 1), np.float32), np.dtype(np.float32), "y")
    b.converted_id_type_features2embedding_tensor(True)
    return b, ids


def surface_steps(pc, ctx, rng, B, steps, oracle_worker=None, card=40, n_raw=0, before_forward=None):
    """`steps` training steps through get_embedding_from_data and Backward, gradients made in torch (a raw slot's
    [U, dim] f32 one as persia/ctx.py builds it); the summation outputs are compared with the oracle worker's (one
    request of all 300 slots) when one is given.  before_forward(batch) runs before each forward.  Returns the outputs
    of every step (f16 arrays: the summation slots', then each raw slot's distinct-sign table) and the signs seen."""
    import torch
    import torch.utils.dlpack as dl

    names = [f"s{i}" for i in range(300)]
    bwd = pc.backward.Backward(4)
    outs, seen = [], set()
    for step in range(steps):
        b, ids = surface_batch(pc, rng, B, card, n_raw)
        if before_forward is not None:
            before_forward(b)
        tb = ctx.get_embedding_from_data(b, 0)
        keep = [e.get_raw_embedding()[0] if e.is_raw_embedding() else e.get_sum_embedding()
                for e in tb.consume_all_id_type_feature_embedding_tensors()]
        gb = tb.create_gradient_batch()
        grads, got = {}, {}
        skipped = {f"s{(step * 37) % 300}", "s60"}  # a skipped slot inside feature group ga
        for t in keep:
            n, x = t.name, dl.from_dlpack(t.dlpack)
            got[n] = x.cpu().numpy()
            outs.append(got[n])
            if n in skipped:
                gb.add_skipped_gradient(n)
            elif n in ids and n not in names:  # a raw slot: rows [1, U] of its table are its distinct signs
                if x.shape[0] > 1:
                    g = torch.from_numpy((rng.standard_normal((x.shape[0] - 1, x.shape[1])) * 1e-2)
                                         .astype(np.float32)).to(x.device)
                    grads[n] = g
                    gb.add_gradient(n, g.data_ptr(), list(g.shape), False, 1.0)
            else:
                g = torch.from_numpy((rng.standard_normal(tuple(x.shape)) * 1e-2).astype(np.float16)).to(x.device)
                grads[n] = g
                gb.add_gradient(n, g.data_ptr(), list(g.shape), True, 1.0)
        torch.cuda.synchronize()
        bwd.update_id_type_feature_gradient_batched(gb)
        torch.cuda.synchronize()
        assert bwd.dropped == 0
        if oracle_worker is not None:
            ro = full_row_off(300, B)
            want, octx = oracle_worker.forward(np.concatenate([ids[n] for n in names]), ro, B, training=True)
            for i, n in enumerate(names):
                assert same_bits(got[n], want[i]), (step, n)
                seen.update(oracle_worker.ctx_signs(octx, i).tolist())
            g_all = [grads[n].cpu().numpy() if n in grads else np.zeros((B, 16), np.float16) for n in names]
            oracle_worker.backward(octx, g_all, skip=[int(n in skipped) for n in names])
    return outs, seen


def _surface(impl):
    pc = impl.install()
    ctx = pc.PersiaCommonContext(10, 0, 1, 0)
    opt = pc.optim.OptimizerBase()
    opt.init_adam(0.01, (0.9, 0.999), 1e-8)
    opt.apply()
    ctx.configure_embedding_parameter_servers(-0.01, 0.01, 1.0, True, 10.0)
    return pc, ctx


def test_surface_more_than_128_slots_of_one_dim(oracle):
    """300 summation slots of one dim through set_embedding_config, get_embedding_from_data and Backward, with Adam,
    against one oracle worker holding all 300 slots: persia_core serves them with three contexts of at most 128 slots,
    each feature group whole in one of them (a split group would advance its beta powers twice per step)."""
    from persia_b200 import persia_core as impl
    from persia_b200.persia_core import _S, parse_embedding_config

    impl.reset()
    try:
        cfg = surface_config()
        impl.set_embedding_config(cfg)
        pc, ctx = _surface(impl)
        _, slots = parse_embedding_config(cfg)
        w = oracle.Worker([oracle.SlotCfg(16, prefix=s.index_prefix) for s in slots], n_ps=1)
        w.configure(-0.01, 0.01, 1.0, True, 10.0)
        w.set_optimizer(oracle.Optim(ADAM, lr=0.01, b1=0.9, b2=0.999, eps=1e-8))
        _, seen = surface_steps(pc, ctx, np.random.default_rng(300), 64, 3, oracle_worker=w)
        g = _S.groups[16]
        assert sorted(len(k) for k in g["ctx"]) == [44, 128, 128]
        entries_equal(None, g["shard"], w, np.array(sorted(seen), np.uint64))
        assert ctx.get_embedding_size() == [w.ps_len(0)]
    finally:
        impl.reset()


def test_surface_stage_more_than_128_slots(monkeypatch):
    """The same 300 summation slots and four raw slots of the dim (304 slots) with a host-memory tier behind the HBM
    rows: the Forward engine's stage (persia_core._stage) runs before every forward and issues pb_tier_stage in calls of
    at most 128 slots.  It moves tier-held signs back (its counters move), and every output and entry equals the
    unstaged run's.  Sizes: ~600 signs per step and 7 requests per step, under the 768 rows the table keeps free
    (PERSIA_B200_HBM_ROWS / 16), so neither run ever refuses an admission; ~20000 signs over the run, so most steps after
    the 20th need rows that eviction moved to the tier."""
    from persia_b200 import persia_core as impl
    from persia_b200.persia_core import _S

    def run(staged):
        impl.reset()
        try:
            impl.set_embedding_config(surface_config(n_raw=4))
            pc, ctx = _surface(impl)
            outs, _ = surface_steps(pc, ctx, np.random.default_rng(304), 2, 40, card=200, n_raw=4,
                                    before_forward=impl._stage if staged else None)
            sh = _S.groups[16]["shard"]
            assert sh.host_tier is not None
            ts = sh.tier_stats()
            assert sh.counters()["capacity_refused"] == 0 and ts["refused"] == 0 and ts["dropped"] == 0, ts
            assert ts["restored"] > 0, ts  # (the tier was used, staged or not)
            signs = sh.export_signs()[0].cpu().numpy().view(np.uint64)
            tier = sh._export_table(sh.host_tier.h)[0].cpu().numpy().view(np.uint64)
            keys = np.unique(np.concatenate([signs, tier]))
            ent, found = sh.get_entries(to_dev_ids(keys, DEV))
            assert bool(found.all())
            return outs, keys, ent.cpu().numpy(), sh.stage_stats()
        finally:
            impl.reset()

    monkeypatch.setenv("PERSIA_B200_CAPACITY", str(1 << 16))
    monkeypatch.setenv("PERSIA_B200_HBM_ROWS", "12288")
    o0, k0, e0, st0 = run(False)
    o1, k1, e1, st1 = run(True)
    assert st0 == {"staged": 0, "skipped": 0} and st1["staged"] > 0, (st0, st1)
    assert len(o0) == len(o1) == 40 * 304
    for k, (a, b) in enumerate(zip(o0, o1)):
        assert same_bits(a, b), (k // 304, k % 304)
    assert k0.tobytes() == k1.tobytes() and e0.tobytes() == e1.tobytes()


def _two_process_rank(rank, world, port, result_dir):
    """One rank of test_two_process_more_than_128_slots_matches_oracle: three steps of the surface, then its outputs
    and the rows its table holds, saved for the oracle replay."""
    import torch
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    from persia_b200 import persia_core as impl
    from persia_b200.persia_core import _S

    impl.reset()
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        impl.set_embedding_config(surface_config())
        pc = impl.install()
        ctx = pc.PersiaCommonContext(10, rank, world, rank)
        opt = pc.optim.OptimizerBase()
        opt.init_adam(0.01, (0.9, 0.999), 1e-8)
        opt.apply()
        ctx.configure_embedding_parameter_servers(-0.01, 0.01, 1.0, True, 10.0)
        outs, _ = surface_steps(pc, ctx, np.random.default_rng(500 + rank), 64, 3)
        g = _S.groups[16]
        assert len(g["workers"]) == 3
        signs = g["shard"].export_signs()[0].cpu().numpy().view(np.uint64)
        ent = g["shard"].get_entries(to_dev_ids(signs, f"cuda:{rank}"))[0].cpu().numpy()
        outs = np.stack(outs)
        np.savez(os.path.join(result_dir, f"r{rank}.npz"), outs=outs, signs=signs, ent=ent)
        dist.barrier()
    finally:
        impl.reset()
        dist.destroy_process_group()


def test_two_process_more_than_128_slots_matches_oracle(torch_cuda, oracle, tmp_path):
    """Two processes (one per GPU), 300 summation slots of one dim with Adam: each rank serves them with three sharded
    workers on its one table, in chunk order.  Each rank's outputs and the union of the ranks' rows equal an oracle
    worker with two parameter servers driven by the same batches."""
    torch = torch_cuda
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import socket

    from persia_b200 import persia_core as impl
    from persia_b200.persia_core import parse_embedding_config

    import torch.multiprocessing as mp

    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    mp.spawn(_two_process_rank, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    # the oracle: the same batches (each rank's seeded draws), two parameter servers, ranks applied in rank order
    names = [f"s{i}" for i in range(300)]
    _, slots = parse_embedding_config(surface_config())
    w = oracle.Worker([oracle.SlotCfg(16, prefix=s.index_prefix) for s in slots], n_ps=2)
    w.configure(-0.01, 0.01, 1.0, True, 10.0)
    w.set_optimizer(oracle.Optim(ADAM, lr=0.01, b1=0.9, b2=0.999, eps=1e-8))
    impl.reset()
    pc = impl.install()
    rngs = [np.random.default_rng(500 + r) for r in range(2)]
    res = [np.load(tmp_path / f"r{r}.npz") for r in range(2)]
    for step in range(3):
        octx, grads, skips = [], [], []
        for r in range(2):
            b, ids = surface_batch(pc, rngs[r], 64)
            want, c = w.forward(np.concatenate([ids[n] for n in names]), full_row_off(300, 64), 64, training=True)
            octx.append(c)
            skipped = {f"s{(step * 37) % 300}", "s60"}
            g = []
            for i, n in enumerate(names):
                got = res[r]["outs"][step * 300 + i]
                assert same_bits(got, want[i]), (step, r, n)
                if n in skipped:
                    g.append(np.zeros((64, 16), np.float16))
                else:
                    g.append((rngs[r].standard_normal((64, 16)) * 1e-2).astype(np.float16))
            grads.append(g)
            skips.append([int(n in skipped) for n in names])
        for r in range(2):
            w.backward(octx[r], grads[r], skip=skips[r])
    for r in range(2):
        for k, x in enumerate(res[r]["signs"]):
            assert res[r]["ent"][k].tobytes() == w.get_entry(int(x)).tobytes(), (r, k)
    impl.reset()
