"""GPU: the hash sets a batch goes through before any row is read, at clustered homes, at region and set ends, and the
index prefix at every prefix width.

Nothing downstream of these sets sees a sign again, only its cell and its item number, so a probe that wraps wrongly, a
reserved cell that is missed or a prefix that differs at one residue changes which rows a batch reads and steps.  The
keys come from tests/hash_set_keys.py, whose docstring restates every home formula used here:

  k_dedup        every slot holds many distinct signs homed on its region's last cell (off + size - 1), so the probes
                 wrap to `off` and fill the region; a prefix-0 slot also holds the sign 2^64-1, whose reserved cell
                 (off + size) follows that cluster.  Multiplicities put clustered items in the cold, warm and hot lists.
  k_link_items   slots of one feature group hold the same clustered signs: on R virtual ranks a sign is found again in the
                 other slots' regions by find_in_slot, which must follow k_dedup's probe sequence.
  k_raw_insert   a cluster on the raw set's last cell (cells - 1, wrapping to 0) and the sign 2^64-1 (cell `cells`).
  inc_find / inc_claim   more than 8 signs whose path starts in the incremental set's last bucket: the path wraps to
                 cell 0.  Marking the same signs again must find every one of them.
  indices_add_prefix  prefix bits 1..63 at ids 0, 1, m-1, m, m+1, multiples of m, 2^63 and 2^64-1 (m = 2^(64-b) - 1).
                 Ids equal mod m are one sign and so one item of their slot; at b = 63 (m = 1) a slot is one hot item.

Everything is compared bit for bit with the oracle (Adagrad and Adam in its exact-rsqrt mode): forward outputs, slot
statuses and every touched entry; BatchContext.batch_stats() is compared with counts made in numpy.  The oracle, like
the reference, dedups raw ids before it adds the prefix; the prefix-width tests give it each id's residue mod m (the
same sign), so that it sees the one item the GPU keeps.  Every set keeps more free cells than it holds signs, so a
correct probe always ends."""
import numpy as np
import pytest

import hash_set_keys as K
from util import DEV, _gpu_optim, _read_rows, entries_equal, full_row_off, to_dev_i32, to_dev_ids

pytestmark = pytest.mark.gpu
U64 = np.uint64
M64 = K.M64


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
       3: dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8)}


def _shard(pb, oracle, dim, kind, cap=1 << 14, tier_rows=0):
    s = pb.EmbeddingShard(dim, cap, 0, tier_rows=tier_rows)
    s.set_optimizer(**_gpu_optim(kind, OPT[kind]))
    s.configure()
    return s


def _worker(oracle, cfgs, kind, n_ps=1, prefix_bit=8):
    w = oracle.Worker(cfgs, n_ps=n_ps, prefix_bit=prefix_bit)
    w.configure()
    w.set_optimizer(oracle.Optim(kind, **OPT[kind]))
    return w


def _class_counts(slot_signs):
    """batch_stats() of a batch whose slots hold these (prefixed) signs, one entry per occurrence."""
    out = dict(items=0, cold=0, warm=0, hot=0)
    for s in slot_signs:
        c = np.unique(np.asarray(s, U64), return_counts=True)[1]
        out["items"] += c.size
        out["cold"] += int((c == 1).sum())
        out["warm"] += int(((c >= 2) & (c <= 32)).sum())
        out["hot"] += int((c > 32).sum())
    return out


def _check_stats(ctx, slot_signs):
    st = ctx.batch_stats()
    want = _class_counts(slot_signs)
    assert {k: st[k] for k in want} == want, (st, want)
    assert st["occurrences"] == sum(len(s) for s in slot_signs)
    return want


def _grads(rng, shape, f32):
    return (rng.standard_normal(shape) * 1e-2).astype(np.float32 if f32 else np.float16)


def _step(torch, s, ctx, w, ids, oracle_ids, slot_off, B, g):
    """One batched training step on the GPU (ids) and in the oracle (oracle_ids): outputs and statuses bit for bit."""
    S = ctx.n_slots
    got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B).cpu().numpy()
    want, octx = w.forward(oracle_ids, full_row_off(S, B), B, training=True)
    for i in range(S):
        assert got[i].tobytes() == want[i].tobytes(), f"forward, slot {i}"
    stats = ctx.batch_stats()
    st = ctx.backward(s, [torch.from_numpy(np.ascontiguousarray(g[i])).to(DEV) for i in range(S)],
                      want_status=True).cpu().numpy().tolist()
    assert st == w.backward(octx, [g[i] for i in range(S)]) == [0] * S
    return stats


def _cluster_slot(rng, counts, homed, extra=()):
    """One slot's ids: homed[k] repeated counts[k] times (every other homed id once), plus `extra`, shuffled."""
    reps = np.ones(homed.size, np.int64)
    reps[:len(counts)] = counts
    ids = np.concatenate([np.repeat(homed, reps), np.asarray(extra, U64)])
    return ids[rng.permutation(ids.size)]


# ---------------------------------------------------------------------------------------------- k_dedup
@pytest.mark.parametrize("dim,kind,f32", [(12, 1, False), (64, 1, True), (64, 0, False), (12, 3, True), (33, 1, False)])
def test_dedup_clusters_at_region_ends(torch_cuda, pb, oracle, dim, kind, f32):
    """Three slots of B ids; in each, every distinct sign is homed on the region's last cell.  Slot 1 has no prefix and
    also carries 2^64-1 three times (the reserved cell right after the cluster's home)."""
    torch = torch_cuda
    rng = np.random.default_rng(dim * 10 + kind)
    S, B = 3, 300
    pf = [oracle.index_prefix(0), 0, oracle.index_prefix(1)]
    slot_off = [i * B for i in range(S + 1)]
    counts = [40, 33, 32, 17, 2]  # hot, hot, warm at its bound, warm, warm; then cold
    homed = []
    for i in range(S):
        off, size = K.set_region(slot_off, i)
        n_distinct = B - sum(counts) + len(counts) - (3 if pf[i] == 0 else 0)
        h = K.homed_ids(lambda x: K.dedup_home(x, off, size), off + size - 1, n_distinct, 8, pf[i], start=(i + 1) << 40)
        assert n_distinct + (pf[i] == 0) <= B < size  # within the region's load bound
        homed.append(h)
    s = _shard(pb, oracle, dim, kind)
    ctx = pb.BatchContext(S * B, S * B, pf)
    w = _worker(oracle, [oracle.SlotCfg(dim, prefix=p) for p in pf], kind)
    seen = set()
    for step in range(3):
        ids = [_cluster_slot(rng, counts, homed[i], [M64] * 3 if pf[i] == 0 else ()) for i in range(S)]
        signs = [K.prefix_np(ids[i], 8, pf[i]) for i in range(S)]
        flat = np.concatenate(ids)
        stats = _step(torch, s, ctx, w, flat, flat, slot_off, B, _grads(rng, (S, B, dim), f32))
        want = _class_counts(signs)
        assert {k: stats[k] for k in want} == want
        assert want["hot"] == 6 and want["warm"] == 3 * 3 + 1  # (2^64-1 is warm)
        seen.update(int(x) for x in np.concatenate(signs))
    assert M64 in seen
    entries_equal(torch, s, w, np.array(sorted(seen), U64))


# ---------------------------------------------------------------------------------------------- k_link_items
def _group_batch(rng, homed, S, B):
    """S slots of one feature group over the same clustered signs: slot 0 holds all of them, slot 1 the first two
    thirds, slot 2 every other one; the first signs are hot and warm in every slot."""
    out = []
    for i in range(S):
        h = [homed, homed[:2 * homed.size // 3], homed[::2]][i % 3]
        counts = [36, 12, 3]
        h = h[:B - sum(counts) + len(counts)]
        ids = _cluster_slot(rng, counts, h)
        pad = B - ids.size  # fresh cold signs of the slot's own
        out.append(np.concatenate([ids, np.arange(1 << 50, (1 << 50) + pad, dtype=U64) + U64(i << 20)]))
    return out


@pytest.mark.parametrize("R", [1, 2, 3])
def test_shared_feature_group_clusters(torch_cuda, pb, oracle, R):
    """Slots of one feature group hold the same signs, every one homed on the last cell of its slot's region (the
    regions are the same size, so a sign has the same home in each).  The reference steps such a sign once per slot, in
    slot order (R = 1), and once per (rank, slot) on R ranks, where the requester links a sign's entries by finding it
    again in the other slots' regions."""
    torch = torch_cuda
    rng = np.random.default_rng(R)
    S, B, dim, kind = 3, 200, 16, 1
    pf0 = oracle.index_prefix(0)
    slot_off = [i * B for i in range(S + 1)]
    off, size = K.set_region(slot_off, 0)
    homed = K.homed_ids(lambda x: K.dedup_home(x, off, size), off + size - 1, 150, 8, pf0)
    for i in range(S):  # the same home in every slot's region
        o, sz = K.set_region(slot_off, i)
        assert np.all(K.dedup_home(K.prefix_np(homed, 8, pf0), o, sz) == o + sz - 1)
    w = _worker(oracle, [oracle.SlotCfg(dim, prefix=pf0) for _ in range(S)], kind, n_ps=R)
    seen = set()
    if R == 1:
        s = _shard(pb, oracle, dim, kind)
        ctx = pb.BatchContext(S * B, S * B, [pf0] * S)
        for step in range(3):
            ids = _group_batch(rng, homed, S, B)
            flat = np.concatenate(ids)
            stats = _step(torch, s, ctx, w, flat, flat, slot_off, B, _grads(rng, (S, B, dim), step == 1))
            want = _class_counts([K.prefix_np(x, 8, pf0) for x in ids])
            assert {k: stats[k] for k in want} == want
            seen.update(int(x) for x in K.prefix_np(flat, 8, pf0))
        entries_equal(torch, s, w, np.array(sorted(seen), U64))
        return
    from persia_b200.worker import ShardedEmbeddingWorker as W
    from test_gpu_worker_groups import _check_rows, _group

    ws, w, _ = _group(torch, oracle, R, [0] * S, dim, kind, B)
    for step in range(3):
        ids = [np.concatenate(_group_batch(rng, homed, S, B)) for _ in range(R)]
        torch.cuda.synchronize()
        outs = W.group_forward(ws, [to_dev_ids(x, DEV) for x in ids], B, training=True)
        torch.cuda.synchronize()
        octx = []
        for r in range(R):
            want, c = w.forward(ids[r], full_row_off(S, B), B, training=True)
            octx.append(c)
            got = outs[r].cpu().numpy()
            for i in range(S):
                assert got[i].tobytes() == want[i].tobytes(), (step, r, i)
            signs = [K.prefix_np(ids[r][i * B:(i + 1) * B], 8, pf0) for i in range(S)]
            _check_stats(ws[r].ctx, signs)
            seen.update(int(x) for x in np.concatenate(signs))
        g = _grads(rng, (R, S, B, dim), step == 1)
        sts = W.group_backward(ws, [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)],
                               want_status=True)
        torch.cuda.synchronize()
        for r in range(R):
            assert sts[r].cpu().numpy().tolist() == w.backward(octx[r], [g[r, i] for i in range(S)]) == [0] * S
    _check_rows(torch, oracle, ws, w, seen, R)


# ---------------------------------------------------------------------------------------------- k_raw_insert
def _raw_batch(rng, B, max_ids, homed, n_special, start):
    """A ragged raw batch of B samples (0..max_ids ids each): the homed signs 1..4 times each, 2^64-1 n_special times,
    fresh ids for the rest."""
    row_off = np.zeros(B + 1, np.uint32)
    row_off[1:] = np.cumsum(rng.integers(0, max_ids + 1, size=B))
    n = int(row_off[-1])
    ids = np.concatenate([np.repeat(homed, rng.integers(1, 5, size=homed.size)), np.full(n_special, M64, U64)])
    assert ids.size <= n
    ids = np.concatenate([ids, np.arange(start, start + n - ids.size, dtype=U64)])
    return ids[rng.permutation(n)], row_off


def _raw_compare(got, wt, wi, wne, wnum):
    table, index, non_empty, num, counts = got
    U, ne = counts.cpu().numpy().tolist()
    assert U == wt.shape[0] - 1
    assert table[:U + 1].cpu().numpy().tobytes() == wt.tobytes()
    np.testing.assert_array_equal(index.cpu().numpy(), wi)
    assert ne == wne.size
    np.testing.assert_array_equal(non_empty[:ne].cpu().numpy(), wne)
    np.testing.assert_array_equal(num.cpu().numpy().view(np.uint32), wnum)
    return U


@pytest.mark.parametrize("path", ["local", "sharded2"])
@pytest.mark.parametrize("group", [None, 0])
def test_raw_set_cluster_at_the_last_cell(torch_cuda, pb, oracle, path, group):
    """40 signs homed on the raw set's last cell (their probes wrap to cell 0) and the sign 2^64-1 (its own cell past
    the end), in ragged samples longer than sample_fixed_size."""
    torch = torch_cuda
    rng = np.random.default_rng(7 + (group or 0) + (path == "local"))
    dim, kind, fixed, B, max_ids = 16, 1, 3, 128, 6
    pf = oracle.index_prefix(group) if group is not None else 0
    cells = K.raw_cells(B * max_ids)
    homed = K.homed_ids(lambda x: K.raw_home(x, cells), cells - 1, 40, 8, pf)
    cfg = [oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=pf)]
    seen = set()
    if path == "local":
        s = _shard(pb, oracle, dim, kind)
        ctx = pb.BatchContext(B * max_ids, B * max_ids, [pf])
        w = _worker(oracle, cfg, kind)
        for step in range(3):
            ids, ro = _raw_batch(rng, B, max_ids, homed, 3, (1 << 44) + step * 1000)
            got = ctx.forward_raw(s, to_dev_ids(ids, DEV), B, fixed, row_off=to_dev_i32(ro, DEV))
            wt, wi, wne, wnum, octx = w.forward_raw(0, ids, ro, B)
            U = _raw_compare(got, wt, wi, wne, wnum)
            g = _grads(rng, (U, dim), step != 1)
            assert ctx.backward_raw(s, torch.from_numpy(g).to(DEV), want_status=True).item() == 0
            assert w.backward_raw(0, octx, g) == 0
            seen.update(int(x) for x in K.prefix_np(ids, 8, pf))
        entries_equal(torch, s, w, np.array(sorted(seen), U64))
        return
    from persia_b200.worker import ShardedRawWorker as RW

    R = 2
    ws = RW.local_group(R, 1, dim, [pf], 1 << 14, cap=B * max_ids, optimizer=_gpu_optim(kind, OPT[kind]), hyper={},
                        max_batch=B, max_ids_per_sample=max_ids)
    w = _worker(oracle, cfg, kind, n_ps=R)
    shards = [x.shard for x in ws]
    for x in shards:  # table storage is allocated on first use, with a device-wide sync: not while a peer waits
        x.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    for step in range(3):
        batches = [_raw_batch(rng, B, max_ids, homed, 2 + r, (1 << 44) + (step * R + r) * 1000) for r in range(R)]
        res = RW.group_forward_raw(ws, [to_dev_ids(b[0], DEV) for b in batches], B, fixed,
                                   row_offs=[to_dev_i32(b[1], DEV) for b in batches])
        torch.cuda.synchronize()
        octx, grads = [], []
        for r, (ids, ro) in enumerate(batches):
            wt, wi, wne, wnum, c = w.forward_raw(0, ids, ro, B)
            U = _raw_compare(res[r], wt, wi, wne, wnum)
            octx.append(c)
            grads.append(_grads(rng, (U, dim), True))
            seen.update(int(x) for x in K.prefix_np(ids, 8, pf))
        sts = RW.group_backward_raw(ws, [torch.from_numpy(g).to(DEV) for g in grads], want_status=True)
        torch.cuda.synchronize()
        for r in range(R):
            assert sts[r].item() == w.backward_raw(0, octx[r], grads[r]) == 0
    for x in ws:
        assert x.status() == (False, False)
    got, want = _read_rows(torch, oracle, shards, w, np.array(sorted(seen), U64), R)
    assert got.tobytes() == want.tobytes()


# ---------------------------------------------------------------------------------------------- inc_find / inc_claim
def _take_equals(s, model):
    st = s.incremental_stats()
    assert st["held"] == len(model), (st, len(model))
    signs, ent, skipped = s.take_incremental()
    assert skipped == 0 and signs.view(U64).tolist() == sorted(model)
    again, found = s.get_entries(to_dev_ids(signs.view(U64), DEV))
    assert bool(found.all()) and again.cpu().numpy().tobytes() == ent.tobytes()
    assert s.incremental_stats()["held"] == 0 and s.incremental_held() == 0


def test_incremental_set_wraps_past_the_last_bucket(torch_cuda, pb, oracle):
    """Signs whose paths start in the set's last bucket (cells n-8..n-1), marked by pb_backward (12 prefixed signs),
    pb_update (4) and a raw backward (4 and the sign 2^64-1, which has a reserved cell): 20 > 8, so the path wraps to
    cell 0.  Marking them all again holds nothing new; a take returns exactly the model's set and empties it; the same
    signs are then marked again from empty."""
    torch = torch_cuda
    rng = np.random.default_rng(3)
    dim, kind, B = 8, 1, 64
    cap = 128
    n = K.inc_cells(cap)
    last = n // K.BUCKET - 1
    pf = oracle.index_prefix(0)
    home = lambda x: K.inc_bucket(x, n)  # noqa: E731
    a_ids = K.homed_ids(home, last, 12, 8, pf)
    a = K.prefix_np(a_ids, 8, pf)
    b = K.prefix_np(K.homed_ids(home, last, 4, 0, 0, start=1 << 40, avoid=a), 0, 0)
    c = K.prefix_np(K.homed_ids(home, last, 4, 0, 0, start=1 << 41, avoid=np.concatenate([a, b])), 0, 0)
    s = _shard(pb, oracle, dim, kind)
    ctx = pb.BatchContext(B, B, [pf])
    rctx = pb.BatchContext(B, B, [0])
    s.lookup(to_dev_ids(b, DEV), training=True)  # pb_update marks signs that have a row
    s.enable_incremental(cap)

    def mark_all():
        ids = np.concatenate([a_ids, a_ids[:4], np.arange(1 << 45, (1 << 45) + B - 16, dtype=U64)])
        ctx.forward(s, to_dev_ids(ids, DEV), [0, B], B)
        ctx.backward(s, [torch.from_numpy(_grads(rng, (B, dim), False)).to(DEV)])
        fresh = K.prefix_np(ids[16:], 8, pf)
        s.update(to_dev_ids(b, DEV), torch.from_numpy(_grads(rng, (b.size, dim), True)).to(DEV))
        rids = np.concatenate([c, [M64], c[:2]]).astype(U64)
        ro = np.arange(rids.size + 1, dtype=np.uint32)
        _, _, _, _, counts = rctx.forward_raw(s, to_dev_ids(rids, DEV), rids.size, 1, row_off=to_dev_i32(ro, DEV))
        U = int(counts[0])
        assert U == 5
        assert rctx.backward_raw(s, torch.from_numpy(_grads(rng, (U, dim), True)).to(DEV), want_status=True).item() == 0
        return set(int(x) for x in np.concatenate([a, fresh, b, c, [M64]]))

    model = mark_all()
    st = s.incremental_stats()
    assert st["held"] == len(model) == st["inserted"] and st["dropped"] == 0
    assert mark_all() == model
    st = s.incremental_stats()
    assert st["held"] == len(model) == st["inserted"] and st["dropped"] == 0
    _take_equals(s, model)
    model = mark_all()
    _take_equals(s, model)
    assert s.incremental_stats()["dropped"] == 0


def test_incremental_cluster_fills_the_set_exactly(torch_cuda, pb, oracle):
    """A set of capacity 16 (1024 cells): 12 signs of the last bucket, then the same 12 and 8 more.  The 12 are found
    again, so exactly 4 of the 8 get a place and 4 are dropped."""
    torch = torch_cuda
    rng = np.random.default_rng(4)
    dim, cap = 8, 16
    n = K.inc_cells(cap)
    first = K.homed_ids(lambda x: K.inc_bucket(x, n), n // K.BUCKET - 1, 20, 0, 0)
    s = _shard(pb, oracle, dim, 0)
    s.lookup(to_dev_ids(first, DEV), training=True)
    s.enable_incremental(cap)
    s.update(to_dev_ids(first[:12], DEV), torch.from_numpy(_grads(rng, (12, dim), True)).to(DEV))
    st = s.incremental_stats()
    assert (st["held"], st["inserted"], st["dropped"]) == (12, 12, 0)
    again = first[rng.permutation(20)]
    s.update(to_dev_ids(again, DEV), torch.from_numpy(_grads(rng, (20, dim), True)).to(DEV))
    st = s.incremental_stats()
    assert (st["held"], st["inserted"], st["dropped"]) == (16, 16, 4), st
    signs, _, _ = s.take_incremental()
    got = set(signs.view(U64).tolist())
    assert len(got) == 16 and set(first[:12].tolist()) <= got <= set(first.tolist())


# ---------------------------------------------------------------------------------------------- prefix widths
def _width_ids(rng, b, n):
    """n ids (with repeats) drawn from the edge ids of width b and from groups of ids equal mod m."""
    m = K.spacing(b)
    pool = set(int(x) for x in K.edge_ids(b, rng))
    for r in rng.integers(0, m, size=6, dtype=U64, endpoint=False) if m > 1 else [0]:
        for k in rng.integers(0, M64 // m, size=3, dtype=U64, endpoint=True):
            if int(r) + int(k) * m <= M64:
                pool.add(int(r) + int(k) * m)
    pool = np.array(sorted(pool), U64)
    return pool[rng.integers(0, pool.size, size=n)]


def _width_prefixes(oracle, b):
    return [oracle.index_prefix(g, b) for g in ([0, 1] if b > 1 else [0])]


@pytest.mark.parametrize("b", K.PREFIX_BITS)
def test_add_prefix_at_width(torch_cuda, pb, oracle, b):
    rng = np.random.default_rng(b)
    ids = np.concatenate([K.edge_ids(b, rng, n_random=200), _width_ids(rng, b, 300)])
    pf = _width_prefixes(oracle, b) + [0]
    offs = [0, 150, 400, ids.size] if len(pf) == 3 else [0, 300, ids.size]
    got = pb.add_prefix(to_dev_ids(ids, DEV), offs, pf, prefix_bit=b).cpu().numpy().view(U64)
    want = [K.prefix_int(x, b, pf[i]) for i in range(len(pf)) for x in ids[offs[i]:offs[i + 1]].tolist()]
    assert [int(x) for x in got] == want


@pytest.mark.parametrize("b", K.PREFIX_BITS)
def test_training_step_at_width(torch_cuda, pb, oracle, b):
    """Ids equal mod m are one item of their slot; the oracle gets each id's residue."""
    torch = torch_cuda
    rng = np.random.default_rng(100 + b)
    dim, kind, B = 16, 1, 256
    pf = _width_prefixes(oracle, b)
    S = len(pf)
    slot_off = [i * B for i in range(S + 1)]
    s = _shard(pb, oracle, dim, kind)
    ctx = pb.BatchContext(S * B, S * B, pf, prefix_bit=b)
    w = _worker(oracle, [oracle.SlotCfg(dim, prefix=p) for p in pf], kind, prefix_bit=b)
    seen = set()
    for step in range(2):
        ids = [_width_ids(rng, b, B) for _ in range(S)]
        res = np.concatenate([K.residues(ids[i], b, pf[i]) for i in range(S)])
        signs = [K.prefix_np(ids[i], b, pf[i]) for i in range(S)]
        stats = _step(torch, s, ctx, w, np.concatenate(ids), res, slot_off, B, _grads(rng, (S, B, dim), step == 1))
        want = _class_counts(signs)
        assert {k: stats[k] for k in want} == want
        assert want["items"] < sum(np.unique(x).size for x in ids)  # some ids did fold into one sign
        if b == 63:
            assert want == dict(items=S, cold=0, warm=0, hot=S)
        seen.update(int(x) for x in np.concatenate(signs))
    entries_equal(torch, s, w, np.array(sorted(seen), U64))


@pytest.mark.parametrize("b", K.PREFIX_BITS)
def test_raw_slot_at_width(torch_cuda, pb, oracle, b):
    torch = torch_cuda
    rng = np.random.default_rng(200 + b)
    dim, kind, B, fixed = 8, 1, 64, 3
    pf = oracle.index_prefix(0, b)
    s = _shard(pb, oracle, dim, kind)
    ctx = pb.BatchContext(4 * B, 4 * B, [pf], prefix_bit=b)
    w = _worker(oracle, [oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=pf)], kind, prefix_bit=b)
    seen = set()
    for step in range(2):
        ro = np.zeros(B + 1, np.uint32)
        ro[1:] = np.cumsum(rng.integers(0, 5, size=B))
        ids = _width_ids(rng, b, int(ro[-1]))
        got = ctx.forward_raw(s, to_dev_ids(ids, DEV), B, fixed, row_off=to_dev_i32(ro, DEV))
        wt, wi, wne, wnum, octx = w.forward_raw(0, K.residues(ids, b, pf), ro, B)
        U = _raw_compare(got, wt, wi, wne, wnum)
        assert U == np.unique(K.prefix_np(ids, b, pf)).size
        g = _grads(rng, (U, dim), step == 0)
        assert ctx.backward_raw(s, torch.from_numpy(g).to(DEV), want_status=True).item() == 0
        assert w.backward_raw(0, octx, g) == 0
        seen.update(int(x) for x in K.prefix_np(ids, b, pf))
    entries_equal(torch, s, w, np.array(sorted(seen), U64))


def _table_signs(s, h):
    return set(s._export_table(h)[0].cpu().numpy().view(U64).tolist())


@pytest.mark.parametrize("b", K.PREFIX_BITS)
def test_stage_at_width(torch_cuda, pb, oracle, b):
    """Two tiered tables take the same steps: X trained, then aged out into the tier by filler steps.  One stages the
    next batch (pb_tier_stage prefixes the ids itself) before its forward, the other does not: the stage restores
    exactly what the unstaged forward restores, and outputs and entries stay equal bit for bit."""
    torch = torch_cuda
    rng = np.random.default_rng(300 + b)
    dim, C, B = 16, 64, 64
    pf = oracle.index_prefix(0, b)
    x0, x1 = _width_ids(rng, b, B), _width_ids(rng, b, B)
    fill = [np.arange(k, k + 4, dtype=U64) % U64(min(pf, 1000)) for k in range(3)]  # prefix 0: signs below pf
    tables = []
    for _ in range(2):
        s = _shard(pb, oracle, dim, 0, cap=C, tier_rows=1024)
        s.set_eviction(check_every=1, low_water=C, target_free=C, keep_batches=1)
        ctx = pb.BatchContext(B, B, [pf], prefix_bit=b)
        fctx = pb.BatchContext(B, B, [0], prefix_bit=b)
        for cx, ids in [(ctx, x0)] + [(fctx, f) for f in fill]:
            cx.forward(s, to_dev_ids(ids, DEV), [0, ids.size], ids.size)
            cx.backward(s, [torch.full((ids.size, dim), 1e-3, dtype=torch.float16, device=DEV)])
        tables.append((s, ctx))
    aged = set(int(x) for x in K.prefix_np(x0, b, pf))
    for s, _ in tables:
        assert aged <= _table_signs(s, s.host_tier.h)
    (sa, ca), (sb, cb) = tables
    want = len(set(int(x) for x in K.prefix_np(x1, b, pf)) & aged)
    ra, rb = sa.tier_stats()["restored"], sb.tier_stats()["restored"]
    sa.stage(to_dev_ids(x1, DEV), [0, B], [pf], prefix_bit=b)
    assert sa.stage_stats() == {"staged": want, "skipped": 0}
    assert set(int(x) for x in K.prefix_np(x1, b, pf)) & aged <= _table_signs(sa, sa.h)
    outs = [cx.forward(s, to_dev_ids(x1, DEV), [0, B], B).cpu().numpy() for s, cx in tables]
    assert outs[0].tobytes() == outs[1].tobytes()
    assert sa.tier_stats()["restored"] - ra == want == sb.tier_stats()["restored"] - rb
    g = torch.from_numpy(_grads(rng, (B, dim), False)).to(DEV)
    for s, cx in tables:
        cx.backward(s, [g])
    every = np.array(sorted(aged | set(int(x) for x in K.prefix_np(x1, b, pf))), U64)
    ea, fa = sa.get_entries(to_dev_ids(every, DEV))
    eb, fb = sb.get_entries(to_dev_ids(every, DEV))
    assert bool(fa.all()) and bool(fb.all()) and ea.cpu().numpy().tobytes() == eb.cpu().numpy().tobytes()


@pytest.mark.parametrize("b", K.PREFIX_BITS)
def test_sharded_step_at_width(torch_cuda, pb, oracle, b):
    """R = 2 virtual ranks route each distinct sign by farmhash64 of the prefixed sign."""
    torch = torch_cuda
    from persia_b200.worker import ShardedEmbeddingWorker as W

    rng = np.random.default_rng(400 + b)
    R, dim, kind, B = 2, 16, 1, 128
    pf = _width_prefixes(oracle, b)
    S = len(pf)
    ws = W.local_group(R, S, dim, pf, 1 << 14, cap=S * B, optimizer=_gpu_optim(kind, OPT[kind]), max_batch=B,
                       prefix_bit=b)
    w = _worker(oracle, [oracle.SlotCfg(dim, prefix=p) for p in pf], kind, n_ps=R, prefix_bit=b)
    shards = [x.shard for x in ws]
    for x in shards:
        x.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    seen = set()
    for step in range(2):
        ids = [[_width_ids(rng, b, B) for _ in range(S)] for _ in range(R)]
        torch.cuda.synchronize()
        outs = W.group_forward(ws, [to_dev_ids(np.concatenate(x), DEV) for x in ids], B, training=True)
        torch.cuda.synchronize()
        octx = []
        for r in range(R):
            res = np.concatenate([K.residues(ids[r][i], b, pf[i]) for i in range(S)])
            want, c = w.forward(res, full_row_off(S, B), B, training=True)
            octx.append(c)
            got = outs[r].cpu().numpy()
            for i in range(S):
                assert got[i].tobytes() == want[i].tobytes(), (step, r, i)
            signs = [K.prefix_np(ids[r][i], b, pf[i]) for i in range(S)]
            _check_stats(ws[r].ctx, signs)
            seen.update(int(x) for x in np.concatenate(signs))
        g = _grads(rng, (R, S, B, dim), step == 1)
        sts = W.group_backward(ws, [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)],
                               want_status=True)
        torch.cuda.synchronize()
        for r in range(R):
            assert sts[r].cpu().numpy().tolist() == w.backward(octx[r], [g[r, i] for i in range(S)]) == [0] * S
    for x in ws:
        assert x.status() == (False, False)
    got, want = _read_rows(torch, oracle, shards, w, np.array(sorted(seen), U64), R)
    assert got.tobytes() == want.tobytes()
