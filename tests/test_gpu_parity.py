"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Bar (SURVEY.md §8c): bit-exact for hashes, prefixes, shard ids, partitions, looked-up rows, single-id
pooled f16 outputs, SGD and (against the oracle's exact-rsqrt mode) Adagrad updates; <= 1 f16 ulp for
multi-id pooled sums (f32 summation order differs), which are bit-exact against util.pool_model; Adagrad vs
the reference's _mm256_rsqrt_ps mode within 3.7e-4 of the step.
"""
import numpy as np
import pytest

from util import entries_equal as _entries_equal
from util import (f16_ulp_diff, full_row_off, held_rows, make_batch, pool_model, same_bits, slot_signs, to_dev_i32,
                  to_dev_ids)
from util import fwd_both as _fwd_both
from util import pair as _pair
from util import train_steps as _train_steps

pytestmark = pytest.mark.gpu


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


DEV = "cuda:0"


def _np_u64(t):
    return t.cpu().numpy().view(np.uint64)


# ---------------------------------------------------------------------------------------------- A1-A3
def test_farmhash_prefix_shard_bit_exact(torch_cuda, pb, oracle):
    rng = np.random.default_rng(11)
    x = np.concatenate([rng.integers(0, 2**63, size=100000, dtype=np.uint64) * 2 + 1,
                        np.array([0, 1, 12, 23, 34, 56, 78, 90, 2**64 - 1], np.uint64)])
    d = to_dev_ids(x, DEV)
    np.testing.assert_array_equal(_np_u64(pb.farmhash64(d)), oracle.farmhash64(x))
    for R in (1, 2, 3, 8, 255):
        np.testing.assert_array_equal(pb.shard_of(d, R).cpu().numpy().view(np.uint32), oracle.shard_of(x, R))
    # reference KAT (embedding_worker_service/mod.rs:1615-1660), prefix_bit 12
    raw = np.array([12, 23, 34, 56, 78, 90, 16000000000000000, 56], np.uint64)
    got = _np_u64(pb.add_prefix(to_dev_ids(raw, DEV), [0, 8], [100 << 52], prefix_bit=12))
    assert got.tolist() == [450359962737049612, 450359962737049623, 450359962737049634, 450359962737049656,
                            450359962737049678, 450359962737049690, 452849163854938115, 450359962737049656]
    # per-slot prefixes over a ragged layout, incl. an empty slot
    offs = [0, 1000, 1000, 50000, x.size]
    pf = [oracle.index_prefix(g) for g in (0, 1, 2, 3)]
    want = np.concatenate([oracle.add_prefix(x[offs[i]:offs[i + 1]], 8, pf[i]) for i in range(4)])
    np.testing.assert_array_equal(_np_u64(pb.add_prefix(d, offs, pf, prefix_bit=8)), want)


def test_hash_stack_on_device_matches_reference_vector(torch_cuda, pb):
    """A1 on the device (pb_hash_stack): the reference's own vector (embedding_worker_service/mod.rs:1570-1613, in
    tests/golden/farmhash64_kat.json) and, at size, the chained farmhash modulo rule."""
    import json
    import os

    fx = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "farmhash64_kat.json")))
    ids = np.array([int(k) for k in fx["hashstack_rounds2_size10"]], np.uint64)
    got = _np_u64(pb.hash_stack(to_dev_ids(ids, DEV), 2, 10)).reshape(-1, 2)
    assert got.tolist() == [list(v) for v in fx["hashstack_rounds2_size10"].values()]
    rng = np.random.default_rng(3)
    x = rng.integers(0, 2**63, size=50000, dtype=np.uint64)
    d = to_dev_ids(x, DEV)
    got = _np_u64(pb.hash_stack(d, 3, 1000003)).reshape(-1, 3)
    h = d
    for r in range(3):
        h = pb.farmhash64(h)
        np.testing.assert_array_equal(got[:, r], _np_u64(h) % np.uint64(1000003) + np.uint64(r * 1000003))
    assert pb.hash_stack(to_dev_ids(np.zeros(0, np.uint64), DEV), 2, 10).numel() == 0


@pytest.mark.parametrize("n,R", [(0, 2), (1, 1), (1000, 2), (100003, 8), (300000, 3)])
def test_partition_by_shard_stable(torch_cuda, pb, oracle, n, R):
    rng = np.random.default_rng(n + R)
    x = rng.integers(0, 2**62, size=n, dtype=np.uint64)
    perm, counts = pb.partition_by_shard(to_dev_ids(x, DEV), R)
    perm, counts = perm.cpu().numpy(), counts.cpu().numpy()
    sh = oracle.shard_of(x, R)
    want = np.argsort(sh, kind="stable")  # (slot, index_batch) order kept inside a shard (mod.rs:454-479)
    np.testing.assert_array_equal(perm, want)
    np.testing.assert_array_equal(counts, np.bincount(sh, minlength=R))


# ---------------------------------------------------------------------------------------------- A4
def _shard(pb, oracle, dim, cap, kind, **kw):
    s = pb.EmbeddingShard(dim, cap, 0)
    s.set_optimizer(kind, **kw)
    s.configure()
    return s


def test_set_get_lookup_rows(torch_cuda, pb, oracle):
    torch = torch_cuda
    rng = np.random.default_rng(3)
    dim, n = 16, 5000
    s = _shard(pb, oracle, dim, 20000, oracle.ADAGRAD)
    assert s.entry_len == 2 * dim
    signs = np.unique(rng.integers(0, 2**64 - 1, size=n, dtype=np.uint64))
    signs = np.concatenate([signs, np.array([2**64 - 1, 0], np.uint64)])  # incl. the empty-marker collision
    ent = rng.standard_normal((signs.size, 2 * dim)).astype(np.float32)
    s.set_entries(to_dev_ids(signs, DEV), torch.from_numpy(ent).to(DEV))
    assert len(s) == signs.size
    got, found = s.get_entries(to_dev_ids(signs, DEV))
    assert found.all()
    np.testing.assert_array_equal(got.cpu().numpy(), ent)
    # inference lookup: present -> emb, absent -> zeros (PS mod.rs:231-251)
    absent = np.array([5, 6, 7], np.uint64)
    q = np.concatenate([signs[:100], absent, signs[:100]])
    out = s.lookup(to_dev_ids(q, DEV), training=False).cpu().numpy()
    np.testing.assert_array_equal(out[:100], ent[:100, :dim])
    np.testing.assert_array_equal(out[100:103], 0)
    np.testing.assert_array_equal(out[103:], ent[:100, :dim])
    assert len(s) == signs.size
    # overwrite replaces (EvictionMap::insert, eviction_map.rs:76-97)
    s.set_entries(to_dev_ids(signs[:10], DEV), torch.from_numpy(ent[10:20]).to(DEV))
    got, _ = s.get_entries(to_dev_ids(signs[:10], DEV))
    np.testing.assert_array_equal(got.cpu().numpy(), ent[10:20])
    assert len(s) == signs.size


@pytest.mark.parametrize("kind,dim", [(0, 16), (1, 64), (2, 12), (3, 8)])
def test_training_lookup_admits_and_initialises(torch_cuda, pb, oracle, kind, dim):
    """New rows: emb = the (unpinned) restated init stream of the sign, state = optimizer initialisation
    (PS mod.rs:193-206, optim.rs:299-302).  Duplicates inside one request see the same row."""
    rng = np.random.default_rng(5)
    s = _shard(pb, oracle, dim, 4096, kind, initialization=0.25)
    signs = rng.integers(0, 2**60, size=1000, dtype=np.uint64)
    q = np.concatenate([signs, signs[::-1]])
    out = s.lookup(to_dev_ids(q, DEV), training=True).cpu().numpy()
    want = np.stack([oracle.init_row(int(x), dim, -0.01, 0.01) for x in signs])
    np.testing.assert_array_equal(out[:1000], want)
    np.testing.assert_array_equal(out[1000:], want[::-1])
    assert len(s) == np.unique(signs).size
    ent, found = s.get_entries(to_dev_ids(signs, DEV))
    assert found.all()
    ent = ent.cpu().numpy()
    np.testing.assert_array_equal(ent[:, :dim], want)
    state = ent[:, dim:]
    np.testing.assert_array_equal(state, 0.25 if kind in (1, 2) else 0.0)
    # second lookup hits
    out2 = s.lookup(to_dev_ids(signs, DEV), training=True).cpu().numpy()
    np.testing.assert_array_equal(out2, want)
    assert len(s) == np.unique(signs).size


def test_lookup_matches_oracle_ps(torch_cuda, pb, oracle):
    rng = np.random.default_rng(8)
    dim = 32
    s = _shard(pb, oracle, dim, 1 << 15, oracle.SGD)
    w = oracle.Worker([oracle.SlotCfg(dim)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD))
    for step in range(5):
        signs = rng.integers(0, 5000, size=3000, dtype=np.uint64)
        train = step % 2 == 0
        got = s.lookup(to_dev_ids(signs, DEV), training=train).cpu().numpy()
        want = w.ps_lookup(0, signs, np.full(signs.size, dim, np.uint32), train).reshape(-1, dim)
        np.testing.assert_array_equal(got, want)
        assert len(s) == w.ps_len(0)


def test_capacity_refusal_is_counted(torch_cuda, pb, oracle):
    s = _shard(pb, oracle, 8, 100, oracle.SGD)
    signs = np.arange(1, 301, dtype=np.uint64)
    out = s.lookup(to_dev_ids(signs, DEV), training=True).cpu().numpy()
    c = s.counters()
    assert c["admitted"] == 100 and c["capacity_refused"] == 200
    assert (np.abs(out).sum(axis=1) > 0).sum() == 100  # refused signs read as zeros


def test_errors(torch_cuda, pb, oracle):
    from persia_b200.native import PersiaB200Error

    torch = torch_cuda
    s = pb.EmbeddingShard(8, 100, 0)
    ids = to_dev_ids(np.arange(4, dtype=np.uint64), DEV)
    with pytest.raises(PersiaB200Error):  # OptimizerNotFoundError (PS mod.rs:180-182)
        s.lookup(ids, training=True)
    np.testing.assert_array_equal(s.lookup(ids, training=False).cpu().numpy(), 0)
    s.set_optimizer(oracle.SGD)
    with pytest.raises(PersiaB200Error):  # NotConfiguredError (PS mod.rs:150-158)
        s.lookup(ids, training=True)
    s.configure()
    s.lookup(ids, training=True)
    ctx = pb.BatchContext(1 << 17, 1 << 17, [1 << 56])
    big = to_dev_ids(np.zeros(65536, np.uint64), DEV)
    with pytest.raises(PersiaB200Error):  # persia-common lib.rs:49-51
        ctx.forward(s, big, [0, 65536], 65536)
    with pytest.raises(PersiaB200Error):  # backward without a pending forward
        ctx.backward(s, [torch.zeros(4, 8, device=DEV)])


def test_misaligned_pointers_are_refused(torch_cuda, pb, oracle):
    """Gradient, output and update buffers must be 16-byte aligned (the kernels use vector accesses): a raw pointer that
    is not is refused before anything is enqueued, and the tensor wrappers copy such a view instead."""
    from persia_b200 import native as N
    from persia_b200.native import PersiaB200Error

    torch = torch_cuda
    lib = N.load()
    rng = np.random.default_rng(12)
    S, B, dim, card = 2, 257, 12, [5, 1000]  # slot 1 of an [S, B, dim] f16 tensor starts B * dim * 2 = 6168 bytes in
    kw = dict(lr=0.05)
    s, ctx, w, _ = _pair(pb, oracle, S, dim, oracle.SGD, optim_kw=kw)
    s2, ctx2, _, _ = _pair(pb, oracle, S, dim, oracle.SGD, optim_kw=kw)  # the same steps with aligned gradients
    ids, _, slot_off = make_batch(rng, S, B, card)
    d_ids = to_dev_ids(ids, DEV)
    out = torch.empty(S * B * dim + 8, dtype=torch.float16, device=DEV)[1:1 + S * B * dim].view(S, B, dim)
    torch.cuda.synchronize()
    n0 = lib.pb_launch_count()
    with pytest.raises(PersiaB200Error):
        ctx.forward(s, d_ids, slot_off, B, out=out)
    assert lib.pb_launch_count() == n0
    ctx.forward(s, d_ids, slot_off, B)
    ctx2.forward(s2, d_ids, slot_off, B)
    _, octx = w.forward(ids, full_row_off(S, B), B, training=True)
    signs = np.concatenate([w.ctx_signs(octx, i) for i in range(S)])
    before = s.get_entries(to_dev_ids(signs, DEV))[0].cpu().numpy()
    g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
    g_dev = torch.from_numpy(g).to(DEV)
    views = [g_dev[i] for i in range(S)]
    assert views[1].is_contiguous() and views[1].data_ptr() % 16 != 0
    torch.cuda.synchronize()
    n0 = lib.pb_launch_count()
    with pytest.raises(PersiaB200Error):
        ctx.backward_ptrs(s, [v.data_ptr() for v in views], True)
    assert lib.pb_launch_count() == n0
    np.testing.assert_array_equal(s.get_entries(to_dev_ids(signs, DEV))[0].cpu().numpy(), before)
    # the refused call left the batch pending: the tensor form copies the misaligned slot and applies it
    ctx.backward(s, views)
    ctx2.backward(s2, [v.clone() for v in views])
    w.backward(octx, [g[i] for i in range(S)])
    got = s.get_entries(to_dev_ids(signs, DEV))[0].cpu().numpy()
    assert got.tobytes() == s2.get_entries(to_dev_ids(signs, DEV))[0].cpu().numpy().tobytes()
    assert not np.array_equal(got, before)
    _entries_equal(torch, s, w, signs)
    # pb_update (update_gradient_mixed) reads its f32 gradients with 16-byte loads too
    g32 = torch.zeros(dim * 2 + 1, dtype=torch.float32, device=DEV)[1:].view(2, dim)
    torch.cuda.synchronize()
    n0 = lib.pb_launch_count()
    with pytest.raises(PersiaB200Error):
        s.update(to_dev_ids(signs[:2], DEV), g32)
    assert lib.pb_launch_count() == n0
    np.testing.assert_array_equal(s.get_entries(to_dev_ids(signs, DEV))[0].cpu().numpy(), got)


# ---------------------------------------------------------------------------------------------- A5
def test_forward_single_id_bit_exact(torch_cuda, pb, oracle):
    """C1 shape: 4 slots, dim 16, batch 512, rows pre-seeded through set_embedding."""
    torch = torch_cuda
    rng = np.random.default_rng(1)
    S, dim, B, card = 4, 16, 512, 25000
    s, ctx, w, pf = _pair(pb, oracle, S, dim, oracle.SGD, cap=1 << 17)
    seed_rng = np.random.default_rng(7)
    for i in range(S):
        signs = oracle.add_prefix(np.arange(card, dtype=np.uint64), 8, pf[i])
        ent = seed_rng.uniform(-0.01, 0.01, size=(card, dim)).astype(np.float32)
        s.set_entries(to_dev_ids(signs, DEV), torch.from_numpy(ent).to(DEV))
        w.set_embedding(signs, ent, dim)
    for _ in range(3):
        ids, row_off, slot_off = make_batch(rng, S, B, card)
        got, want, _ = _fwd_both(torch, s, ctx, w, ids, row_off, slot_off, B, training=True)
        for i in range(S):
            np.testing.assert_array_equal(got[i].view(np.uint16), want[i].view(np.uint16))


@pytest.mark.parametrize("dim", [12, 64, 96, 128, 200])
def test_forward_multi_id_ragged(torch_cuda, pb, oracle, dim):
    """Ragged LIL with empty samples, sqrt scaling on some slots, admission on the fly, eval and train."""
    torch = torch_cuda
    rng = np.random.default_rng(dim)
    S, B = 5, 257
    sqrt = [False, True, False, True, True]
    s, ctx, w, pf = _pair(pb, oracle, S, dim, oracle.ADAGRAD, sqrt=sqrt)
    for it in range(4):
        ids, row_off, slot_off = make_batch(rng, S, B, [3, 50, 1000, 100000, 7], max_ids=6, allow_empty=True)
        training = it != 2
        got, want, _ = _fwd_both(torch, s, ctx, w, ids, row_off, slot_off, B, training=training)
        signs = slot_signs(oracle, ids, slot_off, pf)
        model = pool_model(held_rows(torch, oracle, [s], signs), signs, row_off, B, sqrt, dim=dim)
        for i in range(S):
            assert same_bits(got[i], model[i])  # sample order, bit for bit
            assert f16_ulp_diff(got[i], want[i]) <= 1  # f32 sum order differs for multi-id samples
        assert len(s) == w.ps_len(0)
        counts = np.diff(row_off)
        single = (counts <= 1).reshape(S, B)
        for i in range(S):  # samples with <= 1 id are pure copies: bit-exact
            np.testing.assert_array_equal(got[i][single[i]].view(np.uint16), want[i][single[i]].view(np.uint16))


def test_forward_empty_and_tiny(torch_cuda, pb, oracle):
    torch = torch_cuda
    s, ctx, w, _ = _pair(pb, oracle, 2, 8, oracle.SGD)
    # batch of one sample, one id
    ids = np.array([5, 9], np.uint64)
    got, want, _ = _fwd_both(torch, s, ctx, w, ids, None, [0, 1, 2], 1)
    np.testing.assert_array_equal(got.view(np.uint16).reshape(-1), np.concatenate(want).view(np.uint16).reshape(-1))
    # every sample empty
    row_off = np.zeros(2 * 4 + 1, np.uint32)
    got = ctx.forward(s, to_dev_ids(np.zeros(0, np.uint64), DEV), [0, 0, 0], 4, row_off=to_dev_i32(row_off, DEV))
    assert got.shape == (2, 4, 8) and not got.cpu().numpy().any()


# ---------------------------------------------------------------------------------------------- A8 + A9
def test_sgd_training_bit_exact_c1(torch_cuda, pb, oracle):
    """BASELINE config 1: 4 slots, 1e5-row dim-16 table, batch 512, forward + SGD vs the oracle.
    Duplicate ids inside a batch are reduced in reference order, so every entry is bit-identical."""
    torch = torch_cuda
    rng = np.random.default_rng(1)
    S, dim, B, card = 4, 16, 512, 25000
    s, ctx, w, pf = _pair(pb, oracle, S, dim, oracle.SGD, cap=1 << 17, optim_kw=dict(lr=0.01, wd=0.0))
    seed_rng = np.random.default_rng(7)
    for i in range(S):
        signs = oracle.add_prefix(np.arange(card, dtype=np.uint64), 8, pf[i])
        ent = seed_rng.uniform(-0.01, 0.01, size=(card, dim)).astype(np.float32)
        s.set_entries(to_dev_ids(signs, DEV), torch.from_numpy(ent).to(DEV))
        w.set_embedding(signs, ent, dim)
    touched = _train_steps(torch, s, ctx, w, rng, S, B, dim, card, steps=100)
    for t in touched:
        _entries_equal(torch, s, w, t[:3000])


@pytest.mark.parametrize("dim,kw", [(12, dict(lr=0.05, wd=0.01)), (64, dict(lr=0.01, wd=0.001))])
def test_sgd_heavy_duplicates_weight_decay_scale(torch_cuda, pb, oracle, dim, kw):
    """Tiny cardinalities (long duplicate runs), multi-id ragged samples, loss scale, sqrt scaling,
    a NaN slot, a skipped slot, +-inf gradients, dim with an unfused tail."""
    torch = torch_cuda
    rng = np.random.default_rng(dim)
    S, B = 4, 300
    s, ctx, w, _ = _pair(pb, oracle, S, dim, oracle.SGD, sqrt=[False, True, False, True], optim_kw=kw,
                         hyper_kw=dict(wb=0.05))
    touched = _train_steps(torch, s, ctx, w, rng, S, B, dim, [3, 40, 5000, 11], steps=6, max_ids=4,
                           allow_empty=False, scale=[128.0, 1.0, 1024.0, 3.0], nan_slot=(2, 1), skip_slot=(3, 0))
    for t in touched:
        _entries_equal(torch, s, w, t)


@pytest.mark.parametrize("dim", [12, 64])
def test_adagrad_training_matches_exact_mode_bitwise(torch_cuda, pb, oracle, dim):
    """Adagrad: the GPU reproduces the reference's fused/unfused structure with an exact 1/sqrt, i.e. the
    oracle's exact-rsqrt mode bit for bit; the accumulator is bit-exact against the reference mode too and
    the weights stay within the documented _mm256_rsqrt_ps error of it."""
    torch = torch_cuda
    S, B, card = 3, 256, [5, 300, 100000]
    kw = dict(lr=0.01, mom=1.0, init_acc=0.01, eps=1e-10)
    for exact in (True, False):
        oracle.set_rsqrt_exact(exact)
        try:
            rng = np.random.default_rng(99)
            s, ctx, w, _ = _pair(pb, oracle, S, dim, oracle.ADAGRAD, optim_kw=kw)
            touched = _train_steps(torch, s, ctx, w, rng, S, B, dim, card, steps=5, max_ids=3)
            for t in touched:
                if exact:
                    _entries_equal(torch, s, w, t)
                else:
                    ent, _ = s.get_entries(to_dev_ids(t, DEV))
                    ent = ent.cpu().numpy()
                    ref = np.stack([w.get_entry(int(x)) for x in t])
                    np.testing.assert_allclose(ent[:, :dim], ref[:, :dim], rtol=0, atol=2e-4)
                    np.testing.assert_array_equal(ent[:, dim:], ref[:, dim:])  # accumulator never sees rsqrt
        finally:
            oracle.set_rsqrt_exact(False)


def test_adagrad_vectorwise_and_f32_grads(torch_cuda, pb, oracle):
    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(21)
        S, B, dim = 2, 128, 20
        s, ctx, w, _ = _pair(pb, oracle, S, dim, oracle.ADAGRAD_VW, optim_kw=dict(lr=0.02, mom=0.9, init_acc=0.1, eps=1e-8))
        touched = _train_steps(torch, s, ctx, w, rng, S, B, dim, [7, 1000], steps=4, max_ids=2, f32=True)
        for t in touched:
            _entries_equal(torch, s, w, t)
    finally:
        oracle.set_rsqrt_exact(False)


def test_shared_feature_group_updates_sequentially(torch_cuda, pb, oracle):
    """Two slots of one feature group share signs: the reference applies one optimizer step per slot, in
    slot order (embedding_worker_service/mod.rs:720-822)."""
    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(4)
        S, B, dim = 3, 200, 16
        s, ctx, w, _ = _pair(pb, oracle, S, dim, oracle.ADAGRAD, groups=[0, 0, 1], optim_kw=dict(lr=0.05))
        touched = _train_steps(torch, s, ctx, w, rng, S, B, dim, [30, 30, 30], steps=5, max_ids=2)
        for t in touched:
            _entries_equal(torch, s, w, t)
    finally:
        oracle.set_rsqrt_exact(False)


def test_direct_update_matches_oracle_ps(torch_cuda, pb, oracle):
    """pb_update == update_gradient_mixed on distinct signs, incl. absent ones (counted, skipped)."""
    torch = torch_cuda
    rng = np.random.default_rng(17)
    dim = 24
    for kind in (oracle.SGD, oracle.ADAGRAD):
        oracle.set_rsqrt_exact(True)
        try:
            s = _shard(pb, oracle, dim, 4096, kind, lr=0.1, wd=0.01 if kind == 0 else 0.0)
            w = oracle.Worker([oracle.SlotCfg(dim)], n_ps=1)
            w.configure()
            w.set_optimizer(oracle.Optim(kind, lr=0.1, wd=0.01 if kind == 0 else 0.0))
            w.set_faithful_miss(False)
            signs = np.arange(100, 1100, dtype=np.uint64)
            s.lookup(to_dev_ids(signs, DEV), training=True)
            w.ps_lookup(0, signs, np.full(signs.size, dim, np.uint32), True)
            upd = np.concatenate([signs[::3], np.array([5, 6], np.uint64)])  # two absent signs
            rng.shuffle(upd)
            g = rng.standard_normal((upd.size, dim)).astype(np.float32)
            s.update(to_dev_ids(upd, DEV), torch.from_numpy(g).to(DEV))
            w.ps_update(0, upd, np.full(upd.size, dim, np.uint32), g)
            _entries_equal(torch, s, w, signs)
            assert s.counters()["gradient_id_miss"] == 2 == w.grad_miss()
        finally:
            oracle.set_rsqrt_exact(False)


@pytest.mark.parametrize("dim,kind,f32,max_ids", [(64, 0, False, 1), (16, 1, False, 1), (128, 1, False, 1), (12, 0, False, 1),
                                                  (200, 2, False, 1), (96, 3, True, 1), (13, 0, False, 1),
                                                  (64, 1, False, 3), (128, 2, True, 2), (72, 1, True, 1)])
def test_heavy_multiplicity_bit_exact(torch_cuda, pb, oracle, dim, kind, f32, max_ids):
    """Tiny-cardinality slots repeat a sign thousands of times in a batch: those signs go through the hot path of the
    backward (bitmap order, then producer warps fill a shared-memory ring that chain warps add in order; element-wise
    loads when a gradient row is not a whole number of 16-byte vectors).  The
    gradient sum keeps the reference order for any multiplicity, so every row is bit-identical to the oracle's, with
    f16 and f32 gradients, every optimizer, one-id and ragged layouts (sqrt scaling and a loss scale on some slots)."""
    torch = torch_cuda
    oracle.set_rsqrt_exact(True)
    try:
        S, B, card = 4, 4096 if max_ids == 1 else 1500, [3, 40, 700, 100000]
        kw = dict(lr=0.05) if kind != 3 else dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8)
        rng = np.random.default_rng(2024 + dim)
        sqrt = [True, False, True, False] if max_ids > 1 else None
        scale = [1.0, 128.0, 1.0, 1024.0] if max_ids > 1 else None
        s, ctx, w, _ = _pair(pb, oracle, S, dim, kind, optim_kw=kw, cap=1 << 16, sqrt=sqrt)
        touched = _train_steps(torch, s, ctx, w, rng, S, B, dim, card, steps=3, f32=f32, max_ids=max_ids, scale=scale)
        for t in touched:
            _entries_equal(torch, s, w, t)
        assert s.counters()["wait_errors"] == 0
    finally:
        oracle.set_rsqrt_exact(False)


def test_overlapping_batches_two_contexts(torch_cuda, pb, oracle):
    """Two training batches in flight on one table (fwd A, fwd B, bwd A, bwd B), as persia_core.Forward prefetches
    them, with heavily overlapping signs: what a batch keeps between its forward and its backward lives in its own
    context, so the gradients of A reach A's signs (the table-wide leader words of round 1 could not guarantee that)."""
    torch = torch_cuda
    rng = np.random.default_rng(99)
    S, B, dim, card = 3, 512, 32, [5, 300, 20000]
    s, ctx_a, w, pf = _pair(pb, oracle, S, dim, oracle.SGD, optim_kw=dict(lr=0.05, wd=0.001))
    ctx_b = pb.BatchContext(1 << 16, 1 << 16, pf)
    seen = [set() for _ in range(S)]
    for it in range(4):
        ia, _, slot_off = make_batch(rng, S, B, card)
        ib, _, _ = make_batch(rng, S, B, card)
        ga = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
        gb = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
        oa = ctx_a.forward(s, to_dev_ids(ia, DEV), slot_off, B, training=True).cpu().numpy()
        ob = ctx_b.forward(s, to_dev_ids(ib, DEV), slot_off, B, training=True).cpu().numpy()
        wa, octx_a = w.forward(ia, full_row_off(S, B), B, training=True)
        wb, octx_b = w.forward(ib, full_row_off(S, B), B, training=True)
        for i in range(S):
            np.testing.assert_array_equal(oa[i].view(np.uint16), wa[i].view(np.uint16))
            np.testing.assert_array_equal(ob[i].view(np.uint16), wb[i].view(np.uint16))
            seen[i].update(w.ctx_signs(octx_a, i).tolist())
            seen[i].update(w.ctx_signs(octx_b, i).tolist())
        ctx_a.backward(s, [torch.from_numpy(ga[i]).to(DEV) for i in range(S)])
        ctx_b.backward(s, [torch.from_numpy(gb[i]).to(DEV) for i in range(S)])
        w.backward(octx_a, [ga[i] for i in range(S)])
        w.backward(octx_b, [gb[i] for i in range(S)])
    for t in seen:
        _entries_equal(torch, s, w, np.array(sorted(t), np.uint64))


def test_graph_capture_replay_same_result(torch_cuda, pb, oracle):
    """A step (pb_forward + pb_backward, including the work pb_backward forks onto the context's own stream) captured
    once in a CUDA graph and replayed gives bit-identical rows; nothing per-batch is baked into the launches."""
    torch = torch_cuda
    rng = np.random.default_rng(31)
    S, B, dim, card = 6, 1024, 64, [3, 17, 900, 50000, 50000, 11]
    s, ctx, w, pf = _pair(pb, oracle, S, dim, oracle.SGD, cap=1 << 17, optim_kw=dict(lr=0.05, wd=0.001))
    touched = _train_steps(torch, s, ctx, w, rng, S, B, dim, card, steps=4)
    for t in touched:
        _entries_equal(torch, s, w, t[:2000])
    # the same step captured once and replayed: inputs are refreshed in place between replays
    ids_np, _, slot_off = make_batch(rng, S, B, card)
    ids_dev = to_dev_ids(ids_np, DEV)
    g_dev = torch.zeros((S, B, dim), dtype=torch.float16, device=DEV)
    out = torch.empty((S, B, dim), dtype=torch.float16, device=DEV)
    grads = [g_dev[i] for i in range(S)]
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        ctx.forward(s, ids_dev, slot_off, B, training=True, out=out)  # warm-up (allocations happen here)
        ctx.backward(s, grads)
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            ctx.forward(s, ids_dev, slot_off, B, training=True, out=out)
            ctx.backward(s, grads)
    # bring the oracle to the same state: one step with zero gradients happened above (plus the capture's none)
    _, octx = w.forward(ids_np, full_row_off(S, B), B, training=True)
    w.backward(octx, [np.zeros((B, dim), np.float16)] * S)
    seen = [set() for _ in range(S)]
    for it in range(3):
        ids_np, _, _ = make_batch(rng, S, B, card)
        g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
        ids_dev.copy_(to_dev_ids(ids_np, DEV))
        g_dev.copy_(torch.from_numpy(g).to(DEV))
        graph.replay()
        torch.cuda.synchronize()
        want, octx = w.forward(ids_np, full_row_off(S, B), B, training=True)
        got = out.cpu().numpy()
        for i in range(S):
            np.testing.assert_array_equal(got[i].view(np.uint16), want[i].view(np.uint16))
            seen[i].update(w.ctx_signs(octx, i).tolist())
        w.backward(octx, [g[i] for i in range(S)])
    for t in seen:
        _entries_equal(torch, s, w, np.array(sorted(t), np.uint64)[:2000])


@pytest.mark.parametrize("dim", [12, 64])
def test_adam_training_bit_exact(torch_cuda, pb, oracle, dim):
    """Adam (persia-simd adam_avx2 + the per-feature-group beta powers of optim.rs:155-197), incl. two slots that
    share one feature group (their power advances once per request)."""
    torch = torch_cuda
    rng = np.random.default_rng(dim + 7)
    S, B, card = 3, 200, [30, 30, 5000]
    s, ctx, w, _ = _pair(pb, oracle, S, dim, oracle.ADAM, groups=[0, 0, 1],
                         optim_kw=dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8))
    touched = _train_steps(torch, s, ctx, w, rng, S, B, dim, card, steps=5, max_ids=2)
    for t in touched:
        _entries_equal(torch, s, w, t)


def test_adam_nan_and_skipped_slots_do_not_advance_their_group(torch_cuda, pb, oracle):
    """A slot dropped for a NaN gradient (mod.rs:731-746) or skipped sends nothing to the parameter server, so its
    feature group's beta powers stay where they are for that request (get_batch_level_state only sees the signs sent)."""
    torch = torch_cuda
    rng = np.random.default_rng(91)
    S, B, dim, card = 3, 200, 16, [30, 500, 5000]
    s, ctx, w, _ = _pair(pb, oracle, S, dim, oracle.ADAM, optim_kw=dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8))
    touched = _train_steps(torch, s, ctx, w, rng, S, B, dim, card, steps=6, nan_slot=(2, 1), skip_slot=(3, 0))
    for t in touched:
        _entries_equal(torch, s, w, t)


def test_adam_graph_replay_advances_beta_powers(torch_cuda, pb, oracle):
    """The beta powers live on the device: a captured forward+backward replayed k times equals k oracle steps."""
    torch = torch_cuda
    rng = np.random.default_rng(77)
    S, B, dim, card = 2, 256, 32, [40, 3000]
    s, ctx, w, _ = _pair(pb, oracle, S, dim, oracle.ADAM, optim_kw=dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8))
    ids_np, _, slot_off = make_batch(rng, S, B, card)
    ids_dev = to_dev_ids(ids_np, DEV)
    g_dev = torch.zeros((S, B, dim), dtype=torch.float16, device=DEV)
    out = torch.empty((S, B, dim), dtype=torch.float16, device=DEV)
    grads = [g_dev[i] for i in range(S)]

    def oracle_step(ids, g):
        _, octx = w.forward(ids, full_row_off(S, B), B, training=True)
        w.backward(octx, [g[i] for i in range(S)])

    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        ctx.forward(s, ids_dev, slot_off, B, training=True, out=out)  # eager step (allocations happen here)
        ctx.backward(s, grads)
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):  # capture launches nothing
            ctx.forward(s, ids_dev, slot_off, B, training=True, out=out)
            ctx.backward(s, grads)
    oracle_step(ids_np, np.zeros((S, B, dim), np.float16))
    seen = [set() for _ in range(S)]
    for it in range(4):
        ids_np, _, _ = make_batch(rng, S, B, card)
        g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
        ids_dev.copy_(to_dev_ids(ids_np, DEV))
        g_dev.copy_(torch.from_numpy(g).to(DEV))
        graph.replay()
        torch.cuda.synchronize()
        oracle_step(ids_np, g)
        for i in range(S):
            seen[i].update(oracle.add_prefix(ids_np[i * B:(i + 1) * B], 8, oracle.index_prefix(i)).tolist())
    for t in seen:
        _entries_equal(torch, s, w, np.array(sorted(t), np.uint64))


def test_capacity_eviction_keeps_recent_rows(torch_cuda, pb, oracle):
    """EvictionMap semantics (eviction_map.rs:76-97), batch-granular: least recently used rows go first, rows used
    in the recent batches and a hot set touched every batch survive, the shard never refuses an admission, and a
    re-admitted sign starts again from its initial value."""
    torch = torch_cuda
    dim, cap = 8, 4096
    s = _shard(pb, oracle, dim, cap, oracle.SGD)
    s.set_eviction(check_every=1, low_water=600, target_free=1200, keep_batches=1)
    hot = np.arange(10_000_000, 10_000_050, dtype=np.uint64)
    batches = []
    for k in range(60):
        cold = np.arange(k * 300, (k + 1) * 300, dtype=np.uint64) + np.uint64(1)
        q = np.concatenate([cold, hot])
        batches.append(cold)
        out = s.lookup(to_dev_ids(q, DEV), training=True).cpu().numpy()
        assert np.abs(out).sum(axis=1).min() > 0  # every sign got storage (nothing refused, nothing read as zeros)
        if k == 0:
            first_val = out[:300].copy()
    c = s.counters()
    assert c["capacity_refused"] == 0
    assert 0 < len(s) <= cap
    _, found_hot = s.get_entries(to_dev_ids(hot, DEV))
    assert found_hot.all()
    for k in range(52, 60):  # the most recent batches are all resident
        _, f = s.get_entries(to_dev_ids(batches[k], DEV))
        assert f.all(), k
    _, f0 = s.get_entries(to_dev_ids(batches[0], DEV))
    assert not f0.any()  # the oldest batch is gone
    np.testing.assert_array_equal(s.lookup(to_dev_ids(batches[0], DEV), training=False).cpu().numpy(), 0)
    # dirty a few hot rows, then check an evicted sign comes back with its initial value (seeded by the sign)
    again = s.lookup(to_dev_ids(batches[0], DEV), training=True).cpu().numpy()
    np.testing.assert_array_equal(again, first_val)
    np.testing.assert_array_equal(again, np.stack([oracle.init_row(int(x), dim, -0.01, 0.01) for x in batches[0]]))
