"""GPU: what the Python bindings do between a tensor and the C ABI, in both forms of a call (`local`: an EmbeddingShard
and its BatchContexts; `sharded`: rank 0 of two virtual ranks of one GPU, ShardedEmbeddingWorker.local_group).  Slot
gradients: a misaligned slot view is copied and applies as an aligned one would, its pointer form is refused before
anything is launched, and mixed dtypes are refused before anything is launched.  An empty raw gradient is a request,
not a skip.  Every counter reader returns its fields, in order."""
import numpy as np
import pytest

from util import to_dev_ids

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S, B, DIM = 2, 64, 16


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def _group(torch, oracle, n_slots=S, dim=DIM, batch=B):
    """Two virtual ranks, their tables allocated (a first use allocates with a device-wide sync: not while a peer spins)."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker

    pf = [oracle.index_prefix(i) for i in range(n_slots)]
    ws = ShardedEmbeddingWorker.local_group(2, n_slots, dim, pf, 1 << 12, cap=n_slots * batch,
                                            optimizer=dict(kind=N.OPT_SGD, lr=0.1), max_batch=batch)
    for w in ws:
        w.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    return ws


def _local(oracle, n_slots=S, dim=DIM, **kw):
    from persia_b200 import native as N
    from persia_b200 import shard as SH

    s = SH.EmbeddingShard(dim, 1 << 12, 0, **kw)
    s.set_optimizer(N.OPT_SGD, lr=0.1)
    s.configure()
    return s, SH.BatchContext(n_slots * B, n_slots * B, [oracle.index_prefix(i) for i in range(n_slots)])


def _close(torch, *objs):
    torch.cuda.synchronize()
    for o in objs:
        o.close()


def test_sharded_misaligned_slot_view_applies_as_an_aligned_clone(torch_cuda, oracle):
    """Slot 1 of an f16 [2, 257, 12] gradient starts 257 * 12 * 2 = 6168 bytes in, 8 bytes off 16: the worker copies it
    on its stream, and the tables end bit for bit as with aligned clones.  Its pointer form is refused with nothing
    launched, and the batch stays pending for the tensor form.  Rank 0 passes slot views, rank 1 the whole tensor."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    lib = N.load()
    b, dim = 257, 12
    rng = np.random.default_rng(12)
    ids = [rng.integers(0, 1000, size=S * b, dtype=np.uint64) for _ in range(2)]
    d_ids = [to_dev_ids(x, DEV) for x in ids]
    pf = [oracle.index_prefix(i) for i in range(S)]
    signs = to_dev_ids(np.unique(np.concatenate([oracle.add_prefix(x.reshape(S, b)[i], 8, pf[i])
                                                 for x in ids for i in range(S)])), DEV)
    ga, gb = _group(torch, oracle, dim=dim, batch=b), _group(torch, oracle, dim=dim, batch=b)
    try:
        W.group_forward(ga, d_ids, b)
        W.group_forward(gb, d_ids, b)
        g = [torch.from_numpy((rng.standard_normal((S, b, dim)) * 1e-2).astype(np.float16)).to(DEV) for _ in range(2)]
        views = [g[0][i] for i in range(S)]
        assert views[1].is_contiguous() and views[1].data_ptr() % 16 != 0
        torch.cuda.synchronize()
        before = ga[0].shard.get_entries(signs)[0].cpu().numpy()
        n0 = lib.pb_launch_count()
        with pytest.raises(N.PersiaB200Error) as ei:
            ga[0].backward_ptrs([v.data_ptr() for v in views], True)
        assert ei.value.code == N.PB_ERR_INVALID
        assert lib.pb_launch_count() == n0
        W.group_backward(ga, [views, g[1]])
        W.group_backward(gb, [[v.clone() for v in views], g[1].clone()])
        torch.cuda.synchronize()
        for r in range(2):
            got, found = ga[r].shard.get_entries(signs)
            want, want_found = gb[r].shard.get_entries(signs)
            assert got.cpu().numpy().tobytes() == want.cpu().numpy().tobytes()
            assert found.cpu().numpy().tolist() == want_found.cpu().numpy().tolist()
        assert not np.array_equal(ga[0].shard.get_entries(signs)[0].cpu().numpy(), before)
        assert ga[0].status() == (False, False)
    finally:
        _close(torch, *ga, *gb)


@pytest.mark.parametrize("form", ["local", "sharded"])
def test_mixed_slot_gradient_dtypes_are_refused_before_any_launch(torch_cuda, oracle, form):
    """f16 and f32 slot gradients in one request raise before anything is launched; the batch then takes a request
    of one dtype."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    lib = N.load()
    d_ids = to_dev_ids(np.arange(S * B, dtype=np.uint64), DEV)
    g16 = torch.zeros((B, DIM), dtype=torch.float16, device=DEV)
    g32 = torch.zeros((B, DIM), dtype=torch.float32, device=DEV)
    off = [s * B for s in range(S + 1)]
    if form == "local":
        s, ctx = _local(oracle)
        objs = (ctx, s)
    else:
        objs = ws = _group(torch, oracle)
    try:
        if form == "local":
            ctx.forward(s, d_ids, off, B)
        else:
            W.group_forward(ws, [d_ids, d_ids], B)
        torch.cuda.synchronize()
        n0 = lib.pb_launch_count()
        with pytest.raises(AssertionError):
            if form == "local":
                ctx.backward(s, [g16, g32])
            else:
                ws[0].backward([g16, g32], phases=N.PHASE_SEND)
        assert lib.pb_launch_count() == n0
        if form == "local":
            assert ctx.backward(s, [g32, g32], want_status=True).tolist() == [0, 0]
        else:
            assert [st.tolist() for st in W.group_backward(ws, [[g16, g16]] * 2, want_status=True)] == [[0, 0]] * 2
    finally:
        _close(torch, *objs)


def test_local_empty_raw_gradient_is_a_request(torch_cuda, oracle):
    """A batch without ids (U = 0) takes a [0, dim] gradient, f32 or f16, as an applied request (status 0); None is the
    skipped one (status 1)."""
    torch = torch_cuda
    s, ctx = _local(oracle, n_slots=1)
    empty = torch.zeros(0, dtype=torch.int64, device=DEV)
    row_off = torch.zeros(B + 1, dtype=torch.int32, device=DEV)
    try:
        for grad, want in ((torch.zeros((0, DIM), dtype=torch.float32, device=DEV), 0),
                           (torch.zeros((0, DIM), dtype=torch.float16, device=DEV), 0), (None, 1)):
            _, _, _, _, counts = ctx.forward_raw(s, empty, B, 2, row_off=row_off)
            assert counts.tolist() == [0, 0]
            assert ctx.backward_raw(s, grad, want_status=True).tolist() == [want]
    finally:
        _close(torch, ctx, s)


COUNTERS = ("admitted", "lookup_miss", "gradient_id_miss", "capacity_refused", "wait_errors")
INDEX_STATS = ("live", "tomb", "empty")
TIER_STATS = ("host_rows", "moved_out", "restored", "dropped", "refused")
STAGE_STATS = ("staged", "skipped")
INCREMENTAL_STATS = ("held", "inserted", "dropped", "taken")
BATCH_STATS = ("items", "cold", "warm", "hot", "repeated_occurrences", "occurrences")
HOT_GEOMETRY = ("EPL", "CH", "PW", "vec", "vshift", "lean", "R1", "R", "S", "cols", "stride", "passes")


def _keys_and_ints(d, keys):
    assert tuple(d) == keys
    assert all(type(v) is int for v in d.values())
    return d


@pytest.mark.parametrize("form", ["local", "sharded"])
def test_counter_readers_return_their_fields_in_order(torch_cuda, oracle, form):
    """After one training step of S * B distinct signs, each looked up and stepped once by its owner."""
    from persia_b200 import shard as SH
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    d_ids = to_dev_ids(np.arange(S * B, dtype=np.uint64), DEV)
    grads = [torch.full((B, DIM), 1e-2, dtype=torch.float16, device=DEV)] * S
    signs = np.concatenate([oracle.add_prefix(np.arange(i * B, (i + 1) * B, dtype=np.uint64), 8, oracle.index_prefix(i))
                            for i in range(S)])
    if form == "local":
        s, ctx = _local(oracle, tier_rows=1 << 12)
        objs, table, mine = (ctx, s), s, S * B
    else:
        ws = _group(torch, oracle)
        objs, table, ctx = ws, ws[0].shard, ws[0].ctx
        mine = int((oracle.shard_of(signs, 2) == 0).sum())
    try:
        if form == "local":
            s.enable_incremental(1 << 10)
            ctx.forward(s, d_ids, [i * B for i in range(S + 1)], B)
            ctx.backward(s, grads)
            incremental = s.incremental_stats()
        else:
            for w in ws:
                w.enable_incremental(1 << 10)
            W.group_forward(ws, [d_ids, d_ids], B)
            W.group_backward(ws, [grads, grads])
            incremental = ws[0].incremental_stats()
            assert ws[0].status() == (False, False)
        torch.cuda.synchronize()
        assert _keys_and_ints(table.counters(), COUNTERS)["admitted"] == mine
        assert _keys_and_ints(table.index_stats(), INDEX_STATS)["live"] == mine
        assert _keys_and_ints(table.tier_stats(), TIER_STATS)["host_rows"] == 0
        assert _keys_and_ints(table.stage_stats(), STAGE_STATS) == dict.fromkeys(STAGE_STATS, 0)
        assert _keys_and_ints(incremental, INCREMENTAL_STATS)["held"] == mine
        assert _keys_and_ints(ctx.batch_stats(), BATCH_STATS)["occurrences"] == S * B
        _keys_and_ints(SH.hot_geometry(DIM, True), HOT_GEOMETRY)
    finally:
        _close(torch, *objs)
