"""GPU: growable tables (pb_table_set_growth).  Every run is checked bit for bit against an eager twin of the same
capacity fed the same seeded calls: outputs, entries, counters and the resident list.  storage_stats shows the growth
events, and the allocator's refusals of rows that are not backed stay 0."""
import ctypes as C

import numpy as np
import pytest

from util import DEV, make_batch, same_bits, to_dev_i32, to_dev_ids

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return torch


@pytest.fixture(scope="module")
def lib(torch):
    from persia_b200 import native as N

    lib = N.load()
    lib.pb_debug_owned.restype = C.c_int
    lib.pb_debug_owned.argtypes = [C.POINTER(C.c_uint64)]
    lib.pb_debug_refuse_after.restype = None
    lib.pb_debug_refuse_after.argtypes = [C.c_int64]
    return lib


def _owned(lib):
    out = (C.c_uint64 * 2)()
    assert lib.pb_debug_owned(out) == 0
    return int(out[0]), int(out[1])


OPTIM = {  # kind -> EmbeddingShard.set_optimizer kwargs
    "sgd": dict(kind=0, lr=0.05),
    "adagrad": dict(kind=1, lr=0.02, initialization=0.01),
    "adagrad_intel": dict(kind=1, lr=0.02, initialization=0.01),
    "adagrad_vw": dict(kind=2, lr=0.02, initialization=0.01),
    "adam": dict(kind=3, lr=0.01, eps=1e-8),
}


def _shard(pb, dim, capacity, kind, grow, evict=None):
    s = pb.EmbeddingShard(dim, capacity, 0, grow=grow)
    s.set_optimizer(**OPTIM[kind])
    if kind == "adagrad_intel":
        s.set_rsqrt("intel")
    s.configure()
    if evict:
        s.set_eviction(**evict)
    return s


def _same_tables(torch, a, b, extra_signs=None):
    """a and b hold the same entries, counters and resident list (signs and their recency)."""
    ca, cb = a.counters(), b.counters()
    assert ca == cb, (ca, cb)
    sa, ra = a.export_signs()
    sb, rb = b.export_signs()
    assert torch.equal(sa, sb) and torch.equal(ra, rb)
    signs = sa if extra_signs is None else torch.cat([sa, extra_signs])
    if signs.numel():
        ea, fa = a.get_entries(signs)
        eb, fb = b.get_entries(signs)
        assert torch.equal(fa, fb)
        assert same_bits(ea.cpu().numpy(), eb.cpu().numpy())


class _Storage:
    """storage_stats over a run: growth events of the rows and of the index, and the refused-unmapped counter."""

    def __init__(self, s):
        self.s, self.row_growths, self.index_growths = s, 0, 0
        st = s.storage_stats()
        self.rows, self.cells = st["mapped_rows"], st["index_cells"]

    def note(self):
        st = self.s.storage_stats()
        assert st["refused_unmapped"] == 0
        assert st["mapped_rows"] <= st["reserved_rows"]
        self.row_growths += st["mapped_rows"] > self.rows
        self.index_growths += st["index_cells"] > self.cells
        self.rows, self.cells = st["mapped_rows"], st["index_cells"]


# ----------------------------------------------------------------------------------------------------- 1. parity
@pytest.mark.parametrize("kind", list(OPTIM))
def test_parity_with_growth(torch, kind):
    """Summation slots (ragged, single-id, two sharing a feature group) and a raw slot train both twins until the
    capacity is reached and eviction runs; pb_set_rows and a re-inserted checkpoint of entries (pb_image_insert's own
    path, pb_set_rows) land in between."""
    import persia_b200.shard as pb

    rng = np.random.default_rng(7)
    dim, cap, B = 8, 200_000, 2048
    pf = [1 << 56, 2 << 56, 2 << 56, 3 << 56]  # slots 1 and 2 share a feature group
    raw_pf = 4 << 56
    # every request checks, and low water exceeds what one call admits: no admission ever finds the table full (which
    # of several racing admissions gets the last free row is not deterministic, on any table)
    evict = dict(check_every=1, low_water=cap // 4, target_free=cap // 2, keep_batches=2)
    twins = [_shard(pb, dim, cap, kind, grow, evict) for grow in (False, True)]
    ctxs = [pb.BatchContext(1 << 16, 1 << 14, pf) for _ in twins]
    raws = [pb.BatchContext(1 << 14, 1 << 13, [raw_pf]) for _ in twins]
    track = _Storage(twins[1])
    seen = set()
    for step in range(26):
        ids, row_off, slot_off = make_batch(rng, 4, B, [1 << 20, 1 << 20, 1 << 20, 400], max_ids=3)
        ro = to_dev_i32(row_off, DEV)
        g = (rng.standard_normal((4, B, dim)) * 1e-2).astype(np.float16)
        raw_n = rng.integers(1, 4, size=B)
        raw_off = np.zeros(B + 1, np.uint32)
        raw_off[1:] = np.cumsum(raw_n)
        raw_ids = rng.integers(0, 1 << 22, size=int(raw_off[-1]), dtype=np.uint64)
        for k in range(4):
            seen.update((ids[slot_off[k]:slot_off[k + 1]] + np.uint64(k << 50)).tolist())
        outs, raw_outs = [], []
        for s, ctx, rctx in zip(twins, ctxs, raws):
            outs.append(ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=ro).cpu().numpy())
            ctx.backward(s, [torch.from_numpy(g[i]).to(DEV) for i in range(4)])
            table, index, non_empty, sample_id_num, counts = rctx.forward_raw(s, to_dev_ids(raw_ids, DEV), B, 4,
                                                                             row_off=to_dev_i32(raw_off, DEV))
            u = int(counts[0])
            raw_outs.append((table[:u + 1].cpu().numpy(), index.cpu().numpy(), counts.cpu().numpy()))
            rg = torch.from_numpy((np.random.default_rng(step).standard_normal((u, dim)) * 1e-2).astype(np.float32))
            rctx.backward_raw(s, rg.to(DEV))
        assert same_bits(outs[0], outs[1]), step
        for x, y in zip(raw_outs[0], raw_outs[1]):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), step
        if step in (5, 17):  # set_embedding of fresh and resident signs, as a checkpoint load inserts them
            signs = np.concatenate([rng.integers(1 << 40, 1 << 41, size=30_000, dtype=np.uint64),
                                    ids[:1000]])
            signs = np.unique(signs)
            ent = torch.from_numpy(rng.standard_normal((signs.size, twins[0].entry_len)).astype(np.float32)).to(DEV)
            for s in twins:
                s.set_entries(to_dev_ids(signs, DEV), ent)
        track.note()
    torch.cuda.synchronize()
    _same_tables(torch, twins[0], twins[1])
    assert len(seen) > cap and twins[1].counters()["capacity_refused"] == 0  # so eviction ran
    assert track.row_growths >= 5 and track.index_growths >= 2, (track.row_growths, track.index_growths)
    assert twins[1].storage_stats()["mapped_rows"] <= cap
    for x in ctxs + raws + twins:
        x.close()


# --------------------------------------------------------------------------------------- 2. batches in flight
@pytest.mark.parametrize("n_streams", [2, 4])
def test_batches_in_flight(torch, n_streams):
    """n_streams training batches in flight at once, each on its own stream and context, each admitting new signs
    across a chunk boundary: equal to the same batches run one after another on an eager table."""
    import persia_b200.shard as pb

    rng = np.random.default_rng(11 + n_streams)
    dim, cap, B, S = 16, 1_000_000, 4096, 2
    pf = [1 << 56, 2 << 56]
    grow, eager = _shard(pb, dim, cap, "adagrad", True), _shard(pb, dim, cap, "adagrad", False)
    streams = [torch.cuda.Stream() for _ in range(n_streams)]
    gctx = [pb.BatchContext(S * B, S * B, pf) for _ in range(n_streams)]
    ectx = pb.BatchContext(S * B, S * B, pf)
    track = _Storage(grow)
    for rnd in range(6):
        # batch i of every round draws from its own key range: batches in flight share no sign
        batches = []
        for i in range(n_streams):
            ids = (rng.integers(0, 40_000 * (rnd + 1), size=S * B, dtype=np.uint64) + np.uint64(i << 40))
            g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
            batches.append((ids, g))
        outs = [None] * n_streams
        for i, (ids, g) in enumerate(batches):
            with torch.cuda.stream(streams[i]):
                outs[i] = gctx[i].forward(grow, to_dev_ids(ids, DEV), [0, B, 2 * B], B)
        for i, (ids, g) in enumerate(batches):
            with torch.cuda.stream(streams[i]):
                gctx[i].backward(grow, [torch.from_numpy(g[k]).to(DEV) for k in range(S)])
        torch.cuda.synchronize()
        for i, (ids, g) in enumerate(batches):
            want = ectx.forward(eager, to_dev_ids(ids, DEV), [0, B, 2 * B], B)
            ectx.backward(eager, [torch.from_numpy(g[k]).to(DEV) for k in range(S)])
            assert same_bits(outs[i].cpu().numpy(), want.cpu().numpy()), (rnd, i)
        track.note()
    torch.cuda.synchronize()
    _same_tables(torch, eager, grow)
    assert track.row_growths >= 2
    for x in gctx + [ectx, grow, eager]:
        x.close()


# ------------------------------------------------------------------------------- 3. a capacity no card reserves
def test_capacity_beyond_hbm(torch, lib):
    """capacity 1e9 at dim 64 with SGD would reserve 256 GB of rows and a 2^31-cell index (32 GB): a growable table
    trains 100 steps over ~1e6 distinct signs, equal to an eager table large enough for them, and holds at most
    twice what its resident rows and its index need."""
    import persia_b200.shard as pb

    rng = np.random.default_rng(3)
    dim, B, S = 64, 4096, 4
    pf = [(i + 1) << 56 for i in range(S)]
    eager = _shard(pb, dim, 1 << 21, "sgd", False)
    ectx, gctx = pb.BatchContext(S * B, S * B, pf), pb.BatchContext(S * B, S * B, pf)
    eager.get_entries(to_dev_ids(np.zeros(1, np.uint64), DEV))  # the eager twin's storage, before the count starts
    torch.cuda.synchronize()
    before = _owned(lib)[1]
    grow = _shard(pb, dim, 1_000_000_000, "sgd", True)
    grow.get_entries(to_dev_ids(np.zeros(1, np.uint64), DEV))  # (the twin's miss, counted alike)
    stride = dim
    for step in range(100):
        ids = rng.integers(0, 250_000, size=S * B, dtype=np.uint64)
        g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
        off = [k * B for k in range(S + 1)]
        got = gctx.forward(grow, to_dev_ids(ids, DEV), off, B)
        gctx.backward(grow, [torch.from_numpy(g[k]).to(DEV) for k in range(S)])
        want = ectx.forward(eager, to_dev_ids(ids, DEV), off, B)
        ectx.backward(eager, [torch.from_numpy(g[k]).to(DEV) for k in range(S)])
        if step % 10 == 9:
            assert same_bits(got.cpu().numpy(), want.cpu().numpy()), step
            st = grow.storage_stats()
            live = grow.counters()["admitted"]
            need = live * (stride * 4 + 20) + st["index_cells"] * 16
            assert _owned(lib)[1] - before <= 2 * need + (64 << 20), (step, _owned(lib)[1] - before, need)
            assert st["refused_unmapped"] == 0 and st["reserved_rows"] == 1_000_000_000
    torch.cuda.synchronize()
    assert grow.counters()["admitted"] > 750_000  # (1.6e6 draws from 1e6 keys)
    _same_tables(torch, eager, grow)
    for x in (gctx, ectx, grow, eager):
        x.close()


# ------------------------------------------------------------------------------------------------- 4. capture
def test_capture_maps_full_capacity(torch):
    """A step captured on a growable table backs its whole capacity first; its replays equal eager steps."""
    import persia_b200.shard as pb

    rng = np.random.default_rng(5)
    dim, cap, B, S = 16, 300_000, 1024, 2
    pf = [1 << 56, 2 << 56]
    grow, eager = _shard(pb, dim, cap, "adam", True), _shard(pb, dim, cap, "adam", False)
    gctx, ectx = pb.BatchContext(S * B, S * B, pf), pb.BatchContext(S * B, S * B, pf)
    ids_dev = torch.zeros(S * B, dtype=torch.int64, device=DEV)
    g_dev = torch.zeros((S, B, dim), dtype=torch.float16, device=DEV)
    out = torch.empty((S, B, dim), dtype=torch.float16, device=DEV)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        gctx.forward(grow, ids_dev, [0, B, 2 * B], B, out=out)  # warm-up: a real step
        gctx.backward(grow, [g_dev[k] for k in range(S)])
        stream.synchronize()
        assert grow.storage_stats()["mapped_rows"] < cap
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            gctx.forward(grow, ids_dev, [0, B, 2 * B], B, out=out)
            gctx.backward(grow, [g_dev[k] for k in range(S)])
    st = grow.storage_stats()
    assert st["mapped_rows"] == cap and st["index_cells"] == 1 << 19, st
    ectx.forward(eager, ids_dev, [0, B, 2 * B], B)
    ectx.backward(eager, [g_dev[k] for k in range(S)])
    for it in range(8):
        ids = rng.integers(0, 1 << 30, size=S * B, dtype=np.uint64)
        g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
        ids_dev.copy_(to_dev_ids(ids, DEV))
        g_dev.copy_(torch.from_numpy(g).to(DEV))
        torch.cuda.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        want = ectx.forward(eager, ids_dev, [0, B, 2 * B], B)
        ectx.backward(eager, [g_dev[k] for k in range(S)])
        torch.cuda.synchronize()
        assert same_bits(out.cpu().numpy(), want.cpu().numpy()), it
    _same_tables(torch, eager, grow)
    del graph
    for x in (gctx, ectx, grow, eager):
        x.close()


# ------------------------------------------------------------------------------------------------- 5. refusals
def test_refused_growth_leaves_the_table_as_it_was(torch, lib):
    """Every chunk a growing call acquires (rows, row recency, free-row stack, rebuild pairs, index) is refused in
    turn: each try fails with PB_ERR_CUDA, holds nothing new, enqueues nothing; the run then goes on and ends equal to
    an unrefused one.  Closing gives everything back."""
    import persia_b200.shard as pb
    from persia_b200 import native as N

    import gc

    rng = np.random.default_rng(9)
    dim, cap = 32, 2_000_000
    gc.collect()
    torch.cuda.synchronize()
    start = _owned(lib)
    grow, eager = _shard(pb, dim, cap, "adagrad", True), _shard(pb, dim, cap, "adagrad", False)
    for s in (grow, eager):  # first allocation and a scratch for every call below: only growth acquires in the loop
        s.get_entries(to_dev_ids(np.zeros(500_000, np.uint64), DEV))
    refused = 0
    for rnd in range(3):
        signs = np.unique(rng.integers(0, 1 << 50, size=150_000 * (rnd + 1), dtype=np.uint64))
        ent = torch.from_numpy(rng.standard_normal((signs.size, grow.entry_len)).astype(np.float32)).to(DEV)
        eager.set_entries(to_dev_ids(signs, DEV), ent)
        for k in range(64):
            torch.cuda.synchronize()
            held = _owned(lib)
            lib.pb_debug_refuse_after(k)
            try:
                grow.set_entries(to_dev_ids(signs, DEV), ent)
            except N.PersiaB200Error as e:
                assert e.code == N.PB_ERR_CUDA
                torch.cuda.synchronize()
                assert _owned(lib) == held, k
                refused += 1
                continue
            finally:
                lib.pb_debug_refuse_after(-1)
            break
        assert grow.storage_stats()["refused_unmapped"] == 0
    assert refused >= 6, refused  # the rows' five regions and the index, at least once each
    torch.cuda.synchronize()
    _same_tables(torch, eager, grow)
    grow.close()
    eager.close()
    torch.cuda.synchronize()
    assert _owned(lib) == start


def test_refused_calls(torch):
    """Growth chosen after the first allocation or on a host table, and exports or a tier of a growable table, are
    refused with PB_ERR_STATE."""
    import persia_b200.shard as pb
    from persia_b200 import native as N

    lib = N.load()
    s = _shard(pb, 8, 1 << 16, "sgd", False)
    s.lookup(to_dev_ids(np.arange(10, dtype=np.uint64), DEV))
    assert lib.pb_table_set_growth(s.h, 1) == -3
    host = pb.EmbeddingShard(8, 1 << 16, 0, host=True)
    assert lib.pb_table_set_growth(host.h, 1) == -3
    g = _shard(pb, 8, 1 << 16, "sgd", True)
    g.lookup(to_dev_ids(np.arange(10, dtype=np.uint64), DEV))
    buf = C.create_string_buffer(int(lib.pb_table_view_bytes()))
    assert lib.pb_table_export_view(g.h, buf) == -3
    assert lib.pb_table_export_live_view(g.h, buf) == -3
    host.set_optimizer(**OPTIM["sgd"])
    assert lib.pb_table_attach_tier(g.h, host.h) == -3
    with pytest.raises(ValueError):
        pb.EmbeddingShard(8, 1 << 16, 0, tier_rows=100, grow=True)
    for x in (s, g, host):
        x.close()


# ---------------------------------------------------------------------------------------------- 7. R-GPU owners
@pytest.mark.parametrize("R", [2, 4])
def test_r_gpu_owners(torch, R):
    """R virtual ranks on one GPU with growable owner tables, summation and raw slots: equal to eager owners."""
    import persia_b200.shard as pb
    from persia_b200.worker import ShardedEmbeddingWorker as SW, ShardedRawWorker as RW

    rng = np.random.default_rng(21 + R)
    dim, B, cap = 16, 2048, 1_000_000
    pf = [1 << 56, 2 << 56]
    opt = OPTIM["adagrad"]
    groups = {}
    for grow in (False, True):
        sw = SW.local_group(R, 2, dim, pf, cap, cap=2 * B, optimizer=opt, max_batch=B, grow=grow)
        rw = RW.local_group(R, 1, dim, [3 << 56], cap, cap=3 * B, optimizer=opt, max_batch=B, max_ids_per_sample=3,
                            shards=[w.shard for w in sw])
        groups[grow] = (sw, rw)
    tracks = [_Storage(w.shard) for w in groups[True][0]]
    for step in range(12):
        ids = [rng.integers(0, 30_000 * (step + 1), size=2 * B, dtype=np.uint64) for _ in range(R)]
        g = [(rng.standard_normal((2, B, dim)) * 1e-2).astype(np.float16) for _ in range(R)]
        raw = []
        for _ in range(R):
            n = rng.integers(1, 4, size=B)
            off = np.zeros(B + 1, np.uint32)
            off[1:] = np.cumsum(n)
            raw.append((rng.integers(0, 1 << 30, size=int(off[-1]), dtype=np.uint64), off))
        res = {}
        for grow, (sw, rw) in groups.items():
            outs = SW.group_forward(sw, [to_dev_ids(x, DEV) for x in ids], B, training=True)
            routs = RW.group_forward_raw(rw, [to_dev_ids(x, DEV) for x, _ in raw], B, 4,
                                         row_offs=[to_dev_i32(o, DEV) for _, o in raw])
            torch.cuda.synchronize()
            res[grow] = ([o.cpu().numpy() for o in outs], [[t.cpu().numpy() for t in ro] for ro in routs])
            SW.group_backward(sw, [[torch.from_numpy(g[r][k]).to(DEV) for k in range(2)] for r in range(R)])
            us = [int(ro[4][0]) for ro in routs]
            rg = [torch.from_numpy((np.random.default_rng(step * 8 + r).standard_normal((us[r], dim)) * 1e-2)
                                   .astype(np.float32)).to(DEV) for r in range(R)]
            RW.group_backward_raw(rw, rg)
            torch.cuda.synchronize()
        for r in range(R):
            assert same_bits(res[False][0][r], res[True][0][r]), (step, r)
            u = int(res[False][1][r][4][0])
            assert same_bits(res[False][1][r][0][:u + 1], res[True][1][r][0][:u + 1]), (step, r)
            assert np.array_equal(res[False][1][r][1], res[True][1][r][1])
        for t in tracks:
            t.note()
    for r in range(R):
        _same_tables(torch, groups[False][0][r].shard, groups[True][0][r].shard)
    assert sum(t.row_growths for t in tracks) >= R
    for sw, rw in groups.values():
        for w in rw + sw:
            w.close()
