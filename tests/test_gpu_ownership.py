"""GPU: the CUDA resources the C ABI's objects hold (persia_b200/csrc/pb_own.cuh).  Every object gives back all it
holds when it is closed, and a create or lazy step whose acquisition fails leaves nothing allocated by it and no gate
set: the object stays usable, and a later call acquires afresh.  The failures are refusals the library makes itself
(pb_debug_refuse_after), before any CUDA call: no device state is touched."""
import ctypes as C
import gc

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S, B, DIM, CARD, FIXED = 2, 64, 32, 600, 3
PF = [s << 56 for s in range(S)]
SLOT_OFF = [s * B for s in range(S + 1)]
# HBM rows of the tables that evict, and a check before every training request that leaves room for two whole batches
# (S * B signs each): no admission is refused, so which signs get rows never depends on the order the device serves
# them in, while the signs of a few steps (CARD per slot) still outgrow the rows
ROWS = 512
EVICT = dict(check_every=1, low_water=2 * S * B, target_free=2 * S * B + 32, keep_batches=1)


@pytest.fixture(scope="module")
def torch():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


@pytest.fixture(scope="module")
def lib(torch):
    from persia_b200 import native as N

    lib = N.load()
    lib.pb_debug_owned.restype = C.c_int
    lib.pb_debug_owned.argtypes = [C.POINTER(C.c_uint64)]
    lib.pb_debug_refuse_after.restype = None
    lib.pb_debug_refuse_after.argtypes = [C.c_int64]
    lib.pb_debug_table_seq.restype = C.c_int
    lib.pb_debug_table_seq.argtypes = [C.c_void_p, C.POINTER(C.c_uint32)]
    return lib


def _owned(lib):
    """(resources, device + host bytes) every live object holds."""
    from persia_b200 import native as N

    out = (C.c_uint64 * 2)()
    N.check(lib.pb_debug_owned(out))
    return int(out[0]), int(out[1])


def _attempt(torch, lib, refuse, call, steps=1):
    """call() once (refuse False), or with the (n+1)-th acquisition refused for n = 0, 1, ... until it succeeds: every
    refused try raises PB_ERR_CUDA and leaves what the objects hold as it was.  Returns (result, refused tries).
    steps > 1: the call acquires in that many steps, each committed on its own once it has succeeded (a later call
    needs them and does not acquire them again); a refused try then leaves at most what its earlier steps hold, and the
    test's last check (everything given back once closed) shows that none of it leaks."""
    from persia_b200 import native as N

    if not refuse:
        return call(), 0
    for n in range(1000):
        gc.collect()
        torch.cuda.synchronize()
        before = _owned(lib)
        gc.disable()  # (no object of an earlier step is closed during the call)
        lib.pb_debug_refuse_after(n)
        try:
            res = call()
        except N.PersiaB200Error as e:
            assert e.code == N.PB_ERR_CUDA, str(e)
            after = _owned(lib)
            assert after == before if steps == 1 else after[0] >= before[0], (n, str(e))
            continue
        finally:
            lib.pb_debug_refuse_after(-1)
            gc.enable()
        return res, n
    raise AssertionError("never succeeded")


def _opt(N, kind):
    if kind == N.OPT_ADAM:
        return dict(kind=kind, lr=0.01, beta1=0.9, beta2=0.999, eps=1e-8)
    return dict(kind=kind, lr=0.02, initialization=0.01, eps=1e-10)


def _shard(N, SH, kind=None, capacity=1 << 12, **kw):
    s = SH.EmbeddingShard(DIM, capacity, 0, **kw)
    s.set_optimizer(**_opt(N, N.OPT_ADAGRAD if kind is None else kind))
    s.configure()
    return s


def _steps(torch, seed, n=3, batch=B):
    rng = np.random.default_rng(seed)
    return [(torch.from_numpy(rng.integers(0, CARD, size=S * batch, dtype=np.uint64).view(np.int64)).to(DEV),
             torch.from_numpy((rng.standard_normal((S, batch, DIM)) * 1e-2).astype(np.float16)).to(DEV))
            for _ in range(n)]


def _train(ctx, s, steps):
    outs = []
    for ids, g in steps:
        outs.append(ctx.forward(s, ids, SLOT_OFF, B).cpu().numpy())
        ctx.backward(s, g)
    return outs


def _entries(torch, SH, s, steps):
    signs = torch.cat([SH.add_prefix(ids, [k * (ids.numel() // S) for k in range(S + 1)], PF) for ids, _ in steps])
    ent, found = s.get_entries(signs)
    return [ent.cpu().numpy(), found.cpu().numpy()]


def _ctx(SH, n_slots=S):
    return SH.BatchContext(n_slots * B * 4, n_slots * B, PF[:n_slots])


# ---- every object, closed: back to what was held before ---------------------------------------------------------------
def test_every_object_gives_back_what_it_holds(torch, lib):
    from persia_b200 import native as N, shard as SH
    from persia_b200.checkpoint import _Image, _Pinned
    from persia_b200.worker import RemoteReader, ShardedEmbeddingWorker as W, TierStager

    gc.collect()
    torch.cuda.synchronize()
    start = _owned(lib)
    steps = _steps(torch, 1)
    closers = []
    # an Adam table with a host tier: eviction churning, incremental updates taken, a dump part written, index stats
    t = _shard(N, SH, N.OPT_ADAM, capacity=ROWS, tier_rows=1 << 12)
    t.set_eviction(**EVICT)
    t.enable_incremental(1 << 12)
    ctx = _ctx(SH)
    _train(ctx, t, steps)
    assert len(t.take_incremental()[0]) > 0
    t.dump_reserve(1 << 20)
    image = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    meta = torch.zeros(2, dtype=torch.int64, device=DEV)
    t.dump_part(0, 1, image, meta)
    torch.cuda.synchronize()
    nbytes = int(meta[0])
    assert nbytes > 28
    t.index_stats()
    # an untiered table exported live (a tiered one refuses every export)
    u = _shard(N, SH)
    _train(ctx, u, steps[:1])
    u.export_live_view()
    with pytest.raises(N.PersiaB200Error):
        t.export_live_view()
    # a vectorwise-Adagrad table trained once (its context's vectorwise stage)
    v = _shard(N, SH, N.OPT_ADAGRAD_VW)
    _train(ctx, v, steps[:1])
    # summation and raw training on one context
    rctx = _ctx(SH, 1)
    rctx.forward(u, steps[0][0][:B], [0, B], B)
    rctx.backward(u, steps[0][1][:1])
    counts = rctx.forward_raw(u, steps[0][0][:B], B, FIXED)[4]
    rctx.backward_raw(u, torch.full((int(counts[0]), DIM), 0.01, device=DEV))
    # 2 ranks: prepare, resize, train; a stager; remote readers over untiered shards
    ws = W.local_group(2, S, DIM, PF, 1 << 12, cap=8, optimizer=_opt(N, N.OPT_ADAGRAD), max_batch=B)
    for w in ws:
        w.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    ids = [steps[r][0] for r in range(2)]
    need, f32 = W.group_prepare(ws, ids, B)
    assert W.group_resize(ws, need, f32)
    W.group_forward(ws, ids, B)
    W.group_backward(ws, [steps[r][1] for r in range(2)])
    stagers = TierStager.local_group([w.shard for w in ws], cap=S * B)
    readers = RemoteReader.local_group([w.shard for w in ws])
    readers[0].forward(ids[0], B, PF)
    torch.cuda.synchronize()
    # a checkpoint image: the dumped part, indexed from pinned host memory and inserted
    buf = _Pinned(nbytes)
    buf.view[:] = image[:nbytes].cpu().numpy()
    im = _Image(torch.device(DEV), 1 << 12)
    stream = torch.cuda.current_stream()
    summary = im.index(buf, nbytes, 0, 0xFFFFFFFF, 1, 0, stream)
    dest = _shard(N, SH, N.OPT_ADAM)
    im.insert(dest, DIM, 0, summary[0][2], False, stream)
    torch.cuda.synchronize()
    assert _owned(lib)[0] > start[0]
    for rd in readers:  # views before the tables they view
        rd.close()
    closers += stagers + ws + [im, buf, ctx, rctx, t, u, v, dest]
    for x in closers:
        x.close()
    torch.cuda.synchronize()
    assert _owned(lib) == start


# ---- refused acquisitions leave nothing behind ---------------------------------------------------------------------
def _path(torch, lib, name, refuse):
    """One seeded workload that runs the call `name` names once, refused acquisition by acquisition when `refuse`.
    Returns (what it computed, refused tries, objects to close)."""
    from persia_b200 import native as N, shard as SH
    from persia_b200.checkpoint import _Image, _Pinned
    from persia_b200.worker import RemoteReader, ShardedEmbeddingWorker as W, TierStager

    def attempt(call, steps=1):
        res, n = _attempt(torch, lib, refuse, call, steps)
        tries.append(n)
        return res

    tries, keep = [], []
    steps = _steps(torch, 7, 4)
    warm = _ctx(SH)  # a context whose backward stage is grown already (by a table of this dim)
    _train(warm, _shard(N, SH), steps[:1])
    keep.append(warm)
    out = []
    if name == "table_create":
        s = attempt(lambda: SH.EmbeddingShard(DIM, 1 << 12, 0))
        s.set_optimizer(**_opt(N, N.OPT_ADAGRAD))
        s.configure()
        out = _train(warm, s, steps)
    elif name == "first_forward":
        s = _shard(N, SH)
        out = [attempt(lambda: warm.forward(s, steps[0][0], SLOT_OFF, B)).cpu().numpy()]
        warm.backward(s, steps[0][1])
        out += _train(warm, s, steps[1:])
    elif name == "adam":
        s = SH.EmbeddingShard(DIM, 1 << 12, 0)
        attempt(lambda: s.set_optimizer(**_opt(N, N.OPT_ADAM)))
        s.configure()
        out = _train(warm, s, steps)
    elif name == "attach_tier":
        s = SH.EmbeddingShard(DIM, ROWS, 0, tier_rows=1 << 12)
        attempt(lambda: s.set_optimizer(**_opt(N, N.OPT_ADAGRAD)))
        s.configure()
        s.set_eviction(**EVICT)
        out = _train(warm, s, steps) + [np.array(list(s.tier_stats().values()))]
    elif name == "evict_ws":
        s = _shard(N, SH, capacity=ROWS)
        s.set_eviction(**EVICT)
        s.get_entries(steps[0][0])  # storage and scratch: the forward's only new resources are the sweep's
        out = [attempt(lambda: warm.forward(s, steps[0][0], SLOT_OFF, B)).cpu().numpy()]
        warm.backward(s, steps[0][1])
        out += _train(warm, s, steps[1:]) + [np.array(list(s.counters().values()))]
    elif name == "incremental":
        s = _shard(N, SH)
        out = _train(warm, s, steps[:1])
        attempt(lambda: s.enable_incremental(1 << 12))
        out += _train(warm, s, steps[1:])
        out += list(s.take_incremental()[:2])
    elif name in ("dump_reserve", "image_index"):
        s = _shard(N, SH)
        out = _train(warm, s, steps)
        if name == "dump_reserve":
            attempt(lambda: s.dump_reserve(1 << 20))
        else:
            s.dump_reserve(1 << 20)
        image = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
        meta = torch.zeros(2, dtype=torch.int64, device=DEV)
        s.dump_part(0, 1, image, meta)
        torch.cuda.synchronize()
        nbytes = int(meta[0])
        out.append(image[:nbytes].cpu().numpy())
        if name == "image_index":
            buf = _Pinned(nbytes)
            buf.view[:] = out[-1]
            im = _Image(torch.device(DEV), 1 << 12)
            stream = torch.cuda.current_stream()
            # (three steps: the summary words, the position arrays, and the inserts' staging once the summary is read)
            summary = attempt(lambda: im.index(buf, nbytes, 0, 0xFFFFFFFF, 1, 0, stream), steps=3)
            dest = _shard(N, SH)
            im.insert(dest, DIM, 0, summary[0][2], False, stream)
            out += _entries(torch, SH, dest, steps)
            keep += [im, buf, dest]
    elif name == "export_live":
        s = _shard(N, SH)
        out = _train(warm, s, steps[:1])
        attempt(lambda: s.export_live_view())
        seq = C.c_uint32(1)
        N.check(lib.pb_debug_table_seq(s.h, C.byref(seq)))
        assert seq.value == 0
        out += _train(warm, s, steps[1:])
    elif name == "ctx_create":
        s = _shard(N, SH)
        ctx = attempt(lambda: _ctx(SH))
        out = _train(ctx, s, steps)
        keep.append(ctx)
    elif name == "raw":  # ensure_raw (an inference forward), then the training forward's raw stage
        s = _shard(N, SH)
        _train(warm, s, steps[:1])
        rctx = _ctx(SH, 1)
        ids = steps[1][0][:B]
        out = [x.cpu().numpy() for x in attempt(lambda: rctx.forward_raw(s, ids, B, FIXED, training=False))]
        got = attempt(lambda: rctx.forward_raw(s, ids, B, FIXED))
        out += [x.cpu().numpy() for x in got]
        rctx.backward_raw(s, torch.full((int(got[4][0]), DIM), 0.01, device=DEV))
        keep.append(rctx)
    elif name == "hot_stage":
        s = _shard(N, SH)
        s.get_entries(steps[0][0])
        ctx = _ctx(SH)
        out = [attempt(lambda: ctx.forward(s, steps[0][0], SLOT_OFF, B)).cpu().numpy()]
        ctx.backward(s, steps[0][1])
        out += _train(ctx, s, steps[1:])
        keep.append(ctx)
    elif name == "vw_stage":
        s = _shard(N, SH, N.OPT_ADAGRAD_VW)
        out = [warm.forward(s, steps[0][0], SLOT_OFF, B).cpu().numpy()]
        attempt(lambda: warm.backward(s, steps[0][1]))
        out += _train(warm, s, steps[1:])
    elif name == "remote_stage":
        shards = [_shard(N, SH) for _ in range(2)]
        for sh in shards:
            _train(warm, sh, steps)
        readers = RemoteReader.local_group(shards)
        readers[0]._ctx(("sum", tuple(PF), None, 8), S * B, S * B)  # the context only: the forward's stage is new
        out = [attempt(lambda: readers[0].forward(steps[0][0], B, PF)).cpu().numpy()]
        torch.cuda.synchronize()
        for rd in readers:
            rd.close()
        keep += shards
    elif name in ("xchg_create", "xchg_create_stage"):
        ws = W.local_group(2, S, DIM, PF, ROWS, cap=8, optimizer=_opt(N, N.OPT_ADAGRAD), max_batch=B,
                           tier_rows=1 << 12)
        for w in ws:
            w.shard.set_eviction(**EVICT)
            w.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
        torch.cuda.synchronize()
        stagers = None
        if name == "xchg_create_stage":
            areas, bases = W._local_areas(2, TierStager.area_bytes(2, S * B), torch.device(DEV))
            stagers = [attempt(lambda r=r: TierStager(ws[r].shard, r, 2, S * B, areas[r], bases)) for r in range(2)]
        for k in range(2):
            ids = [steps[k + r][0] for r in range(2)]
            need, f32 = W.group_prepare(ws, ids, B)
            to = ws[0]._resize_to(need, f32)
            if to is not None:  # group_resize, each rank's new exchange under refusals
                areas, bases = W._local_areas(2, W.area_bytes(2, to[0], DIM, to[1]), torch.device(DEV))
                for r, w in enumerate(ws):
                    if name == "xchg_create":
                        attempt(lambda w=w, r=r: w._replace_xchg(*to, areas[r], bases))
                    else:
                        w._replace_xchg(*to, areas[r], bases)
            outs = W.group_forward(ws, ids, B)
            if stagers:
                TierStager.group_stage(stagers, [steps[k + 1 + r][0] for r in range(2)], [SLOT_OFF] * 2, PF)
            W.group_backward(ws, [steps[k + r][1] for r in range(2)])
            out += [o.cpu().numpy() for o in outs]
        out += [x for w in ws for x in _entries(torch, SH, w.shard, steps)]
        keep += (stagers or []) + ws
    elif name == "view_open":
        s = _shard(N, SH)
        out = _train(warm, s, steps)
        view = attempt(lambda: SH.TableView(s.export_view()))
        keep += [s, view]
        return out, tries, keep
    else:
        raise AssertionError(name)
    if name not in ("remote_stage", "xchg_create", "xchg_create_stage", "image_index") and "s" in locals():
        out += _entries(torch, SH, s, steps)
        keep.append(s)
    return out, tries, keep


PATHS = ["table_create", "first_forward", "adam", "attach_tier", "evict_ws", "incremental", "dump_reserve",
         "export_live", "ctx_create", "raw", "hot_stage", "vw_stage", "remote_stage", "xchg_create", "xchg_create_stage",
         "image_index", "view_open"]


@pytest.mark.parametrize("name", PATHS)
def test_refused_acquisitions_leave_nothing_behind(torch, lib, name):
    """The call is refused at its first, second, ... acquisition until it succeeds.  Every refused try fails with
    PB_ERR_CUDA and leaves what the objects hold as it was; the object stays usable, and the run's outputs and entries
    equal those of a run without refusals bit for bit."""
    gc.collect()
    torch.cuda.synchronize()
    start = _owned(lib)
    runs = []
    for refuse in (False, True):
        out, tries, keep = _path(torch, lib, name, refuse)
        torch.cuda.synchronize()
        runs.append(out)
        for x in reversed(keep):
            x.close()
        if refuse:
            assert all(n >= 1 for n in tries) or name == "view_open", tries
    gc.collect()
    torch.cuda.synchronize()
    assert len(runs[0]) == len(runs[1])
    for a, b in zip(*runs):
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    assert _owned(lib) == start
