"""GPU: J batches in flight on J streams against one table (embedding_staleness J: one context and one stream per
batch, calls pipelined as bench.py's in-flight legs issue them, forward k+1 before backward k, no syncs between the
streams), against a model that applies the same batches one after another.

Every result here is independent of the order the batches are applied in, so one answer is right: SGD with wd 0 and
lr 2^-4, rows set to dyadic values of a few bits, gradients that are small integers times 2^-10 (f16 and f32), loss
scales that are powers of two, ragged samples of 1 or 4 ids (1/sqrt(n) exact) and the weight bound out of reach.  Every
f32 sum and step is then exact, and every entry must match the oracle's serial run bit for bit, and a float64 sum of
each sign's gradients that does not go through the oracle.  A lost update (two backwards stepping one row at once) or a
torn entry shows up as a wrong bit pattern.

  reduce classes      cold / warm / hot / huge / giant signs, the hottest ones in every batch, dims of each hot-reduce
                      geometry (16, 64, 128, 130 f16; 64 f32)
  other steps         pb_backward_raw beside the summation backwards, pb_update on a stream of its own, with and
                      without a host tier
  Adam                N requests over J streams, then one serial step on fresh rows: it exposes the beta powers
  incremental set     batches of different sizes (different mark grids): the mirror, the take, one more mark
  eviction            check_every 1, keep 1: the same as the same calls on one stream, no sign in two cells
  one capture         J contexts forked onto side streams of one CUDA graph capture, replayed

Every wait on the device is bounded (_drain): a run that does not finish ends the process instead of waiting forever.
"""
import os
import sys
import time

import numpy as np
import pytest

from util import DEV, to_dev_i32, to_dev_ids

pytestmark = pytest.mark.gpu

SGD, ADAM = 0, 3
LR = 2.0 ** -4
GU = 2.0 ** -10          # gradient unit
COUNTS = [1500, 400, 100, 12]  # occurrences per 4096 of ids 0..3: giant, huge, hot, warm; the rest of a slot is drawn
POOL = 3000                    # from ids 4..POOL-1 (cold and warm)
SCALES = [2.0, 0.5]            # loss scale of slot 0 (one id per sample) and slot 1 (ragged, sqrt scaling)
HYPER = dict(enable_weight_bound=True, weight_bound=1e30)
RAW_FIXED = 4


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


def _drain(torch, streams, timeout=120.0):
    """Waits for the work enqueued so far on `streams` and the current stream, polling with a deadline.  A run that is
    still going after `timeout` seconds (a probe walking a corrupt index) ends the process: a hung kernel cannot be
    cancelled, and a test that went on would only wait on it again."""
    evs = []
    for st in list(streams) + [torch.cuda.current_stream()]:
        ev = torch.cuda.Event()
        ev.record(st)
        evs.append(ev)
    end = time.monotonic() + timeout
    while not all(ev.query() for ev in evs):
        if time.monotonic() > end:
            sys.stderr.write(f"test_gpu_streams: device work still running after {timeout:.0f} s; exiting\n")
            sys.stderr.flush()
            os._exit(3)
        time.sleep(0.001)


def _gate(torch, streams, cycles=200_000_000):
    """Holds `streams` behind one spinning kernel (about 0.1 s) so that the calls issued next are all queued before any
    of them runs: the batches then overlap on the device instead of each finishing while the host issues the next."""
    gate = torch.cuda.Stream()
    with torch.cuda.stream(gate):
        torch.cuda._sleep(cycles)
    for st in streams:
        st.wait_stream(gate)


# ---- batches ---------------------------------------------------------------------------------------------------------
def _slot_ids(rng, n, base):
    """n ids: ids base+0..3 at COUNTS (scaled to n) positions, the rest drawn from base+4..base+POOL-1."""
    ids = rng.integers(len(COUNTS), POOL, size=n).astype(np.uint64)
    pos = rng.permutation(n)
    o = 0
    for k, c in enumerate(COUNTS):
        c = max(1, c * n // 4096)
        ids[pos[o:o + c]] = k
        o += c
    return ids + np.uint64(base)


def _batch(rng, B, f32, dim, base=0):
    """Slot 0: one id per sample; slot 1: 1 or 4 ids per sample (sqrt scaling).  Gradients are integers in -4..4
    times 2^-10."""
    cnt1 = rng.choice(np.array([1, 4], np.uint32), size=B)
    ids0, ids1 = _slot_ids(rng, B, base), _slot_ids(rng, int(cnt1.sum()), base)
    row_off = np.zeros(2 * B + 1, np.uint32)
    row_off[1:] = np.cumsum(np.concatenate([np.ones(B, np.uint32), cnt1]))
    g = (rng.integers(-4, 5, size=(2, B, dim)) * GU).astype(np.float32 if f32 else np.float16)
    return dict(ids=np.concatenate([ids0, ids1]), slots=[ids0, ids1], cnt1=cnt1, row_off=row_off,
                slot_off=[0, B, B + ids1.size], B=B, g=g)


def _raw_batch(rng, B, dim):
    """A raw slot: 1..3 ids per sample from 64 ids (so its signs repeat across batches); f32 gradient rows of the
    distinct ids in first-occurrence order."""
    cnt = rng.integers(1, 4, size=B).astype(np.uint32)
    row_off = np.zeros(B + 1, np.uint32)
    row_off[1:] = np.cumsum(cnt)
    ids = rng.integers(0, 64, size=int(row_off[-1])).astype(np.uint64)
    _, first = np.unique(ids, return_index=True)
    distinct = ids[np.sort(first)]
    g = (rng.integers(-4, 5, size=(distinct.size, dim)) * GU).astype(np.float32)
    return dict(ids=ids, row_off=row_off, B=B, distinct=distinct, g=g)


class Run:
    """One table driven from several streams, the oracle driven serially in the same issue order, and a float64
    running total of every sign's gradients."""

    def __init__(self, torch, pb, oracle, dim, kind=SGD, cap=1 << 15, tier_rows=0, optim=None):
        self.torch, self.pb, self.oracle, self.dim, self.kind = torch, pb, oracle, dim, kind
        self.pf = [oracle.index_prefix(0), oracle.index_prefix(1)]
        self.raw_pf = oracle.index_prefix(2)
        optim = optim or dict(lr=LR, wd=0.0)
        self.s = pb.EmbeddingShard(dim, cap, 0, tier_rows=tier_rows)
        self.s.set_optimizer(kind, **optim)
        self.s.configure(**HYPER)
        self.w = oracle.Worker([oracle.SlotCfg(dim, sqrt_scaling=i == 1, prefix=self.pf[i]) for i in range(2)], n_ps=1)
        self.w.configure(wb=1e30)
        self.w.set_optimizer(oracle.Optim(kind, **{{"beta1": "b1", "beta2": "b2"}.get(k, k): v for k, v in optim.items()}))
        self.seed = {}
        self.total = {}
        self.keep = []  # device tensors the enqueued work still reads or writes

    def signs(self, b):
        return [self.oracle.add_prefix(b["slots"][i], 8, self.pf[i]) for i in range(2)]

    def raw_signs(self, r):
        return self.oracle.add_prefix(r["distinct"], 8, self.raw_pf)

    def set_rows(self, signs, rng):
        """Dyadic rows of a few bits (and zero optimizer state) for `signs`, on the GPU table and in the oracle."""
        signs = np.unique(np.asarray(signs, np.uint64))
        L = self.s.entry_len
        ent = np.zeros((signs.size, L), np.float32)
        ent[:, :self.dim] = rng.integers(-64, 65, size=(signs.size, self.dim)) * 2.0 ** -6
        self.s.set_entries(to_dev_ids(signs, DEV), self.torch.from_numpy(ent).to(DEV))
        self.w.set_embedding(signs, ent, self.dim)
        for k, x in enumerate(signs):
            self.seed[int(x)] = ent[k, :self.dim].astype(np.float64)
        return signs

    # float64 totals (applied to the model's rows as w - lr * total)
    def _add(self, signs, v):
        for k, x in enumerate(signs):
            x = int(x)
            self.total[x] = self.total.get(x, 0.0) + v[k]

    def add_batch(self, b):
        B = b["B"]
        for i, signs in enumerate(self.signs(b)):
            sample = np.arange(B) if i == 0 else np.repeat(np.arange(B), b["cnt1"])
            v = b["g"][i][sample].astype(np.float64) / SCALES[i]
            if i == 1:
                v /= np.sqrt(b["cnt1"][sample].astype(np.float64))[:, None]
            u, inv = np.unique(signs, return_inverse=True)
            tot = np.zeros((u.size, self.dim))
            np.add.at(tot, inv, v)
            self._add(u, tot)

    # ---- the GPU side --------------------------------------------------------------------------------------------
    def dev_batch(self, b):
        torch = self.torch
        d = dict(ids=to_dev_ids(b["ids"], DEV), row_off=to_dev_i32(b["row_off"], DEV),
                 g=[torch.from_numpy(np.ascontiguousarray(b["g"][i])).to(DEV) for i in range(2)])
        self.keep.append(d)
        return d

    def dev_raw(self, r):
        d = dict(ids=to_dev_ids(r["ids"], DEV), row_off=to_dev_i32(r["row_off"], DEV),
                 g=self.torch.from_numpy(r["g"]).to(DEV))
        self.keep.append(d)
        return d

    def forward(self, ctx, b, d):
        self.keep.append(ctx.forward(self.s, d["ids"], b["slot_off"], b["B"], row_off=d["row_off"], training=True))

    def backward(self, ctx, d):
        ctx.backward(self.s, d["g"], scales=SCALES)

    def forward_raw(self, ctx, r, d):
        self.keep.append(ctx.forward_raw(self.s, d["ids"], r["B"], RAW_FIXED, row_off=d["row_off"], training=True))

    def backward_raw(self, ctx, d):
        ctx.backward_raw(self.s, d["g"])

    # ---- the serial model ----------------------------------------------------------------------------------------
    def model_forward(self, b):
        _, octx = self.w.forward(b["ids"], b["row_off"], b["B"], training=True)
        return octx

    def model_backward(self, octx, b):
        self.w.backward(octx, [b["g"][0], b["g"][1]], scale=np.array(SCALES, np.float32))
        self.add_batch(b)

    def model_update(self, signs, g):
        """pb_update and a raw backward with scale 1 both step each (distinct) sign once with its gradient row."""
        self.w.ps_update(0, signs, np.full(signs.size, self.dim, np.uint32), g)
        self._add(signs, g.astype(np.float64))

    # ---- checks --------------------------------------------------------------------------------------------------
    def check(self, signs, f64=True, what=""):
        signs = np.unique(np.asarray(signs, np.uint64))
        ent, found = self.s.get_entries(to_dev_ids(signs, DEV))
        ent, found = ent.cpu().numpy(), found.cpu().numpy()
        assert found.all(), f"{what}: {int((~found).sum())} signs have no entry"
        ref = np.stack([self.w.get_entry(int(x)) for x in signs])
        bad = np.flatnonzero((ent.view(np.uint32) != ref.view(np.uint32)).any(axis=1))
        assert bad.size == 0, (f"{what}: {bad.size} of {signs.size} entries differ from the serial model; worst "
                               f"signs {[hex(int(x)) for x in signs[bad[:4]]]}: got {ent[bad[0], :4]} want "
                               f"{ref[bad[0], :4]}")
        if f64:
            want = np.stack([self.seed[int(x)] - LR * self.total.get(int(x), 0.0) for x in signs])
            got = ent[:, :self.dim].astype(np.float64)
            bad = np.flatnonzero((got != want).any(axis=1))
            assert bad.size == 0, (f"{what}: {bad.size} of {signs.size} rows differ from w - lr * (float64 sum of "
                                   f"their gradients); sign {int(signs[bad[0]]):#x}: got {got[bad[0], :4]} want "
                                   f"{want[bad[0], :4]}")


def _pipeline(run, ctxs, streams, batches, raws=None, raw_ctxs=None, updates=None, upd_stream=None):
    """Issues batch k on ctxs[k % J] and streams[k % J]: forward k+1 before backward k, raw batch k right after
    summation batch k on the same stream, and update k on `upd_stream`; the model applies the same calls in the same
    order.  Nothing waits between streams."""
    torch = run.torch
    J = len(ctxs)
    dev = [run.dev_batch(b) for b in batches]
    draw = [run.dev_raw(r) for r in raws] if raws else None
    dupd = [(to_dev_ids(s, DEV), torch.from_numpy(g).to(DEV)) for s, g in updates] if updates else None
    run.keep.append(dupd)
    if raws:  # a raw context's first training forward allocates its staging buffer and synchronises: not behind the gate
        for j in range(min(J, len(raws))):
            with torch.cuda.stream(streams[j]):
                run.forward_raw(raw_ctxs[j], raws[j], draw[j])
    _drain(torch, [])  # the inputs are on the device before other streams read them
    _gate(torch, streams + ([upd_stream] if updates else []))
    N = len(batches)

    def fwd(k):
        with torch.cuda.stream(streams[k % J]):
            run.forward(ctxs[k % J], batches[k], dev[k])
            if raws:
                run.forward_raw(raw_ctxs[k % J], raws[k], draw[k])

    def bwd(k):
        with torch.cuda.stream(streams[k % J]):
            run.backward(ctxs[k % J], dev[k])
            if raws:
                run.backward_raw(raw_ctxs[k % J], draw[k])
        if updates:
            with torch.cuda.stream(upd_stream):
                run.s.update(*dupd[k])

    fwd(0)
    for k in range(N):
        if k + 1 < N:
            fwd(k + 1)
        bwd(k)
    # the model, in the same order
    octx = {0: run.model_forward(batches[0])}
    for k in range(N):
        if k + 1 < N:
            octx[k + 1] = run.model_forward(batches[k + 1])
        run.model_backward(octx.pop(k), batches[k])
        if raws:
            run.model_update(run.raw_signs(raws[k]), raws[k]["g"])
        if updates:
            run.model_update(*updates[k])


def _setup(torch, pb, oracle, J, dim, f32=False, n_mult=3, seed=0, **kw):
    rng = np.random.default_rng(1000 * J + dim + 7 * f32 + seed)
    run = Run(torch, pb, oracle, dim, **kw)
    batches = [_batch(rng, 4096, f32, dim) for _ in range(n_mult * J)]
    universe = np.unique(np.concatenate([np.concatenate(run.signs(b)) for b in batches]))
    run.set_rows(universe, rng)
    ctxs = [pb.BatchContext(1 << 15, 1 << 14, run.pf, [False, True]) for _ in range(J)]
    streams = [torch.cuda.Stream() for _ in range(J)]
    return rng, run, batches, universe, ctxs, streams


@pytest.mark.parametrize("J", [2, 3, 4])
@pytest.mark.parametrize("dim,f32", [(16, False), (64, False), (128, False), (130, False), (64, True)])
def test_summation_batches_in_flight(torch_cuda, pb, oracle, J, dim, f32):
    """3J batches of 4096 samples over J streams, every one holding the same giant, huge, hot and warm signs: every
    entry equals the serial run bit for bit, and w - lr * (float64 sum of its gradients)."""
    torch = torch_cuda
    rng, run, batches, universe, ctxs, streams = _setup(torch, pb, oracle, J, dim, f32)
    _pipeline(run, ctxs, streams, batches)
    _drain(torch, streams)
    assert ctxs[0].batch_stats()["hot"] >= 3  # giant, huge and hot signs took the hot reduce
    run.check(universe, what=f"J={J} dim={dim} {'f32' if f32 else 'f16'}")
    assert run.s.counters()["wait_errors"] == 0


@pytest.mark.parametrize("J", [2, 3, 4])
@pytest.mark.parametrize("tier", [False, True])
def test_raw_and_update_beside_summation(torch_cuda, pb, oracle, J, tier):
    """Each batch also carries a raw slot (pb_backward_raw on the batch's stream) and a pb_update of the hottest
    summation signs, the raw signs and some others on a stream of its own; with and without a host tier."""
    torch = torch_cuda
    dim = 64
    rng, run, batches, universe, ctxs, streams = _setup(torch, pb, oracle, J, dim, tier_rows=(1 << 15) if tier else 0)
    raws = [_raw_batch(rng, 512, dim) for _ in batches]
    raw_universe = run.set_rows(np.unique(np.concatenate([run.raw_signs(r) for r in raws])), rng)
    raw_ctxs = [pb.BatchContext(1 << 12, 1 << 12, [run.raw_pf]) for _ in range(J)]
    updates = []
    hot = np.concatenate([oracle.add_prefix(np.arange(4, dtype=np.uint64), 8, p) for p in run.pf])
    for b in batches:
        s = np.unique(np.concatenate([hot, raw_universe[:16], rng.choice(universe, 64, replace=False)]))
        updates.append((s, (rng.integers(-4, 5, size=(s.size, dim)) * GU).astype(np.float32)))
    _pipeline(run, ctxs, streams, batches, raws=raws, raw_ctxs=raw_ctxs, updates=updates, upd_stream=torch.cuda.Stream())
    _drain(torch, streams)
    run.check(np.concatenate([universe, raw_universe]), what=f"J={J} tier={tier}")
    assert run.s.counters()["wait_errors"] == 0
    if tier:
        assert run.s.tier_stats()["host_rows"] == 0


@pytest.mark.parametrize("J", [2, 3, 4])
def test_adam_beta_powers_in_flight(torch_cuda, pb, oracle, J):
    """Adam: 3J requests over J streams advance each feature group's (beta1^t, beta2^t) 3J times.  One more request,
    issued alone on rows set fresh (m = v = 0), steps with beta^(3J+1): its rows equal the oracle's bit for bit only if
    no advance was lost."""
    torch = torch_cuda
    dim = 64
    optim = dict(lr=0.01, beta1=0.9, beta2=0.999, eps=1e-8)
    rng, run, batches, universe, ctxs, streams = _setup(torch, pb, oracle, J, dim, kind=ADAM, optim=optim)
    _pipeline(run, ctxs, streams, batches)
    _drain(torch, streams)
    last = _batch(rng, 1024, False, dim, base=POOL)  # signs no earlier batch used
    fresh = run.set_rows(np.concatenate(run.signs(last)), rng)
    d = run.dev_batch(last)
    run.forward(ctxs[0], last, d)
    run.backward(ctxs[0], d)
    run.w.backward(run.model_forward(last), [last["g"][0], last["g"][1]], scale=np.array(SCALES, np.float32))
    _drain(torch, [])
    run.check(fresh, f64=False, what=f"Adam J={J}: the step after the in-flight requests")


@pytest.mark.parametrize("J", [2, 3, 4])
def test_incremental_set_in_flight(torch_cuda, pb, oracle, J):
    """The incremental set marked from J streams by batches of different sizes (so the mark launches have different
    grids), raw backwards and updates: after a sync the mirror equals the held count, the take returns exactly the
    signs stepped, and one more mark afterwards still moves the mirror."""
    torch = torch_cuda
    dim = 32
    rng = np.random.default_rng(77 + J)
    run = Run(torch, pb, oracle, dim)
    sizes = [4096, 1024, 300, 2048, 64, 700]
    batches = [_batch(rng, sizes[k % len(sizes)], False, dim) for k in range(3 * J)]
    raws = [_raw_batch(rng, 64 + 100 * k, dim) for k in range(len(batches))]
    universe = run.set_rows(np.concatenate([np.concatenate(run.signs(b)) for b in batches]), rng)
    raw_universe = run.set_rows(np.unique(np.concatenate([run.raw_signs(r) for r in raws])), rng)
    updates = []
    for k in range(len(batches)):
        s = np.unique(rng.choice(universe, 10 + 40 * k, replace=False))
        updates.append((s, (rng.integers(-4, 5, size=(s.size, dim)) * GU).astype(np.float32)))
    run.s.enable_incremental(1 << 16)
    ctxs = [pb.BatchContext(1 << 15, 1 << 14, run.pf, [False, True]) for _ in range(J)]
    raw_ctxs = [pb.BatchContext(1 << 12, 1 << 12, [run.raw_pf]) for _ in range(J)]
    streams = [torch.cuda.Stream() for _ in range(J)]
    _pipeline(run, ctxs, streams, batches, raws=raws, raw_ctxs=raw_ctxs, updates=updates, upd_stream=torch.cuda.Stream())
    _drain(torch, streams)
    stepped = set()
    for b, r, (u, _) in zip(batches, raws, updates):
        stepped.update(int(x) for x in np.concatenate(run.signs(b) + [run.raw_signs(r), u]))
    st = run.s.incremental_stats()
    assert run.s.incremental_held() == st["held"] == len(stepped), (run.s.incremental_held(), st, len(stepped))
    assert st["dropped"] == 0
    signs, _, skipped = run.s.take_incremental(1 << 16)
    assert skipped == 0
    assert set(int(x) for x in signs.view(np.uint64)) == stepped
    run.check(np.concatenate([universe, raw_universe]), what=f"incremental J={J}")
    one = universe[:5]
    run.s.update(to_dev_ids(one, DEV), torch.zeros((one.size, dim), dtype=torch.float32, device=DEV))
    _drain(torch, [])
    assert run.s.incremental_held() == run.s.incremental_stats()["held"] == one.size


def _evict_table(pb, oracle, dim, cap):
    s = pb.EmbeddingShard(dim, cap, 0)
    s.set_optimizer(SGD, lr=LR, wd=0.0)
    s.configure(**HYPER)
    s.set_eviction(check_every=1, low_water=cap // 3, target_free=cap // 2, keep_batches=1)
    return s


@pytest.mark.parametrize("J", [2, 3, 4])
def test_eviction_in_flight_matches_one_stream(torch_cuda, pb, oracle, J):
    """A capacity-bounded table (an eviction check before every training request, keep 1) trained by J streams ends
    exactly where the same calls issued on one stream end: the same export list in the same order, the same index
    statistics and counters, bit-identical entries, and no sign in two cells."""
    torch = torch_cuda
    dim, cap, B = 32, 8192, 512
    rng = np.random.default_rng(500 + J)
    pf = [oracle.index_prefix(0), oracle.index_prefix(1)]
    batches = []
    for _ in range(6 * J):
        b = _batch(rng, B, False, dim)
        for i in range(2):  # a wider pool than the capacity holds
            b["slots"][i] = b["slots"][i] + np.uint64(POOL) * rng.integers(0, 32, size=b["slots"][i].size).astype(np.uint64)
        b["ids"] = np.concatenate(b["slots"])
        batches.append(b)
    keep = []
    dev = []
    for b in batches:
        dev.append(dict(ids=to_dev_ids(b["ids"], DEV), row_off=to_dev_i32(b["row_off"], DEV),
                        g=[torch.from_numpy(np.ascontiguousarray(b["g"][i])).to(DEV) for i in range(2)]))
    _drain(torch, [])
    tables = []
    for streams in ([torch.cuda.Stream() for _ in range(J)], [torch.cuda.Stream()] * J):
        s = _evict_table(pb, oracle, dim, cap)
        ctxs = [pb.BatchContext(1 << 14, 1 << 12, pf, [False, True]) for _ in range(J)]
        _gate(torch, set(streams))

        def fwd(k):
            with torch.cuda.stream(streams[k % J]):
                keep.append(ctxs[k % J].forward(s, dev[k]["ids"], batches[k]["slot_off"], B, row_off=dev[k]["row_off"]))

        def bwd(k):
            with torch.cuda.stream(streams[k % J]):
                ctxs[k % J].backward(s, dev[k]["g"], scales=SCALES)

        fwd(0)
        for k in range(len(batches)):
            if k + 1 < len(batches):
                fwd(k + 1)
            bwd(k)
        _drain(torch, streams)
        tables.append((s, ctxs))
    (a, _), (b, _) = tables
    sa, ra = a.export_signs()
    sb, rb = b.export_signs()
    sa, ra, sb, rb = sa.cpu().numpy(), ra.cpu().numpy(), sb.cpu().numpy(), rb.cpu().numpy()
    ca, cb = a.counters(), b.counters()
    assert cb["capacity_refused"] == 0 and cb["wait_errors"] == 0
    assert np.array_equal(sa, sb) and np.array_equal(ra, rb)
    assert ca == cb
    # (whether an admission takes a tombstone or an EMPTY cell can depend on the order of the admissions racing in one
    # probe, on one stream too: only the live count is fixed)
    ia, ib = a.index_stats(), b.index_stats()
    assert ia["live"] == ib["live"] == np.unique(sa).size == sa.size, (ia, ib, sa.size)
    seen = np.unique(np.concatenate([oracle.add_prefix(b["slots"][i], 8, pf[i]) for b in batches for i in range(2)]))
    assert ca["admitted"] == sa.size <= cap < seen.size  # rows were evicted along the way
    ea, fa = a.get_entries(torch.from_numpy(sa).to(DEV))
    eb, fb = b.get_entries(torch.from_numpy(sb).to(DEV))
    assert fa.all() and fb.all()
    assert torch.equal(ea.view(torch.int32), eb.view(torch.int32))


@pytest.mark.parametrize("J", [2, 3, 4])
def test_one_capture_side_streams(torch_cuda, pb, oracle, J):
    """J contexts forked onto side streams of one CUDA graph capture: the table's ordering becomes edges of that graph,
    so one replay gives the serial result."""
    torch = torch_cuda
    dim = 64
    rng, run, batches, universe, ctxs, streams = _setup(torch, pb, oracle, J, dim, n_mult=2, seed=1)
    dev = [run.dev_batch(b) for b in batches]
    outs = [torch.empty((2, b["B"], dim), dtype=torch.float16, device=DEV) for b in batches]
    _drain(torch, [])
    main = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    N = len(batches)
    with torch.cuda.graph(graph, stream=main):
        for st in streams:
            st.wait_stream(main)

        def fwd(k):
            with torch.cuda.stream(streams[k % J]):
                ctxs[k % J].forward(run.s, dev[k]["ids"], batches[k]["slot_off"], batches[k]["B"],
                                    row_off=dev[k]["row_off"], out=outs[k])

        fwd(0)
        for k in range(N):
            if k + 1 < N:
                fwd(k + 1)
            with torch.cuda.stream(streams[k % J]):
                run.backward(ctxs[k % J], dev[k])
        for st in streams:
            main.wait_stream(st)
    _drain(torch, streams + [main])
    # the capture ran nothing: the rows are still the seeds
    run.check(universe[:64], what="after the capture")
    with torch.cuda.stream(main):
        graph.replay()
    _drain(torch, [main])
    octx = {0: run.model_forward(batches[0])}
    for k in range(N):
        if k + 1 < N:
            octx[k + 1] = run.model_forward(batches[k + 1])
        run.model_backward(octx.pop(k), batches[k])
    run.check(universe, what=f"one capture J={J}")
