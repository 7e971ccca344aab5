"""GPU: every path at the batch context's occurrence limit (pb_ctx_create: 2^24), against the oracle bit for bit.

The batches come from tests/scale_cases.py (tests/test_scale_cases.py checks their shape on the CPU):
  1. one summation slot of 2^24 - 3 occurrences: items of 1 to ~4 M occurrences, 2048 bitmap windows of k_reduce_hot,
     spans across window boundaries and inside the last window, the hot staging and the giant/huge lists filled;
  2. the bitmap pool both ways: 48 hot items in a slot of 4 M occurrences, 32 bitmaps fit, 16 items get occurrence lists;
     36000 hot items that together ask for more than 2^32 bitmap words; the warm list, the hot list and the giants'
     region filled to their sizes at 2^24 occurrences;
  3. 128 slots x 65535 samples of one id (8,388,480 occurrences and output rows), Adam over shared feature groups;
  4. U = N: 16 M distinct ids in 65535 samples admitted in one forward;
  5. raw slots past one spine trip of the numbering scan (k_scan_spine carries), up to 2^24 - 5 ids;
  6. raw gradient staging at the sizes persia_core makes a raw context (twice the batch's ids), at dims 128 and 1024.
Outputs are compared with the sample-order model of the pooled forward (util.pool_model) or the oracle, raw tables,
indices and counts with oracle.Worker.forward_raw, statuses with the oracle, entries after the steps with the oracle (in
exact-rsqrt mode).  Every case frees its context and shard.  Each prints its wall time and peak device memory (torch's
allocations and the library's own cudaMallocs, from the device's free memory) when run with -s."""
import time

import numpy as np
import pytest

import scale_cases as SC
from util import (DEV, full_row_off, pair, pool_model, same_bits, slot_signs, to_dev_i32, to_dev_ids)

pytestmark = pytest.mark.gpu
SGD, ADAGRAD, ADAGRAD_VW, ADAM = 0, 1, 2, 3
OPT = {SGD: dict(lr=0.05, wd=0.0), ADAGRAD: dict(lr=0.02, init_acc=0.01, eps=1e-10),
       ADAM: dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8)}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    if torch.cuda.get_device_properties(0).total_memory < 70e9:
        pytest.skip("batches at the context's limit need an 80 GB-class GPU")
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


class Meter:
    """Wall time and peak device memory of one case: torch's peak allocation, and the growth of the device's used
    memory (torch's and the library's cudaMallocs) over the case's start, sampled after the forwards and backwards only.
    The second figure also counts whatever else allocates on the device meanwhile, and misses what is freed between
    samples: an estimate, not a bound."""

    def __init__(self, torch, name):
        self.torch, self.name = torch, name
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        free, total = torch.cuda.mem_get_info()
        self.base, self.peak, self.t0 = total - free, 0, time.perf_counter()

    def sample(self):
        self.torch.cuda.synchronize()
        free, total = self.torch.cuda.mem_get_info()
        self.peak = max(self.peak, total - free - self.base)

    def report(self):
        t = time.perf_counter() - self.t0
        print(f"\nSCALE {self.name}: wall {t:.1f} s, peak torch {self.torch.cuda.max_memory_allocated() / 1e9:.2f} GB, "
              f"peak device {self.peak / 1e9:.2f} GB")


def _free(torch, *objs):
    for o in objs:
        o.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _held(torch, s, signs, dim):
    """(distinct signs ascending, f32 [n, dim]) of the signs the table holds: pool_model's array form of held_rows."""
    keys = np.unique(np.asarray(signs, np.uint64))
    ent, found = s.get_entries(to_dev_ids(keys, DEV))
    found = found.cpu().numpy().astype(bool)
    return keys[found], ent[:, :dim].cpu().numpy()[found]


def _entries_equal(torch, s, w, signs):
    """Every entry of `signs` on the GPU equals the oracle's bit for bit (one bulk read, then the oracle's)."""
    signs = np.asarray(signs, np.uint64)
    ent, found = s.get_entries(to_dev_ids(signs, DEV))
    assert bool(found.all())
    ent = ent.cpu().numpy()
    want = np.stack([w.get_entry(int(x)) for x in signs])
    bad = np.flatnonzero((ent.view(np.uint32) != want.view(np.uint32)).any(axis=1))
    assert bad.size == 0, (bad.size, int(signs[bad[0]]), ent[bad[0]], want[bad[0]])


def _class_counts(signs, slot_off):
    want = dict(items=0, cold=0, warm=0, hot=0)
    warm_occ = 0
    for i in range(len(slot_off) - 1):
        c = np.unique(signs[slot_off[i]:slot_off[i + 1]], return_counts=True)[1]
        want["items"] += c.size
        want["cold"] += int((c == 1).sum())
        want["warm"] += int(((c >= 2) & (c <= SC.WARM_MAX)).sum())
        want["hot"] += int((c > SC.WARM_MAX).sum())
        warm_occ += int(c[(c >= 2) & (c <= SC.WARM_MAX)].sum())
    return want, warm_occ


def _summation_step(torch, oracle, s, ctx, w, pf, ids, row_off, B, dim, rng, f32=False, sqrt=None, scale=None):
    """One training step of one summation slot: outputs against the sample-order model, batch statistics against the
    batch, status against the oracle.  Returns (batch statistics, occurrences of warm items, gradient, signs, rows the
    table held at forward time)."""
    n = ids.size
    slot_off = [0, n]
    got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=to_dev_i32(row_off, DEV), training=True)
    got = got.cpu().numpy()
    signs = slot_signs(oracle, ids, slot_off, pf)
    st = ctx.batch_stats()
    want, warm_occ = _class_counts(signs, slot_off)
    assert {k: st[k] for k in want} == want and st["occurrences"] == n, (st, want)
    held = _held(torch, s, signs, dim)
    model = pool_model(held, signs, row_off, B, sqrt, dim=dim)
    assert same_bits(got[0], model[0])
    _, octx = w.forward(ids, row_off, B, training=True)
    g = (rng.standard_normal((1, B, dim)) * 1e-2).astype(np.float32 if f32 else np.float16)
    scales = [scale] if scale else None
    status = ctx.backward(s, [torch.from_numpy(g[0]).to(DEV)], scales=scales, want_status=True).cpu().numpy().tolist()
    assert status == w.backward(octx, [g[0]], scale=scales) == [0]
    return st, warm_occ, g[0], signs, held


def _sequential_sum(rows):
    """Sum of f32 rows in order, one addition at a time (np.cumsum over float32 adds in sequence), in chunks."""
    acc = np.zeros(rows.shape[1], np.float32)
    for lo in range(0, rows.shape[0], 1 << 20):
        c = rows[lo:lo + (1 << 20)].astype(np.float32)
        c[0] = acc + c[0]
        acc = np.cumsum(c, axis=0, dtype=np.float32)[-1]
    return acc


# ---------------------------------------------------------------------------------------------- 1. the context limit
@pytest.mark.parametrize("kind,dim,f32,steps", [(SGD, 64, False, 2), (ADAGRAD, 64, False, 2), (ADAGRAD, 128, True, 1)])
def test_summation_slot_at_the_context_limit(torch_cuda, pb, oracle, kind, dim, f32, steps):
    """One ragged slot of 65535 samples, 2^24 - 3 occurrences in a context of exactly 2^24 (SUM_ITEMS: multiplicities
    1 .. ~4 M, spans across window boundaries and inside the last window, ~2 M warm and cold fill ids).  The f32 case
    adds sqrt scaling and a loss scale.  Every hot item gets a bitmap (9 x 2^19 words of a 2^24-word pool): the
    occurrence lists hold the warm items' occurrences only.  The SGD case restates the ~4 M item's step in numpy: its
    f16 gradient rows summed in f32 in ascending occurrence order, then w - lr * (sum + w * 0) as one fused
    multiply-add, within the weight bound."""
    torch = torch_cuda
    m = Meter(torch, f"summation kind={kind} dim={dim} f32={f32}")
    rng = np.random.default_rng(100 + kind + dim)
    sqrt = [True] if f32 else None
    s, ctx, w, pf = pair(pb, oracle, 1, dim, kind, cap=1 << 22, sqrt=sqrt, optim_kw=OPT[kind], max_occ=SC.CTX_LIMIT)
    seen = set()
    try:
        for step in range(steps):
            ids, row_off = SC.summation_case(step)
            st, warm_occ, g, signs, held = _summation_step(torch, oracle, s, ctx, w, pf, ids, row_off, SC.SUM_B, dim,
                                                           rng, f32=f32, sqrt=sqrt, scale=4.0 if f32 else None)
            m.sample()
            assert st["hot"] == 9 and st["repeated_occurrences"] == warm_occ  # no hot item in list mode
            seen.update(np.unique(signs).tolist())
            if kind == SGD and step == 0:  # the oracle's sum of the ~4 M item against a plain sequential one
                big = signs[ids == np.uint64(7)][0]
                occ = np.flatnonzero(ids == np.uint64(7))
                sample = np.searchsorted(row_off, occ, side="right") - 1
                total = _sequential_sum(g[sample].astype(np.float32))
                w0 = held[1][np.searchsorted(held[0], big)]
                # decayed_sgd's 8-wide form: fma(-lr, fma(wd, w, g), w), one rounding (the f32 product is exact in
                # f64; dim 64 has no scalar tail); then the weight bound (10, on by default)
                dg = total + w0 * np.float32(0)
                want = (w0.astype(np.float64) - np.float64(np.float32(OPT[SGD]["lr"])) * dg).astype(np.float32)
                want = np.clip(want, np.float32(-10), np.float32(10))
                assert w.get_entry(int(big)).tobytes() == want.astype(np.float32).tobytes()
        _entries_equal(torch, s, w, np.array(sorted(seen), np.uint64))
        assert s.counters()["wait_errors"] == 0
    finally:
        m.report()
        _free(torch, ctx, s)


# ---------------------------------------------------------------------------------------------- 2. the bitmap pool
def test_bitmap_pool_both_ways(torch_cuda, pb, oracle):
    """48 hot items in one slot of 4 M occurrences (POOL_ITEMS): each wants ceil(4e6 / 32) bitmap words of a pool of
    max(4096, max_occurrences) words, so 32 get bitmaps and 16 get occurrence lists.  The lists show in the batch
    statistics: the occurrence-list entries exceed the warm items' occurrences by the list-mode items' occurrences.  A
    second batch on the same context matches too: no bitmap bit or cursor is left behind."""
    torch = torch_cuda
    m = Meter(torch, "bitmap pool")
    rng = np.random.default_rng(2)
    dim = 32
    words = (SC.POOL_N + 31) // 32
    assert 32 * words <= max(4096, SC.POOL_N) < 33 * words  # pb_ctx_create's pool: 32 bitmaps of this slot
    s, ctx, w, pf = pair(pb, oracle, 1, dim, ADAGRAD, cap=1 << 21, optim_kw=OPT[ADAGRAD], max_occ=SC.POOL_N)
    seen = set()
    try:
        for step in range(2):
            ids, row_off = SC.pool_case(10 + step)
            st, warm_occ, _, signs, _ = _summation_step(torch, oracle, s, ctx, w, pf, ids, row_off, SC.POOL_B, dim, rng)
            m.sample()
            assert st["hot"] == 48
            listed = st["repeated_occurrences"] - warm_occ  # occurrences of the hot items that got lists
            smallest16 = sum(sorted(SC.POOL_ITEMS)[:16])
            assert listed >= smallest16, (listed, smallest16)
            seen.update(np.unique(signs).tolist())
        _entries_equal(torch, s, w, np.array(sorted(seen), np.uint64))
        assert s.counters()["wait_errors"] == 0
    finally:
        m.report()
        _free(torch, ctx, s)


def test_bitmap_pool_counter_past_2_pow_32(torch_cuda, pb, oracle):
    """36000 hot items of 40 occurrences in one slot of 4 M (WRAP_CASE): together they ask for 4.5e9 bitmap words.  A
    32-bit count of the words asked for wraps past 2^32, and the items that ask after the wrap would get bitmaps again:
    offsets already handed out (two items summing each other's occurrences) or, with the pool's bit 31 flag, far past
    the pool.  Exactly 32 items get bitmaps, so the occurrence lists hold the other 35968 items' 40 occurrences each on
    top of the warm items'.  Outputs, status and every entry equal the oracle's, and so does a second batch on the same
    context (no bitmap bit left behind)."""
    torch = torch_cuda
    m = Meter(torch, "bitmap pool counter past 2^32")
    rng = np.random.default_rng(36)
    dim = 16
    words = (SC.POOL_N + 31) // 32
    assert SC.WRAP_HOT * words > 2 ** 32
    s, ctx, w, pf = pair(pb, oracle, 1, dim, SGD, cap=1 << 21, optim_kw=OPT[SGD], max_occ=SC.POOL_N)
    seen = set()
    try:
        for step in range(2):
            ids, row_off = SC.wrap_case(20 + step)
            st, warm_occ, _, signs, _ = _summation_step(torch, oracle, s, ctx, w, pf, ids, row_off, SC.POOL_B, dim, rng)
            m.sample()
            assert st["hot"] == SC.WRAP_HOT
            assert st["repeated_occurrences"] - warm_occ == (SC.WRAP_HOT - SC.POOL_BITMAPS) * SC.WRAP_MULT
            seen.update(np.unique(signs).tolist())
        _entries_equal(torch, s, w, np.array(sorted(seen), np.uint64))
        assert s.counters()["wait_errors"] == 0
    finally:
        m.report()
        _free(torch, ctx, s)


@pytest.mark.parametrize("kind,opt", [("pairs", ADAGRAD), ("hot33", SGD), ("giant", ADAM)])
def test_lists_filled_to_their_sizes(torch_cuda, pb, oracle, kind, opt):
    """128 ragged slots of 65535 samples, 2^24 occurrences, every item of one multiplicity (capacity_case): the warm
    list holds 2^23 pairs (n / 2 + 1 entries), the hot list 508,400 items of 33 (n / 33 entries below the giants'), the
    giants' region 16,368 items of 1025 (n / 1024 + 1 entries), each with its occurrence lists, hot_stage rows and
    bitmaps (4095 fit, the rest get lists).  Outputs against the sample-order model, statuses, and entries after one
    step against the oracle: every entry, but a sample of 2^18 of the pairs' 8.4 M."""
    torch = torch_cuda
    m = Meter(torch, f"lists filled: {kind}")
    rng = np.random.default_rng(len(kind))
    S, B, dim = SC.CAP_S, SC.CAP_B, 16
    mult = SC.CAP_KINDS[kind]
    s, ctx, w, pf = pair(pb, oracle, S, dim, opt, cap=1 << 24, optim_kw=OPT[opt], max_occ=SC.CTX_LIMIT)
    try:
        ids, row_off, slot_off = SC.capacity_case(kind, 9)
        got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=to_dev_i32(row_off, DEV), training=True)
        got = got.cpu().numpy()
        m.sample()
        signs = slot_signs(oracle, ids, slot_off, pf)
        st = ctx.batch_stats()
        items = SC.CTX_LIMIT // mult
        cls = "warm" if mult <= SC.WARM_MAX else "hot"
        assert st[cls] == items and st["items"] == items + SC.CTX_LIMIT - items * mult, st
        assert st["occurrences"] == SC.CTX_LIMIT
        if kind == "pairs":
            assert st["repeated_occurrences"] == SC.CTX_LIMIT  # seg_occ filled whole
        keys = np.unique(signs)
        ent = s.get_entries(to_dev_ids(keys, DEV))[0][:, :dim].cpu().numpy()
        assert same_bits(got, pool_model((keys, ent), signs, row_off, B, None, dim=dim))
        del ent
        _, octx = w.forward(ids, row_off, B, training=True)
        g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
        status = ctx.backward(s, [torch.from_numpy(g[i]).to(DEV) for i in range(S)], want_status=True)
        m.sample()
        assert status.cpu().numpy().tolist() == w.backward(octx, [g[i] for i in range(S)]) == [0] * S
        check = keys if keys.size <= 1 << 20 else np.unique(rng.choice(keys, size=1 << 18, replace=False))
        _entries_equal(torch, s, w, check)
        assert s.counters()["wait_errors"] == 0
    finally:
        m.report()
        _free(torch, ctx, s)


# ---------------------------------------------------------------------------------------------- 3. 128 x 65535
def test_128_slots_of_65535_samples(torch_cuda, pb, oracle):
    """128 slots x 65535 samples of one Zipf id each: 8,388,480 occurrences and output rows in one context.  Feature
    groups of 8 slots (0..7, 60..67 across a slot-mask word, 120..127), Adam: the beta powers advance per group.  A NaN
    in slot 64 (inside group 60..67) and slot 3 skipped (inside group 0..7): their groups still advance."""
    torch = torch_cuda
    m = Meter(torch, "128 slots x 65535")
    S, B, dim = SC.MANY_S, SC.MANY_B, 16
    rng = np.random.default_rng(3)
    groups = SC.many_slots_groups()
    s, ctx, w, pf = pair(pb, oracle, S, dim, ADAM, cap=1 << 22, groups=groups, optim_kw=OPT[ADAM], max_occ=S * B)
    try:
        ids = SC.many_slots_case(3)
        slot_off = [i * B for i in range(S + 1)]
        got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, training=True).cpu().numpy()
        m.sample()
        signs = slot_signs(oracle, ids, slot_off, pf)
        st = ctx.batch_stats()
        want_cls, _ = _class_counts(signs, slot_off)
        assert {k: st[k] for k in want_cls} == want_cls and st["occurrences"] == S * B, (st, want_cls)
        want, octx = w.forward(ids, full_row_off(S, B), B, training=True)
        for i in range(S):
            assert same_bits(got[i], want[i]), i  # one id per sample: f16(0 + row), the oracle's order is moot
        g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
        g[64, B // 2, 3] = np.nan
        grads = [None if i == 3 else torch.from_numpy(g[i]).to(DEV) for i in range(S)]
        status = ctx.backward(s, grads, want_status=True).cpu().numpy().tolist()
        m.sample()
        assert status == w.backward(octx, [g[i] for i in range(S)], skip=[int(i == 3) for i in range(S)])
        assert [i for i in range(S) if status[i]] == [3, 64]
        _entries_equal(torch, s, w, np.unique(signs))
        assert len(s) == w.ps_len(0) and s.counters()["wait_errors"] == 0
    finally:
        m.report()
        _free(torch, ctx, s)


# ---------------------------------------------------------------------------------------------- 4. U = N
def test_sixteen_million_distinct_ids(torch_cuda, pb, oracle):
    """One ragged slot of 16 M distinct ids in 65535 samples, in a table of 2^24 rows at dim 16 (Adagrad): the forward
    admits every one (k_dedup regions of 2 n + 1 cells, k_probe_items' grid over 16 M items, every item cold,
    k_gather_items over samples of ~244 ids).  Outputs equal the sample-order model over the rows the table holds; the
    admission count is exact; 4096 sampled entries equal the oracle's as admitted and after one step (each id occurs
    once, so a fresh oracle given a batch of the sampled ids alone, each with its sample's gradient row, admits and
    steps them the same way)."""
    torch = torch_cuda
    m = Meter(torch, "U = N")
    N, B, dim = SC.UNIQUE_N, SC.UNIQUE_B, 16
    rng = np.random.default_rng(4)
    s, ctx, _, pf = pair(pb, oracle, 1, dim, ADAGRAD, cap=1 << 24, optim_kw=OPT[ADAGRAD], max_occ=N)
    try:
        ids, row_off = SC.unique_case(4)
        got = ctx.forward(s, to_dev_ids(ids, DEV), [0, N], B, row_off=to_dev_i32(row_off, DEV), training=True)
        got = got.cpu().numpy()
        m.sample()
        st = ctx.batch_stats()
        assert (st["items"], st["cold"], st["warm"], st["hot"]) == (N, N, 0, 0)
        c = s.counters()
        assert c["admitted"] == N and c["capacity_refused"] == 0 and c["wait_errors"] == 0 and len(s) == N
        signs = slot_signs(oracle, ids, [0, N], pf)
        ent, found = s.get_entries(to_dev_ids(signs, DEV))
        assert bool(found.all())
        ent = ent.cpu().numpy()
        order = np.argsort(signs)
        assert same_bits(got[0], pool_model((signs[order], ent[order]), signs, row_off, B, None, dim=dim)[0])
        pick = np.sort(rng.choice(N, size=4096, replace=False))
        before = ent[pick]
        del ent
        g = (rng.standard_normal((B, dim)) * 1e-2).astype(np.float16)
        status = ctx.backward(s, [torch.from_numpy(g).to(DEV)], want_status=True).cpu().numpy().tolist()
        m.sample()
        assert status == [0]
        w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf[0])], n_ps=1)
        w.configure()
        w.set_optimizer(oracle.Optim(ADAGRAD, **OPT[ADAGRAD]))
        _, octx = w.forward(ids[pick], full_row_off(1, pick.size), pick.size, training=True)  # admits them afresh
        want = np.stack([w.get_entry(int(x)) for x in signs[pick]])
        assert before.tobytes() == want.tobytes()  # the admitted rows: the oracle's initial values and state
        sample = np.searchsorted(row_off, pick, side="right") - 1
        assert w.backward(octx, [g[sample]]) == [0]
        _entries_equal(torch, s, w, signs[pick])
        assert s.counters()["wait_errors"] == 0
    finally:
        m.report()
        _free(torch, ctx, s)


# ---------------------------------------------------------------------------------------------- 5. raw scan trips
def _first_order(ids):
    """The distinct ids in first-occurrence order (the raw numbering)."""
    return ids[np.sort(np.unique(ids, return_index=True)[1])]


@pytest.mark.parametrize("n", SC.RAW_SIZES)
def test_raw_slot_past_one_spine_trip(torch_cuda, pb, oracle, n):
    """A raw slot of n ids (RAW_SIZES: one spine trip of the numbering scan exactly, one id past it, a partial second
    trip, 16 trips) in 65535 samples, without an index prefix, holding the three marker-valued ids, samples far longer
    than sample_fixed_size and empty ones.  The table, index, non_empty_index, sample_id_num and both counts equal the
    oracle's; an f16 gradient with +inf and -inf steps the rows (SGD) as the oracle does."""
    torch = torch_cuda
    m = Meter(torch, f"raw n={n}")
    rng = np.random.default_rng(n)
    dim, fixed = 16, SC.RAW_FIXED
    ids, row_off = SC.raw_case(n, n)
    B = row_off.size - 1
    s = pb.EmbeddingShard(dim, 1 << 24, 0)
    s.set_optimizer(SGD, lr=OPT[SGD]["lr"])
    s.configure()
    ctx = pb.BatchContext(n, B, [0])
    w = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=0)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(SGD, **OPT[SGD]))
    try:
        table, index, non_empty, num, counts = ctx.forward_raw(s, to_dev_ids(ids, DEV), B, fixed,
                                                               row_off=to_dev_i32(row_off, DEV))
        m.sample()
        U, placed = (int(x) for x in counts.cpu().numpy())
        wt, wi, wn, wnum, octx = w.forward_raw(0, ids, row_off, B)
        assert U == wt.shape[0] - 1 and placed == wn.size
        assert same_bits(table[:U + 1].cpu().numpy(), wt)
        assert np.array_equal(index.cpu().numpy(), wi) and np.array_equal(non_empty[:placed].cpu().numpy(), wn)
        assert np.array_equal(num.cpu().numpy().view(np.uint32), wnum)
        uniq = _first_order(ids)
        assert uniq.size == U and set(SC.MARKERS.tolist()) <= set(uniq.tolist())
        g = (rng.standard_normal((U, dim)) * 1e-2).astype(np.float16)
        g[0, 0], g[U - 1, dim - 1] = np.inf, -np.inf
        status = ctx.backward_raw(s, torch.from_numpy(g).to(DEV), want_status=True).item()
        m.sample()
        assert status == w.backward_raw(0, octx, g) == 0
        check = uniq if U <= 1 << 20 else np.concatenate([uniq[:1 << 18], uniq[-(1 << 18):], SC.MARKERS])
        _entries_equal(torch, s, w, np.unique(check))
        assert s.counters()["wait_errors"] == 0
    finally:
        m.report()
        _free(torch, ctx, s)


# ---------------------------------------------------------------------------------------------- 6. raw staging
@pytest.mark.parametrize("dim", [128, 1024])
def test_raw_staging_at_persia_core_sizes(torch_cuda, pb, oracle, dim):
    """A raw batch of 2^23 - 7 ids in a context made as persia_core makes it (ctx_size: twice the ids, here
    2^24 - 14 occurrences).  The backward stages the [U, dim] gradient in f32.  Sized by the context that staging was
    2^24 x 1024 x 4 bytes = 64 GB at dim 1024, beside the 17 GB f16 table of the forward: more than the GPU holds.
    Sized by the batch it is half that.  Outputs against the oracle on the distinct ids in first-occurrence order (the
    same numbering, the same table rows) and the index against the numbering; entries after one f32 step with a loss
    scale against the oracle (a raw gradient row steps its own sign only)."""
    from persia_b200.persia_core import ctx_size

    torch = torch_cuda
    m = Meter(torch, f"raw staging dim={dim}")
    rng = np.random.default_rng(dim)
    fixed = 4
    ids, row_off = SC.stage_case(6)
    n, B = ids.size, row_off.size - 1
    cap, rows = ctx_size(n, B)
    pf = oracle.index_prefix(0)
    s = pb.EmbeddingShard(dim, 1 << 13, 0)
    s.set_optimizer(SGD, lr=OPT[SGD]["lr"])
    s.configure()
    ctx = pb.BatchContext(cap, rows, [pf])
    try:
        table, index, non_empty, num, counts = ctx.forward_raw(s, to_dev_ids(ids, DEV), B, fixed,
                                                               row_off=to_dev_i32(row_off, DEV))
        m.sample()
        U, placed = (int(x) for x in counts.cpu().numpy())
        uniq = _first_order(ids)
        lens = np.diff(row_off.astype(np.int64))
        assert U == uniq.size == SC.STAGE_POOL and placed == int(np.minimum(lens, fixed).sum())
        rank = np.empty(int(uniq.max()) + 1, np.int64)
        rank[uniq.astype(np.int64)] = np.arange(U)
        want_index = np.zeros(B * fixed, np.int64)
        sample = np.repeat(np.arange(B), lens)
        col = np.arange(n) - row_off[sample].astype(np.int64)
        keep = col < fixed
        want_index[sample[keep] * fixed + col[keep]] = rank[ids[keep].astype(np.int64)] + 1
        assert np.array_equal(index.cpu().numpy(), want_index)
        assert np.array_equal(non_empty[:placed].cpu().numpy(), np.flatnonzero(want_index))
        assert np.array_equal(num.cpu().numpy(), np.minimum(lens, fixed).astype(np.int32))
        w = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=1, prefix=pf)], n_ps=1)
        w.configure()
        w.set_optimizer(oracle.Optim(SGD, **OPT[SGD]))
        wt, _, _, _, octx = w.forward_raw(0, uniq, full_row_off(1, U), U)
        assert same_bits(table[:U + 1].cpu().numpy(), wt)
        del table
        g = (rng.standard_normal((U, dim)) * 1e-2).astype(np.float32)
        status = ctx.backward_raw(s, torch.from_numpy(g).to(DEV), scale=2.0, want_status=True).item()
        m.sample()
        assert status == w.backward_raw(0, octx, g, scale=2.0) == 0
        _entries_equal(torch, s, w, oracle.add_prefix(uniq, 8, pf))
        assert s.counters()["wait_errors"] == 0
    finally:
        m.report()
        _free(torch, ctx, s)
