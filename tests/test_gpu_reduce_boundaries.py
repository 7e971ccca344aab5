"""GPU: the backward reduce (csrc/pb_reduce.cu) at the thresholds where its code path changes, against the CPU oracle
bit for bit (Adagrad against the oracle's exact-rsqrt mode) and, for SGD, against a float64 computation of the
reference operation that does not go through the oracle.

  multiplicity classes   1 cold / 2..32 warm / 33.. hot (257.. huge, 1025.. giant, started first); chunk tails
  hot geometries         lean 16-byte producer loop (dim 16..256 f16), vector loads with a vector count per row that
                         is not a power of two (dim 24, 264 f16; dim 20 f32), element-wise loads (dim 130 f16)
  bitmap windows         an item's occurrences are ordered HOT_WIN at a time: B around and past 8192, items that
                         straddle a window boundary or sit in a later window only, ragged slots (occurrence windows)
  column passes          dim > HOT_COLS: several passes per item, a short last column block (520, 1027)
  occurrence-list mode   hot items that found no room in the bitmap pool (context sized to the batch)
  bitmap reuse           an abandoned forward, a NaN slot and a skipped slot leave no stale bits behind
"""
import numpy as np
import pytest

from util import (DEV, batch_with_multiplicities, entries_equal, fwd_both, pair, ragged_with_multiplicities, to_dev_i32,
                  to_dev_ids)

pytestmark = pytest.mark.gpu

HOT_WIN = 8192  # occurrences of a slot per bitmap window of k_reduce_hot
HOT_COLS = 512  # columns of a row per pass
WARM_MAX = 32   # items of more occurrences are hot
SGD, ADAGRAD, ADAGRAD_VW, ADAM = 0, 1, 2, 3
OPT = {SGD: dict(lr=0.01, wd=0.0), ADAGRAD: dict(lr=0.01, init_acc=0.01, eps=1e-10),
       ADAGRAD_VW: dict(lr=0.02, mom=0.9, init_acc=0.1, eps=1e-8), ADAM: dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8)}
HYPER = dict(wb=1e30)  # the weight bound stays out of reach: the float64 check computes w - lr * sum
U = 2.0 ** -24


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


def _layout(slots, B):
    """slots: per slot (ids, row_off or None) -> flat ids, CSR row offsets (None when every slot has one id per sample)
    and the slot boundaries in the flat ids."""
    slot_off = [0]
    for ids, _ in slots:
        slot_off.append(slot_off[-1] + ids.size)
    ids = np.concatenate([x[0] for x in slots])
    if all(x[1] is None for x in slots):
        return ids, None, slot_off
    parts = [x[1] if x[1] is not None else np.arange(B + 1, dtype=np.uint32) for x in slots]
    row_off = np.concatenate([[0]] + [p[1:].astype(np.int64) + slot_off[i] for i, p in enumerate(parts)]).astype(np.uint32)
    return ids, row_off, slot_off


def _rows(s, signs, dim):
    return s.get_entries(to_dev_ids(signs, DEV))[0].cpu().numpy()[:, :dim]


def _check_f64(torch, s, oracle, pf, slots, g, before, B, dim, lr, scale, sqrt):
    """SGD (wd 0, weight bound out of reach) against the reference operation in float64: per occurrence the f16
    gradient with +-inf clamped to +-65504, times 1/scale and the sample's 1/sqrt(ids), summed per sign; w - lr * sum.
    The GPU sums n terms in f32 in a fixed order (at most gamma_{n-1} * sum|g| off, Higham) after up to four roundings
    per term (1/scale, the sqrt factor, two products) and rounds lr * sum and the difference once each: gamma_{n+6}
    covers all but the last rounding, 2^-24 |w| that one."""
    for i, (ids, ro) in enumerate(slots):
        signs = oracle.add_prefix(ids, 8, pf[i])
        sample = np.arange(B) if ro is None else np.repeat(np.arange(B), np.diff(ro))
        v = g[i][sample].astype(np.float64)
        if g.dtype == np.float16:
            v = np.clip(v, -65504.0, 65504.0)
        if scale is not None:
            v /= scale[i]
        if sqrt is not None and sqrt[i] and ro is not None:
            v /= np.sqrt(np.diff(ro)[sample].astype(np.float64))[:, None]
        u, inv, n = np.unique(signs, return_inverse=True, return_counts=True)
        order = np.argsort(inv, kind="stable")
        starts = np.concatenate([[0], np.cumsum(n)[:-1]])
        total = np.add.reduceat(v[order], starts, axis=0)
        mag = np.add.reduceat(np.abs(v[order]), starts, axis=0)
        w0 = before[i].astype(np.float64)
        want = w0 - lr * total
        m = (n + 6) * U
        tol = lr * (m / (1 - m))[:, None] * mag + U * np.abs(w0)
        got = _rows(s, u, dim).astype(np.float64)
        bad = np.abs(got - want) > tol
        assert not bad.any(), (i, u[np.argmax(bad.any(axis=1))], np.abs(got - want)[bad][:4], tol[bad][:4])


def _train(torch, s, ctx, w, oracle, pf, slots, B, dim, rng, kind, f32=False, scale=None, sqrt=None, nan=None, skip=None,
           stats=None):
    """One training step of the GPU path and the oracle on the same batch; SGD steps are also checked in float64.
    slots: per slot (ids, row_off or None); nan: slot whose gradient gets a NaN at an occurrence of its id 0; skip:
    slot passed as skipped; stats: expected cold/warm/hot counts of BatchContext.batch_stats().  Returns the signs
    touched, per slot."""
    ids, row_off, slot_off = _layout(slots, B)
    S = len(slots)
    _, _, octx = fwd_both(torch, s, ctx, w, ids, row_off, slot_off, B, training=True)
    if stats is not None:
        st = ctx.batch_stats()
        assert {k: st[k] for k in stats} == stats
    touched = [np.sort(w.ctx_signs(octx, i)) for i in range(S)]
    g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float32 if f32 else np.float16)
    if not f32:
        g[0, 0, 0] = np.inf  # clamps to 65504 (persia-common lib.rs:163-180)
        g[0, 1, min(1, dim - 1)] = -np.inf
    if nan is not None:  # at a sample holding the slot's id 0, its most frequent one
        first = int(np.flatnonzero(slots[nan][0] == 0)[0])
        sample = first if slots[nan][1] is None else int(np.searchsorted(slots[nan][1], first, side="right") - 1)
        g[nan, sample, dim - 1] = np.nan
    f64 = kind == SGD and nan is None and skip is None
    before = [_rows(s, t, dim) for t in touched] if f64 else None
    grads = [torch.from_numpy(g[i]).to(DEV) for i in range(S)]
    oskip = None
    if skip is not None:
        grads[skip] = None
        oskip = [int(i == skip) for i in range(S)]
    st = ctx.backward(s, grads, scales=scale, want_status=True).cpu().numpy().tolist()
    assert st == w.backward(octx, [g[i] for i in range(S)], scale=scale, skip=oskip)
    if f64:
        _check_f64(torch, s, oracle, pf, slots, g, before, B, dim, OPT[SGD]["lr"], scale, sqrt)
    return touched


def _abandon(torch, s, ctx, w, slots, B):
    """A training forward whose backward never comes (on both sides)."""
    ids, row_off, slot_off = _layout(slots, B)
    ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=to_dev_i32(row_off, DEV) if row_off is not None else None,
                training=True)
    w.forward(ids, row_off if row_off is not None else np.arange(len(slots) * B + 1, dtype=np.uint32), B, training=True,
              keep_ctx=False)


def _check(torch, s, w, touched):
    for t in touched:
        entries_equal(torch, s, w, np.unique(np.concatenate(t)) if isinstance(t, list) else t)
    assert s.counters()["wait_errors"] == 0


def _run(torch, pb, oracle, make_slots, S, B, dim, kind, steps=2, f32=False, scale=None, sqrt=None, cap=1 << 16,
         max_occ=1 << 18, stats=None):
    rng = np.random.default_rng(1000 * dim + B + kind)
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, cap=cap, sqrt=sqrt, optim_kw=OPT[kind], hyper_kw=HYPER, max_occ=max_occ)
    touched = [[] for _ in range(S)]
    for _ in range(steps):
        t = _train(torch, s, ctx, w, oracle, pf, make_slots(rng), B, dim, rng, kind, f32=f32, scale=scale, sqrt=sqrt,
                   stats=stats)
        for i in range(S):
            touched[i].append(t[i])
    _check(torch, s, w, touched)
    return s, ctx, w


# ---------------------------------------------------------------------------------------------- classes, geometries
CLASS_COUNTS = [1, 2, 31, 32, 33, 34, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025, 2049]


@pytest.mark.parametrize("dim,f32,kind", [(16, False, SGD), (64, False, ADAGRAD), (128, False, SGD), (24, False, SGD),
                                          (130, False, ADAGRAD), (256, False, SGD), (264, False, ADAGRAD),
                                          (20, True, SGD)])
def test_multiplicity_classes_and_chunk_tails(torch_cuda, pb, oracle, dim, f32, kind):
    """Every multiplicity class boundary and chunk tails (a hot item's count not a multiple of the chunk's rows or of
    four) in two slots, at dims that select each hot-path geometry; the work lists hold what numpy counts."""
    S, B = 2, 8000
    counts = np.array(CLASS_COUNTS)
    fresh = B - int(counts.sum())
    stats = {"cold": S * (int((counts == 1).sum()) + fresh), "warm": S * int(((counts >= 2) & (counts <= WARM_MAX)).sum()),
             "hot": S * int((counts > WARM_MAX).sum())}
    _run(torch_cuda, pb, oracle, lambda rng: [(batch_with_multiplicities(rng, B, CLASS_COUNTS), None) for _ in range(S)],
         S, B, dim, kind, f32=f32, stats=stats)


# ---------------------------------------------------------------------------------------------- bitmap windows
def _window_items(n):
    """(counts, spans) of items placed against the HOT_WIN boundaries of a slot of n positions."""
    counts, spans = [], {}
    lo, hi = HOT_WIN - 48, min(n, HOT_WIN + 48)
    spans[0] = (lo, hi)
    counts.append(min(64, hi - lo))  # straddles the first boundary (n = 8193: holds position 8192, window 2's only one)
    if n >= HOT_WIN + 400:
        spans[len(counts)] = (HOT_WIN, min(n, 2 * HOT_WIN))
        counts.append(300)  # every occurrence in the second window
    if n > 2 * HOT_WIN:
        spans[len(counts)] = (n - 200, n)
        counts.append(100)  # the last window (and the one before when n % HOT_WIN < 200)
    return counts + [4100, 1025, 33, 32, 2], spans


@pytest.mark.parametrize("kind", [SGD, ADAGRAD])
@pytest.mark.parametrize("B", [8191, 8192, 8193, 16389, 65535])
def test_windows_one_id_per_sample(torch_cuda, pb, oracle, B, kind):
    counts, spans = _window_items(B)
    _run(torch_cuda, pb, oracle, lambda rng: [(batch_with_multiplicities(rng, B, counts, spans), None)], 1, B, 64, kind,
         cap=1 << 18)


@pytest.mark.parametrize("kind", [SGD, ADAGRAD])
def test_windows_ragged_sqrt_and_scale(torch_cuda, pb, oracle, kind):
    """A ragged slot of > 8192 occurrences with sqrt scaling and a loss scale (the producers' general loop, windows over
    occurrences, occ_outrow set) beside a one-id slot that the ragged layout also takes off the lean loop."""
    B = 3000
    counts, spans = _window_items(HOT_WIN + 2000)  # the spans fit any slot of >= 10192 occurrences
    counts[counts.index(4100)] = 3000

    def make(rng):
        ids, ro = ragged_with_multiplicities(rng, B, counts, max_ids=6, spans=spans)
        assert ro[-1] > HOT_WIN + 2000
        return [(ids, ro), (batch_with_multiplicities(rng, B, [700, 40, 3]), None)]

    _run(torch_cuda, pb, oracle, make, 2, B, 64, kind, scale=[3.0, 128.0], sqrt=[True, False])


# ---------------------------------------------------------------------------------------------- column passes
@pytest.mark.parametrize("kind", [SGD, ADAGRAD, ADAGRAD_VW, ADAM])
@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("dim", [520, 640, 1027, 2048])
def test_column_passes(torch_cuda, pb, oracle, dim, f32, kind):
    B = 1200
    counts = [300, 100, 40, 33, 20, 2]
    _run(torch_cuda, pb, oracle, lambda rng: [(batch_with_multiplicities(rng, B, counts), None)], 1, B, dim, kind, f32=f32,
         cap=1 << 13)


@pytest.mark.parametrize("kind", [SGD, ADAGRAD])
def test_column_passes_across_windows(torch_cuda, pb, oracle, kind):
    B = 9000
    counts, spans = _window_items(B)
    _run(torch_cuda, pb, oracle, lambda rng: [(batch_with_multiplicities(rng, B, counts, spans), None)], 1, B, 640, kind,
         cap=1 << 15)


# ---------------------------------------------------------------------------------------------- bitmap pool
@pytest.mark.parametrize("kind", [SGD, ADAGRAD])
def test_bitmap_pool_exhaustion_list_mode(torch_cuda, pb, oracle, kind):
    """A context sized to the batch (as bench.py and worker.py size theirs) has a bitmap pool of max(4096, S * B) words;
    a hot item takes ceil(B / 32) of them.  With hundreds of hot items most find no room and come with occurrence lists
    (the reduce sets their bits itself), beside the ones in bitmap mode, across two windows."""
    S, B, dim = 1, 16384, 64
    counts = [40] * 300 + [1500, 2]
    hot = sum(c > WARM_MAX for c in counts)
    assert hot * ((B + 31) // 32) > max(4096, S * B)
    _run(torch_cuda, pb, oracle, lambda rng: [(batch_with_multiplicities(rng, B, counts), None)], S, B, dim, kind,
         max_occ=S * B)


# ---------------------------------------------------------------------------------------------- bitmap reuse
def test_bitmap_reuse_after_abandoned_forward_nan_and_skip(torch_cuda, pb, oracle):
    """The forward sets the bits of its hot items; the backward (or the next forward, for a batch whose backward never
    came) zeroes them, a dead slot's items included.  A stale bit would add a foreign row into the next batch's sum."""
    torch = torch_cuda
    S, B, dim = 2, 12000, 64
    counts = [2000, 700, 300, 40, 33]
    rng = np.random.default_rng(5)
    s, ctx, w, pf = pair(pb, oracle, S, dim, SGD, cap=1 << 18, optim_kw=OPT[SGD], hyper_kw=HYPER, max_occ=S * B)

    def slots():
        return [(batch_with_multiplicities(rng, B, counts), None) for _ in range(S)]

    touched = []
    _abandon(torch, s, ctx, w, slots(), B)
    touched += _train(torch, s, ctx, w, oracle, pf, slots(), B, dim, rng, SGD)
    touched += _train(torch, s, ctx, w, oracle, pf, slots(), B, dim, rng, SGD, nan=0)
    touched += _train(torch, s, ctx, w, oracle, pf, slots(), B, dim, rng, SGD)
    touched += _train(torch, s, ctx, w, oracle, pf, slots(), B, dim, rng, SGD, skip=0)
    _abandon(torch, s, ctx, w, slots(), B)
    touched += _train(torch, s, ctx, w, oracle, pf, slots(), B, dim, rng, SGD)
    _check(torch, s, w, [np.unique(np.concatenate(touched))])
