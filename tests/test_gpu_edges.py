"""GPU: every path that steps a row, at the edges of its arithmetic, against the oracle and against closed forms.

The rest of the suite draws gradients from N(0, 1) * 1e-2 and rows from +-0.01, with the weight bound at 10.  Here the
rows are seeded (set_entries on the GPU, set_embedding in the oracle) at the bound, past it with the bound off, at
FLT_MIN, at -0 and at the f16 limits, and the gradients hold +-65504, +-inf in f16 and f32, subnormals, -0, sums that
overflow and degenerate optimizer settings.  Each case runs through every path (util.EDGE_PATHS): the batched step with
cold, warm and hot items, pb_update, the raw step, the sharded step at R = 2 and 3 (dims 64 and 128 step rows in
k_owner_update_all, 12, 130 and 256 in k_owner_update), a shared feature group and sharded raw.  Entries compare bit
for bit with the oracle in exact-rsqrt mode, NaN matching any NaN.  The special values also get closed forms written
from the reference's formulas (persia-simd lib.rs, optim.rs, the EW's gradient preparation in
embedding_worker_service/mod.rs), so that a mistake the oracle shares cannot pass."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from util import (DEV, EDGE_COUNTS, EDGE_PATHS, batch_with_multiplicities, full_row_off, pool_lists,  # noqa: E402
                  run_edge_path, same_bits, to_dev_i32, to_dev_ids)

pytestmark = pytest.mark.gpu
FLT_MIN = np.float32(np.finfo(np.float32).tiny)
ONE_STEP = ("batch", "direct", "raw")  # paths on which every seeded row takes exactly one optimizer step


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def _mask(ids, dim, mod, off=0):
    """Elements picked by (id + element + off) % mod == 0: every occurrence of a sign gets the same pattern."""
    k = (np.asarray(ids, np.uint64) % np.uint64(mod)).astype(np.int64)
    return (k[:, None] + np.arange(dim)[None, :] + off) % mod == 0


def _uniform(lo, hi):
    return lambda signs, dim: np.random.default_rng(len(signs) + dim).uniform(lo, hi, (len(signs), dim)).astype(np.float32)


def _run_all(torch, oracle, kind, dim, seed_fn, grad_fn, paths=EDGE_PATHS, **kw):
    return {p: run_edge_path(torch, oracle, p, kind, dim, seed_fn, grad_fn, **kw) for p in paths}


def _same(res):
    for p, (signs, got, want) in res.items():
        for k in range(signs.size):
            assert same_bits(got[k], want[k]), (p, k, int(signs[k]), got[k], want[k])


# ---- the weight bound -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [12, 64, 130, 256])
@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_weight_bound_engaged(torch_cuda, oracle, kind, dim):
    """wb = 0.02, rows just inside it and steps far past it: every element ends in [-wb, wb] and most sit on it
    (persia-simd weight_bound: min(max(w, -b), b))."""
    wb = 0.02
    g = lambda rng, ids, d: (rng.standard_normal((len(ids), d)) * 10).astype(np.float16)  # noqa: E731
    res = _run_all(torch_cuda, oracle, kind, dim, _uniform(-0.019, 0.019), g, opt=dict(lr=0.5),
                   hyper=dict(wb=wb), steps=2)
    _same(res)
    for p, (_, got, _) in res.items():
        emb = got[:, :dim]
        assert (np.abs(emb) <= np.float32(wb)).all(), p
        assert (np.abs(emb) == np.float32(wb)).mean() > 0.5, p


@pytest.mark.parametrize("dim", [64, 130])
@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_weight_bound_off(torch_cuda, oracle, kind, dim):
    """enable_weight_bound = 0: rows past 10 stay there."""
    def seed(signs, d):
        x = _uniform(12.0, 14.0)(signs, d)
        return np.where(_mask(signs, d, 2), -x, x)
    g = lambda rng, ids, d: (rng.standard_normal((len(ids), d)) * 1e-2).astype(np.float16)  # noqa: E731
    res = _run_all(torch_cuda, oracle, kind, dim, seed, g, hyper=dict(enable_wb=False), steps=2)
    _same(res)
    for p, (_, got, _) in res.items():
        assert (np.abs(got[:, :dim]) > 11).all(), p


# ---- gradient values --------------------------------------------------------------------------------------------------
def _f16_extremes(rng, ids, dim):
    g = (rng.standard_normal((len(ids), dim)) * 1e-2).astype(np.float16)
    big = _mask(ids, dim, 5)
    g[big] = np.where(np.nonzero(big)[1] % 2 == 0, 65504, -65504)
    g[_mask(ids, dim, 7, 3)] = np.inf
    g[_mask(ids, dim, 7, 5)] = -np.inf
    hot = np.flatnonzero(np.asarray(ids, np.uint64) == 0)  # a hot sign whose occurrences mix +inf and -inf
    g[hot[0::2], 0] = np.inf
    g[hot[1::2], 0] = -np.inf
    return g


@pytest.mark.parametrize("kind,dim", [(0, 64), (1, 130), (2, 12), (3, 256), (1, 64), (0, 130)])
def test_f16_extreme_gradients(torch_cuda, oracle, kind, dim):
    """f16 +-65504 and +-inf: the EW clamps +-inf to +-65504 before it sums (persia-common lib.rs:163-180).  The hot
    sign's element 0 takes as many +inf as -inf, so it sums to exactly 0 and SGD leaves it as it was; Adagrad's state
    stays finite wherever a row took one f16 gradient (raw); pb_update takes the f32 inf as given."""
    seed = _uniform(-0.01, 0.01)
    res = _run_all(torch_cuda, oracle, kind, dim, seed, _f16_extremes, steps=2)
    _same(res)
    if kind == 0:
        signs, got, _ = res["batch"]
        k = int(np.flatnonzero(signs == oracle.add_prefix(np.zeros(1, np.uint64), 8, oracle.index_prefix(0))[0])[0])
        assert got[k, 0] == seed(signs, dim)[k, 0]
    if kind == 1:
        assert np.isfinite(res["raw"][1][:, dim:]).all()
        assert np.isinf(res["direct"][1][:, dim:]).any()


@pytest.mark.parametrize("kind,dim", [(0, 64), (1, 12), (2, 130), (3, 64)])
def test_f16_subnormal_gradients(torch_cuda, oracle, kind, dim):
    """f16 subnormal gradients on rows of the same scale: a flush anywhere changes the row."""
    def g(rng, ids, d):
        return (rng.integers(-1023, 1024, (len(ids), d)) * 2.0**-24).astype(np.float16)
    _same(_run_all(torch_cuda, oracle, kind, dim, _uniform(-1e-6, 1e-6), g, opt=dict(lr=0.5), steps=2))


def _f32_inf(rng, ids, dim):
    g = (rng.standard_normal((len(ids), dim)) * 1e-2).astype(np.float32)
    g[_mask(ids, dim, 7)] = np.inf
    g[_mask(ids, dim, 7, 3)] = -np.inf
    return g


@pytest.mark.parametrize("dim", [64, 130])
@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_f32_inf_gradients(torch_cuda, oracle, kind, dim):
    """f32 +-inf are not clamped.  One step of w - lr * (+-inf) is -+inf for SGD and (with the old accumulator) both
    Adagrads, and the bound takes it to -+wb; Adam's descent is inf / inf = NaN, which the bound maps to -wb
    (_mm256_max_ps(w, -b) / fmax return -b for a NaN w).  Adagrad's accumulator becomes inf."""
    wb = np.float32(10)
    res = _run_all(torch_cuda, oracle, kind, dim, _uniform(-0.01, 0.01), _f32_inf)
    _same(res)
    for p in ONE_STEP:
        signs, got, _ = res[p]
        ids = signs - np.uint64(oracle.index_prefix(0))
        pos, neg = _mask(ids, dim, 7), _mask(ids, dim, 7, 3)
        emb = got[:, :dim]
        if kind == 3:
            assert (emb[pos | neg] == -wb).all(), p
        else:
            assert (emb[pos] == -wb).all() and (emb[neg] == wb).all(), p
        if kind == 1:
            assert np.isposinf(got[:, dim:][pos | neg]).all(), p
        if kind == 2:
            assert np.isposinf(got[:, dim][(pos | neg).any(axis=1)]).all(), p


@pytest.mark.parametrize("kind,dim", [(0, 64), (1, 130), (3, 12), (2, 256)])
def test_f32_sums_overflow(torch_cuda, oracle, kind, dim):
    """3e38 in the same elements of every occurrence: the hot and warm sums overflow to inf inside the reduce."""
    def g(rng, ids, d):
        x = (rng.standard_normal((len(ids), d)) * 1e-2).astype(np.float32)
        x[_mask(ids, d, 4)] = 3e38
        return x
    res = _run_all(torch_cuda, oracle, kind, dim, _uniform(-0.01, 0.01), g)
    _same(res)
    if kind == 0:
        signs, got, _ = res["batch"]
        ids = signs - np.uint64(oracle.index_prefix(0))
        assert (got[:, :dim][_mask(ids, dim, 4)] == -10).all()


def _tiny_rows(signs, dim):
    x = FLT_MIN * ((np.arange(dim) % 8) + 1) / np.float32(8)  # 1/8 .. 1 of FLT_MIN: subnormal rows too
    return np.where(_mask(signs, dim, 3), -x, x).astype(np.float32) * np.ones((len(signs), 1), np.float32)


def _tiny_grad(ids, dim):
    """Multiples of 2^-135 below FLT_MIN in magnitude (f32 subnormals), the same for every occurrence of a sign."""
    k = (np.asarray(ids, np.uint64) % np.uint64(1009)).astype(np.int64)
    return ((((k[:, None] * 7 + np.arange(dim)[None, :] * 13) % 2001) - 1000) * 2.0**-135).astype(np.float32)


@pytest.mark.parametrize("kind,dim", [(0, 64), (0, 130), (1, 12), (2, 64), (3, 256)])
def test_f32_subnormal_gradients_near_flt_min(torch_cuda, oracle, kind, dim):
    """Rows at FLT_MIN and f32 subnormal gradients.  For SGD with lr = 0.5 and wd = 0 every product and sum is exact,
    so the row is w - 0.5 * n * g with n the sign's multiplicity, much of it subnormal: a flush to zero anywhere fails."""
    res = _run_all(torch_cuda, oracle, kind, dim, _tiny_rows, lambda rng, ids, d: _tiny_grad(ids, d),
                   opt=dict(lr=0.5))
    _same(res)
    if kind != 0:
        return
    for p in ONE_STEP:
        signs, got, _ = res[p]
        ids = signs - np.uint64(oracle.index_prefix(0))
        n = np.ones(ids.size)
        if p == "batch":
            for i, c in enumerate(EDGE_COUNTS):
                n[ids == i] = c
        want = (_tiny_rows(signs, dim).astype(np.float64) - 0.5 * n[:, None] * _tiny_grad(ids, dim)).astype(np.float32)
        assert same_bits(got[:, :dim], want), p
        sub = (np.abs(got[:, :dim]) < FLT_MIN) & (got[:, :dim] != 0)
        assert sub.mean() > 0.2, p


@pytest.mark.parametrize("dtype", [np.float16, np.float32])
@pytest.mark.parametrize("kind", [0, 1])
def test_negative_zero_gradient_on_negative_zero_row(torch_cuda, oracle, kind, dtype):
    """The EW adds every gradient into a zeroed row — summed (mod.rs:800-812) and raw (mod.rs:780-798) alike — so a -0
    gradient reaches the step as +0, and w = -0 - lr * (+0) stays -0.  pb_update takes the gradient as given, as the PS
    does (PS mod.rs:359-427): -0 - lr * (-0) = +0.  The f32 raw gradient without a loss scale is staged for this too."""
    seed = lambda signs, d: np.full((len(signs), d), -0.0, np.float32)  # noqa: E731
    g = lambda rng, ids, d: np.full((len(ids), d), -0.0, dtype)  # noqa: E731
    res = _run_all(torch_cuda, oracle, kind, 64, seed, g, opt=dict(wd=0.0))
    _same(res)
    for p, (_, got, _) in res.items():
        bits = got[:, :64].view(np.uint32)
        assert (bits == (0 if p == "direct" else 0x80000000)).all(), (p, np.unique(bits))


@pytest.mark.parametrize("dim", [64, 130])
@pytest.mark.parametrize("kind", [0, 1])
def test_scaled_negative_subnormal_gradient_on_negative_zero_row(torch_cuda, oracle, kind, dim):
    """Loss scale 2 on f32 gradients of -2^-149 (even elements) and -k * 2^-149, k = 2..7 (odd elements).  The EW
    multiplies by 1/scale first (mod.rs:751-755): -2^-149 * 0.5 rounds to -0, and only then adds into zeros
    (mod.rs:780-812), which makes it +0; so a -0 row stays -0 in the even elements.  A single fma(g, 0.5, +0) would
    round the exact -2^-150 to -0 and step the row to +0.  pb_update has no loss scale: -0 - lr * (-2^-149) = +0."""
    seed = lambda signs, d: np.full((len(signs), d), -0.0, np.float32)  # noqa: E731

    def g(rng, ids, d):
        x = -(rng.integers(2, 8, (len(ids), d)) * 2.0**-149).astype(np.float32)
        x[:, 0::2] = -np.float32(2.0**-149)
        return x
    res = _run_all(torch_cuda, oracle, kind, dim, seed, g, opt=dict(wd=0.0), scale=2.0)
    _same(res)
    for p, (_, got, _) in res.items():
        bits = got[:, :dim:2].view(np.uint32)
        assert (bits == (0 if p == "direct" else 0x80000000)).all(), (p, np.unique(bits))


# ---- degenerate optimizer settings ------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [64, 130])
def test_adagrad_zero_eps_zero_state_zero_gradient(torch_cuda, oracle, dim):
    """eps = 0, initialization = 0, g = 0: 1/sqrt(0) = inf and 0 * inf = NaN; the bound maps NaN to -wb."""
    g = lambda rng, ids, d: np.zeros((len(ids), d), np.float32)  # noqa: E731
    res = _run_all(torch_cuda, oracle, 1, dim, _uniform(-0.01, 0.01), g, opt=dict(eps=0.0, init_acc=0.0))
    _same(res)
    for p, (_, got, _) in res.items():
        assert (got[:, :dim] == -10).all() and (got[:, dim:] == 0).all(), p


@pytest.mark.parametrize("dim", [64, 130])
def test_vectorwise_adagrad_dot_overflow(torch_cuda, oracle, dim):
    """g = 1e20: dot(g, g) overflows, the shared state becomes inf; the step that used the old state hits the bound,
    and a later one scales by 1/sqrt(inf) = 0 and leaves the row there."""
    g = lambda rng, ids, d: np.full((len(ids), d), 1e20, np.float32)  # noqa: E731
    res = _run_all(torch_cuda, oracle, 2, dim, _uniform(-0.01, 0.01), g)
    _same(res)
    for p, (_, got, _) in res.items():
        assert (got[:, :dim] == -10).all() and np.isposinf(got[:, dim]).all(), p


@pytest.mark.parametrize("dim", [64, 130])
def test_adam_zero_eps_zero_gradient(torch_cuda, oracle, dim):
    """eps = 0, g = 0 on fresh state: the descent is 0 / (0 + sqrt(0)) = NaN, bound to -wb; m and v stay 0."""
    g = lambda rng, ids, d: np.zeros((len(ids), d), np.float32)  # noqa: E731
    res = _run_all(torch_cuda, oracle, 3, dim, _uniform(-0.01, 0.01), g, opt=dict(eps=0.0))
    _same(res)
    for p, (_, got, _) in res.items():
        assert (got[:, :dim] == -10).all() and (got[:, dim:] == 0).all(), p


# ---- the f16 rounding of the forward ----------------------------------------------------------------------------------
EDGE_VALUES = np.array([65504.0, 65519.996, 65520.0, 1e-7, -0.0, 32752.0, -32760.0, 3e-5, -1e-7, 0.5], np.float32)


def _edge_rows(signs, dim):
    k = (np.asarray(signs, np.uint64) % np.uint64(len(EDGE_VALUES))).astype(np.int64)
    return EDGE_VALUES[(k[:, None] + np.arange(dim)[None, :]) % len(EDGE_VALUES)]


def _seed(torch, oracle, shards, w, signs, dim, R):
    ent = _edge_rows(signs, dim)
    owner = oracle.shard_of(signs, R) if R > 1 else np.zeros(signs.size, np.uint32)
    for r, s in enumerate(shards):
        m = owner == r
        if m.any():
            s.set_entries(to_dev_ids(signs[m], DEV), torch.from_numpy(ent[m].copy()).to(DEV))
    w.set_embedding(signs, ent, dim)
    torch.cuda.synchronize()
    return ent


@pytest.mark.parametrize("dim", [64, 130])
def test_forward_f16_rounding_edges(torch_cuda, oracle, dim):
    """Rows at 65504, 65519.996 (rounds down), 65520 (rounds to inf), f16 subnormals and -0: single-id copies are
    f16(0 + row) (-0 -> +0), pooled sums with and without sqrt scaling overflow to inf, the raw table is f16(row) (-0
    stays), and the sharded forward over f16 and f32 row exchanges gives the same."""
    from persia_b200 import shard as SH
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    rng = np.random.default_rng(dim)
    pf = oracle.index_prefix(0)
    B, n_ids = 64, 40
    ids1 = rng.integers(0, n_ids, B, dtype=np.uint64)
    counts = rng.integers(0, 3, B)  # up to two ids: the sum does not depend on their order
    row_off = np.zeros(2 * B + 1, np.uint32)
    row_off[1:B + 1] = np.arange(1, B + 1)
    row_off[B + 1:] = B + np.cumsum(counts)
    ids2 = rng.integers(0, n_ids, int(counts.sum()), dtype=np.uint64)
    signs = oracle.add_prefix(np.arange(n_ids, dtype=np.uint64), 8, pf)
    rows = _edge_rows(signs, dim)
    lists = [[int(x) for x in ids2[row_off[B + b] - B:row_off[B + b + 1] - B]] for b in range(B)]
    for sqrt in (False, True):
        s = SH.EmbeddingShard(dim, 1 << 12, 0)
        s.set_optimizer(0, lr=0.1)
        s.configure()
        w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf), oracle.SlotCfg(dim, sqrt_scaling=sqrt, prefix=pf)], n_ps=1)
        w.configure()
        w.set_optimizer(oracle.Optim(0, lr=0.1))
        _seed(torch, oracle, [s], w, signs, dim, 1)
        ctx = SH.BatchContext(4 * B, 2 * B, [pf, pf], [False, sqrt])
        ids = np.concatenate([ids1, ids2])
        got = ctx.forward(s, to_dev_ids(ids, DEV), [0, B, ids.size], B, row_off=to_dev_i32(row_off, DEV),
                          training=False).cpu().numpy()
        want, _ = w.forward(ids, row_off, B, training=False)
        assert same_bits(got[0], want[0]) and same_bits(got[1], want[1])
        assert same_bits(got[0], pool_lists(rows, [[int(k)] for k in ids1], False))
        assert same_bits(got[1], pool_lists(rows, lists, sqrt))
        assert np.isposinf(got[0]).any() and not (got[0].view(np.uint16) == 0x8000).any()
    # the raw table: f16(row), -0 kept
    s = SH.EmbeddingShard(dim, 1 << 12, 0)
    s.set_optimizer(0, lr=0.1)
    s.configure()
    w = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=3, prefix=pf)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(0, lr=0.1))
    _seed(torch, oracle, [s], w, signs, dim, 1)
    ctx = SH.BatchContext(4 * B, 4 * B, [pf])
    ro = row_off[B:] - B
    table, _, _, _, cnt = ctx.forward_raw(s, to_dev_ids(ids2, DEV), B, 3, row_off=to_dev_i32(ro, DEV), training=False)
    U = int(cnt[0])
    wt = w.forward_raw(0, ids2, ro, B, training=False)[0]
    first = ids2[np.sort(np.unique(ids2, return_index=True)[1])].astype(np.int64)
    with np.errstate(over="ignore"):
        closed = np.concatenate([np.zeros((1, dim), np.float16), rows[first].astype(np.float16)])
    assert same_bits(table[:U + 1].cpu().numpy(), wt) and same_bits(wt, closed)
    assert (wt.view(np.uint16) == 0x8000).any()
    # sharded, one id per sample: f16 and f32 row exchanges
    for rows_f32 in (False, True):
        R = 2
        ws = W.local_group(R, 1, dim, [pf], 1 << 12, cap=B, optimizer=dict(kind=0, lr=0.1), max_batch=B,
                           rows_f32=rows_f32)
        w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf)], n_ps=R)
        w.configure()
        w.set_optimizer(oracle.Optim(0, lr=0.1))
        for x in ws:
            x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
        _seed(torch, oracle, [x.shard for x in ws], w, signs, dim, R)
        batches = [rng.integers(0, n_ids, B, dtype=np.uint64) for _ in range(R)]
        torch.cuda.synchronize()
        outs = W.group_forward(ws, [to_dev_ids(b, DEV) for b in batches], B, training=False)
        torch.cuda.synchronize()
        for r in range(R):
            want, _ = w.forward(batches[r], full_row_off(1, B), B, training=False)
            got = outs[r][0].cpu().numpy()
            assert same_bits(got, want[0]), (rows_f32, r)
            assert same_bits(got, pool_lists(rows, [[int(k)] for k in batches[r]], False)), (rows_f32, r)


# ---- init range -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lo,hi", [(0.5, 0.75), (1.0, float(np.nextafter(np.nextafter(np.float32(1), np.float32(2)),
                                                                           np.float32(2))))])
@pytest.mark.parametrize("dim", [12, 64])
def test_first_touch_rows_in_init_range(torch_cuda, oracle, dim, lo, hi):
    """A new row is init_row(sign, dim, lo, hi) (emb_entry.rs:28-68) on every admitting path: the batched forward,
    pb_lookup(training = 1), the raw forward and sharded admission.  The two-ulp range runs uniform_scale's shrink loop."""
    from persia_b200 import shard as SH
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    pf = oracle.index_prefix(0)
    lo32, hi32 = float(np.float32(lo)), float(np.float32(hi))
    hyper = dict(init_lower=lo32, init_upper=hi32)
    B = 50
    ids = np.arange(B, dtype=np.uint64) * np.uint64(7919) + np.uint64(3)
    signs = oracle.add_prefix(ids, 8, pf)
    want = np.stack([oracle.init_row(int(x), dim, lo32, hi32) for x in signs])
    assert ((want >= np.float32(lo)) & (want < np.float32(hi))).all()

    def shard():
        s = SH.EmbeddingShard(dim, 1 << 12, 0)
        s.set_optimizer(1, lr=0.1, initialization=0.25)
        s.configure(**hyper)
        return s

    def check(s, sg, what):
        ent, found = s.get_entries(to_dev_ids(sg, DEV))
        ent = ent.cpu().numpy()
        assert found.all(), what
        rows = np.stack([oracle.init_row(int(x), dim, lo32, hi32) for x in sg])
        assert same_bits(ent[:, :dim], rows), what
        assert (ent[:, dim:] == np.float32(0.25)).all(), what

    s = shard()
    ctx = SH.BatchContext(B, B, [pf])
    out = ctx.forward(s, to_dev_ids(ids, DEV), [0, B], B, training=True).cpu().numpy()
    check(s, signs, "batched forward")
    assert same_bits(out[0], want.astype(np.float16))
    s = shard()
    got = s.lookup(to_dev_ids(signs, DEV), training=True).cpu().numpy()
    assert same_bits(got, want)
    check(s, signs, "pb_lookup")
    s = shard()
    ctx = SH.BatchContext(B, B, [pf])
    ctx.forward_raw(s, to_dev_ids(ids, DEV), B, 1, training=True)
    check(s, signs, "raw forward")
    R = 2
    ws = W.local_group(R, 1, dim, [pf], 1 << 12, cap=B, optimizer=dict(kind=1, lr=0.1, initialization=0.25),
                       hyper=hyper, max_batch=B)
    for x in ws:
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    W.group_forward(ws, [to_dev_ids(ids, DEV)] * R, B, training=True)
    torch.cuda.synchronize()
    owner = oracle.shard_of(signs, R)
    for r in range(R):
        check(ws[r].shard, signs[owner == r], f"sharded rank {r}")


# ---- admit_probability < 1 --------------------------------------------------------------------------------------------
def test_admit_probability_properties(torch_cuda, oracle):
    """The reference draws admission from an unpinned RNG, so only properties are checked: the admitted fraction lies
    within a binomial bound; a sign that was not admitted reads zeros, holds no row and counts one gradient_id_miss
    per applied entry; inference admits nothing; and the resident rows match the oracle replaying the step on them."""
    from persia_b200 import shard as SH

    torch = torch_cuda
    p, B, dim = 0.3, 4000, 16
    pf = oracle.index_prefix(0)
    s = SH.EmbeddingShard(dim, 1 << 14, 0)
    s.set_optimizer(1, lr=0.02, initialization=0.01, eps=1e-10)
    s.configure(admit_probability=p)
    ctx = SH.BatchContext(B, B, [pf])
    rng = np.random.default_rng(3)
    ids = rng.permutation(np.arange(B, dtype=np.uint64) + np.uint64(1 << 20))  # every id once: one entry per sign
    signs = oracle.add_prefix(ids, 8, pf)
    before = s.counters()
    out = ctx.forward(s, to_dev_ids(ids, DEV), [0, B], B, training=True).cpu().numpy()[0]
    n = len(s)
    assert abs(n - p * B) < 5 * np.sqrt(B * p * (1 - p)), n
    ent, found = s.get_entries(to_dev_ids(signs, DEV))
    ent, found = ent.cpu().numpy(), found.cpu().numpy().astype(bool)
    assert found.sum() == n
    assert (out[~found].view(np.uint16) == 0).all()
    assert same_bits(out[found], ent[found, :dim].astype(np.float16))
    # the oracle, seeded with the GPU's resident rows, replays the step (its own admission decides nothing here:
    # a row's step does not depend on which other signs hold rows)
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(1, lr=0.02, init_acc=0.01, eps=1e-10))
    w.set_embedding(signs[found], ent[found], dim)
    g = (rng.standard_normal((B, dim)) * 1e-2).astype(np.float16)
    oracle.set_rsqrt_exact(True)
    try:
        _, octx = w.forward(ids, np.arange(B + 1, dtype=np.uint32), B, training=True)
        w.backward(octx, [g])
        ctx.backward(s, [torch.from_numpy(g).to(DEV)])
        after = s.counters()
        assert after["gradient_id_miss"] - before["gradient_id_miss"] == B - n
        got = s.get_entries(to_dev_ids(signs[found], DEV))[0].cpu().numpy()
        for k, sign in enumerate(signs[found]):
            assert same_bits(got[k], w.get_entry(int(sign))), k
    finally:
        oracle.set_rsqrt_exact(False)
    fresh = np.arange(B, dtype=np.uint64) + np.uint64(1 << 30)
    ctx.forward(s, to_dev_ids(fresh, DEV), [0, B], B, training=False)
    torch.cuda.synchronize()
    assert len(s) == n
