"""GPU: the short hot items (33..128 occurrences) of batches of 8192 samples or more, which k_reduce_hot_short sums a
warp per item, against the CPU oracle bit for bit (Adagrad in the oracle's exact-rsqrt mode) and, for SGD, against a
float64 computation of the reference operation.  Every batch holds items either side of the edges (33, 34, 64, 65, 128
beside 129, 255, 256 and the huge 257, which k_reduce_hot sums), so both hot kernels stage sums into one staging buffer
that one k_step_hot reads.

  dims                 1, 3 (element loads), 64, 127, 128, 513 (a lane takes several column blocks); f16 and f32
  ragged               several ids per sample with sqrt scaling and a loss scale (occ_outrow and row_off read per row)
  two windows          a slot of more than HOT_WIN samples: items in both windows and across the boundary
  list mode            the bitmap pool runs out: most short items come with unsorted occurrence lists
  NaN / skipped slots  dead slots' items are skipped with their bits cleared: the next batches are exact
  rounds               slots of one feature group: the reduce runs once per round, other rounds' bits are kept
  graph                a captured backward, replayed, then eager steps
"""
import numpy as np
import pytest

from test_gpu_reduce_boundaries import HOT_WIN, HYPER, OPT, WARM_MAX, _check, _run, _train, _window_items
from util import DEV, batch_with_multiplicities, fwd_both, pair, ragged_with_multiplicities

pytestmark = pytest.mark.gpu

SGD, ADAGRAD, ADAGRAD_VW, ADAM = 0, 1, 2, 3
EDGES = [257, 256, 255, 129, 128, 65, 64, 34, 33, 32, 2]  # k_reduce_hot | k_reduce_hot_short | warm
MANY = [33 + (37 * k) % 224 for k in range(16)]  # hot items of many lengths


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


def _one_id(counts, S, B):
    return lambda rng: [(batch_with_multiplicities(rng, B, counts), None) for _ in range(S)]


@pytest.mark.parametrize("kind", [SGD, ADAGRAD])
@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("dim", [1, 3, 64, 127, 128, 513])
def test_class_edges_by_dim(torch_cuda, pb, oracle, dim, f32, kind):
    B = 8192
    counts = EDGES + MANY
    stats = {"hot": 2 * sum(c > WARM_MAX for c in counts)}
    _run(torch_cuda, pb, oracle, _one_id(counts, 2, B), 2, B, dim, kind, f32=f32, cap=1 << 16, stats=stats)


@pytest.mark.parametrize("dim,f32", [(64, False), (128, False), (127, True)])
def test_ragged_sqrt_and_scale(torch_cuda, pb, oracle, dim, f32):
    B = 8192

    def make(rng):
        return [ragged_with_multiplicities(rng, B, EDGES + MANY[:20], max_ids=3, min_ids=2),
                ragged_with_multiplicities(rng, B, EDGES, max_ids=4)]

    _run(torch_cuda, pb, oracle, make, 2, B, dim, SGD, f32=f32, scale=[3.0, 128.0], sqrt=[True, False], cap=1 << 17,
         max_occ=2 * 4 * B)


@pytest.mark.parametrize("kind", [SGD, ADAGRAD])
def test_two_windows(torch_cuda, pb, oracle, kind):
    """Slots of more than HOT_WIN samples: a short item across the window boundary, one in the last window only."""
    B = HOT_WIN + 3000
    counts, spans = _window_items(B)

    def make(rng):
        return [(batch_with_multiplicities(rng, B, counts + EDGES, spans), None),
                (batch_with_multiplicities(rng, B, EDGES + MANY), None)]

    _run(torch_cuda, pb, oracle, make, 2, B, 128, kind, cap=1 << 16)


@pytest.mark.parametrize("f32", [False, True])
def test_bitmap_pool_exhaustion_list_mode(torch_cuda, pb, oracle, f32):
    """A context sized to the batch: most of the hot items find no room in the bitmap pool and come with unsorted
    occurrence lists, beside the ones that do."""
    S, B = 1, 16384
    counts = [256, 129, 128, 127] + [33 + k % 32 for k in range(200)] + [1500, 2]
    assert sum(c > WARM_MAX for c in counts) * ((B + 31) // 32) > max(4096, S * B)
    _run(torch_cuda, pb, oracle, _one_id(counts, S, B), S, B, 128, ADAGRAD, f32=f32, max_occ=S * B)


@pytest.mark.parametrize("kind", [ADAGRAD, ADAM])
def test_nan_and_skipped_then_clean(torch_cuda, pb, oracle, kind):
    """A NaN slot and a skipped slot hold short items: their rows stay, their bits go back to zero, and the clean
    batches after them (the same signs, the same bitmap words) are exact."""
    torch = torch_cuda
    S, B, dim = 3, 8192, 128
    rng = np.random.default_rng(40 + kind)
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, cap=1 << 18, optim_kw=OPT[kind], hyper_kw=HYPER, max_occ=S * B)
    make = _one_id(EDGES + MANY, S, B)
    touched = []
    for nan, skip in [(None, None), (0, 2), (None, None), (1, None), (None, 0), (None, None)]:
        touched += _train(torch, s, ctx, w, oracle, pf, make(rng), B, dim, rng, kind, nan=nan, skip=skip)
    _check(torch, s, w, [np.unique(np.concatenate(touched))])


@pytest.mark.parametrize("groups", [[0, 0], [0, 1, 0]])
def test_shared_feature_group(torch_cuda, pb, oracle, groups):
    torch = torch_cuda
    S, B, dim = len(groups), 8192, 64
    rng = np.random.default_rng(70 + S)
    s, ctx, w, pf = pair(pb, oracle, S, dim, ADAGRAD, cap=1 << 16, groups=groups, optim_kw=OPT[ADAGRAD], max_occ=S * B)
    touched = []
    for nan in [None, S - 1, None]:
        t = _train(torch, s, ctx, w, oracle, pf, _one_id(EDGES + MANY, S, B)(rng), B, dim, rng, ADAGRAD, nan=nan)
        touched.append(np.concatenate(t))
    _check(torch, s, w, [np.unique(np.concatenate(touched))])


def test_captured_backward_replayed(torch_cuda, pb, oracle):
    torch = torch_cuda
    S, B, dim, kind = 2, 8192, 128, ADAGRAD
    rng = np.random.default_rng(9)
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, cap=1 << 16, optim_kw=OPT[kind], hyper_kw=HYPER, max_occ=S * B)
    make = _one_id(EDGES + MANY, S, B)
    touched = _train(torch, s, ctx, w, oracle, pf, make(rng), B, dim, rng, kind)
    ids = np.concatenate([x[0] for x in make(rng)])
    _, _, octx = fwd_both(torch, s, ctx, w, ids, None, [0, B, 2 * B], B, training=True)
    touched += [w.ctx_signs(octx, i) for i in range(S)]
    g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
    grads = [torch.from_numpy(g[i]).to(DEV) for i in range(S)]
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ctx.backward(s, grads)
    graph.replay()
    torch.cuda.synchronize()
    w.backward(octx, [g[i] for i in range(S)])
    _check(torch, s, w, [np.unique(np.concatenate(touched))])
    touched += _train(torch, s, ctx, w, oracle, pf, make(rng), B, dim, rng, kind)
    _check(torch, s, w, [np.unique(np.concatenate(touched))])
