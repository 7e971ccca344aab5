"""GPU: the hot-sign backward in two kernels — k_reduce_hot stages every hot item's ordered sum without reading the NaN
marks (it runs beside the NaN scan), k_step_hot applies the NaN rule and steps the rows once the scan is done — against
the CPU oracle bit for bit (Adagrad in the oracle's exact-rsqrt mode).

  NaN / skipped slots   slots holding giant, huge and hot items get a NaN gradient or none beside applied slots: their
                        rows stay, the others step, and the next batches (the same hot signs, their bitmaps reused) are
                        exact; every optimizer, f16 and f32 gradients, dims of each hot geometry and two column passes
  rows missing          hot signs that hold no row: gradient_id_miss counts the applied slots' items only
  rounds                slots of one feature group with a NaN slot: reduce, then step, round by round on one stream
  graph capture         a captured backward with no eager backward before it, then eager steps
"""
import numpy as np
import pytest

from test_gpu_reduce_boundaries import HYPER, OPT, _check, _train
from util import DEV, _seed_rows, batch_with_multiplicities, fwd_both, pair

pytestmark = pytest.mark.gpu

SGD, ADAGRAD, ADAGRAD_VW, ADAM = 0, 1, 2, 3
COUNTS = [1500, 1100, 300, 40, 33, 5]  # ids 0..: giant, giant, huge, hot, hot, warm; the rest of a slot is cold


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


def _slots(S, B):
    return lambda rng: [(batch_with_multiplicities(rng, B, COUNTS), None) for _ in range(S)]


@pytest.mark.parametrize("kind", [SGD, ADAGRAD, ADAGRAD_VW, ADAM])
@pytest.mark.parametrize("dim,f32", [(16, False), (64, False), (128, False), (130, False), (640, False), (128, True),
                                     (640, True)])
def test_nan_and_skipped_slots_beside_applied(torch_cuda, pb, oracle, dim, f32, kind):
    torch = torch_cuda
    S, B = 3, 4096
    rng = np.random.default_rng(100 * dim + 10 * kind + f32)
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, cap=1 << 16, optim_kw=OPT[kind], hyper_kw=HYPER, max_occ=S * B)
    make = _slots(S, B)
    touched = []
    for nan, skip in [(None, None), (0, None), (None, 1), (2, 0), (None, None)]:
        touched += _train(torch, s, ctx, w, oracle, pf, make(rng), B, dim, rng, kind, f32=f32, nan=nan, skip=skip)
    _check(torch, s, w, [np.unique(np.concatenate(touched))])


@pytest.mark.parametrize("kind", [ADAGRAD, ADAGRAD_VW])
def test_hot_signs_without_rows(torch_cuda, pb, oracle, kind):
    """Nothing is admitted (admit_probability 0): of every slot only the seeded signs hold rows, among them some of the
    hot ones.  gradient_id_miss counts one per item of an applied slot without a row — the NaN slot's and the skipped
    slot's items are not counted — and the seeded rows step as the oracle's do."""
    torch = torch_cuda
    S, B, dim = 3, 4096, 64
    rng = np.random.default_rng(7 + kind)
    hyper = dict(HYPER, admit_p=0.0)
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, cap=1 << 15, optim_kw=OPT[kind], hyper_kw=hyper, max_occ=S * B)
    w.set_faithful_miss(False)  # a sign without a row consumes its gradient, as on the GPU
    seeded = np.concatenate([oracle.add_prefix(np.array([0, 2, 3, 5], np.uint64), 8, pf[i]) for i in range(S)])
    seed = lambda signs, d: rng.uniform(-0.1, 0.1, (signs.size, d))  # noqa: E731
    _seed_rows(torch, oracle, [s], w, seeded, dim, kind, OPT[kind], seed, 1)
    make = _slots(S, B)
    miss0 = s.counters()["gradient_id_miss"]
    want_miss = 0
    for nan, skip in [(None, None), (1, None), (None, 2), (None, None)]:
        slots = make(rng)
        _train(torch, s, ctx, w, oracle, pf, slots, B, dim, rng, kind, nan=nan, skip=skip)
        for i, (ids, _) in enumerate(slots):
            if i not in (nan, skip):
                want_miss += int(np.setdiff1d(oracle.add_prefix(np.unique(ids), 8, pf[i]), seeded).size)
    assert s.counters()["gradient_id_miss"] - miss0 == want_miss == w.grad_miss()
    _check(torch, s, w, [seeded])


@pytest.mark.parametrize("kind", [ADAGRAD, ADAM])
def test_shared_feature_group_with_nan_slot(torch_cuda, pb, oracle, kind):
    """Slots 0 and 2 of one feature group (two rounds) beside slot 1; the second round's slot holds a NaN in one step,
    the first round's in another."""
    torch = torch_cuda
    groups, B, dim = [0, 1, 0], 4096, 64
    S = len(groups)
    rng = np.random.default_rng(31 + kind)
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, cap=1 << 16, groups=groups, optim_kw=OPT[kind], max_occ=S * B)
    make = _slots(S, B)
    touched = []
    for nan in [None, 2, None, 0, None]:
        touched += _train(torch, s, ctx, w, oracle, pf, make(rng), B, dim, rng, kind, nan=nan)
    _check(torch, s, w, [np.unique(np.concatenate(touched))])


def test_captured_backward_first(torch_cuda, pb, oracle):
    """A backward captured into a CUDA graph right after the context's first (eager) forward, replayed once, then eager
    steps over the same hot signs."""
    torch = torch_cuda
    S, B, dim, kind = 2, 4096, 128, ADAGRAD
    rng = np.random.default_rng(3)
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, cap=1 << 16, optim_kw=OPT[kind], hyper_kw=HYPER, max_occ=S * B)
    slots = _slots(S, B)(rng)
    ids = np.concatenate([x[0] for x in slots])
    _, _, octx = fwd_both(torch, s, ctx, w, ids, None, [0, B, 2 * B], B, training=True)
    touched = [w.ctx_signs(octx, i) for i in range(S)]
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
    for _ in range(2):
        touched += _train(torch, s, ctx, w, oracle, pf, _slots(S, B)(rng), B, dim, rng, kind)
    _check(torch, s, w, [np.unique(np.concatenate(touched))])
