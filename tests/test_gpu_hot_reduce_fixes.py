"""GPU: k_reduce_hot (csrc/pb_reduce.cu) against the CPU oracle bit for bit (Adagrad in the oracle's exact-rsqrt mode),
at the cases two defects hid in.

  f32 gradients, dim 128   the producers' lean loop converts at most four parts of a ring chunk; a chunk of 64 rows in
                           parts of 8 (32 f32 vectors per row) left rows 32..63 of every chunk unwritten
  shared feature groups    two slots of one group on one GPU run the hot reduce once per round; the first round saw the
                           second round's items as dead and zeroed their bitmaps, so that round summed nothing
Beside them, the longest chains of the metric workload's shape: items either side of 256 and 1024 occurrences and one
of 4080, at dims with each producer mode, f16 and f32.
"""
import numpy as np
import pytest

from test_gpu_reduce_boundaries import OPT, _check, _run, _train
from util import batch_with_multiplicities, pair

pytestmark = pytest.mark.gpu

SGD, ADAGRAD, ADAGRAD_VW, ADAM = 0, 1, 2, 3
LONG = [4080, 1025, 1024, 257, 256, 40, 33, 2]


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


def _one_id(counts, S=1, B=8192):
    return lambda rng: [(batch_with_multiplicities(rng, B, counts), None) for _ in range(S)]


@pytest.mark.parametrize("dim,f32", [(16, False), (64, False), (128, False), (130, False), (256, False), (520, False),
                                     (64, True), (128, True), (256, True)])
def test_long_chains_by_dim(torch_cuda, pb, oracle, dim, f32):
    _run(torch_cuda, pb, oracle, _one_id(LONG), 1, 8192, dim, ADAGRAD, f32=f32, cap=1 << 15)


@pytest.mark.parametrize("kind", [SGD, ADAGRAD, ADAGRAD_VW, ADAM])
def test_f32_dim128_every_optimizer(torch_cuda, pb, oracle, kind):
    _run(torch_cuda, pb, oracle, _one_id([2100, 300, 64, 40], S=2, B=4096), 2, 4096, 128, kind, f32=True, cap=1 << 14)


@pytest.mark.parametrize("kind", [ADAGRAD, ADAGRAD_VW, ADAM])
@pytest.mark.parametrize("groups", [[0, 0], [0, 1, 0]])
def test_shared_feature_group_one_gpu(torch_cuda, pb, oracle, groups, kind):
    """Slots of one feature group on one GPU, hot signs in each: every round finds its items' bits, and none is left
    set for the next batch.  (No SGD: _train's float64 check models one step per slot, not a row stepped per slot.)"""
    torch = torch_cuda
    S, B, dim = len(groups), 4096, 64
    rng = np.random.default_rng(11 + kind + S)
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, cap=1 << 15, groups=groups, optim_kw=OPT[kind], max_occ=S * B)
    touched = []
    for _ in range(3):
        t = _train(torch, s, ctx, w, oracle, pf, _one_id([2000, 1100, 300, 40], S=S, B=B)(rng), B, dim, rng, kind)
        touched.append(np.concatenate(t))
    _check(torch, s, w, [np.unique(np.concatenate(touched))])
