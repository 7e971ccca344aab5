"""GPU: the hot-sign reduce (k_reduce_hot) at every geometry its launcher chooses (tests/hot_geometry_cases.py; the
CPU test tests/test_hot_geometry_classes.py keeps that list complete), against the CPU oracle bit for bit in
exact-rsqrt mode and, for SGD, against a float64 computation of the reference operation.

The item counts come from the geometry pb_hot_geometry returns (PW producer warps, parts of R1 rows, ring slots of R
rows, S slots), one item each in a slot of B = 8192 samples:
  33                      the smallest hot item
  PW*R1, PW*R1 + 1        the last window of R1-row chunks, and the first cut into larger ones
  2*PW*R1, 2*PW*R1 + 1    the same for chunks of two parts (where 2*R1 <= R)
  S*R + 1                 the chunks wrap the ring once
  2*S*R + 3               twice (the barrier parity flips back), ending on a tail that is not a multiple of four
  a multiple of R         whole chunks only
Counts of 32 or less are warm items and are left out.  A second slot holds 200 items of 33..40 occurrences: blocks take
several items in a row, carrying the ring position across items and column passes, and with the context sized to the
batch most of them come with occurrence lists instead of bitmaps."""
import numpy as np
import pytest

from hot_geometry_cases import ONE_ID_CASES, RAGGED_CASES, SEND_CASES, WINDOW_CASES
from test_gpu_reduce_boundaries import SGD, WARM_MAX, _run, _window_items
from test_gpu_worker import _check_rows, _group
from util import batch_with_multiplicities, full_row_off, ragged_with_multiplicities, to_dev_ids

pytestmark = pytest.mark.gpu

B = 8192
MANY = [33 + k % 8 for k in range(200)]
KIND_NAMES = {0: "sgd", 1: "adagrad", 2: "adagrad_vw", 3: "adam"}


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


def _hot_counts(g):
    PW, R1, R, S = g["PW"], g["R1"], g["R"], g["S"]
    counts = [33, PW * R1, PW * R1 + 1]
    if 2 * R1 <= R:
        counts += [2 * PW * R1, 2 * PW * R1 + 1]
    counts += [S * R + 1, 2 * S * R + 3, R * (WARM_MAX // R + 2)]
    return [c for c in counts if c > WARM_MAX]


def _name(dim, f16):
    return f"{'f16' if f16 else 'f32'}-{dim}"


CLASS_RUNS = [(d, f16, k) for d, f16, kinds in ONE_ID_CASES for k in kinds]


@pytest.mark.parametrize("dim,f16,kind", CLASS_RUNS, ids=[f"{_name(d, f)}-{KIND_NAMES[k]}" for d, f, k in CLASS_RUNS])
def test_every_geometry_class(torch_cuda, pb, oracle, dim, f16, kind):
    counts = _hot_counts(pb.hot_geometry(dim, f16))
    _run(torch_cuda, pb, oracle,
         lambda rng: [(batch_with_multiplicities(rng, B, counts), None), (batch_with_multiplicities(rng, B, MANY), None)],
         2, B, dim, kind, steps=1, f32=not f16, cap=1 << 14, max_occ=2 * B)


@pytest.mark.parametrize("dim,f16", RAGGED_CASES, ids=[_name(d, f) for d, f in RAGGED_CASES])
def test_ragged_sqrt_and_scale(torch_cuda, pb, oracle, dim, f16):
    """The dims whose one-id batches take the producers' lean loop, with several ids per sample, sqrt scaling and a loss
    scale: the general loop.  2..3 ids per sample keep both slots inside one window."""
    counts = _hot_counts(pb.hot_geometry(dim, f16, ragged=True))
    n = 2700

    def make(rng):
        return [ragged_with_multiplicities(rng, n, counts, max_ids=3, min_ids=2),
                ragged_with_multiplicities(rng, n, MANY[:140], max_ids=3, min_ids=2)]

    _run(torch_cuda, pb, oracle, make, 2, n, dim, SGD, steps=1, f32=not f16, scale=[3.0, 128.0], sqrt=[True, False],
         cap=1 << 14, max_occ=2 * 3 * n)


@pytest.mark.parametrize("dim,f16", WINDOW_CASES, ids=[_name(d, f) for d, f in WINDOW_CASES])
def test_two_windows(torch_cuda, pb, oracle, dim, f16):
    """A slot of 9000 samples: items across the HOT_WIN boundary and in the second window only, beside the geometry's
    counts."""
    n = 9000
    counts, spans = _window_items(n)
    counts = counts + _hot_counts(pb.hot_geometry(dim, f16))
    _run(torch_cuda, pb, oracle, lambda rng: [(batch_with_multiplicities(rng, n, counts, spans), None)], 1, n, dim, SGD,
         steps=1, f32=not f16, cap=1 << 14, max_occ=n)


@pytest.mark.parametrize("dim,f16", SEND_CASES, ids=[_name(d, f) for d, f in SEND_CASES])
def test_sharded_requester(torch_cuda, pb, oracle, dim, f16):
    """The requester's instantiation (SEND): two virtual ranks, the reduced gradients go to the owners' receive areas and
    the owners apply them (Adagrad)."""
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, S, n = 2, 2, 4096
    counts = _hot_counts(pb.hot_geometry(dim, f16))
    rng = np.random.default_rng(2 * dim + f16)
    ws, w, pf = _group(torch, oracle, R, S, dim, oracle.ADAGRAD, n)
    outs = [torch.empty((S, n, dim), dtype=torch.float16, device="cuda:0") for _ in range(R)]
    seen = set()
    for step in range(2):
        ids = [np.concatenate([batch_with_multiplicities(rng, n, counts), batch_with_multiplicities(rng, n, MANY[:100])])
               for _ in range(R)]
        torch.cuda.synchronize()
        W.group_forward(ws, [to_dev_ids(x, "cuda:0") for x in ids], n, training=True, outs=outs)
        torch.cuda.synchronize()
        octx = []
        for r in range(R):
            want, c = w.forward(ids[r], full_row_off(S, n), n, training=True)
            octx.append(c)
            got = outs[r].cpu().numpy()
            for i in range(S):
                np.testing.assert_array_equal(got[i].view(np.uint16), want[i].view(np.uint16))
                seen.update(w.ctx_signs(c, i).tolist())
        g = (rng.standard_normal((R, S, n, dim)) * 1e-2).astype(np.float16 if f16 else np.float32)
        dg = [[torch.from_numpy(g[r, i]).to("cuda:0") for i in range(S)] for r in range(R)]
        torch.cuda.synchronize()
        W.group_backward(ws, dg)
        torch.cuda.synchronize()
        for r in range(R):
            w.backward(octx[r], [g[r, i] for i in range(S)])
    _check_rows(torch, oracle, ws, w, seen, R)
