"""GPU: the exchange checks of pb_backward_sharded.  An exchange sized for another dim is refused before anything is
enqueued, as pb_backward_raw_sharded refuses one (test_gpu_worker_raw.py::test_raw_sharded_abi_refusals): the reduces
would otherwise write the gradients into a receive area laid out for the other dim."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from util import to_dev_ids  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def test_backward_sharded_refuses_an_exchange_of_another_dim(torch_cuda, oracle):
    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    lib = N.load()
    S, B, dim = 2, 16, 16
    pf = [oracle.index_prefix(i) for i in range(S)]
    x = W.local_group(1, S, dim, pf, 1 << 10, cap=S * B, optimizer=dict(kind=N.OPT_SGD, lr=0.1), max_batch=B)[0]
    other = W.local_group(1, S, 32, pf, 1 << 10, cap=S * B, optimizer=dict(kind=N.OPT_SGD, lr=0.1), max_batch=B)[0]
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pf], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1))
    g = (np.random.default_rng(0).standard_normal((S, B, dim)) * 0.1).astype(np.float16)
    dg = [torch.from_numpy(g[i]).to(DEV) for i in range(S)]
    ptrs, is_f16, _ = SH._slot_grads(dg, S)
    st = C.c_void_p(x.stream.cuda_stream)

    def bwd(xchg):
        return lib.pb_backward_sharded(x.shard.h, x.ctx.h, xchg, ptrs, int(is_f16), None, None, st, 0)

    torch.cuda.synchronize()
    launches = lib.pb_launch_count()
    assert bwd(other.h) == N.PB_ERR_STATE  # no batch pending: refused for that first, as before the exchange checks
    assert lib.pb_launch_count() == launches

    ids = np.arange(S * B, dtype=np.uint64) % B
    out = x.forward(to_dev_ids(ids, DEV), B)
    want, octx = w.forward(ids, np.arange(S * B + 1, dtype=np.uint32), B, training=True)
    torch.cuda.synchronize()
    for i in range(S):
        assert out[i].cpu().numpy().tobytes() == want[i].tobytes()
    signs = np.concatenate([oracle.add_prefix(np.arange(B, dtype=np.uint64), 8, p) for p in pf])
    before = x.shard.get_entries(to_dev_ids(signs, DEV))[0].cpu().numpy()
    n_before = len(x.shard)
    torch.cuda.synchronize()
    launches = lib.pb_launch_count()
    assert bwd(other.h) == N.PB_ERR_INVALID
    assert "another embedding dim" in lib.pb_last_error().decode()
    torch.cuda.synchronize()
    assert lib.pb_launch_count() == launches
    assert len(x.shard) == n_before
    assert x.shard.get_entries(to_dev_ids(signs, DEV))[0].cpu().numpy().tobytes() == before.tobytes()

    # the pending batch still takes its gradient, as the oracle applies it; a second backward is "backward_ref_id not found"
    x.backward(dg)
    w.backward(octx, [g[i] for i in range(S)])
    got = x.shard.get_entries(to_dev_ids(signs, DEV))[0].cpu().numpy()
    for k, sign in enumerate(signs):
        ref = w.get_entry(int(sign))
        assert ref is not None and got[k].tobytes() == ref.tobytes(), k
    assert got.tobytes() != before.tobytes()
    with pytest.raises(N.PersiaB200Error):
        x.backward(dg)
    assert x.status() == (False, False)
    x.close()
    other.close()
