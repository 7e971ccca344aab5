"""GPU: what the local and sharded entry points of the C ABI share.  Each rejected input gets the same PB_ERR_* code
from both forms of a call, before the call launches anything; a sharded raw backward refuses a batch looked up in
another table, as the local one does; and a stage (pb_tier_stage) starts after every earlier call on its table,
whatever their streams.

The sharded forms run on rank 0 of two virtual ranks of one GPU (ShardedEmbeddingWorker.local_group).  Only inputs
that are refused before anything is launched are used, so a refused call leaves no peer waiting."""
import ctypes as C

import numpy as np
import pytest

from util import to_dev_ids

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
S, B, DIM, FIXED, MAX_IDS = 2, 64, 16, 2, 2


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def _sgd(N):
    return dict(kind=N.OPT_SGD, lr=0.1)


def _warm(torch, workers):
    for w in workers:  # table storage is allocated on first use, with a device-wide sync: not while a peer spins
        w.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()


class Form:
    """The summation and raw forward and backward of one form (`local`: pb_forward & co. on an EmbeddingShard;
    `sharded`: pb_*_sharded on rank 0 of two virtual ranks), called straight through the ABI so that every input
    reaches the library as given.  Each call returns the library's code."""

    def __init__(self, torch, oracle, form):
        from persia_b200 import native as N
        from persia_b200 import shard as SH
        from persia_b200.worker import ShardedEmbeddingWorker, ShardedRawWorker

        self.torch, self.lib, self.sharded = torch, N.load(), form == "sharded"
        pf, rpf = [oracle.index_prefix(0), oracle.index_prefix(1)], oracle.index_prefix(2)
        if self.sharded:
            self.ws = ShardedEmbeddingWorker.local_group(2, S, DIM, pf, 1 << 12, cap=S * B, optimizer=_sgd(N),
                                                         max_batch=B)
            self.rws = ShardedRawWorker.local_group(2, 1, DIM, [rpf], 1 << 12, cap=B * MAX_IDS, optimizer=_sgd(N),
                                                    max_batch=B, max_ids_per_sample=MAX_IDS,
                                                    shards=[w.shard for w in self.ws])
            _warm(torch, self.ws)
            w, rw = self.ws[0], self.rws[0]
            self.table, self.ctx, self.rctx = w.shard, w.ctx, rw.ctx
            self.st = C.c_void_p(w.stream.cuda_stream)
        else:
            self.table = SH.EmbeddingShard(DIM, 1 << 12, 0)
            self.table.set_optimizer(N.OPT_SGD, lr=0.1)
            self.table.configure()
            self.ctx = SH.BatchContext(S * B, S * B, pf)
            self.rctx = SH.BatchContext(B * MAX_IDS, B, [rpf])
            self.st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.ids = to_dev_ids(np.arange(S * B, dtype=np.uint64), DEV)
        self.out = torch.empty((S, B + 1, DIM), dtype=torch.float16, device=DEV)
        self.raw_out = [torch.empty(n, dtype=d, device=DEV) for n, d in
                        (((B * MAX_IDS + 1) * DIM, torch.float16), (B * FIXED, torch.int64),
                         (B * FIXED, torch.int64), (B, torch.int32), (2, torch.int32))]
        self.grads = torch.zeros((S, B, DIM), dtype=torch.float16, device=DEV)
        self.raw_grad = torch.zeros((B + 1, DIM), dtype=torch.float32, device=DEV)

    def forward(self, n_occ=S * B, off=None, batch=B, out_shift=0):
        off = (C.c_uint32 * (S + 1))(*(off if off is not None else [s * B for s in range(S + 1)]))
        args = (self.ids.data_ptr(), n_occ, None, off, batch, 1, self.out.data_ptr() + out_shift, self.st)
        if self.sharded:
            return self.lib.pb_forward_sharded(self.table.h, self.ctx.h, self.ws[0].h, *args, 0)
        return self.lib.pb_forward(self.table.h, self.ctx.h, *args)

    def forward_raw(self, n_occ=B, batch=B, out_shift=0):
        table, index, non_empty, num, counts = (t.data_ptr() for t in self.raw_out)
        args = (self.ids.data_ptr(), n_occ, None, batch, FIXED, 1, table + out_shift, index, non_empty, num, counts,
                self.st)
        if self.sharded:
            return self.lib.pb_forward_raw_sharded(self.table.h, self.rctx.h, self.rws[0].h, *args, 0)
        return self.lib.pb_forward_raw(self.table.h, self.rctx.h, *args)

    def backward(self, shift=0):
        ptrs = (C.c_void_p * S)(self.grads[0].data_ptr() + shift, self.grads[1].data_ptr())
        if self.sharded:
            return self.lib.pb_backward_sharded(self.table.h, self.ctx.h, self.ws[0].h, ptrs, 1, None, None, self.st, 0)
        return self.lib.pb_backward(self.table.h, self.ctx.h, ptrs, 1, None, None, self.st)

    def backward_raw(self, shift=0):
        g = self.raw_grad.data_ptr() + shift
        if self.sharded:
            return self.lib.pb_backward_raw_sharded(self.table.h, self.rctx.h, self.rws[0].h, g, 0, 1.0, None, self.st, 0)
        return self.lib.pb_backward_raw(self.table.h, self.rctx.h, g, 0, 1.0, None, self.st)

    def train(self):
        """A summation training forward on every rank: the context's batch is then pending."""
        from persia_b200.worker import ShardedEmbeddingWorker

        ids = self.ids
        if self.sharded:
            ShardedEmbeddingWorker.group_forward(self.ws, [ids, ids], B)
        else:
            self.ctx.forward(self.table, ids, [s * B for s in range(S + 1)], B)
        self.torch.cuda.synchronize()

    def train_raw(self):
        from persia_b200.worker import ShardedRawWorker

        ids = self.ids[:B]
        if self.sharded:
            ShardedRawWorker.group_forward_raw(self.rws, [ids, ids], B, FIXED)
        else:
            self.rctx.forward_raw(self.table, ids, B, FIXED)
        self.torch.cuda.synchronize()

    def close(self):
        self.torch.cuda.synchronize()
        for w in (self.rws + self.ws) if self.sharded else ():
            w.close()
        if not self.sharded:
            self.rctx.close()
            self.ctx.close()
            self.table.close()


# case -> (what is done before the call, the call, the code both forms return)
CASES = {
    "slot_offsets_short": (None, lambda f: f.forward(off=[0, B, 2 * B - 1]), "PB_ERR_INVALID"),
    "slot_offsets_descend": (None, lambda f: f.forward(off=[0, 2 * B + 1, 2 * B]), "PB_ERR_INVALID"),
    "batch_over_65535": (None, lambda f: f.forward(batch=65536), "PB_ERR_BATCH"),
    "batch_over_capacity": (None, lambda f: f.forward(n_occ=S * (B + 1), off=[0, B + 1, 2 * (B + 1)], batch=B + 1),
                            "PB_ERR_CAPACITY"),
    "no_row_offsets": (None, lambda f: f.forward(n_occ=S * B - 1, off=[0, B, 2 * B - 1]), "PB_ERR_INVALID"),
    "misaligned_output": (None, lambda f: f.forward(out_shift=2), "PB_ERR_INVALID"),
    "raw_batch_over_65535": (None, lambda f: f.forward_raw(batch=65536), "PB_ERR_BATCH"),
    "raw_batch_over_capacity": (None, lambda f: f.forward_raw(n_occ=B + 1, batch=B + 1), "PB_ERR_CAPACITY"),
    "raw_no_row_offsets": (None, lambda f: f.forward_raw(n_occ=B - 1), "PB_ERR_INVALID"),
    "raw_misaligned_output": (None, lambda f: f.forward_raw(out_shift=2), "PB_ERR_INVALID"),
    "backward_not_pending": (None, lambda f: f.backward(), "PB_ERR_STATE"),
    "backward_misaligned_gradient": (Form.train, lambda f: f.backward(shift=4), "PB_ERR_INVALID"),
    "raw_backward_not_pending": (None, lambda f: f.backward_raw(), "PB_ERR_STATE"),
    "raw_backward_misaligned_gradient": (Form.train_raw, lambda f: f.backward_raw(shift=4), "PB_ERR_INVALID"),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("form", ["local", "sharded"])
def test_rejected_input_same_code_in_both_forms(torch_cuda, oracle, form, case):
    from persia_b200 import native as N

    setup, call, code = CASES[case]
    f = Form(torch_cuda, oracle, form)
    try:
        if setup is not None:
            setup(f)
        launches = f.lib.pb_launch_count()
        assert call(f) == getattr(N, code), f.lib.pb_last_error()
        assert f.lib.pb_launch_count() == launches
    finally:
        f.close()


def test_sharded_raw_backward_refuses_another_table(torch_cuda, oracle):
    """A raw batch looked up through one table and exchange takes its gradients through those only: the sharded raw
    backward with another table and exchange of the same dim is refused, with nothing launched, and the batch still
    takes its gradients through its own."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedRawWorker

    torch = torch_cuda
    lib = N.load()
    pf = oracle.index_prefix(0)
    a, b = (ShardedRawWorker.local_group(1, 1, DIM, [pf], 1 << 12, cap=B, optimizer=_sgd(N), max_batch=B)[0]
            for _ in range(2))
    try:
        _warm(torch, [a, b])
        _, _, _, _, counts = a.forward_raw(to_dev_ids(np.arange(B, dtype=np.uint64), DEV), B, FIXED)
        g = torch.zeros((int(counts[0]), DIM), dtype=torch.float32, device=DEV)
        torch.cuda.synchronize()
        launches = lib.pb_launch_count()
        rc = lib.pb_backward_raw_sharded(b.shard.h, a.ctx.h, b.h, g.data_ptr(), 0, 1.0, None,
                                         C.c_void_p(b.stream.cuda_stream), 0)
        assert rc == N.PB_ERR_INVALID, lib.pb_last_error()
        assert lib.pb_launch_count() == launches
        a.backward_raw(g)
        torch.cuda.synchronize()
    finally:
        torch.cuda.synchronize()
        a.close()
        b.close()


def test_stage_waits_for_a_forward_on_another_stream(torch_cuda, oracle):
    """A stage starts after every earlier call on its table: a training forward still running on one stream (behind a
    sleep) and a backward already finished on another come before a stage captured on a third, so the capture fails
    with PB_ERR_STATE rather than record a dependency on work outside it.  Outside a capture the same stage waits."""
    from persia_b200 import native as N
    from persia_b200 import shard as SH

    torch = torch_cuda
    pf = [oracle.index_prefix(0), oracle.index_prefix(1)]
    off = [s * B for s in range(S + 1)]
    s = SH.EmbeddingShard(DIM, 1 << 10, 0, tier_rows=1 << 12)
    s.set_optimizer(N.OPT_SGD, lr=0.1)
    s.configure()
    ctx_a, ctx_b = SH.BatchContext(S * B, S * B, pf), SH.BatchContext(S * B, S * B, pf)
    ids_a = to_dev_ids(np.arange(S * B, dtype=np.uint64), DEV)
    ids_b = to_dev_ids(np.arange(S * B, 2 * S * B, dtype=np.uint64), DEV)
    nxt = to_dev_ids(np.arange(2 * S * B, 3 * S * B, dtype=np.uint64), DEV)
    grads = [torch.zeros((B, DIM), dtype=torch.float16, device=DEV) for _ in range(S)]
    s1, s2, s3 = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    try:
        # every kernel below runs once first: a kernel's first launch loads its module, which may wait for the whole
        # device, the sleep included
        ctx_a.forward(s, ids_a, off, B, training=True)
        ctx_a.backward(s, grads)
        s.stage(nxt, off, pf)
        ctx_a.forward(s, ids_a, off, B, training=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(s1):
            torch.cuda._sleep(200_000_000)
            ctx_b.forward(s, ids_b, off, B, training=True)
        with torch.cuda.stream(s2):
            ctx_a.backward(s, grads)
        s2.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s3):
            graph.capture_begin()
            try:
                with pytest.raises(N.PersiaB200Error) as ei:
                    s.stage(nxt, off, pf)
            finally:
                graph.capture_end()
        assert ei.value.code == N.PB_ERR_STATE, ei.value
        with torch.cuda.stream(s3):
            s.stage(nxt, off, pf)
        with torch.cuda.stream(s1):
            ctx_b.backward(s, grads)
        torch.cuda.synchronize()
    finally:
        torch.cuda.synchronize()
        ctx_a.close()
        ctx_b.close()
        s.close()
