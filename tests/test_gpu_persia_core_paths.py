"""GPU: persia_core's three placements of a batch's lookups (a pooled context on one GPU, the collective workers on R
GPUs, the remote readers for lookups that do not train on R GPUs), driven through the public surface as
tests/test_gpu_persia_core.py drives it, against the oracle's embedding worker."""
import os
import socket
import sys
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu

HYPER = (-0.01, 0.01, 1.0, True, 10.0)


def _surface(cfg, replica_size=1):
    from persia_b200 import persia_core as impl

    impl.reset()
    pc = impl.install()
    pc.set_embedding_config(cfg)
    return impl, pc, pc.PersiaCommonContext(10, 0, replica_size, 0)


def _register(pc, ctx):
    opt = pc.optim.OptimizerBase()
    opt.init_sgd(0.05, 0.0)
    opt.apply()
    ctx.configure_embedding_parameter_servers(*HYPER)


def _oracle_worker(oracle, slots, n_ps=1):
    w = oracle.Worker(slots, n_ps=n_ps)
    w.configure(*HYPER)
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.05, wd=0.0))
    return w


def _csr(lils, B):
    rows = []
    for v in lils:
        rows.extend([np.array([x], np.uint64) for x in v] if isinstance(v, np.ndarray) else v)
    off = np.zeros(len(rows) + 1, np.uint32)
    off[1:] = np.cumsum([len(r) for r in rows])
    return (np.concatenate(rows) if rows else np.zeros(0, np.uint64)), off


def _batch(pc, lil, requires_grad):
    b = pc.data.PersiaBatch()
    for name, v in lil.items():
        if isinstance(v, np.ndarray):
            b.add_id_type_feature_with_single_id(v, name)
        else:
            b.add_id_type_feature(v, name)
    B = len(next(iter(lil.values())))
    b.add_label(np.zeros((B, 1), np.float32), np.dtype(np.float32), "y")
    b.converted_id_type_features2embedding_tensor(requires_grad)
    return b


def test_refused_raw_forward_releases_the_group_lock():
    """An inference forward of a raw slot before an optimizer is registered raises; the group's lock is free after it,
    so the other threads that take it (backward workers, dumps, loads, flushes) do not block for ever."""
    impl, pc, ctx = _surface({"slots_config": {"seq": {"dim": 16, "embedding_summation": False}}})
    try:
        B = 4
        lil = {"seq": [np.array([1, 2, 3], np.uint64)] * B}
        with pytest.raises(RuntimeError, match="optimizer not registered"):
            ctx.get_embedding_from_data(_batch(pc, lil, False), 0)
        lock = impl._S.groups[16]["lock"]
        got = []

        def take():
            ok = lock.acquire(timeout=5)
            got.append(ok)
            if ok:
                lock.release()

        t = threading.Thread(target=take)
        t.start()
        t.join()
        assert got == [True]
        assert len(impl._S.groups[16]["ctx"][("raw", "seq")]) == 1  # (the refused forward gave its context back)
    finally:
        impl.reset()


def test_pooled_context_is_not_reused_for_more_rows(oracle):
    """One summation slot, inference: a ragged batch of 8 samples x 200 ids makes a pooled context of 3200 occurrences
    and 1024 output rows; a later batch of 2048 samples of one id each has fewer ids but more rows, so it needs a context
    of its own.  Its outputs equal the oracle's bit for bit.  Then 8 samples x 1250 ids (more ids than that context
    holds, few rows): a context made for it also covers the pool's top, so batches that keep alternating these shapes
    reuse it and the pool stops growing."""
    import torch.utils.dlpack as dl

    impl, pc, ctx = _surface({"slots_config": {"s": {"dim": 16}}})
    try:
        _register(pc, ctx)
        prefix = impl._S.by_name["s"].index_prefix
        card = 1000
        signs = oracle.add_prefix(np.arange(card, dtype=np.uint64), 8, prefix)
        rng = np.random.default_rng(5)
        ent = (rng.standard_normal((card, 16)) * 0.05).astype(np.float32)
        ctx.set_embedding([(int(s), ent[k], np.zeros(0, np.float32)) for k, s in enumerate(signs)])
        w = _oracle_worker(oracle, [oracle.SlotCfg(16, prefix=prefix)])
        w.set_embedding(signs, ent, 16)
        pooled = []
        for _ in range(3):
            for B, per in ((8, 200), (2048, 1), (8, 1250)):
                lil = (rng.integers(0, card, size=B, dtype=np.uint64) if per == 1 else
                       [rng.integers(0, card, size=per, dtype=np.uint64) for _ in range(B)])
                tb = ctx.get_embedding_from_data(_batch(pc, {"s": lil}, False), 0)
                (e,) = tb.consume_all_id_type_feature_embedding_tensors()
                got = dl.from_dlpack(e.get_sum_embedding().dlpack).cpu().numpy()
                ids, off = _csr([lil], B)
                (want,), _ = w.forward(ids, off, B, training=False, keep_ctx=False)
                if per == 1:
                    assert got.tobytes() == want.tobytes()
                else:
                    assert np.abs(got.astype(np.float32) - want.astype(np.float32)).max() <= 2e-5
            pooled.append(len(impl._S.groups[16]["ctx"][("s",)]))
        assert pooled == [3, 3, 3]
    finally:
        impl.reset()


# The R-GPU placements on one GPU: one process, a gloo process group of world size 1, replica_size 2.  The workers are
# then R = 1 over plain device memory, and the remote readers probe this rank's own table.
PATH_CFG = {
    "feature_index_prefix_bit": 8,
    "slots_config": {
        "user": {"dim": 16},
        "seq": {"dim": 32, "embedding_summation": False, "sample_fixed_size": 4},
        "item": {"dim": 16, "sqrt_scaling": True},
        "hs": {"dim": 16, "hash_stack_config": {"hash_stack_rounds": 2, "embedding_size": 1000}},
        "fa": {"dim": 32},
        "fb": {"dim": 32},
    },
    "feature_groups": {"fg": ["fa", "fb"]},
}
CARD = {"user": 500, "seq": 60, "item": 40, "hs": 100000, "fa": 30, "fb": 30}
KEYS = dict(CARD, hs=2000)  # resident key space per slot (hash stack: rounds x embedding_size)
SINGLE = ("user", "hs", "fa")


def _path_batch(rng, B):
    lil = {}
    for n in PATH_CFG["slots_config"]:
        if n in SINGLE:
            lil[n] = rng.integers(0, CARD[n], size=B, dtype=np.uint64)
        else:
            lil[n] = [rng.integers(0, CARD[n], size=rng.integers(0, 6), dtype=np.uint64) for _ in range(B)]
    return lil


@pytest.fixture()
def one_rank():
    import torch
    import torch.distributed as dist

    torch.cuda.set_device(0)
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=0, world_size=1)
    try:
        yield
    finally:
        dist.destroy_process_group()


def test_r_gpu_placements_on_one_rank(oracle, one_rank):
    """Training batches take the collective workers and the lookup that does not train takes the remote readers, with
    two dims, a ragged slot, a hash-stacked slot, two slots of one feature group and a raw slot (one gradient skipped).
    Outputs and entries equal the oracle's with one parameter server.  Every worker starts at cap 8, and its first
    step's agreement gives it the cap its own prepared need grows to."""
    import torch
    import torch.utils.dlpack as dl

    from persia_b200.worker import ShardedEmbeddingWorker as W
    from util import to_dev_ids

    impl, pc, ctx = _surface(PATH_CFG, replica_size=2)
    agree, first = impl._agree_and_resize, []  # first: the first step's (worker, its prepare's (need, rows_f32))

    def record(plan, dev):
        if not first:
            first.extend((wk, need) for _, wk, need in plan)
        return agree(plan, dev)

    impl._agree_and_resize = record
    try:
        _register(pc, ctx)  # (the process group is up: the tables are exported live here)
        S = impl._S
        by = S.by_name
        sums = {d: [n for n in PATH_CFG["slots_config"] if by[n].dim == d and by[n].embedding_summation] for d in (16, 32)}
        ws = {d: _oracle_worker(oracle, [oracle.SlotCfg(d, sqrt_scaling=by[n].sqrt_scaling, prefix=by[n].index_prefix,
                                                        hs_rounds=by[n].hash_stack_rounds,
                                                        hs_size=by[n].hash_stack_embedding_size) for n in names])
              for d, names in sums.items()}
        w_raw = _oracle_worker(oracle, [oracle.SlotCfg(32, summation=False, sample_fixed_size=4,
                                                       prefix=by["seq"].index_prefix)])
        bwd = pc.backward.Backward(8)
        rng = np.random.default_rng(17)
        B, fixed, scale = 64, 4, 128.0

        def close(n, got, want):
            if n in SINGLE and n != "hs":
                assert got.tobytes() == want.tobytes(), n
            else:
                assert np.abs(got.astype(np.float32) - want.astype(np.float32)).max() <= 2e-5, n

        for step in range(3):
            lil = _path_batch(rng, B)
            tb = ctx.get_embedding_from_data(_batch(pc, lil, True), 0)
            embs = dict(zip(lil, tb.consume_all_id_type_feature_embedding_tensors()))
            keep, xs = [], {}
            for n, e in embs.items():
                if n == "seq":
                    continue
                t = e.get_sum_embedding()
                keep.append(t)
                xs[n] = dl.from_dlpack(t.dlpack)
                xs[n].requires_grad = True
            octx = {}
            for d, names in sums.items():
                ids, off = _csr([lil[n] for n in names], B)
                want, octx[d] = ws[d].forward(ids, off, B, training=True)
                for n, wv in zip(names, want):
                    close(n, xs[n].detach().cpu().numpy(), wv)
            raw, index, non_empty, num = embs["seq"].get_raw_embedding()
            keep += [raw, index, non_empty]
            table, index_t, ne_t = (dl.from_dlpack(x.dlpack) for x in (raw, index, non_empty))
            ids, off = _csr([lil["seq"]], B)
            wt, wi, wne, wnum, rctx = w_raw.forward_raw(0, ids, off, B, training=True)
            assert table.cpu().numpy().tobytes() == wt.tobytes()
            np.testing.assert_array_equal(index_t.cpu().numpy(), wi)
            np.testing.assert_array_equal(ne_t.cpu().numpy(), wne)
            assert num == wnum.tolist()
            # a loss over every output (persia/ctx.py builds the raw slot's [B, fixed, dim] input like this)
            sel = table.index_select(0, index_t.view(-1))
            sel.requires_grad = True
            loss = sum((x.float() * (i + 1)).sum() for i, x in enumerate(xs.values()))
            loss = (loss + sel.float().sum() * 0.5) * scale * 1e-3
            loss.backward()
            gb = tb.create_gradient_batch()
            for n, x in xs.items():
                gb.add_gradient(n, x.grad.data_ptr(), list(x.grad.shape), True, scale)
            skip_raw = step == 1
            if skip_raw:
                gb.add_skipped_gradient("seq")
            else:
                grad = torch.zeros_like(table, dtype=torch.float32)
                nz = sel.grad.index_select(0, ne_t.view(-1)).float()
                grad.index_add_(0, index_t.view(-1)[ne_t.view(-1)], nz)
                grad = grad[1:, :].contiguous()
                gb.add_gradient("seq", grad.data_ptr(), list(grad.shape), False, scale)
            torch.cuda.synchronize()
            bwd.update_id_type_feature_gradient_batched(gb)
            for d, names in sums.items():
                ws[d].backward(octx[d], [xs[n].grad.cpu().numpy() for n in names], scale=[scale] * len(names))
            if skip_raw:
                w_raw.backward_raw(0, rctx, None, skip=True)
            else:
                w_raw.backward_raw(0, rctx, grad.cpu().numpy(), scale=scale)
            if step == 0:  # the raw slot, the dim-16 chunk (with the hash-stacked slot) and the dim-32 chunk
                assert sorted((wk.dim, wk.S) for wk, _ in first) == [(16, 3), (32, 1), (32, 2)]
                for wk, (need, f32) in first:
                    assert need > 8 and (wk.cap, wk.rows_f32) == (W.grown_cap(need, 8), f32), (wk.dim, wk.S, need)
        torch.cuda.synchronize()
        # the path the training batches took: the collective workers, no pooled context
        for d in (16, 32):
            g = S.groups[d]
            assert len(g["workers"]) == 1 and g["ctx"] == {}
        assert set(S.groups[32]["raw_workers"]) == {"seq"}
        # the entries, bit for bit
        for d in (16, 32):
            sh = S.groups[d]["shard"]
            for n in sums[d] + (["seq"] if d == 32 else []):
                w = w_raw if n == "seq" else ws[d]
                signs = oracle.add_prefix(np.arange(KEYS[n], dtype=np.uint64), 8, by[n].index_prefix)
                ent, found = sh.get_entries(to_dev_ids(signs, "cuda:0"))
                ent, found = ent.cpu().numpy(), found.cpu().numpy()
                for k, s in enumerate(signs):
                    ref = w.get_entry(int(s))
                    assert (ref is not None) == bool(found[k]), (n, k)
                    if ref is not None:
                        assert ent[k].tobytes() == ref.tobytes(), (n, k)
        # a lookup that does not train: this rank's remote readers, no collective and no pooled context
        assert S.remote is not None and all(not rd._ctxs for rd in S.remote.values())
        lil = _path_batch(rng, B)
        tb = ctx.get_embedding_from_data(_batch(pc, lil, False), 0)
        embs = dict(zip(lil, tb.consume_all_id_type_feature_embedding_tensors()))
        assert all(rd._ctxs for rd in S.remote.values())
        assert all(S.groups[d]["ctx"] == {} for d in (16, 32))
        for d, names in sums.items():
            ids, off = _csr([lil[n] for n in names], B)
            want, _ = ws[d].forward(ids, off, B, training=False, keep_ctx=False)
            for n, wv in zip(names, want):
                close(n, embs[n].get_sum_embedding().numpy(), wv)
        table, index, _, num = embs["seq"].get_raw_embedding()
        table, index = table.numpy(), index.numpy()
        ids, off = _csr([lil["seq"]], B)
        wt, wi, _, wnum, _ = w_raw.forward_raw(0, ids, off, B, training=False, keep_ctx=False)
        assert num == wnum.tolist()
        assert ((index != 0) == (wi != 0)).all()
        held = wi != 0  # the row at every index position, whatever numbering either side chose
        assert table[index[held]].tobytes() == wt[wi[held]].tobytes()
    finally:
        impl._agree_and_resize = agree
        impl.reset()
