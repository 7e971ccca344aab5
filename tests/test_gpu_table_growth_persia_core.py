"""GPU: a persia_core Train job with dims 8, 32 and 128 under PERSIA_B200_GROW=1 equals the same job without it, bit for
bit: every pooled output, every entry, and the checkpoint files it dumps, before and after a load of that checkpoint
(checkpoint.DeviceLoader: pb_image_insert) into the cleared tables.  Each dim's growable table backs about what that
dim's resident signs need, far below `capacity`, while the eager tables back all of it."""
import os

import numpy as np
import pytest

from util import DEV

pytestmark = pytest.mark.gpu

CFG = {"feature_index_prefix_bit": 8,
       "slots_config": {"a": {"dim": 8}, "b": {"dim": 32}, "c": {"dim": 128}, "d": {"dim": 32, "sqrt_scaling": True}}}
KEYS = {"a": 200_000, "b": 60_000, "c": 6_000, "d": 30_000}  # each dim resident at its own scale
CAPACITY = 1 << 21
B, STEPS = 1024, 24


def _emb_files(d):
    out = {}
    for root, _, files in os.walk(d):
        for f in files:
            if f.endswith(".emb"):
                with open(os.path.join(root, f), "rb") as fh:
                    out[os.path.relpath(os.path.join(root, f), d)] = fh.read()
    return out


def _job(monkeypatch, tmp, grow):
    """The job: STEPS training steps (half through get_embedding_from_data, half through the Forward engine's
    dataflow), a dump, clear, a load of that dump, and a second dump.  Returns (outputs per step, entries after the
    run, the two dumps, [(dim, resident, mapped, capacity, occurrences of the dim per step)] per step)."""
    import torch
    import torch.utils.dlpack as dl

    from persia_b200 import persia_core as impl

    monkeypatch.setenv("PERSIA_B200_CAPACITY", str(CAPACITY))
    monkeypatch.delenv("PERSIA_B200_HBM_ROWS", raising=False)
    if grow:
        monkeypatch.setenv("PERSIA_B200_GROW", "1")
    else:
        monkeypatch.delenv("PERSIA_B200_GROW", raising=False)
    impl.reset()
    pc = impl.install()
    try:
        pc.set_embedding_config(CFG)
        ctx = pc.PersiaCommonContext(10, 0, 1, 0)
        opt = pc.optim.OptimizerBase()
        opt.init_sgd(0.05, 0.0)
        opt.apply()
        ctx.configure_embedding_parameter_servers(-0.01, 0.01, 1.0, True, 10.0)
        bwd = pc.backward.Backward(8)  # not launched: updates apply in this thread, in step order
        ch = pc.utils.PersiaBatchDataChannel(4)
        pc.nats.initialize_dataflow(1, ch.get_sender())
        fwd = pc.forward.Forward(8, True, 1)
        fwd.set_input_channel(ch.get_receiver())
        fwd.launch(2)
        rng = np.random.default_rng(17)
        outs, storage = [], []
        from persia_b200.persia_core import _S

        for step in range(STEPS):
            b = pc.data.PersiaBatch()
            b.add_id_type_feature_with_single_id(rng.integers(0, KEYS["a"], size=B, dtype=np.uint64), "a")
            b.add_id_type_feature([rng.integers(0, KEYS["b"], size=rng.integers(1, 4), dtype=np.uint64)
                                   for _ in range(B)], "b")
            b.add_id_type_feature_with_single_id(rng.integers(0, KEYS["c"], size=B, dtype=np.uint64), "c")
            b.add_id_type_feature([rng.integers(0, KEYS["d"], size=rng.integers(0, 3), dtype=np.uint64)
                                   for _ in range(B)], "d")
            b.add_label(np.zeros((B, 1), np.float32), np.dtype(np.float32), "y")
            b.converted_id_type_features2embedding_tensor(True)
            if step % 2 == 0:
                tb = ctx.get_embedding_from_data(b, 0)
            else:  # one batch in the engine at a time: its prefetch never runs beside the previous backward
                ctx.send_id_type_features_to_embedding_worker(b)
                ctx.send_non_id_type_features_to_nn_worker(b)
                tb = fwd.get_batch(10_000)
            embs = {t.name: t for t in (e.get_sum_embedding() for e in tb.consume_all_id_type_feature_embedding_tensors())}
            outs.append({n: dl.from_dlpack(t.dlpack).cpu().numpy().copy() for n, t in embs.items()})
            gb = tb.create_gradient_batch()
            keep = []
            for n in sorted(embs):
                g = torch.from_numpy((rng.standard_normal((B, CFG["slots_config"][n]["dim"])) * 1e-2)
                                     .astype(np.float16)).to(DEV)
                keep.append(g)
                gb.add_gradient(n, g.data_ptr(), list(g.shape), True, 1.0)
            torch.cuda.synchronize()
            bwd.update_id_type_feature_gradient_batched(gb)
            torch.cuda.synchronize()
            rows = []
            for dim in (8, 32, 128):
                sh = _S.groups[dim]["shard"]
                st = sh.storage_stats()
                assert st["refused_unmapped"] == 0
                occ = B if dim != 32 else 5 * B
                rows.append((dim, sh.counters()["admitted"], st["mapped_rows"], st["reserved_rows"], occ))
            storage.append(rows)
        groups = {d: _S.groups[d]["shard"] for d in (8, 32, 128)}
        entries = {}
        for d, sh in groups.items():
            signs, _ = sh.export_signs()
            ent, found = sh.get_entries(signs)
            assert bool(found.all())
            entries[d] = (signs.cpu().numpy(), ent.cpu().numpy())
        d1, d2 = os.path.join(tmp, "dump1"), os.path.join(tmp, "dump2")
        ctx.dump(d1)
        ctx.clear_embeddings()
        assert ctx.get_embedding_size() == [0, 0, 0]
        ctx.load(d1)
        ctx.dump(d2)
        return outs, entries, _emb_files(d1), _emb_files(d2), storage
    finally:
        impl.reset()


def test_persia_core_grow_equals_eager(monkeypatch, tmp_path):
    from persia_b200 import checkpoint as CK

    eager = _job(monkeypatch, str(tmp_path / "eager"), False)
    grow = _job(monkeypatch, str(tmp_path / "grow"), True)
    for step, (a, b) in enumerate(zip(eager[0], grow[0])):
        assert a.keys() == b.keys()
        for n in a:
            assert np.array_equal(a[n].view(np.uint16), b[n].view(np.uint16)), (step, n)
    for d in (8, 32, 128):
        assert np.array_equal(eager[1][d][0], grow[1][d][0])
        assert eager[1][d][1].tobytes() == grow[1][d][1].tobytes(), d
    assert eager[2] and eager[2].keys() == grow[2].keys()
    for f in eager[2]:
        assert eager[2][f] == grow[2][f], f  # the job's dump
        assert eager[3][f] == grow[3][f], f  # the dump after loading it into the cleared tables
        # the load brought back every entry of the dump (its list order follows the load's recency, not the job's)
        s1, _, e1 = CK.decode_list(grow[2][f])
        s2, _, e2 = CK.decode_list(grow[3][f])
        o1, o2 = np.argsort(s1, kind="stable"), np.argsort(s2, kind="stable")
        assert np.array_equal(s1[o1], s2[o2]) and np.asarray(e1)[o1].tobytes() == np.asarray(e2)[o2].tobytes(), f
    # storage: an eager table backs its whole capacity; a growable one about what its dim's resident signs need
    for rows in eager[4]:
        for dim, resident, mapped, reserved, occ in rows:
            assert mapped == reserved == CAPACITY
    mapped_last = {}
    for rows in grow[4]:
        for dim, resident, mapped, reserved, occ in rows:
            chunk = (2 << 20) // (4 * dim)  # rows of one 2 MB chunk (SGD: stride = dim)
            assert reserved == CAPACITY and resident <= mapped < CAPACITY, (dim, resident, mapped)
            assert mapped <= 2 * (resident + 3 * occ) + chunk, (dim, resident, mapped)
            mapped_last[dim] = (resident, mapped)
    # every dim backs its own entries only, each far below the capacity every eager table backs
    assert len({r for r, _ in mapped_last.values()}) == 3
    for dim, (resident, mapped) in mapped_last.items():
        assert mapped < CAPACITY // 8, (dim, resident, mapped)
