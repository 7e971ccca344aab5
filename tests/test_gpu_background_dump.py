"""GPU: background embedding dumps (persia_b200/checkpoint.py BackgroundDumper over pb_table_dump_part, pb_dump.cu).

Every part file must be byte for byte the reference's list encoding (checkpoint.encode_list) of the table's entries
whose sign falls in that part, in export_signs' order, as the table held them at one point of its call order; the
synchronous dump, now encoded on the device (pb_dump_nodes), keeps its files byte for byte."""
import os
import threading

import numpy as np
import pytest

from util import full_row_off, make_batch, to_dev_ids

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ODD = np.array([2**64 - 1, 2**64 - 2, 2**64 - 3], np.uint64)  # signs equal to the index's markers: reserved cells


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def _state(sh):
    """(signs u64, entries f32 [n, L]) of the table now, in export order."""
    signs, _ = sh.export_signs()
    ent, found = sh.get_entries(signs)
    assert bool(found.all())
    return signs.cpu().numpy().view(np.uint64), ent.cpu().numpy()


def _part_bytes(CK, state, dim, n_parts, k):
    s, e = state
    m = CK.part_of(s, n_parts) == np.uint64(k)
    return CK.encode_list(s[m], e[m], dim)


def _read(path):
    with open(path, "rb") as f:
        return f.read()


def _filled_shard(torch, pb, N, dim, kind, rng, n=700, capacity=4096, tier_rows=0, odd=True):
    sh = pb.EmbeddingShard(dim, capacity, 0, tier_rows=tier_rows)
    sh.set_optimizer(kind, lr=0.05, initialization=0.01)
    sh.configure()
    L = sh.entry_len
    signs = np.unique(rng.integers(1, 2**63, size=n, dtype=np.uint64) | (rng.integers(0, 2, size=n, dtype=np.uint64) << 63))
    if odd:
        signs = np.concatenate([signs, ODD])
    ent = rng.standard_normal((signs.size, L)).astype(np.float32)
    sh.set_entries(to_dev_ids(signs, DEV), torch.from_numpy(ent).to(DEV))
    for k in range(3):  # three requests of growing recency over subsets: the order mixes requests and sign order
        pick = signs[rng.random(signs.size) < 0.3]
        if pick.size:
            sh.lookup(to_dev_ids(pick, DEV), training=True)
    return sh


KINDS = [0, 1, 2, 3]  # SGD, Adagrad, Adagrad (vector-wise), Adam


@pytest.mark.parametrize("n_parts", [1, 3, 100])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("dim", [1, 12, 64, 128, 130])
def test_quiescent_parts_equal_the_export(torch_cuda, tmp_path, dim, kind, n_parts):
    torch = torch_cuda
    from persia_b200 import checkpoint as CK
    from persia_b200 import native as N
    from persia_b200 import shard as pb

    rng = np.random.default_rng(dim * 10 + kind)
    sh = _filled_shard(torch, pb, N, dim, kind, rng)
    state = _state(sh)
    d = CK.BackgroundDumper(str(tmp_path / "bg"), [sh], n_parts=n_parts).start()
    d.wait()
    assert d.status() == ("Idle", 1.0)
    files = sorted(os.listdir(tmp_path / "bg" / "s0"))
    assert files == sorted([CK.DONE_FILE] + [CK.part_file(0, 0, n_parts, k) for k in range(n_parts)])
    union = []
    for k in range(n_parts):
        got = _read(tmp_path / "bg" / "s0" / CK.part_file(0, 0, n_parts, k))
        assert got == _part_bytes(CK, state, dim, n_parts, k), k
        union.append(CK.decode_list(got)[0])
    # the synchronous dump: one file, the whole export, byte for byte; the parts hold exactly its signs
    CK.dump_shards(str(tmp_path / "sync"), [sh])
    whole = _read(tmp_path / "sync" / "s0" / "replica_0_shard_0.emb")
    assert whole == CK.encode_list(state[0], state[1], dim)
    np.testing.assert_array_equal(np.sort(np.concatenate(union)), np.sort(state[0]))
    assert (tmp_path / "bg" / CK.DONE_FILE).is_file()
    sh.close()


def test_empty_table_and_a_table_with_a_host_tier(torch_cuda, tmp_path):
    torch = torch_cuda
    from persia_b200 import checkpoint as CK
    from persia_b200 import native as N
    from persia_b200 import shard as pb

    empty = pb.EmbeddingShard(16, 1024, 0)
    empty.set_optimizer(N.OPT_ADAGRAD)
    empty.configure()
    rng = np.random.default_rng(1)
    tiered = _filled_shard(torch, pb, N, 24, N.OPT_ADAM, rng, n=1500, capacity=512, tier_rows=4096)
    assert tiered.tier_stats()["host_rows"] > 0  # the entries beyond the HBM rows live in the tier
    states = [_state(empty), _state(tiered)]
    assert states[0][0].size == 0
    n_parts = 5
    CK.BackgroundDumper(str(tmp_path), [empty, tiered], n_parts=n_parts).start().wait()
    for d, (sh, st) in enumerate(zip([empty, tiered], states)):
        for k in range(n_parts):
            got = _read(tmp_path / "s0" / CK.part_file(0, d, n_parts, k))
            assert got == _part_bytes(CK, st, sh.dim, n_parts, k), (d, k)
    assert _read(tmp_path / "s0" / CK.part_file(0, 0, n_parts, 0)) == CK.encode_list(np.zeros(0, np.uint64),
                                                                                      np.zeros((0, 32), np.float32), 16)
    CK.dump_shards(str(tmp_path / "sync"), [empty, tiered])
    for i, (sh, st) in enumerate(zip([empty, tiered], states)):
        assert _read(tmp_path / "sync" / "s0" / f"replica_0_shard_{i}.emb") == CK.encode_list(st[0], st[1], sh.dim)
    # the synchronous dump's slices: a list staged in several pieces gives the same file
    CK.dump_shards(str(tmp_path / "sliced"), [tiered], chunk=97)
    assert _read(tmp_path / "sliced" / "s0" / "replica_0_shard_0.emb") == CK.encode_list(states[1][0], states[1][1], 24)
    # the checkpoint loads back (load_shards reads every .emb of the directory)
    fresh = pb.EmbeddingShard(24, 4096, 0)
    fresh.set_optimizer(N.OPT_ADAM)
    fresh.configure()
    fresh16 = pb.EmbeddingShard(16, 1024, 0)
    fresh16.set_optimizer(N.OPT_ADAGRAD)
    fresh16.configure()
    assert CK.load_shards(str(tmp_path), {24: fresh, 16: fresh16}) == states[1][0].size
    ent, found = fresh.get_entries(to_dev_ids(states[1][0], DEV))
    assert bool(found.all())
    np.testing.assert_array_equal(ent.cpu().numpy(), states[1][1])


def test_a_part_larger_than_its_buffer_is_issued_again(torch_cuda, tmp_path):
    torch = torch_cuda
    from persia_b200 import checkpoint as CK
    from persia_b200 import native as N
    from persia_b200 import shard as pb

    sh = _filled_shard(torch, pb, N, 32, N.OPT_ADAGRAD, np.random.default_rng(2), n=900)
    state = _state(sh)
    d = CK.BackgroundDumper(str(tmp_path), [sh], n_parts=3, part_bytes=256)  # far too small: every part grows it
    d.start().wait()
    for k in range(3):
        assert _read(tmp_path / "s0" / CK.part_file(0, 0, 3, k)) == _part_bytes(CK, state, 32, 3, k)


def test_parts_between_training_steps_are_snapshots(torch_cuda, oracle, tmp_path):
    """BatchContext training with eviction into a host tier; one part between steps (step-driven dumper).  Each part
    equals the table after the step it followed (its own read-back, whose values the oracle confirms), restricted to
    the part, in (last-use request, sign) order."""
    torch = torch_cuda
    from persia_b200 import checkpoint as CK
    from persia_b200 import native as N
    from persia_b200 import shard as pb

    dim, S, B, n_parts = 16, 3, 256, 6
    pf = [oracle.index_prefix(i) for i in range(S)]
    # HBM rows for every request's signs after each check (a restore refused for want of a row would skip a step the
    # unbounded oracle takes), fewer than the run's signs: entries move out to the tier and back
    sh = pb.EmbeddingShard(dim, 2048, 0, tier_rows=8192)
    sh.set_optimizer(N.OPT_ADAGRAD, lr=0.05, initialization=0.01)
    sh.configure()
    sh.set_eviction(check_every=1, low_water=900, target_free=1200, keep_batches=1)
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf[i]) for i in range(S)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.ADAGRAD, lr=0.05, init_acc=0.01, eps=1e-10))
    oracle.set_rsqrt_exact(True)
    ctx = pb.BatchContext(S * B, S * B, pf)
    rng = np.random.default_rng(9)
    d = CK.BackgroundDumper(str(tmp_path), [sh], n_parts=n_parts)
    seen = set()
    try:
        for step in range(n_parts):
            ids, _, slot_off = make_batch(rng, S, B, [40, 700, 5000])
            ctx.forward(sh, to_dev_ids(ids, DEV), slot_off, B, training=True)
            _, octx = w.forward(ids, full_row_off(S, B), B, training=True)
            for i in range(S):
                seen.update(int(x) for x in w.ctx_signs(octx, i))
            g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float32)
            ctx.backward(sh, [torch.from_numpy(g[i]).to(DEV) for i in range(S)])
            w.backward(octx, [g[i] for i in range(S)])
            assert d.step() == (step + 1 < n_parts)
            state = _state(sh)  # nothing ran on the table since the part
            got = _read(tmp_path / "s0" / CK.part_file(0, 0, n_parts, step))
            assert got == _part_bytes(CK, state, dim, n_parts, step), step
            assert sh.tier_stats()["refused"] == 0 and sh.counters()["capacity_refused"] == 0
            # the oracle's table after this step, restricted to the part: the same signs (it drops none: every entry
            # the HBM rows release moves to the tier) and every entry bit for bit
            signs, _, ents = CK.decode_list(got)
            all_seen = np.array(sorted(seen), np.uint64)
            want = all_seen[CK.part_of(all_seen, n_parts) == np.uint64(step)]
            np.testing.assert_array_equal(np.sort(signs), want)
            for sgn, e in zip(signs, ents):
                ref = w.get_entry(int(sgn))
                assert ref is not None and e.tobytes() == ref.tobytes()
        assert sh.tier_stats()["moved_out"] > 0
        assert d.status() == ("Idle", 1.0) and (tmp_path / CK.DONE_FILE).is_file()
    finally:
        oracle.set_rsqrt_exact(False)


@pytest.mark.parametrize("R", [2, 3])
def test_virtual_ranks_dump_on_their_worker_streams(torch_cuda, oracle, tmp_path, R):
    torch = torch_cuda
    from persia_b200 import checkpoint as CK
    from persia_b200 import native as N
    from persia_b200 import shard as pb
    from persia_b200.worker import ShardedEmbeddingWorker as W

    dim, S, B, n_parts = 32, 3, 300, 4
    pf = [oracle.index_prefix(i) for i in range(S)]
    ws = W.local_group(R, S, dim, pf, 1 << 14, cap=S * B, optimizer=dict(kind=N.OPT_ADAGRAD, lr=0.05, initialization=0.01),
                       max_batch=B)
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf[i]) for i in range(S)], n_ps=R)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.ADAGRAD, lr=0.05, init_acc=0.01, eps=1e-10))
    oracle.set_rsqrt_exact(True)
    for x in ws:
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    rng = np.random.default_rng(R)
    dumpers = [CK.BackgroundDumper(str(tmp_path), [CK.DumpTable(ws[r].shard, None, ws[r].stream)], r, R, n_parts=n_parts)
               for r in range(R)]
    outs = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(R)]
    union = []
    try:
        for step in range(n_parts):
            ids = [make_batch(rng, S, B, [30, 500, 4000])[0] for _ in range(R)]
            W.group_forward(ws, [to_dev_ids(x, DEV) for x in ids], B, training=True, outs=outs)
            torch.cuda.synchronize()
            octx = [w.forward(ids[r], full_row_off(S, B), B, training=True)[1] for r in range(R)]
            g = (rng.standard_normal((R, S, B, dim)) * 1e-2).astype(np.float32)
            W.group_backward(ws, [[torch.from_numpy(g[r, i]).to(DEV) for i in range(S)] for r in range(R)])
            torch.cuda.synchronize()
            for r in range(R):
                w.backward(octx[r], [g[r, i] for i in range(S)])
            for r in reversed(range(R)):  # rank 0 last: it waits for every rank's marker after its last part
                dumpers[r].step()
                state = _state(ws[r].shard)
                got = _read(tmp_path / f"s{r}" / CK.part_file(r, 0, n_parts, step))
                assert got == _part_bytes(CK, state, dim, n_parts, step), (r, step)
                signs, _, ents = CK.decode_list(got)
                for sgn, e in zip(signs, ents):
                    assert e.tobytes() == w.get_entry(int(sgn)).tobytes()
                union.append((signs, ents))
        assert (tmp_path / CK.DONE_FILE).is_file()
        # re-sharded into one replica: the union of every rank's parts
        fresh = pb.EmbeddingShard(dim, 1 << 16, 0)
        fresh.set_optimizer(N.OPT_ADAGRAD, lr=0.05, initialization=0.01)
        fresh.configure()
        signs = np.concatenate([u[0] for u in union])
        assert CK.load_shards(str(tmp_path), {dim: fresh}, 0, 1) == signs.size
        ent, found = fresh.get_entries(to_dev_ids(signs, DEV))
        assert bool(found.all())
        np.testing.assert_array_equal(ent.cpu().numpy(), np.stack([e for u in union for e in u[1]]))
    finally:
        oracle.set_rsqrt_exact(False)


# ------------------------------------------------------------------------------------------------ the persia_core surface
@pytest.fixture()
def core(torch_cuda):
    from persia_b200 import persia_core as PC

    PC.reset()
    os.environ.pop("RANK", None)
    os.environ.pop("WORLD_SIZE", None)
    yield torch_cuda, PC
    PC.reset()


def _surface(PC, dims=(8, 32)):
    pc = PC.install()
    pc.set_embedding_config({"feature_index_prefix_bit": 8,
                             "slots_config": {f"s{d}": {"dim": d} for d in dims}})
    ctx = pc.PersiaCommonContext(10, 0, 1, 0)
    opt = pc.optim.OptimizerBase()
    opt.init_adagrad(0.01, 0.0, 1.0, 0.01, 1e-10, False)
    opt.apply()
    ctx.configure_embedding_parameter_servers(-0.01, 0.01, 1.0, True, 10.0)
    rng = np.random.default_rng(8)
    rows = [(int(sign), rng.standard_normal(d).astype(np.float32), rng.random(d).astype(np.float32))
            for d, n in zip(dims, (300, 120)) for sign in rng.integers(1, 2**60, size=n, dtype=np.uint64)]
    ctx.set_embedding(rows)
    return ctx


def test_status_errors_and_waits(core, tmp_path):
    torch, PC = core
    ctx = _surface(PC)
    blocker = tmp_path / "file"
    blocker.write_text("not a directory")
    ctx.dump(str(blocker / "ckpt"), background=True)  # its shard directory cannot be created
    with pytest.raises(RuntimeError, match="emb dump FAILED for server 0, due to"):
        ctx.wait_for_emb_dumping()
    assert ctx.dump_status()[0] == "Failed"
    ctx.set_embedding([(12345, np.ones(8, np.float32), np.ones(8, np.float32))])  # the tables still work
    assert ctx.get_embedding_size() == [301, 120]
    ctx.dump(str(tmp_path / "sync"), background=False)  # a later blocking dump reports its own outcome, not the failure
    ctx.wait_for_emb_dumping()
    assert ctx.dump_status() == ("Idle", 1.0)
    ctx.dump(str(tmp_path / "good"), background=True)
    ctx.wait_for_emb_dumping()
    assert ctx.dump_status() == ("Idle", 1.0)
    assert (tmp_path / "good" / "embedding_dump_done").is_file()
    # a second dump while one runs is refused; load waits for the running one
    g = PC._S.groups[8]
    g["lock"].acquire()  # the dump's first part waits for the group: it is surely running
    try:
        ctx.dump(str(tmp_path / "second"), background=True)
        assert ctx.dump_status()[0] == "Dumping"
        with pytest.raises(RuntimeError, match="already running"):
            ctx.dump(str(tmp_path / "third"), background=True)
        seen = {}

        def load():
            ctx.load(str(tmp_path / "good"))
            seen["status"] = ctx.dump_status()

        t = threading.Thread(target=load)
        t.start()
        t.join(0.5)
        assert t.is_alive()  # blocked behind the dump
    finally:
        g["lock"].release()
    t.join(60)
    assert seen["status"] == ("Idle", 1.0)
    ctx.wait_for_emb_dumping()
    assert ctx.get_embedding_size() == [301, 120]


def test_env_selects_the_background_dump(core, tmp_path, monkeypatch):
    torch, PC = core
    from persia_b200 import checkpoint as CK

    PC.set_global_config({"embedding_parameter_server_config": {"num_hashmap_internal_shards": 4}})
    ctx = _surface(PC)
    monkeypatch.setenv("PERSIA_B200_BACKGROUND_DUMP", "1")
    ctx.dump(str(tmp_path / "bg"))
    ctx.wait_for_emb_dumping()
    assert sorted(os.listdir(tmp_path / "bg" / "s0")) == sorted([CK.DONE_FILE] + [f"replica_0_shard_{i}.emb"
                                                                                  for i in range(8)])
    monkeypatch.setenv("PERSIA_B200_BACKGROUND_DUMP", "0")
    ctx.dump(str(tmp_path / "sync"))
    assert sorted(os.listdir(tmp_path / "sync" / "s0")) == [CK.DONE_FILE, "replica_0_shard_0.emb", "replica_0_shard_1.emb"]
    ctx.clear_embeddings()
    ctx.load(str(tmp_path / "bg"))
    assert ctx.get_embedding_size() == [300, 120]


def _tower_batch(rng, api, names, card, B, n_dense):
    ids = [rng.integers(0, card[i], size=B, dtype=np.uint64) for i in range(len(names))]
    dense = rng.standard_normal((B, n_dense)).astype(np.float32)
    label = (rng.random((B, 1)) > 0.5).astype(np.float32)
    return api.PersiaBatch([api.IDTypeFeatureWithSingleID(names[i], ids[i]) for i in range(len(names))],
                           non_id_type_features=[api.NonIDTypeFeature(dense, name="dense")],
                           labels=[api.Label(label, name="click")], requires_grad=True)


def _train(torch, PC, tmp_path, dump_at=None, steps=30):
    """TrainCtx with the Backward engine running; returns (the states after every forward and every backward when
    dump_at is None, else the checkpoint directory)."""
    from persia_b200 import api
    from persia_b200 import workload as W

    PC.reset()
    names, dim, B, n_dense = [f"slot{i}" for i in range(4)], 16, 256, 8
    card = [20, 300, 3000, 30000]
    PC.set_embedding_config({"slots_config": {n: {"dim": dim} for n in names}})
    PC.set_global_config({"embedding_parameter_server_config": {"num_hashmap_internal_shards": 8}})
    torch.manual_seed(0)
    model = W.make_dlrm_tower(len(names), dim, n_dense=n_dense, bottom=(32,), top=(32,)).cuda()
    rng = np.random.default_rng(11)
    states = []
    ckpt = str(tmp_path / "ckpt")

    def record():
        sh = PC._S.groups[dim]["shard"]
        with PC._S.groups[dim]["lock"]:
            states.append(_state(sh))

    with api.TrainCtx(model=model, embedding_optimizer=api.Adagrad(lr=0.05),
                      dense_optimizer=torch.optim.SGD(model.parameters(), lr=0.1), device_id=0, mixed_precision=False,
                      embedding_config=api.EmbeddingConfig()) as ctx:
        for step in range(steps):
            tb = ctx.get_embedding_from_data(_tower_batch(rng, api, names, card, B, n_dense), 0)
            if dump_at is None:
                record()
            out, labels = ctx.forward(tb)
            loss = torch.nn.functional.binary_cross_entropy_with_logits(out, labels[0].squeeze(1))
            ctx.backward(loss)
            if dump_at is None:
                ctx.backward_engine.flush()
                record()
            if step == dump_at:
                ctx.dump_embedding(ckpt, blocking=False)
        if dump_at is not None:
            ctx.wait_for_dump_embedding()
    return states if dump_at is None else ckpt


def test_threaded_dump_through_the_api(core, tmp_path):
    torch, PC = core
    from persia_b200 import checkpoint as CK

    ckpt = _train(torch, PC, tmp_path / "a", dump_at=5, steps=30)
    states = _train(torch, PC, tmp_path / "b", dump_at=None, steps=30)
    n_parts, dim = 8, 16
    t_prev = 0
    contents = []
    for k in range(n_parts):
        got = _read(os.path.join(ckpt, "s0", CK.part_file(0, 0, n_parts, k)))
        match = [t for t in range(t_prev, len(states)) if _part_bytes(CK, states[t], dim, n_parts, k) == got]
        assert match, f"part {k} equals no state of the run without a dump from state {t_prev} on"
        t_prev = match[0]
        contents.append(CK.decode_list(got))
    assert os.path.isfile(os.path.join(ckpt, CK.DONE_FILE))
    # a fresh context loads the files' contents back
    PC.reset()
    ctx = _surface(PC, dims=(16, 32))
    ctx.clear_embeddings()
    ctx.load(ckpt)
    signs = np.concatenate([c[0] for c in contents])
    ents = [e for c in contents for e in c[2]]
    got = ctx.get_entries(signs, dim)
    np.testing.assert_array_equal(got, np.stack(ents))


@pytest.mark.parametrize("R", [2, 3])
def test_virtual_ranks_raw_only_dim_parts_follow_the_sharded_calls(torch_cuda, oracle, tmp_path, R):
    """A dim served only by a raw slot over R virtual ranks: its sharded calls run on each rank's worker stream, outside
    the table's chains, and every part runs on the dumper's own stream with no host sync in between: the ShardedFence
    alone orders them.  Each part equals the oracle's R-server state after the step before it, sign set and entries."""
    torch = torch_cuda
    from persia_b200 import checkpoint as CK
    from persia_b200 import native as N
    from persia_b200.worker import ShardedRawWorker as RW

    dim, B, fixed, n_parts, card = 16, 256, 4, 4, 3000
    prefix = oracle.index_prefix(0)
    ws = RW.local_group(R, 1, dim, [prefix], 1 << 14, cap=B, optimizer=dict(kind=N.OPT_ADAGRAD, lr=0.05, initialization=0.01),
                        max_batch=B)
    w = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=fixed, prefix=prefix)], n_ps=R)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.ADAGRAD, lr=0.05, init_acc=0.01, eps=1e-10))
    oracle.set_rsqrt_exact(True)
    for x in ws:
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    torch.cuda.synchronize()
    fences = [CK.ShardedFence() for _ in range(R)]
    dumpers = [CK.BackgroundDumper(str(tmp_path), [CK.DumpTable(ws[r].shard, None, None, fence=fences[r])], r, R,
                                   n_parts=n_parts) for r in range(R)]
    rng = np.random.default_rng(30 + R)
    seen = set()
    try:
        for step in range(n_parts):
            ids = [rng.integers(0, card, size=B, dtype=np.uint64) for _ in range(R)]
            octx, grads = [], []
            for r in range(R):
                wt, _, _, _, c = w.forward_raw(0, ids[r], np.arange(B + 1, dtype=np.uint32), B, training=True)
                octx.append(c)
                grads.append((rng.standard_normal((wt.shape[0] - 1, dim)) * 1e-2).astype(np.float32))
                seen.update(int(x) for x in oracle.add_prefix(ids[r], 8, prefix))
            d_ids = [to_dev_ids(x, DEV) for x in ids]
            dg = [torch.from_numpy(g).to(DEV) for g in grads]
            torch.cuda.synchronize()  # (inputs in place; from here on nothing synchronises until the parts are issued)
            streams = [x._torch_stream() for x in ws]
            for r in range(R):
                fences[r].call_begin(streams[r])
            RW.group_forward_raw(ws, d_ids, B, fixed, training=True)
            for r in range(R):
                fences[r].call_end(streams[r])
                fences[r].call_begin(streams[r])
            RW.group_backward_raw(ws, dg)
            for r in range(R):
                fences[r].call_end(streams[r])
            for r in range(R):
                w.backward_raw(0, octx[r], grads[r])
            all_seen = np.array(sorted(seen), np.uint64)
            owner = oracle.shard_of(all_seen, R)
            for r in reversed(range(R)):  # rank 0 last: it waits for every rank's marker after its last part
                dumpers[r].step()
                signs, _, ents = CK.decode_list(_read(tmp_path / f"s{r}" / CK.part_file(r, 0, n_parts, step)))
                mine = all_seen[(owner == r) & (CK.part_of(all_seen, n_parts) == np.uint64(step))]
                np.testing.assert_array_equal(np.sort(signs), mine)
                for sgn, e in zip(signs, ents):
                    assert e.tobytes() == w.get_entry(int(sgn)).tobytes(), (r, step, int(sgn))
        assert (tmp_path / CK.DONE_FILE).is_file()
        for x in ws:
            assert x.status() == (False, False)
    finally:
        oracle.set_rsqrt_exact(False)


def _two_process_rank(rank, world, port, ckpt, steps, dump_at):
    import time

    import torch

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    from persia_b200 import api
    from persia_b200 import persia_core as PC
    from persia_b200 import workload as W

    PC.reset()
    names, dim, B, n_dense = [f"slot{i}" for i in range(4)], 16, 256, 8
    card = [20, 300, 3000, 30000]
    PC.set_embedding_config({"slots_config": {n: {"dim": dim} for n in names}})
    PC.set_global_config({"embedding_parameter_server_config": {"num_hashmap_internal_shards": 8}})
    torch.manual_seed(0)
    model = W.make_dlrm_tower(len(names), dim, n_dense=n_dense, bottom=(32,), top=(32,)).cuda()
    rng = np.random.default_rng(11)
    with api.TrainCtx(model=model, embedding_optimizer=api.Adagrad(lr=0.05),
                      dense_optimizer=torch.optim.SGD(model.parameters(), lr=0.1), device_id=rank, mixed_precision=False,
                      embedding_config=api.EmbeddingConfig()) as ctx:
        for step in range(steps):
            batches = [_tower_batch(rng, api, names, card, B, n_dense) for _ in range(world)]  # all drawn, own kept
            out, labels = ctx.forward(ctx.get_embedding_from_data(batches[rank], 0))
            ctx.backward(torch.nn.functional.binary_cross_entropy_with_logits(out, labels[0].squeeze(1)))
            if step == dump_at:
                if rank == 1:
                    time.sleep(1.0)  # rank 1's shard marker comes late: rank 0's root marker must wait for it
                ctx.dump_embedding(ckpt, blocking=False)
        ctx.wait_for_dump_embedding()
        ctx.backward_engine.flush()
        torch.cuda.synchronize()
        import torch.distributed as dist

        dist.barrier()


def test_two_process_background_dump_loads_resharded(core, tmp_path):
    torch, PC = core
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket

    import torch.multiprocessing as mp

    from persia_b200 import checkpoint as CK

    world, n_parts, dim = 2, 8, 16
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ckpt = str(tmp_path / "ckpt")
    mp.spawn(_two_process_rank, args=(world, port, ckpt, 12, 3), nprocs=world, join=True)
    root = os.stat(os.path.join(ckpt, CK.DONE_FILE)).st_mtime_ns
    for q in range(world):
        assert os.stat(os.path.join(ckpt, f"s{q}", CK.DONE_FILE)).st_mtime_ns <= root
    assert CK.checkpoint_info(ckpt) == (world, n_parts)
    contents = [CK.decode_list(_read(os.path.join(ckpt, f"s{q}", CK.part_file(q, 0, n_parts, k))))
                for q in range(world) for k in range(n_parts)]
    signs = np.concatenate([c[0] for c in contents])
    assert signs.size > 0
    for q in range(world):  # every rank dumped only the signs it owns
        mine = np.concatenate([c[0] for c in contents[q * n_parts:(q + 1) * n_parts]])
        assert (CK._farmhash64(mine) % np.uint64(world) == np.uint64(q)).all()
    # re-sharded into one replica: the union of both ranks' parts
    PC.reset()
    ctx = _surface(PC, dims=(16, 32))
    ctx.clear_embeddings()
    ctx.load(ckpt)
    got = ctx.get_entries(signs, dim)
    np.testing.assert_array_equal(got, np.stack([e for c in contents for e in c[2]]))
