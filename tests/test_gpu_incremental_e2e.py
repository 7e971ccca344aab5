"""GPU end to end: training through TrainCtx with incremental updates on writes `.inc` flushes beside a checkpoint, and an
Infer job started from that checkpoint catches up by applying the later flushes: its tables then hold the trained
entries bit for bit and its inference forward gives the trained side's f16 outputs."""
import os
import shutil

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture()
def env(oracle):
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    from persia_b200 import persia_core as PC

    PC.reset()
    os.environ.pop("RANK", None)
    os.environ.pop("WORLD_SIZE", None)
    yield torch, PC
    PC.reset()


NAMES = ["a", "b", "c", "d"]
CFG = {"slots_config": {"a": {"dim": 16}, "b": {"dim": 16}, "c": {"dim": 8, "sqrt_scaling": True}, "d": {"dim": 8}},
       "feature_groups": {"ab": ["a", "b"]}}
CARD = [60, 60, 800, 5000]


def _batch(api, rng, B, requires_grad=True):
    ids = [rng.integers(0, CARD[i], size=B, dtype=np.uint64) for i in range(len(NAMES))]
    dense = rng.standard_normal((B, 4)).astype(np.float32)
    label = (rng.random((B, 1)) > 0.5).astype(np.float32)
    return api.PersiaBatch([api.IDTypeFeatureWithSingleID(NAMES[i], ids[i]) for i in range(len(NAMES))],
                           non_id_type_features=[api.NonIDTypeFeature(dense, name="dense")],
                           labels=[api.Label(label, name="click")], requires_grad=requires_grad)


def _tables(PC):
    """{dim: (signs u64 sorted, entries)} of every resident sign."""
    out = {}
    for dim in sorted(PC._S.groups):
        sh = PC._S.groups[dim]["shard"]
        signs, _ = sh.export_signs()
        signs = signs.cpu().numpy().view(np.uint64)
        signs = np.sort(signs)
        ent = PC.PersiaCommonContext(1, 0, 1).get_entries(signs, dim) if signs.size else np.zeros((0, sh.entry_len))
        out[dim] = (signs, np.asarray(ent))
    return out


def _infer_outputs(api, common, batch):
    tb = common.get_embedding_from_data(batch.data, 0)
    return [e.get_sum_embedding().numpy().copy() for e in tb.consume_all_id_type_feature_embedding_tensors()]


def test_train_flush_checkpoint_then_infer_catches_up(env, tmp_path):
    torch, PC = env
    from persia_b200 import api
    from persia_b200 import incremental as INC

    rng = np.random.default_rng(7)
    B, inc, ckpt = 256, str(tmp_path / "inc"), str(tmp_path / "ckpt")
    PC.set_embedding_config(CFG)
    PC.set_global_config({"common_config": {"checkpointing_config": {"num_workers": 3}},
                          "embedding_parameter_server_config": {"enable_incremental_update": True,
                                                                "incremental_buffer_size": 400,
                                                                "incremental_dir": inc}})
    torch.manual_seed(0)
    emb_opt = api.Adagrad(lr=0.05)

    class Tower(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(4 + 16 * 2 + 8 * 2, 1)

        def forward(self, non_id, embs):
            return self.lin(torch.cat([non_id[0]] + [e.float() for e in embs], dim=1)).squeeze(1)

    model = Tower().cuda()
    loss_fn = torch.nn.BCEWithLogitsLoss()
    probe = _batch(api, np.random.default_rng(99), B, requires_grad=False)
    with api.TrainCtx(model=model, embedding_optimizer=emb_opt, dense_optimizer=torch.optim.SGD(model.parameters(), lr=0.1),
                      device_id=0, mixed_precision=False, embedding_config=api.EmbeddingConfig()) as ctx:
        def train(n):
            for _ in range(n):
                out, labels = ctx.forward(ctx.get_embedding_from_data(_batch(api, rng, B), 0))
                ctx.backward(loss_fn(out, labels[0].squeeze(1)))

        train(3)
        first = ctx.common_context.flush_incremental()
        assert first is not None
        ctx.common_context.dump(ckpt)
        pre = set(os.listdir(os.path.join(inc, "s0")))
        train(8)
        ctx.common_context.flush_incremental()
        post = sorted(set(os.listdir(os.path.join(inc, "s0"))) - pre)
        assert len(post) >= 3, post  # automatic flushes past the threshold, then the forced one
        for d in post:
            files = sorted(os.listdir(os.path.join(inc, "s0", d)))
            assert files[-1] == INC.DONE_FILE and 1 <= len(files) - 1 <= 3
        for g in PC._S.groups.values():
            assert g["shard"].incremental_stats()["dropped"] == 0
        torch.cuda.synchronize()
        trained = _tables(PC)
        want_out = _infer_outputs(api, ctx.common_context, probe)
    PC.reset()

    # Infer: the checkpoint, then the flushes written after it.  The flushes already present at start are not applied
    infer_dir = str(tmp_path / "inc_infer")
    os.makedirs(os.path.join(infer_dir, "s0"))
    for d in pre:
        shutil.copytree(os.path.join(inc, "s0", d), os.path.join(infer_dir, "s0", d))
    PC.set_embedding_config(CFG)
    PC.set_global_config({"common_config": {"job_type": "Infer", "infer_config": {"embedding_checkpoint": ckpt}},
                          "embedding_parameter_server_config": {"incremental_dir": infer_dir}})
    common = PC.PersiaCommonContext(1, 0, 1, 0)
    api.Adagrad(lr=0.05).apply()  # registering the optimizer starts the servers: checkpoint load + scanner
    loader = common.incremental_loader
    assert loader is not None and loader.poll() == []
    for d in post:
        shutil.copytree(os.path.join(inc, "s0", d), os.path.join(infer_dir, "s0", d))
    assert loader.poll() == post
    assert loader.entries_dropped == 0
    torch.cuda.synchronize()
    served = _tables(PC)
    for dim, (signs, ent) in trained.items():
        s2, e2 = served[dim]
        assert s2.tolist() == signs.tolist()
        assert e2.tobytes() == ent.tobytes()
    got_out = _infer_outputs(api, common, probe)
    assert len(got_out) == len(want_out)
    for a, b in zip(got_out, want_out):
        assert a.dtype == np.float16 and a.tobytes() == b.tobytes()


def test_two_virtual_ranks_flush_own_dirs_and_infer_catches_up(oracle, tmp_path):
    """R = 2 virtual ranks on one GPU, with the calls persia_core makes at R > 1: each owner table's set is taken by
    persia_core's flush (device take + gather, host half on the dumper thread) and written by a dumper of its replica
    index, a checkpoint of both shards sits between the flushes, and an Infer start of each replica (load_shards of its
    s{r}, then the loader on incremental_dir/s{r}) reproduces that rank's entries bit for bit."""
    import functools
    import threading

    import torch

    from persia_b200 import checkpoint as CK
    from persia_b200 import incremental as INC
    from persia_b200 import persia_core as PC
    from persia_b200 import shard as SH
    from persia_b200.worker import ShardedEmbeddingWorker as W
    from util import DEV, make_batch, to_dev_ids

    R, S, B, dim, cap, set_cap = 2, 2, 256, 16, 1 << 14, 1 << 13
    pfs = [oracle.index_prefix(0), oracle.index_prefix(1)]
    gopt = dict(kind=1, lr=0.02, initialization=0.01, eps=1e-10)
    ws = W.local_group(R, S, dim, pfs, cap, cap=S * B, optimizer=gopt, max_batch=B)
    for x in ws:
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))  # (allocation syncs the device: not mid-step)
        x.enable_incremental(set_cap)
    groups = [{dim: {"shard": x.shard, "lock": threading.RLock(), "device": 0}} for x in ws]
    inc, ckpt, infer_dir = str(tmp_path / "inc"), str(tmp_path / "ckpt"), str(tmp_path / "inc_infer")
    dumpers = [INC.IncrementalDumper(inc, r, num_workers=3) for r in range(R)]
    rng = np.random.default_rng(41)

    def train(n):
        for _ in range(n):
            batches = [make_batch(rng, S, B, [300, 5000])[0] for _ in range(R)]
            torch.cuda.synchronize()
            W.group_forward(ws, [to_dev_ids(b, DEV) for b in batches], B)
            torch.cuda.synchronize()
            g = [[torch.from_numpy((rng.standard_normal((B, dim)) * 1e-2).astype(np.float16)).to(DEV) for _ in range(S)]
                 for _ in range(R)]
            W.group_backward(ws, g)
            torch.cuda.synchronize()

    def flush():
        for r in range(R):
            with torch.cuda.stream(ws[r].stream):
                dumpers[r].submit(PC._take_flush(groups[r], set_cap))
        for d in dumpers:
            d.flush()

    train(2)
    flush()
    for r in range(R):
        CK.dump_shards(ckpt, [ws[r].shard], r, R)
    pre = [set(os.listdir(os.path.join(inc, f"s{r}"))) for r in range(R)]
    for _ in range(3):
        train(2)
        flush()
    assert sorted(os.listdir(inc)) == ["s0", "s1"]
    post = [sorted(set(os.listdir(os.path.join(inc, f"s{r}"))) - pre[r]) for r in range(R)]
    for r in range(R):
        assert len(post[r]) == 3
        for d in post[r] + sorted(pre[r]):
            path = os.path.join(inc, f"s{r}", d)
            files = sorted(f for f in os.listdir(path) if f.endswith(".inc"))
            assert files and all(f.startswith(f"{r}_") for f in files)
            for f in files:  # every flushed sign is owned by the rank that wrote it
                signs = INC.decode_packet(open(os.path.join(path, f), "rb").read())[0]
                assert signs.size and (oracle.shard_of(signs, R) == r).all()
    trained = []
    for x in ws:
        signs, _ = x.shard.export_signs()
        signs = np.sort(signs.cpu().numpy().view(np.uint64))
        trained.append((signs, x.shard.get_entries(torch.from_numpy(signs.view(np.int64)).to(DEV))[0].cpu().numpy()))
    for d in dumpers:
        d.close()
    for x in ws:
        x.close()

    for r in range(R):  # Infer, replica r
        os.makedirs(os.path.join(infer_dir, f"s{r}"))
        for d in pre[r]:
            shutil.copytree(os.path.join(inc, f"s{r}", d), os.path.join(infer_dir, f"s{r}", d))
        sh = SH.EmbeddingShard(dim, cap, 0)
        sh.set_optimizer(**gopt)
        sh.configure()
        CK.load_shards(ckpt, {dim: sh}, r, R)
        grp = {dim: {"shard": sh, "lock": threading.RLock(), "device": 0}}
        loader = INC.IncrementalLoader(os.path.join(infer_dir, f"s{r}"),
                                       functools.partial(PC._apply_incremental, groups=grp))
        assert loader.poll() == []
        for d in post[r]:
            shutil.copytree(os.path.join(inc, f"s{r}", d), os.path.join(infer_dir, f"s{r}", d))
        assert loader.poll() == post[r] and loader.entries_dropped == 0 and loader.failed_files == 0
        signs, _ = sh.export_signs()
        signs = np.sort(signs.cpu().numpy().view(np.uint64))
        assert signs.tolist() == trained[r][0].tolist()
        ent = sh.get_entries(torch.from_numpy(signs.view(np.int64)).to(DEV))[0].cpu().numpy()
        assert ent.tobytes() == trained[r][1].tobytes()
        sh.close()
