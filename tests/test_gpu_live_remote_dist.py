"""GPU, two processes on two GPUs: TrainCtx with replica_size = 2 where rank 0 alone runs eval batches through eval_ctx in
the middle of training and rank 1 does not.  The eval forwards read the peers' live tables in place, with no collective,
so both ranks finish; rank 0's eval outputs equal the oracle with 2 parameter servers at that point; and every entry at
the end equals, bit for bit, a run without the eval (an eval admits nothing and refreshes no recency).  Skipped with
fewer than two GPUs."""
import os
import pickle
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu
NAMES, DIM, CARD = ["slot0", "slot1", "slot2"], 32, [50, 4000, 1 << 30]
B, STEPS, EVAL_AT, K = 256, 5, 2, 3  # rank 0 evaluates K batches after training step EVAL_AT


def _ids(rng):
    return [rng.integers(0, c, size=B, dtype=np.uint64) for c in CARD]


def _rank(rank, world, port, result_dir, with_eval):
    import torch

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    import torch.distributed as dist

    from persia_b200 import api
    from persia_b200 import persia_core as PC

    class Tower(torch.nn.Module):  # a small DLRM-style tower: dense bottom MLP, embeddings concatenated, top MLP
        def __init__(self):
            super().__init__()
            self.bottom = torch.nn.Linear(4, 8)
            self.top = torch.nn.Sequential(torch.nn.Linear(8 + len(NAMES) * DIM, 16), torch.nn.ReLU(), torch.nn.Linear(16, 1))

        def forward(self, non_id, emb):
            x = torch.relu(self.bottom(non_id[0]))
            return self.top(torch.cat([x] + [e.float() for e in emb], dim=1)).squeeze(1)

    PC.reset()
    PC.set_embedding_config({"slots_config": {n: {"dim": DIM} for n in NAMES}})
    torch.manual_seed(0)
    model = Tower().cuda()
    rng = np.random.default_rng(5)
    erng = np.random.default_rng(100)
    rec, evals = [], []
    loss_fn = torch.nn.BCEWithLogitsLoss()
    with api.TrainCtx(model=model, embedding_optimizer=api.SGD(lr=0.1), dense_optimizer=torch.optim.SGD(model.parameters(), lr=0.1),
                      device_id=rank, mixed_precision=False, embedding_config=api.EmbeddingConfig()) as ctx:
        for step in range(STEPS):
            feats = [_ids(rng) for _ in range(world)]  # all drawn, own kept
            mine = feats[rank]
            dense = rng.standard_normal((world, B, 4)).astype(np.float32)[rank]
            label = (rng.random((world, B, 1)) < 0.5).astype(np.float32)[rank]
            pb = api.PersiaBatch([api.IDTypeFeatureWithSingleID(n, f) for n, f in zip(NAMES, mine)],
                                 non_id_type_features=[api.NonIDTypeFeature(dense, name="dense")],
                                 labels=[api.Label(label, name="y")], requires_grad=True)
            out, labels = ctx.forward(ctx.get_embedding_from_data(pb, 0))
            ctx.backward(loss_fn(out, labels[0].squeeze(1)))
            grads = np.stack([c[-1].grad.detach().cpu().numpy()
                              for c in ctx.current_batch.id_type_feature_embedding_cache_torch_tensors])
            ctx.backward_engine.flush()
            torch.cuda.synchronize()
            rec.append((feats, grads))
            if step == EVAL_AT and rank == 0 and with_eval:  # rank 1 goes on training meanwhile, then waits below
                with api.eval_ctx(model=model, embedding_config=api.EmbeddingConfig()) as ev:
                    for _ in range(K):
                        ef = _ids(erng)  # (signs of the training batches and new ones)
                        epb = api.PersiaBatch([api.IDTypeFeatureWithSingleID(n, f) for n, f in zip(NAMES, ef)],
                                              non_id_type_features=[api.NonIDTypeFeature(np.zeros((B, 4), np.float32),
                                                                                         name="dense")],
                                              requires_grad=False)
                        ev.forward(ev.get_embedding_from_data(epb, 0))
                        embs = np.stack([e.detach().cpu().numpy()
                                         for e in ev.current_batch.id_type_feature_embedding_torch_tensors])
                        evals.append((ef, embs))
        dist.barrier()
        import oracle

        signs = []
        _, slots = PC.parse_embedding_config({"slots_config": {n: {"dim": DIM} for n in NAMES}})
        pf = {s.name: s.index_prefix for s in slots}
        for feats, _ in rec:
            for r in range(world):
                for n, f in zip(NAMES, feats[r]):
                    signs.append(oracle.add_prefix(f, 8, pf[n]))
        signs = np.unique(np.concatenate(signs).astype(np.uint64))
        ent = ctx.common_context.get_entries(signs, DIM, missing_ok=True)
        keep = [k for k, e in enumerate(ent) if e is not None]
        with open(os.path.join(result_dir, f"rank{rank}.pkl"), "wb") as f:
            pickle.dump((rec, evals, signs[keep], np.stack([ent[k] for k in keep])), f)
        dist.barrier()  # (both ranks stop together: the views close before either table)
    PC.reset()


def _spawn(tmp, with_eval):
    import torch.multiprocessing as mp

    os.makedirs(tmp, exist_ok=True)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_rank, args=(2, port, tmp, with_eval), nprocs=2, join=True)
    out = []
    for r in range(2):
        with open(os.path.join(tmp, f"rank{r}.pkl"), "rb") as f:
            out.append(pickle.load(f))
    return out


def test_rank_zero_alone_evaluates_mid_training(oracle, tmp_path):
    import torch

    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from persia_b200 import persia_core as PC

    world = 2
    res = _spawn(str(tmp_path / "eval"), True)
    base = _spawn(str(tmp_path / "plain"), False)
    assert len(res[0][1]) == K and len(res[1][1]) == 0
    for r in range(world):  # the eval moved nothing: every entry as in the run without it
        np.testing.assert_array_equal(res[r][2], base[r][2])
        assert res[r][3].tobytes() == base[r][3].tobytes(), r
    _, slots = PC.parse_embedding_config({"slots_config": {n: {"dim": DIM} for n in NAMES}})
    w = oracle.Worker([oracle.SlotCfg(DIM, prefix=s.index_prefix) for s in slots], n_ps=world)
    w.configure(wb=10.0)
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1, wd=0.0))
    row_off = np.arange(len(NAMES) * B + 1, dtype=np.uint32)
    for step in range(STEPS):
        octx = []
        for r in range(world):
            feats, _ = res[r][0][step]
            _, c = w.forward(np.concatenate(feats[r]).astype(np.uint64), row_off, B, training=True)
            octx.append(c)
        for r in range(world):
            w.backward(octx[r], list(res[r][0][step][1]))
        if step == EVAL_AT:
            for ef, embs in res[0][1]:
                want, _ = w.forward(np.concatenate(ef).astype(np.uint64), row_off, B, training=False, keep_ctx=False)
                for i in range(len(NAMES)):
                    assert embs[i].tobytes() == want[i].tobytes(), i
