"""GPU, two processes on two GPUs: TrainCtx with replica_size = 2 whose first batch is small (B = 8, one id per sample),
then a ragged batch of B = 1024 and an eval batch larger still.  Every step is sized from its own batch (the symmetric
areas are rendezvoused again when an exchange grows), and the embeddings and rows match the oracle with 2 parameter
servers.  Skipped with fewer than two GPUs."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu
NAMES, DIM, CARD = ["slot0", "slot1", "slot2"], 32, [20, 3000, 1 << 30]
STEPS = [(8, 1, True), (1024, 6, True), (4096, 1, False)]  # (B, most ids per sample, training)


def _ids(rng, B, max_ids):
    """Per slot: B samples of 1..max_ids ids (exactly one when max_ids == 1)."""
    out = []
    for c in CARD:
        n = rng.integers(1, max_ids + 1, size=B) if max_ids > 1 else np.ones(B, np.int64)
        out.append([rng.integers(0, c, size=k, dtype=np.uint64) for k in n])
    return out


def _rank(rank, world, port, result_dir):
    import torch

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    from persia_b200 import api
    from persia_b200 import persia_core as PC

    PC.reset()
    PC.set_embedding_config({"slots_config": {n: {"dim": DIM} for n in NAMES}})
    torch.manual_seed(0)
    model = torch.nn.Linear(len(NAMES) * DIM, 1).cuda()
    rng = np.random.default_rng(5)
    rec = []
    with api.TrainCtx(model=model, embedding_optimizer=api.SGD(lr=0.1), dense_optimizer=torch.optim.SGD(model.parameters(), lr=0.1),
                      device_id=rank, mixed_precision=False, embedding_config=api.EmbeddingConfig()) as ctx:
        for B, max_ids, training in STEPS:
            feats = [_ids(rng, B, max_ids) for _ in range(world)][rank]  # all drawn, own kept
            pb = api.PersiaBatch([api.IDTypeFeature(n, f) for n, f in zip(NAMES, feats)],
                                 labels=[api.Label(np.zeros((B, 1), np.float32), name="y")], requires_grad=training)
            tb = ctx.get_embedding_from_data(pb, 0)
            out, labels = ctx.forward(tb)
            embs = np.stack([e.detach().cpu().numpy() for e in ctx.current_batch.id_type_feature_embedding_torch_tensors])
            grads = None
            if training:
                ctx.backward(((out - 1.0) ** 2).mean())
                grads = np.stack([c[-1].grad.detach().cpu().numpy()
                                  for c in ctx.current_batch.id_type_feature_embedding_cache_torch_tensors])
                ctx.backward_engine.flush()
            torch.cuda.synchronize()
            rec.append((feats, embs, grads))
    np.save(os.path.join(result_dir, f"rank{rank}.npy"), np.array(rec, dtype=object), allow_pickle=True)
    PC.reset()


def test_two_process_steps_sized_from_their_batches(oracle, tmp_path):
    import torch

    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from persia_b200 import persia_core as PC

    world = 2
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    mp.spawn(_rank, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    res = [np.load(os.path.join(str(tmp_path), f"rank{r}.npy"), allow_pickle=True) for r in range(world)]
    _, slots = PC.parse_embedding_config({"slots_config": {n: {"dim": DIM} for n in NAMES}})
    w = oracle.Worker([oracle.SlotCfg(DIM, prefix=s.index_prefix) for s in slots], n_ps=world)
    w.configure(wb=10.0)
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1, wd=0.0))
    for step, (B, max_ids, training) in enumerate(STEPS):
        octx = []
        for r in range(world):
            feats, embs, _ = res[r][step]
            counts = np.array([len(x) for f in feats for x in f], np.uint32)
            row_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
            ids = np.concatenate([x for f in feats for x in f]).astype(np.uint64)
            want, c = w.forward(ids, row_off, B, training=training)
            octx.append(c)
            for i in range(len(NAMES)):
                if max_ids == 1:
                    assert embs[i].tobytes() == want[i].tobytes(), (step, r, i)
                else:  # the f32 sum order of a sample's ids differs (sample order here, shard order in the oracle)
                    np.testing.assert_allclose(embs[i].astype(np.float32), want[i].astype(np.float32), rtol=2e-3, atol=8e-3)
        if training:
            for r in range(world):
                w.backward(octx[r], list(res[r][step][2]))
