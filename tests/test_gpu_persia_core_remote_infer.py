"""GPU, two processes: an Infer job of persia_core with replica_size = 2 serves each rank's requests alone.

Each process is one replica (on cuda:0 and cuda:1 with two GPUs, else both on cuda:0: CUDA IPC opens a handle in
another process on the same device too).  Both load one checkpoint (written here with one shard, so each replica keeps
its farmhash64(sign) % 2 part), export their tables and exchange the view blobs (_start_remote), then apply an `.inc`
packet of their own signs (inserted through the sequence word).  Then rank 0 calls get_embedding_from_bytes while rank 1
waits in a barrier, and the other way round: neither call has a peer taking part.  The summation slots' outputs must be
the oracle's with 2 parameter servers bit for bit, and the raw slot's rows the oracle's for every index position."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = pytest.mark.gpu
DIM, B, FIXED = 16, 64, 3
CFG = {"slots_config": {"a": {"dim": DIM}, "b": {"dim": DIM},
                        "r": {"dim": DIM, "embedding_summation": False, "sample_fixed_size": FIXED}}}
CARD = {"a": 50, "b": 400, "r": 300}  # ids below CARD are in the checkpoint; the batches draw up to 2 x CARD


def _entry(signs, salt):
    s = (np.asarray(signs, np.uint64) % np.uint64(1 << 20)).astype(np.float64)
    return (np.cos(s[:, None] * 0.013 + np.arange(DIM)[None, :] * 0.7 + salt) * 0.25).astype(np.float32)


def _rank(rank, world, port, tmp, devices):
    import torch
    import torch.distributed as dist

    dev = devices[rank]
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    from persia_b200 import api
    from persia_b200 import incremental as INC
    from persia_b200 import persia_core as PC

    PC.reset()
    PC.set_embedding_config(CFG)
    inc = os.path.join(tmp, "inc")
    PC.set_global_config({"common_config": {"job_type": "Infer", "infer_config": {"embedding_checkpoint": os.path.join(tmp, "ckpt")}},
                          "embedding_parameter_server_config": {"incremental_dir": inc}})
    common = PC.PersiaCommonContext(1, rank, world, dev)
    api.SGD(lr=0.1).apply()  # the servers start: checkpoint load, export and blob exchange, scanner
    assert PC._S.remote is not None
    loader = common.incremental_loader
    d = os.path.join(inc, f"s{rank}", INC.flush_dir_name())  # a flush that appears after the start
    os.makedirs(d)
    with open(os.path.join(tmp, f"packet{rank}.inc"), "rb") as f, open(os.path.join(d, f"{rank}_0.inc"), "wb") as g:
        g.write(f.read())
    open(os.path.join(d, INC.DONE_FILE), "w").close()
    loader.poll()
    assert os.path.basename(d) in loader.applied and loader.failed_files == 0 and loader.entries_dropped == 0
    torch.cuda.synchronize()
    dist.barrier()
    batch = np.load(os.path.join(tmp, f"batch{rank}.npy"), allow_pickle=True).item()
    data = api.PersiaBatch([api.IDTypeFeatureWithSingleID("a", batch["a"]), api.IDTypeFeatureWithSingleID("b", batch["b"]),
                            api.IDTypeFeature("r", list(batch["r"]))], requires_grad=False).to_bytes()
    for turn in range(world):  # one rank serves, the other idles in the barrier
        if turn == rank:
            tb = common.get_embedding_from_bytes(data, dev)
            embs = tb.consume_all_id_type_feature_embedding_tensors()
            out = {"a": embs[0].get_sum_embedding().numpy(), "b": embs[1].get_sum_embedding().numpy()}
            table, index, non_empty, num = embs[2].get_raw_embedding()
            out.update(r_table=table.numpy(), r_index=index.numpy(), r_num=np.asarray(num))
            torch.cuda.synchronize()
        dist.barrier()
    out["wait_errors"] = sum(int(g["shard"].counters()["wait_errors"]) for g in PC._S.groups.values())
    np.save(os.path.join(tmp, f"out{rank}.npy"), out, allow_pickle=True)
    PC._close_remote()
    dist.barrier()  # every view closed before any table goes
    PC.reset()
    dist.destroy_process_group()


def test_infer_job_two_replicas_serve_alone(oracle, tmp_path):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import torch.multiprocessing as mp
    from persia_b200 import checkpoint as CK
    from persia_b200 import incremental as INC
    from persia_b200 import persia_core as PC

    world, tmp = 2, str(tmp_path)
    _, slots = PC.parse_embedding_config(CFG)
    pf = {s.name: s.index_prefix for s in slots}
    # the checkpoint: every id below CARD of every slot, one shard (each replica keeps its part when it loads)
    ck_signs = np.concatenate([oracle.add_prefix(np.arange(CARD[n], dtype=np.uint64), 8, pf[n]) for n in CARD])
    ck_ent = _entry(ck_signs, 0.0)
    os.makedirs(os.path.join(tmp, "ckpt", "s0"))
    with open(os.path.join(tmp, "ckpt", "s0", "replica_0_shard_0.emb"), "wb") as f:
        f.write(CK.encode_list(ck_signs, ck_ent, DIM))
    for path in (os.path.join(tmp, "ckpt", "s0", CK.DONE_FILE), os.path.join(tmp, "ckpt", CK.DONE_FILE)):
        with open(path, "w") as f:
            f.write(CK.done_yaml(1, 1))
    # the packet: every third checkpoint sign rewritten, and new signs; each replica's directory holds its own signs
    new = np.concatenate([oracle.add_prefix(np.arange(CARD[n], CARD[n] + CARD[n] // 2, dtype=np.uint64), 8, pf[n])
                          for n in CARD])
    pk_signs = np.concatenate([ck_signs[::3], new])
    pk_ent = _entry(pk_signs, 1.0)
    owner = oracle.shard_of(pk_signs, world)
    for r in range(world):
        with open(os.path.join(tmp, f"packet{r}.inc"), "wb") as f:
            f.write(INC.encode_packet(pk_signs[owner == r], DIM, pk_ent[owner == r]))
    rng = np.random.default_rng(3)
    batches = []
    for r in range(world):
        b = {n: rng.integers(0, 2 * CARD[n], size=B, dtype=np.uint64) for n in ("a", "b")}
        b["r"] = np.array([rng.integers(0, 2 * CARD["r"], size=int(k), dtype=np.uint64)
                           for k in rng.integers(0, FIXED + 2, size=B)], dtype=object)
        np.save(os.path.join(tmp, f"batch{r}.npy"), b, allow_pickle=True)
        batches.append(b)
    devices = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    mp.spawn(_rank, args=(world, port, tmp, devices), nprocs=world, join=True)

    w_sum = oracle.Worker([oracle.SlotCfg(DIM, prefix=pf["a"]), oracle.SlotCfg(DIM, prefix=pf["b"])], n_ps=world)
    w_raw = oracle.Worker([oracle.SlotCfg(DIM, summation=False, sample_fixed_size=FIXED, prefix=pf["r"])], n_ps=world)
    for w in (w_sum, w_raw):
        w.configure()
        w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1, wd=0.0))
        w.set_embedding(ck_signs, ck_ent, DIM)
        w.set_embedding(pk_signs, pk_ent, DIM)  # the packet overwrites
    for r in range(world):
        out = np.load(os.path.join(tmp, f"out{r}.npy"), allow_pickle=True).item()
        assert out["wait_errors"] == 0
        b = batches[r]
        want, _ = w_sum.forward(np.concatenate([b["a"], b["b"]]), np.arange(2 * B + 1, dtype=np.uint32), B,
                                training=False, keep_ctx=False)
        assert out["a"].tobytes() == want[0].tobytes(), r
        assert out["b"].tobytes() == want[1].tobytes(), r
        counts = np.array([len(x) for x in b["r"]], np.uint32)
        row_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
        ids = np.concatenate([np.asarray(x, np.uint64) for x in b["r"]])
        otable, oindex, _, onum, _ = w_raw.forward_raw(0, ids, row_off, B, training=False, keep_ctx=False)
        assert (out["r_num"] == onum).all()
        assert ((out["r_index"] != 0) == (oindex != 0)).all()
        held = oindex != 0  # the row at every index position, whatever numbering either side chose
        assert out["r_table"][out["r_index"][held]].tobytes() == otable[oindex[held]].tobytes(), r
