"""Exportable growable owners (EmbeddingShard(grow="shared")) against eager owners on R = 2 virtual ranks of one GPU.

Reports, with the card's name and power limit read in the same run:
  * the remote forward (RemoteReader.forward, rank 0 reading both owners) on owners that trained to the same state,
    grown against eager, at two shapes: 26 slots x batch 8192 x dim 128 ("large") and 1 slot x batch 256 x dim 16
    ("small"), from CUDA events on the reader's stream over --reads calls each (median);
  * the steady sharded training step (group_forward + group_backward) at the large shape, grown against eager,
    alternating table sets step by step (either first half the time), over --steps steps (median per set).
Views of owners in the same process map everything their owners map, so these remote calls never take the stale
check's host synchronisation; a reader in a second process, and a call that meets a stale item, are not measured here.
Virtual ranks share one GPU: peer reads are local HBM reads, not NVLink.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--reads", type=int, default=100)
    a = ap.parse_args()
    import torch

    from persia_b200.shard import TableView
    from persia_b200.worker import RemoteReader, ShardedEmbeddingWorker as SW

    assert torch.cuda.is_available(), "needs a GPU"
    R, S, B, dim = 2, 26, 8192, 128
    pf = [(i + 1) << 56 for i in range(S)]
    opt = dict(kind=1, lr=0.02, initialization=0.01)
    rng = np.random.default_rng(0)
    sets = {}
    for grow in (False, "shared"):
        ws = SW.local_group(R, S, dim, pf, 1 << 22, cap=S * B, optimizer=opt, max_batch=B, grow=grow)
        for w in ws:
            w.shard.get_entries(torch.zeros(1, dtype=torch.int64, device="cuda:0"))
        torch.cuda.synchronize()
        blobs = [w.shard.export_live_view() for w in ws]
        rd = RemoteReader(ws[0].shard, [None, TableView(blobs[1], 0)], 0, stream=torch.cuda.Stream())
        sets[grow] = (ws, rd)
    step_ms = {k: [] for k in sets}
    for step in range(a.steps + 5):
        ids = [torch.from_numpy(rng.integers(0, 400_000, size=S * B, dtype=np.uint64).view(np.int64)).cuda()
               for _ in range(R)]
        g = [[torch.from_numpy((rng.standard_normal((B, dim)) * 1e-2).astype(np.float16)).cuda() for _ in range(S)]
             for _ in range(R)]
        order = list(sets) if step % 2 == 0 else list(sets)[::-1]
        for k in order:
            ws = sets[k][0]
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            SW.group_forward(ws, ids, B, training=True)
            SW.group_backward(ws, g)
            e1.record()
            torch.cuda.synchronize()
            if step >= 5:
                step_ms[k].append(e0.elapsed_time(e1))
    read_ms = {}
    for shape, (s, b, d_slots) in {"large": (S, B, S), "small": (1, 256, 1)}.items():
        q = torch.from_numpy(rng.integers(0, 800_000, size=s * b, dtype=np.uint64).view(np.int64)).cuda()
        for k, (_, rd) in sets.items():
            st = rd.stream
            for _ in range(5):
                rd.forward(q, b, pf[:d_slots])
            st.synchronize()
            ms = []
            for _ in range(a.reads):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                rd.forward(q, b, pf[:d_slots])
                e1.record(st)
                st.synchronize()
                ms.append(e0.elapsed_time(e1))
            read_ms[f"{shape}_{'grown' if k else 'eager'}_ms"] = round(float(np.median(ms)), 4)
    out = {"card": card(), "R": R, "remote_forward": read_ms,
           "train_step": {("grown" if k else "eager") + "_ms": round(float(np.median(v)), 4) for k, v in step_ms.items()},
           "mapped_rows": [w.shard.storage_stats()["mapped_rows"] for w in sets["shared"][0]],
           "second_process_reader": "not measured", "stale_call": "not measured"}
    for ws, rd in sets.values():
        rd.close()
        for w in ws:
            w.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
