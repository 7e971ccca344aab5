"""Per-request latency and requests/s of inference on R GPUs: the remote path (RemoteReader, one rank alone reads the
owners' shards in place) against the collective path (ShardedEmbeddingWorker.group_forward(training=False), every rank
in one step).  R = 2 virtual ranks on one GPU, 26 slots at dim 128, one id per sample, at batch 512 and 4096 (--batches).

  collective  one step serves R requests (one per rank): latency = the step's time, requests/s = R / step time
  remote      one rank's request alone (ranks take turns): latency = the call's time, requests/s = 1 / latency

The tables are filled by one collective training step, then exported; the two paths then alternate on the same tables.
Every call is timed with a host clock around work that ends in a device synchronise; median and p99 are printed.  Both
paths' outputs are compared bit for bit once per batch size.  Virtual ranks share one GPU, so the remote path's peer
reads are local HBM reads here: the cost of an NVLink hop per row is not measured by this script.  Prints one JSON line
with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(ts):
    ts = np.sort(np.asarray(ts) * 1e3)
    return {"median_ms": round(float(np.median(ts)), 4), "p99_ms": round(float(ts[int(0.99 * (len(ts) - 1))]), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batches", default="512,4096")
    ap.add_argument("--slots", type=int, default=26)
    ap.add_argument("--dim", type=int, default=128)
    args = ap.parse_args()
    import torch

    from persia_b200 import native as N
    from persia_b200.worker import RemoteReader
    from persia_b200.worker import ShardedEmbeddingWorker as W

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing is measured")
    R, S, dim, dev = 2, args.slots, args.dim, torch.device("cuda", 0)
    Bs = [int(b) for b in args.batches.split(",")]
    Bmax = max(Bs)
    pf = [(i + 1) << 56 for i in range(S)]
    rng = np.random.default_rng(0)
    card_ids = [int(10 ** (2 + 5 * i / S)) for i in range(S)]  # 100 .. ~10^7 distinct ids per slot

    def ids_for(B):
        return [torch.from_numpy(np.stack([rng.integers(0, c, size=B, dtype=np.uint64) for c in card_ids])
                                 .reshape(-1).view(np.int64)).to(dev) for _ in range(R)]

    ws = W.local_group(R, S, dim, pf, 1 << 22, cap=S * Bmax, optimizer=dict(kind=N.OPT_SGD, lr=0.01), max_batch=Bmax)
    for w in ws:
        w.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=dev))
    torch.cuda.synchronize()
    W.group_forward(ws, ids_for(Bmax), Bmax, training=True)  # admits the rows the inference batches find
    W.group_backward(ws, [torch.zeros((S, Bmax, dim), dtype=torch.float16, device=dev) for _ in range(R)])
    torch.cuda.synchronize()
    readers = RemoteReader.local_group([w.shard for w in ws])
    res = {"card": card(), "R": R, "slots": S, "dim": dim, "virtual_ranks_on_one_gpu": True, "results": {}}
    try:
        for B in Bs:
            ids = ids_for(B)
            outs = [torch.empty((S, B, dim), dtype=torch.float16, device=dev) for _ in range(R)]
            mine = [torch.empty((S, B, dim), dtype=torch.float16, device=dev) for _ in range(R)]
            coll, rem = [], []
            for it in range(args.warmup + args.reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                W.group_forward(ws, ids, B, training=False, outs=outs)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                r = it % R
                readers[r].forward(ids[r], B, pf, out=mine[r])
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                if it >= args.warmup:
                    coll.append(t1 - t0)
                    rem.append(t2 - t1)
                if it == 0:
                    for q in range(R):
                        readers[q].forward(ids[q], B, pf, out=mine[q])
                    torch.cuda.synchronize()
                    same = all(torch.equal(outs[q].view(torch.int16), mine[q].view(torch.int16)) for q in range(R))
            c, m = stats(coll), stats(rem)
            res["results"][str(B)] = {
                "collective_step": c, "collective_requests_per_s": round(R / float(np.median(coll)), 1),
                "remote_request": m, "remote_requests_per_s": round(1 / float(np.median(rem)), 1),
                "remote_us_per_row": round(float(np.median(rem)) * 1e6 / (S * B), 5),
                "collective_us_per_row": round(float(np.median(coll)) * 1e6 / (R * S * B), 5),
                "outputs_bit_identical": bool(same)}
    finally:
        for rd in readers:
            rd.close()
    for w in ws:
        assert w.shard.counters()["wait_errors"] == 0
    print(json.dumps(res))


if __name__ == "__main__":
    main()
