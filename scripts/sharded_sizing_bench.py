"""What sizing every sharded step from its own batch costs: R = 2 virtual ranks on one GPU at the metric shape (26 slots,
B = 8192, dim 128, one id per sample), SGD.

  fixed   the step as a fixed-cap exchange runs it: forward (SEND / SERVE / FINISH) + backward, every rank
  sized   the same step after PREPARE, pb_xchg_need (a host sync per rank), the agreement (max over the ranks) and a
          resize check that finds the exchange large enough — what persia_core adds per step on R GPUs, minus the
          all-reduce between processes
  resize  one exchange replacement (drain, new areas, new exchanges) for every rank

Steps alternate fixed / sized on the same workers, timed with a host clock around work that ends in a device
synchronise.  Prints one JSON line with the card's name and power limit read in the same run.  The cost on R real GPUs
(with the all-reduce) is not measured here."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=8192)
    args = ap.parse_args()
    import torch

    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    assert torch.cuda.is_available(), "needs a GPU"
    R, S, B, dim = 2, 26, args.batch, 128
    rng = np.random.default_rng(0)
    card_sizes = rng.integers(10, 2_000_000, size=S)
    pf = [(i + 1) << 56 for i in range(S)]
    ws = W.local_group(R, S, dim, pf, 1 << 22, cap=S * B, optimizer=dict(kind=N.OPT_SGD, lr=0.01), max_batch=B)
    for x in ws:
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device="cuda"))
    batches = [[torch.from_numpy(np.concatenate([rng.integers(0, c, size=B, dtype=np.uint64) for c in card_sizes])
                                 .view(np.int64)).cuda() for _ in range(R)] for _ in range(4)]
    grads = [torch.full((S, B, dim), 1e-3, dtype=torch.float16, device="cuda") for _ in range(R)]
    outs = [torch.empty((S, B, dim), dtype=torch.float16, device="cuda") for _ in range(R)]

    def step(i, sized):
        ids = batches[i % len(batches)]
        if sized:
            need = W.group_prepare(ws, ids, B)
            W.group_resize(ws, *need)
        W.group_forward(ws, ids, B, outs=outs)
        W.group_backward(ws, grads)

    times = {"fixed": [], "sized": []}
    for i in range(args.warmup + args.steps):
        for kind in ("fixed", "sized"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            step(i, kind == "sized")
            torch.cuda.synchronize()
            if i >= args.warmup:
                times[kind].append(time.perf_counter() - t0)
    resize = []
    for k in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        W.group_resize(ws, ws[0].cap + 1, False)
        torch.cuda.synchronize()
        resize.append(time.perf_counter() - t0)
        step(k, False)
    assert all(x.status() == (False, False) for x in ws)
    med = {k: float(np.median(v)) * 1e3 for k, v in times.items()}
    print(json.dumps({"card_and_power_limit": card(), "R_virtual": R, "slots": S, "batch": B, "dim": dim,
                      "fixed_step_ms": round(med["fixed"], 3), "sized_step_ms": round(med["sized"], 3),
                      "sizing_overhead_ms": round(med["sized"] - med["fixed"], 3),
                      "spread_ms": {k: [round(float(np.min(v)) * 1e3, 3), round(float(np.max(v)) * 1e3, 3)]
                                    for k, v in times.items()},
                      "resize_ms": [round(x * 1e3, 2) for x in resize], "final_cap": ws[0].cap}))


if __name__ == "__main__":
    main()
