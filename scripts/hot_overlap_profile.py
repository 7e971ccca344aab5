"""torch.profiler view of the metric leg's backward: the hot-sign reduce beside the NaN scan.

Runs bench.py's metric-leg workload (table, batches and gradients built as run_leg builds them), kernel by kernel, in
two phases of --steps steps each:
  beside  the usual stream layout: k_reduce_hot starts on the context's side stream with the backward and, at 8192
          samples per slot or more, k_reduce_hot_short (the items of up to 128 occurrences) on its third one, both
          beside k_nan_scan; k_step_hot follows the scan and the short sums on the first
  alone   a kernel family being timed (pb_profile_enable): the backward runs its kernels one after another on one stream
and prints, per phase, the mean duration of k_nan_scan, k_reduce_hot, k_reduce_hot_short and k_step_hot from the CUDA
kernel records, and in how many steps k_reduce_hot started before k_nan_scan ended.  The chrome traces go to --out.
  python scripts/hot_overlap_profile.py [--steps 20] [--out DIR] [bench.py's workload flags: --rows --dim --batch ...]"""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import bench
from persia_b200 import native as N
from persia_b200 import shard as SH
from persia_b200 import workload as W

KERNELS = ("k_nan_scan", "k_reduce_hot_short", "k_reduce_hot", "k_step_hot")  # (a name matches its first entry)


def kernel_records(path):
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    out = []
    for e in ev:
        if e.get("cat") != "kernel":
            continue
        name = next((k for k in KERNELS if k in e["name"]), None)
        if name:
            out.append((name, float(e["ts"]), float(e["ts"]) + float(e["dur"])))
    return sorted(out, key=lambda r: r[1])


def summarize(recs):
    """Mean duration per kernel (us); and, pairing the i-th k_nan_scan with the i-th k_reduce_hot (one of each per
    step), the steps whose hot reduce started before their scan ended."""
    by = {k: [r for r in recs if r[0] == k] for k in KERNELS}
    mean = {k: float(np.mean([r[2] - r[1] for r in v])) if v else None for k, v in by.items()}
    pairs = list(zip(by["k_nan_scan"], by["k_reduce_hot"]))
    early = sum(1 for scan, hot in pairs if hot[1] < scan[2])
    lead = [scan[2] - hot[1] for scan, hot in pairs]
    return {"mean_us": mean, "steps": len(pairs), "hot_started_before_scan_ended": early,
            "hot_start_before_scan_end_us": float(np.mean(lead)) if lead else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None, help="directory for the chrome traces (default: a temporary directory)")
    mine, rest = ap.parse_known_args()
    sys.argv = [sys.argv[0]] + rest
    args = bench.parse_args()
    out_dir = mine.out or tempfile.mkdtemp(prefix="hot_overlap_")
    os.makedirs(out_dir, exist_ok=True)

    lib = N.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    S, B, dim, rows = args.slots, args.batch, args.dim, int(args.rows)
    card = W.scaled_cardinalities(rows, S)
    pf = W.index_prefixes(S)
    slot_off = [s * B for s in range(S + 1)]
    sh = SH.EmbeddingShard(dim, rows + 1024, dev)
    sh.set_optimizer(N.OPT_ADAGRAD, lr=0.01, initialization=0.01, eps=1e-10)
    sh.configure()
    ctx = SH.BatchContext(S * B, S * B, pf, device=dev)
    bench.fill_table(torch, SH, sh, card, pf, dev, dim)
    n_sets = 4
    ids_host = W.make_batches(2, card, B, n_sets, args.alpha)
    ids_dev = [torch.from_numpy(ids_host[k].view(np.int64)).to(dev) for k in range(n_sets)]
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    grads_all = (torch.randn((n_sets, S, B, dim), generator=g, device=dev) * 1e-2).half()
    grads = [[grads_all[k, s] for s in range(S)] for k in range(n_sets)]
    outs = [torch.empty((S, B, dim), dtype=torch.float16, device=dev) for _ in range(n_sets)]
    stream = torch.cuda.Stream(device=dev)

    def steps(n):
        with torch.cuda.stream(stream):
            for i in range(n):
                ctx.forward(sh, ids_dev[i % n_sets], slot_off, B, training=True, out=outs[i % n_sets])
                ctx.backward(sh, grads[i % n_sets])
        torch.cuda.synchronize()

    gpu = bench.gpu_info(torch, dev.index or 0)
    res = {"gpu": gpu, "workload": f"{S} slots, {rows:.3g} rows, dim {dim}, batch {B}, Adagrad, eager"}
    for phase in ("beside", "alone"):
        if phase == "alone":
            lib.pb_profile_enable(1 << 3)  # any family: the backward then runs on one stream
        steps(5)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            steps(mine.steps)
        if phase == "alone":
            lib.pb_profile_enable(0)
        path = os.path.join(out_dir, f"hot_overlap_{phase}.pt.trace.json")
        prof.export_chrome_trace(path)
        res[phase] = summarize(kernel_records(path))
    res["traces"] = out_dir
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
