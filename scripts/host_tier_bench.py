"""A table larger than HBM on one GPU: an HBM table with a host-memory tier behind it (pb_table_attach_tier) against the
same workload HBM-only, where eviction drops rows (BASELINE.json configs[4], scaled to one GPU).

Workload: dim 96, Adagrad, 26 Zipf(1.05) slots, batch 8192, a key space of `--keys-per-hbm-row` times the HBM rows;
every training request runs an eviction check.  The tier is sized to a quarter of the host's available memory (capped
at the key space) and printed.  A step is captured in a CUDA graph and its replays are timed with device events; ids
come from pre-generated batches copied in before each replay:
    forward(cur) -> [side stream: pb_tier_stage(next)] || [dense stand-in, backward(cur)] -> join
The dense stand-in is a fixed loop of fp16 matmuls (sized and printed) standing in for the dense tower's step, which is
what a stage overlaps in training.  Legs, all with the same stand-in unless named otherwise: the tier unstaged (no
side stream), the tier staged, HBM-only (where eviction drops rows), and the tier staged without the stand-in.  Reports
step time, samples/s, the GPU hit ratio, rows restored / moved out per step, the bytes they move over PCIe, stage
counters per step, the move kernels' achieved rate (torch.profiler, a separate unstaged run), and the card's name and
power limit.  --stage-blocks times the staged leg once more for each listed grid of the stage's kernels.

    python scripts/host_tier_bench.py [--hbm-rows 1048576] [--steps 100] [--warmup 80] [--stage-blocks 16,64,132]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:  # no nvidia-smi: the torch name alone
        import torch

        return torch.cuda.get_device_name(0) + ", power limit unknown"


def host_available_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    raise RuntimeError("MemAvailable not in /proc/meminfo")


def dense_standin(args):
    """A fixed loop of fp16 matmuls [batch, n] @ [n, n]: the dense step a stage runs beside."""
    import torch

    x = torch.randn((args.batch, args.dense_n), device="cuda:0").half()
    w = (torch.randn((args.dense_n, args.dense_n), device="cuda:0") / args.dense_n ** 0.5).half()

    def step():
        y = x
        for _ in range(args.dense_iters):
            y = y @ w
        return y

    return step


def run(args, tier, batches_dev, slot_off, profile=False, staged=False, dense=None, stage_blocks=None):
    import torch

    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200.workload import index_prefixes

    S, B, dim = args.slots, args.batch, args.dim
    if stage_blocks:
        N.load().pb_debug_stage_blocks(int(stage_blocks))
    sh = SH.EmbeddingShard(dim, args.hbm_rows, 0, tier_rows=tier)
    sh.set_optimizer(N.OPT_ADAGRAD, lr=0.01, initialization=0.01, eps=1e-10)
    sh.configure()
    sh.set_eviction(check_every=1, low_water=args.hbm_rows // 8, target_free=args.hbm_rows // 4, keep_batches=1)
    prefixes = index_prefixes(S)
    ctx = SH.BatchContext(S * B, S * B, prefixes)
    ids = torch.empty(S * B, dtype=torch.int64, device="cuda:0")
    nxt = torch.empty(S * B, dtype=torch.int64, device="cuda:0")  # the next step's ids (the stage's)
    out = torch.empty((S, B, dim), dtype=torch.float16, device="cuda:0")
    g = (torch.randn((S, B, dim), device="cuda:0") * 1e-3).half()
    grads = [g[i] for i in range(S)]
    stream, side = torch.cuda.Stream(), torch.cuda.Stream()
    n_sets = batches_dev.shape[0]

    def step():
        ctx.forward(sh, ids, slot_off, B, training=True, out=out)
        if staged:
            side.wait_stream(stream)
            with torch.cuda.stream(side):
                sh.stage(nxt, slot_off, prefixes)
        if dense is not None:
            dense()
        ctx.backward(sh, grads)
        if staged:
            stream.wait_stream(side)

    with torch.cuda.stream(stream):
        for k in range(args.warmup):  # eager: fills HBM and the tier to a steady state
            ids.copy_(batches_dev[k % n_sets])
            nxt.copy_(batches_dev[(k + 1) % n_sets])
            step()
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            step()
        stream.synchronize()
        items = ctx.batch_stats()["items"]
        st0, res0, sg0 = sh.tier_stats(), int(sh.counters()["admitted"]), sh.stage_stats()
        starts = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps)]
        ends = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps)]
        prof = None
        if profile:
            from torch.profiler import ProfilerActivity, profile as tprofile

            prof = tprofile(activities=[ProfilerActivity.CUDA])
            prof.__enter__()
        for k in range(args.steps):
            ids.copy_(batches_dev[(args.warmup + k) % n_sets])
            nxt.copy_(batches_dev[(args.warmup + k + 1) % n_sets])
            starts[k].record(stream)
            graph.replay()
            ends[k].record(stream)
        stream.synchronize()
        if prof is not None:
            prof.__exit__(None, None, None)
    ms = sum(a.elapsed_time(b) for a, b in zip(starts, ends)) / args.steps
    st1, res1, sg1 = sh.tier_stats(), int(sh.counters()["admitted"]), sh.stage_stats()
    steps = args.steps
    restored = (st1["restored"] - st0["restored"]) / steps
    moved = (st1["moved_out"] - st0["moved_out"]) / steps
    # signs new to the union this step: what it holds more, plus what its sweeps dropped
    new = ((res1 + st1["host_rows"] + st1["dropped"]) - (res0 + st0["host_rows"] + st0["dropped"])) / steps
    row_bytes = 4 * (dim + dim)  # embedding ++ Adagrad state
    res = {"tier_rows": tier, "step_ms": ms, "samples_per_s": B / (ms * 1e-3), "distinct_per_step": items,
           "restored_per_step": restored, "moved_out_per_step": moved, "pcie_bytes_per_step": (restored + moved) * row_bytes}
    if staged:
        res["staged_per_step"] = (sg1["staged"] - sg0["staged"]) / steps
        res["stage_skipped_per_step"] = (sg1["skipped"] - sg0["skipped"]) / steps
        res["stage_blocks"] = int(stage_blocks or 132)
    if tier:  # (HBM-only: the sweeps' drops are not counted, so neither are the misses)
        res["new_signs_per_step"] = new
        res["gpu_hit_ratio"] = 1.0 - (restored + new) / max(items, 1)
    if prof is not None:
        move_us = sum(e.device_time_total for e in prof.key_averages() if "k_tier_restore" in e.key or "k_tier_move" in e.key
                      or "k_tier_stage" in e.key)
        res["move_kernels_us_per_step"] = move_us / steps
        res["move_kernels_GBps"] = res["pcie_bytes_per_step"] / max(move_us / steps * 1e-6, 1e-12) / 1e9
    sh.close()
    if stage_blocks:
        N.load().pb_debug_stage_blocks(0)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hbm-rows", type=int, default=1 << 20)
    ap.add_argument("--keys-per-hbm-row", type=float, default=10.0)
    ap.add_argument("--slots", type=int, default=26)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--dim", type=int, default=96)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=80)
    ap.add_argument("--sets", type=int, default=240, help="pre-generated batches (fresh ids for every step)")
    ap.add_argument("--dense-n", type=int, default=4096, help="dense stand-in: [batch, n] @ [n, n] fp16 matmuls")
    ap.add_argument("--dense-iters", type=int, default=3, help="dense stand-in: matmuls per step")
    ap.add_argument("--stage-blocks", default="", help="comma-separated grids to time the staged leg at, besides the default (132)")
    args = ap.parse_args()
    import torch

    from persia_b200.workload import make_batches

    if not torch.cuda.is_available():
        raise SystemExit("host_tier_bench needs a CUDA device")
    keys = int(args.hbm_rows * args.keys_per_hbm_row)
    avail = host_available_bytes()
    row_bytes = 4 * 2 * args.dim
    tier = int(min(keys, avail // 4 // row_bytes))
    print(f"card: {card()}")
    print(f"host MemAvailable {avail / 2**30:.1f} GiB -> tier of {tier} rows ({tier * row_bytes / 2**30:.1f} GiB pinned); "
          f"HBM rows {args.hbm_rows}, key space {keys} ({args.slots} slots)", flush=True)
    cards = [keys // args.slots] * args.slots
    batches = make_batches(1, cards, args.batch, args.sets)
    batches_dev = torch.from_numpy(batches.view(np.int64)).to("cuda:0")
    slot_off = [s * args.batch for s in range(args.slots + 1)]
    dense = dense_standin(args)
    dense()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(20):
        dense()
    b.record()
    torch.cuda.synchronize()
    dense_ms = a.elapsed_time(b) / 20
    print(f"dense stand-in: {args.dense_iters} x [{args.batch}, {args.dense_n}] @ [{args.dense_n}, {args.dense_n}] fp16 "
          f"matmuls, {dense_ms:.3f} ms alone", flush=True)
    out = {"dense_standin_ms": dense_ms,
           "tier_unstaged": run(args, tier, batches_dev, slot_off, dense=dense),
           "tier_staged": run(args, tier, batches_dev, slot_off, staged=True, dense=dense),
           "hbm_only": run(args, 0, batches_dev, slot_off, dense=dense),
           "tier_staged_no_standin": run(args, tier, batches_dev, slot_off, staged=True)}
    for blocks in [int(x) for x in args.stage_blocks.split(",") if x]:
        out[f"tier_staged_blocks_{blocks}"] = run(args, tier, batches_dev, slot_off, staged=True, dense=dense,
                                                  stage_blocks=blocks)
    out["tier_unstaged_profiled"] = run(args, tier, batches_dev, slot_off, profile=True, dense=dense)
    out["card"] = card()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
