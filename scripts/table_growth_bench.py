"""Growable tables (pb_table_set_growth) against eagerly allocated ones on one GPU.

Three legs, each printed as one JSON object with the card's name, power limit and top SM clock:

  steady  — step time of a fully grown growable table against an eager one at the same capacity, both holding
            --rows resident rows (Adagrad, 26 Criteo-shaped slots, one id per sample, Zipf(1.05) ids), at configs[1]'s
            shape (dim 64, batch 4096) and at the metric shape (dim 128, batch 8192).  The two kinds alternate, --reps
            times each; every repetition builds its table, fills it (pb_lookup training over every row), warms up and
            times --steps training forward + backward steps with device events.  Only one table exists at a time (two
            tables of 5e7 rows at dim 128 would not fit in 80 GB).  The kernels address both tables alike; what may
            differ is how the chunked mappings translate.
  growth  — the time of the calls that grow a table: training lookups of 2^20 fresh signs each fill a growable table
            (dim 64, Adagrad, capacity --rows); every call is timed with a host clock around a device synchronise.
            Calls that mapped rows and calls that doubled the index are reported with the live entries they started
            from, nearest 1e6, 1e7 and 5e7 (or --rows), beside the median of the calls that grew nothing.
  memory  — the bytes a growable table holds (pb_debug_owned) after --zipf-steps training steps at configs[1]'s shape
            over a capacity of --rows, against what an eager table of that capacity allocates.

    python scripts/table_growth_bench.py [--rows 50000000] [--steps 100] [--warmup 20] [--reps 2] [--legs steady,growth,memory]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SLOTS = 26


def gpu_info(torch):
    """Name, power limit and top SM clock of the card the numbers were measured on."""
    info = {"name": torch.cuda.get_device_name(0), "power_limit": None, "max_sm_clock": None}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
    except (OSError, subprocess.SubprocessError):
        return info
    if len(out) == 2:
        info["power_limit"], info["max_sm_clock"] = out[0].strip(), out[1].strip()
    return info


def owned_bytes(lib):
    from persia_b200 import native as N

    lib.pb_debug_owned.restype = C.c_int
    lib.pb_debug_owned.argtypes = [C.POINTER(C.c_uint64)]
    out = (C.c_uint64 * 2)()
    N.check(lib.pb_debug_owned(out))
    return int(out[1])


def new_table(SH, N, dim, rows, grow):
    sh = SH.EmbeddingShard(dim, rows, 0, grow=grow)
    sh.set_optimizer(N.OPT_ADAGRAD, lr=0.01, initialization=0.01, eps=1e-10)
    sh.configure()
    return sh


def fill(torch, SH, sh, card, pf, dim, timed=None):
    """Every row of ids [0, card[s]) of every slot resident, 2^20 signs per training lookup.  timed: a list that
    receives (live entries before the call, seconds, rows mapped before / after, index cells before / after) per call."""
    chunk = 1 << 20
    buf = torch.empty((chunk, dim), dtype=torch.float32, device="cuda:0")
    live = 0
    for s in range(len(card)):
        for lo in range(0, int(card[s]), chunk):
            hi = min(int(card[s]), lo + chunk)
            signs = SH.add_prefix(torch.arange(lo, hi, dtype=torch.int64, device="cuda:0"), [0, hi - lo], [pf[s]])
            if timed is None:
                sh.lookup(signs, training=True, out=buf[: signs.numel()])
                continue
            before = sh.storage_stats()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sh.lookup(signs, training=True, out=buf[: signs.numel()])
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            after = sh.storage_stats()
            timed.append((live, dt, before["mapped_rows"], after["mapped_rows"], before["index_cells"],
                          after["index_cells"]))
            live += hi - lo
    torch.cuda.synchronize()


def steady_leg(args, torch, SH, N, W, dim, B, name):
    card = W.scaled_cardinalities(args.rows, SLOTS)
    pf = W.index_prefixes(SLOTS)
    batches = W.make_batches(1, card, B, 8)
    ids = [torch.from_numpy(b.view(np.int64)).to("cuda:0") for b in batches]
    grads = [torch.randn((B, dim), device="cuda:0").half() * 1e-2 for _ in range(SLOTS)]
    off = [s * B for s in range(SLOTS + 1)]
    times = {"eager": [], "grown": []}
    for rep in range(args.reps):
        for kind in ("eager", "grown"):
            sh = new_table(SH, N, dim, args.rows, kind == "grown")
            ctx = SH.BatchContext(SLOTS * B, SLOTS * B, pf)
            fill(torch, SH, sh, card, pf, dim)
            if kind == "grown":
                st = sh.storage_stats()
                assert st["mapped_rows"] == st["reserved_rows"] and st["refused_unmapped"] == 0, st
            for k in range(args.warmup):
                ctx.forward(sh, ids[k % len(ids)], off, B)
                ctx.backward(sh, grads)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for k in range(args.steps):
                ctx.forward(sh, ids[k % len(ids)], off, B)
                ctx.backward(sh, grads)
            e1.record()
            torch.cuda.synchronize()
            times[kind].append(e0.elapsed_time(e1) / args.steps)
            ctx.close()
            sh.close()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    return {"leg": "steady", "shape": name, "dim": dim, "batch": B, "slots": SLOTS, "resident_rows": args.rows,
            "ms_per_step": {k: v for k, v in times.items()},
            "grown_over_eager": float(np.median(times["grown"]) / np.median(times["eager"]))}


def growth_leg(args, torch, SH, N, W):
    dim = 64
    pf = W.index_prefixes(SLOTS)
    card = W.scaled_cardinalities(args.rows, SLOTS)
    sh = new_table(SH, N, dim, args.rows, True)
    calls = []
    fill(torch, SH, sh, card, pf, dim, timed=calls)
    sh.close()
    rows_grew = [c for c in calls if c[3] > c[2]]
    index_grew = [c for c in calls if c[5] > c[4]]
    plain = [c[1] for c in calls if c[3] == c[2] and c[5] == c[4]]

    def nearest(cs, target):
        if not cs:
            return None
        c = min(cs, key=lambda c: abs(c[0] - target))
        return {"live_entries": c[0], "ms": c[1] * 1e3, "rows_mapped": [c[2], c[3]], "index_cells": [c[4], c[5]]}

    targets = [t for t in (1_000_000, 10_000_000, 50_000_000) if t <= args.rows] or [args.rows]
    return {"leg": "growth", "dim": dim, "signs_per_call": 1 << 20, "capacity": args.rows,
            "row_growth_calls": len(rows_grew), "index_doublings": len(index_grew),
            "row_growth": {str(t): nearest(rows_grew, t) for t in targets},
            "index_doubling": {str(t): nearest(index_grew, t) for t in targets},
            "plain_call_ms_median": float(np.median(plain) * 1e3) if plain else None}


def memory_leg(args, torch, SH, N, W):
    dim, B = 64, 4096
    lib = N.load()
    pf = W.index_prefixes(SLOTS)
    card = W.scaled_cardinalities(args.rows, SLOTS)
    batches = W.make_batches(2, card, B, args.zipf_steps)
    grads = [torch.randn((B, dim), device="cuda:0").half() * 1e-2 for _ in range(SLOTS)]
    off = [s * B for s in range(SLOTS + 1)]
    torch.cuda.synchronize()
    base = owned_bytes(lib)
    sh = new_table(SH, N, dim, args.rows, True)
    ctx = SH.BatchContext(SLOTS * B, SLOTS * B, pf)
    ctx_bytes = owned_bytes(lib) - base
    for b in batches:
        ctx.forward(sh, torch.from_numpy(b.view(np.int64)).to("cuda:0"), off, B)
        ctx.backward(sh, grads)
    torch.cuda.synchronize()
    st, live = sh.storage_stats(), sh.counters()["admitted"]
    mapped = owned_bytes(lib) - base - ctx_bytes
    stride = 2 * dim  # Adagrad: emb ++ per-element state
    cells = 1
    while cells < max(1024, args.rows + args.rows // 2):
        cells *= 2
    eager = args.rows * (4 * stride + 4) + 16 * (cells + 3)  # rows, row_tick, index (no eviction: no sweep workspace)
    ctx.close()
    sh.close()
    return {"leg": "memory", "dim": dim, "batch": B, "steps": args.zipf_steps, "capacity": args.rows,
            "live_entries": live, "mapped_rows": st["mapped_rows"], "index_cells": st["index_cells"],
            "growable_bytes": mapped, "eager_bytes": eager, "growable_over_eager": mapped / eager}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rows", type=int, default=50_000_000, help="resident rows (steady), capacity (growth, memory)")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=2, help="alternating repetitions of each kind (steady)")
    ap.add_argument("--zipf-steps", type=int, default=200)
    ap.add_argument("--legs", default="steady,growth,memory")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("no GPU: every number here is a GPU measurement")
    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200 import workload as W

    gpu = gpu_info(torch)
    legs = args.legs.split(",")
    if "steady" in legs:
        for dim, B, name in ((64, 4096, "configs[1]"), (128, 8192, "metric")):
            print(json.dumps({**steady_leg(args, torch, SH, N, W, dim, B, name), "gpu": gpu}), flush=True)
    if "growth" in legs:
        print(json.dumps({**growth_leg(args, torch, SH, N, W), "gpu": gpu}), flush=True)
    if "memory" in legs:
        print(json.dumps({**memory_leg(args, torch, SH, N, W), "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
