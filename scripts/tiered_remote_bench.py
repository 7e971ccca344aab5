"""Remote reads of owners with a shared host tier (pb_table_create_host_shared + RemoteReader).

R = 2 virtual ranks on one GPU, one slot, dim 64, SGD (one entry = 256 B).  Reports, with the card's name and power
limit read in the same run:
  * frozen: a lone reader request's latency (rank 0, --read-batch distinct signs, CUDA events on its stream, median and
    p99) for signs its owners hold in HBM against signs they hold in their tiers (host rows read over PCIe);
  * live: training steps of the same tables exported live (an eviction check every step, HBM a fraction of the signs, so
    every step restores and moves): the step time, how many times per step the write-sequence word went odd
    (pb_debug_table_seq), the device time of the kernels inside those windows (the eviction check's and the restore's,
    torch.profiler), and a reader request's latency issued beside each step;
  * a second process opening rank 0's tiered view (the tier's memfd through /proc, mapped and registered): the open's
    wall time per GB of tier;
  * one GPU, no export: the same tiered training step with a shared tier against a private one (pb_table_create_host),
    alternating: the step time (events), and in a profiled run of its own per table the device time per step of the
    kernels that touch host rows, k_tier_restore_items (restores), k_tier_move (moves out) and k_tier_collect
    (torch.profiler), to show what memfd pages cost them.
Virtual ranks share one GPU: peer HBM reads are local HBM reads here, not NVLink; host rows are read over PCIe as on R
GPUs.  Prints one JSON line."""
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

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(ms):
    ms = np.sort(np.asarray(ms))
    return {"median_ms": round(float(np.median(ms)), 4), "p99_ms": round(float(ms[int(0.99 * (len(ms) - 1))]), 4)}


_OPENER = r"""
import sys, time
from persia_b200 import native as N, shard as SH
import torch
torch.cuda.init()
N.load()
blob = bytes.fromhex(sys.stdin.readline().strip())
t0 = time.perf_counter()
v = SH.TableView(blob, 0)
t1 = time.perf_counter()
v.close()
print(t1 - t0, flush=True)
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dim", type=int, default=64)
    ap.add_argument("--hbm-rows", type=int, default=1 << 18, help="HBM rows per rank")
    ap.add_argument("--tier-rows", type=int, default=1 << 21, help="host-tier rows per rank (entries held: 3/4 of it)")
    ap.add_argument("--read-batch", type=int, default=4096)
    ap.add_argument("--reads", type=int, default=200)
    ap.add_argument("--batch", type=int, default=8192, help="training ids per rank and step")
    ap.add_argument("--train-hbm-rows", type=int, default=1 << 15,
                    help="HBM rows per rank of the training parts (steps draw from 8x as many signs: they restore and move)")
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()
    import torch

    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200.worker import RemoteReader
    from persia_b200.worker import ShardedEmbeddingWorker as W

    assert torch.cuda.is_available(), "needs a GPU"
    R, dim, H, T = 2, args.dim, args.hbm_rows, args.tier_rows
    out = {"card": card(), "R": R, "dim": dim, "hbm_rows": H, "train_hbm_rows": args.train_hbm_rows, "tier_rows": T,
           "batch": args.batch, "read_batch": args.read_batch}
    lib = N.load()
    lib.pb_debug_table_seq.restype = C.c_int
    lib.pb_debug_table_seq.argtypes = [C.c_void_p, C.POINTER(C.c_uint32)]

    def group():
        return W.local_group(R, 1, dim, [0], H, cap=args.batch, optimizer=dict(kind=N.OPT_SGD, lr=0.0, wd=0.0),
                             max_batch=args.batch, tier_rows=T, shared_tier=True)

    # ---- frozen: HBM-held against tier-held signs ----
    ws = group()
    total = R * ((3 * T) // 4)
    n_hbm = (9 * R * H) // 10  # signs [0, n_hbm) are set first, alone: they fit the HBM rows; the rest go to the tiers
    for lo, hi in [(0, n_hbm)] + [(a, min(total, a + (1 << 20))) for a in range(n_hbm, total, 1 << 20)]:
        signs = torch.arange(lo, hi, dtype=torch.int64, device=DEV)
        own = SH.shard_of(signs, R)
        for r, x in enumerate(ws):
            sel = signs[own == r]
            x.shard.set_entries(sel, torch.rand((sel.numel(), dim), device=DEV))
    torch.cuda.synchronize()
    out["tier_stats"] = [x.shard.tier_stats() for x in ws]
    readers = RemoteReader.local_group([x.shard for x in ws])
    rd = readers[0]
    rng = np.random.default_rng(0)

    def time_reads(pool_lo, pool_hi, n):
        ms = []
        for i in range(n + 10):
            q = torch.from_numpy(rng.integers(pool_lo, pool_hi, size=args.read_batch).astype(np.int64)).to(DEV)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(rd.stream)
            rd.forward(q, args.read_batch, [0])
            e1.record(rd.stream)
            e1.synchronize()
            if i >= 10:
                ms.append(e0.elapsed_time(e1))
        return stats(ms)

    out["frozen_read_hbm"] = time_reads(0, n_hbm, args.reads)
    out["frozen_read_tier"] = time_reads(n_hbm, total, args.reads)

    # ---- a second process opens rank 0's tiered view ----
    blob = ws[0].shard.export_view()  # (exported frozen already: the same blob again)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.Popen([sys.executable, "-c", _OPENER], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True,
                         env=env)
    got, _ = p.communicate(blob.hex() + "\n", timeout=600)
    open_s = float(got.strip().splitlines()[-1])
    gb = T * dim * 4 / 1e9
    out["view_open_s"] = round(open_s, 4)
    out["view_open_s_per_gb"] = round(open_s / gb, 4)
    out["tier_gb"] = round(gb, 3)
    for x in readers:
        x.close()
    for x in ws:
        x.close()
    torch.cuda.synchronize()

    # ---- live: steps with restores and moves, the word's windows, a reader beside each step ----
    HT = args.train_hbm_rows
    card_ids = 8 * R * HT  # signs a step draws from: HBM holds an eighth of them
    ws = W.local_group(R, 1, dim, [0], HT, cap=args.batch, optimizer=dict(kind=N.OPT_SGD, lr=0.0, wd=0.0),
                       max_batch=args.batch, tier_rows=T, shared_tier=True)
    for x in ws:
        x.shard.set_eviction(check_every=1, low_water=args.batch, target_free=args.batch + args.batch // 2, keep_batches=1)
    blobs = [x.shard.export_live_view() for x in ws]
    readers = [RemoteReader(x.shard, [SH.TableView(b, 0) if q != r else None for q, b in enumerate(blobs)], r,
                            stream=torch.cuda.Stream(device=DEV)) for r, x in enumerate(ws)]
    zeros = [[torch.zeros((args.batch, dim), dtype=torch.float16, device=DEV)] for _ in range(R)]

    def seq(x):
        v = C.c_uint32()
        N.check(lib.pb_debug_table_seq(x.shard.h, C.byref(v)))
        return v.value

    step_ms, read_ms, windows = [], [], []
    for i in range(args.steps + 5):
        ids = [torch.from_numpy(rng.integers(0, card_ids, size=args.batch).astype(np.int64)).to(DEV) for _ in range(R)]
        q = torch.from_numpy(rng.integers(0, card_ids, size=args.read_batch).astype(np.int64)).to(DEV)
        torch.cuda.synchronize()
        s0 = [seq(x) for x in ws]
        t0 = time.perf_counter()
        W.group_forward(ws, ids, args.batch, training=True, slot_occ_offs=[[0, args.batch]] * R)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(readers[0].stream)
        readers[0].forward(q, args.read_batch, [0])
        e1.record(readers[0].stream)
        W.group_backward(ws, zeros)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if i >= 5:
            step_ms.append((t1 - t0) * 1e3)
            read_ms.append(e0.elapsed_time(e1))
            windows.append(sum((seq(x) - a) // 2 for x, a in zip(ws, s0)) / R)
    out["live_step"] = stats(step_ms)
    out["live_read_beside_step"] = stats(read_ms)
    out["live_windows_per_rank_step"] = float(np.mean(windows))
    out["live_tier_stats"] = [x.shard.tier_stats() for x in ws]
    out["live_wait_errors"] = [x.shard.counters()["wait_errors"] for x in ws]
    # the kernels inside the windows, one profiled step
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ids = [torch.from_numpy(rng.integers(0, card_ids, size=args.batch).astype(np.int64)).to(DEV) for _ in range(R)]
        W.group_forward(ws, ids, args.batch, training=True, slot_occ_offs=[[0, args.batch]] * R)
        W.group_backward(ws, zeros)
        torch.cuda.synchronize()
    inside = ("k_evict", "k_tier_plan", "k_tier_collect", "k_tier_move", "k_rebuild", "k_tier_restore_recv", "k_seq_")
    win_us = sum(e.device_time_total for e in prof.key_averages() if any(k in e.key for k in inside))
    out["live_window_kernels_us_per_rank_step"] = round(win_us / R, 1)
    for x in readers:
        x.close()
    for x in ws:
        x.close()
    torch.cuda.synchronize()

    # ---- one GPU, no export: shared against private host rows ----
    shards = {}
    for shared in (True, False):
        s = SH.EmbeddingShard(dim, HT, 0, tier_rows=T, shared_tier=shared)
        s.set_optimizer(kind=N.OPT_SGD, lr=0.0)
        s.configure()
        s.set_eviction(check_every=1, low_water=args.batch, target_free=args.batch + args.batch // 2, keep_batches=1)
        shards[shared] = (s, SH.BatchContext(args.batch, args.batch, [0], device=0))
    g = torch.zeros((args.batch, dim), dtype=torch.float16, device=DEV)
    times = {True: [], False: []}
    for i in range(2 * (args.steps + 5)):
        shared = i % 2 == 0
        s, ctx = shards[shared]
        ids = torch.from_numpy(rng.integers(0, 8 * HT, size=args.batch).astype(np.int64)).to(DEV)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ctx.forward(s, ids, [0, args.batch], args.batch, training=True)
        ctx.backward(s, [g])
        e1.record()
        e1.synchronize()
        if i >= 10:
            times[shared].append(e0.elapsed_time(e1))
    out["one_gpu_step_shared_tier"] = stats(times[True])
    out["one_gpu_step_private_tier"] = stats(times[False])
    kernels = ("k_tier_restore_items", "k_tier_move", "k_tier_collect")
    for rnd in range(2):  # each table profiled alone, twice, alternating
        for shared in (True, False):
            s, ctx = shards[shared]
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    ids = torch.from_numpy(rng.integers(0, 8 * HT, size=args.batch).astype(np.int64)).to(DEV)
                    ctx.forward(s, ids, [0, args.batch], args.batch, training=True)
                    ctx.backward(s, [g])
                torch.cuda.synchronize()
            us = {k: 0.0 for k in kernels}
            for e in prof.key_averages():
                for k in kernels:
                    if k in e.key:
                        us[k] += e.device_time_total / args.steps
            key = "one_gpu_kernel_us_per_step_" + ("shared" if shared else "private")
            out.setdefault(key, []).append({k: round(v, 1) for k, v in us.items()})
    out["one_gpu_tier_stats"] = {str(k): v[0].tier_stats() for k, v in shards.items()}
    for s, ctx in shards.values():
        ctx.close()
        s.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
