"""Training beside reads of live-exported tables on R GPUs (pb_table_export_live_view + RemoteReader).

R = 2 virtual ranks on one GPU, 26 slots at dim 128, training batch 8192 per rank, one id per sample, an eviction check
on every step (small shards: the sweeps and index rebuilds run throughout).  Reports, with the card's name and power
limit read in the same run:
  * training step time (group_forward + group_backward) on tables without and with a live export, alternating step by
    step on two identical table sets (either first half the time), over --rounds rounds (each round's medians: the run-to-run spread);
  * a lone reader request's latency (rank 0 reads its peer's table, --read-batch samples), alone and issued beside a
    training step of the live tables, from CUDA events on the reader's stream (median and p99);
  * the owners' write windows: how many times per step the write-sequence word went odd (pb_debug_table_seq), and
    the device time of the kernels that keep it odd (k_evict_sweep and the three rebuild kernels, torch.profiler), the
    longest a reader can be sent round again by one window, against the wait budget of PB_WAIT_SPINS rounds.
The reader kernel keeps no retry counter, so retries per request are not counted directly: a request retries only
while it overlaps a window, and the latency beside training against alone shows what those retries cost.
Virtual ranks share one GPU: peer reads are local HBM reads here, not NVLink.  Prints one JSON line."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WAIT_SPINS = 1 << 25  # pb_remote.cu's PB_WAIT_SPINS: rounds a lane group retries before it gives up


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def stats(ms):
    ms = np.sort(np.asarray(ms))
    return {"median_ms": round(float(np.median(ms)), 4), "p99_ms": round(float(ms[int(0.99 * (len(ms) - 1))]), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20, help="timed steps per table set and round")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--read-batch", type=int, default=512)
    ap.add_argument("--reads", type=int, default=200)
    ap.add_argument("--slots", type=int, default=26)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--capacity", type=int, default=1 << 20, help="rows per shard (small: eviction on every step)")
    args = ap.parse_args()
    import torch

    from persia_b200 import native as N
    from persia_b200.shard import TableView
    from persia_b200.worker import RemoteReader
    from persia_b200.worker import ShardedEmbeddingWorker as W

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing is measured")
    R, S, dim, B, dev = 2, args.slots, args.dim, args.batch, torch.device("cuda", 0)
    lib = N.load()
    lib.pb_debug_table_seq.argtypes = [C.c_void_p, C.POINTER(C.c_uint32)]
    pf = [(i + 1) << 56 for i in range(S)]
    rng = np.random.default_rng(0)
    card_ids = [int(10 ** (2 + 5 * i / S)) for i in range(S)]  # 100 .. ~10^7 distinct ids per slot

    def ids_for(n):
        return [torch.from_numpy(np.stack([rng.integers(0, c, size=n, dtype=np.uint64) for c in card_ids])
                                 .reshape(-1).view(np.int64)).to(dev) for _ in range(R)]

    def group():
        ws = W.local_group(R, S, dim, pf, args.capacity, cap=S * B, optimizer=dict(kind=N.OPT_ADAGRAD, lr=0.01),
                           max_batch=B)
        for w in ws:
            w.shard.set_eviction(check_every=1)
            w.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=dev))
        torch.cuda.synchronize()
        return ws

    plain, live = group(), group()
    blobs = [w.shard.export_live_view() for w in live]
    readers = [RemoteReader(w.shard, [TableView(b, dev) if q != r else None for q, b in enumerate(blobs)], r,
                            stream=torch.cuda.Stream(device=dev)) for r, w in enumerate(live)]
    grads = [torch.full((S, B, dim), 1e-3, dtype=torch.float16, device=dev) for _ in range(R)]

    def step(ws, ids):
        W.group_forward(ws, ids, B, training=True)
        W.group_backward(ws, grads)

    def seq():
        out = []
        for w in live:
            v = C.c_uint32()
            N.check(lib.pb_debug_table_seq(w.shard.h, C.byref(v)))
            out.append(v.value)
        return out

    res = {"card": card(), "R": R, "slots": S, "dim": dim, "batch": B, "capacity_per_shard": args.capacity,
           "optimizer": "adagrad", "virtual_ranks_on_one_gpu": True}
    try:
        for _ in range(args.warmup):  # fills the shards to their eviction threshold
            ids = ids_for(B)
            step(plain, ids)
            step(live, ids)
        torch.cuda.synchronize()
        # ---- step time, alternating -------------------------------------------------------------------------------------
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        rounds = []
        for _ in range(args.rounds):
            t = {"plain": [], "live": []}
            for k in range(args.steps):
                ids = ids_for(B)
                order = (("plain", plain), ("live", live))
                for name, ws in (order if k % 2 == 0 else order[::-1]):  # (either goes first half the time)
                    torch.cuda.synchronize()
                    ev[0].record()
                    step(ws, ids)
                    ev[1].record()
                    torch.cuda.synchronize()
                    t[name].append(ev[0].elapsed_time(ev[1]))
            rounds.append({k: round(float(np.median(v)), 4) for k, v in t.items()})
        res["step_ms_median_per_round"] = rounds
        # ---- a lone reader request: alone, and beside a training step -----------------------------------------------
        rb = args.read_batch
        q = ids_for(rb)[0]
        rd = readers[0]
        out = torch.empty((S, rb, dim), dtype=torch.float16, device=dev)
        rev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def read():
            rev[0].record(rd.stream)
            rd.forward(q, rb, pf, out=out)
            rev[1].record(rd.stream)

        alone, beside, windows = [], [], []
        for i in range(args.reads + args.warmup):
            torch.cuda.synchronize()
            read()
            torch.cuda.synchronize()
            if i >= args.warmup:
                alone.append(rev[0].elapsed_time(rev[1]))
        for i in range(args.reads + args.warmup):
            ids = ids_for(B)
            torch.cuda.synchronize()
            s0 = seq()
            W.group_forward(live, ids, B, training=True)  # (the eviction check is enqueued first)
            read()
            W.group_backward(live, grads)
            torch.cuda.synchronize()
            s1 = seq()
            if i >= args.warmup:
                beside.append(rev[0].elapsed_time(rev[1]))
                windows.append(sum((b - a) // 2 for a, b in zip(s0, s1)) / R)
        res["read_batch"] = rb
        res["read_alone"] = stats(alone)
        res["read_beside_training"] = stats(beside)
        res["write_windows_per_step_per_owner"] = round(float(np.mean(windows)), 3)
        # ---- how long a window stays open: the kernels that hold the word odd -------------------------------------------
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                step(live, ids_for(B))
            torch.cuda.synchronize()
        names = ("k_evict_sweep", "k_rebuild_compact", "k_rebuild_clear", "k_rebuild_insert")
        per = {}
        for e in prof.events():
            if e.device_type is not None and "CUDA" in str(e.device_type) and any(n in e.name for n in names):
                key = next(n for n in names if n in e.name)
                per.setdefault(key, []).append(e.device_time / 1e3 if hasattr(e, "device_time") else e.cuda_time / 1e3)
        res["window_kernels_ms_max"] = {k: round(max(v), 4) for k, v in per.items()}
        res["window_ms_upper_bound"] = round(sum(max(v) for v in per.values()), 4)
        res["wait_budget_rounds"] = WAIT_SPINS
        res["wait_errors"] = [int(w.shard.counters()["wait_errors"]) for w in live]
        res["admitted"] = [int(w.shard.counters()["admitted"]) for w in live]
        res["index_stats_rank0"] = live[0].shard.index_stats()
    finally:
        for r in readers:
            r.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
