"""What incremental updates cost at the metric shape (dim 128, 26 slots, batch 8192, Adagrad, one GPU): the training
step with the table's set of updated signs enabled versus not, and one flush at incremental_buffer_size signs: the part
persia_core runs on the training thread (device take + entry gather + one sync) and the part its dumper thread runs
(device-to-host copy + sort).

Both step legs replay CUDA graphs of forward + backward over rotating buffer sets and are timed with device events, as
bench.py times its metric leg; they run on one table, alternating in chunks of --chunk steps, so both see the same
table and clocks.  Between chunks (untimed) the set is emptied once it holds more than the buffer size, as a trainer's
flushes would.  Prints one JSON line.

    python scripts/incremental_bench.py [--rows 5e7] [--steps 200] [--buffer 1000000]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def log(msg):
    print(f"[incremental_bench] {msg}", file=sys.stderr, flush=True)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()
        return dict(zip(q.split(","), [x.strip() for x in out[0].split(",")])) if out else {}
    except (OSError, subprocess.SubprocessError):
        return {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=5e7)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--chunk", type=int, default=4)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--slots", type=int, default=26)
    ap.add_argument("--alpha", type=float, default=1.05)
    ap.add_argument("--sets", type=int, default=8)
    ap.add_argument("--buffer", type=int, default=1_000_000, help="incremental_buffer_size")
    args = ap.parse_args()

    import torch

    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200 import workload as W

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    S, B, dim, rows = args.slots, args.batch, args.dim, int(args.rows)
    card = W.scaled_cardinalities(rows, S)
    pf = W.index_prefixes(S)
    slot_off = [s * B for s in range(S + 1)]
    sh = SH.EmbeddingShard(dim, rows + 1024, dev)
    sh.set_optimizer(N.OPT_ADAGRAD, lr=0.01, initialization=0.01, eps=1e-10)
    sh.configure()
    ctx = SH.BatchContext(S * B, S * B, pf, device=dev)
    chunk = 1 << 21
    buf = torch.empty((chunk, dim), dtype=torch.float32, device=dev)
    for s in range(S):  # every id of every slot resident (bench.py's warm table)
        for lo in range(0, int(card[s]), chunk):
            hi = min(int(card[s]), lo + chunk)
            signs = SH.add_prefix(torch.arange(lo, hi, dtype=torch.int64, device=dev), [0, hi - lo], [pf[s]])
            sh.lookup(signs, training=True, out=buf[:signs.numel()])
    torch.cuda.synchronize()
    del buf
    log(f"table filled: {len(sh)} rows")
    n_sets = max(2, args.sets)
    ids_host = W.make_batches(2, card, B, n_sets, args.alpha)
    ids = [torch.from_numpy(ids_host[k].view(np.int64)).to(dev) for k in range(n_sets)]
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    grads = (torch.randn((n_sets, S, B, dim), generator=g, device=dev) * 1e-2).half()
    outs = [torch.empty((S, B, dim), dtype=torch.float16, device=dev) for _ in range(n_sets)]

    def step(k):
        ctx.forward(sh, ids[k], slot_off, B, training=True, out=outs[k])
        ctx.backward(sh, [grads[k, s] for s in range(S)])

    stream = torch.cuda.Stream(device=dev)
    graphs = {}
    with torch.cuda.stream(stream):
        for on in (False, True):
            sh.enable_incremental(2 * args.buffer if on else 0)
            for i in range(3):
                step(i % n_sets)
            stream.synchronize()
            graphs[on] = []
            for k in range(n_sets):
                gph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gph, stream=stream):
                    step(k)
                graphs[on].append(gph)
        sh.take_incremental()
        log("graphs captured")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ms = {False: 0.0, True: 0.0}
        n = {False: 0, True: 0}
        i = 0
        for warm in (True, False):
            todo = max(args.chunk, args.steps // 10) if warm else args.steps
            done = 0
            while done < todo:
                for on in (False, True):
                    torch.cuda.synchronize()
                    ev[0].record(stream)
                    for j in range(args.chunk):
                        graphs[on][(i + j) % n_sets].replay()
                    ev[1].record(stream)
                    torch.cuda.synchronize()
                    if not warm:
                        ms[on] += ev[0].elapsed_time(ev[1])
                        n[on] += args.chunk
                    if on and sh.incremental_held() > args.buffer:
                        sh.take_incremental()
                i += args.chunk
                done += args.chunk
        stats = sh.incremental_stats()
        log(f"steps timed: {stats}")
        log(f"step ms off {ms[False] / n[False]:.5f} on {ms[True] / n[True]:.5f}")
        # one flush at the buffer size: the rotating batches repeat their signs, so the set is filled past the buffer
        # by stepping that many resident signs of the largest slot with zero gradients (pb_update marks them; an
        # Adagrad step with a zero gradient leaves the entry as it is)
        big = int(np.argmax(card))
        want = min(args.buffer + 1, int(card[big]))
        fill = SH.add_prefix(torch.arange(want, dtype=torch.int64, device=dev), [0, want], [pf[big]])
        zeros = torch.zeros((want, dim), dtype=torch.float32, device=dev)

        def refill():
            sh.take_incremental()
            sh.update(fill, zeros)
            torch.cuda.synchronize()

        refill()
        held = sh.incremental_held()
        log(f"set filled to {held} signs")
        torch.cuda.synchronize()
        # persia_core's flush: the device half runs on the training thread (take, gather, one sync to read the count),
        # the host half (copy out, sort) on the dumper's thread
        import threading

        from persia_b200 import persia_core as PC

        t0 = time.perf_counter()
        host_half = PC._take_flush({dim: {"shard": sh, "lock": threading.RLock()}}, 2 * args.buffer)
        t1 = time.perf_counter()
        taken, ent = host_half()[0][0::2]
        t2 = time.perf_counter()
        skipped = held - taken.size
        # the device take alone, on a set refilled to the same size
        refill()
        count = torch.zeros(1, dtype=torch.int32, device=dev)
        out = torch.empty(2 * args.buffer + 16, dtype=torch.int64, device=dev)
        import ctypes as C

        st = C.c_void_p(stream.cuda_stream)
        ev[0].record(stream)
        N.check(sh.lib.pb_inc_take(sh.h, C.c_void_p(out.data_ptr()), out.numel(), C.c_void_p(count.data_ptr()), st))
        ev[1].record(stream)
        torch.cuda.synchronize()
        take_ms = ev[0].elapsed_time(ev[1])
        sel = torch.from_numpy(taken).to(dev)
        ev[0].record(stream)
        sh.get_entries(sel)
        ev[1].record(stream)
        torch.cuda.synchronize()
        get_ms = ev[0].elapsed_time(ev[1])
    off, on = ms[False] / n[False], ms[True] / n[True]
    res = {
        "workload": f"{S} slots, dim {dim}, batch {B}, {rows:.3g} resident rows, Adagrad, forward + backward, CUDA graphs",
        "gpu": gpu_info(),
        "step_ms_set_off": round(off, 5), "step_ms_set_on": round(on, 5),
        "mark_us_per_step": round((on - off) * 1e3, 2), "mark_share": round((on - off) / off, 4),
        "steps_timed_each": n[False], "set_stats_after_timing": stats,
        "flush": {"signs_held": int(held), "signs_taken_resident": int(taken.size), "skipped": int(skipped),
                  "training_thread_ms": round((t1 - t0) * 1e3, 2), "dumper_thread_ms": round((t2 - t1) * 1e3, 2),
                  "device_take_ms": round(take_ms, 3),
                  "get_entries_ms": round(get_ms, 3), "entry_bytes": int(ent.nbytes)},
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
