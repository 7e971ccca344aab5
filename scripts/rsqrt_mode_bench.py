"""What Adagrad's intel rsqrt mode (EmbeddingShard.set_rsqrt("intel"): a table load per fused element) costs against the
exact mode (an IEEE div + sqrt per element), on one GPU.

  graph    the training step (forward + backward, Adagrad) captured as CUDA graphs on one table, one graph per mode
           (a graph keeps the mode it was captured with), replays timed with device events, the modes alternating
           round by round; at the metric leg's shape (26 slots, dim 128, batch 8192) and configs[1]'s (26 slots, dim
           64, batch 4096), over a resident table of --rows rows of Zipf ids (bench.py's workload)
  kernels  torch.profiler kernel times per mode of k_reduce_cold (one GPU, the metric shape) and k_owner_update_all
           (R = 2 virtual ranks on the GPU, 26 slots, dim 128, batch 8192 per rank, eager steps)

Prints one JSON line with the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def kernel_us(torch, fn, names, reps):
    """Mean device time per call of fn (us) of every kernel whose name holds one of `names`."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        for n in names:
            if n in e.name:
                out[n] += e.device_time / reps if hasattr(e, "device_time") else e.cuda_time / reps
    return out


def local_leg(torch, args, dim, B):
    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200 import workload as W

    dev = torch.device("cuda", 0)
    S = 26
    card_ = W.scaled_cardinalities(args.rows, S)
    pf = W.index_prefixes(S)
    slot_off = [s * B for s in range(S + 1)]
    sh = SH.EmbeddingShard(dim, int(args.rows) + 1024, dev)
    sh.set_optimizer(N.OPT_ADAGRAD, lr=0.01, initialization=0.01, eps=1e-10)
    sh.configure()
    ctx = SH.BatchContext(S * B, S * B, pf, device=dev)
    chunk = 1 << 21
    buf = torch.empty((chunk, dim), dtype=torch.float32, device=dev)
    for s in range(S):
        for lo in range(0, int(card_[s]), chunk):
            hi = min(int(card_[s]), lo + chunk)
            sh.lookup(SH.add_prefix(torch.arange(lo, hi, dtype=torch.int64, device=dev), [0, hi - lo], [pf[s]]),
                      training=True, out=buf[: hi - lo])
    del buf
    n_sets = 4
    ids = [torch.from_numpy(x.view(np.int64)).to(dev) for x in W.make_batches(2, card_, B, n_sets, 1.05)]
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
        for mode in ("exact", "intel"):
            sh.set_rsqrt(mode)
            for i in range(3):
                step(i % n_sets)
            stream.synchronize()
            graphs[mode] = []
            for k in range(n_sets):
                gph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gph, stream=stream):
                    step(k)
                graphs[mode].append(gph)
        ms = {"exact": [], "intel": []}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for r in range(args.rounds):
            for mode in (("exact", "intel") if r % 2 == 0 else ("intel", "exact")):
                for i in range(args.warmup):
                    graphs[mode][i % n_sets].replay()
                e0.record(stream)
                for i in range(args.steps):
                    graphs[mode][i % n_sets].replay()
                e1.record(stream)
                stream.synchronize()
                ms[mode].append(e0.elapsed_time(e1) / args.steps)
        kern = {}
        for mode in ("exact", "intel"):  # eager steps: the kernels the graphs replay
            sh.set_rsqrt(mode)
            it = iter(range(1 << 30))
            kern[mode] = kernel_us(torch, lambda: step(next(it) % n_sets), ["k_reduce_cold", "k_reduce_warm", "k_step_hot"],
                                   args.steps)
    torch.cuda.synchronize()
    return {"dim": dim, "batch": B, "rows": args.rows,
            "ms_per_step": {m: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
                            for m, v in ms.items()},
            "kernel_us_per_step": kern}


def sharded_leg(torch, args):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as WK

    R, S, B, dim = 2, 26, 8192, 128
    rng = np.random.default_rng(0)
    card_ = rng.integers(10, 2_000_000, size=S)
    pf = [(i + 1) << 56 for i in range(S)]
    ws = WK.local_group(R, S, dim, pf, 1 << 22, cap=S * B, max_batch=B,
                        optimizer=dict(kind=N.OPT_ADAGRAD, lr=0.01, initialization=0.01, eps=1e-10))
    for x in ws:
        x.shard.get_entries(torch.zeros(1, dtype=torch.int64, device="cuda"))
    batches = [[torch.from_numpy(np.concatenate([rng.integers(0, c, size=B, dtype=np.uint64) for c in card_])
                                 .view(np.int64)).cuda() for _ in range(R)] for _ in range(4)]
    grads = [(torch.randn((S, B, dim), device="cuda") * 1e-2).half() for _ in range(R)]
    outs = [torch.empty((S, B, dim), dtype=torch.float16, device="cuda") for _ in range(R)]
    it = [0]

    def step():
        ids = batches[it[0] % len(batches)]
        it[0] += 1
        WK.group_forward(ws, ids, B, outs=outs)
        WK.group_backward(ws, grads)

    res = {}
    for _ in range(3):
        step()
    for mode in ("exact", "intel", "exact", "intel"):
        for x in ws:
            x.shard.set_rsqrt(mode)
        step()
        k = kernel_us(torch, step, ["k_owner_update_all", "k_owner_update<"], args.steps)
        res.setdefault(mode, []).append(k)
    torch.cuda.synchronize()
    return {"R": R, "dim": dim, "batch_per_rank": B,
            "kernel_us_per_step": {m: {n: float(np.mean([r[n] for r in v])) for n in v[0]} for m, v in res.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=2e7)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=6)
    args = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "needs a GPU"
    before = card()
    out = {"card_before": before,
           "metric_shape": local_leg(torch, args, 128, 8192),
           "configs1_shape": local_leg(torch, args, 64, 4096),
           "virtual_ranks": sharded_leg(torch, args),
           "card_after": card()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
