"""Tables larger than HBM on R GPUs: every rank's shard with a host-memory tier behind it (pb_table_attach_tier), served
through the sharded calls, unstaged and staged (pb_tier_stage_sharded through worker.TierStager), against the same
workload HBM-only, where eviction drops rows instead of moving them.

Workload: dim 96, Adagrad, `--slots` Zipf(1.05) slots of one id per sample, `--batch` samples per rank, a key space of
`--keys-per-hbm-row` times the HBM rows of all ranks; every training request runs an eviction check.  Each tier holds
every key its owner can own.  Both legs see the same batches and the same HBM rows per rank; their steps alternate in
one process.  A training step is forward (SEND / SERVE / FINISH) of every rank, then on every rank's stream a dense
stand-in (`--dense-iters` fp16 matmuls [batch, n] @ [n, n], standing in for the dense tower's step) and its backward.
The staged leg stages the next batch after the forwards, on the stagers' streams, so the owners' eviction checks and
restores run beside the dense stand-ins and the backwards:
    forward(i) -> [stager streams: stage(i + 1)] || [worker streams: dense stand-in, backward(i)] -> join
An inference step is one training=False forward of every rank.  Step times come from device events around the whole
step of all ranks.  Also reported per training step: restores done by the forwards, signs staged and stage restores
skipped, refused restores and moves out of HBM, and, from a separate torch.profiler run, the device time of
k_tier_restore_recv (unstaged: the forward's; staged: both instantiations), of k_owner_lookup_tier (inference) and of
the untiered leg's k_owner_lookup.  Prints one JSON line with the card's name and power limit read in the same run.

    python scripts/sharded_tier_bench.py [--ranks 2] [--hbm-rows 131072] [--steps 30] [--warmup 10]
        R virtual ranks on one GPU (one host thread drives them phase by phase)
    torchrun --nproc-per-node N scripts/sharded_tier_bench.py [...]
        N real ranks, one process per GPU, receive areas in symmetric memory
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def batches(rng, n, S, B, keys_per_slot):
    """n batches of S Zipf(1.05) slots, B ids each (slot-major), the ranks spread over the key space."""
    out = []
    for _ in range(n):
        z = (rng.zipf(1.05, size=S * B).astype(np.uint64) - np.uint64(1)) % np.uint64(keys_per_slot)
        out.append((z * np.uint64(0x9E3779B97F4A7C15) >> np.uint64(24)) % np.uint64(1 << 40))
    return out


class Leg:
    """The workers of one leg (all ranks of this process), their device batches, outputs and gradients."""

    def __init__(self, name, ws, ids, grads, S, B, dim, dense, pf, stagers=None):
        import torch

        self.name, self.ws, self.ids, self.grads, self.S, self.B = name, ws, ids, grads, S, B
        self.dense, self.pf, self.stagers = dense, pf, stagers or []
        self.outs = [torch.empty((S, B, dim), dtype=torch.float16, device=w.device) for w in ws]
        self.train_ms, self.infer_ms = [], []

    def enqueue(self, i, training):
        from persia_b200 import native as N

        phases = [N.PHASE_SEND, N.PHASE_SERVE, N.PHASE_FINISH] if len(self.ws) > 1 else [0]
        for ph in phases:
            for r, w in enumerate(self.ws):
                w.forward(self.ids[r][i], self.B, training=training, out=self.outs[r], phases=ph)
        if training:
            if self.stagers and i + 1 < len(self.ids[0]):
                so = [s * self.B for s in range(self.S + 1)]
                for ph in ([N.PHASE_SEND, N.PHASE_SERVE] if len(self.stagers) > 1 else [0]):
                    for r, st in enumerate(self.stagers):
                        st.stage(self.ids[r][i + 1], so, self.pf, phases=ph)
            for w in self.ws:
                self.dense(w._torch_stream())
            for ph in ([N.PHASE_SEND, N.PHASE_SERVE] if len(self.ws) > 1 else [0]):
                for r, w in enumerate(self.ws):
                    w.backward(self.grads[r], phases=ph)

    def timed(self, i, training):
        """Device events around the step of every rank of this process: every worker stream starts after `start` and
        `end` is recorded after all of them."""
        import torch

        cur = torch.cuda.current_stream()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record(cur)
        for w in self.ws:
            w._torch_stream().wait_event(start)
        self.enqueue(i, training)
        for s in [w._torch_stream() for w in self.ws] + [st.stream for st in self.stagers]:
            cur.wait_event(s.record_event())
        end.record(cur)
        end.synchronize()
        (self.train_ms if training else self.infer_ms).append(start.elapsed_time(end))

    def tier(self, field):
        if field in ("staged", "skipped"):
            return sum(int(w.shard.stage_stats()[field]) for w in self.ws)
        return sum(int(w.shard.tier_stats()[field]) for w in self.ws)


def dense_standin(n, iters, rows, dev):
    """A fixed loop of fp16 matmuls [rows, n] @ [n, n] on a given stream: the dense step a stage runs beside."""
    import torch

    x = torch.randn((rows, n), device=dev).half()
    w = (torch.randn((n, n), device=dev) / n ** 0.5).half()

    def run(stream):
        with torch.cuda.stream(stream):
            y = x
            for _ in range(iters):
                y = y @ w
        return y

    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ranks", type=int, default=2, help="virtual ranks on one GPU (ignored under torchrun)")
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--dim", type=int, default=96)
    ap.add_argument("--hbm-rows", type=int, default=1 << 17, help="HBM rows per rank")
    ap.add_argument("--keys-per-hbm-row", type=float, default=4.0)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--dense-n", type=int, default=4096, help="dense stand-in: [batch, n] @ [n, n] fp16 matmuls")
    ap.add_argument("--dense-iters", type=int, default=3, help="dense stand-in: matmuls per step and rank")
    args = ap.parse_args()
    import torch

    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W, TierStager

    assert torch.cuda.is_available(), "needs a GPU (there is no CPU fallback)"
    world = int(os.environ.get("WORLD_SIZE", "1"))
    dist_mode = world > 1
    if dist_mode:
        import torch.distributed as dist

        rank = int(os.environ["RANK"])
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dev = torch.device("cuda", torch.cuda.current_device())
        dist.init_process_group("nccl", device_id=dev)
        R, local = world, [rank]
    else:
        dev = torch.device("cuda", 0)
        R, local = args.ranks, list(range(args.ranks))
    S, B, dim, C = args.slots, args.batch, args.dim, args.hbm_rows
    keys = int(args.keys_per_hbm_row * C * R)
    tier_rows = int(keys / R * 1.25) + 4096  # every key its owner can own, with the farmhash spread's headroom
    pf = [(i + 1) << 56 for i in range(S)]
    opt = dict(kind=N.OPT_ADAGRAD, lr=0.01, initialization=0.01, eps=1e-10)
    n_steps = args.warmup + args.steps + args.profile_steps

    def group(tier):
        kw = dict(cap=S * B, optimizer=opt, max_batch=B, tier_rows=tier_rows if tier else 0)
        ws = [W.distributed(S, dim, pf, C, device=dev, **kw)] if dist_mode else W.local_group(R, S, dim, pf, C, **kw)
        for w in ws:
            w.shard.set_eviction(check_every=1, low_water=C // 4, target_free=C // 4, keep_batches=2)
            w.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=dev))  # storage, allocated before any step
        return ws

    ids, grads = [], []
    for r in local:
        rng = np.random.default_rng(1000 + r)
        ids.append([torch.from_numpy(b.view(np.int64)).to(dev) for b in batches(rng, n_steps, S, B, keys // S)])
        grads.append((torch.randn((S, B, dim), device=dev) * 1e-2).half())
    dense = dense_standin(args.dense_n, args.dense_iters, B, dev)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dense(torch.cuda.current_stream())
    a.record()
    for _ in range(20):
        dense(torch.cuda.current_stream())
    b.record()
    b.synchronize()
    dense_ms = a.elapsed_time(b) / 20

    def stagers(ws):
        if dist_mode:
            return [TierStager.distributed(ws[0].shard, S * B)]
        return TierStager.local_group([w.shard for w in ws], S * B)

    staged_ws = group(True)
    legs = [Leg("tier_unstaged", group(True), ids, grads, S, B, dim, dense, pf),
            Leg("tier_staged", staged_ws, ids, grads, S, B, dim, dense, pf, stagers(staged_ws)),
            Leg("hbm_only", group(False), ids, grads, S, B, dim, dense, pf)]
    torch.cuda.synchronize()
    fields = ("restored", "staged", "skipped", "refused", "moved_out")
    counts = {}
    for i in range(args.warmup + args.steps):
        if i == args.warmup:
            counts = {leg.name: {f: leg.tier(f) for f in fields} for leg in legs[:2]}
            for leg in legs:
                leg.train_ms.clear()
                leg.infer_ms.clear()
        for leg in legs:  # alternated: same batch, tier unstaged, tier staged, HBM-only
            leg.timed(i, True)
        for leg in legs:
            leg.timed(i, False)
    per_step = {}
    for leg in legs[:2]:
        d = {f: (leg.tier(f) - counts[leg.name][f]) / args.steps for f in fields}
        d["restored_by_forward"] = d["restored"] - d["staged"]
        per_step[leg.name] = d
    status = [w.status() for leg in legs for w in leg.ws + leg.stagers]

    # kernel time: a separate profiled run of a few steps per leg
    from torch.profiler import ProfilerActivity, profile

    names = ("k_tier_restore_recv<false>", "k_tier_restore_recv<true>", "k_stage_route", "k_owner_lookup_tier",
             "k_owner_lookup<", "k_tier_move", "k_tier_collect")
    kernel_us = {}
    for leg in legs:
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(args.warmup + args.steps, n_steps):
                leg.enqueue(i, True)
                leg.enqueue(i, False)
            torch.cuda.synchronize()
        tot = {n: 0.0 for n in names}
        for e in prof.key_averages():
            for n in names:
                if n in e.key:
                    tot[n] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        kernel_us[leg.name] = {n.rstrip("<"): round(v / max(args.profile_steps, 1), 1) for n, v in tot.items() if v}

    def stats(v):
        v = np.asarray(v)
        return {"median_ms": round(float(np.median(v)), 3), "mean_ms": round(float(v.mean()), 3),
                "min_ms": round(float(v.min()), 3), "max_ms": round(float(v.max()), 3)}

    res = {"card_and_power_limit": card(), "mode": f"torchrun x{R}" if dist_mode else f"{R} virtual ranks on one GPU",
           "slots": S, "batch_per_rank": B, "dim": dim, "hbm_rows_per_rank": C, "keys": keys,
           "tier_rows_per_rank": tier_rows, "steps": args.steps, "warmup": args.warmup,
           "dense_standin": f"{args.dense_iters} x [{B}, {args.dense_n}] @ [{args.dense_n}, {args.dense_n}] fp16 per rank",
           "dense_standin_ms_alone": round(dense_ms, 3),
           "train_step": {leg.name: stats(leg.train_ms) for leg in legs},
           "infer_step": {leg.name: stats(leg.infer_ms) for leg in legs},
           "tier_per_train_step": per_step, "kernel_us_per_step_profiled": kernel_us,
           "status_ok": all(s == (False, False) for s in status)}
    if dist_mode:
        import torch.distributed as dist

        out = [None] * world
        dist.all_gather_object(out, res)
        if dist.get_rank() == 0:
            print(json.dumps({"ranks": out}))
        dist.destroy_process_group()
    else:
        print(json.dumps(res))


if __name__ == "__main__":
    main()
