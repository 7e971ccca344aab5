"""Checkpoint loads at the metric shape (dim 128, Adagrad: 256 floats per entry): checkpoint.load_shards (host decode,
numpy stack) against checkpoint.DeviceLoader (pb_load.cu), and what a background load costs a training job.

Legs (--entries entries each, default 1e7: a 10.5 GB image in the writer layout):
  sync       one synchronous-dump file (dump_shards);
  background a background-dump directory (BackgroundDumper, 100 parts);
  reference  a file laid out as the reference's writer can leave it: list order a random permutation of the nodes,
             1 % free nodes (after the live ones, on the free list), dims 128 and 32 (half each, by node).
For each leg, each loader into fresh tables, both ending in a device synchronise:
  - whole-load wall seconds of load_shards and of the device loader, and image GB/s of the latter;
  - the device loader's split: file reads (reader thread), index calls (the host pass over a whole image plus the
    device selection, wall time) and the gathers and inserts (CUDA events on the loader's stream);
  - the training step's p50 / p99 (a forward + backward of --batch x --slots uniform ids over a separate range of
    signs, under the table's lock, timed to a synchronise) with no load, and beside a background load into the same
    table (the steps run until the load ends).
Files are written right before they are loaded, so the page cache likely still holds them ("repeat" reads: nothing here
drops the cache).  They go to a temporary directory (--dir), removed after each leg.  Prints the card's name and power
limit and one JSON line per leg.

    python scripts/load_bench.py [--entries 1e7] [--dir /scratch]
"""
import argparse
import gc
import json
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
MULT = 0x9E3779B97F4A7C15 - (1 << 64)  # signs k * an odd constant: distinct, spread over the index


def log(msg):
    print(f"[load_bench] {msg}", file=sys.stderr, flush=True)


def gpu_info():
    q = "name,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()
        return dict(zip(q.split(","), [x.strip() for x in out[0].split(",")])) if out else {}
    except (OSError, subprocess.SubprocessError):
        return {}


def pct(xs, q):
    return float(np.percentile(np.asarray(xs), q)) if xs else None


def tables(dims, cap):
    from persia_b200 import native as N
    from persia_b200.shard import EmbeddingShard

    out = {}
    for d in dims:
        sh = EmbeddingShard(d, cap, 0)
        sh.set_optimizer(N.OPT_ADAGRAD, lr=0.01, initialization=0.01)
        sh.configure()
        out[d] = sh
    return out


def release(tabs):
    import torch

    for t in tabs.values():
        t.close()
    tabs.clear()
    gc.collect()
    torch.cuda.empty_cache()


def reference_file(path, n, rng):
    """The reference-layout leg's file, written a block of nodes at a time."""
    from persia_b200 import checkpoint as CK

    n_a = n // 2  # dim 128 (256 floats), then dim 32 (64 floats)
    free = n // 100
    m = n + free
    order = rng.permutation(n).astype(np.int64)  # list position -> node
    nxt = np.zeros(n, np.uint32)
    prv = np.zeros(n, np.uint32)
    nxt[order[:-1]] = (order[1:] + 1).astype(np.uint32)
    prv[order[1:]] = (order[:-1] + 1).astype(np.uint32)
    with open(path, "wb") as f:
        f.write(np.array([n], "<u8").tobytes() + np.array([order[0] + 1, order[-1] + 1, n + 1 if free else 0, m, m],
                                                          "<u4").tobytes())
        for lo_g, hi_g, dim in ((0, n_a, 128), (n_a, n, 32)):
            L = 2 * dim
            for lo in range(lo_g, hi_g, 1 << 20):
                hi = min(hi_g, lo + (1 << 20))
                nodes = np.zeros(hi - lo, CK._node_dtype(L))
                nodes["next"], nodes["prev"], nodes["flag"], nodes["len"] = nxt[lo:hi], prv[lo:hi], 1, L
                nodes["inner"] = rng.standard_normal((hi - lo, L), dtype=np.float32)
                nodes["dim"] = dim
                nodes["sign"] = (np.arange(lo + 1, hi + 1, dtype=np.uint64) * np.uint64(MULT & (2**64 - 1)))
                f.write(nodes.tobytes())
        fr = np.zeros(free, np.dtype([("next", "<u4"), ("prev", "<u4"), ("flag", "u1")]))
        fr["next"] = np.arange(n + 2, m + 2, dtype=np.uint32)
        if free:
            fr["next"][-1] = 0
        f.write(fr.tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entries", type=float, default=1e7)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--slots", type=int, default=26)
    ap.add_argument("--steps", type=int, default=200, help="timed steps without a load")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--dir", default=None)
    ap.add_argument("--legs", default="sync,background,reference")
    args = ap.parse_args()

    import torch

    from persia_b200 import checkpoint as CK
    from persia_b200 import shard as SH

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    info = gpu_info()
    log(f"card: {info.get('name', torch.cuda.get_device_name(0))}, power limit {info.get('power.limit', 'unknown')}")
    n, B, S = int(args.entries), args.batch, args.slots
    train_rows = 1 << 20
    root = tempfile.mkdtemp(prefix="load_bench_", dir=args.dir)
    rng = np.random.default_rng(0)
    try:
        for leg in args.legs.split(","):
            d = os.path.join(root, leg)
            t0 = time.perf_counter()
            if leg in ("sync", "background"):
                src = tables((128,), n + 1024)
                for lo in range(0, n, 1 << 20):
                    k = torch.arange(lo + 1, min(n, lo + (1 << 20)) + 1, dtype=torch.int64, device=dev)
                    src[128].set_entries(k * MULT, torch.rand((k.numel(), 256), device=dev) * 0.02 - 0.01)
                if leg == "sync":
                    CK.dump_shards(d, [src[128]])
                else:
                    bg = CK.BackgroundDumper(d, [src[128]], n_parts=100)
                    while bg.step():
                        pass
                release(src)
                dims = (128,)
            else:
                os.makedirs(os.path.join(d, "s0"))
                reference_file(os.path.join(d, "s0", "replica_0_shard_0.emb"), n, rng)
                for p in (os.path.join(d, "s0", CK.DONE_FILE), os.path.join(d, CK.DONE_FILE)):
                    with open(p, "w") as f:
                        f.write(CK.done_yaml(1, 1))
                dims = (32, 128)
            files = [os.path.join(d, "s0", x) for x in os.listdir(os.path.join(d, "s0")) if x.endswith(".emb")]
            nbytes = sum(os.path.getsize(p) for p in files)
            log(f"{leg}: {len(files)} files, {nbytes / 1e9:.2f} GB written in {time.perf_counter() - t0:.1f} s")
            row = {"leg": leg, "entries": n, "files": len(files), "image_gb": nbytes / 1e9}

            def timed(fn):
                torch.cuda.synchronize()
                t = time.perf_counter()
                out = fn()
                torch.cuda.synchronize()
                return time.perf_counter() - t, out

            tabs = tables(dims, n + train_rows + 1024)
            row["load_shards_s"], _ = timed(lambda: CK.load_shards(d, tabs))
            release(tabs)
            tabs = tables(dims, n + train_rows + 1024)
            ld = CK.DeviceLoader(d, tabs)
            row["device_s"], _ = timed(ld.run)
            row["device_gb_s"] = nbytes / row["device_s"] / 1e9
            row["device_split"] = {k: round(v, 3) for k, v in ld.timings.items()}
            release(tabs)
            log(f"{leg}: load_shards {row['load_shards_s']:.2f} s, device {row['device_s']:.2f} s "
                f"({row['device_gb_s']:.2f} GB/s; {row['device_split']})")

            # training beside a background load into the same dim-128 table
            tabs = tables(dims, n + train_rows + 1024)
            sh, lock = tabs[128], threading.Lock()
            ctx = SH.BatchContext(S * B, S * B, [0] * S, device=0)
            ids = [(torch.randint(0, train_rows, (S * B,), device=dev) + n + 2) * MULT for _ in range(4)]
            grads = [(torch.randn((S, B, 128), device=dev) * 1e-3).half() for _ in range(4)]
            slot_off = [s * B for s in range(S + 1)]

            def step(i):
                t = time.perf_counter()
                with lock:
                    ctx.forward(sh, ids[i % 4], slot_off, B, training=True)
                with lock:
                    ctx.backward(sh, [grads[i % 4][s] for s in range(S)])
                torch.cuda.synchronize()
                return (time.perf_counter() - t) * 1e3

            for i in range(args.warmup):
                step(i)
            base = [step(i) for i in range(args.steps)]
            ld = CK.DeviceLoader(d, tabs, locks={128: lock})
            t = time.perf_counter()
            ld.start()
            during, i = [], 0
            while ld.running():
                during.append(step(i))
                i += 1
            ld.wait()
            row["background_load_s"] = time.perf_counter() - t
            row["step_ms_no_load"] = {"p50": pct(base, 50), "p99": pct(base, 99), "steps": len(base)}
            row["step_ms_background_load"] = {"p50": pct(during, 50), "p99": pct(during, 99), "steps": len(during)}
            ctx.close()
            release(tabs)
            shutil.rmtree(d)
            row.update(card=info.get("name"), power_limit=info.get("power.limit"))
            print(json.dumps(row), flush=True)
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
