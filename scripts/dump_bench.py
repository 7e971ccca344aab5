"""What an embedding checkpoint costs a training job at the metric shape (dim 128, Adagrad, 26 slots, batch 8192, one
GPU): the training step's median and p99 time with no dump and with a background dump in flight
(checkpoint.BackgroundDumper), the background dump's wall time, its encoder's rate (image bytes plus entry bytes read,
over the part kernels' time from CUDA events, timed in a run of their own), and the synchronous dump's wall time.

The table holds --rows resident entries (default 1e7: a 10.5 GB image, so that the file system can hold it); each step is
a forward + backward of uniform ids over them, issued under the table's lock as persia_core issues them, and timed from
its first call to a synchronise after its last.  The dump files go to a temporary directory (--dump-dir), removed after
each dump.  Prints the card's name and power limit and one JSON line, also written to --out/dump_bench.json.

    python scripts/dump_bench.py --out <dir> [--rows 1e7] [--steps 200]
"""
import argparse
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


def log(msg):
    print(f"[dump_bench] {msg}", file=sys.stderr, flush=True)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rows", type=float, default=1e7)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--slots", type=int, default=26)
    ap.add_argument("--steps", type=int, default=200, help="timed steps without a dump")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--n-parts", type=int, default=None, help="parts per table (default: the dumper's rule)")
    ap.add_argument("--timed-parts", type=int, default=20, help="parts timed with CUDA events for the encoder's rate")
    ap.add_argument("--dump-dir", default=None, help="where the dump files are written (default: a temporary directory)")
    args = ap.parse_args()

    import torch

    from persia_b200 import checkpoint as CK
    from persia_b200 import native as N
    from persia_b200 import shard as SH

    assert torch.cuda.is_available(), "needs a CUDA device"
    os.makedirs(args.out, exist_ok=True)
    dev = torch.device("cuda", 0)
    info = gpu_info()
    log(f"card: {info.get('name', torch.cuda.get_device_name(0))}, power limit {info.get('power.limit', 'unknown')}")
    rows, dim, B, S = int(args.rows), args.dim, args.batch, args.slots

    sh = SH.EmbeddingShard(dim, rows + rows // 8 + 1024, 0)
    sh.set_optimizer(N.OPT_ADAGRAD, lr=0.01, initialization=0.01)
    sh.configure()
    L = sh.entry_len
    mult = 0x9E3779B97F4A7C15 - (1 << 64)  # resident signs: k * an odd constant (distinct, spread over the index)
    fill = 1 << 20
    for lo in range(0, rows, fill):
        k = torch.arange(lo, min(rows, lo + fill), dtype=torch.int64, device=dev)
        sh.set_entries(k * mult, torch.rand((k.numel(), L), device=dev) * 0.02 - 0.01)
    torch.cuda.synchronize()
    log(f"{rows} rows resident ({len(sh)} counted), entry {L} floats, node {sh.node_bytes()} B")

    lock = threading.Lock()
    ctx = SH.BatchContext(S * B, S * B, [0] * S, device=0)
    n_sets = 4
    ids = [torch.randint(0, rows, (S * B,), device=dev) * mult for _ in range(n_sets)]
    grads = [(torch.randn((S, B, dim), device=dev) * 1e-3).half() for _ in range(n_sets)]
    slot_off = [s * B for s in range(S + 1)]

    def step(i):
        t0 = time.perf_counter()
        with lock:
            ctx.forward(sh, ids[i % n_sets], slot_off, B, training=True)
        with lock:
            ctx.backward(sh, [grads[i % n_sets][s] for s in range(S)])
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    for i in range(args.warmup):
        step(i)
    base = [step(i) for i in range(args.steps)]
    log(f"no dump: median {pct(base, 50):.3f} ms, p99 {pct(base, 99):.3f} ms")

    dump_root = tempfile.mkdtemp(prefix="dump_bench_", dir=args.dump_dir)
    try:
        # background dump in flight: steps go on until it ends
        d = CK.BackgroundDumper(os.path.join(dump_root, "bg"), [CK.DumpTable(sh, lock)], n_parts=args.n_parts)
        n_parts = d.n_parts
        t0 = time.perf_counter()
        d.start()
        during, i = [], 0
        while d.running():
            during.append(step(i))
            i += 1
        bg_wall = time.perf_counter() - t0
        d.wait()
        bg_bytes = sum(os.path.getsize(os.path.join(dump_root, "bg", "s0", f)) for f in os.listdir(os.path.join(dump_root, "bg", "s0")))
        log(f"background dump: {n_parts} parts, {bg_bytes / 1e9:.2f} GB in {bg_wall:.2f} s; {len(during)} steps beside it, "
            f"median {pct(during, 50):.3f} ms, p99 {pct(during, 99):.3f} ms")
        shutil.rmtree(os.path.join(dump_root, "bg"))

        # the encoder alone: parts timed with CUDA events (collect + sort + encode of one part)
        cap = 2 * (bg_bytes // n_parts) + 4096
        sh.dump_reserve(cap)
        image = torch.empty(cap, dtype=torch.uint8, device=dev)
        meta = torch.zeros(2, dtype=torch.int64, device=dev)
        st = torch.cuda.Stream(dev)
        ms, img_bytes, read_bytes = 0.0, 0, 0
        for k in range(min(args.timed_parts, n_parts)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            sh.dump_part(k, n_parts, image, meta, st)
            e1.record(st)
            e1.synchronize()
            ms += e0.elapsed_time(e1)
            nb = int(meta[0])
            assert nb <= cap
            img_bytes += nb
            read_bytes += (nb - 28) // sh.node_bytes() * L * 4
        sh.dump_release()
        del image
        enc_gbs = (img_bytes + read_bytes) / (ms * 1e-3) / 1e9
        log(f"encoder: {min(args.timed_parts, n_parts)} parts, {img_bytes / 1e9:.3f} GB image + {read_bytes / 1e9:.3f} GB "
            f"read in {ms:.2f} ms: {enc_gbs:.1f} GB/s")

        # the synchronous dump (training stopped)
        t0 = time.perf_counter()
        CK.dump_shards(os.path.join(dump_root, "sync"), [sh])
        sync_wall = time.perf_counter() - t0
        log(f"synchronous dump: {sync_wall:.2f} s")
        shutil.rmtree(os.path.join(dump_root, "sync"))
    finally:
        shutil.rmtree(dump_root, ignore_errors=True)

    res = dict(bench="dump_bench", card=info.get("name", torch.cuda.get_device_name(0)),
               power_limit=info.get("power.limit"), rows=rows, dim=dim, batch=B, slots=S, entry_floats=L,
               image_gb=bg_bytes / 1e9, n_parts=n_parts,
               step_ms_no_dump={"median": pct(base, 50), "p99": pct(base, 99), "steps": len(base)},
               step_ms_background_dump={"median": pct(during, 50), "p99": pct(during, 99), "steps": len(during)},
               background_dump_s=bg_wall, encoder_gb_s=enc_gbs, encoder_part_ms=ms / max(1, min(args.timed_parts, n_parts)),
               sync_dump_s=sync_wall)
    with open(os.path.join(args.out, "dump_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
