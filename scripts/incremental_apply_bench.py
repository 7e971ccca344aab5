"""Applying incremental-update packets on an Infer job at the metric shape (dim 128, Adagrad: 256 floats per entry):
the host path (read the file, incremental.decode_packet, persia_core._apply_incremental: set_entries, then get_entries
to count drops) against the device path (persia_core._apply_packet_file: one pinned buffer, pb_image_packet, the
inserts through pb_image_insert, drops from the tables' counters).

The packets are one flush as training writes it (IncrementalDumper.write): --files files of --entries entries each,
default 4 x 2.5e5 (one file of the default 1e6-sign flush across 4 writers, about 261 MB).  For each path, into a fresh
table of its own:
  - the wall time of each file, applied alone, up to a device synchronise (the first file of the device path also
    allocates its pinned buffer);
  - the p50 / p99 of the inference forwards (pb_forward, training = 0, --batch x --slots ids drawn from the flushed
    signs, under the table's lock as persia_core serves them, each timed to a synchronise of its own stream) that a
    second thread makes on the same table: with no packet applying, and while the files apply again into a fresh
    table (the forwards run until the last file is applied).
The files go to a temporary directory (--dir), removed at the end; they are read right after they are written, so the
page cache likely still holds them.  Prints the card's name and power limit and one JSON line per path.

    python scripts/incremental_apply_bench.py [--entries 2.5e5] [--files 4] [--dir /scratch]
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
MULT = 0x9E3779B97F4A7C15 - (1 << 64)  # signs k * an odd constant: distinct, spread over the index


def log(msg):
    print(f"[incremental_apply_bench] {msg}", file=sys.stderr, flush=True)


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
    ap.add_argument("--entries", type=float, default=2.5e5, help="entries per file")
    ap.add_argument("--files", type=int, default=4)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--slots", type=int, default=26)
    ap.add_argument("--forwards", type=int, default=200, help="timed forwards with no packet applying")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--dir", default=None)
    args = ap.parse_args()

    import torch

    from persia_b200 import incremental as INC
    from persia_b200 import native as N
    from persia_b200 import persia_core as PC
    from persia_b200 import shard as SH

    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    info = gpu_info()
    log(f"card: {info.get('name', torch.cuda.get_device_name(0))}, power limit {info.get('power.limit', 'unknown')}")
    n, F, B, S, dim = int(args.entries), args.files, args.batch, args.slots, 128
    total = n * F
    root = tempfile.mkdtemp(prefix="incremental_apply_bench_", dir=args.dir)
    try:
        t0 = time.perf_counter()
        rng = np.random.default_rng(0)
        signs = np.arange(1, total + 1, dtype=np.uint64) * np.uint64(MULT & (2**64 - 1))
        entries = rng.standard_normal((total, 2 * dim), dtype=np.float32) * np.float32(0.01)
        flush = INC.IncrementalDumper(root, 0, num_workers=F).write([(signs, dim, entries)], timestamp=1)
        del entries
        paths = [os.path.join(flush, f"0_{i}.inc") for i in range(F)]
        nbytes = [os.path.getsize(p) for p in paths]
        log(f"{F} files of {n} entries ({nbytes[0] / 1e6:.0f} MB each) written in {time.perf_counter() - t0:.1f} s")

        def table():
            sh = SH.EmbeddingShard(dim, total + 1024, 0)
            sh.set_optimizer(N.OPT_ADAGRAD, lr=0.01, initialization=0.01)
            sh.configure()
            return {dim: {"shard": sh, "lock": threading.RLock(), "device": 0}}

        def host_apply(path, groups):
            with open(path, "rb") as f:
                s, d, e, _ = INC.decode_packet(f.read())
            return PC._apply_incremental(s, d, e, groups=groups)

        paths_of = {"host": host_apply, "device": lambda p, g: PC._apply_packet_file(p, groups=g)[0]}
        sign_dev = torch.from_numpy(signs.view(np.int64)).to(dev)
        ids = [sign_dev[torch.randint(0, total, (S * B,), device=dev)] for _ in range(4)]
        slot_off = [s * B for s in range(S + 1)]
        for name, apply in paths_of.items():
            row = {"path": name, "files": F, "entries_per_file": n, "file_mb": nbytes[0] / 1e6}
            groups = table()
            walls, dropped = [], 0
            for p in paths:
                torch.cuda.synchronize()
                t = time.perf_counter()
                dropped += apply(p, groups)
                torch.cuda.synchronize()
                walls.append(time.perf_counter() - t)
            assert dropped == 0 and len(groups[dim]["shard"]) == total
            row["file_s"] = [round(w, 4) for w in walls]
            row["file_s_median"] = float(np.median(walls))
            row["file_gb_s_median"] = nbytes[0] / row["file_s_median"] / 1e9
            groups[dim]["shard"].close()

            # inference forwards on a second thread, on the table being applied to
            groups = table()
            sh, lock = groups[dim]["shard"], groups[dim]["lock"]
            ctx = SH.BatchContext(S * B, S * B, [0] * S, device=0)
            fs = torch.cuda.Stream(dev)

            def forward(i):
                t = time.perf_counter()
                with torch.cuda.stream(fs):
                    with lock:
                        ctx.forward(sh, ids[i % 4], slot_off, B, training=False)
                    fs.synchronize()
                return (time.perf_counter() - t) * 1e3

            for i in range(args.warmup):
                forward(i)
            base = [forward(i) for i in range(args.forwards)]
            done = threading.Event()
            during = []

            def serve():
                i = 0
                while not done.is_set():
                    during.append(forward(i))
                    i += 1

            th = threading.Thread(target=serve)
            th.start()
            t = time.perf_counter()
            try:
                for p in paths:
                    apply(p, groups)
                torch.cuda.synchronize()
            finally:
                done.set()
                th.join()
            row["apply_beside_forwards_s"] = time.perf_counter() - t
            row["forward_ms_no_apply"] = {"p50": pct(base, 50), "p99": pct(base, 99), "forwards": len(base)}
            row["forward_ms_during_apply"] = {"p50": pct(during, 50), "p99": pct(during, 99), "forwards": len(during)}
            ctx.close()
            sh.close()
            row.update(card=info.get("name"), power_limit=info.get("power.limit"))
            log(f"{name}: file median {row['file_s_median']:.3f} s; forward p50/p99 {row['forward_ms_no_apply']['p50']:.2f}/"
                f"{row['forward_ms_no_apply']['p99']:.2f} ms alone, {row['forward_ms_during_apply']['p50']:.2f}/"
                f"{row['forward_ms_during_apply']['p99']:.2f} ms during")
            print(json.dumps(row), flush=True)
    finally:
        PC.reset()
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
