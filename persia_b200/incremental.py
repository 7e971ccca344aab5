"""Incremental updates in the reference's `.inc` packet format: how a model trained online reaches serving without full
checkpoints (persia-incremental-update-manager/src/lib.rs).

Training side: the tables keep the set of signs the optimizer stepped (pb_table_enable_incremental, on the device);
once the replica's sets hold more than `incremental_buffer_size` signs, persia_core takes them and hands one flush (the
signs' current entries) to an `IncrementalDumper`, which writes it on a thread of its own:

    incremental_dir/s{replica_index}/inc_%Y%m%d%H%M%S_{seq}/{replica_index}_{i}.inc   one file per writer, i = 0, 1, ...
    incremental_dir/s{replica_index}/inc_%Y%m%d%H%M%S_{seq}/inc_update_done           written once every file is

Each file is the persia-speedy encoding of PerisaIncrementalPacket { content: Vec<HashMapEmbeddingEntry>, timestamps }:
`count u32 | entry x count | unix seconds u64`, every entry laid out as in a checkpoint (checkpoint.entry_fields).

Serving side: an `IncrementalLoader` applies every complete directory (one with `inc_update_done`) it has not applied
yet, and skips the directories present when it started (lib.rs:314-364).

Deliberate differences from the reference (DESIGN.md §4 "Incremental update"): one directory per flush, named once
(the reference names it per file, so a flush can straddle two seconds); a `seq` suffix, unique within the process,
makes the names sort in flush order; no empty file when a flush holds fewer signs than writers (the reference's
`chunks(n / threads)` panics then); entries in ascending sign order (the reference: HashSet order); the loader applies
directories in name order and the files of one in index order, one after another (the reference's thread pool lets
two packets that hold one sign race), and comes back to a directory whose done file is not there yet (the reference
never looks at it again).
"""
import datetime
import itertools
import os
import queue
import re
import sys
import threading
import time

import numpy as np

from .checkpoint import entry_fields

DONE_FILE = "inc_update_done"
SCAN_INTERVAL_S = 10  # inc_dir_scan_thread's sleep (lib.rs:340)
JOB_TYPES = ("Train", "Eval", "Infer")  # PerisaJobType (persia-embedding-config/src/lib.rs:173-177)


# ------------------------------------------------------------------------------------------------ global config
def parse_global_config(gc):
    """The keys of the reference's global config (PERSIA_GLOBAL_CONFIG) this project reads, with the reference's
    defaults (persia-embedding-config/src/lib.rs:262-276, 298-375, 417-447).  capacity is None when unset."""
    gc = gc or {}
    common = gc.get("common_config") or {}
    ps = gc.get("embedding_parameter_server_config") or {}
    job = str(common.get("job_type", "Train"))
    if job not in JOB_TYPES:
        raise RuntimeError(f"common_config.job_type must be one of {JOB_TYPES}, got {job!r}")
    ck = common.get("checkpointing_config") or {}
    infer = common.get("infer_config") or {}
    cfg = dict(job_type=job, num_workers=int(ck.get("num_workers", 4)),
               embedding_checkpoint=infer.get("embedding_checkpoint") or None,
               capacity=int(ps["capacity"]) if ps.get("capacity") else None,
               enable_incremental_update=bool(ps.get("enable_incremental_update", False)),
               incremental_buffer_size=int(ps.get("incremental_buffer_size", 1_000_000)),
               incremental_dir=str(ps.get("incremental_dir", "/workspace/incremental_dir/")),
               incremental_channel_capacity=int(ps.get("incremental_channel_capacity", 1000)))
    if cfg["num_workers"] <= 0 or cfg["incremental_buffer_size"] <= 0 or cfg["incremental_channel_capacity"] <= 0:
        raise RuntimeError("checkpointing_config.num_workers, incremental_buffer_size and incremental_channel_capacity "
                           "must be positive")
    return cfg


# ------------------------------------------------------------------------------------------------ packet format
def records(signs, dim, entries):
    """Entries of one embedding dim as packet records: signs u64 [n], entries f32 [n, L]."""
    entries = np.asarray(entries, np.float32)
    n = np.asarray(signs).size
    rec = np.zeros(n, np.dtype(entry_fields(entries.shape[1] if entries.ndim == 2 else 0)))
    rec["len"], rec["dim"] = rec.dtype["inner"].shape[0], dim
    rec["sign"] = np.asarray(signs).view(np.uint64) if np.asarray(signs).dtype == np.int64 else signs
    if n:
        rec["inner"] = entries
    return rec


def packet_bytes(runs, timestamp):
    """A packet whose entries are the given record arrays (see `records`), one after another."""
    n = sum(r.size for r in runs)
    return b"".join([np.array([n], "<u4").tobytes()] + [r.tobytes() for r in runs] +
                    [np.array([int(timestamp)], "<u8").tobytes()])


def encode_packet(signs, dims, entries, timestamp=None):
    """PerisaIncrementalPacket of the given entries, in the given order.  signs u64 [n], dims embedding dim per entry,
    entries: f32 arrays (one per entry, any lengths) or one [n, L] array."""
    signs = np.ascontiguousarray(signs, np.uint64)
    dims = np.broadcast_to(np.asarray(dims, np.uint64), signs.shape)
    ts = int(time.time()) if timestamp is None else timestamp
    if isinstance(entries, np.ndarray) and entries.ndim == 2:
        return packet_bytes([records(signs, dims, entries)], ts)
    runs = []
    k = 0
    while k < signs.size:  # runs of one entry length
        L = np.asarray(entries[k]).size
        j = k
        while j < signs.size and np.asarray(entries[j]).size == L:
            j += 1
        runs.append(records(signs[k:j], dims[k:j], np.stack([np.asarray(e, np.float32) for e in entries[k:j]])))
        k = j
    return packet_bytes(runs, ts)


def decode_packet(buf):
    """Inverse of encode_packet: (signs u64 [n], dims u64 [n], entries list of f32 arrays, timestamp)."""
    buf = memoryview(buf)
    if len(buf) < 12:
        raise ValueError("truncated packet")
    n = int(np.frombuffer(buf[:4], "<u4")[0])
    off = 4
    signs, dims = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    entries = []
    k = 0
    while k < n:
        if len(buf) < off + 4:
            raise ValueError("truncated packet: entry")
        L = int(np.frombuffer(buf[off:off + 4], "<u4")[0])
        dt = np.dtype(entry_fields(L))
        # the longest run of entries of this length that fits (one vectorised view)
        m = min(n - k, (len(buf) - off - 8) // dt.itemsize)
        if m <= 0:
            raise ValueError("truncated packet: entry")
        rec = np.frombuffer(buf[off:off + m * dt.itemsize], dt)
        m = int(np.argmax(rec["len"] != L)) if (rec["len"] != L).any() else m
        rec = rec[:m]
        signs[k:k + m], dims[k:k + m] = rec["sign"], rec["dim"]
        entries.extend(np.array(rec["inner"], np.float32))
        off += m * dt.itemsize
        k += m
    if len(buf) != off + 8:
        raise ValueError("packet length does not match its entries")
    return signs, dims, entries, int(np.frombuffer(buf[off:off + 8], "<u8")[0])


# ------------------------------------------------------------------------------------------------ training side
_SEQ = itertools.count()
_SEQ_LOCK = threading.Lock()


def flush_dir_name(now=None):
    """inc_%Y%m%d%H%M%S + a sequence number unique within the process, zero-padded so that names sort in flush order.
    The time is UTC (the reference: chrono::Local): the loader applies directories in name order, and local time goes
    back an hour when daylight saving time ends."""
    with _SEQ_LOCK:
        seq = next(_SEQ)
    now = datetime.datetime.now(datetime.timezone.utc) if now is None else now
    return f"{now.strftime('inc_%Y%m%d%H%M%S')}_{seq:08d}"


class IncrementalDumper:
    """Writes flushes under incremental_dir/s{replica_index}: `submit` hands one over to a writer thread behind a
    queue of `channel_capacity` flushes (the reference's buffer_channel_output; a flush that finds it full is dropped
    with a warning, as there: lib.rs:286-288), `write` writes one in the calling thread.  A submitted flush may be a
    callable that returns the parts: the writer thread calls it (persia_core hands over device buffers that way, so that
    their copy to the host and the sort run here rather than on the training thread)."""

    def __init__(self, incremental_dir, replica_index=0, num_workers=4, channel_capacity=1000):
        self.dir = os.path.join(incremental_dir, f"s{int(replica_index)}")
        self.replica_index, self.num_workers = int(replica_index), max(1, int(num_workers))
        self._q = queue.Queue(maxsize=max(1, int(channel_capacity)))
        self._thread = None
        self.dropped_flushes = 0
        self.failed_flushes = 0
        self.written = []  # directories written, in flush order

    def write(self, parts, timestamp=None):
        """parts: [(signs u64 [n], dim, entries f32 [n, L])], one per table.  Returns the directory written, or None
        when the flush holds no sign (nothing is written)."""
        parts = [(np.asarray(s).view(np.uint64) if np.asarray(s).dtype == np.int64 else np.asarray(s, np.uint64), d, e)
                 for s, d, e in parts]
        recs = [records(s, d, e) for s, d, e in parts if np.asarray(s).size]
        if not recs:
            return None
        every = np.concatenate([r["sign"] for r in recs])
        table = np.concatenate([np.full(r.size, t, np.int32) for t, r in enumerate(recs)])
        row = np.concatenate([np.arange(r.size) for r in recs])
        order = np.argsort(every, kind="stable")
        n = order.size
        ts = int(time.time()) if timestamp is None else timestamp
        path = os.path.join(self.dir, flush_dir_name())
        os.makedirs(path, exist_ok=True)
        for i, chunk in enumerate(np.array_split(order, min(self.num_workers, n))):  # never an empty file
            tb = table[chunk]
            cuts = np.concatenate([[0], np.flatnonzero(np.diff(tb)) + 1, [chunk.size]])
            runs = [recs[tb[a]][row[chunk[a:b]]] for a, b in zip(cuts[:-1], cuts[1:])]
            with open(os.path.join(path, f"{self.replica_index}_{i}.inc"), "wb") as f:
                f.write(packet_bytes(runs, ts))
        with open(os.path.join(path, DONE_FILE), "w"):
            pass
        self.written.append(path)
        return path

    def submit(self, parts):
        if self._thread is None:
            self._thread = threading.Thread(target=self._run, name="persia-incremental-dump", daemon=True)
            self._thread.start()
        try:
            self._q.put_nowait(parts)
        except queue.Full:
            self.dropped_flushes += 1
            sys.stderr.write("[persia_b200] incremental update dropped: the dump queue is full, "
                             "try a bigger incremental_channel_capacity\n")

    def wait_queued(self, n):
        """Returns once at most `n` submitted flushes are waiting for the writer thread."""
        while self._thread is not None and self._q.qsize() > n:
            time.sleep(0.001)

    def flush(self):
        """Returns once every flush submitted so far is written."""
        if self._thread is not None:
            self._q.join()

    def close(self):
        if self._thread is not None:
            self.flush()
            self._q.put(None)
            self._thread.join(timeout=60)
            self._thread = None

    def _run(self):
        while True:
            parts = self._q.get()
            try:
                if parts is None:
                    return
                self.write(parts() if callable(parts) else parts)
            except Exception as e:  # noqa: BLE001 — logged, as the reference logs a failed packet (lib.rs:204-212)
                self.failed_flushes += 1
                sys.stderr.write(f"[persia_b200] failed to write an incremental update: {e!r}\n")
            finally:
                self._q.task_done()


# ------------------------------------------------------------------------------------------------ serving side
_INC_FILE = re.compile(r"^(\d+)_(\d+)\.inc$")


class IncrementalLoader:
    """Applies the flushes that appear under `directory` (incremental_dir/s{replica_index}).  apply(signs u64 [n],
    dims u64 [n], entries list) stores one packet's entries, decoded here, and returns how many it could not store;
    apply_file(path), when given instead, reads, decodes and stores one packet file itself (persia_core: on the device)
    and returns (how many it could not store, how many entries the packet held).  A file that cannot be read or applied is logged and counted (failed_files) and the scan goes
    on, as the reference's scanner does."""

    def __init__(self, directory, apply=None, interval=SCAN_INTERVAL_S, apply_file=None):
        if (apply is None) == (apply_file is None):
            raise ValueError("give one of apply and apply_file")
        self.dir, self.apply, self.apply_file, self.interval = directory, apply, apply_file, interval
        self.seen = set(self._dirs())  # present at start: not applied (lib.rs:324-333)
        self.applied = []
        self.entries_applied = 0
        self.entries_dropped = 0
        self.failed_files = 0
        self._lock = threading.Lock()
        self._stop = threading.Event()
        self._thread = None

    def _dirs(self):
        if not os.path.isdir(self.dir):
            return []
        return sorted(d for d in os.listdir(self.dir) if os.path.isdir(os.path.join(self.dir, d)))

    def poll(self):
        """Applies every complete directory not applied yet: directories in name order, the files of one in index
        order.  Returns the directories applied by this call."""
        done = []
        with self._lock:
            for d in self._dirs():
                path = os.path.join(self.dir, d)
                if d in self.seen or not os.path.isfile(os.path.join(path, DONE_FILE)):
                    continue  # (an incomplete directory is looked at again by the next poll)
                files = sorted((int(m.group(2)), f) for f in os.listdir(path) for m in [_INC_FILE.match(f)] if m)
                for _, f in files:
                    try:
                        if self.apply_file is not None:
                            dropped, n = (int(x) for x in self.apply_file(os.path.join(path, f)))
                        else:
                            with open(os.path.join(path, f), "rb") as fh:
                                signs, dims, entries, _ = decode_packet(fh.read())
                            dropped, n = int(self.apply(signs, dims, entries)), signs.size
                        self.entries_dropped += dropped
                        self.entries_applied += n
                    except Exception as e:  # noqa: BLE001 — a bad packet does not stop the catch-up (lib.rs:216-227)
                        self.failed_files += 1
                        sys.stderr.write(f"[persia_b200] failed to load incremental packet {os.path.join(path, f)}: {e!r}\n")
                self.seen.add(d)
                self.applied.append(d)
                done.append(d)
        return done

    def start(self):
        """Polls every `interval` seconds on a daemon thread until stop()."""
        if self._thread is None:
            self._stop.clear()
            self._thread = threading.Thread(target=self._run, name="persia-incremental-load", daemon=True)
            self._thread.start()

    def stop(self):
        if self._thread is not None:
            self._stop.set()
            self._thread.join(timeout=60)
            self._thread = None

    def _run(self):
        while not self._stop.wait(self.interval):
            try:
                self.poll()
            except Exception as e:  # noqa: BLE001 — a bad packet is logged, the scanner goes on
                sys.stderr.write(f"[persia_b200] failed to load an incremental update: {e!r}\n")
