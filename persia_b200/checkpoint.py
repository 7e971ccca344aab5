"""Embedding checkpoints in the reference's on-disk format (SURVEY.md N2).

What the reference writes (persia-model-manager/src/lib.rs:242-343): under `<dir>/s{replica_index}/` one file
`replica_{r}_shard_{i}.emb` per internal shard of the parameter server, each the persia-speedy encoding
(little endian, `usize` as u64, u32 length prefixes — persia-speedy/src/writable_impl.rs:158-162,
private.rs:110-116) of that shard's `ArrayLinkedList<HashMapEmbeddingEntry>`:

    count u64 | first_index u32 | last_index u32 | free_index u32 | end_index u32 | n_nodes u32 | nodes...
    node  = next_index u32 | prev_index u32 | flag u8 | [entry if flag != 0]          (array_linked_list.rs:137-213)
    entry = len u32 | len x f32 (embedding ++ optimizer state) | embedding_dim u64 | sign u64   (emb_entry.rs:17-25)

Node indices are 1-based positions in the node array, 0 = none; the list runs from `first_index` along
`next_index` (least recently used first), unused nodes hang off `free_index` with flag 0
(array_linked_list.rs:215-272).  `embedding_dump_done` (YAML: num_shards, num_internal_shards, datetime) marks a
complete shard directory and, written by replica 0, a complete checkpoint (lib.rs:150-198).  A server loads every
`.emb` of its own `s{r}` directory and inserts the entries in list order (lib.rs:259-273, PS mod.rs:460-466).

PARITY UNPINNED: the reference cannot run here and ships no checkpoint fixture, so the byte layout above is a
restatement of its (de)serialisation code; tests pin this module against hand-laid-out bytes and round trips.

This module is host-side file format code over EmbeddingShard.export_signs / get_entries / set_entries; the rows
themselves never leave the GPU except through those calls.
"""
import os
import time

import numpy as np

DONE_FILE = "embedding_dump_done"


# ------------------------------------------------------------------------------------------------ format
def entry_fields(entry_len):
    """One HashMapEmbeddingEntry as speedy writes it (emb_entry.rs:17-25): len u32 | f32 x len | embedding_dim u64 |
    sign u64.  Incremental-update packets (persia_b200/incremental.py) carry the same entries."""
    return [("len", "<u4"), ("inner", "<f4", (entry_len,)), ("dim", "<u8"), ("sign", "<u8")]


def _node_dtype(entry_len):
    return np.dtype([("next", "<u4"), ("prev", "<u4"), ("flag", "u1")] + entry_fields(entry_len))


def encode_list(signs, entries, dims):
    """One ArrayLinkedList whose list order is the given order.  signs u64 [n]; entries: list of float32 arrays
    (or one [n, L] array); dims: embedding_dim per entry (scalar or [n])."""
    signs = np.ascontiguousarray(signs, dtype=np.uint64)
    n = signs.size
    dims = np.broadcast_to(np.asarray(dims, dtype=np.uint64), (n,))
    head = np.zeros(1, np.dtype([("count", "<u8"), ("first", "<u4"), ("last", "<u4"), ("free", "<u4"), ("end", "<u4"),
                                 ("n", "<u4")]))
    head["count"], head["first"], head["last"], head["n"] = n, (1 if n else 0), n, n
    out = [head.tobytes()]
    if isinstance(entries, np.ndarray) and entries.ndim == 2:  # uniform entry length: one vectorised block
        nodes = np.zeros(n, _node_dtype(entries.shape[1]))
        nodes["next"] = np.arange(2, n + 2, dtype=np.uint32)
        if n:
            nodes["next"][-1] = 0
        nodes["prev"] = np.arange(0, n, dtype=np.uint32)
        nodes["flag"], nodes["len"] = 1, entries.shape[1]
        nodes["inner"], nodes["dim"], nodes["sign"] = entries, dims, signs
        out.append(nodes.tobytes())
    else:
        for i in range(n):
            e = np.ascontiguousarray(entries[i], dtype="<f4")
            out.append(np.array([i + 2 if i + 1 < n else 0, i], "<u4").tobytes() + b"\x01" +
                       np.array([e.size], "<u4").tobytes() + e.tobytes() +
                       np.array([dims[i], signs[i]], "<u8").tobytes())
    return b"".join(out)


def decode_list(buf):
    """Inverse of the reference's writer for any ArrayLinkedList<HashMapEmbeddingEntry> (free nodes, arbitrary node
    order).  Returns (signs u64 [n], dims u64 [n], entries list of float32 arrays) in list order."""
    buf = memoryview(buf)
    if len(buf) < 28:
        raise ValueError("truncated checkpoint: header")
    count = int(np.frombuffer(buf[:8], "<u8")[0])
    first, last, free, end, n_nodes = (int(x) for x in np.frombuffer(buf[8:28], "<u4"))
    off = 28
    # fast path: every node in use and of one length -> one structured view
    if n_nodes and count == n_nodes and len(buf) >= off + 13:
        L = int(np.frombuffer(buf[off + 9:off + 13], "<u4")[0])
        dt = _node_dtype(L)
        if buf[off + 8] == 1 and len(buf) - off == n_nodes * dt.itemsize:
            nodes = np.frombuffer(buf[off:], dt)
            if (nodes["flag"] == 1).all() and (nodes["len"] == L).all():
                order = _walk(nodes["next"], first, count)
                return nodes["sign"][order].copy(), nodes["dim"][order].copy(), list(nodes["inner"][order])
    nxt = np.zeros(n_nodes, np.uint32)
    signs, dims, entries, live = np.zeros(n_nodes, np.uint64), np.zeros(n_nodes, np.uint64), [None] * n_nodes, []
    for i in range(n_nodes):
        if len(buf) < off + 9:
            raise ValueError("truncated checkpoint: node")
        nxt[i] = np.frombuffer(buf[off:off + 4], "<u4")[0]
        flag = buf[off + 8]
        off += 9
        if flag:
            L = int(np.frombuffer(buf[off:off + 4], "<u4")[0])
            if len(buf) < off + 4 + 4 * L + 16:
                raise ValueError("truncated checkpoint: entry")
            entries[i] = np.frombuffer(buf[off + 4:off + 4 + 4 * L], "<f4").copy()
            dims[i], signs[i] = np.frombuffer(buf[off + 4 + 4 * L:off + 20 + 4 * L], "<u8")
            off += 20 + 4 * L
            live.append(i)
    if off != len(buf):
        raise ValueError("trailing bytes after the node array")
    if len(live) != count:
        raise ValueError(f"checkpoint says {count} entries, {len(live)} nodes hold one")
    order = _walk(nxt, first, count)
    if any(entries[i] is None for i in order):
        raise ValueError("the list runs through an unused node")
    return signs[order], dims[order], [entries[i] for i in order]


def _walk(nxt, first, count):
    order = np.empty(count, np.int64)
    cur = first
    for k in range(count):
        if cur == 0 or cur > nxt.size:
            raise ValueError("broken list: it ends before `count` entries")
        order[k] = cur - 1
        cur = int(nxt[cur - 1])
    if cur != 0:
        raise ValueError("broken list: it continues past `count` entries")
    return order


def done_yaml(num_shards, num_internal_shards, now=None):
    """EmbeddingModelInfo as serde_yaml writes it (lib.rs:52-61, 150-170)."""
    now = time.time() if now is None else now
    secs = int(now)
    return (f"---\nnum_shards: {num_shards}\nnum_internal_shards: {num_internal_shards}\ndatetime:\n"
            f"  secs_since_epoch: {secs}\n  nanos_since_epoch: {int((now - secs) * 1e9)}\n")


def list_header(n):
    """The 28-byte header of a list of n entries in list order (encode_list's, without the nodes)."""
    return np.array([n], "<u8").tobytes() + np.array([1 if n else 0, n, 0, 0, n], "<u4").tobytes()


# ------------------------------------------------------------------------------------------------ dump / load
SLICE_BYTES = 256 << 20  # device staging of one slice of the synchronous dump, and the part size a background dump aims at


def dump_shards(dst_dir, shards, replica_index=0, replica_size=1, chunk=1 << 20, locks=None, fences=None):
    """EmbeddingModelManager.dump_embedding for one parameter-server replica.  `shards`: the EmbeddingShards (one per
    embedding dim) this replica holds; each becomes one `.emb` file ("internal shard").  The nodes are encoded on the
    device (pb_dump_nodes) at most `chunk` entries and SLICE_BYTES at a time, in export_signs' order.  locks: one lock per
    shard, held while that shard is read (the calls on a table come from one host thread at a time); fences: one
    ShardedFence (or None) per shard, ordering the reads against the sharded calls of R GPUs."""
    import contextlib

    import torch

    shard_dir = os.path.join(dst_dir, f"s{replica_index}")
    os.makedirs(shard_dir, exist_ok=True)
    for i, sh in enumerate(shards):
        path = os.path.join(shard_dir, f"replica_{replica_index}_shard_{i}.emb")
        fence = fences[i] if fences else None
        with (locks[i] if locks else contextlib.nullcontext()), open(path, "wb") as f:
            if fence is not None:  # (the reads run on the current stream; their host syncs end them under the lock)
                fence.dump_begin(torch.cuda.current_stream(sh.device))
                fence.dump_end(torch.cuda.current_stream(sh.device))
            signs, _ = sh.export_signs()
            n, nb = signs.numel(), sh.node_bytes()
            f.write(list_header(n))
            if not n:
                continue
            step = max(1, min(chunk, n, SLICE_BYTES // nb))
            sh.dump_reserve(28 + step * nb)
            try:
                out = torch.empty(step * nb, dtype=torch.uint8, device=sh.device)
                host = torch.empty(step * nb, dtype=torch.uint8, pin_memory=True)
                for lo in range(0, n, step):  # entries leave the GPU a slice at a time
                    k = min(step, n - lo)
                    sh.dump_nodes(signs, lo, k, out)
                    host[:k * nb].copy_(out[:k * nb])
                    f.write(memoryview(host.numpy())[:k * nb])
            finally:
                sh.dump_release()
    with open(os.path.join(shard_dir, DONE_FILE), "w") as f:  # mark_embedding_dump_done
        f.write(done_yaml(replica_size, len(shards)))
    if replica_index == 0 and replica_size == 1:
        with open(os.path.join(dst_dir, DONE_FILE), "w") as f:
            f.write(done_yaml(replica_size, len(shards)))


# ------------------------------------------------------------------------------------------------ background dump
# The reference's server dumps in the background: one file per internal shard, each written under that shard's read
# lock on a thread pool while training goes on (persia-model-manager/src/lib.rs:286-343); the caller polls its status
# (persia-core/src/rpc.rs:211-280).  Here each table (one per dim) is split into n_parts parts by part(sign); a part is
# collected, ordered and encoded on the device at one point of the table's call order (pb_table_dump_part), then copied
# out and written by the dumper's thread while training goes on.
DEFAULT_INTERNAL_SHARDS = 100  # num_hashmap_internal_shards' serde default (persia-embedding-config/src/lib.rs)
MARKER_TIMEOUT = 600.0         # waiting_for_all_embedding_server_dump's bound on the root marker's wait (lib.rs:172-198)


def splitmix64(x):
    """splitmix64 of each u64 (include/persia_b200.h, pb_table_dump_part)."""
    z = np.ascontiguousarray(x, dtype=np.uint64).copy()
    with np.errstate(over="ignore"):
        z += np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def part_of(signs, n_parts):
    """The part of each sign in a background dump of n_parts parts."""
    return splitmix64(signs) % np.uint64(n_parts)


def internal_shards(global_config=None):
    """embedding_parameter_server_config.num_hashmap_internal_shards of a global config dict (the reference's number of
    dump files per server), DEFAULT_INTERNAL_SHARDS when unset."""
    ps = (global_config or {}).get("embedding_parameter_server_config") or {}
    n = int(ps.get("num_hashmap_internal_shards", DEFAULT_INTERNAL_SHARDS))
    if n <= 0:
        raise RuntimeError(f"num_hashmap_internal_shards must be positive, got {n}")
    return n


def table_bytes(sh):
    """Bytes of the entries a table (HBM rows and its host tier) can hold."""
    rows = sh.capacity + (sh.host_tier.capacity if sh.host_tier is not None else 0)
    return rows * sh.entry_len * 4


def num_parts(table_sizes, shards=DEFAULT_INTERNAL_SHARDS, part_bytes=SLICE_BYTES):
    """Parts per table: at least the internal shard count, and enough that a full table's part stays near part_bytes."""
    return max([int(shards), 1] + [-(-int(b) // part_bytes) for b in table_sizes])


def part_file(replica_index, table_index, n_parts, part):
    """File of part `part` of the table of the table_index-th smallest dim."""
    return f"replica_{replica_index}_shard_{table_index * n_parts + part}.emb"


def wait_for_markers(dst_dir, replica_size, timeout=MARKER_TIMEOUT, poll=0.05, clock=time.monotonic, sleep=time.sleep):
    """Rank 0's wait for every shard directory's embedding_dump_done (waiting_for_all_embedding_server_dump); raises
    TimeoutError after `timeout` seconds."""
    deadline = clock() + timeout
    paths = [os.path.join(dst_dir, f"s{q}", DONE_FILE) for q in range(replica_size)]
    while True:
        missing = [p for p in paths if not os.path.isfile(p)]
        if not missing:
            return
        if clock() >= deadline:
            raise TimeoutError(f"waited {timeout:.0f} s for the dump of every server: {missing} missing")
        sleep(poll)


class ShardedFence:
    """Orders a table's dump calls against the calls its chains do not order (the sharded calls of R GPUs,
    include/persia_b200.h), whatever streams either runs on.  A sharded call waits for the last dump call issued before
    it; a dump call waits for the last sharded call issued before it on every stream.  Sharded calls on different
    streams stay unordered among themselves.  Every method is called under the table's lock; none synchronises the
    host."""

    def __init__(self):
        import torch

        self._torch = torch
        self._calls = {}  # stream handle -> event recorded after the latest sharded call issued on that stream
        self._dump = torch.cuda.Event()  # recorded after the latest dump call
        self._dumped = False

    def call_begin(self, stream):
        if self._dumped:
            stream.wait_event(self._dump)

    def call_end(self, stream):
        ev = self._calls.get(stream.cuda_stream)
        if ev is None:
            ev = self._calls[stream.cuda_stream] = self._torch.cuda.Event()
        ev.record(stream)

    def dump_begin(self, stream):
        for ev in self._calls.values():
            stream.wait_event(ev)

    def dump_end(self, stream):
        self._dump.record(stream)
        self._dumped = True


class DumpTable:
    """One table a background dump reads: the shard, the lock its calls are issued under, the stream its parts go on
    (None: a stream of the dumper's own) and, on R GPUs, the table's ShardedFence (the parts are then ordered against the
    sharded calls on any stream)."""

    def __init__(self, shard, lock=None, stream=None, fence=None):
        import threading

        self.shard, self.lock, self.stream = shard, lock if lock is not None else threading.Lock(), stream
        self.fence = fence


class BackgroundDumper:
    """A background dump of one replica's tables (one per dim, `tables` in ascending dim order) into dst_dir.

    Each part is issued under its table's lock on the part stream, with no host synchronisation or allocation under the
    lock; the image is copied to pinned host memory on a copy stream of its own and written by the dumper's thread.  Two
    device images and two pinned buffers alternate, so part k + 1 is encoded while part k is copied and written.  A part
    larger than its buffer grows the buffers (outside the lock) and is issued again, a later snapshot.  Device memory is
    allocated when the dump starts and freed when it ends.  Then `s{r}/embedding_dump_done` is written and, on replica
    0, the root marker once every replica's marker exists.

    start() runs it on a thread; step() issues and writes one part in the caller's thread (tests interleave parts with
    training steps).  status(): ("Idle", 1.0) done, ("Dumping", fraction), ("Failed", message)."""

    def __init__(self, dst_dir, tables, replica_index=0, replica_size=1, n_parts=None, shards=DEFAULT_INTERNAL_SHARDS,
                 part_bytes=None, marker_timeout=MARKER_TIMEOUT):
        self.dst_dir, self.tables = dst_dir, [t if isinstance(t, DumpTable) else DumpTable(t) for t in tables]
        self.replica_index, self.replica_size = int(replica_index), int(replica_size)
        self.n_parts = int(n_parts) if n_parts else num_parts([table_bytes(t.shard) for t in self.tables], shards)
        self.part_bytes, self.marker_timeout = part_bytes, marker_timeout
        self.jobs = [(d, k) for d in range(len(self.tables)) for k in range(self.n_parts)]
        self.done = 0
        self.requests = {}  # (table, part) -> the table's request number at the part's snapshot
        self.error = None
        self.finished = False
        self._thread = None
        self._stop = False
        self._opened = False
        self._ahead = False  # a part is issued in the other buffer while this one is finished

    # ---- surface ------------------------------------------------------------------------------------------------------
    def status(self):
        if self.error is not None:
            return ("Failed", self.error)
        if self.finished:
            return ("Idle", 1.0)
        return ("Dumping", self.done / max(1, len(self.jobs) + 1))

    def start(self):
        import threading

        self._thread = threading.Thread(target=self._run, name="persia-emb-dump", daemon=True)
        self._thread.start()
        return self

    def running(self):
        return self._thread is not None and self._thread.is_alive()

    def wait(self):
        """Blocks until the dump ends; RuntimeError when it failed."""
        if self._thread is not None:
            self._thread.join()
        if self.error is not None:
            raise RuntimeError(f"emb dump FAILED for server {self.replica_index}, due to {self.error}")

    def stop(self):
        """Abandons the dump after the part in hand (files already written stay)."""
        self._stop = True
        if self._thread is not None:
            self._thread.join()
        self._close()

    def step(self):
        """Issues and writes the next part in the caller's thread (and the markers after the last one); returns whether
        parts remain."""
        try:
            if self.finished:
                return False
            if not self._opened:
                self._open()
            if self.done < len(self.jobs):
                slot = self.done % 2
                self._issue(self.done, slot)
                self._finish(self.done, slot)
            if self.done == len(self.jobs):
                self._markers()
                self._close()
            return not self.finished
        except Exception as e:  # noqa: BLE001 — recorded as the dump's status
            self._fail(e)
            raise

    # ---- the dump -----------------------------------------------------------------------------------------------------
    def _run(self):
        try:
            self._open()
            n = len(self.jobs)
            if n:
                self._issue(0, 0)
            for i in range(n):
                if self._stop:
                    return
                self._ahead = i + 1 < n
                if self._ahead:
                    self._issue(i + 1, (i + 1) % 2)
                self._finish(i, i % 2)
            self._markers()
        except Exception as e:  # noqa: BLE001 — recorded as the dump's status, raised by wait()
            self._fail(e)
        finally:
            self._close()

    def _fail(self, e):
        self.error = f"{type(e).__name__}: {e}"
        self._close()

    def _open(self):
        import torch

        os.makedirs(os.path.join(self.dst_dir, f"s{self.replica_index}"), exist_ok=True)
        if not self.tables:  # nothing to read: the markers only
            return
        self.device = self.tables[0].shard.device
        self._own_stream = torch.cuda.Stream(self.device)
        self._copy_stream = torch.cuda.Stream(self.device)
        self._cap = 0
        if self.part_bytes:
            self._cap = int(self.part_bytes)
        else:  # an average part of the fullest table, with room for the spread of the parts' sizes
            for t in self.tables:
                rows = table_bytes(t.shard) // (4 * t.shard.entry_len) / self.n_parts
                self._cap = max(self._cap, 28 + int(rows + 6 * rows ** 0.5 + 64) * t.shard.node_bytes())
        self._cap = max(self._cap, 64)
        self._opened = True
        self._alloc(self._cap)

    def _alloc(self, cap):
        import torch

        self._cap = (int(cap) + 15) // 16 * 16
        self._images = [torch.empty(self._cap, dtype=torch.uint8, device=self.device) for _ in range(2)]
        self._host = [torch.empty(self._cap, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
        self._meta = [torch.zeros(2, dtype=torch.int64, device=self.device) for _ in range(2)]
        self._meta_host = [torch.zeros(2, dtype=torch.int64, pin_memory=True) for _ in range(2)]
        self._ev_part = [torch.cuda.Event() for _ in range(2)]
        self._ev_meta = [torch.cuda.Event() for _ in range(2)]
        self._ev_copy = [torch.cuda.Event() for _ in range(2)]
        for t in self.tables:
            t.shard.dump_reserve(self._cap)

    def _close(self):
        if not self._opened:
            return
        self._opened = False
        import torch

        torch.cuda.synchronize(self.device)  # (the parts and copies in flight use the buffers)
        for t in self.tables:
            try:
                t.shard.dump_release()
            except Exception:  # noqa: BLE001 — a closed table frees its workspace itself
                pass
        self._images = self._host = self._meta = self._meta_host = None

    def _issue(self, i, slot):
        """Part i of the job list into buffer `slot`: the part under the table's lock, then (copy stream) its size."""
        import torch

        d, k = self.jobs[i]
        t = self.tables[d]
        st = t.stream if t.stream is not None else self._own_stream
        with t.lock:
            if t.fence is not None:
                t.fence.dump_begin(st)
            t.shard.dump_part(k, self.n_parts, self._images[slot], self._meta[slot], st)
            self._ev_part[slot].record(st)
            if t.fence is not None:
                t.fence.dump_end(st)
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(self._ev_part[slot])
            self._meta_host[slot].copy_(self._meta[slot], non_blocking=True)
            self._ev_meta[slot].record(self._copy_stream)

    def _finish(self, i, slot):
        """Waits for part i's image, copies it out and writes its file; a part too large for the buffers grows them
        and is issued again (a part issued after it in the other buffer is then issued again too)."""
        import torch

        d, k = self.jobs[i]
        while True:
            self._ev_meta[slot].synchronize()
            nbytes, req = int(self._meta_host[slot][0]), int(self._meta_host[slot][1]) & 0xFFFFFFFF
            if nbytes <= self._cap:
                break
            # new buffers in both slots, the parts in them issued again; the part issued ahead may still write into
            # the old image, so nothing is dropped before it ends
            torch.cuda.synchronize(self.device)
            self._alloc(2 * nbytes)
            self._issue(i, slot)
            if self._ahead:
                self._issue(i + 1, (i + 1) % 2)
        with torch.cuda.stream(self._copy_stream):
            self._host[slot][:nbytes].copy_(self._images[slot][:nbytes], non_blocking=True)
            self._ev_copy[slot].record(self._copy_stream)
        self._ev_copy[slot].synchronize()
        path = os.path.join(self.dst_dir, f"s{self.replica_index}", part_file(self.replica_index, d, self.n_parts, k))
        with open(path, "wb") as f:
            f.write(memoryview(self._host[slot].numpy())[:nbytes])
        self.requests[(d, k)] = req
        self.done = i + 1

    def _sleep(self, s):
        if self._stop:
            raise RuntimeError("the dump was stopped")
        time.sleep(s)

    def _markers(self):
        shard_dir = os.path.join(self.dst_dir, f"s{self.replica_index}")
        with open(os.path.join(shard_dir, DONE_FILE), "w") as f:  # mark_embedding_dump_done
            f.write(done_yaml(self.replica_size, len(self.tables) * self.n_parts))
        if self.replica_index == 0:
            wait_for_markers(self.dst_dir, self.replica_size, self.marker_timeout, sleep=self._sleep)
            with open(os.path.join(self.dst_dir, DONE_FILE), "w") as f:
                f.write(done_yaml(self.replica_size, len(self.tables) * self.n_parts))
        self.finished = True


def checkpoint_info(src_dir):
    """load_embedding_checkpoint_info (persia-model-manager/src/lib.rs:200-240): the `embedding_dump_done` marker of the
    checkpoint (the root's, else shard 0's) -> (num_shards, num_internal_shards)."""
    for path in (os.path.join(src_dir, DONE_FILE), os.path.join(src_dir, "s0", DONE_FILE)):
        if os.path.isfile(path):
            info = {}
            for line in open(path):
                if ":" in line and not line.startswith(" "):
                    k, v = line.split(":", 1)
                    if v.strip().isdigit():
                        info[k.strip()] = int(v.strip())
            if "num_shards" in info:
                return info["num_shards"], info.get("num_internal_shards", 1)
    raise RuntimeError(f"LoadingFromUncompeleteCheckpoint({src_dir!r})")


def _farmhash64(x):
    """farmhash 1.1.5 hash64 of the 8 LE bytes of each u64 (sign_to_shard_modulo, embedding_worker_service/mod.rs:341-345)."""
    x = np.ascontiguousarray(x, dtype=np.uint64)
    k2 = np.uint64(0x9AE16A3B2F90404F)
    mul = k2 + np.uint64(16)

    def rotr(v, s):
        return (v >> np.uint64(s)) | (v << np.uint64(64 - s))

    with np.errstate(over="ignore"):
        a = x + k2
        c = rotr(x, 37) * mul + a
        d = (rotr(a, 25) + x) * mul
        h = (c ^ d) * mul
        h ^= h >> np.uint64(47)
        g = (d ^ h) * mul
        g ^= g >> np.uint64(47)
        return g * mul


def load_files(src_dir, replica_index=0, replica_size=1):
    """The `.emb` files load_shards reads, in its order, and how it selects: (files, error, R, rank).  error: the
    exception load_shards raises when it reaches the first incomplete shard directory (after the files before it;
    None: all complete).  Entries are kept when farmhash64(sign) % R == rank."""
    num_shards, _ = checkpoint_info(src_dir)
    reshard = num_shards != replica_size
    dirs = [os.path.join(src_dir, f"s{k}") for k in range(num_shards)] if reshard else [os.path.join(src_dir, f"s{replica_index}")]
    files = []
    for shard_dir in dirs:
        names = sorted(x for x in os.listdir(shard_dir) if x.endswith(".emb")) if os.path.isdir(shard_dir) else []
        if not os.path.isfile(os.path.join(shard_dir, DONE_FILE)) or not names:
            return files, RuntimeError(f"LoadingFromUncompeleteCheckpoint({shard_dir!r})"), 1, 0
        files += [os.path.join(shard_dir, x) for x in names]
    if reshard and replica_size > 1:
        return files, None, int(replica_size), int(replica_index)
    return files, None, 1, 0


def load_shards(src_dir, shards_by_dim, replica_index=0, replica_size=1, chunk=1 << 20):
    """EmbeddingWorker::load (embedding_worker_service/mod.rs:1150-1259).  A checkpoint written by as many shards as there
    are replicas now is loaded shard by shard: replica r reads `s{r}` (load_embedding_via_emb_servers ->
    EmbeddingModelManager.load_embedding_from_dir, lib.rs:259-273).  Any other shard count goes "via the embedding
    worker": every `.emb` of every shard directory is read and its entries are re-sharded by sign exactly as
    set_embedding does (farmhash64(sign) % replica_size, mod.rs:1197-1259); here every replica reads all files and
    keeps what it owns.  shards_by_dim: {embedding_dim: EmbeddingShard}.  Returns the number of entries loaded into
    this replica.  Errors mirror the reference's (lib.rs:343-372)."""
    import torch

    num_shards, _ = checkpoint_info(src_dir)
    reshard = num_shards != replica_size
    dirs = [os.path.join(src_dir, f"s{k}") for k in range(num_shards)] if reshard else [os.path.join(src_dir, f"s{replica_index}")]
    total = 0
    for shard_dir in dirs:
        if not os.path.isfile(os.path.join(shard_dir, DONE_FILE)):
            raise RuntimeError(f"LoadingFromUncompeleteCheckpoint({shard_dir!r})")
        files = sorted(x for x in os.listdir(shard_dir) if x.endswith(".emb"))
        if not files:
            raise RuntimeError(f"LoadingFromUncompeleteCheckpoint({shard_dir!r})")
        for name in files:
            with open(os.path.join(shard_dir, name), "rb") as f:
                signs, dims, entries = decode_list(f.read())
            keep = np.ones(signs.size, bool)
            if reshard and replica_size > 1:
                keep = (_farmhash64(signs) % np.uint64(replica_size)) == np.uint64(replica_index)
            for dim in np.unique(dims[keep]) if keep.any() else []:
                sh = shards_by_dim.get(int(dim))
                if sh is None:
                    raise RuntimeError(f"checkpoint holds dim-{int(dim)} embeddings but no slot has that dim")
                pick = np.nonzero((dims == dim) & keep)[0]
                lens = {entries[i].size for i in pick}
                if lens != {sh.entry_len}:
                    raise RuntimeError(f"dim-{int(dim)} entries of {sorted(lens)} floats, the registered optimizer needs "
                                       f"{sh.entry_len} (embedding ++ state)")
                if getattr(sh, "host_tier", None) is not None:
                    # HBM rows + a host tier: the newest entries take the HBM rows, the oldest overflow to the tier (the
                    # reference's LRU map, filled in list order beyond its capacity, would keep the newest)
                    pick = pick[::-1]
                for lo in range(0, pick.size, chunk):
                    sel = pick[lo:lo + chunk]
                    ent = torch.from_numpy(np.stack([entries[i] for i in sel])).to(sh.device)
                    sg = torch.from_numpy(signs[sel].view(np.int64)).to(sh.device)
                    sh.set_entries(sg, ent)
                total += pick.size
    return total


# ------------------------------------------------------------------------------------------------ device load
# The reference's server loads a checkpoint in the background: one job per file, each decoded whole and inserted in
# list order, while the server reports Loading(progress) (persia-model-manager/src/lib.rs:375-425,
# embedding_parameter_service/mod.rs:264-280); the caller polls wait_for_emb_loading (persia-core/src/rpc.rs:154-176,
# 235-283).  Here the entries are decoded, selected and gathered on the device (pb_image_*, pb_load.cu) and offered to
# the tables in load_shards' order, so the tables end as load_shards leaves them.
LOAD_SUMMARY_ROWS = 64  # (dim, entry length) pairs one image may hold (pb_load.cu LOAD_PAIRS)
_FORMAT_ERRORS = {"ValueError": ValueError, "IndexError": IndexError}


def writer_layout(size, head):
    """(n_nodes, entry_len) when a file of `size` bytes whose first 41 bytes (header and first node's header) are
    `head` may be in the writer layout: count = n_nodes > 0, the list from node 1, the first node live, size =
    28 + n_nodes (29 + 4 entry_len).  None: any other layout.  The nodes themselves are checked as their windows are
    read."""
    if size < 41 or len(head) < 41:
        return None
    count = int(np.frombuffer(head[:8], "<u8")[0])
    first, _, _, _, n = (int(x) for x in np.frombuffer(head[8:28], "<u4"))
    L = int(np.frombuffer(head[37:41], "<u4")[0])
    if not n or count != n or first != 1 or head[36] != 1 or size != 28 + n * (29 + 4 * L):
        return None
    return n, L


def windows(n_nodes, node_bytes, buffer_bytes, newest_first=False):
    """Node ranges [lo, hi) of a writer-layout file read through a buffer of buffer_bytes: whole nodes, at least one
    per window.  newest_first: from the end of the file, cut from the end (so that, as in load_shards' reversed
    chunks, only the last window offered is short)."""
    w = max(1, int(buffer_bytes) // int(node_bytes))
    if newest_first:
        return [(max(0, hi - w), hi) for hi in range(n_nodes, 0, -w)]
    return [(lo, min(lo + w, n_nodes)) for lo in range(0, n_nodes, w)]


def check_dims(summary, shards_by_dim):
    """load_shards' checks of one image's selected entries, dims ascending: summary rows (dim, entry length,
    entries).  Returns [(dim, entries)] of the dims with selected entries."""
    out = []
    for dim in sorted({d for d, _, k in summary if k}):
        sh = shards_by_dim.get(dim)
        if sh is None:
            raise RuntimeError(f"checkpoint holds dim-{dim} embeddings but no slot has that dim")
        lens = sorted({ln for d, ln, k in summary if d == dim and k})
        if lens != [sh.entry_len]:
            raise RuntimeError(f"dim-{dim} entries of {lens} floats, the registered optimizer needs {sh.entry_len} "
                               f"(embedding ++ state)")
        out.append((dim, sum(k for d, _, k in summary if d == dim)))
    return out


class LoadStatus:
    """The reference's server status while it loads (embedding_parameter_service/mod.rs:264-280): ("Loading", fraction)
    as work is done, ("Idle", 1.0) once done, ("Failed", "Type: message") when it failed."""

    def __init__(self, total):
        self.total, self.done, self.error, self.finished = max(1, int(total)), 0, None, False

    def advance(self, amount):
        self.done = min(self.total, self.done + int(amount))

    def fail(self, e):
        self.error = f"{type(e).__name__}: {e}"

    def finish(self):
        self.finished = True

    def __call__(self):
        if self.error is not None:
            return ("Failed", self.error)
        if self.finished:
            return ("Idle", 1.0)
        return ("Loading", min(self.done / self.total, 0.999))


class _Pinned:
    """Pinned host memory of the library's own (pb_host_alloc), mapped into the device's address space and freed on
    close(): the image buffers of a load, released when the load ends rather than kept by a caching allocator."""

    def __init__(self, nbytes):
        import ctypes as C

        from . import native as N

        self.N, self.lib = N, N.load()
        p = C.c_void_p()
        N.check(self.lib.pb_host_alloc(int(nbytes), C.byref(p)))
        self.ptr, self.size = p.value, int(nbytes)
        self.view = np.ctypeslib.as_array((C.c_uint8 * max(1, self.size)).from_address(self.ptr))

    def data_ptr(self):
        return self.ptr

    def close(self):
        if self.ptr:
            self.view = None
            self.N.check(self.lib.pb_host_free(self.ptr))
            self.ptr = 0


class _Image:
    """A pb_image: one list image (or writer-layout window, or incremental-update packet) in pinned host memory,
    indexed, selected and inserted on the device."""

    def __init__(self, device, chunk):
        import ctypes as C

        from . import native as N

        self.C, self.N, self.lib = C, N, N.load()
        h = C.c_void_p()
        N.check(self.lib.pb_image_create(device.index or 0, int(chunk), C.byref(h)))
        self.h = h
        self._rows = (C.c_uint64 * (3 * LOAD_SUMMARY_ROWS))()

    def _summary(self, n):
        return [(int(self._rows[3 * i]), int(self._rows[3 * i + 1]), int(self._rows[3 * i + 2])) for i in range(n)]

    def _check(self, rc):
        if rc == self.N.PB_ERR_FORMAT:  # decode_list's (decode_packet's) exception
            kind, msg = self.lib.pb_last_error().decode().split(": ", 1)
            raise _FORMAT_ERRORS[kind](msg)
        self.N.check(rc)

    def index(self, buf, nbytes, p_lo, p_hi, R, rank, stream):
        C = self.C
        rows = C.c_uint32()
        self._check(self.lib.pb_image_index(self.h, C.c_void_p(buf.data_ptr()), int(nbytes), int(p_lo), int(p_hi), R,
                                            rank, self._rows, LOAD_SUMMARY_ROWS, C.byref(rows),
                                            C.c_void_p(stream.cuda_stream)))
        return self._summary(rows.value)

    def packet(self, buf, nbytes, R, rank, stream):
        """An incremental-update packet's (summary, timestamp); decode_packet's exception when it is malformed."""
        C = self.C
        rows, ts = C.c_uint32(), C.c_uint64()
        self._check(self.lib.pb_image_packet(self.h, C.c_void_p(buf.data_ptr()), int(nbytes), R, rank, self._rows,
                                             LOAD_SUMMARY_ROWS, C.byref(rows), C.byref(ts),
                                             C.c_void_p(stream.cuda_stream)))
        return self._summary(rows.value), int(ts.value)

    def window(self, buf, node0, n, n_total, entry_len, dim, R, rank, stream):
        """The window's summary, or None when a node of it is not in the writer layout."""
        C = self.C
        rows, ok = C.c_uint32(), C.c_int()
        self.N.check(self.lib.pb_image_window(self.h, C.c_void_p(buf.data_ptr()), int(node0), int(n), int(n_total),
                                              int(entry_len), int(dim), R, rank, self._rows, LOAD_SUMMARY_ROWS,
                                              C.byref(rows), C.byref(ok), C.c_void_p(stream.cuda_stream)))
        return self._summary(rows.value) if ok.value else None

    def insert(self, shard, dim, lo, hi, newest_first, stream):
        self.N.check(self.lib.pb_image_insert(self.h, shard.h, int(dim), int(lo), int(hi), int(bool(newest_first)),
                                              self.C.c_void_p(stream.cuda_stream)))

    def close(self):
        if getattr(self, "h", None):
            self.lib.pb_image_destroy(self.h)
            self.h = None


class DeviceLoader:
    """load_shards on the device, in the foreground or in the background: the same files, entries, order and errors,
    and the same tables at the end.

    A file in the writer layout (writer_layout) is read through the pinned buffers a window of whole nodes at a time
    (windows: from the end of the file for a table with a host tier, whose entries go newest first); each window's
    nodes are checked on the device before any of it is inserted.  A window that is not in the writer layout sends the
    loader to the whole file, which then gives decode_list's error, or the entries not yet inserted.  Any other file is
    read whole.  A reader thread reads window or file k + 1 into one of two alternating pinned buffers while k is
    decoded.  The entries of each dim go to its table in chunks of at most `chunk`, each under the table's lock
    (locks: {dim: lock}), on a stream of the loader's own, and at R > 1 between the table's ShardedFence calls
    (fences: {dim: fence}).  Device workspace lives while the load runs.

    run() loads in the caller's thread and raises what load_shards raises; start() runs it on a thread; step()
    handles one window or file in the caller's thread (tests interleave training steps); wait() blocks and raises
    RuntimeError("emb dump FAILED for server {r}, due to ...") (the reference's text) when it failed; status():
    LoadStatus.  Files and windows inserted before a failure stay."""

    def __init__(self, src_dir, shards_by_dim, replica_index=0, replica_size=1, chunk=1 << 20, buffer_bytes=SLICE_BYTES,
                 locks=None, fences=None):
        self.src_dir, self.shards = src_dir, dict(shards_by_dim)
        self.replica_index, self.replica_size = int(replica_index), int(replica_size)
        self.chunk, self.buffer_bytes = int(chunk), max(64, int(buffer_bytes))
        self.locks, self.fences = locks or {}, fences or {}
        self.loaded = 0
        self.error = None
        self._status = LoadStatus(1)
        self._planned = False
        self._tasks, self._next = [], 0
        self._thread = None
        self._stop = False
        self._opened = False

    # ---- surface ------------------------------------------------------------------------------------------------------
    def status(self):
        return self._status()

    def start(self):
        import threading

        self._thread = threading.Thread(target=self._run, name="persia-emb-load", daemon=True)
        self._thread.start()
        return self

    def running(self):
        return self._thread is not None and self._thread.is_alive()

    def join(self):
        if self._thread is not None:
            self._thread.join()

    def wait(self):
        self.join()
        if self.error is not None:
            raise RuntimeError(f"emb dump FAILED for server {self.replica_index}, due to {self._status.error}")

    def stop(self):
        """Abandons the load after the window or file in hand (what was inserted stays); a load that had not finished
        then reports ("Failed", "RuntimeError: the load was stopped")."""
        self._stop = True
        self.join()
        self._close()

    def run(self):
        """Loads everything in the caller's thread; raises the load's exception.  Returns the entries loaded."""
        try:
            self._open()
            pending = self._submit(0)
            for i in range(len(self._tasks)):
                if self._stop:
                    raise RuntimeError("the load was stopped")
                got = pending.result()
                pending = self._submit(i + 1)
                self._handle(i, got)
            self._status.finish()
            return self.loaded
        except Exception as e:  # noqa: BLE001 — recorded as the load's status, then raised
            self.error = e
            self._status.fail(e)
            raise
        finally:
            self._close()

    def step(self):
        """Handles the next window or file in the caller's thread; returns whether any remain."""
        try:
            if not self._opened:
                self._open()
            if self._next < len(self._tasks):
                i = self._next
                self._handle(i, self._read(i))
            if self._next >= len(self._tasks):
                self._status.finish()
                self._close()
                return False
            return True
        except Exception as e:  # noqa: BLE001
            self.error = e
            self._status.fail(e)
            self._close()
            raise

    # ---- the load -----------------------------------------------------------------------------------------------------
    def _run(self):
        try:
            self.run()
        except Exception:  # noqa: BLE001 — recorded as the load's status, raised by wait()
            pass

    def _open(self):
        import concurrent.futures

        import torch

        files, self._dir_error, self.R, self.rank = load_files(self.src_dir, self.replica_index, self.replica_size)
        tasks = []  # (file, kind, lo, hi, info): kind "window" (writer layout, nodes [lo, hi)) or "whole"
        for f in files:
            size = os.path.getsize(f)
            with open(f, "rb") as fh:
                w = writer_layout(size, fh.read(41))
                if w is not None:
                    n, L = w
                    fh.seek(41 + 4 * L)
                    dim = int(np.frombuffer(fh.read(8), "<u8")[0])
            if w is None:
                tasks.append((f, "whole", 0, 0, size))
                continue
            sh = self.shards.get(dim)
            newest = sh is not None and getattr(sh, "host_tier", None) is not None
            tasks += [(f, "window", lo, hi, (n, L, dim, newest)) for lo, hi in windows(n, 29 + 4 * L, self.buffer_bytes, newest)]
        if self._dir_error is not None:
            tasks.append((None, "error", 0, 0, 0))
        self._tasks = tasks
        self._skip = set()  # files loaded whole after a window was not in the writer layout
        self._status = LoadStatus(sum(self._task_bytes(t) for t in tasks))
        self.device = next(iter(self.shards.values())).device if self.shards else torch.device("cuda", torch.cuda.current_device())
        self._stream = torch.cuda.Stream(self.device)
        self._bufs = [None, None]
        self._done = [torch.cuda.Event(), torch.cuda.Event()]  # the inserts that read each buffer
        # where the time goes: file reads (reader thread), index calls (host pass + device selection, wall time), and
        # the device time of the gathers and inserts (CUDA events, from the end of each index call to its last insert)
        self.timings = {"read_s": 0.0, "index_s": 0.0, "insert_ms": 0.0}
        self._events = []
        self._image = _Image(self.device, self.chunk)
        self._pool = concurrent.futures.ThreadPoolExecutor(1, thread_name_prefix="persia-emb-read")
        self._opened = True

    def _close(self):
        if not self._opened:
            return
        self._opened = False
        self._pool.shutdown(wait=True)
        self._stream.synchronize()
        self._image.close()
        self.timings["insert_ms"] += sum(a.elapsed_time(b) for a, b in self._events)
        self._events = []
        for b in self._bufs:
            if b is not None:
                b.close()
        self._bufs = [None, None]

    @staticmethod
    def _task_bytes(t):
        f, kind, lo, hi, info = t
        if kind == "window":
            return (hi - lo) * (29 + 4 * info[1])
        return info if kind == "whole" else 0

    def _buffer(self, slot, nbytes):
        buf = self._bufs[slot]
        if buf is None or buf.size < nbytes:
            self._done[slot].synchronize()
            if buf is not None:
                buf.close()
            cap = max(64, min(int(nbytes) * 2, max(int(nbytes), self.buffer_bytes)))
            buf = self._bufs[slot] = _Pinned(cap)
        return buf

    def _read(self, i):
        """Task i's bytes into buffer i % 2 (once the inserts that read that buffer before have run)."""
        f, kind, lo, hi, info = self._tasks[i]
        slot = i % 2
        self._done[slot].synchronize()
        if kind == "error" or f in self._skip:
            return slot, 0
        if kind == "window":
            nb = 29 + 4 * info[1]
            start, nbytes = 28 + lo * nb, (hi - lo) * nb
        else:
            start, nbytes = 0, info
        buf = self._buffer(slot, nbytes)
        t0 = time.perf_counter()
        with open(f, "rb") as fh:
            fh.seek(start)
            got = fh.readinto(memoryview(buf.view)[:nbytes])
        self.timings["read_s"] += time.perf_counter() - t0
        if got != nbytes:
            raise RuntimeError(f"{f} changed while it was loaded")
        return slot, nbytes

    def _submit(self, i):
        import concurrent.futures

        if i >= len(self._tasks):
            done = concurrent.futures.Future()
            done.set_result(None)
            return done
        return self._pool.submit(self._read, i)

    def _insert(self, summary, newest_of=None):
        """load_shards' checks of the image's dims, then their entries, dims ascending, a chunk at a time."""
        import contextlib

        for dim, k in check_dims(summary, self.shards):
            sh = self.shards[dim]
            newest = getattr(sh, "host_tier", None) is not None if newest_of is None else newest_of
            fence = self.fences.get(dim)
            for lo in range(0, k, self.chunk):
                with self.locks.get(dim) or contextlib.nullcontext():
                    if fence is not None:
                        fence.dump_begin(self._stream)
                    self._image.insert(sh, dim, lo, min(lo + self.chunk, k), newest, self._stream)
                    if fence is not None:
                        fence.dump_end(self._stream)
            self.loaded += k

    def _handle(self, i, got):
        f, kind, lo, hi, info = self._tasks[i]
        self._next = i + 1
        slot, nbytes = got
        if kind == "error":
            raise self._dir_error
        if f not in self._skip:
            import torch

            buf = self._bufs[slot]
            t0 = time.perf_counter()
            if kind == "whole":
                summary = self._image.index(buf, nbytes, 0, 0xFFFFFFFF, self.R, self.rank, self._stream)
            else:
                n, L, dim, newest = info
                summary = self._image.window(buf, lo, hi - lo, n, L, dim, self.R, self.rank, self._stream)
            self.timings["index_s"] += time.perf_counter() - t0
            ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[0].record(self._stream)
            if kind == "whole":
                self._insert(summary)
            elif summary is not None:
                self._insert(summary, newest)
            else:
                self._whole_rest(i)
            ev[1].record(self._stream)
            self._events.append(ev)
            self._done[slot].record(self._stream)
        self._status.advance(self._task_bytes(self._tasks[i]))

    def _whole_rest(self, i):
        """Window i of its file is not in the writer layout: the whole file, less the windows already inserted (they
        hold list positions [0, lo), or [hi, n) newest first, whenever the file is a valid list)."""
        f, _, lo, hi, (n, _, _, newest) = self._tasks[i]
        self._skip.add(f)
        self._stream.synchronize()
        size = os.path.getsize(f)
        buf = _Pinned(max(64, size))
        try:
            with open(f, "rb") as fh:
                fh.readinto(memoryview(buf.view)[:size])
            p_lo, p_hi = (0, hi) if newest else (lo, n)
            self._insert(self._image.index(buf, size, p_lo, p_hi, self.R, self.rank, self._stream))
            self._stream.synchronize()  # (the inserts read buf)
        finally:
            buf.close()
