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
