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


# ------------------------------------------------------------------------------------------------ dump / load
def dump_shards(dst_dir, shards, replica_index=0, replica_size=1, chunk=1 << 20):
    """EmbeddingModelManager.dump_embedding for one parameter-server replica.  `shards`: the EmbeddingShards (one per
    embedding dim) this replica holds; each becomes one `.emb` file ("internal shard")."""
    import torch

    shard_dir = os.path.join(dst_dir, f"s{replica_index}")
    os.makedirs(shard_dir, exist_ok=True)
    for i, sh in enumerate(shards):
        signs, _ = sh.export_signs()
        n, L = signs.numel(), sh.entry_len
        path = os.path.join(shard_dir, f"replica_{replica_index}_shard_{i}.emb")
        with open(path, "wb") as f:
            head = encode_list(np.zeros(0, np.uint64), np.zeros((0, L), np.float32), sh.dim)
            hdr = np.frombuffer(head[:28], np.uint8).copy()
            hdr[:8] = np.frombuffer(np.array([n], "<u8").tobytes(), np.uint8)
            hdr[8:28] = np.frombuffer(np.array([1 if n else 0, n, 0, 0, n], "<u4").tobytes(), np.uint8)
            f.write(hdr.tobytes())
            for lo in range(0, n, chunk):  # entries leave the GPU a chunk at a time
                part = signs[lo:lo + chunk]
                ent, found = sh.get_entries(part)
                assert bool(found.all())
                nodes = np.zeros(part.numel(), _node_dtype(L))
                idx = np.arange(lo, lo + part.numel(), dtype=np.uint32)
                nodes["next"] = np.where(idx + 1 < n, idx + 2, 0)
                nodes["prev"] = idx
                nodes["flag"], nodes["len"], nodes["dim"] = 1, L, sh.dim
                nodes["inner"] = ent.cpu().numpy()
                nodes["sign"] = part.cpu().numpy().view(np.uint64)
                f.write(nodes.tobytes())
        torch.cuda.synchronize(sh.device)
    with open(os.path.join(shard_dir, DONE_FILE), "w") as f:  # mark_embedding_dump_done
        f.write(done_yaml(replica_size, len(shards)))
    if replica_index == 0 and replica_size == 1:
        with open(os.path.join(dst_dir, DONE_FILE), "w") as f:
            f.write(done_yaml(replica_size, len(shards)))


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
