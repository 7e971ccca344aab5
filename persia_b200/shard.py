"""EmbeddingShard / BatchContext: thin torch-facing wrappers over the C ABI.

`EmbeddingShard` is one embedding-parameter-server replica resident in one GPU's HBM
(reference: rust/persia-embedding-server/src/embedding_parameter_service/mod.rs +
rust/persia-embedding-holder).  `BatchContext` is what the embedding worker keeps between the forward
and the backward of one batch (embedding_worker_service/mod.rs:1087-1119).  torch only owns device
memory and the current stream here; all compute is in libpersia_b200.so.
"""
import ctypes as C

import torch

from . import native as N


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def aligned(t, stream=None):
    """The library refuses gradient buffers that are not 16-byte aligned (include/persia_b200.h).  A contiguous view at
    such a storage offset (one slot of an [S, B, dim] tensor, say) is copied: on `stream`, the stream the call that
    reads it runs on, so that the copy is ordered like the call and its memory is not reused before the call has read it."""
    if t is None or t.data_ptr() % 16 == 0:
        return t
    if stream is None:
        return t.clone()
    with torch.cuda.stream(stream):
        return t.clone()


def _as_i64_bits(t):
    """uint64 ids travel as int64 bit patterns inside torch (torch has no full uint64 support)."""
    if t.dtype == torch.uint64:
        t = t.view(torch.int64)
    assert t.dtype == torch.int64, "ids must be uint64/int64 bit patterns"
    return t.contiguous()


# Marshalling shared by the local wrappers here and the sharded ones (worker.py): tensors -> the C ABI's arguments.
def _slot_offsets(slot_off, n_slots):
    return (C.c_uint32 * (n_slots + 1))(*[int(x) for x in slot_off])


def _prefixes(prefixes):
    return (C.c_uint64 * len(prefixes))(*[int(p) for p in prefixes])


def _grad_ptrs(ptrs, n_slots):
    """Per-slot device pointers (None or 0 = skipped slot) as the backward's c_void_p[n_slots] array."""
    return (C.c_void_p * n_slots)(*[(int(p) if p else None) for p in ptrs])


def _slot_grads(grads, n_slots, stream=None):
    """Per-slot gradients (device tensors [batch, dim], all f16 or all f32; None = skipped slot) -> (pointer array,
    is_f16, the tensors to hold through the call).  A misaligned tensor is copied on `stream`, the stream the call runs
    on (None: the current one; see aligned)."""
    grads = [aligned(g, stream) for g in grads]
    is_f16 = None
    for g in grads:
        if g is not None:
            assert g.is_contiguous() and g.dtype in (torch.float16, torch.float32)
            f16 = g.dtype == torch.float16
            assert is_f16 is None or is_f16 == f16, "all slot gradients of one request share a dtype"
            is_f16 = f16
    return _grad_ptrs([g.data_ptr() if g is not None else None for g in grads], n_slots), bool(is_f16), grads


def _scales(scales, n_slots):
    """Per-slot loss scales as the backward's c_float[n_slots] array; None when none are given."""
    return (C.c_float * n_slots)(*[float(s) for s in scales]) if scales is not None else None


def _raw_grad(grad, is_f16, owner, stream=None):
    """A raw backward's gradient (tensor, device pointer or None) -> (pointer, is_f16, the tensor to hold through the
    call).  A misaligned tensor is copied on `stream` (see aligned).  An empty one (U = 0: nothing is read, but the
    request is not a skipped one) points at `owner._dummy`, made on first use: one per wrapper object."""
    if grad is None or isinstance(grad, int):
        return grad, is_f16, None
    grad = aligned(grad, stream)
    assert grad.is_contiguous() and grad.dtype in (torch.float16, torch.float32)
    is_f16 = grad.dtype == torch.float16
    if not grad.numel():
        if getattr(owner, "_dummy", None) is None:
            owner._dummy = torch.zeros(4, dtype=torch.float32, device=owner.device)
        grad = owner._dummy
    return grad.data_ptr(), is_f16, grad


def _raw_outputs(n, batch, fixed, dim, device):
    """The five output buffers of a raw forward of n ids (see BatchContext.forward_raw)."""
    return (torch.empty((n + 1, dim), dtype=torch.float16, device=device),
            torch.empty(batch * fixed, dtype=torch.int64, device=device),
            torch.empty(max(batch * fixed, 1), dtype=torch.int64, device=device),
            torch.empty(max(batch, 1), dtype=torch.int32, device=device),
            torch.empty(2, dtype=torch.int32, device=device))


def _raw_row_off(row_off, batch):
    """A raw forward's CSR offsets (device int32 [batch + 1]; None: one id per sample), checked, as a pointer."""
    if row_off is not None:
        assert row_off.dtype == torch.int32 and row_off.is_contiguous() and row_off.numel() == batch + 1
    return _ptr(row_off)


def _read_block(fields, call, ctype=C.c_uint64):
    """`call(pointer)` fills len(fields) counters of `ctype` and returns a pb status; the counters keyed by `fields`."""
    out = (ctype * len(fields))()
    N.check(call(C.byref(out)))
    return dict(zip(fields, out))


COUNTER_FIELDS = ("admitted", "lookup_miss", "gradient_id_miss", "capacity_refused", "wait_errors")
INDEX_STATS_FIELDS = ("live", "tomb", "empty")
STORAGE_STATS_FIELDS = ("reserved_rows", "mapped_rows", "index_cells", "refused_unmapped")
TIER_STATS_FIELDS = ("host_rows", "moved_out", "restored", "dropped", "refused")
STAGE_STATS_FIELDS = ("staged", "skipped")
INCREMENTAL_STATS_FIELDS = ("held", "inserted", "dropped", "taken")
BATCH_STATS_FIELDS = ("items", "cold", "warm", "hot", "repeated_occurrences", "occurrences")


def _capturing(stream):
    with torch.cuda.stream(stream):
        return torch.cuda.is_current_stream_capturing()


class StreamMark:
    """An event recorded on one stream for work on another to wait for, as the library's table marks do it: a wait never
    crosses a stream-capture boundary.  Work recorded outside a capture must have completed before the capture starts
    (synchronise first); work recorded inside one graph is ordered within it, and graphs among themselves by whoever
    launches them."""

    def __init__(self):
        self.ev, self.captured = None, False

    def record(self, stream):
        if self.ev is None:
            self.ev = torch.cuda.Event()
        self.captured = _capturing(stream)
        self.ev.record(stream)

    def wait(self, stream):
        if self.ev is not None and self.captured == _capturing(stream):
            stream.wait_event(self.ev)


def rsqrt_mode(mode):
    """pb_rsqrt_mode of "exact" / "intel" (or of the mode itself)."""
    modes = {"exact": N.RSQRT_EXACT, "intel": N.RSQRT_INTEL}
    if isinstance(mode, str):
        if mode not in modes:
            raise ValueError(f"unknown rsqrt mode {mode!r}: expected 'exact' or 'intel'")
        return modes[mode]
    if mode not in modes.values():
        raise ValueError(f"unknown rsqrt mode {mode!r}")
    return int(mode)


def grow_mode(grow):
    """EmbeddingShard's `grow` as a pb_table_set_growth mode: False / None / 0 / "0" / "" off, True / 1 / "1" growable,
    "shared" / 2 growable and exportable."""
    if grow is None or grow is False or str(grow).strip() in ("", "0"):
        return N.GROW_OFF
    if grow is True or str(grow).strip() == "1":
        return N.GROW_ON
    if str(grow).strip() in ("shared", "2"):
        return N.GROW_SHARED
    raise ValueError(f"unknown growth mode {grow!r}: expected False, True or 'shared'")


class EmbeddingShard:
    def __init__(self, dim, capacity, device=0, tier_rows=0, host=False, shared_tier=False, grow=False):
        """capacity: rows in HBM.  tier_rows > 0: a host-memory tier of that many rows behind them (include/persia_b200.h,
        pb_table_attach_tier), attached once the optimizer is registered.  host: this table's rows live in host memory
        (the tier itself).  shared_tier: the tier's rows are shared memory other processes can map
        (pb_table_create_host_shared), so that the table can be exported and its peers read the tier in place.
        grow: capacity bounds the table instead of reserving it: HBM backs rows and index cells as entries are admitted
        (pb_table_set_growth; no tier).  True or "1": no export; "shared": exportable (growth mode 2), so that peers
        read it in place while it grows (register their views with add_readers)."""
        if grow and (host or tier_rows):
            raise ValueError("a growable table has no host tier and is not one")
        mode = grow_mode(grow)
        self.lib = N.load()
        self.dim, self.capacity = int(dim), int(capacity)
        self.device = torch.device("cuda", device) if not isinstance(device, torch.device) else device
        h = C.c_void_p()
        cfg = N.TableCfg(self.dim, self.capacity)
        create = self.lib.pb_table_create
        if host:
            create = self.lib.pb_table_create_host_shared if shared_tier else self.lib.pb_table_create_host
        N.check(create(self.device.index or 0, C.byref(cfg), C.byref(h)))
        self.h = h
        self.grow = mode != N.GROW_OFF
        self.grow_shared = mode == N.GROW_SHARED
        if self.grow:
            N.check(self.lib.pb_table_set_growth(h, mode))
        self._entry_len = None
        self.shared_tier = bool(shared_tier and tier_rows)
        self.host_tier = EmbeddingShard(dim, tier_rows, device, host=True, shared_tier=shared_tier) if tier_rows else None
        self._tier_attached = False
        # R GPUs (worker.TierStager): the sharded forwards of this shard's workers, keyed by worker, and its stager's
        # last stage.  A stage waits for the forwards before it; a forward waits for the stage before it.
        self._forward_marks = {}
        self._stage_mark = StreamMark()

    # register_optimizer (PS mod.rs:429-438)
    def set_optimizer(self, kind, lr=0.01, wd=0.0, g_square_momentum=1.0, initialization=0.01, eps=1e-10,
                      beta1=0.9, beta2=0.999):
        cfg = N.OptimCfg(kind, lr, wd, g_square_momentum, initialization, eps, beta1, beta2)
        N.check(self.lib.pb_table_set_optimizer(self.h, C.byref(cfg)))
        self._entry_len = None
        if self.host_tier is not None:  # one entry layout in both tables
            N.check(self.lib.pb_table_set_optimizer(self.host_tier.h, C.byref(cfg)))
            if not self._tier_attached:
                N.check(self.lib.pb_table_attach_tier(self.h, self.host_tier.h))
                self._tier_attached = True

    def set_rsqrt(self, mode):
        """Adagrad's 1/sqrt(s + eps) on the fused lanes (elements < 8 * (dim // 8)): "exact" (N.RSQRT_EXACT, the
        default) or "intel" (N.RSQRT_INTEL: _mm256_rsqrt_ps as Intel CPUs compute it, so that steps match the reference's
        bit for bit as run on an Intel CPU).  Applies to every step enqueued after the call (pb_table_set_rsqrt); the host
        tier gets the same mode."""
        m = rsqrt_mode(mode)
        N.check(self.lib.pb_table_set_rsqrt(self.h, m))
        if self.host_tier is not None:
            N.check(self.lib.pb_table_set_rsqrt(self.host_tier.h, m))

    # configure (PS mod.rs:440-451)
    def configure(self, init_lower=-0.01, init_upper=0.01, admit_probability=1.0, enable_weight_bound=True,
                  weight_bound=10.0):
        cfg = N.HyperCfg(init_lower, init_upper, admit_probability, int(enable_weight_bound), weight_bound)
        N.check(self.lib.pb_table_configure(self.h, C.byref(cfg)))

    def set_eviction(self, check_every=4, low_water=None, target_free=None, keep_batches=2):
        """Recency-based capacity policy (EvictionMap semantics, batch-granular); see persia_b200.h."""
        low = (self.capacity // 16 if low_water is None else low_water) if check_every else 0
        tgt = (self.capacity // 8 if target_free is None else target_free) if check_every else 0
        N.check(self.lib.pb_table_set_eviction(self.h, check_every, low, tgt, keep_batches))

    @property
    def entry_len(self):
        if self._entry_len is None:
            v = C.c_uint32()
            N.check(self.lib.pb_table_entry_len(self.h, C.byref(v)))
            self._entry_len = v.value
        return self._entry_len

    def counters(self):
        return _read_block(COUNTER_FIELDS, lambda out: self.lib.pb_table_counters(self.h, out, _stream(self.device)))

    def index_stats(self):
        """Cells of the hash index (host sync): live signs, tombstones of evicted signs, and EMPTY cells."""
        return _read_block(INDEX_STATS_FIELDS, lambda out: self.lib.pb_table_index_stats(self.h, out, _stream(self.device)))

    def storage_stats(self):
        """Storage of the table (host sync): rows reserved (capacity) and backed by HBM, index cells, and admissions
        refused because their row was not backed yet (stays 0).  A table without growth backs its whole capacity."""
        return _read_block(STORAGE_STATS_FIELDS, lambda out: self.lib.pb_table_storage_stats(self.h, out, _stream(self.device)))

    def tier_stats(self):
        """The host tier's counters (host sync); all zero without a tier."""
        return _read_block(TIER_STATS_FIELDS, lambda out: self.lib.pb_tier_stats(self.h, out, _stream(self.device)))

    def stage(self, ids, slot_off, prefixes, prefix_bit=8):
        """pb_tier_stage on the current stream: the eviction check and the tier restores of an upcoming training request,
        one batch ahead.  ids: flat device slot ids (slot-major, hash-stacked where a slot hash-stacks), slot_off: host
        list of n_slots + 1 offsets, prefixes: each slot's index prefix (0 = ids taken as they are).  Values never
        change, only where entries live; without a tier nothing runs."""
        ids = _as_i64_bits(ids)
        S = len(prefixes)
        N.check(self.lib.pb_tier_stage(self.h, _ptr(ids), ids.numel(), _slot_offsets(slot_off, S), _prefixes(prefixes), S,
                                       int(prefix_bit), _stream(self.device)))

    def stage_stats(self):
        """Stage counters (host sync): signs moved into HBM by stages (also counted in tier_stats()["restored"]), and
        stage restores skipped for want of a free HBM row (left to the request's own restore)."""
        return _read_block(STAGE_STATS_FIELDS, lambda out: self.lib.pb_tier_stage_stats(self.h, out, _stream(self.device)))

    # incremental updates (PerisaIncrementalUpdateManager, persia-incremental-update-manager/src/lib.rs:251-312)
    def enable_incremental(self, capacity):
        """Keep the set of signs the optimizer steps from now on (at most `capacity`; further new signs are dropped and
        counted), for take_incremental().  capacity 0 frees the set.  With a host tier, the set covers both tables."""
        N.check(self.lib.pb_table_enable_incremental(self.h, int(capacity)))

    def incremental_stats(self):
        """The set's counters (host sync): signs held now, inserted, dropped because the set was full, and taken."""
        return _read_block(INCREMENTAL_STATS_FIELDS, lambda out: self.lib.pb_inc_stats(self.h, out, _stream(self.device)))

    def incremental_held(self):
        """Signs held, read without a sync: may lag the work still in flight on the stream."""
        v = C.c_uint64()
        N.check(self.lib.pb_inc_held(self.h, C.byref(v)))
        return int(v.value)

    def take_incremental_device(self, capacity):
        """Empties the set (at most `capacity` signs: the capacity it was enabled with) on the current stream and returns
        (signs int64 [n], entries f32 [n, entry_len], found bool [n]) on the device, in no particular order; found is
        False for a held sign no table holds any more.  The only host sync is the read of n.  None (and the set left as
        it is) when it holds more than `capacity` signs."""
        buf = torch.empty(max(int(capacity), 1), dtype=torch.int64, device=self.device)
        count = torch.zeros(1, dtype=torch.int32, device=self.device)
        N.check(self.lib.pb_inc_take(self.h, _ptr(buf), int(capacity), _ptr(count), _stream(self.device)))
        n = int(count)
        if n > capacity:
            return None
        signs = buf[:n]
        if not n:
            return signs, torch.zeros((0, self.entry_len), dtype=torch.float32, device=self.device), \
                torch.zeros(0, dtype=torch.bool, device=self.device)
        ent, found = self.get_entries(signs)
        return signs, ent, found

    def take_incremental(self, capacity=None):
        """Empties the set.  Returns (signs, entries, skipped): the held signs that are still resident (HBM or tier),
        int64 bit patterns sorted ascending as u64, on the host; their entries (f32 [n, entry_len], on the host); and
        the number of held signs no table holds any more (evicted and dropped since they were marked), which are
        skipped as the reference skips them (lib.rs:187-192).  capacity: the set's (None: sized by a first call)."""
        while True:
            n = capacity
            if n is None:
                count = torch.zeros(1, dtype=torch.int32, device=self.device)
                N.check(self.lib.pb_inc_take(self.h, None, 0, _ptr(count), _stream(self.device)))
                n = int(count)
            got = self.take_incremental_device(n)
            if got is not None:  # (marks enqueued from another thread since the sizing call can grow the set)
                return host_entries(*got)
            if capacity is not None:
                raise RuntimeError("the set holds more signs than the capacity given")

    def __len__(self):
        """Entries held: the HBM rows plus the host tier's."""
        n = int(self.counters()["admitted"])
        return n + int(self.tier_stats()["host_rows"]) if self.host_tier is not None else n

    def clear(self):
        N.check(self.lib.pb_table_clear(self.h, _stream(self.device)))

    # lookup_mixed (PS mod.rs:344-357)
    def lookup(self, signs, training=True, out=None):
        signs = _as_i64_bits(signs)
        n = signs.numel()
        if out is None:
            out = torch.empty((n, self.dim), dtype=torch.float32, device=self.device)
        N.check(self.lib.pb_lookup(self.h, _ptr(signs), n, int(training), _ptr(out), _stream(self.device)))
        return out

    # update_gradient_mixed (PS mod.rs:359-427); signs must be distinct within one call
    def update(self, signs, grads):
        signs = _as_i64_bits(signs)
        grads = grads.contiguous()
        assert grads.dtype == torch.float32 and grads.numel() == signs.numel() * self.dim
        N.check(self.lib.pb_update(self.h, _ptr(signs), _ptr(grads), signs.numel(), _stream(self.device)))

    # set_embedding (PS mod.rs:287-306)
    def set_entries(self, signs, entries):
        signs = _as_i64_bits(signs)
        entries = entries.contiguous()
        assert entries.dtype == torch.float32 and entries.numel() == signs.numel() * self.entry_len
        N.check(self.lib.pb_set_rows(self.h, _ptr(signs), _ptr(entries), signs.numel(), _stream(self.device)))

    def get_entries(self, signs):
        signs = _as_i64_bits(signs)
        n = signs.numel()
        ent = torch.empty((n, self.entry_len), dtype=torch.float32, device=self.device)
        found = torch.empty(n, dtype=torch.uint8, device=self.device)
        N.check(self.lib.pb_get_rows(self.h, _ptr(signs), n, _ptr(ent), _ptr(found), _stream(self.device)))
        return ent, found.bool()

    def _export_table(self, h):
        count = torch.zeros(1, dtype=torch.int32, device=self.device)
        N.check(self.lib.pb_table_export_signs(h, None, None, 0, _ptr(count), _stream(self.device)))
        n = int(count)
        signs = torch.empty(n, dtype=torch.int64, device=self.device)
        rec = torch.empty(n, dtype=torch.int32, device=self.device)
        if n:
            N.check(self.lib.pb_table_export_signs(h, _ptr(signs), _ptr(rec), n, _ptr(count), _stream(self.device)))
            assert int(count) == n, "the table changed during the export"
        return signs, rec

    def export_signs(self):
        """Resident signs (int64 bit patterns) and the training-request number each was last used in, on the device,
        sorted oldest first (ties by sign): the order the reference's LRU list is dumped in.  With a host tier, the
        signs of both tables (they share one clock)."""
        signs, rec = self._export_table(self.h)
        if self.host_tier is not None:
            ts, tr = self._export_table(self.host_tier.h)
            signs, rec = torch.cat([signs, ts]), torch.cat([rec, tr])
        if signs.numel():
            order = torch.argsort(signs, stable=True)           # deterministic file: by sign ...
            order = order[torch.argsort(rec[order].to(torch.int64) & 0xFFFFFFFF, stable=True)]  # ... inside a request
            signs, rec = signs[order], rec[order]
        return signs, rec

    # checkpoint images on the device (include/persia_b200.h, pb_table_dump_*)
    def node_bytes(self):
        """Bytes of one entry's node in a `.emb` list: 29 + 4 * entry_len."""
        return 29 + 4 * self.entry_len

    def dump_reserve(self, max_bytes):
        """Allocates the dump workspace for images of up to max_bytes (synchronises the device)."""
        N.check(self.lib.pb_table_dump_reserve(self.h, int(max_bytes)))

    def dump_release(self):
        N.check(self.lib.pb_table_dump_release(self.h))

    def dump_part(self, part, n_parts, image, meta, stream=None):
        """Enqueues part `part` of `n_parts` on `stream` (None: the current one): its image into `image` (device uint8,
        16-byte aligned; its size is the image bound), its size into meta[0] and the table's request number into the low
        word of meta[1] (meta: device int64 [2])."""
        st = C.c_void_p((stream or torch.cuda.current_stream(self.device)).cuda_stream)
        base = meta.data_ptr()
        N.check(self.lib.pb_table_dump_part(self.h, int(part), int(n_parts), _ptr(image), image.numel(), C.c_void_p(base),
                                            C.c_void_p(base + 8), st))

    def dump_nodes(self, signs, lo, n, out):
        """Nodes [lo, lo + n) of the list of `signs` (device int64, in list order) into `out` (device uint8, 16-byte
        aligned, n * node_bytes()), on the current stream."""
        signs = _as_i64_bits(signs)
        N.check(self.lib.pb_dump_nodes(self.h, _ptr(signs), signs.numel(), int(lo), int(n), _ptr(out),
                                       _stream(self.device)))

    def export_view(self):
        """The table's view blob (bytes) for peers that read it in place (pb_table_export_view).  From now on the table
        is read-only but for set_entries and checkpoint / packet inserts, and it must outlive every view of it.  With a
        shared tier the tier's blob follows the table's in the same bytes (pb_table_export_tier_view)."""
        return self._export(self.lib.pb_table_export_view)

    def export_live_view(self):
        """The table's view blob (bytes) for peers that read it in place while it keeps training
        (pb_table_export_live_view): the blob export_view gives, read by the same TableView and RemoteReader, but the
        table stays writable.  Sweeps, index rebuilds, set_entries and clear are bracketed for the readers (with a shared
        tier, every move between the table and its tier too); a read beside an optimizer step may see each element before
        or after it.  One table, one export mode; the table must outlive every view of it."""
        return self._export(self.lib.pb_table_export_live_view)

    def add_readers(self, addresses):
        """Registers the views of this exported table opened in other processes (TableView.address of each; "" and
        None are skipped) so that they receive its chunks as it grows (pb_table_add_reader).  Only a table created with
        grow="shared" has readers; for any other this does nothing."""
        if not self.grow_shared:
            return
        for a in addresses:
            if a:
                N.check(self.lib.pb_table_add_reader(self.h, a.encode() if isinstance(a, str) else bytes(a)))

    def _export(self, call):
        buf = C.create_string_buffer(int(self.lib.pb_table_view_bytes()))
        N.check(call(self.h, buf))
        if not self.shared_tier:
            return buf.raw
        tier = C.create_string_buffer(int(self.lib.pb_tier_view_bytes()))
        N.check(self.lib.pb_table_export_tier_view(self.h, tier))
        return buf.raw + tier.raw

    def close(self):
        if getattr(self, "h", None):
            self.lib.pb_table_destroy(self.h)
            self.h = None
        if getattr(self, "host_tier", None) is not None:  # after the table it stands behind
            self.host_tier.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class TableView:
    """Another rank's exported table as this process reads it on `device` (pb_view_open / pb_view_close): through CUDA
    IPC when the blob comes from another process, through its own pointers when from this one.  A blob of a table with a
    shared tier opens both (pb_view_open_tiered; from another process the tier's rows are mapped through /proc)."""

    def __init__(self, blob, device=0):
        self.lib = N.load()
        self.device = torch.device("cuda", device) if not isinstance(device, torch.device) else device
        blob = bytes(blob)
        n = int(self.lib.pb_table_view_bytes())
        h = C.c_void_p()
        if len(blob) == n + int(self.lib.pb_tier_view_bytes()):  # a table with a shared tier: its blob, then the tier's
            N.check(self.lib.pb_view_open_tiered(self.device.index or 0, blob[:n], blob[n:], C.byref(h)))
        else:
            assert len(blob) == n, "not a table view blob"
            N.check(self.lib.pb_view_open(self.device.index or 0, blob, C.byref(h)))
        self.h = h

    @property
    def address(self):
        """The socket address the owner of a growable table (grow="shared") in another process sends its chunks to
        (EmbeddingShard.add_readers); "" for every other view.  Chunks that have arrived are mapped by each remote
        call itself."""
        buf = C.create_string_buffer(108)
        N.check(self.lib.pb_view_address(self.h, buf, len(buf)))
        return buf.value.decode()

    def close(self):
        if getattr(self, "h", None):
            self.lib.pb_view_close(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BatchContext:
    """Device-side per-batch context + workspace for the batched forward/backward of one shard."""

    def __init__(self, max_occurrences, max_out_rows, prefixes, sqrt_scaling=None, prefix_bit=8, device=0):
        if len(prefixes) > N.PB_MAX_SLOTS:
            raise ValueError(f"a batch context serves at most PB_MAX_SLOTS = {N.PB_MAX_SLOTS} slots, got {len(prefixes)}")
        self.lib = N.load()
        self.device = torch.device("cuda", device) if not isinstance(device, torch.device) else device
        self.n_slots = len(prefixes)
        self.prefixes, self.prefix_bit = [int(p) for p in prefixes], int(prefix_bit)
        h = C.c_void_p()
        N.check(self.lib.pb_ctx_create(self.device.index or 0, int(max_occurrences), int(max_out_rows), C.byref(h)))
        self.h = h
        cfg = N.SlotsCfg()
        cfg.n_slots, cfg.prefix_bit = self.n_slots, prefix_bit
        for i, p in enumerate(prefixes):
            cfg.prefix[i] = int(p)
            cfg.sqrt_scaling[i] = int(bool(sqrt_scaling[i])) if sqrt_scaling is not None else 0
        N.check(self.lib.pb_ctx_set_slots(self.h, C.byref(cfg)))

    def batch_stats(self):
        """Dedup statistics of the last training batch (host sync): distinct items and their multiplicity classes."""
        return _read_block(BATCH_STATS_FIELDS, lambda out: self.lib.pb_ctx_batch_stats(self.h, out, _stream(self.device)),
                           C.c_uint32)

    def forward(self, shard, ids, slot_occ_off, batch, row_off=None, training=True, out=None):
        """ids: flat device int64-bit ids (slot-major); slot_occ_off: host list, n_slots+1;
        row_off: device int32 CSR offsets [n_slots*batch+1] or None (one id per sample per slot).
        Returns f16 [n_slots, batch, dim]."""
        ids = _as_i64_bits(ids)
        if out is None:
            out = torch.empty((self.n_slots, batch, shard.dim), dtype=torch.float16, device=self.device)
        if row_off is not None:
            assert row_off.dtype == torch.int32 and row_off.is_contiguous()
        N.check(self.lib.pb_forward(shard.h, self.h, _ptr(ids), ids.numel(), _ptr(row_off),
                                    _slot_offsets(slot_occ_off, self.n_slots), int(batch), int(training), _ptr(out),
                                    _stream(self.device)))
        return out

    def backward(self, shard, grads, scales=None, want_status=False):
        """grads: list (per slot) of device tensors [batch, dim] (all f16 or all f32) or None (skipped), or an
        [n_slots, batch, dim] tensor.  A tensor that is not 16-byte aligned is copied first."""
        ptrs, is_f16, held = _slot_grads(grads, self.n_slots)  # (held through the call)
        status = torch.empty(self.n_slots, dtype=torch.int32, device=self.device) if want_status else None
        N.check(self.lib.pb_backward(shard.h, self.h, ptrs, int(is_f16), _scales(scales, self.n_slots), _ptr(status),
                                     _stream(self.device)))
        return status

    def backward_ptrs(self, shard, ptrs, is_f16, scales=None):
        """GradientBatch form (persia-core/src/backward.rs:86-105): raw device pointers, None = skipped slot.  A pointer
        that is not 16-byte aligned is refused (PersiaB200Error)."""
        N.check(self.lib.pb_backward(shard.h, self.h, _grad_ptrs(ptrs, self.n_slots), int(bool(is_f16)),
                                     _scales(scales, self.n_slots), None, _stream(self.device)))

    def forward_raw(self, shard, ids, batch, sample_fixed_size, row_off=None, training=True):
        """Raw (embedding_summation: false) slot; the context must have been built with ONE prefix.
        Returns (table f16 [n_occ+1, dim] of which rows [0, U] are valid, index i64 [batch*fixed],
        non_empty i64 [batch*fixed] of which counts[1] entries are valid, sample_id_num i32 [batch],
        counts i32 [2] = (U, non-empty entries)), all on the device (mod.rs:586-623, forward.rs:336-347)."""
        assert self.n_slots == 1, "a raw context serves one slot"
        ids = _as_i64_bits(ids)
        n, fixed = ids.numel(), int(sample_fixed_size)
        out = _raw_outputs(n, batch, fixed, shard.dim, self.device)
        N.check(self.lib.pb_forward_raw(shard.h, self.h, _ptr(ids), n, _raw_row_off(row_off, batch), int(batch), fixed,
                                        int(training), *map(_ptr, out), _stream(self.device)))
        table, index, non_empty, sample_id_num, counts = out
        return table, index, non_empty, sample_id_num[:batch], counts

    def backward_raw(self, shard, grad, scale=1.0, want_status=False, is_f16=None):
        """grad: device tensor [U, dim] (f32 as persia/ctx.py:970-980 builds it, or f16), a raw device pointer
        (then pass is_f16), or None (add_skipped_gradient)."""
        ptr, is_f16, held = _raw_grad(grad, is_f16, self)  # (held through the call)
        status = torch.empty(1, dtype=torch.int32, device=self.device) if want_status else None
        N.check(self.lib.pb_backward_raw(shard.h, self.h, ptr, int(bool(is_f16)), float(scale), _ptr(status),
                                         _stream(self.device)))
        return status

    def close(self):
        if getattr(self, "h", None):
            self.lib.pb_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def host_entries(signs, ent, found):
    """take_incremental_device's result on the host: (signs int64 sorted ascending as u64, entries, skipped) of the
    signs found."""
    import numpy as np

    found = found.cpu().numpy()
    signs = signs.cpu().numpy()[found]
    ent = ent.cpu().numpy()[found]
    order = np.argsort(signs.view(np.uint64), kind="stable")
    return signs[order], ent[order], int((~found).sum())


def add_prefix(ids, slot_occ_off, prefixes, prefix_bit=8):
    lib = N.load()
    ids = _as_i64_bits(ids)
    out = torch.empty_like(ids)
    S = len(prefixes)
    N.check(lib.pb_add_prefix(_ptr(ids), ids.numel(), _slot_offsets(slot_occ_off, S), _prefixes(prefixes), S, prefix_bit,
                              _ptr(out), _stream(ids.device)))
    return out


def shard_of(signs, R):
    lib = N.load()
    signs = _as_i64_bits(signs)
    out = torch.empty(signs.numel(), dtype=torch.int32, device=signs.device)
    N.check(lib.pb_shard_of(_ptr(signs), signs.numel(), R, _ptr(out), _stream(signs.device)))
    return out


def hash_stack(ids, rounds, embedding_size, out=None):
    """indices_to_hashstack_indices (mod.rs:347-400) on the device: [n] ids -> [n * rounds] keys, id-major."""
    lib = N.load()
    ids = _as_i64_bits(ids)
    if out is None:
        out = torch.empty(ids.numel() * int(rounds), dtype=torch.int64, device=ids.device)
    N.check(lib.pb_hash_stack(_ptr(ids), ids.numel(), int(rounds), int(embedding_size), _ptr(out), _stream(ids.device)))
    return out


def farmhash64(x):
    lib = N.load()
    x = _as_i64_bits(x)
    out = torch.empty_like(x)
    N.check(lib.pb_farmhash64(_ptr(x), x.numel(), _ptr(out), _stream(x.device)))
    return out


HOT_GEOMETRY_FIELDS = ("EPL", "CH", "PW", "vec", "vshift", "lean", "R1", "R", "S", "cols", "stride", "passes")


def hot_geometry(dim, f16, ragged=False):
    """The geometry the backward gives its reduce of hot signs (include/persia_b200.h, pb_hot_geometry) as a dict keyed
    by HOT_GEOMETRY_FIELDS.  Host-only."""
    return _read_block(HOT_GEOMETRY_FIELDS,
                       lambda out: N.load().pb_hot_geometry(int(dim), int(bool(f16)), int(bool(ragged)), out), C.c_uint32)


def partition_by_shard(signs, R):
    """Stable partition: returns (perm int32[n], counts int32[R])."""
    lib = N.load()
    signs = _as_i64_bits(signs)
    n = signs.numel()
    perm = torch.empty(n, dtype=torch.int32, device=signs.device)
    counts = torch.empty(R, dtype=torch.int32, device=signs.device)
    wb = int(lib.pb_partition_workspace(n))
    work = torch.empty(wb, dtype=torch.uint8, device=signs.device)
    N.check(lib.pb_partition_by_shard(_ptr(signs), n, R, _ptr(perm), _ptr(counts), _ptr(work), wb, _stream(signs.device)))
    return perm, counts
