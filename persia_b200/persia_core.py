"""`persia_core` surface over libpersia_b200.so — the module `persia/prelude.py:6` imports.

The reference's `persia_core` is a PyO3 cdylib (rust/persia-core/src/lib.rs:461-497) whose engines talk to an
embedding worker and parameter servers over HTTP/NATS.  This module keeps the names, arities, ownership rules
and error behaviour of that surface (SURVEY.md §8b) for a single box: the "servers" are pb_tables in this
process's GPU, `get_embedding_from_data` / `Forward.get_batch` run pb_forward, `Backward` runs pb_backward on
the raw device pointers `GradientBatch.add_gradient` receives.  `install()` registers it (and its submodules)
in `sys.modules` as `persia_core`, after which the reference's own `persia` package runs unchanged on top.

Scope: summation and raw slots (no hash-stack on raw slots), one process per GPU.  A batch's units (_units) are its raw
slots and its summation slots of each dim in chunks of at most PB_MAX_SLOTS slots, a feature group never split
(slot_chunks); each unit is served by one placement (forward, backward, release): a pooled batch context (_Local) or,
with `replica_size > 1`, its ShardedEmbeddingWorker or ShardedRawWorker (_ShardedPart, persia_b200.worker), all of one
dim on the rank's one table; summation slots there may share a feature group (each rank's entries of a shared sign are
applied in slot order, the ranks in rank order), but a raw slot may not share its feature group with another slot.
Their calls are collective, so every rank issues them in one fixed order (_units): the raw slots in batch order, then
the summation dims in ascending order, in the forward and again in the backward; every batch must carry the same raw
slots in the same order.  Every step on R GPUs is sized from its own batch (_sharded_step): each worker prepares its
batch locally (PB_PHASE_PREPARE), one all_reduce(MAX) agrees on every worker's need, and the exchanges that do not cover
it are replaced before any rank sends; an exchange overflow or a wait that gave up is then an internal error.  `Forward` prefetches on worker threads with the reference's ordering and
staleness rules (persia_b200/engine.py), `Backward` applies updates in the caller's thread; `to_bytes()` is a private encoding (the speedy wire format is N4); `dump`/`load`
write and read the reference's `.emb` checkpoint files (persia_b200/checkpoint.py).  With the global config's
`enable_incremental_update` on a Train job, the signs the tables step are flushed as the reference's `.inc` packets; an
Infer job loads its checkpoint and applies them as they appear (persia_b200/incremental.py, `set_global_config`).
At `replica_size > 1` every forward that does not train is served by its rank alone, reading the owners' shards in place
(_start_remote, _Remote): no collective.  An Infer job exports its tables frozen once its checkpoint is
loaded; a Train job exports them live when its optimizer is registered, and its training forwards and backwards stay
collective.

Host tiers (PERSIA_B200_HBM_ROWS: a table larger than that keeps the rest of `capacity` in host memory behind each
rank's HBM rows) serve one GPU only unless PERSIA_B200_SHARED_TIER=1.  With it set, every dim group's shard is created
with a shared tier (pb_table_create_host_shared) at any replica_size, and at replica_size > 1 both exports carry it: an
Infer job's frozen one (checkpoint loads and incremental packets included) and a Train job's live one, so a forward that
does not train reads tier-held signs from their owners' host rows in place.  It is an opt-in because shared host memory
costs more than private pinned memory: it is shmem charged to the owning rank's memory cgroup, every peer that reads
it pins it again, and the ranks must run as one user in one PID namespace (a peer maps the owner's memfd through
/proc/<pid>/fd).  Tier staging (worker.TierStager) stays off at replica_size > 1.

PERSIA_B200_GROW=1 (growth_on) makes every dim group's table growable: `capacity` bounds each table instead of
reserving HBM for it, and HBM backs rows and index cells as entries are admitted, so a config with several dims or the
reference's default capacity of 1e9 costs what its resident entries cost.  Every dim still has its own `capacity`.  It
is an opt-in, read when a dim group is created, so that the default stays today's allocation.  At replica_size > 1
tables are exported for remote reads, which PERSIA_B200_GROW=1's tables cannot be: there PERSIA_B200_GROW=shared is
needed, which makes them growable and exportable (growth mode 2: each rank's peers receive its chunks as they are
mapped, over a socket, and read while the table grows, _start_remote).  It works at any replica_size, for Train jobs
(live exports) and Infer jobs (frozen exports, grown by checkpoint loads and incremental packets).  Both are refused
together with PERSIA_B200_HBM_ROWS, before any table exists.
"""
import os
import queue
import sys
import threading
import types

import numpy as np

_SUPPORTED = {np.dtype(t) for t in (np.bool_, np.float32, np.float64, np.int8, np.int16, np.int32, np.int64,
                                     np.uint8, np.uint16, np.uint32, np.uint64)}  # data.rs:117-131
MAX_BATCH_SIZE = 65535  # persia-common/src/lib.rs:49-51


# ---------------------------------------------------------------------------------------------------------
# process-wide state: what the embedding worker + parameter servers hold in the reference
# ---------------------------------------------------------------------------------------------------------
class SlotConfig:
    def __init__(self, name, dim, embedding_summation=True, sqrt_scaling=False, sample_fixed_size=10,
                 hash_stack_rounds=0, hash_stack_embedding_size=0):
        self.name, self.dim = name, int(dim)
        self.embedding_summation, self.sqrt_scaling = bool(embedding_summation), bool(sqrt_scaling)
        self.sample_fixed_size = int(sample_fixed_size)
        self.hash_stack_rounds, self.hash_stack_embedding_size = int(hash_stack_rounds), int(hash_stack_embedding_size)
        self.index_prefix = 0


def parse_embedding_config(cfg):
    """persia-embedding-config/src/lib.rs:600-650: slots not named in a feature group form their own group
    (appended in slot order); index_prefix = (group index + 1) << (64 - feature_index_prefix_bit)."""
    bits = int(cfg.get("feature_index_prefix_bit", 8))
    if bits <= 0:
        raise RuntimeError("feature_index_prefix_bit must > 0")
    slots = []
    for name, sc in cfg["slots_config"].items():
        hs = sc.get("hash_stack_config") or {}
        if sc.get("index_prefix", 0):
            raise RuntimeError("please do not set index_prefix manually")
        slots.append(SlotConfig(name, sc["dim"], sc.get("embedding_summation", True), sc.get("sqrt_scaling", False),
                                sc.get("sample_fixed_size", 10), hs.get("hash_stack_rounds", 0), hs.get("embedding_size", 0)))
    groups = [(g, list(names)) for g, names in (cfg.get("feature_groups") or {}).items()]
    grouped = {n for _, names in groups for n in names}
    group_names = {g for g, _ in groups}
    for s in slots:
        if s.name not in grouped:
            if s.name in group_names:
                raise RuntimeError("a slot name can not same with feature group name")
            groups.append((s.name, [s.name]))
    of = {n: gi for gi, (_, names) in enumerate(groups) for n in names}
    for s in slots:
        v = (of[s.name] + 1) << (64 - bits)
        if v >= 1 << 64:
            raise RuntimeError("slot index_prefix overflow, please try a bigger feature_index_prefix_bit")
        s.index_prefix = v
    return bits, slots


def hbm_split(capacity, hbm_rows, replica_size=1, shared=False):
    """(rows in HBM, rows of the host-memory tier behind them) of a table of `capacity` entries.  hbm_rows
    (PERSIA_B200_HBM_ROWS; None or "" = unset): a table larger than that keeps the rest in host memory, moved in and out
    by the kernels (include/persia_b200.h, pb_table_attach_tier); unset or >= capacity: everything in HBM, no tier.
    At replica_size > 1 a tier needs `shared` (PERSIA_B200_SHARED_TIER=1): its rows are then shared memory the peers'
    remote reads map (pb_table_create_host_shared)."""
    capacity = int(capacity)
    if hbm_rows is None or str(hbm_rows).strip() == "":
        return capacity, 0
    hbm_rows = int(hbm_rows)
    if hbm_rows <= 0:
        raise RuntimeError(f"PERSIA_B200_HBM_ROWS must be positive, got {hbm_rows}")
    if hbm_rows >= capacity:
        return capacity, 0
    if (replica_size or 1) > 1 and not shared:
        raise RuntimeError("PERSIA_B200_HBM_ROWS (a host-memory tier behind the HBM rows) is supported on one GPU only "
                           f"(replica_size = 1, got {replica_size}): unset it or raise it to the capacity ({capacity})")
    return hbm_rows, capacity - hbm_rows


def adagrad_rsqrt():
    """PERSIA_B200_ADAGRAD_RSQRT: "intel" steps Adagrad's fused lanes with _mm256_rsqrt_ps as Intel CPUs compute it, so
    that training matches the reference's bit for bit as run on an Intel CPU; unset or "exact": exact 1/sqrt.  Read when
    the optimizer is registered; every rank must see the same value."""
    v = os.environ.get("PERSIA_B200_ADAGRAD_RSQRT", "").strip() or "exact"
    if v not in ("exact", "intel"):
        raise RuntimeError(f"PERSIA_B200_ADAGRAD_RSQRT must be 'exact' or 'intel', got {v!r}")
    return v


def growth_on(grow, replica_size=1, hbm_rows=None):
    """PERSIA_B200_GROW (`grow`; "1" or "shared" on, None, "" or "0" off): every dim group's table is growable
    (pb_table_set_growth): `capacity` bounds it and HBM backs its rows and index as entries are admitted, so the
    reference's capacities (1e9 by default) can be configured as they are.  Returns False, True ("1") or "shared"
    (EmbeddingShard's `grow`).  "1" is refused at replica_size > 1 (a Train job exports its tables live, an Infer job
    frozen, and its tables cannot be exported); "shared" makes them exportable and works at any replica_size.  Both are
    refused together with PERSIA_B200_HBM_ROWS (`hbm_rows`: a growable table has no host tier)."""
    v = "" if grow is None else str(grow).strip()
    if v not in ("", "0", "1", "shared"):
        raise RuntimeError(f"PERSIA_B200_GROW must be '1', 'shared' or '0', got {v!r}")
    if v in ("", "0"):
        return False
    if v == "1" and (replica_size or 1) > 1:
        raise RuntimeError("PERSIA_B200_GROW=1 (tables that grow with their entries) is supported on one GPU only "
                           f"(replica_size = 1, got {replica_size}): its tables are exported for remote reads there; "
                           "PERSIA_B200_GROW=shared makes them exportable")
    if hbm_rows is not None and str(hbm_rows).strip() != "":
        raise RuntimeError(f"PERSIA_B200_GROW={v} cannot be combined with PERSIA_B200_HBM_ROWS: a growable table has no "
                           "host-memory tier")
    return True if v == "1" else "shared"


def shared_tier_on():
    """PERSIA_B200_SHARED_TIER=1: host tiers are created in shared memory (see the module docstring)."""
    return os.environ.get("PERSIA_B200_SHARED_TIER", "").strip() == "1"


class _State:
    def __init__(self):
        self.reset()

    def reset(self):
        self.prefix_bit, self.slots, self.by_name = 8, [], {}
        self.groups = {}  # dim -> dict(shard, ctx pool, slot indices)
        self.capacity = int(os.environ.get("PERSIA_B200_CAPACITY", 1 << 22))
        self.optimizer = None
        self.rsqrt = "exact"  # adagrad_rsqrt() when the optimizer was registered
        self.hyper = None
        self.device_id = None
        self.replica_index, self.replica_size = 0, 1
        self.dataflow_sender = None
        self.next_batch_id = 0
        self.forward_id_buffer = {}
        self.raw_order = None  # replica_size > 1: the raw slots of the first batch, in order (every batch must match)
        self.gcfg = None  # the global config's keys this project reads (incremental.parse_global_config)
        self.dumper = None  # Train with enable_incremental_update: the writer of this replica's flushes
        self.loader = None  # Infer: the scanner of this replica's incremental directory
        self.inc_lock = threading.Lock()
        self.packet_readers = {}  # device index -> _PacketReader (_apply_packet_file)
        self.packet_lock = threading.Lock()
        self.gcfg_raw = None  # the global config dict itself (keys parse_global_config does not carry)
        self.emb_dump = None  # the latest background dump (checkpoint.BackgroundDumper)
        self.emb_load = None  # the latest load (checkpoint.DeviceLoader)
        self.remote = None  # replica_size > 1: dim -> RemoteReader (_start_remote): one rank serves alone

    def global_config(self):
        """set_global_config's dict, else the PERSIA_GLOBAL_CONFIG yaml, else the reference's defaults."""
        if self.gcfg is None:
            from . import incremental as INC

            gc = {}
            g = os.environ.get("PERSIA_GLOBAL_CONFIG")
            if g and os.path.isfile(g):
                import yaml

                gc = yaml.safe_load(open(g)) or {}
            self.gcfg = INC.parse_global_config(gc)
            self.gcfg_raw = gc
        return self.gcfg

    def internal_shards(self):
        """num_hashmap_internal_shards of the global config: the least number of parts of a background dump."""
        from . import checkpoint as CK

        self.global_config()
        return CK.internal_shards(self.gcfg_raw)

    def wait_dump(self):
        """Returns once no background dump runs (its outcome stays in emb_dump for wait_for_emb_dumping)."""
        d = self.emb_dump
        if d is not None and d.running():
            d._thread.join()

    def wait_load(self):
        """Returns once no background load runs (its outcome stays in emb_load for wait_for_emb_loading)."""
        if self.emb_load is not None:
            self.emb_load.join()

    def device_loader(self, src_dir):
        """A checkpoint.DeviceLoader of src_dir into this replica's tables, under their groups' locks and fences."""
        from . import checkpoint as CK

        groups = {d: self.group(d) for d in sorted({s.dim for s in self.slots})}
        return CK.DeviceLoader(src_dir, {d: g["shard"] for d, g in groups.items()}, self.replica_index or 0,
                               max(1, self.replica_size or 1), locks={d: g["lock"] for d, g in groups.items()},
                               fences={d: g["fence"] for d, g in groups.items() if g.get("fence") is not None})

    def incremental_on(self):
        c = self.global_config()
        return c["job_type"] == "Train" and c["enable_incremental_update"]

    def set_config(self, cfg):
        self.prefix_bit, self.slots = parse_embedding_config(cfg)
        self.by_name = {s.name: s for s in self.slots}
        self.groups = {}

    def ensure_config(self):
        if self.slots:
            return
        path = os.environ.get("PERSIA_EMBEDDING_CONFIG")
        if not path or not os.path.isfile(path):
            raise RuntimeError("embedding config not found: set PERSIA_EMBEDDING_CONFIG or call "
                               "persia_core.set_embedding_config(dict)")
        import yaml

        self.set_config(yaml.safe_load(open(path)))
        g = os.environ.get("PERSIA_GLOBAL_CONFIG")
        if g and os.path.isfile(g) and "PERSIA_B200_CAPACITY" not in os.environ:
            gc = yaml.safe_load(open(g)) or {}
            cap = (gc.get("embedding_parameter_server_config") or {}).get("capacity")
            if cap:
                self.capacity = int(cap)

    def group(self, dim):
        """The shard (one per distinct dim) and its batch contexts, created on first use."""
        g = self.groups.get(dim)
        if g is None:
            from . import shard as SH

            dev = self.device_id if self.device_id is not None else 0
            shared = shared_tier_on()
            hbm_rows = os.environ.get("PERSIA_B200_HBM_ROWS")
            grow = growth_on(os.environ.get("PERSIA_B200_GROW"), self.replica_size, hbm_rows)
            hbm, tier = hbm_split(self.capacity, hbm_rows, self.replica_size, shared=shared)
            sh = SH.EmbeddingShard(dim, hbm, dev, tier_rows=tier, shared_tier=shared, grow=grow)
            sh.set_eviction()  # the reference's holder is an LRU map bounded by `capacity` (eviction_map.rs:76-97)
            if self.optimizer is not None:
                sh.set_optimizer(**self.optimizer)
                sh.set_rsqrt(self.rsqrt)
            if self.hyper is not None:
                sh.configure(**self.hyper)
            if self.incremental_on():  # twice the flush threshold: the set fills while a flush is being taken
                sh.enable_incremental(2 * self.global_config()["incremental_buffer_size"])
            g = self.groups[dim] = {"shard": sh, "ctx": {}, "device": dev, "lock": threading.RLock()}
            if (self.replica_size or 1) > 1:  # orders dumps against the sharded calls, whatever their streams
                from . import checkpoint as CK

                g["fence"] = CK.ShardedFence()
        return g

    def all_groups(self):
        self.ensure_config()
        return [self.group(d) for d in sorted({s.dim for s in self.slots})]


_S = _State()


def set_embedding_config(cfg):
    """Programmatic stand-in for the PERSIA_EMBEDDING_CONFIG yaml the reference's servers read
    (persia-embedding-config/src/lib.rs:566-585)."""
    _S.set_config(cfg)


def set_global_config(cfg):
    """Programmatic stand-in for the PERSIA_GLOBAL_CONFIG yaml (persia-embedding-config/src/lib.rs:355-447): of it this
    project reads embedding_parameter_server_config.{enable_incremental_update, incremental_buffer_size,
    incremental_dir, incremental_channel_capacity} and common_config.{job_type, checkpointing_config.num_workers,
    infer_config.embedding_checkpoint}.  (capacity keeps coming from PERSIA_B200_CAPACITY or the yaml.)  Set it before
    the first batch: the tables are created with it."""
    from . import incremental as INC

    _S.gcfg = INC.parse_global_config(cfg)
    _S.gcfg_raw = cfg or {}


def reset():
    """Drop every table and configuration (tests).  A running background dump is stopped first."""
    if _S.emb_dump is not None:
        _S.emb_dump.stop()
    if _S.emb_load is not None:
        _S.emb_load.stop()
    if _S.loader is not None:
        _S.loader.stop()
    if _S.dumper is not None:
        _S.dumper.close()
    for rd in _S.packet_readers.values():
        rd.close()
    _close_remote()  # (the views before the tables)
    for g in _S.groups.values():
        g["shard"].close()
    _S.reset()


def _close_remote():
    """Closes the remote readers (their contexts and views of the peers' tables), if any: by reset(), and at interpreter
    exit before any table (an atexit hook, so that the views never outlive this process's tables whatever order the
    objects are collected in).  A peer's table must outlive this rank's views of it, so the ranks of an Infer or a Train
    job stop together: end with a barrier (or dist.destroy_process_group after one) before any rank exits."""
    if _S.remote is not None:
        for rd in _S.remote.values():
            rd.close()
        _S.remote = None


def _maybe_flush_incremental():
    """After a batch's updates are enqueued: the reference dumps once its set holds more than incremental_buffer_size
    signs (lib.rs:265-275), one set per parameter server across every dim, so the threshold counts the signs of all of
    this replica's tables.  The held counts are read without a sync and may lag by the batches still in flight."""
    if not _S.incremental_on():
        return
    groups = [g for g in _S.groups.values()]
    if sum(g["shard"].incremental_held() for g in groups) > _S.global_config()["incremental_buffer_size"]:
        _flush_incremental()


def _flush_incremental():
    """Takes every table's set and hands one flush to the dumper.  Only device work is done here, under each group's
    lock and on the update stream: the take (one pass over the set) and the gather of the taken signs' entries into a
    device buffer, then one host sync to read how many signs there are.  The copy to the host, the sort and the files
    are the dumper thread's: it waits for an event recorded after the gathers.  A queued flush keeps its signs and
    entries in device memory (~1 GB per 10^6 signs at dim 128 with Adagrad) until the dumper has copied them out, so
    at most MAX_QUEUED_FLUSHES wait: past that the training thread waits for the writer rather than drop updates."""
    from . import incremental as INC

    c = _S.global_config()
    with _S.inc_lock:
        parts = _take_flush(_S.groups, 2 * c["incremental_buffer_size"])
        if _S.dumper is None:
            _S.dumper = INC.IncrementalDumper(c["incremental_dir"], _S.replica_index or 0, c["num_workers"],
                                              c["incremental_channel_capacity"])
        _S.dumper.wait_queued(MAX_QUEUED_FLUSHES - 1)
        _S.dumper.submit(parts)
    return _S.dumper


MAX_QUEUED_FLUSHES = 2  # flushes whose device buffers may wait for the dumper thread at once


def _take_flush(groups, capacity):
    """The device half of a flush over `groups` ({dim: group}, each a table of `capacity`-sign set and its lock);
    returns the host half, a callable that waits for the device work and gives the dumper's parts."""
    import torch

    from . import shard as SH

    taken = []
    for dim in sorted(groups):
        g = groups[dim]
        with g["lock"]:
            got = g["shard"].take_incremental_device(capacity)
        taken.append((dim, got))
    ready = torch.cuda.Event()
    ready.record()

    def parts():  # (on the dumper's thread)
        ready.synchronize()
        out = []
        for dim, (signs, ent, found) in taken:
            s, e, _ = SH.host_entries(signs, ent, found)
            out.append((s, dim, e))
        return out

    return parts


def _start_infer():
    """Infer: load infer_config.embedding_checkpoint, then scan incremental_dir/s{replica_index} for flushes
    (persia-embedding-parameter-server.rs:111-117, lib.rs:163-170).  Runs once the optimizer is registered (the entry
    layout is known then)."""
    from . import checkpoint as CK
    from . import incremental as INC

    c = _S.global_config()
    if c["job_type"] != "Infer" or _S.loader is not None:
        return
    _S.ensure_config()
    if c["embedding_checkpoint"]:
        _S.device_loader(c["embedding_checkpoint"]).run()
    if (_S.replica_size or 1) > 1:  # before the first packet: from the export on, inserts are bracketed for readers
        _start_remote()
    directory = os.path.join(c["incremental_dir"], f"s{_S.replica_index or 0}")
    _S.loader = INC.IncrementalLoader(directory, apply_file=_apply_packet_file)
    _S.loader.start()


def _start_remote(live=False):
    """R GPUs: every dim group exports its table and the ranks exchange the blobs once (collective: every rank registers
    its optimizer alike, an Infer job once its checkpoint is loaded, a Train job as its TrainCtx enters).  From then on a
    forward that does not train is served by the dim's RemoteReader (persia_b200/worker.py) on this rank alone: no
    _sharded_step, no all_reduce, so each rank answers its own requests whatever its peers do, as the reference's servers
    answer each request alone.  Infer (live = False): the tables are then read-only but for checkpoint loads and
    incremental packets, which the readers see whole or not at all.  Train (live = True): the tables keep training
    through the collective path; a read never returns another sign's row, and beside an optimizer step it may see each
    element before or after that step (include/persia_b200.h, pb_table_export_live_view)."""
    import torch.distributed as dist

    from .worker import RemoteReader

    if not dist.is_initialized():
        raise RuntimeError("replica_size > 1 needs torch.distributed (TrainCtx initialises it; else call init_process_group)")
    groups = {d: _S.group(d) for d in sorted({s.dim for s in _S.slots})}
    blobs = {}
    for d, g in groups.items():
        with g["lock"]:
            blobs[d] = g["shard"].export_live_view() if live else g["shard"].export_view()
    got = [None] * dist.get_world_size()
    dist.all_gather_object(got, blobs)  # one exchange for every dim
    rank = dist.get_rank()
    from . import shard as SH

    readers = {}
    for d, g in groups.items():
        views = [SH.TableView(got[q][d], g["shard"].device) if q != rank else None for q in range(len(got))]
        readers[d] = RemoteReader(g["shard"], views, rank)
    if any(g["shard"].grow_shared for g in groups.values()):  # (PERSIA_B200_GROW=shared: the same on every rank)
        addrs = [None] * len(got)  # each rank's view addresses, per dim and owner
        dist.all_gather_object(addrs, {d: [v.address if v is not None else "" for v in r.views]
                                       for d, r in readers.items()})
        for d, g in groups.items():
            with g["lock"]:
                g["shard"].add_readers([a[d][rank] for a in addrs])
    dist.barrier()  # (no rank reads before every view is open)
    _S.remote = readers
    global _CLOSE_AT_EXIT
    if not _CLOSE_AT_EXIT:
        import atexit

        atexit.register(_close_remote)
        _CLOSE_AT_EXIT = True


_CLOSE_AT_EXIT = False  # _close_remote is registered to run at interpreter exit


def _start_train_remote():
    """Train on R GPUs: once the optimizer is registered (every rank's TrainCtx registers it as it enters, in step), the
    tables are exported live and the views exchanged (_start_remote), once.  Where torch.distributed is not initialised
    nothing starts: the collective path, which needs it as well, then raises at the first forward, as before."""
    import torch.distributed as dist

    if _S.global_config()["job_type"] != "Train" or (_S.replica_size or 1) <= 1 or _S.remote is not None:
        return
    if not dist.is_initialized():
        return
    _S.ensure_config()
    _start_remote(live=True)


PACKET_CHUNK = 1 << 16  # entries of one pb_image_insert of a packet (device staging: PACKET_CHUNK x entry length floats)


class _PacketReader:
    """What _apply_packet_file keeps across the files it applies on one device: the pinned buffer a file is read into
    (grown when a file needs more), the pb_image that indexes it, the stream its inserts run on, and an event recorded
    after them, which the next file waits for before it overwrites the buffer."""

    def __init__(self, device):
        import torch

        from . import checkpoint as CK

        self.CK = CK
        self.stream = torch.cuda.Stream(device)
        self.done = torch.cuda.Event()
        self.image = CK._Image(device, PACKET_CHUNK)
        self.buf = None

    def read(self, path):
        """The file's bytes into the buffer; returns their count."""
        size = os.path.getsize(path)
        self.done.synchronize()
        if self.buf is None or self.buf.size < size:
            if self.buf is not None:
                self.buf.close()
            self.buf = self.CK._Pinned(max(64, size))
        with open(path, "rb") as fh:
            got = fh.readinto(memoryview(self.buf.view)[:size])
        if got != size:
            raise RuntimeError(f"{path} changed while it was read")
        return size

    def close(self):
        self.stream.synchronize()
        self.image.close()
        if self.buf is not None:
            self.buf.close()
            self.buf = None


def _dropped_so_far(sh, stream):
    """Entries the table and its tier have refused since creation: admissions the HBM table refused for capacity (with
    a tier, pb_set_rows gives each back when the tier stores the entry) plus the tier's drops.  Statistics calls are
    table calls: the caller holds the table's group lock.  Synchronises `stream`."""
    import torch

    with torch.cuda.stream(stream):
        return int(sh.counters()["capacity_refused"]) + int(sh.tier_stats()["dropped"])


def _apply_packet_file(path, groups=None, chunk=PACKET_CHUNK):
    """One packet file into the tables of its dims (groups: {dim: group}, None = this replica's), as
    _apply_incremental(*decode_packet(bytes)[:3], groups) applies it — the same checks and errors, dims ascending, each
    dim's entries in packet order through pb_set_rows, what was applied before an error kept — but decoded, selected and
    gathered on the device (pb_image_packet, pb_load.cu).  The file is read into a pinned buffer and indexed outside
    every lock; a group's lock is held while its dim's inserts (chunk entries each) are enqueued and the table's counters
    are read before and after them.  Returns (entries neither the HBM table nor its tier had room for, from those
    counters; entries the packet holds).  A packet of more dims or (dim, entry length) pairs than one device summary
    holds (pb_image_packet's PB_ERR_CAPACITY) is decoded on the host and applied by _apply_incremental instead."""
    import torch

    from . import incremental as INC
    from . import native as N

    groups = _S.groups if groups is None else groups
    dev = torch.device("cuda", next(iter(groups.values()))["device"] if groups else torch.cuda.current_device())
    chunk = max(1, min(int(chunk), PACKET_CHUNK))
    with _S.packet_lock:
        rd = _S.packet_readers.get(dev.index)
        if rd is None:
            rd = _S.packet_readers[dev.index] = _PacketReader(dev)
        nbytes = rd.read(path)
        try:
            try:
                summary, _ = rd.image.packet(rd.buf, nbytes, 1, 0, rd.stream)
            except N.PersiaB200Error as e:
                if e.code != N.PB_ERR_CAPACITY:
                    raise
                signs, dims, entries, _ = INC.decode_packet(rd.buf.view[:nbytes].tobytes())
                return _apply_incremental(signs, dims, entries, groups), int(signs.size)
            dropped = 0
            for dim in sorted({d for d, _, k in summary if k}):
                g = groups.get(dim)
                if g is None:
                    raise RuntimeError(f"incremental packet holds dim-{dim} entries but no slot has that dim")
                lens = {ln for d, ln, k in summary if d == dim and k}
                if len(lens) > 1:  # (np.stack's error in _apply_incremental)
                    raise ValueError("all input arrays must have the same shape")
                sh = g["shard"]
                if lens != {sh.entry_len}:
                    raise RuntimeError(f"dim-{dim} entries of {lens.pop()} floats, the registered optimizer needs "
                                       f"{sh.entry_len}")
                k = sum(n for d, _, n in summary if d == dim)
                with g["lock"]:
                    before = _dropped_so_far(sh, rd.stream)
                    for lo in range(0, k, chunk):
                        rd.image.insert(sh, dim, lo, min(lo + chunk, k), False, rd.stream)
                    dropped += (_dropped_so_far(sh, rd.stream) - before) % (1 << 32)  # (32-bit device counters)
            return dropped, sum(n for _, _, n in summary)
        finally:
            rd.done.record(rd.stream)


def _apply_incremental(signs, dims, entries, groups=None):
    """One packet into the tables of its dims (groups: {dim: group}, None = this replica's), through set_entries (HBM
    first, then the tier); returns the entries neither table had room for."""
    import torch

    dropped = 0
    groups = _S.groups if groups is None else groups
    for dim in np.unique(dims):
        g = groups.get(int(dim))
        if g is None:
            raise RuntimeError(f"incremental packet holds dim-{int(dim)} entries but no slot has that dim")
        pick = np.flatnonzero(dims == dim)
        ent = np.stack([entries[i] for i in pick])
        sh = g["shard"]
        if ent.shape[1] != sh.entry_len:
            raise RuntimeError(f"dim-{int(dim)} entries of {ent.shape[1]} floats, the registered optimizer needs "
                               f"{sh.entry_len}")
        dev = torch.device("cuda", g["device"])
        sg = torch.from_numpy(np.ascontiguousarray(signs[pick]).view(np.int64)).to(dev)
        with g["lock"]:
            sh.set_entries(sg, torch.from_numpy(ent).to(dev))
            dropped += int((~sh.get_entries(sg)[1]).sum())
    return dropped


def is_cuda_feature_available():  # lib.rs:452-459
    return True


# ---------------------------------------------------------------------------------------------------------
# forward.Tensor / Dtype
# ---------------------------------------------------------------------------------------------------------
class Dtype:
    _IDS = {"bool": 1, "float16": 2, "float32": 3, "float64": 4, "int8": 5, "int16": 6, "int32": 7, "int64": 8,
            "uint8": 9, "uint16": 10, "uint32": 11, "uint64": 12}

    def __init__(self, name):
        self._name = name

    @property
    def type_id(self):
        return self._IDS.get(self._name, 0)

    @property
    def type_name(self):
        return self._name


class Tensor:
    """forward.rs:119-254: a named buffer handed to torch through DLPack.  The wrapper must outlive the torch view
    (ctx.py keeps it in `emb_slots`); here it also owns the storage."""

    def __init__(self, data, name=None):
        import torch

        if isinstance(data, np.ndarray):  # #[new] from_numpy(&PyArray2<f32>)
            if data.dtype != np.float32 or data.ndim != 2:
                raise TypeError("Tensor(ndarray) expects a 2-D float32 array")
            data = torch.from_numpy(np.ascontiguousarray(data))
        self._t = data
        self._name = name

    @property
    def dlpack(self):
        import torch.utils.dlpack as dl

        return dl.to_dlpack(self._t)

    def check_dlpack(self, capsule):
        return None

    @property
    def data_ptr(self):
        return self._t.data_ptr()

    @property
    def shape(self):
        return list(self._t.shape)

    @property
    def dtype(self):
        return Dtype(str(self._t.dtype).replace("torch.", ""))

    @property
    def name(self):
        return self._name or ""

    @property
    def device(self):
        return "cuda" if self._t.is_cuda else "cpu"

    def numpy(self):
        return self._t.detach().cpu().numpy()


class Embedding:  # forward.rs:57-99
    def __init__(self, tensor, raw=None):
        self._inner = tensor   # sum: Tensor; raw: (Tensor table, Tensor index, Tensor non_empty_index, [sample_id_num])
        self._raw = raw is not None
        if self._raw:
            self._inner = raw

    def is_raw_embedding(self):
        return self._raw

    def get_sum_embedding(self):
        if self._raw:
            raise RuntimeError("AttrError: raw embedding can not convert to sum embedding")
        if self._inner is None:
            raise RuntimeError("embedding already taken")  # Option::take().unwrap() panics in the reference
        t, self._inner = self._inner, None
        return t

    def get_raw_embedding(self):
        if not self._raw:
            raise RuntimeError("AttrError: sum embedding can not convert to raw embedding")
        if self._inner is None:
            raise RuntimeError("embedding already taken")
        t, self._inner = self._inner, None
        return t


# ---------------------------------------------------------------------------------------------------------
# data.PersiaBatch
# ---------------------------------------------------------------------------------------------------------
def _as_array(obj, dtype, name):
    if not isinstance(dtype, np.dtype):
        raise RuntimeError(f"PersiaBatch datatype parse error {name or 'unknow_data'}, check PersiaBatch datatype "
                           f"support list to prevent datatype parse error.")
    if dtype not in _SUPPORTED:
        raise RuntimeError("Unsupport datatype of ndarray")
    return np.ascontiguousarray(obj, dtype=dtype)


def check_pyarray_dtype_valid(py_object, dtype, name=None):  # data.rs:137-140
    _as_array(py_object, dtype, name)


class PersiaBatch:  # data.rs:142-266
    def __init__(self):
        self.non_id_type_features, self.labels = [], []
        self.id_type_features = []       # taken by converted_id_type_features2embedding_tensor
        self.embedding_tensor = None     # ("ids", requires_grad, features) | ("ref", batch_id)
        self.meta_data = None
        self._batch_id = None

    def add_non_id_type_feature(self, pyarray_object, dtype, name=None):
        self.non_id_type_features.append((name, _as_array(pyarray_object, dtype, name)))

    def add_label(self, py_object, dtype, name=None):
        self.labels.append((name, _as_array(py_object, dtype, name)))

    def _push(self, name, lil):
        if self.id_type_features is None:
            raise RuntimeError("id_type_features already been taken")
        if len(lil) > MAX_BATCH_SIZE:
            raise RuntimeError(f"batch size cannot be larger than {MAX_BATCH_SIZE}")  # FeatureBatch::new panics
        self.id_type_features.append((name, lil))

    def add_id_type_feature(self, id_type_feature, id_type_feature_name):
        self._push(id_type_feature_name, [np.ascontiguousarray(x, dtype=np.uint64) for x in id_type_feature])

    def add_id_type_feature_with_single_id(self, id_type_feature, id_type_feature_name):
        self._push(id_type_feature_name, np.ascontiguousarray(id_type_feature, dtype=np.uint64))

    def converted_id_type_features2embedding_tensor(self, requires_grad=None):
        requires_grad = True if requires_grad is None else bool(requires_grad)
        if requires_grad and not self.labels:
            raise RuntimeError("add label data when requires_grad set to true.")
        feats, self.id_type_features = self.id_type_features, None
        self.embedding_tensor = ("ids", requires_grad, feats)

    def add_meta(self, data=None):
        self.meta_data = bytes(data) if data is not None else None

    def to_bytes(self):  # data.rs:256-258: the persia-speedy encoding of PersiaBatchImpl (persia_b200/speedy.py)
        from . import speedy

        e = self.embedding_tensor
        if e is None and self.id_type_features:
            raise RuntimeError("call converted_id_type_features2embedding_tensor before to_bytes")
        return speedy.encode_batch(self.non_id_type_features, e, self.labels, self.meta_data, self._batch_id)

    @staticmethod
    def _from_bytes(b):  # lib.rs:400-407 get_embedding_from_bytes: PersiaBatchImpl::read_from_buffer
        from . import speedy

        try:
            non_id, idf, labels, meta, batch_id = speedy.decode_batch(b)
        except speedy.SpeedyError as e:
            raise RuntimeError(f"PersiaBatch deserialization failed: {e}")
        p = PersiaBatch()
        p.non_id_type_features, p.labels, p.meta_data, p._batch_id = non_id, labels, meta, batch_id
        p.embedding_tensor = idf if idf is None or idf[0] == "ids" else ("ref", idf[1])
        p.id_type_features = None
        return p

    def batch_id(self):
        if self._batch_id is None:
            raise RuntimeError("please call forward_id before get batch_id")
        return self._batch_id


# ---------------------------------------------------------------------------------------------------------
# the forward itself: LIL id features -> pb_forward per dim group -> PersiaTrainingBatch
# ---------------------------------------------------------------------------------------------------------
class _Pending:
    """What the EW keeps under backward_ref_id (mod.rs:1087-1098): the placement of each of the batch's units
    (_Local or _ShardedPart), in the order of its forward."""

    def __init__(self):
        self.parts = []

    def release(self):
        for part in self.parts:
            part.release()
        self.parts = []


def farmhash64_np(x):
    """farmhash 1.1.5 hash64 of the 8 LE bytes of each u64 (FarmHash HashLen0to16, 8..16 branch), vectorised."""
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


def _hashstack(feature, slot):
    """indices_to_hashstack_indices (embedding_worker_service/mod.rs:347-400) as an id expansion: every id becomes
    `rounds` keys, key_r = farmhash64^(r+1)(id) % embedding_size + r * embedding_size; sample_num_signs grows by the
    same factor, which is what the sqrt scaling then counts."""
    R, size = slot.hash_stack_rounds, np.uint64(slot.hash_stack_embedding_size)
    rows = [np.array([v], np.uint64) for v in feature] if isinstance(feature, np.ndarray) else list(feature)
    out = []
    for ids in rows:
        h = np.ascontiguousarray(ids, dtype=np.uint64)
        keys = np.empty((h.size, R), np.uint64)
        for r in range(R):
            h = farmhash64_np(h)
            keys[:, r] = h % size + np.uint64(r) * size
        out.append(keys.reshape(-1))
    return out


def _flatten(feats, batch):
    """[(name, lil | single ids)] of one dim group -> flat ids, CSR offsets (None when one id per sample), slot offsets."""
    single = all(isinstance(x, np.ndarray) and x.ndim == 1 and x.dtype == np.uint64 for _, x in feats)
    if single:
        ids = np.concatenate([x for _, x in feats]) if feats else np.zeros(0, np.uint64)
        return ids, None, [i * batch for i in range(len(feats) + 1)]
    chunks, counts = [], []
    for _, x in feats:
        rows = [np.array([v], np.uint64) for v in x] if isinstance(x, np.ndarray) else x
        counts.extend(len(r) for r in rows)
        chunks.extend(rows)
    row_off = np.zeros(len(counts) + 1, np.uint32)
    row_off[1:] = np.cumsum(counts)
    ids = np.concatenate(chunks) if chunks else np.zeros(0, np.uint64)
    slot_off = [int(row_off[i * batch]) for i in range(len(feats) + 1)]
    return ids, row_off, slot_off


def _to_device_ids(ids, row_off, slot_off, slots, B, dev):
    """Flat host ids of one dim group -> device ids, with indices_to_hashstack_indices (embedding_worker_service/mod.rs:
    347-400) applied ON THE DEVICE to the slots that configure it (pb_hash_stack): every id becomes `rounds` keys next to
    each other, so the slot's samples hold `rounds` times as many ids (sample_num_signs, :393-397) and the CSR offsets
    are scaled on the host.  Returns (d_ids, row_off, slot_off)."""
    import torch

    from . import shard as SH

    d_raw = torch.from_numpy(ids.view(np.int64)).to(dev, non_blocking=True)
    rounds = [max(1, sc.hash_stack_rounds) for sc in slots]
    if all(r == 1 for r in rounds):
        return d_raw, row_off, slot_off
    n_in = [slot_off[i + 1] - slot_off[i] for i in range(len(slots))]
    new_off = [0]
    for n, r in zip(n_in, rounds):
        new_off.append(new_off[-1] + n * r)
    d_out = torch.empty(new_off[-1], dtype=torch.int64, device=dev)
    for i, sc in enumerate(slots):
        src = d_raw[slot_off[i]:slot_off[i + 1]]
        dst = d_out[new_off[i]:new_off[i + 1]]
        if rounds[i] == 1:
            dst.copy_(src)
        elif n_in[i]:
            SH.hash_stack(src, rounds[i], sc.hash_stack_embedding_size, out=dst)
    counts = np.ones(len(slots) * B, np.int64) if row_off is None else np.diff(row_off.astype(np.int64))
    counts = counts * np.repeat(np.array(rounds, np.int64), B)
    new_row_off = np.zeros(counts.size + 1, np.uint32)
    new_row_off[1:] = np.cumsum(counts)
    return d_out, new_row_off, new_off


def slot_chunks(prefixes):
    """The summation slots of one dim, given by their index prefixes in batch order, split into the batch contexts that
    serve them (a context holds at most PB_MAX_SLOTS slots): lists of slot indices, each in batch order.  A feature group
    (the slots of one index prefix) is never split: Adam advances a group's beta powers once per request, so a group
    served by two backwards would advance twice.  Groups are packed in the order of their first slot, so the split
    depends on the slots alone and every rank issues the same calls."""
    from .native import PB_MAX_SLOTS

    members = {}  # (insertion order: the order of each group's first slot)
    for i, p in enumerate(prefixes):
        members.setdefault(p, []).append(i)
    chunks, cur = [], []
    for idx in members.values():
        if len(idx) > PB_MAX_SLOTS:
            raise RuntimeError(f"a feature group of {len(idx)} summation slots of one dim: one batch context serves at "
                               f"most {PB_MAX_SLOTS} slots and a feature group is not split across contexts")
        if len(cur) + len(idx) > PB_MAX_SLOTS:
            chunks.append(sorted(cur))
            cur = []
        cur += idx
    if cur:
        chunks.append(sorted(cur))
    return chunks


MAX_CTX_OCCURRENCES = 1 << 24  # id occurrences one batch context holds (pb_ctx_create)


def ctx_occurrences(n_ids, rows=0):
    """Id occurrences of a pooled batch context made for a batch of n_ids ids in `rows` output rows (slots x samples):
    twice the larger of the two, so that later batches fit, but at most what one context holds.  A batch of more ids
    than that is refused."""
    if n_ids > MAX_CTX_OCCURRENCES:
        raise RuntimeError(f"a batch holds {n_ids} ids in the slots one batch context serves: at most "
                           f"{MAX_CTX_OCCURRENCES} (2^24) fit, split the batch")
    return min(max(2 * max(n_ids, rows), 1024), MAX_CTX_OCCURRENCES)


def ctx_size(n_ids, rows, held=(0, 0)):
    """(occurrences, output rows) of a batch context for n_ids ids in `rows` output rows, never less than the `held`
    (occurrences, rows) of the context it replaces: ctx_occurrences for the ids, twice the rows (at least 1024) for the
    outputs.  Every batch context persia_core and its workers make is sized by it."""
    return max(ctx_occurrences(n_ids, rows), held[0]), max(2 * rows, 1024, held[1])


_STATE_LOCK = threading.RLock()  # configuration / group creation; GPU work takes the lock of the table it touches
_BACKWARDS = []                   # live Backward engines (direct lookups wait for their queues to drain)


class _Sharded:
    """A sharded call on group g's table through worker wk (under the group's lock): ordered against the group's dumps
    by its ShardedFence (the table's chains do not order sharded calls)."""

    def __init__(self, g, wk):
        self.fence, self.wk = g.get("fence"), wk

    def __enter__(self):
        if self.fence is not None:
            self.st = self.wk._torch_stream()
            self.fence.call_begin(self.st)
        return self.wk

    def __exit__(self, *exc):
        if self.fence is not None:
            self.fence.call_end(self.st)


def _forward(batch, device_id, training, direct=False):
    if direct:  # forward_directly (forward.rs:782-831) carries no staleness permit: see every update already handed over
        for b in list(_BACKWARDS):
            b.flush()
    return _forward_locked(batch, device_id, training)


def _forward_locked(batch, device_id, training):
    import torch

    _S.ensure_config()
    if batch.embedding_tensor is None:
        raise RuntimeError("PersiaBatch holds no id_type_features: call converted_id_type_features2embedding_tensor first")
    if batch.embedding_tensor[0] == "ref":
        stored = _S.forward_id_buffer.pop(batch.embedding_tensor[1], None)
        if stored is None:
            raise RuntimeError("forward id not found")  # EmbeddingWorkerError::ForwardIdNotFound
        requires_grad, feats = stored
    else:
        _, requires_grad, feats = batch.embedding_tensor
    training = bool(training and requires_grad)
    if _S.device_id is None:
        _S.device_id = device_id if device_id is not None else 0
    dev = torch.device("cuda", _S.device_id)
    sizes = {len(x) for _, x in feats}
    if len(sizes) > 1:
        raise RuntimeError("id_type_features of one batch must share the batch size")
    B = sizes.pop() if sizes else 0
    for name, _ in feats:
        if name not in _S.by_name:
            raise RuntimeError(f"slot: {name} not found")  # get_slot_by_feature_name expect()
        sc = _S.by_name[name]
        if not sc.embedding_summation and sc.hash_stack_rounds > 0:
            raise RuntimeError(f"slot {name}: a raw (embedding_summation: false) slot with hash_stack is not supported")
    sharded = (_S.replica_size or 1) > 1
    if sharded:  # the collective calls of a step must come in the same order on every rank
        raw_names = tuple(n for n, _ in feats if not _S.by_name[n].embedding_summation)
        for n in raw_names:
            if sum(_S.by_name[m].index_prefix == _S.by_name[n].index_prefix for m, _ in feats) > 1:
                raise RuntimeError(f"slot {n}: on R GPUs a raw slot cannot share its feature group with another slot "
                                   "of the batch")
        if _S.raw_order is None:
            _S.raw_order = raw_names
        elif _S.raw_order != raw_names:
            raise RuntimeError("on R GPUs every batch must carry the same raw slots, in the same order")
    units = _units(feats, B)
    # R GPUs: a forward that does not train is read from the owners' shards by this rank alone (_start_remote), in Infer
    # and Train jobs; a training forward takes the collective path
    if sharded and not training and _S.remote is not None:
        parts = [_Remote(u, dev) for u in units]
    elif sharded:
        parts = _sharded_step(units, training, dev)
    else:
        parts = [_Local(u, dev) for u in units]
    pending = _Pending()
    by_slot, raw_out = {}, {}
    for u, part in zip(units, parts):
        with u.g["lock"]:
            out = part.forward(training)
            if u.raw:  # the distinct-sign table is sized on the host, like the reference's CPU tensors
                U, ne = out[4].tolist()
            if not training:
                part.release()
        if u.raw:  # one request per raw slot (FeatureRawEmbeddingBatch, mod.rs:586-623)
            (n,), (table, index, non_empty, num, _) = u.names, out
            raw_out[n] = (Tensor(table[:U + 1], n), Tensor(index, f"{n}_index"),
                          Tensor(non_empty[:ne], f"{n}_non_empty_index"), num.tolist())
        else:
            by_slot.update(zip(u.names, out))
        if training:
            pending.parts.append(part)
    emb = [Embedding(None, raw=raw_out[n]) if n in raw_out else Embedding(Tensor(by_slot[n], n)) for n, _ in feats]
    to_dev = lambda items: [Tensor(torch.from_numpy(a).to(dev), n) for n, a in items]  # noqa: E731
    return PersiaTrainingBatch(to_dev(batch.non_id_type_features), emb, to_dev(batch.labels), batch.meta_data,
                               pending if training else None)


class _Unit:
    """One lookup of a batch: a raw slot, or a chunk of one dim's summation slots (slot_chunks), with the dim's group.
    k: the chunk's index among its dim's chunks; dim_names: the dim's summation slots in batch order."""

    def __init__(self, feats, B, raw, k=0, dim_names=()):
        self.names = [n for n, _ in feats]
        self.slots = [_S.by_name[n] for n in self.names]
        self.dim, self.B, self.raw, self.k, self.dim_names = self.slots[0].dim, B, raw, k, dim_names
        self.key = ("raw", self.names[0]) if raw else tuple(self.names)  # (of its contexts in the group's pool)
        self.prefixes = [sc.index_prefix for sc in self.slots]
        self.sqrt = None if raw else [sc.sqrt_scaling for sc in self.slots]
        with _STATE_LOCK:
            self.g = _S.group(self.dim)
        self.ids, self.row_off, self.slot_off = _flatten(feats, B)

    def device_ids(self, dev):
        """(device ids, device CSR offsets or None, slot offsets), hash stack applied."""
        import torch

        d_ids, row_off, slot_off = _to_device_ids(self.ids, self.row_off, self.slot_off, self.slots, self.B, dev)
        d_off = torch.from_numpy(row_off.view(np.int32)).to(dev, non_blocking=True) if row_off is not None else None
        return d_ids, d_off, slot_off


def _units(feats, B):
    """A batch's lookups (_Unit) in the order every rank issues them on R GPUs: the raw slots in batch order, then the
    summation dims ascending, each chunk by chunk."""
    units = [_Unit([(n, x)], B, True) for n, x in feats if not _S.by_name[n].embedding_summation]
    for dim in sorted({_S.by_name[n].dim for n, _ in feats if _S.by_name[n].embedding_summation}):
        part = [(n, x) for n, x in feats if _S.by_name[n].dim == dim and _S.by_name[n].embedding_summation]
        names = tuple(n for n, _ in part)
        for k, chunk in enumerate(slot_chunks([_S.by_name[n].index_prefix for n in names])):
            units.append(_Unit([part[i] for i in chunk], B, False, k, names))
    return units


# A unit's placement: forward(training), under the group's lock, returns the outputs (summation) or forward_raw's five
# tensors (raw); backward(grad, is_f16, scale) steps a training forward's batch (_grad_args); release() follows the
# backward, or the forward at once when it does not train.
class _Local:
    """replica_size 1: a batch context from the group's pool on the group's own table, given back by release."""

    def __init__(self, u, dev):
        self.u, self.dev, self.ctx = u, dev, None

    def forward(self, training):
        from . import shard as SH

        u = self.u
        ids, off, slot_off = u.device_ids(self.dev)
        n, rows = int(ids.numel()), len(u.names) * u.B
        pool = u.g["ctx"].setdefault(u.key, [])
        if pool and n <= pool[-1]._size[0] and rows <= pool[-1]._size[1]:
            self.ctx = pool.pop()
        else:  # (covers the pool's top as well: batches of alternating shapes end up reusing one context)
            size = ctx_size(n, rows, pool[-1]._size if pool else (0, 0))
            self.ctx = SH.BatchContext(*size, u.prefixes, u.sqrt, _S.prefix_bit, self.dev)
            self.ctx._size = size
        try:
            if u.raw:
                return self.ctx.forward_raw(u.g["shard"], ids, u.B, u.slots[0].sample_fixed_size, row_off=off,
                                            training=training)
            return self.ctx.forward(u.g["shard"], ids, slot_off, u.B, row_off=off, training=training)
        except Exception:
            self.release()  # (a refused forward gives its context back)
            raise

    def backward(self, grad, is_f16, scale):
        if self.u.raw:
            self.ctx.backward_raw(self.u.g["shard"], grad, scale=scale, is_f16=is_f16)
        else:
            self.ctx.backward_ptrs(self.u.g["shard"], grad, is_f16, scale)

    def release(self):
        self.u.g["ctx"][self.u.key].append(self.ctx)


class _ShardedPart:
    """R GPUs: the unit's ShardedEmbeddingWorker or ShardedRawWorker (created by the first batch), its batch prepared
    here (local work: _sharded_step sizes the exchange after every unit is prepared).  Every later call is collective
    and ordered against the group's dumps (_Sharded); the worker keeps its one context."""

    def __init__(self, u, training, dev):
        g, self.u = u.g, u
        if u.k == 0 and not u.raw and g.setdefault("names", u.dim_names) != u.dim_names:
            raise RuntimeError("on R GPUs every batch must carry the same summation slots of a dim, in the same order")
        with g["lock"]:
            self.ids, self.off, self.slot_off = u.device_ids(dev)
            self.wk = _worker(u, dev)
            if u.raw:
                self.need = self.wk.prepare_raw(self.ids, u.B, u.slots[0].sample_fixed_size, row_off=self.off,
                                                training=training)
            else:
                self.need = self.wk.prepare(self.ids, u.B, row_off=self.off, slot_occ_off=self.slot_off,
                                            training=training)

    def forward(self, training):
        u = self.u
        with _Sharded(u.g, self.wk) as wk:
            if u.raw:
                out = wk.forward_raw(self.ids, u.B, u.slots[0].sample_fixed_size, row_off=self.off, training=training)
            else:
                out = wk.forward(self.ids, u.B, training=training, row_off=self.off, slot_occ_off=self.slot_off)
        _check_exchange(self.wk)
        return out

    def backward(self, grad, is_f16, scale):
        with _Sharded(self.u.g, self.wk) as wk:
            if self.u.raw:  # (a collective, even when skipped)
                wk.backward_raw(grad, scale=scale, is_f16=is_f16)
            else:
                wk.backward_ptrs(grad, is_f16, scale)

    def release(self):
        pass


class _Remote:
    """R GPUs, a forward that does not train: the dim's RemoteReader reads the owners' shards, for this rank alone."""

    def __init__(self, u, dev):
        self.u, self.dev, self.rd = u, dev, _S.remote[u.dim]
        self.raw_ids = u.device_ids(dev) if u.raw else None  # (a raw slot's ids are copied before the lock is taken)

    def forward(self, training):
        u = self.u
        if u.raw:
            ids, off, _ = self.raw_ids
            return self.rd.forward_raw(ids, u.B, u.slots[0].sample_fixed_size, u.prefixes[0], _S.prefix_bit,
                                       row_off=off)
        ids, off, slot_off = u.device_ids(self.dev)
        return self.rd.forward(ids, u.B, u.prefixes, u.sqrt, _S.prefix_bit, row_off=off, slot_occ_off=slot_off)

    def release(self):
        pass


def _grad_args(u, grads):
    """(gradient, is_f16, scale) of unit u's backward from the GradientBatch's items ((ptr, shape, is_f16, scale), or
    None when skipped): a raw slot's pointer to its [U, dim] gradient of the distinct-sign table (persia/ctx.py:970-980)
    or None, or a pointer (or None) and a scale per summation slot."""
    items = [grads.get(n) for n in u.names]
    dtypes = {it[2] for it in items if it is not None}
    if len(dtypes) > 1:
        raise RuntimeError("gradients of one batch must share a dtype")
    ptrs = [it[0] if it else None for it in items]
    scales = [it[3] if it else 1.0 for it in items]
    is16 = dtypes.pop() if dtypes else None
    return (ptrs[0], is16, scales[0]) if u.raw else (ptrs, bool(is16), scales)


def _sharded_step(units, training, dev):
    """R GPUs: sizes this step's exchanges from its own batch, agreed by every rank before any rank sends.  Every unit's
    worker is prepared (its batch context grown if need be, the batch deduplicated: local work) in the collective
    order (_units), and then _agree_and_resize sizes them all with one all-reduce.  Returns the units' placements
    (_ShardedPart)."""
    parts = [_ShardedPart(u, training, dev) for u in units]
    _agree_and_resize([(p.u.g, p.wk, p.need) for p in parts], dev)
    return parts


def _agree_and_resize(plan, dev):
    """plan: [(group, worker, (need, rows_f32))] of one step, in the collective order.  Every rank's needs are packed into
    one tensor and reduced by ONE all_reduce(MAX), so every rank gets the same agreed (need, rows_f32) per worker; then,
    in that order, each worker resizes where the agreed need exceeds its exchange (a collective of its own, which every
    rank enters alike: the decision depends only on agreed values and the exchange every rank shares).  Returns the
    agreed pairs."""
    import torch
    import torch.distributed as dist

    if not plan:
        return []
    packed = [v for _, _, (need, f32) in plan for v in (int(need), int(bool(f32)))]
    t = torch.tensor(packed, dtype=torch.int64, device=dev if dist.get_backend() == "nccl" else "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    v = t.tolist()
    agreed = [(v[2 * i], bool(v[2 * i + 1])) for i in range(len(plan))]
    for (g, wk, _), (need, f32) in zip(plan, agreed):
        with g["lock"]:
            wk.resize(need, f32)
    return agreed


def _check_exchange(wk):
    """After a sharded forward: a step sized by _agree_and_resize never overflows its exchange and never waits in vain,
    so either status flag is an internal error."""
    overflowed, gave_up = wk.status()
    if overflowed or gave_up:
        raise RuntimeError("internal error in the sharded exchange: " + ("a batch overflowed the size every rank agreed on"
                           if overflowed else "a wait for a peer gave up"))


def _stage(batch):
    """Forward's stage (ForwardEngine): for every dim group whose table has a host-memory tier, the host-tier moves the
    batch's training forward will need (pb_tier_stage) are issued now, while the batches before it still train: the
    signs of the group's summation slots (hash-stacked as _to_device_ids does) and raw slots, on a stream the group owns,
    under the group's lock.  Results do not change; the forward finds its entries in HBM.  Nothing runs for tables
    without a tier, inference batches, or on R GPUs (there a shared tier is not staged: on virtual ranks staging did not
    shorten a step, and it waits for a measurement on R real GPUs)."""
    import torch

    from .native import PB_MAX_SLOTS

    if (_S.replica_size or 1) > 1 or batch.embedding_tensor is None or not _S.slots:
        return
    if batch.embedding_tensor[0] == "ref":
        stored = _S.forward_id_buffer.get(batch.embedding_tensor[1])
        if stored is None:
            return
        requires_grad, feats = stored
    else:
        _, requires_grad, feats = batch.embedding_tensor
    sizes = {len(x) for _, x in feats}
    if not requires_grad or len(sizes) != 1 or any(n not in _S.by_name for n, _ in feats):
        return
    B = sizes.pop()
    dev = torch.device("cuda", _S.device_id if _S.device_id is not None else 0)
    for dim in sorted({_S.by_name[n].dim for n, _ in feats}):
        with _STATE_LOCK:
            g = _S.groups.get(dim)  # (a group is created by its first forward: nothing is held in a tier before)
        if g is None or g["shard"].host_tier is None:
            continue
        summ = [(n, x) for n, x in feats if _S.by_name[n].dim == dim and _S.by_name[n].embedding_summation]
        raw = [(n, x) for n, x in feats if _S.by_name[n].dim == dim and not _S.by_name[n].embedding_summation]
        with g["lock"]:
            if g.get("stage_stream") is None:
                g["stage_stream"] = torch.cuda.Stream(dev)
            with torch.cuda.stream(g["stage_stream"]):
                parts, off, prefixes = [], [0], []
                if summ:
                    ids, row_off, slot_off = _flatten(summ, B)
                    slots = [_S.by_name[n] for n, _ in summ]
                    d_ids, _, slot_off = _to_device_ids(ids, row_off, slot_off, slots, B, dev)
                    parts.append(d_ids)
                    off += [int(x) for x in slot_off[1:]]
                    prefixes += [sc.index_prefix for sc in slots]
                for n, x in raw:
                    ids, _, _ = _flatten([(n, x)], B)
                    parts.append(torch.from_numpy(ids.view(np.int64)).to(dev, non_blocking=True))
                    off.append(off[-1] + int(ids.size))
                    prefixes.append(_S.by_name[n].index_prefix)
                d = torch.cat(parts) if len(parts) > 1 else parts[0]
                for lo in range(0, len(prefixes), PB_MAX_SLOTS):  # pb_tier_stage takes at most PB_MAX_SLOTS slots
                    hi = min(lo + PB_MAX_SLOTS, len(prefixes))
                    g["shard"].stage(d[off[lo]:off[hi]], [o - off[lo] for o in off[lo:hi + 1]], prefixes[lo:hi],
                                     _S.prefix_bit)


def _worker(u, dev):
    """Unit u's worker (persia_b200/worker.py) over the rank's table of its dim: a ShardedRawWorker for a raw slot
    (g["raw_workers"], by slot name), a ShardedEmbeddingWorker for a summation chunk (g["workers"], by chunk u.k).  The
    first batch that carries the unit creates it: a collective — every rank's first lookup of the unit must happen in
    the same step (it does: the ranks train in lockstep).  It starts with the smallest exchange and context; its first
    prepare grows the context (ctx_size) and _agree_and_resize sizes the exchange, as they do at every later step."""
    workers = u.g.setdefault("raw_workers" if u.raw else "workers", {})
    key = u.names[0] if u.raw else u.k
    if key in workers:
        return workers[key]
    import torch.distributed as dist

    from .worker import ShardedEmbeddingWorker, ShardedRawWorker

    if not dist.is_initialized():
        raise RuntimeError("replica_size > 1 needs torch.distributed (TrainCtx initialises it; else call init_process_group)")
    cls = ShardedRawWorker if u.raw else ShardedEmbeddingWorker
    # the group's table is the rank's shard: every worker of the dim serves it
    workers[key] = cls.distributed(len(u.names), u.dim, u.prefixes, _S.capacity, 8, _S.optimizer or {}, dev,
                                   hyper=_S.hyper, max_batch=1, sqrt_scaling=u.sqrt, prefix_bit=_S.prefix_bit,
                                   shard=u.g["shard"])
    return workers[key]


class PersiaTrainingBatch:  # forward.rs:256-306, #[pyclass(dict)]: python attaches attributes to it
    def __init__(self, non_id, emb, labels, meta, pending):
        self._non_id, self._emb, self._labels, self._meta, self._pending = non_id, emb, labels, meta, pending
        self._permit = None  # embedding staleness permit (forward.rs:316): moves into the gradient batch

    def __del__(self):  # a batch dropped without an update gives its permit back, like the Rust Drop
        permit = getattr(self, "_permit", None)
        if permit is not None:
            permit.release()

    def embedding_worker_addr(self):
        return "local"

    def consume_all_non_id_type_feature_tensors(self):
        x, self._non_id = self._non_id, []
        return x

    def consume_all_id_type_feature_embedding_tensors(self):
        x, self._emb = self._emb, []
        return x

    def consume_all_label_tensors(self):
        x, self._labels = self._labels, []
        return x

    def consume_all_meta_data(self):
        return self._meta

    def create_gradient_batch(self):
        p, self._pending = self._pending, None
        gb = GradientBatch(p)
        gb._permit, self._permit = self._permit, None  # forward.rs:299-305
        return gb


# ---------------------------------------------------------------------------------------------------------
# backward.GradientBatch / Backward
# ---------------------------------------------------------------------------------------------------------
class GradientBatch:  # backward.rs:60-106
    def __init__(self, pending):
        self._pending = pending
        self._grads = {}
        self._permit = None

    def add_skipped_gradient(self, slot_name):
        self._grads[slot_name] = None

    def add_gradient(self, slot_name, data_ptr, shape, is_f16_gradient, scale_factor):
        self._grads[slot_name] = (int(data_ptr), tuple(shape), bool(is_f16_gradient), float(scale_factor))


class Backward:  # backward.rs:203-405
    """The NN worker's backward engine: `update_id_type_feature_gradient_batched` hands the gradient batch to a bounded
    queue (backward.rs:357-405; the reference's first stage copies the gradients to the host there — here they stay
    on the device, the raw pointers are simply passed on) and returns; `num_backward_worker` threads take batches off
    the queue, enqueue pb_backward on the table's stream and give the staleness permit back (backward.rs:304-354).
    A failing update is logged and the batch dropped, as in the reference (backward.rs:332-339).  Before `launch`
    (or after `shutdown`) updates are applied in the caller's thread."""

    def __init__(self, queue_size):
        self.queue_size = max(1, int(queue_size))
        self._q = queue.Queue(maxsize=self.queue_size)
        self._threads = []
        self._running = False
        self.dropped = 0

    def launch(self, num_backward_worker):
        if self._running:
            return
        self._running = True
        for i in range(max(1, int(num_backward_worker))):
            t = threading.Thread(target=self._worker, name=f"persia-backward-{i}", daemon=True)
            t.start()
            self._threads.append(t)
        _BACKWARDS.append(self)

    def shutdown(self):
        if not self._running:
            return
        self.flush()
        self._running = False
        for _ in self._threads:
            self._q.put(None)
        for t in self._threads:
            t.join(timeout=10)
        self._threads = []
        if self in _BACKWARDS:
            _BACKWARDS.remove(self)

    def flush(self):
        """Returns once every gradient batch handed over so far has been enqueued on the GPU."""
        if self._running:
            self._q.join()

    def _worker(self):
        import torch

        if _S.device_id is not None:
            torch.cuda.set_device(_S.device_id)  # every helper thread selects the device itself (backward.rs:240-244)
        while True:
            item = self._q.get()
            try:
                if item is None:
                    return
                try:
                    self._apply(*item)
                except Exception as e:  # noqa: BLE001 — logged and dropped, the trainer goes on (backward.rs:332-339)
                    self.dropped += 1
                    sys.stderr.write(f"[persia_b200] update_gradient_batched failed, batch dropped: {e!r}\n")
            finally:
                self._q.task_done()

    @staticmethod
    def _apply(p, grads, permit, ready=None):
        try:
            if ready is not None:  # the gradients were produced on the caller's stream: this thread's stream follows it
                import torch

                torch.cuda.current_stream().wait_event(ready)
            for part in p.parts:
                with part.u.g["lock"]:
                    part.backward(*_grad_args(part.u, grads))
            _maybe_flush_incremental()
        finally:
            p.release()
            if permit is not None:  # the update is enqueued: the batch no longer counts as in flight (backward.rs:341-343)
                permit.release()

    def update_id_type_feature_gradient_batched(self, gradients):
        p, gradients._pending = gradients._pending, None
        permit, gradients._permit = gradients._permit, None
        if p is None:
            if permit is not None:
                permit.release()
            raise RuntimeError("cannot find gradient batch")
        ready = getattr(gradients, "_ready", None)
        if self._running:
            self._q.put((p, gradients._grads, permit, ready))  # blocks when the queue is full (bounded channel)
        else:
            self._apply(p, gradients._grads, permit, ready)


# ---------------------------------------------------------------------------------------------------------
# optim.OptimizerBase
# ---------------------------------------------------------------------------------------------------------
class OptimizerBase:  # optim.rs:8-66
    def __init__(self):
        self._cfg = None

    def init_adagrad(self, lr, wd, g_square_momentum, initialization, eps, vectorwise_shared=None):
        from . import native as N

        kind = N.OPT_ADAGRAD_VW if vectorwise_shared else N.OPT_ADAGRAD
        self._cfg = dict(kind=kind, lr=lr, wd=wd, g_square_momentum=g_square_momentum, initialization=initialization, eps=eps)

    def init_sgd(self, lr, wd):
        from . import native as N

        self._cfg = dict(kind=N.OPT_SGD, lr=lr, wd=wd)

    def init_adam(self, lr, betas, eps):
        from . import native as N

        self._cfg = dict(kind=N.OPT_ADAM, lr=lr, beta1=betas[0], beta2=betas[1], eps=eps)

    def apply(self):  # register_optimizer on every PS (embedding_parameter_service/mod.rs:429-438)
        if self._cfg is None:
            raise RuntimeError("optimizer is not initialized")
        _S.optimizer = dict(self._cfg)
        _S.rsqrt = adagrad_rsqrt()
        for g in _S.groups.values():
            g["shard"].set_optimizer(**_S.optimizer)
            g["shard"].set_rsqrt(_S.rsqrt)  # the R-GPU workers serve this shard: an owner steps with its mode
        _start_infer()  # job_type Infer: the servers load their checkpoint and start scanning for incremental updates
        _start_train_remote()  # job_type Train on R GPUs: export the tables live for forwards that do not train


# ---------------------------------------------------------------------------------------------------------
# utils: channels / message queues (utils.rs:9-137)
# ---------------------------------------------------------------------------------------------------------
class PersiaBatchDataSender:
    def __init__(self, q):
        self._q = q

    def send(self, batch_data):
        self._q.put(batch_data)


class PersiaBatchDataReceiver:
    def __init__(self, q):
        self._q = q


class PersiaBatchDataChannel:
    def __init__(self, capacity):
        self._q = queue.Queue(maxsize=capacity)

    def get_sender(self):
        return PersiaBatchDataSender(self._q)

    def get_receiver(self):
        return PersiaBatchDataReceiver(self._q)


_MQ = {}
_MQ_LOCK = threading.Lock()


class PersiaMessageQueueServer:
    def __init__(self, port, cap):
        with _MQ_LOCK:
            self._q = _MQ.setdefault(int(port), queue.Queue(maxsize=cap))

    def put(self, data):
        self._q.put(bytes(data))

    def get(self):
        return self._q.get()


class PersiaMessageQueueClient:
    def __init__(self, server_addr):
        port = int(str(server_addr).rsplit(":", 1)[-1])
        with _MQ_LOCK:
            self._q = _MQ.setdefault(port, queue.Queue())

    def put(self, data):
        self._q.put(bytes(data))

    def get(self):
        return self._q.get()


# ---------------------------------------------------------------------------------------------------------
# forward.Forward (forward.rs:833-907): input channel -> lookup -> training batch
# ---------------------------------------------------------------------------------------------------------
class Forward:  # forward.rs:833-907 over persia_b200.engine.ForwardEngine (reorder, prefetch, staleness permits)
    def __init__(self, forward_buffer_size, reproducible, embedding_staleness=None):
        from .engine import ForwardEngine

        self.forward_buffer_size, self.reproducible, self.embedding_staleness = forward_buffer_size, reproducible, embedding_staleness

        def lookup(batch, permit):
            tb = _forward(batch, _S.device_id, training=True)
            tb._permit = permit
            return tb

        def stage(batch):
            _stage(batch)

        self._engine = ForwardEngine(lookup, forward_buffer_size, reproducible, embedding_staleness,
                                     world_size=max(1, _S.replica_size or 1), rank=_S.replica_index or 0, stage=stage)
        self._engine.is_remote_ref = lambda b: b.embedding_tensor is not None and b.embedding_tensor[0] == "ref"

    def set_input_channel(self, receiver):
        self._engine.set_input(receiver._q)

    def launch(self, num_workers):
        self._engine.launch(num_workers)

    def shutdown(self):
        self._engine.shutdown()

    def get_batch(self, timeout_ms):
        return self._engine.get_batch(timeout_ms)


# ---------------------------------------------------------------------------------------------------------
# PersiaCommonContext (lib.rs:190-450)
# ---------------------------------------------------------------------------------------------------------
class PersiaCommonContext:
    def __init__(self, num_coroutines_worker, replica_index, replica_size, device_id=None):
        # replica_size > 1: one process per GPU; the dim groups are then served by ShardedEmbeddingWorkers (rows
        # hash-sharded over the ranks, summation slots only), created by the first batch
        _S.replica_index, _S.replica_size = int(replica_index), int(replica_size)
        if device_id is not None:
            _S.device_id = int(device_id)
        self._master_addr = "127.0.0.1:0"

    def init_nats_publisher(self, world_size=None):
        return None

    def init_master_discovery_service(self, master_addr=None):
        if master_addr:
            self._master_addr = master_addr

    @property
    def master_addr(self):
        return self._master_addr

    def get_embedding_worker_addr_list(self):
        return ["local"]

    def init_rpc_client_with_addr(self, embedding_worker_addr):
        return None

    def wait_servers_ready(self):
        return "local"

    def get_embedding_size(self):
        return [len(g["shard"]) for g in _S.all_groups()]

    def clear_embeddings(self):
        _S.wait_dump()
        _S.wait_load()
        for g in _S.all_groups():
            g["shard"].clear()

    def dump(self, dst_dir, background=None):  # lib.rs:356-366 -> PS dump (mod.rs:453-458): the reference's .emb files
        """background: True starts a background dump (checkpoint.BackgroundDumper: the tables are dumped part by part
        while training goes on; wait_for_emb_dumping / dump_status follow it) and returns; False dumps now, one file per
        dim, each table read under its group's lock; None: background when PERSIA_B200_BACKGROUND_DUMP=1."""
        from . import checkpoint as CK

        if background is None:
            background = os.environ.get("PERSIA_B200_BACKGROUND_DUMP", "") == "1"
        _S.ensure_config()
        _S.wait_load()
        if _S.emb_dump is not None and _S.emb_dump.running():
            raise RuntimeError("an embedding dump is already running: wait_for_emb_dumping() first")
        groups = _S.all_groups()
        r, R = _S.replica_index or 0, max(1, _S.replica_size or 1)
        if not background:
            _S.emb_dump = None  # an earlier background dump's outcome no longer describes the latest dump
            CK.dump_shards(dst_dir, [g["shard"] for g in groups], r, R, locks=[g["lock"] for g in groups],
                           fences=[g.get("fence") for g in groups])
            return
        tables = [CK.DumpTable(g["shard"], g["lock"], fence=g.get("fence")) for g in groups]
        _S.emb_dump = CK.BackgroundDumper(dst_dir, tables, r, R, shards=_S.internal_shards()).start()

    def dump_status(self):
        """Not part of the reference surface (its servers report it through wait_for_emb_dumping's polling, rpc.rs:211-280):
        ("Idle", 1.0), ("Dumping", fraction done) or ("Failed", message) of this replica's latest background dump."""
        return _S.emb_dump.status() if _S.emb_dump is not None else ("Idle", 1.0)

    def load(self, src_dir, background=None):  # lib.rs:368-378 -> PS load (mod.rs:460-466)
        """Loads the checkpoint on the device (checkpoint.DeviceLoader: the tables end as load_shards leaves them).
        background: True starts the load and returns (wait_for_emb_loading / load_status follow it, as the reference's
        load_embedding_from_dir spawns one job per file, lib.rs:375-425); False loads now and raises what load_shards
        raises; None: background when PERSIA_B200_BACKGROUND_LOAD=1."""
        if background is None:
            background = os.environ.get("PERSIA_B200_BACKGROUND_LOAD", "") == "1"
        _S.wait_dump()
        _S.wait_load()
        _S.ensure_config()
        if _S.optimizer is None:
            raise RuntimeError("optimizer not registered: the entry layout (embedding ++ state) is unknown")
        _S.emb_load = _S.device_loader(src_dir)
        if background:
            _S.emb_load.start()
        else:
            _S.emb_load.run()

    def load_status(self):
        """The reference's server status of this replica's latest load (embedding_parameter_service/mod.rs:264-280):
        ("Loading", fraction done), ("Idle", 1.0) or ("Failed", "Type: message")."""
        return _S.emb_load.status() if _S.emb_load is not None else ("Idle", 1.0)

    def flush_incremental(self):
        """Not part of the reference surface (its manager flushes only on the threshold): takes every table's set of
        updated signs now, writes them as one incremental update and returns once it is on disk — for the end of
        training and for tests.  Returns the directory written (None when no sign was updated since the last flush)."""
        if not _S.incremental_on():
            raise RuntimeError("incremental updates are off: set embedding_parameter_server_config."
                               "enable_incremental_update on a Train job (set_global_config / PERSIA_GLOBAL_CONFIG)")
        for b in list(_BACKWARDS):
            b.flush()
        n = len(_S.dumper.written) if _S.dumper is not None else 0
        d = _flush_incremental()
        d.flush()
        return d.written[-1] if len(d.written) > n else None

    @property
    def incremental_loader(self):
        """Infer: the IncrementalLoader scanning this replica's incremental directory (poll() applies what is new)."""
        return _S.loader

    def wait_for_serving(self):
        """Blocks while a load runs (the reference's server is not ready_for_serving while it loads)."""
        _S.wait_load()

    def wait_for_emb_loading(self):
        """Blocks until this replica's load is done; RuntimeError("emb dump FAILED for server {r}, due to ...") (the
        reference's text, persia-core/src/rpc.rs:154-176) when it failed."""
        if _S.emb_load is not None:
            _S.emb_load.wait()

    def wait_for_emb_dumping(self):
        """Blocks until this replica's background dump is done (on replica 0: until the root marker is written, after
        every replica's); RuntimeError("emb dump FAILED for server {r}, due to ...") when it failed."""
        if _S.emb_dump is not None:
            _S.emb_dump.wait()

    def shutdown_servers(self):
        return None

    def send_id_type_features_to_embedding_worker(self, batch):  # lib.rs:342-354 -> EW forward_batch_id buffer
        if batch.embedding_tensor is None or batch.embedding_tensor[0] != "ids":
            raise RuntimeError("PersiaBatch holds no id_type_features to send")
        bid = _S.next_batch_id
        _S.next_batch_id += 1
        _, requires_grad, feats = batch.embedding_tensor
        _S.forward_id_buffer[bid] = (requires_grad, feats)
        batch.embedding_tensor = ("ref", bid)
        batch._batch_id = bid

    def send_non_id_type_features_to_nn_worker(self, batch):  # lib.rs:356-365 -> dataflow channel
        if _S.dataflow_sender is None:
            raise RuntimeError("dataflow is not initialized (nats.initialize_dataflow)")
        _S.dataflow_sender.send(batch)

    def configure_embedding_parameter_servers(self, initialize_lower, initialize_upper, admit_probability,
                                               enable_weight_bound, weight_bound):
        _S.hyper = dict(init_lower=initialize_lower, init_upper=initialize_upper, admit_probability=admit_probability,
                        enable_weight_bound=bool(enable_weight_bound), weight_bound=weight_bound)
        for g in _S.groups.values():
            g["shard"].configure(**_S.hyper)

    def get_embedding_from_data(self, batch, device_id=None):  # forward_directly (forward.rs:782-831)
        """forward_directly: this rank's pending backwards are flushed first.  On R GPUs a batch that does not train is
        then read from the owners' shards by this rank alone (_start_remote): it sees every update this rank handed
        over, but updates its peers' owners have not applied yet may still be missing, the staleness the reference's
        asynchronous backward workers give too."""
        return _forward(batch, device_id, training=True, direct=True)

    def get_embedding_from_bytes(self, data, device_id=None):
        return _forward(PersiaBatch._from_bytes(bytes(data)), device_id, training=True, direct=True)

    def read_from_file(self, file_path):
        with open(file_path, "rb") as f:
            return f.read()

    def dump_to_file(self, content, file_dir, file_name):
        os.makedirs(file_dir, exist_ok=True)
        with open(os.path.join(file_dir, file_name), "wb") as f:
            f.write(bytes(content))

    def get_entries(self, signs, dim, missing_ok=False):
        """Not part of the reference surface: reads back whole entries (embedding ++ optimizer state) of the given signs
        from the table of `dim` (tests; the reference has no read-back besides dump).  missing_ok: a list with None
        for the signs this replica does not hold."""
        import torch

        g = _S.group(int(dim))
        dev = torch.device("cuda", g["device"])
        with g["lock"]:
            ent, found = g["shard"].get_entries(torch.from_numpy(np.ascontiguousarray(signs, np.uint64).view(np.int64)).to(dev))
            if missing_ok:
                f, e = found.cpu().numpy().astype(bool), ent.cpu().numpy()
                return [e[k] if f[k] else None for k in range(e.shape[0])]
            if not bool(found.all()):
                raise RuntimeError("sign not resident")
            return ent.cpu().numpy()

    def set_embedding(self, embeddings):  # lib.rs:433-449: [(sign, emb f32 ndarray, opt f32 ndarray)]
        import torch

        _S.wait_dump()
        _S.ensure_config()
        by_dim = {}
        for sign, emb, opt in embeddings:
            emb = np.asarray(emb, np.float32).reshape(-1)
            opt = np.asarray(opt, np.float32).reshape(-1)
            by_dim.setdefault(emb.size, []).append((int(sign), np.concatenate([emb, opt])))
        for dim, items in by_dim.items():
            g = _S.group(dim)
            sh = g["shard"]
            dev = torch.device("cuda", g["device"])
            ent = np.stack([e for _, e in items])
            if ent.shape[1] != sh.entry_len:
                raise RuntimeError(f"entry length {ent.shape[1]} does not match dim + optimizer state = {sh.entry_len}")
            signs = np.array([s for s, _ in items], np.uint64)
            sh.set_entries(torch.from_numpy(signs.view(np.int64)).to(dev), torch.from_numpy(ent).to(dev))


def initialize_dataflow(world_size, channel):  # nats.rs:409-423
    _S.dataflow_sender = channel


# ---------------------------------------------------------------------------------------------------------
# module layout of the reference: persia_core.{data,forward,backward,optim,utils,nats}
# ---------------------------------------------------------------------------------------------------------
def _submodule(name, **objs):
    m = types.ModuleType(f"persia_core.{name}")
    for k, v in objs.items():
        setattr(m, k, v)
    return m


data = _submodule("data", PersiaBatch=PersiaBatch, check_pyarray_dtype_valid=check_pyarray_dtype_valid)
forward = _submodule("forward", Forward=Forward, Tensor=Tensor, PersiaTrainingBatch=PersiaTrainingBatch,
                     Embedding=Embedding, Dtype=Dtype)
backward = _submodule("backward", Backward=Backward, GradientBatch=GradientBatch)
optim = _submodule("optim", OptimizerBase=OptimizerBase)
utils = _submodule("utils", PersiaMessageQueueServer=PersiaMessageQueueServer, PersiaMessageQueueClient=PersiaMessageQueueClient,
                   PersiaBatchDataChannel=PersiaBatchDataChannel, PersiaBatchDataSender=PersiaBatchDataSender,
                   PersiaBatchDataReceiver=PersiaBatchDataReceiver)
nats = _submodule("nats", initialize_dataflow=initialize_dataflow)


_PUBLIC = ("PersiaCommonContext", "is_cuda_feature_available", "set_embedding_config", "set_global_config", "reset",
           "parse_embedding_config")
_facade = None


def install():
    """Make `import persia_core` resolve to this surface (what persia/prelude.py:6 imports).  The registered module
    is a facade holding only the public names and the six submodules: prelude.register_submodule walks every
    module-typed attribute recursively, so the implementation module (which imports os, numpy, ...) cannot be it."""
    global _facade
    if _facade is None:
        me = sys.modules[__name__]
        f = types.ModuleType("persia_core")
        f.__doc__ = __doc__
        for n in _PUBLIC:
            setattr(f, n, getattr(me, n))
        for n in ("data", "forward", "backward", "optim", "utils", "nats"):
            setattr(f, n, getattr(me, n))
        _facade = f
    sys.modules["persia_core"] = _facade
    for n in ("data", "forward", "backward", "optim", "utils", "nats"):
        sys.modules[f"persia_core.{n}"] = getattr(_facade, n)
    return _facade
