"""`persia_core` surface over libpersia_b200.so — the module `persia/prelude.py:6` imports.

The reference's `persia_core` is a PyO3 cdylib (rust/persia-core/src/lib.rs:461-497) whose engines talk to an
embedding worker and parameter servers over HTTP/NATS.  This module keeps the names, arities, ownership rules
and error behaviour of that surface (SURVEY.md §8b) for a single box: the "servers" are pb_tables in this
process's GPU, `get_embedding_from_data` / `Forward.get_batch` run pb_forward, `Backward` runs pb_backward on
the raw device pointers `GradientBatch.add_gradient` receives.  `install()` registers it (and its submodules)
in `sys.modules` as `persia_core`, after which the reference's own `persia` package runs unchanged on top.

Scope: summation and raw slots (no hash-stack on raw slots), one process per GPU.  With `replica_size > 1` every dim
group is served by a ShardedEmbeddingWorker and every raw slot by its own ShardedRawWorker (persia_b200.worker), all
of one dim on the rank's one table; summation slots there may share a feature group (each rank's entries of a shared
sign are applied in slot order, the ranks in rank order), but a raw slot may not share its feature group with another
slot of the batch.
Their calls are collective, so every rank issues them in one fixed order: the raw slots in batch order, then the
summation dims in ascending order, in the forward and again in the backward; every batch must carry the same raw
slots in the same order.  `Forward` prefetches on worker threads with the reference's ordering and
staleness rules (persia_b200/engine.py), `Backward` applies updates in the caller's thread; `to_bytes()` is a private encoding (the speedy wire format is N4); `dump`/`load`
write and read the reference's `.emb` checkpoint files (persia_b200/checkpoint.py).
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


class _State:
    def __init__(self):
        self.reset()

    def reset(self):
        self.prefix_bit, self.slots, self.by_name = 8, [], {}
        self.groups = {}  # dim -> dict(shard, ctx pool, slot indices)
        self.capacity = int(os.environ.get("PERSIA_B200_CAPACITY", 1 << 22))
        self.optimizer = None
        self.hyper = None
        self.device_id = None
        self.replica_index, self.replica_size = 0, 1
        self.dataflow_sender = None
        self.next_batch_id = 0
        self.forward_id_buffer = {}
        self.raw_order = None  # replica_size > 1: the raw slots of the first batch, in order (every batch must match)

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
            sh = SH.EmbeddingShard(dim, self.capacity, dev)
            sh.set_eviction()  # the reference's holder is an LRU map bounded by `capacity` (eviction_map.rs:76-97)
            if self.optimizer is not None:
                sh.set_optimizer(**self.optimizer)
            if self.hyper is not None:
                sh.configure(**self.hyper)
            g = self.groups[dim] = {"shard": sh, "ctx": {}, "device": dev, "lock": threading.RLock()}
        return g

    def all_groups(self):
        self.ensure_config()
        return [self.group(d) for d in sorted({s.dim for s in self.slots})]


_S = _State()


def set_embedding_config(cfg):
    """Programmatic stand-in for the PERSIA_EMBEDDING_CONFIG yaml the reference's servers read
    (persia-embedding-config/src/lib.rs:566-585)."""
    _S.set_config(cfg)


def reset():
    """Drop every table and configuration (tests)."""
    for g in _S.groups.values():
        g["shard"].close()
    _S.reset()


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
    """What the EW keeps under backward_ref_id (mod.rs:1087-1098): per dim group, the device context."""

    def __init__(self):
        self.parts = []  # (group, ctx, [slot names in order], is_raw)

    def release(self):
        for g, ctx, _, _ in self.parts:
            if ctx is not None:  # sharded groups keep their one context inside the worker
                g["ctx"].setdefault(ctx._pool_key, []).append(ctx)
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


_STATE_LOCK = threading.RLock()  # configuration / group creation; GPU work takes the lock of the table it touches
_BACKWARDS = []                   # live Backward engines (direct lookups wait for their queues to drain)


def _forward(batch, device_id, training, direct=False):
    if direct:  # forward_directly (forward.rs:782-831) carries no staleness permit: see every update already handed over
        for b in list(_BACKWARDS):
            b.flush()
    return _forward_locked(batch, device_id, training)


def _forward_locked(batch, device_id, training):
    import torch

    from . import shard as SH

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
    pending = _Pending()
    by_slot = {}
    raw_out = {}
    for n, x in feats:  # raw slots: one request each (FeatureRawEmbeddingBatch, mod.rs:586-623)
        sc = _S.by_name[n]
        if sc.embedding_summation:
            continue
        with _STATE_LOCK:
            g = _S.group(sc.dim)
        if sharded:  # R GPUs: one request per owner, through the slot's raw worker
            with g["lock"]:
                ids, row_off, _ = _flatten([(n, x)], B)
                wk = _sharded_raw_worker(g, sc, B, ids, row_off, dev)
                d_ids = torch.from_numpy(ids.view(np.int64)).to(dev, non_blocking=True)
                d_off = torch.from_numpy(row_off.view(np.int32)).to(dev, non_blocking=True) if row_off is not None else None
                table, index, non_empty, num, counts = wk.forward_raw(d_ids, B, sc.sample_fixed_size, row_off=d_off,
                                                                      training=training)
                if wk.status()[0]:
                    raise RuntimeError("a batch requested more distinct signs of one shard than the exchange holds: raise "
                                       "PERSIA_B200_XCHG_CAP")
                U, ne = counts.tolist()
            raw_out[n] = (Tensor(table[:U + 1], n), Tensor(index, f"{n}_index"),
                          Tensor(non_empty[:ne], f"{n}_non_empty_index"), num.tolist())
            if training:
                pending.parts.append((g, None, [n], True))
            continue
        key = ("raw", n)
        pool = g["ctx"].setdefault(key, [])
        ids, row_off, _ = _flatten([(n, x)], B)
        g["lock"].acquire()
        if pool and pool[-1]._cap >= max(len(ids), B):
            ctx = pool.pop()
        else:
            cap = max(2 * len(ids), 2 * B, 1024)
            ctx = SH.BatchContext(cap, cap, [sc.index_prefix], None, _S.prefix_bit, dev)
            ctx._pool_key, ctx._cap = key, cap
        d_ids = torch.from_numpy(ids.view(np.int64)).to(dev, non_blocking=True)
        d_off = torch.from_numpy(row_off.view(np.int32)).to(dev, non_blocking=True) if row_off is not None else None
        table, index, non_empty, num, counts = ctx.forward_raw(g["shard"], d_ids, B, sc.sample_fixed_size, row_off=d_off,
                                                               training=training)
        U, ne = counts.tolist()  # the distinct-sign table is sized on the host, like the reference's CPU tensors
        raw_out[n] = (Tensor(table[:U + 1], n), Tensor(index, f"{n}_index"),
                      Tensor(non_empty[:ne], f"{n}_non_empty_index"), num.tolist())
        if training:
            pending.parts.append((g, ctx, [n], True))
        else:
            pool.append(ctx)
        g["lock"].release()
    for dim in sorted({_S.by_name[n].dim for n, _ in feats if _S.by_name[n].embedding_summation}):
        part = [(n, x) for n, x in feats if _S.by_name[n].dim == dim and _S.by_name[n].embedding_summation]
        names = [n for n, _ in part]
        with _STATE_LOCK:
            g = _S.group(dim)
        key = tuple(names)
        pool = g["ctx"].setdefault(key, [])
        ids, row_off, slot_off = _flatten(part, B)
        slots = [_S.by_name[n] for n in names]
        if (_S.replica_size or 1) > 1:  # R GPUs: the embedding worker's fan-out runs inside the sharded worker
            with g["lock"]:
                d_ids, row_off, slot_off = _to_device_ids(ids, row_off, slot_off, slots, B, dev)
                if g.get("worker") is None and any(sc.hash_stack_rounds > 0 for sc in slots):
                    ids = d_ids.cpu().numpy().view(np.uint64)  # (the first batch sizes the exchange from its keys)
                wk = _sharded_worker(g, dim, names, B, ids, row_off, slot_off, dev)
                d_off = torch.from_numpy(row_off.view(np.int32)).to(dev, non_blocking=True) if row_off is not None else None
                out = wk.forward(d_ids, B, training=training, row_off=d_off, slot_occ_off=slot_off)
                if wk.status()[0]:
                    raise RuntimeError("a batch requested more distinct signs of one shard than the exchange holds: raise "
                                       "PERSIA_B200_XCHG_CAP")
            for i, n in enumerate(names):
                by_slot[n] = out[i]
            if training:
                pending.parts.append((g, None, names, False))
            continue
        g["lock"].acquire()
        d_ids, row_off, slot_off = _to_device_ids(ids, row_off, slot_off, slots, B, dev)
        if pool and pool[-1]._cap >= d_ids.numel():
            ctx = pool.pop()
        else:
            cap = max(int(d_ids.numel()), len(names) * max(B, 1), 1)
            ctx = SH.BatchContext(max(cap * 2, 1024), max(len(names) * max(B, 1) * 2, 1024),
                                  [_S.by_name[n].index_prefix for n in names],
                                  [_S.by_name[n].sqrt_scaling for n in names], _S.prefix_bit, dev)
            ctx._pool_key, ctx._cap = key, max(cap * 2, 1024)
        d_off = torch.from_numpy(row_off.view(np.int32)).to(dev, non_blocking=True) if row_off is not None else None
        out = ctx.forward(g["shard"], d_ids, slot_off, B, row_off=d_off, training=training)
        for i, n in enumerate(names):
            by_slot[n] = out[i]
        if training:
            pending.parts.append((g, ctx, names, False))
        else:
            pool.append(ctx)
        g["lock"].release()
    emb = [Embedding(None, raw=raw_out[n]) if n in raw_out else Embedding(Tensor(by_slot[n], n)) for n, _ in feats]
    to_dev = lambda items: [Tensor(torch.from_numpy(a).to(dev), n) for n, a in items]  # noqa: E731
    return PersiaTrainingBatch(to_dev(batch.non_id_type_features), emb, to_dev(batch.labels), batch.meta_data,
                               pending if training else None)


def _sharded_worker(g, dim, names, B, ids, row_off, slot_off, dev):
    """The dim group's ShardedEmbeddingWorker (persia_b200/worker.py), created by the first batch: a collective —
    every rank's first lookup of the group must happen in the same step (it does: the ranks train in lockstep)."""
    wk = g.get("worker")
    if wk is not None:
        if wk.names != tuple(names):
            raise RuntimeError("on R GPUs every batch must carry the same summation slots of a dim, in the same order")
        return wk
    import torch
    import torch.distributed as dist

    from .worker import ShardedEmbeddingWorker as W

    if not dist.is_initialized():
        raise RuntimeError("replica_size > 1 needs torch.distributed (TrainCtx initialises it; else call init_process_group)")
    slots = [_S.by_name[n] for n in names]
    cap = _exchange_cap([(ids[slot_off[i]:slot_off[i + 1]], sc.index_prefix) for i, sc in enumerate(slots)], dev)
    ragged = row_off is not None
    per_sample = max(1, -(-len(ids) // max(1, len(names) * B)))
    max_batch = int(os.environ.get("PERSIA_B200_MAX_BATCH", B))
    # the group's table is the rank's shard: raw workers of this dim serve it too
    wk = W.distributed(len(names), dim, [sc.index_prefix for sc in slots], _S.capacity, cap, _S.optimizer or {}, dev,
                       hyper=_S.hyper, max_batch=max(B, max_batch), sqrt_scaling=[sc.sqrt_scaling for sc in slots],
                       rows_f32=ragged, prefix_bit=_S.prefix_bit, max_ids_per_sample=2 * per_sample if ragged else 1,
                       shard=g["shard"])
    wk.names = tuple(names)
    g["worker"] = wk
    return wk


def _sharded_raw_worker(g, sc, B, ids, row_off, dev):
    """Raw slot `sc`'s ShardedRawWorker (persia_b200/worker.py) over the rank's table of its dim, created by the first
    batch that carries the slot: a collective, like _sharded_worker."""
    wk = g.setdefault("raw_workers", {}).get(sc.name)
    if wk is not None:
        return wk
    import torch.distributed as dist

    from .worker import ShardedRawWorker

    if not dist.is_initialized():
        raise RuntimeError("replica_size > 1 needs torch.distributed (TrainCtx initialises it; else call init_process_group)")
    cap = _exchange_cap([(ids, sc.index_prefix)], dev)
    ragged = row_off is not None
    per_sample = max(1, -(-len(ids) // max(1, B)))
    max_batch = int(os.environ.get("PERSIA_B200_MAX_BATCH", B))
    wk = ShardedRawWorker.distributed(1, sc.dim, [sc.index_prefix], _S.capacity, cap, _S.optimizer or {}, dev,
                                      hyper=_S.hyper, max_batch=max(B, max_batch, 1), prefix_bit=_S.prefix_bit,
                                      max_ids_per_sample=2 * per_sample if ragged else 1, shard=g["shard"])
    g["raw_workers"][sc.name] = wk
    return wk


def _exchange_cap(slot_ids, dev):
    """Slots per (source, owner) pair of a new exchange: PERSIA_B200_XCHG_CAP, else from this first batch — the
    distinct signs it requests of one owner, largest over the ranks (a collective), with a generous margin.
    slot_ids: [(flat ids of one slot, its index_prefix)]."""
    import torch
    import torch.distributed as dist

    cap = int(os.environ.get("PERSIA_B200_XCHG_CAP", 0))
    if cap:
        return cap
    R = dist.get_world_size()
    counts = np.zeros(R, np.int64)
    spacing = np.uint64((1 << (64 - _S.prefix_bit)) - 1)
    for x, prefix in slot_ids:
        u = np.unique(x % spacing + np.uint64(prefix) if prefix else x)
        counts += np.bincount((farmhash64_np(u) % np.uint64(R)).astype(np.int64), minlength=R)
    t = torch.tensor([int(counts.max())], dtype=torch.int64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return (int(int(t) * 1.5) + 1024 + 7) // 8 * 8


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
            for g, ctx, names, is_raw in p.parts:
                with g["lock"]:
                    if is_raw:  # [U, dim] gradient of the distinct-sign table (persia/ctx.py:970-980)
                        item = grads.get(names[0])
                        if ctx is None:  # R GPUs: the slot's raw worker (a collective, even when skipped)
                            wk = g["raw_workers"][names[0]]
                            if item is None:
                                wk.backward_raw(None)
                            else:
                                ptr, shape, is16, sc = item
                                wk.backward_raw(ptr, scale=sc, is_f16=is16)
                        elif item is None:
                            ctx.backward_raw(g["shard"], None)
                        else:
                            ptr, shape, is16, sc = item
                            ctx.backward_raw(g["shard"], ptr, scale=sc, is_f16=is16)
                        continue
                    ptrs, scales, f16 = [], [], None
                    for n in names:
                        item = grads.get(n)
                        if item is None:
                            ptrs.append(None)
                            scales.append(1.0)
                            continue
                        ptr, shape, is16, sc = item
                        if f16 is not None and f16 != is16:
                            raise RuntimeError("gradients of one batch must share a dtype")
                        f16 = is16
                        ptrs.append(ptr)
                        scales.append(sc)
                    if g.get("worker") is not None:
                        g["worker"].backward_ptrs(ptrs, bool(f16), scales)
                    else:
                        ctx.backward_ptrs(g["shard"], ptrs, bool(f16), scales)
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
        for g in _S.groups.values():
            g["shard"].set_optimizer(**_S.optimizer)


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

        self._engine = ForwardEngine(lookup, forward_buffer_size, reproducible, embedding_staleness,
                                     world_size=max(1, _S.replica_size or 1), rank=_S.replica_index or 0)
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
        for g in _S.all_groups():
            g["shard"].clear()

    def dump(self, dst_dir):  # lib.rs:356-366 -> PS dump (mod.rs:453-458): the reference's .emb files
        from . import checkpoint as CK

        _S.ensure_config()
        CK.dump_shards(dst_dir, [g["shard"] for g in _S.all_groups()], _S.replica_index or 0, max(1, _S.replica_size or 1))

    def load(self, src_dir):  # lib.rs:368-378 -> PS load (mod.rs:460-466)
        from . import checkpoint as CK

        _S.ensure_config()
        if _S.optimizer is None:
            raise RuntimeError("optimizer not registered: the entry layout (embedding ++ state) is unknown")
        dims = sorted({s.dim for s in _S.slots})
        CK.load_shards(src_dir, {d: _S.group(d)["shard"] for d in dims}, _S.replica_index or 0, max(1, _S.replica_size or 1))

    def wait_for_serving(self):
        return None

    def wait_for_emb_loading(self):
        return None

    def wait_for_emb_dumping(self):
        return None

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


_PUBLIC = ("PersiaCommonContext", "is_cuda_feature_available", "set_embedding_config", "reset", "parse_embedding_config")
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
