"""ShardedEmbeddingWorker — the embedding worker's fan-out over the R GPUs of one box.

Reference: rust/persia-embedding-server/src/embedding_worker_service/mod.rs.  There the EW shards a batch's distinct
signs by farmhash64(sign) % R and issues one HTTP `lookup_mixed` / `update_gradient_mixed` per parameter server
(:886-919, :835-859).  Here every rank is at once a data-parallel trainer (its own batches), the embedding worker of
those batches and parameter server `rank` (its pb_table).  The fan-out is inside libpersia_b200's kernels
(pb_forward_sharded / pb_backward_sharded, csrc/pb_shard.cu): signs, rows and reduced gradients are stored straight
into the receiver's area over NVLink peer mappings.  What is left on the host is set-up: sizing the areas, mapping
them (torch symmetric memory) and choosing `cap`, the slots per (source, owner) pair.

Semantics (DESIGN.md §Multi-GPU): a rank's batch is one request per owner — the reference's picture with R NN
workers.  An owner serves a step's R lookup requests together and applies its R gradient requests one after another
in rank order.  Both calls are collective.

Two ways to build the ranks of a box:
  * `ShardedEmbeddingWorker.distributed(...)`: one process per GPU (torchrun), areas in symmetric memory.
  * `ShardedEmbeddingWorker.local_group(R, ...)`: R virtual ranks on ONE GPU in one process, each with its own table,
    context and stream, areas in plain device memory.  Same kernels, same protocol; lets a single-GPU box run the
    R > 1 parity tests.  One host thread drives them phase by phase (group_forward / group_backward: all ranks send,
    then all serve, then all finish), so a rank never spins on a flag whose raising has not been enqueued yet.
"""
import ctypes as C
import os

import numpy as np
import torch

from . import native as N
from . import shard as SH


def distinct_per_owner(slot_ids, prefixes, R, prefix_bit=8):
    """Host-side (numpy) count of the distinct signs one batch requests of every owner: what `cap` must cover.
    slot_ids: each slot's uint64 ids (any lengths).  Mirrors indices_add_prefix + FeatureBatch::new + sign_to_shard_modulo."""
    from .persia_core import farmhash64_np

    spacing = np.uint64((1 << (64 - prefix_bit)) - 1)
    counts = np.zeros(R, np.int64)
    for x, prefix in zip(slot_ids, prefixes):
        x = np.asarray(x, dtype=np.uint64)
        u = np.unique(x % spacing + np.uint64(prefix) if prefix else x)
        counts += np.bincount((farmhash64_np(u) % np.uint64(R)).astype(np.int64), minlength=R)
    return counts


XCHG_STATUS_FIELDS = ("overflowed", "wait_gave_up")


def _by_phase(workers, *phases):
    """(rank, worker, phase) in the order one host thread drives the virtual ranks of one GPU: every phase is enqueued
    for all ranks before the next."""
    return ((r, w, ph) for ph in phases for r, w in enumerate(workers))


class ShardedEmbeddingWorker:
    def __init__(self, n_slots, dim, prefixes, capacity, device, rank, world, cap, area, peer_bases, optimizer,
                 hyper=None, max_batch=4096, sqrt_scaling=None, rows_f32=False, prefix_bit=8, stream=None,
                 max_ids_per_sample=1, shard=None, tier_rows=0, shared_tier=False, rsqrt=None, grow=False):
        """shard: an existing EmbeddingShard of this rank to serve (configured by its owner, who also closes it), so
        that the workers of one dim — summation slots and raw slots — share one table; None: a new one.  tier_rows > 0:
        the new shard has a host-memory tier of that many rows behind its `capacity` HBM rows (EmbeddingShard; a
        caller's `shard` brings its own tier or none); shared_tier: that tier is shared memory, so the shard can be exported
        to a RemoteReader (EmbeddingShard).  rsqrt: the new shard's Adagrad rsqrt mode (EmbeddingShard.set_rsqrt; None:
        exact).  grow: the new shard's storage grows with its entries (EmbeddingShard; not with a tier): True, or
        "shared" so that it can also be exported to a RemoteReader.  Statistics: `self.shard.tier_stats()`, `self.shard.storage_stats()`."""
        self.S, self.dim, self.rank, self.R, self.cap = n_slots, dim, rank, world, int(cap)
        self.device = device if isinstance(device, torch.device) else torch.device("cuda", device)
        self.lib = N.load()
        self.stream = stream
        self.area = area  # keeps the receive area alive
        self._own_shard = shard is None
        if shard is None:
            shard = SH.EmbeddingShard(dim, capacity, self.device, tier_rows=tier_rows, shared_tier=shared_tier, grow=grow)
            shard.set_optimizer(**optimizer)
            if rsqrt is not None:
                shard.set_rsqrt(rsqrt)
            shard.configure(**(hyper or {}))
        assert shard.dim == dim, "the shard holds another embedding dim"
        self.shard = shard
        self._ctx_args = (prefixes, sqrt_scaling, prefix_bit)
        self._new_ctx(n_slots * max_batch * max_ids_per_sample, n_slots * max_batch)
        self.rows_f32 = bool(rows_f32)
        self.h = None
        self._create_xchg(self.cap, self.rows_f32, peer_bases)

    def _new_ctx(self, max_occurrences, max_out_rows):
        self.ctx = SH.BatchContext(max_occurrences, max_out_rows, *self._ctx_args, self.device)
        self.ctx_occ, self.ctx_rows = int(max_occurrences), int(max_out_rows)

    def _create_xchg(self, cap, rows_f32, peer_bases):
        bases = (C.c_uint64 * self.R)(*[int(p) for p in peer_bases])
        h = C.c_void_p()
        N.check(self.lib.pb_xchg_create(self.device.index or 0, self.R, self.rank, int(cap), self.dim, int(rows_f32), bases,
                                        C.byref(h)))
        self.h = h

    # ---- set-up helpers --------------------------------------------------------------------------------------------
    @staticmethod
    def area_bytes(world, cap, dim, rows_f32=False):
        b = int(N.load().pb_xchg_bytes(world, int(cap), dim, int(rows_f32)))
        assert b > 0, "bad exchange geometry"
        return b

    @classmethod
    def local_group(cls, world, n_slots, dim, prefixes, capacity, cap, optimizer, device=0, shards=None, tier_rows=0,
                    shared_tier=False, **kw):
        """R virtual ranks on one GPU (tests; also a way to exercise the protocol without a multi-GPU box).
        shards: the R ranks' existing EmbeddingShards (e.g. `[w.shard for w in group]` of another group of this dim).
        tier_rows: host-tier rows behind each new shard (0: none); shared_tier: those tiers are shared memory.  grow=True
        (in **kw): each new shard's storage grows with its entries."""
        dev = torch.device("cuda", device)
        areas, bases = cls._local_areas(world, cls.area_bytes(world, cap, dim, kw.get("rows_f32", False)), dev)
        return [cls(n_slots, dim, prefixes, capacity, dev, r, world, cap, areas[r], bases, optimizer,
                    stream=torch.cuda.Stream(device=dev), shard=shards[r] if shards else None, tier_rows=tier_rows,
                    shared_tier=shared_tier, **kw)
                for r in range(world)]

    @staticmethod
    def _local_areas(world, nbytes, dev):
        """The zeroed receive areas of `world` virtual ranks on one GPU, in plain device memory, and their bases."""
        areas = [torch.zeros(nbytes + 256, dtype=torch.uint8, device=dev) for _ in range(world)]
        torch.cuda.synchronize(dev)
        return areas, [(a.data_ptr() + 255) // 256 * 256 for a in areas]

    @classmethod
    def distributed(cls, n_slots, dim, prefixes, capacity, cap, optimizer, device, group=None, tier_rows=0,
                    shared_tier=False, **kw):
        """One process per GPU: the receive areas live in torch symmetric memory (every peer's area mapped here).
        tier_rows: host-tier rows behind this rank's new shard (0: none); shared_tier: that tier is shared memory.  grow=True
        (in **kw): the new shard's storage grows with its entries."""
        import torch.distributed as dist

        grp = group if group is not None else dist.group.WORLD
        world, rank = dist.get_world_size(grp), dist.get_rank(grp)
        dev = device if isinstance(device, torch.device) else torch.device("cuda", device)
        area, bases = cls._symmetric_area(cls.area_bytes(world, cap, dim, kw.get("rows_f32", False)), dev, grp)
        w = cls(n_slots, dim, prefixes, capacity, dev, rank, world, cap, area, bases, optimizer, tier_rows=tier_rows,
                shared_tier=shared_tier, **kw)
        w.group = grp
        return w

    @staticmethod
    def _symmetric_area(nbytes, dev, grp):
        """A zeroed receive area of nbytes in symmetric memory and every rank's base (collective over grp); a plain
        device area when the group has one rank."""
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm

        if dist.get_world_size(grp) == 1:
            area = torch.zeros(nbytes + 256, dtype=torch.uint8, device=dev)
            return area, [(area.data_ptr() + 255) // 256 * 256]
        area = symm.empty(nbytes, dtype=torch.uint8, device=dev)
        area.zero_()
        hdl = symm.rendezvous(area, grp)
        bases = [int(p) for p in hdl.buffer_ptrs]
        assert all(b % 256 == 0 for b in bases)
        torch.cuda.synchronize(dev)
        dist.barrier(group=grp)
        return (area, hdl), bases

    @staticmethod
    def calibrate_cap(id_batches, batch, prefixes, world, margin=1.15, extra=64, group=None):
        """Slots per (source, owner) pair from sample batches (host ids, uint64 [n_slots * batch] each): the largest
        number of distinct signs any batch requests of one owner, plus a margin.  With a process group: the maximum
        over its ranks (collective).  A later batch that still overflows raises the status flag; the caller then
        re-runs it on a worker built with a larger cap."""
        worst = 0
        for ids in id_batches:
            slot_ids = np.ascontiguousarray(ids, dtype=np.uint64).reshape(len(prefixes), batch)
            worst = max(worst, int(distinct_per_owner(slot_ids, prefixes, world).max()))
        if group is not None or (torch.distributed.is_available() and torch.distributed.is_initialized()):
            import torch.distributed as dist

            t = torch.tensor([worst], dtype=torch.int64)
            if dist.get_backend(group) == "nccl":
                t = t.cuda()
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
            worst = int(t)
        return (int(worst * margin) + extra + 7) // 8 * 8

    # ---- incremental updates: the owner table's set of stepped signs (EmbeddingShard.enable_incremental) ---------------
    def _on_stream(self, fn, *args):
        with torch.cuda.stream(self._torch_stream()):
            return fn(*args)

    def enable_incremental(self, capacity):
        return self._on_stream(self.shard.enable_incremental, capacity)

    def incremental_stats(self):
        return self._on_stream(self.shard.incremental_stats)

    def incremental_held(self):
        return self.shard.incremental_held()

    def take_incremental(self):
        return self._on_stream(self.shard.take_incremental)

    # ---- forward_batched_direct / update_gradient_batched ------------------------------------------------------------
    def _torch_stream(self):
        """The stream this worker's calls run on: its own, else the current one."""
        return self.stream if self.stream is not None else torch.cuda.current_stream(self.device)

    def _st(self):
        return C.c_void_p(self._torch_stream().cuda_stream)

    def forward(self, ids, batch, training=True, row_off=None, slot_occ_off=None, out=None, phases=0):
        """ids: device int64-bit ids, slot-major; one id per sample per slot unless row_off (device int32 CSR offsets,
        [n_slots*batch+1]) and slot_occ_off (host list) are given.  Returns f16 [n_slots, batch, dim].
        phases: see PB_PHASE_* in persia_b200.h (0 = the whole call; virtual ranks are driven phase by phase)."""
        ids = SH._as_i64_bits(ids)
        if slot_occ_off is None:
            slot_occ_off = [s * batch for s in range(self.S + 1)]
        if out is None:
            out = torch.empty((self.S, batch, self.dim), dtype=torch.float16, device=self.device)
        self._after_stage()
        N.check(self.lib.pb_forward_sharded(self.shard.h, self.ctx.h, self.h, SH._ptr(ids), ids.numel(), SH._ptr(row_off),
                                            SH._slot_offsets(slot_occ_off, self.S), int(batch), int(training),
                                            SH._ptr(out), self._st(), int(phases)))
        self._forward_done(phases)
        return out

    def _after_stage(self):
        """A forward starts after the last stage of this rank's shard (TierStager); nothing without one."""
        self.shard._stage_mark.wait(self._torch_stream())

    def _forward_done(self, phases):
        """Once a forward's last phase is enqueued, the shard's next stage starts after it (TierStager)."""
        if phases == 0 or phases & N.PHASE_FINISH:
            self.shard._forward_marks.setdefault(id(self), SH.StreamMark()).record(self._torch_stream())

    def backward(self, grads, scales=None, want_status=False, phases=0, status=None):
        """grads: f16/f32 tensor [n_slots, batch, dim] or a list of per-slot tensors (None = skipped slot).  A slot
        tensor that is not 16-byte aligned (a slot of [n_slots, batch, dim] when batch * dim * 2 is not a multiple of
        16) is copied first, on the worker's stream."""
        if torch.is_tensor(grads):
            grads = [grads[i] for i in range(self.S)]
        ptrs, is_f16, held = SH._slot_grads(grads, self.S, self._torch_stream())  # (held through the call)
        if status is None and want_status:
            status = torch.empty(self.S, dtype=torch.int32, device=self.device)
        N.check(self.lib.pb_backward_sharded(self.shard.h, self.ctx.h, self.h, ptrs, int(is_f16), SH._scales(scales, self.S),
                                             SH._ptr(status), self._st(), int(phases)))
        return status

    def backward_ptrs(self, ptrs, is_f16, scales=None):
        """GradientBatch form (persia-core/src/backward.rs:86-105): raw device pointers, None = skipped slot.  A pointer
        that is not 16-byte aligned is refused (PersiaB200Error)."""
        N.check(self.lib.pb_backward_sharded(self.shard.h, self.ctx.h, self.h, SH._grad_ptrs(ptrs, self.S),
                                             int(bool(is_f16)), SH._scales(scales, self.S), None, self._st(), 0))

    @staticmethod
    def group_forward(workers, ids, batch, training=True, row_offs=None, slot_occ_offs=None, outs=None):
        """Virtual ranks of one GPU, driven by one host thread: every phase is enqueued for all ranks before the next."""
        outs = outs if outs is not None else [None] * len(workers)
        for r, w, ph in _by_phase(workers, N.PHASE_SEND, N.PHASE_SERVE, N.PHASE_FINISH):
            outs[r] = w.forward(ids[r], batch, training, row_offs[r] if row_offs else None,
                                slot_occ_offs[r] if slot_occ_offs else None, outs[r], phases=ph)
        return outs

    @staticmethod
    def group_backward(workers, grads, scales=None, want_status=False):
        sts = [torch.empty(w.S, dtype=torch.int32, device=w.device) if want_status else None for w in workers]
        for r, w, ph in _by_phase(workers, N.PHASE_SEND, N.PHASE_SERVE):
            w.backward(grads[r], scales, want_status, phases=ph, status=sts[r])
        return sts

    # ---- sizing each step from its own batch (PB_PHASE_PREPARE, pb_xchg_need) ---------------------------------------
    def _fit_ctx(self, n_occ, rows):
        """Grows the batch context when a batch of n_occ ids in `rows` output rows does not fit, as persia_core.ctx_size
        sizes it (local to this rank; the context holds one batch)."""
        if n_occ <= self.ctx_occ and rows <= self.ctx_rows:
            return
        from .persia_core import ctx_size

        size = ctx_size(n_occ, rows, (self.ctx_occ, self.ctx_rows))
        self._torch_stream().synchronize()
        self.ctx.close()
        self._new_ctx(*size)

    def _need(self):
        out = (C.c_uint32 * 1)()
        N.check(self.lib.pb_xchg_need(self.h, self.ctx.h, out, self._st()))
        return int(out[0])

    def prepare(self, ids, batch, row_off=None, slot_occ_off=None, training=True):
        """Local part of a forward, run before it: grows this rank's batch context if the batch needs it, then
        deduplicates the batch (PB_PHASE_PREPARE: no table state, no peer).  Returns (need, rows_f32): the most distinct
        items it sends one owner, and whether it needs f32 rows (ragged).  The forward of the same batch follows, after
        every rank has agreed on the exchange's size (resize)."""
        ids = SH._as_i64_bits(ids)
        self._fit_ctx(ids.numel(), self.S * batch)
        if slot_occ_off is None:
            slot_occ_off = [s * batch for s in range(self.S + 1)]
        if getattr(self, "_dummy_out", None) is None:  # (PREPARE writes no output; the call wants an aligned pointer)
            self._dummy_out = torch.empty(8, dtype=torch.float16, device=self.device)
        N.check(self.lib.pb_forward_sharded(self.shard.h, self.ctx.h, self.h, SH._ptr(ids), ids.numel(), SH._ptr(row_off),
                                            SH._slot_offsets(slot_occ_off, self.S), int(batch), int(training),
                                            SH._ptr(self._dummy_out), self._st(), N.PHASE_PREPARE))
        return self._need(), row_off is not None

    @staticmethod
    def grown_cap(need, cap):
        """The cap an exchange of `cap` slots grows to for an agreed need: never smaller, and with headroom over the
        need (1.5x + 1024, a multiple of 8) so that drift does not resize every step."""
        return cap if need <= cap else max(cap, (need * 3 // 2 + 1024 + 7) // 8 * 8)

    def _resize_to(self, need, rows_f32):
        """(cap, rows_f32) of the exchange this worker needs for the agreed (need, rows_f32), or None when its own
        suffices.  Every rank holds the same exchange geometry, so every rank reaches the same answer."""
        cap, f32 = self.grown_cap(int(need), self.cap), self.rows_f32 or bool(rows_f32)
        return None if (cap, f32) == (self.cap, self.rows_f32) else (cap, f32)

    def _replace_xchg(self, cap, rows_f32, area, bases):
        """The exchange replaced by one of (cap, rows_f32) over `area` (include/persia_b200.h, pb_xchg_destroy): the
        table, its Adam powers and its incremental set stay; a prepared batch stays in the context."""
        self._torch_stream().synchronize()
        old = self.h
        self._create_xchg(cap, rows_f32, bases)  # (sets self.h once created: a failure leaves the old one in place)
        self.lib.pb_xchg_destroy(old)
        self.cap, self.rows_f32, self.area = int(cap), bool(rows_f32), area

    def resize(self, need, rows_f32):
        """Collective over the worker's group: every rank passes the same agreed (need, rows_f32).  When this exchange
        does not cover them, every rank drains its stream and passes a barrier (no peer still writes the old areas),
        then a new symmetric area is rendezvoused and a new exchange created; the old area is released after that.
        Grows only.  Returns whether it resized."""
        to = self._resize_to(need, rows_f32)
        if to is None:
            return False
        import torch.distributed as dist

        grp = getattr(self, "group", None)
        if grp is None:
            assert self.R == 1, "a virtual rank resizes through group_resize"
            area, bases = self._local_areas(1, self.area_bytes(1, to[0], self.dim, to[1]), self.device)
            self._replace_xchg(*to, area[0], bases)
            return True
        self._torch_stream().synchronize()
        dist.barrier(group=grp)
        area, bases = self._symmetric_area(self.area_bytes(self.R, to[0], self.dim, to[1]), self.device, grp)
        self._replace_xchg(*to, area, bases)
        return True

    @staticmethod
    def group_prepare(workers, ids, batch, training=True, row_offs=None, slot_occ_offs=None):
        """Virtual ranks of one GPU: every rank's prepare, and their agreement (the max over the ranks, as the
        all-reduce of persia_core computes it over processes)."""
        needs = [w.prepare(ids[r], batch, row_offs[r] if row_offs else None, slot_occ_offs[r] if slot_occ_offs else None,
                           training) for r, w in enumerate(workers)]
        return max(n for n, _ in needs), any(f for _, f in needs)

    @staticmethod
    def group_resize(workers, need, rows_f32):
        """Virtual ranks of one GPU: resize (same rule) with plain device areas for all ranks.  Returns whether it did."""
        to = workers[0]._resize_to(need, rows_f32)
        if to is None:
            return False
        w0 = workers[0]
        areas, bases = w0._local_areas(len(workers), w0.area_bytes(len(workers), to[0], w0.dim, to[1]), w0.device)
        for r, w in enumerate(workers):
            w._replace_xchg(*to, areas[r], bases)
        return True

    def status(self):
        """(overflowed, wait_gave_up) — host sync."""
        out = SH._read_block(XCHG_STATUS_FIELDS, lambda out: self.lib.pb_xchg_status(self.h, out, self._st()), C.c_uint32)
        return bool(out["overflowed"]), bool(out["wait_gave_up"])

    def close(self):
        if getattr(self, "h", None):
            self.lib.pb_xchg_destroy(self.h)
            self.h = None
        if getattr(self, "shard", None) is not None:
            self.shard._forward_marks.pop(id(self), None)
        self.ctx.close()
        if self._own_shard:
            self.shard.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ShardedRawWorker(ShardedEmbeddingWorker):
    """One raw (embedding_summation: false) slot over the R GPUs of one box: pb_forward_raw_sharded /
    pb_backward_raw_sharded.  Built like ShardedEmbeddingWorker with n_slots == 1 (its one prefix is the slot's
    index_prefix); its exchange always carries f32 rows, which the requester rounds to the f16 table.  Pass `shard=` /
    `shards=` to serve the table of the rank's summation worker of the same dim.  Every call is collective, including
    batches without ids; each raw slot of a model has its own worker (its own exchange)."""

    def __init__(self, n_slots, dim, prefixes, capacity, device, rank, world, cap, area, peer_bases, optimizer, **kw):
        assert n_slots == 1 and len(prefixes) == 1, "a raw worker serves one slot"
        kw["rows_f32"] = True
        kw.pop("sqrt_scaling", None)  # (a raw slot's sqrt_scaling only matters with hash-stack, which it cannot have)
        super().__init__(1, dim, prefixes, capacity, device, rank, world, cap, area, peer_bases, optimizer, **kw)

    @staticmethod
    def area_bytes(world, cap, dim, rows_f32=True):
        return ShardedEmbeddingWorker.area_bytes(world, cap, dim, True)

    def forward_raw(self, ids, batch, sample_fixed_size, row_off=None, training=True, out=None, phases=0):
        """What BatchContext.forward_raw returns: (table f16 [n_occ+1, dim] of which rows [0, U] are valid, index i64
        [batch*fixed], non_empty i64 of which counts[1] entries are valid, sample_id_num i32 [batch], counts i32 [2] =
        (U, non-empty entries)), on the device.  out: those five buffers from an earlier call (phase-split and
        captured calls reuse them)."""
        ids = SH._as_i64_bits(ids)
        n, fixed = ids.numel(), int(sample_fixed_size)
        if out is None:  # (after prepare_raw: the buffers it numbered the batch into)
            out = getattr(self, "_prepared_out", None) or SH._raw_outputs(n, batch, fixed, self.dim, self.device)
        if phases == 0 or phases & N.PHASE_FINISH:
            self._prepared_out = None
        table, index, non_empty, num, counts = out
        self._after_stage()
        N.check(self.lib.pb_forward_raw_sharded(self.shard.h, self.ctx.h, self.h, SH._ptr(ids), n,
                                                SH._raw_row_off(row_off, batch), int(batch), fixed, int(training),
                                                *map(SH._ptr, out), self._st(), int(phases)))
        self._forward_done(phases)
        return table, index, non_empty, num[:batch], counts

    def backward_raw(self, grad, scale=1.0, want_status=False, is_f16=None, phases=0, status=None):
        """grad: device tensor [U, dim] (f32 as persia/ctx.py:970-980 builds it, or f16), a raw device pointer (then
        pass is_f16), or None (add_skipped_gradient).  A tensor that is not 16-byte aligned is copied first."""
        ptr, is_f16, held = SH._raw_grad(grad, is_f16, self, self._torch_stream())  # (held through the call)
        if status is None and want_status:
            status = torch.empty(1, dtype=torch.int32, device=self.device)
        N.check(self.lib.pb_backward_raw_sharded(self.shard.h, self.ctx.h, self.h, ptr, int(bool(is_f16)), float(scale),
                                                 SH._ptr(status), self._st(), int(phases)))
        return status

    def prepare_raw(self, ids, batch, sample_fixed_size, row_off=None, training=True):
        """prepare() of a raw slot: grows the context if needed, numbers the slot's distinct signs (PB_PHASE_PREPARE) into
        the output buffers the next forward_raw of this batch takes over.  Returns (need, True): raw exchanges carry f32
        rows always."""
        ids = SH._as_i64_bits(ids)
        n, fixed = ids.numel(), int(sample_fixed_size)
        self._fit_ctx(n, batch)
        out = SH._raw_outputs(n, batch, fixed, self.dim, self.device)
        N.check(self.lib.pb_forward_raw_sharded(self.shard.h, self.ctx.h, self.h, SH._ptr(ids), n,
                                                SH._raw_row_off(row_off, batch), int(batch), fixed, int(training),
                                                *map(SH._ptr, out), self._st(), N.PHASE_PREPARE))
        self._prepared_out = out
        return self._need(), True

    @staticmethod
    def group_prepare_raw(workers, ids, batch, sample_fixed_size, training=True, row_offs=None):
        """Virtual ranks of one GPU: every rank's prepare_raw, and their agreement (max over the ranks)."""
        needs = [w.prepare_raw(ids[r], batch, sample_fixed_size, row_offs[r] if row_offs else None, training)
                 for r, w in enumerate(workers)]
        return max(n for n, _ in needs), True

    @staticmethod
    def group_forward_raw(workers, ids, batch, sample_fixed_size, training=True, row_offs=None, outs=None):
        """Virtual ranks of one GPU, driven by one host thread: every phase is enqueued for all ranks before the next.
        Returns one forward_raw result per rank."""
        outs = list(outs) if outs is not None else [None] * len(workers)
        for r, w, ph in _by_phase(workers, N.PHASE_SEND, N.PHASE_SERVE, N.PHASE_FINISH):
            outs[r] = w.forward_raw(ids[r], batch, sample_fixed_size, row_offs[r] if row_offs else None, training,
                                    out=outs[r], phases=ph)
        return outs

    @staticmethod
    def group_backward_raw(workers, grads, scales=None, want_status=False):
        """grads: per rank a [U_r, dim] tensor or None (add_skipped_gradient); scales: per rank (default 1)."""
        sts = [torch.empty(1, dtype=torch.int32, device=w.device) if want_status else None for w in workers]
        for r, w, ph in _by_phase(workers, N.PHASE_SEND, N.PHASE_SERVE):
            w.backward_raw(grads[r], scales[r] if scales is not None else 1.0, phases=ph, status=sts[r])
        return sts


class TierStager:
    """The next batch's host-tier moves on R GPUs, one step early (pb_tier_stage_sharded): every rank sends the signs of
    its next training batch to their owners, and each owner runs the eviction check that batch would run and moves the
    tier-held signs it received back into HBM, on a stream of its own, beside the current batch's backward and dense
    step.  One stager per rank and table, shared by the summation and raw workers of that dim (they serve its shard).
    Values never change: a staged run equals the unstaged one bit for bit.

    Ordering is kept on the EmbeddingShard, so callers handle no events: stage() waits for the last forward of every
    worker of the shard, and their next forward / forward_raw waits for the stage.  Each call is collective, like the
    workers' (one process per GPU: `distributed`; virtual ranks of one GPU: `local_group` and `group_stage`).

    cap: the most signs one rank stages one owner in one call; the stage area holds R x cap signs.  Pass the most ids one
    stage() call brings and no sign is ever over cap.  Signs over it are not staged (status()[0]): the forward restores
    them as it would unstaged."""

    def __init__(self, shard, rank, world, cap, area, peer_bases, stream=None):
        self.lib = N.load()
        self.shard, self.rank, self.R, self.cap = shard, int(rank), int(world), int(cap)
        self.device = shard.device
        self.area = area  # keeps the stage area alive
        self.stream = stream if stream is not None else torch.cuda.Stream(device=self.device)
        bases = (C.c_uint64 * self.R)(*[int(p) for p in peer_bases])
        h = C.c_void_p()
        N.check(self.lib.pb_xchg_create_stage(self.device.index or 0, self.R, self.rank, self.cap, bases, C.byref(h)))
        self.h = h

    @staticmethod
    def area_bytes(world, cap):
        b = int(N.load().pb_xchg_stage_bytes(world, int(cap)))
        assert b > 0, "bad stage geometry"
        return b

    @classmethod
    def local_group(cls, shards, cap, streams=None):
        """One stager per virtual rank of one GPU, over the ranks' shards (e.g. `[w.shard for w in workers]`)."""
        dev = shards[0].device
        areas, bases = ShardedEmbeddingWorker._local_areas(len(shards), cls.area_bytes(len(shards), cap), dev)
        return [cls(s, r, len(shards), cap, areas[r], bases, stream=streams[r] if streams else None)
                for r, s in enumerate(shards)]

    @classmethod
    def distributed(cls, shard, cap, group=None, stream=None):
        """One process per GPU: the stage area lives in symmetric memory, like the workers' receive areas (collective)."""
        import torch.distributed as dist

        grp = group if group is not None else dist.group.WORLD
        world, rank = dist.get_world_size(grp), dist.get_rank(grp)
        area, bases = ShardedEmbeddingWorker._symmetric_area(cls.area_bytes(world, cap), shard.device, grp)
        st = cls(shard, rank, world, cap, area, bases, stream=stream)
        st.group = grp
        return st

    def stage(self, ids, slot_occ_off, prefixes, prefix_bit=8, phases=0):
        """Stages the next training batch of this rank: ids flat device slot ids (slot-major, hash-stacked where a slot
        hash-stacks; the summation and raw slots of the table may come in one call), slot_occ_off host list of
        n_slots + 1 offsets, prefixes each slot's index prefix (0 = ids taken as they are).  Runs on the stager's
        stream.  phases: PHASE_SEND, PHASE_SERVE or 0 = both (virtual ranks: group_stage)."""
        ids = SH._as_i64_bits(ids)
        S = len(prefixes)
        st = self.stream
        if phases == 0 or phases & N.PHASE_SEND:
            for m in self.shard._forward_marks.values():
                m.wait(st)
        N.check(self.lib.pb_tier_stage_sharded(self.shard.h, self.h, SH._ptr(ids), ids.numel(),
                                               SH._slot_offsets(slot_occ_off, S), SH._prefixes(prefixes), S,
                                               int(prefix_bit), C.c_void_p(st.cuda_stream), int(phases)))
        if phases == 0 or phases & N.PHASE_SERVE:
            self.shard._stage_mark.record(st)

    @staticmethod
    def group_stage(stagers, ids, slot_occ_offs, prefixes, prefix_bit=8):
        """Virtual ranks of one GPU, driven by one host thread: SEND for every rank, then SERVE for every rank."""
        for r, s, ph in _by_phase(stagers, N.PHASE_SEND, N.PHASE_SERVE):
            s.stage(ids[r], slot_occ_offs[r], prefixes, prefix_bit, phases=ph)

    def stage_stats(self):
        """This rank's owner counters (host sync): signs staged into HBM, and stage restores skipped for want of a free
        row."""
        return self.shard.stage_stats()

    def status(self):
        """(overflowed, wait_gave_up) — host sync.  overflowed: a stage had more than cap signs for one owner."""
        out = SH._read_block(XCHG_STATUS_FIELDS, lambda out: self.lib.pb_xchg_status(self.h, out,
                                                                                     C.c_void_p(self.stream.cuda_stream)),
                             C.c_uint32)
        return bool(out["overflowed"]), bool(out["wait_gave_up"])

    def close(self):
        if getattr(self, "h", None):
            self.lib.pb_xchg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def exchange_readers(shard, views, group=None):
    """R GPUs with exportable growable owners (grow="shared"): every rank's view addresses (TableView.address, one per
    owner) are exchanged with one all_gather_object, and this rank's shard registers the views of it its peers opened
    (EmbeddingShard.add_readers), so that they receive its chunks as it grows.  Collective; after every view is open.
    Skipped on every rank when no rank's shard grows shared (the same on all ranks)."""
    import torch.distributed as dist

    if not shard.grow_shared:
        return
    grp = group if group is not None else dist.group.WORLD
    rank = dist.get_rank(grp)
    addrs = [None] * dist.get_world_size(grp)
    dist.all_gather_object(addrs, [v.address if v is not None else "" for v in views], group=grp)
    shard.add_readers([a[rank] for a in addrs])


class RemoteReader:
    """Inference on R GPUs one rank at a time (pb_forward_remote / pb_forward_raw_remote): this rank's requests are
    served alone, whatever its peers do.  The requesting GPU probes each owner's index and reads its rows in place,
    through views of the owners' exported tables (EmbeddingShard.export_view, TableView); no flag, no collective, no
    kernel on the owner.  Outputs are bit for bit the collective path's inference forwards (ShardedEmbeddingWorker /
    ShardedRawWorker with training=False).

    export_view makes every table read-only but for set_entries and checkpoint / incremental-packet inserts, which the
    reads see whole or not at all (include/persia_b200.h): an Infer job's export.  A training job's tables are exported
    live instead (EmbeddingShard.export_live_view, built into readers with this class's constructor): they keep training
    collectively, and a read never returns another sign's row.  The views close before the tables (close() first), and
    every owner outlives its peers' views.

    One batch context per slot chunk (the slots one call serves, keyed by their prefixes), grown when a larger batch
    comes.  Two ways to build the readers of a box, like ShardedEmbeddingWorker's:
      * `RemoteReader.distributed(shard, group)`: one process per GPU; the blobs are exchanged with one all_gather_object.
      * `RemoteReader.local_group(shards)`: R virtual ranks on one GPU in one process (views from blobs of this pid)."""

    def __init__(self, shard, views, rank, stream=None):
        """shard: this rank's EmbeddingShard (exported); views: one TableView per rank (None at `rank`: its own table is
        probed directly)."""
        self.lib = N.load()
        self.shard, self.views, self.rank, self.R = shard, list(views), int(rank), len(views)
        self.device, self.dim, self.stream = shard.device, shard.dim, stream
        self._views = (C.c_void_p * self.R)(*[(v.h.value if v is not None else None) for v in self.views])
        self._ctxs = {}  # (kind, prefixes, sqrt_scaling, prefix_bit) -> [BatchContext, max occurrences, max rows]

    @classmethod
    def local_group(cls, shards, streams=None):
        """R virtual ranks on one GPU: every shard is exported and viewed by the others (same process).  streams: one per
        rank (default: a new stream each)."""
        blobs = [s.export_view() for s in shards]
        return [cls(s, [SH.TableView(b, s.device) if q != r else None for q, b in enumerate(blobs)], r,
                    stream=streams[r] if streams else torch.cuda.Stream(device=s.device))
                for r, s in enumerate(shards)]

    @classmethod
    def distributed(cls, shard, group=None, stream=None):
        """One process per GPU: exports this rank's shard and exchanges the blobs with one all_gather_object over the
        group (collective); the peers' tables are then opened through CUDA IPC."""
        import torch.distributed as dist

        grp = group if group is not None else dist.group.WORLD
        world, rank = dist.get_world_size(grp), dist.get_rank(grp)
        blobs = [None] * world
        dist.all_gather_object(blobs, shard.export_view(), group=grp)
        views = [SH.TableView(b, shard.device) if q != rank else None for q, b in enumerate(blobs)]
        exchange_readers(shard, views, grp)
        dist.barrier(group=grp)  # (no rank reads before every view is open)
        return cls(shard, views, rank, stream=stream)

    def _torch_stream(self):
        return self.stream if self.stream is not None else torch.cuda.current_stream(self.device)

    def _st(self):
        return C.c_void_p(self._torch_stream().cuda_stream)

    def _ctx(self, key, n_occ, rows):
        """The batch context of `key`, grown (persia_core.ctx_size) when n_occ ids in `rows` rows do not fit."""
        from .persia_core import ctx_size

        got = self._ctxs.get(key)
        if got is not None and n_occ <= got[1] and rows <= got[2]:
            return got[0]
        occ, out_rows = ctx_size(n_occ, rows, got[1:] if got else (0, 0))
        if got is not None:
            self._torch_stream().synchronize()
            got[0].close()
        _, prefixes, sqrt, prefix_bit = key
        ctx = SH.BatchContext(occ, out_rows, list(prefixes), list(sqrt) if sqrt else None, prefix_bit, self.device)
        self._ctxs[key] = [ctx, occ, out_rows]
        return ctx

    def forward(self, ids, batch, prefixes, sqrt_scaling=None, prefix_bit=8, row_off=None, slot_occ_off=None, out=None):
        """ShardedEmbeddingWorker.forward(training=False) of this rank alone: ids slot-major (device int64 bits), one id
        per sample per slot unless row_off (device int32 CSR offsets) and slot_occ_off (host list) are given; the slots'
        index prefixes and sqrt scaling.  Returns f16 [n_slots, batch, dim]."""
        ids = SH._as_i64_bits(ids)
        S = len(prefixes)
        if slot_occ_off is None:
            slot_occ_off = [s * batch for s in range(S + 1)]
        key = ("sum", tuple(int(p) for p in prefixes), tuple(bool(x) for x in sqrt_scaling) if sqrt_scaling else None,
               int(prefix_bit))
        ctx = self._ctx(key, ids.numel(), S * batch)
        if out is None:
            out = torch.empty((S, batch, self.dim), dtype=torch.float16, device=self.device)
        if row_off is not None:
            assert row_off.dtype == torch.int32 and row_off.is_contiguous()
        N.check(self.lib.pb_forward_remote(self.shard.h, self._views, self.R, self.rank, ctx.h, SH._ptr(ids), ids.numel(),
                                           SH._ptr(row_off), SH._slot_offsets(slot_occ_off, S), int(batch), SH._ptr(out),
                                           self._st()))
        return out

    def forward_raw(self, ids, batch, sample_fixed_size, prefix, prefix_bit=8, row_off=None, out=None):
        """ShardedRawWorker.forward_raw(training=False) of this rank alone, for the raw slot of index prefix `prefix`:
        (table f16 [n_occ+1, dim] of which rows [0, U] are valid, index i64 [batch*fixed], non_empty i64 of which
        counts[1] entries are valid, sample_id_num i32 [batch], counts i32 [2] = (U, non-empty entries)), on the device.
        out: those five buffers from an earlier call of the same sizes (captured calls reuse them)."""
        ids = SH._as_i64_bits(ids)
        n, fixed = ids.numel(), int(sample_fixed_size)
        ctx = self._ctx(("raw", (int(prefix),), None, int(prefix_bit)), n, batch)
        if out is None:
            out = SH._raw_outputs(n, batch, fixed, self.dim, self.device)
        N.check(self.lib.pb_forward_raw_remote(self.shard.h, self._views, self.R, self.rank, ctx.h, SH._ptr(ids), n,
                                               SH._raw_row_off(row_off, batch), int(batch), fixed, *map(SH._ptr, out),
                                               self._st()))
        table, index, non_empty, num, counts = out
        return table, index, non_empty, num[:batch], counts

    def close(self):
        """Closes the contexts and the views (before the tables they view: their owners close those)."""
        for ctx, _, _ in self._ctxs.values():
            ctx.close()
        self._ctxs = {}
        for v in self.views:
            if v is not None:
                v.close()
        self.views = [None] * self.R

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
