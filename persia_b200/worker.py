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


def distinct_per_owner(ids, batch, prefixes, R, prefix_bit=8):
    """Host-side (numpy) count of the distinct signs one batch requests of every owner: what `cap` must cover.
    ids: uint64 [n_slots * batch] slot-major.  Mirrors indices_add_prefix + FeatureBatch::new + sign_to_shard_modulo."""
    from .persia_core import farmhash64_np

    S = len(prefixes)
    ids = np.ascontiguousarray(ids, dtype=np.uint64).reshape(S, batch)
    spacing = np.uint64((1 << (64 - prefix_bit)) - 1)
    counts = np.zeros(R, np.int64)
    for s in range(S):
        signs = ids[s] % spacing + np.uint64(prefixes[s]) if prefixes[s] else ids[s]
        u = np.unique(signs)
        counts += np.bincount((farmhash64_np(u) % np.uint64(R)).astype(np.int64), minlength=R)
    return counts


class ShardedEmbeddingWorker:
    def __init__(self, n_slots, dim, prefixes, capacity, device, rank, world, cap, area, peer_bases, optimizer,
                 hyper=None, max_batch=4096, sqrt_scaling=None, rows_f32=False, prefix_bit=8, stream=None,
                 max_ids_per_sample=1, shard=None):
        """shard: an existing EmbeddingShard of this rank to serve (configured by its owner, who also closes it), so
        that the workers of one dim — summation slots and raw slots — share one table; None: a new one."""
        self.S, self.dim, self.rank, self.R, self.cap = n_slots, dim, rank, world, int(cap)
        self.device = device if isinstance(device, torch.device) else torch.device("cuda", device)
        self.lib = N.load()
        self.stream = stream
        self.area = area  # keeps the receive area alive
        self._own_shard = shard is None
        if shard is None:
            shard = SH.EmbeddingShard(dim, capacity, self.device)
            shard.set_optimizer(**optimizer)
            shard.configure(**(hyper or {}))
        assert shard.dim == dim, "the shard holds another embedding dim"
        self.shard = shard
        n = n_slots * max_batch * max_ids_per_sample
        self.ctx = SH.BatchContext(n, n_slots * max_batch, prefixes, sqrt_scaling, prefix_bit, self.device)
        bases = (C.c_uint64 * world)(*[int(p) for p in peer_bases])
        h = C.c_void_p()
        N.check(self.lib.pb_xchg_create(self.device.index or 0, world, rank, self.cap, dim, int(rows_f32), bases, C.byref(h)))
        self.h = h

    # ---- set-up helpers --------------------------------------------------------------------------------------------
    @staticmethod
    def area_bytes(world, cap, dim, rows_f32=False):
        b = int(N.load().pb_xchg_bytes(world, int(cap), dim, int(rows_f32)))
        assert b > 0, "bad exchange geometry"
        return b

    @classmethod
    def local_group(cls, world, n_slots, dim, prefixes, capacity, cap, optimizer, device=0, shards=None, **kw):
        """R virtual ranks on one GPU (tests; also a way to exercise the protocol without a multi-GPU box).
        shards: the R ranks' existing EmbeddingShards (e.g. `[w.shard for w in group]` of another group of this dim)."""
        dev = torch.device("cuda", device)
        nbytes = cls.area_bytes(world, cap, dim, kw.get("rows_f32", False))
        areas = [torch.zeros(nbytes + 256, dtype=torch.uint8, device=dev) for _ in range(world)]
        bases = [(a.data_ptr() + 255) // 256 * 256 for a in areas]
        torch.cuda.synchronize(dev)
        return [cls(n_slots, dim, prefixes, capacity, dev, r, world, cap, areas[r], bases, optimizer,
                    stream=torch.cuda.Stream(device=dev), shard=shards[r] if shards else None, **kw)
                for r in range(world)]

    @classmethod
    def distributed(cls, n_slots, dim, prefixes, capacity, cap, optimizer, device, group=None, **kw):
        """One process per GPU: the receive areas live in torch symmetric memory (every peer's area mapped here)."""
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm

        grp = group if group is not None else dist.group.WORLD
        world, rank = dist.get_world_size(grp), dist.get_rank(grp)
        dev = device if isinstance(device, torch.device) else torch.device("cuda", device)
        nbytes = cls.area_bytes(world, cap, dim, kw.get("rows_f32", False))
        if world == 1:
            area = torch.zeros(nbytes + 256, dtype=torch.uint8, device=dev)
            bases = [(area.data_ptr() + 255) // 256 * 256]
            return cls(n_slots, dim, prefixes, capacity, dev, 0, 1, cap, area, bases, optimizer, **kw)
        area = symm.empty(nbytes, dtype=torch.uint8, device=dev)
        area.zero_()
        hdl = symm.rendezvous(area, grp)
        bases = [int(p) for p in hdl.buffer_ptrs]
        assert all(b % 256 == 0 for b in bases)
        torch.cuda.synchronize(dev)
        dist.barrier(group=grp)
        w = cls(n_slots, dim, prefixes, capacity, dev, rank, world, cap, (area, hdl), bases, optimizer, **kw)
        w.group = grp
        return w

    @staticmethod
    def calibrate_cap(id_batches, batch, prefixes, world, margin=1.15, extra=64, group=None):
        """Slots per (source, owner) pair from sample batches (host ids, uint64 [n_slots * batch] each): the largest
        number of distinct signs any batch requests of one owner, plus a margin.  With a process group: the maximum
        over its ranks (collective).  A later batch that still overflows raises the status flag; the caller then
        re-runs it on a worker built with a larger cap."""
        worst = 0
        for ids in id_batches:
            worst = max(worst, int(distinct_per_owner(ids, batch, prefixes, world).max()))
        if group is not None or (torch.distributed.is_available() and torch.distributed.is_initialized()):
            import torch.distributed as dist

            t = torch.tensor([worst], dtype=torch.int64)
            if dist.get_backend(group) == "nccl":
                t = t.cuda()
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
            worst = int(t)
        return (int(worst * margin) + extra + 7) // 8 * 8

    # ---- forward_batched_direct / update_gradient_batched ------------------------------------------------------------
    def _st(self):
        s = self.stream if self.stream is not None else torch.cuda.current_stream(self.device)
        return C.c_void_p(s.cuda_stream)

    def forward(self, ids, batch, training=True, row_off=None, slot_occ_off=None, out=None, phases=0):
        """ids: device int64-bit ids, slot-major; one id per sample per slot unless row_off (device int32 CSR offsets,
        [n_slots*batch+1]) and slot_occ_off (host list) are given.  Returns f16 [n_slots, batch, dim].
        phases: see PB_PHASE_* in persia_b200.h (0 = the whole call; virtual ranks are driven phase by phase)."""
        ids = SH._as_i64_bits(ids)
        if slot_occ_off is None:
            slot_occ_off = [s * batch for s in range(self.S + 1)]
        if out is None:
            out = torch.empty((self.S, batch, self.dim), dtype=torch.float16, device=self.device)
        off = (C.c_uint32 * (self.S + 1))(*[int(v) for v in slot_occ_off])
        N.check(self.lib.pb_forward_sharded(self.shard.h, self.ctx.h, self.h, SH._ptr(ids), ids.numel(), SH._ptr(row_off), off,
                                            int(batch), int(training), SH._ptr(out), self._st(), int(phases)))
        return out

    def backward(self, grads, scales=None, want_status=False, phases=0, status=None):
        """grads: f16/f32 tensor [n_slots, batch, dim] or a list of per-slot tensors (None = skipped slot).  A slot
        tensor that is not 16-byte aligned (a slot of [n_slots, batch, dim] when batch * dim * 2 is not a multiple of
        16) is copied first, on the worker's stream."""
        if torch.is_tensor(grads):
            grads = [grads[i] for i in range(self.S)]
        st = self.stream if self.stream is not None else torch.cuda.current_stream(self.device)
        grads = [SH.aligned(g, st) for g in grads]  # (kept alive until the call has enqueued its reads)
        ptrs = (C.c_void_p * self.S)()
        is_f16 = None
        for i, g in enumerate(grads):
            if g is None:
                ptrs[i] = None
                continue
            assert g.is_contiguous() and g.dtype in (torch.float16, torch.float32)
            f16 = g.dtype == torch.float16
            assert is_f16 is None or is_f16 == f16, "all slot gradients of one request share a dtype"
            is_f16 = f16
            ptrs[i] = g.data_ptr()
        sc = (C.c_float * self.S)(*[float(v) for v in scales]) if scales is not None else None
        if status is None and want_status:
            status = torch.empty(self.S, dtype=torch.int32, device=self.device)
        N.check(self.lib.pb_backward_sharded(self.shard.h, self.ctx.h, self.h, ptrs, int(bool(is_f16)), sc, SH._ptr(status),
                                             self._st(), int(phases)))
        return status

    def backward_ptrs(self, ptrs, is_f16, scales=None):
        """GradientBatch form (persia-core/src/backward.rs:86-105): raw device pointers, None = skipped slot.  A pointer
        that is not 16-byte aligned is refused (PersiaB200Error)."""
        arr = (C.c_void_p * self.S)(*[(int(p) if p else None) for p in ptrs])
        sc = (C.c_float * self.S)(*[float(v) for v in scales]) if scales is not None else None
        N.check(self.lib.pb_backward_sharded(self.shard.h, self.ctx.h, self.h, arr, int(bool(is_f16)), sc, None, self._st(), 0))

    @staticmethod
    def group_forward(workers, ids, batch, training=True, row_offs=None, slot_occ_offs=None, outs=None):
        """Virtual ranks of one GPU, driven by one host thread: every phase is enqueued for all ranks before the next."""
        R = len(workers)
        outs = outs if outs is not None else [None] * R
        for ph in (N.PHASE_SEND, N.PHASE_SERVE, N.PHASE_FINISH):
            for r, w in enumerate(workers):
                outs[r] = w.forward(ids[r], batch, training, row_offs[r] if row_offs else None,
                                    slot_occ_offs[r] if slot_occ_offs else None, outs[r], phases=ph)
        return outs

    @staticmethod
    def group_backward(workers, grads, scales=None, want_status=False):
        R = len(workers)
        sts = [torch.empty(w.S, dtype=torch.int32, device=w.device) if want_status else None for w in workers]
        for ph in (N.PHASE_SEND, N.PHASE_SERVE):
            for r, w in enumerate(workers):
                w.backward(grads[r], scales, want_status, phases=ph, status=sts[r])
        return sts

    def status(self):
        """(overflowed, wait_gave_up) — host sync."""
        out = (C.c_uint32 * 2)()
        N.check(self.lib.pb_xchg_status(self.h, C.byref(out), self._st()))
        return bool(out[0]), bool(out[1])

    def close(self):
        if getattr(self, "h", None):
            self.lib.pb_xchg_destroy(self.h)
            self.h = None
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
        self._dummy = None

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
        if out is None:
            out = (torch.empty((n + 1, self.dim), dtype=torch.float16, device=self.device),
                   torch.empty(batch * fixed, dtype=torch.int64, device=self.device),
                   torch.empty(max(batch * fixed, 1), dtype=torch.int64, device=self.device),
                   torch.empty(max(batch, 1), dtype=torch.int32, device=self.device),
                   torch.empty(2, dtype=torch.int32, device=self.device))
        table, index, non_empty, num, counts = out
        if row_off is not None:
            assert row_off.dtype == torch.int32 and row_off.is_contiguous() and row_off.numel() == batch + 1
        N.check(self.lib.pb_forward_raw_sharded(self.shard.h, self.ctx.h, self.h, SH._ptr(ids), n, SH._ptr(row_off),
                                                int(batch), fixed, int(training), SH._ptr(table), SH._ptr(index),
                                                SH._ptr(non_empty), SH._ptr(num), SH._ptr(counts), self._st(),
                                                int(phases)))
        return table, index, non_empty, num[:batch], counts

    def backward_raw(self, grad, scale=1.0, want_status=False, is_f16=None, phases=0, status=None):
        """grad: device tensor [U, dim] (f32 as persia/ctx.py:970-980 builds it, or f16), a raw device pointer (then
        pass is_f16), or None (add_skipped_gradient).  A tensor that is not 16-byte aligned is copied first."""
        ptr = None
        if grad is not None and not isinstance(grad, int):
            st = self.stream if self.stream is not None else torch.cuda.current_stream(self.device)
            grad = SH.aligned(grad, st)
            assert grad.is_contiguous() and grad.dtype in (torch.float16, torch.float32)
            is_f16 = grad.dtype == torch.float16
            if grad.numel():
                ptr = grad.data_ptr()
            else:  # U = 0: nothing is read, but the request is not a skipped one
                if self._dummy is None:
                    self._dummy = torch.zeros(4, dtype=torch.float32, device=self.device)
                ptr = self._dummy.data_ptr()
        elif grad is not None:
            ptr = grad
        if status is None and want_status:
            status = torch.empty(1, dtype=torch.int32, device=self.device)
        N.check(self.lib.pb_backward_raw_sharded(self.shard.h, self.ctx.h, self.h, ptr, int(bool(is_f16)), float(scale),
                                                 SH._ptr(status), self._st(), int(phases)))
        return status

    @staticmethod
    def group_forward_raw(workers, ids, batch, sample_fixed_size, training=True, row_offs=None, outs=None):
        """Virtual ranks of one GPU, driven by one host thread: every phase is enqueued for all ranks before the next.
        Returns one forward_raw result per rank."""
        R = len(workers)
        outs = list(outs) if outs is not None else [None] * R
        for ph in (N.PHASE_SEND, N.PHASE_SERVE, N.PHASE_FINISH):
            for r, w in enumerate(workers):
                outs[r] = w.forward_raw(ids[r], batch, sample_fixed_size, row_offs[r] if row_offs else None, training,
                                        out=outs[r], phases=ph)
        return outs

    @staticmethod
    def group_backward_raw(workers, grads, scales=None, want_status=False):
        """grads: per rank a [U_r, dim] tensor or None (add_skipped_gradient); scales: per rank (default 1)."""
        sts = [torch.empty(1, dtype=torch.int32, device=w.device) if want_status else None for w in workers]
        for ph in (N.PHASE_SEND, N.PHASE_SERVE):
            for r, w in enumerate(workers):
                w.backward_raw(grads[r], scales[r] if scales is not None else 1.0, phases=ph, status=sts[r])
        return sts
