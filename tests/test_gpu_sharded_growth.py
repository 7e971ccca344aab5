"""GPU: exportable growable tables (pb_table_set_growth(t, 2), EmbeddingShard(grow="shared")) read in place while they
grow.

Virtual ranks on cuda:0 train owners through row growths and index doublings while each rank's reader serves forwards
that do not train, and every read equals the same read of an eager twin bit for bit; frozen exports grow through
set_entries under their readers.  Two processes on one device: the reader maps the owner's chunks as they arrive over
its socket, including every chunk mapped before it registered, and a read that meets a chunk the owner has kept back
waits for it and reads again, exactly (the owner sends only once the reader's process has counted the stale retry)."""
import ctypes as C
import os
import sys
import tempfile
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from util import same_bits, to_dev_i32, to_dev_ids  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
OPT = dict(kind=1, lr=0.02, initialization=0.01)  # Adagrad


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _fd_handles():
    """Whether this device can export growable tables (POSIX file descriptor handles)."""
    import persia_b200.shard as SH
    from persia_b200 import native as N

    s = SH.EmbeddingShard(8, 1024, 0)
    try:
        return N.load().pb_table_set_growth(s.h, 2) == 0
    finally:
        s.close()


def _live_readers(torch, shards):
    from persia_b200.shard import TableView
    from persia_b200.worker import RemoteReader

    blobs = [s.export_live_view() for s in shards]
    return [RemoteReader(s, [TableView(b, s.device) if q != r else None for q, b in enumerate(blobs)], r,
                         stream=torch.cuda.Stream(device=s.device)) for r, s in enumerate(shards)]


class _Growth:
    """storage_stats of a shard over a run: row growths and index doublings; refusals of unbacked rows stay 0."""

    def __init__(self, s):
        st = s.storage_stats()
        self.s, self.rows, self.cells, self.row_growths, self.doublings = s, st["mapped_rows"], st["index_cells"], 0, 0

    def note(self):
        st = self.s.storage_stats()
        assert st["refused_unmapped"] == 0
        self.row_growths += st["mapped_rows"] > self.rows
        self.doublings += st["index_cells"] > self.cells
        self.rows, self.cells = st["mapped_rows"], st["index_cells"]


def _reads(rd, q, pf, raw_pf):
    """One rank's pooled and raw remote forwards of a query (host arrays: slot-major ids, raw ids and their CSR
    offsets)."""
    ids, raw_ids, raw_off = q
    out = rd.forward(to_dev_ids(ids, DEV), ids.size // len(pf), pf)
    table, index, non_empty, num, counts = rd.forward_raw(to_dev_ids(raw_ids, DEV), raw_off.size - 1, 4, raw_pf,
                                                          row_off=to_dev_i32(raw_off, DEV))
    rd.stream.synchronize()
    u = int(counts[0])
    return out.cpu().numpy(), table[:u + 1].cpu().numpy(), index.cpu().numpy(), counts.cpu().numpy()


def _same_reads(a, b, where):
    """_reads of two table sets: pooled outputs and raw rows bit for bit, raw index and counts equal."""
    assert same_bits(a[0], b[0]) and same_bits(a[1], b[1]), where
    assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3]), where


# ---- 1. virtual ranks: live exports grow under their readers ------------------------------------------------------------
@pytest.mark.parametrize("R", [2, 4])
def test_live_owners_grow_under_readers(torch_cuda, R):
    import persia_b200.shard as SH
    from persia_b200.worker import ShardedEmbeddingWorker as SW, ShardedRawWorker as RW

    torch = torch_cuda
    if not _fd_handles():
        pytest.skip("the device cannot export memory as POSIX file descriptors")
    rng = np.random.default_rng(40 + R)
    dim, B, cap = 16, 4096, 1 << 22
    pf, raw_pf = [1 << 56, 2 << 56], 3 << 56
    groups = {}
    for grow in (False, "shared"):
        sw = SW.local_group(R, 2, dim, pf, cap, cap=2 * B, optimizer=OPT, max_batch=B, grow=grow)
        rw = RW.local_group(R, 1, dim, [raw_pf], cap, cap=3 * B, optimizer=OPT, max_batch=B, max_ids_per_sample=3,
                            shards=[w.shard for w in sw])
        for w in sw:
            w.shard.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
        torch.cuda.synchronize()
        groups[grow] = (sw, rw, _live_readers(torch, [w.shard for w in sw]))
    tracks = [_Growth(w.shard) for w in groups["shared"][0]]
    try:
        for step in range(16):
            ids = [rng.integers(0, 80_000 * (step + 1), size=2 * B, dtype=np.uint64) for _ in range(R)]
            g = [(rng.standard_normal((2, B, dim)) * 1e-2).astype(np.float16) for _ in range(R)]
            raw = []
            for _ in range(R):
                n = rng.integers(1, 4, size=B)
                off = np.zeros(B + 1, np.uint32)
                off[1:] = np.cumsum(n)
                raw.append((rng.integers(0, 1 << 30, size=int(off[-1]), dtype=np.uint64), off))
            # queries: signs trained so far and never trained
            qs = []
            for _ in range(R):
                n = rng.integers(1, 4, size=B)
                off = np.zeros(B + 1, np.uint32)
                off[1:] = np.cumsum(n)
                qs.append((rng.integers(0, 160_000 * (step + 1), size=2 * B, dtype=np.uint64),
                           rng.integers(0, 1 << 30, size=int(off[-1]), dtype=np.uint64), off))
            res = {}
            for grow, (sw, rw, readers) in groups.items():
                SW.group_forward(sw, [to_dev_ids(x, DEV) for x in ids], B, training=True)
                routs = RW.group_forward_raw(rw, [to_dev_ids(x, DEV) for x, _ in raw], B, 4,
                                             row_offs=[to_dev_i32(o, DEV) for _, o in raw])
                torch.cuda.synchronize()
                SW.group_backward(sw, [[torch.from_numpy(g[r][k]).to(DEV) for k in range(2)] for r in range(R)])
                us = [int(ro[4][0]) for ro in routs]
                rg = [torch.from_numpy((np.random.default_rng(step * 8 + r).standard_normal((us[r], dim)) * 1e-2)
                                       .astype(np.float32)).to(DEV) for r in range(R)]
                RW.group_backward_raw(rw, rg)
                torch.cuda.synchronize()
                res[grow] = [_reads(readers[r], qs[r], pf, raw_pf) for r in range(R)]
            for r in range(R):
                _same_reads(res[False][r], res["shared"][r], (step, r))
            for t in tracks:
                t.note()
        for grow, (sw, _, _) in groups.items():
            for w in sw:
                c = w.shard.counters()
                assert c["wait_errors"] == 0
        assert [w.shard.counters()["lookup_miss"] for w in groups[False][0]] == \
            [w.shard.counters()["lookup_miss"] for w in groups["shared"][0]]
        assert all(t.row_growths >= 2 and t.doublings >= 2 for t in tracks), \
            [(t.row_growths, t.doublings) for t in tracks]
    finally:
        for sw, rw, readers in groups.values():
            for rd in readers:
                rd.close()
            for w in rw + sw:
                w.close()


# ---- 2. virtual ranks: frozen exports grow through set_entries under their readers ------------------------------------
@pytest.mark.parametrize("R", [2, 4])
def test_frozen_owners_grow_through_inserts(torch_cuda, R):
    import persia_b200.shard as SH
    from persia_b200 import native as N
    from persia_b200.persia_core import farmhash64_np
    from persia_b200.worker import RemoteReader

    torch = torch_cuda
    if not _fd_handles():
        pytest.skip("the device cannot export memory as POSIX file descriptors")
    rng = np.random.default_rng(70 + R)
    dim, B = 32, 4096
    pf, raw_pf = [1 << 56], 2 << 56
    twins = {}
    for grow in (False, "shared"):
        shards = []
        for _ in range(R):
            s = SH.EmbeddingShard(dim, 1 << 21, 0, grow=grow)
            s.set_optimizer(**OPT)
            s.configure()
            shards.append(s)
        twins[grow] = (shards, RemoteReader.local_group(shards))
    tracks = [_Growth(s) for s in twins["shared"][0]]
    try:
        # a mode-1 table still refuses export
        m1 = SH.EmbeddingShard(8, 1 << 16, 0, grow=True)
        m1.set_optimizer(**OPT)
        with pytest.raises(N.PersiaB200Error):
            m1.export_view()
        m1.close()
        for step in range(10):
            signs = rng.integers(0, 1 << 40, size=30_000 * (step + 1), dtype=np.uint64)
            signs = np.unique(np.concatenate([signs | np.uint64(1 << 56), signs[: len(signs) // 2] | np.uint64(raw_pf)]))
            owner = farmhash64_np(signs) % np.uint64(R)
            ent_len = twins[False][0][0].entry_len
            ent = (rng.standard_normal((signs.size, ent_len)) * 0.05).astype(np.float32)
            for grow, (shards, _) in twins.items():
                for r, s in enumerate(shards):
                    k = owner == r
                    s.set_entries(to_dev_ids(signs[k], DEV), torch.from_numpy(ent[k]).to(DEV))
            torch.cuda.synchronize()
            qids = np.concatenate([rng.choice(signs, size=B) & np.uint64((1 << 56) - 1),
                                   rng.integers(0, 1 << 40, size=B, dtype=np.uint64)])
            n = rng.integers(1, 4, size=B)
            off = np.zeros(B + 1, np.uint32)
            off[1:] = np.cumsum(n)
            raw_q = rng.choice(signs, size=int(off[-1])) & np.uint64((1 << 56) - 1)
            res = {grow: [_reads(rd, (qids, raw_q, off), pf, raw_pf) for rd in readers]
                   for grow, (_, readers) in twins.items()}
            for r in range(R):
                _same_reads(res[False][r], res["shared"][r], (step, r))
            for t in tracks:
                t.note()
        assert all(t.row_growths >= 2 and t.doublings >= 2 for t in tracks), \
            [(t.row_growths, t.doublings) for t in tracks]
        for s in twins["shared"][0]:
            assert s.counters()["wait_errors"] == 0
    finally:
        for shards, readers in twins.values():
            for rd in readers:
                rd.close()
            for s in shards:
                s.close()


# ---- 3. two processes on one device ------------------------------------------------------------------------------------
def _values(signs, ent_len):
    """Entries as a function of the sign, exact in f16: what any reader must read back."""
    v = ((signs % np.uint64(997)).astype(np.int64) - 498).astype(np.float32) / 256.0
    return np.repeat(v[:, None], ent_len, axis=1) + np.arange(ent_len, dtype=np.float32)[None, :] / 64.0


def _two_process_rank(rank, store_path, out_q):
    import time

    import torch
    import torch.distributed as dist

    import persia_b200.shard as SH
    from persia_b200 import native as N
    from persia_b200.persia_core import farmhash64_np
    from persia_b200.worker import RemoteReader, exchange_readers

    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", init_method=f"file://{store_path}", rank=rank, world_size=2)
        lib = N.load()
        lib.pb_debug_owned.argtypes = [C.POINTER(C.c_uint64)]
        lib.pb_debug_defer_sends.argtypes = [C.c_void_p, C.c_int]
        lib.pb_debug_stale_retries.restype = C.c_uint64
        owned0 = (C.c_uint64 * 2)()
        lib.pb_debug_owned(owned0)
        dim, B = 16, 8192
        sh = SH.EmbeddingShard(dim, 1 << 22, 0, grow="shared")
        sh.set_optimizer(**OPT)
        sh.configure()
        ent_len = sh.entry_len
        rng = np.random.default_rng(5)
        pool = np.unique(rng.integers(0, 1 << 40, size=2_000_000, dtype=np.uint64)) | np.uint64(1 << 56)
        mine = pool[farmhash64_np(pool) % np.uint64(2) == np.uint64(rank)]

        def insert(lo, hi):
            x = mine[lo:hi]
            sh.set_entries(to_dev_ids(x, DEV), torch.from_numpy(_values(x, ent_len)).to(DEV))
            torch.cuda.synchronize()

        # before the reader registers: several chunks and doublings (rank 0 only), sent on registration
        done = 0
        if rank == 0:
            for hi in (20_000, 60_000, 140_000):
                insert(done, hi)
                done = hi
        else:
            insert(0, 1000)
            done = 1000
        dist.barrier()
        views = [None, None]
        blobs = [None, None]
        dist.all_gather_object(blobs, sh.export_live_view())
        views[1 - rank] = SH.TableView(blobs[1 - rank], 0)
        exchange_readers(sh, views)
        dist.barrier()
        rd = RemoteReader(sh, views, rank, stream=torch.cuda.Stream(device=0))

        def query(counts):
            """B pooled ids drawn from every sign both ranks inserted so far, and the outputs they must read."""
            ins = np.concatenate([pool[farmhash64_np(pool) % np.uint64(2) == np.uint64(q)][:counts[q]] for q in (0, 1)])
            q = np.random.default_rng(int(ins.size)).choice(ins, size=B) & np.uint64((1 << 56) - 1)
            return q, _values(q | np.uint64(1 << 56), ent_len)[:, :dim].astype(np.float16)

        def read(q):
            out = rd.forward(to_dev_ids(q, DEV), B, [1 << 56])
            rd.stream.synchronize()
            return out.cpu().numpy()[0]

        def check():
            """rank 1 reads every sign both ranks inserted so far; the results equal their values."""
            got_all = [None, None]
            dist.all_gather_object(got_all, int(done))
            if rank == 1:
                q, want = query(got_all)
                assert same_bits(read(q), want), "a remote read differs from the owner's entries"
            dist.barrier()  # (the owner changes nothing before the read is done)

        check()
        # the owner grows while the other process reads
        for hi in (200_000, 260_000, 340_000, 440_000):
            if rank == 0:
                insert(done, hi)
                done = hi
            dist.barrier()
            check()
        # a stale read, in this order: the owner grows and keeps the new chunks; the reader's call meets rows or cells
        # it has not mapped (its process counts a stale retry, and the call waits); only then does the owner send them
        retries0 = lib.pb_debug_stale_retries()
        if rank == 0:
            lib.pb_debug_defer_sends(sh.h, 1)
            hi = min(len(mine), done + 2 * int(sh.storage_stats()["mapped_rows"]))  # (past every row mapped so far)
            insert(done, hi)
            done = hi
        dist.barrier()
        got_all = [None, None]
        dist.all_gather_object(got_all, int(done))
        if rank == 0:
            dist.barrier()  # (the reader's call has met a stale item and waits)
            lib.pb_debug_defer_sends(sh.h, 0)
        else:
            q, want = query(got_all)
            box = {}

            def call():
                try:
                    box["out"] = read(q)
                except BaseException as e:  # noqa: BLE001 (raised below, in this thread)
                    box["err"] = e

            th = threading.Thread(target=call)
            th.start()
            t0 = time.monotonic()
            while lib.pb_debug_stale_retries() == retries0 and th.is_alive() and time.monotonic() - t0 < 15:
                time.sleep(0.005)
            met = lib.pb_debug_stale_retries() > retries0
            dist.barrier()  # the owner sends its kept chunks now
            th.join(timeout=60)
            assert not th.is_alive(), "the read did not return"
            if "err" in box:
                raise box["err"]
            assert met, "the read never met the chunks the owner kept"
            assert same_bits(box["out"], want), "a read after a stale retry differs from the owner's entries"
        dist.barrier()
        st = sh.storage_stats()
        assert st["refused_unmapped"] == 0
        assert sh.counters()["wait_errors"] == 0
        rd.close()
        dist.barrier()  # (every view closed before any table)
        sh.close()
        torch.cuda.synchronize()
        owned1 = (C.c_uint64 * 2)()
        lib.pb_debug_owned(owned1)
        assert tuple(owned1) == tuple(owned0), (tuple(owned0), tuple(owned1))
        dist.barrier()
        dist.destroy_process_group()
        out_q.put((rank, "ok"))
    except BaseException as e:  # noqa: BLE001 (reported to the parent)
        import traceback

        out_q.put((rank, "".join(traceback.format_exception(e))))
        raise


def test_two_processes_one_device(torch_cuda):
    import multiprocessing as mp

    if not _fd_handles():
        pytest.skip("the device cannot export memory as POSIX file descriptors")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    with tempfile.TemporaryDirectory() as d:
        store = os.path.join(d, "store")
        ps = [ctx.Process(target=_two_process_rank, args=(r, store, q)) for r in range(2)]
        for p in ps:
            p.start()
        results = {}
        try:
            for _ in range(2):
                r, msg = q.get(timeout=600)
                results[r] = msg
                if msg != "ok":
                    break
            for p in ps:
                p.join(timeout=60)
        finally:
            for p in ps:
                if p.is_alive():
                    p.terminate()
                    p.join(timeout=30)
    assert results == {0: "ok", 1: "ok"}, results
    assert all(p.exitcode == 0 for p in ps), [p.exitcode for p in ps]
