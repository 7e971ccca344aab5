"""GPU: remote reads of owners whose tables hold most of their entries in a shared host tier
(pb_table_create_host_shared, pb_view_open_tiered, k_remote_lookup<TIER>).

R virtual ranks share cuda:0, as in test_gpu_remote_infer.py.  Each rank's table keeps a few dozen rows in HBM and the
rest in its tier.  Frozen: remote reads of every layout equal the collective path's inference forwards bit for bit, and
the owners' miss counters grow alike; inserts beside reads are seen whole or not at all.  Live: SGD at lr 0 with an
eviction check every step keeps every entry its sign's initial row while entries move in and out of the tiers; a read
returns that row or zeros, never another sign's row.  A live tiered step adds the launches the header states.  A
refused shared mapping leaves nothing behind, and a second process opens a rank's tier through /proc.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from util import make_batch, same_bits, to_dev_i32, to_dev_ids  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HBM, TIER = 48, 1 << 14  # HBM rows per rank, far fewer than the entries each rank holds


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def _misses(ws):
    return [int(w.shard.counters()["lookup_miss"]) for w in ws]


def _populate(torch, shards, prefixes, n_ids, rng):
    """Entries for ids [0, n_ids) of every prefix, each set on its owner (HBM rows first, the rest into the tier)."""
    from persia_b200 import shard as SH

    R, dim = len(shards), shards[0].dim
    for p in sorted(set(prefixes)):
        ids = torch.arange(n_ids, dtype=torch.int64, device=DEV)
        signs = SH.add_prefix(ids, [0, n_ids], [p])
        owner = SH.shard_of(signs, R)
        for r, s in enumerate(shards):
            sel = signs[owner == r]
            ent = torch.from_numpy((rng.standard_normal((sel.numel(), s.entry_len)) * 0.1).astype(np.float32)).to(DEV)
            s.set_entries(sel, ent)
    torch.cuda.synchronize()
    for s in shards:
        st = s.tier_stats()
        assert st["host_rows"] > 4 * HBM and st["dropped"] == 0, st


def _tiered_group(torch, R, S, dim, pf, B, ragged=False, max_ids=1):
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    return W.local_group(R, S, dim, pf, HBM, cap=S * B * max_ids, optimizer=dict(kind=N.OPT_SGD, lr=0.05, wd=0.0),
                         max_batch=B, sqrt_scaling=[i % 2 == 0 for i in range(S)] if ragged else None, rows_f32=ragged,
                         max_ids_per_sample=max_ids, tier_rows=TIER, shared_tier=True)


# ---- 1. frozen, bit for bit --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,dim,layout", [(2, 64, "one"), (4, 8, "one"), (2, 128, "one"), (2, 13, "one"),
                                          (2, 12, "ragged"), (4, 128, "ragged"), (2, 13, "ragged")])
def test_tiered_remote_matches_collective(torch_cuda, oracle, R, dim, layout):
    from persia_b200.worker import RemoteReader
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    rng = np.random.default_rng(17 * R + dim)
    S, B, known = 3, 256, 1500
    ragged = layout == "ragged"
    max_ids = 4 if ragged else 1
    pf = [oracle.index_prefix(i) for i in range(S)]
    sqrt = [i % 2 == 0 for i in range(S)] if ragged else [False] * S
    ws = _tiered_group(torch, R, S, dim, pf, B, ragged, max_ids)
    _populate(torch, [x.shard for x in ws], pf, known, rng)
    # ids beyond `known` are held nowhere: misses on their owners
    bs = [make_batch(rng, S, B, 2 * known, max_ids=max_ids, allow_empty=ragged) for _ in range(R)]
    d_ids = [to_dev_ids(b[0], DEV) for b in bs]
    d_off = [to_dev_i32(b[1], DEV) for b in bs] if ragged else None
    m0 = _misses(ws)
    want = W.group_forward(ws, d_ids, B, training=False, row_offs=d_off, slot_occ_offs=[b[2] for b in bs])
    torch.cuda.synchronize()
    want = [x.cpu().numpy() for x in want]
    m1 = _misses(ws)
    assert sum(m1) > sum(m0)
    readers = RemoteReader.local_group([x.shard for x in ws])
    try:
        for r in range(R):  # one rank at a time: nothing runs on the others
            got = readers[r].forward(d_ids[r], B, pf, sqrt, row_off=d_off[r] if ragged else None, slot_occ_off=bs[r][2])
            readers[r].stream.synchronize()
            assert same_bits(got.cpu().numpy(), want[r]), (r, layout)
        m2 = _misses(ws)
        assert [b - a for a, b in zip(m1, m2)] == [b - a for a, b in zip(m0, m1)]
        for x in ws:
            assert x.shard.counters()["wait_errors"] == 0
            assert x.shard.tier_stats()["restored"] == 0  # inference moved nothing
    finally:
        for rd in readers:
            rd.close()


@pytest.mark.parametrize("R,dim", [(2, 12), (4, 64), (2, 13)])
def test_tiered_remote_raw_matches_collective(torch_cuda, oracle, R, dim):
    from persia_b200 import native as N
    from persia_b200.worker import RemoteReader, ShardedRawWorker

    torch = torch_cuda
    rng = np.random.default_rng(R * dim + 1)
    B, fixed, known = 300, 5, 2000
    prefix = oracle.index_prefix(3)
    ws = ShardedRawWorker.local_group(R, 1, dim, [prefix], HBM, cap=B * 6,
                                      optimizer=dict(kind=N.OPT_SGD, lr=0.05, wd=0.0), max_batch=B, max_ids_per_sample=6,
                                      tier_rows=TIER, shared_tier=True)
    _populate(torch, [x.shard for x in ws], [prefix], known, rng)
    bs = [make_batch(rng, 1, B, 2 * known, max_ids=6, allow_empty=True) for _ in range(R)]
    ids, offs = [to_dev_ids(b[0], DEV) for b in bs], [to_dev_i32(b[1], DEV) for b in bs]
    m0 = _misses(ws)
    want = ShardedRawWorker.group_forward_raw(ws, ids, B, fixed, training=False, row_offs=offs)
    torch.cuda.synchronize()
    want = [[t.cpu().numpy() for t in x] for x in want]
    m1 = _misses(ws)
    readers = RemoteReader.local_group([x.shard for x in ws])
    try:
        for r in range(R):
            got = readers[r].forward_raw(ids[r], B, fixed, prefix, row_off=offs[r])
            readers[r].stream.synchronize()
            table, index, non_empty, num, counts = [t.cpu().numpy() for t in got]
            U, ne = counts.tolist()
            assert counts.tolist() == want[r][4].tolist()
            assert same_bits(table[:U + 1], want[r][0][:U + 1])
            assert (index == want[r][1]).all() and (non_empty[:ne] == want[r][2][:ne]).all()
            assert (num == want[r][3]).all()
        m2 = _misses(ws)
        assert [b - a for a, b in zip(m1, m2)] == [b - a for a, b in zip(m0, m1)]
        assert all(x.shard.counters()["wait_errors"] == 0 for x in ws)
    finally:
        for rd in readers:
            rd.close()


# ---- 2. inserts beside frozen reads --------------------------------------------------------------------------------------
def test_inserts_beside_frozen_tiered_reads(torch_cuda, tmp_path):
    """set_entries and `.inc` packets (pb_image_insert, as an Infer job applies them) on the owners, alternately:
    restores out of the tier, HBM and tier inserts, while every rank reads.  Each row read is the entry before the
    insert or after it (f16 of either), never a mix and never another sign's."""
    import threading

    from persia_b200 import incremental as INC
    from persia_b200 import persia_core as PC
    from persia_b200 import shard as SH
    from persia_b200.worker import RemoteReader

    torch = torch_cuda
    rng = np.random.default_rng(3)
    R, B, dim, known = 2, 1024, 32, 3000
    ws = _tiered_group(torch, R, 1, dim, [0], B)
    shards = [x.shard for x in ws]
    _populate(torch, shards, [0], known, rng)
    signs = torch.arange(2 * known, dtype=torch.int64, device=DEV)
    owner = SH.shard_of(signs, R)
    cur = np.zeros((2 * known, dim), np.float16)  # what each sign reads as now (zeros: held nowhere)
    for r, s in enumerate(shards):
        sel = signs[owner == r]
        ent, found = s.get_entries(sel)
        cur[sel.cpu().numpy()[found.cpu().numpy()]] = ent[found].half().cpu().numpy()
    readers = RemoteReader.local_group(shards)
    try:
        for it in range(12):
            q = rng.integers(0, 2 * known, size=B).astype(np.uint64)
            d_q = to_dev_ids(q, DEV)
            upd = rng.choice(2 * known, size=400, replace=False)  # known signs and new ones alike
            new = (rng.standard_normal((400, dim)) * 0.1).astype(np.float32)
            d_upd = torch.from_numpy(upd.astype(np.int64)).to(DEV)
            d_new = torch.from_numpy(new).to(DEV)
            d_own = SH.shard_of(d_upd, R)
            torch.cuda.synchronize()
            outs = [readers[r].forward(d_q, B, [0]) for r in range(R)]
            own = d_own.cpu().numpy()
            for r, s in enumerate(shards):
                m = d_own == r
                if it % 2 == 0:
                    s.set_entries(d_upd[m], d_new[m])
                else:  # the owner's signs as one packet, inserted on the packet reader's stream
                    path = str(tmp_path / f"p{it}_{r}.inc")
                    with open(path, "wb") as f:
                        f.write(INC.encode_packet(upd[own == r].astype(np.uint64), dim, new[own == r]))
                    group = {"shard": s, "lock": threading.RLock(), "device": 0}
                    assert PC._apply_packet_file(path, {dim: group}) == (0, int((own == r).sum()))
            outs += [readers[r].forward(d_q, B, [0]) for r in range(R)]
            torch.cuda.synchronize()
            after = cur.copy()
            after[upd] = new.astype(np.float16)
            before_bits, after_bits = cur[q.astype(np.int64)].view(np.uint16), after[q.astype(np.int64)].view(np.uint16)
            for o in outs:
                ov = o[0].cpu().numpy().view(np.uint16)
                ok = np.all(ov == before_bits, axis=1) | np.all(ov == after_bits, axis=1)
                assert ok.all(), it
            cur = after
        assert all(s.counters()["wait_errors"] == 0 for s in shards)
    finally:
        for rd in readers:
            rd.close()
        PC.reset()  # (its packet reader)


# ---- 3. live churn --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tier_rows,staged", [(TIER, False), (TIER, True), (600, False)])
def test_live_tiered_reads_across_moves(torch_cuda, tier_rows, staged):
    """SGD at lr 0: every entry stays its sign's initial row (a function of the sign alone) wherever it lives.  HBM holds
    a third of each rank's signs and an eviction check runs every step, so every step restores signs from the tier and
    moves others out.  Reads issued before, beside and after each step return, per item, exactly the sign's initial row,
    or zeros only for a sign no step had admitted before the read (or, with a tier too small to hold every entry, one it
    may have dropped), i.e. a sign its owner held before the read and holds after it is never read as a miss.
    staged: a TierStager stages the next step's signs beside the backward (its eviction check and restores on the
    stagers' streams), and reads are issued beside the stage too."""
    from persia_b200 import native as N
    from persia_b200.shard import EmbeddingShard, TableView
    from persia_b200.worker import RemoteReader, TierStager
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    R, B, dim, card, cap = 2, 512, 64, 3000, 1024
    rng = np.random.default_rng(tier_rows)
    ws = W.local_group(R, 1, dim, [0], cap, cap=B, optimizer=dict(kind=N.OPT_SGD, lr=0.0, wd=0.0), max_batch=B,
                       tier_rows=tier_rows, shared_tier=True)
    for x in ws:
        x.shard.set_eviction(check_every=1, low_water=cap // 3, target_free=cap // 2, keep_batches=1)
    ref = EmbeddingShard(dim, 1 << 16, 0)
    ref.set_optimizer(kind=N.OPT_SGD, lr=0.0, wd=0.0)
    ref.configure()
    blobs = [x.shard.export_live_view() for x in ws]
    readers = [RemoteReader(x.shard, [TableView(b, 0) if q != r else None for q, b in enumerate(blobs)], r,
                            stream=torch.cuda.Stream(device=DEV)) for r, x in enumerate(ws)]
    stagers = TierStager.local_group([x.shard for x in ws], B) if staged else None
    steps = [[rng.integers(0, card, size=B, dtype=np.uint64) for _ in range(R)] for _ in range(81)]
    if staged:
        first = [to_dev_ids(b, DEV) for b in steps[0]]
        torch.cuda.synchronize()
        TierStager.group_stage(stagers, first, [[0, B]] * R, [0])

    def held(d_q):  # whether the owners hold each sign (in HBM or the tier), read between steps
        from persia_b200 import shard as SH

        own = SH.shard_of(d_q, R)
        out = torch.zeros(d_q.numel(), dtype=torch.bool, device=DEV)
        for r, x in enumerate(ws):
            m = own == r
            out[m] = x.shard.get_entries(d_q[m])[1]
        return out.cpu().numpy()

    try:
        rows_seen = zeros_seen = 0
        for step in range(80):
            ids = steps[step]
            q = rng.integers(0, card, size=B, dtype=np.uint64)
            d_q = to_dev_ids(q, DEV)
            d_ids = [to_dev_ids(b, DEV) for b in ids]
            d_next = [to_dev_ids(b, DEV) for b in steps[step + 1]]
            zeros = [[torch.zeros((B, dim), dtype=torch.float16, device=DEV)] for _ in range(R)]
            torch.cuda.synchronize()
            before = held(d_q)
            outs = [(readers[r].forward(d_q, B, [0]), before) for r in range(R)]
            step_out = W.group_forward(ws, d_ids, B, training=True, slot_occ_offs=[[0, B]] * R)
            outs += [(readers[r].forward(d_q, B, [0]), before) for r in range(R)]
            if staged:  # the next step's moves beside this step's backward, and reads beside them
                TierStager.group_stage(stagers, d_next, [[0, B]] * R, [0])
                outs += [(readers[r].forward(d_q, B, [0]), before) for r in range(R)]
            W.group_backward(ws, zeros)
            torch.cuda.synchronize()
            del step_out, zeros, d_ids, d_next
            after = held(d_q)
            outs += [(readers[r].forward(d_q, B, [0]), after) for r in range(R)]
            torch.cuda.synchronize()
            want = ref.lookup(d_q, training=True).half().cpu().numpy().view(np.uint16)
            drops = sum(x.shard.tier_stats()["dropped"] for x in ws)
            for o, adm in outs:
                ov = o[0].cpu().numpy().view(np.uint16)
                zero = np.all(ov == 0, axis=1)
                mine = np.all(ov == want, axis=1)
                assert np.all(zero | mine), step
                if not drops:
                    assert not np.any(zero & ~mine & adm), step  # an admitted sign is never a false miss
                rows_seen += int(mine.sum())
                zeros_seen += int((zero & ~mine).sum())
        assert rows_seen > 0
        for x in ws:
            st = x.shard.tier_stats()
            assert st["restored"] > 0 and st["moved_out"] > 0, st
            assert (st["dropped"] > 0) == (tier_rows < card), st
            assert x.shard.counters()["wait_errors"] == 0
            if staged:
                assert x.shard.stage_stats()["staged"] > 0
        if staged:
            assert not any(any(s.status()) for s in stagers)
    finally:
        for rd in readers:
            rd.close()
        for s in stagers or []:
            s.close()
        ref.close()


# ---- 4. launches a live tiered step adds -------------------------------------------------------------------------------
def test_live_tiered_step_launch_count(torch_cuda):
    """Two groups on the same batches, one exported live: each step of the exported one launches 4 more kernels per
    rank (k_seq_begin / k_seq_end around the SEND's eviction check and around the SERVE's restore), and nothing else."""
    from persia_b200 import native as N
    from persia_b200.worker import ShardedEmbeddingWorker as W

    torch = torch_cuda
    # room for two whole batches per owner after every check: no admission or restore is refused, so which signs hold
    # rows never depends on the order the device serves them in, and the two groups stay equal
    R, B, dim, card, cap = 2, 256, 16, 6000, 2048
    lib = N.load()
    groups = []
    for _ in range(2):
        ws = W.local_group(R, 1, dim, [0], cap, cap=B, optimizer=dict(kind=N.OPT_SGD, lr=0.0, wd=0.0), max_batch=B,
                           tier_rows=TIER, shared_tier=True)
        for x in ws:
            x.shard.set_eviction(check_every=1, low_water=2 * R * B, target_free=2 * R * B + 32, keep_batches=1)
        groups.append(ws)
    for x in groups[1]:
        x.shard.export_live_view()
    rng = np.random.default_rng(4)
    torch.cuda.synchronize()
    for step in range(12):
        ids = [to_dev_ids(rng.integers(0, card, size=B, dtype=np.uint64), DEV) for _ in range(R)]
        zeros = [[torch.zeros((B, dim), dtype=torch.float16, device=DEV)] for _ in range(R)]
        n = []
        for ws in groups:
            torch.cuda.synchronize()
            l0 = lib.pb_launch_count()
            W.group_forward(ws, ids, B, training=True, slot_occ_offs=[[0, B]] * R)
            W.group_backward(ws, zeros)
            torch.cuda.synchronize()
            n.append(lib.pb_launch_count() - l0)
        assert n[1] - n[0] == 4 * R, (step, n)
    assert all(x.shard.tier_stats()["moved_out"] > 0 for ws in groups for x in ws)
    for a, b in zip(*groups):  # and the two computed the same
        ids = torch.arange(card, dtype=torch.int64, device=DEV)
        ea, fa = a.shard.get_entries(ids)
        eb, fb = b.shard.get_entries(ids)
        assert torch.equal(fa, fb) and torch.equal(ea[fa], eb[fb])


def test_live_tiered_captured_step_equals_eager(torch_cuda):
    """One GPU's training step on a live-exported table with a shared tier (an eviction check every step, so entries
    move out to the tier and back every step) captured once in a CUDA graph and replayed on new batches, against the
    same steps eager on a like table that is not exported: the windows' launches run inside the graph, and every output
    and entry (HBM and tier) stays the eager table's."""
    from persia_b200 import native as N
    from persia_b200.shard import BatchContext, EmbeddingShard

    torch = torch_cuda
    S, B, dim, cap = 2, 512, 32, 4096
    pf = [1 << 56, 2 << 56]
    shards = []
    for _ in range(2):
        s = EmbeddingShard(dim, cap, 0, tier_rows=TIER, shared_tier=True)
        s.set_optimizer(kind=N.OPT_ADAGRAD, lr=0.05, initialization=0.01)
        s.configure()
        # every check frees all but the rows of the last two requests (<= 2 x S * B), so a step's restores and
        # admissions (S * B at most) always find a free row: no outcome depends on which lane pops one first; the
        # 6000 signs the batches draw outgrow the HBM rows, so every step moves entries out and back
        s.set_eviction(check_every=1, low_water=cap, target_free=cap, keep_batches=1)
        shards.append(s)
    plain, live = shards
    live.export_live_view()
    ctxs = [BatchContext(S * B, S * B, pf) for _ in range(2)]
    rng = np.random.default_rng(6)
    slot_off = [0, B, 2 * B]
    ids_dev = torch.empty(S * B, dtype=torch.int64, device=DEV)
    g_dev = torch.zeros((S, B, dim), dtype=torch.float16, device=DEV)
    outs = [torch.empty((S, B, dim), dtype=torch.float16, device=DEV) for _ in range(2)]
    seen = set()

    def draw():
        ids = rng.integers(0, 3000, size=S * B, dtype=np.uint64)
        seen.update(ids.tolist())
        ids_dev.copy_(to_dev_ids(ids, DEV))
        g_dev.copy_(torch.from_numpy((rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)).to(DEV))
        torch.cuda.synchronize()

    stream = torch.cuda.Stream()
    draw()
    with torch.cuda.stream(stream):
        for k in range(2):
            ctxs[k].forward(shards[k], ids_dev, slot_off, B, training=True, out=outs[k])  # warm-up: a real step
            ctxs[k].backward(shards[k], [g_dev[i] for i in range(S)])
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            ctxs[1].forward(live, ids_dev, slot_off, B, training=True, out=outs[1])
            ctxs[1].backward(live, [g_dev[i] for i in range(S)])
    for it in range(12):
        draw()
        with torch.cuda.stream(stream):
            ctxs[0].forward(plain, ids_dev, slot_off, B, training=True, out=outs[0])  # eager
            ctxs[0].backward(plain, [g_dev[i] for i in range(S)])
            graph.replay()
            stream.synchronize()
        assert same_bits(outs[1].cpu().numpy(), outs[0].cpu().numpy()), it
    for s in shards:
        st = s.tier_stats()
        assert st["moved_out"] > 0 and st["restored"] > 0 and st["refused"] == 0 and st["dropped"] == 0, st
        assert s.counters()["capacity_refused"] == 0
    from persia_b200.shard import add_prefix

    ids = to_dev_ids(np.array(sorted(seen), np.uint64), DEV)
    signs = torch.cat([add_prefix(ids, [0, ids.numel()], [p]) for p in pf])
    (pa, pf_), (la, lf) = plain.get_entries(signs), live.get_entries(signs)
    assert torch.equal(pf_, lf) and int(pf_.sum()) > cap  # (more than HBM holds: the rest in the tiers)
    assert same_bits(pa[pf_].cpu().numpy(), la[lf].cpu().numpy())
    for c in ctxs:
        c.close()
    for s in shards:
        s.close()


# ---- 5. ownership, and a second process ----------------------------------------------------------------------------------
def _owned(lib):
    out = (C.c_uint64 * 2)()
    assert lib.pb_debug_owned(out) == 0
    return int(out[0]), int(out[1])


def _debug(lib):
    lib.pb_debug_owned.restype = C.c_int
    lib.pb_debug_owned.argtypes = [C.POINTER(C.c_uint64)]
    lib.pb_debug_refuse_after.restype = None
    lib.pb_debug_refuse_after.argtypes = [C.c_int64]


def test_refused_shared_tier_leaves_nothing_behind(torch_cuda):
    from persia_b200 import native as N
    from persia_b200.shard import EmbeddingShard

    lib = N.load()
    _debug(lib)
    sh = EmbeddingShard(16, 64, 0, tier_rows=1 << 12, shared_tier=True)
    msgs = []
    try:
        for n in range(64):
            o0 = _owned(lib)
            lib.pb_debug_refuse_after(n)
            try:
                sh.set_optimizer(kind=N.OPT_SGD, lr=0.0)  # attaches the tier: both tables' storage, the shared rows
                break
            except N.PersiaB200Error as e:
                msgs.append(str(e))
                assert _owned(lib) == o0, n
            finally:
                lib.pb_debug_refuse_after(-1)
        assert any("shared host mapping" in m for m in msgs), msgs
        assert sh.tier_stats()["host_rows"] == 0
    finally:
        sh.close()


_CHILD = r"""
import sys
import numpy as np
import torch
from persia_b200 import native as N, shard as SH
sh = SH.EmbeddingShard(16, 64, 0, tier_rows=1 << 12, shared_tier=True)
sh.set_optimizer(kind=N.OPT_SGD, lr=0.0)
sh.configure()
signs = torch.arange(3000, dtype=torch.int64, device="cuda:0")
mine = signs[SH.shard_of(signs, 2) == 1]
val = (mine.double().unsqueeze(1) * 1e-3 + torch.arange(16, device="cuda:0").double() * 1e-2).float()
sh.set_entries(mine, val)
print(sh.export_view().hex(), flush=True)
sys.stdin.readline()
"""


def test_second_process_reads_a_shared_tier(torch_cuda):
    """Rank 1 is another process with most of its entries in its tier; rank 0 opens its view (the tier's rows through
    /proc/<pid>/fd) and reads its signs alone.  A refused peer mapping leaves nothing behind."""
    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200.worker import RemoteReader

    torch = torch_cuda
    lib = N.load()
    _debug(lib)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    child = subprocess.Popen([sys.executable, "-c", _CHILD], stdin=subprocess.PIPE, stdout=subprocess.PIPE, env=env,
                             text=True)
    own = view = reader = None
    try:
        blob = bytes.fromhex(child.stdout.readline().strip())
        own = SH.EmbeddingShard(16, 64, 0, tier_rows=1 << 12, shared_tier=True)
        own.set_optimizer(kind=N.OPT_SGD, lr=0.0)
        own.configure()
        msgs = []
        for n in range(16):
            o0 = _owned(lib)
            lib.pb_debug_refuse_after(n)
            try:
                view = SH.TableView(blob, 0)
                break
            except N.PersiaB200Error as e:
                msgs.append(str(e))
                assert _owned(lib) == o0, n
            finally:
                lib.pb_debug_refuse_after(-1)
        assert view is not None and any("shared host mapping" in m for m in msgs), msgs
        reader = RemoteReader(own, [None, view], 0, stream=torch.cuda.Stream(device=DEV))
        q = torch.arange(3000, dtype=torch.int64, device=DEV)
        out = reader.forward(q, 3000, [0])
        reader.stream.synchronize()
        theirs = (SH.shard_of(q, 2) == 1).cpu().numpy()
        want = (q.double().unsqueeze(1) * 1e-3 + torch.arange(16, device=DEV).double() * 1e-2).float().half()
        got = out[0].cpu().numpy().view(np.uint16)
        assert np.array_equal(got[theirs], want.cpu().numpy().view(np.uint16)[theirs])
        assert not got[~theirs].any()  # rank 0's own table holds nothing
    finally:
        if reader is not None:
            reader.close()
        elif view is not None:
            view.close()
        if own is not None:
            own.close()
        try:
            child.stdin.write("\n")
            child.stdin.flush()
        except OSError:
            pass
        try:
            child.wait(timeout=120)
        except subprocess.TimeoutExpired:
            child.kill()
            child.wait()
