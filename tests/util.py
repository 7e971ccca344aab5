"""Shared helpers for the parity tests: seeded synthetic id batches in the reference's LIL shape,
flattened to the slot-major CSR the C ABI takes, and the GPU-vs-oracle training harness."""
import numpy as np

DEV = "cuda:0"


def make_batch(rng, n_slots, batch, cardinality, max_ids=1, allow_empty=False):
    """Returns (ids u64 [N], row_off u32 [S*B+1] or None, slot_occ_off list[S+1]).
    max_ids == 1 and not allow_empty -> single-id slots (row_off None)."""
    card = [cardinality] * n_slots if np.isscalar(cardinality) else list(cardinality)
    if max_ids == 1 and not allow_empty:
        ids = np.stack([rng.integers(0, card[s], size=batch, dtype=np.uint64) for s in range(n_slots)]).reshape(-1)
        slot_off = [s * batch for s in range(n_slots + 1)]
        return ids, None, slot_off
    counts = rng.integers(0 if allow_empty else 1, max_ids + 1, size=n_slots * batch)
    row_off = np.zeros(n_slots * batch + 1, np.uint32)
    row_off[1:] = np.cumsum(counts)
    ids = np.empty(int(row_off[-1]), np.uint64)
    for s in range(n_slots):
        lo, hi = int(row_off[s * batch]), int(row_off[(s + 1) * batch])
        ids[lo:hi] = rng.integers(0, card[s], size=hi - lo, dtype=np.uint64)
    slot_off = [int(row_off[s * batch]) for s in range(n_slots + 1)]
    return ids, row_off, slot_off


def full_row_off(n_slots, batch):
    return np.arange(n_slots * batch + 1, dtype=np.uint32)


def to_dev_ids(ids, device):
    import torch

    return torch.from_numpy(np.ascontiguousarray(ids).view(np.int64)).to(device)


def to_dev_i32(a, device):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).to(device)


def batch_with_multiplicities(rng, n, counts, spans=None):
    """One slot with one id per position (sample, or occurrence of a ragged slot): id k (k = 0, 1, ...) sits at exactly
    counts[k] distinct random positions, drawn from range(*spans[k]) when spans (a dict) has k, every other position
    holds a fresh id of its own.  Ids are placed in the order given: constrained ones should come first.
    Returns uint64 ids [n]."""
    spans = spans or {}
    free = np.ones(n, bool)
    ids = np.empty(n, np.uint64)
    for k, c in enumerate(counts):
        lo, hi = spans.get(k, (0, n))
        cand = np.flatnonzero(free[lo:hi]) + lo
        assert c <= cand.size, (k, c, cand.size)
        pos = rng.choice(cand, size=c, replace=False)
        ids[pos] = k
        free[pos] = False
    ids[free] = np.uint64(int(rng.integers(1 << 32, 1 << 48))) + np.arange(int(free.sum()), dtype=np.uint64)
    return ids


def ragged_with_multiplicities(rng, batch, counts, max_ids, min_ids=1, spans=None):
    """batch_with_multiplicities over the occurrences of a ragged slot whose samples hold min_ids..max_ids ids each
    (spans are occurrence ranges).  Returns (ids uint64 [N], row_off uint32 [batch + 1])."""
    row_off = np.zeros(batch + 1, np.uint32)
    row_off[1:] = np.cumsum(rng.integers(min_ids, max_ids + 1, size=batch))
    return batch_with_multiplicities(rng, int(row_off[-1]), counts, spans), row_off


def f16_ulp_diff(a, b):
    """Max distance in f16 representable steps between two float16 arrays (sign-magnitude -> ordered ints)."""
    def key(x):
        u = x.view(np.uint16).astype(np.int32)
        return np.where(u & 0x8000, -(u & 0x7FFF), u & 0x7FFF)
    return int(np.max(np.abs(key(np.ascontiguousarray(a)) - key(np.ascontiguousarray(b))))) if a.size else 0


# ---- GPU shard + context against an oracle worker (R = 1) ----------------------------------------------------------
def pair(pb, oracle, n_slots, dim, kind, cap=1 << 16, sqrt=None, groups=None, optim_kw=None, hyper_kw=None,
         max_occ=1 << 18):
    """A GPU shard + context and an oracle worker (R=1) with the same slot table."""
    groups = groups or list(range(n_slots))
    pf = [oracle.index_prefix(g) for g in groups]
    sq = sqrt or [False] * n_slots
    optim_kw, hyper_kw = optim_kw or {}, hyper_kw or {}
    s = pb.EmbeddingShard(dim, cap, 0)
    s.set_optimizer(kind, **{{"mom": "g_square_momentum", "init_acc": "initialization", "b1": "beta1",
                              "b2": "beta2"}.get(k, k): v for k, v in optim_kw.items()})
    s.configure(**{{"lo": "init_lower", "hi": "init_upper", "admit_p": "admit_probability",
                    "enable_wb": "enable_weight_bound", "wb": "weight_bound"}.get(k, k): v for k, v in hyper_kw.items()})
    ctx = pb.BatchContext(max_occ, max_occ, pf, sq)
    w = oracle.Worker([oracle.SlotCfg(dim, sqrt_scaling=sq[i], prefix=pf[i]) for i in range(n_slots)], n_ps=1)
    w.configure(**hyper_kw)
    w.set_optimizer(oracle.Optim(kind, **optim_kw))
    return s, ctx, w, pf


def fwd_both(torch, s, ctx, w, ids, row_off, slot_off, B, training=True):
    n_slots = ctx.n_slots
    ro_dev = to_dev_i32(row_off, DEV) if row_off is not None else None
    got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=ro_dev, training=training).cpu().numpy()
    ro = row_off if row_off is not None else full_row_off(n_slots, B)
    want, octx = w.forward(ids, ro, B, training=training)
    return got, want, octx


def entries_equal(torch, s, w, signs, exact=True, rtol=0.0, atol=0.0):
    ent, found = s.get_entries(to_dev_ids(signs, DEV))
    ent = ent.cpu().numpy()
    assert found.all()
    for k, sign in enumerate(signs):
        ref = w.get_entry(int(sign))
        assert ref is not None
        if exact:
            assert ent[k].tobytes() == ref.tobytes(), (k, sign, ent[k], ref)
        else:
            np.testing.assert_allclose(ent[k], ref, rtol=rtol, atol=atol)


def slot_signs(oracle, ids, slot_off, prefixes, prefix_bit=8):
    """The signs of slot-major ids: every slot's index prefix added (indices_add_prefix)."""
    ids = np.asarray(ids, np.uint64)
    out = np.empty(ids.size, np.uint64)
    for s, p in enumerate(prefixes):
        lo, hi = int(slot_off[s]), int(slot_off[s + 1])
        out[lo:hi] = oracle.add_prefix(ids[lo:hi], prefix_bit, p)
    return out


def held_rows(torch, oracle, shards, signs):
    """{sign: f32 [dim]} of the signs the table holds now (HBM or tier); with R > 1 shards each sign is read from its
    owner.  A sign without a row is absent."""
    signs = np.unique(np.asarray(signs, np.uint64))
    R, dim = len(shards), shards[0].dim
    owner = oracle.shard_of(signs, R) if R > 1 else np.zeros(signs.size, np.uint32)
    rows = {}
    for r, s in enumerate(shards):
        mine = signs[owner == r]
        if not mine.size:
            continue
        ent, found = s.get_entries(to_dev_ids(mine, DEV))
        ent, found = ent.cpu().numpy(), found.cpu().numpy().astype(bool)
        rows.update((int(x), ent[k, :dim]) for k, x in enumerate(mine) if found[k])
    return rows


def pool_model(rows, ids, row_off, batch, sqrt, dim=None, order="sample", per_row=False, factor=None):
    """The pooled forward of summation slots (k_gather_items, k_expand_pool), step by step in f32: every output row
    sums the rows of its sample's signs into +0 in ascending occurrence order, skipping signs without a row; a slot with
    sqrt scaling then multiplies by f32(1 / f32(sqrt(max(n, 1)))); the result rounds to f16 (RNE).  One-id layouts
    (row_off None) give f16(0 + row).
      rows     {sign: f32 [dim]}: what the table held at forward time, or (signs u64 [n] ascending, f32 [n, >= dim])
               for batches of millions of distinct signs
      ids      u64 [N] signs (prefixed), slot-major;  row_off  u32 [S*B+1] or None;  sqrt  per-slot bools or None
    Variants that the kernels must NOT match (tests use them to show their inputs discriminate):
      order    "reversed" / "sorted" (by sign) within each sample;  per_row  scale every row before adding it;
      factor   n (int array) -> f32 sqrt factor, instead of the double-rounded one.
    Returns f16 [S, B, dim]."""
    ids = np.asarray(ids, np.uint64)
    if isinstance(rows, tuple):
        keys, held = np.asarray(rows[0], np.uint64), np.asarray(rows[1], np.float32)
        dim = held.shape[1] if dim is None else dim
        table = np.zeros((keys.size + 1, dim), np.float32)  # the last row stands for "no row" (never added)
        table[:-1] = held[:, :dim]
    else:
        keys = np.array(sorted(rows), np.uint64)
        if dim is None:
            dim = len(next(iter(rows.values())))
        table = np.zeros((keys.size + 1, dim), np.float32)
        for k, x in enumerate(keys):
            table[k] = np.asarray(rows[int(x)], np.float32)[:dim]
    pos = np.searchsorted(keys, ids)
    hit = pos < keys.size
    hit[hit] = keys[pos[hit]] == ids[hit]
    idx = np.where(hit, pos, keys.size)
    n_out = ids.size if row_off is None else len(row_off) - 1
    S = n_out // batch if batch else 0
    with np.errstate(over="ignore", invalid="ignore"):
        if row_off is None:
            return (np.float32(0) + table[idx]).astype(np.float16).reshape(S, batch, dim)
        ro = np.asarray(row_off, np.int64)
        cnt = np.diff(ro)
        sample = np.repeat(np.arange(n_out), cnt)
        first = ro[:-1][sample]
        if order == "sample":
            perm = np.arange(ids.size)
        elif order == "reversed":
            perm = 2 * first + cnt[sample] - 1 - np.arange(ids.size)
        else:
            assert order == "sorted", order
            perm = np.lexsort((ids, sample))
        scale = np.ones(n_out, np.float32)
        sq = np.repeat(np.asarray(sqrt if sqrt is not None else [False] * S, bool), batch)
        if sq.any():
            n = np.maximum(cnt[sq], 1)
            scale[sq] = factor(n) if factor else np.float32(1) / np.sqrt(n.astype(np.float32))
        acc = np.zeros((n_out, dim), np.float32)
        for k in range(int(cnt.max(initial=0))):
            m = np.flatnonzero(cnt > k)
            j = perm[ro[m] + k]
            sel, j = m[hit[j]], j[hit[j]]
            v = table[idx[j]]
            acc[sel] = acc[sel] + (v * scale[sel, None] if per_row else v)
        if not per_row:
            acc = acc * scale[:, None]
        return acc.astype(np.float16).reshape(S, batch, dim)


def pool_lists(rows, lists, sqrt):
    """The EW's forward over one slot, in closed form: rows f32 [n, dim], lists the row numbers of every sample; sum into
    zeros in f32, x 1/sqrt(max(n, 1)), RNE to f16 (mod.rs:547-579)."""
    out = np.zeros((len(lists), rows.shape[1]), np.float32)
    for b, ks in enumerate(lists):
        acc = np.zeros(rows.shape[1], np.float32)
        for k in ks:
            acc = acc + rows[k]
        if sqrt:
            acc = acc * (np.float32(1) / np.sqrt(np.float32(max(len(ks), 1))))
        out[b] = acc
    with np.errstate(over="ignore"):
        return out.astype(np.float16)


def same_bits(a, b):
    """Bit equality of two float arrays, except that NaN matches any NaN (CUDA's canonical NaN and x86's default NaN
    differ in payload and sign)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    u = np.uint32 if a.dtype == np.float32 else np.uint16
    return bool((na == nb).all() and (a.view(u)[~na] == b.view(u)[~nb]).all())


# ---- every path that steps a row, on seeded rows (tests/test_gpu_edges.py) ------------------------------------------
EDGE_PATHS = ("batch", "direct", "raw", "shard2", "shard3", "group2", "sraw2")
# multiplicities of ids 0, 1, ... in one batched step: hot past 256 and past 32, two warm, then cold
EDGE_COUNTS = [260, 34, 6, 2]
EDGE_B = 320


def edge_configs(oracle, kind, opt=None, hyper=None):
    """(optimizer kwargs in the oracle's names, hyper kwargs in the oracle's names) with defaults per optimizer."""
    base = {oracle.SGD: dict(lr=0.05, wd=0.0), oracle.ADAGRAD: dict(lr=0.02, init_acc=0.01, eps=1e-10),
            oracle.ADAGRAD_VW: dict(lr=0.02, init_acc=0.01, eps=1e-10),
            oracle.ADAM: dict(lr=0.01, b1=0.9, b2=0.999, eps=1e-8)}[kind]
    return {**base, **(opt or {})}, dict(hyper or {})


def _gpu_optim(kind, o):
    return dict(kind=kind, lr=o["lr"], wd=o.get("wd", 0.0), g_square_momentum=o.get("mom", 1.0),
                initialization=o.get("init_acc", 0.01), eps=o.get("eps", 1e-10), beta1=o.get("b1", 0.9),
                beta2=o.get("b2", 0.999))


def _gpu_hyper(h):
    names = {"lo": "init_lower", "hi": "init_upper", "admit_p": "admit_probability", "enable_wb": "enable_weight_bound",
             "wb": "weight_bound"}
    return {names[k]: v for k, v in h.items()}


def _seed_rows(torch, oracle, shards, w, signs, dim, kind, o, seed_fn, R):
    """Rows seed_fn(signs, dim) (f32 [n, dim]) with fresh optimizer state, on their owners and in the oracle."""
    signs = np.unique(np.asarray(signs, np.uint64))
    opt = oracle.Optim(kind, **o)
    emb = np.asarray(seed_fn(signs, dim), np.float32)
    ent = np.stack([opt.new_entry(e) for e in emb]) if signs.size else np.zeros((0, dim), np.float32)
    owner = oracle.shard_of(signs, R) if R > 1 else np.zeros(signs.size, np.uint32)
    for r, s in enumerate(shards):
        m = owner == r
        if m.any():
            s.set_entries(to_dev_ids(signs[m], DEV), torch.from_numpy(np.ascontiguousarray(ent[m])).to(DEV))
    w.set_embedding(signs, ent, dim)
    torch.cuda.synchronize()
    return signs


def _read_rows(torch, oracle, shards, w, signs, R):
    signs = np.asarray(signs, np.uint64)
    owner = oracle.shard_of(signs, R) if R > 1 else np.zeros(signs.size, np.uint32)
    got = np.zeros((signs.size, shards[0].entry_len), np.float32)
    for r, s in enumerate(shards):
        m = owner == r
        if m.any():
            ent, found = s.get_entries(to_dev_ids(signs[m], DEV))
            assert found.all()
            got[m] = ent.cpu().numpy()
    want = np.stack([w.get_entry(int(x)) for x in signs])
    return got, want


def _out_equal(got, want, what):
    assert same_bits(np.asarray(got), np.asarray(want)), what


def run_edge_path(torch, oracle, path, kind, dim, seed_fn, grad_fn, opt=None, hyper=None, steps=1, rng_seed=0,
                  scale=1.0):
    """One path that steps a row, on rows seeded by seed_fn(signs, dim), with per-row gradients
    grad_fn(rng, ids, dim) (ids: the unprefixed id of every gradient row; the dtype of the result is the request's).
    scale: the loss scale of every gradient request (pb_update has none).
    Outputs, statuses and every seeded entry are compared with the oracle (exact-rsqrt mode); returns
    (signs, GPU entries, oracle entries).  Paths:
      batch   one GPU, the batched step; ids at multiplicities EDGE_COUNTS (hot, warm) and cold
      direct  pb_update with the f32 gradient as given
      raw     pb_forward_raw / pb_backward_raw (f16 gradients are staged, f32 ones too)
      shard2  R = 2 virtual ranks, f16 row exchange;  shard3  R = 3, f32 row exchange
      group2  R = 2, two slots of one feature group (the chained owner walk)
      sraw2   R = 2 sharded raw"""
    from persia_b200 import shard as SH
    from persia_b200.worker import ShardedEmbeddingWorker as W, ShardedRawWorker as RW

    o, h = edge_configs(oracle, kind, opt, hyper)
    rng = np.random.default_rng(rng_seed)
    pf = oracle.index_prefix(0)
    sign = lambda ids: oracle.add_prefix(np.asarray(ids, np.uint64), 8, pf)  # noqa: E731
    gopt, ghyp = _gpu_optim(kind, o), _gpu_hyper(h)
    cap = 1 << 12
    oracle.set_rsqrt_exact(True)
    try:
        if path in ("batch", "direct", "raw"):
            s = SH.EmbeddingShard(dim, cap, 0)
            s.set_optimizer(**gopt)
            s.configure(**ghyp)
            w = oracle.Worker([oracle.SlotCfg(dim, summation=path != "raw", sample_fixed_size=4, prefix=pf)], n_ps=1)
            w.configure(**h)
            w.set_optimizer(oracle.Optim(kind, **o))
            if path == "batch":
                batches = [batch_with_multiplicities(rng, EDGE_B, EDGE_COUNTS) for _ in range(steps)]
                signs = _seed_rows(torch, oracle, [s], w, sign(np.concatenate(batches)), dim, kind, o, seed_fn, 1)
                ctx = SH.BatchContext(EDGE_B, EDGE_B, [pf])
                for ids in batches:
                    got, want, octx = fwd_both(torch, s, ctx, w, ids, None, [0, EDGE_B], EDGE_B)
                    _out_equal(got[0], want[0], "batched forward")
                    g = grad_fn(rng, ids, dim)
                    st = ctx.backward(s, [torch.from_numpy(g).to(DEV)], scales=[scale], want_status=True).cpu().numpy()
                    assert st.tolist() == w.backward(octx, [g], scale=[scale]), "status"
            elif path == "direct":
                ids = np.arange(64, dtype=np.uint64)
                signs = _seed_rows(torch, oracle, [s], w, sign(ids), dim, kind, o, seed_fn, 1)
                for _ in range(steps):
                    g = np.ascontiguousarray(grad_fn(rng, ids, dim), np.float32)
                    s.update(to_dev_ids(sign(ids), DEV), torch.from_numpy(g).to(DEV))
                    w.ps_update(0, sign(ids), np.full(ids.size, dim, np.uint32), g)
            else:
                B = 100
                batches = [ragged_with_multiplicities(rng, B, [5, 3], 3) for _ in range(steps)]
                signs = _seed_rows(torch, oracle, [s], w, sign(np.concatenate([b[0] for b in batches])), dim, kind, o,
                                   seed_fn, 1)
                ctx = SH.BatchContext(3 * B, 3 * B, [pf])
                for ids, ro in batches:
                    table, _, _, _, counts = ctx.forward_raw(s, to_dev_ids(ids, DEV), B, 4, row_off=to_dev_i32(ro, DEV))
                    U = int(counts[0])
                    wt, _, _, _, octx = w.forward_raw(0, ids, ro, B)
                    _out_equal(table[:U + 1].cpu().numpy(), wt, "raw table")
                    uniq = ids[np.sort(np.unique(ids, return_index=True)[1])]  # numbered by first occurrence
                    g = grad_fn(rng, uniq, dim)
                    st = ctx.backward_raw(s, torch.from_numpy(g).to(DEV), scale=scale, want_status=True).item()
                    assert st == w.backward_raw(0, octx, g, scale=scale), "status"
            return (signs,) + _read_rows(torch, oracle, [s], w, signs, 1)

        R = int(path[-1])
        if path == "sraw2":
            B = 100
            ws = RW.local_group(R, 1, dim, [pf], cap, cap=3 * B, optimizer=gopt, hyper=ghyp, max_batch=B,
                                max_ids_per_sample=3)
            w = oracle.Worker([oracle.SlotCfg(dim, summation=False, sample_fixed_size=4, prefix=pf)], n_ps=R)
            batches = [[ragged_with_multiplicities(rng, B, [5, 3], 3) for _ in range(R)] for _ in range(steps)]
            every = np.concatenate([b[0] for st in batches for b in st])
        else:
            S = 2 if path == "group2" else 1
            B = EDGE_B
            ws = W.local_group(R, S, dim, [pf] * S, cap, cap=S * B, optimizer=gopt, hyper=ghyp, max_batch=B,
                               rows_f32=path == "shard3")
            w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf) for _ in range(S)], n_ps=R)
            # ranks and slots share the multiplied ids: a row is stepped by several requests and chain entries
            batches = [[np.concatenate([batch_with_multiplicities(rng, B, EDGE_COUNTS) for _ in range(S)])
                        for _ in range(R)] for _ in range(steps)]
            every = np.concatenate([b for st in batches for b in st])
        w.configure(**h)
        w.set_optimizer(oracle.Optim(kind, **o))
        shards = [x.shard for x in ws]
        for x in shards:  # table storage is allocated on first use, with a device-wide sync: not while a peer waits
            x.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
        signs = _seed_rows(torch, oracle, shards, w, sign(every), dim, kind, o, seed_fn, R)
        for step in batches:
            if path == "sraw2":
                torch.cuda.synchronize()
                res = RW.group_forward_raw(ws, [to_dev_ids(b[0], DEV) for b in step], B, 4,
                                           row_offs=[to_dev_i32(b[1], DEV) for b in step])
                torch.cuda.synchronize()
                octx, grads = [], []
                for r, (ids, ro) in enumerate(step):
                    U = int(res[r][4][0])
                    wt, _, _, _, c = w.forward_raw(0, ids, ro, B)
                    _out_equal(res[r][0][:U + 1].cpu().numpy(), wt, "sharded raw table")
                    octx.append(c)
                    grads.append(grad_fn(rng, ids[np.sort(np.unique(ids, return_index=True)[1])], dim))
                sts = RW.group_backward_raw(ws, [torch.from_numpy(g).to(DEV) for g in grads], scales=[scale] * R,
                                            want_status=True)
                torch.cuda.synchronize()
                for r in range(R):
                    assert sts[r].item() == w.backward_raw(0, octx[r], grads[r], scale=scale), "status"
            else:
                torch.cuda.synchronize()
                outs = W.group_forward(ws, [to_dev_ids(b, DEV) for b in step], B, training=True)
                torch.cuda.synchronize()
                octx = []
                for r in range(R):
                    want, c = w.forward(step[r], full_row_off(S, B), B, training=True)
                    octx.append(c)
                    for i in range(S):
                        _out_equal(outs[r][i].cpu().numpy(), want[i], "sharded forward")
                grads = [[grad_fn(rng, step[r][i * B:(i + 1) * B], dim) for i in range(S)] for r in range(R)]
                torch.cuda.synchronize()
                sts = W.group_backward(ws, [[torch.from_numpy(g).to(DEV) for g in gr] for gr in grads], scales=[scale] * S,
                                       want_status=True)
                torch.cuda.synchronize()
                for r in range(R):
                    assert sts[r].cpu().numpy().tolist() == w.backward(octx[r], grads[r], scale=[scale] * S), "status"
        for x in ws:
            assert x.status() == (False, False)
        return (signs,) + _read_rows(torch, oracle, shards, w, signs, R)
    finally:
        oracle.set_rsqrt_exact(False)


def train_steps(torch, s, ctx, w, rng, S, B, dim, card, steps, max_ids=1, allow_empty=False, scale=None,
                f32=False, nan_slot=None, skip_slot=None):
    touched = [set() for _ in range(S)]
    for it in range(steps):
        ids, row_off, slot_off = make_batch(rng, S, B, card, max_ids=max_ids, allow_empty=allow_empty)
        got, want, octx = fwd_both(torch, s, ctx, w, ids, row_off, slot_off, B, training=True)
        for i in range(S):
            touched[i].update(w.ctx_signs(octx, i).tolist())
        g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float32 if f32 else np.float16)
        if f32 is False and it == 1:
            g[0, 0, 0] = np.inf  # clamps to 65504 (persia-common lib.rs:163-180)
            g[0, 1, 1] = -np.inf
        if nan_slot is not None and it == nan_slot[0]:
            g[nan_slot[1], B // 2, dim - 1] = np.nan
        grads = [torch.from_numpy(g[i]).to(DEV) for i in range(S)]
        ograds = [g[i] for i in range(S)]
        skip = None
        if skip_slot is not None and it == skip_slot[0]:
            grads[skip_slot[1]] = None
            skip = [int(i == skip_slot[1]) for i in range(S)]
        st = ctx.backward(s, grads, scales=scale, want_status=True).cpu().numpy().tolist()
        ost = w.backward(octx, ograds, scale=scale, skip=skip)
        assert st == ost, (it, st, ost)
    return [np.array(sorted(t), np.uint64) for t in touched]
