"""GPU: pooled forward outputs bit for bit against util.pool_model, the sample-order model of the pooled forward.

Every path that pools (k_gather_items on one GPU, its tier-reading instantiation, k_expand_copy / k_expand_pool on the
sharded path and shared feature groups) sums a sample's rows into +0 in f32 in ascending occurrence order, skips
signs without a row, multiplies by f32(1 / f32(sqrt(max(n, 1)))) on sqrt-scaled slots and rounds to f16 (RNE).  The
oracle adds a sample's ids in another order, so it only bounds multi-id outputs; the model pins them.

The inputs are built so that a wrong order or a wrong scale shows, and every test asserts that they do, with numpy
only: rows are either "big" (every element +-2^12, in pairs of signs whose rows cancel exactly) or "small" (magnitudes
in [2^-10, 2^-6), some -0).  A sample mixes pairs and small signs in random order, so its f32 partial sums absorb
small terms into big ones and round differently in any other order; sample lengths include n whose double-rounded
sqrt factor differs from the single-rounded one.  Shapes: dims 1 to 4096 (vec_group's VEC 1 and 4, G = 1..32, the
owner's f16 row store at dim % 8 == 0, % 4 == 0 and otherwise), sample lengths 0..1000 in one batch, a sign repeated 40
times in one sample and present in others, a slot of empty samples, B = 257, 3 and 1 (S * B a multiple of neither 4
nor 256), sqrt scaling on and off, one-id and ragged layouts, training and inference."""
import numpy as np
import pytest

from util import DEV, held_rows, pool_model, same_bits, slot_signs, to_dev_i32, to_dev_ids

pytestmark = pytest.mark.gpu

DIMS = [1, 2, 3, 4, 5, 7, 8, 9, 12, 13, 64, 128, 130, 4095, 4096]
LENGTHS = [0, 1, 2, 3, 31, 32, 33, 100, 1000]
FILL = [3, 4, 5, 6, 7, 17, 18, 21, 24]  # 6, 7, 17, 18, 21, 24: f32(1/f32(sqrt(n))) != f32(1/sqrt(n))
SQRT = [False, True, True]  # slot 2: every sample empty in the ragged layout
N_PAIRS, N_SMALL = 48, 64
HOT = 40  # repeats of one pair's signs inside the length-100 sample
MAX_OCC = 1 << 14
OPT = dict(kind=0, lr=0.1)


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def _double_rounded():
    n = np.arange(2, 1001)
    twice = np.float32(1) / np.sqrt(n.astype(np.float32))
    return n[twice != (1.0 / np.sqrt(n.astype(np.float64))).astype(np.float32)]


DOUBLE_ROUNDED = _double_rounded()  # sample lengths whose sqrt factor the kernels must round twice
PROBE_N = [6, 7, 17, 24]  # lengths of the sqrt-factor probes (in DOUBLE_ROUNDED)


def once_rounded(n):
    """The sqrt factor rounded once, f32(1 / sqrt(n)): what an exact rsqrt would give."""
    return (1.0 / np.sqrt(n.astype(np.float64))).astype(np.float32)


def _probe_value(n):
    """A multiple v of 2^-16 such that n * v is exact in f32 and f16(n v * factor) differs between the twice-rounded
    and the once-rounded sqrt factor of n: a sample of n copies of a sign whose row is v shows which one a kernel used."""
    v = np.arange(1, 1 << 16, dtype=np.float32) * np.float32(2.0**-16)
    acc = np.float32(n) * v
    twice = np.float32(1) / np.sqrt(np.float32(n))
    k = np.flatnonzero((acc * twice).astype(np.float16) != (acc * once_rounded(np.array([n]))[0]).astype(np.float16))
    assert k.size, n
    return v[k[k.size // 2]]


class Pool:
    """The ids a test draws from: N_PAIRS pairs of big signs (P_k, N_k with row(N_k) = -row(P_k)), N_SMALL small signs,
    their unprefixed ids a random permutation (so that sorting by sign is another order), one probe sign per PROBE_N
    length, and fresh ids nobody seeds."""

    def __init__(self, rng, dim):
        n = 2 * N_PAIRS + N_SMALL
        self.ids = (rng.permutation(n) + 1000).astype(np.uint64)
        self.P, self.N, self.small = self.ids[:N_PAIRS], self.ids[N_PAIRS:2 * N_PAIRS], self.ids[2 * N_PAIRS:]
        big = np.where(rng.random((N_PAIRS, dim)) < 0.5, -4096.0, 4096.0).astype(np.float32)
        small = (rng.uniform(2.0**-10, 2.0**-6, (N_SMALL, dim)) * rng.choice([-1, 1], (N_SMALL, dim))).astype(np.float32)
        small[rng.random((N_SMALL, dim)) < 0.05] = -0.0
        self.probe = {n: np.uint64(500 + i) for i, n in enumerate(PROBE_N)}
        self.ids = np.concatenate([self.ids, np.array(list(self.probe.values()), np.uint64)])
        self.emb = np.concatenate([big, -big, small, np.stack([np.full(dim, _probe_value(n)) for n in PROBE_N])])
        self.fresh = np.uint64(1 << 40)

    def absent(self):
        self.fresh += np.uint64(1)
        return self.fresh

    def sample(self, rng, n, hot=False):
        """n ids: pairs and small signs (at least n / 3 of them, one of them sometimes an unseeded id), shuffled."""
        if hot:
            ids = [self.P[0]] * HOT + [self.N[0]] * HOT
        else:
            k = rng.integers(0, N_PAIRS, n // 3)
            ids = list(self.P[k]) + list(self.N[k])
        ids += list(self.small[rng.integers(0, N_SMALL, n - len(ids))])
        if n >= 3 and rng.random() < 0.3:
            ids[-1] = self.absent()
        return [ids[i] for i in rng.permutation(n)]

    def ragged(self, rng, B, lengths=None):
        """Three slots: two of B samples (every LENGTHS entry once when B allows, the rest FILL; the length-100 sample
        holds the hot pair; when B allows, the sqrt-scaled slot 1 holds every probe sign n times in a sample of its
        own) and one of B empty samples.  Returns (ids u64, row_off u32 [3B + 1], slot_off)."""
        samples = []
        for slot in range(2):
            ls = lengths if lengths is not None else list(LENGTHS) + list(rng.choice(FILL, B - len(LENGTHS)))
            ss = [self.sample(rng, n, hot=n == 100) for n in ls]
            if slot == 1 and lengths is None:
                ss[len(LENGTHS):len(LENGTHS) + len(PROBE_N)] = [[q] * n for n, q in self.probe.items()]
            samples += [ss[i] for i in rng.permutation(len(ss))]
        samples += [[]] * B
        for s in samples[:B]:  # the hot pair also occurs in other samples
            if len(s) >= 3:
                s[:2] = [self.P[0], self.N[0]]
                break
        row_off = np.zeros(3 * B + 1, np.uint32)
        row_off[1:] = np.cumsum([len(s) for s in samples])
        ids = np.array([x for s in samples for x in s], np.uint64)
        return ids, row_off, [int(row_off[s * B]) for s in range(4)]

    def one_id(self, rng, B):
        ids = [self.ids[rng.integers(0, self.ids.size)] if rng.random() < 0.9 else self.absent() for _ in range(3 * B)]
        return np.array(ids, np.uint64), None, [s * B for s in range(4)]


class Discrimination:
    """Counts, over a test, the multi-id outputs that the reversed-order and the sorted-order models change, and the
    sqrt-scaled outputs that scaling every row first or a once-rounded sqrt factor change: the test's inputs must let a
    wrong kernel fail."""

    def __init__(self):
        self.multi = self.rev = self.srt = self.per_row = self.factor = self.sqrt_n = 0

    def add(self, rows, signs, row_off, B, sqrt, want):
        cnt = np.diff(row_off.astype(np.int64)).reshape(3, B)
        multi = cnt >= 2
        for what, kw in (("rev", dict(order="reversed")), ("srt", dict(order="sorted")), ("per_row", dict(per_row=True)),
                         ("factor", dict(factor=once_rounded))):
            other = pool_model(rows, signs, row_off, B, sqrt, dim=want.shape[-1], **kw)
            diff = (other.view(np.uint16) != want.view(np.uint16)).any(axis=-1)
            setattr(self, what, getattr(self, what) + int((diff & (multi if what in ("rev", "srt") else True)).sum()))
        self.multi += int(multi.sum())
        self.sqrt_n += int(sum(np.isin(cnt[s], DOUBLE_ROUNDED).sum() for s in range(3) if sqrt[s]))

    def check(self):
        assert self.multi > 0 and self.rev >= self.multi / 2 and self.srt >= self.multi / 2, vars(self)
        assert self.per_row > 0 and self.factor >= len(PROBE_N) and self.sqrt_n > 0, vars(self)


def _seed(torch, oracle, shards, w, pool, signs_of):
    """The pool's rows on their owners and in the oracle, under the signs of every slot."""
    signs = np.concatenate([signs_of(pool.ids, s) for s in range(3)])
    emb = np.concatenate([pool.emb] * 3)
    signs, k = np.unique(signs, return_index=True)
    emb = emb[k]
    R = len(shards)
    owner = oracle.shard_of(signs, R) if R > 1 else np.zeros(signs.size, np.uint32)
    for r, s in enumerate(shards):
        m = owner == r
        if m.any():
            s.set_entries(to_dev_ids(signs[m], DEV), torch.from_numpy(np.ascontiguousarray(emb[m])).to(DEV))
    w.set_embedding(signs, emb, pool.emb.shape[1])
    torch.cuda.synchronize()
    return signs


def _compare(got, want, model, row_off, B, what):
    """got bit for bit with the model; the oracle bit for bit where a sample holds at most two ids (their sum does
    not depend on the order).  Longer samples only get a loose sanity bound against the oracle (n^2 * 2^-12, which at
    n = 1000 exceeds any output here): the model assertion is the check."""
    assert same_bits(got, model), what
    cnt = np.ones(3 * B, np.int64) if row_off is None else np.diff(row_off.astype(np.int64))
    cnt = cnt.reshape(3, B)
    few = cnt <= 2
    assert same_bits(got[few], want[few]), what
    bound = (cnt[~few].astype(np.float64) ** 2 * 2.0**-12)[:, None]
    assert (np.abs(got[~few].astype(np.float64) - want[~few].astype(np.float64)) <= bound).all(), what


def _batches(pool, rng, layout):
    for B in (257, 3, 1):
        if layout == "one":
            yield B, pool.one_id(rng, B)
        else:
            yield B, pool.ragged(rng, B, None if B == 257 else list(rng.choice(LENGTHS, B)))


# ---- a. pb_forward on one GPU -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", DIMS)
def test_pooled_forward_one_gpu(torch_cuda, oracle, dim):
    """k_gather_items, one-id and ragged, inference then training (rows read after the training forward: it admits
    the unseeded ids and steps nothing)."""
    from persia_b200 import shard as SH

    torch = torch_cuda
    rng = np.random.default_rng(dim)
    pool = Pool(rng, dim)
    pf = [oracle.index_prefix(g) for g in range(3)]
    s = SH.EmbeddingShard(dim, 1 << 12, 0)
    s.set_optimizer(**OPT)
    s.configure()
    ctx = SH.BatchContext(MAX_OCC, 3 * 257, pf, SQRT)
    w = oracle.Worker([oracle.SlotCfg(dim, sqrt_scaling=SQRT[i], prefix=pf[i]) for i in range(3)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1))
    _seed(torch, oracle, [s], w, pool, lambda ids, i: oracle.add_prefix(ids, 8, pf[i]))
    disc = Discrimination()
    for training in (False, True):
        for layout in ("one", "ragged"):
            for B, (ids, row_off, slot_off) in _batches(pool, rng, layout):
                ro = to_dev_i32(row_off, DEV) if row_off is not None else None
                got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=ro, training=training).cpu().numpy()
                signs = slot_signs(oracle, ids, slot_off, pf)
                rows = held_rows(torch, oracle, [s], signs)
                model = pool_model(rows, signs, row_off, B, SQRT, dim=dim)
                want, _ = w.forward(ids, row_off if row_off is not None else np.arange(3 * B + 1, dtype=np.uint32), B,
                                    training=training)
                _compare(got, np.stack(want), model, row_off, B, (training, layout, B))
                if row_off is not None:
                    disc.add(rows, signs, row_off, B, SQRT, model)
    assert len(s) == w.ps_len(0)
    disc.check()


# ---- b. inference with a host tier: k_gather_items<TIER> ---------------------------------------------------------------
@pytest.mark.parametrize("dim", [1, 3, 8, 13, 130, 4096])
def test_pooled_forward_tier(torch_cuda, oracle, dim):
    """An HBM table of 96 rows with a host tier behind it: the seeded rows that HBM has no room for are stored in the
    tier, so a batch reads HBM-held, tier-held and absent signs.  Inference reads the tier in place."""
    from persia_b200 import shard as SH

    torch = torch_cuda
    rng = np.random.default_rng(100 + dim)
    pool = Pool(rng, dim)
    pf = [oracle.index_prefix(g) for g in range(3)]
    s = SH.EmbeddingShard(dim, 96, 0, tier_rows=1 << 10)
    s.set_optimizer(**OPT)
    s.configure()
    ctx = SH.BatchContext(MAX_OCC, 3 * 257, pf, SQRT)
    w = oracle.Worker([oracle.SlotCfg(dim, sqrt_scaling=SQRT[i], prefix=pf[i]) for i in range(3)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1))
    seeded = _seed(torch, oracle, [s], w, pool, lambda ids, i: oracle.add_prefix(ids, 8, pf[i]))
    tier = s._export_table(s.host_tier.h)[0].cpu().numpy().view(np.uint64)
    assert 0 < tier.size < seeded.size and len(s) == seeded.size
    disc = Discrimination()
    for layout in ("one", "ragged"):
        for B, (ids, row_off, slot_off) in _batches(pool, rng, layout):
            ro = to_dev_i32(row_off, DEV) if row_off is not None else None
            got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=ro, training=False).cpu().numpy()
            signs = slot_signs(oracle, ids, slot_off, pf)
            rows = held_rows(torch, oracle, [s], signs)
            if B == 257:
                in_tier, have = np.isin(signs, tier), np.isin(signs, np.array(list(rows), np.uint64))
                assert in_tier.any() and (have & ~in_tier).any() and not have.all()  # tier, HBM and absent signs
            model = pool_model(rows, signs, row_off, B, SQRT, dim=dim)
            want, _ = w.forward(ids, row_off if row_off is not None else np.arange(3 * B + 1, dtype=np.uint32), B,
                                training=False)
            _compare(got, np.stack(want), model, row_off, B, (layout, B))
            if row_off is not None:
                disc.add(rows, signs, row_off, B, SQRT, model)
    assert s.tier_stats()["restored"] == 0 and len(s) == seeded.size
    disc.check()


# ---- c, d. sharded virtual ranks and shared feature groups --------------------------------------------------------------
def _sharded(torch, oracle, R, dim, groups, rows_f32, layouts, seed):
    from persia_b200.worker import ShardedEmbeddingWorker as W

    rng = np.random.default_rng(seed)
    pool = Pool(rng, dim)
    pf = [oracle.index_prefix(g) for g in groups]
    ws = W.local_group(R, 3, dim, pf, 1 << 12, cap=1024, optimizer=OPT, max_batch=257, sqrt_scaling=SQRT,
                       rows_f32=rows_f32, max_ids_per_sample=MAX_OCC // (3 * 257))
    w = oracle.Worker([oracle.SlotCfg(dim, sqrt_scaling=SQRT[i], prefix=pf[i]) for i in range(3)], n_ps=R)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1))
    shards = [x.shard for x in ws]
    for x in shards:  # table storage is allocated on first use, with a device-wide sync: not while a peer waits
        x.get_entries(torch.zeros(1, dtype=torch.int64, device=DEV))
    _seed(torch, oracle, shards, w, pool, lambda ids, i: oracle.add_prefix(ids, 8, pf[i]))
    disc = Discrimination()
    for training in (False, True):
        for layout in layouts:
            for B in (257, 3, 1):
                step = [(pool.one_id(rng, B) if layout == "one" else
                         pool.ragged(rng, B, None if B == 257 else list(rng.choice(LENGTHS, B)))) for _ in range(R)]
                torch.cuda.synchronize()
                outs = W.group_forward(ws, [to_dev_ids(b[0], DEV) for b in step], B, training=training,
                                       row_offs=[to_dev_i32(b[1], DEV) for b in step] if layout != "one" else None,
                                       slot_occ_offs=[b[2] for b in step])
                torch.cuda.synchronize()
                signs = [slot_signs(oracle, b[0], b[2], pf) for b in step]
                rows = held_rows(torch, oracle, shards, np.concatenate(signs))
                for r, (ids, row_off, slot_off) in enumerate(step):
                    model = pool_model(rows, signs[r], row_off, B, SQRT, dim=dim)
                    want, _ = w.forward(ids, row_off if row_off is not None else np.arange(3 * B + 1, dtype=np.uint32),
                                        B, training=training)
                    _compare(outs[r].cpu().numpy(), np.stack(want), model, row_off, B, (training, layout, B, r))
                    if row_off is not None:
                        disc.add(rows, signs[r], row_off, B, SQRT, model)
    for x in ws:
        assert x.status() == (False, False)
    if "ragged" in layouts:
        disc.check()


@pytest.mark.parametrize("R,dim", [(2, 1), (2, 13), (2, 4096), (3, 12), (3, 64), (8, 5), (8, 128)])
def test_pooled_forward_sharded_f32_rows(torch_cuda, oracle, R, dim):
    """f32 row exchange: k_expand_pool sums the received rows of ragged samples and copies one-id ones."""
    _sharded(torch_cuda, oracle, R, dim, [0, 1, 2], True, ("one", "ragged"), 10 * R + dim)


@pytest.mark.parametrize("R,dim", [(2, 64), (2, 13), (3, 8), (3, 12), (8, 4096), (8, 7)])
def test_pooled_forward_sharded_f16_rows(torch_cuda, oracle, R, dim):
    """f16 row exchange, one id per sample: the owner stores f16(0 + row) (dim % 8, % 4 and other branches), the
    requester copies it (k_expand_copy at dim % 8 == 0, k_expand_pool's copy branch otherwise)."""
    _sharded(torch_cuda, oracle, R, dim, [0, 1, 2], False, ("one",), 20 * R + dim)


@pytest.mark.parametrize("dim", [3, 64])
def test_pooled_forward_shared_group(torch_cuda, oracle, dim):
    """R = 2, slots 0 and 1 in one feature group (the same signs in both), f32 rows."""
    _sharded(torch_cuda, oracle, 2, dim, [0, 0, 1], True, ("one", "ragged"), 30 + dim)
