"""CPU: util.pool_model, the sample-order model of the pooled forward that the GPU tests hold the kernels to bit for bit,
against the oracle's forward (which adds a sample's ids in another order) and against util.pool_lists."""
import numpy as np

from util import f16_ulp_diff, pool_lists, pool_model, same_bits, slot_signs


def test_pool_model_against_oracle(oracle):
    """Three slots (sqrt off, on, on) of samples holding 0..40 ids over seeded rows in +-0.5, some signs absent (an
    inference miss): within 1 f16 ulp of the oracle, and bit for bit where a sample holds at most two ids (the sum of
    two does not depend on the order); bit for bit with
    pool_lists."""
    rng = np.random.default_rng(0)
    dim, B, S, card = 13, 200, 3, 400
    sqrt = [False, True, True]
    pf = [oracle.index_prefix(g) for g in range(S)]
    counts = rng.choice([0, 1, 2, 3, 5, 17, 40], size=S * B)
    row_off = np.zeros(S * B + 1, np.uint32)
    row_off[1:] = np.cumsum(counts)
    ids = rng.integers(0, card, size=int(row_off[-1]), dtype=np.uint64)
    slot_off = [int(row_off[s * B]) for s in range(S + 1)]
    signs = slot_signs(oracle, ids, slot_off, pf)
    held = np.unique(signs)
    held = held[rng.random(held.size) < 0.9]  # the rest have no row
    emb = rng.uniform(-0.5, 0.5, (held.size, dim)).astype(np.float32)
    w = oracle.Worker([oracle.SlotCfg(dim, sqrt_scaling=sqrt[s], prefix=pf[s]) for s in range(S)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.SGD, lr=0.1))
    w.set_embedding(held, emb, dim)
    want, _ = w.forward(ids, row_off, B, training=False)
    rows = {int(x): emb[k] for k, x in enumerate(held)}
    got = pool_model(rows, signs, row_off, B, sqrt)
    assert got.shape == (S, B, dim) and got.dtype == np.float16
    few = (counts <= 2).reshape(S, B)
    for s in range(S):
        assert f16_ulp_diff(got[s], want[s]) <= 1, s
        assert same_bits(got[s][few[s]], want[s][few[s]]), s
        table = np.concatenate([emb, np.zeros((1, dim), np.float32)])
        k = np.searchsorted(held, signs)
        k[(k >= held.size) | (held[np.minimum(k, held.size - 1)] != signs)] = held.size
        lists = [[int(x) for x in k[row_off[s * B + b]:row_off[s * B + b + 1]] if x < held.size] for b in range(B)]
        # pool_lists takes n from the ids it is given: only the samples whose every sign has a row
        full = np.diff(row_off[s * B:(s + 1) * B + 1]) == np.array([len(x) for x in lists])
        assert same_bits(got[s][full], pool_lists(table, lists, sqrt[s])[full]), s
    assert (few & (counts == 2).reshape(S, B)).any() and (counts > 2).any()
    # one id per sample: f16(0 + row)
    one = slot_signs(oracle, ids[:S * B], [s * B for s in range(S + 1)], pf)
    want1, _ = w.forward(ids[:S * B], np.arange(S * B + 1, dtype=np.uint32), B, training=False)
    got1 = pool_model(rows, one, None, B, sqrt, dim=dim)
    for s in range(S):
        assert same_bits(got1[s], want1[s]), s
