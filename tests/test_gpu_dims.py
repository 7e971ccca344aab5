"""GPU: every path that steps a row, and the host tier, at the embedding dims the rest of the suite leaves out.

The kernels branch on dim: vec_group takes VEC 4 only at dim % 4 == 0 and G = 1..32 lanes; below dim 8 the fused
8-element blocks of the row update are empty and every element takes the unfused tail; k_reduce_hot picks 2 or 4
elements per lane and runs 8 column passes at 4096 (the ABI's largest dim); the owner's f16 row store branches on
dim % 8 and dim % 4; the tier moves whole entries of round4(dim + state) floats.  Here dims 1, 2, 3, 5, 7, 9, 4095 and
4096 run with ordinary values (rows in +-0.5, N(0, 1e-2) gradients) through util.EDGE_PATHS against the oracle in
exact-rsqrt mode, and a short parity-over-churn runs the tier at dims 1, 7 and 4095."""
import numpy as np
import pytest

from util import (DEV, EDGE_PATHS, f16_ulp_diff, full_row_off, held_rows, make_batch, pool_model, run_edge_path,
                  same_bits, slot_signs, to_dev_i32, to_dev_ids)

pytestmark = pytest.mark.gpu

# all four optimizers at dims 1, 5, 9 and 4096; SGD and Adagrad at 2, 3, 7 and 4095
CASES = [(d, k) for d in (1, 5, 9, 4096) for k in (0, 1, 2, 3)] + [(d, k) for d in (2, 3, 7, 4095) for k in (0, 1)]


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def _rows(signs, dim):
    return np.random.default_rng(len(signs) + dim).uniform(-0.5, 0.5, (len(signs), dim)).astype(np.float32)


@pytest.mark.parametrize("dtype", [np.float16, np.float32])
@pytest.mark.parametrize("dim,kind", CASES)
def test_every_path_at_dim(torch_cuda, oracle, dim, kind, dtype):
    """Two steps of every path; every seeded entry bit for bit with the oracle."""
    def grad(rng, ids, d):
        return (rng.standard_normal((len(ids), d)) * 1e-2).astype(dtype)
    for p in EDGE_PATHS:
        signs, got, want = run_edge_path(torch_cuda, oracle, p, kind, dim, _rows, grad, steps=2, rng_seed=dim)
        for k in range(signs.size):
            assert same_bits(got[k], want[k]), (p, k, int(signs[k]))


def _entries_match(s, w, signs, what):
    ent, found = s.get_entries(to_dev_ids(signs, DEV))
    ent, found = ent.cpu().numpy(), found.cpu().numpy()
    assert found.all(), what
    for k, sign in enumerate(signs):
        assert same_bits(ent[k], w.get_entry(int(sign))), (what, k, int(sign))


@pytest.mark.parametrize("dim", [1, 7, 4095])
@pytest.mark.parametrize("kind_name,kw", [("ADAM", {"lr": 0.001}), ("ADAGRAD_VW", {"lr": 0.02})])
def test_tier_churn_at_dim(torch_cuda, oracle, kind_name, kw, dim):
    """HBM rows C = 512 over ~4 C keys with a host tier behind them, one eviction check per request: rows move out
    and back.  Outputs match the sample-order model bit for bit (and the oracle: single ids exactly, several within
    1 f16 ulp), and every entry seen equals the unbounded oracle's, wherever it lives."""
    from persia_b200 import shard as SH

    torch = torch_cuda
    kind = getattr(oracle, kind_name)
    C, S, B = 512, 2, 16
    pf = [oracle.index_prefix(g) for g in range(S)]
    oracle.set_rsqrt_exact(True)
    try:
        s = SH.EmbeddingShard(dim, C, 0, tier_rows=1 << 12)
        s.set_optimizer(kind, **kw)
        s.configure()
        s.set_eviction(check_every=1, low_water=C // 2, target_free=C // 2, keep_batches=2)
        ctx = SH.BatchContext(1 << 10, S * B, pf)
        w = oracle.Worker([oracle.SlotCfg(dim, prefix=p) for p in pf], n_ps=1)
        w.configure()
        w.set_optimizer(oracle.Optim(kind, **kw))
        rng = np.random.default_rng(dim)
        seen = set()
        for step in range(24):
            ids, row_off, slot_off = make_batch(rng, S, B, 1000, max_ids=3 if step % 2 else 1)
            ro_dev = to_dev_i32(row_off, DEV) if row_off is not None else None
            got = ctx.forward(s, to_dev_ids(ids, DEV), slot_off, B, row_off=ro_dev, training=True).cpu().numpy()
            ro = row_off if row_off is not None else full_row_off(S, B)
            want, octx = w.forward(ids, ro, B, training=True)
            signs = slot_signs(oracle, ids, slot_off, pf)
            model = pool_model(held_rows(torch, oracle, [s], signs), signs, row_off, B, None, dim=dim)
            one = (np.diff(ro) <= 1).reshape(S, B)
            for i in range(S):
                assert same_bits(got[i], model[i]), step
                assert same_bits(got[i][one[i]], want[i][one[i]]), step
                assert f16_ulp_diff(got[i], want[i]) <= 1, step
                seen.update(w.ctx_signs(octx, i).tolist())
            g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float32 if step % 4 >= 2 else np.float16)
            st = ctx.backward(s, [torch.from_numpy(g[i]).to(DEV) for i in range(S)], want_status=True)
            assert st.cpu().numpy().tolist() == w.backward(octx, [g[i] for i in range(S)]), step
            if step % 8 == 7:
                _entries_match(s, w, np.array(sorted(seen), np.uint64), step)
                assert len(s) == len(seen), (step, len(s), len(seen))
        ts = s.tier_stats()
        assert ts["moved_out"] > 0 and ts["restored"] > 0 and ts["dropped"] == 0 and ts["refused"] == 0, ts
    finally:
        oracle.set_rsqrt_exact(False)
