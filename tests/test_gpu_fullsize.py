"""GPU, BASELINE.json configs[1] at full size: 26 Criteo-shaped slots, a 1e8-row dim-64 Adagrad shard (51 GB of
HBM), batch 4096, Zipf(1.05) ids.  The oracle cannot hold 1e8 rows, so parity is anchored in two ways:

* a real training step is replayed on the oracle for exactly the rows the batch touches (the oracle's rows are
  seeded from the GPU's with set_embedding — the reference's own debug loader, lib.rs:433-449), then every touched
  row is compared bit for bit (the gradient sums keep the reference order for every multiplicity);
* size-independent properties: a repeated forward is idempotent and admits nothing, the batched forward equals the
  f16 rounding of the direct lookup, zero gradients leave Adagrad rows untouched (momentum 1), and a batch whose
  samples are permuted produces the same rows when the gradient sums are exact in f32.
"""
import numpy as np
import pytest

from util import to_dev_ids

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROWS, S, B, DIM = 100_000_000, 26, 4096, 64


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    if torch.cuda.get_device_properties(0).total_memory < 70e9:
        pytest.skip("the full-size shard needs an 80 GB-class GPU")
    return torch


@pytest.fixture(scope="module")
def full(torch_cuda):
    from persia_b200 import native as N
    from persia_b200 import shard as pb
    from persia_b200 import workload as W

    card = W.scaled_cardinalities(ROWS, S)
    pf = W.index_prefixes(S)
    s = pb.EmbeddingShard(DIM, ROWS, 0)
    s.set_optimizer(N.OPT_ADAGRAD, lr=0.01, initialization=0.01, eps=1e-10, g_square_momentum=1.0)
    s.configure()
    ctx = pb.BatchContext(S * B, S * B, pf)
    ids = W.make_batches(2, card, B, 6)  # [6, S*B]
    slot_off = [i * B for i in range(S + 1)]
    yield s, ctx, ids, slot_off, pf, card
    ctx.close()
    s.close()


def _oracle_for(oracle, pf):
    w = oracle.Worker([oracle.SlotCfg(DIM, prefix=pf[i]) for i in range(S)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(oracle.ADAGRAD, lr=0.01, init_acc=0.01, eps=1e-10, mom=1.0))
    return w


def _signs(oracle, ids, pf):
    return np.concatenate([oracle.add_prefix(ids[i * B:(i + 1) * B], 8, pf[i]) for i in range(S)])


@pytest.mark.parametrize("which", [0, 1])
def test_full_size_step_matches_oracle(torch_cuda, full, oracle, which):
    torch = torch_cuda
    s, ctx, ids, slot_off, pf, _ = full
    oracle.set_rsqrt_exact(True)
    try:
        rng = np.random.default_rng(17 + which)
        b = ids[which]
        d_ids = to_dev_ids(b, DEV)
        out = ctx.forward(s, d_ids, slot_off, B, training=True)  # admits what is new
        signs = np.unique(_signs(oracle, b, pf))
        ent, found = s.get_entries(to_dev_ids(signs, DEV))
        assert found.all()
        w = _oracle_for(oracle, pf)
        w.set_embedding(signs, ent.cpu().numpy(), DIM)
        want, octx = w.forward(b, np.arange(S * B + 1, dtype=np.uint32), B, training=True)
        got = out.cpu().numpy()
        for i in range(S):
            np.testing.assert_array_equal(got[i].view(np.uint16), want[i].view(np.uint16))
        g = (rng.standard_normal((S, B, DIM)) * 1e-2).astype(np.float16)
        st = ctx.backward(s, [torch.from_numpy(g[i]).to(DEV) for i in range(S)], want_status=True).cpu().numpy()
        assert st.tolist() == w.backward(octx, [g[i] for i in range(S)])
        ent2 = s.get_entries(to_dev_ids(signs, DEV))[0].cpu().numpy()
        ref = np.stack([w.get_entry(int(x)) for x in signs])
        # every sign, whatever its multiplicity (tiny slots repeat one id thousands of times): reference order
        assert ent2.tobytes() == ref.tobytes()
        assert s.counters()["wait_errors"] == 0
    finally:
        oracle.set_rsqrt_exact(False)


def test_full_size_properties(torch_cuda, full, oracle):
    torch = torch_cuda
    s, ctx, ids, slot_off, pf, _ = full
    b = ids[2]
    d_ids = to_dev_ids(b, DEV)
    out1 = ctx.forward(s, d_ids, slot_off, B, training=True).clone()
    size1 = len(s)
    ctx.backward(s, [None] * S)  # add_skipped_gradient for every slot: the pending batch is dropped
    out2 = ctx.forward(s, d_ids, slot_off, B, training=True).clone()
    assert len(s) == size1  # nothing new to admit
    assert torch.equal(out1, out2)
    # batched forward == f16(direct lookup) for one-id samples (pure copy + RNE, mod.rs:547-561)
    signs = _signs(oracle, b, pf)
    rows = s.lookup(to_dev_ids(signs, DEV), training=False)
    assert torch.equal(rows.half().view(S, B, DIM), out2)
    # zero gradients: Adagrad leaves weights and (momentum 1) accumulators as they are
    usigns = np.unique(signs)
    before = s.get_entries(to_dev_ids(usigns, DEV))[0].clone()
    zero = torch.zeros((B, DIM), dtype=torch.float16, device=DEV)
    ctx.backward(s, [zero] * S)
    assert torch.equal(before, s.get_entries(to_dev_ids(usigns, DEV))[0])
    # permuting the samples of a batch changes nothing when the gradient sums are exact (multiples of 2^-10, |.|<=1)
    rng = np.random.default_rng(5)
    b3 = ids[3]
    g = (rng.integers(-8, 9, size=(S, B, DIM)) / 1024.0).astype(np.float16)
    perm = rng.permutation(B)
    b3p = b3.reshape(S, B)[:, perm].reshape(-1)
    gp = g[:, perm]
    us = np.unique(_signs(oracle, b3, pf))
    d_us = to_dev_ids(us, DEV)
    ctx.forward(s, to_dev_ids(b3, DEV), slot_off, B, training=True)
    ctx.backward(s, [None] * S)
    snap = s.get_entries(d_us)[0].clone()

    def step(bb, gg):
        s.set_entries(d_us, snap)
        ctx.forward(s, to_dev_ids(bb, DEV), slot_off, B, training=True)
        ctx.backward(s, [torch.from_numpy(np.ascontiguousarray(gg[i])).to(DEV) for i in range(S)])
        return s.get_entries(d_us)[0].clone()

    assert torch.equal(step(b3, g), step(b3p, gp))
