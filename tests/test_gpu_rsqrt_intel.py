"""GPU: Adagrad's intel rsqrt mode (EmbeddingShard.set_rsqrt("intel"), pb_table_set_rsqrt) against the CPU oracle in
table mode (tests/rsqrt_oracle.py), bit for bit with NaN matching NaN, on every path that steps a row.

The table mode reproduces the reference's golden vectors on any host, so these tests do not depend on the CPU that runs
them.  Covered: the golden vectors through pb_update; both Adagrad kinds at dims with no fused lanes (1, 7), only fused
lanes (8, 64, 96, 128, 256) and a tail (12, 130; 130 and 256 take the owners' striding kernel) on the local batched step
(cold, warm and hot items), pb_update, raw slots, R = 2 and 4 virtual ranks, a shared feature group and a sharded raw
slot; batches of 8192 samples (k_reduce_hot_short); a tier-held row stepped in place; the special inputs of the
approximation; a captured, replayed backward; tables never switched or switched back (today's bits); persia_core with
PERSIA_B200_ADAGRAD_RSQRT=intel."""
import numpy as np
import pytest

import rsqrt_oracle as RO
from test_gpu_hot_short import EDGES, MANY, _one_id
from test_gpu_reduce_boundaries import HYPER, _check, _run, _train
from test_oracle_golden import ADAGRAD_GOLD, ADAGRAD_VW_GOLD, GRADS, INIT
from util import DEV, fwd_both, pair, run_edge_path, same_bits, to_dev_ids

pytestmark = pytest.mark.gpu

ADAGRAD, ADAGRAD_VW = 1, 2
DIMS = [1, 7, 8, 12, 64, 96, 128, 130, 256]
PATHS = ("batch", "direct", "raw", "shard2", "shard4", "group2", "sraw2")
LOCAL = ("batch", "direct", "raw")
OPT = {ADAGRAD: dict(lr=0.01, init_acc=0.01, eps=1e-10), ADAGRAD_VW: dict(lr=0.02, mom=0.9, init_acc=0.1, eps=1e-8)}


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


@pytest.fixture(scope="module")
def pb(torch_cuda):
    from persia_b200 import shard

    return shard


@pytest.fixture
def table_oracle(monkeypatch, oracle):
    """The oracle in table mode; the shared helpers' requests for its exact mode are ignored."""
    with RO.table_mode(oracle):
        monkeypatch.setattr(oracle, "set_rsqrt_exact", lambda on: None)
        yield oracle


def _intel_shards(monkeypatch, via_worker=False):
    """Every shard the helpers create steps in intel mode: set right after its optimizer, or (via_worker) passed to the
    sharded workers that create them."""
    from persia_b200 import shard as SH
    from persia_b200.worker import ShardedEmbeddingWorker as W

    if via_worker:
        init = W.__init__

        def worker_init(self, *a, **k):
            k.setdefault("rsqrt", "intel")
            init(self, *a, **k)

        monkeypatch.setattr(W, "__init__", worker_init)
        return
    set_opt = SH.EmbeddingShard.set_optimizer

    def set_optimizer(self, *a, **k):
        set_opt(self, *a, **k)
        self.set_rsqrt("intel")

    monkeypatch.setattr(SH.EmbeddingShard, "set_optimizer", set_optimizer)


def _rows(signs, dim):
    return np.random.default_rng(len(signs) + dim).uniform(-0.5, 0.5, (len(signs), dim)).astype(np.float32)


def _grad(dtype):
    return lambda rng, ids, d: (rng.standard_normal((len(ids), d)) * 1e-2).astype(dtype)


def _opt_names(o):
    ren = {"mom": "g_square_momentum", "init_acc": "initialization"}
    return {ren.get(k, k): v for k, v in o.items()}


@pytest.mark.parametrize("kind,gold", [(ADAGRAD, ADAGRAD_GOLD), (ADAGRAD_VW, ADAGRAD_VW_GOLD)])
def test_golden_vectors_through_pb_update(torch_cuda, pb, oracle, kind, gold):
    """persia-common/src/optim.rs:362-445: dim 12 (8 fused lanes and a tail of 4), three steps."""
    torch = torch_cuda
    o = dict(lr=0.01, wd=0.0, mom=1.0, init_acc=0.01, eps=1e-10)
    s = pb.EmbeddingShard(12, 64, 0)
    s.set_optimizer(kind, **_opt_names(o))
    s.set_rsqrt("intel")
    s.configure()
    sign = np.array([12345], np.uint64)
    ent = oracle.Optim(kind, **o).new_entry(np.array(INIT, np.float32))
    s.set_entries(to_dev_ids(sign, DEV), torch.from_numpy(ent[None, :]).to(DEV))
    for g in GRADS:
        s.update(to_dev_ids(sign, DEV), torch.tensor([g], dtype=torch.float32, device=DEV))
    got = s.get_entries(to_dev_ids(sign, DEV))[0].cpu().numpy()[0]
    assert got.tobytes() == np.array(gold, np.float32).tobytes()


@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("kind", [ADAGRAD, ADAGRAD_VW])
@pytest.mark.parametrize("dim", DIMS)
def test_every_path(torch_cuda, table_oracle, monkeypatch, dim, kind, path):
    """Three steps; every seeded entry bit for bit (outputs and statuses are checked by run_edge_path)."""
    _intel_shards(monkeypatch, via_worker=path not in LOCAL)
    dtype = np.float32 if dim in (7, 96, 256) else np.float16
    signs, got, want = run_edge_path(torch_cuda, table_oracle, path, kind, dim, _rows, _grad(dtype), opt=OPT[kind],
                                     steps=3, rng_seed=dim + 10 * kind)
    for k in range(signs.size):
        assert same_bits(got[k], want[k]), (k, int(signs[k]))


@pytest.mark.parametrize("kind", [ADAGRAD, ADAGRAD_VW])
@pytest.mark.parametrize("dim", [64, 130])
def test_hot_short_batches(torch_cuda, pb, table_oracle, monkeypatch, dim, kind):
    """Slots of 8192 samples with items of 33..257 occurrences: k_reduce_hot, k_reduce_hot_short, then k_step_hot."""
    _intel_shards(monkeypatch)
    _run(torch_cuda, pb, table_oracle, _one_id(EDGES + MANY, 2, 8192), 2, 8192, dim, kind, steps=3)


@pytest.mark.parametrize("kind", [ADAGRAD, ADAGRAD_VW])
@pytest.mark.parametrize("dim", [12, 130])
def test_tier_held_rows_stepped_in_place(torch_cuda, pb, table_oracle, monkeypatch, dim, kind):
    """256 HBM rows over 1000 keys with a host tier behind them and an eviction check per request (at most 32 new rows
    a request, so that none is refused), then pb_update of every key seen: most rows are stepped where the tier holds
    them."""
    torch = torch_cuda
    _intel_shards(monkeypatch)
    oracle = table_oracle
    o = OPT[kind]
    pf = oracle.index_prefix(0)
    s = pb.EmbeddingShard(dim, 256, 0, tier_rows=1 << 12)
    s.set_optimizer(kind, **_opt_names(o))
    s.configure()
    s.set_eviction(check_every=1, low_water=128, target_free=128, keep_batches=2)
    ctx = pb.BatchContext(32, 32, [pf])
    w = oracle.Worker([oracle.SlotCfg(dim, prefix=pf)], n_ps=1)
    w.configure()
    w.set_optimizer(oracle.Optim(kind, **o))
    rng = np.random.default_rng(dim + kind)
    seen = set()
    for _ in range(48):
        ids = rng.integers(0, 1000, size=32, dtype=np.uint64)
        _, _, octx = fwd_both(torch, s, ctx, w, ids, None, [0, 32], 32)
        g = (rng.standard_normal((32, dim)) * 1e-2).astype(np.float16)
        ctx.backward(s, [torch.from_numpy(g).to(DEV)])
        w.backward(octx, [g])
        seen.update(oracle.add_prefix(ids, 8, pf).tolist())
    signs = np.array(sorted(seen), np.uint64)
    torch.cuda.synchronize()
    assert s.tier_stats()["host_rows"] > signs.size // 2  # most of them live in the tier now
    assert s.counters()["capacity_refused"] == 0
    for _ in range(2):
        g = (rng.standard_normal((signs.size, dim)) * 1e-2).astype(np.float32)
        s.update(to_dev_ids(signs, DEV), torch.from_numpy(g).to(DEV))
        w.ps_update(0, signs, np.full(signs.size, dim, np.uint32), g)
    ent, found = s.get_entries(to_dev_ids(signs, DEV))
    ent, found = ent.cpu().numpy(), found.cpu().numpy()
    assert found.all()
    for k, sign in enumerate(signs):
        assert same_bits(ent[k], w.get_entry(int(sign))), (k, int(sign))


def _const_rows(v):
    return lambda signs, dim: np.full((len(signs), dim), v, np.float32)


SPECIALS = {
    # s + eps == 0: rsqrt +inf, the step NaN or +-inf, then the weight bound
    "zero_state": (dict(init_acc=0.0, eps=0.0), _grad(np.float16)),
    # s == +inf: rsqrt +0
    "inf_state": (dict(init_acc=float("inf")), _grad(np.float16)),
    # s + eps denormal: the table gives +inf where exact 1/sqrt is finite
    "denormal_state": (dict(init_acc=1e-40, eps=0.0), _grad(np.float16)),
    # +-65504 f16 gradients (g^2 overflows the state to +inf after one step)
    "f16_max_grad": (dict(), lambda rng, ids, d: np.where(rng.random((len(ids), d)) < 0.5, 65504.0, -65504.0)
                     .astype(np.float16)),
    # f32 gradients whose squares overflow
    "f32_huge_grad": (dict(), lambda rng, ids, d: (rng.standard_normal((len(ids), d)) * 1e30).astype(np.float32)),
}


@pytest.mark.parametrize("path", ["batch", "direct", "shard2", "group2"])
@pytest.mark.parametrize("kind", [ADAGRAD, ADAGRAD_VW])
@pytest.mark.parametrize("case", list(SPECIALS))
def test_special_inputs(torch_cuda, table_oracle, monkeypatch, case, kind, path):
    _intel_shards(monkeypatch, via_worker=path not in LOCAL)
    opt, grad = SPECIALS[case]
    o = {**OPT[kind], **opt}
    for dim in (12, 130):
        signs, got, want = run_edge_path(torch_cuda, table_oracle, path, kind, dim, _const_rows(0.25), grad, opt=o,
                                         hyper=dict(wb=1e30), steps=2, rng_seed=dim)
        for k in range(signs.size):
            assert same_bits(got[k], want[k]), (dim, k, int(signs[k]))


@pytest.mark.parametrize("kind", [ADAGRAD, ADAGRAD_VW])
def test_captured_backward_replayed(torch_cuda, pb, table_oracle, monkeypatch, kind):
    torch = torch_cuda
    _intel_shards(monkeypatch)
    oracle = table_oracle
    S, B, dim = 2, 8192, 128
    rng = np.random.default_rng(90 + kind)
    s, ctx, w, pf = pair(pb, oracle, S, dim, kind, cap=1 << 16, optim_kw=OPT[kind], hyper_kw=HYPER, max_occ=S * B)
    make = _one_id(EDGES + MANY, S, B)
    touched = _train(torch, s, ctx, w, oracle, pf, make(rng), B, dim, rng, kind)
    for _ in range(2):  # a graph per batch: the forward is eager, the captured backward replayed once
        ids = np.concatenate([x[0] for x in make(rng)])
        _, _, octx = fwd_both(torch, s, ctx, w, ids, None, [0, B, 2 * B], B, training=True)
        touched += [w.ctx_signs(octx, i) for i in range(S)]
        g = (rng.standard_normal((S, B, dim)) * 1e-2).astype(np.float16)
        grads = [torch.from_numpy(g[i]).to(DEV) for i in range(S)]
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ctx.backward(s, grads)
        graph.replay()
        torch.cuda.synchronize()
        w.backward(octx, [g[i] for i in range(S)])
    _check(torch, s, w, [np.unique(np.concatenate(touched))])


@pytest.mark.parametrize("switch", ["never", "back"])
@pytest.mark.parametrize("path", ["batch", "direct", "shard2"])
@pytest.mark.parametrize("kind", [ADAGRAD, ADAGRAD_VW])
def test_exact_mode_keeps_todays_bits(torch_cuda, oracle, monkeypatch, kind, path, switch):
    """A table never switched, and one switched to intel and back before any step, against the oracle's exact mode."""
    from persia_b200 import shard as SH

    if switch == "back":
        set_opt = SH.EmbeddingShard.set_optimizer

        def set_optimizer(self, *a, **k):
            set_opt(self, *a, **k)
            self.set_rsqrt("intel")
            self.set_rsqrt("exact")

        monkeypatch.setattr(SH.EmbeddingShard, "set_optimizer", set_optimizer)
    for dim in (12, 130):
        signs, got, want = run_edge_path(torch_cuda, oracle, path, kind, dim, _rows, _grad(np.float16), opt=OPT[kind],
                                         steps=2, rng_seed=dim)
        for k in range(signs.size):
            assert same_bits(got[k], want[k]), (dim, k, int(signs[k]))


def test_persia_core_env(torch_cuda, table_oracle, monkeypatch):
    """The persia_core surface with PERSIA_B200_ADAGRAD_RSQRT=intel, one process on one GPU, Adagrad: every entry of
    every slot bit for bit with the oracle in table mode."""
    import torch
    import torch.utils.dlpack as dl

    from persia_b200 import persia_core as impl
    from persia_b200.persia_core import _S
    from test_gpu_persia_core import CFG, KEYS, _batch, _csr

    oracle = table_oracle
    monkeypatch.setenv("PERSIA_B200_ADAGRAD_RSQRT", "intel")
    impl.reset()
    pc = impl.install()
    try:
        pc.set_embedding_config(CFG)
        ctx = pc.PersiaCommonContext(10, 0, 1, 0)
        opt = pc.optim.OptimizerBase()
        opt.init_adagrad(0.01, 0.0, 1.0, 0.01, 1e-10)
        opt.apply()
        assert _S.rsqrt == "intel"
        ctx.configure_embedding_parameter_servers(-0.01, 0.01, 1.0, True, 10.0)
        bwd = pc.backward.Backward(8)
        from persia_b200.persia_core import parse_embedding_config

        _, slots = parse_embedding_config(CFG)
        ws = {}
        for dim in sorted({s.dim for s in slots}):
            part = [s for s in slots if s.dim == dim]
            w = oracle.Worker([oracle.SlotCfg(dim, sqrt_scaling=s.sqrt_scaling, prefix=s.index_prefix,
                                              hs_rounds=s.hash_stack_rounds, hs_size=s.hash_stack_embedding_size)
                               for s in part], n_ps=1)
            w.configure(-0.01, 0.01, 1.0, True, 10.0)
            w.set_optimizer(oracle.Optim(oracle.ADAGRAD, lr=0.01, wd=0.0, mom=1.0, init_acc=0.01, eps=1e-10))
            ws[dim] = (w, [s.name for s in part])
        rng = np.random.default_rng(5)
        B = 96
        for step in range(4):
            b, lil = _batch(pc, rng, B)
            tb = ctx.get_embedding_from_data(b, 0)
            keep, xs = [], {}
            for e in tb.consume_all_id_type_feature_embedding_tensors():
                t = e.get_sum_embedding()
                keep.append(t)
                x = dl.from_dlpack(t.dlpack)
                x.requires_grad = True
                xs[t.name] = x
            octx = {}
            for dim, (w, names) in ws.items():
                ids, off = _csr([lil[n] for n in names], B)
                _, octx[dim] = w.forward(ids, off, B, training=True)
            scale = 128.0
            # a loss linear in the embeddings: its gradients do not depend on the forward's values
            loss = sum((x.float() * (i + 1)).sum() for i, x in enumerate(xs.values())) * scale * 1e-3
            loss.backward()
            gb = tb.create_gradient_batch()
            for n, x in xs.items():
                gb.add_gradient(n, x.grad.data_ptr(), list(x.grad.shape), True, scale)
            torch.cuda.synchronize()
            bwd.update_id_type_feature_gradient_batched(gb)
            for dim, (w, names) in ws.items():
                w.backward(octx[dim], [xs[n].grad.cpu().numpy() for n in names], scale=[scale] * len(names))
        torch.cuda.synchronize()
        for dim, (w, names) in ws.items():
            sh = _S.groups[dim]["shard"]
            for n in names:
                signs = oracle.add_prefix(np.arange(KEYS[n], dtype=np.uint64), 8, _S.by_name[n].index_prefix)
                ent, found = sh.get_entries(to_dev_ids(signs, DEV))
                ent, found = ent.cpu().numpy(), found.cpu().numpy()
                for k, s in enumerate(signs):
                    ref = w.get_entry(int(s))
                    assert (ref is not None) == bool(found[k])
                    if ref is not None:
                        assert same_bits(ent[k], ref), (n, k)
        del ws, w
    finally:
        impl.reset()
