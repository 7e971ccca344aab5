"""GPU: checkpoint loads on the device (persia_b200/checkpoint.py DeviceLoader over pb_image_*, pb_load.cu).

Every case loads one directory into two fresh tables per dim, one with checkpoint.load_shards (the host decoder, the
model) and one with the device loader, and compares them bit for bit: size, export order and recency, every entry,
counters and host-tier statistics.  Malformed files give decode_list's exception and message."""
import os
import threading

import numpy as np
import pytest

from emb_layouts import reference_layout
from util import to_dev_ids

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ODD = np.array([2**64 - 1, 2**64 - 2, 2**64 - 3], np.uint64)


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


def _tables(dims, capacity=8192, tier_rows=0):
    from persia_b200 import native as N
    from persia_b200.shard import EmbeddingShard

    out = {}
    for d in dims:
        sh = EmbeddingShard(d, capacity, 0, tier_rows=tier_rows)
        sh.set_optimizer(N.OPT_ADAGRAD, lr=0.05, initialization=0.01)
        sh.configure()
        out[d] = sh
    return out


def _snap(sh):
    signs, rec = sh.export_signs()
    ent, found = sh.get_entries(signs)
    return (len(sh), signs.cpu().numpy(), rec.cpu().numpy(), ent.cpu().numpy(), found.cpu().numpy(), sh.counters(),
            sh.tier_stats())


def _same(a, b):
    for ta, tb in zip(a, b):
        if isinstance(ta, np.ndarray):
            assert ta.dtype == tb.dtype and ta.shape == tb.shape
            assert ta.tobytes() == tb.tobytes()
        else:
            assert ta == tb


def _compare(torch, src, dims, r=0, R=1, capacity=8192, tier_rows=0, **kw):
    from persia_b200 import checkpoint as CK

    ref, dev = _tables(dims, capacity, tier_rows), _tables(dims, capacity, tier_rows)
    chunk = kw.pop("chunk", 1 << 20)
    n_ref = CK.load_shards(src, ref, r, R, chunk=chunk)
    n_dev = CK.DeviceLoader(src, dev, r, R, chunk=chunk, **kw).run()
    torch.cuda.synchronize()
    assert n_ref == n_dev
    for d in dims:
        _same(_snap(ref[d]), _snap(dev[d]))
    return ref, dev


def _write(path, shard_images, num_shards=None):
    """A checkpoint directory: shard_images[k] = {file name: bytes} of s{k}."""
    from persia_b200 import checkpoint as CK

    R = num_shards or len(shard_images)
    for k, files in enumerate(shard_images):
        d = os.path.join(path, f"s{k}")
        os.makedirs(d, exist_ok=True)
        for name, img in files.items():
            with open(os.path.join(d, name), "wb") as f:
                f.write(img)
        with open(os.path.join(d, CK.DONE_FILE), "w") as f:
            f.write(CK.done_yaml(R, len(files)))
    with open(os.path.join(path, CK.DONE_FILE), "w") as f:
        f.write(CK.done_yaml(R, 1))
    return str(path)


def _signs(rng, n, odd=False):
    s = np.unique(rng.integers(1, 2**64 - 4, size=n, dtype=np.uint64))
    return np.concatenate([s, ODD]) if odd else s


def _filled(torch, rng, dims, n=600, tier_rows=0, capacity=8192):
    tabs = _tables(dims, capacity, tier_rows)
    for d, sh in tabs.items():
        s = _signs(rng, n, odd=True)
        sh.set_entries(to_dev_ids(s, DEV), torch.from_numpy(rng.standard_normal((s.size, sh.entry_len)).astype(np.float32)).to(DEV))
        sh.lookup(to_dev_ids(s[rng.random(s.size) < 0.3], DEV), training=True)
    return tabs


# ------------------------------------------------------------------------------------------------ writer layout
def test_synchronous_dump_two_dims(torch_cuda, tmp_path):
    from persia_b200 import checkpoint as CK

    rng = np.random.default_rng(1)
    tabs = _filled(torch_cuda, rng, (8, 32))
    CK.dump_shards(str(tmp_path), [tabs[8], tabs[32]])
    _compare(torch_cuda, str(tmp_path), (8, 32))


def test_background_dump_directory(torch_cuda, tmp_path):
    from persia_b200 import checkpoint as CK

    rng = np.random.default_rng(2)
    tabs = _filled(torch_cuda, rng, (8, 32))
    d = CK.BackgroundDumper(str(tmp_path), [tabs[8], tabs[32]], n_parts=5)
    while d.step():
        pass
    _compare(torch_cuda, str(tmp_path), (8, 32))


def test_files_of_zero_and_one_entries(torch_cuda, tmp_path):
    from persia_b200 import checkpoint as CK

    rng = np.random.default_rng(3)
    one = CK.encode_list(np.array([2**64 - 2], np.uint64), rng.standard_normal((1, 16)).astype(np.float32), 8)
    src = _write(tmp_path, [{"a.emb": CK.list_header(0), "b.emb": one, "c.emb": CK.encode_list([], np.zeros((0, 16), np.float32), 8)}])
    _compare(torch_cuda, src, (8,))


@pytest.mark.parametrize("per", [1, 2, 3, 7, 16, 49, 50, 64])
def test_window_sizes(torch_cuda, tmp_path, per):
    """Windows of `per` whole nodes (the last one shorter unless per divides 50) from buffers whose size ends at
    several bytes of a node, forward and newest first (a host tier)."""
    from persia_b200 import checkpoint as CK

    rng = np.random.default_rng(4)
    n, L, nb = 50, 16, 93
    s = _signs(rng, n)
    src = _write(tmp_path, [{"a.emb": CK.encode_list(s, rng.standard_normal((s.size, L)).astype(np.float32), 8)}])
    for tier in ((0, 64) if 32 % per == 0 else (0,)):  # with a tier: HBM (32 rows) fills at a call boundary
        ref = _tables((8,), capacity=32 if tier else 8192, tier_rows=tier)
        CK.load_shards(src, ref, chunk=per)
        want = _snap(ref[8])
        for b in (0, 1, 45, 92):
            dev = _tables((8,), capacity=32 if tier else 8192, tier_rows=tier)
            ld = CK.DeviceLoader(src, dev, chunk=per, buffer_bytes=per * nb + b)
            assert [(lo, hi) for _, _, lo, hi, _ in ld_tasks(ld)] == CK.windows(n, nb, per * nb + b, bool(tier))
            ld.run()
            _same(want, _snap(dev[8]))


def ld_tasks(ld):
    ld._open()
    try:
        return list(ld._tasks)
    finally:
        ld._close()


# ------------------------------------------------------------------------------------------------ reference layouts
@pytest.mark.parametrize("case", ["permuted", "free", "mixed", "markers"])
def test_reference_layouts(torch_cuda, tmp_path, case):
    from persia_b200 import checkpoint as CK

    rng = np.random.default_rng(5)
    n = 700
    s = _signs(rng, n, odd=case == "markers")
    dims = np.full(s.size, 8, np.uint64)
    if case == "mixed":
        dims[rng.random(s.size) < 0.4] = 32
    ent = [rng.standard_normal(2 * int(d)).astype(np.float32) for d in dims]
    files = {}
    for k in range(3):
        pick = np.arange(k, s.size, 3)
        img = reference_layout(s[pick], dims[pick], [ent[i] for i in pick], rng, permute=case != "free",
                               free=pick.size // 10 if case in ("free", "mixed") else 0)
        got = CK.decode_list(img)
        np.testing.assert_array_equal(got[0], s[pick])
        assert CK.writer_layout(len(img), img[:41]) is None
        files[f"replica_0_shard_{k}.emb"] = img
    src = _write(tmp_path, [files])
    _compare(torch_cuda, src, (8, 32))


# ------------------------------------------------------------------------------------------------ re-sharding
@pytest.mark.parametrize("R", [1, 3])
def test_resharding_load(torch_cuda, tmp_path, R):
    from persia_b200 import checkpoint as CK

    rng = np.random.default_rng(6)
    shards = []
    for k in range(2):
        s = _signs(rng, 400, odd=k == 1)
        shards.append({"replica_%d_shard_0.emb" % k: CK.encode_list(s, rng.standard_normal((s.size, 16)).astype(np.float32), 8),
                       "replica_%d_shard_1.emb" % k: reference_layout(
                           s[:50], [32] * 50, list(rng.standard_normal((50, 64)).astype(np.float32)), rng, free=7)})
    src = _write(tmp_path, shards)
    for r in range(R):
        _compare(torch_cuda, src, (8, 32), r, R)


# ------------------------------------------------------------------------------------------------ host tier
@pytest.mark.parametrize("layout", ["writer", "reference"])
def test_host_tier_newest_first(torch_cuda, tmp_path, layout):
    from persia_b200 import checkpoint as CK

    rng = np.random.default_rng(7)
    n, cap = 3072, 1024  # windows and chunks of 1024: the first (newest) fills HBM exactly, the rest go to the tier
    s = np.arange(1, n + 1, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    ent = rng.standard_normal((s.size, 16)).astype(np.float32)
    img = CK.encode_list(s, ent, 8) if layout == "writer" else reference_layout(s, [8] * s.size, list(ent), rng, free=30)
    src = _write(tmp_path, [{"a.emb": img}])
    _, dev = _compare(torch_cuda, src, (8,), capacity=cap, tier_rows=4096, chunk=1024, buffer_bytes=1024 * 93)
    assert dev[8].tier_stats()["host_rows"] == s.size - cap


# ------------------------------------------------------------------------------------------------ malformed files
def _malformed(CK, rng):
    s = _signs(rng, 6)
    ent = rng.standard_normal((6, 16)).astype(np.float32)
    good = CK.encode_list(s, ent, 8)
    nb = 93
    out = {"header": good[:20], "node": good[:28 + 2 * nb + 5], "entry": good[:28 + 2 * nb + 40],
           "trailing": good + b"\0", "len-index": good[:28 + 9], "len-short": good[:28 + 11]}
    head = bytearray(good)
    head[0] = 5  # count 5, six live nodes
    out["count"] = bytes(head)
    ends = bytearray(good)
    ends[28 + 2 * nb:28 + 2 * nb + 4] = np.array([0], "<u4").tobytes()  # node 3 ends the list early
    out["ends"] = bytes(ends)
    cyc = bytearray(good)
    cyc[28 + 3 * nb:28 + 3 * nb + 4] = np.array([2], "<u4").tobytes()  # node 4 -> node 2: a cycle
    out["cycle"] = bytes(cyc)
    free = reference_layout(s, [8] * 6, list(ent), rng, permute=False, free=2)
    # the list runs through a free node: live p2 -> free F -> live p3, and p4 ends it (p5 is live but unlisted)
    b = bytearray(free)
    off, offs, live = 28, [], []
    for i in range(8):
        offs.append(off)
        if free[off + 8]:
            live.append(i)
        off += 9 + (20 + 64 if free[off + 8] else 0)
    f0 = int(np.frombuffer(free[16:20], "<u4")[0]) - 1
    for node, nxt in ((live[2], f0 + 1), (f0, live[3] + 1), (live[4], 0)):
        b[offs[node]:offs[node] + 4] = np.array([nxt], "<u4").tobytes()
    out["unused"] = bytes(b)
    late = bytearray(CK.encode_list(_signs(rng, 40), rng.standard_normal((40, 16)).astype(np.float32), 8))
    late[28 + 30 * nb:28 + 30 * nb + 4] = np.array([40], "<u4").tobytes()  # node 31 skips to node 40
    out["late"] = bytes(late)
    return out


def test_malformed_files_give_decode_list_errors(torch_cuda, tmp_path):
    from persia_b200 import checkpoint as CK

    rng = np.random.default_rng(8)
    for name, img in _malformed(CK, rng).items():
        try:
            CK.decode_list(img)
            raise AssertionError(f"{name}: decode_list accepted it")
        except (ValueError, IndexError) as e:
            want = e
        src = _write(tmp_path / name, [{"a.emb": img}])
        dev = _tables((8,))
        with pytest.raises(type(want)) as got:
            CK.DeviceLoader(src, dev, buffer_bytes=10 * 93).run()
        assert str(got.value) == str(want), name
        if name == "late":  # a streamed file keeps the windows before the malformed one
            assert len(dev[8]) == 30
        else:
            assert len(dev[8]) == 0, name


def test_unknown_dim_and_entry_length(torch_cuda, tmp_path):
    from persia_b200 import checkpoint as CK

    rng = np.random.default_rng(9)
    s = _signs(rng, 20)
    for layout in ("writer", "reference"):
        for dim, L, msg in ((16, 32, "checkpoint holds dim-16 embeddings but no slot has that dim"),
                            (8, 17, r"dim-8 entries of \[17\] floats, the registered optimizer needs 16")):
            ent = rng.standard_normal((s.size, L)).astype(np.float32)
            img = CK.encode_list(s, ent, dim) if layout == "writer" else reference_layout(s, [dim] * s.size, list(ent), rng)
            src = _write(tmp_path / f"{layout}{dim}{L}", [{"a.emb": img}])
            for load in (lambda t: CK.load_shards(src, t), lambda t: CK.DeviceLoader(src, t).run()):
                t = _tables((8,))
                with pytest.raises(RuntimeError, match=msg):
                    load(t)
                assert len(t[8]) == 0


# ------------------------------------------------------------------------------------------------ background
def test_status_rises_and_steps_interleave_with_training(torch_cuda, tmp_path):
    from persia_b200 import checkpoint as CK

    torch = torch_cuda
    rng = np.random.default_rng(10)
    tabs = _filled(torch, rng, (8, 32))
    CK.dump_shards(str(tmp_path), [tabs[8], tabs[32]])
    train = _signs(np.random.default_rng(99), 64)  # signs outside the checkpoint
    grads = torch.from_numpy(rng.standard_normal((train.size, 8)).astype(np.float32)).to(DEV)

    def train_step(t):
        t[8].lookup(to_dev_ids(train, DEV), training=True)
        t[8].update(to_dev_ids(train, DEV), grads)

    ref = _tables((8, 32))
    CK.load_shards(str(tmp_path), ref)
    for _ in range(3):
        train_step(ref)
    dev = _tables((8, 32))
    ld = CK.DeviceLoader(str(tmp_path), dev, buffer_bytes=50 * 93)
    seen = [ld.status()]
    k = 0
    while ld.step():
        seen.append(ld.status())
        if k < 3:
            train_step(dev)
            k += 1
    seen.append(ld.status())
    while k < 3:
        train_step(dev)
        k += 1
    assert seen[-1] == ("Idle", 1.0)
    fr = [f for st, f in seen[:-1]]
    assert all(st == "Loading" for st, _ in seen[:-1]) and fr == sorted(fr) and fr[-1] > fr[0]
    for d in (8, 32):  # (the loaded rows' recency is pb_set_rows', the request number at their insert)
        a, b = _snap(ref[d]), _snap(dev[d])
        assert a[0] == b[0] and a[5] == b[5] and a[6] == b[6]
        order = np.argsort(a[1].view(np.uint64))
        got = b[1].view(np.uint64)
        np.testing.assert_array_equal(np.sort(got), a[1].view(np.uint64)[order])
        ent_b = dict(zip(got.tolist(), b[3]))
        for sg, e in zip(a[1].view(np.uint64).tolist(), a[3]):
            assert ent_b[sg].tobytes() == e.tobytes()


@pytest.fixture()
def core(torch_cuda):
    from persia_b200 import persia_core as PC

    PC.reset()
    os.environ.pop("RANK", None)
    os.environ.pop("WORLD_SIZE", None)
    yield torch_cuda, PC
    PC.reset()


def _surface(PC, dims=(8, 32)):
    pc = PC.install()
    pc.set_embedding_config({"feature_index_prefix_bit": 8, "slots_config": {f"s{d}": {"dim": d} for d in dims}})
    ctx = pc.PersiaCommonContext(10, 0, 1, 0)
    opt = pc.optim.OptimizerBase()
    opt.init_adagrad(0.01, 0.0, 1.0, 0.01, 1e-10, False)
    opt.apply()
    ctx.configure_embedding_parameter_servers(-0.01, 0.01, 1.0, True, 10.0)
    return ctx


def test_background_load_through_persia_core(core, tmp_path):
    torch, PC = core
    from persia_b200 import api

    ctx = _surface(PC)
    rng = np.random.default_rng(11)
    ctx.set_embedding([(int(sg), rng.standard_normal(d).astype(np.float32), rng.random(d).astype(np.float32))
                       for d, n in ((8, 300), (32, 120)) for sg in rng.integers(1, 2**60, size=n, dtype=np.uint64)])
    ctx.dump(str(tmp_path / "ck"), background=False)
    ctx.clear_embeddings()
    assert ctx.get_embedding_size() == [0, 0]
    g = PC._S.groups[8]
    g["lock"].acquire()  # the load's first insert waits for the group: it is surely running
    try:
        ctx.load(str(tmp_path / "ck"), background=True)
        assert ctx.load_status()[0] == "Loading"
        waited = threading.Thread(target=ctx.wait_for_serving)
        waited.start()
        waited.join(0.3)
        assert waited.is_alive()
    finally:
        g["lock"].release()
    ctx.wait_for_emb_loading()
    waited.join(60)
    assert ctx.load_status() == ("Idle", 1.0)
    assert ctx.get_embedding_size() == [300, 120]
    # failure: the reference's text
    (tmp_path / "bad" / "s0").mkdir(parents=True)
    (tmp_path / "bad" / "s0" / "replica_0_shard_0.emb").write_bytes(b"\0" * 20)
    (tmp_path / "bad" / "s0" / "embedding_dump_done").write_text("---\nnum_shards: 1\nnum_internal_shards: 1\n")
    ctx.load(str(tmp_path / "bad"), background=True)
    with pytest.raises(RuntimeError, match=r"^emb dump FAILED for server 0, due to ValueError: truncated checkpoint: header$"):
        ctx.wait_for_emb_loading()
    assert ctx.load_status() == ("Failed", "ValueError: truncated checkpoint: header")
    with pytest.raises(ValueError, match="truncated checkpoint: header"):  # blocking raises what load_shards raises
        ctx.load(str(tmp_path / "bad"), background=False)
    # api: load_embedding(blocking=False) returns before the load is done
    ctx.clear_embeddings()
    ectx = api.EmbeddingCtx.__new__(api.EmbeddingCtx)
    ectx.common_context = ctx
    g["lock"].acquire()
    try:
        ectx.load_embedding(str(tmp_path / "ck"), blocking=False)
        assert ctx.load_status()[0] == "Loading"
    finally:
        g["lock"].release()
    ctx.wait_for_emb_loading()
    assert ctx.get_embedding_size() == [300, 120]


def test_training_launches_unchanged_without_a_load(torch_cuda, tmp_path):
    """A training request issues as many kernel launches after a load has run and closed on its table as before."""
    from persia_b200 import checkpoint as CK
    from persia_b200 import native as N

    lib = N.load()
    rng = np.random.default_rng(12)
    src = _write(tmp_path, [{"a.emb": CK.encode_list(_signs(rng, 300), rng.standard_normal((300, 16)).astype(np.float32), 8),
                             "b.emb": reference_layout(_signs(rng, 40), [8] * 40,
                                                       list(rng.standard_normal((40, 16)).astype(np.float32)), rng, free=3)}])
    t = _tables((8,))[8]
    s = to_dev_ids(_signs(np.random.default_rng(13), 100), DEV)
    g = torch_cuda.zeros((100, 8), device=DEV)

    def step():
        torch_cuda.cuda.synchronize()
        a = lib.pb_launch_count()
        t.lookup(s, training=True)
        t.update(s, g)
        torch_cuda.cuda.synchronize()
        return lib.pb_launch_count() - a

    step()
    before = step()
    CK.DeviceLoader(src, {8: t}).run()
    assert step() == before
