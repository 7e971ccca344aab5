"""GPU: incremental-update packets applied on the device (persia_core._apply_packet_file over pb_image_packet, pb_load.cu)
against the host path (persia_core._apply_incremental of incremental.decode_packet), which is the reference here.

Every case builds two identical sets of tables, applies the same packet files, one set through each path, and then
requires identical export_signs (signs and recency), identical entry bytes and equal dropped counts; malformed packets
must raise decode_packet's error and leave the tables as they were, and a bad dim or entry length the same error after
the same partial application."""
import os
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
U64 = np.uint64
SGD, ADAGRAD, ADAM = 0, 1, 3


@pytest.fixture(scope="module")
def torch_cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.fail("GPU tests need a CUDA device (there is no CPU fallback)")
    return torch


@pytest.fixture()
def env(torch_cuda):
    from persia_b200 import incremental as INC
    from persia_b200 import persia_core as PC
    from persia_b200 import shard as SH

    made = []

    def tables(spec, cap=1 << 12, tier=0):
        """{dim: group} of fresh tables: spec {dim: optimizer kind}."""
        out = {}
        for dim, kind in spec.items():
            sh = SH.EmbeddingShard(dim, cap, 0, tier_rows=tier)
            sh.set_optimizer(kind, lr=0.01)
            sh.configure()
            made.append(sh)
            out[dim] = {"shard": sh, "lock": threading.RLock(), "device": 0}
        return out

    yield torch_cuda, INC, PC, tables
    torch_cuda.cuda.synchronize()
    for sh in made:
        sh.close()


def _state(torch, groups):
    """{dim: (signs, recency, entry bytes)} of every entry held, HBM and tier."""
    torch.cuda.synchronize()
    out = {}
    for dim, g in sorted(groups.items()):
        sh = g["shard"]
        signs, rec = sh.export_signs()
        ent = sh.get_entries(signs)[0] if signs.numel() else torch.zeros((0, sh.entry_len))
        out[dim] = (signs.cpu().numpy().tolist(), rec.cpu().numpy().tolist(), ent.cpu().numpy().tobytes())
    return out


def _write(tmp_path, name, data):
    path = os.path.join(str(tmp_path), name)
    with open(path, "wb") as f:
        f.write(data)
    return path


def _entries(rng, n, L):
    return rng.standard_normal((n, L)).astype(np.float32)


def _signs(rng, n):
    return np.unique(rng.integers(1, 1 << 63, size=2 * n, dtype=np.int64).astype(U64))[:n]


def _apply_both(env, paths, host, dev, chunk=None):
    """Each file through both paths; returns the dropped counts, equal on both."""
    _, INC, PC, _ = env
    drops = []
    for p in paths:
        with open(p, "rb") as f:
            signs, dims, ent, _ = INC.decode_packet(f.read())
        a = PC._apply_incremental(signs, dims, ent, groups=host)
        b, n = PC._apply_packet_file(p, groups=dev) if chunk is None else PC._apply_packet_file(p, groups=dev, chunk=chunk)
        assert a == b and n == signs.size, (p, a, b, n, signs.size)
        drops.append(b)
    return drops


def _same(torch, host, dev):
    a, b = _state(torch, host), _state(torch, dev)
    assert a.keys() == b.keys()
    for dim in a:
        assert a[dim][0] == b[dim][0], f"dim {dim}: signs"
        assert a[dim][1] == b[dim][1], f"dim {dim}: recency"
        assert a[dim][2] == b[dim][2], f"dim {dim}: entries"
    return a


@pytest.mark.parametrize("kind", [SGD, ADAGRAD, ADAM])
def test_one_dim_each_optimizer(env, tmp_path, kind):
    torch, INC, PC, tables = env
    rng = np.random.default_rng(kind)
    host, dev = tables({16: kind}), tables({16: kind})
    L = host[16]["shard"].entry_len
    paths = []
    for i in range(3):
        s = _signs(rng, 700)
        paths.append(_write(tmp_path, f"0_{i}.inc", INC.encode_packet(s, 16, _entries(rng, s.size, L), 100 + i)))
    assert _apply_both(env, paths, host, dev) == [0, 0, 0]
    st = _same(torch, host, dev)
    assert len(st[16][0]) == 2100


def test_several_dims_in_runs_of_different_lengths(env, tmp_path):
    """One packet interleaving three dims whose entry lengths differ (the host walk), and one whose two dims share an
    entry length (arithmetic offsets with two dims)."""
    torch, INC, PC, tables = env
    rng = np.random.default_rng(1)
    spec = {8: ADAGRAD, 16: SGD, 4: ADAM}
    host, dev = tables(spec), tables(spec)
    lens = {d: host[d]["shard"].entry_len for d in spec}
    assert lens[8] == lens[16] != lens[4]
    s = _signs(rng, 900)
    dims = rng.choice([8, 16, 4], size=s.size)
    dims[:5] = 4  # runs of every length, one of them at the start
    ent = [rng.standard_normal(lens[int(d)]).astype(np.float32) for d in dims]
    mixed = _write(tmp_path, "0_0.inc", INC.encode_packet(s, dims, ent, 7))
    s2 = _signs(rng, 500)
    d2 = rng.choice([8, 16], size=s2.size)
    same_len = _write(tmp_path, "0_1.inc", INC.encode_packet(s2, d2, _entries(rng, s2.size, lens[8]), 8))
    assert _apply_both(env, [mixed, same_len], host, dev) == [0, 0]
    st = _same(torch, host, dev)
    assert sum(len(v[0]) for v in st.values()) == len(set(s.tolist()) | set(s2.tolist()))


def test_empty_packet(env, tmp_path):
    torch, INC, PC, tables = env
    host, dev = tables({8: SGD}), tables({8: SGD})
    p = _write(tmp_path, "0_0.inc", INC.packet_bytes([], 5))
    assert _apply_both(env, [p], host, dev) == [0]
    assert _same(torch, host, dev)[8][0] == []


def test_marker_valued_signs(env, tmp_path):
    torch, INC, PC, tables = env
    rng = np.random.default_rng(2)
    host, dev = tables({8: ADAGRAD}), tables({8: ADAGRAD})
    L = host[8]["shard"].entry_len
    s = np.concatenate([_signs(rng, 40), np.array([~U64(0), ~U64(0) - U64(1), ~U64(0) - U64(2), 0], U64)])
    p = _write(tmp_path, "0_0.inc", INC.encode_packet(s, 8, _entries(rng, s.size, L), 5))
    assert _apply_both(env, [p], host, dev) == [0]
    got = _same(torch, host, dev)[8][0]
    assert {int(x) for x in np.array(got, np.int64).view(U64)} == {int(x) for x in s}


def test_same_sign_in_consecutive_packets_later_wins(env, tmp_path):
    torch, INC, PC, tables = env
    rng = np.random.default_rng(3)
    host, dev = tables({8: SGD}), tables({8: SGD})
    s = _signs(rng, 50)
    first, second = _entries(rng, 50, 8), _entries(rng, 50, 8)
    paths = [_write(tmp_path, "0_0.inc", INC.encode_packet(s, 8, first, 1)),
             _write(tmp_path, "0_1.inc", INC.encode_packet(s[::2], 8, second[::2], 2))]
    _apply_both(env, paths, host, dev)
    _same(torch, host, dev)
    got = dev[8]["shard"].get_entries(torch.from_numpy(s.view(np.int64)).cuda())[0].cpu().numpy()
    want = first.copy()
    want[::2] = second[::2]
    assert got.tobytes() == want.tobytes()


def test_hbm_full_without_tier_counts_drops(env, tmp_path):
    """The first packet fills the table; of the second, the signs it already holds are set and the new ones dropped."""
    torch, INC, PC, tables = env
    rng = np.random.default_rng(4)
    cap = 64
    host, dev = tables({8: ADAGRAD}, cap=cap), tables({8: ADAGRAD}, cap=cap)
    L = host[8]["shard"].entry_len
    s = _signs(rng, cap + 30)
    old, new = s[:cap], s[cap:]
    again = np.concatenate([old[:20], new])
    paths = [_write(tmp_path, "0_0.inc", INC.encode_packet(old, 8, _entries(rng, cap, L), 1)),
             _write(tmp_path, "0_1.inc", INC.encode_packet(again, 8, _entries(rng, again.size, L), 2))]
    assert _apply_both(env, paths, host, dev) == [0, 30]
    assert len(_same(torch, host, dev)[8][0]) == cap


def test_host_tier_holds_what_hbm_cannot(env, tmp_path):
    """PERSIA_B200_HBM_ROWS below the entries: HBM first, then the tier; then a packet that overflows both, whose drops
    are equal (which entries are dropped among those of one insert is not ordered, so only the counts are compared)."""
    torch, INC, PC, tables = env
    rng = np.random.default_rng(5)
    host, dev = tables({16: ADAGRAD}, cap=128, tier=1024), tables({16: ADAGRAD}, cap=128, tier=1024)
    L = host[16]["shard"].entry_len
    paths = []
    for i in range(2):
        s = _signs(rng, 400)
        paths.append(_write(tmp_path, f"0_{i}.inc", INC.encode_packet(s, 16, _entries(rng, s.size, L), i)))
    assert _apply_both(env, paths, host, dev, chunk=96) == [0, 0]
    assert len(_same(torch, host, dev)[16][0]) == 800
    for g in (host, dev):
        assert g[16]["shard"].tier_stats()["host_rows"] == 800 - 128
    s = _signs(rng, 600)
    over = _write(tmp_path, "0_2.inc", INC.encode_packet(s, 16, _entries(rng, s.size, L), 3))
    (d,) = _apply_both(env, [over], host, dev, chunk=96)
    assert d == 800 + 600 - 128 - 1024
    assert len(host[16]["shard"]) == len(dev[16]["shard"]) == 128 + 1024


def test_packet_larger_than_the_insert_chunk(env, tmp_path):
    torch, INC, PC, tables = env
    rng = np.random.default_rng(6)
    host, dev = tables({32: ADAM}), tables({32: ADAM})
    L = host[32]["shard"].entry_len
    s = _signs(rng, 3000)
    p = _write(tmp_path, "0_0.inc", INC.encode_packet(s, 32, _entries(rng, s.size, L), 1))
    assert _apply_both(env, [p], host, dev, chunk=257) == [0]
    assert len(_same(torch, host, dev)[32][0]) == 3000


def test_two_virtual_ranks_apply_their_own_directories(env, tmp_path, oracle):
    """Flushes written by the dumpers of two replicas, each scanned by its own loader: one through decode_packet and
    _apply_incremental, one through _apply_packet_file."""
    import functools

    torch, INC, PC, tables = env
    rng = np.random.default_rng(7)
    R, spec = 2, {8: SGD, 16: ADAGRAD}
    inc = str(tmp_path / "inc")
    sets = [(tables(spec), tables(spec)) for _ in range(R)]
    loaders = [(INC.IncrementalLoader(os.path.join(inc, f"s{r}"), functools.partial(PC._apply_incremental, groups=h)),
                INC.IncrementalLoader(os.path.join(inc, f"s{r}"),
                                      apply_file=functools.partial(PC._apply_packet_file, groups=d)))
               for r, (h, d) in enumerate(sets)]
    lens = {d: sets[0][0][d]["shard"].entry_len for d in spec}
    for _ in range(3):
        s = _signs(rng, 1200)
        own = oracle.shard_of(s, R)
        for r in range(R):
            mine = s[own == r]
            half = mine.size // 2
            parts = [(mine[:half], 8, _entries(rng, half, lens[8])),
                     (mine[half:], 16, _entries(rng, mine.size - half, lens[16]))]
            INC.IncrementalDumper(inc, r, num_workers=3).write(parts)
    for r, (lh, ld) in enumerate(loaders):
        assert lh.poll() == ld.poll() and len(lh.applied) == 3
        assert (lh.entries_applied, lh.entries_dropped, lh.failed_files) == \
            (ld.entries_applied, ld.entries_dropped, ld.failed_files)
        assert ld.entries_applied > 0 and ld.failed_files == 0
        _same(torch, *sets[r])


def test_malformed_packets_raise_decode_packet_errors_and_change_nothing(env, tmp_path):
    """Cut at every byte, and one trailing byte, of a uniform and of a mixed-length packet; then through the loader."""
    torch, INC, PC, tables = env
    rng = np.random.default_rng(8)
    spec = {4: SGD, 8: ADAGRAD}
    host, dev = tables(spec), tables(spec)
    seed = _write(tmp_path, "seed.inc", INC.encode_packet(_signs(rng, 20), 4, _entries(rng, 20, 4), 1))
    _apply_both(env, [seed], host, dev)
    before = _same(torch, host, dev)
    uniform = INC.encode_packet(_signs(rng, 3), 4, _entries(rng, 3, 4), 2)
    mixed = INC.encode_packet(_signs(rng, 3), [4, 8, 4], [np.ones(4, np.float32), np.ones(16, np.float32),
                                                          np.ones(4, np.float32)], 3)
    n = 0
    for good in (uniform, mixed):
        for bad in [good[:cut] for cut in range(len(good))] + [good + b"\0"]:
            with pytest.raises(ValueError) as want:
                INC.decode_packet(bad)
            p = _write(tmp_path, "bad.inc", bad)
            with pytest.raises(ValueError) as got:
                PC._apply_packet_file(p, groups=dev)
            assert str(got.value) == str(want.value), len(bad)
            n += 1
    assert n == len(uniform) + len(mixed) + 2
    assert _state(torch, dev) == before
    # through the loader: counted as failed, the good file beside it applied
    import functools

    d = tmp_path / "inc" / "s0"
    lh = INC.IncrementalLoader(str(d), functools.partial(PC._apply_incremental, groups=host))
    ld = INC.IncrementalLoader(str(d), apply_file=functools.partial(PC._apply_packet_file, groups=dev))
    os.makedirs(d / "inc_1")
    good = INC.encode_packet(_signs(rng, 10), 4, _entries(rng, 10, 4), 4)
    (d / "inc_1" / "0_0.inc").write_bytes(uniform[:-1])
    (d / "inc_1" / "0_1.inc").write_bytes(good)
    (d / "inc_1" / INC.DONE_FILE).write_bytes(b"")
    assert lh.poll() == ld.poll() == ["inc_1"]
    assert (ld.failed_files, ld.entries_applied, ld.entries_dropped) == (lh.failed_files, lh.entries_applied, 0) == (1, 10, 0)
    _same(torch, host, dev)


@pytest.mark.parametrize("case", ["unknown_dim", "wrong_length", "two_lengths_one_dim"])
def test_bad_dim_or_length_raises_after_the_same_partial_application(env, tmp_path, case):
    torch, INC, PC, tables = env
    rng = np.random.default_rng(9)
    spec = {4: SGD, 16: ADAGRAD, 64: SGD}
    host, dev = tables(spec), tables(spec)
    s = _signs(rng, 60)
    if case == "unknown_dim":  # dims 4 (applied), 8 (no table), 16 (not reached)
        dims = np.repeat([16, 8, 4], 20)
        ent = [np.full({16: 32, 8: 8, 4: 4}[int(d)], i, np.float32) for i, d in enumerate(dims)]
    elif case == "wrong_length":  # dim 16 entries of 16 floats, the table's are 32
        dims = np.repeat([4, 16, 64], 20)
        ent = [np.full({4: 4, 16: 16, 64: 64}[int(d)], i, np.float32) for i, d in enumerate(dims)]
    else:  # dim 16 entries of two lengths
        dims = np.repeat([4, 16, 16], 20)
        ent = [np.full(4 if d == 4 else (32 if i < 40 else 16), i, np.float32) for i, d in enumerate(dims)]
    p = _write(tmp_path, "0_0.inc", INC.encode_packet(s, dims, ent, 1))
    signs, dd, ee, _ = INC.decode_packet(open(p, "rb").read())
    with pytest.raises((RuntimeError, ValueError)) as want:
        PC._apply_incremental(signs, dd, ee, groups=host)
    with pytest.raises((RuntimeError, ValueError)) as got:
        PC._apply_packet_file(p, groups=dev)
    assert type(got.value) is type(want.value) and str(got.value) == str(want.value)
    st = _same(torch, host, dev)
    assert len(st[4][0]) == 20 and st[16][0] == [] and st[64][0] == []


def test_uniform_packet_and_one_with_a_corrupted_length_in_the_middle(env, tmp_path):
    """A uniform packet is read at arithmetic offsets; the same packet with one `len` changed fails the device check
    and takes the host walk, which gives decode_packet's error."""
    torch, INC, PC, tables = env
    rng = np.random.default_rng(10)
    host, dev = tables({16: ADAGRAD}), tables({16: ADAGRAD})
    L = host[16]["shard"].entry_len
    s = _signs(rng, 1000)
    good = INC.encode_packet(s, 16, _entries(rng, s.size, L), 1)
    assert len(good) == 12 + s.size * (20 + 4 * L)
    nb = 20 + 4 * L
    for new_len in (L - 1, L + 1, 0, 3 * L, 0x7FFFFFFF, 0x80000000):
        bad = bytearray(good)
        bad[4 + 500 * nb:8 + 500 * nb] = np.array([new_len], "<u4").tobytes()
        p = _write(tmp_path, "bad.inc", bytes(bad))
        with pytest.raises(ValueError) as want:
            INC.decode_packet(bytes(bad))
        with pytest.raises(ValueError) as got:
            PC._apply_packet_file(p, groups=dev)
        assert str(got.value) == str(want.value), new_len
    assert _state(torch, dev)[16][0] == []
    p = _write(tmp_path, "0_0.inc", good)
    assert _apply_both(env, [p], host, dev) == [0]
    assert len(_same(torch, host, dev)[16][0]) == 1000


def test_packet_of_more_dims_than_one_device_summary_is_applied_on_the_host(env, tmp_path):
    """33 dims (the device summary holds 32): the packet goes through decode_packet and _apply_incremental, and the
    tables end as the host path leaves them."""
    torch, INC, PC, tables = env
    rng = np.random.default_rng(11)
    spec = {d: SGD for d in range(1, 34)}
    host, dev = tables(spec, cap=64), tables(spec, cap=64)
    s = _signs(rng, 33 * 4)
    dims = np.repeat(np.arange(1, 34), 4)
    ent = [rng.standard_normal(int(d)).astype(np.float32) for d in dims]
    p = _write(tmp_path, "0_0.inc", INC.encode_packet(s, dims, ent, 1))
    assert _apply_both(env, [p], host, dev) == [0]
    st = _same(torch, host, dev)
    assert all(len(st[d][0]) == 4 for d in spec)


def test_forwards_beside_packets_read_whole_entries(env, tmp_path):
    """A second thread serves inference forwards of the packets' signs on the same table, under its lock, while
    packets that rewrite those signs apply: every pooled row is one packet's entry (or the zeros of a sign not yet
    inserted), never a mix, and the table ends as the host path leaves it."""
    from persia_b200 import shard as SH

    torch, INC, PC, tables = env
    rng = np.random.default_rng(12)
    dim, B = 16, 4096
    host, dev = tables({dim: SGD}, cap=1 << 14), tables({dim: SGD}, cap=1 << 14)
    s = _signs(rng, B)
    vals = [_entries(rng, B, dim) for _ in range(6)]
    paths = [_write(tmp_path, f"0_{k}.inc", INC.encode_packet(s, dim, v, k)) for k, v in enumerate(vals)]
    allowed = np.stack([np.zeros((B, dim), np.float16)] + [v.astype(np.float16) for v in vals])  # [7, B, dim]
    sh, lock = dev[dim]["shard"], dev[dim]["lock"]
    ctx = SH.BatchContext(B, B, [0], device=0)
    ids = torch.from_numpy(s.view(np.int64)).cuda()
    fs = torch.cuda.Stream()
    done, bad, served = threading.Event(), [], [0]

    def serve():
        while not done.is_set():
            with torch.cuda.stream(fs):
                with lock:
                    out = ctx.forward(sh, ids, [0, B], B, training=False)
                fs.synchronize()
            got = out[0].cpu().numpy()
            ok = (allowed.view(np.uint16) == got.view(np.uint16)[None]).all(axis=2).any(axis=0)
            if not ok.all():
                bad.append(int((~ok).sum()))
            served[0] += 1

    th = threading.Thread(target=serve)
    th.start()
    try:
        for p in paths:
            with open(p, "rb") as f:
                sg, dd, ee, _ = INC.decode_packet(f.read())
            PC._apply_incremental(sg, dd, ee, groups=host)
            assert PC._apply_packet_file(p, groups=dev) == (0, B)
    finally:
        done.set()
        th.join()
        ctx.close()
    assert served[0] > 0 and not bad, bad[:5]
    _same(torch, host, dev)
