"""CPU: incremental-update packets, the dumper's directory layout, the loader's order, and the global-config keys
(persia_b200/incremental.py)."""
import os
import struct

import numpy as np
import pytest

from persia_b200 import incremental as INC


# ------------------------------------------------------------------------------------------------ packet codec
def _entry(sign, dim, inner):
    return struct.pack("<I", len(inner)) + struct.pack(f"<{len(inner)}f", *inner) + struct.pack("<QQ", dim, sign)


def test_two_entry_packet_mixed_dims_against_hand_laid_bytes():
    want = (struct.pack("<I", 2) + _entry(5, 2, [1.0, 2.0]) + _entry(0xFFFFFFFFFFFFFFFF, 1, [3.0, 0.5, -0.25]) +
            struct.pack("<Q", 1_700_000_000))
    got = INC.encode_packet(np.array([5, 0xFFFFFFFFFFFFFFFF], np.uint64), [2, 1],
                            [np.array([1.0, 2.0], np.float32), np.array([3.0, 0.5, -0.25], np.float32)], 1_700_000_000)
    assert got == want
    signs, dims, ent, ts = INC.decode_packet(want)
    assert signs.tolist() == [5, 0xFFFFFFFFFFFFFFFF] and dims.tolist() == [2, 1] and ts == 1_700_000_000
    assert [e.tolist() for e in ent] == [[1.0, 2.0], [3.0, 0.5, -0.25]]


def test_zero_entry_packet():
    want = struct.pack("<I", 0) + struct.pack("<Q", 42)
    assert INC.encode_packet(np.zeros(0, np.uint64), [], [], 42) == want
    signs, dims, ent, ts = INC.decode_packet(want)
    assert signs.size == 0 and dims.size == 0 and ent == [] and ts == 42


def test_uniform_packet_matches_checkpoint_entry_layout():
    """The entries are laid out exactly as a checkpoint node's entry (checkpoint.entry_fields)."""
    from persia_b200 import checkpoint as CK

    rng = np.random.default_rng(0)
    signs = rng.integers(0, 1 << 63, 5, dtype=np.uint64)
    ent = rng.standard_normal((5, 6)).astype(np.float32)
    buf = INC.encode_packet(signs, 3, ent, 9)
    node = CK.encode_list(signs, ent, 3)[28:]  # the checkpoint's nodes: next u32 | prev u32 | flag u8 | entry
    L = 4 + 6 * 4 + 16
    for k in range(5):
        assert buf[4 + k * L:4 + (k + 1) * L] == node[k * (9 + L) + 9:(k + 1) * (9 + L)]


@pytest.mark.parametrize("lens", [[4], [4, 4, 2, 2, 2, 9], [1, 3, 1, 3]])
def test_round_trips(lens):
    rng = np.random.default_rng(len(lens))
    signs = rng.integers(0, 1 << 64, len(lens), dtype=np.uint64)
    ent = [rng.standard_normal(L).astype(np.float32) for L in lens]
    dims = [max(1, L // 2) for L in lens]
    s, d, e, ts = INC.decode_packet(INC.encode_packet(signs, dims, ent, 7))
    assert s.tolist() == signs.tolist() and d.tolist() == dims and ts == 7
    assert all(a.tobytes() == b.tobytes() for a, b in zip(e, ent))


def test_truncated_packets_raise():
    buf = INC.encode_packet(np.array([1, 2], np.uint64), 2, np.ones((2, 2), np.float32), 1)
    for cut in (3, 10, len(buf) - 1):
        with pytest.raises(ValueError):
            INC.decode_packet(buf[:cut])
    with pytest.raises(ValueError):
        INC.decode_packet(buf + b"\0")


# ------------------------------------------------------------------------------------------------ dumper
def _parts(rng, n_by_dim):
    parts = []
    for dim, n in n_by_dim.items():
        signs = rng.choice(1 << 40, n, replace=False).astype(np.uint64) | np.uint64(dim << 56)
        parts.append((signs, dim, rng.standard_normal((n, 2 * dim)).astype(np.float32)))
    return parts


def test_dumper_layout_done_last_and_sorted(tmp_path):
    rng = np.random.default_rng(1)
    d = INC.IncrementalDumper(str(tmp_path), replica_index=3, num_workers=4)
    parts = _parts(rng, {8: 50, 2: 31})
    order = []
    real_open = open

    def spy(path, mode="r", *a, **kw):  # the order files are created in
        order.append(os.path.basename(path))
        return real_open(path, mode, *a, **kw)

    import builtins

    builtins.open, saved = spy, builtins.open
    try:
        path = d.write(parts, timestamp=11)
    finally:
        builtins.open = saved
    assert os.path.dirname(path) == os.path.join(str(tmp_path), "s3")
    assert order == ["3_0.inc", "3_1.inc", "3_2.inc", "3_3.inc", INC.DONE_FILE]
    assert sorted(os.listdir(path)) == sorted(order)
    signs, dims, ents = [], [], []
    sizes = []
    for i in range(4):
        s, dm, e, ts = INC.decode_packet(open(os.path.join(path, f"3_{i}.inc"), "rb").read())
        assert ts == 11
        sizes.append(s.size)
        signs.append(s), dims.append(dm), ents.extend(e)
    signs, dims = np.concatenate(signs), np.concatenate(dims)
    assert np.all(signs[:-1] < signs[1:])  # ascending across the flush's files
    assert sorted(sizes) == [20, 20, 20, 21]
    want = {int(x): (dim, e[k]) for x0, dim, e in parts for k, x in enumerate(x0)}
    for k, x in enumerate(signs):
        assert want[int(x)][0] == dims[k] and want[int(x)][1].tobytes() == ents[k].tobytes()


def test_dumper_no_empty_files_and_empty_flush(tmp_path):
    d = INC.IncrementalDumper(str(tmp_path), replica_index=0, num_workers=4)
    rng = np.random.default_rng(2)
    path = d.write(_parts(rng, {4: 2}))
    assert sorted(os.listdir(path)) == ["0_0.inc", "0_1.inc", INC.DONE_FILE]
    assert d.write([(np.zeros(0, np.uint64), 4, np.zeros((0, 8), np.float32))]) is None
    assert os.listdir(os.path.join(str(tmp_path), "s0")) == [os.path.basename(path)]


def test_dir_names_unique_and_in_flush_order_within_one_second(tmp_path):
    import datetime

    now = datetime.datetime(2026, 1, 2, 3, 4, 5)
    names = [INC.flush_dir_name(now) for _ in range(12)]
    assert len(set(names)) == 12 and names == sorted(names)
    assert all(n.startswith("inc_20260102030405_") for n in names)
    d = INC.IncrementalDumper(str(tmp_path), num_workers=1)
    rng = np.random.default_rng(3)
    paths = [d.write(_parts(rng, {2: 3})) for _ in range(12)]
    assert len(set(paths)) == 12 and paths == sorted(paths)


def test_dumper_thread_and_full_queue(tmp_path):
    d = INC.IncrementalDumper(str(tmp_path), num_workers=2, channel_capacity=2)
    rng = np.random.default_rng(4)
    for _ in range(3):
        d.submit(_parts(rng, {2: 5}))
    d.flush()
    assert len(d.written) + d.dropped_flushes == 3 and len(d.written) >= 2
    d.close()


# ------------------------------------------------------------------------------------------------ loader
def test_loader_order_incomplete_and_seen_at_start(tmp_path):
    rng = np.random.default_rng(5)
    d = INC.IncrementalDumper(str(tmp_path), replica_index=1, num_workers=3)
    pre = d.write(_parts(rng, {2: 4}))  # present at start: never applied
    applied = []

    def apply(signs, dims, entries):
        applied.append((signs.copy(), [e.copy() for e in entries]))
        return 0

    loader = INC.IncrementalLoader(os.path.join(str(tmp_path), "s1"), apply)
    assert loader.poll() == []
    # one sign in two flushes, with different values: the later flush must be applied last
    sign = np.array([77], np.uint64)
    a = d.write([(sign, 2, np.full((1, 4), 1.0, np.float32))] + _parts(rng, {2: 5}))
    b = d.write([(sign, 2, np.full((1, 4), 2.0, np.float32))] + _parts(rng, {2: 5}))
    os.remove(os.path.join(b, INC.DONE_FILE))  # b is still being written
    assert loader.poll() == [os.path.basename(a)]
    assert loader.poll() == []
    open(os.path.join(b, INC.DONE_FILE), "w").close()
    assert loader.poll() == [os.path.basename(b)]
    assert os.path.basename(pre) not in loader.applied
    last = {}
    for signs, ents in applied:
        for k, x in enumerate(signs):
            last[int(x)] = ents[k]
    assert last[77].tolist() == [2.0] * 4
    # files are applied in index order
    sizes = [s.size for s, _ in applied]
    assert sizes[:3] == [2, 2, 2] and sum(sizes) == 12


def test_loader_background_thread_stops(tmp_path):
    loader = INC.IncrementalLoader(os.path.join(str(tmp_path), "s0"), lambda *a: 0, interval=0.05)
    loader.start()
    d = INC.IncrementalDumper(str(tmp_path), num_workers=1)
    d.write(_parts(np.random.default_rng(6), {2: 3}))
    import time

    for _ in range(100):
        if loader.applied:
            break
        time.sleep(0.05)
    loader.stop()
    assert len(loader.applied) == 1 and loader._thread is None


# ------------------------------------------------------------------------------------------------ global config
def test_global_config_defaults_match_the_reference():
    c = INC.parse_global_config({})
    assert c == dict(job_type="Train", num_workers=4, embedding_checkpoint=None, capacity=None,
                     enable_incremental_update=False, incremental_buffer_size=1_000_000,
                     incremental_dir="/workspace/incremental_dir/", incremental_channel_capacity=1000)


def test_global_config_train_and_infer():
    t = INC.parse_global_config({"common_config": {"job_type": "Train", "checkpointing_config": {"num_workers": 2}},
                                 "embedding_parameter_server_config": {
                                     "capacity": 1000, "enable_incremental_update": True,
                                     "incremental_buffer_size": 10, "incremental_dir": "/x",
                                     "incremental_channel_capacity": 3}})
    assert (t["job_type"], t["num_workers"], t["capacity"], t["enable_incremental_update"], t["incremental_buffer_size"],
            t["incremental_dir"], t["incremental_channel_capacity"]) == ("Train", 2, 1000, True, 10, "/x", 3)
    i = INC.parse_global_config({"common_config": {"job_type": "Infer", "infer_config": {"embedding_checkpoint": "/c"}}})
    assert i["job_type"] == "Infer" and i["embedding_checkpoint"] == "/c"
    with pytest.raises(RuntimeError):
        INC.parse_global_config({"common_config": {"job_type": "Serve"}})


def test_persia_core_reads_the_global_config(tmp_path, monkeypatch):
    from persia_b200 import persia_core as pc

    pc.reset()
    try:
        p = tmp_path / "global.yml"
        p.write_text("common_config:\n  job_type: Infer\nembedding_parameter_server_config:\n"
                     "  enable_incremental_update: true\n  incremental_dir: /tmp/inc\n")
        monkeypatch.setenv("PERSIA_GLOBAL_CONFIG", str(p))
        c = pc._S.global_config()
        assert c["job_type"] == "Infer" and c["incremental_dir"] == "/tmp/inc" and not pc._S.incremental_on()
        pc.set_global_config({"embedding_parameter_server_config": {"enable_incremental_update": True}})
        assert pc._S.incremental_on() and pc._S.global_config()["job_type"] == "Train"
        with pytest.raises(RuntimeError):
            pc.set_global_config({"common_config": {"job_type": "nope"}})
    finally:
        pc.reset()
    assert not pc._S.incremental_on() or os.environ.get("PERSIA_GLOBAL_CONFIG")


def test_loader_logs_a_bad_packet_and_goes_on(tmp_path):
    rng = np.random.default_rng(8)
    d = INC.IncrementalDumper(str(tmp_path), num_workers=2)
    applied = []
    loader = INC.IncrementalLoader(os.path.join(str(tmp_path), "s0"), lambda s, dm, e: applied.append(s.size) or 0)
    a = d.write(_parts(rng, {2: 6}))
    b = d.write(_parts(rng, {2: 4}))
    with open(os.path.join(a, "0_0.inc"), "r+b") as f:  # truncate one packet of the first flush
        f.truncate(10)
    assert loader.poll() == [os.path.basename(a), os.path.basename(b)]
    assert loader.failed_files == 1 and applied == [3, 2, 2]
    assert loader.poll() == []


def test_dir_names_use_utc():
    import datetime

    name = INC.flush_dir_name()
    now = datetime.datetime.now(datetime.timezone.utc)
    stamp = datetime.datetime.strptime(name.split("_")[1], "%Y%m%d%H%M%S").replace(tzinfo=datetime.timezone.utc)
    assert abs((now - stamp).total_seconds()) < 5
