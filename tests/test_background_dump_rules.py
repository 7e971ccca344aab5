"""CPU: the host-side rules of the background embedding dump (persia_b200/checkpoint.py): the part of a sign, the
number of parts, the file numbering and the root marker's wait."""
import os

import numpy as np
import pytest

from persia_b200 import checkpoint as CK


def test_splitmix64_matches_the_published_constants():
    # splitmix64 of 0 and 1 (Vigna's reference generator seeded with x, first output)
    assert int(CK.splitmix64(np.array([0], np.uint64))[0]) == 0xE220A8397B1DCDAF
    assert int(CK.splitmix64(np.array([1], np.uint64))[0]) == 0x910A2DEC89025CC1


def test_part_rule_is_deterministic_and_covers_every_part():
    rng = np.random.default_rng(5)
    signs = rng.integers(0, 2**64, size=100_000, dtype=np.uint64)
    a, b = CK.part_of(signs, 100), CK.part_of(signs.copy(), 100)
    np.testing.assert_array_equal(a, b)
    assert a.max() < 100 and np.unique(a).size == 100


@pytest.mark.parametrize("R", [2, 3, 8])
def test_every_owner_part_pair_is_populated(R):
    # the owner rule farmhash64 % R would put every sign of rank r in part r % n_parts: splitmix64 is independent of it
    rng = np.random.default_rng(R)
    signs = rng.integers(0, 2**64, size=100_000, dtype=np.uint64)
    owner = CK._farmhash64(signs) % np.uint64(R)
    part = CK.part_of(signs, 100)
    pairs = np.unique(owner.astype(np.int64) * 100 + part.astype(np.int64))
    assert pairs.size == R * 100


def test_num_parts_follows_the_config_key_its_default_and_the_size_term():
    assert CK.internal_shards(None) == 100
    assert CK.internal_shards({}) == 100
    assert CK.internal_shards({"embedding_parameter_server_config": {"num_hashmap_internal_shards": 7}}) == 7
    with pytest.raises(RuntimeError):
        CK.internal_shards({"embedding_parameter_server_config": {"num_hashmap_internal_shards": 0}})
    mib = 1 << 20
    assert CK.num_parts([10 * mib], 100) == 100
    assert CK.num_parts([10 * mib], 1) == 1
    assert CK.num_parts([256 * mib], 1) == 1
    assert CK.num_parts([256 * mib + 1], 1) == 2
    # 5e7 rows of dim 128 with Adagrad: 51.2 GB of entries
    assert CK.num_parts([50_000_000 * 256 * 4, 10 * mib], 100) == -(-50_000_000 * 256 * 4 // (256 * mib))


def test_num_parts_reads_the_global_config_without_changing_the_parsed_dict():
    from persia_b200 import incremental as INC

    gc = {"embedding_parameter_server_config": {"num_hashmap_internal_shards": 12, "capacity": 1000}}
    parsed = INC.parse_global_config(gc)
    assert "num_hashmap_internal_shards" not in parsed
    assert CK.internal_shards(gc) == 12


def test_file_numbering():
    assert CK.part_file(0, 0, 100, 0) == "replica_0_shard_0.emb"
    assert CK.part_file(2, 1, 100, 7) == "replica_2_shard_107.emb"
    assert CK.part_file(1, 3, 5, 4) == "replica_1_shard_19.emb"
    names = {CK.part_file(0, d, 3, k) for d in range(4) for k in range(3)}
    assert names == {f"replica_0_shard_{i}.emb" for i in range(12)}


class _Clock:
    def __init__(self):
        self.t = 0.0

    def __call__(self):
        return self.t


def test_marker_wait_completes_when_the_markers_appear(tmp_path):
    clock = _Clock()
    for q in range(3):
        os.makedirs(tmp_path / f"s{q}")
    (tmp_path / "s0" / CK.DONE_FILE).write_text("x")
    late = iter([1, 2])

    def sleep(s):  # a shard marker appears at each poll
        clock.t += s
        q = next(late, None)
        if q is not None:
            (tmp_path / f"s{q}" / CK.DONE_FILE).write_text("x")

    CK.wait_for_markers(str(tmp_path), 3, timeout=10, poll=1, clock=clock, sleep=sleep)
    assert clock.t == 2


def test_marker_wait_times_out(tmp_path):
    clock = _Clock()
    os.makedirs(tmp_path / "s0")
    (tmp_path / "s0" / CK.DONE_FILE).write_text("x")

    def sleep(s):
        clock.t += s

    with pytest.raises(TimeoutError):
        CK.wait_for_markers(str(tmp_path), 2, timeout=5, poll=1, clock=clock, sleep=sleep)
    assert clock.t >= 5


def test_a_dump_whose_markers_time_out_ends_failed(tmp_path):
    """The dumper records the root marker's timeout as its status; wait() raises the reference's message."""
    d = CK.BackgroundDumper(str(tmp_path), [], replica_index=0, replica_size=2, n_parts=1, marker_timeout=0.0)
    d.start()
    with pytest.raises(RuntimeError, match="emb dump FAILED for server 0, due to"):
        d.wait()
    state, msg = d.status()
    assert state == "Failed" and "TimeoutError" in msg
    assert (tmp_path / "s0" / CK.DONE_FILE).is_file() and not (tmp_path / CK.DONE_FILE).exists()
