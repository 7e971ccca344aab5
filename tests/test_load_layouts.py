"""CPU-only: the host-side planning of device checkpoint loads (persia_b200/checkpoint.py DeviceLoader): which files
stream in windows of whole nodes, the windows, the reference-layout generator the GPU tests use, the per-dim checks
and the load status."""
import numpy as np
import pytest

from emb_layouts import reference_layout
from persia_b200 import checkpoint as CK


def _entries(rng, n, L):
    return rng.standard_normal((n, L)).astype(np.float32)


@pytest.mark.parametrize("n", [1, 2, 7])
def test_writer_files_are_detected(n):
    rng = np.random.default_rng(n)
    img = CK.encode_list(rng.integers(0, 2**63, n, dtype=np.uint64), _entries(rng, n, 16), 8)
    assert CK.writer_layout(len(img), img[:41]) == (n, 16)
    assert CK.writer_layout(len(img) + 1, img[:41]) is None  # trailing bytes
    assert CK.writer_layout(len(img), img[:40]) is None


def test_other_layouts_are_not_writer_files():
    rng = np.random.default_rng(1)
    signs = rng.integers(0, 2**63, 20, dtype=np.uint64)
    assert CK.writer_layout(28, CK.list_header(0)) is None  # the empty list: read whole
    for permute, free in ((True, 0), (False, 3), (True, 4)):
        img = reference_layout(signs, [8] * 20, list(_entries(rng, 20, 16)), rng, permute=permute, free=free)
        assert CK.writer_layout(len(img), img[:41]) is None
    mixed = [_entries(rng, 1, 16)[0] if k % 2 else _entries(rng, 1, 64)[0] for k in range(20)]
    img = reference_layout(signs, [8 if k % 2 else 32 for k in range(20)], mixed, rng, permute=False)
    assert CK.writer_layout(len(img), img[:41]) is None


@pytest.mark.parametrize("permute,free", [(True, 0), (False, 5), (True, 9), (False, 0)])
def test_generator_decodes_to_its_list(permute, free):
    rng = np.random.default_rng(7 + free)
    n = 40
    signs = np.concatenate([rng.integers(0, 2**63, n - 3, dtype=np.uint64),
                            np.array([2**64 - 1, 2**64 - 2, 2**64 - 3], np.uint64)])
    dims = np.where(np.arange(n) % 3 == 0, 32, 8).astype(np.uint64)
    ent = [rng.standard_normal(2 * int(d)).astype(np.float32) for d in dims]
    s, d, e = CK.decode_list(reference_layout(signs, dims, ent, rng, permute=permute, free=free))
    np.testing.assert_array_equal(s, signs)
    np.testing.assert_array_equal(d, dims)
    for a, b in zip(e, ent):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("nb", [45, 93, 1053])
def test_windows_are_whole_nodes(nb):
    n = 37
    for extra in range(nb):
        for buf in (3 * nb + extra, nb + extra, extra or 1):
            for newest in (False, True):
                w = CK.windows(n, nb, buf, newest)
                per = max(1, buf // nb)
                assert all(hi - lo <= per and (hi - lo) * nb <= max(buf, nb) for lo, hi in w)
                flat = [i for lo, hi in (w[::-1] if newest else w) for i in range(lo, hi)]
                assert flat == list(range(n))  # every node once, the windows in file order or its reverse
                if newest:
                    assert w[0][1] == n and w[-1][0] == 0
                else:
                    assert w[0][0] == 0 and w[-1][1] == n


def test_newest_first_windows_run_from_the_end():
    assert CK.windows(10, 100, 300) == [(0, 3), (3, 6), (6, 9), (9, 10)]
    assert CK.windows(10, 100, 300, newest_first=True) == [(7, 10), (4, 7), (1, 4), (0, 1)]
    assert CK.windows(3, 100, 1) == [(0, 1), (1, 2), (2, 3)]
    assert CK.windows(0, 100, 300) == []


class _Table:
    def __init__(self, entry_len):
        self.entry_len = entry_len


def test_dim_checks_give_load_shards_messages():
    tables = {8: _Table(16), 32: _Table(64)}
    assert CK.check_dims([(32, 64, 5), (8, 16, 3)], tables) == [(8, 3), (32, 5)]
    with pytest.raises(RuntimeError, match=r"^checkpoint holds dim-16 embeddings but no slot has that dim$"):
        CK.check_dims([(8, 16, 3), (16, 32, 1)], tables)
    with pytest.raises(RuntimeError, match=r"^dim-8 entries of \[16, 17\] floats, the registered optimizer needs 16 "
                                           r"\(embedding \+\+ state\)$"):
        CK.check_dims([(8, 17, 1), (8, 16, 3)], tables)
    # dims ascending: the first failing dim is the one load_shards reaches first
    with pytest.raises(RuntimeError, match="dim-8 entries of"):
        CK.check_dims([(8, 20, 1), (16, 32, 1)], tables)


def test_status_machine():
    st = CK.LoadStatus(200)
    assert st() == ("Loading", 0.0)
    st.advance(50)
    assert st() == ("Loading", 0.25)
    st.advance(500)
    assert st()[0] == "Loading" and st()[1] < 1.0  # done only when finished
    st.finish()
    assert st() == ("Idle", 1.0)
    bad = CK.LoadStatus(0)
    bad.fail(ValueError("truncated checkpoint: node"))
    assert bad() == ("Failed", "ValueError: truncated checkpoint: node")
