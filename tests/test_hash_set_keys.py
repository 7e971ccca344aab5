"""CPU: the key-crafting helpers of tests/hash_set_keys.py do what the GPU hash-set tests rely on.  Without these, a GPU
test could pass without any cluster ever forming: mix64 is MurmurHash3's fmix64, the numpy prefix equals the oracle's
indices_add_prefix at every prefix width, and the search returns ids whose signs land where it says."""
import numpy as np
import pytest

import hash_set_keys as K

M64 = K.M64


def test_mix64_is_fmix64():
    # fmix64 values (MurmurHash3_x64_128's finaliser), independent of numpy
    known = {0: 0x0, 1: 0xB456BCFC34C2CB2C, 2: 0x3ABF2A20650683E7, 0xDEADBEEF: 0xD24BD59F862A1DAC,
             1 << 63: 0x8F780810AF31A493, M64: 0x64B5720B4B825F21}
    got = K.mix64(np.array(list(known), np.uint64))
    assert [int(x) for x in got] == list(known.values())

    def fmix64(k):
        k ^= k >> 33
        k = (k * 0xFF51AFD7ED558CCD) & M64
        k ^= k >> 33
        k = (k * 0xC4CEB9FE1A85EC53) & M64
        return k ^ (k >> 33)

    x = np.random.default_rng(0).integers(0, M64, size=2000, dtype=np.uint64, endpoint=True)
    assert [int(v) for v in K.mix64(x)] == [fmix64(int(v)) for v in x]


@pytest.mark.parametrize("b", range(1, 64))
def test_prefix_matches_the_oracle_at_every_width(oracle, b):
    rng = np.random.default_rng(b)
    ids = K.edge_ids(b, rng, n_random=64)
    m = K.spacing(b)
    assert m == 2 ** (64 - b) - 1
    for g in range(min(3, (1 << b) - 1)):
        p = oracle.index_prefix(g, b)
        assert p == (g + 1) << (64 - b)
        want = oracle.add_prefix(ids, b, p)
        assert [int(x) for x in K.prefix_np(ids, b, p)] == [int(x) for x in want]
        assert [K.prefix_int(x, b, p) for x in ids.tolist()] == [int(x) for x in want]
        # an id's residue is the one id of its sign; the residue of m is 0, not m
        assert K.prefix_np(K.residues(ids, b, p), b, p).tobytes() == want.tobytes()
        assert K.prefix_int(m, b, p) == K.prefix_int(0, b, p) == p
        assert K.prefix_int(2 * m + 5, b, p) == K.prefix_int(5 % m, b, p)
    # prefix 0: ids pass through, 2^64-1 included
    assert K.prefix_np(ids, b, 0).tobytes() == oracle.add_prefix(ids, b, 0).tobytes() == ids.tobytes()


def test_edge_ids_cover_the_residue_edges():
    rng = np.random.default_rng(1)
    for b in K.PREFIX_BITS:
        m = K.spacing(b)
        ids = set(int(x) for x in K.edge_ids(b, rng))
        assert {0, 1, m - 1, m, m + 1, 2 * m, 1 << 63, M64} <= ids
        assert sum(1 for x in ids if x % m == 0) >= 3  # 0, m, 2m at least: one sign
    assert K.edge_ids(1, rng).max() == M64 and K.spacing(1) * 3 > M64


def test_set_layouts():
    # regions: slot s of n_s occurrences owns 2 n_s + 1 cells, then the reserved cell; the next region starts after it
    occ = [0, 5, 5, 12]
    regions = [K.set_region(occ, s) for s in range(3)]
    assert regions == [(0, 11), (12, 1), (14, 15)]
    for (off, size), (nxt, _) in zip(regions, regions[1:]):
        assert off + size + 1 == nxt
    assert K.raw_cells(100) == 1024 and K.raw_cells(513) == 2048 and K.raw_cells(1024) == 2048
    assert K.inc_cells(16) == 1024 and K.inc_cells(1500) == 4096
    signs = np.random.default_rng(2).integers(0, M64, size=5000, dtype=np.uint64)
    h = K.dedup_home(signs, 100, 37)
    assert h.min() >= 100 and h.max() < 137 and np.unique(h).size == 37


@pytest.mark.parametrize("b,g", [(0, None), (8, 0), (8, 5), (31, 1)])
def test_search_lands_every_sign_on_its_target(oracle, b, g):
    p = oracle.index_prefix(g, b) if g is not None else 0
    # a region's last cell: the probes of all but the first sign wrap to the region's first cell
    off, size = K.set_region([0, 40, 140], 1)
    ids = K.homed_ids(lambda s: K.dedup_home(s, off, size), off + size - 1, 30, b, p)
    signs = K.prefix_np(ids, b, p)
    assert signs.tobytes() == oracle.add_prefix(ids, b, p).tobytes()
    assert np.unique(signs).size == ids.size == 30 and np.all(ids[1:] > ids[:-1])
    assert np.all(K.dedup_home(signs, off, size) == off + size - 1)
    assert sorted(K.probe_cells(K.dedup_home(signs, off, size), off, size)) == [off + k for k in range(29)] + [off + size - 1]
    # the raw set's last cell and the incremental set's last bucket
    cells = K.raw_cells(1000)
    r = K.prefix_np(K.homed_ids(lambda s: K.raw_home(s, cells), cells - 1, 5, b, p), b, p)
    assert np.all(K.raw_home(r, cells) == cells - 1)
    n = K.inc_cells(500)
    last = n // K.BUCKET - 1
    i = K.prefix_np(K.homed_ids(lambda s: K.inc_bucket(s, n), last, 12, b, p, avoid=r), b, p)
    assert np.all(K.inc_bucket(i, n) == last) and not set(i.tolist()) & set(r.tolist())
