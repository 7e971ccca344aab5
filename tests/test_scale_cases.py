"""CPU-only: the batches of tests/test_gpu_scale.py (tests/scale_cases.py) are what their cases say they are."""
import numpy as np
import pytest

import scale_cases as SC


def _positions(ids, k):
    return np.flatnonzero(ids == np.uint64(k))


@pytest.fixture(scope="module")
def summation():
    return SC.summation_case(1)


def test_summation_case_fills_the_context(summation):
    ids, row_off = summation
    assert ids.size == SC.SUM_N and int(row_off[-1]) == SC.SUM_N and row_off.size == SC.SUM_B + 1
    assert 0 < SC.CTX_LIMIT - SC.SUM_N <= 4
    lens = np.diff(row_off.astype(np.int64))
    assert sorted(np.flatnonzero(lens == 0).tolist()) == sorted(SC.SUM_EMPTY)
    assert SC.CTX_LIMIT // SC.HOT_WIN == 2048  # windows of the slot: far more than the 8 any other test reaches


def test_summation_case_multiplicities_and_spans(summation):
    ids, _ = summation
    n_windows = -(-SC.SUM_N // SC.HOT_WIN)
    last = (n_windows - 1) * SC.HOT_WIN
    for k, (count, span) in enumerate(SC.SUM_ITEMS):
        pos = _positions(ids, k)
        assert pos.size == count, (k, pos.size, count)
        if span is not None:
            assert span[0] <= pos.min() and pos.max() < span[1], (k, span)
    # straddling: the item holds occurrences on both sides of a window boundary
    for k in (0, 2, 3, 4, 5, 6):
        w = _positions(ids, k) // SC.HOT_WIN
        assert w.min() < w.max(), k
    assert _positions(ids, 0).size == SC.HOT_WIN + 1 and np.unique(_positions(ids, 0) // SC.HOT_WIN).size == 2
    # one item inside the last (short) window, and the ~4 M item in every window
    assert (_positions(ids, 1) >= last).all() and SC.SUM_N - last < SC.HOT_WIN
    assert np.unique(_positions(ids, 7) // SC.HOT_WIN).size == n_windows
    assert SC.SUM_ITEMS[7][0] > 4_000_000 and SC.SUM_ITEMS[8][0] > 1_000_000 - 10


def test_summation_case_only_named_items_are_hot(summation):
    ids, _ = summation
    fill = ids[ids >= SC.FILL_BASE]
    c = np.unique(fill, return_counts=True)[1]
    assert c.max() <= SC.WARM_MAX and (c == 1).any() and (c > 1).any()
    assert fill.size + sum(x for x, _ in SC.SUM_ITEMS) == SC.SUM_N
    assert 1_500_000 < c.size <= SC.SUM_POOL


def test_pool_case_needs_both_modes():
    ids, row_off = SC.pool_case(2)
    assert ids.size == SC.POOL_N and int(row_off[-1]) == SC.POOL_N
    for k, count in enumerate(SC.POOL_ITEMS):
        assert _positions(ids, k).size == count, k
    hot = [c for c in SC.POOL_ITEMS if c > SC.WARM_MAX]
    words = (SC.POOL_N + 31) // 32
    assert SC.POOL_BITMAPS == 32 and len(hot) == len(SC.POOL_ITEMS) == 48
    assert len(hot) * words > max(4096, SC.POOL_N) >= SC.POOL_BITMAPS * words  # some bitmaps fit, the rest do not
    c = np.unique(ids[ids >= SC.FILL_BASE], return_counts=True)[1]
    assert c.max() <= SC.WARM_MAX


def test_wrap_case_passes_2_pow_32_words():
    ids, row_off = SC.wrap_case(7)
    assert ids.size == SC.POOL_N and int(row_off[-1]) == SC.POOL_N
    c = np.unique(ids, return_counts=True)
    hot = c[0][c[1] > SC.WARM_MAX]
    assert hot.tolist() == list(range(SC.WRAP_HOT)) and (c[1][c[1] > SC.WARM_MAX] == SC.WRAP_MULT).all()
    words = (SC.POOL_N + 31) // 32
    assert SC.WRAP_HOT * words > 2 ** 32  # the words asked for pass what a 32-bit counter holds
    assert SC.POOL_BITMAPS * words <= max(4096, SC.POOL_N) < (SC.POOL_BITMAPS + 1) * words


@pytest.mark.parametrize("kind", sorted(SC.CAP_KINDS))
def test_capacity_case_fills_its_list(kind):
    ids, row_off, slot_off = SC.capacity_case(kind, 8)
    mult = SC.CAP_KINDS[kind]
    assert ids.size == int(row_off[-1]) == SC.CTX_LIMIT and row_off.size == SC.CAP_S * SC.CAP_B + 1
    items, singles = 0, 0
    for s in range(SC.CAP_S):
        c = np.unique(ids[slot_off[s]:slot_off[s + 1]], return_counts=True)[1]
        assert set(c.tolist()) <= {1, mult}
        items += int((c == mult).sum())
        singles += int((c == 1).sum())
    # the list each kind fills, at the sizes pb_ctx_create gives it for 2^24 occurrences
    n = SC.CTX_LIMIT
    want = {"pairs": (n // 2, n // 2 + 1), "hot33": (n // 33, n // 33), "giant": (n // 1025, n // 1024 + 1)}[kind]
    assert items == want[0] and want[0] <= want[1] and want[1] - want[0] <= 17, (items, want)
    assert items * mult + singles == n and singles < mult


def test_many_slots_case_shape():
    ids = SC.many_slots_case(3)
    assert ids.size == SC.MANY_S * SC.MANY_B == 8_388_480 <= SC.CTX_LIMIT
    per_slot = ids.reshape(SC.MANY_S, SC.MANY_B)
    top = [np.unique(per_slot[s], return_counts=True)[1].max() for s in (0, 63, 127)]
    assert min(top) > 4096  # every slot has a giant hot id (> 1024 occurrences), of thousands of occurrences
    g = SC.many_slots_groups()
    assert len(set(g)) < SC.MANY_S and g.count(1) == 8 and {g[31], g[32]} != {g[63], g[64]}


def test_unique_case_is_distinct():
    ids, row_off = SC.unique_case(4)
    assert ids.size == SC.UNIQUE_N and np.unique(ids).size == SC.UNIQUE_N
    assert row_off.size == SC.UNIQUE_B + 1 == 65536 and int(row_off[-1]) == SC.UNIQUE_N
    assert SC.UNIQUE_N < SC.CTX_LIMIT


@pytest.mark.parametrize("n", SC.RAW_SIZES)
def test_raw_case_scan_trips(n):
    ids, row_off = SC.raw_case(5, n)
    assert ids.size == n and int(row_off[-1]) == n
    tiles, trips = SC.scan_geometry(n)
    want = {(1 << 20) - 1: (1024, 1), 1 << 20: (1024, 1), (1 << 20) + 1: (1025, 2), (1 << 20) + 1025: (1026, 2)}
    if n in want:
        assert (tiles, trips) == want[n]
    else:
        assert trips == 16 and n > SC.CTX_LIMIT - 8
    assert row_off.size == SC.RAW_B + 1
    lens = np.diff(row_off.astype(np.int64))
    assert (lens == 0).any() and (lens > SC.RAW_FIXED).any()
    assert set(SC.MARKERS.tolist()) <= set(ids[[0, n // 2, n - 1]].tolist())
    assert np.unique(ids).size > n // 3


def test_stage_case_sizes():
    from persia_b200.persia_core import ctx_occurrences

    ids, row_off = SC.stage_case(6)
    assert ids.size == SC.STAGE_N and int(row_off[-1]) == SC.STAGE_N and row_off.size == SC.STAGE_B + 1 == 65536
    assert np.unique(ids).size == SC.STAGE_POOL
    cap = ctx_occurrences(SC.STAGE_N, SC.STAGE_B)
    assert SC.CTX_LIMIT - 16 < cap <= SC.CTX_LIMIT
    # f32 staging at dim 1024: the context's max_occ would want 64 GB; the batch's ids want half of that
    assert cap * 1024 * 4 > 60e9 and SC.STAGE_N * 1024 * 4 < 35e9
