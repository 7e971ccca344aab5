"""CPU: how persia_core splits the summation slots of one dim into batch contexts (slot_chunks), how it sizes a pooled
context (ctx_occurrences), and that a batch context refuses more than PB_MAX_SLOTS slots."""
import numpy as np
import pytest

from persia_b200.native import PB_MAX_SLOTS
from persia_b200.persia_core import MAX_CTX_OCCURRENCES, ctx_occurrences, ctx_size, parse_embedding_config, slot_chunks


def _check(prefixes, chunks):
    """Every chunk holds at most PB_MAX_SLOTS slots in batch order, every slot sits in exactly one chunk and every
    feature group in one chunk; groups come in the order of their first slot."""
    flat = [i for c in chunks for i in c]
    assert sorted(flat) == list(range(len(prefixes)))
    for c in chunks:
        assert 0 < len(c) <= PB_MAX_SLOTS and c == sorted(c)
    where = {}
    for k, c in enumerate(chunks):
        for i in c:
            assert where.setdefault(prefixes[i], k) == k, "a feature group split across contexts"
    first = {}
    for i, p in enumerate(prefixes):
        first.setdefault(p, i)
    order = sorted(first, key=first.get)
    assert [where[p] for p in order] == sorted(where[p] for p in order)


@pytest.mark.parametrize("n", [1, 127, 128])
def test_up_to_128_slots_is_one_context_in_batch_order(n):
    """At most PB_MAX_SLOTS slots: one context holding them all, as before the split existed."""
    rng = np.random.default_rng(n)
    prefixes = rng.integers(0, 20, size=n).tolist()
    assert slot_chunks(prefixes) == [list(range(n))]


@pytest.mark.parametrize("n,want", [(129, [128, 1]), (256, [128, 128]), (300, [128, 128, 44])])
def test_single_slot_groups_fill_contexts_in_order(n, want):
    chunks = slot_chunks(list(range(n)))
    assert [len(c) for c in chunks] == want
    assert [i for c in chunks for i in c] == list(range(n))


def test_groups_are_never_split_and_packing_is_deterministic():
    """220 single-slot groups, one group of 50 slots and one of 30, interleaved: a group that does not fit the current
    context opens the next one, whole."""
    rng = np.random.default_rng(7)
    prefixes = [100 + i for i in range(220)] + [1] * 50 + [2] * 30
    perm = rng.permutation(len(prefixes))
    prefixes = [prefixes[i] for i in perm]
    chunks = slot_chunks(prefixes)
    _check(prefixes, chunks)
    assert len(chunks) == 3
    assert slot_chunks(list(prefixes)) == chunks  # the same slots give the same split (every rank issues the same calls)


def test_exactly_full_context_and_group_on_the_bound():
    """A group of exactly PB_MAX_SLOTS slots fills one context; the slots before it close theirs."""
    prefixes = [0, 1] + [9] * PB_MAX_SLOTS + [2]
    chunks = slot_chunks(prefixes)
    assert chunks == [[0, 1], list(range(2, 2 + PB_MAX_SLOTS)), [2 + PB_MAX_SLOTS]]
    _check(prefixes, chunks)


@pytest.mark.parametrize("seed", range(20))
def test_random_group_layouts(seed):
    rng = np.random.default_rng(seed)
    n_groups = int(rng.integers(1, 80))
    sizes = rng.integers(1, 60, size=n_groups)
    prefixes = np.repeat(np.arange(n_groups), sizes)
    prefixes = prefixes[rng.permutation(prefixes.size)].tolist()
    _check(prefixes, slot_chunks(prefixes))


def test_group_of_129_slots_is_refused():
    with pytest.raises(RuntimeError, match="129 summation slots"):
        slot_chunks([5] + [3] * (PB_MAX_SLOTS + 1))
    _check([3] * PB_MAX_SLOTS, slot_chunks([3] * PB_MAX_SLOTS))


def test_configured_feature_groups_map_to_chunks():
    """The prefixes parse_embedding_config gives: configured groups first, then one group per remaining slot."""
    cfg = {"slots_config": {f"s{i}": {"dim": 8} for i in range(300)},
           "feature_groups": {"a": [f"s{i}" for i in range(10, 60)], "b": [f"s{i}" for i in range(200, 230)]}}
    _, slots = parse_embedding_config(cfg)
    prefixes = [s.index_prefix for s in slots]
    assert len(set(prefixes)) == 222
    chunks = slot_chunks(prefixes)
    _check(prefixes, chunks)
    assert len(chunks) == 3


def test_context_sizing_is_clamped():
    """Twice the larger of the batch's ids and output rows, at least 1024, at most what pb_ctx_create accepts; a batch
    of more ids than that is refused with a message that counts its ids."""
    assert MAX_CTX_OCCURRENCES == 1 << 24
    assert ctx_occurrences(1) == 1024
    assert ctx_occurrences(5000) == 10000
    assert ctx_occurrences(100, 5000) == 10000  # (a ragged batch with empty samples)
    assert ctx_occurrences(1 << 23) == 1 << 24
    assert ctx_occurrences((1 << 23) + 1) == 1 << 24
    assert ctx_occurrences(1 << 24) == 1 << 24
    assert ctx_occurrences(1000, 128 * 65535) == 2 * 128 * 65535  # rows alone never refuse a batch
    with pytest.raises(RuntimeError, match=f"holds {(1 << 24) + 1} ids.*2\\^24"):
        ctx_occurrences((1 << 24) + 1)
    # (occurrences, output rows): twice the rows, at least 1024, never less than the context being replaced holds
    assert ctx_size(1600, 8) == (3200, 1024)
    assert ctx_size(2048, 2048) == (4096, 4096)
    assert ctx_size(10, 3, held=(5000, 2000)) == (5000, 2000)


def test_batch_context_refuses_more_than_128_slots():
    from persia_b200 import shard as SH

    with pytest.raises(ValueError, match="PB_MAX_SLOTS = 128"):
        SH.BatchContext(1024, 1024, list(range(PB_MAX_SLOTS + 1)))
