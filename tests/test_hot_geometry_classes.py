"""CPU-only: the geometry classes of the hot-sign reduce (k_reduce_hot) and the GPU cases that cover them.

pb_hot_geometry returns the geometry the launcher gives the kernel for a dim, a gradient dtype and a layout.  Over dims
1..4096, f16 and f32, one id per sample and ragged, it takes 78 classes (hot_geometry_cases.geometry_class).  Every class
must hold a dim that tests/test_gpu_hot_geometry.py runs in that layout."""
import collections

import pytest

from hot_geometry_cases import (ALL, HOT_COLS, ONE_ID_CASES, RAGGED_CASES, SEND_CASES, SGD, WINDOW_CASES,
                                geometry_class)

CLASSES = 78  # of the launcher at the time of writing; a change makes test_class_count say so


@pytest.fixture(scope="module")
def geo():
    from persia_b200 import build, shard

    build.build()
    return {(d, f16, rag): shard.hot_geometry(d, f16, rag) for d in range(1, 4097) for f16 in (False, True)
            for rag in (False, True)}


def _classes(geo):
    cl = collections.defaultdict(list)
    for (d, f16, rag), g in geo.items():
        cl[(f16,) + geometry_class(d, g)].append((d, rag))
    return cl


def test_class_count(geo):
    assert len(_classes(geo)) == CLASSES, f"{len(_classes(geo))} hot-reduce geometry classes (was {CLASSES})"


def test_every_class_has_a_gpu_case(geo):
    covered = {(f16,) + geometry_class(d, geo[(d, f16, False)]) for d, f16, _ in ONE_ID_CASES}
    covered |= {(f16,) + geometry_class(d, geo[(d, f16, True)]) for d, f16 in RAGGED_CASES}
    cl = _classes(geo)
    missing = {k: sorted(cl[k])[:4] for k in cl if k not in covered}
    assert not missing, f"{len(missing)} of {len(cl)} hot-reduce geometry classes have no GPU case: {missing}"


def test_optimizers_per_class(geo):
    """SGD at every case; per class one other optimizer, and all four at a dim with dim % EPL != 0 and at CH >= 3."""
    by_class = collections.defaultdict(list)
    for d, f16, kinds in ONE_ID_CASES:
        assert SGD in kinds, (d, f16)
        by_class[(f16,) + geometry_class(d, geo[(d, f16, False)])].append((d, kinds))
    for k, cases in by_class.items():
        assert any(len(kinds) > 1 for _, kinds in cases), k
        EPL, CH = k[1], k[2]
        if CH >= 3 or any(d % EPL for d, _ in cases):
            assert any(kinds == ALL and (CH >= 3 or d % EPL) for d, kinds in cases), k


def test_ragged_cases_are_the_lean_classes(geo):
    lean = {(d, f16) for d in range(1, 4097) for f16 in (False, True) if geo[(d, f16, False)]["lean"]}
    lean_classes = {(f16,) + geometry_class(d, geo[(d, f16, False)]) for d, f16 in lean}
    assert {(f16,) + geometry_class(d, geo[(d, f16, False)]) for d, f16 in RAGGED_CASES} == lean_classes
    for d, f16 in RAGGED_CASES:
        assert not geo[(d, f16, True)]["lean"]


def _mode(g):
    return "lean" if g["lean"] else ("pow2" if g["vec"] and g["vshift"] < 32 else ("vec" if g["vec"] else "elem"))


def test_window_and_send_cases_cover_their_groups(geo):
    one = {(d, f16): g for (d, f16, rag), g in geo.items() if not rag}
    modes = {(g["S"], _mode(g)) for g in one.values()}
    assert {(one[c]["S"], _mode(one[c])) for c in WINDOW_CASES} == modes
    groups = collections.defaultdict(set)
    for (d, f16), g in one.items():
        groups[(f16, g["EPL"], g["CH"], g["vec"], g["S"])].add(d)
    send = {(f16, one[(d, f16)]["EPL"], one[(d, f16)]["CH"], one[(d, f16)]["vec"], one[(d, f16)]["S"]): d
            for d, f16 in SEND_CASES}
    assert set(send) == set(groups)
    for k, d in send.items():
        assert d % 2 or not any(x % 2 for x in groups[k]), (k, d)


def test_geometry_values(geo):
    """Spot values of the launcher's arithmetic, and what every geometry must satisfy."""
    from persia_b200 import native as N, shard

    g = geo[(128, False, False)]  # f32 dim 128: chunks of 32 rows in four parts of 8
    assert (g["EPL"], g["CH"], g["PW"], g["R1"], g["R"], g["S"], g["lean"], g["vshift"]) == (2, 2, 6, 8, 32, 8, 1, 5)
    g = geo[(72, True, False)]
    assert (g["R1"], g["R"], g["S"], g["vec"], g["vshift"]) == (28, 112, 6, 1, 32)
    for (d, f16, rag), g in geo.items():
        assert g["cols"] == min(d, HOT_COLS) and g["stride"] == (g["cols"] + 3) // 4 * 4
        assert g["passes"] == (d + HOT_COLS - 1) // HOT_COLS
        assert g["CH"] * 32 * g["EPL"] >= g["cols"] and g["PW"] == min(8 - g["CH"], g["S"])
        assert g["R"] % 4 == 0 and g["R1"] <= 32 and g["R"] % g["R1"] == 0 and g["R"] // g["R1"] <= 4
        assert g["S"] * g["R"] * g["stride"] * 4 <= 6 * 32768
    for bad in (0, 4097):
        with pytest.raises(N.PersiaB200Error):
            shard.hot_geometry(bad, True)
