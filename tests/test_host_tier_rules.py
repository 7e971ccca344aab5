"""CPU: how persia_core splits a table between HBM and a host-memory tier (PERSIA_B200_HBM_ROWS), before any GPU work."""
import pytest


def test_split_rules():
    from persia_b200.persia_core import hbm_split

    assert hbm_split(1 << 20, None) == (1 << 20, 0)  # unset: everything in HBM, as before
    assert hbm_split(1 << 20, "") == (1 << 20, 0)
    assert hbm_split(1 << 20, str(1 << 20)) == (1 << 20, 0)  # HBM rows >= capacity: no tier
    assert hbm_split(1000, "5000", replica_size=4) == (1000, 0)
    assert hbm_split(1 << 20, "4096") == (4096, (1 << 20) - 4096)
    with pytest.raises(RuntimeError, match="one GPU only"):
        hbm_split(1 << 20, "4096", replica_size=2)
    with pytest.raises(RuntimeError, match="positive"):
        hbm_split(1 << 20, "0")


def test_tier_on_r_gpus_is_refused_before_any_table_exists(monkeypatch):
    from persia_b200 import persia_core

    monkeypatch.setenv("PERSIA_B200_HBM_ROWS", "1024")
    persia_core.reset()
    try:
        pc = persia_core.install()
        pc.set_embedding_config({"slots_config": {"s": {"dim": 8}}})
        pc.PersiaCommonContext(10, 0, 2, None)
        with pytest.raises(RuntimeError, match="PERSIA_B200_HBM_ROWS"):
            persia_core._S.group(8)
        assert not persia_core._S.groups
    finally:
        persia_core.reset()
