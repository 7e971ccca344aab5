"""CPU: PERSIA_B200_GROW (growable tables in persia_core) and its refusals, before any GPU work, and the growth
entry points in the symbol list."""
import pytest


def test_grow_parsing():
    from persia_b200.persia_core import growth_on

    assert growth_on(None) is False  # unset: tables reserve their capacity, as before
    assert growth_on("") is False
    assert growth_on("0") is False
    assert growth_on("1") is True
    assert growth_on(" 1 ", replica_size=1, hbm_rows="") is True
    with pytest.raises(RuntimeError, match="PERSIA_B200_GROW must be"):
        growth_on("yes")


def test_grow_refusals():
    from persia_b200.persia_core import growth_on

    with pytest.raises(RuntimeError, match="one GPU only"):
        growth_on("1", replica_size=2)
    with pytest.raises(RuntimeError, match="PERSIA_B200_HBM_ROWS"):
        growth_on("1", hbm_rows="4096")
    assert growth_on("0", replica_size=4, hbm_rows="4096") is False  # off: nothing to refuse


@pytest.mark.parametrize("env", [{"PERSIA_B200_GROW": "1"},
                                 {"PERSIA_B200_GROW": "1", "PERSIA_B200_HBM_ROWS": "1024"}])
def test_grow_refused_before_any_table_exists(monkeypatch, env):
    from persia_b200 import persia_core

    monkeypatch.delenv("PERSIA_B200_HBM_ROWS", raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    persia_core.reset()
    try:
        pc = persia_core.install()
        pc.set_embedding_config({"slots_config": {"s": {"dim": 8}}})
        pc.PersiaCommonContext(10, 0, 2 if len(env) == 1 else 1, None)
        with pytest.raises(RuntimeError, match="PERSIA_B200_GROW"):
            persia_core._S.group(8)
        assert not persia_core._S.groups
    finally:
        persia_core.reset()


def test_symbols():
    from persia_b200 import native as N

    assert N.SYMBOLS["pb_table_set_growth"][1] == [N._vp, N._i32]
    assert len(N.SYMBOLS["pb_table_storage_stats"][1]) == 3
