"""CPU: the rules `persia_core` enforces for raw slots on R GPUs before any GPU work.  The calls of a step are collective,
so every rank must issue them in one order (raw slots in batch order, then summation dims), and a raw slot may not
share its feature group with another slot of the batch."""
import numpy as np
import pytest


@pytest.fixture()
def pc():
    from persia_b200 import persia_core

    persia_core.reset()
    yield persia_core.install()
    persia_core.reset()


def _batch(pc, feats, B=3):
    b = pc.data.PersiaBatch()
    for name in feats:
        b.add_id_type_feature([np.array([1, 2], np.uint64)] + [np.array([7], np.uint64)] * (B - 1), name)
    b.add_label(np.zeros((B, 1), np.float32), np.dtype(np.float32), "y")
    b.converted_id_type_features2embedding_tensor(True)
    return b


def test_raw_slot_sharing_a_feature_group_is_rejected_on_r_gpus(pc):
    pc.set_embedding_config({"slots_config": {"r": {"dim": 8, "embedding_summation": False}, "s": {"dim": 8}},
                             "feature_groups": {"g": ["r", "s"]}})
    ctx = pc.PersiaCommonContext(10, 0, 2, None)
    with pytest.raises(RuntimeError, match="feature group"):
        ctx.get_embedding_from_data(_batch(pc, ["r", "s"]), 0)


def test_raw_slots_must_keep_their_order_on_r_gpus(pc):
    from persia_b200 import persia_core as PC

    pc.set_embedding_config({"slots_config": {"a": {"dim": 8, "embedding_summation": False},
                                              "b": {"dim": 8, "embedding_summation": False}, "s": {"dim": 8}}})
    ctx = pc.PersiaCommonContext(10, 0, 2, None)
    PC._S.raw_order = ("a", "b")  # what the first batch of this process carried
    for feats in (["b", "a", "s"], ["a", "s"], ["b"], ["s"]):  # another order, a slot missing, no raw slot at all
        with pytest.raises(RuntimeError, match="same raw slots"):
            ctx.get_embedding_from_data(_batch(pc, feats), 0)
