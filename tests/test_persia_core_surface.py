"""CPU: the `persia_core` surface (SURVEY.md §8b): the module layout `persia/prelude.py` expects, the batch
semantics and the host-side hashing."""
import os
import types

import numpy as np
import pytest


@pytest.fixture()
def pc():
    from persia_b200 import persia_core

    persia_core.reset()
    yield persia_core.install()
    persia_core.reset()


def test_module_layout_matches_prelude(pc):
    import persia_core
    from persia_core import PersiaCommonContext, is_cuda_feature_available  # noqa: F401
    from persia_core.backward import Backward  # noqa: F401
    from persia_core.data import PersiaBatch, check_pyarray_dtype_valid  # noqa: F401
    from persia_core.forward import Forward, PersiaTrainingBatch, Tensor  # noqa: F401
    from persia_core.nats import initialize_dataflow  # noqa: F401
    from persia_core.optim import OptimizerBase  # noqa: F401
    from persia_core.utils import (PersiaBatchDataChannel, PersiaBatchDataReceiver, PersiaBatchDataSender,  # noqa: F401
                                   PersiaMessageQueueClient, PersiaMessageQueueServer)

    for sub in ("data", "forward", "backward", "optim", "utils", "nats"):
        assert isinstance(getattr(persia_core, sub), types.ModuleType)
    ctx = PersiaCommonContext(10, 0, 1, None)
    for name in ("init_nats_publisher", "init_master_discovery_service", "get_embedding_worker_addr_list",
                 "init_rpc_client_with_addr", "wait_servers_ready", "get_embedding_size", "clear_embeddings", "dump", "load",
                 "wait_for_serving", "wait_for_emb_loading", "wait_for_emb_dumping", "shutdown_servers",
                 "send_id_type_features_to_embedding_worker", "send_non_id_type_features_to_nn_worker",
                 "configure_embedding_parameter_servers", "get_embedding_from_data", "get_embedding_from_bytes",
                 "read_from_file", "dump_to_file", "set_embedding"):
        assert callable(getattr(ctx, name)), name
    assert isinstance(ctx.master_addr, str)
    two = PersiaCommonContext(10, 1, 2, None)  # R GPUs: accepted; the sharded worker is built by the first batch
    assert two.get_embedding_worker_addr_list() == ["local"]
    PersiaCommonContext(10, 0, 1, None)


def test_prefix_rule_and_batch_semantics(pc):
    from persia_b200.persia_core import parse_embedding_config

    bits, slots = parse_embedding_config({
        "feature_index_prefix_bit": 12,
        "slots_config": {"a": {"dim": 8}, "b": {"dim": 8}, "c": {"dim": 16, "sqrt_scaling": True}},
        "feature_groups": {"g": ["b", "c"]},
    })
    by = {s.name: s for s in slots}
    assert bits == 12
    assert by["b"].index_prefix == by["c"].index_prefix == 1 << 52  # explicit groups first
    assert by["a"].index_prefix == 2 << 52                          # then one group per remaining slot
    b = pc.data.PersiaBatch()
    b.add_id_type_feature_with_single_id(np.arange(4, dtype=np.uint64), "a")
    with pytest.raises(RuntimeError):  # data.rs:236-240
        b.converted_id_type_features2embedding_tensor(True)
    b = pc.data.PersiaBatch()
    b.add_id_type_feature([np.array([1, 2], np.uint64), np.array([], np.uint64)], "a")
    b.add_label(np.zeros((2, 1), np.float32), np.dtype(np.float32), "y")
    b.converted_id_type_features2embedding_tensor(True)
    assert isinstance(b.to_bytes(), bytes)
    with pytest.raises(RuntimeError):
        b.batch_id()
    with pytest.raises(RuntimeError):  # FeatureBatch::new panics above u16::MAX samples
        pc.data.PersiaBatch().add_id_type_feature_with_single_id(np.zeros(65536, np.uint64), "a")
    ch = pc.utils.PersiaBatchDataChannel(4)
    fwd = pc.forward.Forward(8, False, 1)
    fwd.set_input_channel(ch.get_receiver())
    with pytest.raises(RuntimeError):
        fwd.set_input_channel(ch.get_receiver())
    fwd.launch(2)
    with pytest.raises(TimeoutError):  # forward.rs:875
        fwd.get_batch(5)


def test_farmhash_numpy_matches_golden(pc):
    import json

    from persia_b200.persia_core import SlotConfig, _hashstack, farmhash64_np

    fx = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "farmhash64_kat.json")))
    ids = np.array([int(k) for k in fx["hash64"]], np.uint64)
    np.testing.assert_array_equal(farmhash64_np(ids), np.array([int(v, 16) for v in fx["hash64"].values()], np.uint64))
    slot = SlotConfig("t", 32, hash_stack_rounds=2, hash_stack_embedding_size=10)
    got = _hashstack(ids, slot)  # the reference's own test vector (mod.rs:1570-1613)
    assert [g.tolist() for g in got] == [list(v) for v in fx["hashstack_rounds2_size10"].values()]
