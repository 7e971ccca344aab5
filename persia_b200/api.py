"""The `persia` Python API over libpersia_b200 — host-side mirror of the reference's user-facing layer.

The reference's `persia/ctx.py`, `persia/embedding/{__init__,optim,data}.py` sit on the PyO3 module `persia_core`.
persia_b200.persia_core re-exposes that module surface (tests/test_persia_core_surface.py).  This module provides
the same names, arguments and behaviour as the reference's `persia` package, written from scratch against the same
surface, so that a user script

    from persia_b200.api import TrainCtx, PersiaBatch, IDTypeFeatureWithSingleID, Label, NonIDTypeFeature, Adagrad, EmbeddingConfig

reads like one written against `persia.ctx` / `persia.embedding.*` (reference line numbers in every docstring).
The dense tower is the user's `torch.nn.Module`, called as `model(non_id_type_tensors, embedding_tensors)`
(persia/ctx.py:446-448); at world size > 1 it is wrapped in DistributedDataParallel (persia/distributed.py:174-191)
and the sparse path goes through the sharded worker.
"""
import os
from enum import Enum
from queue import Queue

import numpy as np
import torch

from . import persia_core as PC

MAX_BATCH_SIZE = 65535  # persia/embedding/data.py:14


# ---- persia/embedding/__init__.py:4-26 ------------------------------------------------------------------------------
class EmbeddingConfig:
    def __init__(self, emb_initialization=(-0.01, 0.01), admit_probability=1.0, weight_bound=10):
        self.emb_initialization = emb_initialization
        self.admit_probability = admit_probability
        self.weight_bound = weight_bound


def get_default_embedding_config():
    return EmbeddingConfig()


# ---- persia/embedding/optim.py --------------------------------------------------------------------------------------
class Optimizer:
    def __init__(self):
        self.optimizer_base = PC.OptimizerBase()

    def apply(self):  # optim.py:11-16: register on every parameter server
        self.optimizer_base.apply()


class SGD(Optimizer):  # optim.py:18-33
    def __init__(self, lr, momentum=0.0, weight_decay=0.0):
        super().__init__()
        self.lr, self.momentum, self.weight_decay = lr, momentum, weight_decay
        self.optimizer_base.init_sgd(self.lr, self.weight_decay)


class Adam(Optimizer):  # optim.py:35-58
    def __init__(self, lr=1e-3, betas=(0.9, 0.999), weight_decay=0, eps=1e-8):
        super().__init__()
        self.lr, self.betas, self.weight_decay, self.eps = lr, betas, weight_decay, eps
        self.optimizer_base.init_adam(self.lr, self.betas, self.eps)


class Adagrad(Optimizer):  # optim.py:60-96
    def __init__(self, lr=1e-2, initial_accumulator_value=1e-2, weight_decay=0, g_square_momentum=1, eps=1e-10,
                 vectorwise_shared=False):
        super().__init__()
        self.lr, self.initial_accumulator_value, self.weight_decay = lr, initial_accumulator_value, weight_decay
        self.g_square_momentum, self.eps, self.vectorwise_shared = g_square_momentum, eps, vectorwise_shared
        self.optimizer_base.init_adagrad(self.lr, self.weight_decay, self.g_square_momentum, self.initial_accumulator_value,
                                         self.eps, self.vectorwise_shared)


# ---- persia/embedding/data.py -----------------------------------------------------------------------------------------
_ND_TYPES = (np.bool_, np.int8, np.int16, np.int32, np.int64, np.float32, np.float64, np.uint8)  # data.py:20-29


def _batch_size_check(batch_size, target_batch_size, data_type, name):  # data.py:59-66
    assert batch_size == target_batch_size, \
        f"expected {data_type}: {name} batch_size equal to {target_batch_size} but got {batch_size}"
    assert batch_size <= MAX_BATCH_SIZE, \
        f"expected {data_type}:{name} batch_size <= MAX_BATCH_SIZE: {MAX_BATCH_SIZE} but got {batch_size}"


class IDTypeFeature:  # data.py:69-113: LIL, a variable number of ids per sample
    def __init__(self, name, data):
        (x.dtype == np.uint64 for x in data)
        for x in data:
            assert isinstance(x, np.ndarray) and x.ndim == 1 and x.dtype == np.uint64, \
                "IDTypeFeature expects a list of 1-D uint64 ndarrays"
        self.name, self.data = name, data

    @property
    def batch_size(self):
        return len(self.data)


class IDTypeFeatureWithSingleID:  # data.py:116-157: one id per sample
    def __init__(self, name, data):
        assert isinstance(data, np.ndarray) and data.ndim == 1 and data.dtype == np.uint64, \
            "IDTypeFeatureWithSingleID expects a 1-D uint64 ndarray"
        self.name, self.data = name, data

    @property
    def batch_size(self):
        return len(self.data)


class NdarrayDataBase:  # data.py:160-214
    DEFAULT_NAME = "ndarray_base"

    def __init__(self, data, name=None):
        assert isinstance(data, np.ndarray), f"expected ndarray but got {type(data)}"
        assert data.ndim > 0 and data.dtype.type in _ND_TYPES, f"unsupported ndarray {data.dtype} with ndim {data.ndim}"
        self.data, self._name = data, name

    @property
    def batch_size(self):
        return self.data.shape[0]

    @property
    def name(self):
        return self._name or self.DEFAULT_NAME

    def __len__(self):
        return len(self.data)


class Label(NdarrayDataBase):  # data.py:217-253
    DEFAULT_NAME = "label_anonymous"


class NonIDTypeFeature(NdarrayDataBase):  # data.py:256-276
    DEFAULT_NAME = "non_id_type_feature_anonymous"


class PersiaBatch:  # data.py:279-411
    def __init__(self, id_type_features, non_id_type_features=None, labels=None, batch_size=None, requires_grad=True,
                 meta=None):
        assert len(id_type_features) > 0, "id_type_features should not be empty"
        batch_size = batch_size or id_type_features[0].batch_size
        self.batch = PC.PersiaBatch()
        for f in id_type_features:
            _batch_size_check(f.batch_size, batch_size, "id_type_feature", f.name)
            if isinstance(f, IDTypeFeatureWithSingleID):
                self.batch.add_id_type_feature_with_single_id(f.data, f.name)
            elif isinstance(f, IDTypeFeature):
                self.batch.add_id_type_feature(f.data, f.name)
            else:
                raise TypeError("expected type of id_type_feature to be Union[IDTypeFeatureWithSingleID, IDTypeFeature] "
                                f"but got {type(f)}")
        for f in non_id_type_features or []:
            _batch_size_check(f.batch_size, batch_size, "non_id_type_feature", f.name)
            self.batch.add_non_id_type_feature(f.data, f.data.dtype, f.name)
        for lb in labels or []:
            _batch_size_check(lb.batch_size, batch_size, "label", lb.name)
            self.batch.add_label(lb.data, lb.data.dtype, lb.name)
        if meta is not None and isinstance(meta, bytes):
            self.batch.add_meta(meta)
        self.batch_size = batch_size
        self.batch.converted_id_type_features2embedding_tensor(requires_grad)

    @property
    def data(self):
        return self.batch

    def to_bytes(self):
        return self.data.to_bytes()


# ---- persia/ctx.py ------------------------------------------------------------------------------------------------------
class PreprocessMode(Enum):  # ctx.py:57-72
    TRAIN = 1
    EVAL = 2
    INFERENCE = 3


_CURRENT_CXT = None


def cnt_ctx():  # ctx.py:1058-1060
    return _CURRENT_CXT


def _to_torch(tensor, requires_grad=False):
    """ctx.py:40-55 `_cast_dlpack2torch_tensor`: the surface's Tensor -> torch view through DLPack."""
    import torch.utils.dlpack as dl

    t = dl.from_dlpack(tensor.dlpack)
    t.requires_grad = requires_grad
    return t


def _prepare_feature(batch, mode=PreprocessMode.TRAIN):
    """ctx.py:75-199.  Summation slots: the f16 [batch, dim] tensor, requires_grad in training.  Raw slots:
    index_select of the distinct-sign table + the mask channel, [batch, sample_fixed_size, dim + 1]."""
    if mode == PreprocessMode.INFERENCE:
        batch.label_torch_tensors = None
    else:
        batch.label_tensors = batch.consume_all_label_tensors()
        batch.label_torch_tensors = [_to_torch(t) for t in batch.label_tensors]
    training = mode == PreprocessMode.TRAIN
    batch.non_id_type_feature_tensors = batch.consume_all_non_id_type_feature_tensors()
    batch.non_id_type_feature_torch_tensors = [_to_torch(t) for t in batch.non_id_type_feature_tensors]
    batch.id_type_feature_embedding_tensors = batch.consume_all_id_type_feature_embedding_tensors()
    batch.emb_slots = []  # keeps the surface tensors alive while torch views exist
    cache, feats = [], []
    for e in batch.id_type_feature_embedding_tensors:
        if e.is_raw_embedding():
            raw, index, non_empty, sample_id_num = e.get_raw_embedding()
            batch.emb_slots.append([raw, index, non_empty])
            distinct = _to_torch(raw)
            index_t = _to_torch(index)
            assert index_t.max() < distinct.shape[0], "raw embedding select index larger than tensor"
            non_empty_t = _to_torch(non_empty)
            bsz, dim = len(sample_id_num), distinct.shape[-1]
            fixed = index_t.shape[-1] // bsz
            sel = distinct.index_select(0, index_t.view(-1))
            sel.requires_grad = training
            mask = (index_t.view(bsz, fixed, 1) != 0).half()
            cache.append((raw.name, distinct, index_t, non_empty_t, sel))
            feats.append(torch.cat([sel.view(-1, fixed, dim), mask], dim=2))
        else:
            emb = e.get_sum_embedding()
            batch.emb_slots.append([emb])
            t = _to_torch(emb, requires_grad=training)
            feats.append(t)
            cache.append((emb.name, None, None, None, t))
    batch.id_type_feature_embedding_torch_tensors = feats
    batch.id_type_feature_embedding_cache_torch_tensors = cache
    return batch.non_id_type_feature_torch_tensors, feats, batch.label_torch_tensors


def _check_finite(tensors):  # ctx.py:58 helper
    return all(bool(torch.isfinite(t).all()) for t in tensors if t is not None)


def _rank_world():
    """persia/env.py:29-56: RANK / WORLD_SIZE (torchrun) or REPLICA_INDEX / REPLICA_SIZE."""
    if "RANK" in os.environ:
        return int(os.environ["RANK"]), int(os.environ.get("WORLD_SIZE", "1"))
    return int(os.environ.get("REPLICA_INDEX", "0")), int(os.environ.get("REPLICA_SIZE", "1"))


class BaseCtx:  # ctx.py:202-271
    def __init__(self, threadpool_worker_size=10, device_id=None):
        self.origin_context = None
        if device_id is not None and device_id >= 0:
            assert torch.cuda.is_available() and 0 <= device_id < torch.cuda.device_count(), f"device_id: {device_id} invalid!"
            torch.cuda.set_device(device_id)
        else:
            device_id = None
        self.device_id = device_id
        rank, world = _rank_world()
        self.common_context = PC.PersiaCommonContext(threadpool_worker_size, rank, world, device_id)

    def _enter(self):
        ...

    def _exit(self):
        ...

    def __enter__(self):
        global _CURRENT_CXT
        self._enter()
        self.origin_context = _CURRENT_CXT
        _CURRENT_CXT = self
        return self

    def __exit__(self, exc_type, value, trace):
        global _CURRENT_CXT
        self._exit()
        _CURRENT_CXT = self.origin_context


class EmbeddingCtx(BaseCtx):  # ctx.py:345-652
    def __init__(self, preprocess_mode, model=None, embedding_config=None, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.preprocess_mode = preprocess_mode
        self.model = model
        self.embedding_config = embedding_config or get_default_embedding_config()
        self.current_batch = None

    def _enter(self):
        if self.embedding_config is not None:
            self.configure_embedding_parameter_servers(self.embedding_config)

    def configure_embedding_parameter_servers(self, embedding_config):  # ctx.py:415-431
        self.common_context.configure_embedding_parameter_servers(
            embedding_config.emb_initialization[0], embedding_config.emb_initialization[1],
            embedding_config.admit_probability, embedding_config.weight_bound > 0, embedding_config.weight_bound)

    def forward(self, batch):  # ctx.py:433-448
        assert self.model is not None, "model not found, please init context with model"
        non_id, emb, labels = self.prepare_features(batch)
        return self.model(non_id, emb), labels

    def prepare_features(self, batch):  # ctx.py:450-476
        self.current_batch = batch
        return _prepare_feature(batch, self.preprocess_mode)

    def get_embedding_from_data(self, persia_batch, device_id=None):  # ctx.py:620-635
        return self.common_context.get_embedding_from_data(persia_batch.data, device_id if device_id is not None else self.device_id)

    def get_embedding_from_bytes(self, data, device_id=None):  # ctx.py:637-652
        return self.common_context.get_embedding_from_bytes(data, device_id if device_id is not None else self.device_id)

    def dump_embedding(self, dst_dir, blocking=True):  # ctx.py:535-553
        self.common_context.dump(dst_dir)
        if blocking:
            self.common_context.wait_for_emb_dumping()

    def load_embedding(self, src_dir, blocking=True):  # ctx.py:515-533
        self.common_context.load(src_dir)
        if blocking:
            self.common_context.wait_for_emb_loading()

    def get_embedding_size(self):
        return self.common_context.get_embedding_size()

    def clear_embeddings(self):
        self.common_context.clear_embeddings()


def eval_ctx(*args, **kwargs):  # ctx.py:1063-1074
    return EmbeddingCtx(PreprocessMode.EVAL, *args, **kwargs)


class TrainCtx(EmbeddingCtx):  # ctx.py:655-1055
    def __init__(self, embedding_optimizer, dense_optimizer, grad_scalar_update_factor=4, backward_buffer_size=10,
                 backward_workers_size=8, grad_update_buffer_size=60, lookup_emb_directly=True, mixed_precision=True,
                 distributed_option=None, *args, **kwargs):
        super().__init__(PreprocessMode.TRAIN, *args, **kwargs)
        assert embedding_optimizer is not None, "EmbeddingOptimizer should not be none in train context"
        assert grad_scalar_update_factor > 0, "grad scalar should greater than zero"
        assert self.model is not None, "Model not found, please init context with pytorch model"
        self.rank_id, self.world_size = _rank_world()
        assert not mixed_precision or torch.cuda.is_available(), "Mixed precision training only support on cuda device."
        self.mixed_precision = mixed_precision
        if mixed_precision:
            self.grad_scalar_update_factor = grad_scalar_update_factor
            self.grad_scaler = torch.amp.GradScaler("cuda")
            self.update_times = 0
        if self.world_size > 1:
            # persia/distributed.py:174-191 (DDPOption.convert2distributed_model): the dense tower is data parallel
            import torch.distributed as dist

            if not dist.is_initialized():
                backend = (distributed_option or {}).get("backend", "nccl") if isinstance(distributed_option, dict) else "nccl"
                dist.init_process_group(backend, rank=self.rank_id, world_size=self.world_size)
            ids = [self.device_id] if self.device_id is not None else None
            self.model = torch.nn.parallel.DistributedDataParallel(self.model, device_ids=ids, find_unused_parameters=True)
        self.dense_optimizer = dense_optimizer
        self.embedding_optimizer = embedding_optimizer
        self.common_context.wait_servers_ready()
        self.backward_workers_size = backward_workers_size
        self.grad_queue = Queue(grad_update_buffer_size)  # keeps the gradient tensors alive (ctx.py:851, 935-936, 999)
        self.backward_engine = PC.Backward(backward_buffer_size)

    def _enter(self):
        super()._enter()
        self.embedding_optimizer.apply()
        self.backward_engine.launch(self.backward_workers_size)

    def _exit(self):
        super()._exit()
        self.backward_engine.shutdown()

    def backward(self, loss, embedding_gradient_check_frequency=20):  # ctx.py:893-924
        if self.mixed_precision:
            loss = self.grad_scaler.scale(loss)
            scale = self.grad_scaler.get_scale()
        else:
            scale = 1
        loss.backward()
        finite = self._on_backward(scale, embedding_gradient_check_frequency)
        if self.mixed_precision:
            self.grad_scaler.step(self.dense_optimizer)
            if finite:
                self.grad_scaler.update()
            else:
                self.grad_scaler.update(scale / self.grad_scalar_update_factor)
        else:
            self.dense_optimizer.step()
        self.dense_optimizer.zero_grad()
        return loss

    def _on_backward(self, loss_scale, embedding_gradient_check_frequency):  # ctx.py:926-1005
        if self.grad_queue.full():
            self.grad_queue.get()
        finite = True
        if self.mixed_precision and self.update_times % embedding_gradient_check_frequency == 0:
            finite = _check_finite([c[-1].grad for c in self.current_batch.id_type_feature_embedding_cache_torch_tensors])
            self.update_times += 1
        grad_slots = []
        gradient_batch = self.current_batch.create_gradient_batch()
        for name, distinct, index, non_zero_index, emb in self.current_batch.id_type_feature_embedding_cache_torch_tensors:
            if emb.grad is None:
                gradient_batch.add_skipped_gradient(name)
                continue
            if distinct is not None:  # raw slot: [U, dim] f32 gradient of the distinct-sign table without its row 0
                if distinct.shape[0] > 1:
                    grad = torch.zeros_like(distinct, dtype=torch.float32)
                    nz = emb.grad.index_select(0, non_zero_index.view(-1)).float()
                    grad.index_add_(0, index.view(-1)[non_zero_index.view(-1)], nz)
                    grad = grad[1:, :].contiguous()
                    is_f16 = False
                else:
                    grad = None
            else:
                grad = emb.grad
                is_f16 = True
            if grad is not None:
                grad_slots.append(grad)
                gradient_batch.add_gradient(name, grad.data_ptr(), grad.shape, is_f16, loss_scale)
        # The reference synchronises the device here (ctx.py:995-996): its backward engine copies the gradients to the host
        # on another stream.  Here the engine's workers enqueue pb_backward on the SAME stream the autograd kernels ran on
        # (the device's default stream), after them in host order, so stream order already makes the gradients ready;
        # grad_queue keeps the tensors alive until the update has been enqueued.  Should the caller have run autograd on
        # another stream, the event recorded here orders the worker's stream after it.
        if self.device_id is not None:
            ready = torch.cuda.Event()
            ready.record()
            gradient_batch._ready = ready
        self.backward_engine.update_id_type_feature_gradient_batched(gradient_batch)
        self.grad_queue.put(grad_slots)
        return finite

    def dump_checkpoint(self, dst_dir, dense_model_filename="dense.pt", jit_dense_model_filename="jit_dense.pt",
                        opt_filename="opt.pt", blocking=True, with_jit_model=False):  # ctx.py:1007-1037
        os.makedirs(dst_dir, exist_ok=True)
        torch.save(self.model.state_dict(), os.path.join(dst_dir, dense_model_filename))
        torch.save(self.dense_optimizer.state_dict(), os.path.join(dst_dir, opt_filename))
        self.dump_embedding(dst_dir, blocking=blocking)

    def load_checkpoint(self, src_dir, map_location=None, dense_model_filename="dense.pt", opt_filename="opt.pt",
                        blocking=True):  # ctx.py:1039-1055
        mp = os.path.join(src_dir, dense_model_filename)
        if os.path.exists(mp):
            self.model.load_state_dict(torch.load(mp, map_location=map_location))
        op = os.path.join(src_dir, opt_filename)
        if os.path.exists(op):
            self.dense_optimizer.load_state_dict(torch.load(op, map_location=map_location))
        self.load_embedding(src_dir, blocking=blocking)
