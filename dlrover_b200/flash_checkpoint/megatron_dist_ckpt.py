"""Megatron-LM checkpoint save/load that keeps the DISTRIBUTED optimizer state
distributed: every rank checkpoints its own main_param / exp_avg / exp_avg_sq
shards instead of gathering them on data-parallel rank 0.

Reference @ 468d632: dlrover/trainer/torch/flash_checkpoint/megatron_dist_ckpt.py
  save_checkpoint (:178-299), get_dist_optimizer_checkpoint_name (:300-313:
  "<save>/iter_XXXXXXX/rank_NNNNN/distrib_optim.pt"), get_parameter_state
  (:316-358), load_checkpoint (:372-583), _load_checkpoint_from_memory (:585),
  _load_base_checkpoint (:594-651), load_parameter_state_from_state_dict
  (:654-683), deletion strategies keyed on "iter_XXXXXXX" (:78-141).

What changes underneath: the per-rank shard dict goes through the gather
kernel like any other state dict, and on restore from memory the optimizer
shards are scattered into the live fp32 tensors by ONE DMA fill + scatter
kernel (`CheckpointEngine.load_into`) instead of one `copy_` per tensor (:683).

Megatron-LM is resolved lazily through `_mlm()`; nothing here imports it at
module import time.
"""

from __future__ import annotations

import os
import random
import sys
from types import SimpleNamespace
from typing import List

import numpy as np
import torch
import torch.distributed as dist

from ..common.constants import CheckpointConstant
from ..common.log import default_logger as logger
from ..common.singleton import Singleton
from ..common.storage import (
    CheckpointDeletionStrategy,
    PosixDiskStorage,
    PosixStorageWithDeletion,
)
from .api import StorageType
from .engine import MegatronCheckpointEngine, MegatronDistCheckpointEngine

_MODEL = CheckpointConstant.MODEL_STATES_NAME
_OPTIM = CheckpointConstant.OPTIM_STATES_NAME

_bindings = None


def _mlm():
    """Megatron-LM symbols this module needs (new `megatron.training` layout
    first, then the pre-core layout).  Override with `bind_megatron(ns)`."""
    global _bindings
    if _bindings is not None:
        return _bindings
    ns = SimpleNamespace()
    try:
        from megatron.core import mpu, tensor_parallel
        from megatron.core.num_microbatches_calculator import update_num_microbatches
        from megatron.core.optimizer.optimizer import ChainedOptimizer
        from megatron.training import checkpointing as ck
        from megatron.training import get_args
        from megatron.training.utils import print_rank_0, unwrap_model
    except ImportError:
        from megatron import checkpointing as ck
        from megatron import get_args, mpu, update_num_microbatches
        from megatron.core import tensor_parallel
        from megatron.optimizer.optimizer import ChainedOptimizer
        from megatron.utils import print_rank_0, unwrap_model
    ns.mpu, ns.tensor_parallel, ns.get_args = mpu, tensor_parallel, get_args
    ns.update_num_microbatches, ns.ChainedOptimizer = update_num_microbatches, ChainedOptimizer
    ns.print_rank_0, ns.unwrap_model = print_rank_0, unwrap_model
    for name in ("check_checkpoint_args", "find_checkpoint_rank_0",
                 "fix_query_key_value_ordering", "get_checkpoint_name",
                 "get_checkpoint_tracker_filename", "get_checkpoint_version", "get_rng_state",
                 "read_metadata", "set_checkpoint_version"):
        setattr(ns, name, getattr(ck, name))
    _bindings = ns
    return ns


def bind_megatron(namespace):
    """Inject the Megatron symbols (tests, forks with a different layout)."""
    global _bindings
    _bindings = namespace


def _iter_dir(step: int) -> str:
    return "iter_{:07d}".format(step)


class KeepStepIntervalStrategy(CheckpointDeletionStrategy):
    """Keep only iterations that are multiples of `keep_interval`
    (Megatron directory naming: iter_XXXXXXX)."""

    def __init__(self, keep_interval: int, checkpoint_dir: str):
        self._keep_interval = keep_interval
        self._checkpoint_dir = checkpoint_dir

    def clean_up(self, step, delete_func):
        if step % self._keep_interval == 0:
            return
        victim = os.path.join(self._checkpoint_dir, _iter_dir(step))
        try:
            delete_func(victim)
            logger.info(f"Clean path {victim}")
        except Exception:
            logger.warning(f"Fail to clean path {victim}!")


class KeepLatestStepStrategy(CheckpointDeletionStrategy):
    """Keep the newest `max_to_keep` iterations."""

    def __init__(self, max_to_keep: int, checkpoint_dir: str):
        self._max_to_keep = max(max_to_keep, 1)
        self._checkpoint_dir = checkpoint_dir
        self._steps: List[int] = []

    def clean_up(self, step, delete_func):
        self._steps.append(step)
        if len(self._steps) != self._max_to_keep:
            return
        victim = os.path.join(self._checkpoint_dir, _iter_dir(self._steps.pop(0)))
        try:
            delete_func(victim)
            logger.info(f"Clean path {victim}")
        except Exception:
            logger.warning(f"Fail to clean path {victim}!")


def get_checkpoint_storage(deletion_strategy=None):
    if deletion_strategy:
        return PosixStorageWithDeletion(tracker_file=CheckpointConstant.TRACER_FILE_NAME,
                                        deletion_strategy=deletion_strategy)
    return PosixDiskStorage()


class MegatronDistCheckpointer(Singleton):
    def __init__(self, checkpoint_dir, storage=None, comm_backend="",
                 use_distributed_optimizer=False, save_timeout=CheckpointConstant.SAVE_TIMEOUT,
                 async_drain=None):
        self.storage = storage if storage else PosixDiskStorage()
        engine_cls = (MegatronDistCheckpointEngine if use_distributed_optimizer
                      else MegatronCheckpointEngine)
        self.engine = engine_cls(checkpoint_dir=checkpoint_dir, storage=self.storage,
                                 comm_backend=comm_backend, save_timeout=save_timeout,
                                 async_drain=async_drain)


def get_dist_optimizer_checkpoint_name(checkpoints_path, iteration, release=False):
    directory = "release" if release else _iter_dir(iteration)
    rank = dist.get_rank() if dist.is_initialized() else 0
    return os.path.join(checkpoints_path, directory, f"rank_{rank:05d}", "distrib_optim.pt")


# ------------------------------------------------- distributed-optimizer shards --


def _walk_param_shards(dist_optimizer):
    """Yield (bucket_idx, group_index, group_order, tensors) for every model
    parameter this rank owns a shard of; tensors = {"param": main_param,
    **optimizer.state[main_param]} (live tensors, not copies)."""
    for gbuf_range_maps in dist_optimizer.gbuf_ranges:
        assert len(gbuf_range_maps) == 1, "single dtype supported, for now."
        for _dtype, per_bucket in gbuf_range_maps.items():
            for bucket_idx, gbuf_range_map in enumerate(per_bucket):
                for model_param in gbuf_range_map["param_map"]:
                    group_index, group_order = \
                        dist_optimizer.model_param_group_index_map[model_param]
                    main_param = \
                        dist_optimizer.optimizer.param_groups[group_index]["params"][group_order]
                    tensors = {"param": main_param, **dist_optimizer.optimizer.state[main_param]}
                    yield bucket_idx, group_index, group_order, tensors


def get_parameter_state(dist_optimizer):
    """{bucket: {group: {order: {"param", "exp_avg", "exp_avg_sq", ...}}}} of
    THIS rank's shards — no gather to DP rank 0."""
    state = {}
    for bucket, group, order, tensors in _walk_param_shards(dist_optimizer):
        state.setdefault(bucket, {}).setdefault(group, {})[order] = tensors
    return state


def get_chained_optimizer_parameter_state(chained_optimizer):
    return [get_parameter_state(opt) if hasattr(opt, "get_parameter_state") else None
            for opt in chained_optimizer.chained_optimizers]


def load_parameter_state_from_state_dict(dist_optimizer, state_dict):
    """Copy restored shards into the live main params / optimizer states."""
    for bucket, group, order, tensors in _walk_param_shards(dist_optimizer):
        restored = state_dict[bucket][group][order]
        for key, live in tensors.items():
            live.data.copy_(restored[key])


def load_chained_optimizer_parameter_state(chained_optimizer, states):
    for idx, opt in enumerate(chained_optimizer.chained_optimizers):
        if hasattr(opt, "load_parameter_state_from_state_dict"):
            load_parameter_state_from_state_dict(opt, states[idx] if states else None)


def _restore_shards_from_memory(engine, optimizer) -> bool:
    """Fast path: scatter the in-memory optimizer shards into the live tensors
    with one DMA fill + one scatter kernel.  False when not applicable (falls
    back to the per-tensor copy)."""
    m = _mlm()
    try:
        if isinstance(optimizer, m.ChainedOptimizer):
            target = get_chained_optimizer_parameter_state(optimizer)
        else:
            target = get_parameter_state(optimizer)
        step, _ = engine.load_into({_OPTIM: target}, strict=False)
        return step > 0
    except (KeyError, ValueError, RuntimeError) as e:
        logger.info(f"In-memory shard scatter not applicable ({e}); copying per tensor.")
        return False


# -------------------------------------------------------------------------- save --


def save_checkpoint(iteration, model, optimizer, opt_param_scheduler,
                    num_floating_point_operations_so_far, storage_type=StorageType.DISK,
                    comm_backend="", deletion_strategy=None,
                    save_timeout=CheckpointConstant.SAVE_TIMEOUT):
    """Megatron's save_checkpoint, with the optimizer shards kept per rank.

    deletion_strategy: KeepLatestStepStrategy / KeepStepIntervalStrategy of this
    module, or None; save_timeout: seconds agent rank 0 waits for all shards."""
    m = _mlm()
    args = m.get_args()
    checkpointer = MegatronDistCheckpointer.singleton_instance(
        args.save, storage=get_checkpoint_storage(deletion_strategy), comm_backend=comm_backend,
        use_distributed_optimizer=args.use_distributed_optimizer, save_timeout=save_timeout)
    if checkpointer.engine.refuse_non_finite:
        raise NotImplementedError("refuse_non_finite does not cover megatron_dist_ckpt saves: "
                                  "switch it off for this checkpointer")
    model = m.unwrap_model(model)
    m.print_rank_0("saving checkpoint at iteration {:7d} to {}".format(iteration, args.save))
    rng_state = m.get_rng_state()  # collective across DP ranks

    shard_state = {}
    if args.use_distributed_optimizer and not args.no_save_optim and optimizer is not None:
        if isinstance(optimizer, m.ChainedOptimizer):
            shard_state = get_chained_optimizer_parameter_state(optimizer)
        else:
            shard_state = get_parameter_state(optimizer)

    model_state = {}
    if not dist.is_initialized() or m.mpu.get_data_modulo_expert_parallel_rank() == 0:
        model_state = _collect_model_state(m, args, iteration, model, optimizer,
                                           opt_param_scheduler, rng_state,
                                           num_floating_point_operations_so_far)
    state_dicts, paths = {}, {}
    if model_state:
        state_dicts[_MODEL] = model_state
        paths[_MODEL] = m.get_checkpoint_name(args.save, iteration)
    if shard_state:
        state_dicts[_OPTIM] = shard_state
        paths[_OPTIM] = get_dist_optimizer_checkpoint_name(args.save, iteration)
    checkpointer.engine.guard_if_in_place(optimizer)
    if storage_type == StorageType.MEMORY:
        checkpointer.engine.save_to_memory(iteration, state_dicts, paths)
    else:
        checkpointer.engine.save_to_storage(iteration, state_dicts, paths)
    if dist.is_initialized():
        dist.barrier()


def _collect_model_state(m, args, iteration, model, optimizer, opt_param_scheduler, rng_state,
                         flops):
    sd = {"args": args, "checkpoint_version": 3.0, "iteration": iteration,
          "num_floating_point_operations_so_far": flops}
    if len(model) == 1:
        sd["model"] = model[0].state_dict_for_save_checkpoint()
    else:
        for i, chunk in enumerate(model):
            m.mpu.set_virtual_pipeline_model_parallel_rank(i)
            sd["model%d" % i] = chunk.state_dict_for_save_checkpoint()
    if not args.no_save_optim:
        if optimizer is not None:
            sd["optimizer"] = optimizer.state_dict()
        if opt_param_scheduler is not None:
            sd["opt_param_scheduler"] = opt_param_scheduler.state_dict()
    if not args.no_save_rng:
        sd["rng_state"] = rng_state
    return sd


# -------------------------------------------------------------------------- load --


def _load_checkpoint_from_memory(checkpointer):
    step, state_dict = checkpointer.engine.load()
    return (state_dict.get(_MODEL, {}), state_dict.get(_OPTIM, {}), _iter_dir(step), False)


def _load_base_checkpoint(load_dir, rank0=False):
    """(model_state, optim_shards, checkpoint_name, release) from storage, or
    (None, None, "", False) when there is no tracker file."""
    m = _mlm()
    tracker = m.get_checkpoint_tracker_filename(load_dir)
    if not os.path.isfile(tracker):
        if not rank0:
            m.print_rank_0("WARNING: could not find the metadata file {} ".format(tracker))
            m.print_rank_0("    will not load any checkpoints and will start from random")
        return None, None, "", False
    iteration, release = m.read_metadata(tracker)
    if rank0:
        name = m.find_checkpoint_rank_0(load_dir, iteration, release)
    else:
        name = m.get_checkpoint_name(load_dir, iteration, release)
        m.print_rank_0(f" loading release checkpoint from {load_dir}" if release else
                       f" loading checkpoint from {load_dir} at iteration {iteration}")
    shard_name = get_dist_optimizer_checkpoint_name(load_dir, iteration, release)
    try:
        model_state = torch.load(name, map_location="cpu")
        shards = torch.load(shard_name, map_location="cpu") if os.path.exists(shard_name) else {}
    except BaseException as e:
        m.print_rank_0("could not load the checkpoint")
        m.print_rank_0(e)
        sys.exit()
    return model_state, shards, name, release


def load_checkpoint(model, optimizer, opt_param_scheduler, load_arg="load", strict=True,
                    comm_backend="", deletion_strategy=None,
                    save_timeout=CheckpointConstant.SAVE_TIMEOUT):
    """Load a checkpoint (shared memory first, then storage) and return
    (iteration, num_floating_point_operations_so_far)."""
    m = _mlm()
    args = m.get_args()
    load_dir = getattr(args, load_arg)
    checkpointer = MegatronDistCheckpointer.singleton_instance(
        args.save, storage=get_checkpoint_storage(deletion_strategy), comm_backend=comm_backend,
        use_distributed_optimizer=args.use_distributed_optimizer, save_timeout=save_timeout)
    model = m.unwrap_model(model)
    model_state, shards, name, release = _load_checkpoint_from_memory(checkpointer)
    from_memory = bool(model_state)
    if not from_memory:
        model_state, shards, name, release = _load_base_checkpoint(load_dir, rank0=False)
    if model_state is None:
        if args.exit_on_missing_checkpoint:
            m.print_rank_0(">> '--exit-on-missing-checkpoint' set ... exiting. <<")
            dist.barrier()
            sys.exit()
        return 0, 0

    m.set_checkpoint_version(model_state.get("checkpoint_version", 0))
    iteration = 0
    if not (args.finetune or release):
        iteration = model_state.get("iteration", model_state.get("total_iters"))
        if iteration is None:
            m.print_rank_0("A metadata file exists but unable to load iteration from "
                           "checkpoint {}, exiting".format(name))
            sys.exit()
    flops = model_state.get("num_floating_point_operations_so_far", 0)

    assert args.consumed_train_samples == 0
    assert args.consumed_valid_samples == 0
    if "args" in model_state and not args.finetune:
        saved_args = model_state["args"]
        m.check_checkpoint_args(saved_args)
        args.consumed_train_samples = getattr(saved_args, "consumed_train_samples", 0)
        m.update_num_microbatches(consumed_samples=args.consumed_train_samples)
        args.consumed_valid_samples = getattr(saved_args, "consumed_valid_samples", 0)
    else:
        m.print_rank_0("could not find arguments in the checkpoint ...")

    if args.retro_add_retriever or args.transformer_impl == "transformer_engine":
        strict = False
    if len(model) == 1:
        model[0].load_state_dict(model_state["model"], strict=strict)
    else:
        for i, chunk in enumerate(model):
            m.mpu.set_virtual_pipeline_model_parallel_rank(i)
            chunk.load_state_dict(model_state["model%d" % i], strict=strict)
    version = m.get_checkpoint_version()
    m.print_rank_0(f" checkpoint version {version}")
    m.fix_query_key_value_ordering(model, version)

    if not release and not args.finetune and not args.no_load_optim:
        try:
            _restore_optimizer(m, args, checkpointer, optimizer, opt_param_scheduler,
                               model_state, shards, from_memory)
        except KeyError:
            m.print_rank_0("Unable to load optimizer from checkpoint {}. Specify "
                           "--no-load-optim or --finetune to prevent attempting to load the "
                           "optimizer state, exiting ...".format(name))
            sys.exit()
    elif (args.fp16 or args.bf16) and optimizer is not None:
        optimizer.reload_model_params()

    if not release and not args.finetune and not args.no_load_rng:
        try:
            _restore_rng(m, args, model_state)
        except KeyError:
            m.print_rank_0("Unable to load rng state from checkpoint {}. Specify "
                           "--no-load-rng or --finetune to prevent attempting to load the rng "
                           "state, exiting ...".format(name))
            sys.exit()
    if dist.is_initialized():
        dist.barrier()
    m.print_rank_0(f"  successfully loaded checkpoint from {args.load} at iteration {iteration}")
    return iteration, flops


def _restore_optimizer(m, args, checkpointer, optimizer, opt_param_scheduler, model_state,
                       shards, from_memory):
    if optimizer is not None:
        optimizer.load_state_dict(model_state["optimizer"])
    if args.use_distributed_optimizer and optimizer is not None:
        done = from_memory and _restore_shards_from_memory(checkpointer.engine, optimizer)
        if not done:
            if isinstance(optimizer, m.ChainedOptimizer):
                load_chained_optimizer_parameter_state(optimizer, shards)
            else:
                load_parameter_state_from_state_dict(optimizer, shards)
    if opt_param_scheduler is not None:
        key = "lr_scheduler" if "lr_scheduler" in model_state else "opt_param_scheduler"
        opt_param_scheduler.load_state_dict(model_state[key])


def _restore_rng(m, args, model_state):
    if "rng_state" in model_state:
        which = m.mpu.get_data_parallel_rank() if args.data_parallel_random_init else 0
        rng = model_state["rng_state"][which]
    else:  # checkpoints older than the per-DP-rank list
        rng = model_state
    random.setstate(rng["random_rng_state"])
    np.random.set_state(rng["np_rng_state"])
    torch.set_rng_state(rng["torch_rng_state"])
    torch.cuda.set_rng_state(rng["cuda_rng_state"])
    if not rng["rng_tracker_states"]:
        raise KeyError("rng_tracker_states")
    m.tensor_parallel.get_cuda_rng_tracker().set_states(rng["rng_tracker_states"])


def wait_latest_checkpoint(timeout=1800):
    checkpointer = MegatronDistCheckpointer.singleton_instance(
        checkpoint_dir=_mlm().get_args().save)
    checkpointer.engine.wait_latest_checkpoint(timeout)
