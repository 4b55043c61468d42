"""Flash checkpointers for FSDP modules.

Reference @ 468d632: dlrover/trainer/torch/flash_checkpoint/fsdp.py —
FsdpShardCheckpointer (:36-157, SHARDED_STATE_DICT through DCP, every rank a
shard, no cross-rank tensor traffic) and FsdpFullCheckpointer (:160-300,
FULL_STATE_DICT(rank0_only=False): torch FSDP all-gathers the flat parameters
over NCCL/NVSwitch — the only place a full replica is required — and the
result is saved like a DDP state dict).
"""

from __future__ import annotations

import os

import torch.distributed as dist
import torch.distributed.checkpoint as dist_cp
from torch.distributed.checkpoint.optimizer import load_sharded_optimizer_state_dict
from torch.distributed.fsdp import FullStateDictConfig
from torch.distributed.fsdp import FullyShardedDataParallel as FSDP
from torch.distributed.fsdp import StateDictType
from torch.distributed.fsdp.api import FullOptimStateDictConfig

from ..common.constants import CheckpointConstant
from ..common.storage import get_checkpoint_storage
from .api import Checkpointer, StorageType
from .engine import FullCheckpointEngine
from .fsdp_engine import FsdpCheckpointEngine

_MODEL = CheckpointConstant.MODEL_STATES_NAME


def _dcp_load(state_dict, reader):
    if hasattr(dist_cp, "load"):
        return dist_cp.load(state_dict, storage_reader=reader)
    return dist_cp.load_state_dict(state_dict=state_dict, storage_reader=reader)


def _dispatch(engine, storage_type, step, state_dict, paths):
    if storage_type == StorageType.MEMORY:
        return engine.save_to_memory(step, state_dict, paths)
    if storage_type == StorageType.DISK:
        if not paths[_MODEL]:
            raise ValueError("path cannot be empty if storage type is disk!")
        return engine.save_to_storage(step, state_dict, paths)
    raise ValueError(f"No support storage type {storage_type}")


class FsdpShardCheckpointer(Checkpointer):
    """Saves / loads the SHARDED state of an FSDP module and its optimizer.

    Example::
        ckpt = FsdpShardCheckpointer(checkpoint_dir)
        ckpt.save_checkpoint(step, model, optimizer, {"epoch": e},
                             storage_type=StorageType.MEMORY)
        extra = ckpt.load_checkpoint(model, optimizer)
    """

    def __init__(self, checkpoint_dir: str, comm_backend="", deletion_strategy=None,
                 save_timeout=CheckpointConstant.SAVE_TIMEOUT, async_drain=None):
        self.checkpoint_dir = checkpoint_dir
        self.storage = get_checkpoint_storage(deletion_strategy)
        self._engine = FsdpCheckpointEngine(checkpoint_dir, self.storage, comm_backend,
                                            save_timeout, async_drain=async_drain)

    def save_checkpoint(self, step, model, optimizer, extra_sd={}, path="",
                        storage_type=StorageType.DISK):
        self._engine.guard_if_in_place(optimizer)
        with FSDP.state_dict_type(model, StateDictType.SHARDED_STATE_DICT):
            state_dict = {"model": model.state_dict(),
                          "optim": FSDP.optim_state_dict(model, optimizer)}
            state_dict.update(extra_sd)
            if not path:
                path = os.path.join(self.checkpoint_dir, str(step))
            _dispatch(self._engine, storage_type, step, state_dict, {_MODEL: path})

    def load_checkpoint(self, model, optimizer, resume_path=""):
        return self._load(model, optimizer, lambda: self._engine.load(resume_path))

    def rollback_checkpoint(self, model, optimizer):
        """load_checkpoint from this process's own last memory checkpoint, for a rollback
        (a loss spike, a NaN step, a survivor resetting to the last consistent step).
        Each of the two passes (model, optimizer) scatters its tensor items from the HBM
        snapshot of that save when every rank's snapshot covers them: nothing crosses
        PCIe.  Otherwise every rank reads that pass from its segment, as load_checkpoint
        does; the bytes are the same either way.  FSDP hands the sharded optimizer state
        to save_checkpoint as host copies (ShardedOptimStateDictConfig's default
        offload_to_cpu=True), so it is never in the snapshot: its pass reads the segment,
        and like every restore from the segment it retires the snapshot and the
        incremental baseline.  Returns what load_checkpoint returns, or {} when the ranks
        hold no common step in memory (storage is not consulted).
        engine.last_rollback_stats() tells which path each pass took.  Every rank must
        call it."""
        return self._load(model, optimizer, self._engine.rollback_reader)

    def _load(self, model, optimizer, get_reader):
        with FSDP.state_dict_type(model, StateDictType.SHARDED_STATE_DICT):
            # the optimizer state cannot be loaded in the same pass as the model
            state_dict = {"model": model.state_dict(), "step": 0}
            reader = get_reader()
            if not reader:
                return {}
            _dcp_load(state_dict, reader)
            model_sd = state_dict.pop("model", None)
            if model_sd:
                model.load_state_dict(model_sd)
            optim_state = load_sharded_optimizer_state_dict(
                model_state_dict=model_sd, optimizer_key="optim", storage_reader=reader)
            optim_sd = optim_state.pop("optim", None)
            if optim_sd:
                optimizer.load_state_dict(FSDP.optim_state_dict_to_load(model, optimizer,
                                                                        optim_sd))
            return state_dict

    def wait_latest_checkpoint(self, timeout=1800):
        self._engine.wait_latest_checkpoint(timeout)

    def wait_memory_save(self, timeout=None):
        return self._engine.wait_memory_save(timeout)

    @property
    def engine(self):
        return self._engine


class FsdpFullCheckpointer(Checkpointer):
    """Saves / loads the FULL (unsharded) state of an FSDP module: every rank
    materialises the whole model (NCCL all-gather inside torch FSDP), local
    rank 0 of each node writes it to shared memory."""

    def __init__(self, checkpoint_dir: str, comm_backend="", deletion_strategy=None,
                 save_timeout: int = CheckpointConstant.SAVE_TIMEOUT, async_drain=None):
        self.checkpoint_dir = checkpoint_dir
        self._rank = dist.get_rank() if dist.is_initialized() else 0
        self.storage = get_checkpoint_storage(deletion_strategy)
        self._engine = FullCheckpointEngine(
            checkpoint_dir=checkpoint_dir, storage=self.storage, local_shard_num=1,
            global_shard_num=1, comm_backend=comm_backend, save_timeout=save_timeout,
            async_drain=async_drain)

    @staticmethod
    def _full_state(model):
        return FSDP.state_dict_type(model, StateDictType.FULL_STATE_DICT,
                                    FullStateDictConfig(rank0_only=False),
                                    FullOptimStateDictConfig(rank0_only=False))

    def _from_shards(self) -> bool:
        """The FULL checkpoint can be assembled from every rank's SHARDED state dict
        (no FULL_STATE_DICT all-gather, no full replica in every rank's HBM) when the
        ranks of the job all sit on this node and save cooperatively."""
        return os.getenv("DLROVER_B200_FULL_FROM_SHARDS", "1") not in ("0", "false", "False") \
            and self._engine.full_from_shards_supported()

    def save_checkpoint(self, step, model, optimizer, extra_sd={}, path="",
                        storage_type=StorageType.DISK):
        if path == "":
            # one image per node, written under the node's saving rank (local rank 0)
            path = os.path.join(self.checkpoint_dir, f"{step}/rank_{self._rank}.pt")
        self._engine.guard_if_in_place(optimizer)
        if self._from_shards():
            path = os.path.join(os.path.dirname(path), "rank_0.pt") if path.endswith(
                f"rank_{self._rank}.pt") else path
            with FSDP.state_dict_type(model, StateDictType.SHARDED_STATE_DICT):
                state_dict = {"model": model.state_dict(),
                              "optimizer": FSDP.optim_state_dict(model, optimizer)}
            state_dict.update(extra_sd)
            if storage_type == StorageType.MEMORY:
                return self._engine.save_shards_to_memory(step, {_MODEL: state_dict},
                                                          {_MODEL: path})
            if storage_type == StorageType.DISK:
                if not path:
                    raise ValueError("path cannot be empty if storage type is disk!")
                if self._rank == 0:
                    self.storage.safe_rmtree(os.path.dirname(path))
                return self._engine.save_shards_to_storage(step, {_MODEL: state_dict},
                                                           {_MODEL: path})
            raise ValueError(f"No support storage type {storage_type}")
        with self._full_state(model):
            state_dict = {"model": model.state_dict(),
                          "optimizer": FSDP.optim_state_dict(model, optimizer)}
        state_dict.update(extra_sd)
        if storage_type == StorageType.DISK and path and self._rank == 0:
            self.storage.safe_rmtree(os.path.dirname(path))
        _dispatch(self._engine, storage_type, step, {_MODEL: state_dict}, {_MODEL: path})

    def load_checkpoint(self, model, optimizer, resume_path=""):
        state_dict = self._engine.load(resume_path)
        if not state_dict:
            return {}
        model_sd = state_dict.pop("model", {})
        optim_sd = state_dict.pop("optimizer", {})
        with self._full_state(model):
            optim_sd = FSDP.optim_state_dict_to_load(model=model, optim=optimizer,
                                                     optim_state_dict=optim_sd)
        model.load_state_dict(model_sd)
        optimizer.load_state_dict(optim_sd)
        return state_dict

    def wait_latest_checkpoint(self, timeout=1800):
        self._engine.wait_latest_checkpoint(timeout)

    def wait_memory_save(self, timeout=None):
        return self._engine.wait_memory_save(timeout)

    @property
    def engine(self):
        return self._engine
