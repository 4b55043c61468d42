"""User-facing checkpointer contract + the DDP checkpointer.

Reference @ 468d632: dlrover/trainer/torch/flash_checkpoint/checkpointer.py
(StorageType :18-20, Checkpointer :23-65) and ddp.py (DdpCheckpointer :25-125).
"""

from __future__ import annotations

import os
from abc import ABCMeta, abstractmethod
from enum import Enum, auto

import torch.distributed as dist

from ..common.constants import CheckpointConstant
from ..common.storage import get_checkpoint_storage
from .engine import FullCheckpointEngine


class StorageType(Enum):
    MEMORY = auto()
    DISK = auto()


class Checkpointer(metaclass=ABCMeta):
    """Saves to shared memory first (cheap, every few steps) and lets the agent
    persist to storage asynchronously; loads from memory when the node
    survived, from storage otherwise."""

    @abstractmethod
    def save_checkpoint(self, step, state_dict, path, storage_type=StorageType.DISK):
        """step: global iteration; state_dict: model/optimizer state; path:
        where the agent persists it (also used for the breakpoint save after a
        failure); storage_type: MEMORY or DISK."""

    @abstractmethod
    def load_checkpoint(self, resuming_path=None):
        """Return the state dict of `resuming_path`, or of the latest step."""


class DdpCheckpointer(Checkpointer):
    """Flash checkpointer for DDP models / any full (replicated) state dict.

    Args:
        checkpoint_dir: directory of the checkpoints.
        local_shard_num / global_shard_num: 1/1 for replicated state; set to
            ranks-per-node / world size if every rank holds different state.
        comm_backend: backend of the control group ("" = default group's).
        deletion_strategy: KeepLatestStepStrategy / KeepStepIntervalStrategy /
            None (keep everything).
        save_timeout: seconds agent rank 0 waits for all shards.
        replica_count: in-memory replicas on other nodes.
        cooperative: replicated state (local_shard_num=1) on a node with several local
            ranks: every local rank drains 1/n of the one image into the one segment
            (n PCIe links instead of one).  None = on when possible
            (DLROVER_B200_COOP_DRAIN=0 turns it off), False = the reference's policy
            (only local rank 0 writes).

    Example::
        ckpt = DdpCheckpointer("/tmp/checkpoint/")
        for step, batch in enumerate(loader):
            ...
            if step % 5 == 0:
                ckpt.save_checkpoint(step, model.state_dict(), storage_type=StorageType.MEMORY)
            if step % 100 == 0:
                ckpt.save_checkpoint(step, model.state_dict(), storage_type=StorageType.DISK)
        sd = ckpt.load_checkpoint()
    """

    def __init__(self, checkpoint_dir: str, local_shard_num=1, global_shard_num=1,
                 comm_backend="", deletion_strategy=None,
                 save_timeout=CheckpointConstant.SAVE_TIMEOUT, replica_count=0,
                 async_drain=None, cooperative=None):
        self.checkpoint_dir = checkpoint_dir
        self._rank = dist.get_rank() if dist.is_initialized() else 0
        self.storage = get_checkpoint_storage(deletion_strategy)
        self._engine = FullCheckpointEngine(
            checkpoint_dir=checkpoint_dir,
            storage=self.storage,
            local_shard_num=local_shard_num,
            global_shard_num=global_shard_num,
            comm_backend=comm_backend,
            save_timeout=save_timeout,
            replica_count=replica_count,
            async_drain=async_drain,
            cooperative=cooperative,
        )

    def save_checkpoint(self, step, state_dict, path="", storage_type=StorageType.DISK):
        if path == "":
            path = os.path.join(self.checkpoint_dir, f"{step}/rank_{self._rank}.pt")
        name = CheckpointConstant.MODEL_STATES_NAME
        wrapped, paths = {name: state_dict}, {name: path}
        if storage_type == StorageType.MEMORY:
            self._engine.save_to_memory(step, wrapped, paths)
        elif storage_type == StorageType.DISK:
            if not path:
                raise ValueError("path cannot be empty if storage type is disk!")
            self._engine.save_to_storage(step, wrapped, paths)
        else:
            raise ValueError(f"No support storage type {storage_type}")

    def load_checkpoint(self, resume_path=""):
        return self._engine.load(resume_path)

    def load_checkpoint_into(self, state_dict, stream=None, strict=True):
        """Scatter the in-memory checkpoint into the live tensors of
        `state_dict` (e.g. model.state_dict()); returns the restored step, 0 if
        memory holds nothing usable (then fall back to load_storage_into() or
        load_checkpoint())."""
        step, _ = self._engine.load_into({CheckpointConstant.MODEL_STATES_NAME: state_dict},
                                         stream=stream, strict=strict)
        return step

    def rollback_into(self, state_dict, stream=None, strict=True):
        """Roll the live tensors of `state_dict` back to the in-memory checkpoint this
        process saved: from the HBM snapshot of that save when every rank still holds
        it (no PCIe transfer, the incremental baseline survives), else exactly as
        load_checkpoint_into.  Returns the restored step, 0 if memory holds nothing
        usable."""
        step, _ = self._engine.rollback_into({CheckpointConstant.MODEL_STATES_NAME: state_dict},
                                             stream=stream, strict=strict)
        return step

    def load_storage_into(self, state_dict, resume_path="", stream=None, strict=True):
        """Restore the persisted checkpoint (`resume_path`, else the latest tracked step)
        straight into the live tensors of `state_dict`, without torch.load: for a node
        whose shared memory lost the checkpoint (load_checkpoint_into returned 0).
        Returns the restored step, 0 if nothing is tracked."""
        step, _ = self._engine.load_storage_into(
            {CheckpointConstant.MODEL_STATES_NAME: state_dict}, resume_path=resume_path,
            stream=stream, strict=strict)
        return step

    def wait_memory_save(self, timeout=None):
        """Block until the last save_checkpoint(MEMORY) is fully in shared memory."""
        return self._engine.wait_memory_save(timeout)

    def wait_latest_checkpoint(self, timeout=1800):
        self._engine.wait_latest_checkpoint(timeout)

    @property
    def engine(self):
        return self._engine
