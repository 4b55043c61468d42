"""Agent-side consumers: persist the shared-memory checkpoint to storage
asynchronously, off the training critical path.

Public surface and on-disk protocol follow the reference @ 468d632,
dlrover/python/elastic_agent/torch/ckpt_saver.py:
  AsyncCheckpointSaver (:399-936)  factory thread on SharedQueue("factory")
      (:476-536), event loop over SAVE / UPDATE_SHARD / EXIT (:619-650), shard
      persist under the shard lock (:680-746), breakpoint save (:795-852),
      SIGTERM-save / SIGINT-cleanup (:569-592), reset on trainer restart (:883).
  CommonDirCheckpointSaver (:939-1122)  done-file commit in
      <dir>/._dlrover_ckpt_stage/<step>.done/<rank> and tracker update.
  TempDirCheckpointSaver (:1125-1338)  write under the stage dir, then move.
  DdpCheckpointSaver / MegatronCheckpointSaver / DeepSpeedCheckpointSaver
      (:1341-1447) tracker-file flavours; FsdpDcpSaver (:1450-1494) raw
      "__<rank>_0.distcp" bytes + pickled ".metadata".
The serialisation side (TensorMeta, SharedMemoryHandler...) lives in
shm_handler.py and is re-exported here so `ckpt_saver.X` names resolve as in
the reference.
"""

from __future__ import annotations

import importlib
import json
import os
import pickle
import re
import signal
import sys
import threading
import time
from abc import ABCMeta, abstractmethod
from concurrent.futures import Future, ThreadPoolExecutor
from dataclasses import dataclass
from datetime import datetime
from enum import Enum, auto
from pathlib import Path
from typing import List, Optional

import torch

from .common import env_utils
from .common.constants import CheckpointConstant, EventReportConstants, TrainingExceptionLevel
from .common.log import default_logger as logger
from .common.multi_process import SharedDict, SharedLock, SharedMemory, SharedQueue  # noqa: F401
from .common.serialize import ClassMeta
from .shm_handler import (  # noqa: F401  (re-exported names)
    DLROVER_CKPT_CONFIG_KEY,
    CheckpointConfig,
    CheckpointSharedObjPrefix,
    PendingSave,
    SharedMemoryHandler,
    TensorMeta,
    _create_shared_memory,
    _read_state_dict_from_shm,
    _read_tensor_from_buf,
    _traverse_state_dict,
    plan_layout,
    report_local_event,
)


class CheckpointEventType(Enum):
    SAVE = auto()
    UPDATE_SHARD = auto()
    EXIT = auto()


@dataclass
class CheckpointEvent:
    type: CheckpointEventType = CheckpointEventType.SAVE
    step: int = 0
    global_shard_num: int = 0


def _reference_master_client():
    try:
        from dlrover.python.elastic_agent.master_client import MasterClient  # type: ignore
    except Exception:
        return None
    try:
        return MasterClient.singleton_instance()
    except Exception:
        return None


def _same_path(a: str, b: str) -> bool:
    return os.path.normpath(a) == os.path.normpath(b)


class AsyncCheckpointSaver(metaclass=ABCMeta):
    """Persists the state dict held in shared memory to storage.

    Args:
        checkpoint_dir: root directory of the job's checkpoints (tracker file,
            stage directory).
        storage_meta: ClassMeta of the CheckpointStorage to instantiate here.
        local_shard_num / global_shard_num: shards on this node / in the job.
        save_timeout: seconds agent rank 0 waits for all shards of a step.
        rank: rank of the training process that asked for this saver.
    """

    _saver_instance: Optional["AsyncCheckpointSaver"] = None
    _STAGE_DIR = "._dlrover_ckpt_stage"
    _factory_guard = threading.Lock()

    def __init__(self, checkpoint_dir, storage_meta: ClassMeta, local_shard_num=1,
                 global_shard_num=1, save_timeout=CheckpointConstant.SAVE_TIMEOUT, rank=0):
        logger.info(
            f"Initializing the AsyncSaver: checkpoint_dir={checkpoint_dir}, "
            f"local_shard_num={local_shard_num}, global_shard_num={global_shard_num}, "
            f"save_timeout={save_timeout}, rank={rank}")
        self.checkpoint_dir = checkpoint_dir
        self.local_shard_num = local_shard_num
        self.global_shard_num = global_shard_num
        self._node_rank = env_utils.get_rank()
        self._rank = rank
        self._is_agent_rank_0 = rank == 0
        self._save_timeout = save_timeout
        self._stop_commit = False
        self._writing_storage = False
        self._latest_step = 0
        self._master_client = None

        storage_cls = getattr(importlib.import_module(storage_meta.module_path),
                              storage_meta.class_name)
        self.storage = storage_cls(**storage_meta.kwargs)

        self._event_queue = SharedQueue(
            name=CheckpointSharedObjPrefix.SAVE_STEP_QNAME + "0", create=True)
        self._shm_handlers: List[SharedMemoryHandler] = []
        self._shm_locks: List[SharedLock] = []
        for i in range(local_shard_num):
            self._shm_handlers.append(SharedMemoryHandler(i))
            self._shm_locks.append(
                SharedLock(name=CheckpointSharedObjPrefix.SHM_LOCK_NAME + str(i), create=True))
        self._executor = ThreadPoolExecutor(max_workers=local_shard_num,
                                            thread_name_prefix="ckpt_saver-")
        self._closed = False
        logger.info(f"AsyncSaver({type(self).__name__}) initialized.")

    def __del__(self, _finalizing=sys.is_finalizing):
        if _finalizing():
            return  # the agent exits: segments are left for the next incarnation
        try:
            self.close()
        except Exception:
            pass

    # -- factory -------------------------------------------------------------------------
    @classmethod
    def start_async_saving_ckpt(cls):
        """Serve SharedQueue("factory"): each ClassMeta a trainer puts there
        names the saver class to run (trainer side: engine.py:295-324)."""
        factory_queue = SharedQueue(name="factory", create=True)

        def run_saver(meta: ClassMeta):
            if cls._saver_instance is not None:
                cls._saver_instance.close()
                cls._saver_instance = None
            saver_cls = getattr(importlib.import_module(meta.module_path), meta.class_name)
            saver: AsyncCheckpointSaver = saver_cls(**meta.kwargs)
            cls._saver_instance = saver
            saver._sync_shm_to_storage()

        def factory_loop():
            logger.info("Start the checkpoint saver factory.")
            worker: Optional[threading.Thread] = None
            while True:
                meta: ClassMeta = factory_queue.get()
                with cls._factory_guard:
                    live = cls._saver_instance
                    if live is not None and worker is not None and worker.is_alive():
                        # a restarted trainer re-announces itself: only the
                        # directory and the announcing rank may have changed
                        live.checkpoint_dir = meta.kwargs.get("checkpoint_dir")
                        live._rank = meta.kwargs.get("rank")
                        live._is_agent_rank_0 = live._rank == 0
                        continue
                    worker = threading.Thread(target=run_saver, args=(meta,),
                                              name="checkpoint-saver", daemon=True)
                    worker.start()

        threading.Thread(target=factory_loop, name="checkpoint-saver-factory",
                         daemon=True).start()

    @classmethod
    def get_ckpt_saver(cls):
        return cls._saver_instance

    @classmethod
    def register_signal_handler(cls):
        prev_int = signal.getsignal(signal.SIGINT)
        prev_term = signal.getsignal(signal.SIGTERM)

        def on_sigint(signum, frame):
            # ^C / killall: drop the segments, then die the default way
            if cls._saver_instance:
                cls._saver_instance.close()
            signal.signal(signal.SIGINT, prev_int)
            os.kill(os.getpid(), signum)

        def on_sigterm(signum, frame):
            # pod eviction: flush memory to storage first
            if cls._saver_instance:
                cls._saver_instance.save_shm_to_storage()
                cls._saver_instance.close()
            signal.signal(signal.SIGTERM, prev_term)
            os.kill(os.getpid(), signum)

        signal.signal(signal.SIGINT, on_sigint)
        signal.signal(signal.SIGTERM, on_sigterm)

    @classmethod
    def reset(cls):
        """Training processes are being restarted: forget mappings, free locks
        a dead trainer may still hold, keep the segments."""
        saver = cls._saver_instance
        if saver is None:
            return
        saver.reset_shared_memory()
        logger.info("Reset all shared memory of shards.")
        saver.release_locks()

    # -- small accessors -------------------------------------------------------------------
    def get_master_client(self):
        """The job master's client, if there is one: an injected object
        (set_master_client), else — when this code runs inside the reference's
        agent (`dlrover-run`) — the reference's MasterClient singleton."""
        if self._master_client is None:
            self._master_client = _reference_master_client()
        return self._master_client

    def set_master_client(self, client):
        self._master_client = client

    def ucp(self, input_dir: str, output_dir: str, ucp_device_type: str):
        """universal checkpoint conversion hook (DeepSpeed only)"""

    def get_latest_start_saving_step(self):
        steps = [h.get_checkpoint_config(CheckpointConfig()).step for h in self._shm_handlers]
        return steps[0] if steps else self._latest_step

    def get_latest_success_save_dir(self):
        tracker = os.path.join(self.checkpoint_dir, CheckpointConstant.TRACER_FILE_NAME)
        try:
            with open(tracker, "r") as f:
                return self.checkpoint_dir, int(f.read())
        except FileNotFoundError:
            return None, None

    def wait_saving_checkpoint(self):
        """True while a step is being written to storage."""
        return self._writing_storage

    def close(self):
        """Stop the event loop and destroy the shared objects (segments too)."""
        if self._closed:
            return
        self._closed = True
        if not self._event_queue.empty():
            try:
                self._event_queue.queue.get_nowait()
            except Exception:
                pass
        self._event_queue.put(CheckpointEvent(type=CheckpointEventType.EXIT))
        for handler, lock in zip(self._shm_handlers, self._shm_locks):
            if handler:
                handler.close()
                handler.unlink()
            lock.unlink()
        self._event_queue.unlink()
        self._executor.shutdown(wait=False)

    def release_locks(self):
        for lock in self._shm_locks:
            lock.release()

    def reset_shared_memory(self):
        self._stop_commit = True
        for handler in self._shm_handlers:
            handler.reset()

    # -- event loop --------------------------------------------------------------------------
    def _sync_shm_to_storage(self):
        logger.info("Async flash checkpoint saver starts!")
        while True:
            event: Optional[CheckpointEvent] = None
            try:
                event = self._event_queue.get()
                if event.type == CheckpointEventType.EXIT:
                    break
                if event.type == CheckpointEventType.UPDATE_SHARD:
                    logger.info(f"The number of global shards is {event.global_shard_num}.")
                    self.global_shard_num = event.global_shard_num
                elif event.type == CheckpointEventType.SAVE:
                    logger.info(f"Save checkpoint to storage, event {event}")
                    self.save_step_checkpoint(event.step)
            except Exception as e:
                logger.error(f"Unexpected exception during checkpointing {event}: {e}",
                             exc_info=True)
                self._report_failure_to_master(str(e))

    def _report_failure_to_master(self, error_msg):
        client = self.get_master_client()
        if client is None:
            return
        try:
            payload = json.dumps({
                "node_rank": self._node_rank, "local_rank": -1,
                "message": "Async checkpoint saver got failure:" + (error_msg or "Unknown"),
                "time": datetime.now().strftime("%m/%d/%Y %H:%M:%S"),
            })
            client.report_failures(payload, level=TrainingExceptionLevel.PROCESS_ERROR)
        except Exception as e:
            logger.warning(f"Failed to report failure to master in ckpt saver: {e}.")

    # -- helpers shared by the concrete savers -----------------------------------------------
    def _save_shard(self, step, local_shard_id: int, ckpt_config: CheckpointConfig,
                    step_done_dir: str):
        """Persist one shard under its lock; drop a done-file named after the
        shard's global rank."""
        handler = self._shm_handlers[local_shard_id]
        lock = self._shm_locks[local_shard_id]
        held = False
        try:
            # blocks while the trainer is still filling/draining this shard
            held = bool(lock.acquire())
            # only now: the trainer may have re-created the segment (size change)
            handler.refresh_mapping()
            config = handler.get_checkpoint_config(CheckpointConfig())
            if config.step != step:
                logger.error(f"The step {step} in event is no equal to step {config.step} "
                             "in memory.")
                return False
            if config.writing_shm:
                # the trainer died (its lock was dropped with its connection)
                # while filling the segment: the bytes are not a checkpoint.  The
                # reference persists nothing here but still commits the step.
                logger.error(f"Shard {local_shard_id} of step {step} is only partly written "
                             "(writing_shm is set): not persisting it.")
                return False
            logger.info(f"Saves the checkpoint shard {local_shard_id} of rank "
                        f"{ckpt_config.rank} from the shared memory into the storage "
                        f"{ckpt_config}.")
            report_local_event(EventReportConstants.TYPE_INFO, str(ckpt_config.rank),
                               EventReportConstants.ACTION_SAVE_SHARD_START,
                               f"local_id={local_shard_id}, step={step}")
            self.persist_to_storage(local_shard_id, ckpt_config)
            report_local_event(EventReportConstants.TYPE_INFO, str(ckpt_config.rank),
                               EventReportConstants.ACTION_SAVE_SHARD_COMPLETE,
                               f"local_id={local_shard_id}, step={step}")
            # release BEFORE the done-file so the trainer can refill the segment
            # while the (possibly slow) storage acknowledges; released once only
            # — a second release could drop a lock the trainer has just taken.
            lock.release()
            held = False
            self.storage.write("done", os.path.join(step_done_dir, str(ckpt_config.rank)))
            logger.info(f"Finish saving the checkpoint shard {local_shard_id} of rank "
                        f"{ckpt_config.rank}.")
            return True
        except Exception as e:
            logger.error(f"Fail to save the checkpoint shard {local_shard_id} of rank "
                         f"{ckpt_config.rank}, error: {e}", exc_info=True)
            report_local_event(EventReportConstants.TYPE_ERROR, str(ckpt_config.rank),
                               EventReportConstants.ACTION_SAVE_SHARD_ERROR,
                               f"local_id={local_shard_id}, step={step}, error={e}")
            return False
        finally:
            if held:
                lock.release()

    def _dist_make_dir(self, path, timeout=30):
        """Rank 0 (re)creates `path`; the others wait for it to show up."""
        if self._rank == 0:
            logger.info(f"Create path by rank0 worker: {path}.")
            self.storage.safe_rmtree(path)
            self.storage.safe_makedirs(path)
            return
        for _ in range(timeout):
            if self.storage.exists(path):
                return
            time.sleep(1)
        logger.warning(f"Worker {self._rank} can't find path {path} with timeout {timeout}.")

    def _any_rank_locked(self):
        return any([lock.locked() for lock in self._shm_locks])

    def _get_checkpoint_done_dir(self, step):
        return os.path.join(self.checkpoint_dir, self._STAGE_DIR, f"{step}.done")

    def _check_shard_step_consistence(self, step, timeout=15):
        """All local shards that hold anything must hold `step`."""
        deadline = time.time() + timeout
        while True:
            steps = []
            for handler in self._shm_handlers:
                s = handler.get_checkpoint_config(CheckpointConfig()).step
                if s > 0:
                    steps.append(s)
            # (at least one shard must hold the step: right after the first save of a
            # run the agent can be ahead of the trainer's deferred meta publication)
            if steps and all(s == step for s in steps):
                return True
            time.sleep(1)
            if time.time() > deadline:
                logger.info(f"The cached steps are {steps}")
                return False

    def save_shm_to_storage(self, timeout=60, master_client=None):
        """Breakpoint save: the agent calls this when workers failed or are
        about to be restarted, to persist whatever consistent step is in memory."""
        if any(h.no_checkpoint_state() for h in self._shm_handlers):
            logger.info("Skip because no any memory buffer with the state dict.")
            return
        steps = [h.get_checkpoint_config(CheckpointConfig()).step for h in self._shm_handlers]
        if len(set(steps)) > 1:
            logger.error(f"Skip because steps in shards are not inconsistent: {steps}")
            return
        step = steps[0]
        if master_client is not None and not self._sync_node_checkpoint(master_client, step,
                                                                        timeout):
            # another node is gone: its shards are missing, ours are useless
            logger.info("Skip saving the checkpoint from the memory to the storage.")
            self._stop_commit = True
            return
        # A held lock means a trainer died mid-write (or the saver is busy):
        # the segment may be half written.
        if self._writing_storage or self._any_rank_locked():
            logger.info("Saver is writing the checkpoint to storage and skips saving at "
                        "the breakpoint.")
            return
        if step > self._latest_step:
            self.save_step_checkpoint(step)
            logger.info(f"Save the checkpointing state dict from the shared memory to "
                        f"storage, step: {step}.")
        else:
            logger.info(f"The checkpoint of step {step} has been saved.")

    def _sync_node_checkpoint(self, master_client, step: int, timeout: int):
        start = time.time()
        while True:
            if master_client.sync_checkpoint(step):
                return True
            time.sleep(3)
            if time.time() - start > timeout:
                logger.info("It is timeout to sync checkpoint because some nodes may fail.")
                return False

    def _remove_sub_dir_of_target_path(self, path):
        if not os.path.exists(path):
            return
        for entry in os.listdir(path):
            full = os.path.join(path, entry)
            if os.path.isdir(full):
                self.storage.safe_rmtree(full)

    def _submit_local_shards(self, step, step_done_dir, prepare=None, skip_empty=True):
        """Queue _save_shard for every local shard; returns #ok == #submitted."""
        futures: List[Future] = []
        for i, handler in enumerate(self._shm_handlers):
            conf = handler.get_checkpoint_config(CheckpointConfig())
            if skip_empty and conf.step == 0:
                continue
            if prepare is not None:
                prepare(conf)
            futures.append(self._executor.submit(self._save_shard, step, i, conf, step_done_dir))
        ok = 0
        for i, fut in enumerate(futures):
            if fut.result():
                ok += 1
            else:
                logger.error(f"Fail to save checkpoint shard {i} for step {step}")
        return ok == len(futures)

    # -- abstract ----------------------------------------------------------------------------
    @abstractmethod
    def save_step_checkpoint(self, step: int):
        """Persist the checkpoint of `step` from memory to storage."""

    @abstractmethod
    def persist_to_storage(self, local_shard_id, ckpt_config):
        """Write the state dict of one local shard to ckpt_config.paths."""

    @abstractmethod
    def commit_checkpoint(self, step: int, step_done_dir: str, timeout=600):
        """Agent rank 0: publish the step once every shard reported done."""

    @abstractmethod
    def update_tracker_file(self, step: int):
        """Record `step` as the latest complete checkpoint."""


class CommonDirCheckpointSaver(AsyncCheckpointSaver):
    """Shards are written straight to the paths the trainer chose; a step is
    committed (tracker updated) when the number of done-files equals the
    global shard count."""

    def update_tracker_file(self, step):
        self.storage.write(str(step),
                           os.path.join(self.checkpoint_dir, CheckpointConstant.TRACER_FILE_NAME))

    def save_step_checkpoint(self, step: int):
        if not self._check_shard_step_consistence(step):
            logger.warning(f"Skip persisting the checkpoint of step {step} because the cached "
                           "step in memory are not consistent.")
            return
        self._writing_storage = True
        try:
            step_done_dir = self._get_checkpoint_done_dir(step)
            self._dist_make_dir(step_done_dir)
            if not self._submit_local_shards(step, step_done_dir):
                logger.error(f"Rank {self._node_rank} save checkpoint failed for step {step}")
                return
            self._latest_step = step
            if self._is_agent_rank_0:
                self._stop_commit = False
                self.commit_checkpoint(step, step_done_dir, timeout=self._save_timeout)
        finally:
            self._writing_storage = False

    def commit_checkpoint(self, step: int, step_done_dir: str, timeout=600):
        start = time.time()
        success = False
        while True:
            if self._stop_commit:
                logger.info("Stop committing the checkpoint because the training processes "
                            "restarted.")
                break
            done_files = self.storage.listdir(step_done_dir)
            if len(done_files) == self.global_shard_num:
                logger.info(f"All agents finish saving checkpoint for step {step}")
                self.update_tracker_file(step)
                self.storage.safe_rmtree(step_done_dir)
                success = True
                break
            logger.info(f"The number of ready shards is {len(done_files)} != "
                        f"{self.global_shard_num}.")
            elapsed = round(time.time() - start, 2)
            if elapsed > timeout:
                logger.error(f"Commit checkpoint timeout for step {step}, elapsed_time: "
                             f"{elapsed}. The done files are {done_files}.")
                self.storage.safe_rmtree(step_done_dir)
                break
            time.sleep(5)
        self.storage.commit(step, success)

    def persist_to_storage(self, local_shard_id: int, ckpt_config: CheckpointConfig):
        if ckpt_config is None or not ckpt_config.paths:
            logger.info("Skip persisting checkpoint because checkpoint config is missing.")
            return
        state_dict = self._shm_handlers[local_shard_id].load_state_dict()
        safe_serialization = state_dict.pop("safe_serialization", None)
        for state_name, sd in state_dict.items():
            if not sd or state_name not in ckpt_config.paths:
                continue
            path = ckpt_config.paths[state_name]
            # same bytes as torch.save, written and CRC'd by several threads
            writer = _torch_save_writer()
            if safe_serialization:
                path, writer = _hf_safetensors_target(state_name, path)
            self.storage.write_state_dict(sd, path, writer)


def _torch_save_writer():
    """`write_func(state_dict, path)` producing exactly torch.save's file.
    DLROVER_B200_FAST_PERSIST=0 selects plain torch.save."""
    if os.getenv("DLROVER_B200_FAST_PERSIST", "1") in ("0", "false", "False"):
        return torch.save
    from . import fast_torch_save

    # at most 4 writers: page-cache / tmpfs targets gain nothing from more, they contend
    threads = int(os.getenv("DLROVER_B200_PERSIST_THREADS", "0") or 0) or \
        max(1, min(4, (os.cpu_count() or 1) // 2))
    return lambda sd, path: fast_torch_save.save(sd, path, threads=threads)


def _hf_safetensors_target(state_name: str, path: str):
    """HF Trainer naming: weights asked for as *.bin are stored as safetensors
    when `safe_serialization` travels in the state dict."""
    from safetensors.torch import save_file as safe_save_file
    from transformers.utils import (
        ADAPTER_SAFE_WEIGHTS_NAME,
        ADAPTER_WEIGHTS_NAME,
        SAFE_WEIGHTS_NAME,
        WEIGHTS_NAME,
    )

    if state_name.endswith(ADAPTER_WEIGHTS_NAME):
        return path.replace(ADAPTER_WEIGHTS_NAME, ADAPTER_SAFE_WEIGHTS_NAME), safe_save_file
    if state_name.endswith(WEIGHTS_NAME):
        return path.replace(WEIGHTS_NAME, SAFE_WEIGHTS_NAME), safe_save_file
    if re.fullmatch(r"(.*?)-\d{5}-of-\d{5}.bin", state_name):
        return (path.replace("pytorch_model", "model").replace(".bin", ".safetensors"),
                safe_save_file)
    if state_name.endswith(".safetensors"):
        # recorded from transformers' own safetensors writer (hf_trainer.py)
        return path, lambda sd, p: safe_save_file(sd, p, metadata={"format": "pt"})
    return path, _torch_save_writer()


class TempDirCheckpointSaver(AsyncCheckpointSaver):
    """Shards are first written under <dir>/._dlrover_ckpt_stage/<step>/ and the
    directory is moved to its final place when every shard is done."""

    def __init__(self, checkpoint_dir, storage_meta: ClassMeta, local_shard_num=1,
                 global_shard_num=1, save_timeout=CheckpointConstant.SAVE_TIMEOUT, rank=0):
        super().__init__(checkpoint_dir, storage_meta, local_shard_num, global_shard_num,
                         save_timeout, rank=rank)
        if self._node_rank == 0:
            # leftovers of an earlier incarnation
            self._remove_sub_dir_of_target_path(os.path.join(self.checkpoint_dir, self._STAGE_DIR))

    def update_tracker_file(self, step):
        self.storage.write(str(step),
                           os.path.join(self.checkpoint_dir, CheckpointConstant.TRACER_FILE_NAME))

    def persist_to_storage(self, local_shard_id, ckpt_config):
        CommonDirCheckpointSaver.persist_to_storage(self, local_shard_id, ckpt_config)

    def save_step_checkpoint(self, step):
        logger.info(f"Rank {self._node_rank} start save checkpoint to storage, step: {step}")
        if not self._check_shard_step_consistence(step):
            logger.warning(f"Skip persisting the checkpoint of step {step} because the cached "
                           "step in memory are not consistent.")
            return
        self._writing_storage = True
        try:
            mkdir_timeout = int(self._save_timeout / 2)
            temp_dir = self._get_tmp_ckpt_dir(step)
            self._dist_make_dir(temp_dir, mkdir_timeout)
            step_done_dir = self._get_checkpoint_done_dir(step)
            self._dist_make_dir(step_done_dir, mkdir_timeout)
            target = {"dir": ""}

            def redirect(conf):
                target["dir"] = self._replace_path_dir(conf, temp_dir)

            if not self._submit_local_shards(step, step_done_dir, prepare=redirect,
                                             skip_empty=False):
                logger.error(f"Rank {self._node_rank} save checkpoint failed for step {step}")
                return
            self._latest_step = step
            if self._is_agent_rank_0:
                self.commit_checkpoint(step, step_done_dir=step_done_dir, tmp_path=temp_dir,
                                       target_path=target["dir"], timeout=self._save_timeout)
        finally:
            self._writing_storage = False

    def _replace_path_dir(self, ckpt_config: CheckpointConfig, temp_dir: str):
        """Point every path of the config into temp_dir; returns the original
        (common) directory."""
        origin = ""
        if not ckpt_config.paths:
            return origin
        moved = {}
        for name, path in ckpt_config.paths.items():
            path = str(path)
            parent = os.path.dirname(path)
            moved[name] = path.replace(parent, temp_dir)
            if not origin:
                origin = parent
            elif not _same_path(origin, parent):
                raise ValueError(f"The directories must be same. The latest dir is {origin} "
                                 f"and the current dir  of {name} is {parent}")
        ckpt_config.paths = moved
        return origin

    def _get_tmp_ckpt_dir(self, step: int):
        return os.path.join(self.checkpoint_dir, self._STAGE_DIR, str(step))

    def commit_checkpoint(self, step: int, step_done_dir: str, tmp_path: str,  # type: ignore
                          target_path: str, timeout=600):
        logger.info(f"Start commit checkpoint tmp_path: {tmp_path}, path: {target_path}")
        start = time.time()
        success = False
        while True:
            done_files = self.storage.listdir(step_done_dir)
            if len(done_files) == self.global_shard_num:
                logger.info(f"All agents finish saving checkpoint for step {step}")
                if os.path.exists(target_path):
                    if os.path.isdir(target_path):
                        self.storage.safe_rmtree(target_path)
                    else:
                        self.storage.safe_remove(target_path)
                self.storage.safe_move(tmp_path, target_path)
                self.storage.safe_rmtree(step_done_dir)
                self.update_tracker_file(step)
                success = True
                break
            logger.info(f"The number of ready shards is {len(done_files)} != "
                        f"{self.global_shard_num}.")
            elapsed = time.time() - start
            if elapsed > timeout:
                logger.error(f"Commit checkpoint timeout for step {step}, elapsed_time: "
                             f"{elapsed}. The done files are {done_files}.")
                self.storage.safe_rmtree(tmp_path)
                self.storage.safe_rmtree(step_done_dir)
                break
            time.sleep(5)
        self.storage.commit(step, success)


class DdpCheckpointSaver(CommonDirCheckpointSaver):
    """Persist the (replicated) DDP checkpoint from shared memory."""


class _ExtraTrackerSaver(CommonDirCheckpointSaver):
    """Also writes the framework's own "latest step" file next to ours."""

    TRACER_FILE = ""

    def update_tracker_file(self, step):
        super().update_tracker_file(step)
        self.storage.write(str(step), os.path.join(self.checkpoint_dir, self.TRACER_FILE))


class MegatronCheckpointSaver(_ExtraTrackerSaver):
    TRACER_FILE = "latest_checkpointed_iteration.txt"


class DeepSpeedCheckpointSaver(_ExtraTrackerSaver):
    TRACER_FILE = "latest"

    def get_deepspeed_install_dir(self):
        spec = importlib.util.find_spec("deepspeed")
        return os.path.dirname(spec.origin) if spec and spec.origin else ""

    def ucp(self, input_dir: str, output_dir: str, ucp_device_type: str):
        """Convert a saved checkpoint to DeepSpeed's universal format by running
        deepspeed/checkpoint/ds_to_universal.py in a child process (started with
        torchelastic's SubprocessHandler, like the agent's workers)."""
        import sys

        from packaging import version
        from torch.distributed.elastic.multiprocessing.api import SubprocessHandler

        script = self.get_deepspeed_install_dir() + "/checkpoint/ds_to_universal.py"
        args = [script, "--input_folder", f"{input_dir}", "--output_folder", f"{output_dir}",
                "--inject_missing_state"]
        if ucp_device_type != "cpu":
            args += ["--device", ucp_device_type]
        python = os.getenv("PYTHON_EXEC", sys.executable)
        # SubprocessHandler grew a local_rank_id argument after torch 2.2
        torch_release = version.parse(version.parse(torch.__version__).base_version)
        if torch_release <= version.parse("2.2.2"):
            handler = SubprocessHandler(python, tuple(args), {}, "", "")
        else:
            handler = SubprocessHandler(python, tuple(args), {}, "", "", 0)
        ret = handler.proc.wait()
        if ret != 0:
            logger.error(f"ds_to_universal returned non-zero exit code {ret}")
            return False
        return True


class FsdpDcpSaver(CommonDirCheckpointSaver):
    """torch.distributed.checkpoint layout: the segment IS the shard file."""

    def persist_to_storage(self, local_shard_id: int, ckpt_config: CheckpointConfig):
        handler = self._shm_handlers[local_shard_id]
        path = ckpt_config.paths[CheckpointConstant.MODEL_STATES_NAME]
        checkpoint_dir = os.path.dirname(path)
        leader = self._is_agent_rank_0 and local_shard_id == 0
        if leader:
            self._dist_make_dir(checkpoint_dir)
        else:
            while not self.storage.exists(checkpoint_dir):
                time.sleep(1)
        handler.refresh_mapping()
        assert handler.shared_memory is not None
        self.storage.write(handler.shared_memory.buf, path)
        if leader:
            meta_dict = handler.metadata.get()
            dcp_metadata = meta_dict.get("dcp_metadata", {})
            if dcp_metadata:
                self.storage.write(pickle.dumps(dcp_metadata), Path(checkpoint_dir) / ".metadata")
            self.storage.write(
                str(ckpt_config.step),
                os.path.join(self.checkpoint_dir, CheckpointConstant.TRACER_FILE_NAME))
