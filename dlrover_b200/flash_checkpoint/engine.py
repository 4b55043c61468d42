"""Trainer-side checkpoint engines.

API follows the reference @ 468d632 (dlrover/trainer/torch/flash_checkpoint/):
  engine.py            CheckpointEngine ABC (:154-520), check_all_rank_ready
                       (:57-71), verify_all_rank_step_consistent (:74-95),
                       timer (:98-109), start_saver_process (:118-137)
  full_ckpt_engine.py  FullCheckpointEngine (:33-220)  — the "DDP engine"
  deepspeed_engine.py  DeepSpeedCheckpointEngine (:31-162)
  megatron_engine.py   MegatronCheckpointEngine (:28-157),
                       MegatronDistCheckpointEngine (:160-278)

Behavioural differences, all on the device path:
  * save_state_dict_to_memory enqueues ONE gather kernel on the caller's CUDA
    stream and returns; the PCIe drain, the writing_shm=False meta update and
    the release of the shard lock happen on a completion thread (set
    async_drain=False, or env DLROVER_B200_ASYNC_DRAIN=0, for the reference's
    "bytes are in shared memory when the call returns" behaviour).  While a
    drain is in flight the shard lock is still ours, so the next non-blocking
    save is skipped exactly like a save that finds the agent persisting
    (engine.py:366-375) and the agent's SAVE handler simply blocks on the lock.
  * the readiness all-reduce runs on a side stream and only that stream is
    synchronised, so the check no longer waits for the training stream.
  * load_into(): scatter the in-memory checkpoint straight into live tensors.
"""

from __future__ import annotations

import copy
import os
import threading
import time
from abc import ABCMeta, abstractmethod
from datetime import timedelta
from multiprocessing import Process
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from ..common.ctl_segment import ControlSegment
from ..shm_handler import CoopContext
from ..ckpt_saver import (
    DLROVER_CKPT_CONFIG_KEY,
    AsyncCheckpointSaver,
    CheckpointConfig,
    CheckpointEvent,
    CheckpointEventType,
    CheckpointSharedObjPrefix,
    DdpCheckpointSaver,
    DeepSpeedCheckpointSaver,
    MegatronCheckpointSaver,
    SharedMemoryHandler,
)
from ..common import env_utils
from ..common.constants import CheckpointConstant
from ..common.log import default_logger as logger
from ..common.multi_process import LocalSocketComm, SharedLock, SharedQueue
from ..common.serialize import ClassMeta
from ..common.storage import CheckpointStorage
from .replica import CkptReplicaManger

_side_streams: Dict[int, "torch.cuda.Stream"] = {}
_ready_flags: Dict[str, torch.Tensor] = {}


def _sync_device(backend: str) -> str:
    return "cpu" if backend == "gloo" else f"cuda:{env_utils.get_local_rank()}"


class _OffTrainingStream:
    """Run tiny control collectives on a private CUDA stream so reading their
    result does not synchronise the training stream."""

    def __init__(self, device: str):
        self._ctx = None
        self._stream = None
        if device != "cpu":
            idx = torch.device(device).index or 0
            s = _side_streams.get(idx)
            if s is None:
                s = _side_streams[idx] = torch.cuda.Stream(device=idx)
            self._stream = s
            self._ctx = torch.cuda.stream(s)

    def __enter__(self):
        if self._ctx is not None:
            self._ctx.__enter__()
        return self

    def __exit__(self, *exc):
        if self._ctx is not None:
            self._ctx.__exit__(*exc)
            self._stream.synchronize()
        return False


def check_all_rank_ready(group: Optional[dist.ProcessGroup], ready: bool):
    """True iff every rank of `group` reports ready (SUM all-reduce of 0/1)."""
    if not group and not dist.is_initialized():
        return ready
    device = _sync_device(dist.get_backend(group))
    flag = _ready_flags.get(device)
    with _OffTrainingStream(device):
        if flag is None:
            flag = _ready_flags[device] = torch.zeros(1, dtype=torch.int32, device=device)
        flag.fill_(0 if ready else 1)
        dist.all_reduce(flag, group=group)
        not_ready = int(flag.item())
    return not_ready == 0


def all_reduce_flags(group: Optional[dist.ProcessGroup], flags: List[int]) -> List[int]:
    """SUM all-reduce of a few small non-negative ints (readiness + "my plan changed"
    in ONE collective), on the side stream like check_all_rank_ready."""
    if not group and not dist.is_initialized():
        return list(flags)
    device = _sync_device(dist.get_backend(group))
    with _OffTrainingStream(device):
        t = torch.tensor(flags, dtype=torch.int32, device=device)
        dist.all_reduce(t, group=group)
        out = [int(v) for v in t.tolist()]
    return out


def verify_all_rank_step_consistent(group: Optional[dist.ProcessGroup], step):
    """True iff every rank holds the same in-memory step (all-gather of step)."""
    if not group and not dist.is_initialized():
        return True
    device = _sync_device(dist.get_backend(group))
    world = group.size() if group else dist.get_world_size()
    with _OffTrainingStream(device):
        mine = torch.tensor([float(step)], device=device)
        everyone = [torch.zeros(1, device=device) for _ in range(world)]
        dist.all_gather(everyone, mine, group=group)
        values = [float(t.item()) for t in everyone]
    return all(v == values[0] for v in values)


class ShardLockClaim:
    """The shard lock as one save holds it (`acquired`: the save took it).  Whichever way
    the save ends first (skipped, completed, failed drain, exception) gives it back;
    release() releases at most once, so the paths need not know about each other."""

    def __init__(self, lock: SharedLock, acquired: bool):
        self._lock = lock if acquired else None
        self._mutex = threading.Lock()

    def release(self):
        with self._mutex:
            lock, self._lock = self._lock, None
        if lock is not None:
            lock.release()


def timer(func):
    def wrapper(*args, **kwargs):
        start = time.time()
        result = func(*args, **kwargs)
        logger.info(f"Local rank {env_utils.get_local_rank()} execute {func.__name__} in "
                    f"{round(time.time() - start, 3)}s.")
        return result

    wrapper.__name__ = getattr(func, "__name__", "wrapped")
    wrapper.__doc__ = func.__doc__
    return wrapper


class _EventForwarder:
    """Delivers checkpoint events to the agent's bounded queue from a daemon thread,
    in submission order (see CheckpointEngine._notify_save_event)."""

    def __init__(self, shared_queue):
        import queue
        import threading

        self._target = shared_queue
        self._backlog = queue.Queue()
        self._pending = 0
        self._lock = threading.Lock()
        threading.Thread(target=self._run, name="ckpt-event-forwarder", daemon=True).start()

    def idle(self) -> bool:
        with self._lock:
            return self._pending == 0

    def submit(self, event):
        with self._lock:
            self._pending += 1
        self._backlog.put(event)

    def _run(self):
        while True:
            event = self._backlog.get()
            try:
                self._target.put(event)  # blocks while the agent is busy
            except Exception as e:  # agent gone: nothing to notify
                logger.warning(f"could not deliver {event}: {e}")
            finally:
                with self._lock:
                    self._pending -= 1


def _torch_optimizers(obj, depth=0):
    """The torch.optim.Optimizer objects under a (possibly wrapped) optimizer."""
    if obj is None or depth > 4:
        return
    if hasattr(obj, "register_step_pre_hook"):
        yield obj
        return
    for attr in ("optimizer", "base_optimizer"):
        inner = getattr(obj, attr, None)
        if inner is not None and inner is not obj:
            yield from _torch_optimizers(inner, depth + 1)
            return
    for attr in ("chained_optimizers", "optimizers"):
        inner = getattr(obj, attr, None)
        if isinstance(inner, (list, tuple)):
            for o in inner:
                yield from _torch_optimizers(o, depth + 1)
            return


def start_async_save():
    """Body of the stand-alone saver daemon.  It owns the segments like an agent
    does, but nobody outlives it to use them (the meta tree lives in this process):
    when the trainer ends — SIGTERM from multiprocessing's exit handler — or
    vanishes (we get re-parented), the segments are unlinked instead of being left
    behind in /dev/shm (16 GB per rank for an 8B model)."""
    import signal

    parent = os.getppid()

    def shutdown(*_):
        saver = AsyncCheckpointSaver._saver_instance
        if saver is not None:
            try:
                saver.close()
            except Exception:
                pass
        if os.getenv("TORCHELASTIC_RUN_ID", ""):
            # this run's socket namespace was ours alone
            import shutil

            from ..common.multi_process import _socket_root

            shutil.rmtree(_socket_root(), ignore_errors=True)
        os._exit(0)

    signal.signal(signal.SIGTERM, shutdown)
    AsyncCheckpointSaver.start_async_saving_ckpt()
    while os.getppid() == parent:
        time.sleep(2)
    shutdown()


def start_saver_process():
    """Without dlrover-run there is no agent to host the savers: local rank 0
    forks a daemon that does.  (It dies with the trainer, so it cannot do the
    breakpoint save an agent can.)"""
    if env_utils.launched_by_dlrover_run() or env_utils.get_local_rank() != 0:
        return None
    p = Process(target=start_async_save, daemon=True)
    p.start()
    logger.info("Start a process to asynchronously save checkpoint.")
    return p


def wait_socket_server(socket_server: LocalSocketComm, timeout=60):
    """Clients must not talk before the owner created the socket."""
    start = time.time()
    while not socket_server.is_available():
        time.sleep(0.1)
        if time.time() - start > timeout:
            raise TimeoutError(f"Timed out waiting for socket server: {socket_server.name}.")


def _async_drain_default() -> bool:
    return os.getenv("DLROVER_B200_ASYNC_DRAIN", "1") not in ("0", "false", "False")


class CheckpointEngine(metaclass=ABCMeta):
    """Writes the state dict of this rank's shard into shared memory and asks
    the agent to persist it.

    Args:
        checkpoint_dir: directory of the job's checkpoints.
        storage: CheckpointStorage used for fallback loads and handed (by
            class name) to the agent.
        comm_backend: backend of the control group; "" = the default group's.
        save_timeout: seconds the agent waits for all shards of a step.
        replica_count: cross-node in-memory replicas (multi-node only).
        async_drain: see module docstring; None -> env/default (True).
    """

    saver_proc = None
    # engines whose state is REPLICATED across the local ranks may save cooperatively
    # (every local rank drains 1/n of the one image; see _cooperative_save)
    _supports_cooperative = False

    def __init__(self, checkpoint_dir: str, storage: CheckpointStorage, comm_backend: str = "",
                 save_timeout: int = CheckpointConstant.SAVE_TIMEOUT, replica_count=0,
                 async_drain: Optional[bool] = None):
        logger.info(f"Initializing checkpoint engine: {type(self).__name__.lower()}.")
        if not CheckpointEngine.saver_proc:
            CheckpointEngine.saver_proc = start_saver_process()
        self.checkpoint_dir = checkpoint_dir
        self.storage = storage
        self.latest_step = 0
        self.is_skip = False
        self._save_timeout = save_timeout
        self._async_drain = _async_drain_default() if async_drain is None else bool(async_drain)
        self._local_rank = env_utils.get_local_rank()
        self._restart_count = env_utils.get_torch_restart_count()
        self._cached_step = -1
        self._rank = 0
        self._group_rank = 0
        self._world_size = 1
        self._loader_group = None
        self._saver_group = None
        self._coop_wanted = False
        self._coop_established = False
        self._coop_ctl: Optional[ControlSegment] = None
        self._saving_ranks: Optional[List[int]] = None
        self._init_sync_group(comm_backend)

        self._notify_agent_to_create_saver()
        self._event_queue = None
        if self._local_rank == 0:
            # only local rank 0 talks to the agent's event queue
            self._event_queue = SharedQueue(
                name=CheckpointSharedObjPrefix.SAVE_STEP_QNAME + "0", create=False)
        self._update_saver_config()

        self.local_shard_id = self._local_rank % self.get_local_shard_num()
        self._shm_lock = SharedLock(
            name=CheckpointSharedObjPrefix.SHM_LOCK_NAME + str(self.local_shard_id), create=False)
        wait_socket_server(self._shm_lock)  # created by the saver
        self._shm_handler = SharedMemoryHandler(self.local_shard_id, host=False)
        self._replica_manager = CkptReplicaManger.create_replica_manager(
            self.get_global_shard_num(), replica_count)
        logger.info(f"Checkpoint engine initialized with local rank: {self._local_rank}, "
                    f"rank: {self._rank}.")

    def _init_sync_group(self, comm_backend):
        if not dist.is_initialized():
            self._saving_ranks = [0]
            return
        self._rank = dist.get_rank()
        self._group_rank = env_utils.get_group_rank()
        self._world_size = dist.get_world_size()
        default_backend = dist.get_backend()
        backend = comm_backend or default_backend
        if backend != default_backend:
            self._loader_group = dist.new_group(backend=backend, timeout=timedelta(seconds=60))
        self._saving_ranks = self.get_saving_ranks()
        self._coop_wanted = self._cooperative_by_config()
        self._node_group = None  # NCCL group of this node's ranks (cooperative restore)
        self._node_group_ok = False
        if self._coop_wanted and default_backend == "nccl":
            local_world = env_utils.get_local_world_size()
            if self._world_size == local_world:
                self._node_group_ok = True  # the default group IS the node
            elif self._world_size % local_world == 0:
                for node in range(self._world_size // local_world):
                    ranks = list(range(node * local_world, (node + 1) * local_world))
                    g = dist.new_group(ranks=ranks, backend="nccl", timeout=timedelta(seconds=120))
                    if self._rank in ranks:
                        self._node_group, self._node_group_ok = g, True
        everyone_saves = self._saving_ranks is None or len(self._saving_ranks) == self._world_size
        if backend == default_backend and everyone_saves:
            if self._local_rank == 0:
                logger.info("Use the default process group to sync when saving checkpoint.")
            return
        self._saver_group = dist.new_group(ranks=self._saving_ranks, backend=backend,
                                           timeout=timedelta(seconds=60))
        if self._local_rank == 0:
            who = self._saving_ranks if self._saving_ranks else "all ranks"
            logger.info(f"Create a {backend} communication group to save checkpoint. "
                        f"Saving ranks are {who}.")

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def close(self):
        """Finish a drain in flight and unmap the segment (the agent owns it)."""
        handler = getattr(self, "_shm_handler", None)
        if handler is not None:
            handler.close()
        ctl = getattr(self, "_coop_ctl", None)
        if ctl is not None:
            ctl.close()
            self._coop_ctl = None

    def _notify_agent_to_create_saver(self):
        if self._local_rank != 0:
            return
        factory = SharedQueue(name="factory")
        saver_cls = self.get_saver_class()
        meta = ClassMeta(
            module_path=saver_cls.__module__,
            class_name=saver_cls.__name__,
            kwargs={
                "checkpoint_dir": self.checkpoint_dir,
                "storage_meta": self.storage.get_class_meta(),
                "local_shard_num": self.get_local_shard_num(),
                "global_shard_num": self.get_global_shard_num(),
                "save_timeout": self._save_timeout,
                "rank": self._rank,
            },
        )
        wait_socket_server(factory)
        logger.info(f"Notify agent to create a checkpoint saver using: {meta.__dict__}.")
        factory.put(meta)

    def _update_saver_config(self):
        if self._local_rank != 0:
            return
        if self._event_queue is None:
            raise ValueError("The event queue cannot be None on local rank 0.")
        event = CheckpointEvent(type=CheckpointEventType.UPDATE_SHARD,
                                global_shard_num=self.get_global_shard_num())
        wait_socket_server(self._event_queue)
        logger.info(f"Update saver config: {event.__dict__}")
        self._event_queue.put(event)

    # -- cooperative save of a replicated state --------------------------------------------
    def _cooperative_by_config(self) -> bool:
        """One shard per node, several local ranks, all holding the same state: instead of
        the one saving rank pushing the whole image through its one PCIe link
        (reference full_ckpt_engine.py:76-89), every local rank drains 1/n of it.
        DLROVER_B200_COOP_DRAIN=0 (or cooperative=False) keeps the reference's policy."""
        if not self._supports_cooperative or not dist.is_initialized():
            return False
        if os.getenv("DLROVER_B200_COOP_DRAIN", "1") in ("0", "false", "False"):
            return False
        if getattr(self, "_cooperative_arg", None) is False:
            return False
        return self.get_local_shard_num() == 1 and env_utils.get_local_world_size() > 1

    def _cooperative(self) -> bool:
        """Decided once, after the agent's sockets are up: needs the control segment of an
        agent that creates one (with the reference's agent: the reference's policy)."""
        if not self._coop_wanted:
            return False
        if self._coop_ctl is None:
            self._coop_ctl = ControlSegment.attach(self.local_shard_id)
            if self._coop_ctl is None:
                logger.info("No control segment (reference agent?): cooperative saves are off.")
                self._coop_wanted = False
                return False
            if self._local_rank != 0:
                # whatever a previous trainer of this rank left in the slot
                self._coop_ctl.slot_arrive(self._local_rank, 0, False)
        return True

    def full_from_shards_supported(self) -> bool:
        """True when this engine can assemble a FULL checkpoint from a state dict of shards
        without gathering them (save_shards_to_memory): cooperative saves are on and every
        rank of the job is local to this node (each shard must reach THIS node's segment)."""
        return self._cooperative() and self._world_size == env_utils.get_local_world_size()

    def save_shards_to_memory(self, step, sharded_state_dict, paths: Dict[str, str],
                              blocking=False) -> bool:
        """`sharded_state_dict`: {state name: tree whose tensor leaves are this rank's
        SHARDS (DTensor / ShardedTensor) or replicated tensors}.  The segment receives the
        FULL image — what save_to_memory would write for the gathered state dict
        (reference fsdp.py:238-262: FULL_STATE_DICT all-gather, then one rank saves) — each
        rank contributing its shards over its own PCIe link."""
        if not self.full_from_shards_supported():
            raise RuntimeError("save_shards_to_memory needs cooperative saves on a single node")
        conf = CheckpointConfig(step=step, paths=paths)
        done = self._cooperative_save(sharded_state_dict, conf, blocking, shards=True)
        if done is self._SOLO:
            raise RuntimeError("save_shards_to_memory: the other local ranks do not take part")
        return done

    def save_shards_to_storage(self, step, sharded_state_dict, paths: Dict[str, str],
                               blocking=False) -> bool:
        """save_shards_to_memory + tell the agent to persist the step (the file the agent
        writes is the FULL checkpoint, as after save_to_storage of the gathered state)."""
        success = True
        if step > self._cached_step:
            success = self.save_shards_to_memory(step, sharded_state_dict, paths, blocking)
        if dist.is_initialized():
            dist.barrier()
        if success and self._local_rank == 0:
            self._notify_save_event(step)
        if success:
            self.latest_step = step
        return success

    _SOLO = object()  # _cooperative_save: "not everybody takes part, use the reference policy"

    def _cooperative_save(self, state_dict, conf: CheckpointConfig, blocking: bool,
                          shards: bool = False):
        """The local ranks agree through the control segment — no collective: every
        follower (local rank > 0) posts "I am in save number k, ready or not" in its slot
        and waits for the leader's verdict; the leader (local rank 0, the reference's
        saving rank) takes the shard lock, waits for the followers, settles readiness with
        the leaders of the other nodes (the reference's all-reduce among saving ranks,
        fc/engine.py:57-71) and opens the save or calls it off.

        A job that calls save_checkpoint(MEMORY) on rank 0 only — legal with the reference,
        whose other ranks return at once — is recognised by the followers not showing up:
        the leader then saves alone, and keeps doing so."""
        handler, ctl = self._shm_handler, self._coop_ctl
        local_world = env_utils.get_local_world_size()
        leader = self._local_rank == 0
        conf.rank = self._rank - self._local_rank  # the node's saving rank, as in the reference
        conf.group_rank = self._group_rank
        conf.world_size = self._world_size
        pending = handler.pending_save()
        if pending is not None and blocking:
            pending.wait()
            pending = None
        ready = pending is None and bool(state_dict)
        seq = ctl.coop_seq() + 1
        patience = float(self._save_timeout) if blocking else 60.0

        if not leader:
            ctl.slot_arrive(self._local_rank, seq, ready)
            try:
                go = ctl.wait_coop_open(seq, patience)
            except TimeoutError:
                ctl.slot_arrive(self._local_rank, 0, False)  # withdraw
                logger.warning(f"Rank {self._rank}: the node's saving rank did not start save "
                               f"{conf.step} within {patience:.0f}s; not taking part.")
                return False
            if not go or not ready:
                self.is_skip = True
                return False
            state_dict[DLROVER_CKPT_CONFIG_KEY] = conf
            coop = CoopContext(ctl, self._local_rank, local_world, seq - 1,
                               timeout=float(self._save_timeout), opened=True)
            if shards:
                handler.save_shards_as_full(state_dict, coop,
                                            blocking=not self._async_drain or blocking,
                                            stream=self.snapshot_stream)
            else:
                handler.save_state_dict(state_dict, blocking=not self._async_drain or blocking,
                                        stream=self.snapshot_stream, coop=coop)
            self._cached_step = conf.step
            return True

        # ---- leader ----
        acquired = bool(self._shm_lock.acquire(blocking)) if ready else False
        claim = ShardLockClaim(self._shm_lock, acquired)
        try:
            join = patience if self._coop_established else float(
                os.getenv("DLROVER_B200_COOP_JOIN_TIMEOUT_S", "5"))
            arrived, followers_ready = ctl.wait_arrivals(local_world, seq, join)
            if not arrived:
                logger.warning(
                    f"Only rank {self._rank} of this node calls save_checkpoint (waited "
                    f"{join:.0f}s for the other local ranks): saving alone from now on, as the "
                    "reference does.")
                ctl.next_coop_seq(aborted=True)
                self._coop_wanted = False
                claim.release()
                return self._SOLO
            node_ready = acquired and followers_ready
            all_ready = node_ready
            if self._saver_group is not None and dist.get_world_size(self._saver_group) > 1:
                # several nodes: their leaders settle it like the reference's saving ranks
                all_ready = check_all_rank_ready(self._saver_group, node_ready)
            if not all_ready:
                ctl.next_coop_seq(aborted=True)
                self.is_skip = True
                logger.info(f"Rank {self._rank} skips the cooperative save of step {conf.step}: "
                            "not every rank is ready (the agent is persisting, or a drain is "
                            "in flight).")
                claim.release()
                return False
            state_dict[DLROVER_CKPT_CONFIG_KEY] = conf
            coop = CoopContext(ctl, 0, local_world, seq - 1, timeout=float(self._save_timeout))
            # the handler opens save `seq` once the segment has its size and the
            # announcement is out; a failed drain leaves writing_shm set (torn segment)
            # and only gives the lock back
            if shards:
                handler.save_shards_as_full(state_dict, coop,
                                            blocking=not self._async_drain or blocking,
                                            stream=self.snapshot_stream,
                                            on_complete=claim.release, on_error=claim.release)
            else:
                handler.save_state_dict(state_dict, blocking=not self._async_drain or blocking,
                                        on_complete=claim.release, on_error=claim.release,
                                        stream=self.snapshot_stream, coop=coop)
        except BaseException:
            if ctl.coop_seq() < seq:
                ctl.next_coop_seq(aborted=True)  # wherever it failed: nobody is left waiting
            # the handler queues a drain as the last step of a save: one that raised has
            # queued none, and a blocking drain that failed has run on_error already
            claim.release()
            raise
        self._coop_established = True
        self._cached_step = conf.step
        return True

    # -- memory save ---------------------------------------------------------------------
    def _is_saving_rank(self) -> bool:
        if self._saving_ranks is None:
            return self._local_rank == self.local_shard_id
        return not self._saving_ranks or self._rank in self._saving_ranks

    # Optional: a CUDA stream for the gather kernel (default: the current one).
    # With a side stream the snapshot overlaps the next forward/backward (which
    # only read the parameters); the caller must then order its next MUTATION of
    # the saved tensors after the snapshot:
    #     torch.cuda.current_stream().wait_event(engine.pack_done_event())
    # right before optimizer.step().
    snapshot_stream = None

    def pack_done_event(self):
        """torch.cuda.Event recorded after the gather kernel of the last save
        (None after an in-place save: use wait_snapshot())."""
        return self._shm_handler.last_pack_event

    # In-place saves (opt-in; also DLROVER_B200_IN_PLACE=1): no HBM snapshot, the
    # drain DMAs straight from the live tensors, so a state that does not fit in HBM
    # twice (8B weights + fp32 Adam moments = 112 GB) is still saved asynchronously.
    # Parameters and optimizer state are only written by optimizer.step(): guard it
    # with engine.guard_optimizer(optimizer) (or call engine.wait_snapshot() yourself
    # before the first write).  Buffers that the forward pass mutates (BatchNorm
    # statistics) are not covered — keep the default snapshot mode for such models.
    @property
    def in_place(self) -> bool:
        return self._shm_handler.in_place

    @in_place.setter
    def in_place(self, value: bool):
        self._shm_handler.in_place = bool(value)

    @property
    def in_place_snapshot_bytes(self) -> int:
        """HBM an in-place save may spend on snapshotting the tail of the state; the
        rest is drained in place first, so wait_snapshot() returns sooner
        (default 0; DLROVER_B200_IN_PLACE_SNAPSHOT_MB)."""
        return self._shm_handler.in_place_snapshot_bytes

    @in_place_snapshot_bytes.setter
    def in_place_snapshot_bytes(self, value: int):
        self._shm_handler.in_place_snapshot_bytes = int(value)

    # Incremental saves (opt-in; also DLROVER_B200_INCREMENTAL=1): a full-snapshot save
    # compares the state with the image the previous save left in the HBM arena and
    # drains only the chunks that changed (a frozen base model does not cross PCIe
    # again).  The segment's bytes are the same as without it.
    @property
    def incremental(self) -> bool:
        return self._shm_handler.incremental

    @incremental.setter
    def incremental(self, value: bool):
        self._shm_handler.incremental = bool(value)

    def wait_snapshot(self):
        """Call before the first write to tensors handed to the last save."""
        self._shm_handler.wait_snapshot()

    def guard_optimizer(self, optimizer):
        """Make `optimizer.step()` wait until the last save no longer reads the
        parameters / optimizer state (torch.optim step pre-hook).  Framework wrappers
        (Megatron's optimizers, DeepSpeed's ZeRO optimizers) are unwrapped down to the
        torch optimizers whose step() does the writing.  Idempotent; returns the list of
        new hook handles."""
        guarded = getattr(self, "_guarded_optimizers", None)
        if guarded is None:
            guarded = self._guarded_optimizers = set()
        handles = []
        for opt in _torch_optimizers(optimizer):
            if id(opt) in guarded:
                continue
            guarded.add(id(opt))
            handles.append(opt.register_step_pre_hook(lambda *_a, **_k: self.wait_snapshot()))
        return handles

    def guard_if_in_place(self, optimizer):
        """Checkpointers that are handed the optimizer call this on every save: with
        in-place saves switched on, the optimizer is guarded automatically."""
        if self.in_place and optimizer is not None:
            self.guard_optimizer(optimizer)

    def save_state_dict_to_memory(self, state_dict, conf: CheckpointConfig, blocking=False):
        """Returns True when the state dict was (or is being) written to shared
        memory, False when this rank does not save or the save was skipped."""
        if self._cooperative():
            done = self._cooperative_save(state_dict, conf, blocking)
            if done is not self._SOLO:
                return done
        if not self._is_saving_rank():
            return False
        conf.rank = self._rank
        conf.group_rank = self._group_rank
        conf.world_size = self._world_size

        pending = self._shm_handler.pending_save()
        if pending is not None and blocking:
            pending.wait()
            pending = None
        # While our own drain runs we still hold the lock: report "not acquired"
        # without bothering the agent.
        acquired = False if pending is not None else self._shm_lock.acquire(blocking)
        claim = ShardLockClaim(self._shm_lock, acquired)
        logger.info(f"{self._rank}-{self._local_rank} acquired the lock of shared memory: "
                    f"{acquired} for step: {conf.step}.")
        all_rank_ready = check_all_rank_ready(self._saver_group, acquired)
        if not all_rank_ready or not state_dict:
            self.is_skip = True
            logger.info(f"Rank {self._rank} skips the save the checkpoint in CPU memory since "
                        "it is saving the latest checkpoint from the CPU memory into the "
                        "storage.")
            claim.release()
            return False
        state_dict[DLROVER_CKPT_CONFIG_KEY] = conf

        def completed():
            claim.release()
            self._replica_manager.backup(self._shm_handler)

        try:
            # replica backup issues collectives: keep those on the calling thread
            sync = not self._async_drain or self._replica_manager.has_replica()
            # a failed drain leaves the segment torn (writing_shm stays set): the lock
            # goes back so later saves are attempted instead of being skipped forever
            self._shm_handler.save_state_dict(state_dict, blocking=sync, on_complete=completed,
                                              on_error=claim.release,
                                              stream=self.snapshot_stream)
        except BaseException:
            # the handler queues a drain as the last step of a save: one that raised has
            # queued none, and a blocking drain that failed has run on_error already
            claim.release()
            raise
        self._cached_step = conf.step
        return True

    def wait_memory_save(self, timeout: Optional[float] = None) -> bool:
        """Block until the drain of the last save has landed in shared memory."""
        return self._shm_handler.wait_pending(timeout)

    def wait_segment_pinned(self, timeout: float = 120.0) -> bool:
        """Block until the background pinning of this rank's part of the segment is done
        (never required; the first transfers simply go through bounce slots)."""
        return self._shm_handler.wait_segment_pinned(timeout)

    def last_save_timings(self):
        """(pack_ms, drain_ms, total_ms) device times of the last finished save."""
        return self._shm_handler.last_timings

    def last_save_stats(self):
        """{"delta": bool, "drained_bytes": int} of the last finished save when it went
        through the incremental path (delta False: it was a full save), else None."""
        return self._shm_handler.last_save_stats

    # -- memory load ---------------------------------------------------------------------
    def get_state_dict_from_memory(self):
        """(step, state dict) from shared memory; (step, {}) when unusable."""
        self._restore_memory_from_replica()
        state_dict = {}
        config = self._shm_handler.get_checkpoint_config(CheckpointConfig())
        passed = verify_all_rank_step_consistent(self._loader_group, config.step)
        if passed and config.step > 0:
            state_dict = self._shm_handler.load_state_dict()
            state_dict.pop(DLROVER_CKPT_CONFIG_KEY, None)
            logger.info(f"Load checkpoint at step {config.step} from memory.")
        return config.step, state_dict

    def load_into(self, target_state_dict, stream=None, strict=True):
        """Scatter the in-memory checkpoint into the live tensors of
        `target_state_dict` (tree as it was passed to save_to_memory, i.e.
        {state name: state dict}).  Returns (step, stats); step 0 = nothing
        restorable in memory."""
        self._restore_memory_from_replica()
        config = self._shm_handler.get_checkpoint_config(CheckpointConfig())
        passed = verify_all_rank_step_consistent(self._loader_group, config.step)
        if not passed or config.step <= 0:
            return 0, {}
        coop = None
        if self._coop_wanted and self._node_group_ok and \
                os.getenv("DLROVER_B200_COOP_RESTORE", "1") not in ("0", "false", "False"):
            # replicated state, every local rank restores: each reads 1/n from host memory,
            # the slices travel between the GPUs over NVLink
            coop = (self._local_rank, env_utils.get_local_world_size(), self._node_group)
        stats = self._shm_handler.restore_into(target_state_dict, stream=stream, strict=strict,
                                               pin_after=not self._coop_wanted, coop=coop)
        return config.step, stats

    def _restore_memory_from_replica(self):
        if not self._replica_manager.has_replica():
            return
        self._shm_handler.init_shared_memory()
        byte_tensor, meta = self._replica_manager.gather(self._shm_handler)
        if byte_tensor is not None and meta and not self._shm_handler.shared_memory:
            shm_size = byte_tensor.size()[0]
            self._shm_handler.init_shared_memory(create=True, size=shm_size)
            self._shm_handler.metadata.set(meta)
            logger.info(f"Restore the checkpoint shard with size = {shm_size} from the replica "
                        "in the memory of the alive node.")
        dist.barrier()

    def wait_latest_checkpoint(self, timeout=1800, max_steps=None):
        """Poll the tracker file until the agent committed `latest_step`."""
        tracker = os.path.join(self.checkpoint_dir, CheckpointConstant.TRACER_FILE_NAME)
        start = time.time()
        while True:
            try:
                with open(tracker, "r") as f:
                    step = int(f.read())
                if step == self.latest_step:
                    if max_steps is not None and step == max_steps:
                        break
                    if self.is_skip or max_steps is None:
                        break
            except (FileNotFoundError, ValueError):
                pass
            if time.time() - start > timeout:
                logger.info(f"Timeout ({timeout})s to wait for the latest step checkpoint.")
                break
            time.sleep(3)

    def _notify_save_event(self, step):
        """Tell the agent to persist `step`.  The event queue holds ONE event
        (multi_process.py SharedQueue maxsize=1, as in the reference): while the agent
        still chews on the previous one — its step-consistency wait alone is 15 s
        (ckpt_saver.py:777) — a blocking put would park the training thread.  Deliver
        inline when the queue is free, else through a forwarder thread, in order."""
        event = CheckpointEvent(type=CheckpointEventType.SAVE, step=step)
        forwarder = getattr(self, "_event_forwarder", None)
        if forwarder is None or forwarder.idle():
            try:
                if self._event_queue.empty():
                    self._event_queue.put(event)
                    return
            except Exception:
                pass  # fall through: let the forwarder retry
        if forwarder is None:
            forwarder = self._event_forwarder = _EventForwarder(self._event_queue)
        forwarder.submit(event)

    # -- to be provided by concrete engines ------------------------------------------------
    @abstractmethod
    def get_saving_ranks(self):
        """Ranks that write shared memory (None = the default policy)."""

    @abstractmethod
    def get_saver_class(self):
        """The AsyncCheckpointSaver subclass the agent must run."""

    @abstractmethod
    def get_local_shard_num(self):
        """Number of shards on this node."""

    @abstractmethod
    def get_global_shard_num(self):
        """Number of shards in the job."""

    @abstractmethod
    def save_to_memory(self, step, state_dict, paths: Dict[str, str], blocking=False):
        """Write {state name: state dict} to shared memory; `paths` maps state
        names to the storage paths the agent would persist them to."""

    @abstractmethod
    def save_to_storage(self, step, state_dict, paths: Dict[str, str]):
        """save_to_memory + tell the agent to persist the step."""

    @abstractmethod
    def load(self, resume_path=""):
        """Return the checkpoint: from memory when possible, else storage."""


class _ShardedRanksMixin:
    """Policy shared by the DeepSpeed / Megatron engines: the first
    `local_shard_num` local ranks of every node are the saving ranks."""

    def get_saving_ranks(self):
        local_world = env_utils.get_local_world_size()
        shards = self.get_local_shard_num()
        return [r for r in range(dist.get_world_size()) if r % local_world < shards]

    def get_local_shard_num(self):
        return min(env_utils.get_local_world_size(), self.get_global_shard_num())

    def _memory_then_barrier(self, step, state_dict, paths, *args):
        ok = True
        if step > self._cached_step:
            ok = self.save_to_memory(step, state_dict, paths, *args)
        if dist.is_initialized():
            dist.barrier()
        return ok


class FullCheckpointEngine(CheckpointEngine):
    """Replicated (DDP-style) state: `local_shard_num` ranks per node write
    shared memory, agent persists `<dir>/<step>/rank_<r>.pt`.

    Example::
        engine = FullCheckpointEngine("/tmp/ckpt", storage)
        engine.save_to_memory(step, {"model_states": sd}, {"model_states": path})
        engine.save_to_storage(step, {"model_states": sd}, {"model_states": path})
        sd = engine.load()
    """

    _supports_cooperative = True

    def __init__(self, checkpoint_dir, storage, local_shard_num=1, global_shard_num=1,
                 comm_backend="", save_timeout=CheckpointConstant.SAVE_TIMEOUT, replica_count=0,
                 async_drain=None, cooperative=None):
        self._cooperative_arg = cooperative
        if replica_count:
            self._cooperative_arg = False  # replica backup reads the whole segment from one rank
        if global_shard_num < local_shard_num:
            global_shard_num = local_shard_num
            logger.info(f"Set global_shard_num to {local_shard_num}.")
        self._local_shard_num = local_shard_num
        self._global_shard_num = global_shard_num
        super().__init__(checkpoint_dir, storage, comm_backend, save_timeout,
                         replica_count=replica_count, async_drain=async_drain)

    def get_saving_ranks(self):
        local_world = env_utils.get_local_world_size()
        ranks = [node * local_world + j
                 for node in range(env_utils.get_group_world_size())
                 for j in range(self._local_shard_num)]
        logger.info(f"The ranks to save checkpoint are {ranks}.")
        return ranks

    def get_local_shard_num(self):
        return self._local_shard_num

    def get_global_shard_num(self):
        return self._global_shard_num

    def get_saver_class(self):
        return DdpCheckpointSaver

    @timer
    def save_to_memory(self, step, state_dict, paths: Dict[str, str], blocking=False):
        conf = CheckpointConfig(step=step, paths=paths)
        return self.save_state_dict_to_memory(state_dict, conf, blocking)

    @timer
    def save_to_storage(self, step, state_dict, paths, blocking=False):
        success = True
        if step > self._cached_step:
            success = self.save_to_memory(step, state_dict, paths, blocking)
        if dist.is_initialized():
            dist.barrier()
        if success and self._local_rank == 0:
            self._notify_save_event(step)
        if success:
            self.latest_step = step
        return success

    def load(self, resume_path=""):
        _, state_dict = self.get_state_dict_from_memory()
        if state_dict:
            logger.info("Load the state dict from the CPU memory buffer.")
            names = list(state_dict.keys())
            if len(names) > 1:
                raise ValueError("The checkpoint shared memory must has only the"
                                 f"state dict of one path. Now, paths are {names}")
            return state_dict[names[0]]
        return self._load_from_storage(resume_path)

    def _load_from_storage(self, resume_path=""):
        def read(path):
            return torch.load(path, map_location="cpu")

        if resume_path:
            return self.storage.read_state_dict(resume_path, read_func=read)
        tracker = os.path.join(self.checkpoint_dir, CheckpointConstant.TRACER_FILE_NAME)
        content: str = self.storage.read(tracker)
        if not content:
            return {}
        path = self._gen_restore_checkpoint_path(int(content.strip()))
        logger.info(f"Load the state dict from {path}")
        return self.storage.read_state_dict(path, read_func=read)

    def _gen_restore_checkpoint_path(self, iteration):
        # unsharded: everyone reads what rank 0 wrote
        who = 0 if self._global_shard_num == 1 else self._rank
        return os.path.join(self.checkpoint_dir, f"{iteration}/rank_{who}.pt")


# north_star's name for the DDP engine; the reference class is FullCheckpointEngine
DdpCheckpointEngine = FullCheckpointEngine


class DeepSpeedCheckpointEngine(_ShardedRanksMixin, CheckpointEngine):
    """DeepSpeedEngine state; sharded by dp rank under ZeRO (`global_shard_num`
    = dp world size), unsharded otherwise."""

    def __init__(self, checkpoint_dir, storage, global_shard_num=1, zero_stage=0, comm_backend="",
                 save_timeout=CheckpointConstant.SAVE_TIMEOUT, async_drain=None):
        self.global_shard_num = global_shard_num
        self.zero_stage = zero_stage
        super().__init__(checkpoint_dir, storage, comm_backend, save_timeout,
                         async_drain=async_drain)

    def get_global_shard_num(self):
        return self.global_shard_num

    def get_saver_class(self):
        return DeepSpeedCheckpointSaver

    @timer
    def save_to_memory(self, step, state_dict, paths, blocking=False):
        conf = CheckpointConfig(step=step, paths=paths)
        return self.save_state_dict_to_memory(state_dict, conf, blocking)

    @timer
    def save_to_storage(self, step, state_dict, paths, blocking=False):
        success = self._memory_then_barrier(step, state_dict, paths, blocking)
        if success and self._local_rank == 0:
            self._notify_save_event(step)
        if success:
            self.latest_step = step
        return success

    def load(self):
        _, state_dict = self.get_state_dict_from_memory()
        name = CheckpointConstant.MODEL_STATES_NAME
        if state_dict and name not in state_dict and self.zero_stage in (1, 2):
            # ZeRO-1/2 do not partition the module: only local rank 0 saved it.
            # Borrow (a private copy of) it from local rank 0's segment.
            donor = SharedMemoryHandler(0, host=False)
            state_dict[name] = copy.deepcopy(donor.load_state_dict()[name])
        return state_dict


class _MegatronTopology:
    def _read_topology(self):
        self._tp_rank = self._pp_rank = self._dp_rank = 0
        self._tp_world_size = self._pp_world_size = 1
        if not dist.is_initialized():
            return
        try:
            from megatron.core import mpu
        except ImportError:  # older Megatron-LM
            from megatron import mpu
        self._tp_rank = mpu.get_tensor_model_parallel_rank()
        self._pp_rank = mpu.get_pipeline_model_parallel_rank()
        self._dp_rank = mpu.get_data_parallel_rank()
        self._tp_world_size = mpu.get_tensor_model_parallel_world_size()
        self._pp_world_size = mpu.get_pipeline_model_parallel_world_size()


class MegatronCheckpointEngine(_ShardedRanksMixin, _MegatronTopology, CheckpointEngine):
    """Megatron-LM model+optimizer dicts: one shard per (tp, pp) coordinate."""

    def __init__(self, checkpoint_dir, storage, comm_backend="",
                 save_timeout=CheckpointConstant.SAVE_TIMEOUT, replica_count=0, async_drain=None):
        self._read_topology()
        super().__init__(checkpoint_dir, storage, comm_backend, save_timeout,
                         replica_count=replica_count, async_drain=async_drain)

    def get_global_shard_num(self):
        return self._pp_world_size * self._tp_world_size

    def get_saver_class(self):
        return MegatronCheckpointSaver

    @timer
    def save_to_memory(self, step, state_dict, paths):
        conf = CheckpointConfig(step=step, paths=paths)
        return self.save_state_dict_to_memory(state_dict, conf)

    @timer
    def save_to_storage(self, step, state_dict, paths):
        succeed = self._memory_then_barrier(step, state_dict, paths)
        if succeed:
            # (the reference forgets this, so its wait_latest_checkpoint on a
            # Megatron engine always runs into the timeout)
            self.latest_step = step
        # one notifier per node: dp rank 0's local rank 0
        if self._dp_rank != 0 or self._local_rank != 0:
            return
        if succeed:
            self._notify_save_event(step)

    def load(self, resume_path=""):
        return self.get_state_dict_from_memory()


class MegatronDistCheckpointEngine(_ShardedRanksMixin, _MegatronTopology, CheckpointEngine):
    """Megatron with distributed optimizer: EVERY rank is a shard (its own
    main_param/exp_avg/exp_avg_sq slice), no DP gather."""

    def __init__(self, checkpoint_dir, storage, comm_backend="",
                 save_timeout=CheckpointConstant.SAVE_TIMEOUT, async_drain=None):
        self._read_topology()
        super().__init__(checkpoint_dir, storage, comm_backend, save_timeout,
                         async_drain=async_drain)

    def get_saving_ranks(self):
        return None  # all ranks

    def get_global_shard_num(self):
        return dist.get_world_size() if dist.is_initialized() else 1

    def get_saver_class(self):
        return MegatronCheckpointSaver

    @timer
    def save_to_memory(self, step, state_dict, paths):
        conf = CheckpointConfig(step=step, paths=paths)
        return self.save_state_dict_to_memory(state_dict, conf)

    @timer
    def save_to_storage(self, step, state_dict, paths):
        success = self._memory_then_barrier(step, state_dict, paths)
        if success and self._local_rank == 0:
            self._notify_save_event(step)
        if success:
            self.latest_step = step

    def load(self, resume_path=""):
        return self.get_state_dict_from_memory()
