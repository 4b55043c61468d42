"""torch.distributed.checkpoint (DCP) over the checkpoint shared-memory segment.

Contract follows the reference @ 468d632,
dlrover/trainer/torch/flash_checkpoint/fsdp_engine.py:
  * SharedMemoryWriter (:158-232): a DCP StorageWriter whose "file" is this
    rank's shm segment: the items of the local SavePlan are laid out back to
    back in plan order (:85-107, :133-155), each answered with
    WriteResult(index, size, _StorageInfo(relative_path="__<rank>_0.distcp",
    offset, length)); DCP Metadata + non-sharded objects go to the agent's
    SharedDict under "dcp_metadata" / "no_shard_data" (:225-232, :512-520);
  * SharedMemoryReader (:235-340) / FileReader (:362-444): read items back from
    the segment, resp. from "<dir>/__<rank>_0.distcp" + ".metadata" on storage;
  * FsdpCheckpointEngine (:447-602): every rank is a shard.

Underneath, tensor items are not copied one at a time with blocking
`shm_tensor.copy_(data)` (:144-147): all CUDA items of the plan become ONE
descriptor table -> one gather kernel into the HBM arena -> one DMA drain; the
write results are known at planning time, so DCP's metadata exchange overlaps
the drain.
"""

from __future__ import annotations

import dataclasses
import io
import os
import pickle
from dataclasses import dataclass
from pathlib import Path
from typing import Any, Dict, List, Optional, Tuple, Union

import torch
import torch.distributed as dist
import torch.distributed.checkpoint as dist_cp
from torch.distributed.checkpoint.metadata import (
    STORAGE_TYPES,
    Metadata,
    MetadataIndex,
    TensorStorageMetadata,
)
from torch.distributed.checkpoint.planner import (
    LoadItemType,
    LoadPlan,
    LoadPlanner,
    ReadItem,
    SavePlan,
    SavePlanner,
    WriteItem,
    WriteItemType,
)
from torch.distributed.checkpoint.storage import StorageReader, StorageWriter, WriteResult
from torch.futures import Future

from ..ckpt_saver import (
    DLROVER_CKPT_CONFIG_KEY,
    CheckpointConfig,
    FsdpDcpSaver,
    SharedMemoryHandler,
)
from ..common import env_utils
from ..common.constants import CheckpointConstant
from ..common.log import default_logger as logger
from .engine import (
    CheckpointEngine,
    ShardLockClaim,
    all_reduce_flags,
    check_all_rank_ready,
    timer,
    verify_all_rank_step_consistent,
)

try:  # moved around between torch releases
    from torch.distributed.checkpoint.filesystem import DEFAULT_SUFFIX
except ImportError:  # pragma: no cover
    DEFAULT_SUFFIX = ".distcp"
from torch.distributed._shard._utils import narrow_tensor_by_index


@dataclass
class _StorageInfo:
    """Where one item lives: file (segment) name, byte offset, byte length."""

    relative_path: str
    offset: int
    length: int


@dataclass
class _StoragePrefix:
    prefix: str


def _tensor_item_size(item: WriteItem) -> int:
    assert item.tensor_data is not None
    numel = 1
    for s in item.tensor_data.size:
        numel *= s
    return numel * torch._utils._element_size(item.tensor_data.properties.dtype)


def _get_buffer_size(files: List[Tuple[str, WriteItem]], planner: SavePlanner) -> int:
    """Bytes needed for all items: tensors by metadata, BYTE_IO by content."""
    total = 0
    for _, item in files:
        if item.type != WriteItemType.BYTE_IO:
            total += _tensor_item_size(item)
        else:
            total += planner.resolve_data(item).getbuffer().nbytes
    return total


def _stage_items(files: List[Tuple[str, WriteItem]], planner: SavePlanner):
    """Resolve every item once and lay the plan out back to back.

    Returns (write_results, no_shard_data, device_ranges, host_ranges,
    raw_chunks, total_bytes).  Non-SHARD items are also collected in
    `no_shard_data` (only rank 0 plans them; they are broadcast so any rank can
    restore from memory)."""
    results: List[WriteResult] = []
    no_shard: Dict[str, STORAGE_TYPES] = {}
    device_ranges, host_ranges, raw_chunks = [], [], []
    offset = 0
    flat_sd = getattr(planner, "state_dict", None)
    for storage_key, item in files:
        data = None
        if item.type == WriteItemType.SHARD and flat_sd is not None:
            # a DTensor's one local shard: skip the planner's lookup (to_local() through
            # autograd + offset search, ~20 us per item, thousands of items per save)
            obj = flat_sd.get(item.index.fqn)
            local = getattr(obj, "_local_tensor", None) if obj is not None else None
            if local is not None and item.tensor_data is not None and \
                    tuple(local.shape) == tuple(item.tensor_data.chunk.sizes):
                data = local
        if data is None and item.type == WriteItemType.BYTE_IO:
            data = getattr(planner, "_fc_resolved", {}).get(item.index.fqn)
        if data is None:
            data = planner.resolve_data(item)
        if torch.is_tensor(data):
            data = data.detach()
        if item.type != WriteItemType.SHARD:
            no_shard[item.index.fqn] = data
        if item.type == WriteItemType.BYTE_IO:
            assert isinstance(data, io.BytesIO)
            buf = data.getbuffer()
            length = buf.nbytes
            raw_chunks.append((buf, offset))
        else:
            assert isinstance(data, torch.Tensor)
            length = data.numel() * data.element_size()
            if length:
                (device_ranges if data.is_cuda else host_ranges).append((data, offset, length))
        results.append(WriteResult(index=item.index, size_in_bytes=length,
                                   storage_data=_StorageInfo(storage_key, offset, length)))
        offset += length
    return results, no_shard, device_ranges, host_ranges, raw_chunks, offset


def _write_item(shm, offset, data, write_item, storage_key) -> Tuple[int, WriteResult]:
    """Write ONE host-resident item at `offset` of a mapped segment and return
    (next offset, WriteResult) — the reference's per-item helper
    (fsdp_engine.py:133-155), kept for callers that drive a raw SharedMemory.
    Device-resident tensors do not go through here: SharedMemoryWriter batches
    them into one gather kernel."""
    if write_item.type == WriteItemType.BYTE_IO:
        assert isinstance(data, io.BytesIO)
        view = data.getbuffer()
        length = view.nbytes
        shm.buf[offset:offset + length] = view
    else:
        assert isinstance(data, torch.Tensor)
        if data.is_cuda:
            raise ValueError("_write_item handles host tensors only; CUDA items are written "
                             "by SharedMemoryWriter.write_data in one batch")
        length = data.numel() * data.element_size()
        if length:
            src = data.detach().contiguous()
            from .. import _native

            _native.host_pack(shm.address, [src.data_ptr()], [offset], [length], 1)
    result = WriteResult(index=write_item.index, size_in_bytes=length,
                         storage_data=_StorageInfo(storage_key, offset, length))
    return offset + length, result


def _write_memory_from_list(shm_handler=None, files=None, planner=None, blocking: bool = True,
                            shm=None):
    """Write all items of `files` into the handler's segment (sized on demand).
    Returns (write_results, no_shard_data, pending).

    Called with a raw mapped segment (`shm=`, the reference's signature,
    fsdp_engine.py:85-107) it writes host-resident items one by one and
    returns (write_results, no_shard_data)."""
    if shm is not None or not hasattr(shm_handler, "write_ranges"):
        segment = shm if shm is not None else shm_handler
        results, no_shard, offset = [], {}, 0
        for storage_key, item in files:
            data = planner.resolve_data(item)
            if torch.is_tensor(data):
                data = data.detach()
            if item.type != WriteItemType.SHARD:
                no_shard[item.index.fqn] = data
            offset, res = _write_item(segment, offset, data, item, storage_key)
            results.append(res)
        return results, no_shard
    results, no_shard, dev, host, raw, total = _stage_items(files, planner)
    if total > 0:
        shm_handler.ensure_segment(total)
    pending = None
    if total > 0:
        pending = shm_handler.write_ranges(dev, host, raw, blocking=blocking,
                                           keepalive=[d for d, _, _ in dev])
    return results, no_shard, pending


class NoShardData(dict):
    """`no_shard_data` of a shard's meta: fqn -> object for every non-sharded entry of the
    state dict (reference fsdp_engine.py:225-232).  Plain objects are ordinary dict items;
    the tensor-valued entries (e.g. one `step` scalar per parameter) live in ONE bytes blob
    + an index and are rebuilt on access — pickling a few hundred torch tensors one by one
    costs tens of milliseconds per save, this costs microseconds."""

    def __init__(self, plain=None, blob: bytes = b"", index=None):
        super().__init__(plain or {})
        self.blob = blob
        self.index = dict(index or {})  # fqn -> (dtype, shape, offset, nbytes)

    def __reduce__(self):
        return (NoShardData, (dict(super().items()), self.blob, self.index))

    def _tensor(self, fqn):
        dtype, shape, off, n = self.index[fqn]
        if n == 0:
            return torch.empty(shape, dtype=dtype)
        return torch.frombuffer(bytearray(self.blob[off:off + n]), dtype=dtype).reshape(shape)

    def __getitem__(self, fqn):
        if fqn in self.index:
            return self._tensor(fqn)
        return super().__getitem__(fqn)

    def get(self, fqn, default=None):
        try:
            return self[fqn]
        except KeyError:
            return default

    def __contains__(self, fqn):
        return fqn in self.index or super().__contains__(fqn)

    def __iter__(self):
        yield from super().__iter__()
        yield from self.index

    def keys(self):
        return list(self)

    def items(self):
        return [(k, self[k]) for k in self]

    def values(self):
        return [self[k] for k in self]

    def __len__(self):
        return super().__len__() + len(self.index)


def no_shard_lookup(no_shard_data, fqn):
    return no_shard_data[fqn]


class _DeferredHostCopy:
    """The CUDA tensors among a plan's non-sharded objects, snapshotted with one
    device-side concatenation on the caller's stream; `get()` — called from the thread
    that publishes the meta — brings them to the host with one copy on a side stream, so
    the training thread never waits for a device-to-host copy."""

    def __init__(self, objects: Dict[str, Any]):
        self._plain = {k: v for k, v in objects.items() if not torch.is_tensor(v)}
        tensors = [(k, v.detach()) for k, v in objects.items() if torch.is_tensor(v)]
        self._cuda = [(k, v) for k, v in tensors if v.is_cuda]
        self._host = [(k, v) for k, v in tensors if not v.is_cuda]
        self._flat = self._event = None
        self._result: Optional[Dict[str, Any]] = None
        if self._cuda:
            self._flat = torch.cat([v.contiguous().reshape(-1).view(torch.uint8)
                                    for _, v in self._cuda])
            self._event = torch.cuda.Event()
            self._event.record()

    def get(self) -> Dict[str, Any]:
        """NoShardData: plain entries as they are, tensors packed into one blob."""
        if self._result is not None:
            return self._result
        out = dict(self._plain)
        chunks, index, off = [], {}, 0
        if self._cuda:
            side = _copy_stream(self._flat.device)
            with torch.cuda.stream(side):
                side.wait_event(self._event)
                host = self._flat.to("cpu", non_blocking=True)
                self._flat.record_stream(side)
            side.synchronize()
            chunks.append(host.numpy().tobytes())
            for k, v in self._cuda:
                n = v.numel() * v.element_size()
                index[k] = (v.dtype, tuple(v.shape), off, n)
                off += n
            self._flat = None
        for k, v in self._host:
            raw = v.contiguous().reshape(-1).view(torch.uint8).numpy().tobytes()
            index[k] = (v.dtype, tuple(v.shape), off, len(raw))
            chunks.append(raw)
            off += len(raw)
        self._result = NoShardData(out, b"".join(chunks), index)
        return self._result


_copy_streams: Dict[int, "torch.cuda.Stream"] = {}


def _copy_stream(device) -> "torch.cuda.Stream":
    idx = device.index if device.index is not None else torch.cuda.current_device()
    s = _copy_streams.get(idx)
    if s is None:
        s = _copy_streams[idx] = torch.cuda.Stream(device=idx)
    return s


class SharedMemoryWriter(StorageWriter):
    """DCP StorageWriter whose storage is the shared-memory segment.

    Beyond the reference's writer (fsdp_engine.py:158-232):
      * `announce` (set by the engine) publishes "segment is being written" before the
        first byte of the segment changes (SharedMemoryHandler.write_ranges decides
        whether inline or from the completion thread with the drain held);
      * the non-sharded objects of the LOCAL plan (before torch dedups replicated entries
        over the ranks) are kept per rank: replicated means every rank has them, so no
        rank needs another rank's copy to restore from its own memory
        (the reference broadcasts rank 0's, fsdp_engine.py:512-520);
      * last_plan / last_results let the engine reuse the plan when the structure of the
        state dict has not changed (no DCP collective at all on such saves).
    """

    def __init__(self, shm_handler: SharedMemoryHandler, blocking: bool = True) -> None:
        super().__init__()
        self.file_name = ""
        self.shm_handler = shm_handler
        self.metadata: Dict[str, Any] = {}
        self.blocking = blocking
        self.pending = None
        self.last_items: List[Tuple[str, WriteItem]] = []
        self.last_plan: Optional[SavePlan] = None
        self.last_results: List[WriteResult] = []
        self.local_non_shard: List[WriteItem] = []
        self.no_shard: Optional[_DeferredHostCopy] = None
        self.announce = None   # Callable[[], None] or None
        self.on_error = None

    def reset(self, checkpoint_id: Union[str, os.PathLike, None] = None) -> None:
        pass

    @classmethod
    def validate_checkpoint_id(cls, checkpoint_id: Union[str, os.PathLike]) -> bool:
        return True

    def set_up_storage_writer(self, is_coordinator: bool, *args, **kwargs) -> None:
        pass

    def prepare_local_plan(self, plan: SavePlan) -> SavePlan:
        # every non-sharded entry this rank HOLDS (the global plan will leave each of
        # them to one rank only)
        self.local_non_shard = [it for it in plan.items if it.type != WriteItemType.SHARD]
        return plan

    def prepare_global_plan(self, global_plan: List[SavePlan]) -> List[SavePlan]:
        return [dataclasses.replace(plan, storage_data=_StoragePrefix(f"__{i}_"))
                for i, plan in enumerate(global_plan)]

    def write_data(self, plan: SavePlan, planner: SavePlanner) -> Future[List[WriteResult]]:
        prefix: _StoragePrefix = plan.storage_data
        self.file_name = f"{prefix.prefix}0{DEFAULT_SUFFIX}"
        files = [(self.file_name, item) for item in plan.items]
        self.last_items = files  # the final local plan, in segment order
        self.last_plan = plan
        results, written_no_shard, dev, host, raw, total = _stage_items(files, planner)
        objects = dict(written_no_shard)
        for item in self.local_non_shard:
            if item.index.fqn not in objects:
                data = planner.resolve_data(item)
                objects[item.index.fqn] = data.detach() if torch.is_tensor(data) else data
        self.no_shard = _DeferredHostCopy(objects)
        self.pending = None
        if total > 0:
            self.shm_handler.ensure_segment(total)
            self.pending = self.shm_handler.write_ranges(
                dev, host, raw, blocking=self.blocking, keepalive=[d for d, _, _ in dev],
                announce=self.announce, on_error=self.on_error)
        elif self.announce is not None:
            self.announce()
        self.last_results = results
        self.metadata["no_shard_data"] = objects  # (reference attribute; host copies: no_shard.get())
        fut: Future[List[WriteResult]] = Future()
        fut.set_result(results)
        return fut

    def finish(self, metadata: Metadata, results: List[List[WriteResult]]) -> None:
        storage_md = {}
        for per_rank in results:
            storage_md.update({wr.index: wr.storage_data for wr in per_rank})
        metadata.storage_data = storage_md
        self.metadata["dcp_metadata"] = metadata


def _load_item(read_item: ReadItem, item_bytes: io.BytesIO, planner: LoadPlanner,
               tensor_md: Optional[TensorStorageMetadata], pickled: bool = False):
    """Hand one stored item to the planner (bytes) or copy it into the
    planner's destination tensor (narrowed to the requested slice)."""
    if read_item.type == LoadItemType.BYTE_IO:
        planner.load_bytes(read_item, item_bytes)
        return
    if pickled:
        tensor = torch.load(item_bytes)
    else:
        assert tensor_md is not None
        flat = torch.frombuffer(item_bytes.getbuffer(), dtype=tensor_md.properties.dtype)
        tensor = flat.reshape(_chunk_shape(tensor_md, read_item))
    tensor = narrow_tensor_by_index(tensor, read_item.storage_offsets, read_item.lengths)
    target = planner.resolve_tensor(read_item).detach()
    assert target.size() == tensor.size(), (
        f"req {read_item.storage_index} mismatch sizes {target.size()} vs {tensor.size()}")
    target.copy_(tensor)
    planner.commit_tensor(read_item, target)


def _chunk_shape(md: TensorStorageMetadata, read_item: ReadItem):
    """Shape of the STORED chunk the item points at (the request may be a
    sub-box of it when the world was resharded); falls back to the requested
    lengths, which is what the reference always assumes (:293-296)."""
    where = read_item.storage_index.offset
    chunks = getattr(md, "chunks", None) or []
    if where is not None:
        for c in chunks:
            if tuple(c.offsets) == tuple(where):
                return tuple(c.sizes)
    if len(chunks) == 1:
        return tuple(chunks[0].sizes)
    return tuple(read_item.lengths)


class SharedMemoryReader(StorageReader):
    """DCP StorageReader over the shared-memory segment."""

    def __init__(self, shm_handler: SharedMemoryHandler) -> None:
        super().__init__()
        self.storage_data: Dict[MetadataIndex, _StorageInfo] = {}
        self.shm_handler = shm_handler
        self.state_dict_metadata: Dict[str, STORAGE_TYPES] = {}
        self.no_shard_data: Dict[str, STORAGE_TYPES] = {}
        self.last_fast_items = 0  # items of the last read_data served by DMA + scatter

    def _device_fast_path(self, read_item: ReadItem, info: _StorageInfo, planner: LoadPlanner):
        """(target, offset, nbytes) when the item is a whole stored chunk going
        into a contiguous CUDA tensor of the same dtype — then it joins the
        one-shot DMA + scatter instead of a per-item pageable H2D copy_
        (reference fsdp_engine.py:303)."""
        if read_item.type == LoadItemType.BYTE_IO or not read_item.storage_index.offset:
            return None
        md = self.state_dict_metadata.get(read_item.storage_index.fqn)
        if not isinstance(md, TensorStorageMetadata):
            return None
        if any(int(o) != 0 for o in read_item.storage_offsets):
            return None
        if tuple(_chunk_shape(md, read_item)) != tuple(read_item.lengths):
            return None
        target = planner.resolve_tensor(read_item).detach()
        if not (target.is_cuda and target.is_contiguous()) or \
                target.dtype != md.properties.dtype or \
                target.numel() * target.element_size() != info.length or \
                tuple(target.size()) != tuple(read_item.lengths):
            return None
        return target, info.offset, info.length

    def read_data(self, plan: LoadPlan, planner: LoadPlanner) -> Future[None]:
        self.shm_handler.wait_pending()
        if self.shm_handler.shared_memory is None:
            self.shm_handler.init_shared_memory()
        fast = []  # (read_item, target, offset, nbytes)
        for read_item in plan.items:
            info = self.storage_data[read_item.storage_index]
            hit = self._device_fast_path(read_item, info, planner)
            if hit is not None:
                fast.append((read_item,) + hit)
                continue
            pickled = False
            if not read_item.storage_index.offset:
                # non-sharded entry: taken from the broadcast copy, not the segment
                data = no_shard_lookup(self.no_shard_data, read_item.storage_index.fqn)
                if isinstance(data, io.BytesIO):
                    item_bytes = data
                else:
                    item_bytes = io.BytesIO()
                    torch.save(data, item_bytes)
                pickled = True
            else:
                assert self.shm_handler.shared_memory is not None
                item_bytes = io.BytesIO(
                    self.shm_handler.shared_memory.buf[info.offset:info.offset + info.length])
            item_bytes.seek(0)
            md = None
            if read_item.type != LoadItemType.BYTE_IO:
                md = self.state_dict_metadata[read_item.storage_index.fqn]
            _load_item(read_item, item_bytes, planner, md, pickled=pickled)
        self.last_fast_items = len(fast)
        if fast:
            self.shm_handler.read_ranges([(t, off, n) for _, t, off, n in fast])
            for read_item, target, _, _ in fast:
                planner.commit_tensor(read_item, target)
        fut: Future = Future()
        fut.set_result(None)
        return fut

    def read_metadata(self, *args, **kwargs) -> Metadata:
        cached = self.shm_handler.metadata.get()
        self.no_shard_data = cached["no_shard_data"]
        return cached["dcp_metadata"]

    def set_up_storage_reader(self, metadata: Metadata, is_coordinator: bool, *args,
                              **kwargs) -> None:
        self.storage_data = metadata.storage_data
        self.state_dict_metadata = metadata.state_dict_metadata
        assert self.storage_data is not None

    def prepare_local_plan(self, plan: LoadPlan) -> LoadPlan:
        return plan

    def prepare_global_plan(self, global_plan: List[LoadPlan]) -> List[LoadPlan]:
        return global_plan

    def reset(self, checkpoint_id: Union[str, os.PathLike, None] = None) -> None:
        pass

    @classmethod
    def validate_checkpoint_id(cls, checkpoint_id: Union[str, os.PathLike]) -> bool:
        return True


class FileReader(StorageReader):
    """DCP StorageReader over the files the agent wrote from the segments
    ("__<rank>_0.distcp" raw bytes + pickled ".metadata")."""

    def __init__(self, path: Union[str, os.PathLike]) -> None:
        super().__init__()
        self.path = Path(path)
        self.storage_data: Dict[MetadataIndex, _StorageInfo] = {}
        self.state_dict_metadata: Dict[str, STORAGE_TYPES] = {}

    def read_data(self, plan: LoadPlan, planner: LoadPlanner) -> Future[None]:
        by_file: Dict[str, List[ReadItem]] = {}
        for item in plan.items:
            by_file.setdefault(self.storage_data[item.storage_index].relative_path,
                               []).append(item)
        for relative_path, items in by_file.items():
            with (self.path / relative_path).open("rb") as f:
                for item in items:
                    info = self.storage_data[item.storage_index]
                    f.seek(info.offset)
                    item_bytes = io.BytesIO(f.read(info.length))
                    md = None
                    if item.type != LoadItemType.BYTE_IO:
                        md = self.state_dict_metadata[item.storage_index.fqn]
                    _load_item(item, item_bytes, planner, md)
        fut: Future = Future()
        fut.set_result(None)
        return fut

    def read_metadata(self, *args, **kwargs) -> Metadata:
        with (self.path / ".metadata").open("rb") as f:
            return pickle.load(f)

    def set_up_storage_reader(self, metadata: Metadata, is_coordinator: bool, *args,
                              **kwargs) -> None:
        self.storage_data = metadata.storage_data
        self.state_dict_metadata = metadata.state_dict_metadata
        assert self.storage_data is not None

    def prepare_local_plan(self, plan: LoadPlan) -> LoadPlan:
        return plan

    def prepare_global_plan(self, global_plan: List[LoadPlan]) -> List[LoadPlan]:
        return global_plan

    def reset(self, checkpoint_id: Union[str, os.PathLike, None] = None) -> None:
        pass

    @classmethod
    def validate_checkpoint_id(cls, checkpoint_id: Union[str, os.PathLike]) -> bool:
        return True


def _save_planner():
    """torch's DefaultSavePlanner, minus one of its two full traversals of the state dict
    when there is nothing for it to do: `_flatten_sharded_tensors` only rewrites nested
    ShardedTensors (FSDP1 + TP); for DTensor / plain states it is a 4 ms no-op per save."""
    from torch.distributed.checkpoint import default_planner as dp

    class _Planner(dp.DefaultSavePlanner):
        def set_up_planner(self, state_dict, storage_meta=None, is_coordinator=False):
            try:
                from torch.distributed._shard.sharded_tensor import ShardedTensor

                if self.flatten_state_dict:
                    state_dict, self.mappings = dp.flatten_state_dict(state_dict)
                    if self.flatten_sharded_tensors and any(
                            isinstance(v, ShardedTensor) for v in state_dict.values()):
                        state_dict = dp._flatten_sharded_tensors(state_dict)
                    self.state_dict = state_dict
                    self.is_coordinator = is_coordinator
                    return
            except (ImportError, AttributeError):
                pass
            super().set_up_planner(state_dict=state_dict, storage_meta=storage_meta,
                                   is_coordinator=is_coordinator)

    return _Planner()


def _dcp_save(state_dict, writer):
    if hasattr(dist_cp, "save"):
        return dist_cp.save(state_dict, storage_writer=writer)
    return dist_cp.save_state_dict(state_dict=state_dict, storage_writer=writer)


class FsdpCheckpointEngine(CheckpointEngine):
    """Sharded FSDP state through DCP: every rank writes its local shards to its
    own segment; the agent dumps each segment as "__<rank>_0.distcp"."""

    def __init__(self, checkpoint_dir: str, storage, comm_backend="",
                 save_timeout=CheckpointConstant.SAVE_TIMEOUT, async_drain=None):
        super().__init__(checkpoint_dir, storage, comm_backend, save_timeout,
                         async_drain=async_drain)
        self._shm_writer = SharedMemoryWriter(shm_handler=self._shm_handler,
                                              blocking=not self._async_drain)
        self._shm_reader = SharedMemoryReader(self._shm_handler)
        self._plan_cache: Optional[Dict[str, Any]] = None
        self._published_meta: Dict[str, Any] = {}
        self.last_save_reused_plan = False

    def get_saving_ranks(self):
        return None  # every rank holds a shard

    # -- plan reuse ---------------------------------------------------------------------
    @staticmethod
    def _describe(value):
        if torch.is_tensor(value):
            placements = getattr(value, "placements", None)
            if placements is not None:  # DTensor
                local = getattr(value, "_local_tensor", None)
                if local is None:
                    local = value.to_local()
                return ("D", tuple(value.shape), value.dtype, placements,
                        tuple(local.shape), local.device.type)
            return ("T", tuple(value.shape), value.dtype, value.device.type)
        shards = getattr(value, "local_shards", None)
        if callable(shards):  # ShardedTensor (FSDP1 SHARDED_STATE_DICT)
            return ("S", tuple(value.size()), value.dtype,
                    tuple((tuple(sh.metadata.shard_offsets), tuple(sh.metadata.shard_sizes))
                          for sh in shards()))
        return ("O", type(value).__name__)

    def _structure_key(self, planner, cached_plan: Optional[SavePlan]):
        """What the DCP plan of this rank depends on: the flattened names, every tensor's
        global/local shape, dtype and placement, and the pickled size of the byte items
        this rank writes (their offsets follow from it)."""
        flat = planner.state_dict
        key = [(k, self._describe(v)) for k, v in flat.items()]
        if cached_plan is not None:
            resolved = {}
            for item in cached_plan.items:
                if item.type == WriteItemType.BYTE_IO:
                    data = planner.resolve_data(item)  # torch.save into a BytesIO: ~1 ms each
                    resolved[item.index.fqn] = data
                    key.append((item.index.fqn, data.getbuffer().nbytes))
            planner._fc_resolved = resolved  # _stage_items takes them from here
        return key

    @timer
    def save_to_memory(self, step, state_dict, paths: Dict[str, str]):
        """`paths["model_states"]` is the DIRECTORY of the step; the agent
        stores this rank's segment there as "__<rank>_0.distcp".

        The first save of a structure runs torch DCP's planning collectives; later saves
        of the same structure reuse this rank's final plan and the global metadata and
        run NO collective besides the readiness all-reduce (which carries one more int:
        "my plan changed")."""
        if self._local_rank != self.local_shard_id:
            return False
        handler, writer = self._shm_handler, self._shm_writer
        pending = handler.pending_save()
        acquired = False if pending is not None else bool(self._shm_lock.acquire(blocking=False))
        claim = ShardLockClaim(self._shm_lock, acquired)
        planner = _save_planner()
        changed = True
        try:
            planner.set_up_planner(state_dict=state_dict, storage_meta=None,
                                   is_coordinator=self._rank == 0)
            cache = self._plan_cache
            key = self._structure_key(planner, cache["plan"] if cache else None)
            changed = cache is None or key != cache["key"] or \
                os.getenv("DLROVER_B200_FSDP_PLAN_CACHE", "1") == "0"
        except Exception as e:  # planner internals moved: always take the DCP path
            logger.warning(f"cannot fingerprint the DCP plan ({e}); planning every save")
            key = None
        not_ready, n_changed = all_reduce_flags(self._saver_group,
                                                [0 if acquired else 1, 1 if changed else 0])
        if not_ready:
            logger.info(f"Rank {self._rank} skips the save the checkpoint in CPU memory since "
                        "it is saving the latest checkpoint from the CPU memory into the "
                        "storage.")
            claim.release()
            return False

        conf = CheckpointConfig(rank=self._rank, group_rank=self._group_rank,
                                world_size=self._world_size, step=step)
        name = CheckpointConstant.MODEL_STATES_NAME
        reuse = n_changed == 0
        previous = dict(self._published_meta)  # what the agent holds for this shard now

        def announce():
            # before the first byte of the segment changes.  A reused plan already knows
            # the whole meta; a new one is still being agreed on: keep the previous tree
            # under the new step with writing_shm set
            if reuse:
                meta = {DLROVER_CKPT_CONFIG_KEY: conf, "dcp_metadata": cache["dcp_metadata"],
                        "no_shard_data": writer.no_shard.get()}
            else:
                meta = {**previous, DLROVER_CKPT_CONFIG_KEY: conf}
            # the meta plane holds the last save's tree (`previous`; under a reused plan
            # the same tree) if that save's final publication went through
            handler._set_meta(meta, True, handler._meta_published, handler._buffer_size)

        # a failed drain leaves the segment torn: the meta keeps writing_shm=True (the
        # agent and a restarted trainer refuse it); only the lock goes back so later saves run
        writer.announce, writer.on_error = announce, claim.release
        try:
            conf.paths = {name: os.path.join(paths[name], f"__{self._rank}_0{DEFAULT_SUFFIX}")}
            if reuse:
                writer.write_data(cache["plan"], planner)
                if [(r.index, r.size_in_bytes) for r in writer.last_results] != cache["results"]:
                    raise RuntimeError("reused DCP plan produced different item sizes")
                dcp_metadata = cache["dcp_metadata"]
            else:
                if hasattr(dist_cp, "save"):
                    dist_cp.save(state_dict, storage_writer=writer, planner=planner)
                else:
                    dist_cp.save_state_dict(state_dict=state_dict, storage_writer=writer,
                                            planner=planner)
                # the coordinator's global metadata goes to every rank
                shared = [writer.metadata.get("dcp_metadata")]
                if dist.is_initialized():
                    dist.broadcast_object_list(shared, src=0)
                dcp_metadata = shared[0]
                self._plan_cache = None
                if key is not None and writer.last_plan is not None:
                    # the byte-item sizes belong to the key the NEXT save is compared with
                    self._plan_cache = {
                        "plan": writer.last_plan, "dcp_metadata": dcp_metadata,
                        "results": [(r.index, r.size_in_bytes) for r in writer.last_results],
                        "key": self._structure_key(planner, writer.last_plan)}
            conf.paths = {name: os.path.join(paths[name], writer.file_name)}
        except BaseException:
            writer.announce = writer.on_error = None
            # a drain that write_data queued may still read the tensors, and its
            # completion publishes nothing: the lock goes back once it is over
            try:
                handler.wait_pending()
            except BaseException:
                pass
            claim.release()
            raise
        writer.announce = writer.on_error = None
        self.last_save_reused_plan = reuse
        no_shard = writer.no_shard

        def completed():
            try:
                meta = {DLROVER_CKPT_CONFIG_KEY: conf, "dcp_metadata": dcp_metadata,
                        "no_shard_data": no_shard.get()}
                # only the header flips when the announcement already carried this tree
                handler._set_meta(meta, False, reuse, handler._buffer_size)
                self._published_meta = {"dcp_metadata": dcp_metadata,
                                        "no_shard_data": meta["no_shard_data"]}
            finally:
                claim.release()

        drain = writer.pending
        if drain is None or drain.done():
            if drain is not None:
                drain.wait()  # re-raises a drain error (its on_error gave the lock back)
            completed()
        else:
            import threading

            def waiter():
                try:
                    drain.wait()
                except BaseException as e:
                    logger.error(f"FSDP shard drain of step {conf.step} failed: {e}")
                    return  # write_ranges' on_error gave the lock back
                try:
                    completed()
                except BaseException as e:
                    logger.error(f"publishing step {conf.step} failed: {e}", exc_info=True)

            t = threading.Thread(target=waiter, name="fc-fsdp-drain", daemon=True)
            t.start()
            self._finalizer = t
        self._cached_step = conf.step
        return True

    def wait_memory_save(self, timeout: Optional[float] = None) -> bool:
        ok = super().wait_memory_save(timeout)
        t = getattr(self, "_finalizer", None)
        if ok and t is not None:
            t.join(timeout)
            ok = not t.is_alive()
        return ok

    def save_to_storage(self, step, state_dict, paths: Dict[str, str]):
        success = True
        if step > self._cached_step:
            success = self.save_to_memory(step, state_dict, paths)
        if dist.is_initialized():
            dist.barrier()
        if self._local_rank == 0 and success:
            logger.info("Put a save event to notify the agent persists checkpoint.")
            self._notify_save_event(step)
        if success:
            self.latest_step = step

    def get_saver_class(self):
        return FsdpDcpSaver

    def get_local_shard_num(self):
        return env_utils.get_local_world_size()

    def get_global_shard_num(self):
        return dist.get_world_size() if dist.is_initialized() else 1

    def load(self, resume_path=""):
        """A StorageReader: over shared memory when every rank holds the same
        step there, else over the files at `resume_path` / the tracked step;
        None when there is nothing to read."""
        self._shm_handler.wait_pending()
        config = self._shm_handler.get_checkpoint_config(CheckpointConfig())
        passed = verify_all_rank_step_consistent(self._saver_group, config.step)
        if passed and not self._shm_handler.no_checkpoint_state():
            logger.info(f"Create a shared memory reader with step {config.step}.")
            return self._shm_reader
        if not resume_path:
            resume_path = self._get_track_resume_path()
        if resume_path and os.path.exists(resume_path):
            logger.info(f"Create a storage reader with path {resume_path}.")
            return FileReader(resume_path)
        return None

    def _get_track_resume_path(self):
        tracker = os.path.join(self.checkpoint_dir, CheckpointConstant.TRACER_FILE_NAME)
        step = self.storage.read(tracker)
        return os.path.join(self.checkpoint_dir, step) if step else ""
