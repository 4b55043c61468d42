"""Shared-memory handler: serialises a (nested) state_dict into the node-local
POSIX shm segment the agent persists from, and reads it back.

Contract (reference @ 468d632, dlrover/python/elastic_agent/torch/ckpt_saver.py):
  * TensorMeta / CheckpointConfig dataclasses (:88-115) and the config key
    "_DLORVER_CKPT_CONFIG" (:50; the typo is format);
  * layout = traversal order of Mapping/list containers, offset = running sum
    of numel*element_size, NO padding (:118-133, :286-301) — SimpleNet + empty
    SGD state is exactly 9640 bytes;
  * segment name "[<run_id>_]ckpt_shm_<local_shard>" (:247-259), meta tree kept
    in the agent's SharedDict "ckpt_meta_<local_shard>" (:261);
  * save protocol: writing_shm=True -> meta set -> bytes -> writing_shm=False
    -> meta set (:303-333); a reader that sees writing_shm gets {} (:343-347);
  * load returns CPU tensors aliasing the segment (:136-161).

What is different underneath: device-resident leaves are NOT copied one by one
with blocking pageable cudaMemcpy (:221-231).  They are described once to
libflashckpt (a cached plan), gathered by one sm_90a kernel into an HBM arena
on the caller's stream, and drained to the pinned segment by DMA on a side
stream; `save_state_dict(..., blocking=False)` returns as soon as the kernel is
enqueued and finishes the protocol from a completion thread.  Host-resident
leaves go straight into the segment with fc_host_pack.  There is no torch
fallback for CUDA leaves: a missing library raises.
"""

from __future__ import annotations

import atexit
import bisect
import contextlib
import copy
import ctypes
import json
import os
import pickle
import threading
import time
import weakref
from collections.abc import Mapping
from dataclasses import dataclass
from datetime import datetime
from typing import Any, Callable, Dict, List, Optional, Tuple

import torch

from . import _native as native
from .common.constants import EventReportConstants, NodeEnv
from .common.log import default_logger as logger
from .common.ctl_segment import ControlSegment
from .common.multi_process import SharedDict, SharedMemory

DLROVER_CKPT_CONFIG_KEY = "_DLORVER_CKPT_CONFIG"


def report_local_event(event_type="", instance="", action="", msg="", labels=None):
    stamp = datetime.now().strftime("%Y-%m-%d, %H:%M:%S")
    logger.info(f"[{stamp}][{event_type}][{instance}][{action}][{msg}][{json.dumps(labels or {})}]")


class CheckpointSharedObjPrefix:
    SAVE_STEP_QNAME = "ckpt_lock_rank_"
    META_NAME = "ckpt_meta_"
    SHM_NAME = "ckpt_shm_"
    SHM_LOCK_NAME = "shm_lock_"


@dataclass
class TensorMeta:
    shape: Tuple[int, ...] = None  # type: ignore
    dtype: torch.dtype = None  # type: ignore
    element_size: int = 0
    numel: int = 0
    offset: int = 0


@dataclass
class CheckpointConfig:
    """Per-shard header stored under DLROVER_CKPT_CONFIG_KEY in the meta tree.

    step: global iteration; writing_shm: True while the trainer is filling the
    segment (a reader must not trust the bytes); paths: state name -> storage
    path the agent persists that sub-dict to."""

    rank: int = 0
    group_rank: int = 0
    world_size: int = 0
    step: int = 0
    writing_shm: bool = False
    paths: Dict[str, str] = None  # type: ignore


class CoopContext:
    """One local rank's part in a cooperative save of a REPLICATED state: all
    `n` local ranks hold the same state dict and each writes only the byte range
    window(total) of the one image into the one segment — over its own PCIe link,
    from a 1/n-sized arena.  `leader` (local rank 0, the reference's saving rank,
    full_ckpt_engine.py:76-89) sizes the segment, publishes the meta and collects the
    others' completion through the control segment's slots."""

    ALIGN = 2 << 20  # slice boundaries: 2 MiB (page- and huge-page-aligned windows)

    def __init__(self, ctl: ControlSegment, index: int, n: int, base_seq: int,
                 timeout: float = 600.0, opened: bool = False):
        self.ctl, self.index, self.n = ctl, index, n
        self.leader = index == 0
        self.seq = base_seq + 1
        self.timeout = timeout
        self.opened = opened  # a follower that has already seen the leader open save `seq`

    @classmethod
    def slice_bytes(cls, total: int, n: int) -> int:
        """Equal slices of ceil(total / n), rounded up to ALIGN: the save windows and the
        slices of the cooperative restore (NCCL all-gather wants them equal) coincide, so
        the part of the segment a rank has page-locked for saving is the part it reads on
        restore."""
        return (total + n * cls.ALIGN - 1) // (n * cls.ALIGN) * cls.ALIGN

    def window(self, total: int) -> Tuple[int, int]:
        w = self.slice_bytes(total, self.n)
        return min(total, self.index * w), min(total, (self.index + 1) * w)


# ------------------------------------------------------------------- traversal --


def _traverse_state_dict(value, visitor: Callable):
    """Depth-first map over Mapping / list containers (tuples are leaves), dict
    order kept, fresh containers returned."""
    if isinstance(value, Mapping):
        return {k: _traverse_state_dict(v, visitor) for k, v in value.items()}
    if isinstance(value, list):
        return [_traverse_state_dict(v, visitor) for v in value]
    return visitor(value)


class _Layout:
    """Result of one planning walk over a state_dict."""

    __slots__ = ("meta", "total", "device_leaves", "host_leaves", "leaf_metas", "reused",
                 "extras", "shape_hash", "unchanged")

    def __init__(self):
        self.meta: Any = None
        self.total = 0
        self.device_leaves: List[Tuple[torch.Tensor, TensorMeta]] = []
        self.host_leaves: List[Tuple[torch.Tensor, TensorMeta]] = []
        self.leaf_metas: List[TensorMeta] = []  # every tensor leaf, traversal order
        self.reused = 0  # leaves whose TensorMeta was taken over from `prev`
        self.extras: list = []  # non-tensor leaves, traversal order
        self.shape_hash = 0     # hash over the keys / container kinds met by the walk
        self.unchanged = False  # same meta tree as `prev` (keys, TensorMetas, extras)


_IMMUTABLE_LEAVES = frozenset({int, float, str, bool, bytes, type(None), complex, torch.dtype,
                               torch.Size, torch.device})


def plan_layout(state_dict, prev: Optional["_Layout"] = None) -> _Layout:
    """Assign every tensor leaf its byte offset (reference layout,
    ckpt_saver.py:286-301) and sort the leaves into device-resident and
    host-resident.  This runs on the training thread at every save, so the walk
    is kept lean: with `prev` (the layout of the previous save) a leaf that
    still has the same shape/dtype at the same offset takes over its TensorMeta
    instead of building a new one."""
    lay = _Layout()
    metas, dev, host = lay.leaf_metas, lay.device_leaves, lay.host_leaves
    prev_metas = prev.leaf_metas if prev is not None else ()
    nprev = len(prev_metas)
    Tensor = torch.Tensor
    total = 0
    reused = 0
    shape_hash = 0
    extras = lay.extras

    def walk(value):
        nonlocal total, reused, shape_hash
        if isinstance(value, Tensor):
            i = len(metas)
            m = prev_metas[i] if i < nprev else None
            if m is not None and m.offset == total and m.dtype is value.dtype \
                    and m.shape == value.shape:
                reused += 1
            else:
                m = TensorMeta(shape=tuple(value.shape), dtype=value.dtype,
                               element_size=value.element_size(), numel=value.numel(),
                               offset=total)
            metas.append(m)
            nbytes = m.numel * m.element_size
            if nbytes:
                (dev if value.is_cuda else host).append((value, m))
                total += nbytes
            return m
        kind = type(value)
        if kind is dict or (kind is not list and isinstance(value, Mapping)):
            out = {}
            for k, v in value.items():
                shape_hash = hash((shape_hash, k))
                out[k] = walk(v)
            shape_hash = hash((shape_hash, len(out), 1))
            return out
        if kind is list or isinstance(value, list):
            shape_hash = hash((shape_hash, len(value), 2))
            return [walk(v) for v in value]
        # non-tensor leaf (tuples included): carried in the meta tree.  The tree is
        # pickled later, possibly on the completion thread: mutable leaves (an args
        # Namespace, user objects) are copied NOW, on the calling thread, so they are
        # captured from the same iteration as the tensors
        if kind is CheckpointConfig:
            value = copy.copy(value)
            if value.paths is not None:
                value.paths = dict(value.paths)
        elif kind not in _IMMUTABLE_LEAVES:
            try:
                value = copy.deepcopy(value)
            except Exception:
                pass
        extras.append(value)
        return value

    lay.meta = walk(state_dict)
    lay.total = total
    lay.reused = reused
    lay.shape_hash = shape_hash
    if prev is not None and reused == len(metas) == nprev and shape_hash == prev.shape_hash \
            and len(extras) == len(prev.extras):
        try:
            # the CheckpointConfig of the save is one of the extras and differs every
            # time: it travels separately (see _MetaPlane), everything else must be equal
            lay.unchanged = all(
                (isinstance(a, CheckpointConfig) and isinstance(b, CheckpointConfig)) or
                (type(a) is type(b) and a == b)
                for a, b in zip(extras, prev.extras))
        except Exception:
            lay.unchanged = False
    return lay


def _local_boxes(value):
    """A sharded leaf as (full shape, dtype, [(local tensor, offsets in the full tensor)])
    or None for anything else.  Understands DTensor (FSDP2, any mesh / placements torch can
    turn into a global offset) and ShardedTensor (FSDP1 SHARDED_STATE_DICT)."""
    if not torch.is_tensor(value) and not hasattr(value, "local_shards"):
        return None
    placements = getattr(value, "placements", None)
    if placements is not None and hasattr(value, "to_local"):
        from torch.distributed.tensor._utils import compute_local_shape_and_global_offset

        local = value.to_local()
        _, offsets = compute_local_shape_and_global_offset(value.shape, value.device_mesh,
                                                           placements)
        return tuple(value.shape), value.dtype, [(local, tuple(int(o) for o in offsets))]
    shards = getattr(value, "local_shards", None)
    if callable(shards):
        return (tuple(value.size()), value.dtype,
                [(sh.tensor, tuple(int(o) for o in sh.metadata.shard_offsets)) for sh in shards()])
    return None


def _box_ranges(local: torch.Tensor, offsets, full_shape, full_off: int):
    """(tensor piece, segment offset, nbytes) for a local box of a row-major full tensor
    that starts at `full_off` in the segment: the box's rows (_view_rows) at the full
    tensor's strides.  A dim-0 shard (every other dim complete) is one contiguous range;
    anything else is one range per run of complete trailing dims.  Each piece is a row of
    the local tensor in its own dtype."""
    shape = tuple(local.shape)
    if local.numel() == 0:
        return []
    if len(shape) != len(full_shape):
        raise ValueError(f"local shard {shape} vs full tensor {tuple(full_shape)}")
    strides, s = [], 1
    for n in reversed(full_shape):
        strides.insert(0, s)
        s *= n
    first = sum(o * st for o, st in zip(offsets, strides))
    rows = _view_rows(shape, strides, first, local.element_size())
    if rows is None:
        raise ValueError("local shard decomposes into too many rows")
    flat = local.detach().contiguous().reshape(len(rows), -1)
    return [(flat[r], full_off + o, n) for r, (o, n) in enumerate(rows)]


def plan_layout_full_from_shards(state_dict):
    """Layout of the FULL (unsharded) state — the one `plan_layout` gives for the gathered
    state dict (reference fsdp.py:238-262 + ckpt_saver.py:286-301) — computed from a state
    dict whose leaves are this rank's SHARDS.  Returns (_Layout, mine) where the layout's
    device/host leaves are the replicated tensors (every rank holds them) and `mine` the
    (tensor piece, segment offset, nbytes) ranges only this rank can write."""
    lay = _Layout()
    metas = lay.leaf_metas
    mine = []
    total = 0

    def walk(value):
        nonlocal total
        boxes = _local_boxes(value)
        if boxes is not None:
            full_shape, dtype, locals_ = boxes
            numel = 1
            for d in full_shape:
                numel *= d
            es = torch.empty(0, dtype=dtype).element_size()
            m = TensorMeta(shape=tuple(full_shape), dtype=dtype, element_size=es, numel=numel,
                           offset=total)
            metas.append(m)
            for local, offsets in locals_:
                mine.extend(_box_ranges(local, offsets, full_shape, total))
            total += numel * es
            return m
        if isinstance(value, torch.Tensor):
            m = TensorMeta(shape=tuple(value.shape), dtype=value.dtype,
                           element_size=value.element_size(), numel=value.numel(), offset=total)
            metas.append(m)
            nbytes = m.numel * m.element_size
            if nbytes:
                total += nbytes
                (lay.device_leaves if value.is_cuda else lay.host_leaves).append((value, m))
            return m
        if isinstance(value, Mapping):
            return {k: walk(v) for k, v in value.items()}
        if isinstance(value, list):
            return [walk(v) for v in value]
        if type(value) not in _IMMUTABLE_LEAVES:
            try:
                value = copy.deepcopy(value)
            except Exception:
                pass
        lay.extras.append(value)
        return value

    lay.meta = walk(state_dict)
    lay.total = total
    return lay, mine


def _read_tensor_from_buf(value, shm: SharedMemory):
    if not isinstance(value, TensorMeta):
        return value
    if value.numel == 0:
        return torch.tensor([], dtype=value.dtype)
    flat = torch.frombuffer(shm.buf, dtype=value.dtype, offset=value.offset, count=value.numel)
    return flat.reshape(value.shape)


def _read_state_dict_from_shm(meta_dict, shm: SharedMemory):
    return _traverse_state_dict(meta_dict, lambda m: _read_tensor_from_buf(m, shm))


def _create_shared_memory(name, create, size=0):
    """Attach to, or (re)create with the requested size, the named segment."""
    if not create:
        try:
            return SharedMemory(name=name)
        except FileNotFoundError:
            return None
    if size == 0:
        logger.warning("Cannot create the shared memory with size = 0.")
        return None
    try:
        return SharedMemory(name=name, create=True, size=size)
    except FileExistsError:
        old = SharedMemory(name=name)
        if old.size == size:
            return old
        logger.info(f"The old size is {old.size} and create a new memory buffer with size {size}.")
        old.unlink()
        old.close()
        return SharedMemory(name=name, create=True, size=size)


def _host_threads() -> int:
    env = os.getenv("DLROVER_B200_HOST_THREADS", "")
    if env:
        return max(1, int(env))
    # measured on config[0] (GPT-2 small on CPU, tools/cpu_config_bench.py): all cores of an
    # 8-vCPU box give 13.7 ms vs 25 ms with half of them (reference: 16.4 ms)
    return max(1, min(32, os.cpu_count() or 1))


# -------------------------------------------------------------- device staging --


def _numa_remote_share(device_index: int) -> int:
    """Of every 256 2-MiB blocks of the segment, how many to place on the OTHER socket.
    DLROVER_B200_NUMA_REMOTE_PER256 forces a value; "auto" derives it from how the local
    ranks' GPUs are spread over the two sockets (a ranks here, b there, a > b: (a-b)/(2a)
    of this rank's pages go across)."""
    env = os.getenv("DLROVER_B200_NUMA_REMOTE_PER256", "0").strip().lower()
    if env != "auto":
        try:
            return max(0, min(256, int(env or 0)))
        except ValueError:
            return 0
    try:
        local_world = int(os.getenv("LOCAL_WORLD_SIZE", "1") or 1)
        mine, n_nodes = native.device_numa_node(device_index)
        if n_nodes != 2 or mine < 0 or local_world < 3:
            return 0
        here = sum(1 for d in range(local_world) if native.device_numa_node(d)[0] == mine)
        there = local_world - here
        if here < 3 or here <= there:
            return 0
        return int(256 * (here - there) / (2 * here))
    except Exception:
        return 0


def _view_rows(shape, stride, first: int, es: int, max_rows: int = 1 << 16,
               min_row_bytes: int = 0):
    """The bytes of a strided view in logical (row-major) order, as (byte offset, nbytes)
    rows starting from element `first`: one row for a dense view, one per dense row when
    the trailing dims are dense ("row-strided"; size-1 dims count as dense).  None when
    there would be more than `max_rows` rows, rows under `min_row_bytes`, or a negative
    stride among the row dims.  The one row walker: tensors, boxes of row-major tensors
    and views stored in files all map onto it."""
    sizes, strides = list(shape), list(stride)
    k, expect = len(sizes), 1  # dims [k:] form the dense row
    while k > 0 and (sizes[k - 1] == 1 or strides[k - 1] == expect):
        expect *= sizes[k - 1]
        k -= 1
    n_rows = 1
    for d in range(k):
        n_rows *= sizes[d]
    if expect * es < min_row_bytes or n_rows > max_rows or any(s < 0 for s in strides[:k]):
        return None
    out, idx = [], [0] * k
    for _ in range(n_rows):
        out.append(((first + sum(i * s for i, s in zip(idx, strides))) * es, expect * es))
        for d in range(k - 1, -1, -1):
            idx[d] += 1
            if idx[d] < sizes[d]:
                break
            idx[d] = 0
    return out


def _row_ranges(t: torch.Tensor, off: int, max_rows: int = 1 << 16, min_row_bytes: int = 256):
    """A non-contiguous tensor whose trailing dims are dense ("row-strided": w[:, :k],
    w[::2], a transposed-then-sliced view...) as one (ptr, offset, nbytes) range per dense
    row, in logical (row-major) order — exactly the bytes `shm.copy_(t)` deposits
    (reference ckpt_saver.py:228-231) without a device-side .contiguous() copy.
    None for a dense tensor and when the rows would be too many / too small (the caller
    takes the tensor whole or repacks it then)."""
    rows = _view_rows(t.shape, t.stride(), 0, t.element_size(), max_rows, min_row_bytes)
    if rows is None or len(rows) == 1:  # one row: the tensor is dense
        return None
    base = t.data_ptr()
    return [(base + o, off + r * n, n) for r, (o, n) in enumerate(rows)]


def _target_rows(t: torch.Tensor):
    """(address, nbytes) rows of a dense or row-strided restore target in logical order,
    else None.  A dense tensor is one row; CUDA rows follow _row_ranges' minimum row size
    (the scatter kernels); a CPU row is one pread of any size."""
    if t.is_contiguous():
        return [(t.data_ptr(), t.numel() * t.element_size())]
    rows = _row_ranges(t, 0) if t.is_cuda else _row_ranges(t, 0, min_row_bytes=1)
    return None if rows is None else [(p, n) for p, _, n in rows]


# kind of the non-finite scan per dtype: complex as its float components; integers, bool
# and the other float8 kinds are not scanned
_SCAN_KINDS = {
    torch.float16: native.KIND_F16, torch.bfloat16: native.KIND_BF16,
    torch.float32: native.KIND_F32, torch.float64: native.KIND_F64,
    torch.complex64: native.KIND_F32, torch.complex128: native.KIND_F64,
    torch.float8_e5m2: native.KIND_E5M2, torch.float8_e4m3fn: native.KIND_E4M3FN,
}


def _leaf_paths(state_dict) -> List[str]:
    """Dotted path of every tensor leaf (sharded ones included), in the order of the
    layout walks above."""
    out: List[str] = []

    def walk(value, path):
        if isinstance(value, torch.Tensor) or hasattr(value, "local_shards"):
            out.append(path)
        elif isinstance(value, Mapping):
            for k, v in value.items():
                walk(v, f"{path}.{k}" if path else str(k))
        elif isinstance(value, list):
            for i, v in enumerate(value):
                walk(v, f"{path}.{i}" if path else str(i))

    walk(state_dict, "")
    return out


def _triples(leaves):
    return [(t, m.offset, m.numel * m.element_size) for t, m in leaves]


def _clip_triples(triples, lo: int, hi: int):
    """(tensor, segment offset, nbytes) triples cut to segment bytes [lo, hi): the part of
    a tensor that falls inside becomes a uint8 view on its bytes."""
    out = []
    for t, off, n in triples:
        a, b = max(off, lo), min(off + n, hi)
        if b <= a:
            continue
        if a == off and b == off + n:
            out.append((t, off, n))
            continue
        flat = t.detach()
        if not flat.is_contiguous():
            flat = flat.contiguous()
        out.append((flat.reshape(-1).view(torch.uint8)[a - off:b - off], a, b - a))
    return out


def _clip_ranges(prepared, lo: int, hi: int):
    """The parts of (ptrs, offsets, lengths) that fall into segment bytes [lo, hi)."""
    ptrs, offs, lens = [], [], []
    for p, o, n in zip(*prepared):
        a, b = max(o, lo), min(o + n, hi)
        if b > a:
            ptrs.append(p + (a - o))
            offs.append(a)
            lens.append(b - a)
    return ptrs, offs, lens


class _DeviceStager:
    """Owns the libflashckpt context usage for ONE segment: host registration,
    arena sizing and the cached plan."""

    # segments up to this size are pinned inline (tens of ms); larger ones are pinned
    # by a library thread after the first transfer, which goes through bounce slots
    SYNC_PIN_MAX = 256 << 20

    def __init__(self, device_index: int):
        self.device_index = device_index
        self.ctx = native.get_context(device_index)
        self._attached: Optional[Tuple[int, int]] = None  # (address, bytes) of our window
        self._pin_started = False
        self._plans: Dict[str, native.Plan] = {}  # role -> plan
        self.register_seconds = 0.0
        self._warned_no_arena = False

    @staticmethod
    def _pin_mode() -> str:
        # "background" (default) | "sync" (pin inline, as round 1 did) | "none"
        return os.getenv("DLROVER_B200_PIN", "background").strip().lower()

    def attach(self, shm: SharedMemory, lo: int = 0, hi: Optional[int] = None):
        """Prepare the bytes [lo, hi) of the segment (default: all of it) as this
        process's DMA target: NUMA placement now (pages are faulted in by whoever
        writes them first), pinning inline for small windows, else in the background
        after the first transfer (pin_in_background)."""
        hi = shm.size if hi is None else hi
        window = (shm.dma_address + lo, hi - lo)
        if window == self._attached:
            return
        self.detach()
        self._attached = window
        addr, size = window
        if size <= 0:
            return
        self.ctx.host_bind_numa(addr, size, _numa_remote_share(self.device_index))
        if self._pin_mode() == "sync" or (size <= self.SYNC_PIN_MAX and self._pin_mode() != "none"):
            t0 = time.time()
            self.ctx.host_register(addr, size, prefault_threads=_host_threads())
            self.register_seconds = time.time() - t0
            self._pin_started = True
            logger.info(f"Pinned the {size / 2**30:.2f} GiB checkpoint segment for DMA "
                        f"in {self.register_seconds:.2f}s.")

    def pin_in_background(self):
        """Start pinning the window on a library thread (no-op when done/started)."""
        if self._attached is None or self._pin_started or self._pin_mode() == "none":
            return
        addr, size = self._attached
        if size <= 0:
            return
        self.ctx.host_register_background(addr, size)
        self._pin_started = True

    def pinned(self) -> bool:
        return bool(self._attached) and self._pin_started and self.ctx.host_ready(self._attached[0])

    def wait_pinned(self, timeout: float = 120.0) -> bool:
        deadline = time.time() + timeout
        while not self.pinned():
            if not self._pin_started or time.time() > deadline:
                return False
            time.sleep(0.01)
        return True

    def detach(self):
        if self._attached is not None and self._pin_started:
            try:
                self.ctx.host_unregister(self._attached[0])
            except native.NativeError as e:
                logger.warning(f"host_unregister: {e}")
        self._attached = None
        self._pin_started = False

    @staticmethod
    def prepare_ranges(ranges: List[Tuple[torch.Tensor, int, int]], keepalive: list,
                       for_write: bool = False):
        """(tensor, segment offset, nbytes) -> parallel lists (ptrs, offsets, lengths).
        Dense tensors are one range; row-strided ones one range per dense row;
        anything else is repacked on the device first (save only — the copy lives in
        `keepalive` until the gather kernel has consumed it)."""
        ptrs, offs, lens = [], [], []
        for t, off, nbytes in ranges:
            if t.is_contiguous():
                ptrs.append(t.data_ptr())
                offs.append(off)
                lens.append(nbytes)
                continue
            rows = _row_ranges(t, off)
            if rows is None:
                if for_write:
                    raise ValueError("restore needs dense or row-strided CUDA targets "
                                     f"(got shape {tuple(t.shape)}, strides {t.stride()})")
                t = t.detach().contiguous()
                keepalive.append(t)
                ptrs.append(t.data_ptr())
                offs.append(off)
                lens.append(nbytes)
                continue
            for p, o, n in rows:
                ptrs.append(p)
                offs.append(o)
                lens.append(n)
        return ptrs, offs, lens

    def plan_for(self, prepared, role: str = "save", stream=None, base: int = 0,
                 compact: bool = False):
        """prepared: (ptrs, segment offsets, lengths) from prepare_ranges.  `base` is
        subtracted from the offsets (a window of the segment staged on its own: arena
        byte 0 = segment byte `base`, the host base moves by the same amount).
        One plan object per role ("save" / "restore"); when the tensors moved (FSDP
        hands out fresh ones on every state_dict()) the plan is re-targeted in place
        with a stream-ordered table upload."""
        ptrs, offs, lens = prepared
        if base:
            offs = [o - base for o in offs]
        host_offs = None
        if compact:
            # ranges scattered over the segment, packed into a small arena; every arena
            # offset congruent to its source mod 16: all of them take the bulk (TMA) kernel
            host_offs, offs, a = offs, [], 0
            for p, n in zip(ptrs, lens):
                a += (p - a) % 16
                offs.append(a)
                a += n
        key = native._plan_key(ptrs, offs, lens, host_offs)
        plan = self._plans.get(role)
        if plan is not None and plan.key == key:
            return plan
        if plan is None:
            plan = self._plans[role] = self.ctx.plan(ptrs, offs, lens, host_offsets=host_offs)
        else:
            plan.update(ptrs, offs, lens, stream, host_offsets=host_offs)
        return plan

    ARENA_FULL, ARENA_WINDOWED, ARENA_NONE = "full", "windowed", "none"

    @classmethod
    def reserve_arena(cls, ctx: native.Context, end: int) -> str:
        """Make room in the arena of `ctx` for a plan that ends at arena offset `end`.
        "full": the arena covers the plan.  "windowed": DLROVER_B200_ARENA_LIMIT_MB caps
        the arena below the plan, which is then streamed through it window by window.
        "none": HBM has no room for it."""
        if end <= ctx.arena_info()[1]:
            return cls.ARENA_FULL
        forced = int(os.getenv("DLROVER_B200_ARENA_LIMIT_MB", "0") or 0)
        if forced:
            limit = max(8, forced) << 20
            ctx.set_arena_limit(limit)
            ctx.arena_reserve(min(end, limit))
            return cls.ARENA_FULL if end <= limit else cls.ARENA_WINDOWED
        try:
            ctx.arena_reserve(end)
            return cls.ARENA_FULL
        except native.NativeError as e:
            if e.code != native.FC_ENOMEM:
                raise
        return cls.ARENA_NONE

    def ensure_arena(self, plan) -> str:
        """Make room for the snapshot of `plan` in HBM (reserve_arena).  "full": the
        training stream then only waits for the gather kernel.  "windowed": saves and
        restores block.  "none": the caller saves in place instead (DMA straight from
        the tensors)."""
        mode = self.reserve_arena(self.ctx, plan.arena_end)
        if mode == self.ARENA_NONE and not self._warned_no_arena:
            self._warned_no_arena = True
            free, _ = torch.cuda.mem_get_info(self.device_index)
            logger.warning(
                f"No room for a {plan.arena_end / 2**30:.1f} GiB snapshot arena in HBM "
                f"({free / 2**30:.1f} GiB free): checkpoints are drained in place (DMA straight "
                "from the tensors). Saves block until the data is in shared memory unless the "
                "engine runs with in_place=True and the optimizer is guarded (see README, "
                "'in-place saves').")
        return mode

    def close(self):
        for p in self._plans.values():
            p.destroy()
        self._plans.clear()
        self.detach()


class PendingSave:
    """Handle of a save whose drain is still running on the copy stream."""

    def __init__(self, ctx: Optional[native.Context], ticket: int, finish: Callable[[], None],
                 keepalive: list, announce: Optional[Callable[[], None]] = None,
                 on_error: Optional[Callable[[], None]] = None, delta: bool = False):
        self._on_error = on_error
        self._ctx = ctx
        self._ticket = ticket
        self._delta = delta  # issued through save_delta_async: `stats` is filled in
        self._finish = finish
        self._keepalive = keepalive
        self._announce = announce  # set <=> the drain is held until it has run
        self._done = threading.Event()
        self._error: Optional[BaseException] = None
        self._lock = threading.Lock()
        self.timings: Optional[Tuple[float, float, float]] = None
        self.stats: Optional[Dict[str, Any]] = None

    def _complete(self):
        """Wait for the DMA, then close the protocol.  Runs exactly once."""
        with self._lock:
            if self._done.is_set():
                return
            try:
                if self._announce is not None:
                    try:
                        self._announce()  # writing_shm=True to the agent, then raw chunks
                    except BaseException:
                        # the agent does not know the segment is about to change: leave
                        # every byte of it alone (the previous checkpoint stays valid)
                        if not self._ctx.save_cancel(self._ticket):
                            self._ctx.save_release(self._ticket)
                            self._ctx.save_wait(self._ticket)
                        raise
                    self._ctx.save_release(self._ticket)
                if self._ctx is not None:
                    self._ctx.save_wait(self._ticket)
                    self.timings = self._ctx.save_timings(self._ticket)
                    if self._delta:
                        was_delta, nbytes = self._ctx.save_delta_stats(self._ticket)
                        self.stats = {"delta": was_delta, "drained_bytes": nbytes}
                self._finish()
            except BaseException as e:  # surfaced by wait()
                self._error = e
                logger.error(f"flash checkpoint drain failed: {e}", exc_info=True)
                if self._on_error is not None:
                    try:
                        self._on_error()  # e.g. give the shard lock back
                    except BaseException:
                        logger.error("error handler of the failed drain raised", exc_info=True)
            finally:
                self._keepalive.clear()
                self._done.set()

    def done(self) -> bool:
        return self._done.is_set()

    def wait(self, timeout: Optional[float] = None) -> bool:
        ok = self._done.wait(timeout)
        if ok and self._error is not None:
            raise self._error
        return ok


# ------------------------------------------------------------------ meta plane --


def _ctl_enabled() -> bool:
    if os.getenv("DLROVER_B200_WIRE_COMPAT", "0") == "1":
        return False  # the peer is the reference: SharedDict only
    return os.getenv("DLROVER_B200_CTL", "1") not in ("0", "false", "False")


class _MetaPlane:
    """Where the meta tree of a shard lives.  Same surface as the reference's
    SharedDict (get / set / unlink / close; ckpt_saver.py:261, multi_process.py:579-672)
    over two stores:

      * the control segment (common/ctl_segment.py) when the agent created one: the
        pickled tree is rewritten only when it changed, every save just flips the
        seqlock'd header (step, writing_shm, the pickled CheckpointConfig) — no socket
        round trip, no SharedDict.set on the steady-state save path;
      * the agent's SharedDict otherwise (the reference's agent, or
        DLROVER_B200_CTL=0 / DLROVER_B200_WIRE_COMPAT=1).
    """

    def __init__(self, shard_id: int, host: bool):
        self._shard = shard_id
        self._host = host
        self.dict = SharedDict(name=CheckpointSharedObjPrefix.META_NAME + str(shard_id),
                               create=host)
        self._ctl: Optional[ControlSegment] = None
        self._ctl_looked = False
        self.next_unchanged = False   # set by the handler right before a steady-state set()
        self.payload_bytes = 0
        self.ctl_publishes = 0
        self.dict_sets = 0
        if host and _ctl_enabled():
            try:
                self._ctl = ControlSegment.create(shard_id)
            except OSError as e:
                logger.warning(f"no control segment for shard {shard_id}: {e}")
            self._ctl_looked = True

    @property
    def ctl(self) -> Optional[ControlSegment]:
        if not _ctl_enabled():
            return None
        if self._ctl is not None and self._ctl.stale():
            self._ctl.close()
            self._ctl, self._ctl_looked = None, False
        if self._ctl is None and not self._ctl_looked:
            self._ctl = ControlSegment.attach(self._shard)
            self._ctl_looked = True
        return self._ctl

    # keys whose values change at every save: they travel in the small per-save blob
    # next to the CheckpointConfig instead of forcing the big tree to be re-pickled
    VOLATILE_KEYS = ("no_shard_data",)

    def set(self, meta_dict):
        unchanged, self.next_unchanged = self.next_unchanged, False
        ctl = self.ctl
        # the owner keeps a SharedDict-only peer (the reference's trainer) working:
        # it writes through the control segment only once a trainer has used it
        if ctl is not None and (not self._host or ctl.has_meta()):
            if not meta_dict:
                ctl.clear()
                self.dict._dict = {}
                return
            conf = meta_dict.get(DLROVER_CKPT_CONFIG_KEY)
            volatile = {DLROVER_CKPT_CONFIG_KEY: conf}
            for k in self.VOLATILE_KEYS:
                if k in meta_dict:
                    volatile[k] = meta_dict[k]
            small = pickle.dumps(volatile, protocol=pickle.HIGHEST_PROTOCOL)
            in_small = set(volatile)
            if len(small) > ctl.conf_capacity:
                in_small = {DLROVER_CKPT_CONFIG_KEY}
                small = pickle.dumps({DLROVER_CKPT_CONFIG_KEY: conf},
                                     protocol=pickle.HIGHEST_PROTOCOL)
                unchanged = False  # the volatile objects ride in the big blob this time
            blob = None
            if not unchanged or not ctl.has_meta():
                rest = {k: v for k, v in meta_dict.items() if k not in in_small}
                blob = pickle.dumps(rest, protocol=pickle.HIGHEST_PROTOCOL)
            ok = ctl.publish(step=int(getattr(conf, "step", 0) or 0),
                             writing=bool(getattr(conf, "writing_shm", False)),
                             payload_bytes=int(self.payload_bytes), conf_blob=small,
                             meta_blob=blob)
            if ok:
                self.ctl_publishes += 1
                self.dict._dict = meta_dict
                return
            logger.warning("meta tree does not fit the control segment: using the SharedDict")
            ctl.clear()
        self.dict_sets += 1
        self.dict.set(meta_dict)

    def get(self, local: bool = False):
        if local:
            return self.dict.get(local=True)
        ctl = self.ctl
        if ctl is not None:
            snap = ctl.snapshot()
            if snap is not None:
                _step, _writing, _payload, conf_blob, _gen, rest = snap
                out = dict(rest)
                volatile = pickle.loads(conf_blob) if conf_blob else {}
                conf = volatile.pop(DLROVER_CKPT_CONFIG_KEY, None)
                out.update(volatile)
                if conf is not None:
                    out[DLROVER_CKPT_CONFIG_KEY] = conf
                return out
        return self.dict.get()

    def unlink(self):
        self.dict.unlink()
        if self._ctl is not None and self._host:
            self._ctl.unlink()

    def close(self):
        try:
            self.dict.close()
        finally:
            if self._ctl is not None:
                self._ctl.close()
                self._ctl = None

    def __bool__(self):
        return True


# --------------------------------------------------------------------- restores --


def _match_tree(target, tree, leaf_type, sequences, strict: bool):
    """Pair every `leaf_type` leaf of the checkpoint `tree` with the tensor at the same
    place in `target`: the tree rules of every restore.  Mappings match by key (the meta
    header key is skipped; a key on one side only raises when strict), `sequences` by
    position and length; the shape and dtype must be exact; other leaves are ignored.
    Returns [(path, target tensor, leaf)] without 0-element leaves."""
    pairs = []

    def walk(tgt, src, path):
        if isinstance(src, Mapping):
            if not isinstance(tgt, Mapping):
                raise KeyError(f"{path}: checkpoint has a dict, target has {type(tgt).__name__}")
            for k, s in src.items():
                if k == DLROVER_CKPT_CONFIG_KEY:
                    continue
                sub = f"{path}.{k}" if path else str(k)
                if k not in tgt:
                    if strict:
                        raise KeyError(f"{sub}: missing in target")
                    continue
                walk(tgt[k], s, sub)
            if strict:
                extra = [k for k in tgt if k not in src]
                if extra:
                    raise KeyError(f"{path}: target keys not in checkpoint: {extra}")
        elif isinstance(src, sequences):
            if not isinstance(tgt, sequences) or len(tgt) != len(src):
                raise KeyError(f"{path}: list length/type mismatch")
            for i, s in enumerate(src):
                walk(tgt[i], s, f"{path}.{i}" if path else str(i))
        elif isinstance(src, leaf_type):
            if not torch.is_tensor(tgt):
                raise KeyError(f"{path}: checkpoint has a tensor, target has {type(tgt).__name__}")
            if tuple(tgt.shape) != tuple(src.shape) or tgt.dtype != src.dtype:
                raise ValueError(f"{path}: shape/dtype mismatch {tuple(tgt.shape)}/{tgt.dtype} "
                                 f"vs {tuple(src.shape)}/{src.dtype}")
            if src.numel:
                pairs.append((path, tgt, src))

    walk(target, tree, "")
    return pairs


def _timed_restore(ctx: native.Context, plan, enqueue) -> Optional[Dict[str, float]]:
    """Run the restore of `plan` that enqueue() starts and wait for it: device_bytes,
    fill_ms, scatter_ms, wall_ms.  None when enqueue() returns False (nothing started)."""
    t0 = time.perf_counter()
    if enqueue() is False:
        return None
    ctx.restore_wait()
    wall_ms = (time.perf_counter() - t0) * 1e3
    fill, scatter, _ = ctx.restore_timings()
    return {"device_bytes": float(plan.payload_bytes), "fill_ms": fill, "scatter_ms": scatter,
            "wall_ms": wall_ms}


# --------------------------------------------------------------------- handler --


class SharedMemoryHandler:
    """Writes / reads the state dict of one local shard to / from shared memory.

    Args:
        local_rank: index of the local shard (names the segment and meta dict).
        host: True on the agent (owns the SharedDict server), False in a
            training process.
    """

    def __init__(self, local_rank, host=True):
        self._buffer_size = 0
        self._local_rank = local_rank
        run_id = os.getenv(NodeEnv.TORCHELASTIC_RUN_ID, "")
        base = CheckpointSharedObjPrefix.SHM_NAME + str(local_rank)
        self._shm_name = f"{run_id}_{base}" if run_id else base
        self.shared_memory: Optional[SharedMemory] = None
        self.metadata = _MetaPlane(local_rank, host)
        self._need_creation = True
        self._announced_once = False
        self._meta_published = False  # the last save's meta tree reached the meta plane
        self._completion_queue = None
        self._layout: Optional[_Layout] = None  # of the previous save (TensorMeta reuse)
        self._stager: Optional[_DeviceStager] = None
        self._pending: Optional[PendingSave] = None
        self._master_client = None
        self.last_timings: Optional[Tuple[float, float, float]] = None
        # torch.cuda.Event recorded right after the last gather kernel
        self.last_pack_event = None
        # in-place saves (no HBM snapshot): opt-in, see write_ranges
        self.in_place = os.getenv("DLROVER_B200_IN_PLACE", "0") == "1"
        # HBM an in-place save may spend on snapshotting the tail of the state (the rest
        # is drained in place first): shortens the time the tensors stay frozen
        self.in_place_snapshot_bytes = int(os.getenv("DLROVER_B200_IN_PLACE_SNAPSHOT_MB", "0")) << 20
        self.last_save_in_place = False
        # incremental saves: opt-in, see write_ranges
        self.incremental = os.getenv("DLROVER_B200_INCREMENTAL", "0") == "1"
        # {"delta": bool, "drained_bytes": int} of the last finished save when it went
        # through the incremental path (None for any other save)
        self.last_save_stats: Optional[Dict[str, Any]] = None
        self._delta_segment = None  # the mapping the last incremental save wrote to
        self.last_restore_stats: Dict[str, float] = {}
        self.last_hybrid_cut = None
        self._snapshot_ceiling = 0  # largest snapshot arena HBM turned out to have room for
        self._scanned = None  # (state dict, layout, mine) of the last scan_nonfinite
        self._last_ticket = None
        if not host:
            # a drain still in flight when the interpreter exits must finish (the
            # completion thread is a daemon): otherwise the last checkpoint of a
            # run that ends right after save_checkpoint() would stay half written
            ref = weakref.ref(self)
            atexit.register(lambda: ref() is not None and ref()._finish_at_exit())

    # -- lifecycle ------------------------------------------------------------------
    def close(self):
        try:
            self.wait_pending()
        except BaseException as e:  # already logged by the completion thread
            logger.warning(f"closing after a failed drain: {e}")
        if self._completion_queue is not None:
            self._completion_queue.put(None)
            self._completion_queue = None
        if self._stager is not None:
            self._stager.close()
            self._stager = None
        if self.shared_memory:
            self.shared_memory.close()

    def unlink(self):
        if not self.shared_memory:
            self.init_shared_memory()  # may have been created by another process
        if self.shared_memory:
            self.shared_memory.unlink()
        if self.metadata:
            self.metadata.unlink()

    def reset(self):
        self._need_creation = True

    def init_shared_memory(self, create=False, size=0):
        self.shared_memory = _create_shared_memory(self._shm_name, create=create, size=size)
        self._need_creation = False

    def refresh_mapping(self):
        """(Re-)attach when this process has no mapping yet or its mapping is stale: the
        writer re-creates the segment when the payload size changes (optimizer state
        filling in after the first save, DCP byte items whose pickled size drifts), and
        a reader that kept the old mapping would persist old bytes under the new meta.
        Call with the shard lock held / after the meta said writing_shm=False."""
        shm = self.shared_memory
        if shm is not None and not self._need_creation and not shm.stale():
            return
        if self._pending is not None:
            return  # the writer side never refreshes under its own drain
        if shm is not None:
            if self._stager is not None:
                self._stager.detach()
            shm.close()
            self.shared_memory = None
        self._delta_invalidate()
        self.init_shared_memory(create=False)

    def _delta_invalidate(self):
        """The segment was (re-)mapped: the next incremental save must be a full one."""
        self._delta_segment = None
        if self._stager is not None:
            self._stager.ctx.delta_invalidate()

    def _create_tensor_meta(self, value):
        """Meta of one leaf at the current end of the layout (API parity with
        the reference's planner hook, ckpt_saver.py:286-301)."""
        if not torch.is_tensor(value):
            return value
        meta = TensorMeta(shape=tuple(value.shape), dtype=value.dtype,
                          element_size=value.element_size(), numel=value.numel(),
                          offset=self._buffer_size)
        self._buffer_size += value.numel() * value.element_size()
        return meta

    def _finish_at_exit(self):
        try:
            self.wait_pending(timeout=120)
        except BaseException:
            pass
        try:
            # a background registration must not race the CUDA runtime's teardown
            if self._stager is not None:
                self._stager.detach()
        except BaseException:
            pass

    def wait_segment_pinned(self, timeout: float = 120.0) -> bool:
        """True once this process's window of the segment is page-locked (transfers are
        plain DMA from then on).  Large windows are pinned by a library thread after the
        first save / restore; nothing has to wait for it — benchmarks do, to time the
        steady state."""
        self.wait_pending()
        return self._stager is not None and self._stager.wait_pinned(timeout)

    # -- pending drain ----------------------------------------------------------------
    def pending_save(self) -> Optional[PendingSave]:
        p = self._pending
        return p if p is not None and not p.done() else None

    def wait_pending(self, timeout: Optional[float] = None) -> bool:
        p = self._pending
        if p is None:
            return True
        try:
            ok = p.wait(timeout)
        except BaseException:
            self._pending = None  # a failed drain is reported once
            raise
        if ok:
            self._pending = None
        return ok

    # -- save ---------------------------------------------------------------------------
    def _stager_for(self, tensors) -> _DeviceStager:
        dev = tensors[0].device
        index = dev.index if dev.index is not None else torch.cuda.current_device()
        for t in tensors:
            if t.device != dev:
                raise ValueError(
                    "all CUDA tensors of one checkpoint shard must live on one device; "
                    f"got {dev} and {t.device}")
        if self._stager is None or self._stager.device_index != index:
            if self._stager is not None:
                self._stager.close()
            self._stager = _DeviceStager(index)
        return self._stager

    def ensure_segment(self, total: int):
        """Map a segment of exactly `total` bytes (re-creating it on a size
        change)."""
        if self.shared_memory is not None and self.shared_memory.size == total \
                and not self._need_creation:
            return
        if self._stager is not None:
            self._stager.detach()
        if self.shared_memory is not None:
            self.shared_memory.close()
            self.shared_memory = None
        self._delta_invalidate()
        self.init_shared_memory(create=True, size=total)
        self._buffer_size = total

    def write_ranges(self, device_ranges, host_ranges, raw_chunks=(), *, blocking=True,
                     stream=None, finish: Optional[Callable[[], None]] = None,
                     keepalive: Optional[list] = None,
                     announce: Optional[Callable[[], None]] = None,
                     on_error: Optional[Callable[[], None]] = None,
                     in_place: Optional[bool] = None,
                     window: Optional[Tuple[int, int]] = None, compact: bool = False):
        """Move bytes into the (already sized) segment.

        device_ranges / host_ranges: (tensor, segment offset, nbytes) for CUDA /
        CPU tensors; raw_chunks: (bytes-like, offset).  CUDA ranges go through
        one gather kernel + DMA drain, the rest is written by the host right
        away.  `finish` runs once everything has landed — inline when blocking,
        else on the completion thread of the returned PendingSave.
        announce: publishes writing_shm=True; it runs before the first byte of the
        segment changes, inline or, with the drain held, on the completion thread.
        in_place (default: self.in_place): no snapshot — the drain reads the CUDA
        tensors themselves, so they must not be written until the save is done
        (wait_pending / PendingSave.wait).  Also chosen, together with blocking,
        when HBM has no room for the snapshot arena.
        window=(lo, hi): this process is responsible for the segment bytes [lo, hi)
        only (cooperative save of a replicated state: every local rank drains its own
        slice of the same image over its own PCIe link): CUDA ranges are clipped to
        the window, the arena holds hi-lo bytes, only that part of the segment is
        pinned.  Host ranges are clipped the same way (parallel memcpy across the
        ranks); raw chunks are written as given (hand them to one rank only).
        """
        keepalive = keepalive if keepalive is not None else []

        def announce_then_raw():
            if announce is not None:
                announce()
            for chunk, off in raw_chunks:
                view = memoryview(chunk).cast("B")
                self.shared_memory.buf[off:off + view.nbytes] = view

        # The announcement (a pickle, and two socket round trips without a control
        # segment) may wait for the completion thread only when nothing touches the
        # segment before the drain: no host tensors (they are copied now, as the training
        # thread may change them once this call returns), and the immutable byte chunks
        # are written right after it.  The first announcement of a handler goes out
        # inline: until it is out the agent's dict holds no step at all, and a SAVE event
        # that overtakes it would find "no shard has a step"
        # (ckpt_saver._check_shard_step_consistence).
        may_hold = (announce is not None and not blocking and bool(device_ranges)
                    and not host_ranges and self._announced_once)
        held = announce_then_raw if may_hold else None
        if held is None:
            announce_then_raw()
        if announce is not None:
            self._announced_once = True
        if host_ranges:
            keep, ptrs, offs, lens = [], [], [], []
            for t, off, nbytes in host_ranges:
                c = t.detach()
                if not c.is_contiguous():
                    c = c.contiguous()
                keep.append(c)
                ptrs.append(c.data_ptr())
                offs.append(off)
                lens.append(nbytes)
            if window is not None:
                ptrs, offs, lens = _clip_ranges((ptrs, offs, lens), window[0], window[1])
            if ptrs:
                native.host_pack(self.shared_memory.address, ptrs, offs, lens, _host_threads())
            del keep
        ctx, ticket = None, 0
        delta = False
        got = self._save_plan(device_ranges, keepalive, stream, window, compact)
        if got is not None:
            stager, prepared, plan, stream = got
            lo, hi = window if window is not None else (0, self.shared_memory.size)
            stager.attach(self.shared_memory, lo, hi)
            host_addr = self.shared_memory.dma_address + lo
            in_place = (self.in_place if in_place is None else in_place) and not compact
            cut = None  # hybrid: window offset from which the tensors are snapshotted
            if in_place:
                arena = stager.ARENA_NONE
                cut = self._hybrid_cut(stager, plan, prepared[1], lo)
                if cut is not None and cut <= min(prepared[1]) - lo \
                        and stager.ensure_arena(plan) == stager.ARENA_FULL:
                    in_place, cut, arena = False, None, stager.ARENA_FULL  # everything fits
            else:
                arena = stager.ensure_arena(plan)
            if arena == stager.ARENA_NONE and not in_place:
                # nobody promised to keep the tensors unchanged: drain before returning
                in_place = blocking = True
            # bounded-arena saves drain inside save_async: announce first, inline
            windowed = arena == stager.ARENA_WINDOWED
            if windowed and not stager.pinned():
                stager.ctx.host_register(*stager._attached, prefault_threads=_host_threads())
                stager._pin_started = True
            if held is not None and (blocking or windowed):
                held()
                held = None
            hold = held is not None
            # incremental saves need an arena image of the whole plan to compare with:
            # full-snapshot saves only (not in place, not hybrid, not windowed)
            delta = self.incremental and not in_place and arena == stager.ARENA_FULL
            if delta and (self._delta_segment is not self.shared_memory
                          or self.shared_memory.stale()):
                # another mapping than the one the baseline was drained to
                stager.ctx.delta_invalidate()
            if in_place and cut is not None:
                ticket = plan.save_hybrid_async(host_addr, cut, stream, hold=hold)
            elif in_place:
                ticket = plan.save_direct_async(host_addr, stream, hold=hold)
            elif delta:
                ticket = plan.save_delta_async(host_addr, stream, hold=hold)
                self._delta_segment = self.shared_memory
            else:
                ticket = plan.save_async(host_addr, stream, hold=hold)
            self._last_ticket = (stager.ctx, ticket)
            self.last_hybrid_cut = None if cut is None else cut + lo
            self.last_save_in_place = in_place
            if in_place:
                self.last_pack_event = None  # there is no snapshot to wait for, only the drain
            else:
                ev = torch.cuda.Event()
                ev.record(stream)
                self.last_pack_event = ev
            ctx = stager.ctx
        if ctx is None and held is not None:  # the window held no device bytes
            held()
            held = None
        user_finish = finish or (lambda: None)
        if ctx is not None:
            def finish_and_pin():
                user_finish()
                # the first transfer of a large window went through bounce slots; pin the
                # window now, off every critical path, so the next ones are plain DMA
                stager.pin_in_background()
        else:
            finish_and_pin = user_finish
        if delta and ctx is not None:
            pin_after = finish_and_pin

            def finish_and_pin():
                # visible before the caller's completion callback and before wait() returns
                self.last_save_stats = pending.stats
                pin_after()
        pending = PendingSave(ctx, ticket, finish_and_pin, keepalive, announce=held,
                              on_error=on_error, delta=ctx is not None and delta)
        self._pending = pending
        if blocking or ctx is None:
            pending._complete()
            self.last_timings = pending.timings
            self.last_save_stats = pending.stats
            self._pending = None
            pending.wait()  # re-raise a drain error
            return None
        self._completion_worker().put(pending)
        return pending

    def _save_plan(self, device_ranges, keepalive: list, stream, window, compact: bool):
        """(stager, prepared ranges, plan, stream) a save of these CUDA (tensor, segment
        offset, nbytes) ranges runs with (the save's and the non-finite scan's one plan),
        or None when there are no device bytes (in the window).  `stream` (default: the
        current one) is made to wait for the current stream."""
        if not device_ranges:
            return None
        stager = self._stager_for([r[0] for r in device_ranges])
        # a dense repack of an oddly strided leaf runs on the CURRENT stream: do it
        # before a side stream is made to wait for that stream
        prepared = stager.prepare_ranges(device_ranges, keepalive)
        if window is not None:
            prepared = _clip_ranges(prepared, window[0], window[1])
            if not prepared[0]:
                return None
        current = torch.cuda.current_stream(stager.device_index)
        if stream is None:
            stream = current
        elif stream != current:
            # snapshot on a side stream: it must see everything the training
            # stream has enqueued so far, and the caller must make the training
            # stream wait for `last_pack_event` before it MUTATES the tensors
            stream.wait_stream(current)
        lo = window[0] if window is not None else 0
        plan = stager.plan_for(prepared, role="save", stream=stream, base=lo, compact=compact)
        return stager, prepared, plan, stream

    def scan_nonfinite(self, state_dict, stream=None, coop: Optional[CoopContext] = None,
                       shards: bool = False, reuse_for=None) -> Dict[str, int]:
        """{leaf path: NaN/Inf count} of the part of `state_dict` that a save through this
        handler would write from this process ({} when it is finite).  CUDA leaves: the
        plan the save will use (built or reused here) is scanned on `stream` after it
        waited for the current stream; CPU leaves are checked on the host.  coop / shards:
        as save_state_dict(coop=...) / save_shards_as_full.  Touches neither the segment,
        the meta nor the arena.  reuse_for: the state dict whose save follows right away
        takes this walk's layout instead of walking again."""
        mine = None
        if shards:
            lay, mine = plan_layout_full_from_shards(state_dict)
        else:
            lay = plan_layout(state_dict, self._layout)
        self._scanned = (reuse_for, lay, mine)
        metas = [m for m in lay.leaf_metas if m.numel]
        starts = [m.offset for m in metas]
        counts: Dict[int, int] = {}  # index into metas -> count

        def owner(off: int) -> int:
            return bisect.bisect_right(starts, off) - 1

        host = _triples(lay.host_leaves) + [r for r in (mine or ()) if not r[0].is_cuda]
        for t, off, _ in host:
            m = metas[owner(off)]
            if _SCAN_KINDS.get(m.dtype, native.KIND_NONE) == native.KIND_NONE:
                continue
            v = t.detach()
            if v.dtype != m.dtype:  # a byte view of a clipped leaf
                v = v.view(m.dtype)
            bad = int((~torch.isfinite(v.float() if v.element_size() == 1 else v)).sum())
            if bad:
                counts[owner(off)] = counts.get(owner(off), 0) + bad
        dev = _triples(lay.device_leaves)
        window = coop.window(lay.total) if coop is not None else None
        if mine is not None:
            dev = _clip_triples(dev, *window) + [r for r in mine if r[0].is_cuda]
            window = None
        got = self._save_plan(dev, [], stream, window, compact=mine is not None)
        if got is not None:
            _, (_, offs, _), plan, stream = got
            owners = [owner(o) for o in offs]
            plan.set_kinds([_SCAN_KINDS.get(metas[i].dtype, native.KIND_NONE) for i in owners])
            plan.scan_nonfinite_async(stream)
            total, per_range = plan.scan_wait(len(owners))
            if total:
                for i, c in zip(owners, per_range):
                    if c:
                        counts[i] = counts.get(i, 0) + c
        if not counts:
            return {}
        paths = {id(m): p for m, p in zip(lay.leaf_metas, _leaf_paths(state_dict))}
        return {paths.get(id(metas[i]), f"offset {metas[i].offset}"): c
                for i, c in sorted(counts.items())}

    def take_scanned(self, state_dict):
        """(layout, mine) of the scan_nonfinite that ran for `state_dict`, or None; the
        scan's layout is forgotten either way (take_scanned(None) after a skipped save)."""
        scanned, self._scanned = self._scanned, None
        if scanned is not None and scanned[0] is not None and scanned[0] is state_dict:
            return scanned[1], scanned[2]
        return None

    def _completion_worker(self):
        """One long-lived thread per handler finishes the non-blocking saves in order
        (starting a thread per save costs the training thread ~0.1 ms)."""
        q = self._completion_queue
        if q is None:
            import queue

            q = self._completion_queue = queue.SimpleQueue()
            ref = weakref.ref(self)

            def loop():
                while True:
                    pending = q.get()
                    if pending is None:
                        return
                    handler = ref()
                    pending._complete()
                    if handler is not None:
                        handler.last_timings = pending.timings
                        handler.last_save_stats = pending.stats
                    del handler

            threading.Thread(target=loop, name="fc-drain", daemon=True).start()
        return q

    MIN_SNAPSHOT_BYTES = 64 << 20  # below this a snapshot part is not worth a kernel

    def _hybrid_cut(self, stager: _DeviceStager, plan, offsets, base: int = 0) -> Optional[int]:
        """In-place save with a snapshot budget: the (window-relative) offset from which
        the tensors fit into the arena (None: no budget / no arena -> pure in-place)."""
        budget = self.in_place_snapshot_bytes
        if budget <= 0:
            return None
        want = min(budget, plan.arena_end)
        if self._snapshot_ceiling:
            want = min(want, self._snapshot_ceiling)
        while stager.ctx.arena_info()[1] < want:
            try:
                stager.ctx.arena_reserve(want)
            except native.NativeError as e:
                if e.code != native.FC_ENOMEM:
                    raise
                # no room for that much: remember it, try half (a failed grow has
                # released the previous arena to make room)
                self._snapshot_ceiling = want = want // 2
                if want < self.MIN_SNAPSHOT_BYTES:
                    break
        cap = min(stager.ctx.arena_info()[1], budget)
        end, cut = plan.arena_end, None
        for off in sorted((o - base for o in offsets), reverse=True):
            # the arena's byte 0 stands for the cut rounded down to 128 B
            if end - (off & ~127) > cap:
                break
            cut = off
        return cut

    def wait_snapshot(self, stream=None):
        """Order the caller's next WRITE to the saved tensors after the last save
        has read them: with a snapshot (default) `stream` (default: current) waits on
        the GPU for the gather kernel; after an in-place save the host waits for the
        drain.  Cheap no-op when nothing is pending."""
        if self.last_save_in_place:
            if self._last_ticket is not None and self.pending_save() is not None:
                ctx, ticket = self._last_ticket
                try:
                    ctx.save_sources_wait(ticket)  # in-place part drained (+ gather done)
                    return
                except native.NativeError:
                    pass  # a later ticket took over / drain error: fall through
            self.wait_pending()
            return
        ev = self.last_pack_event
        if ev is not None:
            (stream or torch.cuda.current_stream()).wait_event(ev)

    def attach_existing(self, total: int):
        """Map the segment another local process created (cooperative saves); it must
        already have `total` bytes."""
        shm = self.shared_memory
        if shm is None or self._need_creation or shm.stale() or shm.size != total:
            if self._stager is not None:
                self._stager.detach()
            if shm is not None:
                shm.close()
                self.shared_memory = None
            self._delta_invalidate()
            self.init_shared_memory(create=False)
        if self.shared_memory is None or self.shared_memory.size != total:
            have = None if self.shared_memory is None else self.shared_memory.size
            raise RuntimeError(f"cooperative save: the segment has {have} bytes, this rank's "
                               f"state dict needs {total} (replicas differ?)")
        self._buffer_size = total

    def save_state_dict(self, state_dict, blocking: bool = True, stream=None,
                        on_complete: Optional[Callable[[], None]] = None,
                        on_error: Optional[Callable[[], None]] = None,
                        coop: Optional[CoopContext] = None):
        """Serialise `state_dict` into the segment.

        blocking=True (the reference's semantics): returns None after every
        byte is in shared memory and the meta says writing_shm=False.
        blocking=False: returns a PendingSave right after the gather kernel is
        enqueued on `stream` (default: the current stream); a completion thread
        finishes the protocol and then calls `on_complete`.
        coop: this process writes only its slice of the image (see CoopContext); the
        leader runs the meta protocol, the others report through the control segment.
        """
        self.wait_pending()
        scanned = self.take_scanned(state_dict)
        lay = self._layout = scanned[0] if scanned else plan_layout(state_dict, self._layout)
        if coop is not None:
            return self._save_cooperative(state_dict, lay, coop, blocking, stream, on_complete,
                                          on_error)
        if lay.total > 0:
            self.ensure_segment(lay.total)
        meta_dict = lay.meta
        conf: CheckpointConfig = meta_dict[DLROVER_CKPT_CONFIG_KEY]
        unchanged = lay.unchanged and self._meta_published
        self._meta_published = False

        def announce():
            report_local_event(EventReportConstants.TYPE_INFO, str(conf.rank),
                               EventReportConstants.ACTION_MEM_CKPT_START, f"step={conf.step}")
            self._set_meta(meta_dict, True, unchanged, lay.total)

        def finish():
            # the tree went out with the announcement
            self._set_meta(meta_dict, False, True, lay.total)
            report_local_event(EventReportConstants.TYPE_INFO, str(conf.rank),
                               EventReportConstants.ACTION_MEM_CKPT_COMPLETE,
                               f"step={conf.step}")
            if on_complete is not None:
                on_complete()

        # the tensors must outlive the gather kernel
        keepalive = [state_dict] if lay.device_leaves else []
        return self.write_ranges(_triples(lay.device_leaves), _triples(lay.host_leaves),
                                 blocking=blocking, stream=stream, finish=finish,
                                 keepalive=keepalive, announce=announce, on_error=on_error)

    def _set_meta(self, meta_dict, writing: bool, unchanged: bool, payload_bytes: int):
        """Publish the meta tree of the save in progress with writing_shm=`writing`:
        True before the first byte of the segment changes, False once every byte has
        landed.  unchanged: the meta plane already holds this tree (everything but the
        CheckpointConfig), so only the header is rewritten."""
        meta_dict[DLROVER_CKPT_CONFIG_KEY].writing_shm = writing
        self.metadata.payload_bytes = payload_bytes
        self.metadata.next_unchanged = unchanged
        self._meta_published = False
        self.metadata.set(meta_dict)
        self._meta_published = not writing

    def save_shards_as_full(self, state_dict, coop: CoopContext, blocking: bool = True,
                            stream=None, on_complete=None, on_error=None):
        """Cooperative save of the FULL state from a state dict of SHARDS (DTensor /
        ShardedTensor leaves, e.g. FSDP's sharded state dict): the segment gets the image the
        gathered state dict would have produced, but nobody gathers anything — every rank
        drains its own shards to where they belong in the full tensors (plus its slice of
        the replicated leaves).  All ranks that hold shards must be local to this node."""
        self.wait_pending()
        lay, mine = self.take_scanned(state_dict) or plan_layout_full_from_shards(state_dict)
        self._layout = None  # not comparable with a plain layout
        return self._save_cooperative(state_dict, lay, coop, blocking, stream, on_complete,
                                      on_error, mine=mine)

    def _save_cooperative(self, state_dict, lay: _Layout, coop: CoopContext, blocking, stream,
                          on_complete, on_error, mine=None):
        meta_dict = lay.meta
        conf: CheckpointConfig = meta_dict[DLROVER_CKPT_CONFIG_KEY]
        total = lay.total
        if coop.leader:
            try:
                if total > 0:
                    self.ensure_segment(total)
                report_local_event(EventReportConstants.TYPE_INFO, str(conf.rank),
                                   EventReportConstants.ACTION_MEM_CKPT_START,
                                   f"step={conf.step}")
                # before any rank touches the segment
                self._set_meta(meta_dict, True, lay.unchanged and self._meta_published, total)
                self._announced_once = True
            except BaseException:
                coop.ctl.next_coop_seq(aborted=True)  # do not leave the others waiting
                raise
            coop.ctl.next_coop_seq()
        else:
            if not coop.opened and not coop.ctl.wait_coop_open(coop.seq, coop.timeout):
                raise RuntimeError("cooperative save: the leader aborted")
            if total > 0:
                self.attach_existing(total)
        window = coop.window(total)

        def finish():
            coop.ctl.slot_set(coop.index, coop.seq, ok=True)
            if coop.leader:
                if not coop.ctl.wait_slots(coop.n, coop.seq, coop.timeout):
                    raise RuntimeError("cooperative save: a local rank failed or did not "
                                       f"report its slice within {coop.timeout:.0f}s")
                self._set_meta(meta_dict, False, True, total)
                report_local_event(EventReportConstants.TYPE_INFO, str(conf.rank),
                                   EventReportConstants.ACTION_MEM_CKPT_COMPLETE,
                                   f"step={conf.step}")
            if on_complete is not None:
                on_complete()

        def failed():
            try:
                coop.ctl.slot_set(coop.index, coop.seq, ok=False)
            finally:
                if on_error is not None:
                    on_error()

        keepalive = [state_dict] if (lay.device_leaves or mine) else []
        if total == 0:
            finish()
            return None
        try:
            if mine is not None:
                # replicated leaves: my slice of each; sharded leaves: what only I hold
                dev = _clip_triples(_triples(lay.device_leaves), *window) + \
                    [r for r in mine if r[0].is_cuda]
                host = _clip_triples(_triples(lay.host_leaves), *window) + \
                    [r for r in mine if not r[0].is_cuda]
                return self.write_ranges(dev, host, blocking=blocking, stream=stream,
                                         finish=finish, keepalive=keepalive + [dev, host],
                                         on_error=failed, compact=True)
            return self.write_ranges(_triples(lay.device_leaves), _triples(lay.host_leaves),
                                     blocking=blocking, stream=stream, finish=finish,
                                     keepalive=keepalive, on_error=failed, window=window)
        except BaseException:
            if self._pending is None:  # raised before a completion thread took over
                coop.ctl.slot_set(coop.index, coop.seq, ok=False)
            raise

    # -- load ---------------------------------------------------------------------------
    def _consistent_meta(self):
        """The check every read of the in-memory checkpoint starts with: wait for this
        handler's own drain, refuse a checkpoint that is being written, map the segment.
        Returns (meta dict, None), or (None, why there is nothing to read)."""
        self.wait_pending()
        meta_dict = self.metadata.get()
        if not meta_dict or meta_dict.get(DLROVER_CKPT_CONFIG_KEY, CheckpointConfig()).writing_shm:
            return None, "no consistent in-memory checkpoint to restore from"
        self.refresh_mapping()
        if not self.shared_memory:
            return None, "the checkpoint segment does not exist"
        return meta_dict, None

    def load_state_dict(self):
        """Returns the state dict (CPU tensors aliasing the segment), or {} when
        there is no usable in-memory checkpoint."""
        meta_dict, why = self._consistent_meta()
        if why:
            return {}
        config = meta_dict.get(DLROVER_CKPT_CONFIG_KEY, CheckpointConfig())
        report_local_event(EventReportConstants.TYPE_INFO, str(config.rank),
                           EventReportConstants.ACTION_RESUME_MEM_CKPT_START,
                           f"step={config.step}")
        state_dict = _read_state_dict_from_shm(meta_dict, self.shared_memory)
        report_local_event(EventReportConstants.TYPE_INFO, str(config.rank),
                           EventReportConstants.ACTION_RESUME_MEM_CKPT_COMPLETE,
                           f"step={config.step}")
        return state_dict

    def restore_into(self, target, stream=None, strict: bool = True,
                     pin_after: bool = True, coop=None, *,
                     image_first: bool = False) -> Dict[str, float]:
        """Scatter the in-memory checkpoint straight into the live tensors of
        `target` (same tree structure as what was saved; extra keys on either
        side raise when strict).  CUDA leaves: one DMA fill of the arena + one
        scatter kernel; CPU leaves: copied from the segment.  Non-tensor leaves
        of the checkpoint are returned under "extras" untouched.

        Replaces `sd = load_state_dict(); model.load_state_dict(sd)` (per
        parameter H2D copies from pageable memory, reference ckpt_saver.py:
        144-161 + user code).

        coop=(index, n, process_group): a REPLICATED state that all n local ranks
        restore at the same time — each rank reads only 1/n of the image from host
        memory into its arena and the slices are exchanged over NVLink (NCCL
        all-gather, in place) before the scatter kernel; every rank must call.

        image_first: scatter the CUDA leaves from the arena image when it covers them
        (see rollback_into); stats then carry "from_image" (1.0 / 0.0)."""
        device_ranges, host_pairs = self._restore_targets(target, strict)
        with torch.no_grad():
            stats = {"host_bytes": self._restore_host_leaves(host_pairs)}
            stats.update(self.read_ranges(device_ranges, stream, image_first=image_first,
                                          coop=coop, pin_after=pin_after))
        return stats

    def rollback_into(self, target, stream=None, strict: bool = True) -> Dict[str, float]:
        """restore_into for a process that saved the checkpoint itself: after a
        full-snapshot save has drained, the HBM arena still holds the image of what it
        wrote, and the CUDA leaves are scattered from there (one scatter kernel, nothing
        crosses PCIe).  The incremental baseline survives, so the next incremental save
        drains only what changed after the rollback.  Without such an image (in-place,
        hybrid, bounded-arena or cooperative saves, a restore or anything else that
        rewrote the arena since) this is restore_into.  CPU leaves come from the segment
        either way.  stats: those of restore_into plus "from_image" (1.0 / 0.0)."""
        return self.restore_into(target, stream, strict, image_first=True)

    def can_rollback(self, target, strict: bool = True) -> bool:
        """Whether rollback_into(target) would scatter every CUDA leaf from the arena
        image; restores nothing.  False when the tree has no CUDA leaf."""
        device_ranges, _ = self._restore_targets(target, strict)
        return bool(device_ranges) and self.image_covers_ranges(device_ranges)

    def _restore_targets(self, target, strict: bool):
        """The part every restore of the in-memory checkpoint into live tensors shares:
        _consistent_meta (raising when there is nothing to read), then each tensor leaf of
        `target` paired with its meta (_match_tree).  Returns (CUDA (tensor, segment
        offset, nbytes) ranges, CPU (tensor, meta) pairs)."""
        meta_dict, why = self._consistent_meta()
        if why:
            raise RuntimeError(why)
        # tuples are leaves of the memory checkpoint (plan_layout does not descend into them)
        pairs = _match_tree(target, meta_dict, TensorMeta, (list,), strict)
        device_ranges = [(t, m.offset, m.numel * m.element_size) for _, t, m in pairs if t.is_cuda]
        host_pairs = [(t, m) for _, t, m in pairs if not t.is_cuda]
        return device_ranges, host_pairs

    def _restore_host_leaves(self, host_pairs) -> float:
        """CPU leaves straight from the segment; returns their bytes."""
        strided = [(t, m) for t, m in host_pairs if not t.is_contiguous()]
        dense = [(t, m) for t, m in host_pairs if t.is_contiguous()]
        for t, m in strided:  # rare: let torch handle the strides
            t.copy_(_read_tensor_from_buf(m, self.shared_memory))
        if dense:
            native.host_unpack(self.shared_memory.address, [t.data_ptr() for t, _ in dense],
                               [m.offset for _, m in dense],
                               [m.numel * m.element_size for _, m in dense], _host_threads())
        return float(sum(m.numel * m.element_size for _, m in host_pairs))

    def _restore_plan(self, device_ranges, stream):
        """(stager, restore plan, stream) for non-empty (CUDA tensor, segment offset,
        nbytes) ranges, checked against the mapped segment: arena offset = segment offset,
        so the plan lines up with the saves' arena image."""
        self.refresh_mapping()
        if not self.shared_memory:
            raise RuntimeError("the checkpoint segment does not exist")
        size = self.shared_memory.size
        for t, off, nbytes in device_ranges:
            if not t.is_cuda:
                raise ValueError("read_ranges needs CUDA targets")
            if off + nbytes > size or t.nbytes != nbytes:
                raise ValueError("read_ranges: range does not fit the segment / the tensor")
        stager = self._stager_for([t for t, _, _ in device_ranges])
        prepared = stager.prepare_ranges(device_ranges, [], for_write=True)
        if stager._attached is None:
            stager.attach(self.shared_memory)
        if stream is None:
            stream = torch.cuda.current_stream(stager.device_index)
        plan = stager.plan_for(prepared, role="restore", stream=stream)
        return stager, plan, stream

    def _run_rollback(self, stager: _DeviceStager, plan, stream) -> Optional[Dict[str, float]]:
        """One scatter kernel from the arena image; None (nothing done) without one."""
        stats = _timed_restore(stager.ctx, plan, lambda: plan.restore_from_image_async(
            self.shared_memory.dma_address, stream))
        if stats is None:
            return None
        stats.update(fill_ms=0.0, direct=0.0, staged=0.0, from_image=1.0)
        self.last_restore_stats = stats
        return dict(stats)

    def _run_restore_cooperative(self, stager: _DeviceStager, plan, stream, coop):
        """Each of the n local ranks fills 1/n of its arena from the segment (its own PCIe
        link), NCCL all-gathers the slices in place over NVLink, one scatter kernel."""
        import torch.distributed as dist

        index, n, group = coop
        total = self.shared_memory.size
        w = CoopContext.slice_bytes(total, n)   # == the save windows
        stager.ctx.arena_reserve(n * w)
        lo, hi = min(total, index * w), min(total, (index + 1) * w)
        t0 = time.perf_counter()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        with torch.cuda.stream(stream):
            ev[0].record(stream)
            stager.ctx.arena_fill(self.shared_memory.dma_address, lo, hi, stream)
            ev[1].record(stream)
            arena = stager.ctx.arena_tensor(n * w)
            dist.all_gather_into_tensor(arena, arena[index * w:(index + 1) * w], group=group)
            ev[2].record(stream)
            plan.unpack(stream)
            ev[3].record(stream)
        ev[3].synchronize()
        self.last_restore_stats = {
            "device_bytes": float(plan.payload_bytes), "fill_ms": ev[0].elapsed_time(ev[1]),
            "allgather_ms": ev[1].elapsed_time(ev[2]), "scatter_ms": ev[2].elapsed_time(ev[3]),
            "cooperative": float(n), "slice_bytes": float(hi - lo),
            "wall_ms": (time.perf_counter() - t0) * 1e3, "staged": float(not stager.pinned())}
        return dict(self.last_restore_stats)

    DIRECT_RESTORE_MIN_SPAN = 1 << 20  # average span size from which in-place restore wins

    def _run_restore(self, stager: _DeviceStager, plan, stream,
                     pin_after: bool = True) -> Dict[str, float]:
        """Few large spans: H2D DMA straight into the targets.  Many small ones: one
        DMA per merged segment run into the arena + one scatter kernel.
        DLROVER_B200_RESTORE=direct|arena overrides the choice."""
        direct = plan.payload_bytes >= plan.n_spans * self.DIRECT_RESTORE_MIN_SPAN
        forced = os.getenv("DLROVER_B200_RESTORE", "")
        if forced in ("direct", "arena"):
            direct = forced == "direct"
        if not direct and stager.ensure_arena(plan) == stager.ARENA_NONE:
            direct = True
        staged = not stager.pinned()  # e.g. a restarted trainer: bounce slots, no 16 GB pin
        stats = _timed_restore(stager.ctx, plan, lambda: plan.restore_async(
            self.shared_memory.dma_address, stream, direct=direct))
        stats.update(direct=float(direct), staged=float(staged))
        self.last_restore_stats = stats
        if pin_after:
            stager.pin_in_background()  # the next save wants plain DMA
        return dict(stats)

    def read_ranges(self, device_ranges, stream=None, *, image_first: bool = False,
                    coop=None, pin_after: bool = True) -> Dict[str, float]:
        """Inverse of write_ranges for CUDA targets: (tensor, segment offset,
        nbytes) triples are filled by one DMA of the covered segment runs into
        the arena + one scatter kernel into the (contiguous) tensors.  Every restore
        of CUDA tensors from the in-memory checkpoint ends here.

        image_first: scatter from the arena image of this process's last full-snapshot
        save when it covers the ranges (one kernel, nothing crosses PCIe; see
        rollback_into), else as above; the stats then carry "from_image" (1.0 / 0.0).
        coop, pin_after: see restore_into."""
        self.wait_pending()
        if not device_ranges:
            stats = {"device_bytes": 0.0, "fill_ms": 0.0, "scatter_ms": 0.0}
            if image_first:
                stats["from_image"] = 0.0
            return stats
        stager, plan, stream = self._restore_plan(device_ranges, stream)
        got = self._run_rollback(stager, plan, stream) if image_first else None
        if got is None and coop is not None:
            got = self._run_restore_cooperative(stager, plan, stream, coop)
        elif got is None:
            got = self._run_restore(stager, plan, stream, pin_after=pin_after)
            if image_first:
                got["from_image"] = self.last_restore_stats["from_image"] = 0.0
        return got

    def image_covers_ranges(self, device_ranges) -> bool:
        """Whether read_ranges(device_ranges, image_first=True) would scatter every range
        from the arena image; moves nothing.  Raises what read_ranges raises for the same
        ranges.  True when there are no ranges: there is nothing to move."""
        self.wait_pending()
        if not device_ranges:
            return True
        _, plan, _ = self._restore_plan(device_ranges, None)
        return plan.image_covers(self.shared_memory.dma_address)

    # -- queries ------------------------------------------------------------------------
    def no_checkpoint_state(self):
        """True when the meta dict holds no config or step 0.  (The agent-side
        handler maps the segment lazily, so the mapping itself says nothing.)"""
        config = self.metadata.get().get(DLROVER_CKPT_CONFIG_KEY, None)
        return config is None or config.step == 0

    def get_checkpoint_config(self, default_config):
        return self.metadata.get().get(DLROVER_CKPT_CONFIG_KEY, default_config)

    def get_master_client(self):
        return self._master_client

    def set_master_client(self, client):
        self._master_client = client


# -- restore from a torch.save file ----------------------------------------------------
# Both storage readers (restore_file_into here, FileDmaReader for DCP shard files) turn
# their leaves into (target address, file, file offset, n) pieces and share the rest:
# _open_files checks every file's length before a byte moves, _read_pieces reads.


class ShortFileError(OSError, ValueError):
    """A file ends before the last byte a restore reads from it; raised before any target
    changes.  An OSError for restore_file_into, a ValueError for a DCP StorageReader."""


def _pair_rows(src, dst):
    """Zip the source rows (file offset, n) with the target rows (address, n), both in
    logical order and of the same total: (address, file offset, n) pieces."""
    out, i, j, si, dj = [], 0, 0, 0, 0
    while i < len(src) and j < len(dst):
        (f, fn), (p, pn) = src[i], dst[j]
        n = min(fn - si, pn - dj)
        out.append((p + dj, f + si, n))
        si, dj = si + n, dj + n
        if si == fn:
            i, si = i + 1, 0
        if dj == pn:
            j, dj = j + 1, 0
    return out


def _unique_pieces(pieces):
    """(address, file, file offset, n) pieces sorted by file and offset, without those that
    repeat bytes of another piece into the same place (tied weights: two leaves, one
    storage in the file and one in the model)."""
    out, live = [], []  # live: kept pieces of the same file that reach past the offset
    for r in sorted(pieces, key=lambda r: (r[1], r[2], -r[3])):
        a, f, o, n = r
        live = [k for k in live if k[1] == f and k[2] + k[3] > o]
        if any(o + n <= ko + kn and a - ka == o - ko for ka, _, ko, kn in live):
            continue
        out.append(r)
        live.append(r)
    return out


def _disjoint_groups(ranges):
    """Split ranges sorted by file offset into groups without overlapping file bytes (a
    mapped plan reads every file byte once): one group, unless two different tensors are
    restored from the same bytes (overlapping views of one storage, untied targets)."""
    groups = []
    for r in ranges:
        for g in groups:
            if g[-1][1] + g[-1][2] <= r[1]:
                g.append(r)
                break
        else:
            groups.append([r])
    return groups


def _restore_file_groups(ranges, device_index: int, stream, enqueue, stats) -> int:
    """Restore CUDA (address, file offset, nbytes) ranges, sorted by file offset, through
    the arena of `device_index`: one mapped plan per _disjoint_groups group, whose file
    fill enqueue(plan, stream) starts.  Adds device_bytes, read_ms and scatter_ms to
    `stats`; returns the number of plans."""
    ctx = native.get_context(device_index)
    if stream is None:
        stream = torch.cuda.current_stream(device_index)
    groups = _disjoint_groups(ranges)
    for group in groups:
        ptrs, arena, foffs, lens, a = [], [], [], [], 0
        for p, f, n in group:
            a += (p - a) % 16  # congruent to the target mod 16: the bulk kernel
            ptrs.append(p)
            arena.append(a)
            foffs.append(f)
            lens.append(n)
            a += n
        plan = ctx.plan(ptrs, arena, lens, host_offsets=foffs)
        try:
            if _DeviceStager.reserve_arena(ctx, plan.arena_end) == _DeviceStager.ARENA_NONE:
                logger.warning(f"No room for a {plan.arena_end / 2**30:.1f} GiB restore arena "
                               "in HBM: the file is restored window by window.")
                ctx.arena_reserve(64 << 20)
            got = _timed_restore(ctx, plan, lambda: enqueue(plan, stream))
        finally:
            plan.destroy()
        stats["device_bytes"] += got["device_bytes"]
        stats["read_ms"] += got["fill_ms"]
        stats["scatter_ms"] += got["scatter_ms"]
    return len(groups)


def _pread_into(fd: int, buf, offset: int):
    """Fill the writable buffer `buf` from `fd` at `offset`."""
    view = memoryview(buf).cast("B")
    got = 0
    while got < len(view):
        n = os.preadv(fd, [view[got:]], offset + got)
        if n <= 0:
            raise OSError(f"short read at file offset {offset + got}")
        got += n


@contextlib.contextmanager
def _open_files(root, pieces, more=()):
    """Open every file that (address, file, file offset, n) `pieces` and the (file, end)
    pairs of `more` name, relative to `root`, and check each with fstat against the
    highest byte they read from it before any byte moves (ShortFileError).  Yields
    {file: fd}; every fd is closed on the way out."""
    need: Dict[Any, int] = {}
    for f, end in [(f, o + n) for _, f, o, n in pieces] + list(more):
        need[f] = max(need.get(f, 0), end)
    fds: Dict[Any, int] = {}
    try:
        for f in sorted(need):
            path = os.path.join(root, f)
            fds[f] = os.open(path, os.O_RDONLY)
            size = os.fstat(fds[f]).st_size
            if size < need[f]:
                raise ShortFileError(f"{path}: the restore reads bytes up to file offset "
                                     f"{need[f]}, the file ends at {size}")
        yield fds
    finally:
        for fd in fds.values():
            os.close(fd)


def _read_pieces(fds, cuda, host, devices, stream=None) -> Dict[str, float]:
    """Read (address, file, file offset, n) pieces from the files `_open_files` opened.
    CUDA pieces: their targets, (name, device) in `devices`, must share one device; the
    pieces, sorted and without repeats (_unique_pieces), go through the arena in one file
    fill per _disjoint_groups group (fc_restore_files_async over the files' virtual
    concatenation, file k owning [bases[k], bases[k+1]); one file is n = 1, base 0).  CPU
    pieces are pread straight in.  Returns device_bytes, host_bytes, read_ms, scatter_ms,
    plans and files."""
    stats = {"device_bytes": 0.0, "host_bytes": 0.0, "read_ms": 0.0, "scatter_ms": 0.0,
             "plans": 0, "files": len(fds)}
    for name, d in devices:
        if d != devices[0][1]:
            raise ValueError(f"{name}: all CUDA leaves must live on one device; "
                             f"got {devices[0][1]} and {d}")
    if cuda:
        dev = devices[0][1]
        cuda = _unique_pieces(cuda)
        ends: Dict[Any, int] = {}  # in file order: the pieces are sorted by file
        for _, f, o, n in cuda:
            ends[f] = max(ends.get(f, 0), o + n)
        bases, b = {}, 0
        for f, end in ends.items():
            bases[f] = b
            b += end
        ranges = [(a, bases[f] + o, n) for a, f, o, n in cuda]
        stats["plans"] = _restore_file_groups(
            ranges, dev.index if dev.index is not None else torch.cuda.current_device(),
            stream, lambda plan, s: plan.restore_files_async(
                [fds[f] for f in bases], list(bases.values()), s), stats)
    t0 = time.perf_counter()
    host = _unique_pieces(host)
    for a, f, o, n in host:
        _pread_into(fds[f], (ctypes.c_char * n).from_address(a), o)
    stats["host_bytes"] = float(sum(n for _, _, _, n in host))
    stats["read_ms"] += (time.perf_counter() - t0) * 1e3
    return stats


def restore_file_into(path: str, target, stream=None, strict: bool = True,
                      index=None) -> Dict[str, float]:
    """Restore the torch.save file at `path` straight into the live tensors of `target`
    (the tree that was saved: same keys, exact shapes and dtypes, no casts).  The file is
    indexed without reading its payload (`torch_file_index.index_file`, torch's
    weights_only unpickler; pass `index` to reuse one).  CUDA leaves: the library preads
    the file through pinned bounce slots into the arena and scatters it with the unpack
    kernels (fc_restore_files_async); CPU leaves are pread straight into the tensors.
    Non-tensor leaves of the file are ignored.  On a short file (ShortFileError, an
    OSError) or a failed read nothing is scattered and the call raises.  The
    incremental-save baseline and the arena image are forgotten, as by every restore.

    Replaces `sd = torch.load(path, map_location="cpu"); model.load_state_dict(sd)`.
    stats: device_bytes, host_bytes, read_ms, scatter_ms, wall_ms."""
    from .torch_file_index import TensorLeaf, index_file

    t0 = time.perf_counter()
    if index is None:
        index = index_file(path)
    cuda, host, devices = [], [], []
    staging = {}  # CPU targets without dense rows: read into a dense copy, then copy_
    for name, t, leaf in _match_tree(target, index.tree, TensorLeaf, (list, tuple), strict):
        shape, stride = leaf.shape, leaf.stride
        src = _view_rows(shape, stride, leaf.storage_offset, t.element_size())
        if src is None or (shape and shape[-1] != 1 and stride[-1] != 1):
            raise ValueError(f"{name}: the file holds a view that is neither dense nor "
                             f"row-strided (shape {shape}, stride {stride}) in {index.path}")
        dst = _target_rows(t)
        if dst is None and t.is_cuda:
            raise ValueError(f"{name}: restore needs dense or row-strided CUDA targets "
                             f"(got shape {tuple(t.shape)}, strides {t.stride()})")
        if dst is None:  # one dense copy per target tensor: tied leaves share it
            if id(t) not in staging:
                staging[id(t)] = (t, torch.empty(t.shape, dtype=t.dtype))
            dst = _target_rows(staging[id(t)][1])
        if t.is_cuda:
            devices.append((name, t.device))
        (cuda if t.is_cuda else host).extend(
            (p, path, leaf.file_offset + f, n) for p, f, n in _pair_rows(src, dst))
    with _open_files("", cuda + host) as fds, torch.no_grad():
        got = _read_pieces(fds, cuda, host, devices, stream)
        t1 = time.perf_counter()
        for t, s in staging.values():
            t.copy_(s)
    stats = {k: got[k] for k in ("device_bytes", "host_bytes", "read_ms", "scatter_ms")}
    stats["read_ms"] += (time.perf_counter() - t1) * 1e3
    stats["wall_ms"] = (time.perf_counter() - t0) * 1e3
    return stats


