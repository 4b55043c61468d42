"""ctypes binding of ``libflashckpt.so`` (the C-ABI declared in include/flashckpt.h).

This is the only module that touches the shared library.  There is NO CPU
fallback: if the library is missing or a call fails, ``NativeError`` is raised
so a GPU box can never silently run the reference's per-tensor ``copy_`` loop
(dlrover/python/elastic_agent/torch/ckpt_saver.py:198-231) instead of the
sm_90a kernels.
"""

from __future__ import annotations

import ctypes
import os
import threading
from typing import Optional, Sequence, Tuple

_LIB_NAME = "libflashckpt.so"
_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", _LIB_NAME)

FC_OK = 0
FC_EINVAL = -1
FC_ECUDA = -2
FC_ENOMEM = -3
FC_EBUSY = -4
FC_ENOTREADY = 1

VARIANT_AUTO = 0
VARIANT_LSU = 1
VARIANT_TMA = 2

DRAIN_HOST_PACED = 0
DRAIN_PINGPONG = 1

# every symbol include/flashckpt.h declares: (name, restype, argtypes)
_u64 = ctypes.c_uint64
_u32 = ctypes.c_uint32
_vp = ctypes.c_void_p
_fp = ctypes.POINTER(ctypes.c_float)
_SIGNATURES = {
    "fc_version": (ctypes.c_int, []),
    "fc_strerror": (ctypes.c_char_p, [ctypes.c_int]),
    "fc_last_error": (ctypes.c_char_p, []),
    "fc_ctx_create": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(_vp)]),
    "fc_ctx_destroy": (ctypes.c_int, [_vp]),
    "fc_arena_reserve": (ctypes.c_int, [_vp, _u64]),
    "fc_set_arena_limit": (ctypes.c_int, [_vp, _u64]),
    "fc_arena_info": (ctypes.c_int, [_vp, ctypes.POINTER(_vp), ctypes.POINTER(_u64)]),
    "fc_host_register": (ctypes.c_int, [_vp, _vp, _u64, ctypes.c_int]),
    "fc_host_unregister": (ctypes.c_int, [_vp, _vp]),
    "fc_host_register_background": (ctypes.c_int, [_vp, _vp, _u64, _u64]),
    "fc_host_ready": (ctypes.c_int, [_vp, _vp]),
    "fc_host_bind_numa": (ctypes.c_int, [_vp, _vp, _u64, ctypes.c_int]),
    "fc_device_numa_node": (ctypes.c_int, [ctypes.c_int, ctypes.POINTER(ctypes.c_int),
                                           ctypes.POINTER(ctypes.c_int)]),
    "fc_set_stage": (ctypes.c_int, [_vp, ctypes.c_int, _u64]),
    "fc_set_drain_mode": (ctypes.c_int, [_vp, ctypes.c_int]),
    "fc_plan_create": (
        ctypes.c_int,
        [_vp, _u32, ctypes.POINTER(_vp), ctypes.POINTER(_u64), ctypes.POINTER(_u64), _u32,
         ctypes.POINTER(_vp)],
    ),
    "fc_plan_update": (
        ctypes.c_int,
        [_vp, _u32, ctypes.POINTER(_vp), ctypes.POINTER(_u64), ctypes.POINTER(_u64), _vp],
    ),
    "fc_plan_create_mapped": (
        ctypes.c_int,
        [_vp, _u32, ctypes.POINTER(_vp), ctypes.POINTER(_u64), ctypes.POINTER(_u64),
         ctypes.POINTER(_u64), _u32, ctypes.POINTER(_vp)],
    ),
    "fc_plan_update_mapped": (
        ctypes.c_int,
        [_vp, _u32, ctypes.POINTER(_vp), ctypes.POINTER(_u64), ctypes.POINTER(_u64),
         ctypes.POINTER(_u64), _vp],
    ),
    "fc_plan_destroy": (ctypes.c_int, [_vp]),
    "fc_plan_info": (
        ctypes.c_int,
        [_vp, ctypes.POINTER(_u64), ctypes.POINTER(_u32), ctypes.POINTER(_u32),
         ctypes.POINTER(_u64)],
    ),
    "fc_pack_async": (ctypes.c_int, [_vp, _vp, ctypes.c_int]),
    "fc_unpack_async": (ctypes.c_int, [_vp, _vp, ctypes.c_int]),
    "fc_launch_count": (ctypes.c_int, [_vp, ctypes.POINTER(_u64), ctypes.POINTER(_u64)]),
    "fc_set_variant": (ctypes.c_int, [_vp, ctypes.c_int]),
    "fc_set_launch": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "fc_set_shift_launch": (ctypes.c_int, [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    "fc_save_async": (ctypes.c_int, [_vp, _vp, _vp, ctypes.POINTER(_u64)]),
    "fc_save_async_held": (ctypes.c_int, [_vp, _vp, _vp, ctypes.POINTER(_u64)]),
    "fc_save_release": (ctypes.c_int, [_vp, _u64]),
    "fc_save_cancel": (ctypes.c_int, [_vp, _u64]),
    "fc_save_direct_async": (ctypes.c_int, [_vp, _vp, _vp, ctypes.c_int, ctypes.POINTER(_u64)]),
    "fc_save_hybrid_async": (ctypes.c_int, [_vp, _vp, _vp, _u64, ctypes.c_int,
                                            ctypes.POINTER(_u64)]),
    "fc_save_delta_async": (ctypes.c_int, [_vp, _vp, _vp, ctypes.c_int, ctypes.POINTER(_u64)]),
    "fc_save_delta_stats": (ctypes.c_int, [_vp, _u64, ctypes.POINTER(_u64),
                                           ctypes.POINTER(ctypes.c_int)]),
    "fc_delta_invalidate": (ctypes.c_int, [_vp]),
    "fc_save_sources_wait": (ctypes.c_int, [_vp, _u64]),
    "fc_restore_direct_async": (ctypes.c_int, [_vp, _vp, _vp]),
    "fc_plan_spans": (ctypes.c_int, [_vp, ctypes.POINTER(_u32)]),
    "fc_save_pack_done": (ctypes.c_int, [_vp, _u64]),
    "fc_save_poll": (ctypes.c_int, [_vp, _u64]),
    "fc_save_wait": (ctypes.c_int, [_vp, _u64]),
    "fc_save_timings": (ctypes.c_int, [_vp, _u64, _fp, _fp, _fp]),
    "fc_set_drain": (ctypes.c_int, [_vp, _u64, ctypes.c_int]),
    "fc_host_unpack": (
        ctypes.c_int,
        [_vp, _u32, ctypes.POINTER(_vp), ctypes.POINTER(_u64), ctypes.POINTER(_u64), ctypes.c_int],
    ),
    "fc_host_pack": (
        ctypes.c_int,
        [_vp, _u32, ctypes.POINTER(_vp), ctypes.POINTER(_u64), ctypes.POINTER(_u64), ctypes.c_int],
    ),
    "fc_restore_async": (ctypes.c_int, [_vp, _vp, _vp]),
    "fc_arena_fill": (ctypes.c_int, [_vp, _vp, _u64, _u64, _vp]),
    "fc_restore_wait": (ctypes.c_int, [_vp]),
    "fc_restore_timings": (ctypes.c_int, [_vp, _fp, _fp, _fp]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


class NativeError(RuntimeError):
    """A libflashckpt call failed (or the library is not built)."""

    def __init__(self, code: int, what: str, detail: str = ""):
        self.code = code
        super().__init__(f"{what} failed with code {code}: {detail}")


class NativeBusy(NativeError):
    """FC_EBUSY: the previous save/restore on this context is still in flight."""


_lib = None
_lib_lock = threading.Lock()


def library_path() -> str:
    return _LIB_PATH


def load_library():
    """dlopen libflashckpt.so and type every entry point.  Raises loudly if it
    has not been built (``python -c 'import __graft_entry__ as g; g.build()'``)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(_LIB_PATH):
            raise NativeError(
                FC_EINVAL,
                "load_library",
                f"{_LIB_PATH} is not built; run __graft_entry__.build() "
                "(nvcc -gencode arch=compute_90a,code=sm_90a). There is no CPU fallback.",
            )
        lib = ctypes.CDLL(_LIB_PATH, mode=ctypes.RTLD_LOCAL)
        for name, (restype, argtypes) in _SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the .so is stale
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
        return _lib


def _check(rc: int, what: str) -> int:
    if rc < 0:
        lib = load_library()
        detail = lib.fc_last_error().decode("utf-8", "replace") or lib.fc_strerror(rc).decode()
        if rc == FC_EBUSY:
            raise NativeBusy(rc, what, detail)
        raise NativeError(rc, what, detail)
    return rc


def _stream_ptr(stream) -> Optional[int]:
    """Accepts None, an int (cudaStream_t) or a torch.cuda.Stream."""
    if stream is None:
        return None
    if isinstance(stream, int):
        return stream or None
    return int(stream.cuda_stream) or None


def _plan_key(ptrs, offsets, nbytes, host_offsets=None):
    key = ([int(p) for p in ptrs], [int(o) for o in offsets], [int(b) for b in nbytes])
    if host_offsets is not None:
        key += ([int(o) for o in host_offsets],)
    return key


class Plan:
    """Cached descriptor table of one state_dict structure (fc_plan)."""

    def __init__(self, ctx: "Context", handle: int, key):
        self._ctx = ctx
        self._h = handle
        self.key = key
        self._refresh_info()

    def _refresh_info(self):
        lib = load_library()
        payload, items, runs, end = _u64(), _u32(), _u32(), _u64()
        _check(
            lib.fc_plan_info(self._h, ctypes.byref(payload), ctypes.byref(items),
                             ctypes.byref(runs), ctypes.byref(end)),
            "fc_plan_info",
        )
        self.payload_bytes = payload.value
        self.n_items = items.value
        self.n_runs = runs.value
        self.arena_end = end.value
        spans = _u32()
        _check(lib.fc_plan_spans(self._h, ctypes.byref(spans)), "fc_plan_spans")
        self.n_spans = spans.value

    @property
    def handle(self) -> int:
        if not self._h:
            raise NativeError(FC_EINVAL, "Plan", "plan already destroyed")
        return self._h

    def update(self, ptrs: Sequence[int], offsets: Sequence[int], nbytes: Sequence[int],
               stream=None, host_offsets: Optional[Sequence[int]] = None):
        """Re-target the plan (stream-ordered table upload, no device sync)."""
        n = len(ptrs)
        a_ptr = (_vp * max(n, 1))(*[int(p) for p in ptrs])
        a_off = (_u64 * max(n, 1))(*[int(o) for o in offsets])
        a_len = (_u64 * max(n, 1))(*[int(b) for b in nbytes])
        if host_offsets is None:
            _check(load_library().fc_plan_update(self.handle, n, a_ptr, a_off, a_len,
                                                 _stream_ptr(stream)), "fc_plan_update")
        else:
            a_host = (_u64 * max(n, 1))(*[int(o) for o in host_offsets])
            _check(load_library().fc_plan_update_mapped(self.handle, n, a_ptr, a_off, a_host,
                                                        a_len, _stream_ptr(stream)),
                   "fc_plan_update_mapped")
        self.key = _plan_key(ptrs, offsets, nbytes, host_offsets)
        self._refresh_info()

    def pack(self, stream=None, variant: int = VARIANT_AUTO):
        _check(load_library().fc_pack_async(self.handle, _stream_ptr(stream), variant),
               "fc_pack_async")

    def unpack(self, stream=None, variant: int = VARIANT_AUTO):
        _check(load_library().fc_unpack_async(self.handle, _stream_ptr(stream), variant),
               "fc_unpack_async")

    def save_async(self, host_ptr: int, compute_stream=None, hold: bool = False) -> int:
        """hold=True: gather now, but start the drain only at Context.save_release."""
        ticket = _u64()
        fn = load_library().fc_save_async_held if hold else load_library().fc_save_async
        _check(fn(self.handle, host_ptr, _stream_ptr(compute_stream), ctypes.byref(ticket)),
               "fc_save_async")
        return ticket.value

    def save_direct_async(self, host_ptr: int, compute_stream=None, hold: bool = False) -> int:
        """In-place save: no snapshot, the drain reads the tensors themselves, which
        must stay unchanged until the ticket is drained."""
        ticket = _u64()
        _check(load_library().fc_save_direct_async(self.handle, host_ptr,
                                                   _stream_ptr(compute_stream), int(hold),
                                                   ctypes.byref(ticket)),
               "fc_save_direct_async")
        return ticket.value

    def save_hybrid_async(self, host_ptr: int, cut: int, compute_stream=None,
                          hold: bool = False) -> int:
        """Tensors at segment offsets >= cut are snapshotted into the arena, the rest
        is drained in place (first)."""
        ticket = _u64()
        _check(load_library().fc_save_hybrid_async(self.handle, host_ptr,
                                                   _stream_ptr(compute_stream), int(cut),
                                                   int(hold), ctypes.byref(ticket)),
               "fc_save_hybrid_async")
        return ticket.value

    def save_delta_async(self, host_ptr: int, compute_stream=None, hold: bool = False) -> int:
        """Incremental save: compare with the arena image of the last delta save of this
        plan to `host_ptr` and drain only the work items that changed (a full save when
        there is no such baseline).  See Context.save_delta_stats."""
        ticket = _u64()
        _check(load_library().fc_save_delta_async(self.handle, host_ptr,
                                                  _stream_ptr(compute_stream), int(hold),
                                                  ctypes.byref(ticket)),
               "fc_save_delta_async")
        return ticket.value

    def restore_async(self, host_ptr: int, stream=None, direct: bool = False):
        """direct=True: DMA straight into the target tensors (no arena, no kernel)."""
        lib = load_library()
        if direct:
            _check(lib.fc_restore_direct_async(self.handle, host_ptr, _stream_ptr(stream)),
                   "fc_restore_direct_async")
        else:
            _check(lib.fc_restore_async(self.handle, host_ptr, _stream_ptr(stream)),
                   "fc_restore_async")

    def destroy(self):
        if self._h:
            load_library().fc_plan_destroy(self._h)
            self._h = 0

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


class Context:
    """One per (process, device): side stream, events, HBM staging arena."""

    def __init__(self, device: int):
        lib = load_library()
        h = _vp()
        _check(lib.fc_ctx_create(int(device), ctypes.byref(h)), "fc_ctx_create")
        self._h = h.value
        self.device = int(device)
        self._registered = {}

    @property
    def handle(self) -> int:
        if not self._h:
            raise NativeError(FC_EINVAL, "Context", "context already destroyed")
        return self._h

    # -- arena / host segment ------------------------------------------------
    def arena_reserve(self, nbytes: int):
        _check(load_library().fc_arena_reserve(self.handle, int(nbytes)), "fc_arena_reserve")

    def set_arena_limit(self, nbytes: int):
        _check(load_library().fc_set_arena_limit(self.handle, int(nbytes)), "fc_set_arena_limit")

    def arena_info(self) -> Tuple[int, int]:
        p, n = _vp(), _u64()
        _check(load_library().fc_arena_info(self.handle, ctypes.byref(p), ctypes.byref(n)),
               "fc_arena_info")
        return (p.value or 0, n.value)

    def host_register(self, host_ptr: int, nbytes: int, prefault_threads: int = 0):
        _check(
            load_library().fc_host_register(self.handle, host_ptr, int(nbytes),
                                            int(prefault_threads)),
            "fc_host_register",
        )
        self._registered[host_ptr] = nbytes

    def host_register_background(self, host_ptr: int, nbytes: int, slice_bytes: int = 0):
        """Pin the range slice by slice on a library thread; returns at once."""
        _check(load_library().fc_host_register_background(self.handle, host_ptr, int(nbytes),
                                                          int(slice_bytes)),
               "fc_host_register_background")
        self._registered[host_ptr] = nbytes

    def host_ready(self, host_ptr: int) -> bool:
        """True once the range is completely pinned (plain DMA); False while a
        background registration is in progress or the range is unknown."""
        if host_ptr not in self._registered:
            return False
        rc = load_library().fc_host_ready(self.handle, host_ptr)
        if rc == FC_ENOTREADY:
            return False
        _check(rc, "fc_host_ready")
        return True

    def host_bind_numa(self, host_ptr: int, nbytes: int, remote_per256: int = 0):
        _check(load_library().fc_host_bind_numa(self.handle, host_ptr, int(nbytes),
                                                int(remote_per256)), "fc_host_bind_numa")

    def set_stage(self, threads: int = 0, slot_bytes: int = 0):
        _check(load_library().fc_set_stage(self.handle, int(threads), int(slot_bytes)),
               "fc_set_stage")

    def set_drain_mode(self, mode: int):
        _check(load_library().fc_set_drain_mode(self.handle, int(mode)), "fc_set_drain_mode")

    def host_unregister(self, host_ptr: int):
        if host_ptr in self._registered:
            _check(load_library().fc_host_unregister(self.handle, host_ptr),
                   "fc_host_unregister")
            self._registered.pop(host_ptr, None)

    # -- plans ----------------------------------------------------------------
    def plan(self, ptrs: Sequence[int], offsets: Sequence[int], nbytes: Sequence[int],
             chunk_bytes: int = 0, host_offsets: Optional[Sequence[int]] = None) -> Plan:
        """offsets: arena offsets; host_offsets (default: the same — the arena is an image
        of the segment): where each range goes in the host segment."""
        n = len(ptrs)
        if not (n == len(offsets) == len(nbytes)) or \
                (host_offsets is not None and len(host_offsets) != n):
            raise NativeError(FC_EINVAL, "plan", "ptrs/offsets/nbytes differ in length")
        a_ptr = (_vp * max(n, 1))(*[int(p) for p in ptrs])
        a_off = (_u64 * max(n, 1))(*[int(o) for o in offsets])
        a_len = (_u64 * max(n, 1))(*[int(b) for b in nbytes])
        h = _vp()
        if host_offsets is None:
            _check(
                load_library().fc_plan_create(self.handle, n, a_ptr, a_off, a_len,
                                              int(chunk_bytes), ctypes.byref(h)),
                "fc_plan_create",
            )
        else:
            a_host = (_u64 * max(n, 1))(*[int(o) for o in host_offsets])
            _check(
                load_library().fc_plan_create_mapped(self.handle, n, a_ptr, a_off, a_host, a_len,
                                                     int(chunk_bytes), ctypes.byref(h)),
                "fc_plan_create_mapped",
            )
        return Plan(self, h.value, _plan_key(ptrs, offsets, nbytes, host_offsets))

    def launch_count(self) -> Tuple[int, int]:
        k, m = _u64(), _u64()
        _check(load_library().fc_launch_count(self.handle, ctypes.byref(k), ctypes.byref(m)),
               "fc_launch_count")
        return k.value, m.value

    # -- tuning ----------------------------------------------------------------
    def set_variant(self, variant: int):
        _check(load_library().fc_set_variant(self.handle, int(variant)), "fc_set_variant")

    def set_launch(self, lsu_ctas_per_sm: int = 0, tma_ctas_per_sm: int = 0, tma_stages: int = 0,
                   tma_tile_bytes: int = 0):
        _check(
            load_library().fc_set_launch(self.handle, lsu_ctas_per_sm, tma_ctas_per_sm,
                                         tma_stages, tma_tile_bytes),
            "fc_set_launch",
        )

    def set_shift_launch(self, ctas_per_sm: int = 0, in_stages: int = 0, tile_bytes: int = 0):
        _check(load_library().fc_set_shift_launch(self.handle, ctas_per_sm, in_stages,
                                                  tile_bytes), "fc_set_shift_launch")

    def set_drain(self, piece_bytes: int = 0, depth: int = 0):
        _check(load_library().fc_set_drain(self.handle, int(piece_bytes), int(depth)),
               "fc_set_drain")

    # -- save / restore tickets ---------------------------------------------------
    def save_release(self, ticket: int):
        _check(load_library().fc_save_release(self.handle, ticket), "fc_save_release")

    def save_pack_done(self, ticket: int) -> bool:
        return _check(load_library().fc_save_pack_done(self.handle, ticket),
                      "fc_save_pack_done") == FC_OK

    def save_cancel(self, ticket: int) -> bool:
        """Drop a held save before any byte of the segment changed; False when the
        drain had already been released."""
        rc = load_library().fc_save_cancel(self.handle, ticket)
        if rc == FC_EBUSY:
            return False
        _check(rc, "fc_save_cancel")
        return True

    def save_sources_wait(self, ticket: int):
        """Block until save `ticket` no longer reads the source tensors."""
        _check(load_library().fc_save_sources_wait(self.handle, ticket), "fc_save_sources_wait")

    def save_poll(self, ticket: int) -> bool:
        return _check(load_library().fc_save_poll(self.handle, ticket), "fc_save_poll") == FC_OK

    def save_wait(self, ticket: int):
        _check(load_library().fc_save_wait(self.handle, ticket), "fc_save_wait")

    def save_timings(self, ticket: int) -> Tuple[float, float, float]:
        a, b, c = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
        _check(
            load_library().fc_save_timings(self.handle, ticket, ctypes.byref(a), ctypes.byref(b),
                                           ctypes.byref(c)),
            "fc_save_timings",
        )
        return a.value, b.value, c.value

    def save_delta_stats(self, ticket: int) -> Tuple[bool, int]:
        """(incremental, drained bytes) of a drained save."""
        nbytes, delta = _u64(), ctypes.c_int()
        rc = _check(load_library().fc_save_delta_stats(self.handle, ticket, ctypes.byref(nbytes),
                                                       ctypes.byref(delta)),
                    "fc_save_delta_stats")
        if rc == FC_ENOTREADY:
            raise NativeError(rc, "fc_save_delta_stats", "the save has not drained yet")
        return bool(delta.value), nbytes.value

    def delta_invalidate(self):
        """The next incremental save is a full one (something else wrote the arena or
        the segment)."""
        _check(load_library().fc_delta_invalidate(self.handle), "fc_delta_invalidate")

    def arena_fill(self, host_ptr: int, lo: int, hi: int, stream=None):
        """Host bytes [lo, hi) -> arena bytes [lo, hi); `stream` waits for them."""
        _check(load_library().fc_arena_fill(self.handle, host_ptr, int(lo), int(hi),
                                            _stream_ptr(stream)), "fc_arena_fill")

    def arena_tensor(self, nbytes: int):
        """The first nbytes of the arena as a uint8 torch tensor (no copy).  Whoever
        holds it may write the arena, so the incremental baseline is forgotten."""
        import torch

        self.delta_invalidate()
        ptr, size = self.arena_info()
        if nbytes > size:
            raise NativeError(FC_EINVAL, "arena_tensor", "arena smaller than requested")

        class _Arena:
            __cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1",
                                        "data": (ptr, False), "version": 2}

        return torch.as_tensor(_Arena(), device=torch.device("cuda", self.device))

    def restore_wait(self):
        _check(load_library().fc_restore_wait(self.handle), "fc_restore_wait")

    def restore_timings(self) -> Tuple[float, float, float]:
        a, b, c = ctypes.c_float(), ctypes.c_float(), ctypes.c_float()
        _check(
            load_library().fc_restore_timings(self.handle, ctypes.byref(a), ctypes.byref(b),
                                              ctypes.byref(c)),
            "fc_restore_timings",
        )
        return a.value, b.value, c.value

    def destroy(self):
        if self._h:
            load_library().fc_ctx_destroy(self._h)
            self._h = 0
            self._registered.clear()

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


def device_numa_node(device: int) -> Tuple[int, int]:
    """(NUMA node of the CUDA device or -1, number of NUMA nodes of the host)."""
    node, n = ctypes.c_int(-1), ctypes.c_int(0)
    _check(load_library().fc_device_numa_node(int(device), ctypes.byref(node), ctypes.byref(n)),
           "fc_device_numa_node")
    return node.value, n.value


def host_pack(dst_addr: int, ptrs: Sequence[int], offsets: Sequence[int],
              nbytes: Sequence[int], threads: int = 1):
    """Multi-threaded memcpy of host-resident ranges into the segment (no GPU)."""
    n = len(ptrs)
    if n == 0:
        return
    a_ptr = (_vp * n)(*[int(p) for p in ptrs])
    a_off = (_u64 * n)(*[int(o) for o in offsets])
    a_len = (_u64 * n)(*[int(b) for b in nbytes])
    _check(load_library().fc_host_pack(dst_addr, n, a_ptr, a_off, a_len, int(threads)),
           "fc_host_pack")


def host_unpack(src_addr: int, ptrs: Sequence[int], offsets: Sequence[int],
                nbytes: Sequence[int], threads: int = 1):
    """Multi-threaded memcpy out of the segment into host-resident ranges (no GPU)."""
    n = len(ptrs)
    if n == 0:
        return
    a_ptr = (_vp * n)(*[int(p) for p in ptrs])
    a_off = (_u64 * n)(*[int(o) for o in offsets])
    a_len = (_u64 * n)(*[int(b) for b in nbytes])
    _check(load_library().fc_host_unpack(src_addr, n, a_ptr, a_off, a_len, int(threads)),
           "fc_host_unpack")


_contexts = {}
_ctx_lock = threading.Lock()


def get_context(device: int) -> Context:
    """Process-wide context per device index."""
    with _ctx_lock:
        ctx = _contexts.get(device)
        if ctx is None or not ctx._h:
            ctx = Context(device)
            forced = os.getenv("DLROVER_B200_VARIANT", "").lower()
            if forced in ("lsu", "tma"):  # profiling / A-B runs only
                ctx.set_variant(VARIANT_LSU if forced == "lsu" else VARIANT_TMA)
            piece = int(os.getenv("DLROVER_B200_DRAIN_PIECE_MB", "0") or 0)
            depth = int(os.getenv("DLROVER_B200_DRAIN_DEPTH", "0") or 0)
            if piece or depth:  # tuning runs only
                ctx.set_drain(piece << 20, depth)
            mode = os.getenv("DLROVER_B200_DRAIN_MODE", "")
            if mode in ("0", "1"):
                ctx.set_drain_mode(int(mode))
            threads = int(os.getenv("DLROVER_B200_STAGE_THREADS", "0") or 0)
            if not threads:
                # first save / restart restore only; leave cores to the other local ranks
                local_world = int(os.getenv("LOCAL_WORLD_SIZE", "1") or 1)
                # at most 8: more threads fault a fresh segment in more slowly and
                # copy no faster
                threads = max(2, min(8, (os.cpu_count() or 2) // max(1, 2 * local_world)))
            ctx.set_stage(threads, 0)
            _contexts[device] = ctx
        return ctx
