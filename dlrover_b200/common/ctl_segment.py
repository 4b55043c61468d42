"""Control segment: the meta plane of one checkpoint shard in shared memory.

The reference keeps the meta tree of a shard in the agent's ``SharedDict`` and the
trainer re-sends the whole pickled tree twice per save over a unix socket
(ckpt_saver.py:315-327, multi_process.py:579-672; SURVEY §8 f.4).  Here a small POSIX
shm segment next to the data segment — ``[<run_id>_]ckpt_ctl_<shard>`` — holds

  * a header guarded by a seqlock: step, "segment is being written" flag, payload
    size, the length of the per-save blob (the pickled CheckpointConfig of the current
    save and other small per-save objects, up to 1 MiB) and the generation / length of
    the meta area;
  * one slot per local rank for cooperative saves (each rank reports the step whose
    slice it has landed in the data segment);
  * the pickled meta tree, rewritten only when the structure of the state dict (or a
    non-tensor leaf) changed.

A steady-state save therefore costs the trainer two header updates (a few stores) and
no socket round trip; the agent reads the header with a seqlock retry loop.  The data
segment keeps the reference's byte layout — nothing is added to it.  The agent creates
the control segment (that is how a trainer recognises an agent that understands it);
with the reference's agent there is none and the trainer falls back to ``SharedDict``.

Memory ordering: the header is written and read with plain stores / loads from Python
(``struct.pack_into``); the seqlock is sound on hosts with total store order (x86-64, the
host CPU of HGX H100 systems).  On a weakly ordered host (Grace) the odd/even sequence
stores need release / acquire fences — move ``publish`` / ``snapshot`` into the C library
(``std::atomic_thread_fence``) before relying on it there.
"""

from __future__ import annotations

import os
import pickle
import struct
import time
from typing import Any, Optional, Tuple

from .log import default_logger as logger
from .multi_process import SharedMemory

MAGIC = int.from_bytes(b"FCCTL01\0", "little")
VERSION = 1
HEADER_BYTES = 4096
SLOT_BYTES = 64
MAX_SLOTS = 64
# the per-save ("volatile") blob: the pickled CheckpointConfig plus whatever small
# objects change at every save (FSDP: the non-sharded entries of the state dict)
CONF_OFFSET = HEADER_BYTES + SLOT_BYTES * MAX_SLOTS  # 8192
CONF_CAPACITY = 1 << 20
META_OFFSET = CONF_OFFSET + CONF_CAPACITY
DEFAULT_BYTES = 16 << 20

# header field offsets (little-endian u64 unless noted)
_OFF_MAGIC, _OFF_VERSION, _OFF_SEQ, _OFF_STEP, _OFF_WRITING = 0, 8, 16, 24, 32
_OFF_PAYLOAD, _OFF_META_GEN, _OFF_META_LEN, _OFF_CONF_LEN = 40, 48, 56, 64
_OFF_COOP_SEQ = 72  # number of the current cooperative save (the slots answer with it)
_OFF_COOP_ABORT = 80  # 1: the leader gave up on save number COOP_SEQ before it started

SLOT_FAILED = -1


def ctl_name(shard_id: int, run_id: Optional[str] = None) -> str:
    run_id = os.getenv("TORCHELASTIC_RUN_ID", "") if run_id is None else run_id
    base = f"ckpt_ctl_{shard_id}"
    return f"{run_id}_{base}" if run_id else base


class ControlSegment:
    """One mapping of a shard's control segment.  Single writer at a time (whoever
    holds the shard lock / the saving trainer), any number of readers."""

    def __init__(self, shm: SharedMemory):
        self._shm = shm
        self._buf = shm.buf
        self._cached_gen = -1
        self._cached_meta: Any = None

    # -- lifecycle ----------------------------------------------------------------
    @classmethod
    def create(cls, shard_id: int, nbytes: int = DEFAULT_BYTES) -> "ControlSegment":
        """Create the shard's control segment (re-initialising one a previous agent of the
        same name left behind: like the reference's SharedDict, a new agent starts with no
        meta — a leftover segment of an unrelated earlier job must not look loadable)."""
        name = ctl_name(shard_id)
        try:
            shm = SharedMemory(name=name, create=True, size=max(nbytes, META_OFFSET + (1 << 20)))
            fresh = True
        except FileExistsError:
            shm = SharedMemory(name=name)
            fresh = False
            if shm.size < META_OFFSET + (1 << 20):  # left by something else: start over
                shm.unlink()
                shm.close()
                shm = SharedMemory(name=name, create=True,
                                   size=max(nbytes, META_OFFSET + (1 << 20)))
                fresh = True
        seg = cls(shm)
        if fresh or seg._u64(_OFF_MAGIC) != MAGIC:
            struct.pack_into("<QQ", seg._buf, _OFF_VERSION, VERSION, 0)
            for off in (_OFF_STEP, _OFF_WRITING, _OFF_PAYLOAD, _OFF_META_GEN, _OFF_META_LEN,
                        _OFF_CONF_LEN, _OFF_COOP_SEQ, _OFF_COOP_ABORT):
                seg._put(off, 0)
            seg._put(_OFF_MAGIC, MAGIC)
        else:
            seg.clear()  # keeps the sequence numbers monotonic for attached readers
        return seg

    @classmethod
    def attach(cls, shard_id: int) -> Optional["ControlSegment"]:
        try:
            shm = SharedMemory(name=ctl_name(shard_id))
        except FileNotFoundError:
            return None
        seg = cls(shm)
        if shm.size < META_OFFSET or seg._u64(_OFF_MAGIC) != MAGIC:
            shm.close()
            return None
        return seg

    def stale(self) -> bool:
        return self._shm.stale()

    @property
    def meta_capacity(self) -> int:
        return self._shm.size - META_OFFSET

    @property
    def conf_capacity(self) -> int:
        return CONF_CAPACITY

    def close(self):
        self._buf = None
        self._shm.close()

    def unlink(self):
        self._shm.unlink()

    # -- raw access ---------------------------------------------------------------
    def _u64(self, off: int) -> int:
        return struct.unpack_from("<Q", self._buf, off)[0]

    def _put(self, off: int, value: int):
        struct.pack_into("<Q", self._buf, off, value)

    # -- header (seqlock) -----------------------------------------------------------
    def publish(self, *, step: int, writing: bool, payload_bytes: int, conf_blob: bytes,
                meta_blob: Optional[bytes] = None) -> bool:
        """Writer side.  meta_blob=None keeps the meta area (same structure as the last
        save).  False when the blobs do not fit (the caller grows the segment or falls
        back to the SharedDict)."""
        if len(conf_blob) > CONF_CAPACITY or (meta_blob is not None and
                                              len(meta_blob) > self.meta_capacity):
            return False
        seq = self._u64(_OFF_SEQ)
        if seq & 1:  # a writer died mid-update: take over
            seq += 1
        self._put(_OFF_SEQ, seq + 1)
        if meta_blob is not None:
            self._buf[META_OFFSET:META_OFFSET + len(meta_blob)] = meta_blob
            self._put(_OFF_META_LEN, len(meta_blob))
            self._put(_OFF_META_GEN, self._u64(_OFF_META_GEN) + 1)
        self._buf[CONF_OFFSET:CONF_OFFSET + len(conf_blob)] = conf_blob
        self._put(_OFF_CONF_LEN, len(conf_blob))
        self._put(_OFF_STEP, step)
        self._put(_OFF_PAYLOAD, payload_bytes)
        self._put(_OFF_WRITING, 1 if writing else 0)
        self._put(_OFF_SEQ, seq + 2)
        return True

    def clear(self):
        """Forget the checkpoint (meta generation back to 0: readers see "nothing here")."""
        seq = self._u64(_OFF_SEQ) | 1
        self._put(_OFF_SEQ, seq)
        for off in (_OFF_STEP, _OFF_WRITING, _OFF_PAYLOAD, _OFF_META_GEN, _OFF_META_LEN,
                    _OFF_CONF_LEN):
            self._put(off, 0)
        self._put(_OFF_SEQ, seq + 1)
        self._cached_gen, self._cached_meta = -1, None

    def has_meta(self) -> bool:
        return self._u64(_OFF_META_GEN) > 0

    def snapshot(self, timeout: float = 5.0) -> Optional[Tuple[int, bool, int, bytes, int, Any]]:
        """Reader side: a consistent (step, writing, payload_bytes, conf_blob, meta_gen,
        meta tree) or None when the segment holds no meta.  The unpickled meta tree is
        cached per generation."""
        deadline = time.time() + timeout
        while True:
            s1 = self._u64(_OFF_SEQ)
            if not (s1 & 1):
                gen = self._u64(_OFF_META_GEN)
                if gen == 0:
                    if self._u64(_OFF_SEQ) == s1:
                        return None
                    continue
                step, writing = self._u64(_OFF_STEP), bool(self._u64(_OFF_WRITING))
                payload, conf_len = self._u64(_OFF_PAYLOAD), self._u64(_OFF_CONF_LEN)
                meta_len = self._u64(_OFF_META_LEN)
                conf_blob = bytes(self._buf[CONF_OFFSET:CONF_OFFSET + min(conf_len, CONF_CAPACITY)])
                meta_blob = None
                if gen != self._cached_gen:
                    meta_blob = bytes(self._buf[META_OFFSET:META_OFFSET + min(meta_len,
                                                                             self.meta_capacity)])
                if self._u64(_OFF_SEQ) == s1:
                    if meta_blob is not None:
                        self._cached_meta = pickle.loads(meta_blob)
                        self._cached_gen = gen
                    return step, writing, payload, conf_blob, gen, self._cached_meta
            if time.time() > deadline:
                logger.warning("control segment: no consistent snapshot (writer stuck mid-update?)")
                return None
            time.sleep(0.0005)

    # -- cooperative-save slots -------------------------------------------------------
    def next_coop_seq(self, aborted: bool = False) -> int:
        """Leader: open cooperative save number seq+1 — called once the data segment has
        its final size and the "being written" announcement is out; the other local ranks
        spin on coop_seq() and start writing their slices when they see it.  aborted=True
        tells them to give up instead."""
        seq = self._u64(_OFF_COOP_SEQ) + 1
        self._put(_OFF_COOP_ABORT, 1 if aborted else 0)
        self._put(_OFF_COOP_SEQ, seq)
        return seq

    def coop_seq(self) -> int:
        return self._u64(_OFF_COOP_SEQ)

    def wait_coop_open(self, seq: int, timeout: float) -> bool:
        """Follower: block until the leader has opened save `seq`; False = aborted."""
        deadline = time.time() + timeout
        delay = 0.00005
        while self._u64(_OFF_COOP_SEQ) < seq:
            if time.time() > deadline:
                raise TimeoutError(f"cooperative save {seq}: the leader did not open it")
            time.sleep(delay)
            delay = min(delay * 1.5, 0.001)
        return self._u64(_OFF_COOP_ABORT) == 0

    # slot layout: +0 done_seq, +8 status, +16 arrived_seq, +24 ready
    def slot_arrive(self, local_rank: int, seq: int, ready: bool):
        """Follower: "I am in save number `seq`" (seq 0 withdraws), with whether it can
        take part (no drain of its own still in flight)."""
        off = HEADER_BYTES + SLOT_BYTES * local_rank
        struct.pack_into("<Q", self._buf, off + 24, 1 if ready else 0)
        struct.pack_into("<Q", self._buf, off + 16, seq)

    def wait_arrivals(self, n_ranks: int, seq: int, timeout: float) -> Tuple[bool, bool]:
        """Leader: wait until the local ranks 1..n-1 have arrived in save `seq`.
        (all arrived, all ready)."""
        deadline = time.time() + timeout
        delay = 0.00005
        while True:
            arrived = ready = 0
            for r in range(1, n_ranks):
                off = HEADER_BYTES + SLOT_BYTES * r
                a, rd = struct.unpack_from("<QQ", self._buf, off + 16)
                if a == seq:
                    arrived += 1
                    ready += 1 if rd else 0
            if arrived == n_ranks - 1:
                return True, ready == n_ranks - 1
            if time.time() > deadline:
                return False, False
            time.sleep(delay)
            delay = min(delay * 1.5, 0.001)

    def slot_set(self, local_rank: int, step: int, ok: bool = True):
        off = HEADER_BYTES + SLOT_BYTES * local_rank
        struct.pack_into("<q", self._buf, off + 8, 0 if ok else SLOT_FAILED)
        struct.pack_into("<Q", self._buf, off, step)

    def slot_get(self, local_rank: int) -> Tuple[int, int]:
        off = HEADER_BYTES + SLOT_BYTES * local_rank
        return struct.unpack_from("<Qq", self._buf, off)

    def wait_slots(self, n_ranks: int, step: int, timeout: float) -> bool:
        """True once every one of the first n_ranks slots reports `step` without an
        error; False on a reported failure or timeout."""
        deadline = time.time() + timeout
        delay = 0.0002
        while True:
            done = 0
            for r in range(n_ranks):
                s, status = self.slot_get(r)
                if s == step:
                    if status == SLOT_FAILED:
                        return False
                    done += 1
            if done == n_ranks:
                return True
            if time.time() > deadline:
                return False
            time.sleep(delay)
            delay = min(delay * 1.5, 0.002)
