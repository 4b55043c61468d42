"""O_DIRECT writes for the agent's persist step (SURVEY §8 f.1, second half).

The reference persists a shard with one buffered `torch.save` / `f.write`
(ckpt_saver.py:1079-1122, :1453-1494, storage.py:129-141): every byte goes through the
page cache, which on a checkpoint-sized file means a second copy in host memory, dirty-page
throttling and write-back competing with the next memory checkpoint.  On a file system
backed by a block device the payload can bypass the page cache:

  * the file is cut into 4 KiB blocks; a block that lies completely inside one payload
    range is written through an O_DIRECT descriptor, every other block (headers, the
    partial blocks at the edges of a range) through a normal buffered one — no block is
    ever touched by both, so the two views of the file cannot disagree;
  * O_DIRECT wants the memory address aligned like the file offset.  A range whose source
    address is congruent with its file offset mod 4 KiB (the raw `.distcp` segment: page
    aligned, written at offset 0) is written straight from where it lies; any other range
    (tensor payloads inside the torch zip) goes through a page-aligned bounce buffer per
    writer thread;
  * the bytes and their offsets are exactly the buffered writer's — files stay
    byte-identical (tests/test_direct_io.py compares sha256).

`enabled_for(path)`: DLROVER_B200_DIRECT_IO=1 forces it (after a probe write), "auto" uses it on
ext4 / xfs / btrfs / f2fs mounts, the default "0" leaves it off: on an overlay file system O_DIRECT
buys nothing and the buffered writer returns sooner while the page cache absorbs the file — how long
the agent holds the shard lock is what matters there.
"""

from __future__ import annotations

import mmap
import os
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, List, Tuple

import numpy as np

from .log import default_logger as logger

BLOCK = 4096
PIECE = 16 << 20  # bytes per direct write call / bounce buffer size

_probe_cache: Dict[str, bool] = {}


def _fs_type(path: str) -> str:
    best, fstype = "", ""
    try:
        real = os.path.realpath(path)
        with open("/proc/mounts") as f:
            for line in f:
                parts = line.split()
                if len(parts) < 3:
                    continue
                mnt = parts[1]
                if (real == mnt or real.startswith(mnt.rstrip("/") + "/")) and len(mnt) > len(best):
                    best, fstype = mnt, parts[2]
    except OSError:
        pass
    return fstype


def _probe(dirpath: str) -> bool:
    got = _probe_cache.get(dirpath)
    if got is not None:
        return got
    ok = False
    p = os.path.join(dirpath, f".fc_odirect_probe_{os.getpid()}")
    try:
        fd = os.open(p, os.O_WRONLY | os.O_CREAT | os.O_DIRECT, 0o600)
        try:
            buf = mmap.mmap(-1, BLOCK)
            ok = os.pwrite(fd, buf, 0) == BLOCK
            buf.close()
        finally:
            os.close(fd)
    except (OSError, AttributeError):
        ok = False
    finally:
        try:
            os.remove(p)
        except OSError:
            pass
    _probe_cache[dirpath] = ok
    return ok


def enabled_for(path: str) -> bool:
    mode = os.getenv("DLROVER_B200_DIRECT_IO", "0").strip().lower()
    if mode in ("0", "false", "off", ""):
        return False
    d = os.path.dirname(os.path.abspath(path)) or "."
    if mode in ("1", "true", "on"):
        return _probe(d)
    return _fs_type(d) in ("ext4", "ext3", "xfs", "btrfs", "f2fs") and _probe(d)


def _addr(view: memoryview) -> int:
    return np.frombuffer(view, dtype=np.uint8).ctypes.data if view.nbytes else 0


class DirectWriter:
    """Writes byte ranges of ONE file, direct where whole blocks allow it.

        w = DirectWriter(path, total_bytes, threads)
        w.write_small(bytes, offset)        # headers etc.: buffered
        w.add(view, offset)                 # a payload range, queued
        w.run()                             # all queued ranges, in parallel
        w.close()                           # fsync (buffered part) + close
    """

    def __init__(self, path: str, total: int, threads: int = 4):
        self.path, self.total, self.threads = path, total, max(1, threads)
        self.fd = os.open(path, os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o644)
        os.ftruncate(self.fd, total)
        self.dfd = os.open(path, os.O_WRONLY | os.O_DIRECT)
        self._jobs: List[Tuple[memoryview, int, int, int]] = []  # view, lo, hi, file offset of lo
        self.direct_bytes = 0
        self.buffered_bytes = 0

    def write_small(self, data, offset: int):
        view = memoryview(data).cast("B")
        done = 0
        while done < view.nbytes:
            done += os.pwrite(self.fd, view[done:], offset + done)
        self.buffered_bytes += view.nbytes

    def add(self, view: memoryview, offset: int):
        view = view.cast("B")
        n = view.nbytes
        if n == 0:
            return
        first = (offset + BLOCK - 1) // BLOCK * BLOCK   # first whole block
        last = (offset + n) // BLOCK * BLOCK            # end of the last whole block
        if last <= first:
            self._jobs.append((view, 0, n, offset))      # no whole block: all buffered
            return
        if first > offset:
            self._jobs.append((view, 0, first - offset, offset))
        for lo in range(first, last, PIECE):
            hi = min(last, lo + PIECE)
            self._jobs.append((view, lo - offset, hi - offset, lo))
        if offset + n > last:
            self._jobs.append((view, last - offset, n, last))

    def _put(self, job, bounce: mmap.mmap):
        view, lo, hi, off = job
        n = hi - lo
        whole = off % BLOCK == 0 and n % BLOCK == 0
        if not whole:
            done = 0
            while done < n:
                done += os.pwrite(self.fd, view[lo + done:hi], off + done)
            return 0, n
        src = view[lo:hi]
        if _addr(src) % BLOCK != 0:
            # bounce: numpy's copy releases the GIL, the writers really run in parallel
            np.copyto(np.frombuffer(bounce, dtype=np.uint8, count=n),
                      np.frombuffer(src, dtype=np.uint8))
            src = memoryview(bounce)[:n]
        done = 0
        while done < n:
            k = os.pwrite(self.dfd, src[done:], off + done)
            if k % BLOCK and done + k < n:   # short, unaligned progress: finish buffered
                rest = src[done + k:]
                d2 = 0
                while d2 < rest.nbytes:
                    d2 += os.pwrite(self.fd, rest[d2:], off + done + k + d2)
                return done + k, n - done - k
            done += k
        return n, 0

    def run(self):
        jobs, self._jobs = self._jobs, []
        if not jobs:
            return

        def worker(chunk):
            bounce = mmap.mmap(-1, PIECE)
            d = b = 0
            try:
                for job in chunk:
                    dd, bb = self._put(job, bounce)
                    d += dd
                    b += bb
            finally:
                try:
                    bounce.close()
                except BufferError:
                    pass
            return d, b

        nt = min(self.threads, len(jobs))
        chunks = [jobs[i::nt] for i in range(nt)]
        with ThreadPoolExecutor(max_workers=nt) as pool:
            for d, b in pool.map(worker, chunks):
                self.direct_bytes += d
                self.buffered_bytes += b

    def close(self, sync: bool = True):
        try:
            if sync:
                os.fsync(self.fd)  # the buffered edges + metadata; direct blocks are on the device
        finally:
            os.close(self.dfd)
            os.close(self.fd)


def write_buffer(path: str, view: memoryview, threads: int = 4) -> Tuple[int, int]:
    """One big buffer (the raw shm segment of the FSDP/DCP saver) to `path`.
    Returns (direct bytes, buffered bytes)."""
    view = view.cast("B")
    w = DirectWriter(path, view.nbytes, threads)
    try:
        w.add(view, 0)
        w.run()
    finally:
        w.close()
    logger.info(f"O_DIRECT persist of {path}: {w.direct_bytes} B direct, "
                f"{w.buffered_bytes} B buffered")
    return w.direct_bytes, w.buffered_bytes
