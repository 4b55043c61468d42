"""Plain-Python model of a plan (include/flashckpt.h): how fc_plan_create cuts byte
ranges into work items, which kernel table each item goes to, how the drain merges
ranges into DMA runs, and what an incremental save must drain.

A test helper, not a test file.  It models this project's own plan, so it lives
here rather than under oracle/ (which restates the reference).  It is written from
the header's contract; the tests compare the library's counts and bytes with it.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Iterable, List, Sequence

import numpy as np

BOUNDARY = 128        # interior item boundaries are 128-B aligned in arena space
VEC = 16              # the bulk (TMA) kernels move whole 16-B words
SHIFT_MIN = 4096      # a shifted item under this many bytes goes to the LSU kernel

LSU, TMA = 1, 2       # _native.VARIANT_LSU / VARIANT_TMA


@dataclass(frozen=True)
class Range:
    """One input range: n bytes at device address tptr, arena offset aoff, segment
    offset hoff (None: the same as aoff, the identity mapping of fc_plan_create)."""

    tptr: int
    aoff: int
    n: int
    hoff: int = None

    def __post_init__(self):
        if self.hoff is None:
            object.__setattr__(self, "hoff", self.aoff)


@dataclass(frozen=True)
class Item:
    """One work item (or a piece of one: a head, body or tail); index is the position
    of its item in the arena-sorted `all` table."""

    tptr: int
    aoff: int
    n: int
    hoff: int
    index: int = -1


def items(ranges: Iterable[Range], chunk: int) -> List[Item]:
    """Split each non-empty range: the first piece is min(n, chunk - aoff % 128) bytes,
    then whole chunks.  Stable-sorted by arena offset."""
    out = []
    for r in ranges:
        tptr, aoff, hoff, left = r.tptr, r.aoff, r.hoff, r.n
        size = chunk - aoff % BOUNDARY
        while left > 0:
            n = min(left, size)
            out.append((tptr, aoff, n, hoff))
            tptr, aoff, hoff, left, size = tptr + n, aoff + n, hoff + n, left - n, chunk
    out.sort(key=lambda it: it[1])
    return [Item(t, a, n, h, k) for k, (t, a, n, h) in enumerate(out)]


def tables(all_items: Sequence[Item]) -> Dict[str, List[Item]]:
    """Route each item to the tables of the TMA variant.  An item whose source and
    arena offset differ mod 16 goes whole to `shift` (>= 4096 B) or `resid`; any
    other item splits into a head (resid), a body of whole 16-B words (bulk) and a
    tail (resid)."""
    t = {"bulk": [], "resid": [], "shift": []}
    for it in all_items:
        if (it.tptr - it.aoff) % VEC:
            t["shift" if it.n >= SHIFT_MIN else "resid"].append(it)
            continue
        head = min((-it.aoff) % VEC, it.n)
        body = (it.n - head) // VEC * VEC
        tail = it.n - head - body
        for name, start, n in (("resid", 0, head), ("bulk", head, body),
                               ("resid", head + body, tail)):
            if n:
                t[name].append(Item(it.tptr + start, it.aoff + start, n, it.hoff + start,
                                    it.index))
    return t


def runs(ranges: Iterable) -> List[Item]:
    """Merge ranges (anything with aoff, n, hoff), sorted by arena offset, where both
    the arena and the segment continue."""
    out: List[Item] = []
    for r in sorted((r for r in ranges if r.n), key=lambda r: r.aoff):
        if out and out[-1].aoff + out[-1].n == r.aoff and out[-1].hoff + out[-1].n == r.hoff:
            last = out[-1]
            out[-1] = Item(last.tptr, last.aoff, last.n + r.n, last.hoff)
        else:
            out.append(Item(r.tptr, r.aoff, r.n, r.hoff))
    return out


def dirty(all_items: Sequence[Item], old_image: np.ndarray, new_image: np.ndarray,
          origin: int = 0) -> List[Item]:
    """The items with any byte of their extent different between two arena images
    (byte k of an image is arena byte origin + k)."""
    changed = np.flatnonzero(old_image != new_image) + origin
    start = np.array([it.aoff for it in all_items], dtype=np.int64)
    end = start + np.array([it.n for it in all_items], dtype=np.int64)
    hit = np.searchsorted(changed, end) > np.searchsorted(changed, start)
    return [it for it, h in zip(all_items, hit) if h]


def drained_bytes(dirty_items: Iterable[Item]) -> int:
    return sum(it.n for it in dirty_items)


def dma_count(run_list: Iterable, piece: int) -> int:
    """DMA copies the drain issues for these runs (pinned host buffer, no slices):
    every run is cut into pieces of at most `piece` bytes."""
    return sum(-(-r.n // piece) for r in run_list)


def cta_load(table: Sequence[Item], ctas: int, tile: int, shifted: bool = False):
    """(tiles, items) each CTA of a TMA ring kernel walks: the grid is min(len(table),
    ctas) and CTA c takes items c, c + grid, ...; an item is ceil(bytes / tile) tiles.
    shifted: the byte-shift kernel of a pack, whose tiles cover the 16-B words of the
    item after the bytes that bring its arena side to 16-B alignment."""
    grid = min(len(table), ctas)
    load = [[0, 0] for _ in range(grid)]
    for k, it in enumerate(table):
        n = (it.n - min((-it.aoff) % VEC, it.n)) // VEC * VEC if shifted else it.n
        load[k % grid][0] += -(-n // tile)
        load[k % grid][1] += 1
    return [tuple(x) for x in load]


def kernel_count(tbl: Dict[str, List[Item]], variant: int) -> int:
    """Kernels one pack / unpack / gather-compare of the whole plan launches: one per
    non-empty table for TMA, one for LSU, none for an empty plan."""
    if variant == TMA:
        return sum(1 for v in tbl.values() if v)
    return 1 if any(tbl.values()) else 0
