"""The copy and gather-compare kernels against a byte model.

Every GPU test here keeps an exact expected image of every byte the library may
touch: the whole HBM arena, the whole pinned host segment and the whole buffer the
unpack / restore targets live in.  Bytes no operation may write hold a position
pattern (canaries), covered bytes follow oracle.pack_ranges, and tests/plan_model.py
says which work items an incremental save must drain, how many DMA copies that takes
and how many kernels a plan launches.  After every operation the device, the arena
and the host buffers must equal the model byte for byte.

The layouts cover leaf lengths around 16 B, 128 B, 4 KiB, the chunk and multiples of
the active tile sizes, sources and targets at every address mod 16, gaps of 0-17 and
128 B between ranges, a pair of tied leaves (two ranges over the same source bytes) and
a real mixed-dtype state dict.  They run under the default launch shape and four
others the setters accept.  Each generated layout starts with a ring section built
from the launch's grid rule: thousands of small congruent leaves, and large shifted
items on the round-robin slots of one CTA.  So every ring (copy, gather-compare and
byte-shift) walks at least three times its stage count in tiles on a CTA that owns
several items.  Its mbarrier parity thus goes through many phases, and its cursor
crosses into items whose loads are already in flight; the tests assert this from the
model.
"""

import contextlib
import ctypes
import mmap
import os
import time

import numpy as np
import pytest
import torch

from dlrover_b200 import _native as native
from oracle import shm_layout as oracle
from tests import plan_model as pm

gpu = pytest.mark.gpu

GUARD = 256
GAPS = (0, *range(1, 16), 16, 17, 128)
CHUNKS = (4096, 4096 + 128, 64 << 10, 0)  # 0: the library default
DEFAULT_CHUNK = 256 << 10
VARIANTS = (native.VARIANT_LSU, native.VARIANT_TMA)

# name: (set_launch(lsu, tma, stages, tile), set_shift_launch(cps, stages, tile)); None
# keeps the defaults
DEFAULT_LAUNCH = (2, 1, 2, 96 << 10)
DEFAULT_SHIFT_LAUNCH = (2, 2, 16 << 10)
SHAPES = {
    "default": (None, None),
    "tiny_ring": ((1, 1, 2, 16), (1, 2, 4096)),
    "deep_odd_tile": ((8, 2, 8, 4112), (8, 8, 4224)),
    "many_stages": ((2, 1, 32, 6144), (2, 2, 57344)),
    "largest_tile": ((2, 1, 2, 115712), None),
}


def pattern(n, start=0):
    """The canary: byte i of a buffer holds (i * 131 + 7) & 255."""
    return ((np.arange(start, start + n, dtype=np.int64) * 131 + 7) & 255).astype(np.uint8)


def _launch(shape):
    """((lsu, tma CTAs/SM, stages, tile), (shift CTAs/SM, stages, tile)) in force."""
    launch, shift = SHAPES[shape]
    return launch or DEFAULT_LAUNCH, shift or DEFAULT_SHIFT_LAUNCH


def _tiles(shape):
    """(copy tile, gather-compare tile, shift tile) of a launch shape."""
    (_, _, _, tile), (_, _, shift_tile) = _launch(shape)
    return tile, max(128, (tile // 2) & ~127), shift_tile


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _context(shape, variant, arena_limit=0):
    """A private context with the shape applied (it must not leak into other tests)."""
    ctx = native.Context(0)
    try:
        ctx.set_variant(variant)
        ctx.set_arena_limit(arena_limit)
        launch, shift = SHAPES[shape]
        if launch:
            ctx.set_launch(*launch)  # raises if the setter refuses the shape
        if shift:
            ctx.set_shift_launch(*shift)
    except BaseException:
        ctx.destroy()
        raise
    return ctx


def ring_section(shape, sms, shift=True):
    """Leaves (length, (source - arena) class mod 16) that load every TMA ring of the
    shape, to be laid out first and back to back from a 16-B aligned arena offset.

    Bulk: (3 x stages - 1) x grid + 1 congruent 32-B leaves, one bulk item of one or two
    tiles each, so that every CTA of the copy and gather-compare kernels walks about
    3 x stages tiles, item after item.  Shift: the first entries of the shift table
    are a 60000-B item on each of CTA 0's round-robin slots and 4096-B items in between,
    so that CTA 0 walks at least 3 x stages tiles over several items (with a chunk that
    keeps a 60000-B leaf in one item: 64 KiB and up)."""
    (_, tma_cps, stages, _), (shift_cps, shift_stages, shift_tile) = _launch(shape)
    specs = [(32, 0)] * ((3 * stages - 1) * sms * tma_cps + 1)
    if shift:
        per_big = -(-(60_000 - 16) // shift_tile)
        for j in range(max(2, -(-3 * shift_stages // per_big))):
            if j:
                specs += [(4096, 3)] * (sms * shift_cps - 1)
            specs.append((60_000, 3))
    return specs


def _busiest(table, ctas, tile, shifted=False):
    """Tiles of the CTA that walks the most, counting only CTAs that own >= 2 items."""
    return max([t for t, n in pm.cta_load(table, ctas, tile, shifted) if n >= 2], default=0)


def _device_bytes(ptr, n):
    class _A:
        __cuda_array_interface__ = {"shape": (int(n),), "typestr": "|u1",
                                    "data": (int(ptr), False), "version": 2}

    return torch.as_tensor(_A(), device="cuda")


# ------------------------------------------------------------------ CPU: the model --


def test_model_first_item_ends_on_a_128_byte_boundary():
    its = pm.items([pm.Range(tptr=1 << 20, aoff=100, n=10_000)], 4096)
    assert [(i.aoff, i.n, i.index) for i in its] == [(100, 3996, 0), (4096, 4096, 1),
                                                     (8192, 1908, 2)]
    assert [i.tptr for i in its] == [1 << 20, (1 << 20) + 3996, (1 << 20) + 8092]
    # a range that starts on the boundary, and one shorter than its first piece
    assert [i.n for i in pm.items([pm.Range(0, 8192, 4097)], 4096)] == [4096, 1]
    assert [i.n for i in pm.items([pm.Range(0, 130, 50)], 4096)] == [50]
    assert pm.items([pm.Range(0, 0, 0)], 4096) == []


def test_model_items_sort_by_arena_offset_and_skip_empty_ranges():
    its = pm.items([pm.Range(0x9000, 5000, 10), pm.Range(0x8000, 77, 0),
                    pm.Range(0x7000, 0, 5000)], 4096)
    assert [(i.tptr, i.aoff, i.n, i.index) for i in its] == [
        (0x7000, 0, 4096, 0), (0x7000 + 4096, 4096, 904, 1), (0x9000, 5000, 10, 2)]


def test_model_congruent_item_splits_into_head_body_tail():
    # source and arena offset both 3 mod 16: a 13-B head, one 16-B word, an 11-B tail
    its = pm.items([pm.Range(tptr=0x1003, aoff=3, n=40)], 4096)
    t = pm.tables(its)
    assert [(i.tptr, i.aoff, i.n) for i in t["resid"]] == [(0x1003, 3, 13), (0x1020, 32, 11)]
    assert [(i.tptr, i.aoff, i.n) for i in t["bulk"]] == [(0x1010, 16, 16)]
    assert t["shift"] == [] and {i.index for i in t["resid"] + t["bulk"]} == {0}
    # aligned on both ends: body only; shorter than the head: head only
    t = pm.tables(pm.items([pm.Range(0x2000, 32, 64)], 4096))
    assert (len(t["resid"]), [i.n for i in t["bulk"]]) == (0, [64])
    t = pm.tables(pm.items([pm.Range(0x2005, 5, 7)], 4096))
    assert ([i.n for i in t["resid"]], t["bulk"]) == ([7], [])


def test_model_shifted_items_under_4096_bytes_take_the_lsu_kernel():
    # source 3 mod 16, arena offset 0 mod 16
    t = pm.tables(pm.items([pm.Range(0x3003, 0, 4095)], 4096))
    assert ([i.n for i in t["resid"]], t["shift"], t["bulk"]) == ([4095], [], [])
    t = pm.tables(pm.items([pm.Range(0x3003, 0, 4096)], 4096))
    assert (t["resid"], [i.n for i in t["shift"]], t["bulk"]) == ([], [4096], [])
    # 9000 B from arena offset 64: 4032 (resid) + 4096 (shift) + 872 (resid)
    t = pm.tables(pm.items([pm.Range(0x3003, 64, 9000)], 4096))
    assert [i.n for i in t["resid"]] == [4032, 872] and [i.n for i in t["shift"]] == [4096]


def test_model_tied_leaves_are_two_items_of_one_source():
    src = 0x10_0000
    its = pm.items([pm.Range(src, 0, 6000), pm.Range(src, 6000 + 5, 6000)], 4096)
    assert [(i.tptr, i.aoff, i.n) for i in its] == [
        (src, 0, 4096), (src + 4096, 4096, 1904),
        (src, 6005, 3979), (src + 3979, 9984, 2021)]  # 6005 % 128 == 117
    t = pm.tables(its)
    # the first copy is congruent (bulk), the second is shifted by 11 mod 16
    assert [i.index for i in t["bulk"]] == [0, 1]
    assert [i.index for i in t["shift"]] == [] and [i.index for i in t["resid"]] == [2, 3]
    # one changed source byte dirties an item of each copy
    old = np.zeros(12_100, np.uint8)
    new = old.copy()
    new[[5000, 6005 + 5000]] = 1
    d = pm.dirty(its, old, new)
    assert [i.index for i in d] == [1, 3] and pm.drained_bytes(d) == 1904 + 2021


def test_model_mapped_runs_merge_only_where_the_segment_continues():
    rs = [pm.Range(0xA000, 0, 100, hoff=0), pm.Range(0xB000, 100, 50, hoff=1000),
          pm.Range(0xC000, 150, 10, hoff=1050), pm.Range(0xD000, 160, 30, hoff=2000),
          pm.Range(0xE000, 200, 8, hoff=2030)]
    # the arena continues at 100, 150 and 160; the segment only at 1050
    assert [(r.aoff, r.n, r.hoff) for r in pm.runs(rs)] == [
        (0, 100, 0), (100, 60, 1000), (160, 30, 2000), (200, 8, 2030)]
    # identity: everything adjacent merges, in arena order whatever the input order
    rs = [pm.Range(0, 40, 8), pm.Range(0, 0, 40), pm.Range(0, 49, 3)]
    assert [(r.aoff, r.n, r.hoff) for r in pm.runs(rs)] == [(0, 48, 0), (49, 3, 49)]
    # dirty items merge the same way: item 1 and 2 are adjacent in the arena only
    its = pm.items([pm.Range(0xA000, 0, 4096, hoff=8192), pm.Range(0xB000, 4096, 4096, 0),
                    pm.Range(0xC000, 8192, 4096, hoff=4096)], 4096)
    assert [(r.aoff, r.n, r.hoff) for r in pm.runs(its)] == [
        (0, 4096, 8192), (4096, 8192, 0)]


def test_model_cta_load_follows_the_grid_rule():
    t = [pm.Item(0, 0, 100, 0), pm.Item(0, 128, 16, 128), pm.Item(0, 256, 300, 256)]
    # two CTAs: CTA 0 takes items 0 and 2 (2 + 5 tiles of 64 B), CTA 1 item 1
    assert pm.cta_load(t, 2, 64) == [(7, 2), (1, 1)]
    assert pm.cta_load(t, 8, 64) == [(2, 1), (1, 1), (5, 1)]  # grid = 3 items
    # byte-shift pack: 13 bytes bring arena offset 3 to 16-B alignment, 80 B of words
    assert pm.cta_load([pm.Item(0, 3, 100, 3)], 1, 64, shifted=True) == [(2, 1)]
    assert pm.cta_load([], 4, 64) == []


def test_model_dma_and_kernel_counts():
    rs = [pm.Item(0, 0, 100, 0), pm.Item(0, 200, 64, 200), pm.Item(0, 300, 65, 300)]
    assert pm.dma_count(rs, 64) == 2 + 1 + 2
    assert pm.dma_count([], 64) == 0
    t = pm.tables(pm.items([pm.Range(0x1003, 3, 40)], 4096))
    assert pm.kernel_count(t, pm.TMA) == 2 and pm.kernel_count(t, pm.LSU) == 1
    t = pm.tables(pm.items([pm.Range(0x3003, 0, 9000)], 4096))
    assert pm.kernel_count(t, pm.TMA) == 2  # shift + resid, no bulk
    empty = pm.tables([])
    assert pm.kernel_count(empty, pm.TMA) == 0 and pm.kernel_count(empty, pm.LSU) == 0


# ------------------------------------------------------------------------ layouts --


class Buf:
    """A device buffer and the model's copy of what it must hold."""

    def __init__(self, init: np.ndarray):
        self.np = init.copy()
        self.dev = torch.from_numpy(init).cuda()
        self.base = self.dev.data_ptr()

    def read(self, tptr, n):
        i = tptr - self.base
        return self.np[i:i + n]

    def write(self, tptr, data):
        i = tptr - self.base
        self.np[i:i + len(data)] = data
        self.dev[i:i + len(data)].copy_(torch.from_numpy(np.ascontiguousarray(data)))

    def check(self, what):
        got = self.dev.cpu().numpy()
        bad = np.flatnonzero(got != self.np)
        assert bad.size == 0, f"{what}: {bad.size} bytes differ, first at {bad[:8]}"


class Leaf:
    def __init__(self, n, aoff, s, t, hoff=None):
        self.n, self.aoff, self.s, self.t = n, aoff, s, t
        self.hoff = aoff if hoff is None else hoff


class Layout:
    """Leaves over one source buffer and, for unpack / restore, the same leaves (tied
    copies excepted) over one target buffer that holds the canary everywhere else."""

    def __init__(self, leaves, src: Buf, tgt: Buf, mapped):
        self.leaves, self.src, self.tgt, self.mapped = leaves, src, tgt, mapped

    def ranges(self, which, moved=None):
        """Model ranges of the source plan ("P") or the target plan ("Q"); moved maps a
        leaf index to the arena offset it was moved to."""
        out = []
        for k, lf in enumerate(self.leaves):
            if which == "Q" and lf.t is None:
                continue
            buf = self.src if which == "P" else self.tgt
            pos = lf.s if which == "P" else lf.t
            aoff = (moved or {}).get(k, lf.aoff)
            out.append(pm.Range(buf.base + pos, aoff, lf.n, lf.hoff if self.mapped else aoff))
        return out

    @property
    def arena_end(self):
        return max(lf.aoff + lf.n for lf in self.leaves)

    @property
    def host_end(self):
        return max(lf.hoff + lf.n for lf in self.leaves)


def mixed_layout(seed, tiles=(), chunk=4096, target=12 << 20, aoff0=0, mapped=False, ring=()):
    """`ring` (see ring_section) back to back from aoff0, then leaves of the lengths
    where kernels go wrong, each with its own (source - arena) class mod 16; every
    non-zero class once more as a 100-B (LSU) and a 9000-B (shift kernel) leaf;
    zero-length leaves in between; one tied pair; filler leaves, alternately congruent
    and shifted, up to `target`."""
    rng = np.random.default_rng(seed)
    lens = [*range(1, 18), 31, 32, 33, 127, 128, 129, 4095, 4096, 4097,
            chunk - 1, chunk, chunk + 1]
    lens += [k * t + d for t in tiles for k in (1, 3) for d in (0, 1, -1, 15, -15, 16, -16,
                                                                  17, -17)]
    specs = [(n, int(rng.integers(0, 16))) for n in lens if n > 0]
    specs += [(n, d) for d in range(1, 16) for n in (100, 9000)]
    filler = 0
    while sum(n for n, _ in specs) + sum(n for n, _ in ring) < target:
        specs.append((int(rng.integers(1 << 18, 1 << 20)) | 1,
                      0 if filler % 2 == 0 else int(rng.integers(1, 16))))
        filler += 1
    order = rng.permutation(len(specs))
    specs = [specs[i] for i in order]
    for i in range(0, len(specs) + 1, 7):  # interleaved empty leaves
        specs.insert(i, (0, int(rng.integers(0, 16))))
    gaps = [GAPS[i % len(GAPS)] for i in rng.permutation(len(specs) + 1)]
    assert not ring or aoff0 % 16 == 0
    gaps = [0] * len(ring) + gaps
    holes = [0] * len(ring) + [(0, 0, 1, 16, 100, 4096)[int(rng.integers(0, 6))]
                               for _ in specs]
    specs = list(ring) + specs

    total = sum(n for n, _ in specs)
    src = Buf(rng.integers(0, 256, total + 16 * len(specs) + 2 * GUARD, dtype=np.uint8))
    tgt = Buf(pattern(total + 160 * len(specs) + 2 * GUARD))
    leaves, a, s, t, h = [], aoff0, GUARD, GUARD, 64
    for k, (n, d) in enumerate(specs):
        a += gaps[k]
        s += (a + d - (src.base + s)) % 16
        t += gaps[k]
        t += (a + d - (tgt.base + t)) % 16
        hole = holes[k]
        leaves.append(Leaf(n, a, s, t, h + hole if mapped else None))
        h += hole + n
        a, s, t = a + n, s + n, t + n
    # the tied pair: a second range over the bytes of a 9000-B leaf, at the end of the plan
    first = next(lf for lf in leaves if lf.n == 9000)
    a += gaps[-1] + 5
    leaves.append(Leaf(first.n, a, first.s, None, h + 3 if mapped else None))
    assert t + GUARD <= tgt.np.size and s + GUARD <= src.np.size
    return Layout(leaves, src, tgt, mapped)


def state_dict_layout(seed):
    """The layout oracle.plan_layout gives a mixed-dtype state dict with 4-byte step
    scalars, its tensors at 512-B aligned addresses as separate allocations are."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i in range(5):
        sd[f"w{i}"] = torch.randn(701 + i, 1029, generator=g).to(torch.bfloat16)
        sd[f"step{i}"] = torch.tensor(float(i + 1))
        sd[f"exp_avg{i}"] = torch.randn(123_457 + 3 * i, generator=g)
        sd[f"idx{i}"] = torch.randint(0, 1 << 40, (4099 + i,), generator=g)
        sd[f"u8_{i}"] = torch.randint(0, 256, (77_777 + i,), dtype=torch.uint8, generator=g)
        sd[f"mask{i}"] = torch.rand(33_335 + i, generator=g) > 0.5
        sd[f"f8_{i}"] = torch.randn(65_537 + i, generator=g).to(torch.float8_e4m3fn)
    meta, _ = oracle.plan_layout(sd)
    metas = oracle.flatten_tensor_metas(meta)
    raw = [oracle.tensor_bytes(t) for t in sd.values()]
    room = sum((b.size + 511) // 512 * 512 for b in raw) + 2 * GUARD + 512
    src_np = np.random.default_rng(seed).integers(0, 256, room, dtype=np.uint8)
    src = Buf(src_np)
    tgt = Buf(pattern(room))
    leaves, s = [], 512
    for m, b in zip(metas, raw):
        src.write(src.base + s, b)
        leaves.append(Leaf(b.size, m.offset, s, s))
        s += (b.size + 511) // 512 * 512
    assert len({lf.aoff % 16 for lf in leaves}) >= 4
    return Layout(leaves, src, tgt, mapped=False)


# ------------------------------------------------------------------------- the world --


def _copies(ranges):
    """The ranges merged where both the arena and the device buffer continue (the
    model moves each such piece with one slice)."""
    return pm.runs([pm.Range(r.tptr, r.aoff, r.n, hoff=r.tptr) for r in ranges])


class World:
    """One context, a source plan P and a target plan Q over a layout, two pinned host
    buffers A and B, and the model of every byte of the arena, the host buffers and the
    two device buffers.  Each operation runs on the device and in the model."""

    def __init__(self, ctx, layout, chunk, variant, piece=16 << 20, arena_lo=0,
                 spare=0, bounded=False):
        self.ctx, self.lay, self.chunk, self.variant, self.piece = ctx, layout, chunk, variant, piece
        self.model_chunk = chunk or DEFAULT_CHUNK
        self.moved = {}
        self.arena_lo = arena_lo
        self.room = layout.arena_end + spare + GUARD
        ctx.arena_reserve(self.room)
        self.bounded = bounded
        if bounded:
            self.arena = None  # windows reuse the arena: its bytes are not modelled
        else:
            self.arena = pattern(self.room - arena_lo, arena_lo)
            ctx.arena_tensor(self.room)[arena_lo:].copy_(torch.from_numpy(self.arena))
        # a mapped plan's host buffer reaches an arena span past its last range, so that
        # even a wrongly merged DMA run stays inside it
        hsize = (layout.host_end + self.room - arena_lo if layout.mapped else self.room) + GUARD
        self.host_t, self.host = {}, {}
        for name in ("A", "B"):
            self.host[name] = pattern(hsize)
            self.host_t[name] = torch.from_numpy(self.host[name]).pin_memory()
        self.base = None
        self.plans = {}
        try:
            for name in ("P", "Q"):
                self._make(name)
        except BaseException:
            self.close()
            raise
        torch.cuda.synchronize()

    # -- plans -----------------------------------------------------------------------
    def _make(self, name):
        rs = self.lay.ranges(name, self.moved if name == "P" else None)
        hoffs = [r.hoff for r in rs] if self.lay.mapped else None
        plan = self.ctx.plan([r.tptr for r in rs], [r.aoff for r in rs], [r.n for r in rs],
                             self.chunk, host_offsets=hoffs)
        self.plans[name] = dict(plan=plan)  # destroyed by close() whatever follows
        its = pm.items(rs, self.model_chunk)
        assert plan.n_items == len(its)
        assert plan.payload_bytes == sum(r.n for r in rs)
        runs = pm.runs(rs)
        assert plan.n_runs == len(runs)
        self.plans[name].update(ranges=rs, items=its, tables=pm.tables(its), runs=runs,
                                copies=_copies(rs))

    def buf(self, name):
        return self.lay.src if name == "P" else self.lay.tgt

    def _kernels(self, name):
        return pm.kernel_count(self.plans[name]["tables"], self.variant)

    def _gathered(self, name):
        """The arena image after plan `name` gathered its sources."""
        new = self.arena.copy()
        for r in self.plans[name]["copies"]:
            new[r.aoff - self.arena_lo:r.aoff - self.arena_lo + r.n] = self.buf(name).read(r.tptr, r.n)
        return new

    def _drain(self, run_list, host):
        lo = self.arena_lo
        for r in run_list:
            self.host[host][r.hoff:r.hoff + r.n] = self.arena[r.aoff - lo:r.aoff - lo + r.n]

    def _forget(self):
        self.base = None

    # -- operations --------------------------------------------------------------------
    def pack(self, name="P"):
        k0, _ = self.ctx.launch_count()
        self.plans[name]["plan"].pack()
        torch.cuda.synchronize()
        assert self.ctx.launch_count()[0] - k0 == self._kernels(name)
        self.arena = self._gathered(name)
        self._forget()

    def unpack(self, name="Q"):
        k0, _ = self.ctx.launch_count()
        self.plans[name]["plan"].unpack()
        torch.cuda.synchronize()
        assert self.ctx.launch_count()[0] - k0 == self._kernels(name)
        self._scatter(name)
        self._forget()

    def _scatter(self, name):
        b, lo = self.buf(name), self.arena_lo
        for r in self.plans[name]["copies"]:
            b.np[r.tptr - b.base:r.tptr - b.base + r.n] = self.arena[r.aoff - lo:r.aoff - lo + r.n]

    def save(self, name="P", host="A"):
        p = self.plans[name]
        k0, m0 = self.ctx.launch_count()
        self.ctx.save_wait(p["plan"].save_async(self.host_t[host].data_ptr(),
                                                torch.cuda.current_stream()))
        k1, m1 = self.ctx.launch_count()
        if self.bounded:  # the save streams window after window; only the segment counts
            for r in p["ranges"]:
                self.host[host][r.hoff:r.hoff + r.n] = self.buf(name).read(r.tptr, r.n)
        else:
            assert k1 - k0 == self._kernels(name)
            assert m1 - m0 == pm.dma_count(p["runs"], self.piece)
            self.arena = self._gathered(name)
            self._drain(p["runs"], host)
        self._forget()

    def save_direct(self, name="P", host="A"):
        p = self.plans[name]
        self.ctx.save_wait(p["plan"].save_direct_async(self.host_t[host].data_ptr(),
                                                       torch.cuda.current_stream()))
        for r in p["ranges"]:
            self.host[host][r.hoff:r.hoff + r.n] = self.buf(name).read(r.tptr, r.n)
        self._forget()

    def save_hybrid(self, name="P", host="A"):
        """Ranges from a tensor boundary in the middle on are snapshotted into the arena,
        whose byte 0 then stands for that boundary rounded down to 128 B."""
        p = self.plans[name]
        starts = sorted(r.aoff for r in p["ranges"] if r.n)
        cut = starts[len(starts) // 2]
        abase = cut & ~127
        self.ctx.save_wait(p["plan"].save_hybrid_async(self.host_t[host].data_ptr(), cut,
                                                       torch.cuda.current_stream()))
        for r in p["ranges"]:
            data = self.buf(name).read(r.tptr, r.n)
            self.host[host][r.hoff:r.hoff + r.n] = data
            if r.aoff >= cut:
                self.arena[r.aoff - abase:r.aoff - abase + r.n] = data
        self._forget()

    def restore(self, name="Q", host="A", source="segment", src=None):
        """Restore plan `name` from the bytes host buffer `host` holds, read from
        `source`: "segment" (at address `src`, the buffer itself when None), "direct"
        (the same, straight into the tensors), "file" (the open descriptor `src`) or
        "image" (the arena image of the last save).  Returns the DMA copies it issued."""
        p = self.plans[name]
        plan, stream = p["plan"], torch.cuda.current_stream()
        addr = self.host_t[host].data_ptr() if src is None else src
        _, m0 = self.ctx.launch_count()
        if source == "file":
            plan.restore_file_async(src, stream)
        elif source == "image":
            assert plan.restore_from_image_async(addr, stream)
        else:
            plan.restore_async(addr, stream, direct=source == "direct")
        self.ctx.restore_wait()
        torch.cuda.synchronize()
        _, m1 = self.ctx.launch_count()
        if self.bounded or source == "direct":
            b = self.buf(name)
            for r in p["ranges"]:
                b.np[r.tptr - b.base:r.tptr - b.base + r.n] = self.host[host][r.hoff:r.hoff + r.n]
        else:
            lo = self.arena_lo
            if source != "image":
                for r in p["runs"]:
                    self.arena[r.aoff - lo:r.aoff - lo + r.n] = self.host[host][r.hoff:r.hoff + r.n]
            self._scatter(name)
        if source != "image":  # a rollback keeps the baseline
            self._forget()
        return m1 - m0

    def arena_fill(self, host="A"):
        hi = self.lay.arena_end
        self.ctx.arena_fill(self.host_t[host].data_ptr(), 0, hi, torch.cuda.current_stream())
        torch.cuda.synchronize()
        self.arena[:hi] = self.host[host][:hi]
        self._forget()

    def delta(self, name="P", host="A", hold=False):
        """An incremental save, checked against the model: whether it compared, the bytes
        and DMA copies it drained, the kernels it launched."""
        p = self.plans[name]
        is_delta = self.base == (name, host)
        new = self._gathered(name)
        if is_delta:
            d = pm.dirty(p["items"], self.arena, new, self.arena_lo)
            run_list, nbytes = pm.runs(d), pm.drained_bytes(d)
        else:
            run_list, nbytes = p["runs"], sum(r.n for r in p["ranges"])
        k0, m0 = self.ctx.launch_count()
        ticket = p["plan"].save_delta_async(self.host_t[host].data_ptr(),
                                            torch.cuda.current_stream(), hold=hold)
        self.arena = new
        if hold:  # cancelled before the drain: the gather ran, the segment is untouched
            torch.cuda.synchronize()
            assert self.ctx.save_cancel(ticket)
            self.ctx.save_wait(ticket)
            self._forget()
            return
        self.ctx.save_wait(ticket)
        k1, m1 = self.ctx.launch_count()
        assert self.ctx.save_delta_stats(ticket) == (is_delta, nbytes)
        assert m1 - m0 == pm.dma_count(run_list, self.piece)
        assert k1 - k0 == self._kernels(name)
        self._drain(run_list, host)
        self.base = (name, host)

    def update(self, moved):
        """Re-target P; moving a range forgets the baseline of P, keeping every extent
        keeps it."""
        old = [(r.aoff, r.n, r.hoff) for r in self.plans["P"]["ranges"]]
        self.moved = moved
        rs = self.lay.ranges("P", moved)
        hoffs = [r.hoff for r in rs] if self.lay.mapped else None
        p = self.plans["P"]
        p["plan"].update([r.tptr for r in rs], [r.aoff for r in rs], [r.n for r in rs],
                         torch.cuda.current_stream(), host_offsets=hoffs)
        p["ranges"], p["runs"], p["copies"] = rs, pm.runs(rs), _copies(rs)
        p["items"] = pm.items(rs, self.model_chunk)
        p["tables"] = pm.tables(p["items"])
        if old != [(r.aoff, r.n, r.hoff) for r in rs] and self.base and self.base[0] == "P":
            self._forget()

    def recreate(self):
        self.plans["P"]["plan"].destroy()
        if self.base and self.base[0] == "P":
            self._forget()
        self._make("P")

    # -- the check -----------------------------------------------------------------------
    def check(self, what=""):
        torch.cuda.synchronize()
        if self.arena is not None:
            ptr, size = self.ctx.arena_info()
            assert size == self.room
            got = _device_bytes(ptr + self.arena_lo, self.room - self.arena_lo).cpu().numpy()
            bad = np.flatnonzero(got != self.arena)
            assert bad.size == 0, f"{what}: arena differs at {bad[:8] + self.arena_lo}"
        for name in ("A", "B"):
            bad = np.flatnonzero(self.host_t[name].numpy() != self.host[name])
            assert bad.size == 0, f"{what}: host {name} differs at {bad[:8]}"
        self.lay.src.check(f"{what}: sources")
        self.lay.tgt.check(f"{what}: targets")

    def close(self):
        """Destroy the plans (before their context: a plan's handle points into it)."""
        for p in self.plans.values():
            p["plan"].destroy()


@contextlib.contextmanager
def _world(ctx, *args, **kw):
    """A World on `ctx`; its plans and then `ctx` are destroyed whatever happens."""
    w = None
    try:
        w = World(ctx, *args, **kw)
        yield w
    finally:
        if w is not None:
            w.close()
        ctx.destroy()


# -------------------------------------------------------------------- the matrix --


def _coverage(tables):
    """(tables that hold items, (src - dst) % 16 classes of shift, of resid)."""
    cls = {k: {(i.tptr - i.aoff) % 16 for i in v} for k, v in tables.items()}
    return {k for k, v in tables.items() if v}, cls["shift"], cls["resid"]


@gpu
@pytest.mark.parametrize("variant", VARIANTS, ids=["lsu", "tma"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_copy_kernels_write_exactly_the_covered_bytes(cuda_device, shape, variant):
    """pack, unpack, save + restore and a bounded-arena save + restore, for every chunk,
    on the mixed layout and on a state-dict layout."""
    sms = _sms()
    (_, tma_cps, stages, tile), (shift_cps, shift_stages, shift_tile) = _launch(shape)
    ring = ring_section(shape, sms)
    cases = [(chunk, mixed_layout(1, _tiles(shape), chunk or DEFAULT_CHUNK, ring=ring))
             for chunk in CHUNKS]
    cases.append((0, state_dict_layout(2)))
    seen = [set(), set(), set()]
    ring_tiles = [0, 0]
    for chunk, lay in cases:
        with _world(_context(shape, variant), lay, chunk, variant) as w:
            t = w.plans["P"]["tables"]
            for k, got in enumerate(_coverage(t)):
                seen[k] |= got
            ring_tiles[0] = max(ring_tiles[0], _busiest(t["bulk"], sms * tma_cps, tile))
            ring_tiles[1] = max(ring_tiles[1], _busiest(t["shift"], sms * shift_cps,
                                                        shift_tile, shifted=True))
            w.pack()
            w.check(f"pack chunk={chunk}")
            w.unpack()
            w.check(f"unpack chunk={chunk}")
            w.save()
            w.check(f"save chunk={chunk}")
            w.lay.tgt.write(w.lay.tgt.base, pattern(w.lay.tgt.np.size))
            w.restore()
            w.check(f"restore chunk={chunk}")
        # the same plan streamed through an 8 MiB arena (launch_slice with a base > 0)
        lay.tgt.write(lay.tgt.base, pattern(lay.tgt.np.size))
        with _world(_context(shape, variant, 8 << 20), lay, chunk, variant,
                    bounded=True) as w:
            assert w.ctx.arena_info()[1] == 8 << 20 < lay.arena_end
            w.save()
            w.check(f"bounded save chunk={chunk}")
            w.restore()
            w.check(f"bounded restore chunk={chunk}")
    assert seen[0] == {"bulk", "resid", "shift"}
    assert seen[1] == set(range(1, 16)) and seen[2] == set(range(16))
    # the copy ring and the byte-shift ring each wrap three times on a CTA that crosses
    # from item to item (the bulk tiles at chunk 4096, the shift tiles at 64 KiB and up)
    assert ring_tiles[0] >= 3 * stages and ring_tiles[1] >= 3 * shift_stages, ring_tiles


@contextlib.contextmanager
def _plain_mapping(data):
    """The bytes of `data` in an anonymous mapping: pageable memory CUDA knows nothing of."""
    mm = mmap.mmap(-1, data.size)
    view = np.frombuffer(mm, dtype=np.uint8)
    view[:] = data
    anchor = ctypes.c_char.from_buffer(mm)
    try:
        yield ctypes.addressof(anchor)
    finally:
        del view, anchor
        mm.close()


@gpu
@pytest.mark.parametrize("variant", VARIANTS, ids=["lsu", "tma"])
@pytest.mark.parametrize("layout", ["state_dict", "mixed"])
def test_every_restore_source_writes_exactly_the_target_bytes(cuda_device, tmp_path, layout,
                                                              variant):
    """Restores of one saved checkpoint from every source: the pinned segment, a plain
    mapping (bounce slots), a mapping registered slice by slice, in place, a file and the
    arena image; into the full arena and, where the source allows it, through an 8 MiB
    one."""
    lay = (state_dict_layout(9) if layout == "state_dict"
           else mixed_layout(9, _tiles("default"), DEFAULT_CHUNK))
    for bounded in (False, True):
        lay.tgt.write(lay.tgt.base, pattern(lay.tgt.np.size))
        ctx = _context("default", variant, 8 << 20 if bounded else 0)
        ctx.set_stage(3, 1 << 20)
        with _world(ctx, lay, 0, variant, bounded=bounded) as w:
            assert (ctx.arena_info()[1] < lay.arena_end) == bounded
            w.save()
            w.check(f"save bounded={bounded}")
            q, host = w.plans["Q"], w.host["A"]

            def restore(source, src=None):
                lay.tgt.write(lay.tgt.base, pattern(lay.tgt.np.size))
                copies = w.restore(source=source, src=src)
                w.check(f"{source} restore at {src} bounded={bounded}")
                return copies

            if not bounded:  # first: every other restore forgets the image
                assert restore("image") == 0
            copies = restore("segment")
            if not bounded:
                assert copies == pm.dma_count(q["runs"], 256 << 20)
            assert restore("direct") >= q["plan"].n_spans
            with _plain_mapping(host) as addr:
                restore("segment", addr)
                ctx.host_register_background(addr, host.size, slice_bytes=2 << 20)
                deadline = time.time() + 60
                while not ctx.host_ready(addr):
                    assert time.time() < deadline
                    time.sleep(0.01)
                restore("segment", addr)
                ctx.host_unregister(addr)
            path = tmp_path / f"segment_{bounded}.bin"
            path.write_bytes(host.tobytes())
            fd = os.open(path, os.O_RDONLY)
            try:
                restore("file", fd)
            finally:
                os.close(fd)


def _window_dma_counts(items, run_list, arena_bytes, piece):
    """DMA copies of each window of a bounded-arena save: a window takes the items from
    the first one left on while they end within arena_bytes of its start rounded down to
    128 B, and drains the runs clipped to the bytes it covers."""
    counts, i = [], 0
    while i < len(items):
        base = end = items[i].aoff
        abase, j = base & ~127, i
        while j < len(items) and items[j].aoff + items[j].n - abase <= arena_bytes:
            end = max(end, items[j].aoff + items[j].n)
            j += 1
        assert j > i
        counts.append(sum(-(-(min(end, r.aoff + r.n) - max(base, r.aoff)) // piece)
                          for r in run_list if max(base, r.aoff) < min(end, r.aoff + r.n)))
        i = j
    return counts


def _save_forms(w, addr, seg, model, pinned, bounded, rng):
    """Every save form of plan P into the host range at `addr` (its bytes `seg`, their
    model `model`), each from a canary segment except the incremental save, which
    follows the full one.  Checks every host, arena and source byte after each form,
    and the DMA copies where the host range is pinned."""
    ctx, p, stream = w.ctx, w.plans["P"], torch.cuda.current_stream()
    plan, src = p["plan"], w.lay.src
    ranges = [r for r in p["ranges"] if r.n]

    def fresh():
        seg[:] = model[:] = pattern(model.size)

    def saved(rs=ranges):
        for r in rs:
            model[r.hoff:r.hoff + r.n] = src.read(r.tptr, r.n)

    def check(form, copies, expected):
        torch.cuda.synchronize()
        if pinned:
            assert copies == expected, f"{form}: {copies} DMA copies, the model says {expected}"
        bad = np.flatnonzero(seg != model)
        assert bad.size == 0, f"{form}: segment differs at {bad[:8]}"
        w.check(form)

    def run(form, call):
        _, m0 = ctx.launch_count()
        call()
        return ctx.launch_count()[1] - m0

    if bounded:
        fresh()
        copies = run("bounded", lambda: ctx.save_wait(plan.save_async(addr, stream)))
        saved()
        counts = _window_dma_counts(p["items"], p["runs"], ctx.arena_info()[1], w.piece)
        assert len(counts) > 1
        check("bounded save", copies, sum(counts))
        return

    fresh()
    copies = run("save", lambda: ctx.save_wait(plan.save_async(addr, stream)))
    w.arena = w._gathered("P")
    saved()
    check("save", copies, pm.dma_count(p["runs"], w.piece))

    for release in (True, False):
        fresh()

        def held():
            ticket = plan.save_async(addr, stream, hold=True)
            torch.cuda.synchronize()
            if release:
                ctx.save_release(ticket)
            else:
                assert ctx.save_cancel(ticket)
            ctx.save_wait(ticket)

        copies = run("held", held)
        w.arena = w._gathered("P")
        if release:
            saved()
        check(f"held save, release={release}", copies,
              pm.dma_count(p["runs"], w.piece) if release else 0)

    fresh()
    copies = run("direct", lambda: ctx.save_wait(plan.save_direct_async(addr, stream)))
    saved()
    check("in-place save", copies, pm.dma_count(ranges, w.piece))

    starts = sorted(r.aoff for r in ranges)
    for cut in (starts[len(starts) // 3], starts[2 * len(starts) // 3]):
        fresh()
        copies = run("hybrid",
                     lambda: ctx.save_wait(plan.save_hybrid_async(addr, cut, stream)))
        abase = cut & ~127
        for r in ranges:
            if r.aoff >= cut:
                w.arena[r.aoff - abase:r.aoff - abase + r.n] = src.read(r.tptr, r.n)
        saved()
        head = [r for r in ranges if r.hoff < cut]
        tail = pm.runs([r for r in ranges if r.aoff >= cut])
        check(f"hybrid save at {cut}", copies,
              pm.dma_count(head, w.piece) + pm.dma_count(tail, w.piece))

    fresh()
    ticket = [0]

    def delta():
        ticket[0] = plan.save_delta_async(addr, stream)
        ctx.save_wait(ticket[0])

    copies = run("delta", delta)
    w.arena = w._gathered("P")
    saved()
    assert ctx.save_delta_stats(ticket[0]) == (False, sum(r.n for r in ranges))
    check("full incremental save", copies, pm.dma_count(p["runs"], w.piece))
    for kind in ("leaf", "span", "byte"):
        _change(w, rng, kind)
    new = w._gathered("P")
    d = pm.dirty(p["items"], w.arena, new, w.arena_lo)
    assert d
    copies = run("delta", delta)
    w.arena = new
    saved()
    assert ctx.save_delta_stats(ticket[0]) == (True, pm.drained_bytes(d))
    check("incremental save", copies, pm.dma_count(pm.runs(d), w.piece))


@gpu
@pytest.mark.parametrize("mode", [native.DRAIN_HOST_PACED, native.DRAIN_PINGPONG],
                         ids=["host_paced", "pingpong"])
@pytest.mark.parametrize("variant", VARIANTS, ids=["lsu", "tma"])
@pytest.mark.parametrize("layout", ["state_dict", "mixed"])
def test_every_save_form_writes_exactly_the_segment_bytes(cuda_device, layout, variant, mode):
    """Every save form (full, held and released, held and cancelled, in place, hybrid at
    two cuts, incremental full and then incremental, and through an 8 MiB arena) into
    the pinned segment, a plain mapping (bounce slots) and a mapping registered slice by
    slice, in 64-KiB drain pieces."""
    rng = np.random.default_rng(11 + variant * 2 + mode)
    lay = (state_dict_layout(10) if layout == "state_dict"
           else mixed_layout(10, _tiles("default"), DEFAULT_CHUNK))
    piece = 64 << 10
    for bounded in (False, True):
        ctx = _context("default", variant, 8 << 20 if bounded else 0)
        ctx.set_stage(3, 1 << 20)
        ctx.set_drain_mode(mode)
        ctx.set_drain(piece)
        with _world(ctx, lay, 0, variant, piece=piece, bounded=bounded) as w:
            assert (ctx.arena_info()[1] < lay.arena_end) == bounded
            a = w.host_t["A"]
            _save_forms(w, a.data_ptr(), a.numpy(), w.host["A"], True, bounded, rng)
            model = pattern(w.host["A"].size)
            with _plain_mapping(model) as addr:
                seg = np.ctypeslib.as_array((ctypes.c_uint8 * model.size).from_address(addr))
                _save_forms(w, addr, seg, model, False, bounded, rng)
                ctx.host_register_background(addr, model.size, slice_bytes=2 << 20)
                deadline = time.time() + 60
                while not ctx.host_ready(addr):
                    assert time.time() < deadline
                    time.sleep(0.01)
                _save_forms(w, addr, seg, model, False, bounded, rng)
                ctx.host_unregister(addr)
                del seg


@gpu
def test_a_refused_save_keeps_the_baseline_and_the_image(cuda_device):
    """A save refused for its arguments (a hybrid cut inside a tensor) touches neither
    the incremental baseline nor the arena image: the next incremental save compares
    and drains nothing."""
    ctx = _context("default", native.VARIANT_TMA)
    with _world(ctx, _small_layout(5, "default"), 4096, native.VARIANT_TMA) as w:
        w.delta()
        w.check("full incremental save")
        p, addr = w.plans["P"], w.host_t["A"].data_ptr()
        inside = next(r for r in p["ranges"] if r.n > 1).aoff + 1
        for hold in (False, True):
            with pytest.raises(native.NativeError) as e:
                p["plan"].save_hybrid_async(addr, inside, torch.cuda.current_stream(), hold)
            assert e.value.code == native.FC_EINVAL
        assert p["plan"].image_covers(addr)
        w.delta()  # asserts (incremental, 0 bytes drained)
        w.check("incremental save after the refusals")


# --------------------------------------------------------- exact incremental accounting --

OPS = ("pack", "unpack", "arena_fill", "save", "save_direct", "save_hybrid", "restore",
       "arena_tensor", "invalidate", "cancel_held", "update_same", "update_moved",
       "recreate", "delta_other_plan", "delta_other_host")
CHANGES = ("byte", "span", "seam", "leaf", "undo")


def _change(w, rng, kind):
    """Change the sources of P: one byte, a span across an item boundary inside a
    leaf or across the seam of two leaves, a whole leaf, or one byte changed and
    changed back (not dirty)."""
    src = w.lay.src
    leaves = [lf for lf in w.lay.leaves if lf.n]
    weight = np.array([lf.n for lf in leaves], dtype=np.float64)
    lf = leaves[int(rng.choice(len(leaves), p=weight / weight.sum()))]  # a byte at random
    if kind in ("byte", "undo"):
        at = src.base + lf.s + int(rng.integers(0, lf.n))
        old = src.read(at, 1).copy()
        src.write(at, old + 1)
        if kind == "undo":
            torch.cuda.synchronize()
            src.write(at, old)
    elif kind == "leaf":
        src.write(src.base + lf.s, rng.integers(0, 256, lf.n, dtype=np.uint8))
    else:
        # the last bytes of an item and the first bytes of the item that follows it in
        # the arena: of the same range ("span"), or of the next range ("seam"; where the
        # segment side does not continue if the plan has such a seam)
        its = w.plans["P"]["items"]
        pairs = [(a, b) for a, b in zip(its, its[1:]) if b.aoff == a.aoff + a.n
                 and (b.tptr == a.tptr + a.n) == (kind == "span")]
        split = [(a, b) for a, b in pairs if b.hoff != a.hoff + a.n]
        pairs = split or pairs
        a, b = pairs[int(rng.integers(0, len(pairs)))]
        for start, n in ((a.tptr + a.n - min(a.n, int(rng.integers(1, 41))), None),
                         (b.tptr, min(b.n, int(rng.integers(1, 41))))):
            n = n or a.tptr + a.n - start
            src.write(start, src.read(start, n) ^ rng.integers(1, 256, n, dtype=np.uint8))


def _op(w, rng, op):
    ctx = w.ctx
    if op in ("pack", "unpack", "save", "save_direct", "save_hybrid", "restore",
              "arena_fill"):
        getattr(w, op)()
    elif op == "arena_tensor":
        ctx.arena_tensor(w.room)
        w._forget()
    elif op == "invalidate":
        ctx.delta_invalidate()
        w._forget()
    elif op == "cancel_held":
        w.delta(hold=True)
    elif op == "update_same":
        w.update(dict(w.moved))
    elif op == "update_moved":
        # toggle one range between its home and a free spot past the end of the plan
        k = next(i for i, lf in enumerate(w.lay.leaves) if lf.n == 4097)
        w.update({} if w.moved else {k: w.lay.arena_end + 37})
    elif op == "recreate":
        w.recreate()
    elif op == "delta_other_plan":
        w.delta("Q", "A")
    elif op == "delta_other_host":
        w.delta("P", "B")
    else:
        raise AssertionError(op)


def _sequence(w, seed, ops=OPS, steps=40):
    """Each step changes sources, runs one operation that may forget the baseline, or
    does nothing; then an incremental save of P to A, checked against the model."""
    rng = np.random.default_rng(seed)
    plan = list(ops) + [c for c in CHANGES for _ in range(4)]
    plan += ["nothing"] * max(0, steps - len(plan))
    plan = [plan[i] for i in rng.permutation(len(plan))]
    w.delta()
    w.check("first save")
    for step, what in enumerate(plan):
        if what in CHANGES:
            _change(w, rng, what)
        elif what != "nothing":
            _op(w, rng, what)
        w.delta()
        w.check(f"step {step} ({what})")


def _small_layout(seed, shape, mapped=False):
    """About 1 MiB of leaves after the bulk ring section of the shape (an incremental
    save compares shifted ranges with the LSU kernel, so it has no shift ring)."""
    return mixed_layout(seed, _tiles(shape)[:2], 4096, target=1 << 20, mapped=mapped,
                        ring=ring_section(shape, _sms(), shift=False))


def _assert_delta_ring_wraps(w, shape):
    """Every ring of the gather-compare kernel (and of the copy kernel) walks at least
    three times its stages in tiles, crossing from item to item."""
    (_, tma_cps, stages, tile), _ = _launch(shape)
    bulk = w.plans["P"]["tables"]["bulk"]
    for t in (_tiles(shape)[1], tile):
        assert _busiest(bulk, _sms() * tma_cps, t) >= 3 * stages, t


@gpu
@pytest.mark.parametrize("mode", [native.DRAIN_HOST_PACED, native.DRAIN_PINGPONG],
                         ids=["host_paced", "pingpong"])
@pytest.mark.parametrize("variant", VARIANTS, ids=["lsu", "tma"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_incremental_save_drains_exactly_the_changed_items(cuda_device, shape, variant, mode):
    ctx = _context(shape, variant)
    with _world(ctx, _small_layout(3, shape), 4096, variant, piece=64 << 10,
                spare=8192) as w:
        ctx.set_drain_mode(mode)
        ctx.set_drain(64 << 10)
        _assert_delta_ring_wraps(w, shape)
        _sequence(w, seed=list(SHAPES).index(shape) * 4 + variant * 2 + mode)


@gpu
@pytest.mark.parametrize("variant", VARIANTS, ids=["lsu", "tma"])
def test_incremental_save_of_a_mapped_plan(cuda_device, variant):
    """Host offsets scattered with holes: dirty items that continue in the arena merge
    into one DMA only where the segment continues too; the holes are canaries."""
    ctx = _context("default", variant)
    with _world(ctx, _small_layout(4, "default", mapped=True), 4096, variant,
                piece=64 << 10, spare=8192) as w:
        ctx.set_drain(64 << 10)
        its = w.plans["P"]["items"]
        assert any(b.aoff == a.aoff + a.n and b.hoff != a.hoff + a.n
                   for a, b in zip(its, its[1:])), "no run the segment side must split"
        _assert_delta_ring_wraps(w, "default")
        # a hybrid save needs the identity mapping
        _sequence(w, seed=17, ops=[op for op in OPS if op != "save_hybrid"])


# ------------------------------------------------------------------------ limits --


@gpu
@pytest.mark.parametrize("variant", VARIANTS, ids=["lsu", "tma"])
def test_gigabyte_items(cuda_device, variant):
    """Chunk 1 GiB, two leaves of 1 GiB + 4099 B (one congruent, one with its source 3
    mod 16): pack, unpack and an incremental save whose only changes are the last
    bytes of the two 1-GiB items.  Compared on the device."""
    n = (1 << 30) + 4099
    a2 = (n + 127) // 128 * 128
    end = a2 + n
    gaps = [(n, a2), (end, end + GUARD)]
    ctx = native.Context(0)
    plan = back = None
    try:
        ctx.set_variant(variant)
        src = torch.randint(0, 256, (2 * n + 64,), dtype=torch.uint8, device="cuda",
                            generator=torch.Generator("cuda").manual_seed(8))
        s2 = n + (3 - (src.data_ptr() + n)) % 16
        leaves = [src[:n], src[s2:s2 + n]]
        assert leaves[1].data_ptr() % 16 == 3
        ctx.arena_reserve(end + GUARD)
        arena = ctx.arena_tensor(end + GUARD)
        for lo, hi in gaps:
            arena[lo:hi].copy_(torch.from_numpy(pattern(hi - lo, lo)))
        plan = ctx.plan([t.data_ptr() for t in leaves], [0, a2], [n, n], 1 << 30)
        assert plan.n_items == 4
        host = torch.empty(end + GUARD, dtype=torch.uint8, pin_memory=True)
        for lo, hi in gaps:
            host[lo:hi] = torch.from_numpy(pattern(hi - lo, lo))
        k0, _ = ctx.launch_count()
        plan.pack()
        torch.cuda.synchronize()
        assert ctx.launch_count()[0] - k0 == (1 if variant == native.VARIANT_LSU else 3)
        assert torch.equal(arena[:n], leaves[0]) and torch.equal(arena[a2:end], leaves[1])
        for lo, hi in gaps:
            assert np.array_equal(arena[lo:hi].cpu().numpy(), pattern(hi - lo, lo))

        # unpack into views at the same classes inside one canary buffer
        tgt = torch.empty(2 * n + 64 + 2 * GUARD, dtype=torch.uint8, device="cuda")
        t2 = GUARD + n + 16 + (3 - (tgt.data_ptr() + GUARD + n + 16)) % 16
        views = [tgt[GUARD:GUARD + n], tgt[t2:t2 + n]]
        guards = [(0, GUARD), (GUARD + n, t2), (t2 + n, tgt.numel())]
        for lo, hi in guards:
            tgt[lo:hi].copy_(torch.from_numpy(pattern(hi - lo, lo)))
        back = ctx.plan([t.data_ptr() for t in views], [0, a2], [n, n], 1 << 30)
        back.unpack()
        torch.cuda.synchronize()
        assert torch.equal(views[0], leaves[0]) and torch.equal(views[1], leaves[1])
        for lo, hi in guards:
            assert np.array_equal(tgt[lo:hi].cpu().numpy(), pattern(hi - lo, lo))
        back.destroy()
        back = None
        del views, tgt

        stream = torch.cuda.current_stream()
        ticket = plan.save_delta_async(host.data_ptr(), stream)
        ctx.save_wait(ticket)
        assert ctx.save_delta_stats(ticket) == (False, 2 * n)
        for t in leaves:
            t[(1 << 30) - 1] += 1
        _, m0 = ctx.launch_count()
        ticket = plan.save_delta_async(host.data_ptr(), stream)
        ctx.save_wait(ticket)
        _, m1 = ctx.launch_count()
        assert ctx.save_delta_stats(ticket) == (True, 2 << 30)
        assert m1 - m0 == 2 * ((1 << 30) // (16 << 20))
        assert torch.equal(arena[:n], leaves[0]) and torch.equal(arena[a2:end], leaves[1])
        for lo, t in ((0, leaves[0]), (a2, leaves[1])):
            assert torch.equal(host[lo:lo + n].cuda(), t)
        for lo, hi in gaps:
            assert np.array_equal(host[lo:hi].numpy(), pattern(hi - lo, lo))
            assert np.array_equal(arena[lo:hi].cpu().numpy(), pattern(hi - lo, lo))
    finally:
        for p in (back, plan):
            if p is not None:
                p.destroy()
        ctx.destroy()
        torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize("variant", VARIANTS, ids=["lsu", "tma"])
def test_arena_offsets_across_4_gib(cuda_device, variant):
    """A mapped plan whose arena offsets straddle 2**32 and whose segment is compact:
    pack, unpack, save, restore and incremental saves, byte for byte."""
    lo = (1 << 32) - 4096 - 5
    lay = mixed_layout(6, (), 4096, target=256 << 10, aoff0=lo, mapped=True)
    assert min(lf.aoff for lf in lay.leaves) < 1 << 32 < lay.arena_end
    with _world(_context("default", variant), lay, 4096, variant, arena_lo=lo - GUARD) as w:
        assert lay.host_end < 8 << 20
        w.pack()
        w.check("pack")
        w.unpack()
        w.check("unpack")
        w.save()
        w.check("save")
        w.lay.tgt.write(w.lay.tgt.base, pattern(w.lay.tgt.np.size))
        w.restore()
        w.check("restore")
        rng = np.random.default_rng(6)
        w.delta()
        w.check("full delta")
        for kind in ("byte", "span", "leaf", "undo", "span"):
            _change(w, rng, kind)
            w.delta()
            w.check(f"delta after {kind}")
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- setter validation --


@gpu
def test_rejected_launch_shapes_leave_the_previous_shape(cuda_device):
    ctx = _context("deep_odd_tile", native.VARIANT_TMA)
    lay = mixed_layout(7, _tiles("deep_odd_tile"), 4096, target=4 << 20,
                       ring=ring_section("deep_odd_tile", _sms()))
    with _world(ctx, lay, 4096, native.VARIANT_TMA) as w:
        _refuse_and_probe(ctx, w)


def _refuse_and_probe(ctx, w):
    bad = [lambda: ctx.set_launch(0, 0, 1, 0),              # one stage is no ring
           lambda: ctx.set_launch(0, 0, 0, 4100),           # not a multiple of 16
           lambda: ctx.set_launch(0, 0, 32, 8192),          # 256 KiB ring > 227 KB
           lambda: ctx.set_launch(0, 0, 2, 131072 + 16),    # tile over 128 KiB
           lambda: ctx.set_shift_launch(0, 0, 2048),        # shift tile under 4 KiB
           lambda: ctx.set_shift_launch(0, 1, 0),           # one input stage
           lambda: ctx.set_shift_launch(0, 8, 32768)]       # ring > 227 KB
    for call in bad:
        with pytest.raises(native.NativeError) as e:
            call()
        assert e.value.code == native.FC_EINVAL
    # straight afterwards, under the shape the refused calls left in place
    w.pack()
    w.check("pack after refused shapes")
    w.unpack()
    w.check("unpack after refused shapes")
    # the stage counts in force are still 8 (copy ring) and 8 (shift ring): the largest
    # tile each accepts is the one 8 stages fit in 227 KB, neither 32 nor 2 stages
    ctx.set_launch(0, 0, 0, 28000)
    with pytest.raises(native.NativeError):
        ctx.set_launch(0, 0, 0, 29056)
    ctx.set_shift_launch(0, 0, 23040)
    with pytest.raises(native.NativeError):
        ctx.set_shift_launch(0, 0, 23168)
    w.pack()
    w.check("pack under the probed shape")
