"""GPU parity tests of the raw C-ABI (pack / unpack / save / restore) against the
numpy oracle (oracle/shm_layout.py).  Bit-exact: this path is a pure byte copy."""

import ctypes

import numpy as np
import pytest
import torch

from dlrover_b200 import _native as native
from oracle import shm_layout as oracle

pytestmark = pytest.mark.gpu

VARIANTS = [native.VARIANT_LSU, native.VARIANT_TMA]


def _arena_bytes(ctx, n):
    ptr, size = ctx.arena_info()
    assert size >= n
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    # plain cudaMemcpy D2D through torch's ctypes-free path: wrap the arena
    # pointer with a uint8 tensor via __cuda_array_interface__
    class _A:
        __cuda_array_interface__ = {
            "shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 2,
        }
    src = torch.as_tensor(_A(), device="cuda")
    out.copy_(src)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _ragged_case(seed, aligned):
    g = torch.Generator().manual_seed(seed)
    sizes = [0, 1, 3, 15, 16, 17, 4096, 4100, 65537, 300_001, 1_000_003, 5 << 20]
    tensors, offsets, off = [], [], 0
    for i, n in enumerate(sizes):
        t = torch.randint(0, 256, (n,), dtype=torch.uint8, generator=g).cuda()
        if aligned and n:
            off = (off + 15) // 16 * 16
        tensors.append(t)
        offsets.append(off)
        off += n
    return tensors, offsets, off


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("aligned", [True, False])
@pytest.mark.parametrize("chunk", [4096, 0])
def test_pack_matches_oracle(cuda_device, variant, aligned, chunk):
    ctx = native.get_context(0)
    tensors, offsets, total = _ragged_case(1, aligned)
    ctx.arena_reserve(total)
    size = min(ctx.arena_info()[1], total + 4096)  # the shared arena may be far larger
    # canary: the gaps between ranges (aligned case) and the bytes past the last range
    # must keep what they held
    canary = ((np.arange(size) * 131 + 7) & 255).astype(np.uint8)
    ctx.arena_tensor(size).copy_(torch.from_numpy(canary))
    plan = ctx.plan([t.data_ptr() for t in tensors], offsets, [t.numel() for t in tensors], chunk)
    assert plan.payload_bytes == sum(t.numel() for t in tensors)
    plan.pack(torch.cuda.current_stream(), variant)
    torch.cuda.synchronize()
    got = _arena_bytes(ctx, size)
    want = canary.copy()
    for t, o in zip(tensors, offsets):
        want[o:o + t.numel()] = oracle.tensor_bytes(t)
    for t, o in zip(tensors, offsets):
        n = t.numel()
        assert np.array_equal(got[o:o + n], want[o:o + n]), f"range at {o} len {n}"
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"bytes outside the ranges written at {bad[:8]}"
    plan.destroy()


@pytest.mark.parametrize("variant", VARIANTS)
def test_source_misaligned_views(cuda_device, variant):
    """Sources that start at odd byte addresses (views into a bigger buffer):
    exercises every source/destination congruence class mod 16."""
    ctx = native.get_context(0)
    g = torch.Generator().manual_seed(7)
    base = torch.randint(0, 256, (1 << 20,), dtype=torch.uint8, generator=g).cuda()
    tensors, offsets, off = [], [], 0
    for r in range(16):
        for n in (1, 31, 16 * 1024 + r, 100_000 + 3 * r):
            start = 1000 * (r + 1) + r
            tensors.append(base[start:start + n])
            offsets.append(off)
            off += n
    ctx.arena_reserve(off)
    plan = ctx.plan([t.data_ptr() for t in tensors], offsets, [t.numel() for t in tensors], 4096)
    plan.pack(None, variant)
    torch.cuda.synchronize()
    got = _arena_bytes(ctx, off)
    want = oracle.pack_ranges([oracle.tensor_bytes(t) for t in tensors], offsets, off)
    assert np.array_equal(got, want)
    plan.destroy()


@pytest.mark.parametrize("variant", VARIANTS)
def test_unpack_round_trip(cuda_device, variant):
    ctx = native.get_context(0)
    tensors, offsets, total = _ragged_case(3, aligned=False)
    ctx.arena_reserve(total)
    ptrs = [t.data_ptr() for t in tensors]
    lens = [t.numel() for t in tensors]
    plan = ctx.plan(ptrs, offsets, lens)
    plan.pack(None, variant)
    keep = [t.clone() for t in tensors]
    for t in tensors:
        t.zero_()
    plan.unpack(None, variant)
    torch.cuda.synchronize()
    for a, b in zip(tensors, keep):
        assert torch.equal(a, b)
    plan.destroy()


def test_save_and_restore_through_host(cuda_device):
    """fc_save_async -> host segment == oracle image; fc_restore_async brings it
    back bit-exact.  Mixed dtypes incl. int64 index tensor and bf16 payload."""
    ctx = native.get_context(0)
    g = torch.Generator().manual_seed(11)
    sd = {
        "w": (torch.randn(257, 129, generator=g) * 0.02).to(torch.bfloat16).cuda(),
        "idx": torch.arange(1001, dtype=torch.int64).cuda(),
        "step": torch.tensor(7.0).cuda(),
        "m": torch.randn(1001, 33, generator=g).cuda(),
        "u8": torch.randint(0, 256, (12345,), dtype=torch.uint8, generator=g).cuda(),
        "empty": torch.empty(0).cuda(),
    }
    meta, want = oracle.serialize(sd)
    metas = oracle.flatten_tensor_metas(meta)
    leaves = list(sd.values())
    total = want.size
    ctx.arena_reserve(total)
    plan = ctx.plan([t.data_ptr() for t in leaves], [m.offset for m in metas],
                    [m.numel * m.element_size for m in metas])
    host = torch.empty(total, dtype=torch.uint8).pin_memory()
    ticket = plan.save_async(host.data_ptr(), torch.cuda.current_stream())
    ctx.save_wait(ticket)
    assert np.array_equal(host.numpy(), want)
    pack_ms, drain_ms, total_ms = ctx.save_timings(ticket)
    assert pack_ms > 0 and drain_ms > 0 and total_ms >= pack_ms
    # restore into zeroed tensors
    keep = {k: v.clone() for k, v in sd.items()}
    for v in sd.values():
        v.zero_()
    plan.restore_async(host.data_ptr(), torch.cuda.current_stream())
    ctx.restore_wait()
    for k in sd:
        assert torch.equal(sd[k], keep[k]), k
    plan.destroy()


def test_registered_pageable_host(cuda_device):
    """The drain target the product uses: an mmap'd POSIX shm segment pinned
    with fc_host_register."""
    import mmap
    import os
    import _posixshmem

    ctx = native.get_context(0)
    name = f"/fc_test_{os.getpid()}"
    n = 3 << 20
    fd = _posixshmem.shm_open(name, os.O_CREAT | os.O_EXCL | os.O_RDWR, mode=0o600)
    try:
        os.ftruncate(fd, n)
        mm = mmap.mmap(fd, n)
        addr = ctypes.addressof(ctypes.c_char.from_buffer(mm))
        ctx.host_register(addr, n, prefault_threads=2)
        t = torch.randint(0, 256, (n - 5,), dtype=torch.uint8).cuda()
        ctx.arena_reserve(n)
        plan = ctx.plan([t.data_ptr()], [5], [t.numel()])
        ticket = plan.save_async(addr, None)
        ctx.save_wait(ticket)
        assert np.array_equal(np.frombuffer(mm, dtype=np.uint8)[5:], t.cpu().numpy())
        ctx.host_unregister(addr)
        plan.destroy()
    finally:
        _posixshmem.shm_unlink(name)
        os.close(fd)


def test_busy_and_errors(cuda_device):
    ctx = native.get_context(0)
    t = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    with pytest.raises(native.NativeError):
        ctx.plan([t.data_ptr(), t.data_ptr()], [0, 100], [1024, 1024])  # overlap
    with pytest.raises(native.NativeError):
        ctx.plan([0], [0], [16])  # null pointer, non-empty
    ctx.arena_reserve(16)
    big = ctx.plan([t.data_ptr()], [1 << 40], [1024])
    with pytest.raises(native.NativeError):
        big.pack()  # arena smaller than plan
    big.destroy()


@pytest.mark.parametrize("variant", VARIANTS)
def test_plan_update_retargets_without_recreating(cuda_device, variant):
    """fc_plan_update: same plan object, new tensors/offsets/sizes (grow and
    shrink), stream-ordered upload."""
    ctx = native.get_context(0)
    g = torch.Generator().manual_seed(21)
    a = [torch.randint(0, 256, (n,), dtype=torch.uint8, generator=g).cuda()
         for n in (1000, 70_000, 33)]
    ctx.arena_reserve(1 << 22)
    plan = ctx.plan([t.data_ptr() for t in a], [0, 1000, 71_000], [t.numel() for t in a], 4096)
    stream = torch.cuda.current_stream()
    plan.pack(stream, variant)
    b = [torch.randint(0, 256, (n,), dtype=torch.uint8, generator=g).cuda()
         for n in (5, 1 << 20, 4097, 300_000, 16)]
    offs, o = [], 3
    for t in b:
        offs.append(o)
        o += t.numel()
    plan.update([t.data_ptr() for t in b], offs, [t.numel() for t in b], stream)
    assert plan.payload_bytes == sum(t.numel() for t in b) and plan.arena_end == o
    plan.pack(stream, variant)
    torch.cuda.synchronize()
    got = _arena_bytes(ctx, o)
    want = oracle.pack_ranges([oracle.tensor_bytes(t) for t in b], offs, o)
    assert np.array_equal(got[3:], want[3:])
    # shrink again
    plan.update([a[1].data_ptr()], [64], [a[1].numel()], stream)
    plan.pack(stream, variant)
    torch.cuda.synchronize()
    got = _arena_bytes(ctx, 64 + a[1].numel())
    assert np.array_equal(got[64:], oracle.tensor_bytes(a[1]))
    plan.destroy()


def test_bounded_arena_streams_window_by_window(cuda_device):
    """Plan (45 MB, ragged + misaligned) bigger than the arena (8 MiB cap):
    fc_save_async/fc_restore_async stream it through the window; bytes equal the
    oracle image, restore is bit-exact."""
    ctx = native.Context(0)  # private context: the cap must not leak into other tests
    ctx.set_arena_limit(8 << 20)
    g = torch.Generator().manual_seed(5)
    sizes = [3, 5 << 20, 1, 7 << 20, 123_457, 9 << 20, 6 << 20, 17, 12 << 20, 4 << 20, 999]
    tensors = [torch.randint(0, 256, (n,), dtype=torch.uint8, generator=g).cuda() for n in sizes]
    offs, o = [], 0
    for t in tensors:
        offs.append(o)
        o += t.numel()
    ctx.arena_reserve(o)
    assert ctx.arena_info()[1] == 8 << 20
    plan = ctx.plan([t.data_ptr() for t in tensors], offs, sizes)
    host = torch.zeros(o, dtype=torch.uint8).pin_memory()
    k0, m0 = ctx.launch_count()
    ticket = plan.save_async(host.data_ptr(), torch.cuda.current_stream())
    assert ctx.save_poll(ticket)  # windowed saves complete before returning
    k1, m1 = ctx.launch_count()
    assert k1 - k0 >= 6  # ceil(45 MB / 8 MiB) windows, one gather kernel each
    want = oracle.pack_ranges([oracle.tensor_bytes(t) for t in tensors], offs, o)
    assert np.array_equal(host.numpy(), want)
    keep = [t.clone() for t in tensors]
    for t in tensors:
        t.zero_()
    plan.restore_async(host.data_ptr(), torch.cuda.current_stream())
    ctx.restore_wait()
    for a, b in zip(tensors, keep):
        assert torch.equal(a, b)
    plan.destroy()
    ctx.destroy()


def test_in_place_save_and_restore(cuda_device):
    """fc_save_direct_async / fc_restore_direct_async: no arena at all — the DMA
    reads / writes the tensors themselves.  Same oracle image, ragged sizes, many
    small spans sharing a batch, views of one buffer next to each other."""
    ctx = native.get_context(0)
    g = torch.Generator().manual_seed(21)
    # one flat buffer cut into consecutive views ...
    flat = torch.randint(0, 256, (3 << 20,), dtype=torch.uint8, generator=g).cuda()
    cuts = [0, 7, 4096, 1 << 20, (1 << 20) + 13, 3 << 20]
    views = [flat[a:b] for a, b in zip(cuts, cuts[1:])]
    # ... 300 small separate tensors, and a big one (several drain pieces)
    small = [torch.randint(0, 256, (n,), dtype=torch.uint8, generator=g).cuda()
             for n in ([1, 3, 4, 17, 255, 4097] * 50)]
    big = torch.randint(0, 256, (70 << 20,), dtype=torch.uint8, generator=g).cuda()
    leaves = views + small + [big, torch.empty(0, dtype=torch.uint8).cuda()]
    offsets, off = [], 0
    for t in leaves:
        offsets.append(off)
        off += t.numel()
    total = off
    want = oracle.pack_ranges([oracle.tensor_bytes(t) for t in leaves], offsets, total)
    plan = ctx.plan([t.data_ptr() for t in leaves], offsets, [t.numel() for t in leaves])
    assert plan.n_spans == len(views) + len(small) + 1  # empty leaf dropped, nothing merged
    host = torch.zeros(total, dtype=torch.uint8).pin_memory()
    k0, m0 = ctx.launch_count()
    ticket = plan.save_direct_async(host.data_ptr(), torch.cuda.current_stream())
    ctx.save_wait(ticket)
    k1, m1 = ctx.launch_count()
    assert k1 == k0 and m1 - m0 >= plan.n_spans  # DMA only, no kernel
    assert np.array_equal(host.numpy(), want)
    assert ctx.save_pack_done(ticket)
    # held variant: nothing lands before the release
    host.zero_()
    ticket = plan.save_direct_async(host.data_ptr(), torch.cuda.current_stream(), hold=True)
    torch.cuda.synchronize()
    assert not ctx.save_poll(ticket) and not ctx.save_pack_done(ticket)
    assert not host.numpy().any()
    ctx.save_release(ticket)
    ctx.save_wait(ticket)
    assert np.array_equal(host.numpy(), want)
    # in-place restore
    keep = [t.clone() for t in leaves]
    flat.zero_()
    big.zero_()
    for t in small:
        t.zero_()
    plan.restore_async(host.data_ptr(), torch.cuda.current_stream(), direct=True)
    ctx.restore_wait()
    for t, k in zip(leaves, keep):
        assert torch.equal(t, k)
    fill_ms, scatter_ms, total_ms = ctx.restore_timings()
    assert fill_ms > 0 and total_ms >= fill_ms
    plan.destroy()


def test_hybrid_save_snapshot_tail_in_place_head(cuda_device):
    """fc_save_hybrid_async: tensors at offsets >= cut go through the arena (the slices of
    the bulk / shift / resid tables from the cut on, arena byte 0 = the cut rounded down to
    128 B), the rest is drained in place first;
    fc_save_pack_done / fc_save_sources_wait tell when the tensors may change."""
    ctx = native.get_context(0)
    g = torch.Generator().manual_seed(31)
    sizes = [5, 4096, 1 << 20, 3, (2 << 20) + 7, 17, 40 << 20, 1, 300_001, 9 << 20]
    leaves = [torch.randint(0, 256, (n,), dtype=torch.uint8, generator=g).cuda() for n in sizes]
    offsets, off = [], 0
    for t in leaves:
        offsets.append(off)
        off += t.numel()
    total = off
    want = oracle.pack_ranges([oracle.tensor_bytes(t) for t in leaves], offsets, total)
    plan = ctx.plan([t.data_ptr() for t in leaves], offsets, sizes)
    host = torch.zeros(total, dtype=torch.uint8).pin_memory()
    stream = torch.cuda.current_stream()
    for first_snapshotted in (0, 4, 7, len(leaves)):   # all snapshot ... all in place
        cut = offsets[first_snapshotted] if first_snapshotted < len(leaves) else total
        ctx.arena_reserve(max(total - (cut & ~127), 8))
        host.zero_()
        k0, m0 = ctx.launch_count()
        ticket = plan.save_hybrid_async(host.data_ptr(), cut, stream, hold=True)
        torch.cuda.synchronize()
        # held: the in-place part has not been read yet -> the tensors are not free
        if first_snapshotted > 0:
            assert not ctx.save_pack_done(ticket)
        assert not host.numpy().any()
        ctx.save_release(ticket)
        ctx.save_sources_wait(ticket)
        assert ctx.save_pack_done(ticket)
        # from here on the sources may change without touching the checkpoint
        keep = [t.clone() for t in leaves]
        for t in leaves[first_snapshotted:]:
            t.add_(1)
        ctx.save_wait(ticket)
        k1, m1 = ctx.launch_count()
        if first_snapshotted < len(leaves):
            assert 1 <= k1 - k0 <= 3   # bulk / shift / resid slices of the tables
        else:
            assert k1 == k0
        assert np.array_equal(host.numpy(), want), first_snapshotted
        for t, k in zip(leaves, keep):
            t.copy_(k)
    # a cut inside a tensor, or an arena smaller than the snapshot part, is refused
    with pytest.raises(native.NativeError):
        plan.save_hybrid_async(host.data_ptr(), offsets[2] + 1, stream)
    plan.destroy()


def test_held_save_can_be_cancelled(cuda_device):
    """fc_save_cancel: a held save is dropped before a byte of the segment changed;
    once released it cannot be cancelled any more."""
    ctx = native.get_context(0)
    t = torch.arange(1 << 20, dtype=torch.int32).cuda()
    n = t.numel() * 4
    ctx.arena_reserve(n)
    plan = ctx.plan([t.data_ptr()], [0], [n])
    host = torch.full((n,), 7, dtype=torch.uint8).pin_memory()
    stream = torch.cuda.current_stream()
    for direct in (False, True):
        if direct:
            ticket = plan.save_direct_async(host.data_ptr(), stream, hold=True)
        else:
            ticket = plan.save_async(host.data_ptr(), stream, hold=True)
        assert not ctx.save_poll(ticket)
        assert ctx.save_cancel(ticket)
        ctx.save_wait(ticket)                 # returns: the ticket counts as complete
        assert ctx.save_pack_done(ticket)
        torch.cuda.synchronize()
        assert (host.numpy() == 7).all()      # untouched
    ticket = plan.save_async(host.data_ptr(), stream)   # the context is usable again
    assert not ctx.save_cancel(ticket)        # not held: too late
    ctx.save_wait(ticket)
    assert np.array_equal(host.numpy().view(np.int32), np.arange(1 << 20, dtype=np.int32))
    plan.destroy()
