"""Incremental memory saves (fc_save_delta_async / SharedMemoryHandler.incremental).

After a save has drained, the HBM arena is a byte image of the segment; an incremental
save compares every new byte with it, writes and drains only the work items that differ.
Every GPU test checks the whole segment (and the arena) byte for byte against the
oracle image of the current tensors after every save."""

import ctypes
import filecmp
import os
import time

import numpy as np
import pytest
import torch

from dlrover_b200 import _native as native
from dlrover_b200.shm_handler import (DLROVER_CKPT_CONFIG_KEY, CheckpointConfig,
                                      SharedMemoryHandler, _DeviceStager)
from oracle import shm_layout as oracle
from tests import plan_model as pm

CHUNK = 64 << 10
gpu = pytest.mark.gpu


# ------------------------------------------------------------------------ helpers --


def _layout(seed=5, big=1 << 20):
    """Leaves of every alignment class the plan builder knows, with their segment
    offsets: a congruent body with a 5-byte tail residue, a 4-byte step scalar, shifted
    ranges behind it (large: shift table; under 4 KiB: LSU), a congruent range with a
    head residue (source and offset both 7 mod 16), a range under 16 B, and a congruent
    range that ends the plan.  Returns (leaves, offsets, total, keepalive)."""
    g = torch.Generator().manual_seed(seed)

    def rnd(n):
        return torch.randint(0, 256, (n,), dtype=torch.uint8, generator=g).cuda()

    base = rnd(200_007 + 64)
    leaves = [rnd(3 * big + 5), rnd(4), rnd(4 * big + 28), rnd(3000),
              base[7:7 + 200_000], rnd(9), rnd(70_000 + 16)]
    offsets, off = [], 0
    for i, t in enumerate(leaves):
        if i == 4:
            off += (7 - off) % 16  # congruent with its source: a head residue
        if i == 6:
            off += (-off) % 16
        offsets.append(off)
        off += t.numel()
    return leaves, offsets, off, [base]


def _want(leaves, offsets, total):
    return oracle.pack_ranges([oracle.tensor_bytes(t) for t in leaves], offsets, total)


def _arena(ctx, nbytes):
    """The arena's bytes, read without handing the arena out (arena_tensor would
    forget the baseline)."""
    ptr, size = ctx.arena_info()
    assert nbytes <= size

    class _A:
        __cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1",
                                    "data": (ptr, False), "version": 2}

    return torch.as_tensor(_A(), device="cuda").cpu().numpy()


def _check(host, ctx, leaves, offsets, total):
    want = _want(leaves, offsets, total)
    assert np.array_equal(host[:total], want), "segment != oracle image"
    arena = _arena(ctx, total)
    for t, o in zip(leaves, offsets):
        assert np.array_equal(arena[o:o + t.numel()], want[o:o + t.numel()]), "arena"


def _drained(leaves, offsets, total, old):
    """The bytes an incremental save must drain: the items (CHUNK plan) in which the
    oracle image of the current tensors differs from `old`."""
    its = pm.items([pm.Range(t.data_ptr(), o, t.numel()) for t, o in zip(leaves, offsets)],
                   CHUNK)
    return pm.drained_bytes(pm.dirty(its, old, _want(leaves, offsets, total)))


def _save(ctx, plan, host_addr, **kw):
    ticket = plan.save_delta_async(host_addr, torch.cuda.current_stream(), **kw)
    ctx.save_wait(ticket)
    return ctx.save_delta_stats(ticket)


def _bump(t, i):
    t[i] += 1  # uint8: always a different byte


# ------------------------------------------------------------------- kernel parity --


@gpu
@pytest.mark.parametrize("variant", [native.VARIANT_TMA, native.VARIANT_LSU])
def test_delta_parity_through_the_c_abi(cuda_device, variant):
    ctx = native.Context(0)
    ctx.set_variant(variant)
    leaves, offsets, total, _keep = _layout()
    ctx.arena_reserve(total)
    plan = ctx.plan([t.data_ptr() for t in leaves], offsets, [t.numel() for t in leaves],
                    chunk_bytes=CHUNK)
    assert plan.n_items > 100
    host = torch.zeros(total, dtype=torch.uint8).pin_memory()
    hnp = host.numpy()
    addr = host.data_ptr()
    payload = sum(t.numel() for t in leaves)

    assert _save(ctx, plan, addr) == (False, payload)  # no baseline: full
    _check(hnp, ctx, leaves, offsets, total)
    assert _save(ctx, plan, addr) == (True, 0)  # nothing changed
    _check(hnp, ctx, leaves, offsets, total)

    a, step, shifted, small, headed, tiny, last = leaves
    changes = [(a, 0), (a, a.numel() // 2), (a, 3 * CHUNK - 1), (a, 3 * CHUNK),
               (a, a.numel() - 1),                       # tail residue
               (step, 2), (shifted, 12345), (shifted, shifted.numel() - 1), (small, 1500),
               (headed, 0), (headed, 8), (headed, 100_000), (headed, headed.numel() - 1),
               (tiny, 4), (last, last.numel() - 1)]      # the last byte of the plan
    for t, i in changes:
        old = _want(leaves, offsets, total)
        _bump(t, i)
        delta, n = _save(ctx, plan, addr)
        assert delta and n == _drained(leaves, offsets, total, old), (i, n)
        _check(hnp, ctx, leaves, offsets, total)
    old = _want(leaves, offsets, total)
    for t, i in changes:  # all at once
        _bump(t, i)
    delta, n = _save(ctx, plan, addr)
    assert delta and n == _drained(leaves, offsets, total, old)
    _check(hnp, ctx, leaves, offsets, total)

    old = _want(leaves, offsets, total)
    shifted.copy_(torch.randint(0, 256, shifted.shape, dtype=torch.uint8, device="cuda"))
    delta, n = _save(ctx, plan, addr)  # one leaf rewritten
    assert delta and n == _drained(leaves, offsets, total, old)
    _check(hnp, ctx, leaves, offsets, total)

    for t in leaves:  # every item, one byte or two each
        t[::CHUNK // 2] += 1
        t[-1] += 1
    assert _save(ctx, plan, addr) == (True, payload)
    _check(hnp, ctx, leaves, offsets, total)
    plan.destroy()
    ctx.destroy()


# -------------------------------------------------------------------- invalidation --


@gpu
def test_every_invalidation_ends_with_a_correct_segment(cuda_device):
    ctx = native.Context(0)
    leaves, offsets, total, _keep = _layout(seed=9)
    room = total + (1 << 20)
    ctx.arena_reserve(room)
    lens = [t.numel() for t in leaves]
    plan = ctx.plan([t.data_ptr() for t in leaves], offsets, lens, chunk_bytes=CHUNK)
    host = torch.zeros(room, dtype=torch.uint8).pin_memory()
    hnp, addr = host.numpy(), host.data_ptr()
    stream = torch.cuda.current_stream()
    payload = sum(lens)

    def full_then_delta(what):
        delta, n = _save(ctx, plan, addr)
        assert not delta and n == payload, what
        _check(hnp, ctx, leaves, offsets, total)
        _bump(leaves[2], 777)
        delta, n = _save(ctx, plan, addr)
        assert delta and 1 <= n <= CHUNK, what
        _check(hnp, ctx, leaves, offsets, total)

    full_then_delta("first save")

    for o, ln in zip(offsets, lens):  # somebody else wrote the segment, and said so
        hnp[o:o + ln] = 0xAB
    ctx.delta_invalidate()
    full_then_delta("poisoned segment")

    _bump(leaves[0], 5)
    ticket = plan.save_delta_async(addr, stream, hold=True)
    torch.cuda.synchronize()
    assert ctx.save_cancel(ticket)
    full_then_delta("cancelled held save")

    # fresh tensors at the same offsets (FSDP): the baseline survives
    fresh = [t.clone() for t in leaves]
    base = _keep[0].clone()
    fresh[4] = base[7:7 + leaves[4].numel()]
    leaves[:] = fresh
    _keep[0] = base
    plan.update([t.data_ptr() for t in leaves], offsets, lens, stream)
    _bump(leaves[6], 3)
    delta, n = _save(ctx, plan, addr)
    assert delta and 1 <= n <= CHUNK
    _check(hnp, ctx, leaves, offsets, total)

    ctx.arena_reserve(room + (4 << 20))  # regrow: a new, empty arena
    full_then_delta("arena regrow")

    plan.restore_async(addr, stream)
    ctx.restore_wait()
    full_then_delta("restore")

    ctx.arena_tensor(total).fill_(0x77)
    torch.cuda.synchronize()
    full_then_delta("arena handed out")

    ctx.save_wait(plan.save_async(addr, stream))
    full_then_delta("plain save")

    moved = [o + 4096 for o in offsets]  # new offsets: the image moves
    plan.update([t.data_ptr() for t in leaves], moved, lens, stream)
    delta, n = _save(ctx, plan, addr)
    assert not delta and n == payload
    want = _want(leaves, moved, total + 4096)
    for o, ln in zip(moved, lens):
        assert np.array_equal(hnp[o:o + ln], want[o:o + ln])
    plan.destroy()
    ctx.destroy()


# -------------------------------------------------------------------- staged drain --


@gpu
def test_staged_and_sliced_drain_of_dirty_runs(cuda_device):
    from tests.test_gpu_r02 import _Segment

    ctx = native.Context(0)
    ctx.set_stage(3, 1 << 20)
    leaves, offsets, total, _keep = _layout(seed=21, big=2 << 20)
    assert total > (9 << 20)
    seg = _Segment(total)
    try:
        ctx.arena_reserve(total)
        plan = ctx.plan([t.data_ptr() for t in leaves], offsets, [t.numel() for t in leaves],
                        chunk_bytes=CHUNK)
        hnp = seg.bytes()

        def at(off):  # the leaf byte that lands at segment offset `off`
            for t, o in zip(leaves, offsets):
                if o <= off < o + t.numel():
                    return t, off - o
            raise AssertionError(off)

        assert _save(ctx, plan, seg.addr)[0] is False  # pageable: bounce slots
        _check(hnp, ctx, leaves, offsets, total)
        old = _want(leaves, offsets, total)
        for off in (100, (3 << 20) + 7, total - 1):
            _bump(*at(off))
        delta, n = _save(ctx, plan, seg.addr)
        assert delta and n == _drained(leaves, offsets, total, old)
        _check(hnp, ctx, leaves, offsets, total)

        ctx.host_register_background(seg.addr, total, slice_bytes=4 << 20)
        deadline = time.time() + 60
        while not ctx.host_ready(seg.addr):
            assert time.time() < deadline
            time.sleep(0.01)
        ctx.set_drain(3 << 20, 1)
        for mode in (native.DRAIN_HOST_PACED, native.DRAIN_PINGPONG):
            ctx.set_drain_mode(mode)
            # dirty items on both sides of the 4 MiB and 8 MiB slice boundaries: their
            # merged runs straddle a slice, so the drain must cut them there
            old = _want(leaves, offsets, total)
            for off in range((4 << 20) - 2 * CHUNK, (4 << 20) + 2 * CHUNK, CHUNK // 2):
                _bump(*at(off))
            for off in ((8 << 20) - 10, (8 << 20) + 10):
                _bump(*at(off))
            _, m0 = ctx.launch_count()
            delta, n = _save(ctx, plan, seg.addr)
            _, m1 = ctx.launch_count()
            assert delta and n == _drained(leaves, offsets, total, old)
            assert m1 - m0 >= 4  # two runs, each cut at a slice boundary
            _check(hnp, ctx, leaves, offsets, total)
        ctx.host_unregister(seg.addr)
        plan.destroy()
    finally:
        ctx.destroy()
        seg.close()


# ---------------------------------------------------------------------- handler --


@gpu
def test_segment_keeps_the_snapshot_after_wait_snapshot(cuda_device, run_env):
    handler = SharedMemoryHandler(0, host=True)
    handler.incremental = True
    try:
        g = torch.Generator().manual_seed(4)
        sd = {"w": torch.randint(0, 256, (3 << 20,), dtype=torch.uint8, generator=g).cuda(),
              "step": torch.tensor([7], dtype=torch.int32).cuda(),
              "m": torch.randn(123_457, generator=g).cuda()}
        for step in (1, 2, 3):
            sd["w"][step * 1000] += 1
            _, want = oracle.serialize(sd)
            sd[DLROVER_CKPT_CONFIG_KEY] = CheckpointConfig(step=step, paths={})
            pending = handler.save_state_dict(sd, blocking=False)
            handler.wait_snapshot()
            sd["w"].add_(1)  # after the snapshot: must not reach the segment
            sd["m"].mul_(2)
            pending.wait()
            del sd[DLROVER_CKPT_CONFIG_KEY]
            got = np.frombuffer(handler.shared_memory.buf, dtype=np.uint8)
            assert np.array_equal(got, want), step
            del got
            stats = handler.last_save_stats
            assert stats["delta"] is (step > 1)
            if step > 1:  # everything but the step scalar changed since the last snapshot
                assert want.size - (256 << 10) <= stats["drained_bytes"] <= want.size
    finally:
        handler.unlink()
        handler.close()


class _Adapted(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.base = torch.nn.Sequential(torch.nn.Linear(1024, 1024), torch.nn.GELU(),
                                        torch.nn.Linear(1024, 1024))
        self.down = torch.nn.Linear(1024, 16, bias=False)
        self.up = torch.nn.Linear(16, 1024, bias=False)
        for p in self.base.parameters():
            p.requires_grad_(False)

    def forward(self, x):
        return self.base(x) + self.up(self.down(x))


def _train_and_save(ckpt, tmp_path, stats=None):
    from dlrover_b200.flash_checkpoint.api import StorageType

    torch.manual_seed(0)
    model = _Adapted().cuda()
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-2)
    x = torch.randn(32, 1024, device="cuda")
    for step in range(1, 6):
        model(x).square().mean().backward()
        opt.step()
        opt.zero_grad()
        sd = {"model": model.state_dict(), "optim": opt.state_dict()}
        kind = StorageType.DISK if step == 5 else StorageType.MEMORY
        ckpt.save_checkpoint(step, sd, path=str(tmp_path / f"{step}.pt"), storage_type=kind)
        assert ckpt.wait_memory_save(60)
        if stats is not None:
            stats.append(ckpt.engine.last_save_stats())
    ckpt.wait_latest_checkpoint(timeout=120)
    return model, opt, sd


@gpu
def test_ddp_adapter_training_drains_only_the_adapter(cuda_device, run_env, tmp_path):
    from dlrover_b200.ckpt_saver import AsyncCheckpointSaver
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer

    AsyncCheckpointSaver.start_async_saving_ckpt()
    (tmp_path / "on").mkdir()
    (tmp_path / "off").mkdir()
    ckpt = DdpCheckpointer(str(tmp_path / "on"))
    ckpt.engine.incremental = True
    stats = []
    try:
        model, opt, sd = _train_and_save(ckpt, tmp_path / "on", stats)
        adapter = sum(p.numel() * p.element_size() for p in (model.down.weight, model.up.weight))
        moments = sum(v.numel() * v.element_size() for s in opt.state.values()
                      for v in s.values() if torch.is_tensor(v) and v.is_cuda)
        changed = 2 + sum(1 for s in opt.state.values() for v in s.values()
                          if torch.is_tensor(v) and v.is_cuda)
        bound = adapter + moments + changed * (256 << 10)
        assert stats[0]["delta"] is False
        for s in stats[1:]:
            assert s["delta"] is True and 0 < s["drained_bytes"] <= bound, s
        loaded = ckpt.load_checkpoint()
        for k, v in sd["model"].items():
            assert torch.equal(loaded["model"][k], v.cpu()), k
        live = {"model": {k: torch.zeros_like(v) for k, v in sd["model"].items()},
                "optim": sd["optim"]}
        assert ckpt.load_checkpoint_into(live, strict=False) == 5
        for k, v in sd["model"].items():
            assert torch.equal(live["model"][k], v), k
    finally:
        ckpt.engine.close()

    ckpt = DdpCheckpointer(str(tmp_path / "off"))
    try:
        _train_and_save(ckpt, tmp_path / "off")
    finally:
        ckpt.engine.close()
    on, off = tmp_path / "on" / "5.pt", tmp_path / "off" / "5.pt"
    assert on.exists() and filecmp.cmp(on, off, shallow=False)


@gpu
def test_cooperative_incremental_save(cuda_device, monkeypatch):
    """Each local rank drains its own window from its own context and baseline; the
    worker compares the whole segment with the oracle after every save."""
    if torch.cuda.device_count() < 2:
        pytest.skip("cooperative saves need 2 local GPUs")
    from tests.test_multi_gpu import run_case

    monkeypatch.setenv("DLROVER_B200_INCREMENTAL", "1")
    run_case("coop", 2, "nccl", "cuda")


# --------------------------------------------------------------- CPU (no GPU needed) --


def test_entry_points_reject_null_arguments():
    lib = native.load_library()
    ticket = ctypes.c_uint64()
    assert lib.fc_save_delta_async(None, None, None, 0, ctypes.byref(ticket)) == native.FC_EINVAL
    assert b"fc_save_delta_async" in lib.fc_last_error()
    n, d = ctypes.c_uint64(), ctypes.c_int()
    assert lib.fc_save_delta_stats(None, 1, ctypes.byref(n), ctypes.byref(d)) == native.FC_EINVAL
    assert lib.fc_delta_invalidate(None) == native.FC_EINVAL


class _FakeCtx:
    def __init__(self):
        self.invalidated = 0

    def delta_invalidate(self):
        self.invalidated += 1

    def arena_info(self):
        return 0, 1 << 40

    def arena_reserve(self, n):
        pass

    def save_release(self, t):
        pass

    def save_wait(self, t):
        pass

    def save_timings(self, t):
        return 0.0, 0.0, 0.0

    def save_delta_stats(self, t):
        return True, 123


class _FakePlan:
    arena_end = 2000

    def __init__(self):
        self.calls = []

    def _call(self, name):
        self.calls.append(name)
        return 1

    def save_async(self, addr, stream=None, hold=False):
        return self._call("save_async")

    def save_delta_async(self, addr, stream=None, hold=False):
        return self._call("save_delta_async")

    def save_direct_async(self, addr, stream=None, hold=False):
        return self._call("save_direct_async")

    def save_hybrid_async(self, addr, cut, stream=None, hold=False):
        return self._call("save_hybrid_async")


class _FakeStager:
    ARENA_FULL, ARENA_WINDOWED, ARENA_NONE = (_DeviceStager.ARENA_FULL,
                                              _DeviceStager.ARENA_WINDOWED,
                                              _DeviceStager.ARENA_NONE)
    device_index = 0

    def __init__(self, arena):
        self.ctx = _FakeCtx()
        self.plan = _FakePlan()
        self.arena = arena
        self._attached = (0, 2000)

    @staticmethod
    def prepare_ranges(ranges, keepalive, for_write=False):
        return [1 << 20, 2 << 20], [0, 1000], [1000, 1000]

    def attach(self, shm, lo=0, hi=None):
        pass

    def plan_for(self, prepared, **kw):
        return self.plan

    def ensure_arena(self, plan):
        return self.arena

    def pinned(self):
        return True

    def pin_in_background(self):
        pass


class _FakeShm:
    dma_address = 1 << 30
    address = 1 << 30
    size = 2000

    def stale(self):
        return False


class _FakeStream:
    def wait_stream(self, other):
        pass


class _FakeEvent:
    def record(self, stream=None):
        pass


@pytest.mark.parametrize("mode,want", [
    ("snapshot", "save_delta_async"),
    ("in_place", "save_direct_async"),
    ("hybrid", "save_hybrid_async"),
    ("windowed", "save_async"),
    ("no_arena", "save_direct_async"),
])
def test_switch_reaches_only_full_snapshot_saves(run_env, monkeypatch, mode, want):
    monkeypatch.setenv("DLROVER_B200_INCREMENTAL", "1")
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _FakeStream())
    monkeypatch.setattr(torch.cuda, "Event", _FakeEvent)
    handler = SharedMemoryHandler(0, host=True)
    try:
        assert handler.incremental
        arena = {"windowed": _DeviceStager.ARENA_WINDOWED,
                 "no_arena": _DeviceStager.ARENA_NONE}.get(mode, _DeviceStager.ARENA_FULL)
        stager = _FakeStager(arena)
        handler._stager_for = lambda tensors: stager
        handler.shared_memory = _FakeShm()
        if mode in ("in_place", "hybrid"):
            handler.in_place = True
        if mode == "hybrid":
            handler.in_place_snapshot_bytes = 1500  # the tensor at 1000 fits, the one at 0 not
        t = torch.zeros(4)
        for _ in range(2):
            handler.write_ranges([(t, 0, 1000), (t, 1000, 1000)], [], blocking=True)
        assert stager.plan.calls == [want, want]
        if want == "save_delta_async":
            assert handler.last_save_stats == {"delta": True, "drained_bytes": 123}
            assert stager.ctx.invalidated == 1  # first save: a mapping it had not seen
        else:
            assert handler.last_save_stats is None
        handler.incremental = False
        handler.write_ranges([(t, 0, 1000), (t, 1000, 1000)], [], blocking=True)
        assert stager.plan.calls[-1] != "save_delta_async"
    finally:
        handler.shared_memory = None
        handler.close()


def test_engine_attribute_sets_the_switch(run_env, tmp_path):
    from dlrover_b200.ckpt_saver import AsyncCheckpointSaver
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer

    AsyncCheckpointSaver.start_async_saving_ckpt()
    ckpt = DdpCheckpointer(str(tmp_path))
    try:
        assert ckpt.engine.incremental is False
        ckpt.engine.incremental = True
        assert ckpt.engine._shm_handler.incremental is True
        assert ckpt.engine.last_save_stats() is None
    finally:
        ckpt.engine.close()
