"""Rollback from the arena image (fc_restore_from_image_async / rollback_into).

After a full-arena save has drained, the HBM arena is a byte image of what the segment
holds for that plan; a rollback scatters the live tensors from it with the plan's unpack
kernels and moves no byte over PCIe.  The GPU tests run on the byte model of
test_kernel_model.py: after every operation the arena, both pinned host buffers, the
sources and the targets must equal the model byte for byte.  Each test also tracks the
image record by hand and checks that the library answers the same."""

import ctypes
import os

import numpy as np
import pytest
import torch

from dlrover_b200 import _native as native
from tests import plan_model as pm
from tests.test_kernel_model import DEFAULT_CHUNK, _context, _tiles, _world, mixed_layout

gpu = pytest.mark.gpu

VARIANTS = (native.VARIANT_LSU, native.VARIANT_TMA)


# ------------------------------------------------------------------------ helpers --


def _rollback(w, name="Q", host="A", expect=True):
    """Roll plan `name` back from the image for host buffer `host`, in the library and
    in the model.  expect=False: the call must refuse, enqueue nothing and change nothing."""
    p = w.plans[name]
    addr = w.host_t[host].data_ptr()
    assert p["plan"].image_covers(addr) is expect
    saved = {k: v.numpy().copy() for k, v in w.host_t.items()}
    k0, m0 = w.ctx.launch_count()
    got = p["plan"].restore_from_image_async(addr, torch.cuda.current_stream())
    assert got is expect
    if got:
        w.ctx.restore_wait()
        fill, scatter, total = w.ctx.restore_timings()
        assert fill == pytest.approx(0.0, abs=0.05) and scatter >= 0.0 and total >= scatter
        w._scatter(name)  # arena unchanged, the baseline kept
    torch.cuda.synchronize()
    k1, m1 = w.ctx.launch_count()
    assert m1 == m0, "a rollback moves no byte over PCIe"
    assert k1 - k0 == (w._kernels(name) if expect else 0)
    for k, v in w.host_t.items():  # no host byte written
        assert np.array_equal(v.numpy(), saved[k]), k
    w.check(f"rollback {name}/{host} expect={expect}")


def _scribble(buf, seed):
    """New bytes everywhere in a device buffer (model and device)."""
    rng = np.random.default_rng(seed)
    buf.write(buf.base, rng.integers(0, 256, buf.np.size, dtype=np.uint8))


def _layout(seed, chunk=DEFAULT_CHUNK, mapped=False, target=4 << 20):
    # congruent, shifted and residue ranges of every (source - arena) class mod 16
    return mixed_layout(seed, _tiles("default"), chunk, target=target, mapped=mapped)


def _targets_hold_the_segment(w, name="Q", host="A"):
    b, h = w.buf(name), w.host[host]
    for r in w.plans[name]["ranges"]:
        got = b.dev[r.tptr - b.base:r.tptr - b.base + r.n].cpu().numpy()
        assert np.array_equal(got, h[r.hoff:r.hoff + r.n])


# --------------------------------------------------------------- parity, zero PCIe --


@gpu
@pytest.mark.parametrize("variant", VARIANTS, ids=["lsu", "tma"])
@pytest.mark.parametrize("chunk", [4096, 0])
def test_rollback_scatters_the_image_with_no_dma(cuda_device, variant, chunk):
    lay = _layout(3, chunk or DEFAULT_CHUNK)
    with _world(_context("default", variant), lay, chunk, variant) as w:
        t = w.plans["Q"]["tables"]
        if variant == native.VARIANT_TMA:
            assert all(t[k] for k in ("bulk", "resid", "shift"))
        w.save()
        w.check("save")
        _scribble(lay.src, 1)  # training went on
        w.check("sources overwritten")
        _rollback(w, "Q")
        _targets_hold_the_segment(w, "Q")
        # the sources themselves come back (the tied copy writes the same bytes twice)
        _rollback(w, "P")
        _targets_hold_the_segment(w, "P")
        _scribble(lay.tgt, 2)
        _rollback(w, "Q")  # the image is kept: roll back as often as wanted
        _targets_hold_the_segment(w, "Q")


# ------------------------------------------------------------------- record rules --


@gpu
def test_image_record_follows_every_event(cuda_device):
    lay = _layout(5, 64 << 10)
    variant = native.VARIANT_TMA
    with _world(_context("default", variant), lay, 64 << 10, variant, spare=8192) as w:
        stream = torch.cuda.current_stream()
        addr = w.host_t["A"].data_ptr()
        _rollback(w, expect=False)  # nothing saved yet

        def forgotten(what, op):
            w.save()
            _rollback(w)
            _scribble(lay.tgt, sum(map(ord, what)))
            op()
            _rollback(w, expect=False)

        forgotten("pack", w.pack)
        forgotten("unpack", w.unpack)
        forgotten("arena_fill", w.arena_fill)
        forgotten("save_direct", w.save_direct)
        forgotten("save_hybrid", w.save_hybrid)
        forgotten("restore", w.restore)
        forgotten("arena_tensor", lambda: w.ctx.arena_tensor(w.room))
        forgotten("invalidate", w.ctx.delta_invalidate)
        forgotten("cancel_held", lambda: w.delta(hold=True))

        # a held full save that is cancelled leaves no image either
        w.save()
        ticket = w.plans["P"]["plan"].save_async(addr, stream, hold=True)
        torch.cuda.synchronize()
        w.arena = w._gathered("P")
        # queued, not drained: refused as busy, the arena is not read
        with pytest.raises(native.NativeBusy):
            w.plans["Q"]["plan"].restore_from_image_async(addr, stream)
        assert w.ctx.save_cancel(ticket)
        w.ctx.save_wait(ticket)
        w._forget()
        _rollback(w, expect=False)

        # a held save: busy until released and drained, then the image is set
        ticket = w.plans["P"]["plan"].save_async(addr, stream, hold=True)
        torch.cuda.synchronize()
        w.arena = w._gathered("P")
        with pytest.raises(native.NativeBusy):
            w.plans["Q"]["plan"].restore_from_image_async(addr, stream)
        w.ctx.save_release(ticket)
        w.ctx.save_wait(ticket)
        w._drain(w.plans["P"]["runs"], "A")
        w._forget()
        _rollback(w)

        # incremental saves set it, full and delta; a rollback keeps it
        w.delta()
        _rollback(w)
        src = lay.src
        lf = next(lf for lf in lay.leaves if lf.n)
        src.write(src.base + lf.s, src.read(src.base + lf.s, 1) + 1)
        w.delta()
        _rollback(w)
        _rollback(w)

        # re-targeting the tensors only keeps it; moving a range forgets it
        w.update(dict(w.moved))
        _rollback(w)
        k = next(i for i, lf in enumerate(lay.leaves) if lf.n == 4097)
        w.update({k: lay.arena_end + 37})
        _rollback(w, expect=False)
        w.update({})
        _rollback(w, expect=False)  # back home, but the record is gone
        w.delta()
        _rollback(w)

        # destroying the image plan forgets it
        w.recreate()
        _rollback(w, expect=False)

        # the image of another plan: Q's own save covers Q, not P (P has a tied copy
        # past Q's last range); another host buffer is not this one
        w.delta("Q", "A")
        _rollback(w, "Q")
        _rollback(w, "P", expect=False)
        w.delta("P", "B")
        _rollback(w, "Q", "A", expect=False)
        _rollback(w, "Q", "B")

        # arena reallocation: nothing to scatter, nothing enqueued
        k0, m0 = w.ctx.launch_count()
        w.ctx.arena_reserve(w.room + (4 << 20))
        assert not w.plans["Q"]["plan"].restore_from_image_async(w.host_t["B"].data_ptr(), stream)
        torch.cuda.synchronize()
        assert w.ctx.launch_count() == (k0, m0)
        w.lay.tgt.check("targets after a refused rollback")


# ----------------------------------------------------------------------- coverage --


def _sub_plan(w, keep, moved=0, host_shift=0, at=None):
    """A plan over the target leaves `keep` (indices into Q's ranges): arena offsets
    moved by `moved`, segment offsets by `host_shift` (at: both sides at that offset)."""
    rs = [w.plans["Q"]["ranges"][i] for i in keep]
    aoffs = [r.aoff + moved if at is None else at for r in rs]
    hoffs = [r.hoff + host_shift if at is None else at for r in rs]
    plan = w.ctx.plan([r.tptr for r in rs], aoffs, [r.n for r in rs], w.chunk,
                      host_offsets=hoffs)
    return plan, rs


@gpu
def test_coverage_of_subsets_and_refusals(cuda_device):
    lay = _layout(7)
    variant = native.VARIANT_TMA
    stream = torch.cuda.current_stream()
    with _world(_context("default", variant), lay, 0, variant, spare=1 << 20) as w:
        addr = w.host_t["A"].data_ptr()
        w.save()
        _scribble(lay.tgt, 3)
        n = len(w.plans["Q"]["ranges"])
        small = next(i for i, r in enumerate(w.plans["Q"]["ranges"]) if 0 < r.n < (64 << 10))

        # half of the leaves (strict=False, one sub-dict): covered
        half = list(range(0, n, 2))
        plan, rs = _sub_plan(w, half)
        try:
            k0, m0 = w.ctx.launch_count()
            assert plan.image_covers(addr)
            assert plan.restore_from_image_async(addr, stream)
            w.ctx.restore_wait()
            torch.cuda.synchronize()
            k1, m1 = w.ctx.launch_count()
            assert m1 == m0
            assert k1 - k0 == pm.kernel_count(pm.tables(pm.items(rs, DEFAULT_CHUNK)), variant)
            b = lay.tgt
            for r in rs:
                b.np[r.tptr - b.base:r.tptr - b.base + r.n] = w.host["A"][r.hoff:r.hoff + r.n]
            w.check("half of the leaves")
        finally:
            plan.destroy()

        refusals = {
            # arena and segment moved together past the end of the image
            "outside": dict(keep=[small], at=lay.arena_end + 64),
            # the arena side moved, the segment side not
            "moved": dict(keep=half, moved=16),
            # a mapped plan whose arena offsets differ from its segment offsets
            "mapped": dict(keep=half, host_shift=4096),
        }
        for what, kw in refusals.items():
            plan, _ = _sub_plan(w, **kw)
            try:
                k0 = w.ctx.launch_count()
                assert not plan.image_covers(addr), what
                assert not plan.restore_from_image_async(addr, stream), what
                torch.cuda.synchronize()
                assert w.ctx.launch_count() == k0, what
            finally:
                plan.destroy()
            w.check(what)
        _rollback(w)  # nothing above forgot the image

        # saves that leave no image
        for what, op in (("hybrid", w.save_hybrid), ("in place", w.save_direct)):
            w.save()
            op()
            _rollback(w, expect=False)


@gpu
def test_bounded_arena_save_leaves_no_image(cuda_device):
    lay = _layout(9, target=12 << 20)
    variant = native.VARIANT_TMA
    with _world(_context("default", variant, 8 << 20), lay, 0, variant, bounded=True) as w:
        assert w.ctx.arena_info()[1] == 8 << 20 < lay.arena_end
        w.save()
        plan = w.plans["Q"]["plan"]
        k0 = w.ctx.launch_count()
        assert not plan.image_covers(w.host_t["A"].data_ptr())
        assert not plan.restore_from_image_async(w.host_t["A"].data_ptr(),
                                                 torch.cuda.current_stream())
        torch.cuda.synchronize()
        assert w.ctx.launch_count() == k0
        w.check("bounded save, refused rollback")


@gpu
@pytest.mark.parametrize("variant", VARIANTS, ids=["lsu", "tma"])
def test_mapped_plan_rolls_back_through_itself(cuda_device, variant):
    lay = _layout(11, 64 << 10, mapped=True)
    with _world(_context("default", variant), lay, 64 << 10, variant) as w:
        assert any(r.aoff != r.hoff for r in w.plans["P"]["ranges"])
        w.save()
        _scribble(lay.src, 4)
        _rollback(w, "P")
        _targets_hold_the_segment(w, "P")
        _rollback(w, "Q")
        _targets_hold_the_segment(w, "Q")


# ------------------------------------------------------------- incremental interplay --


@gpu
@pytest.mark.parametrize("variant", VARIANTS, ids=["lsu", "tma"])
def test_delta_save_after_a_rollback_drains_nothing(cuda_device, variant):
    lay = _layout(13, 64 << 10)
    with _world(_context("default", variant), lay, 64 << 10, variant) as w:
        w.delta()  # full: the baseline and the image
        w.check("baseline")
        rng = np.random.default_rng(1)
        src = lay.src
        big = [lf for lf in lay.leaves if lf.n > 100_000][:3]
        for lf in big:  # train: three leaves change
            src.write(src.base + lf.s, rng.integers(0, 256, lf.n, dtype=np.uint8))
        _rollback(w, "P")  # the sources are the checkpoint again
        assert w.base == ("P", "A")
        k0, m0 = w.ctx.launch_count()
        ticket = w.plans["P"]["plan"].save_delta_async(w.host_t["A"].data_ptr(),
                                                      torch.cuda.current_stream())
        w.ctx.save_wait(ticket)
        assert w.ctx.save_delta_stats(ticket) == (True, 0)
        assert w.ctx.launch_count()[1] == m0
        w.check("delta save after the rollback")
        # one leaf changes: exactly its dirty items drain (World.delta asserts the model)
        src.write(src.base + big[0].s + 5, src.read(src.base + big[0].s + 5, 1) + 1)
        w.delta()
        w.check("one byte after the rollback")


# ------------------------------------------------------------------ handler and API --


def _tree_tensors(tree, prefix=""):
    if isinstance(tree, dict):
        for k, v in tree.items():
            yield from _tree_tensors(v, f"{prefix}{k}.")
    elif isinstance(tree, (list, tuple)):
        for i, v in enumerate(tree):
            yield from _tree_tensors(v, f"{prefix}{i}.")
    elif torch.is_tensor(tree):
        yield prefix, tree


def _state(model, opt, cpu):
    return {"model": model.state_dict(), "optim": opt.state_dict(), "cpu": cpu}


def _clone(tree):
    return {k: t.clone() for k, t in _tree_tensors(tree)}


def _scribble_tree(tree):
    with torch.no_grad():
        for _, t in _tree_tensors(tree):
            t.copy_(torch.full_like(t, 3) if t.dtype != torch.bool else torch.ones_like(t))


def _same(tree, want):
    got = dict(_tree_tensors(tree))
    assert sorted(got) == sorted(want)
    for k, t in got.items():
        a, b = (x.detach().cpu().contiguous().reshape(-1) for x in (t, want[k]))
        assert a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8)), k


def _train(model, opt, x, steps):
    for _ in range(steps):
        model(x).square().mean().backward()
        opt.step()
        opt.zero_grad()


def _engine_rollback(ckpt, tree):
    from dlrover_b200.common.constants import CheckpointConstant

    return ckpt.engine.rollback_into({CheckpointConstant.MODEL_STATES_NAME: tree})


def _run(ckpt, steps_before=5, steps_after=3):
    """Train, save to memory at step `steps_before`, train on; returns the live tree and
    a copy of it at the save."""
    from dlrover_b200.flash_checkpoint.api import StorageType
    from tests.test_incremental_save import _Adapted

    torch.manual_seed(0)
    model = _Adapted().cuda()
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-2)
    x = torch.randn(32, 1024, device="cuda")
    cpu = torch.arange(1000, dtype=torch.float64)
    _train(model, opt, x, steps_before)
    tree = _state(model, opt, cpu)
    assert any(not t.is_cuda for _, t in _tree_tensors(tree["optim"]))  # AdamW's step
    ckpt.save_checkpoint(steps_before, tree, storage_type=StorageType.MEMORY)
    assert ckpt.wait_memory_save(60)
    at_save = _clone(tree)
    _train(model, opt, x, steps_after)
    cpu.mul_(-1)
    return model, opt, x, tree, at_save


@gpu
def test_ddp_checkpointer_rolls_back_from_hbm(cuda_device, run_env, tmp_path):
    from dlrover_b200.ckpt_saver import AsyncCheckpointSaver
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType

    AsyncCheckpointSaver.start_async_saving_ckpt()
    ckpt = DdpCheckpointer(str(tmp_path / "a"))
    handler = ckpt.engine._shm_handler
    try:
        model, opt, x, tree, at_save = _run(ckpt)
        assert ckpt.rollback_into(tree) == 5
        assert handler.last_restore_stats["from_image"] == 1.0
        assert handler.last_restore_stats["fill_ms"] == 0.0
        _same(tree, at_save)
        _scribble_tree(tree)
        step, stats = _engine_rollback(ckpt, tree)  # the engine's form, stats included
        assert step == 5 and stats["from_image"] == 1.0 and stats["host_bytes"] > 0
        _same(tree, at_save)

        # the same checkpoint over PCIe gives the same bytes
        _scribble_tree(tree)
        assert ckpt.load_checkpoint_into(tree) == 5
        _same(tree, at_save)
        assert handler.last_restore_stats.get("from_image") is None

        # a restore rewrote the arena: the rollback falls back, same bytes
        _scribble_tree(tree)
        step, stats = _engine_rollback(ckpt, tree)
        assert step == 5 and stats["from_image"] == 0.0
        _same(tree, at_save)

        # incremental saves: after a rollback, the next save drains only what changed
        ckpt.engine.incremental = True
        ckpt.save_checkpoint(6, tree, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        assert ckpt.engine.last_save_stats()["delta"] is False
        at6 = _clone(tree)
        _train(model, opt, x, 2)
        assert ckpt.rollback_into(tree) == 6
        assert handler.last_restore_stats["from_image"] == 1.0
        _same(tree, at6)
        ckpt.save_checkpoint(7, tree, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        assert ckpt.engine.last_save_stats() == {"delta": True, "drained_bytes": 0}
        _train(model, opt, x, 1)  # the adapter and its moments change, the base not
        ckpt.save_checkpoint(8, tree, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        adapter = sum(p.numel() * p.element_size() for p in (model.down.weight, model.up.weight))
        moments = sum(v.numel() * v.element_size() for s in opt.state.values()
                      for v in s.values() if torch.is_tensor(v) and v.is_cuda)
        changed = 2 + sum(1 for s in opt.state.values() for v in s.values()
                          if torch.is_tensor(v) and v.is_cuda)
        stats = ckpt.engine.last_save_stats()
        assert stats["delta"] is True
        assert 0 < stats["drained_bytes"] <= adapter + moments + changed * (256 << 10), stats
    finally:
        ckpt.engine.close()


@gpu
def test_in_place_saves_fall_back_to_the_segment(cuda_device, run_env, tmp_path, monkeypatch):
    from dlrover_b200.ckpt_saver import AsyncCheckpointSaver
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer

    monkeypatch.setenv("DLROVER_B200_IN_PLACE", "1")
    AsyncCheckpointSaver.start_async_saving_ckpt()
    ckpt = DdpCheckpointer(str(tmp_path / "b"))
    handler = ckpt.engine._shm_handler
    try:
        assert handler.in_place
        _, _, _, tree, at_save = _run(ckpt)
        assert handler.last_save_in_place
        step, stats = _engine_rollback(ckpt, tree)
        assert step == 5 and stats["from_image"] == 0.0
        _same(tree, at_save)
    finally:
        ckpt.engine.close()


# --------------------------------------------------------------- CPU (no GPU needed) --


def test_rollback_entry_points_reject_null_arguments():
    lib = native.load_library()
    assert lib.fc_restore_from_image_async(None, None, None) == native.FC_EINVAL
    assert b"fc_restore_from_image_async" in lib.fc_last_error()
    assert lib.fc_restore_from_image_async(None, ctypes.c_void_p(4096), None) == native.FC_EINVAL
    assert lib.fc_image_covers(None, None) == native.FC_EINVAL
    assert b"fc_image_covers" in lib.fc_last_error()


def test_strerror_names_the_missing_image():
    lib = native.load_library()
    text = lib.fc_strerror(native.FC_ENOIMAGE)
    assert text and b"image" in text and text != lib.fc_strerror(-99)


def test_a_tree_without_cuda_leaves_cannot_roll_back(run_env):
    """CheckpointEngine.rollback_into sends such a tree to load_into."""
    from dlrover_b200.shm_handler import DLROVER_CKPT_CONFIG_KEY, CheckpointConfig
    from dlrover_b200.shm_handler import SharedMemoryHandler

    handler = SharedMemoryHandler(0, host=True)
    tree = {"w": torch.arange(1000, dtype=torch.float32), "step": torch.tensor(5)}
    try:
        handler.save_state_dict({"model_states": tree, DLROVER_CKPT_CONFIG_KEY:
                                 CheckpointConfig(step=5, paths={"model_states": "/x/rank_0.pt"})})
        assert handler.can_rollback({"model_states": tree}) is False
        stats = handler.restore_into({"model_states": tree})  # the same tree does restore
        assert stats["host_bytes"] == 4008 and stats["device_bytes"] == 0.0
    finally:
        handler.unlink()
        handler.close()


def _gloo_worker(rank, world, port, run_id, ckpt_dir, out_dir, images):
    import sys

    import torch.distributed as dist

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    os.environ.update({
        "RANK": str(rank), "LOCAL_RANK": str(rank), "WORLD_SIZE": str(world),
        "LOCAL_WORLD_SIZE": str(world), "GROUP_WORLD_SIZE": "1", "GROUP_RANK": "0",
        "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "TORCHELASTIC_RUN_ID": run_id,
        "DLROVER_LOG_LEVEL": "WARNING",
    })
    os.environ.pop("ROLE_NAME", None)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType

    result = {"calls": []}
    try:
        ckpt = DdpCheckpointer(ckpt_dir, local_shard_num=world, global_shard_num=world)
        eng = ckpt.engine
        handler = eng._shm_handler
        sd = {"w": torch.full((1000,), float(rank + 1))}
        ckpt.save_checkpoint(3, sd, storage_type=StorageType.MEMORY)
        sd["w"].fill_(-1.0)
        # the image path itself needs a GPU: mock it, keep the decision and load_into real
        handler.can_rollback = lambda target, strict=True: images[rank]
        handler.rollback_into = lambda target, stream=None, strict=True: (
            result["calls"].append("image"), {"from_image": 1.0})[1]
        load_into = eng.load_into

        def spy(*a, **k):
            result["calls"].append("load_into")
            return load_into(*a, **k)

        eng.load_into = spy
        result["step"] = ckpt.rollback_into(sd)
        result["restored"] = bool(torch.equal(sd["w"], torch.full((1000,), float(rank + 1))))
        dist.barrier()
        eng.close()
    finally:
        torch.save(result, os.path.join(out_dir, f"r{rank}.pt"))
        dist.destroy_process_group()


def _gloo_run(images):
    import glob
    import shutil
    import tempfile
    import uuid

    import torch.multiprocessing as mp

    world = 2
    run_id = "rb" + uuid.uuid4().hex[:8]
    port = 29600 + (os.getpid() * 11 + sum(images) * 7) % 1500
    with tempfile.TemporaryDirectory() as ckpt_dir, tempfile.TemporaryDirectory() as out_dir:
        mp.spawn(_gloo_worker, args=(world, port, run_id, ckpt_dir, out_dir, images),
                 nprocs=world, join=True)
        results = [torch.load(os.path.join(out_dir, f"r{r}.pt")) for r in range(world)]
    shutil.rmtree(os.path.join("/tmp/ckpt_sock", run_id), ignore_errors=True)
    for f in glob.glob(f"/dev/shm/{run_id}_*"):
        os.unlink(f)
    return results


@pytest.mark.timeout(300)
def test_one_rank_without_image_sends_every_rank_to_load_into():
    for res in _gloo_run((True, False)):
        assert res["calls"] == ["load_into"]
        assert res["step"] == 3 and res["restored"]


@pytest.mark.timeout(300)
def test_every_rank_with_an_image_rolls_back_from_it():
    for res in _gloo_run((True, True)):
        assert res["calls"] == ["image"]
        assert res["step"] == 3
