"""Rolling a sharded (DCP) checkpoint back from the HBM snapshot of its own last memory
save: FsdpCheckpointEngine.rollback_reader / RollbackReader and
FsdpShardCheckpointer.rollback_checkpoint.

The GPU tests check the bytes against the state at the save and against the restore over
PCIe (load / load_checkpoint), and which path each dcp.load pass took.  The CPU tests run
two gloo ranks with the image path mocked, to check that every rank takes the same path."""

import contextlib
import os
import time

import pytest
import torch
import torch.distributed as dist
import torch.distributed.checkpoint as dist_cp
import torch.nn as nn

from dlrover_b200 import _native as native
from dlrover_b200.ckpt_saver import AsyncCheckpointSaver
from dlrover_b200.common.storage import PosixDiskStorage
from dlrover_b200.flash_checkpoint import fsdp_engine as fe

gpu = pytest.mark.gpu


@pytest.fixture
def gloo(run_env, monkeypatch):
    monkeypatch.setenv("MASTER_ADDR", "127.0.0.1")
    monkeypatch.setenv("MASTER_PORT", str(29500 + (os.getpid() * 7) % 2000))
    for k, v in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0"),
                 ("LOCAL_WORLD_SIZE", "1")):
        monkeypatch.setenv(k, v)
    dist.init_process_group("gloo", rank=0, world_size=1)
    AsyncCheckpointSaver.start_async_saving_ckpt()
    yield
    dist.destroy_process_group()


@pytest.fixture
def nccl(cuda_device, run_env, monkeypatch):
    monkeypatch.setenv("MASTER_ADDR", "127.0.0.1")
    monkeypatch.setenv("MASTER_PORT", str(27500 + (os.getpid() * 13) % 1500))
    for k, v in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0"),
                 ("LOCAL_WORLD_SIZE", "1")):
        monkeypatch.setenv(k, v)
    yield  # the test sets its switches first: the handler reads them when it is built
    if dist.is_initialized():
        dist.destroy_process_group()


def _start_nccl():
    dist.init_process_group("nccl", rank=0, world_size=1)
    AsyncCheckpointSaver.start_async_saving_ckpt()


def _bits(t):
    return t.detach().cpu().contiguous().reshape(-1).view(torch.uint8)


def _same(got, want):
    assert sorted(got) == sorted(want)
    for k in got:
        assert torch.equal(_bits(got[k]), _bits(want[k])), k


# ------------------------------------------------------------ engine, DCP tree --


def _tree(device):
    g = torch.Generator().manual_seed(0)

    def rnd(*shape, dtype=torch.float32):
        return torch.randn(shape, generator=g).to(dtype).to(device)

    return {"model": {"w": rnd(37, 129, dtype=torch.bfloat16), "b": rnd(1001),
                      "cube": rnd(3, 5, 7, dtype=torch.bfloat16), "scale": rnd()},
            "optim": {"m": rnd(333, 3), "v": rnd(17, dtype=torch.bfloat16)},
            "step": 7}


def _tensors(tree):
    return {f"{a}.{b}": t for a, sub in tree.items() if isinstance(sub, dict)
            for b, t in sub.items()}


def _scribble(tree):
    for t in _tensors(tree).values():
        t.fill_(3)
    tree["step"] = 0


def _load(tree, reader):
    dist_cp.load(tree, storage_reader=reader)
    assert tree["step"] == 7


@gpu
def test_engine_rolls_back_from_the_image(cuda_device, gloo, tmp_path):
    engine = fe.FsdpCheckpointEngine(str(tmp_path), PosixDiskStorage(), async_drain=True)
    handler = engine._shm_handler
    try:
        sd = _tree(cuda_device)
        assert engine.save_to_memory(5, sd, {"model_states": str(tmp_path / "5")})
        assert engine.wait_memory_save(60)
        want = {k: t.clone() for k, t in _tensors(sd).items()}
        # every tensor but the 0-dim one is a whole stored chunk: a fast item
        fast = [t for t in _tensors(sd).values() if t.dim()]
        fast_bytes = float(sum(t.numel() * t.element_size() for t in fast))

        for _ in range(2):  # a rollback keeps the image: roll back as often as wanted
            _scribble(sd)
            reader = engine.rollback_reader()
            assert isinstance(reader, fe.RollbackReader)
            _load(sd, reader)
            _same(_tensors(sd), want)
            st = reader.last_read_stats
            assert st["from_image"] == 1.0 and st["fill_ms"] == 0.0, st
            assert st["device_bytes"] == fast_bytes and st["fast_items"] == len(fast)
            assert st["slow_items"] == 2  # the 0-dim leaf and the "step" object
            assert st["scatter_ms"] >= 0.0 and st["wall_ms"] > 0.0
            assert engine.last_rollback_stats() == [st]

        # the same checkpoint over PCIe, through load()
        _scribble(sd)
        reader = engine.load()
        assert type(reader) is fe.SharedMemoryReader
        _load(sd, reader)
        _same(_tensors(sd), want)
        assert "from_image" not in handler.last_restore_stats

        # that restore rewrote the arena: the rollback reads the segment, same bytes
        _scribble(sd)
        reader = engine.rollback_reader()
        _load(sd, reader)
        _same(_tensors(sd), want)
        st = reader.last_read_stats
        assert st["from_image"] == 0.0 and st["device_bytes"] == fast_bytes, st

        # incremental saves: after a rollback, with nothing changed since, the next save
        # finds its baseline and drains nothing
        engine.incremental = True
        assert engine.save_to_memory(6, sd, {"model_states": str(tmp_path / "6")})
        assert engine.wait_memory_save(60)
        assert engine.last_save_stats()["delta"] is False  # the restore forgot the baseline
        _scribble(sd)
        reader = engine.rollback_reader()
        _load(sd, reader)
        assert reader.last_read_stats["from_image"] == 1.0
        _same(_tensors(sd), want)
        assert engine.save_to_memory(7, sd, {"model_states": str(tmp_path / "7")})
        assert engine.wait_memory_save(60)
        assert engine.last_save_stats() == {"delta": True, "drained_bytes": 0}
    finally:
        engine.close()


def _cpu_engine(tmp_path):
    """An engine holding _tree("cpu") in memory at step 5, with a copy of its tensors."""
    engine = fe.FsdpCheckpointEngine(str(tmp_path), PosixDiskStorage(), async_drain=False)
    sd = _tree("cpu")
    assert engine.save_to_memory(5, sd, {"model_states": str(tmp_path / "5")})
    assert engine.wait_memory_save(60)
    return engine, sd, {k: t.clone() for k, t in _tensors(sd).items()}


def test_the_memory_reader_takes_no_vote(gloo, tmp_path, monkeypatch):
    engine, sd, want = _cpu_engine(tmp_path)
    try:
        reader = engine.load()
        assert type(reader) is fe.SharedMemoryReader

        def collective(*args, **kwargs):
            raise AssertionError("load()'s reader must not take part in a collective")

        monkeypatch.setattr(fe, "vote_all_ranks", collective)
        monkeypatch.setattr(fe, "all_reduce_flags", collective)
        _scribble(sd)
        _load(sd, reader)
        _same(_tensors(sd), want)
    finally:
        engine.close()


def test_each_rollback_pass_takes_one_vote(gloo, tmp_path, monkeypatch):
    engine, sd, want = _cpu_engine(tmp_path)
    votes = []
    vote = fe.vote_all_ranks

    def counted(group, check):
        votes.append(group)
        return vote(group, check)

    monkeypatch.setattr(fe, "vote_all_ranks", counted)
    try:
        reader = engine.rollback_reader()
        for n in (1, 2):  # two dcp.load passes through one reader, as rollback_checkpoint
            _scribble(sd)
            _load(sd, reader)
            _same(_tensors(sd), want)
            assert len(votes) == len(engine.last_rollback_stats()) == n
        # CPU targets are no fast items: this rank is covered and reads nothing from HBM
        st = reader.last_read_stats
        assert st["fast_items"] == 0 and st["from_image"] == 1.0 and st["device_bytes"] == 0.0
    finally:
        engine.close()


# ------------------------------------------------------------- a real FSDP job --


class _Net(nn.Module):
    def __init__(self, hidden=128):
        super().__init__()
        self.a = nn.Linear(64, hidden)
        self.b = nn.Linear(hidden, 32)

    def forward(self, x):
        return self.b(torch.relu(self.a(x)))


def _job(device, hidden=128):
    from torch.distributed.fsdp import FullyShardedDataParallel as FSDP

    torch.manual_seed(0)
    model = FSDP(_Net(hidden).to(device), device_id=device)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-2)
    return model, opt, torch.randn(8, 64, device=device)


def _train(model, opt, x, steps):
    for _ in range(steps):
        model(x).square().mean().backward()
        opt.step()
        opt.zero_grad()


def _job_state(model, opt):
    """Every parameter and optimizer-state tensor of the job, by position."""
    out = {f"param{i}": p for i, p in enumerate(model.parameters())}
    for i, p in enumerate(opt.param_groups[0]["params"]):
        for name, v in opt.state[p].items():
            if torch.is_tensor(v):
                out[f"state{i}.{name}"] = v
    return out


def _snapshot(model, opt):
    return {k: t.detach().clone() for k, t in _job_state(model, opt).items()}


@gpu
def test_fsdp_checkpointer_rolls_back_from_hbm(cuda_device, nccl, tmp_path):
    from dlrover_b200.flash_checkpoint.api import StorageType
    from dlrover_b200.flash_checkpoint.fsdp import FsdpShardCheckpointer

    _start_nccl()
    ckpt = FsdpShardCheckpointer(str(tmp_path))
    engine = ckpt.engine
    try:
        model, opt, x = _job(cuda_device)
        _train(model, opt, x, 3)
        ckpt.save_checkpoint(3, model, opt, {"step": 3}, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        want = _snapshot(model, opt)
        _train(model, opt, x, 2)
        assert ckpt.rollback_checkpoint(model, opt).get("step") == 3
        model_pass, optim_pass = engine.last_rollback_stats()
        # the parameters: from the HBM image
        assert model_pass["from_image"] == 1.0 and model_pass["fill_ms"] == 0.0, model_pass
        assert model_pass["device_bytes"] > 0, model_pass
        # FSDP hands the sharded optimizer state over as host copies (its default
        # ShardedOptimStateDictConfig(offload_to_cpu=True)): it never was in the arena,
        # so that pass reads the segment
        assert optim_pass["from_image"] == 0.0 and optim_pass["device_bytes"] > 0, optim_pass
        _same(_job_state(model, opt), want)

        # load_checkpoint restores the same bytes
        _train(model, opt, x, 2)
        assert ckpt.load_checkpoint(model, opt).get("step") == 3
        _same(_job_state(model, opt), want)

        # a later save sets the image again: the rollback takes it for the parameters
        ckpt.save_checkpoint(4, model, opt, {"step": 4}, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        at4 = _snapshot(model, opt)
        _train(model, opt, x, 2)
        assert ckpt.rollback_checkpoint(model, opt).get("step") == 4
        assert [st["from_image"] for st in engine.last_rollback_stats()] == [1.0, 0.0]
        _same(_job_state(model, opt), at4)
    finally:
        engine.close()


@gpu
@pytest.mark.parametrize("mode", ["in_place", "bounded_arena"])
def test_saves_without_an_image_roll_back_from_the_segment(cuda_device, nccl, tmp_path,
                                                          monkeypatch, mode):
    """In-place saves leave no snapshot, bounded-arena saves stream through an arena
    smaller than the state: the rollback reads the segment, with load_checkpoint's bytes."""
    import dlrover_b200.shm_handler as sh
    from dlrover_b200.flash_checkpoint.api import StorageType
    from dlrover_b200.flash_checkpoint.fsdp import FsdpShardCheckpointer

    ctx = None
    if mode == "in_place":
        monkeypatch.setenv("DLROVER_B200_IN_PLACE", "1")
    else:  # a fresh context: an arena left by an earlier test would hold the whole state
        ctx = native.Context(0)
        monkeypatch.setattr(sh.native, "get_context", lambda index: ctx)
        monkeypatch.setenv("DLROVER_B200_ARENA_LIMIT_MB", "8")
    _start_nccl()
    ckpt = FsdpShardCheckpointer(str(tmp_path))
    engine = ckpt.engine
    try:
        model, opt, x = _job(cuda_device, hidden=24576)  # 9.4 MB of parameters
        _train(model, opt, x, 2)
        ckpt.save_checkpoint(2, model, opt, {"step": 2}, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        if mode == "in_place":
            assert engine._shm_handler.last_save_in_place
        else:
            assert ctx.arena_info()[1] == 8 << 20
        want = _snapshot(model, opt)
        _train(model, opt, x, 2)
        assert ckpt.rollback_checkpoint(model, opt).get("step") == 2
        passes = engine.last_rollback_stats()
        assert [st["from_image"] for st in passes] == [0.0, 0.0], passes
        _same(_job_state(model, opt), want)
        _train(model, opt, x, 2)
        assert ckpt.load_checkpoint(model, opt).get("step") == 2
        _same(_job_state(model, opt), want)
    finally:
        engine.close()
        if ctx is not None:
            ctx.destroy()


# --------------------------------------------------------------- CPU, two ranks --


def _gloo_worker(rank, world, port, run_id, ckpt_dir, out_dir, fast, covered):
    import sys

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    os.environ.update({
        "RANK": str(rank), "LOCAL_RANK": str(rank), "WORLD_SIZE": str(world),
        "LOCAL_WORLD_SIZE": str(world), "GROUP_WORLD_SIZE": "1", "GROUP_RANK": "0",
        "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "TORCHELASTIC_RUN_ID": run_id,
        "DLROVER_LOG_LEVEL": "WARNING",
    })
    os.environ.pop("ROLE_NAME", None)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from torch.distributed.checkpoint.planner import LoadItemType
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import Shard, distribute_tensor

    from dlrover_b200.flash_checkpoint import fsdp as fsdp_mod

    result = {"calls": []}
    try:
        ckpt = fsdp_mod.FsdpShardCheckpointer(ckpt_dir)
        engine = ckpt.engine
        if fast is None:  # nothing in memory
            result["reader"] = engine.rollback_reader()
            # a plain module: the checkpointer returns before anything FSDP-specific
            fsdp_mod.FSDP.state_dict_type = lambda *a, **k: contextlib.nullcontext()
            result["extra"] = ckpt.rollback_checkpoint(nn.Linear(2, 2), None)
            return
        mesh = init_device_mesh("cpu", (world,))
        full = torch.arange(4000, dtype=torch.float32).reshape(40, 100)
        w = distribute_tensor(full, mesh, [Shard(0)])
        sd = {"model": {"w": w}, "step": 3}
        assert engine.save_to_memory(3, sd, {"model_states": os.path.join(ckpt_dir, "3")})
        assert engine.wait_memory_save(60)
        w.to_local().fill_(-1.0)
        sd["step"] = 0
        handler = engine._shm_handler
        reader = engine.rollback_reader()
        if fast[rank]:
            # CPU targets stand in for CUDA ones: this rank's shard is a fast item
            reader._device_fast_path = lambda item, info, planner: (
                (planner.resolve_tensor(item).detach(), info.offset, info.length)
                if item.type != LoadItemType.BYTE_IO and item.storage_index.offset else None)
            handler.image_covers_ranges = lambda ranges: covered[rank]

        def read_ranges(ranges, stream=None, *, image_first=False):
            result["calls"].append("image" if image_first else "segment")
            for t, off, n in ranges:
                src = bytes(handler.shared_memory.buf[off:off + n])
                t.reshape(-1).view(torch.uint8).copy_(torch.frombuffer(src, dtype=torch.uint8))
            return {"device_bytes": float(sum(n for _, _, n in ranges)), "fill_ms": 0.0,
                    "scatter_ms": 0.0, "from_image": float(image_first)}

        handler.read_ranges = read_ranges
        dist_cp.load(sd, storage_reader=reader)
        half = full.shape[0] // world
        result["restored"] = bool(torch.equal(w.to_local(), full[rank * half:(rank + 1) * half]))
        result["step"] = sd["step"]
        result["stats"] = dict(reader.last_read_stats)
        dist.barrier()
        engine.close()
    finally:
        torch.save(result, os.path.join(out_dir, f"r{rank}.pt"))
        dist.destroy_process_group()


def _gloo_run(fast, covered):
    import glob
    import shutil
    import tempfile
    import uuid

    import torch.multiprocessing as mp

    world = 2
    run_id = "frb" + uuid.uuid4().hex[:8]
    port = 28000 + (os.getpid() * 17 + int(time.time() * 1000)) % 1500
    with tempfile.TemporaryDirectory() as ckpt_dir, tempfile.TemporaryDirectory() as out_dir:
        mp.spawn(_gloo_worker, args=(world, port, run_id, ckpt_dir, out_dir, fast, covered),
                 nprocs=world, join=True)
        results = [torch.load(os.path.join(out_dir, f"r{r}.pt")) for r in range(world)]
    shutil.rmtree(os.path.join("/tmp/ckpt_sock", run_id), ignore_errors=True)
    for f in glob.glob(f"/dev/shm/{run_id}_*"):
        os.unlink(f)
    return results


@pytest.mark.timeout(300)
def test_one_uncovered_rank_sends_every_rank_to_the_segment():
    for res in _gloo_run((True, True), (True, False)):
        assert res["calls"] == ["segment"], res
        assert res["stats"]["from_image"] == 0.0 and res["restored"] and res["step"] == 3


@pytest.mark.timeout(300)
def test_every_rank_covered_reads_from_the_image():
    for res in _gloo_run((True, True), (True, True)):
        assert res["calls"] == ["image"], res
        assert res["stats"]["from_image"] == 1.0 and res["restored"] and res["step"] == 3
        assert res["stats"]["fast_items"] == 1 and res["stats"]["device_bytes"] == 20 * 100 * 4


@pytest.mark.timeout(300)
def test_a_rank_without_fast_items_does_not_block_the_image_path():
    r0, r1 = _gloo_run((True, False), (True, None))
    assert r0["calls"] == ["image"] and r0["stats"]["from_image"] == 1.0, r0
    assert r1["calls"] == [] and r1["stats"]["fast_items"] == 0, r1
    assert r1["stats"]["from_image"] == 1.0 and r1["stats"]["device_bytes"] == 0.0
    assert r0["restored"] and r1["restored"] and r0["step"] == r1["step"] == 3


@pytest.mark.timeout(300)
def test_nothing_in_memory_gives_no_reader():
    for res in _gloo_run(None, None):
        assert res["reader"] is None and res["extra"] == {}, res
