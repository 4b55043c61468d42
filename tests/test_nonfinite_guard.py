"""Refusing memory saves of a non-finite state: the fc_scan_nonfinite kernel against
torch.isfinite, and the engine's decision point (a refused save leaves no trace: segment,
meta, tracker, HBM image and incremental baseline all stay as they were)."""

import os

import pytest
import torch

from dlrover_b200 import _native as native

gpu = pytest.mark.gpu

KINDS = {
    torch.float16: native.KIND_F16, torch.bfloat16: native.KIND_BF16,
    torch.float32: native.KIND_F32, torch.float64: native.KIND_F64,
    torch.complex64: native.KIND_F32, torch.complex128: native.KIND_F64,
    torch.float8_e5m2: native.KIND_E5M2, torch.float8_e4m3fn: native.KIND_E4M3FN,
}
ITEM = 256 << 10  # the scan's work-item size


def _expected(t: torch.Tensor) -> int:
    if t.dtype == torch.float8_e4m3fn:
        b = t.view(torch.uint8)
        return int(((b & 0x7F) == 0x7F).sum())
    if t.dtype in (torch.complex64, torch.complex128):
        t = torch.view_as_real(t)
    if t.element_size() == 1:
        t = t.float()
    return int((~torch.isfinite(t)).sum())


def _scan(ctx, tensors, kinds=None, ranges=None):
    """Per-range counts of one scan over `ranges` ((ptr, nbytes), default: the tensors)."""
    if ranges is None:
        ranges = [(t.data_ptr(), t.numel() * t.element_size()) for t in tensors]
    kinds = kinds if kinds is not None else [KINDS.get(t.dtype, native.KIND_NONE) for t in tensors]
    offs, o = [], 0
    for _, n in ranges:
        offs.append(o)
        o += n
    plan = ctx.plan([p for p, _ in ranges], offs, [n for _, n in ranges])
    try:
        plan.set_kinds(kinds)
        plan.scan_nonfinite_async(torch.cuda.current_stream())
        return plan.scan_wait(len(ranges))
    finally:
        plan.destroy()


def _specials(dtype):
    if dtype == torch.float8_e4m3fn:
        return [0x7F, 0xFF]  # its only non-finite patterns (NaN)
    f = torch.finfo(dtype if not dtype.is_complex else torch.empty(0, dtype=dtype).real.dtype)
    return [float("nan"), float("inf"), float("-inf")] if f else []


def _poke(t, i, v):
    if t.dtype == torch.float8_e4m3fn:
        t.view(torch.uint8)[i] = v
    else:
        t[i] = v


def _finite_edges(dtype, n, device):
    """n finite values that sit next to the non-finite patterns: max, -max, subnormals,
    -0, tiny; e4m3fn's 0x7E / 0xFE."""
    if dtype == torch.float8_e4m3fn:
        pat = torch.tensor([0x7E, 0xFE, 0x00, 0x80, 0x01, 0x77], dtype=torch.uint8)
        return pat.repeat(n // 6 + 1)[:n].view(dtype).to(device)
    real = torch.empty(0, dtype=dtype).real.dtype if dtype.is_complex else dtype
    fi = torch.finfo(real)
    vals = torch.tensor([fi.max, -fi.max, fi.smallest_normal / 4, -0.0, fi.tiny, 1.0],
                        dtype=torch.float64)
    vals = vals.repeat(n // 6 + 1)[:n]
    if dtype.is_complex:
        return torch.complex(vals, vals.flip(0)).to(dtype).to(device)
    return vals.to(real).to(device)


@gpu
@pytest.mark.parametrize("dtype", list(KINDS), ids=str)
def test_counts_match_isfinite(cuda_device, dtype):
    ctx = native.get_context(0)
    es = torch.empty(0, dtype=dtype).element_size()
    n = 3 * ITEM // es + 7  # three items and a tail
    base = _finite_edges(dtype, n + 64, cuda_device)
    specials = _specials(dtype)
    tensors = []
    # 0: whole tensor with specials at the ends and on both sides of every item boundary
    t = base[:n].clone()
    spots = [0, n - 1] + [k * ITEM // es + d for k in (1, 2, 3) for d in (-1, 0)]
    for j, i in enumerate(spots):
        if i < n:
            _poke(t, i, specials[j % len(specials)])
    tensors.append(t)
    # 1..3: sources at odd element offsets (not 16-B aligned), specials at the ends
    for shift in (1, 3, 5):
        u = base.clone()[shift:shift + n - 11]
        _poke(u, 0, specials[0])
        _poke(u, u.numel() - 1, specials[-1])
        _poke(u, u.numel() // 2, specials[shift % len(specials)])
        tensors.append(u)
    # 4, 5: leaves smaller than 16 B, one clean, one with a special
    small = base.clone()[1:1 + max(1, 8 // es)]
    tensors.append(small)
    bad_small = base.clone()[1:1 + max(1, 8 // es)]
    _poke(bad_small, 0, specials[-1])
    tensors.append(bad_small)
    # 6: only finite edge values
    tensors.append(base.clone())
    total, counts = _scan(ctx, tensors)
    want = [_expected(x) for x in tensors]
    assert counts == want
    assert total == sum(want) and want[0] >= len(spots) - 1 and want[-1] == 0


@gpu
def test_integers_and_bytes_are_not_scanned(cuda_device):
    ctx = native.get_context(0)
    tensors = [torch.full((1 << 16,), 255, dtype=torch.uint8, device="cuda"),
               torch.full((4097,), -1, dtype=torch.int32, device="cuda"),
               torch.full((33,), -1, dtype=torch.int64, device="cuda"),
               torch.ones(100, dtype=torch.bool, device="cuda")]
    total, counts = _scan(ctx, tensors)
    assert total == 0 and counts == [0, 0, 0, 0]
    # the same bytes read as float32 would be NaN: the kind decides, not the bytes
    total, counts = _scan(ctx, tensors[:1], kinds=[native.KIND_F32])
    assert counts == [1 << 14]


@gpu
def test_range_of_more_than_2_31_elements(cuda_device):
    ctx = native.get_context(0)
    n = (1 << 31) + 4099
    t = torch.zeros(n, dtype=torch.uint8, device="cuda")
    for i in (0, (1 << 31) - 1, 1 << 31, (1 << 31) + 3, n - 1):
        t[i] = 0x7C  # float8_e5m2 +Inf
    total, counts = _scan(ctx, [t.view(torch.float8_e5m2)])
    assert total == 5 and counts == [5]
    del t
    torch.cuda.empty_cache()


@gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.bfloat16], ids=str)
def test_a_cut_element_is_counted_by_both_halves(cuda_device, dtype):
    """Two windows of the segment meet inside an element: both scan it whole."""
    ctx = native.get_context(0)
    t = torch.ones(3 * ITEM, dtype=dtype, device="cuda")
    es = t.element_size()
    k = ITEM + 17
    t[k] = float("nan")
    cut = k * es + es // 2
    p, nbytes = t.data_ptr(), t.numel() * es
    kind = KINDS[dtype]
    total, counts = _scan(ctx, [t, t], kinds=[kind, kind],
                          ranges=[(p, cut), (p + cut, nbytes - cut)])
    assert counts == [1, 1] and total == 2
    # a cut right after the element: only the first half holds it
    cut = (k + 1) * es
    _, counts = _scan(ctx, [t, t], kinds=[kind, kind], ranges=[(p, cut), (p + cut, nbytes - cut)])
    assert counts == [1, 0]


@gpu
def test_kinds_survive_a_pointer_update(cuda_device):
    ctx = native.get_context(0)
    a = torch.ones(5000, device="cuda")
    b = torch.ones(5000, device="cuda")
    b[4999] = float("inf")
    plan = ctx.plan([a.data_ptr()], [0], [a.numel() * 4])
    try:
        plan.set_kinds([native.KIND_F32])
        plan.scan_nonfinite_async()
        assert plan.scan_wait(1) == (0, [0])
        plan.update([b.data_ptr()], [0], [b.numel() * 4])
        plan.scan_nonfinite_async()
        assert plan.scan_wait(1) == (1, [1])
    finally:
        plan.destroy()


# ------------------------------------------------------------------ engine contract --


def _tree_tensors(tree, prefix=""):
    if isinstance(tree, dict):
        for k, v in tree.items():
            yield from _tree_tensors(v, f"{prefix}{k}.")
    elif isinstance(tree, (list, tuple)):
        for i, v in enumerate(tree):
            yield from _tree_tensors(v, f"{prefix}{i}.")
    elif torch.is_tensor(tree):
        yield prefix, tree


def _model_state():
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(512, 512), torch.nn.GELU(),
                                torch.nn.Linear(512, 256)).cuda()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-3)
    x = torch.randn(16, 512, device="cuda")
    for _ in range(2):
        model(x).square().mean().backward()
        opt.step()
        opt.zero_grad()
    big = torch.randn(64, 4096, device="cuda")
    state = {"model": model.state_dict(), "optim": opt.state_dict(),
             "cpu": torch.arange(1000, dtype=torch.float64),
             "strided": big[:, :1024]}  # row-strided: one range per row
    return model, opt, state


MODES = {
    "full": {},
    "incremental": {"DLROVER_B200_INCREMENTAL": "1"},
    "in_place": {"DLROVER_B200_IN_PLACE": "1"},
    "hybrid": {"DLROVER_B200_IN_PLACE": "1", "DLROVER_B200_IN_PLACE_SNAPSHOT_MB": "1"},
    "bounded_arena": {"DLROVER_B200_ARENA_LIMIT_MB": "8"},
}


@gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_a_refused_save_leaves_no_trace(cuda_device, run_env, tmp_path, monkeypatch, mode):
    from dlrover_b200.ckpt_saver import AsyncCheckpointSaver
    from dlrover_b200.common.constants import CheckpointConstant
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType
    from dlrover_b200.shm_handler import DLROVER_CKPT_CONFIG_KEY

    for k, v in MODES[mode].items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("DLROVER_B200_REFUSE_NONFINITE", "1")
    AsyncCheckpointSaver.start_async_saving_ckpt()
    ckpt = DdpCheckpointer(str(tmp_path / "ckpt"))
    engine = ckpt.engine
    handler = engine._shm_handler
    assert engine.refuse_non_finite
    try:
        model, opt, state = _model_state()
        ckpt.save_checkpoint(10, state, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        image = bytes(handler.shared_memory.buf)
        at10 = {k: t.clone() for k, t in _tree_tensors(state)}

        leaf = state["optim"]["state"][0]["exp_avg"]
        leaf.view(-1)[7] = float("nan")
        state["strided"][3, 5] = float("inf")
        state["strided"][9, 1000] = float("nan")
        path = {"model_states": str(tmp_path / "ckpt" / "20" / "rank_0.pt")}
        assert engine.save_to_memory(20, {"model_states": state}, path) is False
        for storage in (StorageType.MEMORY, StorageType.DISK):
            ckpt.save_checkpoint(20, state, storage_type=storage)
            assert ckpt.wait_memory_save(60)
            assert bytes(handler.shared_memory.buf) == image
            conf = handler.metadata.get().get(DLROVER_CKPT_CONFIG_KEY)
            assert conf.step == 10 and not conf.writing_shm
            stats = engine.last_save_stats()
            assert stats == {"refused": True,
                             "non_finite": {"model_states.optim.state.0.exp_avg": 1,
                                            "model_states.strided": 2}}, stats
        assert not (tmp_path / "ckpt" / "20").exists()
        assert not (tmp_path / "ckpt" / CheckpointConstant.TRACER_FILE_NAME).exists()

        # back to the state of step 10 from its HBM image (modes that keep one)
        assert ckpt.rollback_into(state) == 10
        if mode in ("full", "incremental", "bounded_arena"):  # the state fits in 8 MiB
            assert handler.last_restore_stats["from_image"] == 1.0
        for k, t in _tree_tensors(state):
            assert torch.equal(t.cpu().view(-1).view(torch.uint8) if t.is_contiguous() else
                               t.contiguous().cpu().view(-1).view(torch.uint8),
                               at10[k].contiguous().cpu().view(-1).view(torch.uint8)), k
        # the lock was given back, and an incremental save finds its baseline
        ckpt.save_checkpoint(21, state, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        assert handler.metadata.get()[DLROVER_CKPT_CONFIG_KEY].step == 21
        if mode == "incremental":
            assert engine.last_save_stats() == {"delta": True, "drained_bytes": 0}
        assert bytes(handler.shared_memory.buf) == image
        del model, opt

        # a NaN in a CPU leaf alone refuses too
        state["cpu"][999] = float("nan")
        ckpt.save_checkpoint(22, state, storage_type=StorageType.MEMORY)
        assert engine.last_save_stats()["non_finite"] == {"model_states.cpu": 1}
        assert handler.metadata.get()[DLROVER_CKPT_CONFIG_KEY].step == 21
    finally:
        engine.close()


@gpu
def test_switched_off_a_nan_state_is_saved_as_today(cuda_device, run_env, tmp_path,
                                                   monkeypatch):
    from dlrover_b200.ckpt_saver import AsyncCheckpointSaver
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType
    from dlrover_b200.shm_handler import DLROVER_CKPT_CONFIG_KEY

    monkeypatch.delenv("DLROVER_B200_REFUSE_NONFINITE", raising=False)
    AsyncCheckpointSaver.start_async_saving_ckpt()
    ckpt = DdpCheckpointer(str(tmp_path / "off"))
    handler = ckpt.engine._shm_handler
    try:
        assert not ckpt.engine.refuse_non_finite
        _, _, state = _model_state()
        state["model"]["0.weight"][0, 0] = float("nan")
        state["cpu"][0] = float("inf")
        ckpt.save_checkpoint(5, state, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        assert handler.metadata.get()[DLROVER_CKPT_CONFIG_KEY].step == 5
        assert ckpt.engine.last_save_stats() is None
        # the segment holds every leaf's bytes at its offset, NaN included
        buf = handler.shared_memory.buf
        for (k, t), m in zip(_tree_tensors(state), handler._layout.leaf_metas):
            n = m.numel * m.element_size
            want = t.detach().contiguous().cpu().reshape(-1).view(torch.uint8).numpy().tobytes()
            assert bytes(buf[m.offset:m.offset + n]) == want, k
    finally:
        ckpt.engine.close()


@gpu
def test_sharded_engines_say_they_do_not_check(cuda_device, run_env, tmp_path, monkeypatch):
    from dlrover_b200.ckpt_saver import AsyncCheckpointSaver
    from dlrover_b200.common.storage import PosixDiskStorage
    from dlrover_b200.flash_checkpoint.fsdp_engine import FsdpCheckpointEngine

    AsyncCheckpointSaver.start_async_saving_ckpt()
    engine = FsdpCheckpointEngine(str(tmp_path / "fsdp"), PosixDiskStorage())
    try:
        engine.refuse_non_finite = True
        with pytest.raises(NotImplementedError):
            engine.save_to_memory(1, {"model": {"w": torch.ones(4, device="cuda")}},
                                  {"model": str(tmp_path / "fsdp" / "1")})
    finally:
        engine.close()


@gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="cooperative saves need 2 GPUs")
@pytest.mark.timeout(600)
def test_cooperative_refusal_two_gpus():
    results = _spawn(_coop_worker, 2)
    for res in results:
        assert res["refused"] is True and res["unchanged"], res
    assert results[1]["non_finite"] == {"model_states.w": 1}


def _coop_worker(rank, world, port, run_id, ckpt_dir, out_dir):
    import torch.distributed as dist

    _worker_env(rank, world, port, run_id)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType

    result = {}
    try:
        ckpt = DdpCheckpointer(ckpt_dir)  # one shard per node: cooperative
        ckpt.engine.refuse_non_finite = True
        sd = {"w": torch.ones(3 << 20, device="cuda")}  # 12 MiB: both ranks hold a window
        ckpt.save_checkpoint(3, sd, storage_type=StorageType.MEMORY)
        ckpt.wait_memory_save(60)
        dist.barrier()
        before = bytes(ckpt.engine._shm_handler.shared_memory.buf)
        if rank == 1:
            sd["w"][-1] = float("nan")  # in rank 1's window only
        result["refused"] = ckpt.engine.save_to_memory(
            4, {"model_states": sd}, {"model_states": ckpt_dir + "/4"}) is False
        dist.barrier()
        result["unchanged"] = bytes(ckpt.engine._shm_handler.shared_memory.buf) == before
        result["non_finite"] = (ckpt.engine.last_save_stats() or {}).get("non_finite")
        ckpt.engine.close()
    finally:
        torch.save(result, os.path.join(out_dir, f"r{rank}.pt"))
        dist.destroy_process_group()


# --------------------------------------------------------------- CPU (no GPU needed) --


def test_scan_entry_points_reject_bad_arguments():
    lib = native.load_library()
    assert lib.fc_scan_nonfinite_async(None, None) == native.FC_EINVAL
    assert b"fc_scan_nonfinite_async" in lib.fc_last_error()
    assert lib.fc_scan_wait(None, None, None, 0) == native.FC_EINVAL
    assert lib.fc_plan_set_kinds(None, 0, None) == native.FC_EINVAL
    assert b"fc_plan_set_kinds" in lib.fc_last_error()


def test_switch_defaults_off_and_follows_the_environment(monkeypatch):
    from dlrover_b200.flash_checkpoint.engine import FullCheckpointEngine

    e = object.__new__(FullCheckpointEngine)
    monkeypatch.delenv("DLROVER_B200_REFUSE_NONFINITE", raising=False)
    assert e.refuse_non_finite is False
    monkeypatch.setenv("DLROVER_B200_REFUSE_NONFINITE", "1")
    assert e.refuse_non_finite is True
    e.refuse_non_finite = False
    assert e.refuse_non_finite is False


def _worker_env(rank, world, port, run_id):
    import sys

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    os.environ.update({
        "RANK": str(rank), "LOCAL_RANK": str(rank), "WORLD_SIZE": str(world),
        "LOCAL_WORLD_SIZE": str(world), "GROUP_WORLD_SIZE": "1", "GROUP_RANK": "0",
        "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "TORCHELASTIC_RUN_ID": run_id,
        "DLROVER_LOG_LEVEL": "WARNING",
    })
    os.environ.pop("ROLE_NAME", None)


def _gloo_worker(rank, world, port, run_id, ckpt_dir, out_dir):
    import torch.distributed as dist

    _worker_env(rank, world, port, run_id)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType
    from dlrover_b200.shm_handler import DLROVER_CKPT_CONFIG_KEY

    result = {}
    try:
        ckpt = DdpCheckpointer(ckpt_dir, local_shard_num=world, global_shard_num=world)
        ckpt.engine.refuse_non_finite = True
        handler = ckpt.engine._shm_handler
        sd = {"w": torch.full((1000,), float(rank + 1)), "i": torch.full((9,), -1)}
        ckpt.save_checkpoint(3, sd, storage_type=StorageType.MEMORY)
        before = bytes(handler.shared_memory.buf)
        if rank == 1:
            sd["w"][10] = float("nan")
        sd["w"].add_(1.0)
        ckpt.save_checkpoint(4, sd, storage_type=StorageType.DISK)
        result["saved"] = ckpt.engine.save_to_memory(4, {"model_states": sd},
                                                     {"model_states": ckpt_dir + "/4"})
        result["unchanged"] = bytes(handler.shared_memory.buf) == before
        result["step"] = handler.metadata.get()[DLROVER_CKPT_CONFIG_KEY].step
        result["stats"] = ckpt.engine.last_save_stats()
        dist.barrier()
        ckpt.engine.close()
    finally:
        torch.save(result, os.path.join(out_dir, f"r{rank}.pt"))
        dist.destroy_process_group()


def _spawn(worker, world):
    import glob
    import shutil
    import tempfile
    import uuid

    import torch.multiprocessing as mp

    run_id = "nf" + uuid.uuid4().hex[:8]
    port = 29600 + (os.getpid() * 13 + world) % 1500
    with tempfile.TemporaryDirectory() as ckpt_dir, tempfile.TemporaryDirectory() as out_dir:
        mp.spawn(worker, args=(world, port, run_id, ckpt_dir, out_dir), nprocs=world, join=True)
        results = [torch.load(os.path.join(out_dir, f"r{r}.pt")) for r in range(world)]
        results[0]["dirs"] = sorted(os.listdir(ckpt_dir))
    shutil.rmtree(os.path.join("/tmp/ckpt_sock", run_id), ignore_errors=True)
    for f in glob.glob(f"/dev/shm/{run_id}_*"):
        os.unlink(f)
    return results


@pytest.mark.timeout(300)
def test_one_rank_with_a_nan_makes_every_rank_refuse():
    results = _spawn(_gloo_worker, 2)
    for rank, res in enumerate(results):
        assert res["saved"] is False and res["unchanged"] and res["step"] == 3, res
        assert res["stats"]["refused"] is True
    assert results[0]["stats"]["non_finite"] == {}
    assert results[1]["stats"]["non_finite"] == {"model_states.w": 1}
    assert "4" not in results[0]["dirs"]
