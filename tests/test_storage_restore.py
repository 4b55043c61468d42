"""Restore a persisted checkpoint (a torch.save archive) straight into live tensors:
the archive index (torch_file_index), the library's file fill (fc_restore_file_async),
shm_handler.restore_file_into and the engine / DdpCheckpointer entry points."""

import ctypes
import fractions
import os
import pickle
import shutil
import zipfile

import pytest
import torch

from dlrover_b200 import _native as native
from dlrover_b200 import fast_torch_save
from dlrover_b200.shm_handler import restore_file_into
from dlrover_b200.torch_file_index import TensorLeaf, index_file
from tests.golden.fixtures import fixture_mixed, pat

gpu = pytest.mark.gpu
WRITERS = {"torch_save": torch.save, "fast_save": fast_torch_save.fast_save}


def _leaves(tree, prefix=""):
    if isinstance(tree, dict):
        for k, v in tree.items():
            yield from _leaves(v, f"{prefix}{k}.")
    elif isinstance(tree, (list, tuple)):
        for i, v in enumerate(tree):
            yield from _leaves(v, f"{prefix}{i}.")
    elif torch.is_tensor(tree) or isinstance(tree, TensorLeaf):
        yield prefix[:-1], tree


def _noise(n, dtype, seed):
    """Random bytes as `dtype`: NaN payloads, infinities and denormals included."""
    g = torch.Generator().manual_seed(seed)
    es = torch.empty((), dtype=dtype).element_size()
    return torch.randint(0, 256, (n * es,), dtype=torch.uint8, generator=g).view(dtype)


def _source_tree():
    """Every dtype of the golden fixtures plus the views a state dict can hold: storage
    offsets (odd ones too), tied storages, row-strided views, 0-element leaves."""
    tree = fixture_mixed()
    tree.pop("transposed")  # neither dense nor row-strided: refused, see below
    tree.pop("strided")
    big = _noise(64 * 96, torch.bfloat16, 1).reshape(64, 96)
    emb = _noise(50 * 128, torch.float32, 2).reshape(50, 128)
    raw = _noise(9001, torch.uint8, 3)
    tree.update({
        "nan_f32": _noise(777, torch.float32, 4),
        "nan_f64": _noise(129, torch.float64, 5),
        "nan_f16": _noise(301, torch.float16, 6),
        "f8": _noise(333, torch.float8_e4m3fn, 7),
        "embed": emb, "lm_head": emb,                   # tied weights
        "rows": big[:, 8:72],                           # row-strided, storage offset 8
        "row_odd": big[3:40, 1:97 - 2],                 # odd element offset
        "u8_odd": raw[3:8003],                          # odd byte offset
        "i8_tail": _noise(99, torch.int8, 8)[1:],
        "zero_rows": big[:0],
        "empty_i64": torch.empty(0, dtype=torch.int64),
        "nested": [{"w": _noise(4096, torch.bfloat16, 9)}, (1.5, None)],
    })
    return tree


def _bits(t):
    return t.detach().cpu().contiguous().reshape(-1).view(torch.uint8)


def _same_bits(got, want):
    a, b = dict(_leaves(got)), dict(_leaves(want))
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and tuple(a[k].shape) == tuple(b[k].shape), k
        assert torch.equal(_bits(a[k]), _bits(b[k])), k


def _like(tree, device, strided=False):
    """Zeroed targets of the same shapes; strided=True makes every 2-D leaf a row-strided
    view of a wider buffer, shifted by one element."""
    def make(t):
        if not torch.is_tensor(t):
            return t
        if strided and t.dim() == 2 and t.numel() and t.shape[1] * t.element_size() >= 256:
            buf = torch.zeros(t.shape[0], t.shape[1] + 5, dtype=t.dtype, device=device)
            return buf[:, 1:1 + t.shape[1]]
        return torch.zeros(t.shape, dtype=t.dtype, device=device)

    def walk(v):
        if isinstance(v, dict):
            return {k: walk(x) for k, x in v.items()}
        if isinstance(v, list):
            return [walk(x) for x in v]
        if isinstance(v, tuple):
            return tuple(walk(x) for x in v)
        return make(v)

    out = walk(tree)
    out["lm_head"] = out["embed"]  # the model ties them too
    return out


# ----------------------------------------------------------------------- CPU ---------


@pytest.mark.parametrize("writer", list(WRITERS))
def test_index_agrees_with_zipfile_and_torch_load(tmp_path, writer):
    path = str(tmp_path / "ckpt.pt")
    src = _source_tree()
    WRITERS[writer](src, path)
    idx = index_file(path)
    loaded = torch.load(path, map_location="cpu", weights_only=True)
    raw = open(path, "rb").read()
    with zipfile.ZipFile(path) as z:
        names = [i.filename for i in z.infolist() if "/data/" in i.filename]
        assert sorted(idx.records) == sorted(n.rsplit("/", 1)[1] for n in names)
        for n in names:
            off, size = idx.records[n.rsplit("/", 1)[1]]
            assert raw[off:off + size] == z.read(n), n
            assert off % 64 == 0
    got, want = dict(_leaves(idx.tree)), dict(_leaves(loaded))
    assert sorted(got) == sorted(want)
    for k, leaf in got.items():
        t = want[k]
        assert (leaf.dtype, leaf.shape, leaf.stride, leaf.storage_offset) == \
            (t.dtype, tuple(t.shape), t.stride(), t.storage_offset()), k
        nbytes = t.untyped_storage().nbytes()
        store = torch.frombuffer(bytearray(raw[leaf.file_offset:leaf.file_offset + nbytes]) or
                                 bytearray(1), dtype=torch.uint8)[:nbytes]
        view = store.view(t.dtype).as_strided(leaf.shape, leaf.stride, leaf.storage_offset)
        assert torch.equal(_bits(view), _bits(t)), k
    assert got["embed"].key == got["lm_head"].key
    assert got["u8_odd"].storage_offset == 3 and got["zero_rows"].numel == 0
    assert idx.tree["nested"][1] == (1.5, None) and idx.tree["list"][2] == 17


@pytest.mark.parametrize("writer", list(WRITERS))
def test_cpu_targets_are_pread_straight_in(tmp_path, writer):
    path = str(tmp_path / "ckpt.pt")
    src = _source_tree()
    WRITERS[writer](src, path)
    tgt = _like(src, "cpu", strided=True)
    stats = restore_file_into(path, tgt)
    _same_bits(tgt, torch.load(path, map_location="cpu", weights_only=True))
    assert stats["device_bytes"] == 0 and stats["host_bytes"] > 0
    assert set(stats) == {"device_bytes", "host_bytes", "read_ms", "scatter_ms", "wall_ms"}


def test_tree_rules_are_those_of_restore_into(tmp_path):
    path = str(tmp_path / "ckpt.pt")
    torch.save({"a": torch.ones(4), "b": torch.ones(2, dtype=torch.int32), "n": "x"}, path)
    with pytest.raises(KeyError):
        restore_file_into(path, {"a": torch.zeros(4)})
    with pytest.raises(KeyError):
        restore_file_into(path, {"a": torch.zeros(4), "b": torch.zeros(2, dtype=torch.int32),
                                 "c": torch.zeros(1)})
    with pytest.raises(ValueError, match="a: shape/dtype"):
        restore_file_into(path, {"a": torch.zeros(4, dtype=torch.float64),
                                 "b": torch.zeros(2, dtype=torch.int32)})
    tgt = {"a": torch.zeros(4), "n": 5}
    restore_file_into(path, tgt, strict=False)
    assert torch.equal(tgt["a"], torch.ones(4)) and tgt["n"] == 5


def test_views_that_are_not_row_strided_are_refused(tmp_path):
    path = str(tmp_path / "ckpt.pt")
    torch.save({"t": pat((6, 10), torch.float32, 1).t()}, path)
    with pytest.raises(ValueError, match="t: the file holds a view"):
        restore_file_into(path, {"t": torch.zeros(10, 6)})


def _repack(src, dst, compression=zipfile.ZIP_STORED, edit=None):
    with zipfile.ZipFile(src) as zin, zipfile.ZipFile(dst, "w", compression) as zout:
        for i in zin.infolist():
            data = zin.read(i.filename)
            if edit:
                data = edit(i.filename, data)
            zout.writestr(i.filename, data)


def test_refusals_name_the_file(tmp_path):
    good = str(tmp_path / "good.pt")
    torch.save({"w": torch.arange(1000, dtype=torch.float32)}, good)
    assert index_file(good).records

    deflated = str(tmp_path / "deflated.pt")
    _repack(good, deflated, zipfile.ZIP_DEFLATED)
    with pytest.raises(ValueError, match="deflated.pt.*compressed"):
        index_file(deflated)

    big = str(tmp_path / "big.pt")
    _repack(good, big, edit=lambda n, d: b"big" if n.endswith("/byteorder") else d)
    with pytest.raises(ValueError, match="big.pt.*byteorder"):
        index_file(big)

    legacy = str(tmp_path / "legacy.pt")
    torch.save({"w": torch.ones(3)}, legacy, _use_new_zipfile_serialization=False)
    with pytest.raises(ValueError, match="legacy.pt.*legacy"):
        index_file(legacy)

    size = os.path.getsize(good)
    for cut in (10, size // 2, size - 30):
        trunc = str(tmp_path / f"trunc{cut}.pt")
        with open(good, "rb") as f, open(trunc, "wb") as g:
            g.write(f.read()[:cut])
        with pytest.raises(ValueError, match=f"trunc{cut}.pt.*truncated"):
            index_file(trunc)


def test_globals_outside_the_allowlist_are_refused_like_torch_load(tmp_path):
    good = str(tmp_path / "good.pt")
    torch.save({"w": torch.ones(3)}, good)
    evil = str(tmp_path / "evil.pt")
    payload = pickle.dumps({"w": fractions.Fraction(1, 3)}, protocol=2)
    _repack(good, evil, edit=lambda n, d: payload if n.endswith("/data.pkl") else d)
    with pytest.raises(pickle.UnpicklingError):
        torch.load(evil, weights_only=True)
    with pytest.raises(pickle.UnpicklingError, match="evil.pt"):
        index_file(evil)


def test_index_reads_no_payload(tmp_path, monkeypatch):
    path = str(tmp_path / "ckpt.pt")
    fast_torch_save.fast_save({"w": torch.zeros(1 << 20)}, path)
    seen = []
    real = os.pread
    monkeypatch.setattr(os, "pread", lambda fd, n, off: seen.append(n) or real(fd, n, off))
    index_file(path)
    assert sum(seen) < 256 << 10


def test_no_tracker_restores_nothing(tmp_path):
    from dlrover_b200.common.storage import PosixDiskStorage
    from dlrover_b200.flash_checkpoint.engine import FullCheckpointEngine

    eng = FullCheckpointEngine.__new__(FullCheckpointEngine)
    eng.checkpoint_dir = str(tmp_path)
    eng.storage = PosixDiskStorage()
    eng._loader_group = None
    eng._global_shard_num = 1
    eng._rank = 0
    assert eng.load_storage_into({"model_states": {"w": torch.zeros(2)}}) == (0, {})


def test_file_restore_entry_point_rejects_null_arguments():
    lib = native.load_library()
    assert lib.fc_restore_file_async(None, 3, None) == native.FC_EINVAL
    assert b"fc_restore_file_async" in lib.fc_last_error()
    assert lib.fc_restore_file_async(ctypes.c_void_p(4096), -1, None) == native.FC_EINVAL
    text = lib.fc_strerror(native.FC_EIO)
    assert text and b"file" in text and text != lib.fc_strerror(-99)


# ----------------------------------------------------------------------- GPU ---------


@pytest.fixture
def variant_ctx(cuda_device):
    ctx = native.get_context(0)
    yield ctx
    ctx.set_variant(native.VARIANT_TMA)


@gpu
@pytest.mark.parametrize("writer", list(WRITERS))
@pytest.mark.parametrize("variant", [native.VARIANT_LSU, native.VARIANT_TMA], ids=["lsu", "tma"])
@pytest.mark.parametrize("strided", [False, True], ids=["dense", "rowstrided"])
def test_restore_is_bitwise_torch_load_then_copy(tmp_path, variant_ctx, writer, variant, strided):
    path = str(tmp_path / "ckpt.pt")
    src = _source_tree()
    WRITERS[writer](src, path)
    variant_ctx.set_variant(variant)
    tgt = _like(src, "cuda", strided=strided)
    tgt["nested"][0]["w"] = tgt["nested"][0]["w"].cpu()  # a CPU leaf in a CUDA tree
    tgt["a"]["i64"] = tgt["a"]["i64"].cpu()
    want = _like(src, "cuda", strided=strided)
    want["nested"][0]["w"] = want["nested"][0]["w"].cpu()
    want["a"]["i64"] = want["a"]["i64"].cpu()
    loaded = torch.load(path, map_location="cpu")
    with torch.no_grad():
        for (k, t), (_, s) in zip(_leaves(want), _leaves(_drop_transposed(loaded))):
            t.copy_(s)
    stats = restore_file_into(path, tgt)
    torch.cuda.synchronize()
    _same_bits(tgt, want)
    assert stats["device_bytes"] > 0 and stats["host_bytes"] > 0
    assert stats["wall_ms"] >= stats["read_ms"] >= 0 and stats["scatter_ms"] >= 0
    assert tgt["lm_head"].data_ptr() == tgt["embed"].data_ptr()


def _drop_transposed(tree):
    tree.pop("transposed", None)
    tree.pop("strided", None)
    return tree


@gpu
def test_windowed_when_the_arena_cannot_hold_the_plan(tmp_path, variant_ctx, monkeypatch):
    path = str(tmp_path / "ckpt.pt")
    src = {f"w{i}": _noise((3 << 20) + 17 * i, torch.bfloat16, i) for i in range(6)}
    src["row"] = _noise(512 * 4096, torch.float32, 9).reshape(512, 4096)[:, 3:4000]
    fast_torch_save.fast_save(src, path)
    monkeypatch.setenv("DLROVER_B200_ARENA_LIMIT_MB", "8")
    try:
        tgt = {k: torch.zeros(v.shape, dtype=v.dtype, device="cuda") for k, v in src.items()}
        restore_file_into(path, tgt)
        torch.cuda.synchronize()
        _same_bits(tgt, src)
    finally:
        variant_ctx.set_arena_limit(0)


@gpu
def test_truncated_after_indexing_changes_nothing(tmp_path, cuda_device):
    path = str(tmp_path / "ckpt.pt")
    src = {"a": _noise(1 << 20, torch.float32, 1), "b": _noise(3 << 20, torch.bfloat16, 2),
           "c": _noise(1000, torch.int32, 3)}
    fast_torch_save.fast_save(src, path)
    idx = index_file(path)
    with open(path, "r+b") as f:
        f.truncate(idx.records[idx.tree["b"].key][0] + 12345)
    tgt = {k: torch.full(v.shape, 7, dtype=v.dtype, device="cuda") for k, v in src.items()}
    tgt["c"] = tgt["c"].cpu()
    with pytest.raises((native.NativeError, OSError), match="offset"):
        restore_file_into(path, tgt, index=idx)
    torch.cuda.synchronize()
    for k, v in tgt.items():
        assert torch.equal(v.cpu(), torch.full(v.shape, 7, dtype=v.dtype)), k

    # the library alone: FC_EIO names the offset, no scatter is enqueued
    ctx = native.get_context(0)
    t = torch.full((3 << 20,), 7, dtype=torch.bfloat16, device="cuda")
    off = idx.records[idx.tree["b"].key][0]
    plan = ctx.plan([t.data_ptr()], [0], [t.numel() * 2], host_offsets=[off])
    ctx.arena_reserve(plan.arena_end)
    fd = os.open(path, os.O_RDONLY)
    try:
        with pytest.raises(native.NativeError, match="offset") as e:
            plan.restore_file_async(fd, torch.cuda.current_stream())
        assert e.value.code == native.FC_EIO
    finally:
        os.close(fd)
        plan.destroy()
    torch.cuda.synchronize()
    assert torch.equal(t, torch.full_like(t, 7))


@gpu
def test_file_over_4_gib_restores(tmp_path, cuda_device):
    free = shutil.disk_usage(str(tmp_path)).free
    if free < (10 << 30):
        pytest.skip(f"needs 10 GB free in the temp directory, {free / 2**30:.1f} GiB there")
    path = str(tmp_path / "big.pt")
    n = (4 << 30) + 4099
    big = torch.arange(251, dtype=torch.uint8).repeat(n // 251 + 1)[:n]
    src = {"head": _noise(1000, torch.float32, 1), "big": big,
           "tail": _noise(5000, torch.bfloat16, 2), "tail_view": big[(4 << 30) + 7:]}
    fast_torch_save.fast_save(src, path)
    del src["big"], src["tail_view"], big
    idx = index_file(path)
    assert idx.size > (4 << 30) and idx.tree["tail"].file_offset > (4 << 30)
    tgt = {"head": torch.zeros(1000, device="cuda"),
           "big": torch.empty(n, dtype=torch.uint8, device="cuda"),
           "tail": torch.zeros(5000, dtype=torch.bfloat16, device="cuda"),
           "tail_view": torch.empty(n - (4 << 30) - 7, dtype=torch.uint8, device="cuda")}
    restore_file_into(path, tgt, index=idx)
    torch.cuda.synchronize()
    want = torch.arange(251, dtype=torch.uint8, device="cuda").repeat(n // 251 + 1)[:n]
    assert torch.equal(tgt["big"], want)
    assert torch.equal(tgt["tail_view"], want[(4 << 30) + 7:])
    del want, tgt["big"]
    _same_bits({"head": tgt["head"], "tail": tgt["tail"]}, src)


@gpu
def test_ddp_checkpointer_restores_a_restarted_node_from_disk(cuda_device, run_env, tmp_path,
                                                              monkeypatch):
    from dlrover_b200.ckpt_saver import AsyncCheckpointSaver, CheckpointConfig
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType
    from tests.test_incremental_save import _Adapted

    AsyncCheckpointSaver.start_async_saving_ckpt()
    ckpt = DdpCheckpointer(str(tmp_path / "ckpt"))
    handler = ckpt.engine._shm_handler
    try:
        ckpt.engine.incremental = True
        torch.manual_seed(0)
        model = _Adapted().cuda()
        opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-2)
        x = torch.randn(32, 1024, device="cuda")
        for _ in range(3):
            model(x).square().mean().backward()
            opt.step()
            opt.zero_grad()
        tree = {"model": model.state_dict(), "optim": opt.state_dict(),
                "cpu": torch.arange(1000, dtype=torch.float64)}
        ckpt.save_checkpoint(5, tree, storage_type=StorageType.DISK)
        ckpt.wait_latest_checkpoint(120)
        assert ckpt.wait_memory_save(60)
        at_save = {k: t.clone() for k, t in _leaves(tree)}
        ckpt.save_checkpoint(6, tree, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        assert ckpt.engine.last_save_stats()["delta"] is True  # a baseline exists

        # a replacement node: its shared memory holds nothing
        with monkeypatch.context() as m:
            m.setattr(handler, "get_checkpoint_config", lambda default: CheckpointConfig())
            assert ckpt.load_checkpoint_into(tree) == 0
            with torch.no_grad():
                for _, t in _leaves(tree):
                    t.zero_()
            assert ckpt.load_storage_into(tree) == 5
        torch.cuda.synchronize()
        got = dict(_leaves(tree))
        assert sorted(got) == sorted(at_save)
        for k, t in got.items():
            assert torch.equal(_bits(t), _bits(at_save[k])), k
        assert any(not t.is_cuda for t in got.values())

        # the file restore rewrote the arena: no image to roll back from, no baseline
        assert not handler.can_rollback({"model_states": tree})
        ckpt.save_checkpoint(7, tree, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(60)
        assert ckpt.engine.last_save_stats()["delta"] is False

        # an explicit path: the step is the name of its directory
        step, stats = ckpt.engine.load_storage_into(
            {"model_states": tree}, resume_path=str(tmp_path / "ckpt" / "5" / "rank_0.pt"))
        assert step == 5 and stats["device_bytes"] > 0 and stats["host_bytes"] > 0
    finally:
        ckpt.engine.close()
