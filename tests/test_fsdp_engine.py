"""DCP-over-shared-memory engine (reference behaviours:
dlrover/trainer/tests/torch/fsdp_ckpt_test.py)."""

import io
import os
import pickle
import time

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.distributed.checkpoint as dist_cp
from torch.distributed.checkpoint.default_planner import DefaultSavePlanner
from torch.distributed.checkpoint.metadata import MetadataIndex
from torch.distributed.checkpoint.planner import SavePlan, WriteItem, WriteItemType
from torch.distributed.checkpoint.planner import TensorWriteData
from torch.distributed.checkpoint.metadata import ChunkStorageMetadata, TensorProperties

from dlrover_b200.ckpt_saver import AsyncCheckpointSaver, DLROVER_CKPT_CONFIG_KEY
from dlrover_b200.common.storage import PosixDiskStorage
from dlrover_b200.flash_checkpoint import fsdp_engine as fe
from dlrover_b200.shm_handler import SharedMemoryHandler
from oracle import shm_layout as oracle


@pytest.fixture
def gloo(run_env, monkeypatch):
    monkeypatch.setenv("MASTER_ADDR", "127.0.0.1")
    monkeypatch.setenv("MASTER_PORT", str(29500 + os.getpid() % 2000))
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("WORLD_SIZE", "1")
    monkeypatch.setenv("LOCAL_RANK", "0")
    monkeypatch.setenv("LOCAL_WORLD_SIZE", "1")
    dist.init_process_group("gloo", rank=0, world_size=1)
    AsyncCheckpointSaver.start_async_saving_ckpt()
    yield
    dist.destroy_process_group()


def _item(fqn, t, kind=WriteItemType.TENSOR):
    if kind == WriteItemType.BYTE_IO:
        return WriteItem(index=MetadataIndex(fqn), type=kind)
    return WriteItem(
        index=MetadataIndex(fqn, [0] * t.dim()), type=kind,
        tensor_data=TensorWriteData(
            chunk=ChunkStorageMetadata(offsets=torch.Size([0] * t.dim()), sizes=t.size()),
            properties=TensorProperties.create_from_tensor(t), size=t.size()))


class _Planner(DefaultSavePlanner):
    def __init__(self, data):
        super().__init__()
        self._data = data

    def resolve_data(self, write_item):
        return self._data[write_item.index.fqn]


def test_item_layout_is_back_to_back(run_env):
    """fsdp_ckpt_test.py:188-209: a 2x4 fp32 item is 32 bytes, offsets 0 -> 32."""
    a = torch.arange(8, dtype=torch.float32).reshape(2, 4)
    b = torch.arange(8, 16, dtype=torch.float32).reshape(2, 4)
    blob = io.BytesIO(b"hello-bytes")
    data = {"a": a, "b": b, "blob": blob}
    files = [("__0_0.distcp", _item("a", a, WriteItemType.SHARD)),
             ("__0_0.distcp", _item("blob", None, WriteItemType.BYTE_IO)),
             ("__0_0.distcp", _item("b", b))]
    planner = _Planner(data)
    assert fe._tensor_item_size(files[0][1]) == 32
    assert fe._get_buffer_size(files, planner) == 32 + 11 + 32
    handler = SharedMemoryHandler(0, host=True)
    results, no_shard, pending = fe._write_memory_from_list(handler, files, planner)
    assert pending is None
    infos = [r.storage_data for r in results]
    assert [(i.offset, i.length) for i in infos] == oracle.dcp_item_offsets([32, 11, 32])
    assert all(i.relative_path == "__0_0.distcp" for i in infos)
    assert [r.size_in_bytes for r in results] == [32, 11, 32]
    seg = np.frombuffer(handler.shared_memory.buf, dtype=np.uint8)
    want = np.concatenate([oracle.tensor_bytes(a), np.frombuffer(b"hello-bytes", np.uint8),
                           oracle.tensor_bytes(b)])
    assert np.array_equal(seg, want)
    # only non-SHARD items are broadcast material
    assert set(no_shard) == {"blob", "b"}
    del seg
    handler.unlink()
    handler.close()


def _state(device="cpu"):
    return {"model": {"w": torch.arange(12, dtype=torch.float32, device=device).reshape(3, 4),
                      "b": torch.arange(5, dtype=torch.bfloat16, device=device)},
            "optim": {"m": torch.arange(7, dtype=torch.int64, device=device)},
            "step": 42, "name": "abc"}


def _engine_roundtrip(tmp_path, device, async_drain):
    engine = fe.FsdpCheckpointEngine(str(tmp_path), PosixDiskStorage(), async_drain=async_drain)
    sd = _state(device)
    paths = {"model_states": str(tmp_path / "100")}
    assert engine.save_to_memory(100, sd, paths) is True
    engine.wait_memory_save()
    time.sleep(0.2)
    meta = engine._shm_handler.metadata.get()
    conf = meta[DLROVER_CKPT_CONFIG_KEY]
    assert conf.step == 100 and conf.writing_shm is False
    assert conf.paths == {"model_states": str(tmp_path / "100" / "__0_0.distcp")}
    assert "dcp_metadata" in meta and "no_shard_data" in meta
    # every tensor's bytes sit in the segment at the offset the metadata says
    seg = bytes(engine._shm_handler.shared_memory.buf)
    storage = meta["dcp_metadata"].storage_data
    flat = {"model.w": sd["model"]["w"], "model.b": sd["model"]["b"], "optim.m": sd["optim"]["m"]}
    seen = 0
    for idx, info in storage.items():
        if idx.fqn in flat:
            want = oracle.tensor_bytes(flat[idx.fqn]).tobytes()
            assert seg[info.offset:info.offset + info.length] == want
            seen += 1
    assert seen == 3
    assert sum(i.length for i in storage.values()) == len(seg)

    # restore from memory through DCP
    target = _state(device)
    for t in (target["model"]["w"], target["model"]["b"], target["optim"]["m"]):
        t.zero_()
    target["step"] = 0
    reader = engine.load()
    assert isinstance(reader, fe.SharedMemoryReader)
    dist_cp.load(target, storage_reader=reader)
    if device == "cuda":
        assert reader.last_fast_items == 3  # all tensors via one DMA fill + scatter kernel
    assert torch.equal(target["model"]["w"], sd["model"]["w"])
    assert torch.equal(target["model"]["b"], sd["model"]["b"])
    assert torch.equal(target["optim"]["m"], sd["optim"]["m"])
    assert target["step"] == 42 and target["name"] == "abc"

    # persist through the agent and reload from files
    engine.save_to_storage(100, sd, paths)
    engine.wait_latest_checkpoint(timeout=60)
    assert sorted(os.listdir(tmp_path)) == ["._dlrover_ckpt_stage", "100", "dlrover_latest.txt"]
    assert sorted(os.listdir(tmp_path / "100")) == [".metadata", "__0_0.distcp"]
    assert (tmp_path / "100" / "__0_0.distcp").read_bytes() == seg
    assert (tmp_path / "dlrover_latest.txt").read_text() == "100"
    file_reader = fe.FileReader(str(tmp_path / "100"))
    target2 = _state(device)
    target2["model"]["w"].zero_()
    dist_cp.load(target2, storage_reader=file_reader)
    assert torch.equal(target2["model"]["w"], sd["model"]["w"])
    assert engine._get_track_resume_path() == str(tmp_path / "100")
    assert engine.get_local_shard_num() == 1 and engine.get_global_shard_num() == 1
    engine.close()


def test_engine_roundtrip_cpu(gloo, tmp_path):
    _engine_roundtrip(tmp_path, "cpu", async_drain=False)


@pytest.mark.gpu
@pytest.mark.parametrize("async_drain", [False, True])
def test_engine_roundtrip_cuda(cuda_device, gloo, tmp_path, async_drain):
    _engine_roundtrip(tmp_path, "cuda", async_drain=async_drain)


def test_failed_publication_gives_the_lock_back(gloo, tmp_path, monkeypatch):
    """If the final writing_shm=False publication fails, the shard lock must not stay
    ours (later saves would be skipped forever) and the error surfaces."""
    engine = fe.FsdpCheckpointEngine(str(tmp_path), PosixDiskStorage(), async_drain=False)
    paths = {"model_states": str(tmp_path / "1")}
    calls = {"n": 0}
    real_set = engine._shm_handler.metadata.set

    def flaky_set(meta):
        calls["n"] += 1
        if calls["n"] == 2:  # the final writing_shm=False publication
            raise RuntimeError("agent went away")
        return real_set(meta)

    monkeypatch.setattr(engine._shm_handler.metadata, "set", flaky_set)
    with pytest.raises(RuntimeError):
        engine.save_to_memory(1, _state(), paths)
    saver = AsyncCheckpointSaver.get_ckpt_saver()
    assert not saver._shm_locks[0].locked()
    monkeypatch.setattr(engine._shm_handler.metadata, "set", real_set)
    assert engine.save_to_memory(2, _state(), paths) is True
    engine.close()


def test_load_without_memory_or_files_returns_none(gloo, tmp_path):
    engine = fe.FsdpCheckpointEngine(str(tmp_path), PosixDiskStorage())
    assert engine.load() is None
    assert engine._get_track_resume_path() == ""
    engine.close()


def _against_reference_golden(tmp_path, device, async_drain):
    """Segment image, per-item (fqn, offset, length) table and target path must
    equal what the REFERENCE's FsdpCheckpointEngine produced for the same state
    dict (tests/golden/make_golden_fsdp.py -> dcp_plain.*)."""
    import hashlib
    import json
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    import fixtures
    from tests.util import GOLDEN, to_device

    info = json.load(open(os.path.join(GOLDEN, "dcp_plain.json")))
    if torch.__version__ != info["torch_version"]:
        pytest.skip("DCP plans / pickled BYTE_IO items are torch-version specific")
    want = np.fromfile(os.path.join(GOLDEN, "dcp_plain.bin"), dtype=np.uint8)
    engine = fe.FsdpCheckpointEngine(str(tmp_path), PosixDiskStorage(), async_drain=async_drain)
    sd = to_device(fixtures.fixture_dcp(), device)
    assert engine.save_to_memory(7, sd, {"model_states": str(tmp_path / "7")})
    engine.wait_memory_save()
    time.sleep(0.3)
    got = np.frombuffer(engine._shm_handler.shared_memory.buf, dtype=np.uint8)
    assert got.size == info["size"]
    assert np.array_equal(got, want)
    assert hashlib.sha256(got.tobytes()).hexdigest() == info["sha256"]
    meta = engine._shm_handler.metadata.get()
    items = sorted([idx.fqn, list(idx.offset) if idx.offset is not None else None,
                    si.relative_path, si.offset, si.length]
                   for idx, si in meta["dcp_metadata"].storage_data.items())
    assert items == info["items"]
    assert sorted(meta["no_shard_data"].keys()) == info["no_shard_keys"]
    conf = meta[DLROVER_CKPT_CONFIG_KEY]
    assert os.path.relpath(conf.paths["model_states"], str(tmp_path)) == info["path"]
    del got
    engine.close()


def test_segment_equals_reference_fsdp_engine_cpu(gloo, tmp_path):
    _against_reference_golden(tmp_path, "cpu", async_drain=False)


@pytest.mark.gpu
def test_segment_equals_reference_fsdp_engine_cuda(cuda_device, gloo, tmp_path):
    _against_reference_golden(tmp_path, "cuda", async_drain=True)
