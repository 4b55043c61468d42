"""Restore a sharded DCP checkpoint (raw "__<rank>_0.distcp" shard files + a pickled
".metadata") from storage through FileDmaReader: the piece builder against a numpy model
of DCP's boxes, the library's multi-file fill (fc_restore_files_async) against the byte
model of test_kernel_model, and whole restores compared bit for bit with FileReader, at
the saved and at other world sizes."""

import io
import os
import pickle

import numpy as np
import pytest
import torch
from torch.distributed._shard._utils import narrow_tensor_by_index
from torch.distributed.checkpoint.metadata import (
    BytesStorageMetadata,
    ChunkStorageMetadata,
    Metadata,
    MetadataIndex,
    TensorProperties,
    TensorStorageMetadata,
)
from torch.distributed.checkpoint.planner import LoadItemType, LoadPlan, ReadItem
from torch.distributed.checkpoint.planner_helpers import create_read_items_for_chunk_list

from dlrover_b200 import _native as native
from dlrover_b200.flash_checkpoint.fsdp_engine import (
    FileDmaReader,
    FileReader,
    _plan_reads,
    _StorageInfo,
    _target_rows,
)

gpu = pytest.mark.gpu
STAT_KEYS = {"device_bytes", "host_bytes", "fallback_items", "files", "plans", "read_ms",
             "scatter_ms", "wall_ms"}


# ------------------------------------------------------------- synthetic checkpoints --


def _noise(shape, dtype, seed):
    """Random bytes as `dtype` (NaN payloads included), as a torch tensor."""
    es = torch.empty((), dtype=dtype).element_size()
    n = int(np.prod(shape, dtype=np.int64))
    raw = np.random.default_rng(seed).integers(0, 256, n * es, dtype=np.uint8)
    return torch.from_numpy(raw).view(dtype).reshape(shape)


def _cuts(n, parts, seed):
    """`parts` uneven (possibly empty-free) pieces of range(n) as (start, length)."""
    parts = max(1, min(parts, n))
    rng = np.random.default_rng(seed)
    inner = sorted(rng.choice(np.arange(1, n), parts - 1, replace=False)) if parts > 1 else []
    edges = [0, *[int(e) for e in inner], n]
    return [(a, b - a) for a, b in zip(edges, edges[1:])]


def _boxes(shape, parts, dim, seed):
    """Chunk boxes (offsets, sizes) of `shape` split into `parts` along `dim`."""
    if not shape:
        return [((), ())]
    return [(tuple(a if d == dim else 0 for d in range(len(shape))),
             tuple(n if d == dim else s for d, s in enumerate(shape)))
            for a, n in _cuts(shape[dim], parts, seed)]


def _box(t, offsets, sizes):
    for d, (o, n) in enumerate(zip(offsets, sizes)):
        t = t.narrow(d, o, n)
    return t


# name: (shape, dtype, split dim)
TENSORS = {
    "w_bf16": ((37, 96), torch.bfloat16, 0),
    "w_f32": ((24, 130), torch.float32, 1),
    "odd_bf16": ((1001,), torch.bfloat16, 0),
    "idx_i64": ((9, 7, 5), torch.int64, 1),
    "c64": ((33, 17), torch.complex64, 0),
    "scalar": ((), torch.float32, 0),
    "one": ((1,), torch.float64, 0),
}


def write_checkpoint(root, tensors, ranks, seed=0):
    """Each tensor split into `ranks` uneven chunks; chunk r goes to "__<r>_0.distcp" after
    a few junk bytes (odd storage offsets), as the agent writes rank files, plus a
    BYTE_IO entry in rank 0's file.  Returns the global tensors."""
    os.makedirs(root, exist_ok=True)
    rng = np.random.default_rng(seed)
    files = [bytearray() for _ in range(ranks)]
    md, storage = {}, {}
    full = {}
    for k, (name, (shape, dtype, dim)) in enumerate(tensors.items()):
        t = _noise(shape, dtype, seed * 100 + k)
        full[name] = t
        chunks = []
        for r, (off, sizes) in enumerate(_boxes(shape, ranks, dim, seed + k)):
            f = files[r % ranks]
            f += rng.integers(0, 256, int(rng.integers(1, 4)), dtype=np.uint8).tobytes()
            data = _box(t, off, sizes).contiguous().reshape(-1).view(torch.uint8).numpy()
            storage[MetadataIndex(name, off)] = _StorageInfo(f"__{r % ranks}_0.distcp", len(f),
                                                             data.size)
            f += data.tobytes()
            chunks.append(ChunkStorageMetadata(offsets=torch.Size(off), sizes=torch.Size(sizes)))
        md[name] = TensorStorageMetadata(properties=TensorProperties(dtype=dtype),
                                         size=torch.Size(shape), chunks=chunks)
    blob = io.BytesIO()
    torch.save({"step": 7}, blob)
    storage[MetadataIndex("extra")] = _StorageInfo("__0_0.distcp", len(files[0]),
                                                   len(blob.getvalue()))
    files[0] += blob.getvalue()
    md["extra"] = BytesStorageMetadata()
    for r, f in enumerate(files):
        with open(os.path.join(root, f"__{r}_0.distcp"), "wb") as fh:
            fh.write(bytes(f))
    with open(os.path.join(root, ".metadata"), "wb") as fh:
        pickle.dump(Metadata(state_dict_metadata=md, storage_data=storage), fh)
    return full


class Planner:
    """The LoadPlanner calls a StorageReader makes: targets keyed by (fqn, local chunk
    offsets); resolve_tensor narrows them by dest_offsets, as DCP's default planner does."""

    def __init__(self, targets):
        self.targets, self.loaded, self.commits = targets, {}, 0

    def resolve_tensor(self, item):
        t = self.targets[(item.dest_index.fqn, tuple(item.dest_index.offset))]
        return narrow_tensor_by_index(t, item.dest_offsets, item.lengths)

    def commit_tensor(self, item, tensor):
        self.commits += 1

    def load_bytes(self, item, value):
        value.seek(0)
        self.loaded[item.dest_index.fqn] = torch.load(value)


def local_layout(tensors, world, rank, dim_of=None, seed=7):
    """The local chunk of emulated `rank` of a `world`-rank job: each tensor split along
    its dim (dim_of overrides) into uneven pieces."""
    out = {}
    for k, (name, (shape, dtype, dim)) in enumerate(tensors.items()):
        dim = (dim_of or {}).get(name, dim)
        boxes = _boxes(shape, world, dim, seed + k)
        out[name] = boxes[rank] if rank < len(boxes) else None
    return out


def read_items(root, local):
    with open(os.path.join(root, ".metadata"), "rb") as fh:
        meta = pickle.load(fh)
    items = []
    for name, box in local.items():
        if box is None:
            continue
        items += create_read_items_for_chunk_list(
            name, meta.state_dict_metadata[name],
            [ChunkStorageMetadata(offsets=torch.Size(box[0]), sizes=torch.Size(box[1]))])
    items.append(ReadItem(type=LoadItemType.BYTE_IO, dest_index=MetadataIndex("extra"),
                          dest_offsets=torch.Size((0,)), storage_index=MetadataIndex("extra"),
                          storage_offsets=torch.Size((0,)), lengths=torch.Size((0,))))
    return meta, items


def make_targets(tensors, local, device, strided=(), dtype_of=None, seed=1):
    """Canary-filled targets of the local boxes.  Names in `strided` get a row-strided
    view (the first columns of a wider buffer); dtype_of overrides a target dtype."""
    out = {}
    for name, box in local.items():
        if box is None:
            continue
        dtype = (dtype_of or {}).get(name, tensors[name][1])
        sizes = box[1]
        if name in strided:
            wide = _noise((*sizes[:-1], sizes[-1] + 24), dtype, seed).to(device)
            t = wide[..., 3:3 + sizes[-1]]
            assert not t.is_contiguous()
        else:
            t = _noise(sizes, dtype, seed).to(device) if sizes else _noise((), dtype, seed).to(device)
        out[(name, tuple(box[0]))] = t
    return out


def run_reader(reader_cls, root, meta, items, targets):
    reader = reader_cls(root)
    reader.set_up_storage_reader(meta, True)
    planner = Planner(targets)
    reader.read_data(LoadPlan(items), planner).wait()
    if targets and next(iter(targets.values())).is_cuda:
        torch.cuda.synchronize()
    return reader, planner


def _bits(t):
    return t.detach().cpu().contiguous().reshape(-1).view(torch.uint8)


def assert_matches_model(full, local, targets, dtype_of=None):
    for (name, off), t in targets.items():
        if name in (dtype_of or {}):
            continue
        want = _box(full[name], local[name][0], local[name][1])
        assert torch.equal(_bits(t), _bits(want)), name


# ------------------------------------------------------------------------- CPU tests --


@pytest.mark.parametrize("saved,world", [(1, 1), (2, 1), (2, 3), (4, 3), (3, 2)])
@pytest.mark.parametrize("dim_swap", [False, True])
def test_cpu_targets_are_pread_from_the_boxes_dcp_asks_for(tmp_path, saved, world, dim_swap):
    """Every emulated rank of a `world`-rank job, its chunks split on another dim than the
    stored ones when dim_swap, reads exactly its box (numpy model) through pread."""
    full = write_checkpoint(tmp_path, TENSORS, saved)
    dims = {n: (len(s) - 1 - d if dim_swap and s else d) for n, (s, _, d) in TENSORS.items()}
    for rank in range(world):
        local = local_layout(TENSORS, world, rank, dims)
        meta, items = read_items(tmp_path, local)
        targets = make_targets(TENSORS, local, "cpu")
        reader, planner = run_reader(FileDmaReader, tmp_path, meta, items, targets)
        assert_matches_model(full, local, targets)
        assert planner.loaded["extra"] == {"step": 7}
        st = reader.last_read_stats
        assert set(st) == STAT_KEYS
        # BYTE_IO, and the boxes whose target is neither dense nor row-strided
        slow = [i for i in items if i.type == LoadItemType.BYTE_IO
                or _target_rows(planner.resolve_tensor(i)) is None]
        assert st["fallback_items"] == len(slow) and st["device_bytes"] == 0
        want = sum(int(np.prod(i.lengths)) * planner.resolve_tensor(i).element_size()
                   for i in items if i not in slow)
        assert st["host_bytes"] == want  # the box only, never a whole stored chunk
        assert planner.commits == sum(1 for i in items if i.type.name != "BYTE_IO")


def test_piece_builder_against_the_numpy_model(tmp_path):
    """Every piece reads, from its file, exactly the bytes the numpy model puts at its
    target address: 2-d boxes cut on both dims, uneven chunks, 0-d and 1-element
    tensors, an odd bf16 count, bf16 / fp32 / int64 / complex64."""
    full = write_checkpoint(tmp_path, TENSORS, 3, seed=4)
    for world, dims in ((2, None), (3, {"w_bf16": 1, "w_f32": 0, "idx_i64": 2})):
        for rank in range(world):
            local = local_layout(TENSORS, world, rank, dims, seed=11)
            meta, items = read_items(tmp_path, local)
            targets = make_targets(TENSORS, local, "cpu")
            where = {}  # address -> (fqn, byte index into the flat local box)
            for (name, _), t in targets.items():
                where[t.data_ptr()] = name
            cuda, host, slow, committed = _plan_reads(items, meta.storage_data,
                                                      meta.state_dict_metadata,
                                                      Planner(targets).resolve_tensor)
            assert not cuda and len(slow) == 1
            files = {}
            for addr, path, off, n in host:
                if path not in files:
                    files[path] = np.fromfile(tmp_path / path, dtype=np.uint8)
                owner = max(a for a in where if a <= addr)
                name = where[owner]
                box = local[name]
                want = _box(full[name], box[0], box[1]).contiguous().reshape(-1).view(
                    torch.uint8).numpy()
                i = addr - owner
                assert np.array_equal(files[path][off:off + n], want[i:i + n]), name
            total = sum(n for _, _, _, n in host)
            assert total == sum(t.numel() * t.element_size() for t in targets.values())


def test_pieces_never_cross_a_file_in_virtual_space(tmp_path, monkeypatch):
    """The virtual concatenation FileDmaReader hands the library: every piece of every
    plan lies inside one file's range, and the bases strictly increase."""
    import dlrover_b200.shm_handler as sh

    write_checkpoint(tmp_path, TENSORS, 4, seed=2)
    local = local_layout(TENSORS, 1, 0)
    meta, items = read_items(tmp_path, local)
    targets = make_targets(TENSORS, local, "cpu")
    seen = {}

    def fake_groups(ranges, device_index, stream, enqueue, stats):
        class _Plan:
            def restore_files_async(self, fds, bases, s):
                seen["fds"], seen["bases"] = list(fds), list(bases)

        enqueue(_Plan(), None)
        seen["ranges"] = list(ranges)
        return 1

    monkeypatch.setattr(sh, "_restore_file_groups", fake_groups)
    # route every tensor item through the CUDA branch of the builder without a GPU
    import dlrover_b200.flash_checkpoint.fsdp_engine as fe

    real = fe._plan_reads

    def as_cuda(*a):
        cuda, host, slow, tg = real(*a)
        return host, [], slow, [(i, _FakeCuda(t)) for i, t in tg]

    class _FakeCuda:
        def __init__(self, t):
            self.t, self.is_cuda, self.device = t, True, torch.device("cuda", 0)

    monkeypatch.setattr(fe, "_plan_reads", as_cuda)
    reader, _ = run_reader(FileDmaReader, tmp_path, meta, items, targets)
    assert seen["fds"] and len(seen["fds"]) == len(seen["bases"])
    bases = seen["bases"]
    assert len(bases) == 4 and all(b > a for a, b in zip(bases, bases[1:]))
    sizes = [os.path.getsize(tmp_path / f"__{r}_0.distcp") for r in range(4)]
    for _, v, n in seen["ranges"]:
        k = max(i for i, b in enumerate(bases) if b <= v)
        end = bases[k + 1] if k + 1 < len(bases) else bases[k] + sizes[k]
        assert v + n <= end and v - bases[k] + n <= sizes[k]
    assert reader.last_read_stats["files"] == 4


def test_a_short_file_is_refused_before_any_write(tmp_path):
    write_checkpoint(tmp_path, TENSORS, 3, seed=5)
    local = local_layout(TENSORS, 1, 0)
    meta, items = read_items(tmp_path, local)
    targets = make_targets(TENSORS, local, "cpu")
    before = {k: t.clone() for k, t in targets.items()}
    path = tmp_path / "__1_0.distcp"
    os.truncate(path, os.path.getsize(path) - 5)
    with pytest.raises(ValueError, match="__1_0.distcp"):
        run_reader(FileDmaReader, tmp_path, meta, items, targets)
    for k, t in targets.items():
        assert torch.equal(_bits(t), _bits(before[k])), k


def test_engine_switch_picks_the_reader(tmp_path, monkeypatch):
    from dlrover_b200.flash_checkpoint.fsdp_engine import FsdpCheckpointEngine

    engine = FsdpCheckpointEngine.__new__(FsdpCheckpointEngine)
    assert engine.storage_dma is False
    monkeypatch.setenv("DLROVER_B200_STORAGE_DMA", "1")
    assert engine.storage_dma is True
    engine.storage_dma = False
    assert engine.storage_dma is False
    assert issubclass(FileDmaReader, FileReader)


def test_files_entry_point_rejects_bad_arguments():
    lib = native.load_library()
    assert lib.fc_restore_files_async(None, 1, None, None, None) == native.FC_EINVAL
    assert b"fc_restore_files_async" in lib.fc_last_error()


# ------------------------------------------------------------------------- GPU tests --


def _compare_with_file_reader(root, tensors, local, device, strided=(), dtype_of=None):
    meta, items = read_items(root, local)
    ref_t = make_targets(tensors, local, device, strided, dtype_of)
    got_t = make_targets(tensors, local, device, strided, dtype_of)
    run_reader(FileReader, root, meta, items, ref_t)
    reader, planner = run_reader(FileDmaReader, root, meta, items, got_t)
    for k in ref_t:
        assert torch.equal(_bits(got_t[k]), _bits(ref_t[k])), k
    assert planner.loaded["extra"] == {"step": 7}
    return reader.last_read_stats


def _mixed(device):
    """Half the tensors on the GPU, the rest on the CPU."""
    return {n: device if i % 3 else "cpu" for i, n in enumerate(TENSORS)}


@gpu
@pytest.mark.parametrize("saved", [2, 4])
@pytest.mark.parametrize("world", [1, 3])
def test_resharded_restore_is_bitwise_file_reader(cuda_device, tmp_path, saved, world):
    """Dense and row-strided CUDA targets, odd storage offsets, a dtype-mismatch
    fallback; every emulated rank of the new world in one process."""
    tensors = dict(TENSORS)
    tensors["wide_bf16"] = ((48, 512), torch.bfloat16, 0)  # 1 KiB rows: row-strided
    tensors["wide_f32"] = ((40, 160), torch.float32, 1)
    full = write_checkpoint(tmp_path, tensors, saved, seed=saved)
    for rank in range(world):
        local = local_layout(tensors, world, rank)
        st = _compare_with_file_reader(tmp_path, tensors, local, cuda_device,
                                       strided=("wide_bf16",),
                                       dtype_of={"w_f32": torch.float64})
        assert set(st) == STAT_KEYS
        assert st["device_bytes"] > 0 and st["plans"] >= 1
        meta, items = read_items(tmp_path, local)
        targets = make_targets(tensors, local, cuda_device, ("wide_bf16",))
        # BYTE_IO, the dtype mismatch, and the boxes whose rows are below _row_ranges'
        # minimum on the device
        planner = Planner(make_targets(tensors, local, cuda_device, ("wide_bf16",),
                                       {"w_f32": torch.float64}))
        slow = [i for i in items if i.type == LoadItemType.BYTE_IO or i.dest_index.fqn == "w_f32"
                or _target_rows(planner.resolve_tensor(i)) is None]
        assert st["fallback_items"] == len(slow)
        assert any(i.dest_index.fqn == "wide_bf16" for i in items if i not in slow)
        run_reader(FileDmaReader, tmp_path, meta, items, targets)
        assert_matches_model(full, local, targets)


@gpu
def test_cpu_and_cuda_targets_in_one_read(cuda_device, tmp_path):
    full = write_checkpoint(tmp_path, TENSORS, 4, seed=9)
    local = local_layout(TENSORS, 3, 1)
    meta, items = read_items(tmp_path, local)
    where = _mixed(cuda_device)
    targets = {}
    for k, t in make_targets(TENSORS, local, "cpu").items():
        targets[k] = t.to(where[k[0]])
    reader, _ = run_reader(FileDmaReader, tmp_path, meta, items, targets)
    assert_matches_model(full, local, targets)
    st = reader.last_read_stats
    assert st["device_bytes"] > 0 and st["host_bytes"] > 0


@gpu
def test_an_8_mib_arena_streams_the_plan(cuda_device, tmp_path, monkeypatch):
    """DLROVER_B200_ARENA_LIMIT_MB=8 caps the arena of a fresh context below the plan."""
    import dlrover_b200.shm_handler as sh

    tensors = {"big": ((3000, 2048), torch.bfloat16, 0), "w": ((512, 300), torch.float32, 1)}
    write_checkpoint(tmp_path, tensors, 4, seed=3)
    ctx = native.Context(0)
    monkeypatch.setattr(sh.native, "get_context", lambda index: ctx)
    monkeypatch.setenv("DLROVER_B200_ARENA_LIMIT_MB", "8")
    try:
        st = _compare_with_file_reader(tmp_path, tensors, local_layout(tensors, 1, 0),
                                       cuda_device)
        assert st["device_bytes"] > 8 << 20 and st["plans"] == 1
        assert ctx.arena_info()[1] == 8 << 20
    finally:
        ctx.destroy()


@gpu
def test_two_targets_reading_the_same_bytes_take_two_plans(cuda_device, tmp_path):
    """Two local chunks of one rank that overlap in the checkpoint: the same file bytes
    go to two targets, so the reader splits them into two disjoint plans."""
    tensors = {"w": ((64, 256), torch.float32, 0)}
    full = write_checkpoint(tmp_path, tensors, 2, seed=6)
    with open(tmp_path / ".metadata", "rb") as fh:
        meta = pickle.load(fh)
    boxes = [((0, 0), (40, 256)), ((20, 0), (44, 256))]  # rows 20..39 read twice
    items = create_read_items_for_chunk_list(
        "w", meta.state_dict_metadata["w"],
        [ChunkStorageMetadata(offsets=torch.Size(o), sizes=torch.Size(s)) for o, s in boxes])
    targets = {("w", o): torch.zeros(s, device=cuda_device) for o, s in boxes}
    reader, _ = run_reader(FileDmaReader, tmp_path, meta, items, targets)
    assert reader.last_read_stats["plans"] == 2
    for o, s in boxes:
        assert torch.equal(_bits(targets[("w", o)]), _bits(_box(full["w"], o, s)))


@gpu
def test_truncated_second_file_changes_no_target(cuda_device, tmp_path):
    write_checkpoint(tmp_path, TENSORS, 3, seed=8)
    local = local_layout(TENSORS, 1, 0)
    meta, items = read_items(tmp_path, local)
    targets = make_targets(TENSORS, local, cuda_device)
    before = {k: _bits(t).clone() for k, t in targets.items()}
    path = tmp_path / "__1_0.distcp"
    os.truncate(path, os.path.getsize(path) - 1)
    with pytest.raises(ValueError, match="__1_0.distcp"):
        run_reader(FileDmaReader, tmp_path, meta, items, targets)
    torch.cuda.synchronize()
    for k, t in targets.items():
        assert torch.equal(_bits(t), before[k]), k


# ---------------------------------------------------- the library against the byte model --


@gpu
@pytest.mark.parametrize("variant", [native.VARIANT_LSU, native.VARIANT_TMA], ids=["lsu", "tma"])
def test_files_restore_writes_exactly_the_planned_bytes(cuda_device, tmp_path, monkeypatch,
                                                        variant):
    """fc_restore_files_async over 3 files, each holding one range of the saved host
    buffer, cut inside runs at odd offsets: the targets, the arena and the canaries equal
    the byte model of a one-file restore, into the full arena and through an 8 MiB one.
    With one file it issues the same copies as fc_restore_file_async."""
    from tests.test_kernel_model import (DEFAULT_CHUNK, _context, _tiles, _world,
                                         mixed_layout, pattern)

    lay = mixed_layout(5, _tiles("default"), DEFAULT_CHUNK, mapped=True)
    for bounded in (False, True):
        lay.tgt.write(lay.tgt.base, pattern(lay.tgt.np.size))
        ctx = _context("default", variant, 8 << 20 if bounded else 0)
        ctx.set_stage(3, 1 << 20)
        with _world(ctx, lay, 0, variant, bounded=bounded) as w:
            host = w.host["A"]  # the checkpoint's bytes: random, the canary elsewhere
            host[:] = np.random.default_rng(bounded).integers(0, 256, host.size, dtype=np.uint8)
            w.host_t["A"].copy_(torch.from_numpy(host))
            end = lay.host_end
            cuts = [0, end // 3 + 1, 2 * end // 3 + 7]
            paths, fds, fd1 = [], [], -1
            for k, lo in enumerate(cuts):
                hi = cuts[k + 1] if k + 1 < len(cuts) else host.size
                p = tmp_path / f"part{k}_{bounded}.bin"
                p.write_bytes(host[lo:hi].tobytes())
                paths.append(p)
            one = tmp_path / f"whole_{bounded}.bin"
            one.write_bytes(host.tobytes())
            plan = w.plans["Q"]["plan"]
            try:
                fds = [os.open(p, os.O_RDONLY) for p in paths]
                fd1 = os.open(one, os.O_RDONLY)
                lay.tgt.write(lay.tgt.base, pattern(lay.tgt.np.size))
                copies_one = w.restore(source="file", src=fd1)
                w.check(f"one file bounded={bounded}")
                lay.tgt.write(lay.tgt.base, pattern(lay.tgt.np.size))
                with monkeypatch.context() as m:
                    m.setattr(plan, "restore_file_async",
                              lambda fd, s: plan.restore_files_async([fd], [0], s))
                    assert w.restore(source="file", src=fd1) == copies_one
                w.check(f"n = 1 bounded={bounded}")
                lay.tgt.write(lay.tgt.base, pattern(lay.tgt.np.size))
                with monkeypatch.context() as m:
                    m.setattr(plan, "restore_file_async",
                              lambda fd, s: plan.restore_files_async(fds, cuts, s))
                    w.restore(source="file", src=fds[0])
                w.check(f"3 files bounded={bounded}")
                # a short middle file: refused before anything moves
                os.truncate(paths[1], (cuts[2] - cuts[1]) // 2)
                lay.tgt.write(lay.tgt.base, pattern(lay.tgt.np.size))
                with pytest.raises(native.NativeError, match="file 1") as e:
                    plan.restore_files_async(fds, cuts, torch.cuda.current_stream())
                assert e.value.code == native.FC_EIO
                w.check(f"short file bounded={bounded}")
            finally:
                for fd in fds + [fd1]:
                    if fd >= 0:
                        os.close(fd)


# ------------------------------------------------------ a real FSDP job, same world --


@gpu
def test_fsdp_shard_checkpointer_restores_from_storage_with_the_switch(cuda_device, run_env,
                                                                        monkeypatch, tmp_path):
    """A world-1 FSDP job saves to DISK; with its shared memory hidden, load() reads the
    shard file.  With storage_dma on, the logits and the AdamW state equal those of the
    restore with the switch off, and only non-tensor entries take the fallback."""
    import torch.distributed as dist
    from torch.distributed.fsdp import FullyShardedDataParallel as FSDP
    from torch.distributed.fsdp import StateDictType

    from dlrover_b200.ckpt_saver import CheckpointConfig
    from dlrover_b200.flash_checkpoint.api import StorageType
    from dlrover_b200.flash_checkpoint.fsdp import FsdpShardCheckpointer
    from tests.test_fsdp_checkpointer import _setup, _train_one_step

    _setup(cuda_device, monkeypatch, "nccl")
    try:
        ckpt = FsdpShardCheckpointer(str(tmp_path))
        model, opt = _train_one_step(cuda_device, 0)
        x = torch.randn(4, 64, device=cuda_device)
        ckpt.save_checkpoint(10, model, opt, {"step": 10}, storage_type=StorageType.DISK)
        ckpt.wait_latest_checkpoint(timeout=120)
        handler = ckpt.engine._shm_handler
        monkeypatch.setattr(handler, "get_checkpoint_config", lambda default: CheckpointConfig())
        monkeypatch.setattr(handler, "no_checkpoint_state", lambda: True)
        readers, got = [], {}
        real_load = ckpt.engine.load

        def load(resume_path=""):
            readers.append(real_load(resume_path))
            return readers[-1]

        monkeypatch.setattr(ckpt.engine, "load", load)
        calls, real_read = [], FileDmaReader.read_data

        def read_data(self, plan, planner):
            fut = real_read(self, plan, planner)
            calls.append((plan, self.last_read_stats, self.state_dict_metadata))
            return fut

        monkeypatch.setattr(FileDmaReader, "read_data", read_data)
        for dma in (False, True):
            ckpt.engine.storage_dma = dma
            model2, opt2 = _train_one_step(cuda_device, 1)
            assert ckpt.load_checkpoint(model2, opt2).get("step") == 10
            with torch.no_grad():
                logits = model2(x).clone()
            with FSDP.state_dict_type(model2, StateDictType.FULL_STATE_DICT):
                optim = FSDP.optim_state_dict(model2, opt2)
            got[dma] = (logits, optim)
        assert type(readers[0]) is FileReader and type(readers[1]) is FileDmaReader
        # the model and then the optimizer state: every tensor item took a direct path
        assert len(calls) == 2
        for plan, st, meta in calls:
            non_tensor = [i for i in plan.items if i.type == LoadItemType.BYTE_IO or
                          not isinstance(meta.get(i.storage_index.fqn), TensorStorageMetadata)]
            assert st["fallback_items"] == len(non_tensor)
            assert st["files"] == 1 and set(st) == STAT_KEYS
        assert calls[0][1]["device_bytes"] > 0 and calls[1][1]["device_bytes"] > 0
        assert torch.equal(got[True][0], got[False][0])
        a, b = got[True][1]["state"], got[False][1]["state"]
        assert sorted(a) == sorted(b)
        for k in a:
            for name in a[k]:
                va, vb = a[k][name], b[k][name]
                if torch.is_tensor(va):
                    assert torch.equal(_bits(va), _bits(vb)), (k, name)
                else:
                    assert va == vb, (k, name)
        ckpt.engine.close()
    finally:
        dist.destroy_process_group()
