"""What the two storage readers (restore_file_into, FileDmaReader) share: the one row
walker (_view_rows) and the rule each caller keeps on top of it, the one-device check of
the piece reader, and the one short-file error."""

import os

import pytest
import torch
from torch.distributed.checkpoint.metadata import (
    ChunkStorageMetadata,
    MetadataIndex,
    TensorProperties,
    TensorStorageMetadata,
)
from torch.distributed.checkpoint.planner import LoadPlan, ReadItem

import dlrover_b200.flash_checkpoint.fsdp_engine as fe
import dlrover_b200.shm_handler as sh
from dlrover_b200.flash_checkpoint.fsdp_engine import FileDmaReader, _item_rows, _StorageInfo
from dlrover_b200.shm_handler import (ShortFileError, _box_ranges, _row_ranges, _target_rows,
                                      _view_rows, restore_file_into)
from dlrover_b200.torch_file_index import index_file
from tests.test_fsdp_storage_restore import (TENSORS, Planner, _bits, local_layout,
                                             make_targets, read_items, write_checkpoint)

# ------------------------------------------------------- the walker, through each caller --


def _rows(t, **kw):
    rows = _row_ranges(t, 1000, **kw)
    return None if rows is None else [(p - t.data_ptr(), o, n) for p, o, n in rows]


def _box(shape, offsets, full):
    return [(o, n) for _, o, n in _box_ranges(torch.zeros(shape), offsets, full, 100)]


def _item(chunk, offsets, lengths):
    md = TensorStorageMetadata(
        properties=TensorProperties(dtype=torch.float32), size=torch.Size(chunk),
        chunks=[ChunkStorageMetadata(offsets=torch.Size([0] * len(chunk)),
                                     sizes=torch.Size(chunk))])
    item = ReadItem(type=fe.LoadItemType.TENSOR, dest_index=MetadataIndex("w", (0,) * len(chunk)),
                    dest_offsets=torch.Size([0] * len(chunk)),
                    storage_index=MetadataIndex("w", (0,) * len(chunk)),
                    storage_offsets=torch.Size(offsets), lengths=torch.Size(lengths))
    return _item_rows(md, item, _StorageInfo("__0_0.distcp", 10, 0))


_SIZE1 = torch.zeros(20).as_strided((3, 1, 4), (8, 99, 1))  # size-1 dim of any stride
_EVEN = torch.zeros(8)[::2]                                  # one-element rows

WALKER_CASES = {
    # the walker itself: (byte offset, nbytes) rows
    "walker-contiguous": (lambda: _view_rows((2, 3), (3, 1), 1, 4), [(4, 24)]),
    "walker-0d": (lambda: _view_rows((), (), 5, 2), [(10, 2)]),
    "walker-size1": (lambda: _view_rows((3, 1, 4), (8, 99, 1), 0, 1), [(0, 4), (8, 4), (16, 4)]),
    "walker-1elem-min0": (lambda: _view_rows((4,), (2,), 0, 4),
                          [(0, 4), (8, 4), (16, 4), (24, 4)]),
    "walker-1elem-min4": (lambda: _view_rows((4,), (2,), 0, 4, min_row_bytes=4),
                          [(0, 4), (8, 4), (16, 4), (24, 4)]),
    "walker-1elem-min5": (lambda: _view_rows((4,), (2,), 0, 4, min_row_bytes=5), None),
    "walker-negative": (lambda: _view_rows((3, 4), (-4, 1), 8, 1), None),
    "walker-max_rows": (lambda: _view_rows((5, 4), (8, 1), 0, 1, max_rows=4), None),
    "walker-at-max_rows": (lambda: len(_view_rows((5, 4), (8, 1), 0, 1, max_rows=5)), 5),
    # _row_ranges: (ptr - data_ptr, segment offset, nbytes); a dense tensor is declined
    "row_ranges-contiguous": (lambda: _rows(torch.zeros(4, 6), min_row_bytes=1), None),
    "row_ranges-0d": (lambda: _rows(torch.zeros(()), min_row_bytes=1), None),
    "row_ranges-size1": (lambda: _rows(_SIZE1, min_row_bytes=1),
                         [(0, 1000, 16), (32, 1016, 16), (64, 1032, 16)]),
    "row_ranges-1elem-min1": (lambda: _rows(_EVEN, min_row_bytes=1),
                              [(0, 1000, 4), (8, 1004, 4), (16, 1008, 4), (24, 1012, 4)]),
    "row_ranges-1elem-min256": (lambda: _rows(_EVEN), None),
    "row_ranges-max_rows": (lambda: _rows(torch.zeros(5, 8)[:, :4], min_row_bytes=1,
                                          max_rows=4), None),
    # _target_rows on the CPU: a dense tensor is one row, a CPU row may be one element
    "target_rows-contiguous": (lambda: len(_target_rows(torch.zeros(4, 6))), 1),
    "target_rows-0d": (lambda: len(_target_rows(torch.zeros(()))), 1),
    "target_rows-1elem": (lambda: [n for _, n in _target_rows(_EVEN)], [4, 4, 4, 4]),
    # _box_ranges: (segment offset, nbytes) of a box in a row-major full tensor
    "box-whole": (lambda: _box((2, 3), (0, 0), (2, 3)), [(100, 24)]),
    "box-0d": (lambda: _box((), (), ()), [(100, 4)]),
    "box-size1": (lambda: _box((2, 1, 4), (1, 2, 3), (3, 5, 8)), [(336, 16), (496, 16)]),
    "box-1elem": (lambda: _box((3, 1), (0, 1), (3, 2)), [(104, 4), (112, 4), (120, 4)]),
    # _item_rows: (file offset, nbytes) of a box of a stored chunk at file offset 10
    "item-whole": (lambda: _item((2, 3), (0, 0), (2, 3)), [(10, 24)]),
    "item-0d": (lambda: _item((), (), ()), [(10, 4)]),
    "item-size1": (lambda: _item((3, 5, 8), (1, 2, 3), (2, 1, 4)), [(246, 16), (406, 16)]),
    "item-1elem": (lambda: _item((3, 2), (0, 1), (3, 1)), [(14, 4), (22, 4), (30, 4)]),
    "item-max_rows": (lambda: _item((65537, 2), (0, 0), (65537, 1)), None),
}


@pytest.mark.parametrize("case", list(WALKER_CASES))
def test_row_walker_results_and_declines_through_each_caller(case):
    got, want = WALKER_CASES[case]
    assert got() == want


def test_box_above_the_row_cap_raises():
    with pytest.raises(ValueError, match="too many rows"):
        _box((65537, 1), (0, 0), (65537, 2))
    assert len(_box((65536, 1), (0, 0), (65536, 2))) == 65536


@pytest.mark.parametrize("view,ok", [
    (lambda: torch.arange(8.0)[::2], False),                # last dim neither dense nor size 1
    (lambda: torch.arange(8.0).reshape(4, 2)[:, :1], True),  # size-1 last dim: 1-element rows
    (lambda: torch.arange(12.0).reshape(3, 4)[:, 1:3], True),  # row-strided
    (lambda: torch.arange(6.0).reshape(2, 3).t(), False),    # transposed
    (lambda: torch.tensor(3.5), True),                       # 0-d
    (lambda: torch.zeros(65537, 2)[:, :1], False),           # above the row cap
    (lambda: torch.zeros(65536, 2)[:, :1], True),
], ids=["strided-last", "size1-last", "row-strided", "transposed", "0d", "rows-above-cap",
        "rows-at-cap"])
def test_file_views_the_torch_save_reader_takes_and_refuses(tmp_path, view, ok):
    """The file caller's own rule on top of the walker: a stored view whose last dim is
    neither dense nor of size 1 is refused, even where the walker has rows for it."""
    v = view()
    path = str(tmp_path / "ckpt.pt")
    torch.save({"v": v}, path)
    tgt = {"v": torch.full(v.shape, -1.0)}
    if not ok:
        with pytest.raises(ValueError, match="v: the file holds a view"):
            restore_file_into(path, tgt)
        assert bool((tgt["v"] == -1).all())
        return
    restore_file_into(path, tgt)
    assert torch.equal(tgt["v"], v)


# --------------------------------------------------------------- the shared piece reader --


class _FakeCuda:
    def __init__(self, t, index):
        self.t, self.is_cuda, self.device = t, True, torch.device("cuda", index)


def test_cuda_targets_on_two_devices_are_refused_before_any_write(tmp_path, monkeypatch):
    """FileDmaReader scatters through one device's arena: targets on two devices raise
    before any file byte moves, fallback items included."""
    write_checkpoint(tmp_path, TENSORS, 2, seed=3)
    local = local_layout(TENSORS, 1, 0)
    meta, items = read_items(tmp_path, local)
    targets = make_targets(TENSORS, local, "cpu")
    before = {k: _bits(t).clone() for k, t in targets.items()}
    groups = []
    monkeypatch.setattr(sh, "_restore_file_groups", lambda *a: groups.append(a) or 1)
    real = fe._plan_reads

    def as_cuda(*a):
        cuda, host, slow, tg = real(*a)
        return host, [], slow, [(i, _FakeCuda(t, k % 2)) for k, (i, t) in enumerate(tg)]

    monkeypatch.setattr(fe, "_plan_reads", as_cuda)
    reader = FileDmaReader(tmp_path)
    reader.set_up_storage_reader(meta, True)
    planner = Planner(targets)
    with pytest.raises(ValueError, match="one device; got cuda:0 and cuda:1"):
        reader.read_data(LoadPlan(items), planner)
    assert not groups and not planner.loaded and planner.commits == 0
    for k, t in targets.items():
        assert torch.equal(_bits(t), before[k]), k


def test_short_files_raise_one_error_for_both_readers(tmp_path):
    """A file too short for the restore raises ShortFileError, an OSError and a
    ValueError with one wording naming the file and the offset, before any target
    changes."""
    path = str(tmp_path / "ckpt.pt")
    torch.save({"w": torch.arange(1000.0)}, path)
    idx = index_file(path)
    os.truncate(path, idx.tree["w"].file_offset + 100)
    tgt = {"w": torch.zeros(1000)}
    wording = r": the restore reads bytes up to file offset \d+, the file ends at \d+"
    with pytest.raises(OSError, match="ckpt.pt" + wording) as e:
        restore_file_into(path, tgt, index=idx)
    assert isinstance(e.value, ValueError) and isinstance(e.value, ShortFileError)
    assert not tgt["w"].any()

    root = tmp_path / "dcp"
    write_checkpoint(root, TENSORS, 2, seed=4)
    local = local_layout(TENSORS, 1, 0)
    meta, items = read_items(root, local)
    targets = make_targets(TENSORS, local, "cpu")
    before = {k: _bits(t).clone() for k, t in targets.items()}
    os.truncate(root / "__1_0.distcp", os.path.getsize(root / "__1_0.distcp") - 1)
    reader = FileDmaReader(root)
    reader.set_up_storage_reader(meta, True)
    with pytest.raises(ValueError, match="__1_0.distcp" + wording) as e:
        reader.read_data(LoadPlan(items), Planner(targets))
    assert isinstance(e.value, OSError) and isinstance(e.value, ShortFileError)
    for k, t in targets.items():
        assert torch.equal(_bits(t), before[k]), k
