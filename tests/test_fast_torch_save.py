"""fast_torch_save.fast_save must produce EXACTLY the bytes of torch.save
(the agent's persist format, reference ckpt_saver.py:1079-1122).  The >4 GiB
zip64 cases (offsets past 4 GiB, one tensor >= 4 GiB) run only
with FC_SLOW_TESTS=1 because each needs ~10 GB of RAM and ~40 s."""

import hashlib
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
import fixtures  # noqa: E402
from dlrover_b200 import fast_torch_save as fts  # noqa: E402
from tests.util import golden  # noqa: E402


def _sha(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for block in iter(lambda: f.read(1 << 24), b""):
            h.update(block)
    return h.hexdigest()


def _same(obj, tmp_path, stem="rank_0", threads=4):
    a, b = tmp_path / "a", tmp_path / "b"
    os.makedirs(a, exist_ok=True)
    os.makedirs(b, exist_ok=True)
    torch.save(obj, str(a / f"{stem}.pt"))
    fts.fast_save(obj, str(b / f"{stem}.pt"), threads=threads)
    return _sha(a / f"{stem}.pt") == _sha(b / f"{stem}.pt"), _sha(b / f"{stem}.pt")


@pytest.mark.parametrize("name", list(fixtures.FIXTURES))
def test_fixtures_identical_to_torch_save(tmp_path, name):
    assert _same(fixtures.FIXTURES[name](), tmp_path)[0]


@pytest.mark.parametrize("name", list(fixtures.FIXTURES))
def test_agent_persist_equals_reference_file(run_env, tmp_path, name):
    """What the agent does: tensors aliasing the shm segment -> file.  The sha256
    must be the one of the file the REFERENCE's agent wrote for the same
    fixture (tests/golden/make_golden.py)."""
    from dlrover_b200.shm_handler import (DLROVER_CKPT_CONFIG_KEY, CheckpointConfig,
                                          SharedMemoryHandler)

    info, _ = golden(name)
    if torch.__version__ != info["torch_version"]:
        pytest.skip("golden written by another torch version")
    handler = SharedMemoryHandler(0, host=True)
    handler.save_state_dict({"model_states": fixtures.FIXTURES[name](),
                             DLROVER_CKPT_CONFIG_KEY: CheckpointConfig(step=5, paths={})})
    loaded = handler.load_state_dict()
    p = str(tmp_path / "rank_0.pt")
    fts.fast_save(loaded["model_states"], p, threads=4)
    assert _sha(p) == info["torch_save_sha256"]
    del loaded
    handler.unlink()
    handler.close()


def test_structures(tmp_path):
    t = torch.arange(10.)
    cases = {
        "empty": {},
        "scalars": {"a": 1, "b": "x", "c": None, "d": (1, 2)},
        "shared_storage": {"x": t, "y": t[2:], "z": [t, {"k": t.view(2, 5)}]},
        "zero_numel": {"e": torch.empty(0), "f": torch.empty(0, dtype=torch.int64), "g": t},
        "many": {f"p{i}": torch.full((i % 7 + 1, 3), float(i)) for i in range(300)},
        "dtypes": {str(d): torch.ones(5, dtype=d) for d in (torch.bool, torch.uint8, torch.int16,
                                                            torch.bfloat16, torch.float64,
                                                            torch.complex64)},
    }
    for stem, obj in cases.items():
        same, _ = _same(obj, tmp_path, stem=stem)
        assert same, stem


def test_file_stem_is_the_archive_prefix(tmp_path):
    for stem in ("model_optim_rng", "x", "mp_rank_00_model_states"):
        same, _ = _same({"w": torch.ones(3)}, tmp_path, stem=stem)
        assert same, stem


def test_multi_piece_records_and_views_on_shared_memory(tmp_path):
    """Payload bigger than one write piece, backed by a buffer we do not own
    (what the agent sees: tensors aliasing the shm segment)."""
    raw = bytearray((200 << 20) + 12)
    for i in range(0, len(raw), 4099):
        raw[i] = i % 251
    big = torch.frombuffer(raw, dtype=torch.uint8, count=200 << 20, offset=4)
    small = torch.frombuffer(raw, dtype=torch.int16, count=4, offset=(200 << 20) + 4)
    same, _ = _same({"big": big, "small": small, "step": 3}, tmp_path, threads=6)
    assert same
    back = torch.load(tmp_path / "b" / "rank_0.pt")
    assert torch.equal(back["big"], big) and back["step"] == 3


def test_unsupported_falls_back_to_torch_save(tmp_path, monkeypatch):
    def boom(*a, **k):
        raise fts.Unsupported("nope")

    monkeypatch.setattr(fts, "fast_save", boom)
    p = str(tmp_path / "f.pt")
    fts.save({"a": torch.ones(2)}, p)
    assert torch.equal(torch.load(p)["a"], torch.ones(2))


@pytest.mark.skipif(os.getenv("FC_SLOW_TESTS") != "1", reason="needs ~10 GB RAM, FC_SLOW_TESTS=1")
def test_zip64(tmp_path):
    far = {f"t{i}": torch.full(((768 << 20) // 2,), float(i), dtype=torch.bfloat16)
           for i in range(7)}
    assert _same(far, tmp_path, stem="far", threads=8)[0]
    del far
    huge = {"h": torch.zeros((4 << 30) + 128, dtype=torch.uint8), "tail": torch.ones(10)}
    assert _same(huge, tmp_path, stem="huge", threads=8)[0]
