import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "timeout: per-test timeout (pytest-timeout)")
    # The suite states what the DEFAULT configuration does (several tests assert that a
    # feature is on): switches left in the caller's shell must not change the outcome.
    # FC_TEST_KEEP_ENV=1 keeps them (running the suite under a non-default switch on purpose).
    if os.getenv("FC_TEST_KEEP_ENV") != "1":
        for k in [k for k in os.environ if k.startswith("DLROVER_B200_")
                  or k in ("FC_DRAIN_MODE", "FC_DRAIN_SPIN", "FC_NO_NUMA", "FC_NO_HUGEPAGE",
                           "FC_NO_STAGING")]:
            del os.environ[k]
    # built artefacts are git-ignored: a fresh checkout has no .so yet
    lib = os.path.join(ROOT, "dlrover_b200", "csrc", "libflashckpt.so")
    ora = os.path.join(ROOT, "oracle", "_ref", "libpack_oracle.so")
    if not (os.path.exists(lib) and os.path.exists(ora)):
        import __graft_entry__

        __graft_entry__.build()


def pytest_collection_modifyitems(config, items):
    # `-m gpu` on a box without CUDA must fail loudly, not skip silently.
    pass


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    assert torch.cuda.is_available(), "gpu-marked test needs a CUDA device"
    torch.cuda.set_device(0)
    return torch.device("cuda", 0)


@pytest.fixture
def run_env(monkeypatch, tmp_path):
    """Isolated IPC namespace: unique TORCHELASTIC_RUN_ID (socket dir + shm
    names), saver hosted in-process (ROLE_NAME=dlrover-trainer)."""
    import shutil
    import uuid

    run_id = "t" + uuid.uuid4().hex[:10]
    monkeypatch.setenv("TORCHELASTIC_RUN_ID", run_id)
    monkeypatch.setenv("ROLE_NAME", "dlrover-trainer")
    for k in ("LOCAL_RANK", "RANK", "LOCAL_WORLD_SIZE", "GROUP_RANK", "GROUP_WORLD_SIZE",
              "NODE_RANK", "NODE_NUM", "WORLD_SIZE"):
        monkeypatch.delenv(k, raising=False)
    yield run_id
    from dlrover_b200.ckpt_saver import AsyncCheckpointSaver

    saver = AsyncCheckpointSaver._saver_instance
    if saver is not None:
        try:
            saver.close()
        except Exception:
            pass
        AsyncCheckpointSaver._saver_instance = None
    shutil.rmtree(os.path.join("/tmp/ckpt_sock", run_id), ignore_errors=True)
    # whatever a failed test left behind (segments are up to 16 GB on the GPU box)
    import glob

    for leftover in glob.glob(f"/dev/shm/{run_id}_*"):
        try:
            os.unlink(leftover)
        except OSError:
            pass
    import glob

    for f in glob.glob(f"/dev/shm/{run_id}_*"):
        try:
            os.unlink(f)
        except OSError:
            pass
