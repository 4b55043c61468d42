"""Interoperability with the REFERENCE's agent half: the reference's own
AsyncCheckpointSaver (its byte code under oracle/_ref/pyref, built by oracle/build_ref.py,
run in a separate process, as `dlrover-run` would host it) serves OUR trainer-side
DdpCheckpointer running in wire-compat mode: lock / queue / dict RPCs, the meta tree, the
saver ClassMeta and the SAVE event all cross the process boundary as the reference's
pickles, and the reference persists our shared-memory bytes with its own code.
Runs only where oracle/_ref/pyref has been built."""

import os
import subprocess
import sys
import time
import uuid

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "pyref")


def _ref_trainer_built():
    return os.path.exists(os.path.join(REF, "dlrover", "trainer", "torch", "flash_checkpoint",
                                       "ddp.pyc"))


pytestmark = pytest.mark.skipif(not _ref_trainer_built(),
                                reason="oracle/_ref/pyref not built (no reference to build it from)")

AGENT = r"""
import sys, time
from unittest import mock
sys.path.insert(0, %r)
sys.modules.setdefault("kubernetes", mock.MagicMock())
from dlrover.python.elastic_agent.torch.ckpt_saver import AsyncCheckpointSaver
AsyncCheckpointSaver.start_async_saving_ckpt()
print("AGENT_READY", flush=True)
time.sleep(120)
"""

TRAINER = r"""
import os, sys, time
sys.path.insert(0, %r)
import torch
import dlrover_b200                       # DLROVER_B200_WIRE_COMPAT=1 -> enable_wire_compat()
from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType
from dlrover_b200.common.multi_process import SocketRequest
assert SocketRequest.__module__ == "dlrover.python.common.multi_process"
d = sys.argv[1]
ckpt = DdpCheckpointer(d)
sd = {"w": torch.arange(1000, dtype=torch.float32), "b": torch.ones(7, dtype=torch.bfloat16),
      "step": 12}
ckpt.save_checkpoint(12, sd, storage_type=StorageType.MEMORY)
back = ckpt.load_checkpoint()
assert torch.equal(back["w"], sd["w"]) and back["step"] == 12
del back
ckpt.save_checkpoint(13, sd, storage_type=StorageType.DISK)
ckpt.wait_latest_checkpoint(timeout=60)
print("TRACKER", open(os.path.join(d, "dlrover_latest.txt")).read())
print("FILES", sorted(os.listdir(os.path.join(d, "13"))))
on_disk = torch.load(os.path.join(d, "13", "rank_0.pt"))
assert torch.equal(on_disk["w"], sd["w"]) and torch.equal(on_disk["b"], sd["b"])
print("TRAINER_OK")
ckpt.engine.close()
"""


def test_our_trainer_against_the_reference_agent(tmp_path):
    run_id = "wire" + uuid.uuid4().hex[:8]
    env = dict(os.environ, TORCHELASTIC_RUN_ID=run_id, ROLE_NAME="dlrover-trainer",
               DLROVER_LOG_LEVEL="WARNING", PYTHONDONTWRITEBYTECODE="1")
    env.pop("PYTHONPATH", None)
    agent = subprocess.Popen([sys.executable, "-c", AGENT % REF], env=env,
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    try:
        line = agent.stdout.readline()
        assert "AGENT_READY" in line
        tenv = dict(env, DLROVER_B200_WIRE_COMPAT="1")
        out = subprocess.run([sys.executable, "-c", TRAINER % ROOT, str(tmp_path)], env=tenv,
                             capture_output=True, text=True, timeout=180)
        assert "TRAINER_OK" in out.stdout, out.stdout[-1500:] + out.stderr[-3000:]
        assert "TRACKER 13" in out.stdout and "FILES ['rank_0.pt']" in out.stdout
    finally:
        agent.kill()
        agent.wait()
        import glob
        import shutil

        shutil.rmtree(os.path.join("/tmp/ckpt_sock", run_id), ignore_errors=True)
        for f in glob.glob(f"/dev/shm/{run_id}_*"):
            os.unlink(f)


OUR_AGENT = r"""
import sys, time
sys.path.insert(0, %r)
import dlrover_b200                       # wire-compat: reference pickles resolve to our classes
from dlrover_b200.ckpt_saver import AsyncCheckpointSaver
AsyncCheckpointSaver.start_async_saving_ckpt()
print("AGENT_READY", flush=True)
time.sleep(120)
"""

REF_TRAINER = r"""
import os, sys, time
from unittest import mock
sys.path.insert(0, %r)
sys.modules.setdefault("kubernetes", mock.MagicMock())
import torch
from dlrover.trainer.torch.flash_checkpoint.ddp import DdpCheckpointer, StorageType
d = sys.argv[1]
ckpt = DdpCheckpointer(d)
sd = {"w": torch.arange(1000, dtype=torch.float32), "step": 21}
ckpt.save_checkpoint(21, sd, storage_type=StorageType.DISK)
ckpt.wait_latest_checkpoint(timeout=60)
print("TRACKER", open(os.path.join(d, "dlrover_latest.txt")).read())
on_disk = torch.load(os.path.join(d, "21", "rank_0.pt"))
assert torch.equal(on_disk["w"], sd["w"]) and on_disk["step"] == 21
print("TRAINER_OK")
"""


def test_the_reference_trainer_against_our_agent(tmp_path):
    run_id = "wire" + uuid.uuid4().hex[:8]
    env = dict(os.environ, TORCHELASTIC_RUN_ID=run_id, ROLE_NAME="dlrover-trainer",
               DLROVER_LOG_LEVEL="WARNING", PYTHONDONTWRITEBYTECODE="1")
    env.pop("PYTHONPATH", None)
    agent = subprocess.Popen([sys.executable, "-c", OUR_AGENT % ROOT],
                             env=dict(env, DLROVER_B200_WIRE_COMPAT="1"),
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    try:
        assert "AGENT_READY" in agent.stdout.readline()
        out = subprocess.run([sys.executable, "-c", REF_TRAINER % REF, str(tmp_path)], env=env,
                             capture_output=True, text=True, timeout=180)
        assert "TRAINER_OK" in out.stdout, out.stdout[-1500:] + out.stderr[-3000:]
        assert "TRACKER 21" in out.stdout
    finally:
        agent.kill()
        agent.wait()
        import glob
        import shutil

        shutil.rmtree(os.path.join("/tmp/ckpt_sock", run_id), ignore_errors=True)
        for f in glob.glob(f"/dev/shm/{run_id}_*"):
            os.unlink(f)
