"""Runs the reference's own unit tests of the hot path with this package
swapped in underneath (tests/run_reference_tests.py, tests/REFERENCE_TESTS.md).
Only where oracle/_ref/reftests (the reference's byte code, oracle/build_ref.py)
has been built."""

import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "reftests")

FILES = [
    "dlrover/python/tests/test_multi_process.py",
    "dlrover/python/tests/test_storage.py",
    "dlrover/python/tests/test_ckpt_saver.py",
    "dlrover/trainer/tests/torch/checkpoint_egine_test.py",
    "dlrover/trainer/tests/torch/ddp_checkpointer_test.py",
    "dlrover/trainer/tests/torch/megatron_ckpt_test.py",
    "dlrover/trainer/tests/torch/checkpoint_backup_test.py",
]


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, "dlrover", "__init__.pyc")),
                    reason="oracle/_ref/reftests not built (no reference to build it from)")
@pytest.mark.timeout(600)
def test_reference_unit_tests_pass_on_this_implementation():
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    for k in ("TORCHELASTIC_RUN_ID", "ROLE_NAME", "PYTHONPATH", "LOCAL_RANK", "RANK"):
        env.pop(k, None)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "run_reference_tests.py")]
                         + FILES, capture_output=True, text=True, env=env, timeout=580)
    # the reference's tests leave their tiny segments behind ("unittest_ckpt_shm_0", ...)
    import glob

    for leftover in glob.glob("/dev/shm/unittest_ckpt_shm_*") + glob.glob("/dev/shm/ckpt_shm_[0-9]") + \
            glob.glob("/dev/shm/unittest_ckpt_ctl_*") + glob.glob("/dev/shm/ckpt_ctl_[0-9]"):
        try:
            os.unlink(leftover)
        except OSError:
            pass
    tail = out.stdout[-3000:]
    m = re.search(r"(\d+) passed", tail)
    assert m and int(m.group(1)) == 47, tail + out.stderr[-3000:]
    assert " failed" not in tail.splitlines()[-1], tail + out.stderr[-3000:]
