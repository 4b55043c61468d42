"""ORACLE recipe (test infrastructure, not product code): the REFERENCE ITSELF for the
memory-save path, compiled from where its sources lie under /root/reference into
oracle/_ref/pyref/ — byte code only (sourceless .pyc), git-ignored, not gpurun-ignored, so it
travels to the GPU box like oracle/_ref/libpack_oracle.so.  No reference source is copied.

    python oracle/build_ref.py            (also: make -C oracle pyref; __graft_entry__.build())

What gets compiled is found, not listed: a clean interpreter imports
dlrover/python/elastic_agent/torch/ckpt_saver.py from /root/reference, runs one tiny
SharedMemoryHandler.save_state_dict + load_state_dict (ckpt_saver.py:303-366) so that lazily
imported modules are loaded too, imports the trainer-side DdpCheckpointer, and reports every
module it loaded from the checkout.  Each is compiled with py_compile to the mirrored
path under pyref/ (`x/y.py` -> `x/y.pyc`, `__init__.py` -> `__init__.pyc`), which Python
imports without the source.  MANIFEST.json records the files and the sha256 of the source each came from.

Used by oracle/ref_real.py (bench.py's `--impl reference` arm and `cpu_baseline`:
kind "reference"), by tests/test_oracle.py to pin ref_port.py / shm_layout.py to it and by
tests/test_wire_compat.py (the reference's agent and trainer against ours).
"""

from __future__ import annotations

import hashlib
import json
import os
import py_compile
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE = os.environ.get("FC_REFERENCE_ROOT", "/root/reference")
OUT = os.path.join(HERE, "_ref", "pyref")
# the whole reference package, its own unit tests included (tests/run_reference_tests.py)
OUT_TESTS = os.path.join(HERE, "_ref", "reftests")

PROBE = r"""
import json, os, sys
sys.path.insert(0, sys.argv[1])
os.environ.setdefault("ROLE_NAME", "dlrover-trainer")
os.environ["TORCHELASTIC_RUN_ID"] = "fcbuildref%d" % os.getpid()
import logging
logging.disable(logging.CRITICAL)
import torch
from dlrover.python.elastic_agent.torch import ckpt_saver as ref
h = ref.SharedMemoryHandler(97, host=True)
sd = {"m": {"w": torch.arange(6, dtype=torch.float32).reshape(2, 3), "n": 3},
      ref.DLROVER_CKPT_CONFIG_KEY: ref.CheckpointConfig(step=1, paths={})}
h.save_state_dict(sd)
back = h.load_state_dict()
assert torch.equal(back["m"]["w"], sd["m"]["w"]) and back["m"]["n"] == 3
del back
h.unlink()
h.close()
# the trainer half of the wire (tests/test_wire_compat.py runs it against our agent)
from unittest import mock
sys.modules.setdefault("kubernetes", mock.MagicMock())
from dlrover.trainer.torch.flash_checkpoint.ddp import DdpCheckpointer
root = os.path.realpath(sys.argv[1]) + os.sep
mods = sorted({os.path.realpath(m.__file__) for m in list(sys.modules.values())
               if getattr(m, "__file__", None)
               and os.path.realpath(m.__file__).startswith(root)
               and m.__file__.endswith(".py")})
print("FCREF " + json.dumps(mods))
os._exit(0)
"""


def build(verbose: bool = True) -> int:
    """Returns the number of modules compiled (0: no reference here, nothing done)."""
    if not os.path.isdir(os.path.join(REFERENCE, "dlrover")):
        if verbose:
            print(f"oracle/build_ref.py: no reference at {REFERENCE}; keeping what is in {OUT}")
        return 0
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    env.pop("PYTHONPATH", None)
    p = subprocess.run([sys.executable, "-c", PROBE, REFERENCE], env=env, cwd="/tmp",
                       capture_output=True, text=True, timeout=600)
    marker = [ln for ln in p.stdout.splitlines() if ln.startswith("FCREF ")]
    if p.returncode != 0 or not marker:
        raise RuntimeError(f"reference probe failed ({p.returncode}):\n{p.stderr[-2000:]}")
    files = json.loads(marker[-1][len("FCREF "):])
    root = os.path.realpath(REFERENCE) + os.sep
    tmp = OUT + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    manifest = {"python": sys.version.split()[0], "files": {}}
    for src in files:
        rel = src[len(root):]
        dst = os.path.join(tmp, rel + "c")          # x.py -> x.pyc, next to where x.py would be
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        py_compile.compile(src, cfile=dst, dfile=os.path.join("<reference>", rel), doraise=True,
                           invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
        with open(src, "rb") as f:
            manifest["files"][rel] = hashlib.sha256(f.read()).hexdigest()
    head = os.path.join(REFERENCE, ".git", "HEAD")
    if os.path.exists(head):
        try:
            ref = open(head).read().strip()
            if ref.startswith("ref: "):
                ref = open(os.path.join(REFERENCE, ".git", ref[5:])).read().strip()
            manifest["commit"] = ref
        except OSError:
            pass
    with open(os.path.join(tmp, "MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1, sort_keys=True)
    shutil.rmtree(OUT, ignore_errors=True)
    os.replace(tmp, OUT)
    if verbose:
        print(f"oracle/build_ref.py: {len(files)} reference modules -> {OUT}")
    return len(files)


def build_tests(verbose: bool = True) -> int:
    """Byte-compiles every module of the reference's `dlrover` package — its unit tests and
    their helpers included — into OUT_TESTS, so that tests/run_reference_tests.py can run the
    reference's own tests of this path without the checkout.  Returns the number of modules
    (0: no reference here, nothing done)."""
    pkg = os.path.join(REFERENCE, "dlrover")
    if not os.path.isdir(pkg):
        if verbose:
            print(f"oracle/build_ref.py: no reference at {REFERENCE}; keeping what is in {OUT_TESTS}")
        return 0
    root = os.path.realpath(REFERENCE) + os.sep
    tmp = OUT_TESTS + ".tmp"
    shutil.rmtree(tmp, ignore_errors=True)
    n = 0
    for dirpath, _, files in os.walk(pkg):
        for f in sorted(files):
            if not f.endswith(".py"):
                continue
            src = os.path.realpath(os.path.join(dirpath, f))
            rel = src[len(root):]
            dst = os.path.join(tmp, rel + "c")
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            py_compile.compile(src, cfile=dst, dfile=os.path.join("<reference>", rel), doraise=True,
                               invalidation_mode=py_compile.PycInvalidationMode.UNCHECKED_HASH)
            n += 1
    shutil.rmtree(OUT_TESTS, ignore_errors=True)
    os.replace(tmp, OUT_TESTS)
    if verbose:
        print(f"oracle/build_ref.py: {n} reference modules -> {OUT_TESTS}")
    return n


if __name__ == "__main__":
    build()
    build_tests()
