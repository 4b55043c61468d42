"""Multi-rank parity: tests/mgpu_worker.py under torch.distributed.run.

  * on CPU (not gpu-marked): world_size 2 over gloo, every case — the host logic of the
    N>1 paths (DCP planning + plan reuse, per-rank segments, cooperative slices, control
    segment handshake, topology stand-ins);
  * on GPUs (gpu-marked): NCCL, one rank per GPU, 2 ranks and — when the machine has
    them — 8 ranks.  A machine with a single GPU skips these (NCCL refuses two ranks on
    one device).

Every rank compares its whole segment byte-for-byte with the oracle image of what it
handed to the engine and restores it (see the worker's docstring)."""

import glob
import json
import os
import shutil
import signal
import subprocess
import sys
import tempfile

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "mgpu_worker.py")
CASES = ["fsdp", "ddp", "coop", "fullshards", "zero3", "megatron"]


def run_case(case, world, backend, device, extra=(), timeout=900):
    out = tempfile.mkdtemp(prefix=f"mg_{case}_")
    port = 29500 + (os.getpid() * 13 + hash((case, world, backend))) % 1500
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
           f"--nproc-per-node={world}", "--master-addr", "127.0.0.1", "--master-port", str(port),
           WORKER, "--case", case, "--out", out, "--backend", backend, "--device", device,
           *extra]
    env = dict(os.environ)
    for k in ("ROLE_NAME", "TORCHELASTIC_RUN_ID", "RANK", "LOCAL_RANK", "WORLD_SIZE"):
        env.pop(k, None)
    try:
        # own session: a case that hangs is taken down with all its ranks (and their saver
        # daemons), not just the launcher — nothing is left holding the GPUs
        p = subprocess.Popen(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                             text=True, start_new_session=True)
        try:
            p.stdout_text, p.stderr_text = p.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            try:
                os.killpg(p.pid, signal.SIGKILL)
            except ProcessLookupError:
                pass
            p.stdout_text, p.stderr_text = p.communicate()
            raise AssertionError(f"{case} x{world} ({backend}): no result after {timeout}s\n"
                                 f"{p.stderr_text[-2000:]}")
        results = [json.load(open(f)) for f in sorted(glob.glob(os.path.join(out, "rank*.json")))]
    finally:
        shutil.rmtree(out, ignore_errors=True)
    errors = [(r["rank"], r.get("error"), r.get("traceback", "")[-1500:]) for r in results
              if not r.get("ok")]
    assert p.returncode == 0 and len(results) == world and not errors, \
        f"{case} x{world} ({backend}): rc={p.returncode} errors={errors}\n{p.stderr_text[-2000:]}"
    return results


@pytest.mark.timeout(600)
@pytest.mark.parametrize("case", CASES)
def test_two_ranks_gloo_cpu(case):
    results = run_case(case, 2, "gloo", "cpu", ("--scale", "0.002", "--flat-mib", "3"))
    if case == "coop":
        (a0, a1), (b0, b1) = results[0]["window"], results[1]["window"]
        assert a0 == 0 and a1 == b0 and a1 % (2 << 20) == 0
        assert all(r["dict_sets"] == 0 for r in results)        # control segment only
        assert results[0]["segment"] == results[1]["segment"]  # one image for the node
    if case == "fsdp":
        assert all(r["reloaded_tensors"] == 873 for r in results)


def _gpus():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.gpu
@pytest.mark.timeout(700)
@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("case", CASES + ["fsdp_full"])
def test_nccl_ranks_on_gpus(case, world):
    if _gpus() < world:
        pytest.skip(f"needs {world} GPUs on one machine, this one has {_gpus()}")
    extra = ("--scale", str(1 / 32), "--flat-mib", "256")
    if case == "zero3":
        extra += ("--in-place", "--snapshot-mib", "300")
    results = run_case(case, world, "nccl", "cuda", extra, timeout=600)
    if case == "fsdp":
        assert all(r["fast_items"] and r["fast_items"] > 0 for r in results)  # DMA + scatter
    if case == "coop":
        assert all(r["dict_sets"] == 0 for r in results)
