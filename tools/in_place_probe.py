"""Exposed stall of a checkpoint whose state does not fit in HBM twice: Llama-3-8B bf16
weights + AdamW fp32 moments (80.3 GB at PROBE_SCALE=1, 40 GB at the default 0.5, which
leaves an 80 GB H100 room for the synthetic step) on one GPU, with a ballast
tensor standing in for activations so that a snapshot arena cannot be allocated.

Modes (one process each, PROBE_MODE):
  windowed   DLROVER_B200_ARENA_LIMIT_MB=4096: stream through a bounded arena, blocking
  fallback   default engine, arena allocation fails -> in-place drain, blocking
  in_place   engine.in_place=True + guarded "optimizer": the drain overlaps the next
             forward/backward; only optimizer.step() waits for it
  hybrid     in_place + engine.in_place_snapshot_bytes (PROBE_SNAPSHOT_GB, default 32): the
             tail of the state is snapshotted into spare HBM, the head is drained in place
             first; optimizer.step() only waits for the head
Synthetic step: PROBE_STEP_MS of bf16 matmuls (forward/backward: reads the parameters
only), then the "optimizer step" (guard, then an in-place update of one parameter), then a
loss.item()-style host read.  stall = (loop wall time with checkpoints - without) / saves.
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("TORCHELASTIC_RUN_ID", f"ipprobe{os.getppid()}")
os.environ.setdefault("DLROVER_LOG_LEVEL", "WARNING")
mode = os.getenv("PROBE_MODE", "in_place")
if mode == "windowed":
    os.environ["DLROVER_B200_ARENA_LIMIT_MB"] = "4096"
import torch

from dlrover_b200 import shapes
from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType

scale = float(os.getenv("PROBE_SCALE", "0.5"))
step_ms = float(os.getenv("PROBE_STEP_MS", "400"))
every = int(os.getenv("PROBE_EVERY", "4"))
rounds = int(os.getenv("PROBE_ROUNDS", "3"))
dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)

params = shapes.build_state_dict(shapes.scale_shapes(shapes.llama3_8b_shapes(), scale),
                                 torch.bfloat16, dev)
optim = shapes.adamw_state(params)
sd = {"model": params, "optimizer": optim}
S = shapes.payload_bytes(sd)
shm_free = os.statvfs("/dev/shm").f_bavail * os.statvfs("/dev/shm").f_frsize
if shm_free < S * 1.05:
    print(json.dumps({"skipped": f"/dev/shm has {shm_free / 1e9:.0f} GB free, need {S / 1e9:.0f}"}))
    sys.exit(0)
a = torch.randn(8192, 8192, device=dev, dtype=torch.bfloat16)
b = torch.randn(8192, 8192, device=dev, dtype=torch.bfloat16) * 0.01
# ballast: leave less free HBM than the state needs for a second copy
free, total = torch.cuda.mem_get_info()
ballast_bytes = max(0, free - S // 2) if mode != "windowed" else 0
ballast = torch.empty(ballast_bytes, dtype=torch.uint8, device=dev) if ballast_bytes else None
free_after = torch.cuda.mem_get_info()[0]

# calibrate the matmul count for the requested step time
def burn(n):
    c = a
    for _ in range(n):
        c = torch.mm(c, b)
    return c

burn(50)  # warm-up (cuBLAS init, clocks) before calibrating
torch.cuda.synchronize()
t0 = time.perf_counter()
burn(50)
torch.cuda.synchronize()
per_mm = (time.perf_counter() - t0) / 50
inner = max(1, int(step_ms / 1e3 / per_mm))

ckpt = DdpCheckpointer(f"/tmp/fc_ipprobe_{os.getenv('TORCHELASTIC_RUN_ID')}")
engine = ckpt.engine
if mode in ("in_place", "hybrid"):
    engine.in_place = True
if mode == "hybrid":
    # spend part of the free HBM on a snapshot of the tail of the state
    engine.in_place_snapshot_bytes = int(float(os.getenv("PROBE_SNAPSHOT_GB", "32")) * 1e9)
first = next(iter(params.values()))


def train_step():
    c = burn(inner)                 # forward/backward: reads parameters only
    engine.wait_snapshot()          # what guard_optimizer() does in optimizer.step()
    first.add_(1)                   # the optimizer writes the parameters
    return float(c[0, 0].item())    # loss.item()


def loop(save):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n_saved, call_s = 0, 0.0
    for i in range(every * rounds):
        train_step()
        if save and i % every == 0:
            c0 = time.perf_counter()
            ckpt.save_checkpoint(100 + i, sd, storage_type=StorageType.MEMORY)
            call_s += time.perf_counter() - c0
            n_saved += 1
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    ckpt.wait_memory_save()
    return dt, n_saved, call_s


t0 = time.perf_counter()
ckpt.save_checkpoint(1, sd, storage_type=StorageType.MEMORY)   # creates + pins the segment
ckpt.wait_memory_save()
first_save_s = time.perf_counter() - t0
for _ in range(3):
    train_step()
base, _, _ = loop(False)
with_ckpt, n, call_s = loop(True)
handler = engine._shm_handler
timings = engine.last_save_timings()
# verify the last checkpoint against the live state at its save point is not possible
# after the fact (the parameters moved on); check the untouched optimizer moments instead
loaded = ckpt.load_checkpoint()
k = list(params)[5]
idx = list(params).index(k)
ok = bool(torch.equal(loaded["optimizer"]["state"][idx]["exp_avg"],
                      optim["state"][idx]["exp_avg"].cpu()))
del loaded
print(json.dumps({
    "mode": mode, "state_GB": round(S / 1e9, 2), "free_hbm_GB_before_saves": round(free_after / 1e9, 1),
    "in_place_used": bool(handler.last_save_in_place),
    "hybrid_cut_GB": None if handler.last_hybrid_cut is None else round(handler.last_hybrid_cut / 1e9, 2), "train_step_ms": round(base / (every * rounds) * 1e3, 1),
    "saves": n, "stall_ms_per_save": round((with_ckpt - base) / max(n, 1) * 1e3, 1),
    "save_call_ms": round(call_s / max(n, 1) * 1e3, 1),
    "drain_ms": round(timings[1], 1) if timings else None,
    "drain_GBps": round(S / timings[1] / 1e6, 1) if timings and timings[1] else None,
    "first_save_s": round(first_save_s, 1), "spot_check": ok,
}), flush=True)
engine.close()
