"""Rollback from the HBM arena image against a restore over PCIe, on one GPU, in the same
process and of the same in-memory checkpoint.

    python tools/rollback_probe.py --out DIR [--reps 10] [--warmup 2] [--scale 1.0]

State: Llama-3-8B weights in bf16 (dlrover_b200/shapes.py, 16.06 GB), saved by
SharedMemoryHandler.save_state_dict into a POSIX shared-memory segment (pinned before
the timed loop).  Each repetition saves, changes every tensor, rolls back with
rollback_into (one scatter kernel from the arena, no DMA), changes every tensor again and
restores with restore_into (DMA from the segment; it rewrites or bypasses the arena, so
the next repetition's save sets the image again).  Both are timed with CUDA events and
with a host clock around a synchronise; the restored tensors are compared with the saved
state every time.  Then one incremental save after a rollback, with nothing changed since.
Writes the record as one line to DIR/h100_rollback_n1.json."""

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("TORCHELASTIC_RUN_ID", f"rbprobe{os.getpid()}")

import torch  # noqa: E402

from dlrover_b200.shapes import build_state_dict, llama3_8b_shapes, scale_shapes  # noqa: E402
from dlrover_b200.shm_handler import (DLROVER_CKPT_CONFIG_KEY, CheckpointConfig,  # noqa: E402
                                      SharedMemoryHandler)


def card():
    try:
        out = subprocess.run(
            ["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
             "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power, sm, sm_max = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the record says so instead of guessing
        return {"name": torch.cuda.get_device_name(0), "error": f"nvidia-smi: {e}"}


def timed(fn):
    """(result, device ms, host ms) of fn() on the current stream."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ev[0].record()
    out = fn()
    ev[1].record()
    torch.cuda.synchronize()
    return out, ev[0].elapsed_time(ev[1]), (time.perf_counter() - t0) * 1e3


def summary(xs):
    return {"median": round(statistics.median(xs), 3), "min": round(min(xs), 3),
            "max": round(max(xs), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the Llama-3-8B rows")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    assert torch.cuda.is_available(), "the probe measures on a GPU"
    torch.cuda.set_device(0)
    card_before = card()

    shapes = llama3_8b_shapes()
    if args.scale != 1.0:
        shapes = scale_shapes(shapes, args.scale)
    sd = build_state_dict(shapes, dtype=torch.bfloat16, device="cuda")
    payload = sum(t.numel() * t.element_size() for t in sd.values())
    saved = {k: t.clone() for k, t in sd.items()}
    tree = {"model_states": sd}
    handler = SharedMemoryHandler(0, host=True)
    step = 0

    def save():
        nonlocal step
        step += 1
        handler.save_state_dict({"model_states": sd,
                                 DLROVER_CKPT_CONFIG_KEY: CheckpointConfig(step=step, paths={})},
                                blocking=True)

    def scribble():
        for t in sd.values():
            t.view(torch.int16).add_(1)  # every element's bits change
        torch.cuda.synchronize()

    def check(what):
        for k, t in sd.items():
            assert torch.equal(t, saved[k]), (what, k)

    try:
        save()
        assert handler.wait_segment_pinned(600), "the segment was not pinned"
        roll, rest = [], []
        for rep in range(args.warmup + args.reps):
            save()
            scribble()
            stats, dev, host = timed(lambda: handler.rollback_into(tree))
            assert stats["from_image"] == 1.0, stats
            check("rollback")
            if rep >= args.warmup:
                roll.append((dev, host, stats["scatter_ms"]))
            scribble()
            stats, dev, host = timed(lambda: handler.restore_into(tree))
            check("restore")
            if rep >= args.warmup:
                rest.append((dev, host, stats["fill_ms"], stats["scatter_ms"], stats["direct"]))

        # an incremental save right after a rollback, nothing changed since
        handler.incremental = True
        save()  # full: sets the baseline and the image
        scribble()
        stats, dev, host = timed(lambda: handler.rollback_into(tree))
        assert stats["from_image"] == 1.0
        check("rollback before the incremental save")
        _, _, save_host = timed(save)
        pack_ms, drain_ms, total_ms = handler.last_timings
        delta = dict(handler.last_save_stats)
        card_after = card()
    finally:
        handler.unlink()
        handler.close()

    rec = {
        "probe": "tools/rollback_probe.py", "state": "llama3_8b bf16 weights",
        "scale": args.scale, "payload_bytes": payload, "leaves": len(sd), "reps": args.reps,
        "warmup": args.warmup, "card_before": card_before, "card_after": card_after,
        "rollback": {"event_ms": summary([x[0] for x in roll]),
                     "host_ms": summary([x[1] for x in roll]),
                     "scatter_ms": summary([x[2] for x in roll]), "pcie_bytes": 0},
        "pcie_restore": {"event_ms": summary([x[0] for x in rest]),
                         "host_ms": summary([x[1] for x in rest]),
                         "fill_ms": summary([x[2] for x in rest]),
                         "scatter_ms": summary([x[3] for x in rest]),
                         "direct": rest[0][4], "pcie_bytes": payload},
        "incremental_save_after_rollback": {
            "delta": delta["delta"], "drained_bytes": delta["drained_bytes"],
            "host_ms": round(save_host, 3), "compare_ms": round(pack_ms, 3),
            "drain_ms": round(drain_ms, 3), "total_ms": round(total_ms, 3)},
        "time": time.strftime("%Y-%m-%dT%H:%M:%S"),
    }
    line = json.dumps(rec)
    print(line)
    with open(os.path.join(args.out, "h100_rollback_n1.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
