"""Cost of refusing non-finite memory saves, on one GPU, in one process.

    python tools/nonfinite_probe.py --out DIR [--reps 10] [--warmup 2]

1. The scan alone (fc_scan_nonfinite_async + fc_scan_wait, CUDA events around it) over
   Llama-3-8B weights in bf16 (dlrover_b200/shapes.py, 16.06 GB), and over a mixed state:
   bf16 weights + fp32 AdamW moments of 0.3 of the model's rows (fits twice in 80 GB).
   Share of the floor = (bytes / 3.35 TB/s) / scan time.
2. A synthetic training loop (bf16 matmuls on the current stream, ~60 ms per step) that
   saves the 16.06 GB state every step through SharedMemoryHandler, switch off and on
   alternated: the save call's host time and the step's exposed stall (step time with the
   save minus the median step time without one).  "On" is what the engine does: the
   scan of the save's plan on the current stream, its result read on the host, then the
   save.  The scan waits for the training work queued before it.
Writes the record as one line to DIR/h100_nonfinite_n1.json."""

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("TORCHELASTIC_RUN_ID", f"nfprobe{os.getpid()}")

import torch  # noqa: E402

from dlrover_b200 import _native as native  # noqa: E402
from dlrover_b200.shapes import build_state_dict, llama3_8b_shapes, scale_shapes  # noqa: E402
from dlrover_b200.shm_handler import (DLROVER_CKPT_CONFIG_KEY, CheckpointConfig,  # noqa: E402
                                      SharedMemoryHandler, _SCAN_KINDS)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(
            ["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
             "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power, sm, sm_max = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the record says so instead of guessing
        return {"name": torch.cuda.get_device_name(0), "error": f"nvidia-smi: {e}"}


def summary(xs):
    return {"median": round(statistics.median(xs), 3), "min": round(min(xs), 3),
            "max": round(max(xs), 3)}


def scan_time(leaves, reps, warmup):
    ctx = native.get_context(0)
    ptrs = [t.data_ptr() for t in leaves]
    lens = [t.numel() * t.element_size() for t in leaves]
    offs, o = [], 0
    for n in lens:
        offs.append(o)
        o += n
    plan = ctx.plan(ptrs, offs, lens)
    plan.set_kinds([_SCAN_KINDS[t.dtype] for t in leaves])
    ms = []
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    try:
        for rep in range(warmup + reps):
            torch.cuda.synchronize()
            ev[0].record()
            plan.scan_nonfinite_async(torch.cuda.current_stream())
            ev[1].record()
            total, _ = plan.scan_wait(len(leaves))
            assert total == 0
            if rep >= warmup:
                ms.append(ev[0].elapsed_time(ev[1]))
    finally:
        plan.destroy()
    floor = o / HBM_BYTES_PER_S * 1e3
    med = statistics.median(ms)
    return {"bytes": o, "ranges": len(leaves), "scan_ms": summary(ms),
            "floor_ms": round(floor, 3), "share_of_floor": round(floor / med, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    assert torch.cuda.is_available(), "the probe measures on a GPU"
    torch.cuda.set_device(0)
    rec = {"probe": "nonfinite", "card": card()}

    # 1a. Llama-3-8B bf16
    sd = build_state_dict(llama3_8b_shapes(), dtype=torch.bfloat16, device="cuda")
    rec["scan_llama3_8b_bf16"] = scan_time(list(sd.values()), args.reps, args.warmup)

    # 2. save loop, switch off / on alternated (the 16.06 GB state of 1a)
    a = torch.randn(8192, 8192, device="cuda", dtype=torch.bfloat16)
    handler = SharedMemoryHandler(0, host=True)
    step = 0

    def train():
        for _ in range(8):
            torch.matmul(a, a)

    def save(on):
        nonlocal step
        step += 1
        tree = {"model_states": sd, DLROVER_CKPT_CONFIG_KEY: CheckpointConfig(step=step, paths={})}
        t0 = time.perf_counter()
        if on:
            assert not handler.scan_nonfinite(tree, reuse_for=tree)
        handler.save_state_dict(tree, blocking=False)
        return (time.perf_counter() - t0) * 1e3

    try:
        save(False)
        handler.wait_pending()
        assert handler.wait_segment_pinned(600), "the segment was not pinned"
        plain, call = [], {False: [], True: []}
        steps = {False: [], True: []}
        for rep in range(args.warmup + args.reps):
            for on in (False, True):
                handler.wait_pending()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                train()
                torch.cuda.synchronize()
                p = (time.perf_counter() - t0) * 1e3
                t0 = time.perf_counter()
                train()
                c = save(on)
                torch.cuda.synchronize()
                s = (time.perf_counter() - t0) * 1e3
                if rep >= args.warmup:
                    plain.append(p)
                    call[on].append(c)
                    steps[on].append(s)
        handler.wait_pending()
        base = statistics.median(plain)
        rec["save_loop"] = {
            "state_bytes": rec["scan_llama3_8b_bf16"]["bytes"],
            "step_without_save_ms": summary(plain),
            "off": {"save_call_ms": summary(call[False]),
                    "exposed_stall_ms": summary([s - base for s in steps[False]])},
            "on": {"save_call_ms": summary(call[True]),
                   "exposed_stall_ms": summary([s - base for s in steps[True]])},
        }
    finally:
        handler.close()
        handler.unlink()
    del sd, a
    torch.cuda.empty_cache()

    # 1b. mixed: bf16 weights + fp32 exp_avg / exp_avg_sq of 0.3 of the rows
    shapes = scale_shapes(llama3_8b_shapes(), 0.3)
    w = build_state_dict(shapes, dtype=torch.bfloat16, device="cuda")
    m1 = build_state_dict(shapes, dtype=torch.float32, device="cuda")
    m2 = build_state_dict(shapes, dtype=torch.float32, device="cuda")
    leaves = []
    for k in w:
        leaves += [w[k], m1[k], m2[k]]
    rec["scan_mixed_bf16_fp32_adamw"] = scan_time(leaves, args.reps, args.warmup)
    rec["card_after"] = card()
    line = json.dumps(rec)
    print(line)
    with open(os.path.join(args.out, "h100_nonfinite_n1.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
