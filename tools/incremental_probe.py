"""Incremental saves on one GPU: gather-compare kernel, drain and save times, drained
bytes, for several shares of changed state, alternated with plain full saves of the same
state in the same process.

    python tools/incremental_probe.py --out DIR [--reps 10] [--scale 1.0]

State: Llama-3-8B weights in bf16 (dlrover_b200/shapes.py, 16.06 GB), saved through the
C-ABI into pinned host memory.  Dirty cases:
  frozen      nothing changed
  leaves_1pct every 100th leaf rewritten (adapter-like)
  leaves_10pct every 10th leaf rewritten
  items_1byte every work item has a changed byte (worst case for the compare)
  all_rewrite every byte changed
Writes one JSON line per case to DIR/incremental_cases.jsonl and the whole record as one
line to DIR/h100_incremental_n1.json.  The HBM figure of a delta save is 2 x payload
(source + old arena read) + the bytes of the drained items: an upper bound of what the
kernels wrote (they store only the 16-B vectors / TMA tiles that differ)."""

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from dlrover_b200 import _native as native  # noqa: E402
from dlrover_b200.shapes import build_state_dict, llama3_8b_shapes, scale_shapes  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(
            ["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
             "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power, sm, sm_max = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the record says so instead of guessing
        return {"name": torch.cuda.get_device_name(0), "error": f"nvidia-smi: {e}"}


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
    leaves = list(sd.values())
    offsets, total = [], 0
    for t in leaves:
        offsets.append(total)
        total += t.numel() * t.element_size()
    ctx = native.Context(0)
    ctx.arena_reserve(total)
    plan = ctx.plan([t.data_ptr() for t in leaves], offsets,
                    [t.numel() * t.element_size() for t in leaves])
    host = torch.empty(total, dtype=torch.uint8).pin_memory()
    addr = host.data_ptr()
    stream = torch.cuda.current_stream()
    chunk = 256 << 10

    def rewrite(ts):
        for t in ts:
            t.view(torch.int16).add_(1)  # every element's bits change

    def one_byte_per_item():
        for t in leaves:
            u = t.view(-1).view(torch.uint8)
            u[::chunk // 2] += 1
            u[-1] += 1

    cases = {
        "frozen": lambda: None,
        "leaves_1pct": lambda: rewrite(leaves[::100]),
        "leaves_10pct": lambda: rewrite(leaves[::10]),
        "items_1byte": one_byte_per_item,
        "all_rewrite": lambda: rewrite(leaves),
    }

    def timed(save):
        ticket = save()
        ctx.save_wait(ticket)
        pack, drain, tot = ctx.save_timings(ticket)
        return ticket, pack, drain, tot

    samples = {name: [] for name in cases}
    full = []
    for rep in range(args.warmup + args.reps):
        for name, mutate in cases.items():
            # a plain full save of the same state (it forgets the baseline) ...
            _, pack, drain, tot = timed(lambda: plan.save_async(addr, stream))
            if rep >= args.warmup:
                full.append((pack, drain, tot))
            # ... a delta save that finds no baseline re-establishes it (full) ...
            ticket, *_ = timed(lambda: plan.save_delta_async(addr, stream))
            assert ctx.save_delta_stats(ticket) == (False, total)
            # ... and the measured one
            mutate()
            torch.cuda.synchronize()
            ticket, pack, drain, tot = timed(lambda: plan.save_delta_async(addr, stream))
            delta, drained = ctx.save_delta_stats(ticket)
            assert delta
            if rep >= args.warmup:
                samples[name].append((pack, drain, tot, drained))
    card_after = card()

    def med(xs, i):
        return statistics.median(x[i] for x in xs)

    records = []
    for name, xs in samples.items():
        pack = med(xs, 0)
        drained = int(med(xs, 3))
        hbm = 2 * total + drained
        records.append({
            "case": name, "payload_bytes": total, "drained_bytes": drained,
            "gather_compare_ms": round(pack, 3), "drain_ms": round(med(xs, 1), 3),
            "save_total_ms": round(med(xs, 2), 3),
            "gather_compare_ms_range": [round(min(x[0] for x in xs), 3),
                                        round(max(x[0] for x in xs), 3)],
            "hbm_bytes_upper": hbm, "hbm_floor_ms": round(hbm / HBM_BPS * 1e3, 3),
            "hbm_share_of_3p35TBs": round(hbm / HBM_BPS * 1e3 / pack, 3),
            "samples": len(xs)})
    full_rec = {
        "case": "full_save", "payload_bytes": total, "drained_bytes": total,
        "gather_ms": round(med(full, 0), 3), "drain_ms": round(med(full, 1), 3),
        "save_total_ms": round(med(full, 2), 3),
        "hbm_floor_ms": round(2 * total / HBM_BPS * 1e3, 3),
        "hbm_share_of_3p35TBs": round(2 * total / HBM_BPS * 1e3 / med(full, 0), 3),
        "samples": len(full)}
    records.append(full_rec)
    with open(os.path.join(args.out, "incremental_cases.jsonl"), "w") as f:
        for r in records:
            f.write(json.dumps(r) + "\n")
            print(json.dumps(r))
    line = {"probe": "tools/incremental_probe.py", "state": "llama3_8b bf16 weights",
            "scale": args.scale, "chunk_bytes": chunk, "reps": args.reps,
            "card_before": card_before, "card_after": card_after,
            "time": time.strftime("%Y-%m-%dT%H:%M:%S"), "cases": records}
    with open(os.path.join(args.out, "h100_incremental_n1.json"), "w") as f:
        f.write(json.dumps(line) + "\n")
    plan.destroy()
    ctx.destroy()


if __name__ == "__main__":
    main()
