"""Restore a persisted checkpoint file into live CUDA tensors, three ways, on one GPU and in
one process, alternating the arms.

    python tools/storage_restore_probe.py --dir TMPDIR --out DIR [--reps 10] [--warmup 2]

State: Llama-3-8B weights in bf16 (dlrover_b200/shapes.py, 16.06 GB), written once with
fast_torch_save into --dir (the rows are scaled down when --dir has less free space; the
record says by how much).  Arms, each into the same live CUDA tensors:
  (a) torch.load(path, map_location="cpu") + one copy_ per leaf (today's path);
  (b) torch.load(path, mmap=True) + one copy_ per leaf;
  (c) shm_handler.restore_file_into: index, pread through pinned bounce slots, scatter.
Every arm is checked against the saved state every time.  All reads come from a WARM page
cache: the file was just written or read, and dropping the cache is a host setting this
probe does not touch; a cold cache or network storage is not measured here.
Writes the record as one line to DIR/h100_storage_restore_n1.json."""

import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from dlrover_b200 import fast_torch_save  # noqa: E402
from dlrover_b200.shapes import build_state_dict, llama3_8b_shapes, scale_shapes  # noqa: E402
from dlrover_b200.shm_handler import restore_file_into  # noqa: E402


def card():
    try:
        out = subprocess.run(
            ["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
             "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power, sm, sm_max = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the record says so instead of guessing
        return {"name": torch.cuda.get_device_name(0), "error": f"nvidia-smi: {e}"}


def fs_type(path):
    """File system type of the mount that holds `path` (longest mount point prefix)."""
    best, kind = "", "unknown"
    try:
        real = os.path.realpath(path)
        with open("/proc/mounts") as f:
            for line in f:
                parts = line.split()
                if len(parts) >= 3 and (real == parts[1] or real.startswith(parts[1].rstrip("/") + "/")) \
                        and len(parts[1]) > len(best):
                    best, kind = parts[1], parts[2]
    except OSError:
        pass
    return {"mount": best, "type": kind}


def summary(xs):
    return {"median": round(statistics.median(xs), 3), "min": round(min(xs), 3),
            "max": round(max(xs), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", required=True, help="where the checkpoint file is written")
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    os.makedirs(args.dir, exist_ok=True)
    assert torch.cuda.is_available(), "the probe measures on a GPU"
    torch.cuda.set_device(0)
    card_before = card()

    shapes = llama3_8b_shapes()
    full = sum(torch.Size(s).numel() * 2 for _, s in shapes)
    free = shutil.disk_usage(args.dir).free
    scale = 1.0
    if free < full * 1.1:
        scale = max(0.01, free / (full * 1.2))
        shapes = scale_shapes(shapes, scale)
    sd = build_state_dict(shapes, dtype=torch.bfloat16, device="cuda")
    payload = sum(t.numel() * t.element_size() for t in sd.values())
    saved = {k: t.cpu() for k, t in sd.items()}
    path = os.path.join(args.dir, "rank_0.pt")
    t0 = time.perf_counter()
    fast_torch_save.fast_save(saved, path, threads=4)
    write_s = time.perf_counter() - t0
    file_bytes = os.path.getsize(path)
    del saved
    want = {k: t.clone() for k, t in sd.items()}

    def scribble():
        for t in sd.values():
            t.zero_()
        torch.cuda.synchronize()

    def check(what):
        for k, t in sd.items():
            assert torch.equal(t, want[k]), (what, k)

    def arm_load():
        loaded = torch.load(path, map_location="cpu")
        t1 = time.perf_counter()
        for k, t in sd.items():
            t.copy_(loaded[k])
        torch.cuda.synchronize()
        return {"copy_ms": (time.perf_counter() - t1) * 1e3}

    def arm_mmap():
        loaded = torch.load(path, map_location="cpu", mmap=True)
        t1 = time.perf_counter()
        for k, t in sd.items():
            t.copy_(loaded[k])
        torch.cuda.synchronize()
        return {"copy_ms": (time.perf_counter() - t1) * 1e3}

    def arm_file():
        stats = restore_file_into(path, sd)
        torch.cuda.synchronize()
        return stats

    arms = {"torch_load_copy": arm_load, "torch_load_mmap_copy": arm_mmap,
            "restore_file_into": arm_file}
    times = {k: [] for k in arms}
    details = {k: [] for k in arms}
    try:
        for rep in range(args.warmup + args.reps):
            for name, fn in arms.items():
                scribble()
                t1 = time.perf_counter()
                extra = fn()
                ms = (time.perf_counter() - t1) * 1e3
                check(name)
                if rep >= args.warmup:
                    times[name].append(ms)
                    details[name].append(extra)
        card_after = card()
    finally:
        os.remove(path)

    def rec_arm(name, keys):
        out = {"wall_ms": summary(times[name]),
               "gb_per_s": round(payload / statistics.median(times[name]) / 1e6, 3)}
        for k in keys:
            out[k] = summary([d[k] for d in details[name]])
        return out

    rec = {
        "probe": "tools/storage_restore_probe.py", "state": "llama3_8b bf16 weights",
        "shape_scale": round(scale, 4), "payload_bytes": payload, "file_bytes": file_bytes,
        "leaves": len(sd), "reps": args.reps, "warmup": args.warmup,
        "file_system": fs_type(args.dir), "page_cache": "warm (cold cache not measured)",
        "write_s": round(write_s, 3), "card_before": card_before, "card_after": card_after,
        "torch_load_copy": rec_arm("torch_load_copy", ["copy_ms"]),
        "torch_load_mmap_copy": rec_arm("torch_load_mmap_copy", ["copy_ms"]),
        "restore_file_into": rec_arm("restore_file_into", ["read_ms", "scatter_ms"]),
        "time": time.strftime("%Y-%m-%dT%H:%M:%S"),
    }
    line = json.dumps(rec)
    print(line)
    with open(os.path.join(args.out, "h100_storage_restore_n1.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
