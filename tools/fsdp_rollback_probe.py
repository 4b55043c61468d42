"""Roll a sharded (DCP) checkpoint back from the HBM arena image against the restore over
PCIe of the same in-memory checkpoint, on one GPU (world size 1), in one process.

    python tools/fsdp_rollback_probe.py --out DIR [--reps 10] [--warmup 2] [--scale 1.0]

State: Llama-3-8B weights in bf16 (dlrover_b200/shapes.py, 16.06 GB, 291 tensors) as an
FSDP job of world size 1 hands them over: DTensors sharded on dim 0 over a one-rank mesh
(shapes.ShardedStateFactory), saved by FsdpCheckpointEngine.save_to_memory through torch
DCP into the shared-memory segment (pinned before the timed loop).  Each repetition saves,
changes every tensor, rolls back with dcp.load over engine.rollback_reader() (scatter from
the arena, no DMA), changes every tensor again and restores with dcp.load over
engine.load() (DMA from the segment; it rewrites or bypasses the arena, so the next
repetition's save sets the image again).  Each call is timed with a host clock around a synchronise, from asking the engine for the
reader to the end of dcp.load; the readers' own figures (read_data wall time, fill,
scatter) are reported beside it, and the difference is DCP's planning around read_data.
The restored tensors are compared with the saved state every time.  Then one incremental
save after a rollback, with nothing changed since.  Writes the record as one line to
DIR/h100_fsdp_rollback_n1.json."""

import argparse
import glob
import json
import os
import shutil
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
RUN_ID = f"fsdprbprobe{os.getpid()}"
os.environ.update({"TORCHELASTIC_RUN_ID": RUN_ID, "RANK": "0", "LOCAL_RANK": "0",
                   "WORLD_SIZE": "1", "LOCAL_WORLD_SIZE": "1", "MASTER_ADDR": "127.0.0.1",
                   "MASTER_PORT": str(29000 + os.getpid() % 1000)})
os.environ.setdefault("DLROVER_LOG_LEVEL", "WARNING")

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.distributed.checkpoint as dist_cp  # noqa: E402
from torch.distributed.device_mesh import init_device_mesh  # noqa: E402

from dlrover_b200.common.storage import PosixDiskStorage  # noqa: E402
from dlrover_b200.flash_checkpoint.fsdp_engine import FsdpCheckpointEngine  # noqa: E402
from dlrover_b200.shapes import ShardedStateFactory, llama3_8b_shapes, scale_shapes  # noqa: E402
from tools.rollback_probe import card, summary  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0, help="fraction of the Llama-3-8B rows")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    assert torch.cuda.is_available(), "the probe measures on a GPU"
    dist.init_process_group("nccl", rank=0, world_size=1)
    ckpt_dir = f"/tmp/fc_{RUN_ID}"
    # the engine forks the saver daemon: before this process touches CUDA
    engine = FsdpCheckpointEngine(ckpt_dir, PosixDiskStorage())
    handler = engine._shm_handler
    torch.cuda.set_device(0)
    card_before = card()

    shapes = llama3_8b_shapes()
    if args.scale != 1.0:
        shapes = scale_shapes(shapes, args.scale)
    mesh = init_device_mesh("cuda", (1,))
    factory = ShardedStateFactory(shapes, 1, 0, torch.device("cuda", 0), mesh,
                                  with_optimizer=False)
    sd = factory.build(0)
    local = factory.local_tensors(sd)
    payload = factory.local_bytes
    saved = {k: t.clone() for k, t in local.items()}
    step = 0

    def save():
        nonlocal step
        step += 1
        assert engine.save_to_memory(step, sd, {"model_states": os.path.join(ckpt_dir, str(step))})
        assert engine.wait_memory_save(600)

    def scribble():
        for t in local.values():
            t.view(torch.int16).add_(1)  # every element's bits change
        torch.cuda.synchronize()

    def check(what):
        for k, t in local.items():
            assert torch.equal(t, saved[k]), (what, k)

    def timed_load(get_reader):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        reader = get_reader()
        dist_cp.load(sd, storage_reader=reader)
        torch.cuda.synchronize()
        return reader, (time.perf_counter() - t0) * 1e3

    try:
        save()
        print("first save done", flush=True)
        assert handler.wait_segment_pinned(600), "the segment was not pinned"
        roll, rest = [], []
        for rep in range(args.warmup + args.reps):
            save()
            scribble()
            reader, ms = timed_load(engine.rollback_reader)
            st = dict(reader.last_read_stats)
            assert st["from_image"] == 1.0 and st["slow_items"] == 0, st
            check("rollback")
            if rep >= args.warmup:
                roll.append((ms, st))
            scribble()
            reader, ms = timed_load(engine.load)
            st = dict(handler.last_restore_stats)
            assert reader.last_fast_items == len(local), reader.last_fast_items
            check("load")
            if rep >= args.warmup:
                rest.append((ms, st))
            print(f"rep {rep}: rollback {roll[-1][0] if roll else 0:.1f} ms, "
                  f"load {ms:.1f} ms", flush=True)

        # an incremental save right after a rollback, nothing changed since
        engine.incremental = True
        save()  # full: sets the baseline and the image
        scribble()
        reader, _ = timed_load(engine.rollback_reader)
        assert reader.last_read_stats["from_image"] == 1.0
        check("rollback before the incremental save")
        t0 = time.perf_counter()
        save()
        save_ms = (time.perf_counter() - t0) * 1e3
        pack_ms, drain_ms, total_ms = handler.last_timings
        delta = dict(engine.last_save_stats())
        card_after = card()
    finally:
        handler.unlink()
        engine.close()
        dist.destroy_process_group()
        for f in glob.glob(f"/dev/shm/{RUN_ID}_*"):
            os.unlink(f)
        shutil.rmtree(ckpt_dir, ignore_errors=True)

    def part(rows, key):
        return summary([st[key] for _, st in rows])

    rec = {
        "probe": "tools/fsdp_rollback_probe.py", "state": "llama3_8b bf16 weights through DCP",
        "scale": args.scale, "payload_bytes": payload, "tensors": len(local), "gpus": 1,
        "reps": args.reps, "warmup": args.warmup, "card_before": card_before,
        "card_after": card_after,
        "rollback": {"call_ms": summary([ms for ms, _ in roll]),
                     "read_data_ms": part(roll, "wall_ms"), "fill_ms": part(roll, "fill_ms"),
                     "scatter_ms": part(roll, "scatter_ms"), "pcie_bytes": 0},
        "load": {"call_ms": summary([ms for ms, _ in rest]),
                 "read_ranges_ms": part(rest, "wall_ms"), "fill_ms": part(rest, "fill_ms"),
                 "scatter_ms": part(rest, "scatter_ms"), "direct": rest[0][1]["direct"],
                 "pcie_bytes": payload},
        "incremental_save_after_rollback": {
            "delta": delta["delta"], "drained_bytes": delta["drained_bytes"],
            "call_ms": round(save_ms, 3), "compare_ms": round(pack_ms, 3),
            "drain_ms": round(drain_ms, 3), "total_ms": round(total_ms, 3)},
        "time": time.strftime("%Y-%m-%dT%H:%M:%S"),
    }
    line = json.dumps(rec)
    print(line)
    with open(os.path.join(args.out, "h100_fsdp_rollback_n1.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
