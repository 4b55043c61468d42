"""Restore a sharded DCP checkpoint from storage into live CUDA tensors through FileReader
and through FileDmaReader, on one GPU and in one process, alternating the arms.

    python tools/fsdp_storage_restore_probe.py --dir TMPDIR --out DIR [--reps 10] [--warmup 2]

State: Llama-3-8B weights in bf16 (dlrover_b200/shapes.py, 16.06 GB; the rows are scaled
down when --dir has less free space for two copies, and the record says by how much),
written as the agent writes shard files: raw "__<rank>_0.distcp" + a pickled ".metadata".
Scenarios, each read with torch's own resharding (create_read_items_for_chunk_list):
  same_world:   one rank file holding every tensor whole -> one rank's full tensors;
  reshard_4_1:  4 rank files, every tensor split on dim 0 -> one rank's full tensors;
  reshard_4_2:  the same 4 files -> rank 0's half (dim 0) of a 2-rank layout.
Every arm is checked against the saved state every time.  All reads come from a WARM page
cache (the files were just written or read; dropping the cache is a host setting this
probe does not touch); a cold cache, network storage and more than one GPU are not
measured here.  Writes the record as one line to DIR/h100_fsdp_storage_restore_n1.json."""

import argparse
import json
import os
import pickle
import shutil
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.distributed._shard._utils import narrow_tensor_by_index  # noqa: E402
from torch.distributed.checkpoint.metadata import (  # noqa: E402
    ChunkStorageMetadata,
    Metadata,
    MetadataIndex,
    TensorProperties,
    TensorStorageMetadata,
)
from torch.distributed.checkpoint.planner import LoadPlan  # noqa: E402
from torch.distributed.checkpoint.planner_helpers import (  # noqa: E402
    create_read_items_for_chunk_list,
)

from dlrover_b200.flash_checkpoint.fsdp_engine import (  # noqa: E402
    FileDmaReader,
    FileReader,
    _StorageInfo,
)
from dlrover_b200.shapes import build_state_dict, llama3_8b_shapes, scale_shapes  # noqa: E402
from tools.storage_restore_probe import card, fs_type, summary  # noqa: E402


def dim0_boxes(shape, parts):
    """(offsets, sizes) of `shape` cut into `parts` near-equal pieces on dim 0."""
    n = shape[0]
    edges = [n * k // parts for k in range(parts + 1)]
    return [((a,) + (0,) * (len(shape) - 1), (b - a,) + tuple(shape[1:]))
            for a, b in zip(edges, edges[1:]) if b > a]


def write_checkpoint(root, sd, ranks):
    """Every tensor cut on dim 0 into `ranks` pieces, piece r appended to rank r's file."""
    os.makedirs(root, exist_ok=True)
    md, storage = {}, {}
    fhs = [open(os.path.join(root, f"__{r}_0.distcp"), "wb") for r in range(ranks)]
    pos = [0] * ranks
    try:
        for name, t in sd.items():
            chunks = []
            for r, (off, sizes) in enumerate(dim0_boxes(tuple(t.shape), ranks)):
                piece = t[off[0]:off[0] + sizes[0]].contiguous().cpu()
                raw = piece.reshape(-1).view(torch.uint8).numpy().tobytes()
                storage[MetadataIndex(name, off)] = _StorageInfo(f"__{r}_0.distcp", pos[r],
                                                                 len(raw))
                fhs[r].write(raw)
                pos[r] += len(raw)
                chunks.append(ChunkStorageMetadata(offsets=torch.Size(off),
                                                   sizes=torch.Size(sizes)))
            md[name] = TensorStorageMetadata(properties=TensorProperties(dtype=t.dtype),
                                             size=t.shape, chunks=chunks)
    finally:
        for f in fhs:
            f.close()
    meta = Metadata(state_dict_metadata=md, storage_data=storage)
    with open(os.path.join(root, ".metadata"), "wb") as f:
        pickle.dump(meta, f)
    return meta


class Planner:
    """The LoadPlanner calls a StorageReader makes, over one rank's local tensors."""

    def __init__(self, targets):
        self.targets = targets

    def resolve_tensor(self, item):
        return narrow_tensor_by_index(self.targets[item.dest_index.fqn], item.dest_offsets,
                                      item.lengths)

    def commit_tensor(self, item, tensor):
        pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", required=True, help="where the shard files are written")
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
    if free < full * 2.2:
        scale = max(0.01, free / (full * 2.4))
        shapes = scale_shapes(shapes, scale)
    sd = build_state_dict(shapes, dtype=torch.bfloat16, device="cuda")
    payload = sum(t.numel() * t.element_size() for t in sd.values())
    one_dir, four_dir = os.path.join(args.dir, "world1"), os.path.join(args.dir, "world4")
    t0 = time.perf_counter()
    metas = {"world1": write_checkpoint(one_dir, sd, 1),
             "world4": write_checkpoint(four_dir, sd, 4)}
    write_s = time.perf_counter() - t0
    want = {k: t.clone() for k, t in sd.items()}
    half = {k: t[:dim0_boxes(tuple(t.shape), 2)[0][1][0]] for k, t in sd.items()}

    def items_for(meta, targets, boxes):
        out = []
        for name in targets:
            off, sizes = boxes(name)
            out += create_read_items_for_chunk_list(
                name, meta.state_dict_metadata[name],
                [ChunkStorageMetadata(offsets=torch.Size(off), sizes=torch.Size(sizes))])
        return out

    whole = lambda name: ((0,) * sd[name].dim(), tuple(sd[name].shape))  # noqa: E731
    first_half = lambda name: dim0_boxes(tuple(sd[name].shape), 2)[0]  # noqa: E731
    scenarios = {
        "same_world": (one_dir, metas["world1"], sd, items_for(metas["world1"], sd, whole)),
        "reshard_4_1": (four_dir, metas["world4"], sd, items_for(metas["world4"], sd, whole)),
        "reshard_4_2": (four_dir, metas["world4"], half,
                        items_for(metas["world4"], half, first_half)),
    }

    def run(reader_cls, root, meta, targets, items):
        for t in targets.values():
            t.zero_()
        torch.cuda.synchronize()
        reader = reader_cls(root)
        reader.set_up_storage_reader(meta, True)
        t1 = time.perf_counter()
        reader.read_data(LoadPlan(items), Planner(targets)).wait()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t1) * 1e3
        for k, t in targets.items():
            assert torch.equal(t, want[k][:t.shape[0]]), (reader_cls.__name__, k)
        return ms, getattr(reader, "last_read_stats", {})

    rec = {
        "probe": "tools/fsdp_storage_restore_probe.py", "state": "llama3_8b bf16 weights",
        "shape_scale": round(scale, 4), "payload_bytes": payload, "leaves": len(sd),
        "reps": args.reps, "warmup": args.warmup, "file_system": fs_type(args.dir),
        "page_cache": "warm (cold cache not measured)", "gpus": 1,
        "write_s": round(write_s, 3), "card_before": card_before,
    }
    try:
        for name, (root, meta, targets, items) in scenarios.items():
            times = {"FileReader": [], "FileDmaReader": []}
            stats = []
            for rep in range(args.warmup + args.reps):
                for cls in (FileReader, FileDmaReader):
                    ms, st = run(cls, root, meta, targets, items)
                    if rep >= args.warmup:
                        times[cls.__name__].append(ms)
                        if st:
                            stats.append(st)
            nbytes = sum(t.numel() * t.element_size() for t in targets.values())
            rec[name] = {
                "target_bytes": nbytes, "read_items": len(items),
                "files": stats[0]["files"], "plans": stats[0]["plans"],
                "fallback_items": stats[0]["fallback_items"],
                **{k: {"wall_ms": summary(v),
                       "gb_per_s": round(nbytes / statistics.median(v) / 1e6, 3)}
                   for k, v in times.items()},
            }
            for key in ("read_ms", "scatter_ms"):
                rec[name]["FileDmaReader"][key] = summary([s[key] for s in stats])
            print(name, json.dumps(rec[name]), flush=True)
        rec["card_after"] = card()
    finally:
        shutil.rmtree(one_dir, ignore_errors=True)
        shutil.rmtree(four_dir, ignore_errors=True)
    rec["time"] = time.strftime("%Y-%m-%dT%H:%M:%S")
    line = json.dumps(rec)
    print(line)
    with open(os.path.join(args.out, "h100_fsdp_storage_restore_n1.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
