"""One rank of the multi-rank parity cases (launched by tests/test_multi_gpu.py under
torch.distributed.run).  NCCL + CUDA on GPUs; the same cases run with `--backend gloo
--device cpu`, so the host logic is covered without a GPU.

Every case ends with EVERY rank comparing its whole segment byte-for-byte with the oracle
image (oracle/shm_layout.py) of what that rank handed to the engine, and restoring it.

  fsdp      BASELINE configs[2]: Llama-shaped state row-sharded 1/N per rank as DTensors
            (+ fp32 AdamW moments) through FsdpCheckpointEngine / torch DCP, fresh tensors
            at every save; DCP-load back into zeroed shards
  ddp       every rank its own full shard (DdpCheckpointer local_shard_num = world)
  coop      replicated state saved cooperatively: each rank drains 1/N of the ONE image
  zero3     BASELINE configs[3] shape: 3 flat fp32 partitions per rank through
            DeepSpeedCheckpointEngine (in-place / hybrid with --in-place)
  megatron  BASELINE configs[4] shape: TP2xPP2 model shard + distributed-optimizer shard
            per rank through MegatronDistCheckpointEngine
"""
import argparse
import json
import os
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--backend", default="nccl")
    ap.add_argument("--device", default="cuda")
    ap.add_argument("--scale", type=float, default=1 / 64, help="fraction of Llama-3-8B rows")
    ap.add_argument("--flat-mib", type=float, default=64.0, help="zero3: MiB per flat partition")
    ap.add_argument("--layers", type=int, default=2, help="megatron: layers per pipeline stage")
    ap.add_argument("--widths", type=float, default=0.0,
                    help="megatron: fraction of the Mixtral widths (default: 8 x --scale)")
    ap.add_argument("--in-place", action="store_true")
    ap.add_argument("--snapshot-mib", type=int, default=0)
    ap.add_argument("--full-compare", type=int, default=1,
                    help="1: whole segment byte-for-byte; 0: 64 KiB head+tail of every tensor "
                         "+ a checksum of checksums (states of tens of GB per rank)")
    return ap.parse_args()


def seg_bytes(handler):
    return np.frombuffer(handler.shared_memory.buf, dtype=np.uint8)


def checksum_np(a):
    return int(np.add.reduce(a.view(np.uint64) if a.size % 8 == 0 else a.astype(np.uint64),
                             dtype=np.uint64))


def checksum_dev(t):
    flat = t.reshape(-1).view(torch.uint8)
    if flat.numel() % 8 == 0:
        v = flat.view(torch.int64)
        return int(v.sum().item()) & 0xFFFFFFFFFFFFFFFF
    return int(flat.to(torch.int64).sum().item())


def compare_with_oracle(handler, state, full):
    """Segment vs oracle image of `state` (the tree handed to the engine, config -> None)."""
    from oracle import shm_layout as oracle

    got = seg_bytes(handler)
    meta, total = oracle.plan_layout(state)
    assert got.size == total, (got.size, total)
    if full:
        _, want = oracle.serialize(state)
        assert np.array_equal(got, want), "segment != oracle image"
        return {"bytes": int(total), "mode": "byte-for-byte"}
    # large states: offsets from the oracle's plan, bytes from the device
    leaves = []

    def walk(v, m):
        if isinstance(v, dict):
            for k in v:
                walk(v[k], m[k])
        elif isinstance(v, list):
            for i, x in enumerate(v):
                walk(x, m[i])
        elif torch.is_tensor(v) and v.numel():
            leaves.append((v, m.offset))

    walk(state, meta)
    dev_sum = host_sum = 0
    for t, off in leaves:
        n = t.numel() * t.element_size()
        flat = t.reshape(-1).view(torch.uint8)
        k = min(n, 1 << 16)
        assert np.array_equal(got[off:off + k], flat[:k].cpu().numpy()), f"head of leaf at {off}"
        assert np.array_equal(got[off + n - k:off + n], flat[-k:].cpu().numpy()), f"tail at {off}"
        if n % 8 == 0 and off % 8 == 0:
            dev_sum = (dev_sum * 31 + checksum_dev(t)) & 0xFFFFFFFFFFFF
            host_sum = (host_sum * 31 + checksum_np(got[off:off + n])) & 0xFFFFFFFFFFFF
    assert dev_sum == host_sum, "checksum of checksums differs"
    return {"bytes": int(total), "mode": "head/tail bytes + checksum of checksums",
            "leaves": len(leaves)}


# ------------------------------------------------------------------------------- cases --


def case_fsdp(args, rank, world, dev, ckpt_dir):
    import torch.distributed.checkpoint as dist_cp
    from torch.distributed.checkpoint.default_planner import DefaultSavePlanner
    from torch.distributed.checkpoint.planner import WriteItemType
    from torch.distributed.device_mesh import init_device_mesh

    from dlrover_b200 import shapes
    from dlrover_b200.common.storage import PosixDiskStorage
    from dlrover_b200.flash_checkpoint.fsdp_engine import FsdpCheckpointEngine
    from oracle import shm_layout as oracle

    mesh = init_device_mesh(dev.type, (world,))
    shp = shapes.scale_shapes(shapes.llama3_8b_shapes(), args.scale)
    factory = shapes.ShardedStateFactory(shp, world, rank, dev, mesh)
    engine = FsdpCheckpointEngine(ckpt_dir, PosixDiskStorage())
    handler = engine._shm_handler
    out = {"payload_bytes": factory.local_bytes, "saves": []}
    sd = None
    for step, variant in ((1, 0), (2, 1), (3, 0)):
        sd = factory.build(variant)
        t0 = time.perf_counter()
        assert engine.save_to_memory(step, sd, {"model_states": os.path.join(ckpt_dir, str(step))})
        call_ms = (time.perf_counter() - t0) * 1e3
        assert engine.wait_memory_save(300)
        dist.barrier()
        # oracle image of MY segment: the items of my final DCP plan, back to back
        items = engine._shm_writer.last_items
        planner = DefaultSavePlanner()
        planner.set_up_planner(sd, None, rank == 0)
        blobs = []
        for _, item in items:
            data = planner.resolve_data(item)
            if item.type == WriteItemType.BYTE_IO:
                blobs.append(np.frombuffer(bytes(data.getbuffer()), dtype=np.uint8))
            else:
                blobs.append(oracle.tensor_bytes(data))
        layout = oracle.dcp_item_offsets([b.size for b in blobs])
        total = layout[-1][0] + layout[-1][1] if layout else 0
        want = oracle.pack_ranges(blobs, [o for o, _ in layout], total)
        got = seg_bytes(handler)
        assert got.size == total and np.array_equal(got, want), f"step {step}: segment != oracle"
        meta = handler.metadata.get()
        assert meta["_DLORVER_CKPT_CONFIG"].step == step
        sdata = meta["dcp_metadata"].storage_data
        for (_, item), (off, n) in zip(items, layout):
            info = sdata[item.index]
            assert (info.relative_path, info.offset, info.length) == (f"__{rank}_0.distcp", off, n)
        out["saves"].append({"step": step, "call_ms": call_ms, "items": len(items),
                             "segment_bytes": int(total),
                             "reused_plan": bool(engine.last_save_reused_plan)})
        del got
    # same structure -> the DCP plan is reused (no planning collective) from the 2nd save on
    assert [s["reused_plan"] for s in out["saves"]] == [False, True, True], out["saves"]
    out["dict_sets"] = handler.metadata.dict_sets
    out["ctl_publishes"] = handler.metadata.ctl_publishes
    # a structure change (one entry less) must be noticed on every rank: planned again once,
    # reused afterwards; then back to the original structure for the reload below
    smaller = {"model": dict(sd["model"]), "optim": sd["optim"]}
    smaller["model"].pop(next(iter(smaller["model"])))
    reuse = []
    for step, tree in ((4, smaller), (5, smaller), (6, sd)):
        assert engine.save_to_memory(step, tree, {"model_states": os.path.join(ckpt_dir, str(step))})
        assert engine.wait_memory_save(300)
        reuse.append(bool(engine.last_save_reused_plan))
        dist.barrier()
    assert reuse == [False, True, False], reuse
    # DCP-load back into zeroed shards (same sharding)
    tgt_factory = shapes.ShardedStateFactory(shp, world, rank, dev, mesh, seed=1)
    tgt_factory._wbuf.zero_()
    tgt_factory._mbuf.zero_()
    tgt = tgt_factory.build(0)
    reader = engine.load()
    assert reader is not None
    load_sd = {"model": tgt["model"], "optim": {"state": tgt["optim"]["state"]}}
    dist_cp.load(load_sd, storage_reader=reader)
    a, b = factory.local_tensors(sd), tgt_factory.local_tensors(tgt)
    for k in a:
        assert torch.equal(a[k], b[k]), f"reload mismatch at {k}"
    out["reloaded_tensors"] = len(a)
    out["fast_items"] = getattr(reader, "last_fast_items", None)
    dist.barrier()
    engine.close()
    return out


def llama_state(args, dev, seed):
    from dlrover_b200 import shapes

    shp = shapes.scale_shapes(shapes.llama3_8b_shapes(), args.scale)
    sd = shapes.build_state_dict(shp, torch.bfloat16, dev, seed=seed)
    sd["index"] = torch.arange(100_003, dtype=torch.int64, device=dev) + seed
    sd["bytes"] = (torch.arange(70_001, device=dev) % 251).to(torch.uint8)
    opt = shapes.adamw_state({k: sd[k] for k in list(sd)[:6]}, seed=seed + 5)
    return {"model": sd, "optimizer": opt, "step": 7}


def case_ddp(args, rank, world, dev, ckpt_dir):
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType

    ckpt = DdpCheckpointer(ckpt_dir, local_shard_num=world, global_shard_num=world)
    sd = llama_state(args, dev, seed=100 + rank)
    out = {}
    for step in (1, 2):
        sd["model"]["index"].add_(1)
        ckpt.save_checkpoint(step, sd, storage_type=StorageType.MEMORY)
        assert ckpt.wait_memory_save(300)
        out = compare_with_oracle(ckpt.engine._shm_handler,
                                  {"model_states": sd, "_DLORVER_CKPT_CONFIG": None},
                                  args.full_compare)
    keep = {k: v.clone() for k, v in sd["model"].items()}
    for v in sd["model"].values():
        v.zero_()
    assert ckpt.load_checkpoint_into(sd) == 2
    assert all(torch.equal(sd["model"][k], keep[k]) for k in keep)
    dist.barrier()
    ckpt.engine.close()
    return out


def case_coop(args, rank, world, dev, ckpt_dir):
    from dlrover_b200.flash_checkpoint.api import DdpCheckpointer, StorageType
    from dlrover_b200.shm_handler import CoopContext

    ckpt = DdpCheckpointer(ckpt_dir)  # replicated state, one image per node
    assert ckpt.engine._cooperative()
    sd = llama_state(args, dev, seed=7)  # the same on every rank
    handler = ckpt.engine._shm_handler
    out = {}
    for step in (1, 2, 3):
        sd["model"]["index"].add_(1)
        t0 = time.perf_counter()
        ckpt.save_checkpoint(step, sd, storage_type=StorageType.MEMORY)
        call_ms = (time.perf_counter() - t0) * 1e3
        assert ckpt.wait_memory_save(300)
        dist.barrier()  # the leader's wait covers every slice; followers sync here
        handler.refresh_mapping()
        out = compare_with_oracle(handler, {"model_states": sd, "_DLORVER_CKPT_CONFIG": None},
                                  args.full_compare)
        meta = handler.metadata.get()
        assert meta["_DLORVER_CKPT_CONFIG"].step == step
        assert meta["_DLORVER_CKPT_CONFIG"].writing_shm is False
        out["call_ms"] = call_ms
        dist.barrier()
    total = handler.shared_memory.size
    out["window"] = CoopContext(None, rank % world, world, 0).window(total)
    out["segment"] = handler.shared_memory.name
    out["dict_sets"], out["ctl_publishes"] = handler.metadata.dict_sets, handler.metadata.ctl_publishes
    keep = {k: v.clone() for k, v in sd["model"].items()}
    for v in sd["model"].values():
        v.zero_()
    assert ckpt.load_checkpoint_into(sd) == 3
    assert all(torch.equal(sd["model"][k], keep[k]) for k in keep)
    dist.barrier()
    ckpt.engine.close()
    return out


def case_zero3(args, rank, world, dev, ckpt_dir):
    from dlrover_b200 import shapes
    from dlrover_b200.common.storage import PosixDiskStorage
    from dlrover_b200.flash_checkpoint.engine import DeepSpeedCheckpointEngine

    numel = int(args.flat_mib * (1 << 20) / 4) + 3

    def flat(seed):
        return shapes.fill_(torch.empty(numel, dtype=torch.float32, device=dev), seed + 10 * rank)

    params = [flat(1)]
    optim = {"optimizer_state_dict": {
        "fp32_flat_groups": params,
        "optimizer_state_dict": {
            "state": {0: {"step": torch.tensor(1000.0), "exp_avg": flat(2), "exp_avg_sq": flat(3)}},
            "param_groups": [{"lr": 1e-5, "betas": (0.9, 0.95), "params": [0]}]},
        "zero_stage": 3, "partition_count": [world], "ds_version": "0.14.0"},
        "ds_config": {"zero_optimization": {"stage": 3}}}
    model = {"module": None, "buffer_names": [], "param_shapes": [{"w": (4096, 4096)}],
             "global_steps": 1000, "dp_world_size": world, "mp_world_size": 1}
    state = {"model_states": model, "optim_states": optim}
    engine = DeepSpeedCheckpointEngine(ckpt_dir, PosixDiskStorage(), global_shard_num=world,
                                       zero_stage=3)
    if args.in_place:
        engine.in_place = True
        engine.in_place_snapshot_bytes = args.snapshot_mib << 20
        opt = torch.optim.SGD([torch.nn.Parameter(params[0][:16].clone())], lr=0.1)
        engine.guard_optimizer(opt)
    paths = {"model_states": os.path.join(ckpt_dir, "1000", f"zero_pp_rank_{rank}_model.pt"),
             "optim_states": os.path.join(ckpt_dir, "1000", f"zero_pp_rank_{rank}_optim.pt")}
    out = {"payload_bytes": 3 * numel * 4}
    for step in (1000, 1001, 1002):
        if step == 1001:
            # the first save went through bounce slots and faulted the segment in; time the
            # steady state (plain DMA into the page-locked segment) from here on
            t0 = time.perf_counter()
            out["pinned"] = bool(engine.wait_segment_pinned(600))
            out["background_pin_s"] = time.perf_counter() - t0
            dist.barrier()
        t0 = time.perf_counter()
        assert engine.save_to_memory(step, dict(state), paths)
        call_s = time.perf_counter() - t0
        t1 = time.perf_counter()
        engine.wait_snapshot()            # when the tensors may be written again
        frozen_s = time.perf_counter() - t1
        assert engine.wait_memory_save(1800)
        total_s = time.perf_counter() - t0
        dist.barrier()
        cmp_ = {}
        if step != 1001 or args.full_compare:   # big states: check the first and the last save
            cmp_ = compare_with_oracle(engine._shm_handler,
                                       {**state, "_DLORVER_CKPT_CONFIG": None}, args.full_compare)
        out[f"step_{step}"] = {"call_s": call_s, "sources_frozen_s": frozen_s, "save_s": total_s,
                               "GBps": out["payload_bytes"] / total_s / 1e9,
                               "in_place": bool(engine._shm_handler.last_save_in_place),
                               "hybrid_cut": engine._shm_handler.last_hybrid_cut, **cmp_}
    loaded = engine.load()
    got = loaded["optim_states"]["optimizer_state_dict"]["fp32_flat_groups"][0]
    k = min(got.numel(), 1 << 20)
    assert torch.equal(got[:k], params[0][:k].cpu()) and torch.equal(got[-k:], params[0][-k:].cpu())
    del loaded, got
    dist.barrier()
    engine.close()
    return out


def install_fake_megatron(rank, world):
    """megatron.core.mpu stand-in: TP=2 (fastest), PP=2, DP = world/4."""
    tp, pp = (2, 2) if world % 4 == 0 else ((2, 1) if world % 2 == 0 else (1, 1))
    mpu = types.SimpleNamespace(
        get_tensor_model_parallel_rank=lambda: rank % tp,
        get_pipeline_model_parallel_rank=lambda: (rank // tp) % pp,
        get_data_parallel_rank=lambda: rank // (tp * pp),
        get_tensor_model_parallel_world_size=lambda: tp,
        get_pipeline_model_parallel_world_size=lambda: pp)
    core = types.ModuleType("megatron.core")
    core.mpu = mpu
    meg = types.ModuleType("megatron")
    meg.core = core
    sys.modules["megatron"], sys.modules["megatron.core"] = meg, core
    sys.modules["megatron.core.mpu"] = mpu
    return tp, pp


def case_megatron(args, rank, world, dev, ckpt_dir):
    from dlrover_b200 import shapes
    from dlrover_b200.common.storage import PosixDiskStorage
    from dlrover_b200.flash_checkpoint.engine import MegatronDistCheckpointEngine

    tp, pp = install_fake_megatron(rank, world)
    scale = args.widths or args.scale * 8  # --scale 1/64 -> 1/8 of the Mixtral layer widths
    h, ffn, experts, layers = int(4096 * scale), int(14336 * scale), 8, args.layers
    model = {"args": {"tp": tp, "pp": pp}, "iteration": 20, "checkpoint_version": 3.0, "model": {}}
    for l in range(layers):
        p = f"decoder.layers.{l}."
        model["model"][p + "self_attention.linear_qkv.weight"] = shapes.fill_(
            torch.empty((3 * h // tp, h), dtype=torch.bfloat16, device=dev), l + 7 * rank)
        model["model"][p + "mlp.router.weight"] = shapes.fill_(
            torch.empty((experts, h), dtype=torch.bfloat16, device=dev), 10 + l + 7 * rank)
        for e in range(experts):
            model["model"][p + f"mlp.experts.local_experts.{e}.linear_fc1.weight"] = shapes.fill_(
                torch.empty((2 * ffn // tp, h), dtype=torch.bfloat16, device=dev), 20 + e + rank)
            model["model"][p + f"mlp.experts.local_experts.{e}.linear_fc2.weight"] = shapes.fill_(
                torch.empty((h, ffn // tp), dtype=torch.bfloat16, device=dev), 40 + e + rank)
    dp = max(1, world // (tp * pp))
    optim = {0: {0: {}}}
    for i, (k, t) in enumerate(model["model"].items()):
        n = t.numel() // dp
        optim[0][0][i] = {s: shapes.fill_(torch.empty(n, dtype=torch.float32, device=dev),
                                          100 * j + i + rank)
                          for j, s in enumerate(("param", "exp_avg", "exp_avg_sq"))}
    state = {"model_states": model, "optim_states": optim}
    engine = MegatronDistCheckpointEngine(ckpt_dir, PosixDiskStorage())
    paths = {"model_states": os.path.join(ckpt_dir, "iter_0000020", f"mp_rank_{rank:02d}", "m.pt"),
             "optim_states": os.path.join(ckpt_dir, "iter_0000020", f"rank_{rank:05d}", "o.pt")}
    from dlrover_b200 import shapes as _s

    out = {"payload_bytes": _s.payload_bytes(state), "tp": tp, "pp": pp, "dp": dp}
    for step in (20, 21, 22):
        if step == 21:
            t0 = time.perf_counter()
            out["pinned"] = bool(engine.wait_segment_pinned(600))
            out["background_pin_s"] = time.perf_counter() - t0
            dist.barrier()
        model["iteration"] = step
        t0 = time.perf_counter()
        assert engine.save_to_memory(step, dict(state), paths)
        call_s = time.perf_counter() - t0
        assert engine.wait_memory_save(1800)
        total_s = time.perf_counter() - t0
        dist.barrier()
        cmp_ = {}
        if step != 21 or args.full_compare:
            cmp_ = compare_with_oracle(engine._shm_handler,
                                       {**state, "_DLORVER_CKPT_CONFIG": None}, args.full_compare)
        out[f"step_{step}"] = {"call_s": call_s, "save_s": total_s,
                               "GBps": out["payload_bytes"] / total_s / 1e9, **cmp_}
    step, loaded = engine.load()
    assert step == 22 and loaded["model_states"]["iteration"] == 22
    del loaded
    dist.barrier()
    engine.close()
    return out


def case_fullshards(args, rank, world, dev, ckpt_dir):
    """G2: the FULL checkpoint of a sharded (FSDP-style) state assembled in ONE segment
    without gathering: every rank drains its own shards to their place in the full
    tensors.  Expected image = oracle image of the gathered state dict."""
    from torch.distributed.device_mesh import init_device_mesh

    from dlrover_b200 import shapes
    from dlrover_b200.common.storage import PosixDiskStorage
    from dlrover_b200.flash_checkpoint.engine import FullCheckpointEngine

    mesh = init_device_mesh(dev.type, (world,))
    shp = shapes.scale_shapes(shapes.llama3_8b_shapes(), args.scale)
    factory = shapes.ShardedStateFactory(shp, world, rank, dev, mesh)
    engine = FullCheckpointEngine(ckpt_dir, PosixDiskStorage())
    assert engine.full_from_shards_supported()
    handler = engine._shm_handler
    out = {"payload_bytes_local": factory.local_bytes}
    for step, variant in ((1, 0), (2, 1)):
        sd = factory.build(variant)
        t0 = time.perf_counter()
        assert engine.save_shards_to_memory(step, {"model_states": sd},
                                            {"model_states": os.path.join(ckpt_dir, f"{step}.pt")})
        out["call_ms"] = (time.perf_counter() - t0) * 1e3
        assert engine.wait_memory_save(600)
        dist.barrier()
        handler.refresh_mapping()

        # what a gather would have produced
        def gathered(t):
            if not hasattr(t, "to_local"):
                return t
            local = t.to_local().contiguous()
            parts = [torch.empty_like(local) for _ in range(world)]
            dist.all_gather(parts, local)
            return torch.cat(parts, dim=0)

        def full_tree(v):
            if isinstance(v, dict):
                return {k: full_tree(x) for k, x in v.items()}
            if isinstance(v, list):
                return [full_tree(x) for x in v]
            return gathered(v) if torch.is_tensor(v) else v

        full = full_tree(sd)
        out.update(compare_with_oracle(handler, {"model_states": full,
                                                 "_DLORVER_CKPT_CONFIG": None}, args.full_compare))
        meta = handler.metadata.get()
        assert meta["_DLORVER_CKPT_CONFIG"].step == step
        assert meta["_DLORVER_CKPT_CONFIG"].writing_shm is False
        dist.barrier()
    loaded = engine.load()
    k = next(iter(full["model"]))
    assert torch.equal(loaded["model"][k], full["model"][k].cpu())
    assert loaded["optim"]["param_groups"][0]["lr"] == 3e-4
    del loaded
    out["segment"] = handler.shared_memory.name
    dist.barrier()
    engine.close()
    return out


def case_fsdp_full(args, rank, world, dev, ckpt_dir):
    """FsdpFullCheckpointer on a real torch FSDP module: the full checkpoint is assembled
    from the ranks' SHARDED state dicts; the segment must equal the oracle image of what
    torch's own FULL_STATE_DICT gather produces, and reloading restores the logits."""
    import torch.nn as nn
    from torch.distributed.fsdp import FullOptimStateDictConfig, FullStateDictConfig
    from torch.distributed.fsdp import FullyShardedDataParallel as FSDP
    from torch.distributed.fsdp import StateDictType

    from dlrover_b200.flash_checkpoint.api import StorageType
    from dlrover_b200.flash_checkpoint.fsdp import FsdpFullCheckpointer

    torch.manual_seed(11)
    model = nn.Sequential(nn.Linear(384, 1000), nn.GELU(), nn.LayerNorm(1000),
                          nn.Linear(1000, 777), nn.GELU(), nn.Linear(777, 33)).to(dev)
    fsdp = FSDP(model, device_id=dev if dev.type == "cuda" else None)
    opt = torch.optim.AdamW(fsdp.parameters(), lr=1e-3)
    x = torch.randn(8, 384, device=dev)
    fsdp(x).sum().backward()
    opt.step()
    opt.zero_grad()
    ckpt = FsdpFullCheckpointer(ckpt_dir)
    assert ckpt._from_shards(), "full-from-shards path is off"
    handler = ckpt.engine._shm_handler
    with torch.no_grad():
        want_logits = fsdp(x).clone()
    ckpt.save_checkpoint(5, fsdp, opt, {"epoch": 3}, storage_type=StorageType.MEMORY)
    assert ckpt.wait_memory_save(300)
    dist.barrier()
    handler.refresh_mapping()
    with FSDP.state_dict_type(fsdp, StateDictType.FULL_STATE_DICT,
                              FullStateDictConfig(rank0_only=False),
                              FullOptimStateDictConfig(rank0_only=False)):
        full = {"model": fsdp.state_dict(), "optimizer": FSDP.optim_state_dict(fsdp, opt)}
    full["epoch"] = 3
    out = compare_with_oracle(handler, {"model_states": full, "_DLORVER_CKPT_CONFIG": None}, 1)
    # perturb, reload through the checkpointer, same logits
    with torch.no_grad():
        for p in fsdp.parameters():
            p.add_(0.5)
    extra = ckpt.load_checkpoint(fsdp, opt)
    assert extra.get("epoch") == 3
    with torch.no_grad():
        got = fsdp(x)
    assert torch.equal(got, want_logits), "logits differ after reload"
    dist.barrier()
    ckpt.engine.close()
    return out


CASES = {"fsdp_full": case_fsdp_full, "fullshards": case_fullshards, "fsdp": case_fsdp, "ddp": case_ddp, "coop": case_coop, "zero3": case_zero3,
         "megatron": case_megatron}


def main():
    args = parse()
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(
        os.environ["WORLD_SIZE"])
    os.environ.setdefault("LOCAL_WORLD_SIZE", str(world))
    os.environ.setdefault("DLROVER_LOG_LEVEL", "WARNING")
    os.environ.pop("ROLE_NAME", None)  # local rank 0 forks the saver daemon
    os.environ["TORCHELASTIC_RUN_ID"] = f"mg{os.getppid()}{args.case}"
    if args.device == "cuda":
        torch.cuda.set_device(local)
        dev = torch.device("cuda", local)
    else:
        dev = torch.device("cpu")
    dist.init_process_group(args.backend)
    ckpt_dir = os.path.join(args.out, "ckpt")
    result = {"rank": rank, "world": world, "case": args.case, "ok": False}
    try:
        result.update(CASES[args.case](args, rank, world, dev, ckpt_dir))
        result["ok"] = True
    except BaseException as e:  # noqa: BLE001
        import traceback

        result["error"] = f"{type(e).__name__}: {e}"
        result["traceback"] = traceback.format_exc()[-3000:]
    finally:
        with open(os.path.join(args.out, f"rank{rank}.json"), "w") as f:
            json.dump(result, f, default=str)
    try:
        if result["ok"]:
            dist.barrier()
        dist.destroy_process_group()
    except Exception:
        pass
    # leftovers of this run's namespace (segments are up to tens of GB on the GPU box)
    if local == 0:
        import glob
        import shutil

        time.sleep(0.5)
        for f in glob.glob(f"/dev/shm/{os.environ['TORCHELASTIC_RUN_ID']}_*"):
            try:
                os.unlink(f)
            except OSError:
                pass
        shutil.rmtree(os.path.join("/tmp/ckpt_sock", os.environ["TORCHELASTIC_RUN_ID"]),
                      ignore_errors=True)
    os._exit(0 if result["ok"] else 1)


if __name__ == "__main__":
    main()
