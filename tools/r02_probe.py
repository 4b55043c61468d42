"""Drain, pinning and hybrid-snapshot measurements on one GPU (prints JSON lines and appends
them to $PROBE_OUT_DIR/r02_probe.jsonl, by default under the system's temporary directory):

  drain     pacing modes x piece sizes: drain GB/s and the latency a foreign `.item()`
            sees while the checkpoint drains (host-paced depth-1 vs two-stream ping-pong)
  pin       what pinning a fresh 16 GB segment costs inline vs in the background, and
            whether background cudaHostRegister stalls the main thread's CUDA calls
  staged    bounce-slot save/restore of an unregistered segment: threads x slot size
  hybrid    AdamW-layout hybrid snapshot (everything behind a 4-byte scalar) through
            the TMA tables vs forced LSU: kernel ms, fraction of the measured peak
  all       everything above
"""
import ctypes
import json
import mmap
import os
import statistics
import sys
import tempfile
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import _posixshmem  # noqa: E402
import torch  # noqa: E402

from dlrover_b200 import _native as native  # noqa: E402
from dlrover_b200 import shapes  # noqa: E402

OUT = os.environ.get("PROBE_OUT_DIR") or os.path.join(tempfile.gettempdir(), "fc_probe")
os.makedirs(OUT, exist_ok=True)
LOG = open(os.path.join(OUT, "r02_probe.jsonl"), "a")


def emit(rec):
    line = json.dumps(rec)
    print(line, flush=True)
    LOG.write(line + "\n")
    LOG.flush()


class Segment:
    def __init__(self, nbytes, tag):
        self.name = f"/fc_probe_{tag}_{os.getpid()}"
        self.fd = _posixshmem.shm_open(self.name, os.O_CREAT | os.O_EXCL | os.O_RDWR, mode=0o600)
        os.ftruncate(self.fd, nbytes)
        self.mm = mmap.mmap(self.fd, nbytes)
        self.addr = ctypes.addressof(ctypes.c_char.from_buffer(self.mm))
        self.nbytes = nbytes

    def close(self):
        self.mm.close()
        os.close(self.fd)
        _posixshmem.shm_unlink(self.name)


def llama_plan(ctx, displacement=0):
    sd = shapes.build_state_dict(shapes.llama3_8b_shapes(), torch.bfloat16, "cuda", fill=False)
    leaves = list(sd.values())
    offs, o = [], displacement
    for t in leaves:
        offs.append(o)
        o += t.numel() * 2
    return sd, leaves, offs, o


def foreign_copies(stop, out, dev_scalar):
    """`.item()` in a loop on the main stream while something else drains."""
    while not stop.is_set():
        t0 = time.perf_counter()
        dev_scalar.item()
        out.append((time.perf_counter() - t0) * 1e3)
        time.sleep(0.002)


def probe_drain():
    ctx = native.Context(0)
    sd, leaves, offs, total = llama_plan(ctx)
    seg = Segment(total, "drain")
    ctx.host_register(seg.addr, total, prefault_threads=16)
    ctx.arena_reserve(total)
    plan = ctx.plan([t.data_ptr() for t in leaves], offs, [t.numel() * 2 for t in leaves])
    stream = torch.cuda.current_stream()
    scalar = torch.ones(1, device="cuda")
    base = []
    for _ in range(200):
        t0 = time.perf_counter()
        scalar.item()
        base.append((time.perf_counter() - t0) * 1e3)
    emit({"probe": "drain", "baseline_item_ms": {"median": statistics.median(base), "max": max(base)}})
    for mode, name in ((native.DRAIN_HOST_PACED, "host_paced"), (native.DRAIN_PINGPONG, "pingpong")):
        for piece_mb in (2, 4, 8, 16, 32, 64):
            ctx.set_drain_mode(mode)
            ctx.set_drain(piece_mb << 20, 1)
            ctx.save_wait(plan.save_async(seg.addr, stream))  # warm
            lat, stop = [], threading.Event()
            drains, totals = [], []
            th = threading.Thread(target=foreign_copies, args=(stop, lat, scalar))
            th.start()
            for _ in range(3):
                tk = plan.save_async(seg.addr, stream)
                ctx.save_wait(tk)
                p, d, tot = ctx.save_timings(tk)
                drains.append(d)
                totals.append(tot)
            stop.set()
            th.join()
            lat.sort()
            emit({"probe": "drain", "mode": name, "piece_MiB": piece_mb,
                  "drain_GBps": total / (sum(drains) / len(drains)) / 1e6,
                  "save_GBps": total / (sum(totals) / len(totals)) / 1e6,
                  "item_ms": {"n": len(lat), "median": lat[len(lat) // 2],
                              "p99": lat[int(len(lat) * 0.99)], "max": lat[-1]}})
    plan.destroy()
    ctx.host_unregister(seg.addr)
    ctx.destroy()
    seg.close()


def launch_latency(stop, out):
    x = torch.zeros(1, device="cuda")
    while not stop.is_set():
        t0 = time.perf_counter()
        x.add_(1)
        torch.cuda.current_stream().synchronize()
        out.append((time.perf_counter() - t0) * 1e3)


def probe_pin():
    total = 16_060_522_496
    ctx = native.Context(0)
    # 1. inline, as round 1: bind + parallel prefault + one cudaHostRegister
    seg = Segment(total, "pin1")
    t0 = time.perf_counter()
    ctx.host_register(seg.addr, total, prefault_threads=16)
    inline_s = time.perf_counter() - t0
    ctx.host_unregister(seg.addr)
    # 2. the same pages (now resident), pinned again: registration alone
    t0 = time.perf_counter()
    ctx.host_register(seg.addr, total, prefault_threads=0)
    pin_only_s = time.perf_counter() - t0
    ctx.host_unregister(seg.addr)
    emit({"probe": "pin", "bytes": total, "inline_prefault_and_pin_s": inline_s,
          "pin_only_resident_pages_s": pin_only_s})
    # 3. background, slice sizes; main thread keeps launching tiny kernels
    for slice_mb in (16, 64, 256, 0):
        lat, stop = [], threading.Event()
        th = threading.Thread(target=launch_latency, args=(stop, lat))
        th.start()
        time.sleep(0.2)
        n_before = len(lat)
        t0 = time.perf_counter()
        ctx.host_register_background(seg.addr, total,
                                     slice_bytes=(slice_mb << 20) if slice_mb else (total + 4095) // 4096 * 4096)
        call_s = time.perf_counter() - t0
        while not ctx.host_ready(seg.addr):
            time.sleep(0.005)
        ready_s = time.perf_counter() - t0
        stop.set()
        th.join()
        during = sorted(lat[n_before:]) or [0.0]
        before = sorted(lat[:n_before]) or [0.0]
        emit({"probe": "pin_background", "slice_MiB": slice_mb or "whole", "call_s": call_s,
              "ready_s": ready_s,
              "launch_sync_ms_before": {"median": before[len(before) // 2], "max": before[-1]},
              "launch_sync_ms_during": {"n": len(during), "median": during[len(during) // 2],
                                        "p99": during[int(len(during) * 0.99)], "max": during[-1]}})
        ctx.host_unregister(seg.addr)
    ctx.destroy()
    seg.close()


def probe_staged():
    for threads, slot_mb in ((4, 8), (8, 4), (8, 8), (8, 16), (16, 8), (16, 16), (32, 8)):
        ctx = native.Context(0)
        ctx.set_stage(threads, slot_mb << 20)
        sd, leaves, offs, total = llama_plan(ctx)
        ctx.arena_reserve(total)
        plan = ctx.plan([t.data_ptr() for t in leaves], offs, [t.numel() * 2 for t in leaves])
        stream = torch.cuda.current_stream()
        seg = Segment(total, f"st{threads}_{slot_mb}")
        ctx.host_bind_numa(seg.addr, total, 0)
        rec = {"probe": "staged", "threads": threads, "slot_MiB": slot_mb, "bytes": total}
        t0 = time.perf_counter()
        ctx.save_wait(plan.save_async(seg.addr, stream))  # first touch of every page
        rec["first_save_fresh_segment_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        ctx.save_wait(plan.save_async(seg.addr, stream))
        rec["save_touched_segment_s"] = time.perf_counter() - t0
        for t in leaves[:3]:
            t.zero_()
        t0 = time.perf_counter()
        plan.restore_async(seg.addr, stream, direct=True)
        ctx.restore_wait()
        torch.cuda.synchronize()
        rec["restore_direct_s"] = time.perf_counter() - t0
        rec["save_GBps"] = total / rec["save_touched_segment_s"] / 1e9
        rec["restore_GBps"] = total / rec["restore_direct_s"] / 1e9
        emit(rec)
        plan.destroy()
        del sd, leaves
        ctx.destroy()
        seg.close()
        torch.cuda.empty_cache()


def probe_hybrid():
    peak = 6590.0
    try:
        peak = float(json.load(open(os.path.join(os.path.dirname(OUT), "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass
    for variant, name in ((native.VARIANT_TMA, "tma_tables"), (native.VARIANT_LSU, "lsu")):
        ctx = native.Context(0)
        ctx.set_variant(variant)
        sd, leaves, offs, end = llama_plan(ctx, displacement=4)
        step = torch.ones(1, dtype=torch.float32, device="cuda")  # the 4-byte AdamW `step`
        ptrs = [step.data_ptr()] + [t.data_ptr() for t in leaves]
        lens = [4] + [t.numel() * 2 for t in leaves]
        plan = ctx.plan(ptrs, [0] + offs, lens)
        cut = 4
        ctx.arena_reserve(end - (cut & ~127))
        host = Segment(end, "hyb")
        ctx.host_register(host.addr, end, prefault_threads=16)
        stream = torch.cuda.current_stream()
        packs = []
        for i in range(6):
            tk = plan.save_hybrid_async(host.addr, cut, stream)
            ctx.save_wait(tk)
            p, d, tot = ctx.save_timings(tk)
            if i:
                packs.append(p)
        ms = sum(packs) / len(packs)
        payload = end - 4
        emit({"probe": "hybrid", "variant": name, "snapshot_bytes": payload, "cut": cut,
              "gather_ms": ms, "achieved_GBps": 2 * payload / ms / 1e6, "peak_GBps": peak,
              "frac_of_measured_peak": 2 * payload / ms / 1e6 / peak})
        plan.destroy()
        ctx.host_unregister(host.addr)
        ctx.destroy()
        host.close()
        del sd, leaves
        torch.cuda.empty_cache()


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    torch.cuda.set_device(0)
    emit({"probe": "env", "which": which, "cpus": os.cpu_count(),
          "gpu": torch.cuda.get_device_name(0), "numa": native.device_numa_node(0)})
    if which in ("drain", "all"):
        probe_drain()
    if which in ("hybrid", "all"):
        probe_hybrid()
    if which in ("staged", "all"):
        probe_staged()
    if which in ("pin", "all"):
        probe_pin()
