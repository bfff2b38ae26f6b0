"""Per-kernel device times of one forward+backward step of a config (developer tool, not the bench).

torch.profiler with CUDA activities, in a run of its own (tracing slows the host, so end-to-end numbers come from bench.py).
A few warm-up steps, then `--steps` profiled steps; every kernel / memset / copy is summed by name and divided by the
number of steps.  Binning kernels are also grouped into the stages raster.py times (bin_scan, bin_sort, class_lists).
Prints one JSON line; `--out FILE` also writes it there."""
import argparse
import json
import os
import re
import sys
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import street_gaussians_ns_b200.synthetic as syn  # noqa: E402
from street_gaussians_ns_b200 import raster  # noqa: E402
from street_gaussians_ns_b200.scene import Frame, Segment  # noqa: E402

# kernel name (shortened) -> binning stage.  The patterns also name kernels of earlier builds (start_offsets, pad_keys,
# class_count / class_compact and their CUB scan), so profiles of two builds group alike.  CUB sorts are told apart by their
# key type, CUB scans by their input (the depth-order scan reads through PermutedCount); CUB's scan-state initialisation
# kernels carry neither and are listed under "scan_init".
STAGES = [
    ("bin_scan", r"^(depth_keys_kernel|start_offsets_kernel|write_total_kernel)$|\[u32\]|DeviceScanKernel\[depth\]"),
    ("bin_sort", r"^(emit_keys_kernel|emit_big_kernel|pad_keys_kernel|bin_edges_kernel|bin_edges_capped_kernel)$|\[u16\]"),
    ("class_lists", r"^(class_count_kernel|class_compact_kernel|class_lists_kernel)$|DeviceScanKernel\[class\]"),
    ("scan_init", r"^DeviceScanInitKernel$"),
]


def short_name(name: str) -> str:
    base = re.sub(r"^void ", "", name)
    base = base.split("<")[0].split("(")[0].split("::")[-1].strip()
    if "Radix" in base or "Onesweep" in base:
        if "unsigned short" in name:
            base += "[u16]"
        elif "unsigned int" in name:
            base += "[u32]"
    if base == "DeviceScanKernel":
        base += "[depth]" if "PermutedCount" in name else "[class]"
    return base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sync-binning", action="store_true", help="read the intersection count back (bench.py does not)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    fr = syn.config_frame(a.cfg)
    frc = Frame(fr.camera, [Segment(s.params.to(dev).requires_grad_(True), s.cls, s.rot, s.center, s.idft, s.name)
                            for s in fr.segments])
    s = raster.RenderSettings(async_binning=not a.sync_binning)
    H, W = fr.camera.height, fr.camera.width
    w, v = syn.cotangents(H, W)
    w, v = w.to(dev), v.to(dev)[..., None]
    leaves = [t for sg in frc.segments for t in sg.params.tensors()]

    def step():
        out, holder = raster.render_frame(frc, s)
        torch.autograd.backward([out["rgb"], out["accumulation"], out["object_acc"]], [w, v, 0.1 * v])
        for t in leaves:
            t.grad = None
        return holder

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            holder = step()
        torch.cuda.synchronize()
    per = defaultdict(float)
    calls = defaultdict(int)
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        n = short_name(e.name)
        per[n] += (e.time_range.end - e.time_range.start) / 1e3 / a.steps  # us -> ms per step
        calls[n] += 1
    kernels = {k: {"ms": round(per[k], 4), "calls_per_step": calls[k] / a.steps} for k in sorted(per, key=per.get, reverse=True)}
    stages = {}
    for stage, pat in STAGES:
        stages[stage] = round(sum(per[k] for k in per if re.search(pat, k)), 4)
    props = torch.cuda.get_device_properties(dev)
    try:
        import subprocess
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    res = dict(cfg=a.cfg, device=props.name, power_limit=power, steps=a.steps, binning="sync" if a.sync_binning else "async",
               M=int(holder.M), device_ms_per_step=round(sum(per.values()), 4), binning_stages_ms=stages, kernels=kernels)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
