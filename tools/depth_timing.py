"""Timing of the lidar depth supervision (csrc/depth.cu) and of what it costs a training step.

  * sgn_lidar_depth_map at 170 k points (about one top-lidar sweep) and 2 M points, 1920x1280, config 3's camera;
  * the depth loss forward + backward at 1920x1280 (a sweep's map as the target);
  * sgn_blend_bwd at config 3 with and without a depth cotangent (the same rgb / accumulation / object_acc cotangents
    otherwise), alternated call by call;
  * config-4 training steps/s with the term off and on (tools/train_cfg4.py, --lidar-depth), in alternated runs.

Medians of warmed calls timed with CUDA events (the C-ABI calls on preallocated buffers, back to back); the card's name and
power limit are read in the same run.

    python tools/depth_timing.py [--reps 50] [--cfg4-runs 2] [--cfg4-steps 30] [--out depth_timing.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import street_gaussians_ns_b200.synthetic as syn  # noqa: E402
from street_gaussians_ns_b200 import _lib, raster  # noqa: E402
from street_gaussians_ns_b200.depth import fused_depth_loss, lidar_depth_map  # noqa: E402
from street_gaussians_ns_b200.scene import Frame, Segment  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def events_median(fn, reps, warmup=5, batch=20):
    """Per-call device time: CUDA events around ``batch`` back-to-back calls (so that the host's launch overhead overlaps
    the device work), ``reps`` times; median / min / max of the per-call means."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(batch):
            fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / batch)
    return {"median": float(np.median(ts)), "min": float(np.min(ts)), "max": float(np.max(ts))}


def raw_calls(P, cs, target, depth):
    """The C-ABI calls alone, on preallocated buffers: the map, and the loss forward + backward."""
    L = _lib.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = torch.empty(cs.height, cs.width, device=P.device)
    loss = torch.empty((), device=P.device)
    n_valid = torch.empty((), device=P.device, dtype=torch.int32)
    v = torch.empty_like(depth)
    sb = L.sgn_depth_scratch_bytes()
    scratch = torch.empty(sb, device=P.device, dtype=torch.uint8)

    def ptr(t):
        return C.c_void_p(t.data_ptr())

    def depth_map():
        _lib.check(L.sgn_lidar_depth_map(ptr(P), P.shape[0], C.byref(cs), None, ptr(out), st), "sgn_lidar_depth_map")

    def loss_fb():
        _lib.check(L.sgn_depth_loss_fwd(cs.height, cs.width, ptr(depth), ptr(target), None, 0.1, ptr(loss), ptr(n_valid), ptr(scratch),
                                        sb, st), "sgn_depth_loss_fwd")
        _lib.check(L.sgn_depth_loss_bwd(cs.height, cs.width, ptr(depth), ptr(target), None, 0.1, ptr(n_valid), None, ptr(v), st),
                   "sgn_depth_loss_bwd")
    return depth_map, loss_fb


def blend_bwd_ab(reps, dev):
    """sgn_blend_bwd at config 3 (1 M + 32 x 10 k Gaussians, 1920x1280), with and without a depth cotangent, alternated."""
    fr = syn.config_frame(3)
    frame = Frame(fr.camera, [Segment(s.params.to(dev), s.cls, s.rot, s.center, s.idft, s.name) for s in fr.segments])
    settings = raster.RenderSettings(class_streams=True)
    cs = raster.camera_struct(frame.camera, settings)
    bo = raster.blend_opts(settings, False)
    params = [seg.params.tensors() for seg in frame.segments]
    table = raster.SegmentTable(frame, params, dev)
    proj = raster.project_fwd(table, cs, dev)
    records, radii, _, _ = proj
    M, sorted_ids, tile_bins = raster.bin_and_sort(cs, records, radii, proj=proj)
    obj_ids, obj_bins = raster.class_lists(cs, M, sorted_ids, tile_bins)
    out = raster.blend_fwd(cs, bo, records, sorted_ids, tile_bins, None, obj_ids, obj_bins)
    H, W = cs.height, cs.width
    w_rgb, w_acc = (t.to(dev) for t in syn.cotangents(H, W))
    g = torch.Generator().manual_seed(3)
    v_obj = (torch.rand(H, W, 1, generator=g) * 1e-3).to(dev)
    target = lidar_depth_map(syn.street_points(170_000, seed=1).to(dev), cs)
    d = out["depth"].clone().requires_grad_(True)
    fused_depth_loss(d, target, None, 0.1).backward()
    v_depth = d.grad
    base = {"rgb": w_rgb, "accumulation": w_acc, "object_acc": v_obj}
    arms = {"without_depth": base, "with_depth": dict(base, depth=v_depth)}
    raster.TIMER = raster.StageTimer()
    ms = {k: [] for k in arms}
    try:
        for i in range(reps + 5):
            for k, v in arms.items():
                raster.TIMER.events.clear()
                raster.blend_bwd(cs, bo, records, sorted_ids, tile_bins, out, None, v, False, obj_ids, obj_bins)
                torch.cuda.synchronize()
                if i >= 5:
                    ms[k].append(raster.TIMER.mean_ms()["blend_bwd"])
    finally:
        raster.TIMER = None
    res = {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in ms.items()}
    res["intersections"] = int(M)
    res["valid_depth_pixels"] = int((target > 0).sum())
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--cfg4-runs", type=int, default=2, help="runs per arm (off / on alternated); 0 skips config 4")
    ap.add_argument("--cfg4-steps", type=int, default=30)
    ap.add_argument("--cfg4-weight", type=float, default=0.1)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "depth_timing measures the GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": args.reps, "sgn_lidar_depth_map_ms": {}}
    cs = raster.camera_struct(syn.make_camera(1920, 1280), raster.RenderSettings())
    target = lidar_depth_map(syn.street_points(170_000, seed=1).to(dev), cs)[..., 0].contiguous()
    res["valid_pixels_170k"] = int((target > 0).sum())
    depth = (torch.rand(1280, 1920, generator=torch.Generator().manual_seed(0)) * 50).to(dev)
    for n in (170_000, 2_000_000):
        P = syn.street_points(n, seed=1).to(dev)
        depth_map, loss_fb = raw_calls(P, cs, target, depth)
        res["sgn_lidar_depth_map_ms"][f"street_{n}"] = events_median(depth_map, args.reps)
    res["sgn_depth_loss_fwd_bwd_ms"] = events_median(loss_fb, args.reps)
    P = syn.street_points(170_000, seed=1).to(dev)

    def python_surface():  # depth.py as the model calls it: map, autograd node, backward
        d = depth.view(1280, 1920, 1).requires_grad_(True)
        fused_depth_loss(d, lidar_depth_map(P, cs), None, 0.1).backward()
    res["python_map_loss_fwd_bwd_ms"] = events_median(python_surface, args.reps, batch=5)
    res["blend_bwd_cfg3_ms"] = blend_bwd_ab(args.reps, dev)
    torch.cuda.empty_cache()

    if args.cfg4_runs > 0:
        from train_cfg4 import run
        runs = {"off": [], "on": []}
        for _ in range(args.cfg4_runs):
            for arm, w in (("off", 0.0), ("on", args.cfg4_weight)):
                r = run(steps=args.cfg4_steps, warmup=5, lidar_depth=w)
                runs[arm].append({"steps_per_s": r["value"], "ms_per_step": r["ms_per_step"], "wall_ms_per_step": r["wall_ms_per_step"]})
                torch.cuda.empty_cache()
        res["cfg4"] = {"weight": args.cfg4_weight, "steps": args.cfg4_steps, "runs": runs,
                       "median_steps_per_s": {k: float(np.median([x["steps_per_s"] for x in v])) for k, v in runs.items()}}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
