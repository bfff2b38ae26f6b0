"""What the camera gradient costs, measured on the device the script runs on (the card's name and power limit are printed
with the numbers).

  * config 3 (1 M background + 32 x 10 k actor Gaussians, 1920 x 1280): ``sgn_project_bwd`` against ``sgn_project_bwd_view`` +
    ``sgn_view_grad_reduce`` over the same record cotangents, alternating, CUDA events around each call, after warm-up;
  * config 4 (tools/train_cfg4.py): training steps/s with the camera optimizer off and on, alternating runs, and the host
    time of the camera terms (view, regulariser and metrics' norms: one launch forward, one backward) around a device
    synchronise.

    python tools/camera_grad_timing.py [--launches 200] [--steps 100] [--repeats 8] [--out result.json]

Prints one JSON line."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from pose_grad_timing import card  # noqa: E402


def kernels(launches: int, warmup: int = 20) -> dict:
    import numpy as np
    import torch

    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200 import raster
    from street_gaussians_ns_b200.scene import Frame, Segment
    dev = torch.device("cuda", 0)
    fr = syn.config_frame(3)
    frc = Frame(fr.camera, [Segment(s.params.to(dev), s.cls, s.rot, s.center, s.idft, s.name) for s in fr.segments])
    st = raster.RenderSettings()
    cs = raster.camera_struct(frc.camera, st)
    w, v = syn.cotangents(cs.height, cs.width)
    cot = {"rgb": w.to(dev), "accumulation": v[..., None].to(dev), "object_acc": (0.1 * v)[..., None].to(dev)}
    _, h = raster.forward_backward(frc, st, cot)
    params = [s.params.tensors() for s in frc.segments]
    arena = torch.empty_like(h.grad_arena)
    view = torch.from_numpy(np.concatenate([frc.camera.viewmat().reshape(-1), frc.camera.cam_pos()]).astype(np.float32)).to(dev)
    v_view = torch.empty(12, device=dev)

    def plain():
        raster.project_bwd(h.table, params, cs, h.records, h.radii, h.v_records, make_views=False, out=arena)

    def with_view():
        raster.project_bwd(h.table, params, cs, h.records, h.radii, h.v_records, make_views=False, out=arena, view=view, v_view=v_view)

    for _ in range(warmup):
        plain()
        with_view()
    torch.cuda.synchronize()
    times = {"plain": [], "view": []}
    events = []
    for _ in range(launches):
        for name, fn in (("plain", plain), ("view", with_view)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            events.append((name, e0, e1))
    torch.cuda.synchronize()
    for name, e0, e1 in events:
        times[name].append(e0.elapsed_time(e1))
    med = {k: statistics.median(x) for k, x in times.items()}
    return {"workload": "config 3", "launches_each": launches, "chunks": int(h.table.num_chunks),
            "project_bwd_ms_median": med["plain"], "project_bwd_view_plus_reduce_ms_median": med["view"],
            "extra_per_cent": 100.0 * (med["view"] / med["plain"] - 1.0)}


def host_costs(reps: int = 200) -> dict:
    """Host time per step (to a device synchronise) of the camera terms: view, regulariser and metrics' norms forward (one
    launch) and their backward (one launch), over the 425 cameras of config 4."""
    import torch

    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200.camera_pose import CameraPoseOptimizer
    dev = torch.device("cuda", 0)
    co = CameraPoseOptimizer(425).to(dev)
    cam = syn.make_camera(1920, 1280)
    cam.index = 7

    def step():
        view, reg, _ = co.terms(cam)
        (view[:12].sum() + reg).backward()

    for _ in range(20):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        step()
    torch.cuda.synchronize()
    return {"camera_terms_fwd_bwd_ms": (time.perf_counter() - t0) * 1e3 / reps}


def training(steps: int, repeats: int) -> dict:
    import train_cfg4
    runs = {"off": [], "on": []}
    for _ in range(repeats):
        for name, flag in (("off", False), ("on", True)):
            res = train_cfg4.run(steps=steps, warmup=10, refine_every=0, camera_opt=flag)
            runs[name].append(res["value"])
    med = {k: statistics.median(v) for k, v in runs.items()}
    return {"workload": "config 4, one GPU, no refinement in the timed steps", "steps_each": steps, "runs_each": repeats,
            "steps_per_s_off": runs["off"], "steps_per_s_on": runs["on"], "median_off": med["off"], "median_on": med["on"],
            "on_over_off": med["on"] / med["off"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=8)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device: a timing is a device measurement"
    assert args.launches >= 100, "time at least 100 launches of each form"
    res = {"card": card(), "kernels": kernels(args.launches), "host": host_costs(), "training": training(args.steps, args.repeats)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
