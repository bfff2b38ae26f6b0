"""What the box gradient costs, measured on the device the script runs on (the card's name and power limit are printed with
the numbers).

  * config 3 (1 M background + 32 x 10 k actor Gaussians, 1920 x 1280): ``sgn_project_bwd`` against ``sgn_project_bwd_pose`` +
    ``sgn_pose_grad_reduce`` over the same record cotangents, alternating, CUDA events around each call, after warm-up;
  * config 4 (tools/train_cfg4.py): training steps/s with the box corrections off and on, alternating runs.

    python tools/pose_grad_timing.py [--launches 200] [--steps 60] [--repeats 2] [--out result.json]

Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # the numbers are still printed, marked as of an unknown card
        return {"name": "unknown", "error": f"{type(e).__name__}: {e}"[:200]}


def kernels(launches: int, warmup: int = 20) -> dict:
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
    v_pose = torch.empty(len(frc.segments), 16, device=dev)

    def plain():
        raster.project_bwd(h.table, params, cs, h.records, h.radii, h.v_records, make_views=False, out=arena)

    def pose():
        raster.project_bwd(h.table, params, cs, h.records, h.radii, h.v_records, make_views=False, out=arena, v_pose=v_pose)

    for _ in range(warmup):
        plain()
        pose()
    torch.cuda.synchronize()
    times = {"plain": [], "pose": []}
    events = []
    for _ in range(launches):
        for name, fn in (("plain", plain), ("pose", pose)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            events.append((name, e0, e1))
    torch.cuda.synchronize()
    for name, e0, e1 in events:
        times[name].append(e0.elapsed_time(e1))
    med = {k: statistics.median(x) for k, x in times.items()}
    posed_chunks = int(sum((s.params.num_points + 127) // 128 for s in frc.segments if s.has_pose))
    return {"workload": "config 3", "launches_each": launches, "chunks": int(h.table.num_chunks), "posed_chunks": posed_chunks,
            "project_bwd_ms_median": med["plain"], "project_bwd_pose_plus_reduce_ms_median": med["pose"],
            "project_bwd_ms_p10_p90": [sorted(times["plain"])[launches // 10], sorted(times["plain"])[launches * 9 // 10]],
            "pose_ms_p10_p90": [sorted(times["pose"])[launches // 10], sorted(times["pose"])[launches * 9 // 10]],
            "extra_per_cent": 100.0 * (med["pose"] / med["plain"] - 1.0)}


def training(steps: int, repeats: int) -> dict:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import train_cfg4
    runs = {"off": [], "on": []}
    for _ in range(repeats):
        for name, flag in (("off", False), ("on", True)):
            res = train_cfg4.run(steps=steps, warmup=10, refine_every=0, bbox_opt=flag)
            runs[name].append(res["value"])
    return {"workload": "config 4, one GPU, no refinement in the timed steps", "steps_each": steps, "steps_per_s_off": runs["off"],
            "steps_per_s_on": runs["on"], "on_over_off": statistics.median(runs["on"]) / statistics.median(runs["off"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device: a timing is a device measurement"
    assert args.launches >= 100, "time at least 100 launches of each form"
    res = {"card": card(), "kernels": kernels(args.launches), "training": training(args.steps, args.repeats)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
