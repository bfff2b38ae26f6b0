"""What the sky's rotation cotangent costs, measured on the device the script runs on (the card's name and power limit are
printed with the numbers).

  * config 3 size (1920 x 1280, R = 1024, training jitter): ``sgn_sky_bwd_view`` against ``sgn_sky_bwd_view_rot`` (the same
    texture gradient plus the direction gradient, its tile sums and the fixed-order reduction), and the deterministic pair
    ``sgn_sky_bwd_det_view`` / ``sgn_sky_bwd_det_view_rot``, alternating, CUDA events around each call, after warm-up;
  * config 4 (tools/train_cfg4.py --sky --camera-opt): training steps/s without and with the sky's rotation cotangent,
    alternating runs.

    python tools/sky_view_grad_timing.py [--launches 200] [--steps 100] [--repeats 6] [--out result.json]

Prints one JSON line."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from pose_grad_timing import card  # noqa: E402


def kernels(launches: int, warmup: int = 20) -> dict:
    import torch

    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200 import raster
    from street_gaussians_ns_b200 import sky as skym
    dev = torch.device("cuda", 0)
    W, H, R = 1920, 1280, 1024
    cam = syn.make_camera(W, H)
    cs = raster.camera_struct(cam, raster.RenderSettings())
    view = torch.tensor(list(cs.viewmat) + list(cs.cam_pos), device=dev, dtype=torch.float32)
    g = torch.Generator(device=dev).manual_seed(0)
    tex = torch.rand(6, R, R, 3, device=dev, generator=g)
    ju, jv = torch.rand(H, W, device=dev, generator=g), torch.rand(H, W, device=dev, generator=g)
    v = torch.randn(H, W, 3, device=dev, generator=g)
    forms = {
        "bwd_view": lambda: skym.sky_backward(cs, R, ju, jv, v, dev, False, view),
        "bwd_view_rot": lambda: skym.sky_backward_rot(cs, tex, ju, jv, v, view, True, False),
        "bwd_det_view": lambda: skym.sky_backward(cs, R, ju, jv, v, dev, True, view),
        "bwd_det_view_rot": lambda: skym.sky_backward_rot(cs, tex, ju, jv, v, view, True, True),
    }
    for _ in range(warmup):
        for fn in forms.values():
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in forms}
    events = []
    for _ in range(launches):
        for name, fn in forms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            events.append((name, e0, e1))
    torch.cuda.synchronize()
    for name, e0, e1 in events:
        times[name].append(e0.elapsed_time(e1))
    med = {k: statistics.median(x) for k, x in times.items()}
    return {"workload": "1920x1280, R = 1024, jittered; each call includes its torch allocations (v_tex zeros, scratch)",
            "launches_each": launches, **{f"{k}_ms_median": x for k, x in med.items()},
            "float_extra_per_cent": 100.0 * (med["bwd_view_rot"] / med["bwd_view"] - 1.0),
            "det_extra_per_cent": 100.0 * (med["bwd_det_view_rot"] / med["bwd_det_view"] - 1.0)}


def training(steps: int, repeats: int) -> dict:
    import train_cfg4
    runs = {"off": [], "on": []}
    for _ in range(repeats):
        for name, flag in (("off", False), ("on", True)):
            res = train_cfg4.run(steps=steps, warmup=10, refine_every=0, sky=True, camera_opt=True, sky_view_grad=flag)
            runs[name].append(res["value"])
    med = {k: statistics.median(v) for k, v in runs.items()}
    return {"workload": "config 4 --sky --camera-opt, one GPU, no refinement in the timed steps", "steps_each": steps,
            "runs_each": repeats, "steps_per_s_off": runs["off"], "steps_per_s_on": runs["on"], "median_off": med["off"],
            "median_on": med["on"], "on_over_off": med["on"] / med["off"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--repeats", type=int, default=6)
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
