"""Per-step metrics (get_metrics_dict) on the config-4 scene (2 M Gaussians in 33 sub-models, 1920 x 1280): the fused call
(loss.fused_metrics, csrc/metrics.cu, one reduction through the frame's device segment table) against the torch statement of
the reference's expressions (sgn_splatfacto.py:1031-1037 over torch.cat of the visible sub-models), alternated in one process.

Times are CUDA events around ``--iters`` calls after a warm-up, ``--repeats`` alternations each; ``model`` is the whole
``get_metrics_dict`` call (host work included).  A torch.profiler pass of its own gives the kernels' device time.  The algorithmic
bytes are 20 B per row (log-scales 12, opacity logit 4, radius 4) plus 12 B per pixel of rgb and 3 B (uint8) or 12 B (float) per
pixel of gt; the achieved bandwidth is those bytes over the kernels' device time (the H100 SXM data sheet gives 3.35 TB/s HBM3
for a card allowed 700 W).  Prints one JSON line; ``--out FILE`` also writes it there."""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import street_gaussians_ns_b200.synthetic as syn  # noqa: E402
from street_gaussians_ns_b200.loss import fused_metrics  # noqa: E402
from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel  # noqa: E402

HBM_BPS = 3.35e12


def torch_statement(model, rgb, gt):
    """The reference's get_metrics_dict expressions over the concatenation of the visible sub-models."""
    subs = [model.all_models._modules[n] for n in model.visible_model_names]
    scales = torch.cat([s.gauss_params["scales"] for s in subs])
    opac = torch.cat([s.gauss_params["opacities"] for s in subs])
    g = gt.float() / 255.0 if gt.dtype == torch.uint8 else gt
    psnr = 10 * torch.log10(1 / torch.mean((rgb - g) ** 2))
    return (psnr, torch.exp(scales).mean(), scales.mean(), torch.sigmoid(opac).mean(), model.radii.float().mean())


def events_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_ms(fn, n=20):
    acc = defaultdict(float)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            acc[e.name.split("(")[0].replace("void ", "")[:80]] += (e.time_range.end - e.time_range.start) / 1e3 / n
    return {k: round(v, 4) for k, v in sorted(acc.items(), key=lambda kv: -kv[1])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--camera", type=int, default=212)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU path)"
    dev = torch.device("cuda", 0)
    props = torch.cuda.get_device_properties(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    sc = syn.WaymoScene(actor_range=45.0)
    frame_list = list(range(sc.num_frames))

    def poses_at(t):
        f = int(t)
        return [ActorPose(str(k), rot, center, f, frame_list) for k, rot, center in sc.boxes_at(f)]

    model = SceneGraphRasterModel(sc.background.to(dev), {k: v.to(dev) for k, v in sc.actors.items()},
                                  SceneGraphConfig(use_sky_sphere=False, async_binning=False), poses_at=poses_at).to(dev)
    model.train()
    model.step = 600
    with torch.no_grad():
        out = model.get_outputs(sc.cameras[a.camera])
    h = model._holder
    rgb = out["rgb"]
    res = dict(device=props.name, power_limit=power, H=sc.height, W=sc.width, rows=h.table.N, segments=h.table.nseg,
               iters=a.iters, repeats=a.repeats, cases={})
    for gt_kind in ("uint8", "float32"):
        g = torch.rand(sc.height, sc.width, 3, generator=torch.Generator().manual_seed(5))
        gt = ((g * 255).to(torch.uint8) if gt_kind == "uint8" else g).to(dev)
        batch = {"image": gt}
        with torch.no_grad():
            calls = {"torch": lambda: torch_statement(model, rgb, gt),
                     "fused": lambda: fused_metrics(rgb, gt, table=h.table, radii=h.radii),
                     "model": lambda: model.get_metrics_dict(out, batch)}
            for fn in calls.values():
                for _ in range(10):
                    fn()
            torch.cuda.synchronize()
            times = defaultdict(list)
            for _ in range(a.repeats):
                for name, fn in calls.items():
                    times[name].append(round(events_ms(fn, a.iters), 4))
            t = torch.stack([x.float() for x in calls["torch"]()]).cpu().tolist()
            f = calls["fused"]().cpu().tolist()
            per = {name: kernel_ms(calls[name]) for name in ("torch", "fused")}
        kern = sum(v for k, v in per["fused"].items() if k.startswith("metrics"))
        nbytes = 20 * h.table.N + sc.height * sc.width * (12 + (3 if gt_kind == "uint8" else 12))
        res["cases"][gt_kind] = dict(
            call_ms=dict(times), call_ms_median={k: sorted(v)[len(v) // 2] for k, v in times.items()},
            kernels=per, torch_kernels_total_ms=round(sum(per["torch"].values()), 4), fused_kernels_ms=round(kern, 4),
            algorithmic_bytes=nbytes, achieved_GBps=round(nbytes / (kern * 1e-3) / 1e9, 1) if kern > 0 else None,
            hbm_bound_ms=round(nbytes / HBM_BPS * 1e3, 4), values_torch=t, values_fused=f)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
