"""What the antialiased rasterize mode costs: classic and antialiased alternated, at config 3 (1 M + 32 x 10 k Gaussians,
1920x1280) unless --config says otherwise.

  * sgn_project_fwd, sgn_project_bwd, sgn_blend_fwd and sgn_blend_bwd (the raster.py wrappers of those calls), each the
    median of CUDA-event-timed batches of launches on the same frame, the two modes alternated round by round;
  * the intersection count M of each mode (the compensated touch test drops tiles the smaller opacity no longer reaches);
  * the fraction of visible rows with comp < 0.5 (a property of the synthetic scene that makes the numbers above readable);
  * config-4 training steps/s, classic and --antialiased in alternated runs (tools/train_cfg4.py), with their spread.

The card's name and power limit are read in the same run.

    python tools/antialias_timing.py [--reps 30] [--rounds 3] [--cfg4-runs 2] [--cfg4-steps 30] [--out antialias_timing.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import street_gaussians_ns_b200.synthetic as syn  # noqa: E402
from street_gaussians_ns_b200 import raster  # noqa: E402
from street_gaussians_ns_b200.scene import Frame, Segment  # noqa: E402
from depth_timing import card, events_median  # noqa: E402


def stages(frame, mode, dev):
    """The four stage calls of one mode on one frame, on buffers of one forward pass, plus M and the comp statistics."""
    settings = raster.RenderSettings(class_streams=True, rasterize_mode=mode)
    cs = raster.camera_struct(frame.camera, settings)
    bo = raster.blend_opts(settings, False)
    params = [seg.params.tensors() for seg in frame.segments]
    table = raster.SegmentTable(frame, params, dev)
    proj = raster.project_fwd(table, cs, dev)
    records, radii, _, _ = proj
    M, sorted_ids, tile_bins = raster.bin_and_sort(cs, records, radii, proj=proj)
    obj_ids, obj_bins = raster.class_lists(cs, M, sorted_ids, tile_bins)
    out = raster.blend_fwd(cs, bo, records, sorted_ids, tile_bins, None, obj_ids, obj_bins)
    g = torch.Generator().manual_seed(3)
    H, W = cs.height, cs.width
    vd = {"rgb": (torch.rand(H, W, 3, generator=g) * 1e-6).to(dev), "accumulation": (torch.rand(H, W, 1, generator=g) * 1e-6).to(dev),
          "depth": None, "object_acc": (torch.rand(H, W, 1, generator=g) * 1e-6).to(dev), "background_acc": None}
    v_records, _ = raster.blend_bwd(cs, bo, records, sorted_ids, tile_bins, out, None, vd, False, obj_ids, obj_bins)
    size = sum(raster.arena_layout(table.static)[0])
    arena = torch.zeros(size, device=dev)
    calls = {
        "sgn_project_fwd": lambda: raster.project_fwd(table, cs, dev),
        "sgn_project_bwd": lambda: raster.project_bwd(table, params, cs, records, radii, v_records, make_views=False, out=arena),
        "sgn_blend_fwd": lambda: raster.blend_fwd(cs, bo, records, sorted_ids, tile_bins, None, obj_ids, obj_bins),
        "sgn_blend_bwd": lambda: raster.blend_bwd(cs, bo, records, sorted_ids, tile_bins, out, None, vd, False, obj_ids, obj_bins),
    }
    vis = radii > 0
    comp = records[:, 11][vis]
    info = {"M": int(M), "visible": int(vis.sum())}
    if mode == "antialiased":
        info["frac_visible_comp_below_0.5"] = float((comp < 0.5).float().mean())
        info["comp_quartiles"] = [float(x) for x in torch.quantile(comp[:1 << 24].float(), torch.tensor([0.25, 0.5, 0.75], device=dev))]
    return calls, info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3, help="classic / antialiased alternations of the stage timings")
    ap.add_argument("--cfg4-runs", type=int, default=2, help="runs per arm (classic / antialiased alternated); 0 skips config 4")
    ap.add_argument("--cfg4-steps", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "antialias_timing measures the GPU"
    dev = torch.device("cuda", 0)
    fr = syn.config_frame(args.config)
    frame = Frame(fr.camera, [Segment(s.params.to(dev), s.cls, s.rot, s.center, s.idft, s.name) for s in fr.segments])
    res = {"card": card(), "config": args.config, "reps": args.reps, "rounds": args.rounds, "stages_ms": {}, "scene": {}}
    modes = ("classic", "antialiased")
    samples = {m: {} for m in modes}
    for m in modes:
        _, res["scene"][m] = stages(frame, m, dev)
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for m in modes:
            calls, _ = stages(frame, m, dev)
            for name, fn in calls.items():
                samples[m].setdefault(name, []).append(events_median(fn, args.reps, batch=5)["median"])
            del calls
            torch.cuda.empty_cache()
    for m in modes:
        res["stages_ms"][m] = {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
                               for k, v in samples[m].items()}
    res["stage_ratio_antialiased_over_classic"] = {
        k: res["stages_ms"]["antialiased"][k]["median"] / res["stages_ms"]["classic"][k]["median"] for k in samples["classic"]}
    if args.cfg4_runs > 0:
        from train_cfg4 import run
        runs = {m: [] for m in modes}
        for _ in range(args.cfg4_runs):
            for m in modes:
                r = run(steps=args.cfg4_steps, warmup=5, antialiased=(m == "antialiased"))
                runs[m].append({"steps_per_s": r["value"], "ms_per_step": r["ms_per_step"]})
                torch.cuda.empty_cache()
        res["cfg4"] = {"steps": args.cfg4_steps, "runs": runs,
                       "median_steps_per_s": {k: float(np.median([x["steps_per_s"] for x in v])) for k, v in runs.items()},
                       "spread_steps_per_s": {k: float(np.ptp([x["steps_per_s"] for x in v])) for k, v in runs.items()}}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
