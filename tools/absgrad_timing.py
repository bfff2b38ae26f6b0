"""Timing of the absolute screen-space gradient (sgn_blend_bwd_absgrad, SceneGraphConfig.absgrad).

  * at config 3: sgn_blend_bwd against sgn_blend_bwd_absgrad on the same frame and cotangents (rgb, accumulation,
    object_acc: what training gives), float atomics and deterministic, CUDA events around each launch, the arms alternated,
    medians over the repetitions;
  * config-4 training, steps 605-704 (the refinement at step 700 included), with absgrad off and on (tools/train_cfg4.py),
    alternated runs per arm: steps/s and the row counts after the refinement.

The card's name, power limit and max SM clock are read in the same run.

    python tools/absgrad_timing.py [--reps 50] [--cfg4-runs 2] [--cfg4-steps 100] [--out absgrad_timing.json]
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
from street_gaussians_ns_b200 import raster  # noqa: E402
from depth_timing import card  # noqa: E402


def blend_bwd_times(reps: int, dev) -> dict:
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200.scene import Frame, Segment
    fr = syn.config_frame(3)
    frame = Frame(fr.camera, [Segment(s.params.to(dev), s.cls, s.rot, s.center, s.idft) for s in fr.segments])
    settings = raster.RenderSettings()
    cs = raster.camera_struct(frame.camera, settings)
    bo = raster.blend_opts(settings, False)
    table = raster.SegmentTable(frame, [seg.params.tensors() for seg in frame.segments], dev)
    proj = raster.project_fwd(table, cs, dev)
    records, radii, _, _ = proj
    M, sorted_ids, tile_bins = raster.bin_and_sort(cs, records, radii, proj=proj)
    cls_ids, cls_bins = raster.class_lists(cs, M, sorted_ids, tile_bins)
    out = raster.blend_fwd(cs, bo, records, sorted_ids, tile_bins, None, cls_ids, cls_bins)
    H, W = frame.camera.height, frame.camera.width
    g = torch.Generator().manual_seed(3)
    v = {"rgb": torch.rand(H, W, 3, generator=g).to(dev), "accumulation": torch.rand(H, W, generator=g).to(dev),
         "object_acc": torch.rand(H, W, generator=g).to(dev)}
    res = {"rows": int(records.shape[0]), "intersections": M if isinstance(M, int) else None, "image": [W, H]}
    for det in (False, True):
        ms = {False: [], True: []}
        for i in range(reps + 3):
            for absgrad in (False, True):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                raster.blend_bwd(cs, bo, records, sorted_ids, tile_bins, out, None, v, False, cls_ids, cls_bins,
                                 deterministic=det, absgrad=absgrad)
                b.record()
                torch.cuda.synchronize()
                if i >= 3:
                    ms[absgrad].append(a.elapsed_time(b))
        key = "deterministic" if det else "float"
        med = {k: float(np.median(x)) for k, x in ms.items()}
        res[key] = {"sgn_blend_bwd_ms": med[False], "sgn_blend_bwd_absgrad_ms": med[True],
                    "spread_ms": {"off": [float(min(ms[False])), float(max(ms[False]))], "on": [float(min(ms[True])), float(max(ms[True]))]},
                    "extra": med[True] / med[False] - 1.0}
    res["note"] = ("each timing spans the Python wrapper's allocations (v_records, and v_absxy / the fixed-point buffers) and "
                   "every launch of the backward, between two CUDA events")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--cfg4-runs", type=int, default=2, help="runs per arm (off / on alternated); 0 skips config 4")
    ap.add_argument("--cfg4-steps", type=int, default=100, help="from step 605: crosses the refinement at step 700")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "absgrad_timing measures the GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card(), "config3_blend_bwd": blend_bwd_times(args.reps, dev)}
    torch.cuda.empty_cache()
    if args.cfg4_runs > 0:
        from train_cfg4 import run
        runs = {"off": [], "on": []}
        for _ in range(args.cfg4_runs):
            for arm in ("off", "on"):
                r = run(steps=args.cfg4_steps, warmup=5, absgrad=arm == "on")
                runs[arm].append({"steps_per_s": r["value"], "ms_per_step": r["ms_per_step"],
                                  "gaussians_before": r["gaussians_before"], "gaussians_after": r["gaussians_after"],
                                  "loss_first": r["loss_first"], "loss_last": r["loss_last"]})
                torch.cuda.empty_cache()
        res["cfg4"] = {"steps": args.cfg4_steps, "runs": runs,
                       "median_steps_per_s": {k: float(np.median([x["steps_per_s"] for x in v])) for k, v in runs.items()},
                       "spread_steps_per_s": {k: [float(min(x["steps_per_s"] for x in v)), float(max(x["steps_per_s"] for x in v))]
                                              for k, v in runs.items()}}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
