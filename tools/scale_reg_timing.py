"""Timing of the scale regularisation (csrc/scale_reg.cu) and of what it costs config-4 training.

  * sgn_scale_reg_fwd and sgn_scale_reg_bwd over the rows of a config-4 frame (1.68 M background + the actors in view), through
    the frame's device segment table: CUDA events around batches of back-to-back calls, the two kernels' batches alternated,
    medians over the repetitions;
  * the HBM traffic they need (12 B of scales read per row in the forward; 12 B read and 12 B read-modify-written per row in
    the backward) over those times;
  * config-4 training steps/s with the term off and on (tools/train_cfg4.py, --scale-reg), in alternated runs.

The card's name, power limit and max SM clock are read in the same run.

    python tools/scale_reg_timing.py [--reps 50] [--cfg4-runs 2] [--cfg4-steps 100] [--out scale_reg_timing.json]
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
from street_gaussians_ns_b200 import _lib, raster  # noqa: E402
from street_gaussians_ns_b200.scene import Frame, Segment  # noqa: E402
from depth_timing import card  # noqa: E402


def kernels(reps: int, batch: int, dev) -> dict:
    sc = syn.WaymoScene()
    fr = sc.frame(5 * 40 + 1)
    frame = Frame(fr.camera, [Segment(s.params.to(dev), s.cls, s.rot, s.center, s.idft, s.name) for s in fr.segments])
    params = [seg.params.tensors() for seg in frame.segments]
    table = raster.SegmentTable(frame, params, dev)
    sizes, _, _ = raster.arena_layout(table.static)
    arena = torch.zeros(sum(sizes), device=dev)
    v = torch.ones((), device=dev)
    L = _lib.load()
    gt = raster._arena_grads_table(arena, table.static, dev)  # built once: the C call alone is timed
    fwd = lambda: raster.scale_reg_fwd(table, 10.0)  # noqa: E731

    def bwd():
        _lib.check(L.sgn_scale_reg_bwd(raster._ptr(table.dev), raster._ptr(gt), table.nseg, table.N, table.num_chunks, 10.0,
                                       raster._ptr(v), raster._stream()), "sgn_scale_reg_bwd")
    for _ in range(10):
        fwd()
        bwd()
    torch.cuda.synchronize()
    ts = {"fwd": [], "bwd": []}
    for _ in range(reps):
        for name, fn in (("fwd", fwd), ("bwd", bwd)):  # alternated, so that both see the same state of the card
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(batch):
                fn()
            b.record()
            b.synchronize()
            ts[name].append(a.elapsed_time(b) / batch)
    N = table.N
    res = {"rows": int(N), "segments": int(table.nseg), "batch": batch}
    for name, nbytes in (("fwd", 12 * N), ("bwd", 36 * N)):
        med = float(np.median(ts[name]))
        res[f"{name}_ms"] = {"median": med, "min": float(np.min(ts[name])), "max": float(np.max(ts[name]))}
        res[f"{name}_bytes"] = int(nbytes)
        res[f"{name}_GBps_at_median"] = nbytes / (med * 1e-3) / 1e9
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--batch", type=int, default=20)
    ap.add_argument("--cfg4-runs", type=int, default=2, help="runs per arm (off / on alternated); 0 skips config 4")
    ap.add_argument("--cfg4-steps", type=int, default=100, help="from step 605: crosses the refinement at step 700")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "scale_reg_timing measures the GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": args.reps, "kernels_cfg4_frame": kernels(args.reps, args.batch, dev)}
    torch.cuda.empty_cache()
    if args.cfg4_runs > 0:
        from train_cfg4 import run
        runs = {"off": [], "on": []}
        for _ in range(args.cfg4_runs):
            for arm in ("off", "on"):
                r = run(steps=args.cfg4_steps, warmup=5, scale_reg=arm == "on")
                runs[arm].append({"steps_per_s": r["value"], "ms_per_step": r["ms_per_step"], "wall_ms_per_step": r["wall_ms_per_step"],
                                  "ratio_above_10_before": r["ratio_above_10_before"], "ratio_above_10_after": r["ratio_above_10_after"]})
                torch.cuda.empty_cache()
        res["cfg4"] = {"steps": args.cfg4_steps, "runs": runs,
                       "median_steps_per_s": {k: float(np.median([x["steps_per_s"] for x in v])) for k, v in runs.items()}}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
