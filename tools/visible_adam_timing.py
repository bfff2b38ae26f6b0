"""Timing of the selective Adam step (sgn_adam_step_visible, TrainStep(visible_adam=True)).

  * at config 4: inside a training run of tools/train_cfg4.py with visible_adam (steps 605-704), at some of its optimizer
    steps, sgn_adam_step against sgn_adam_step_visible over that step's tensors (the frame's sub-models), gradient arena and
    visibility bytes (sgn_visible_flags of the frame's radii).  CUDA events around a batch of
    back-to-back launches, the arms alternated, medians over the repetitions.  Reported per frame: the seen-row fraction, the
    algorithmic bytes (28 B per stepped element, plus 1 B of flags per row of a masked tensor) and their rate against the
    data sheet's 3.35 TB/s; and the all-rows-seen launch against the dense one (the cost of the row test);
  * config-4 training, steps 605-704 (the refinement at step 700 included), with visible_adam off and on (tools/train_cfg4.py),
    alternated runs per arm: steps/s with its spread.

The card's name, power limit and max SM clock are read in the same run.

    python tools/visible_adam_timing.py [--frames 8] [--reps 30] [--cfg4-runs 3] [--cfg4-steps 100] [--out visible_adam_timing.json]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from street_gaussians_ns_b200 import _lib  # noqa: E402
from depth_timing import card  # noqa: E402

HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s


def kernel_times(frames: int, reps: int, batch: int, dev) -> dict:
    """Times the two launches inside a config-4 training run with visible_adam (tools/train_cfg4.py, steps 605-704): at every
    ``100 // frames``-th optimizer step, on that step's tensors, arena and flags, before the step itself runs.  The timed
    launches change the run's parameters (it is not the A/B run)."""
    from train_cfg4 import run
    from street_gaussians_ns_b200.optim import FusedAdam
    L = _lib.load()
    every = max(1, 100 // frames)
    out = {"frames": []}
    real_step = FusedAdam.step
    calls = [0]

    def upload(tab, rows=None):
        raw = tab.view(np.uint8).reshape(-1) if rows is None else np.concatenate([tab.view(np.uint8).reshape(-1), rows.view(np.uint8).reshape(-1)])
        return torch.from_numpy(raw.copy()).to(dev)

    def timed(opt, arena, present, full_layout, flags):
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        steps = opt.steps.copy()
        tab, rows = opt.step_table(present, full_layout=full_layout, visible=True)
        opt.steps[:] = steps  # the timing does not count as a step
        nch = int(tab["chunk0"][-1] + (int(tab["numel"][-1]) + 4095) // 4096)
        d_dense, d_vis = upload(tab), upload(tab, rows)
        r_ptr = C.c_void_p(d_vis.data_ptr() + tab.nbytes)
        seen = flags.cpu().numpy() != 0
        ones = torch.ones_like(flags)
        # algorithmic bytes: 28 B per stepped element; the selective step also reads one flag byte per row
        elems = int(tab["numel"].sum())
        stepped = sum(int(seen[r0:r0 + num // w].sum()) * int(w) for r0, num, w in zip(rows["flag_row0"], tab["numel"], rows["row_width"]))
        flag_bytes = sum(int(num // w) for num, w in zip(tab["numel"], rows["row_width"]))
        ptrs = (C.c_void_p(arena.data_ptr()), C.c_void_p(opt.exp_avg.data_ptr()), C.c_void_p(opt.exp_avg_sq.data_ptr()))

        def dense():
            _lib.check(L.sgn_adam_step(C.c_void_p(d_dense.data_ptr()), len(tab), nch, *ptrs, stream), "dense")

        def selective(vis):
            return lambda: _lib.check(L.sgn_adam_step_visible(C.c_void_p(d_vis.data_ptr()), r_ptr, len(tab), nch, *ptrs,
                                                              C.c_void_p(vis.data_ptr()), stream), "selective")
        arms = {"dense": dense, "visible": selective(flags), "all_visible": selective(ones)}
        ms = {k: [] for k in arms}
        for i in range(reps + 2):
            for k, fn in arms.items():  # alternated
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(batch):
                    fn()
                b.record()
                torch.cuda.synchronize()
                if i >= 2:
                    ms[k].append(a.elapsed_time(b) / batch)
        med = {k: float(np.median(v)) for k, v in ms.items()}
        return {"frame_rows": int(seen.size), "submodels": len(present), "seen_fraction": float(seen.mean()),
                "stepped_element_fraction": stepped / elems, "ms": med,
                "spread_ms": {k: [float(min(v)), float(max(v))] for k, v in ms.items()},
                "speedup": med["dense"] / med["visible"], "all_visible_overhead": med["all_visible"] / med["dense"] - 1.0,
                "bytes": {"dense": 28 * elems, "visible": 28 * stepped + flag_bytes},
                "rate_of_peak": {"dense": 28 * elems / (med["dense"] * 1e-3) / HBM_PEAK,
                                 "visible": (28 * stepped + flag_bytes) / (med["visible"] * 1e-3) / HBM_PEAK}}

    def spy(self, grad_arena, present=None, full_layout=False, **kw):
        vis = kw.get("visible")
        if vis is not None and calls[0] >= 5 and (calls[0] - 5) % every == 0 and len(out["frames"]) < frames and not kw.get("kinds"):
            n = sum(int(self._params[6 * s].shape[0]) for s in present)
            out["frames"].append(timed(self, grad_arena, list(present), full_layout, vis[:n].clone()))
        calls[0] += 1
        return real_step(self, grad_arena, present=present, full_layout=full_layout, **kw)
    FusedAdam.step = spy
    try:
        run(steps=100, warmup=5, visible_adam=True)
    finally:
        FusedAdam.step = real_step
    fr = out["frames"]
    out["median"] = {k: float(np.median([f[k] for f in fr])) for k in ("seen_fraction", "speedup", "all_visible_overhead")}
    out["note"] = (f"per-launch device time: CUDA events around {batch} back-to-back launches, {reps} alternated repetitions; "
                   "the tables are on the device before timing")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=8, help="config-4 frames of the kernel timing; 0 skips it")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--batch", type=int, default=10)
    ap.add_argument("--cfg4-runs", type=int, default=3, help="runs per arm (off / on alternated); 0 skips the training runs")
    ap.add_argument("--cfg4-steps", type=int, default=100, help="from step 605: crosses the refinement at step 700")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "visible_adam_timing measures the GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card()}
    if args.frames > 0:
        res["config4_adam"] = kernel_times(args.frames, args.reps, args.batch, dev)
        torch.cuda.empty_cache()
    if args.cfg4_runs > 0:
        from train_cfg4 import run
        runs = {"off": [], "on": []}
        for _ in range(args.cfg4_runs):
            for arm in ("off", "on"):
                r = run(steps=args.cfg4_steps, warmup=5, visible_adam=arm == "on")
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
