"""Timing of densification by MCMC (csrc/mcmc.cu, mcmc.py) at config-4 sizes.

  * sgn_mcmc_noise over 2 M + 32 x 10 k rows: CUDA events around batches of back-to-back launches, medians over the
    repetitions; achieved bytes/s over the algorithmic traffic of 56 B per row (means read and written, scales, quaternion and
    opacity read), against the H100 SXM's 3.35 TB/s;
  * one refinement of the whole model, MCMC (relocation + growth, gsplat's caps: 1 M for the background, 100 k per actor)
    against the default split / duplicate / cull one (with densification statistics that straddle every threshold), each on a
    fresh model with a FusedAdam, host clock from a synchronise to a synchronise, the two alternated;
  * config-4 training steps/s with --mcmc off and on (tools/train_cfg4.py), in alternated runs.

The card's name, power limit and max SM clock are read in the same run.

    python tools/mcmc_timing.py [--reps 30] [--refine-runs 3] [--cfg4-runs 2] [--cfg4-steps 100] [--out mcmc_timing.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from street_gaussians_ns_b200 import mcmc  # noqa: E402
from street_gaussians_ns_b200.scene import GaussianSet  # noqa: E402
from depth_timing import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
NOISE_BYTES_PER_ROW = 56   # means 12 read + 12 written, scales 12, quats 16, opacity 4


def _sets(dev, n_bg=2_000_000, n_act=10_000, actors=32, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)

    def one(n, F):
        r = lambda *s: torch.randn(s, device=dev, generator=g)  # noqa: E731
        return GaussianSet(r(n, 3) * 20, r(n, 3) * 0.5 - 3, r(n, 4), r(n, F, 3), r(n, 15, 3), r(n, 1) * 2.5 - 1.0)
    return one(n_bg, 1), {str(a): one(n_act, 5) for a in range(actors)}


def noise(reps: int, batch: int, dev) -> dict:
    bg, acts = _sets(dev)
    subs = [bg] + list(acts.values())
    tab = mcmc.NoiseTable()
    entries = [(s.means, s.scales, s.quats, s.opacities, 5e5) for s in subs]
    rows = sum(int(s.means.shape[0]) for s in subs)
    fn = lambda: mcmc.inject_noise(tab, entries, 1.6e-4, seed=0, step=1)  # noqa: E731
    for _ in range(10):
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
    med = float(np.median(ts))
    nbytes = NOISE_BYTES_PER_ROW * rows
    return {"rows": rows, "batch": batch, "ms": {"median": med, "min": float(np.min(ts)), "max": float(np.max(ts))}, "bytes": nbytes,
            "GBps_at_median": nbytes / (med * 1e-3) / 1e9, "share_of_3.35TBps": nbytes / (med * 1e-3) / HBM_BYTES_PER_S}


def one_refinement(strategy: str, dev) -> dict:
    from street_gaussians_ns_b200.model import SceneGraphConfig, SceneGraphRasterModel
    from street_gaussians_ns_b200.optim import FusedAdam
    bg, acts = _sets(dev, seed=1)
    m = SceneGraphRasterModel(bg, acts, SceneGraphConfig(strategy=strategy, use_sky_sphere=False)).to(dev)
    m.train()
    opt = FusedAdam(m.optimizer_params())
    g = torch.Generator(device=dev).manual_seed(3)
    if strategy == "mcmc":
        step = 600
    else:  # densification live (as warm_up_refinement picks it), statistics that straddle the thresholds
        step = 700
        for sub in m.all_models.values():
            n, d = sub.num_points, sub.__dict__
            vis = torch.randint(1, 9, (n,), device=dev, generator=g).float()
            d["vis_counts"] = vis
            d["xys_grad_norm"] = torch.rand(n, device=dev, generator=g) * vis * 2.5e-6
            d["max_2Dsize"] = torch.rand(n, device=dev, generator=g) * 0.2
            d["last_size"] = (1280, 1920)
    m.step = step
    before = sum(s.num_points for s in m.all_models.values())
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m.refinement_after(opt, step, generator=g, seed=7)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    after = sum(s.num_points for s in m.all_models.values())
    del m, opt
    torch.cuda.empty_cache()
    return {"ms": ms, "rows_before": before, "rows_after": after}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--batch", type=int, default=20)
    ap.add_argument("--refine-runs", type=int, default=3, help="refinements per strategy (alternated); the first is a warm-up")
    ap.add_argument("--cfg4-runs", type=int, default=2, help="runs per arm (default / mcmc alternated); 0 skips config 4")
    ap.add_argument("--cfg4-steps", type=int, default=100, help="from step 605: crosses the refinement at step 700")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "mcmc_timing measures the GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card(), "noise": noise(args.reps, args.batch, dev)}
    torch.cuda.empty_cache()
    ref = {"default": [], "mcmc": []}
    for _ in range(args.refine_runs + 1):
        for arm in ("default", "mcmc"):
            ref[arm].append(one_refinement(arm, dev))
    res["refinement"] = {"runs": ref, "median_ms_after_first": {k: float(np.median([x["ms"] for x in v[1:]])) for k, v in ref.items()}}
    if args.cfg4_runs > 0:
        from train_cfg4 import run
        runs = {"default": [], "mcmc": []}
        for _ in range(args.cfg4_runs):
            for arm in ("default", "mcmc"):
                r = run(steps=args.cfg4_steps, warmup=5, mcmc=arm == "mcmc")
                runs[arm].append({"steps_per_s": r["value"], "ms_per_step": r["ms_per_step"], "wall_ms_per_step": r["wall_ms_per_step"],
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
