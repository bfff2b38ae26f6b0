"""Timing of the bilateral-grid kernels (csrc/bilagrid.cu) and of what the grids cost config-4 training.

  * sgn_bilagrid_slice_fwd and sgn_bilagrid_slice_bwd on a 1920 x 1280 image with a 16 x 16 x 8 grid, and the total variation
    forward and backward over 425 such grids: CUDA events around batches of back-to-back calls, the four batches alternated,
    medians over the repetitions;
  * achieved bytes/s over the algorithmic traffic, against the H100 SXM's 3.35 TB/s: slice forward 24 B/px (rgb read, out
    written) plus the grid; slice backward 36 B/px (rgb and d_out read, d_rgb written) plus the grid read and its gradient
    written; total variation forward 4 B per grid element read, backward 8 B (read and gradient written);
  * config-4 training steps/s with --bilateral-grid off and on (tools/train_cfg4.py), in alternated runs.

The card's name, power limit and max SM clock are read in the same run.

    python tools/bilagrid_timing.py [--reps 30] [--cfg4-runs 2] [--cfg4-steps 100] [--out bilagrid_timing.json]
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
from street_gaussians_ns_b200.bilagrid import IDENTITY  # noqa: E402
from depth_timing import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def kernels(reps: int, batch: int, dev, H: int = 1280, W: int = 1920, L: int = 8, Hg: int = 16, Wg: int = 16, n_img: int = 425) -> dict:
    g = torch.Generator(device="cpu").manual_seed(0)
    ident = torch.tensor(IDENTITY).reshape(1, 12, 1, 1, 1)
    grids = (ident + 0.1 * torch.randn(n_img, 12, L, Hg, Wg, generator=g)).to(dev).contiguous()
    grid = grids[7]
    rgb = torch.rand(H, W, 3, generator=g).to(dev)
    d_out = torch.randn(H, W, 3, generator=g).to(dev)
    out, d_rgb, d_grid = torch.empty_like(rgb), torch.empty_like(rgb), torch.empty_like(grid)
    d_grids = torch.empty_like(grids)
    L_ = _lib.load()
    sb = L_.sgn_bilagrid_slice_bwd_scratch_bytes(L, Hg, Wg, H, W)
    scratch = torch.empty(sb, device=dev, dtype=torch.uint8)
    tsb = L_.sgn_bilagrid_tv_scratch_bytes()
    tscratch = torch.empty(tsb, device=dev, dtype=torch.uint8)
    tv = torch.empty(1, device=dev)
    v = torch.ones(1, device=dev)
    s = _stream()

    def fwd():
        _lib.check(L_.sgn_bilagrid_slice_fwd(_ptr(grid), L, Hg, Wg, _ptr(rgb), H, W, _ptr(out), s), "sgn_bilagrid_slice_fwd")

    def bwd():
        _lib.check(L_.sgn_bilagrid_slice_bwd(_ptr(grid), L, Hg, Wg, _ptr(rgb), _ptr(d_out), H, W, _ptr(d_rgb), _ptr(d_grid), _ptr(scratch),
                                             sb, s), "sgn_bilagrid_slice_bwd")

    def tv_fwd():
        _lib.check(L_.sgn_bilagrid_tv_fwd(_ptr(grids), n_img, L, Hg, Wg, _ptr(tv), _ptr(tscratch), tsb, s), "sgn_bilagrid_tv_fwd")

    def tv_bwd():
        _lib.check(L_.sgn_bilagrid_tv_bwd(_ptr(grids), n_img, L, Hg, Wg, _ptr(v), _ptr(d_grids), s), "sgn_bilagrid_tv_bwd")
    fns = {"slice_fwd": fwd, "slice_bwd": bwd, "tv_fwd": tv_fwd, "tv_bwd": tv_bwd}
    for _ in range(10):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for name, fn in fns.items():  # alternated, so that every kernel sees the same state of the card
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(batch):
                fn()
            b.record()
            b.synchronize()
            ts[name].append(a.elapsed_time(b) / batch)
    px, grid_bytes, all_bytes = H * W, 4 * grid.numel(), 4 * grids.numel()
    nbytes = {"slice_fwd": 24 * px + grid_bytes, "slice_bwd": 36 * px + 2 * grid_bytes, "tv_fwd": all_bytes, "tv_bwd": 2 * all_bytes}
    res = {"image": f"{W}x{H}", "grid": f"{Hg}x{Wg}x{L}", "grids_tv": n_img, "batch": batch, "slice_bwd_scratch_bytes": int(sb)}
    for name in fns:
        med = float(np.median(ts[name]))
        res[name] = {"ms": {"median": med, "min": float(np.min(ts[name])), "max": float(np.max(ts[name]))},
                     "bytes": int(nbytes[name]), "GBps_at_median": nbytes[name] / (med * 1e-3) / 1e9,
                     "share_of_3.35TBps": nbytes[name] / (med * 1e-3) / HBM_BYTES_PER_S}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--batch", type=int, default=20)
    ap.add_argument("--cfg4-runs", type=int, default=2, help="runs per arm (off / on alternated); 0 skips config 4")
    ap.add_argument("--cfg4-steps", type=int, default=100, help="from step 605: crosses the refinement at step 700")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bilagrid_timing measures the GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": args.reps, "kernels": kernels(args.reps, args.batch, dev)}
    torch.cuda.empty_cache()
    if args.cfg4_runs > 0:
        from train_cfg4 import run
        runs = {"off": [], "on": []}
        for _ in range(args.cfg4_runs):
            for arm in ("off", "on"):
                r = run(steps=args.cfg4_steps, warmup=5, bilateral_grid=arm == "on")
                runs[arm].append({"steps_per_s": r["value"], "ms_per_step": r["ms_per_step"], "wall_ms_per_step": r["wall_ms_per_step"],
                                  "loss_first": r["loss_first"], "loss_last": r["loss_last"]})
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
