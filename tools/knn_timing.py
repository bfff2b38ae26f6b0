"""Timing of the GPU k-nearest-neighbour search (sgn_knn) and of SceneGraphRasterModel.from_points on seeded clouds:
street-like at 1 M and 2 M points (70 % ground slab, 30 % volume over config 3's box, a few far outliers) and 32 actor clouds
of 10 k points.  Medians of warmed calls timed with CUDA events; the card's name and power limit are read in the same run.
sklearn's NearestNeighbors(4).kneighbors, what the reference runs, is timed on the same clouds when it is installed.

    python tools/knn_timing.py [--reps 50] [--out knn_timing.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import street_gaussians_ns_b200.synthetic as syn  # noqa: E402
from street_gaussians_ns_b200 import _lib  # noqa: E402
from street_gaussians_ns_b200.knn import knn_log_scales  # noqa: E402
from street_gaussians_ns_b200.model import SceneGraphConfig, SceneGraphRasterModel  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def events_median(fn, reps, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))


def raw_knn(P, k=3):
    """One sgn_knn call with preallocated outputs and scratch (the k-NN scales epilogue, as initialisation uses it)."""
    L = _lib.load()
    n = P.shape[0]
    scratch = torch.empty(L.sgn_knn_scratch_bytes(n, 0), dtype=torch.uint8, device=P.device)
    scales = torch.empty(n, 3, device=P.device)

    def run():
        _lib.check(L.sgn_knn(C.c_void_p(P.data_ptr()), n, None, 0, k, None, None, C.c_void_p(scales.data_ptr()),
                             C.c_void_p(scratch.data_ptr()), scratch.numel(), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
                   "sgn_knn")
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    ap.add_argument("--sklearn-max", type=int, default=2_000_000, help="largest cloud sklearn is timed on (one call each)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "knn_timing measures the GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": args.reps, "sgn_knn_ms": {}, "from_points_ms": {}, "sklearn_s": {}}
    clouds = {n: syn.street_points(n, seed=1) for n in (1_000_000, 2_000_000)}
    actors = {str(a): (syn.actor_points(10_000, seed=100 + a), torch.rand(10_000, 3, generator=torch.Generator().manual_seed(a)) * 255)
              for a in range(32)}
    for n, P in clouds.items():
        Pd = P.to(dev)
        res["sgn_knn_ms"][f"street_{n}"] = events_median(raw_knn(Pd), args.reps)
        res["sgn_knn_ms"][f"street_{n}_knn_log_scales"] = events_median(lambda: knn_log_scales(Pd), args.reps)
    act_dev = [xyz.to(dev) for xyz, _ in actors.values()]
    runs = [raw_knn(x) for x in act_dev]
    res["sgn_knn_ms"]["actors_32x10000"] = events_median(lambda: [r() for r in runs], args.reps)
    for n, P in clouds.items():
        rgb = torch.randint(0, 256, (n, 3), generator=torch.Generator().manual_seed(2), dtype=torch.uint8)
        cfg = SceneGraphConfig(use_sky_sphere=False)
        res["from_points_ms"][f"street_{n}+32x10000"] = events_median(
            lambda: SceneGraphRasterModel.from_points((P, rgb), actors, config=cfg, device=dev), max(10, args.reps // 5), warmup=2)

    # kernel breakdown (a separate profiled run of the 2 M cloud)
    from torch.profiler import ProfilerActivity, profile
    run = raw_knn(clouds[2_000_000].to(dev))
    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            run()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
            t = getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)
            if t > 0:
                kern[e.key[:90]] = t / 10 / 1000.0  # ms per call
    res["kernels_2M_ms_per_call"] = dict(sorted(kern.items(), key=lambda kv: -kv[1]))

    try:
        from sklearn.neighbors import NearestNeighbors
        for n, P in clouds.items():
            if n > args.sklearn_max:
                continue
            x = P.numpy()
            t0 = time.perf_counter()
            NearestNeighbors(n_neighbors=4, algorithm="auto", metric="euclidean").fit(x).kneighbors(x)
            res["sklearn_s"][f"street_{n}"] = time.perf_counter() - t0
        res["cpu_threads"] = os.cpu_count()
    except ImportError:
        res["sklearn_s"] = "not installed"
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
