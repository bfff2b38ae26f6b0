"""Timing of the semantic term (csrc/semantic.cu, and the extra-channel blend it rides on) and of what it costs a training step.

  * the semantic loss forward + backward and the confusion pass at 1920x1280, C = 3 and C = 19;
  * sgn_blend_extra_fwd and sgn_blend_extra_bwd at C = 3 on config 3 (1 M + 32 x 10 k Gaussians, 1920x1280): the one more
    traversal of the tile lists a training step with semantics makes in the forward and in the backward;
  * config-4 training steps/s with the term off and on (tools/train_cfg4.py, --semantic), in alternated runs.

Medians of warmed calls timed with CUDA events; the card's name and power limit are read in the same run.

    python tools/semantic_timing.py [--reps 50] [--cfg4-runs 2] [--cfg4-steps 30] [--out semantic_timing.json]
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
import street_gaussians_ns_b200.synthetic as syn  # noqa: E402
from street_gaussians_ns_b200 import _lib, raster  # noqa: E402
from street_gaussians_ns_b200.scene import Frame, Segment  # noqa: E402
from depth_timing import card, events_median  # noqa: E402


def loss_calls(H, W, Cn, dev):
    """The C-ABI calls alone on preallocated buffers: loss forward + backward, and the confusion pass."""
    g = torch.Generator().manual_seed(Cn)
    logits = (torch.randn(H, W, Cn, generator=g) * 3).to(dev)
    labels = torch.randint(0, Cn, (H, W), generator=g).to(dev)
    L = _lib.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    loss = torch.empty((), device=dev)
    n_valid = torch.empty((), device=dev, dtype=torch.int32)
    v = torch.empty_like(logits)
    conf = torch.empty(Cn, Cn, device=dev, dtype=torch.int64)
    sb = L.sgn_semantic_scratch_bytes()
    scratch = torch.empty(sb, device=dev, dtype=torch.uint8)

    def ptr(t):
        return C.c_void_p(t.data_ptr())

    def loss_fb():
        _lib.check(L.sgn_semantic_loss_fwd(H, W, Cn, ptr(logits), ptr(labels), None, 0.1, ptr(loss), ptr(n_valid), ptr(scratch), sb, st),
                   "sgn_semantic_loss_fwd")
        _lib.check(L.sgn_semantic_loss_bwd(H, W, Cn, ptr(logits), ptr(labels), None, 0.1, ptr(n_valid), None, ptr(v), st),
                   "sgn_semantic_loss_bwd")

    def confusion():
        _lib.check(L.sgn_semantic_metrics(H, W, Cn, ptr(logits), ptr(labels), None, ptr(conf), st), "sgn_semantic_metrics")
    return loss_fb, confusion


def blend_extra_cfg3(reps, dev, Cn=3):
    """sgn_blend_extra_fwd / sgn_blend_extra_bwd (float and deterministic) at config 3 with C channels."""
    fr = syn.config_frame(3)
    frame = Frame(fr.camera, [Segment(s.params.to(dev), s.cls, s.rot, s.center, s.idft, s.name) for s in fr.segments])
    settings = raster.RenderSettings(class_streams=True)
    cs = raster.camera_struct(frame.camera, settings)
    bo = raster.blend_opts(settings, False)
    params = [seg.params.tensors() for seg in frame.segments]
    table = raster.SegmentTable(frame, params, dev)
    proj = raster.project_fwd(table, cs, dev)
    records, radii, _, _ = proj
    M, sorted_ids, tile_bins = raster.bin_and_sort(cs, records, radii, proj=proj)
    obj_ids, obj_bins = raster.class_lists(cs, M, sorted_ids, tile_bins)
    out = raster.blend_fwd(cs, bo, records, sorted_ids, tile_bins, None, obj_ids, obj_bins)
    N = records.shape[0]
    extra = torch.randn(N, Cn, generator=torch.Generator().manual_seed(1)).to(dev)
    v_out = (torch.randn(cs.height, cs.width, Cn, generator=torch.Generator().manual_seed(2)) * 1e-6).to(dev)
    v_records = torch.zeros_like(records)
    fwd = lambda: raster.blend_extra_fwd(cs, bo, records, sorted_ids, tile_bins, out["final_T"], out["final_idx"], extra)  # noqa: E731
    bwd = lambda: raster.blend_extra_bwd(cs, bo, records, sorted_ids, tile_bins, out["final_T"], out["final_idx"], extra, v_out,  # noqa: E731
                                         v_records, deterministic=False)
    bwd_det = lambda: raster.blend_extra_bwd(cs, bo, records, sorted_ids, tile_bins, out["final_T"], out["final_idx"], extra,  # noqa: E731
                                             v_out, v_records, deterministic=True)
    return {"C": Cn, "gaussians": int(N), "intersections": int(M),
            "fwd_ms": events_median(fwd, reps, batch=5), "bwd_ms": events_median(bwd, reps, batch=5),
            "bwd_det_ms": events_median(bwd_det, reps, batch=5)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--cfg4-runs", type=int, default=2, help="runs per arm (off / on alternated); 0 skips config 4")
    ap.add_argument("--cfg4-steps", type=int, default=30)
    ap.add_argument("--cfg4-weight", type=float, default=0.1)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "semantic_timing measures the GPU"
    dev = torch.device("cuda", 0)
    res = {"card": card(), "reps": args.reps, "loss_fwd_bwd_ms": {}, "confusion_ms": {}}
    for Cn in (3, 19):
        loss_fb, confusion = loss_calls(1280, 1920, Cn, dev)
        res["loss_fwd_bwd_ms"][f"C{Cn}"] = events_median(loss_fb, args.reps)
        res["confusion_ms"][f"C{Cn}"] = events_median(confusion, args.reps)
    torch.cuda.empty_cache()
    res["blend_extra_cfg3"] = blend_extra_cfg3(args.reps, dev)
    torch.cuda.empty_cache()
    if args.cfg4_runs > 0:
        from train_cfg4 import run
        runs = {"off": [], "on": []}
        for _ in range(args.cfg4_runs):
            for arm, w in (("off", 0.0), ("on", args.cfg4_weight)):
                r = run(steps=args.cfg4_steps, warmup=5, semantic=w)
                runs[arm].append({"steps_per_s": r["value"], "ms_per_step": r["ms_per_step"], "wall_ms_per_step": r["wall_ms_per_step"]})
                torch.cuda.empty_cache()
        res["cfg4"] = {"weight": args.cfg4_weight, "steps": args.cfg4_steps, "runs": runs,
                       "median_steps_per_s": {k: float(np.median([x["steps_per_s"] for x in v])) for k, v in runs.items()}}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
