"""SSIM loss term at 1280 x 1920 (H x W): torch ``model.ssim`` forward + backward (as get_loss_dict calls it) against the
fused kernels (loss.fused_ssim_loss, csrc/ssim.cu), with and without a mask, alternated in one process.

Times are CUDA events around ``--iters`` forward + backward calls after a warm-up, ``--repeats`` alternations each.  A
separate torch.profiler pass gives per-kernel device times.  The algorithmic bytes and FMAs are computed from the shape
(no halo re-reads, no cache effects): the share of the H100 SXM data-sheet bound that binds (3.35 TB/s HBM3, 67 TFLOP/s
FP32, for a card allowed 700 W) over the measured kernel time.  Also timed: the add of the L1 and SSIM rgb cotangents,
which torch does when both terms reach rgb.  Prints one JSON line; ``--out FILE`` also writes it there."""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from street_gaussians_ns_b200.loss import fused_ssim_loss  # noqa: E402
from street_gaussians_ns_b200.model import ssim  # noqa: E402

HBM_BPS, FP32_FLOPS = 3.35e12, 67e12


def inputs(H, W, dev, with_mask):
    g = torch.Generator().manual_seed(0)
    gt = (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8)
    # rendered-like: a blurred version of the image plus noise
    blur = torch.nn.functional.avg_pool2d(gt.permute(2, 0, 1)[None].float() / 255, 5, 1, 2)[0].permute(1, 2, 0)
    rgb = (blur + 0.03 * torch.randn(H, W, 3, generator=g)).clamp(0, 1)
    mask = (torch.rand(H, W, 1, generator=g) > 0.1).float() if with_mask else None
    return gt.to(dev), rgb.to(dev).contiguous(), None if mask is None else mask.to(dev)


def torch_step(rgb, gt, mask, w):
    rgb.grad = None
    gt_img = gt.float() / 255.0
    y = rgb
    if mask is not None:
        gt_img, y = gt_img * mask, y * mask
    loss = w * (1 - ssim(gt_img.permute(2, 0, 1)[None, ...], y.permute(2, 0, 1)[None, ...]))
    loss.backward()


def fused_step(rgb, gt, mask, w):
    rgb.grad = None
    fused_ssim_loss(rgb, gt, mask=mask, weight=w).backward()


def events_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def model_counts(H, W, with_mask):
    """Algorithmic bytes and FMAs of the fused kernels (per call)."""
    P, V = H * W, (H - 10) * (W - 10)
    inp = P * (12 + 3 + (4 if with_mask else 0))  # rgb fp32, gt uint8, mask fp32
    maps = V * 36  # a, b, c per channel
    fwd_bytes, bwd_bytes = inp + maps, inp + maps + P * 12  # the backward also writes v_rgb
    # separable filter: 5 moments x 11 taps x 2 passes per output pixel and channel; backward: 3 maps x 11 x 2 per pixel
    fwd_fma, bwd_fma = 3 * V * (5 * 11 * 2), 3 * P * (3 * 11 * 2)
    return dict(fwd_bytes=fwd_bytes, bwd_bytes=bwd_bytes, fwd_fma=fwd_fma, bwd_fma=bwd_fma)


def bound(bytes_, fma, ms):
    t_mem, t_fp = bytes_ / HBM_BPS * 1e3, 2 * fma / FP32_FLOPS * 1e3
    which = "HBM bandwidth" if t_mem >= t_fp else "FP32 rate"
    return dict(bound=which, bound_ms=round(max(t_mem, t_fp), 4), share=round(max(t_mem, t_fp) / ms, 3) if ms > 0 else None,
                achieved_GBps=round(bytes_ / (ms * 1e-3) / 1e9, 1) if ms > 0 else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=1280)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--weight", type=float, default=0.2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda", 0)
    H, W = a.height, a.width
    props = torch.cuda.get_device_properties(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    res = dict(device=props.name, power_limit=power, H=H, W=W, weight=a.weight, iters=a.iters, repeats=a.repeats, cases={})
    for with_mask in (False, True):
        gt, rgb0, mask = inputs(H, W, dev, with_mask)
        rgb = rgb0.clone().requires_grad_(True)
        steps = {"torch": lambda: torch_step(rgb, gt, mask, a.weight), "fused": lambda: fused_step(rgb, gt, mask, a.weight)}
        for fn in steps.values():  # warm-up: module loads, allocator, cuDNN algorithm choice
            for _ in range(5):
                fn()
        torch.cuda.synchronize()
        times = defaultdict(list)
        for _ in range(a.repeats):
            for name, fn in steps.items():
                times[name].append(round(events_ms(fn, a.iters), 4))
        # per-kernel device times, in a pass of their own
        per = {}
        for name, fn in steps.items():
            acc = defaultdict(float)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    fn()
                torch.cuda.synchronize()
            for e in prof.events():
                if e.device_type == torch.autograd.DeviceType.CUDA:
                    acc[e.name.split("(")[0].replace("void ", "")[:80]] += (e.time_range.end - e.time_range.start) / 1e3 / 10
            per[name] = {k: round(v, 4) for k, v in sorted(acc.items(), key=lambda kv: -kv[1])}
            per[name + "_total_ms"] = round(sum(acc.values()), 4)
        cnt = model_counts(H, W, with_mask)
        kf = per["fused"].get("ssim_fwd_kernel", 0.0)
        kb = per["fused"].get("ssim_bwd_kernel", 0.0)
        res["cases"]["mask" if with_mask else "no_mask"] = dict(
            step_ms=dict(times), step_ms_median={k: sorted(v)[len(v) // 2] for k, v in times.items()},
            kernels=per, counts=cnt,
            fwd_kernel=bound(cnt["fwd_bytes"], cnt["fwd_fma"], kf), bwd_kernel=bound(cnt["bwd_bytes"], cnt["bwd_fma"], kb))
    # the add of two [H,W,3] fp32 cotangents (L1's and SSIM's) that autograd does before rgb's backward
    x, y = torch.rand(H, W, 3, device=dev), torch.rand(H, W, 3, device=dev)
    for _ in range(5):
        x + y
    add_ms = sorted(events_ms(lambda: x + y, a.iters) for _ in range(a.repeats))[a.repeats // 2]
    res["cotangent_add"] = dict(ms=round(add_ms, 4), bytes=H * W * 3 * 4 * 3, **bound(H * W * 3 * 4 * 3, 0, add_ms))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
