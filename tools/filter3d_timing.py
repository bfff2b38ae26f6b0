"""Times Mip-Splatting's 3D smoothing filter (SceneGraphConfig.filter_3d) on one GPU, with CUDA events:

  * compute_filter_3d at config 4 (2 M rows x the 425 rig views), host table build included;
  * sgn_project_fwd / sgn_project_bwd at config 3 with and without the filter, alternated call by call;
  * config-4 training steps/s with and without the filter (tools/train_cfg4.py; the filter run includes its recompute every
    100 steps and after the refinement).

Prints one JSON line."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    import numpy as np
    import torch

    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200 import raster
    from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
    from street_gaussians_ns_b200.scene import Frame, Segment
    import train_cfg4

    dev = torch.device("cuda", 0)
    res = {"gpu": torch.cuda.get_device_name(0)}

    sc = syn.WaymoScene(scale=1.0)

    def poses_at(t):
        f = int(t)
        return [ActorPose(str(a), rot, center, f, list(range(sc.num_frames))) for a, rot, center in sc.boxes_at(f)]
    m = SceneGraphRasterModel(sc.background.to(dev), {k: v.to(dev) for k, v in sc.actors.items()}, SceneGraphConfig(filter_3d=True),
                              poses_at=poses_at)
    m.compute_filter_3d(sc.cameras)
    ms = []
    for _ in range(10):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        m.compute_filter_3d(sc.cameras)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    res["filter_cfg4_ms"] = {"median": float(np.median(ms)), "min": float(min(ms)), "max": float(max(ms)), "runs": len(ms)}
    del m

    fr = syn.config_frame(3)
    frc = Frame(fr.camera, [Segment(s.params.to("cuda"), s.cls, s.rot, s.center, s.idft, s.name) for s in fr.segments])
    rng = np.random.default_rng(0)
    frf = Frame(fr.camera, [Segment(s.params, s.cls, s.rot, s.center, s.idft, s.name,
                                    filter_3d=torch.tensor(rng.uniform(1e-3, 0.03, s.params.num_points), dtype=torch.float32, device=dev))
                            for s in frc.segments])
    cs = raster.camera_struct(fr.camera, raster.RenderSettings())
    tabs = {k: raster.SegmentTable(f, [s.params.tensors() for s in f.segments], dev) for k, f in (("off", frc), ("on", frf))}
    params = [s.params.tensors() for s in frc.segments]
    v = {}
    for k, t in tabs.items():
        p = raster.project_fwd(t, cs, dev)
        v[k] = (p, torch.randn_like(p.records) * (p.radii > 0)[:, None])
    times = {f"{k}_{w}": [] for k in tabs for w in ("fwd", "bwd")}
    out = torch.empty(sum(raster.arena_layout(tabs["off"].static)[0]), device=dev)
    for it in range(60):
        for k, t in tabs.items():
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            p = raster.project_fwd(t, cs, dev)
            e[1].record()
            raster.project_bwd(t, params, cs, p.records, p.radii, v[k][1], make_views=False, out=out)
            e[2].record()
            torch.cuda.synchronize()
            if it >= 10:
                times[f"{k}_fwd"].append(e[0].elapsed_time(e[1]))
                times[f"{k}_bwd"].append(e[1].elapsed_time(e[2]))
    res["project_cfg3_ms"] = {k: {"median": float(np.median(x)), "min": float(min(x)), "max": float(max(x))} for k, x in times.items()}
    del tabs, v, frc, frf
    torch.cuda.empty_cache()

    steps = int(os.environ.get("FILTER3D_TIMING_STEPS", "200"))
    for name, on in (("off", False), ("on", True)):
        r = train_cfg4.run(steps=steps, warmup=5, start_step=595, filter_3d=on)
        res[f"cfg4_{name}"] = {"steps_per_s": r["value"], "ms_per_step": r["ms_per_step"], "gaussians_after": r["gaussians_after"],
                               "step_ms_max": max(r["step_ms_rank0"])}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
