"""BASELINE.json configs 4 and 5 as a runnable loop: Waymo-shape synthetic scene (5 cameras x 85 frames, 1.68 M
background + 32 x 10 k actor Gaussians = 2 M), one training step = render one camera + L1 loss against a seeded target
+ Adam (+ densification statistics every step, refinement every ``--refine-every`` steps); with torchrun and N ranks
(config 5) rank r renders camera (step * N + r) mod 425, the gradient arena is all-reduced and averaged, every rank
applies the same update (SURVEY.md 8d / 8e).

    python tools/train_cfg4.py --steps 50                                                   # config 4, one GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 4 --master-addr 127.0.0.1 \\
        --master-port 29511 tools/train_cfg4.py --steps 50                                  # config 5

Prints one JSON line (rank 0): training steps/s over all ranks (weak scaling: one camera per rank per step), the
device time per step (CUDA events, max over ranks), Gaussian counts before / after, the losses of the first and last
step.  bench.py's headline stays config 3 (the metric BASELINE.json quotes); this is the tool for configs 4 / 5.
Actors are boxes parked on the road grid of SURVEY.md 8d; an actor has a box in a frame only while the ego vehicle is
within ``--actor-range`` metres of it, so the set of sub-models in view changes from frame to frame."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(steps: int = 50, warmup: int = 5, scale: float = 1.0, refine_every: int = 100, start_step: int = 600,
        actor_range: float = 45.0, pipeline_chunks: int = 0, overlap: bool = False, resident_table: bool = True,
        async_binning: bool = True, ssim_lambda: float = 0.0, fused_loss: bool = True, sky: bool = False, metrics: bool = False,
        bbox_opt: bool = False, camera_opt: bool = False, sky_view_grad: bool = False, lidar_depth: float = 0.0,
        semantic: float = 0.0, antialiased: bool = False, scale_reg: bool = False, filter_3d: bool = False,
        bilateral_grid: bool = False, mcmc: bool = False, absgrad: bool = False, visible_adam: bool = False) -> dict:
    """One measurement.  torch.distributed must already be initialised when WORLD_SIZE > 1.  Returns the result dict on
    rank 0 (None elsewhere).  ``sky``: the reference's default learnable sky (use_sky_sphere, a 1024^2 cube map stepped by
    the same Adam launch at the ``sky_sphere`` group's lr 0.005, sgn_config.py:72-75).  ``metrics``: every step also computes
    ``get_metrics_dict`` (psnr, gaussian_count, scale / opacity / radii means), as nerfstudio's training pipeline does.
    ``bbox_opt``: the reference's default box corrections (``bbox_optimizer`` mode "simple": delta_center / delta_yaw per
    (frame, box), stepped by the same Adam launch at the ``bbox_opt`` group's lr 1e-3, sgn_config.py:80-83).
    ``camera_opt``: trainable camera poses (``camera_optimizer`` mode "SO3xR3" over the indexed rig cameras, the ``camera_opt``
    group's lr 1e-3 and its 100-step gradient accumulation, sgn_config.py:30,76-79).  ``sky_view_grad`` (with ``sky`` and
    ``camera_opt``): the sky also gives the camera rotation its gradient (CubeMapSky(view_grad=True)).  ``lidar_depth`` > 0: the
    lidar depth term at that weight (SceneGraphConfig.depth_loss_mult), against a synthetic sweep per step
    (``synthetic.street_points(170_000, seed=step)``, about one top-lidar sweep, all drawn onto the device before the first step)
    ``semantic`` > 0: per-Gaussian semantic logits with 3 classes (the reference's SemanticType) and the cross-entropy term at
    that weight (SceneGraphConfig.semantic_loss_mult), against synthetic labels drawn onto the device before timing; the logits
    are the FusedAdam row group "semantic" at features_dc's lr 0.0025 (a choice: the reference config names no rate) with
    the reference's gradient accumulation of 10
    projected with the step's camera.  ``antialiased``: rasterize_mode "antialiased" (the opacity scaled by the blur
    compensation, forward and backward).  ``scale_reg``: nerfstudio's scale regularisation (use_scale_regularization,
    max_gauss_ratio 10, every tenth step); the result then reports the fraction of rows whose max / min scale ratio is above
    10 before and after the run.  ``filter_3d``: Mip-Splatting's 3D smoothing filter from the 425 rig cameras (SceneGraphConfig
    .filter_3d), recomputed after every refinement that changed a row count and every 100 steps.  ``bilateral_grid``: one
    bilateral grid per rig image (425, bilagrid.BilateralGrid with gsplat's 16 x 16 x 8) corrects every training render, with
    the grids' total-variation term; stepped by the same Adam launch at gsplat's lr 2e-3.  ``mcmc``: densification by MCMC
    (SceneGraphConfig(strategy="mcmc"), gsplat's defaults with the actors' 100 k cap): no densification statistics, relocation
    and 5 % growth at every refinement, position noise every step, the opacity and scale regularisers in the loss.  ``absgrad``:
    the split / duplicate decision reads the absolute screen-space gradient (SceneGraphConfig(absgrad=True)).  ``visible_adam``:
    the selective Adam step (TrainStep(visible_adam=True)): only the rows the step's camera saw are stepped."""
    import torch
    import torch.distributed as dist

    if sky_view_grad and not (sky and camera_opt):
        raise ValueError("sky_view_grad needs sky and camera_opt")
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200 import dp
    from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.refine import RefineSettings
    from street_gaussians_ns_b200.training import TrainStep

    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)

    sc = syn.WaymoScene(scale=scale, actor_range=actor_range)
    W, H, num_frames, cams = sc.width, sc.height, sc.num_frames, sc.cameras
    frame_list = list(range(num_frames))

    def poses_at(t):  # fresh objects per call, as a data manager hands them out
        f = int(t)
        return [ActorPose(str(a), rot, center, f, frame_list, frame_id=f) for a, rot, center in sc.boxes_at(f)]

    rs = RefineSettings(refine_every=refine_every)
    cfg = SceneGraphConfig(use_sky_sphere=sky, ssim_lambda=ssim_lambda, fused_loss=fused_loss, full_gradient_arena=world > 1, refine=rs, async_binning=async_binning,
                           object_refine=RefineSettings(refine_every=refine_every, cull_alpha_thresh=0.005),
                           num_train_data=len(cams), refine_record=True, depth_loss_mult=lidar_depth,
                           semantic_classes=3 if semantic > 0 else 0, semantic_loss_mult=semantic,
                           rasterize_mode="antialiased" if antialiased else "classic", use_scale_regularization=scale_reg,
                           filter_3d=filter_3d, strategy="mcmc" if mcmc else "default", absgrad=absgrad)
    env_map = None
    if sky:
        from street_gaussians_ns_b200.sky import CubeMapSky
        env_map = CubeMapSky(1024, view_grad=sky_view_grad)
    boxes = None
    if bbox_opt:
        from street_gaussians_ns_b200.box_pose import BoxPoseOptimizer
        boxes = BoxPoseOptimizer(num_frames, [str(k) for k in sc.actors], {f: f for f in range(num_frames)}, mode="simple")
    cam_opt = None
    if camera_opt or bilateral_grid:  # both look a training image up by its index
        for i, c in enumerate(cams):
            c.index = i
    if camera_opt:
        from street_gaussians_ns_b200.camera_pose import CameraPoseOptimizer
        cam_opt = CameraPoseOptimizer(len(cams))
    bil = None
    if bilateral_grid:
        from street_gaussians_ns_b200.bilagrid import BilateralGrid
        bil = BilateralGrid(len(cams))
    model = SceneGraphRasterModel(sc.background.to(dev), {k: v.to(dev) for k, v in sc.actors.items()}, cfg, poses_at=poses_at,
                                  sky=env_map, bbox_optimizer=boxes, camera_optimizer=cam_opt, bilateral_grid=bil).to(dev)
    model.train()
    extra = {"sky": (model.env_map.base, 0.005)} if sky else {}
    if bbox_opt:
        extra["bbox_opt.delta_center"] = (boxes.delta_center, 1e-3)
        extra["bbox_opt.delta_yaw"] = (boxes.delta_yaw, 1e-3)
    accumulate = None
    if camera_opt:
        extra["camera_opt.pose_adjustment"] = (cam_opt.pose_adjustment, 1e-3)
        accumulate = {"camera_opt.pose_adjustment": 100}
    if bilateral_grid:
        extra["bilateral_grid.grids"] = (bil.grids, 2e-3)
    rows = None
    if semantic > 0:
        rows = {"semantic": (model.semantic_params(), 0.0025)}
        accumulate = dict(accumulate or {}, semantic=10)
    opt = FusedAdam(model.optimizer_params(), extra=extra, reserve_spare=True, rows=rows)  # no cudaMalloc of moment arenas inside the training loop
    step_fn = TrainStep(model, opt, refine_every=refine_every, pipeline_chunks=pipeline_chunks, overlap=overlap, metrics=metrics,
                        gradient_accumulation_steps=accumulate, filter_cameras=cams if filter_3d else None, visible_adam=visible_adam)
    g = torch.Generator().manual_seed(5)
    gt = (torch.rand(H, W, 3, generator=g) * 255).to(torch.uint8).to(dev)  # get_loss_dict consumes uint8 directly
    counts0 = [sub.num_points for sub in model.all_models.values()]

    def needle_fraction():  # rows whose max / min scale ratio is above max_gauss_ratio, over every sub-model
        with torch.no_grad():
            s = torch.exp(torch.cat([sub.gauss_params["scales"] for sub in model.all_models.values()]))
            return float(((s.amax(-1) / s.amin(-1)) > cfg.max_gauss_ratio).float().mean())
    needles0 = needle_fraction()
    times = [float(f) for f in range(num_frames)]
    if resident_table:
        model.prepare_frames(times)
    if world > 1:
        # NCCL sets up its channels lazily, at the first collective of a size class: the statistics exchange of the first
        # refinement would otherwise pay that one-time cost (tens of ms) inside the timed steps
        warm = torch.zeros(1 << 22, device=dev)
        dist.all_reduce(warm, op=dist.ReduceOp.SUM)
        dist.all_reduce(warm, op=dist.ReduceOp.MAX)
        small = torch.zeros(64, device=dev, dtype=torch.int64)
        dist.all_reduce(small, op=dist.ReduceOp.MIN)
        dist.all_reduce(small, op=dist.ReduceOp.MAX)
        del warm, small
    # CUDA loads a kernel's module at its first launch: the first refinement of a process would pay for ~20 kernels nothing else
    # on the step uses (tens of ms of host time).  One refinement of a throwaway model loads them; best effort, process-local
    try:
        from street_gaussians_ns_b200.training import warm_up_refinement
        info = warm_up_refinement(model)
        refine_warm = {"ok": True, "rows_before": info["rows_before"], "rows_after": info["rows_after"]}
    except Exception as e:  # the measurement is still valid without it (the first refinement then includes the module loads)
        refine_warm = {"ok": False, "error": f"{type(e).__name__}: {e}"[:200]}
    if async_binning:
        # without the per-frame read-back of the intersection count the list buffers have a capacity learnt from earlier frames:
        # look at every rig camera at three points of the drive once (no gradients) so that the capacity covers the widest view
        from street_gaussians_ns_b200 import raster
        model.config.async_binning = False
        with torch.no_grad():
            for f in (0, num_frames // 2, num_frames - 1):
                for c in range(5):
                    model.get_outputs(cams[f * 5 + c])
                    raster.async_learn(dev, int(model._holder.M))
        model.config.async_binning = True
        torch.cuda.synchronize()

    # one sweep per step, drawn before the timed steps as a data loader would have prefetched them
    sweeps = [syn.street_points(170_000, seed=start_step + i).to(dev) for i in range(warmup + steps)] if lidar_depth > 0 else []
    # synthetic segmentations (classes 0..2 and 5 % ignored pixels), drawn before the timed steps
    gl = torch.Generator().manual_seed(6)
    labels = []
    for _ in range(4 if semantic > 0 else 0):
        lab = torch.randint(0, 3, (H, W, 1), generator=gl)
        lab[torch.rand(H, W, 1, generator=gl) < 0.05] = 255
        labels.append(lab.to(dev))

    def one(i):
        step = start_step + i
        mine = [cams[dp.camera_for_rank(step, r, world, len(cams))] for r in range(world)]
        # after a refinement replaced parameter tensors the model drops the resident table; a timestamp's rows are then
        # re-staged (and kept on the device) the first time it is rendered again
        batch = {"image": gt}
        if lidar_depth > 0:
            batch["lidar_points"] = sweeps[i % len(sweeps)]
        if semantic > 0:
            batch["semantic"] = labels[i % len(labels)]
        return step_fn(step, mine[rank], batch, all_cameras=mine if world > 1 else None)

    def sync():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    first = None
    for i in range(warmup):
        losses = one(i)
        first = first if first is not None else float(sum(v.detach() for v in losses.values()))
    sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    marks = [torch.cuda.Event(enable_timing=True) for _ in range(steps)]  # per-step device time: where a refinement's cost lands
    host_ms = []
    profile_refine = os.environ.get("SGN_PROFILE_REFINE") == "1" and rank == 0
    t0 = time.perf_counter()
    e0.record()
    for i in range(steps):
        h0 = time.perf_counter()
        if profile_refine and refine_every > 0 and (start_step + warmup + i) % refine_every == 0:
            import cProfile
            import pstats
            prof = cProfile.Profile()
            prof.enable()
            losses = one(warmup + i)
            torch.cuda.synchronize()
            prof.disable()
            pstats.Stats(prof, stream=sys.stderr).sort_stats("cumulative").print_stats(45)
        else:
            losses = one(warmup + i)
        marks[i].record()
        host_ms.append((time.perf_counter() - h0) * 1e3)
    e1.record()
    sync()
    step_ms = [round((e0 if i == 0 else marks[i - 1]).elapsed_time(marks[i]), 3) for i in range(steps)]
    wall_ms = (time.perf_counter() - t0) * 1e3 / steps
    dev_ms = torch.tensor([e0.elapsed_time(e1) / steps, wall_ms], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(dev_ms, op=dist.ReduceOp.MAX)
    last = float(sum(v.detach() for v in losses.values()))
    replicas_identical = None
    if world > 1:
        try:  # every replica must hold bit-identical parameters after the run: same exchange result, same Adam, same refinements
            chk = torch.stack([p.detach().double().sum() for p in model.all_models["background"].gauss_params.values()])
            lo, hi = chk.clone(), chk.clone()
            dist.all_reduce(lo, op=dist.ReduceOp.MIN)
            dist.all_reduce(hi, op=dist.ReduceOp.MAX)
            replicas_identical = bool(torch.equal(lo, hi))
        except Exception:
            replicas_identical = None
    if rank != 0:
        return None
    counts1 = [sub.num_points for sub in model.all_models.values()]
    ms = float(dev_ms[0].item())
    return {
        "metric": f"training steps/s (render 1 camera per rank + L1{' + SSIM' if ssim_lambda > 0 else ''} + backward + gradient all-reduce + fused Adam + densification "
                  f"statistics, refinement every {refine_every} steps; timed steps {start_step + warmup}..{start_step + warmup + steps - 1})", "value": world / (ms * 1e-3), "unit": "steps/s",
        "n_gpus": world, "steps": steps, "warmup": warmup, "ms_per_step": ms, "wall_ms_per_step": float(dev_ms[1].item()),
        "higher_is_better": True, "scaling": "weak", "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"cfg{4 if world == 1 else 5}: 5 cameras x 85 frames, {sc.n_bg} background + 32 x {sc.n_act} actor Gaussians, "
                               f"{W}x{H}; rank r renders camera (step*g + r) mod 425; actors have a box within {actor_range} m of the ego vehicle",
                   "parallelism": f"camera-sharded dp{world}", "ssim_lambda": ssim_lambda,
                   **({"sky": "CubeMapSky(1024), Adam lr 0.005"} if sky else {}),
                   **({"bbox_opt": "BoxPoseOptimizer(simple), Adam lr 1e-3"} if bbox_opt else {}),
                   **({"camera_opt": "CameraPoseOptimizer(SO3xR3), Adam lr 1e-3, gradient accumulation 100"} if camera_opt else {}),
                   **({"sky_view_grad": "the sky's rotation cotangent reaches the camera"} if sky_view_grad else {}),
                   **({"lidar_depth": f"depth_loss_mult {lidar_depth}, street_points(170_000, seed=step) per step"} if lidar_depth > 0 else {}),
                   **({"semantic": f"3 classes, semantic_loss_mult {semantic}, Adam lr 0.0025, gradient accumulation 10, synthetic labels"}
                      if semantic > 0 else {}),
                   **({"rasterize_mode": "antialiased"} if antialiased else {}),
                   **({"scale_reg": "use_scale_regularization, max_gauss_ratio 10, every tenth step"} if scale_reg else {}),
                   **({"filter_3d": "Mip-Splatting 3D filter from the 425 rig cameras, variance 0.2, recomputed every 100 steps "
                                    "and after refinements"} if filter_3d else {}),
                   **({"bilateral_grid": "BilateralGrid(425, 16 x 16 x 8), 10 * total variation, Adam lr 2e-3"} if bilateral_grid else {}),
                   **({"strategy": "mcmc: relocation + 5 % growth per refinement (caps 1 M / 100 k), noise every step, "
                                   "opacity and scale regularisers 0.01"} if mcmc else {}),
                   **({"absgrad": "split / duplicate on the absolute screen-space gradient, densify_absgrad_thresh 0.0008"}
                      if absgrad else {}),
                   **({"visible_adam": "selective Adam: only the rows with radius > 0 in the step's frame are stepped"} if visible_adam else {}),
                   "loss": "fused kernels" if fused_loss else "torch ops", "metrics": "get_metrics_dict every step" if metrics else "none",
                   "start_step": start_step, "refine_every": refine_every,
                   "refinement_kernels_loaded_before_timing": refine_warm,
                   "binning": "no host read-back of the intersection count" if async_binning else "one read-back per frame",
                   "segment_table": "device-resident (staged up front; re-staged per timestamp on first use after a refinement)" if resident_table else "host build per frame",
                   "collective": ("all-reduce(AVG) of the gradient arena (layout of all sub-models), "
                                  + ("overlapped with project_bwd / Adam over arena ranges" if overlap else
                                     (f"pipelined with Adam over {pipeline_chunks} ranges" if pipeline_chunks else "serial"))) if world > 1 else "none"},
        "gaussians_before": int(sum(counts0)), "gaussians_after": int(sum(counts1)),
        "submodels_changed": int(sum(a != b for a, b in zip(counts0, counts1))),
        "loss_first": first, "loss_last": last, "replicas_identical": replicas_identical,
        "ratio_above_10_before": needles0, "ratio_above_10_after": needle_fraction(),
        **({"metrics_last": {k: (v if isinstance(v, int) else float(v)) for k, v in step_fn.metrics.items()}} if metrics else {}),
        "step_ms_rank0": step_ms, "host_ms_rank0": [round(x, 3) for x in host_ms]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0, help="shrinks Gaussian counts and the image (smoke runs)")
    ap.add_argument("--refine-every", type=int, default=100)
    ap.add_argument("--start-step", type=int, default=600, help="past warmup_length so that refinement is live")
    ap.add_argument("--actor-range", type=float, default=45.0)
    ap.add_argument("--pipeline-chunks", type=int, default=0, help="> 0: all-reduce and Adam pipelined over that many arena ranges")
    ap.add_argument("--overlap", action="store_true", help="all-reduce launched per arena range from project_bwd's ranges (dp.OverlappedStep)")
    ap.add_argument("--host-table", action="store_true", help="build the segment table on the host per frame instead of prepare_frames")
    ap.add_argument("--ssim-lambda", type=float, default=0.0, help="weight of the SSIM term (the reference trains with 0.2)")
    ap.add_argument("--torch-loss", action="store_true", help="loss terms as torch ops (SceneGraphConfig.fused_loss = False)")
    ap.add_argument("--sky", action="store_true", help="train the learnable sky cube map (the reference's use_sky_sphere = True)")
    ap.add_argument("--metrics", action="store_true", help="get_metrics_dict every step, between get_outputs and get_loss_dict")
    ap.add_argument("--bbox-opt", action="store_true", help="train the box corrections (the reference's bbox_optimizer mode 'simple')")
    ap.add_argument("--camera-opt", action="store_true", help="train the camera poses (camera_optimizer mode 'SO3xR3', accumulation 100)")
    ap.add_argument("--sky-view-grad", action="store_true", help="with --sky --camera-opt: the sky also trains the camera rotation")
    ap.add_argument("--lidar-depth", type=float, default=0.0, metavar="W",
                    help="> 0: the lidar depth term at weight W against a synthetic 170 k-point sweep per step")
    ap.add_argument("--semantic", type=float, default=0.0, metavar="W",
                    help="> 0: 3-class semantic logits and the cross-entropy term at weight W against synthetic labels")
    ap.add_argument("--antialiased", action="store_true", help="rasterize_mode 'antialiased': opacities scaled by the blur compensation")
    ap.add_argument("--scale-reg", action="store_true", help="nerfstudio's scale regularisation (max_gauss_ratio 10, every tenth step)")
    ap.add_argument("--filter-3d", action="store_true", help="Mip-Splatting's 3D smoothing filter from the 5 x 85 rig cameras")
    ap.add_argument("--bilateral-grid", action="store_true", help="a bilateral grid per rig image (425) corrects each training render")
    ap.add_argument("--mcmc", action="store_true", help="densification by MCMC (SceneGraphConfig(strategy='mcmc'))")
    ap.add_argument("--absgrad", action="store_true", help="densify on absolute screen-space gradients (SceneGraphConfig(absgrad=True))")
    ap.add_argument("--visible-adam", action="store_true", help="selective Adam: step only the Gaussians the step's camera saw")
    args = ap.parse_args()
    if args.sky_view_grad and not (args.sky and args.camera_opt):
        ap.error("--sky-view-grad needs --sky and --camera-opt")

    import torch
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "needs a CUDA device (no CPU path)"
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    res = run(args.steps, args.warmup, args.scale, args.refine_every, args.start_step, args.actor_range, args.pipeline_chunks,
              args.overlap, not args.host_table, ssim_lambda=args.ssim_lambda, fused_loss=not args.torch_loss, sky=args.sky,
              metrics=args.metrics, bbox_opt=args.bbox_opt, camera_opt=args.camera_opt,
              sky_view_grad=args.sky_view_grad, lidar_depth=args.lidar_depth, semantic=args.semantic, antialiased=args.antialiased,
              scale_reg=args.scale_reg, filter_3d=args.filter_3d, bilateral_grid=args.bilateral_grid, mcmc=args.mcmc,
              absgrad=args.absgrad, visible_adam=args.visible_adam)
    if res is not None:
        print(json.dumps(res))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
