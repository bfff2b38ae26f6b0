"""One training iteration of the scene-graph model on the fused path (BASELINE.json configs 4 and 5).

What nerfstudio's ``Trainer.train_iteration`` plus the model's training callbacks do per step for the reference
(SURVEY.md 3.1): ``step_cb`` -> zero_grad -> ``get_outputs`` -> ``get_loss_dict`` -> backward -> optimizer step ->
``after_train`` (densification statistics, sgn_splatfacto.py:513-541) -> every ``refine_every`` steps ``refinement_after``
(:550-646).  nerfstudio's engine itself (config system, data managers, viewer, checkpoints) is out of scope; this is
the sequence of hot-path calls it makes, so that a step -- and a data-parallel step -- can be run, tested and timed.

Data parallel (SURVEY.md 8e): every replica holds all parameters and renders its own camera; the dense gradient
arena is summed with ONE all-reduce and divided by the world size, then every replica applies the same Adam update.
Replicas see different actors (different timestamps), so the arena has the layout of ALL sub-models
(``SceneGraphConfig.full_gradient_arena``) and Adam steps the UNION of the sub-models in view on any replica -- a
parameter that no replica rendered has no gradient and is skipped, as torch.optim.Adam skips ``grad is None``.  The
union is computed on the host from the cameras of all replicas (the camera assignment is deterministic,
``dp.camera_for_rank``): no extra collective.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist

from . import dp, mcmc
from .model import SceneGraphRasterModel, _FullArenaSink
from .optim import FusedAdam
from .scene import Camera


class TrainStep:
    def __init__(self, model: SceneGraphRasterModel, optimizer: FusedAdam, refine_every: Optional[int] = None,
                 group: Optional[dist.ProcessGroup] = None, pipeline_chunks: int = 0, refine_seed: int = 0,
                 check_replicas: bool = True, overlap: bool = False, exchange: str = "auto", metrics: bool = False,
                 gradient_accumulation_steps: Optional[Dict[str, int]] = None, filter_cameras: Optional[Sequence[Camera]] = None):
        """``pipeline_chunks`` > 0 (data parallel only): all-reduce and Adam are pipelined over that many ranges of the
        arena (dp.allreduce_and_step) instead of running one after the other.  ``metrics``: every step calls
        ``model.get_metrics_dict`` between ``get_outputs`` and ``get_loss_dict`` (nerfstudio's order,
        ``VanillaPipeline.get_train_loss_dict``) and keeps its result on ``self.metrics`` (device tensors, no read-back).
        ``gradient_accumulation_steps``: name of one of the optimizer's extra tensors -> n, nerfstudio's trainer rule (the
        reference sets ``{"camera_opt": 100}``, sgn_config.py:30): the tensor's gradient is zeroed at the steps where
        ``step % n == 0``, summed over the steps in between, and the tensor is stepped where ``step % n == n - 1``.  None (or a
        tensor not named): every step.  A per-row group of the optimizer (``FusedAdam(rows=...)``; the reference sets
        ``{"semantic": 10}``) follows the same rule per sub-model: a sub-model whose gradient is None at the due step is skipped,
        and one that a refinement rebuilt in the middle of a cycle starts over from a zero gradient -- the refinement replaces
        the Parameter, as nerfstudio's does, and the accumulated gradient goes with the old one.
        ``filter_cameras`` (a model with ``SceneGraphConfig.filter_3d``): the training cameras the 3D smoothing filter is
        computed from -- on the first step, right after every refinement that changed a row count, and every
        ``filter_3d_every`` steps otherwise (Mip-Splatting's schedule).  Under data parallelism every replica computes the same
        filter from the same full list, so nothing is exchanged."""
        self.model, self.optimizer, self.group = model, optimizer, group
        self.accumulate = dict(gradient_accumulation_steps or {})
        unknown = sorted(set(self.accumulate) - set(optimizer.extra_tensors()) - set(optimizer.row_tensors()))
        if unknown or any(int(n) < 1 for n in self.accumulate.values()):
            raise ValueError(f"gradient_accumulation_steps names tensors the optimizer does not step ({unknown}) or a count < 1: "
                             f"{self.accumulate}")
        self.want_metrics, self.metrics = metrics, None
        self.pipeline_chunks = pipeline_chunks if pipeline_chunks > 0 or not overlap else 4
        self.refine_seed, self.check_replicas, self._gen = refine_seed, check_replicas, None
        # how the gradient arena is exchanged: "sym" = this library's kernel over symmetric memory (csrc/collective.cu),
        # "nccl" = dist.all_reduce, "auto" = sym on NCCL process groups when the symmetric allocation succeeds
        self.exchange_mode, self._exchange = exchange, None
        # None: every sub-model on its own ``refine_every`` (the reference registers one callback per sub-model with
        # ``update_every_num_iters = config.refine_every``); a number: one cadence for all of them
        self.refine_every = refine_every
        self.filter_cameras = list(filter_cameras) if filter_cameras is not None else None
        if self.filter_cameras is not None and not model.config.filter_3d:
            raise ValueError("filter_cameras needs a model with SceneGraphConfig(filter_3d=True)")
        self._filter_step = None  # the step the filter was last computed at
        assert optimizer.num_segments == len(model.all_models), "build FusedAdam over model.optimizer_params()"

    def world_size(self) -> int:
        return dist.get_world_size(self.group) if (dist.is_available() and dist.is_initialized()) else 1

    def submodels_in_view(self, camera: Camera) -> List[int]:
        """Indices (all_models order) of the sub-models a render of ``camera`` lists: the background and every actor with
        a box at the camera's timestamp and at least one Gaussian (scene graph :332-352)."""
        m = self.model
        index = {n: i for i, n in enumerate(m.all_models._modules)}
        seen = [0]
        for pose in m.poses_at(camera.time):
            name = m.get_object_model_name(pose.track_id)
            if m.all_models[name].num_points > 0:
                seen.append(index[name])
        return seen

    def __call__(self, step: int, camera: Camera, batch: Dict[str, torch.Tensor],
                 all_cameras: Optional[Sequence[Camera]] = None) -> Dict[str, torch.Tensor]:
        """``all_cameras``: this step's cameras of ALL replicas (rank order), needed when the world size is > 1."""
        m, opt = self.model, self.optimizer
        world = self.world_size()
        full = isinstance(m._grad_sink, _FullArenaSink)
        if world > 1:
            assert full, "data parallel needs SceneGraphConfig(full_gradient_arena=True): replicas see different actors"
            assert all_cameras is not None and len(all_cameras) == world
        extras = opt.extra_tensors()                      # the optimizer's further groups (the sky cube map)
        if world > 1 and any(t.requires_grad for t in extras.values()):
            # refused before anything is rendered or exchanged: the gradient exchange covers the arena only
            raise NotImplementedError(f"data-parallel training does not exchange the gradients of {sorted(extras)}: the "
                                      "replicas would diverge")
        if world > 1 and (m.config.semantic_classes > 0 or opt.row_tensors()):
            raise NotImplementedError("data-parallel training does not exchange the gradients of the semantic logits: the "
                                      "replicas would diverge")
        if world > 1 and m.config.use_scale_regularization:
            # the term's gradient reaches background rows no replica saw, which the exchange leaves out, and every replica
            # would normalise by its own visible row count
            raise NotImplementedError("data-parallel training does not exchange the gradient of the scale regularisation: the "
                                      "replicas would diverge")
        if world > 1 and m.config.strategy == "mcmc":
            # the relocation and growth would be exchanged as densification statistics are, and the regularisers' gradients reach
            # rows no replica saw
            raise NotImplementedError("data-parallel training does not support strategy='mcmc': the replicas would diverge")
        if world > 1:
            self._ensure_exchange()
        m.step = step                                     # step_cb (sgn_splatfacto.py:754-755)
        if self.filter_cameras is not None and self._filter_step is None:
            self._update_filter(step)
        # accumulated tensors keep their gradient except where their cycle starts; they step where it ends
        keep = {id(extras[k]) for k, n in self.accumulate.items() if step % n != 0 and k in extras}
        rows = opt.row_tensors()
        keep |= {id(t) for k, n in self.accumulate.items() if step % n != 0 and k in rows for t in rows[k]}
        for p in m.parameters():                          # Optimizers.zero_grad_all()
            if id(p) not in keep:
                p.grad = None
        for t in extras.values():
            if id(t) not in keep:
                t.grad = None
        out = m.get_outputs(camera)
        if world > 1 and self._exchange is not None:  # which background rows this replica sees (rows nobody sees are not exchanged)
            h = m._holder
            n_bg = self._layout[1]
            if h is not None and h.radii is not None and h.radii.shape[0] >= n_bg and m.visible_model_names[:1] == ["background"]:
                self._exchange.publish_visible(h.radii, rows=n_bg)
            else:
                self._exchange.flags.zero_()
                self._exchange._union_fresh = False
                self._exchange._union_rows = n_bg
        if self.want_metrics:
            self.metrics = m.get_metrics_dict(out, batch)
        losses = m.get_loss_dict(out, batch)
        total = sum(losses.values())
        rendered = isinstance(total, torch.Tensor) and total.requires_grad
        kinds = None  # which of the six tensors of a sub-model have a gradient (None: all of them)
        if rendered:
            total.backward()
            h, sink = m._holder, getattr(m, "_grad_sink", None)
            # a loss term of the parameters themselves (the scale regularisation with fused_loss=False) sets .grad before the
            # render's backward runs: the render then adds its share into .grad through a temporary arena, and the arena the
            # optimizer reads is rebuilt from .grad
            outside = (sink is not None and getattr(h, "grad_sink", None) is sink and h.table is not None
                       and (h.grad_arena is None or h.grad_arena is not sink.arena) and any(p.grad is not None for p in sink.params))
            if outside:
                arena, got = sink.collect(h.table.static, m.device)
                kinds = None if len(got) == 6 else got
            elif h is not None and h.grad_arena is not None:
                arena = h.grad_arena
                if getattr(h, "params_only", False):  # only parameter terms reached the render (nothing in view): only their tensors step
                    kinds = list(h.term_kinds)
            # with nothing in view a loss term of another tensor (the camera regulariser) can still carry a gradient
            rendered = outside or (h is not None and h.grad_arena is not None)
        if not rendered:
            # nothing in view on this replica (the reference's early-out, sgn_splatfacto.py:878-886): no gradient here.
            # A single replica skips backward / optimizer / after_train only: the refinement callbacks still run
            # (nerfstudio fires them on the step count, whatever was rendered)
            if world == 1:
                # a loss term of a further tensor (the camera regulariser) may still have left a gradient: that tensor steps
                # on its own step count, as nerfstudio steps a group whatever was rendered
                due = self._due_extra_grads(step, extras)
                due_rows = self._due_row_grads(step)
                base = next(iter(due.values()), None)
                if base is None and due_rows:
                    base = next(g for gs in due_rows.values() for g in gs if g is not None)
                if base is not None:
                    opt.step(base, present=[], full_layout=True, extra_grads=due or None, row_grads=due_rows or None)
                self._maybe_refine(step)
                self._inject_noise(step)
                return losses
            arena = m.zero_gradient_arena()
        # the further tensors of the optimizer (the sky cube map, sky.CubeMapSky.base) step with the gradient autograd left
        extra_grads = self._due_extra_grads(step, extras)
        row_grads = self._due_row_grads(step)             # the per-row groups (the semantic logits), per sub-model
        if world > 1:
            present = sorted(set(i for cam in all_cameras for i in self.submodels_in_view(cam)))
        else:
            present = m.present_submodels()
        everything = len(present) == opt.num_segments and (full or present == list(range(opt.num_segments)))
        if world > 1 and self._exchange is not None:
            self._exchange_and_step(arena, None if everything else present, rendered)
        elif world > 1 and self.pipeline_chunks > 0:
            dp.allreduce_and_step(arena, opt, None if everything else present, self.pipeline_chunks, self.group)
        else:
            if world > 1:
                dp.allreduce_gradients(arena, average=True, group=self.group)
            kw = {"kinds": kinds} if kinds is not None else {}
            if row_grads:
                opt.step(arena, present=None if everything else present, full_layout=full, extra_grads=extra_grads or None,
                         row_grads=row_grads, **kw)
            else:
                opt.step(arena, present=None if everything else present, full_layout=full, extra_grads=extra_grads or None, **kw)
        # a frame with nothing in view (rendered only for the scale regularisation's gradient) has no densification statistics;
        # a count left on the device (async binning) is not read back for this
        M = getattr(m._holder, "M", None)
        if rendered and not (type(M) is int and M == 0):
            m.after_train(step)                           # AFTER_TRAIN_ITERATION callbacks, in the reference's order
        self._maybe_refine(step)
        self._inject_noise(step)
        return losses

    def _due_extra_grads(self, step: int, extras: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        """The gradients of the extra tensors that step at ``step``: every one that has a gradient, an accumulated one only at
        the end of its cycle (``step % n == n - 1``)."""
        return {name: t.grad for name, t in extras.items()
                if t.grad is not None and (name not in self.accumulate or step % self.accumulate[name] == self.accumulate[name] - 1)}

    def _due_row_grads(self, step: int) -> Dict[str, List[Optional[torch.Tensor]]]:
        """The per-row groups that step at ``step`` (every step, or at the end of their accumulation cycle): name -> the
        sub-models' gradients (None = skipped); groups without any gradient are left out."""
        out = {}
        for name, ts in self.optimizer.row_tensors().items():
            n = self.accumulate.get(name)
            if n is not None and step % n != n - 1:
                continue
            gs = [t.grad for t in ts]
            if any(g is not None for g in gs):
                out[name] = gs
        return out

    def _ensure_exchange(self) -> None:
        """(Re)allocates the symmetric gradient arena when the model's layout changed (first step, after a refinement).
        Collective: every replica reaches it at the same step with the same sizes."""
        if self.exchange_mode == "nccl" or dist.get_backend(self.group) != "nccl":
            return
        m = self.model
        sink = m._grad_sink
        sink.bind_model(m.optimizer_params(), [])
        total = sink.total_elems()
        n_bg = m.all_models["background"].num_points
        ex = self._exchange
        layout = (total, n_bg, tuple(int(x) for x in sink.sizes[:6]))
        if ex is not None and getattr(self, "_layout", None) == layout and sink.arena is not None and sink.arena.data_ptr() == ex.arena.data_ptr():
            return
        try:
            sink.exchange_plan = None
            if ex is None or total > ex.numel or n_bg > ex.flag_rows:
                # a symmetric allocation is a collective (allocation + handle exchange + barrier): allocate with headroom so
                # that refinements -- which grow the model by a few per cent at a time -- re-use it; the faster path
                # (multimem / peer) is timed once, later allocations reuse the decision
                self._exchange = None
                ex = dp.SymmetricExchange(int(total * 1.25), m.device, self.group, flag_rows=int(n_bg * 1.25) + 128,
                                          use_multicast=getattr(self, "_use_multicast", "auto"))
                self._use_multicast = bool(ex.multicast_ptr)
            ex.arena[:total].zero_()
            sink.set_arena(ex.arena[:total])
            self._exchange, self._layout = ex, layout
            # the background's six tensors are the first six slices of the full layout: K - 1 row ranges + "everything else"
            K = max(2, self.pipeline_chunks or 4)
            widths = [3, 3, 4, 3 * int(m.all_models["background"].gauss_params["features_dc"].shape[1]),
                      3 * int(m.all_models["background"].gauss_params["features_rest"].shape[1]), 1]
            offs = [int(sink.offsets[k]) for k in range(6)]
            bg_end = int(sink.offsets[5] + sink.sizes[5])
            self._ranges = dp.plan_ranges([n_bg], [offs], [widths], K - 1)  # row ranges of the background, with row descriptions
            self._tail = (bg_end, total - bg_end)
            sink.exchange_plan = self._plan
        except Exception as e:  # no peer access / no symmetric-memory support on this box: the NCCL path is the fallback
            if self.exchange_mode == "sym":
                raise
            self._exchange = None
            self.exchange_mode = "nccl"
            self.exchange_error = f"{type(e).__name__}: {e}"[:300]

    def _plan(self, table):
        """Called by the render's backward (raster._SceneGraphRasterize.backward) with the frame's segment table: the chunk
        ranges project_bwd runs in and the callback that starts range k's exchange as soon as its launch is enqueued."""
        ex = self._exchange
        bg_chunks = self._ranges[-1][1]
        ranges = [(a, b) for a, b, _ in self._ranges]
        slices = [sl for _, _, sl in self._ranges]
        if table.num_chunks > bg_chunks or self._tail[1] > 0:  # the actors' rows of this frame, and every sub-model behind the background
            ranges.append((bg_chunks, table.num_chunks))
            slices.append([self._tail] if self._tail[1] > 0 else [])
        self._planned = slices

        def after_range(k):
            ex.after_range(k, slices[k], average=True, skip_unseen=True)
        return ranges, after_range

    def _exchange_and_step(self, arena: torch.Tensor, present, rendered: bool) -> None:
        """Mean of the arena over the replicas with sgn_allreduce_sym -- range by range behind project_bwd when this replica
        rendered (the exchanges were started by the backward), all ranges here when it did not -- and the fused Adam of range
        k as soon as range k has been exchanged (while range k+1 is on the wire)."""
        ex, opt = self._exchange, self.optimizer
        assert arena.data_ptr() == ex.arena.data_ptr(), "the gradient arena is not the symmetric allocation"
        opt.step_count += 1
        tab = opt.step_table(present, full_layout=True)
        if rendered:
            slices = self._planned
        else:  # nothing in view here: an all-zero arena, exchanged in the same ranges as on the replicas that rendered
            slices = [sl for _, _, sl in self._ranges] + ([[self._tail]] if self._tail[1] > 0 else [])
            for k, sl in enumerate(slices):
                ex.after_range(k, sl, average=True, skip_unseen=True)
        for k, sl in enumerate(slices):
            ex.wait_range(k)
            opt.launch(opt.rows_in_slices(tab, sl), arena)

    def _refine_generator(self, step: int) -> torch.Generator:
        """Split samples must be identical on every replica whatever else consumed the global CUDA generator (a sky
        map, augmentation, a different number of randn calls per rank): a dedicated generator reseeded from
        (base seed, step) before each refinement."""
        if self._gen is None:
            self._gen = torch.Generator(device=self.model.device)
        self._gen.manual_seed((self.refine_seed * 1_000_003 + step) & 0x7FFFFFFFFFFFFFFF)
        return self._gen

    def _inject_noise(self, step: int) -> None:
        """MCMC's position noise, every step after the optimizer step and any refinement (gsplat's MCMCStrategy.step_post_backward),
        with the means' learning rate of this step."""
        if self.model.config.strategy == "mcmc":
            self.model.inject_noise(step, self.optimizer.lrs["means"], seed=self.refine_seed)

    def _maybe_refine(self, step: int) -> None:
        m = self.model
        mc = m.config.strategy == "mcmc"
        if self.refine_every is not None:
            due = self.refine_every > 0 and step % self.refine_every == 0
        elif mc:
            due = any(mcmc.due(st, step) for st in (m.config.mcmc, m.config.object_mcmc))
        else:
            due = any(st.refine_every > 0 and step % st.refine_every == 0 for st in (m.config.refine, m.config.object_refine))
        if not due:
            self._maybe_filter(step, False)
            return
        m.__dict__["refine_changed_rows"] = False
        if mc:
            m.refinement_after(self.optimizer, step, due_only=self.refine_every is None, seed=self.refine_seed)
        else:
            m.refinement_after(self.optimizer, step, generator=self._refine_generator(step), due_only=self.refine_every is None)
        self._maybe_filter(step, bool(m.__dict__.get("refine_changed_rows")))
        if self.world_size() > 1 and self.check_replicas:
            # replicas must have taken identical decisions: same row count in every sub-model
            rows = torch.tensor([sub.num_points for sub in m.all_models.values()], device=m.device, dtype=torch.int64)
            lo, hi = rows.clone(), rows.clone()
            dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=self.group)
            dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=self.group)
            assert torch.equal(lo, hi), "replicas diverged in a refinement (row counts differ)"


    def _maybe_filter(self, step: int, rows_changed: bool) -> None:
        """Mip-Splatting's schedule for the 3D filter: after a refinement that changed a row count, and every
        ``filter_3d_every`` steps."""
        if self.filter_cameras is None:
            return
        every = self.model.config.filter_3d_every
        if rows_changed or (every > 0 and step % every == 0 and self._filter_step != step):
            self._update_filter(step)

    def _update_filter(self, step: int) -> None:
        self.model.compute_filter_3d(self.filter_cameras)
        self._filter_step = step


def warm_up_refinement(model: SceneGraphRasterModel, rows: Sequence[int] = (65536, 10000, 10000), step: Optional[int] = None) -> Dict[str, object]:
    """Runs ONE refinement of a throwaway model (same configuration and tensor widths as ``model``, random rows and
    statistics that straddle every threshold, its own generator) and drops it.  Nothing of ``model`` is touched and no
    collective is issued.

    Why: CUDA loads a kernel's module at its first launch.  The first refinement of a process is the first launch of ~20
    kernels nothing else on the training step uses (the decide / apply kernels, scans, reductions, the normal sampler,
    bitwise and comparison kernels, ...), which cost tens of milliseconds of host time in the middle of training.  Calling this once after the
    model is built moves that one-time cost out of the loop, like the warm-up steps of a benchmark.  With ``strategy="mcmc"`` the
    refinement is the MCMC one (at its first due step unless ``step`` is given), followed by one position-noise launch."""
    from dataclasses import replace

    from .scene import GaussianSet
    dev = model.device
    subs = list(model.all_models.values())
    widths = [subs[0]] + [s for s in subs[1:]][:len(rows) - 1]
    g = torch.Generator(device=dev).manual_seed(12345)

    def rand(*shape):
        return torch.randn(shape, device=dev, generator=g)

    sets = []
    for n, like in zip(rows, widths):
        F, R = int(like.gauss_params["features_dc"].shape[1]), int(like.gauss_params["features_rest"].shape[1])
        sets.append(GaussianSet(rand(n, 3) * 5, rand(n, 3) * 1.5 - 4.0, rand(n, 4), rand(n, F, 3), rand(n, R, 3), rand(n, 1) * 2.5 - 1.0))
    mc = model.config.strategy == "mcmc"
    if mc:
        ms = model.config.mcmc
        step = step if step is not None else (ms.refine_start // ms.refine_every + 1) * ms.refine_every
    else:
        st = model.config.refine
        step = step if step is not None else st.warmup_length + st.refine_every * max(1, -(-(model.config.num_train_data + st.refine_every + 1) // st.refine_every))
    cfg = replace(model.config, full_gradient_arena=False, refine_record=True)
    tmp = SceneGraphRasterModel(sets[0], {str(i): s for i, s in enumerate(sets[1:])}, cfg).to(dev)
    tmp.train()
    tmp.step = step
    if mc:  # a few per cent of the random opacity logits are below logit(min_opacity): every kernel of both phases runs
        opt = FusedAdam(tmp.optimizer_params())
        tmp.refinement_after(opt, step, seed=12345)
        tmp.inject_noise(step, opt.lrs["means"], seed=12345)
        if dev.type == "cuda":
            torch.cuda.synchronize(dev)
        return {"step": step, "rows_before": [int(n) for n in rows[:len(sets)]],
                "rows_after": [s.num_points for s in tmp.all_models.values()],
                "records": [dict(s.refine_record_dict) for s in tmp.all_models.values()]}
    for sub in tmp.all_models.values():
        n, d = sub.num_points, sub.__dict__
        vis = torch.randint(1, 9, (n,), device=dev, generator=g).float()
        d["vis_counts"] = vis
        d["xys_grad_norm"] = torch.rand(n, device=dev, generator=g) * vis * 2.5e-6
        d["max_2Dsize"] = torch.rand(n, device=dev, generator=g) * 0.2
        d["last_size"] = (240, 320)
    opt = FusedAdam(tmp.optimizer_params())
    tmp.refinement_after(opt, step, generator=g, sync_stats=False)
    rowsum = torch.tensor([s.num_points for s in tmp.all_models.values()], device=dev, dtype=torch.int64)
    torch.equal(rowsum, rowsum.clone())  # the replica check of TrainStep._maybe_refine
    if dev.type == "cuda":
        torch.cuda.synchronize(dev)
    return {"step": step, "rows_before": [int(n) for n in rows[:len(sets)]], "rows_after": rowsum.tolist(),
            "records": [dict(s.refine_record_dict) for s in tmp.all_models.values()]}
