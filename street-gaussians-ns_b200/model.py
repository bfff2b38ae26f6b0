"""Level-2 drop-in surface: the nerfstudio ``Model`` methods of the reference's scene-graph model
that sit on the hot path, re-hosted on the fused rasterizer.

Mirrors ``SplatfactoSceneGraphModel`` (street_gaussians_ns/sgn_splatfacto_scene_graph.py:41-401) and the
parts of ``SplatfactoModel`` it inherits (street_gaussians_ns/sgn_splatfacto.py:793-1001, :1042-1094):

  * ``all_models`` ModuleDict: "background", "object_<id>" ... each holding the six ``gauss_params``
    (names/shapes unchanged, so reference checkpoints load: ``all_models.<name>.gauss_params.<p>``);
  * ``get_outputs(camera)`` -> {"rgb","accumulation","depth","sky","object_acc","background_acc"
    (+ "background_rgb","object_rgb" in eval)} with the reference's early-outs;
  * side-effect attributes ``xys`` (with ``.grad`` = pixel-space mean gradient after backward),
    ``depths, radii, conics, num_tiles_hit, last_size`` on the model and split per sub-model
    (``SplatfactoModel.after_train`` reads ``self.xys.grad`` and ``self.radii``, :513-541);
  * ``get_loss_dict`` (L1 + SSIM + sky accumulation + object-accumulation entropy, + the lidar depth term when
    ``depth_loss_mult > 0``, + the bilateral grids' total variation with a ``bilateral_grid``);
  * ``get_metrics_dict`` (per-step psnr, Gaussian count, scale / opacity / radii means: one reduction kernel),
    ``get_image_metrics_and_images`` and ``get_outputs_for_camera`` (eval).

nerfstudio is not a dependency here: ``camera`` is any object with the fields of
``street_gaussians_ns_b200.scene.Camera`` (SURVEY.md 8b lists what the path reads from ``Cameras``).
"""
from __future__ import annotations

import itertools
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from . import mcmc, raster, refine
from .mcmc import MCMCSettings
from .refine import RefineSettings
from .scene import PARAM_NAMES, CLS_BACKGROUND, CLS_OBJECT, Camera, Frame, GaussianSet, Segment, fourier_time, idft_basis


@dataclass
class ActorPose:
    """What the path needs from a reference ``Box`` (data/utils/dynamic_annotation.py): trackId,
    center, rot, frame; plus the actor's frame list for the Fourier time (scene graph :239-245).  ``frame_id``: the integer
    timestamp of the box's annotated frame (``Box.frame_id``), which names its row of the box corrections
    (box_pose.BoxPoseOptimizer); None -- the default -- for a box that is not corrected."""

    track_id: str
    rot: np.ndarray
    center: np.ndarray
    frame: int
    frame_list: Sequence[int]
    frame_id: Optional[int] = None


@dataclass
class SceneGraphConfig:
    sh_degree: int = 3
    sh_degree_interval: int = 1000
    block_width: int = 16
    fourier_features_dim: int = 5
    fourier_features_scale: float = 1.0
    use_sky_sphere: bool = True
    ssim_lambda: float = 0.2
    sky_acc_loss_mult: float = 1.0
    object_acc_entropy_loss_mult: float = 0.001
    alpha_clamp_fwd: float = 0.999
    alpha_clamp_bwd: float = 0.99
    render_background_acc: bool = True
    fused_loss: bool = True  # L1 / sky / entropy and SSIM terms through the loss kernels (loss.py) instead of torch ops
    # weight of the lidar depth term (depth.py): w * mean |depth - target| over the pixels with a return; 0 = off
    depth_loss_mult: float = 0.0
    # per-Gaussian semantic logits (semantic.py): classes per Gaussian, 0 = none (3 for the reference's SemanticType: DEFAULT,
    # GROUND, SKY); with classes the render publishes outputs["semantic"] [H,W,C]
    semantic_classes: int = 0
    # weight of the semantic cross-entropy term against batch["semantic"]; 0 = off
    semantic_loss_mult: float = 0.0
    # refinement (sgn_splatfacto.py:550-646): the sub-model configs of sgn_config.py:46-66 (background / object template)
    refine: RefineSettings = field(default_factory=lambda: RefineSettings(cull_alpha_thresh=0.02))
    object_refine: RefineSettings = field(default_factory=lambda: RefineSettings(cull_alpha_thresh=0.005))
    num_train_data: int = 0      # Model.num_train_data: refinement waits until every image was seen after an opacity reset (:563-566)
    refine_record: bool = False  # fill sub.refine_record_dict (the reference's logging counters; one extra read-back per sub-model)
    # data parallel (SURVEY 8e): gradients are delivered in an arena that has the layout of ALL sub-models (the
    # optimizer's), so that replicas which see different actors can sum their arenas with one all-reduce
    full_gradient_arena: bool = False
    # no host read-back of the intersection count inside get_outputs (raster.RenderSettings.async_binning); None -> SGN_ASYNC_BIN
    async_binning: Optional[bool] = None
    # the reference's rasterize_mode (sgn_splatfacto.py:214-223): "classic", or "antialiased" -- every render blends
    # sigmoid(opacity) * comp, the EWA blur's compensation (raster.RenderSettings.rasterize_mode).  The reference leaves the
    # multiply commented out, so its "antialiased" renders like "classic"; here the mode does what its docstring says.  The
    # refinement's opacity cull / reset and the metrics keep reading sigmoid(opacity), as the reference's do
    rasterize_mode: str = "classic"
    # nerfstudio's scale regularisation (PhysGaussian), which the reference's config turns on (use_scale_regularization = True,
    # max_gauss_ratio = 10, sgn_splatfacto.py:206-211) and its loss never computes: every tenth step, losses["scale_reg"] =
    # 0.1 * mean(max(amax(exp(scales)) / amin(exp(scales)), max_gauss_ratio) - max_gauss_ratio) over the visible rows.  Off here
    # by default; the 0.1 weight and the 10-step cadence are nerfstudio's constants
    use_scale_regularization: bool = False
    max_gauss_ratio: float = 10.0
    # Mip-Splatting's 3D smoothing filter (filter3d.py): every Gaussian is rendered convolved with an isotropic 3D Gaussian whose
    # size comes from the highest rate at which a training camera sampled it, sigma = sqrt(filter_3d_variance) / max(f / z),
    # over the views where z > filter_3d_near and the projection is inside the image with a 15 % margin.  The sizes are a
    # per-sub-model buffer (``filter_3d``, in the state dict only with the filter on) that ``compute_filter_3d`` fills;
    # TrainStep(filter_cameras=...) recomputes it after every refinement that changed a row count and every filter_3d_every
    # steps.  The refinement, densification statistics, metrics and scale regularisation keep reading the raw parameters
    filter_3d: bool = False
    filter_3d_variance: float = 0.2
    filter_3d_near: float = 0.2
    filter_3d_every: int = 100
    # densification strategy: "default" is the reference's split / duplicate / cull / opacity reset (refine, object_refine);
    # "mcmc" is gsplat's MCMCStrategy (mcmc.py): dead rows relocated onto live ones, growth by 5 % per refinement up to a
    # per-sub-model cap, position noise every step (TrainStep), and two regularisers in the loss, every training step:
    # mcmc_opacity_reg = mcmc_opacity_reg * mean(sigmoid(opacities)), mcmc_scale_reg = mcmc_scale_reg * mean(exp(scales)), over the
    # visible sub-models' rows (gsplat averages over all rows).  The weights are those of gsplat's MCMC preset.  The actors' cap of
    # 100 000 is a placeholder that no measurement backs: set it from the actors' sizes in the data
    strategy: str = "default"
    mcmc: MCMCSettings = field(default_factory=MCMCSettings)
    object_mcmc: MCMCSettings = field(default_factory=lambda: MCMCSettings(cap_max=100_000))
    mcmc_opacity_reg: float = 0.01
    mcmc_scale_reg: float = 0.01

    # ``stop_split_at`` of the BACKGROUND sub-model: what the reference's entropy gate reads
    # (``config.background_model.stop_split_at``, scene graph :386).  One source: ``refine.stop_split_at``.
    @property
    def stop_split_at(self) -> int:
        return self.refine.stop_split_at

    @stop_split_at.setter
    def stop_split_at(self, v: int) -> None:
        self.refine.stop_split_at = int(v)


_MISSING = object()


class _FrameSlice:
    """A per-frame side-effect attribute of a sub-model (``xys``, ``depths``, ``radii``, ``conics``, ``num_tiles_hit``;
    sgn_splatfacto.py:513-541 reads them): this sub-model's rows of the frame's arrays, sliced on first access.  Publishing
    them eagerly costs 5 slices x 33 sub-models of host time per frame, and nothing on the hot path reads them (the
    densification statistics work on the frame's arrays directly)."""

    def __init__(self, name: str):
        self.name = name

    def __get__(self, obj, cls=None):
        if obj is None:
            return self
        d = obj.__dict__
        cache = d.get("_fs_cache")
        if cache is not None:
            v = cache.get(self.name, _MISSING)
            if v is not _MISSING:
                return v
        src = d.get("_fs_src")
        if src is None:
            return None
        holder, sl = src
        t = getattr(holder, self.name)[sl]
        if self.name == "xys" and holder.v_records is not None:  # after backward: the reference reads ``self.xys.grad``
            t.grad = holder.v_records[:, 0:2][sl]
        if cache is None:
            cache = d["_fs_cache"] = {}
        cache[self.name] = t
        return t

    def __set__(self, obj, value):
        cache = obj.__dict__.get("_fs_cache")
        if cache is None:
            cache = obj.__dict__["_fs_cache"] = {}
        cache[self.name] = value


class GaussianSubModel(torch.nn.Module):
    """One entry of ``all_models``: the ``gauss_params`` ParameterDict (sgn_splatfacto.py:291-300)."""

    xys = _FrameSlice("xys")
    depths = _FrameSlice("depths")
    radii = _FrameSlice("radii")
    conics = _FrameSlice("conics")
    num_tiles_hit = _FrameSlice("num_tiles_hit")

    def __init__(self, params: GaussianSet, semantic_classes: int = 0, filter_3d: bool = False):
        super().__init__()
        self.gauss_params = torch.nn.ParameterDict(
            {k: torch.nn.Parameter(getattr(params, k).detach().clone()) for k in
             ("means", "scales", "quats", "features_dc", "features_rest", "opacities")})
        # per-Gaussian class logits [n, C], zeros at the start.  Kept outside gauss_params: the six-tensor paths (gradient arena,
        # FusedAdam's six tensors per sub-model, sgn_refine_apply, the data-parallel layout) never see it.  Its gradient comes
        # through autograd (render_frame's ``extra``); the optimizer steps it as the row group "semantic"
        if semantic_classes > 0:
            self.semantic_logits = torch.nn.Parameter(torch.zeros(params.means.shape[0], int(semantic_classes),
                                                                  device=params.means.device, dtype=torch.float32))
        else:
            self.semantic_logits = None
        # the 3D smoothing filter's per-row sizes [n] (SceneGraphConfig.filter_3d): a buffer, so it is saved with the model;
        # zeros (no smoothing) until SceneGraphRasterModel.compute_filter_3d fills it
        if filter_3d:
            self.register_buffer("filter_3d", torch.zeros(params.means.shape[0], device=params.means.device, dtype=torch.float32))
        else:
            self.filter_3d = None
        self.xys = self.depths = self.radii = self.conics = self.num_tiles_hit = None
        self.last_size = None
        # densification statistics (sgn_splatfacto.py:513-541), created by the first after_train
        self.xys_grad_norm = self.vis_counts = self.max_2Dsize = None
        self.refine_record_dict: dict = {}

    @property
    def num_points(self) -> int:
        return int(self.gauss_params["means"].shape[0])

    def as_set(self) -> GaussianSet:
        g = self.gauss_params
        return GaussianSet(g["means"], g["scales"], g["quats"], g["features_dc"], g["features_rest"], g["opacities"])

    def load_state_dict(self, state_dict, **kwargs):  # type: ignore[override]
        """Checkpoints hold whatever number of Gaussians refinement had reached: resize the parameters to the
        checkpoint's row count before loading, and accept the pre-ParameterDict key names
        (sgn_splatfacto.py:425-438)."""
        state_dict = dict(state_dict)
        if "means" in state_dict:
            for k in PARAM_NAMES:
                state_dict[f"gauss_params.{k}"] = state_dict.pop(k)
        if "gauss_params.means" in state_dict:
            rows = state_dict["gauss_params.means"].shape[0]
            for k in PARAM_NAMES:
                old = self.gauss_params[k]
                want = state_dict.get(f"gauss_params.{k}")
                shape = (rows,) + (tuple(want.shape[1:]) if want is not None else tuple(old.shape[1:]))
                if tuple(old.shape) != shape:
                    self.gauss_params[k] = torch.nn.Parameter(torch.zeros(shape, device=old.device, dtype=old.dtype))
            sem = self.semantic_logits
            want = state_dict.get("semantic_logits")
            if sem is not None and want is not None and tuple(sem.shape) != tuple(want.shape):
                self.semantic_logits = torch.nn.Parameter(torch.zeros(tuple(want.shape), device=sem.device, dtype=sem.dtype))
            f3 = self.filter_3d
            want = state_dict.get("filter_3d")
            if f3 is not None and want is not None and tuple(f3.shape) != tuple(want.shape):
                self.filter_3d = torch.zeros(tuple(want.shape), device=f3.device, dtype=f3.dtype)
            d = self.__dict__
            d["xys_grad_norm"] = d["vis_counts"] = d["max_2Dsize"] = None  # statistics of the old rows are meaningless
        return super().load_state_dict(state_dict, **kwargs)


class _GradSink:
    """Delivers the rasterizer's flat gradient arena to the model's ~200 parameter tensors.

    torch.autograd with one leaf per parameter tensor costs ~1.5 ms of host time per step here (198
    AccumulateGrad nodes + 198 views), more than half of the GPU time of the whole step.  Instead the
    render has ONE differentiable input (an anchor), and after backward the sink points every
    ``param.grad`` at its slice of a persistent arena that project_bwd overwrites in place.
    Semantics match autograd's: a parameter whose ``.grad`` is None (after ``zero_grad()``) gets the new
    gradient; if any gradient is still set (no zero_grad between backward calls) the new one is ADDED."""

    def __init__(self):
        self.key = None
        self.arena = None
        self.views: List[torch.Tensor] = []
        self.params: List[torch.Tensor] = []

    def bind(self, params: List[torch.Tensor]):
        key = tuple(map(id, params))
        if key != self.key:
            self.key, self.params, self.arena, self.views = key, list(params), None, []

    allocator = None  # optional callable(total, device) -> float32 tensor: where the persistent arena lives (data parallel: a
    #                   symmetric allocation the exchange kernel can address on every replica)

    def _ensure_arena(self, static: dict, device) -> None:
        sizes, _, _ = raster.arena_layout(static)
        total = sum(sizes)
        if self.arena is None or self.arena.numel() != total or self.arena.device != device:
            self.arena = self.allocator(total, device) if self.allocator is not None else torch.empty(total, device=device, dtype=torch.float32)
            assert self.arena.numel() == total and self.arena.dtype == torch.float32
            self.views = raster.arena_views(self.arena, static)

    def collect(self, static: dict, device) -> tuple:
        """The persistent arena made to hold every bound parameter's ``.grad`` (which then points at its slice), for a fused
        optimizer that reads the arena: needed after a backward in which a gradient reached the parameters outside the render
        (a torch loss term of the parameters themselves), so that ``.grad`` was set before the render's backward ran and the
        render added its share through a temporary arena.  A parameter without a gradient gets a zero slice.  Returns (arena,
        the PARAM_NAMES positions that have a gradient in some bound parameter)."""
        self._ensure_arena(static, device)
        kinds = set()
        for i, (p, v) in enumerate(zip(self.params, self.views)):
            if p.grad is None:
                v.zero_()
                continue
            kinds.add(i % 6)
            if p.grad.data_ptr() != v.data_ptr():
                v.copy_(p.grad)
                p.grad = v
        return self.arena, sorted(kinds)

    def target(self, static: dict, device):
        self._ensure_arena(static, device)
        for p in self.params:
            if p.grad is not None:
                return None  # accumulate: render into a temporary arena, add in publish()
        return self.arena

    def grad_offsets(self, static: dict):
        """Where project_bwd puts the frame's slices inside ``target()``'s arena: None = back to back (the frame's layout)."""
        return None

    def publish(self, arena: torch.Tensor, static: dict):
        if arena is self.arena:
            for p, v in zip(self.params, self.views):
                p.grad = v
            return
        for p, v, pv in zip(self.params, raster.arena_views(arena, static), self.views):
            if p.grad is None:
                pv.copy_(v)
                p.grad = pv
            else:
                p.grad.add_(v)


class _FullArenaSink(_GradSink):
    """Data-parallel form of the sink: the persistent arena has the layout of ALL sub-models (the optimizer's layout,
    ``FusedAdam(model.optimizer_params())``), whatever subset is in view.  Replicas render different cameras at
    different timestamps and therefore see different sets of actors; only with a common layout can ONE all-reduce sum
    their gradients.  The slices of sub-models that are not in this replica's frame are zeroed (their sum over the
    replicas is then the other replicas' gradient), the frame's slices are written in place by project_bwd through
    per-tensor offsets."""

    def __init__(self):
        super().__init__()
        self.model_key = None
        self.sizes = self.offsets = None   # per tensor of the whole model (floats, padded to 4)
        self.present: List[int] = []
        self.all_views: List[torch.Tensor] = []
        self.all_shapes: List[tuple] = []

    def bind_model(self, all_params: List[List[torch.Tensor]], present: List[int]):
        key = tuple((id(t), t.shape[0]) for ps in all_params for t in ps)  # ids can be recycled after a refinement
        if key != self.model_key:
            flat = [t for ps in all_params for t in ps]
            self.model_key, self.arena, self.all_views = key, None, []
            self.all_shapes = [tuple(t.shape) for t in flat]
            self.sizes = np.array([(t.numel() + 3) // 4 * 4 for t in flat], np.int64)
            self.offsets = np.concatenate([[0], np.cumsum(self.sizes)[:-1]]).astype(np.int64)
        self.present = list(present)
        self.params = [t for i in self.present for t in all_params[i]]
        self.key = tuple(map(id, self.params))

    def _tensor_ids(self):
        return [6 * i + k for i in self.present for k in range(6)]

    def grad_offsets(self, static: dict):
        return self.offsets[self._tensor_ids()]

    def total_elems(self) -> int:
        return int(self.sizes.sum())

    def set_arena(self, arena: torch.Tensor) -> None:
        """Install the arena the gradients are delivered in (data parallel: a view of a symmetric allocation, so that the
        exchange kernel of csrc/collective.cu can address every replica's copy)."""
        assert arena.dtype == torch.float32 and arena.is_contiguous() and arena.numel() == self.total_elems()
        self.arena = arena
        chunks = arena.split_with_sizes([int(x) for x in self.sizes])
        self.all_views = [c[:int(np.prod(shp))].view(shp) for c, shp in zip(chunks, self.all_shapes)]

    def _ensure_arena(self, static: dict, device) -> None:
        total = int(self.sizes.sum())
        if self.arena is None or self.arena.numel() != total or self.arena.device != device:
            self.set_arena(torch.zeros(total, device=device, dtype=torch.float32))
        self.views = [self.all_views[t] for t in self._tensor_ids()]

    def collect(self, static: dict, device) -> tuple:
        arena, kinds = super().collect(static, device)
        self._zero_absent()
        return arena, kinds

    def target(self, static: dict, device):
        self._ensure_arena(static, device)
        for p in self.params:
            if p.grad is not None:
                return None  # accumulate: render into a temporary arena (frame layout), add in publish()
        self._zero_absent()
        return self.arena

    def _zero_absent(self) -> None:
        # zero the sub-models that are not in this frame (runs of absent sub-models are contiguous in the arena);
        # after an all-reduce they hold the other replicas' gradients
        nsub = len(self.sizes) // 6
        here = set(self.present)
        i = 0
        while i < nsub:
            if i in here:
                i += 1
                continue
            j = i
            while j < nsub and j not in here:
                j += 1
            lo = int(self.offsets[6 * i])
            hi = int(self.offsets[6 * (j - 1) + 5] + self.sizes[6 * (j - 1) + 5])
            self.arena[lo:hi].zero_()
            i = j


_MODEL_SERIAL = itertools.count()


class SceneGraphRasterModel(torch.nn.Module):
    def __init__(self, background: GaussianSet, actors: Dict[str, GaussianSet], config: Optional[SceneGraphConfig] = None,
                 poses_at: Optional[Callable[[float], List[ActorPose]]] = None,
                 sky: Optional[Callable[[Camera, bool], torch.Tensor]] = None, bbox_optimizer: Optional[torch.nn.Module] = None,
                 camera_optimizer: Optional[torch.nn.Module] = None, bilateral_grid: Optional[torch.nn.Module] = None):
        super().__init__()
        self.config = config or SceneGraphConfig()
        raster.rasterize_mode_flag(self.config.rasterize_mode)  # an unknown mode raises ValueError, as the reference's does
        if self.config.strategy not in ("default", "mcmc"):
            raise ValueError(f"unknown densification strategy {self.config.strategy!r}: expected 'default' or 'mcmc'")
        # trainable camera poses (camera_pose.CameraPoseOptimizer, nerfstudio's attribute name).  None, or one in mode "off":
        # every camera is rendered as given, by the same calls as without it
        if camera_optimizer is not None and camera_optimizer.mode != "off" and sky is not None:
            from .sky import CubeMapSky
            if not isinstance(sky, CubeMapSky):
                raise TypeError("a camera optimizer needs the sky to be a sky.CubeMapSky: the corrected view lives on the device, "
                                f"and {type(sky).__name__} cannot take it")
        self.camera_optimizer = camera_optimizer
        # trainable corrections of the actor boxes (box_pose.BoxPoseOptimizer; the reference's attribute name, scene graph
        # :91).  None, or one in mode "off": the boxes are rendered as annotated, by the same calls as without it
        self.bbox_optimizer = bbox_optimizer
        # per-image appearance correction (bilagrid.BilateralGrid, one grid per training image; gsplat's use_bilateral_grid).
        # None: every image is rendered and trained by the same calls as without it
        self.bilateral_grid = bilateral_grid
        self.all_models = torch.nn.ModuleDict()
        C = int(self.config.semantic_classes)
        f3 = bool(self.config.filter_3d)
        self.all_models["background"] = GaussianSubModel(background, C, f3)
        for obj_id, ps in actors.items():
            self.all_models[self.get_object_model_name(obj_id)] = GaussianSubModel(ps, C, f3)
        self.poses_at = poses_at or (lambda t: [])
        # the learnable sky (EnvLight, sgn_splatfacto.py:109-150): sky.CubeMapSky on this library's kernels, or any callable
        # (camera, train) -> [H, W, 3] such as the reference's EnvLight on nvdiffrast
        self.env_map = sky
        self.step = 0
        self.visible_model_names: List[str] = ["background"]
        self.xys = self.depths = self.radii = self.conics = self.num_tiles_hit = None
        self.last_size = None
        self._holder = None
        self._last_camera = None
        self._frame_cache: dict = {}
        self.__dict__["_serial"] = next(_MODEL_SERIAL)  # names this model in raster's static segment-table cache (ids are recycled)
        self._grad_sink = _FullArenaSink() if self.config.full_gradient_arena else _GradSink()
        self._anchor = None
        self._noise_table = mcmc.NoiseTable()
        # eval's LPIPS (torchmetrics LearnedPerceptualImagePatchSimilarity(normalize=True), sgn_splatfacto.py:331): its AlexNet
        # weights are not part of this library; an integration that has them sets a callable (gt, rgb) -> score here
        self.lpips = None

    @classmethod
    def from_points(cls, background=None, actors: Optional[Dict[str, tuple]] = None, config: Optional[SceneGraphConfig] = None,
                    generator: Optional[torch.Generator] = None, replay_scene_graph_init: bool = True, device=None,
                    cameras: Optional[Sequence[Camera]] = None, **model_kwargs) -> "SceneGraphRasterModel":
        """A model initialised from seed points, as ``SplatfactoSceneGraphModel.populate_modules`` builds its sub-models
        (sgn_splatfacto_scene_graph.py:49-96, each one by ``SplatfactoModel.populate_modules``, see populate.py).

        ``background``: ``(xyz, rgb)`` -- COLMAP / lidar ``points3D``, rgb uint8 or float 0..255 -- with ``fourier_dim`` 1, or
        None for the reference's random initialisation of 50 000 points in a cube of side 10.  ``actors``: ``{track_id:
        (xyz, rgb)}``, one aggregated lidar cloud per tracked actor, with ``config.fourier_features_dim``, in the given order.
        Every sub-model uses ``config.sh_degree``.  The initial scales come from the GPU nearest-neighbour search (knn.py).

        ``cameras`` (a sequence of scene.Camera): with ``config.filter_3d``, the 3D smoothing filter is computed from them once
        the model is built (``compute_filter_3d``).

        Draws come from ``generator`` (default: torch's default CPU generator) in the reference's order.  With
        ``replay_scene_graph_init`` (the default) the draws of the scene graph's own random initialisation, which the reference
        makes and discards before the background (:50-52), are consumed first, so that after ``torch.manual_seed(s)`` the
        sub-models equal those of the reference's populate_modules seeded with ``s``.  Draws the reference makes outside
        populate_modules' initialisation (e.g. by modules its trainer builds in between) are not replayed.  ``device``: where
        the parameters live (default: the current CUDA device).  ``model_kwargs`` go to the constructor (poses_at, sky, ...).
        """
        from . import populate
        config = config or SceneGraphConfig()
        if replay_scene_graph_init:
            populate.replay_scene_graph_init(generator)
        if background is None:
            bg = populate.random_gaussians(50000, 10.0, config.sh_degree, 1, generator=generator, device=device)
        else:
            bg = populate.gaussians_from_points(*background, sh_degree=config.sh_degree, fourier_dim=1, generator=generator,
                                                device=device)
        acts = {tid: populate.gaussians_from_points(xyz, rgb, sh_degree=config.sh_degree, fourier_dim=config.fourier_features_dim,
                                                    generator=generator, device=device)
                for tid, (xyz, rgb) in (actors or {}).items()}
        model = cls(bg, acts, config=config, **model_kwargs)
        if cameras is not None and config.filter_3d:
            model.compute_filter_3d(cameras)
        return model

    @staticmethod
    def get_object_model_name(object_id) -> str:
        return f"object_{object_id}"

    def load_state_dict(self, state_dict, **kwargs):  # type: ignore[override]
        """``SplatfactoSceneGraphModel.load_state_dict`` (scene graph :393-401): every sub-model takes the keys under
        ``all_models.<name>.`` (and resizes itself to the checkpoint's row count), the rest loads non-strictly."""
        state_dict = dict(state_dict)
        for name, sub in self.all_models.items():
            prefix = f"all_models.{name}."
            own = {k[len(prefix):]: state_dict.pop(k) for k in list(state_dict) if k.startswith(prefix)}
            if own:
                sub.load_state_dict(own, **kwargs)
        self.invalidate_frames()
        return torch.nn.Module.load_state_dict(self, state_dict, strict=False)

    @property
    def device(self):
        return self.all_models["background"].gauss_params["means"].device

    def _apply(self, fn, *args, **kwargs):  # .to() / .cuda() / .float(): parameter storage moves, staged pointers are stale
        out = super()._apply(fn, *args, **kwargs)
        if "_frame_cache" in self.__dict__:
            self.invalidate_frames()
        return out

    # ------------------------------------------------------------------------------------------
    @staticmethod
    def _pose_digest(poses) -> tuple:
        """Content key of a timestamp's boxes: an integration may move boxes at a fixed timestamp (the reference's
        ``bbox_optimizer.apply_to_bbox`` rewrites them every training step) or hand out fresh objects whose ``id`` CPython
        recycles -- identity says nothing, the bytes do."""
        return tuple((p.track_id, p.frame, len(p.frame_list), p.frame_list[0], p.frame_list[-1],
                      np.asarray(p.rot, np.float64).tobytes(), np.asarray(p.center, np.float64).tobytes()) for p in poses)

    def _frame(self, camera: Camera) -> Frame:
        """The Frame of ``camera``.  The segment rows of a timestamp (poses, IDFT bases, parameter pointers, row offsets) are
        static data while the parameter tensors stay the same objects and the boxes keep their values: they are kept per
        timestamp -- device-resident when ``prepare_frames`` built them up front -- and validated by content."""
        poses = self.poses_at(camera.time)
        digest = self._pose_digest(poses)
        hit = self._frame_cache.get(camera.time)
        if hit is not None and hit["digest"] == digest and hit["ptr0"] == self.all_models._modules["background"].gauss_params._parameters["means"].data_ptr():
            self.visible_model_names = hit["names"]
            frame = Frame(camera, hit["segments"])
            frame._prebuilt, frame._table_slot, frame._actor_poses = hit["table"], hit, hit["actor_poses"]
            frame._static_key = ("model", self.__dict__["_serial"], self.__dict__.get("_param_epoch", 0), tuple(hit["names"]), str(self.device))
            return frame
        frame = self._build_frame(camera, poses)
        frame._table_slot = self._remember_frame(camera.time, digest, frame, None)
        return frame

    def compute_filter_3d(self, cameras: Sequence[Camera]) -> int:
        """Mip-Splatting's 3D filter sizes from the training ``cameras`` (filter3d.py, one sweep of every row against every
        view on the device): fills every sub-model's ``filter_3d`` buffer in place, resizing the ones whose row count changed.
        Each camera's view is its ``c2w`` as given, actors are placed by ``poses_at(camera.time)`` (box corrections are not
        applied).  Returns the number of rows some view samples (also kept as ``filter_3d_sampled``); when it is 0, no view
        sees any Gaussian and every sigma is 0."""
        from . import filter3d
        c = self.config
        if not c.filter_3d:
            raise ValueError("the model was built without the 3D filter (SceneGraphConfig.filter_3d = False)")
        resized = False
        for sub in self.all_models._modules.values():
            n = sub.num_points
            if sub.filter_3d is None or sub.filter_3d.shape[0] != n or sub.filter_3d.device != self.device:
                sub.filter_3d = torch.zeros(n, device=self.device, dtype=torch.float32)
                resized = True
        if resized:  # the frames' segments hold the old buffers
            self.invalidate_frames()
        n = filter3d.compute(self, list(cameras), c.filter_3d_variance, c.filter_3d_near)
        self.filter_3d_sampled = n
        if n == 0:
            import warnings
            warnings.warn("compute_filter_3d: no camera samples any Gaussian; every filter size is 0")
        return n

    def _filter_of(self, name: str) -> Optional[torch.Tensor]:
        """The sub-model's 3D filter sizes for a frame's segment (None with the filter off)."""
        if not self.config.filter_3d:
            return None
        sub = self.all_models._modules[name]
        f = sub.filter_3d
        if f is None or f.shape[0] != sub.num_points:
            raise RuntimeError(f"the 3D filter of {name} has {None if f is None else f.shape[0]} rows, the sub-model "
                               f"{sub.num_points}: call compute_filter_3d after changing the rows (TrainStep(filter_cameras=...) "
                               "does it after every refinement)")
        return f

    def invalidate_frames(self) -> None:
        """Drop the per-timestamp segment rows (call after replacing parameter tensors by hand; ``refinement_after`` and
        ``load_state_dict`` do it themselves)."""
        self._frame_cache.clear()
        self.__dict__.pop("_frame_table_blob", None)
        self.__dict__["_param_epoch"] = self.__dict__.get("_param_epoch", 0) + 1
        self.__dict__["_sets"] = {}

    def _remember_frame(self, time, digest, frame: Frame, table):
        if len(self._frame_cache) > 4096:
            self._frame_cache.clear()
        slot = self._frame_cache[time] = dict(
            digest=digest, segments=frame.segments, names=list(self.visible_model_names), table=table,
            actor_poses=frame._actor_poses,
            ptr0=self.all_models._modules["background"].gauss_params._parameters["means"].data_ptr())
        return slot

    def prepare_frames(self, times: Sequence[float]) -> int:
        """SURVEY.md 8f rank 4: the segment table of EVERY (timestamp, actor) -- object->world rotation / translation /
        quaternion (``object2world_gs``, scene graph :404-417), IDFT basis (:420-433), Fourier time (:239-245), parameter
        pointers and row offsets -- built once from the annotation table (``poses_at``; for the reference's
        ``InterpolatedAnnotation`` that includes slerp-interpolated boxes with ``frame = -1``,
        dynamic_annotation.py:157-171,252-286) and uploaded with ONE copy.  ``get_outputs`` then indexes it by timestamp: no
        per-frame host build, no per-frame H2D.  Rebuilt by the caller after a refinement replaced parameter tensors
        (the cache is dropped there).  Returns the bytes resident on the device."""
        dev = self.device
        built = []
        for t in times:
            poses = self.poses_at(t)
            frame = self._build_frame(None, poses)
            params = [list(seg.params.tensors()) for seg in frame.segments]
            tab = raster.SegmentTable(frame, params, dev, upload=False)
            built.append((t, self._pose_digest(poses), frame, tab))
        if not built:
            return 0
        blob = np.concatenate([tab.host.view(np.uint8).reshape(-1) for _, _, _, tab in built])
        resident = torch.from_numpy(blob).to(dev)
        off = 0
        for t, digest, frame, tab in built:
            nbytes = tab.host.nbytes
            tab.dev = resident[off:off + nbytes]
            off += nbytes
            self.visible_model_names = [seg.name for seg in frame.segments]
            self._remember_frame(t, digest, frame, tab)
        self.__dict__["_frame_table_blob"] = resident
        return int(resident.numel())

    def _set_of(self, name: str) -> GaussianSet:
        sets = self.__dict__.setdefault("_sets", {})
        g = sets.get(name)
        if g is None:
            g = sets[name] = self.all_models._modules[name].as_set()
        return g

    def _build_frame(self, camera: Camera, poses) -> Frame:
        segs = [Segment(self._set_of("background"), CLS_BACKGROUND, name="background", filter_3d=self._filter_of("background"))]
        names = ["background"]
        kept = []
        for pose in poses:
            name = self.get_object_model_name(pose.track_id)
            assert name not in names
            ps = self._set_of(name)
            if ps.means.shape[0] == 0:  # "prevent empty object" (scene graph :337-338)
                continue
            basis = None
            F = ps.features_dc.shape[1]
            if F > 1:
                t = fourier_time(pose.frame, pose.frame_list, self.config.fourier_features_scale)
                basis = idft_basis(t, F)
            segs.append(Segment(ps, CLS_OBJECT, rot=pose.rot, center=pose.center, idft=basis, name=name, filter_3d=self._filter_of(name)))
            names.append(name)
            kept.append(pose)
        self.visible_model_names = names
        frame = Frame(camera, segs)
        frame._actor_poses = kept
        frame._static_key = ("model", self.__dict__["_serial"], self.__dict__.get("_param_epoch", 0), tuple(names), str(self.device))
        return frame

    def _settings(self, class_streams: bool) -> raster.RenderSettings:
        c = self.config
        n = min(self.step // c.sh_degree_interval, c.sh_degree) if self.training else c.sh_degree
        return raster.RenderSettings(sh_degree=c.sh_degree, sh_degree_to_use=n, block_width=c.block_width,
                                     alpha_clamp_fwd=c.alpha_clamp_fwd, alpha_clamp_bwd=c.alpha_clamp_bwd,
                                     class_streams=class_streams, training=self.training, async_binning=c.async_binning,
                                     rasterize_mode=c.rasterize_mode)

    def _box_poses(self, frame: Frame) -> Optional[torch.Tensor]:
        """The corrected poses of the frame's actors, [actors, 16], from ``bbox_optimizer`` -- in training and in eval alike,
        as the reference applies the correction whenever the box has an annotated frame (scene graph :340-341).  The
        annotated poses and parameter rows of a timestamp are staged on the device once and kept with its segment rows."""
        bo = self.bbox_optimizer
        boxes = frame._actor_poses
        if bo is None or bo.mode == "off" or not boxes:
            return None
        slot = getattr(frame, "_table_slot", None)
        staged = slot.get("box_stage") if slot is not None else None
        if staged is None:
            fi, bi = bo.indices(boxes)
            staged = bo.stage(fi, bi, [b.rot for b in boxes], [b.center for b in boxes], device=self.device)
            if slot is not None:
                slot["box_stage"] = staged
        return bo(staged)

    def _camera_view(self, camera: Camera) -> Optional[torch.Tensor]:
        """The corrected device view of ``camera`` from ``camera_optimizer`` -- in training, for a camera with an index
        (nerfstudio applies the correction to the training cameras, which carry ``cam_idx``); None otherwise.  The same
        launch yields the regulariser and the metrics' norms: kept for this step's get_loss_dict / get_metrics_dict."""
        self._camera_terms = None
        co = self.camera_optimizer
        if co is None or co.mode == "off" or not self.training or camera.index is None:
            return None
        view, reg, norms = co.terms(camera)
        self._camera_terms = (reg, norms)
        return view

    def get_outputs(self, camera: Camera) -> Dict[str, torch.Tensor]:
        """``SplatfactoSceneGraphModel.get_outputs`` (scene graph :305-374)."""
        assert camera.time is not None
        frame = self._frame(camera)
        H, W = camera.height, camera.width
        self.last_size = (H, W)
        self._last_camera = camera  # the nominal camera: a batch's lidar sweep is projected with it (_depth_target)
        view = self._camera_view(camera)
        if self.config.use_sky_sphere and self.env_map is not None:
            sky = self.env_map(camera, self.training) if view is None else self.env_map(camera, self.training, view=view)
        else:
            sky = None
        sink = anchor = None
        if torch.is_grad_enabled():
            flat = [t for seg in frame.segments for t in seg.params.tensors()]
            if all(t.requires_grad and t.is_leaf for t in flat):  # the normal case: the model's own nn.Parameters
                sink = self._grad_sink
                if isinstance(sink, _FullArenaSink):
                    sink.bind_model(self.optimizer_params(), self.present_submodels())
                else:
                    sink.bind(flat)
                if self._anchor is None or self._anchor.device != flat[0].device:
                    self._anchor = torch.zeros(1, device=flat[0].device, requires_grad=True)
                anchor = self._anchor
        pose = self._box_poses(frame)
        extra = self._semantic_rows(frame)
        kw = {}
        if extra is not None:
            kw["extra"] = extra
        # the scale regularisation of this step comes out of the render (raster.render_frame, scale_reg=); get_loss_dict takes it
        # from here, so ``outputs`` keeps its keys
        self.__dict__["_scale_reg"] = None
        if self._fused_scale_reg_due():
            kw["scale_reg"] = self.config.max_gauss_ratio
        # likewise MCMC's regularisers, every training step
        self.__dict__["_mcmc_reg"] = None
        if self._fused_mcmc_reg_due():
            kw["terms"] = (raster.MCMCRegTerm(self.config.mcmc_opacity_reg, self.config.mcmc_scale_reg),)
        out, holder = raster.render_frame(frame, self._settings(class_streams=True), sky=sky, grad_sink=sink, anchor=anchor,
                                          pose=pose, view=view, **kw)
        if extra is not None:
            out["semantic"] = out.pop("extra")
        if "scale_reg" in kw:
            self.__dict__["_scale_reg"] = out.pop("scale_reg")
        if "terms" in kw:
            self.__dict__["_mcmc_reg"] = {k: out.pop(k) for k in raster.MCMCRegTerm.names}
        self._holder = holder
        self._publish_side_effects(frame, holder)
        if isinstance(holder.M, raster.LazyCount):
            # rendered without the count's read-back (RenderSettings.async_binning): the reference's early-out for "nothing in
            # view" (depth 0 instead of the 10 of an empty pixel, sgn_splatfacto.py:878-886) is applied on the device
            out["depth"] = out["depth"] * (holder.M.device_count > 0).to(out["depth"].dtype)
        elif holder.M == 0:
            # reference early-out when nothing is visible (sgn_splatfacto.py:878-886): background colour
            # (zeros), zero accumulation and ZERO depth
            dev = self.device
            res = {"rgb": torch.zeros(H, W, 3, device=dev), "accumulation": torch.zeros(H, W, 1, device=dev),
                   "depth": torch.zeros(H, W, 1, device=dev)}
            if sky is not None:
                res["sky"] = sky
            res["object_acc"] = torch.zeros(H, W, 1, device=dev)
            res["background_acc"] = torch.zeros(H, W, 1, device=dev)
            if extra is not None:
                res["semantic"] = torch.zeros(H, W, extra.shape[1], device=dev)
            return self._correct_appearance(res, camera)
        if not self.training:
            # eval-only extra renders (scene graph :367-372): per-class rgb
            with torch.no_grad():
                out["background_rgb"] = self._class_rgb(frame, CLS_BACKGROUND, sky)
                out["object_rgb"] = self._class_rgb(frame, CLS_OBJECT, None, pose)
                if not any(s.cls == CLS_OBJECT for s in frame.segments):
                    # without actors the reference's objects-only render returns {'rgb': zeros[H,W,1], 'depth': zeros[H,W,1]}
                    # (scene graph :264-267), which get_outputs publishes as object_rgb AND object_depth (:371-372)
                    out["object_depth"] = torch.zeros(H, W, 1, device=self.device)
        return self._correct_appearance(out, camera)

    def _correct_appearance(self, out: Dict[str, torch.Tensor], camera: Camera) -> Dict[str, torch.Tensor]:
        """In training, for a camera with an index: ``out["rgb"]`` (the render with the sky composited) replaced by its slice with
        that image's bilateral grid, so the losses, the per-step psnr and every other consumer see the corrected image.  In eval,
        or for a camera without an index (a novel view has no grid of its own), the raw render."""
        bg = self.bilateral_grid
        if bg is not None and self.training and camera.index is not None:
            out["rgb"] = bg.slice(out["rgb"], camera.index)
        return out

    def _fused_scale_reg_due(self) -> bool:
        """Whether this step's scale regularisation comes out of the render: switched on, a step that is a multiple of 10 (as
        nerfstudio's), the fused loss path (``fused_loss=False`` computes it with torch ops in get_loss_dict), and a training
        render that records gradients (an eval loss takes the value alone, see ``_scale_reg_loss``)."""
        c = self.config
        return (c.use_scale_regularization and self.step % 10 == 0 and c.fused_loss and self.training
                and torch.is_grad_enabled())

    def _scale_reg_loss(self, fused: bool) -> torch.Tensor:
        """losses["scale_reg"] (SplatfactoModel.get_loss_dict of nerfstudio 1.0) over the visible sub-models' rows, in the frame's
        concatenation order; a zero without gradient on the steps that are not a multiple of 10."""
        c = self.config
        if self.step % 10 != 0:
            return torch.zeros((), device=self.device)
        if fused:
            reg = self.__dict__.get("_scale_reg")
            if reg is not None:
                return reg
            h = self._holder
            if (self.training and torch.is_grad_enabled()) or h is None or h.table is None:
                raise RuntimeError("the scale regularisation of this step was not rendered: call get_outputs at the same model.step "
                                   "before get_loss_dict")
            return raster.scale_reg_fwd(h.table, c.max_gauss_ratio)  # eval / no_grad: the value alone, from the last frame's rows
        scales = torch.cat([self.all_models._modules[n].gauss_params["scales"] for n in self.visible_model_names])
        scale_exp = torch.exp(scales)
        scale_reg = torch.maximum(scale_exp.amax(dim=-1) / scale_exp.amin(dim=-1),
                                  torch.tensor(c.max_gauss_ratio, device=scales.device)) - c.max_gauss_ratio
        return 0.1 * scale_reg.mean()

    def _fused_mcmc_reg_due(self) -> bool:
        """Whether this step's MCMC regularisers come out of the render: the MCMC strategy, the fused loss path and a training
        render that records gradients."""
        c = self.config
        return c.strategy == "mcmc" and c.fused_loss and self.training and torch.is_grad_enabled()

    def _mcmc_reg_losses(self, fused: bool) -> Dict[str, torch.Tensor]:
        """losses["mcmc_opacity_reg"] and losses["mcmc_scale_reg"] over the visible sub-models' rows: from the render (fused), from
        the last frame's rows without a gradient (eval / no_grad), or with torch ops over ``torch.cat`` of their parameters."""
        c = self.config
        if fused:
            reg = self.__dict__.get("_mcmc_reg")
            if reg is not None:
                return dict(reg)
            h = self._holder
            if (self.training and torch.is_grad_enabled()) or h is None or h.table is None:
                raise RuntimeError("the MCMC regularisers of this step were not rendered: call get_outputs before get_loss_dict")
            out = raster.mcmc_reg_fwd(h.table, c.mcmc_opacity_reg, c.mcmc_scale_reg)
            return {"mcmc_opacity_reg": out[0], "mcmc_scale_reg": out[1]}
        mods = self.all_models._modules
        opac = torch.cat([mods[n].gauss_params["opacities"] for n in self.visible_model_names])
        scales = torch.cat([mods[n].gauss_params["scales"] for n in self.visible_model_names])
        return {"mcmc_opacity_reg": c.mcmc_opacity_reg * torch.sigmoid(opac).mean(),
                "mcmc_scale_reg": c.mcmc_scale_reg * torch.exp(scales).mean()}

    def _semantic_rows(self, frame: Frame) -> Optional[torch.Tensor]:
        """The frame's semantic logits [N, C] in its row order (the visible sub-models' ``semantic_logits``, concatenated in
        segment order), or None without semantic classes.  The logits are static per Gaussian: actors carry no time
        dependence for them."""
        if self.config.semantic_classes <= 0:
            return None
        mods = self.all_models._modules
        return torch.cat([mods[seg.name].semantic_logits for seg in frame.segments])

    def _class_rgb(self, frame: Frame, cls: int, sky, pose=None):
        segs = [s for s in frame.segments if s.cls == cls]
        H, W = frame.camera.height, frame.camera.width
        if not segs:
            return torch.zeros(H, W, 1, device=self.device) if sky is None else sky
        sub, _ = raster.render_frame(Frame(frame.camera, segs), self._settings(class_streams=False), sky=sky, pose=pose)
        return sub["rgb"]

    def _refine_settings_of(self, sub) -> RefineSettings:
        return self.config.refine if sub is self.all_models._modules["background"] else self.config.object_refine

    def _publish_side_effects(self, frame: Frame, holder) -> None:
        # plain tensors, not parameters/buffers: write the instance dicts directly (nn.Module.__setattr__ costs
        # ~5 us per attribute, x6 attributes x33 sub-models per frame)
        d = self.__dict__
        d["xys"], d["depths"], d["radii"] = holder.xys, holder.depths, holder.radii
        d["conics"], d["num_tiles_hit"] = holder.conics, holder.num_tiles_hit
        mods = self.all_models._modules
        visible = set(self.visible_model_names)
        for name, sub in mods.items():
            if name not in visible:
                sd = sub.__dict__
                sd["_fs_src"], sd["_fs_cache"] = None, None
        row = 0
        slices = []
        for seg in frame.segments:
            sub = mods[seg.name]
            n = seg.params.means.shape[0]
            sl = slice(row, row + n)
            sd = sub.__dict__
            sd["_fs_src"], sd["_fs_cache"], sd["last_size"] = (holder, sl), None, self.last_size  # sliced on first access
            slices.append((sub, sl))
            row += n
        d["_slices"] = slices
        holder.post_backward = self._split_xys_grad(slices)

    def after_train(self, step: int) -> None:
        """The ``after_train`` callbacks of all visible sub-models (sgn_splatfacto.py:513-541; the scene graph
        registers one per sub-model, :127-137) as one launch of ``sgn_densify_stats`` over the frame's rows:
        running ||xys.grad|| sums, visibility counts and the max screen-space radius ratio, per sub-model."""
        assert step == self.step
        h = self._holder
        if h is None or h.v_records is None or self.config.strategy == "mcmc":  # MCMC keeps no densification statistics
            return
        import ctypes as C
        from . import _lib
        L = _lib.load()
        # every sub-model's callback reads ITS OWN config.stop_split_at (sgn_splatfacto.py:516-518)
        slices = [(sub, sl) for sub, sl in (self.__dict__.get("_slices") or [])
                  if self.step < self._refine_settings_of(sub).stop_split_at]
        if not slices:
            return
        tab = (_lib.DensifySegment * len(slices))()
        dev = h.v_records.device
        for j, (sub, sl) in enumerate(slices):
            n = sl.stop - sl.start
            first = sub.xys_grad_norm is None or sub.xys_grad_norm.shape[0] != n
            if first:
                d = sub.__dict__
                d["xys_grad_norm"], d["vis_counts"], d["max_2Dsize"] = (torch.empty(n, device=dev) for _ in range(3))
            tab[j].row0, tab[j].count, tab[j].first = sl.start, n, int(first)
            tab[j].xys_grad_norm, tab[j].vis_counts = sub.xys_grad_norm.data_ptr(), sub.vis_counts.data_ptr()
            tab[j].max_2Dsize = sub.max_2Dsize.data_ptr()
        raw = torch.frombuffer(bytearray(bytes(tab)), dtype=torch.uint8).to(dev, non_blocking=True)
        H, W = self.last_size
        _lib.check(L.sgn_densify_stats(raster._ptr(raw), len(slices), h.v_records.shape[0], raster._ptr(h.v_records),
                                       raster._ptr(h.radii), H, W, raster._stream()), "sgn_densify_stats")

    # ------------------------------------------------------------------------------------------
    def refinement_after(self, optimizers, step: int, generator: Optional[torch.Generator] = None, sync_stats: bool = True,
                         due_only: bool = False, seed: int = 0) -> None:
        """The ``refinement_after`` callbacks of all sub-models (sgn_splatfacto.py:550-646; the scene graph registers one
        per sub-model, :127-137): split / duplicate / cull / opacity reset, with the optimizer state carried along
        (dup_in_optim / remove_from_optim, :459-511).  ``optimizers`` is a ``FusedAdam`` built over
        ``self.optimizer_params()``, or the reference's form -- an object (or dict) mapping the six group names to
        ``torch.optim.Adam`` instances whose ``param_groups[0]["params"][i]`` is sub-model i's tensor -- or None.

        Two phases so that nothing is copied twice and the host waits once: decide every sub-model (all launches first,
        then ONE read-back of all the counts), then lay out the new tensors / moment arenas and let ``sgn_refine_apply``
        write each sub-model's rows into them.

        ``due_only``: nerfstudio runs each sub-model's callback every ITS OWN ``refine_every`` steps
        (``update_every_num_iters=self.config.refine_every``, sgn_splatfacto.py:773-781); with ``due_only`` a sub-model
        whose ``refine_every`` does not divide ``step`` is left alone (callers that run on a global cadence pass False).

        With ``strategy="mcmc"`` the sub-models are refined by MCMC instead (``_mcmc_refinement``, draws keyed by ``seed``)."""
        assert step == self.step
        names = list(self.all_models._modules)
        subs = [self.all_models[n] for n in names]
        adapter = _optimizer_adapter(optimizers, len(subs))
        if self.config.strategy == "mcmc":
            self._mcmc_refinement(adapter, step, seed, due_only)
            return
        if sync_stats:
            self._sync_densification_stats(subs)
        # phase 1: every sub-model's decision pass is launched, then ALL totals come back with one read-back
        decided, resets = [], []
        for name, sub in zip(names, subs):
            st = self.config.refine if name == "background" else self.config.object_refine
            densify, cull_only, reset = refine.phase(st, step, self.config.num_train_data)
            if due_only and (st.refine_every <= 0 or step % st.refine_every != 0):
                decided.append(None)
                resets.append(None)
                continue
            sub.__dict__["refine_record_dict"] = {}
            if step <= st.warmup_length or sub.xys_grad_norm is None:  # :552-555
                decided.append(None)
                resets.append(None)
                continue
            entry = None
            if densify or cull_only:
                size = sub.last_size or self.last_size
                cfg = refine.make_config(st, step, size, densify)
                g = sub.gauss_params
                flags, scan = refine.decide_submodel(g["scales"].data, g["opacities"].data, sub.xys_grad_norm if densify else None,
                                                     sub.vis_counts if densify else None,
                                                     sub.max_2Dsize if cfg.use_screen_size else None, cfg)
                entry = (flags, scan, cfg)
            decided.append(entry)
            resets.append(st if reset else None)
            d = sub.__dict__
            d["xys_grad_norm"] = d["vis_counts"] = d["max_2Dsize"] = None  # :644-646
        totals = iter(refine.read_totals([e[1] for e in decided if e is not None]))
        plans, records = [], []
        for sub, entry in zip(subs, decided):  # split samples are drawn in sub-model order, as the reference's callbacks run
            plan = None
            if entry is not None:
                plan = refine.finish_plan(entry[0], entry[1], next(totals), entry[2], generator)
                if self.config.refine_record:
                    records.append((sub, plan, plan.record_counts()))
                if not plan.changed:
                    plan = None
            plans.append(plan)
        old = [[sub.gauss_params[k].data for k in PARAM_NAMES] for sub in subs]
        new = [o if p is None else [torch.empty((p.out_rows,) + tuple(t.shape[1:]), device=t.device, dtype=t.dtype) for t in o]
               for o, p in zip(old, plans)]
        # the semantic logits ride along: the same row map as features_dc (sgn_refine_carry), with their moments
        sem = self.config.semantic_classes > 0
        old_sem = [sub.semantic_logits.data for sub in subs] if sem else None
        new_sem = [o if p is None else torch.empty((p.out_rows,) + tuple(o.shape[1:]), device=o.device, dtype=o.dtype)
                   for o, p in zip(old_sem, plans)] if sem else None
        if any(p is not None for p in plans):
            from .semantic import refine_carry
            changed = [p is not None for p in plans]
            src_m, dst_m = adapter.relayout(new, changed, {"semantic": new_sem} if sem else None)
            for i, p in enumerate(plans):
                if p is not None:
                    refine.apply_plan(p, old[i], new[i], src_m[i], dst_m[i])
                    for k, t in zip(PARAM_NAMES, new[i]):
                        subs[i].gauss_params[k] = torch.nn.Parameter(t)
                    if sem:
                        ms, md = adapter.row_moments("semantic", i)
                        refine_carry(p, old_sem[i], new_sem[i], ms, md)
                        subs[i].semantic_logits = torch.nn.Parameter(new_sem[i])
                    if subs[i].filter_3d is not None:  # sized to the new rows; compute_filter_3d fills it (TrainStep does, next)
                        subs[i].filter_3d = torch.zeros(p.out_rows, device=self.device, dtype=torch.float32)
            adapter.commit([[sub.gauss_params[k] for k in PARAM_NAMES] for sub in subs], changed,
                           {"semantic": [sub.semantic_logits for sub in subs]} if sem else None)
            self.invalidate_frames()
        self.__dict__["refine_changed_rows"] = any(p is not None for p in plans)
        for i, st in enumerate(resets):
            if st is not None:  # opacity reset on the survivors (:629-642); the semantic logits are left alone
                subs[i].gauss_params["opacities"].data.clamp_(max=refine.opacity_reset_logit(st))
                adapter.zero_moments(i, 5)
        if records:  # the logged counters of all sub-models: one read-back, after everything else has been enqueued
            for (sub, plan, _), counts in zip(records, torch.stack([r[2] for r in records]).tolist()):
                sub.__dict__["refine_record_dict"] = plan.record_from(counts)

    def _mcmc_settings_of(self, name: str) -> MCMCSettings:
        return self.config.mcmc if name == "background" else self.config.object_mcmc

    def _mcmc_refinement(self, adapter, step: int, seed: int, due_only: bool) -> None:
        """gsplat's MCMCStrategy._refine per sub-model inside its window (mcmc.py): relocate the dead rows, then draw the added
        rows; then ONE relayout of the optimizer for the sub-models that grew, whose new rows copy the drawn ones in draw order
        with zero moments (the semantic logits and the 3D filter sizes ride along).  No opacity reset.  Nothing is read back but
        the relocation counts with ``refine_record``."""
        names = list(self.all_models._modules)
        subs = [self.all_models[n] for n in names]
        sem = self.config.semantic_classes > 0
        relocated, added = [], []
        for i, (name, sub) in enumerate(zip(names, subs)):
            st = self._mcmc_settings_of(name)
            if not mcmc.in_window(st, step) or (due_only and (st.refine_every <= 0 or step % st.refine_every != 0)):
                relocated.append(None)
                added.append(None)
                continue
            sub.__dict__["refine_record_dict"] = {}
            params = [sub.gauss_params[k].data for k in PARAM_NAMES]
            carried = ([sub.semantic_logits.data] if sem else []) + ([sub.filter_3d] if sub.filter_3d is not None else [])
            relocated.append(mcmc.relocate(params, carried, mcmc.moment_tensors(adapter.moments(i)), st, seed, step, i))
            A = mcmc.num_added(sub.num_points, st)
            added.append((A, mcmc.draw_added(params, A, st, seed, step, i)) if A > 0 else None)
        grow = [a is not None for a in added]
        if any(grow):
            old = [[sub.gauss_params[k].data for k in PARAM_NAMES] for sub in subs]
            new = [o if a is None else [torch.empty((o[0].shape[0] + a[0],) + tuple(t.shape[1:]), device=t.device, dtype=t.dtype) for t in o]
                   for o, a in zip(old, added)]
            old_sem = [sub.semantic_logits.data for sub in subs] if sem else None
            new_sem = [o if a is None else torch.empty((o.shape[0] + a[0],) + tuple(o.shape[1:]), device=o.device, dtype=o.dtype)
                       for o, a in zip(old_sem, added)] if sem else None
            src_m, dst_m = adapter.relayout(new, grow, {"semantic": new_sem} if sem else None)
            for i, a in enumerate(added):
                if a is None:
                    continue
                n = old[i][0].shape[0]
                pairs = [(old[i], new[i])]
                moments = list(zip(src_m[i] or [], dst_m[i] or []))
                if sem:
                    pairs.append(([old_sem[i]], [new_sem[i]]))
                    ms, md = adapter.row_moments("semantic", i)
                    if md is not None:
                        moments.append((ms, md))
                sub = subs[i]
                f_new = None
                if sub.filter_3d is not None:
                    f_new = torch.empty(n + a[0], device=self.device, dtype=torch.float32)
                    pairs.append(([sub.filter_3d], [f_new]))
                for src, dst in pairs:
                    for s_, d_ in zip(src, dst):
                        d_[:n].copy_(s_)
                for src, dst in moments:  # the old rows keep their moments, the appended rows start from zero
                    for s_, d_ in zip(src, dst):
                        d_[:n].copy_(s_)
                        d_[n:].zero_()
                rows = [d_ for _, dst in pairs for d_ in dst]
                mcmc.copy_rows(rows, a[1], a[0], dst_row0=n)
                for k, t in zip(PARAM_NAMES, new[i]):
                    sub.gauss_params[k] = torch.nn.Parameter(t)
                if sem:
                    sub.semantic_logits = torch.nn.Parameter(new_sem[i])
                if f_new is not None:
                    sub.filter_3d = f_new
            adapter.commit([[sub.gauss_params[k] for k in PARAM_NAMES] for sub in subs], grow,
                           {"semantic": [sub.semantic_logits for sub in subs]} if sem else None)
            self.invalidate_frames()
        self.__dict__["refine_changed_rows"] = any(grow)
        if self.config.refine_record:
            done = [i for i, r in enumerate(relocated) if r is not None]
            counts = torch.stack([relocated[i] for i in done]).tolist() if done else []
            for i, c in zip(done, counts):
                subs[i].__dict__["refine_record_dict"] = {"mcmc_relocated": int(c), "mcmc_added": added[i][0] if added[i] else 0}

    def inject_noise(self, step: int, lr: float, seed: int = 0, normals: Optional[torch.Tensor] = None) -> None:
        """gsplat's ``inject_noise_to_position`` on every row of every sub-model, one launch (actors in object coordinates):
        means += Sigma (eps * gate(1 - opacity) * lr * noise_lr), with the sub-model's noise_lr and ``lr`` the means' learning
        rate at this step.  eps ~ N(0, I) from Philox keyed by (seed, step, sub-model, row), or ``normals`` [rows, 3] (the
        sub-models' rows back to back, all_models order)."""
        d = self.__dict__
        # the sub-model list and its device table change only with the parameter tensors (invalidate_frames): this runs every
        # step, and rebuilding them costs more host time than the rest of the step's MCMC work
        key = (d.get("_param_epoch", 0), self.all_models._modules["background"].gauss_params._parameters["means"].data_ptr())
        if d.get("_noise_key") != key:
            subs = []
            for name, sub in self.all_models._modules.items():
                g = sub.gauss_params
                subs.append((g["means"].data, g["scales"].data, g["quats"].data, g["opacities"].data,
                             self._mcmc_settings_of(name).noise_lr))
            d["_noise_subs"], d["_noise_key"] = subs, key
            self._noise_table.get(subs, self.device)
        mcmc.inject_noise(self._noise_table, d["_noise_subs"], lr, seed, step, normals, rebuild=False)

    def _sync_densification_stats(self, subs) -> None:
        """Replicas rendered different cameras: identical split / cull decisions need identical statistics (SURVEY.md 8e).
        SUM / SUM / MAX per sub-model; a replica that has not seen a sub-model since the last refinement contributes
        zeros, and a sub-model nobody saw stays without statistics (the collectives are the same on every replica)."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
            return
        dev = self.device
        has = torch.tensor([float(sub.xys_grad_norm is not None) for sub in subs], device=dev)
        dist.all_reduce(has, op=dist.ReduceOp.MAX)
        live = []
        for sub, h in zip(subs, has.tolist()):
            if not h:
                continue
            if sub.xys_grad_norm is None:
                d = sub.__dict__
                d["xys_grad_norm"], d["vis_counts"], d["max_2Dsize"] = (torch.zeros(sub.num_points, device=dev) for _ in range(3))
                d["last_size"] = sub.last_size or self.last_size
            live.append(sub)
        if not live:
            return
        # TWO collectives for all sub-models (33 x 3 small ones cost ~3 ms per refinement at eight GPUs): the SUM statistics and the
        # MAX statistic are packed into flat buffers, reduced, and copied back
        sums = torch.cat([t for sub in live for t in (sub.xys_grad_norm, sub.vis_counts)])
        maxs = torch.cat([sub.max_2Dsize for sub in live])
        dist.all_reduce(sums, op=dist.ReduceOp.SUM)
        dist.all_reduce(maxs, op=dist.ReduceOp.MAX)
        o = m_ = 0
        for sub in live:
            n = sub.num_points
            sub.xys_grad_norm.copy_(sums[o:o + n])
            sub.vis_counts.copy_(sums[o + n:o + 2 * n])
            sub.max_2Dsize.copy_(maxs[m_:m_ + n])
            o += 2 * n
            m_ += n

    def zero_gradient_arena(self) -> torch.Tensor:
        """Data parallel: this replica rendered nothing (early-out) but the others did -- its contribution to the
        all-reduce is an all-zero arena in the common layout."""
        sink = self._grad_sink
        assert isinstance(sink, _FullArenaSink), "only with SceneGraphConfig(full_gradient_arena=True)"
        sink.bind_model(self.optimizer_params(), [])
        return sink.target(None, self.device)

    def optimizer_params(self) -> List[List[torch.Tensor]]:
        """Per sub-model (all_models order: background, then objects), the six tensors in gradient-arena order: what
        ``FusedAdam`` is built over.  ``present_submodels()`` names the ones in the last frame's gradient arena."""
        return [[sub.gauss_params[k] for k in PARAM_NAMES] for sub in self.all_models._modules.values()]

    def semantic_params(self) -> List[torch.Tensor]:
        """Per sub-model (all_models order) its ``semantic_logits``: the row group ``FusedAdam(..., rows={"semantic":
        (model.semantic_params(), lr)})`` steps (and ``refinement_after`` carries)."""
        assert self.config.semantic_classes > 0, "the model has no semantic logits (SceneGraphConfig.semantic_classes = 0)"
        return [sub.semantic_logits for sub in self.all_models._modules.values()]

    def present_submodels(self) -> List[int]:
        index = {n: i for i, n in enumerate(self.all_models._modules)}
        return [index[n] for n in self.visible_model_names]

    @staticmethod
    def _split_xys_grad(slices):
        """After ``loss.backward()``: ``sub.xys.grad`` for every visible sub-model, as the reference's
        ``set_split_tensor_variable(..., retain_grad=True)`` provides (scene graph :153-179).  ``sub.xys`` is sliced on access
        (with its gradient, once the backward has run); only a ``sub.xys`` that was read BEFORE the backward needs it set here."""
        def hook(h):
            v_xy = None
            for sub, sl in slices:
                cache = sub.__dict__.get("_fs_cache")
                if cache:
                    t = cache.get("xys")
                    if t is not None:
                        v_xy = h.v_records[:, 0:2] if v_xy is None else v_xy
                        t.grad = v_xy[sl]
        return hook

    # ------------------------------------------------------------------------------------------
    def get_loss_dict(self, outputs, batch, metrics_dict=None) -> Dict[str, torch.Tensor]:
        """sgn_splatfacto.py:1042-1094 + scene graph :376-391.  ``batch["image"]`` may be the float image or the
        uint8 one the data loader holds (converted as the reference does: ``.float() / 255``).

        With ``depth_loss_mult > 0`` and a lidar target in the batch (see ``_depth_target``), ``depth_loss`` =
        depth_loss_mult * mean |depth - target| over the pixels with a return (and mask != 0): Street Gaussians' lidar depth
        term, which the reference's nerfstudio port dropped.  Its gradient reaches the geometry through the rendered depth,
        ``where(alpha > 1e-3, d / alpha, 10)``: a return on a pixel with alpha <= 1e-3 adds to the loss value but pulls on
        nothing.

        With ``semantic_loss_mult > 0``, semantic classes and ``batch["semantic"]``, ``semantic_loss`` = semantic_loss_mult *
        mean cross-entropy of ``outputs["semantic"]`` against the labels over the pixels with a label in [0, C) (and mask != 0).
        Sky-labelled pixels are supervised like any other class: the semantic map there is the blend of whatever Gaussians the
        pixel sees, and ``sky_accumulation`` separately pushes their accumulation towards 0, which also shrinks the blended logits
        (weights sum to the accumulation).  The two terms therefore pull against each other on sky pixels; nothing special-cases
        that, as a segmentation with a sky class gives both signals.

        With ``use_scale_regularization``, ``scale_reg`` is present on every call, as nerfstudio emits it: at a step that is a
        multiple of 10, 0.1 * mean(max(amax(s) / amin(s), max_gauss_ratio) - max_gauss_ratio) with s = exp(scales) over the rows
        of the visible sub-models (the render computed it, sgn_scale_reg_fwd; torch ops over ``torch.cat`` of their scales
        with ``fused_loss=False``), and a zero without gradient on the other steps.

        With a ``bilateral_grid``, in training: ``bilagrid_tv`` = 10 * the total variation of all grids
        (bilagrid.BilateralGrid.tv_loss), every step.

        With ``strategy="mcmc"``: ``mcmc_opacity_reg`` = mcmc_opacity_reg * mean(sigmoid(opacities)) and ``mcmc_scale_reg`` =
        mcmc_scale_reg * mean(exp(scales)) over the rows of the visible sub-models, every call (the render computed them,
        sgn_mcmc_reg_fwd; torch ops with ``fused_loss=False``)."""
        c = self.config
        want_sky = "semantic" in batch and c.sky_acc_loss_mult > 0
        want_ent = c.object_acc_entropy_loss_mult > 0.0 and self.step > c.refine.stop_split_at  # background_model.stop_split_at (:386)
        fused = c.fused_loss and outputs["rgb"].is_cuda
        losses = {}

        def float_pair():  # (gt, rgb) as the torch ops consume them
            gt_img, rgb = batch["image"], outputs["rgb"]
            if gt_img.dtype == torch.uint8:
                gt_img = gt_img.float() / 255.0
            if "mask" in batch:
                gt_img, rgb = gt_img * batch["mask"], rgb * batch["mask"]
            return gt_img, rgb

        if fused:
            # one forward + one backward kernel for the three image-space terms (loss.py)
            from .loss import fused_image_losses
            l1, sky, ent = fused_image_losses(
                outputs["rgb"], batch["image"], accumulation=outputs["accumulation"] if want_sky else None,
                object_acc=outputs["object_acc"] if want_ent else None, mask=batch.get("mask"),
                sky_mask=(batch["semantic"] == 2) if want_sky else None,  # SemanticType.SKY (data/utils/data_utils.py:26-29)
                w_l1=1 - c.ssim_lambda, w_sky=c.sky_acc_loss_mult if want_sky else 0.0,
                w_entropy=c.object_acc_entropy_loss_mult if want_ent else 0.0)
            losses["Ll1"] = l1
        else:
            gt_img, rgb = float_pair()
            losses["Ll1"] = (1 - c.ssim_lambda) * torch.abs(gt_img - rgb).mean()
        if c.ssim_lambda > 0 and fused:
            # SSIM forward + backward kernels (loss.py, csrc/ssim.cu); a uint8 image is read as it is
            from .loss import fused_ssim_loss
            losses["simloss"] = fused_ssim_loss(outputs["rgb"], batch["image"], mask=batch.get("mask"), weight=c.ssim_lambda)
        elif c.ssim_lambda > 0:
            gt_img, rgb = float_pair()
            simloss = 1 - ssim(gt_img.permute(2, 0, 1)[None, ...], rgb.permute(2, 0, 1)[None, ...])
            losses["simloss"] = c.ssim_lambda * simloss
        else:
            # the reference always emits the key (sgn_splatfacto.py:1085-1087); with ssim_lambda == 0 its value is 0 * simloss:
            # an exact zero that contributes no gradient, so the SSIM convolutions are not run for it
            losses["simloss"] = torch.zeros((), device=outputs["rgb"].device)
        if want_sky:
            if fused:
                losses["sky_accumulation"] = sky
            else:
                sky_mask = (batch["semantic"] == 2)
                losses["sky_accumulation"] = c.sky_acc_loss_mult * (sky_mask * outputs["accumulation"]).mean()
        if want_ent:
            if fused:
                losses["object_acc_entropy_loss"] = ent
            else:
                oa = torch.clamp(outputs["object_acc"], min=1e-5, max=1 - 1e-5)
                losses["object_acc_entropy_loss"] = c.object_acc_entropy_loss_mult * -(
                    oa * torch.log(oa) + (1.0 - oa) * torch.log(1.0 - oa)).mean()
        if c.depth_loss_mult > 0:
            target = self._depth_target(batch)
            if target is not None:
                from .depth import depth_loss_torch, fused_depth_loss
                term = fused_depth_loss if fused else depth_loss_torch
                losses["depth_loss"] = term(outputs["depth"], target, batch.get("mask"), c.depth_loss_mult)
        if c.semantic_loss_mult > 0 and "semantic" in batch and "semantic" in outputs:
            from .semantic import fused_semantic_loss, semantic_loss_torch
            term = fused_semantic_loss if fused else semantic_loss_torch
            losses["semantic_loss"] = term(outputs["semantic"], batch["semantic"], batch.get("mask"), c.semantic_loss_mult)
        if c.use_scale_regularization:
            losses["scale_reg"] = self._scale_reg_loss(fused)
        if c.strategy == "mcmc":
            losses.update(self._mcmc_reg_losses(fused))
        co = self.camera_optimizer
        if self.training and co is not None and co.mode != "off":
            terms = getattr(self, "_camera_terms", None)
            losses["camera_opt_regularizer"] = terms[0] if terms is not None else co.regularizer()
        if self.training and self.bilateral_grid is not None:
            losses["bilagrid_tv"] = 10.0 * self.bilateral_grid.tv_loss()  # gsplat's tv_loss weight
        return losses

    def _depth_target(self, batch) -> Optional[torch.Tensor]:
        """The lidar depth target [H,W,1] of ``batch``, or None: ``batch["depth_image"]`` as it is (0 = no measurement), else
        ``batch["lidar_points"]`` [M,3] (with the optional 3x4 ``batch["lidar_to_world"]``) projected by ``depth.lidar_depth_map``
        with the nominal camera of the last ``get_outputs``: the sweep is registered with the dataset's vehicle pose and
        calibration, not with the camera optimizer's correction (which still feels the term through the rendered depth)."""
        if "depth_image" in batch:
            return batch["depth_image"]
        if "lidar_points" not in batch:
            return None
        from .depth import lidar_depth_map
        return lidar_depth_map(batch["lidar_points"], self._last_camera, batch.get("lidar_to_world"), self._settings(class_streams=True))

    def _fused_metrics_ok(self, rgb: torch.Tensor) -> bool:
        return self.config.fused_loss and rgb.is_cuda

    def get_metrics_dict(self, outputs, batch) -> Dict[str, object]:
        """``SplatfactoModel.get_metrics_dict`` as the scene graph inherits it (sgn_splatfacto.py:1015-1040; num_downscales = 0):
        psnr of ``outputs["rgb"]`` against ``batch["image"]`` (no mask), ``gaussian_count`` (host int: rows of the visible
        sub-models), the scene graph's own refine counters (always empty: refinement runs on the sub-models), then the means of
        exp(scales), scales, sigmoid(opacities) and radii over the visible rows, under the reference's key names.

        Fused path: the five values are 0-d device tensors of ONE ``sgn_metrics`` launch that reads the parameters through the
        frame's device segment table -- no concatenation, no read-back.  ``fused_loss=False`` or CPU tensors: the reference's
        torch expressions over ``torch.cat`` of the visible sub-models."""
        rgb, gt = outputs["rgb"], batch["image"]
        h = self._holder
        d: Dict[str, object] = {}
        if self._fused_metrics_ok(rgb) and h is not None and h.table is not None:
            from .loss import fused_metrics
            psnr, scale_mean, log_scale_mean, sig, radii_mean = fused_metrics(rgb, gt, table=h.table, radii=h.radii).unbind()
            d["psnr"] = psnr
            d["gaussian_count"] = int(h.table.N)
        else:
            visible = [self.all_models._modules[n] for n in self.visible_model_names]
            with torch.no_grad():
                g = gt.float() / 255.0 if gt.dtype == torch.uint8 else gt
                d["psnr"] = _psnr(rgb.detach(), g)
                d["gaussian_count"] = sum(sub.num_points for sub in visible)
                scales = torch.cat([sub.gauss_params["scales"] for sub in visible])
                opacities = torch.cat([sub.gauss_params["opacities"] for sub in visible])
                scale_mean, log_scale_mean = torch.exp(scales).mean(), scales.mean()
                sig = torch.sigmoid(opacities).mean()
                radii_mean = self.radii.float().mean()
        d["scale_mean"] = scale_mean
        d["log_scale_mean"] = log_scale_mean
        d["sigmoid_opacity"] = sig
        d["self.radii"] = radii_mean  # sic: the reference's key
        co = self.camera_optimizer
        if co is not None and co.mode != "off":
            terms = getattr(self, "_camera_terms", None)
            d.update(co.metrics_of(terms[1]) if terms is not None else co.metrics())
        return d

    def get_image_metrics_and_images(self, outputs, batch):
        """``SplatfactoModel.get_image_metrics_and_images`` (sgn_splatfacto.py:1109-1187; num_downscales = 0).

        Metrics (Python floats): ``psnr`` and ``ssim`` of gt*mask against rgb*mask (no mask: the images as they are), and
        ``lpips`` when ``self.lpips`` is a callable (it receives the masked [1,3,H,W] gt and rgb, in that order).  Fused path:
        psnr from ``sgn_metrics``, ssim = 1 - the SSIM loss kernel at weight 1.  Images: ``img`` = cat([gt, rgb], dim=1), built
        before masking as the reference does; ``accumulation`` and ``depth`` as the model's [H,W,1] maps, not colour-mapped.
        Unlike the reference, ``outputs["rgb"]`` and ``batch["image"]`` are not multiplied by the mask in place.  When the batch
        carries a lidar target (``depth_image`` or ``lidar_points``, see ``_depth_target``), the depth metrics of
        ``depth.depth_metrics`` over the pixels with a return (and mask != 0) are added as ``depth_abs_rel``, ``depth_sq_rel``,
        ``depth_rmse``, ``depth_rmse_log``, ``depth_a1``, ``depth_a2`` and ``depth_a3`` (NaN when no pixel has a return).  With
        semantic classes and ``batch["semantic"]``: ``semantic_acc`` (pixel accuracy of the argmax) and ``semantic_miou`` (mean IoU
        over the classes whose union is > 0) over the pixels with a label in [0, C) (and mask != 0)."""
        rgb, gt = outputs["rgb"], batch["image"]
        gt_f = gt.float() / 255.0 if gt.dtype == torch.uint8 else gt
        mask = batch.get("mask")
        if mask is not None:
            mask = mask.to(rgb.device).float()
        with torch.no_grad():
            img = torch.cat([gt_f, rgb], dim=1)
            masked = None
            if self._fused_metrics_ok(rgb):
                from .loss import fused_metrics, fused_ssim_loss
                psnr = fused_metrics(rgb, gt, mask)[0]
                ssim_v = 1.0 - fused_ssim_loss(rgb, gt, mask, weight=1.0)
            else:
                masked = (gt_f * mask, rgb * mask) if mask is not None else (gt_f, rgb)
                psnr = _psnr(masked[1], masked[0])
                ssim_v = ssim(masked[0].permute(2, 0, 1)[None], masked[1].permute(2, 0, 1)[None])
            metrics = {"psnr": float(psnr.item()), "ssim": float(ssim_v)}
            if callable(self.lpips):
                if masked is None:
                    masked = (gt_f * mask, rgb * mask) if mask is not None else (gt_f, rgb)
                metrics["lpips"] = float(self.lpips(torch.moveaxis(masked[0], -1, 0)[None], torch.moveaxis(masked[1], -1, 0)[None]))
            target = self._depth_target(batch)
            if target is not None:
                # the depth_result the reference's eval calls but never defines (sgn_splatfacto.py:1160-1168)
                from .depth import METRIC_NAMES, depth_metrics
                vals = depth_metrics(outputs["depth"], target, mask).tolist()
                metrics.update({f"depth_{k}": v for k, v in zip(METRIC_NAMES[:7], vals[:7])})
            if "semantic" in batch and "semantic" in outputs:
                from .semantic import semantic_metrics
                metrics.update(semantic_metrics(outputs["semantic"], batch["semantic"], mask))
        images = {"img": img, "accumulation": outputs["accumulation"], "depth": outputs["depth"]}
        return metrics, images

    def get_outputs_for_camera(self, camera: Camera, obb_box=None) -> Dict[str, torch.Tensor]:
        """``SplatfactoModel.get_outputs_for_camera`` (sgn_splatfacto.py:1096-1107): ``get_outputs`` under ``no_grad``.  The
        scene graph supports no crop box outside training (scene graph :361): a box raises."""
        if obb_box is not None:
            raise ValueError("crop boxes are not supported by the scene-graph model")
        with torch.no_grad():
            return self.get_outputs(camera)


def _psnr(preds: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """torchmetrics PeakSignalNoiseRatio(data_range=1.0) on one pair: 10 log10(1 / mean((preds - target)^2)), +inf when equal."""
    mse = torch.sum((preds - target) ** 2) / target.numel()
    return 10.0 * torch.log10(1.0 / mse)


class _NoOptimizer:
    """refinement_after(None, ...): parameters only."""

    def relayout(self, new, changed, rows=None):
        return [None] * len(new), [None] * len(new)

    def row_moments(self, name: str, sub: int):
        """(old (exp_avg, exp_avg_sq), new pair) of a changed sub-model's tensor of row group ``name``, or (None, None)."""
        return None, None

    def commit(self, params, changed, rows=None):
        pass

    def zero_moments(self, sub: int, k: int):
        pass

    def moments(self, sub: int):
        """The (exp_avg, exp_avg_sq) pairs of sub-model ``sub``'s six tensors and of its per-row groups, those that exist."""
        return []


class _FusedAdamAdapter(_NoOptimizer):
    """Moments live in two flat arenas: ``relayout`` allocates the arenas of the new layout, hands out views of the old
    and new ones for the sub-models that change (sgn_refine_apply writes the new ones) and block-copies the rest."""

    def __init__(self, opt):
        self.opt = opt
        self._rows = {}

    def relayout(self, new, changed, rows=None):
        """``rows``: the row groups' tensors after the refinement (name -> one per sub-model: new ones for the changed
        sub-models), for the groups the model carries; a group the optimizer does not hold is left out."""
        opt = self.opt
        old_params = opt._params
        rows = {k: v for k, v in (rows or {}).items() if k in opt.row_index}
        old_index = dict(opt.row_index)
        old_m, old_v, old_off = opt.rebuild(new, rows)
        self._rows = {}
        for name, ts in rows.items():  # changed sub-models: old moments (old layout) -> new moment views (zeroed) for the carry
            pairs = []
            for i, ch in enumerate(changed):
                if not ch:
                    pairs.append(None)
                    continue
                t, o = old_params[old_index[name] + i], int(old_off[old_index[name] + i])
                pairs.append(((old_m[o:o + t.numel()].view(t.shape), old_v[o:o + t.numel()].view(t.shape)),
                              opt.row_moment_views(name, i)))
            self._rows[name] = pairs
        src, dst = [], []
        for i, ch in enumerate(changed):
            if ch:
                pairs = []
                for k in range(6):
                    t, o = old_params[6 * i + k], int(old_off[6 * i + k])
                    pairs.append((old_m[o:o + t.numel()].view(t.shape), old_v[o:o + t.numel()].view(t.shape)))
                src.append(pairs)
                dst.append([opt.moment_views(6 * i + k) for k in range(6)])
            else:  # same tensors, new offsets: one block copy per arena
                a, b = int(old_off[6 * i]), int(opt.offsets[6 * i])
                size = int(opt.sizes[6 * i:6 * i + 6].sum())
                opt.exp_avg[b:b + size].copy_(old_m[a:a + size])
                opt.exp_avg_sq[b:b + size].copy_(old_v[a:a + size])
                src.append(None)
                dst.append(None)
        return src, dst

    def row_moments(self, name: str, sub: int):
        pairs = self._rows.get(name)
        return (None, None) if pairs is None or pairs[sub] is None else pairs[sub]

    def commit(self, params, changed, rows=None):
        self.opt.rebuild_pointers(params, {k: v for k, v in (rows or {}).items() if k in self.opt.row_index})
        self._rows = {}

    def zero_moments(self, sub: int, k: int):
        m, v = self.opt.moment_views(6 * sub + k)
        m.zero_()
        v.zero_()

    def moments(self, sub: int):
        return [self.opt.moment_views(6 * sub + k) for k in range(6)] + [self.opt.row_moment_views(n, sub) for n in self.opt.row_index]


class _TorchAdamGroupsAdapter(_NoOptimizer):
    """The reference's form (nerfstudio ``Optimizers``): one torch.optim.Adam per group name, sub-model i's tensor at
    ``param_groups[0]["params"][i]`` (sgn_splatfacto.py:459-511 index it with ``_model_idx_in_scene_graph``)."""

    def __init__(self, groups):
        self.groups = groups
        self._new_state = {}
        self._row_state = {}

    def _state(self, k: int, i: int):
        opt = self.groups[PARAM_NAMES[k]]
        return opt, opt.state.get(opt.param_groups[0]["params"][i], {})

    def relayout(self, new, changed, rows=None):
        src, dst = [], []
        for i, ch in enumerate(changed):
            states = [self._state(k, i)[1] for k in range(6)] if ch else []
            if not ch or not all("exp_avg" in st for st in states):  # unchanged, or never stepped: nothing to carry
                src.append(None)
                dst.append(None)
                continue
            src.append([(st["exp_avg"], st["exp_avg_sq"]) for st in states])
            dst.append([(torch.empty_like(t), torch.empty_like(t)) for t in new[i]])
            self._new_state[i] = dst[-1]
        self._row_state = {}
        for name, ts in (rows or {}).items():  # a row group with its own Adam in the dict ("semantic"): carried likewise
            if name not in self.groups:
                continue
            opt = self.groups[name]
            for i, ch in enumerate(changed):
                st = opt.state.get(opt.param_groups[0]["params"][i], {}) if ch else {}
                if "exp_avg" in st:
                    self._row_state[(name, i)] = ((st["exp_avg"], st["exp_avg_sq"]),
                                                  (torch.empty_like(ts[i]), torch.empty_like(ts[i])))
        return src, dst

    def row_moments(self, name: str, sub: int):
        return self._row_state.get((name, sub), (None, None))

    def commit(self, params, changed, rows=None):
        for name, ts in (rows or {}).items():
            if name not in self.groups:
                continue
            opt = self.groups[name]
            plist = opt.param_groups[0]["params"]
            for i, ch in enumerate(changed):
                if not ch:
                    continue
                st = opt.state.pop(plist[i], {})
                moved = self._row_state.get((name, i))
                if moved is not None:
                    st = dict(st)
                    st["exp_avg"], st["exp_avg_sq"] = moved[1]
                plist[i] = ts[i]
                if st:
                    opt.state[ts[i]] = st
        self._row_state = {}
        for i, ch in enumerate(changed):
            if not ch:
                continue
            for k in range(6):
                opt, st = self._state(k, i)
                plist = opt.param_groups[0]["params"]
                opt.state.pop(plist[i], None)
                if i in self._new_state:
                    st = dict(st)
                    st["exp_avg"], st["exp_avg_sq"] = self._new_state[i][k]
                plist[i] = params[i][k]
                if st:
                    opt.state[params[i][k]] = st
        self._new_state = {}

    def zero_moments(self, sub: int, k: int):
        _, st = self._state(k, sub)
        if "exp_avg" in st:
            st["exp_avg"] = torch.zeros_like(st["exp_avg"])
            st["exp_avg_sq"] = torch.zeros_like(st["exp_avg_sq"])

    def moments(self, sub: int):
        states = [self._state(k, sub)[1] for k in range(6)]
        if "semantic" in self.groups:
            opt = self.groups["semantic"]
            states.append(opt.state.get(opt.param_groups[0]["params"][sub], {}))
        return [(st["exp_avg"], st["exp_avg_sq"]) for st in states if "exp_avg" in st]


def _optimizer_adapter(optimizers, num_submodels: int):
    from .optim import FusedAdam
    if optimizers is None:
        return _NoOptimizer()
    if isinstance(optimizers, FusedAdam):
        assert optimizers.num_segments == num_submodels, "FusedAdam must be built over model.optimizer_params()"
        return _FusedAdamAdapter(optimizers)
    groups = getattr(optimizers, "optimizers", optimizers)
    assert all(k in groups for k in PARAM_NAMES), f"expected Adam optimizers for the groups {PARAM_NAMES}"
    return _TorchAdamGroupsAdapter(groups)


def _gauss_window(size: int, sigma: float, device, dtype):
    x = torch.arange(size, device=device, dtype=dtype) - size // 2
    g = torch.exp(-(x ** 2) / (2 * sigma ** 2))
    return (g / g.sum())


def ssim(x: torch.Tensor, y: torch.Tensor, data_range: float = 1.0, size: int = 11, sigma: float = 1.5) -> torch.Tensor:
    """pytorch_msssim.SSIM(data_range=1.0, size_average=True, channel=3) as the reference configures it
    (sgn_splatfacto.py:393): separable 11-tap Gaussian, valid padding, mean over the map."""
    C = x.shape[1]
    w = _gauss_window(size, sigma, x.device, x.dtype)
    wh = w.view(1, 1, size, 1).repeat(C, 1, 1, 1)
    ww = w.view(1, 1, 1, size).repeat(C, 1, 1, 1)

    def filt(t):
        return F.conv2d(F.conv2d(t, wh, groups=C), ww, groups=C)

    K1, K2 = 0.01, 0.03
    C1, C2 = (K1 * data_range) ** 2, (K2 * data_range) ** 2
    mu1, mu2 = filt(x), filt(y)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1 = filt(x * x) - mu1_sq
    s2 = filt(y * y) - mu2_sq
    s12 = filt(x * y) - mu12
    cs_map = (2 * s12 + C2) / (s1 + s2 + C2)
    ssim_map = ((2 * mu12 + C1) / (mu1_sq + mu2_sq + C1)) * cs_map
    return ssim_map.flatten(2).mean(-1).mean()
