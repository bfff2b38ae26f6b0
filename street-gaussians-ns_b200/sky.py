"""Learnable sky cube map on the library's kernels (csrc/sky.cu): the reference's ``EnvLight`` (sgn_splatfacto.py:109-150,
``use_sky_sphere = True`` by default) without nvdiffrast.

    model = SceneGraphRasterModel(background, actors, config, poses_at, sky=CubeMapSky())
    opt = FusedAdam(model.optimizer_params(), extra={"sky": (model.env_map.base, 0.005)})   # sgn_config.py:72-75

``CubeMapSky.base`` is the reference's parameter (``env_map.base`` [6, R, R, 3], initialised to 0.5), so checkpoints load
either way.  ``forward(camera, train)`` returns the [H, W, 3] sky; in training the per-pixel jitter is drawn with two
``torch.rand`` calls of [H, W] on the current CUDA generator (u's first), as ``EnvLight.get_world_directions`` draws it, so a
seeded run consumes the generator exactly as the reference does.

The gradient for ``base`` uses float atomics by default.  In deterministic mode -- ``CubeMapSky(deterministic=True)``, or
``deterministic=None`` (the default) with the switch the blend reads, ``raster.DETERMINISTIC`` (``SGN_DETERMINISTIC=1``),
looked up when the backward runs -- it goes through ``sgn_sky_bwd_det``: every addend is rounded once to 64-bit fixed point
(2^32 units per unit of the largest cotangent) and added as an integer, so the gradient is bit-identical from run to run.
The same holds for ``cube_texture`` (and so ``nvdiffrast_compat.texture``).  The fixed-point scratch, int64 [6, R, R, 3]
(151 MB at R = 1024), comes from torch's caching allocator for the duration of the backward.

The lookup is also differentiable in its direction, as nvdiffrast's ``dr.texture`` is in ``uv``: ``cube_texture`` returns
the uv gradient when ``uv`` requires one, and ``CubeMapSky(view_grad=True)`` gives a device ``view`` that requires a
gradient (a ``camera_pose.CameraPoseOptimizer``'s) the sky's share of its rotation cotangent, in the same launch as the
texture gradient (sgn_sky_bwd_view_rot).  That is the reference's chain: ``EnvLight.forward`` looks up
``c2w[:3,:3] @ normalize(d)`` with a ``c2w`` that is not detached.  The switch is off by default: the view is then detached
and the launches and results are those of the texture-only backward."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib, raster
from .raster import RenderSettings, camera_struct
from .scene import Camera


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check_tex(tex: torch.Tensor) -> int:
    if not (tex.is_cuda and tex.dtype == torch.float32 and tex.dim() == 4 and tex.shape[0] == 6 and tex.shape[1] == tex.shape[2]
            and tex.shape[3] == 3):
        raise _lib.SgnError(f"the cube map must be a CUDA float32 [6, R, R, 3] tensor, got {tuple(tex.shape)} {tex.dtype} on {tex.device}")
    return int(tex.shape[1])


def sky_forward(cs: _lib.CameraStruct, tex: torch.Tensor, ju: Optional[torch.Tensor], jv: Optional[torch.Tensor],
                want_dirs: bool = False, view: Optional[torch.Tensor] = None):
    """(sky [H, W, 3], dirs [H, W, 3] or None) through sgn_sky_fwd -- or sgn_sky_fwd_view, with the camera's rotation taken
    from ``view`` (a device view, raster.check_view)."""
    R = _check_tex(tex)
    tex = tex.contiguous()
    sky = torch.empty(cs.height, cs.width, 3, device=tex.device)
    dirs = torch.empty_like(sky) if want_dirs else None
    L = _lib.load()
    if view is not None:
        _lib.check(L.sgn_sky_fwd_view(C.byref(cs), _ptr(view), _ptr(ju), _ptr(jv), _ptr(tex), R, _ptr(sky), _ptr(dirs), _stream()),
                   "sgn_sky_fwd_view")
    else:
        _lib.check(L.sgn_sky_fwd(C.byref(cs), _ptr(ju), _ptr(jv), _ptr(tex), R, _ptr(sky), _ptr(dirs), _stream()), "sgn_sky_fwd")
    return sky, dirs


def _deterministic(flag: Optional[bool]) -> bool:
    return raster.DETERMINISTIC if flag is None else flag


def _det_scratch(R: int, device) -> torch.Tensor:
    """Device scratch of sgn_sky_det_scratch_bytes(R) bytes (the library zeroes it itself)."""
    return torch.empty(_lib.load().sgn_sky_det_scratch_bytes(R), dtype=torch.uint8, device=device)


def sky_backward_rot(cs: _lib.CameraStruct, tex: torch.Tensor, ju, jv, v_sky: torch.Tensor, view: torch.Tensor, want_tex: bool = True,
                     deterministic: Optional[bool] = None):
    """(v_tex [6, R, R, 3] or None, v_view [15]) through sgn_sky_bwd_view_rot, or sgn_sky_bwd_det_view_rot when
    ``deterministic``: the texture gradient of sky_backward(view=view) and the view's cotangent from the sky's dependence on
    the rotation (viewmat[:, :3]; the translation and cam_pos entries are 0).  ``want_tex`` False skips the texture gradient."""
    R = _check_tex(tex)
    L = _lib.load()
    device = tex.device
    v_tex = torch.zeros(6, R, R, 3, device=device) if want_tex else None
    v_view = torch.zeros(raster.VIEW_LEN, device=device)
    v_sky = v_sky.contiguous()
    tex = tex.contiguous()
    partials = torch.empty(L.sgn_sky_rot_scratch_bytes(cs.width, cs.height) // 4, device=device)
    if _deterministic(deterministic) and want_tex:
        scratch = _det_scratch(R, device)
        _lib.check(L.sgn_sky_bwd_det_view_rot(C.byref(cs), _ptr(view), _ptr(ju), _ptr(jv), _ptr(tex), R, _ptr(v_sky), _ptr(v_tex),
                                              _ptr(scratch), scratch.numel(), _ptr(partials), 4 * partials.numel(), _ptr(v_view),
                                              _stream()), "sgn_sky_bwd_det_view_rot")
    else:
        _lib.check(L.sgn_sky_bwd_view_rot(C.byref(cs), _ptr(view), _ptr(ju), _ptr(jv), _ptr(tex), R, _ptr(v_sky), _ptr(v_tex),
                                          _ptr(partials), 4 * partials.numel(), _ptr(v_view), _stream()), "sgn_sky_bwd_view_rot")
    return v_tex, v_view


def sky_backward(cs: _lib.CameraStruct, R: int, ju, jv, v_sky: torch.Tensor, device, deterministic: Optional[bool] = None,
                 view: Optional[torch.Tensor] = None) -> torch.Tensor:
    """v_tex [6, R, R, 3] through sgn_sky_bwd, or sgn_sky_bwd_det when ``deterministic`` (None: raster.DETERMINISTIC); the
    ``_view`` entry points when ``view`` is given (as in sky_forward)."""
    L = _lib.load()
    v_tex = torch.zeros(6, R, R, 3, device=device)
    v_sky = v_sky.contiguous()
    if _deterministic(deterministic):
        scratch = _det_scratch(R, device)
        if view is not None:
            _lib.check(L.sgn_sky_bwd_det_view(C.byref(cs), _ptr(view), _ptr(ju), _ptr(jv), R, _ptr(v_sky), _ptr(v_tex), _ptr(scratch),
                                              scratch.numel(), _stream()), "sgn_sky_bwd_det_view")
        else:
            _lib.check(L.sgn_sky_bwd_det(C.byref(cs), _ptr(ju), _ptr(jv), R, _ptr(v_sky), _ptr(v_tex), _ptr(scratch), scratch.numel(),
                                         _stream()), "sgn_sky_bwd_det")
    elif view is not None:
        _lib.check(L.sgn_sky_bwd_view(C.byref(cs), _ptr(view), _ptr(ju), _ptr(jv), R, _ptr(v_sky), _ptr(v_tex), _stream()),
                   "sgn_sky_bwd_view")
    else:
        _lib.check(L.sgn_sky_bwd(C.byref(cs), _ptr(ju), _ptr(jv), R, _ptr(v_sky), _ptr(v_tex), _stream()), "sgn_sky_bwd")
    return v_tex


class _CubeMapSky(torch.autograd.Function):
    @staticmethod
    def forward(ctx, base: torch.Tensor, cs: _lib.CameraStruct, ju, jv, deterministic: Optional[bool], view: Optional[torch.Tensor]):
        if view is not None:
            view = raster.check_view(view, base.device)
        sky, _ = sky_forward(cs, base.detach(), ju, jv, view=view)
        ctx.cs, ctx.R, ctx.device, ctx.deterministic, ctx.view = cs, int(base.shape[1]), base.device, deterministic, view
        # a view that requires a gradient (CubeMapSky(view_grad=True)) also needs the map's texels in the backward
        ctx.rot = view is not None and ctx.needs_input_grad[5]
        ctx.save_for_backward(*(t for t in (ju, jv) if t is not None), *((base,) if ctx.rot else ()))
        return sky

    @staticmethod
    def backward(ctx, v_sky):
        saved = ctx.saved_tensors
        ju, jv = (saved[0], saved[1]) if len(saved) >= 2 else (None, None)
        if ctx.rot:
            v_tex, v_view = sky_backward_rot(ctx.cs, saved[-1].detach(), ju, jv, v_sky, ctx.view, ctx.needs_input_grad[0],
                                             ctx.deterministic)
            return v_tex, None, None, None, None, v_view
        v_tex = sky_backward(ctx.cs, ctx.R, ju, jv, v_sky, ctx.device, ctx.deterministic, ctx.view) if ctx.needs_input_grad[0] else None
        return v_tex, None, None, None, None, None  # the view is detached unless CubeMapSky(view_grad=True)


class CubeMapSky(torch.nn.Module):
    """Drop-in replacement of the reference's ``EnvLight`` on this library's kernels (see the module docstring)."""

    def __init__(self, resolution: int = 1024, deterministic: Optional[bool] = None, view_grad: bool = False):
        """``deterministic``: the fixed-point gradient (True), float atomics (False), or None: whatever ``raster.DETERMINISTIC``
        says when the backward runs.  ``view_grad``: give a ``view`` that requires a gradient the sky's share of it (the
        rotation cotangent, sgn_sky_bwd_view_rot); off, the view is detached, as before."""
        super().__init__()
        self.base = torch.nn.Parameter(0.5 * torch.ones(6, resolution, resolution, 3))
        self.deterministic = deterministic
        self.view_grad = bool(view_grad)

    def jitter(self, camera: Camera):
        """The two training draws of EnvLight.get_world_directions: torch.rand_like(u), then torch.rand_like(v), [H, W]."""
        ju = torch.rand(camera.height, camera.width, device=self.base.device)
        jv = torch.rand(camera.height, camera.width, device=self.base.device)
        return ju, jv

    def forward(self, camera: Camera, train: bool = False, view: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``view``: a device view (raster.render_frame's ``view``) whose rotation orients the sky in place of the camera's, so
        that a corrected camera sees geometry and sky alike.  The sky gives the view a gradient only with ``view_grad``."""
        ju, jv = self.jitter(camera) if train else (None, None)
        if view is not None and not self.view_grad:
            view = view.detach()
        return _CubeMapSky.apply(self.base, camera_struct(camera, RenderSettings()), ju, jv, self.deterministic, view)


def cube_texture(tex: torch.Tensor, uv: torch.Tensor, deterministic: Optional[bool] = None) -> torch.Tensor:
    """The sampler on given directions: tex [6, R, R, 3], uv [..., 3] float32 CUDA -> [..., 3], differentiable in tex and
    in uv (nvdiffrast's uv gradient, sgn_cube_texture_bwd_uv, when uv requires one).  ``deterministic`` selects the texture
    gradient as in ``CubeMapSky`` (None: raster.DETERMINISTIC at backward time); the uv gradient is bit-reproducible."""
    return _CubeTexture.apply(tex, uv, deterministic)


class _CubeTexture(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tex, uv, deterministic: Optional[bool] = None):
        R = _check_tex(tex)
        uv = uv.detach().contiguous()
        if not (uv.is_cuda and uv.dtype == torch.float32 and uv.shape[-1] == 3):
            raise _lib.SgnError(f"uv must be a CUDA float32 [..., 3] tensor, got {tuple(uv.shape)} {uv.dtype} on {uv.device}")
        out = torch.empty_like(uv)
        P = uv.numel() // 3
        _lib.check(_lib.load().sgn_cube_texture_fwd(P, _ptr(uv), _ptr(tex.detach().contiguous()), R, _ptr(out), _stream()),
                   "sgn_cube_texture_fwd")
        ctx.save_for_backward(uv, *((tex,) if ctx.needs_input_grad[1] else ()))
        ctx.R, ctx.P, ctx.deterministic = R, P, deterministic
        return out

    @staticmethod
    def backward(ctx, v_out):
        if ctx.needs_input_grad[1]:
            return _CubeTexture.backward_uv(ctx, v_out)
        (uv,) = ctx.saved_tensors
        v_tex = None
        if ctx.needs_input_grad[0]:
            L = _lib.load()
            v_tex = torch.zeros(6, ctx.R, ctx.R, 3, device=uv.device)
            v_out = v_out.contiguous()
            if _deterministic(ctx.deterministic):
                scratch = _det_scratch(ctx.R, uv.device)
                _lib.check(L.sgn_cube_texture_bwd_det(ctx.P, _ptr(uv), ctx.R, _ptr(v_out), _ptr(v_tex), _ptr(scratch), scratch.numel(),
                                                      _stream()), "sgn_cube_texture_bwd_det")
            else:
                _lib.check(L.sgn_cube_texture_bwd(ctx.P, _ptr(uv), ctx.R, _ptr(v_out), _ptr(v_tex), _stream()), "sgn_cube_texture_bwd")
        return v_tex, None, None

    @staticmethod
    def backward_uv(ctx, v_out):
        """Both gradients from one launch: sgn_cube_texture_bwd_uv (or _det for the texture gradient)."""
        uv, tex = ctx.saved_tensors
        L = _lib.load()
        want_tex = ctx.needs_input_grad[0]
        v_tex = torch.zeros(6, ctx.R, ctx.R, 3, device=uv.device) if want_tex else None
        v_uv = torch.empty_like(uv)
        v_out = v_out.contiguous()
        tex = tex.detach().contiguous()
        if want_tex and _deterministic(ctx.deterministic):
            scratch = _det_scratch(ctx.R, uv.device)
            _lib.check(L.sgn_cube_texture_bwd_uv_det(ctx.P, _ptr(uv), _ptr(tex), ctx.R, _ptr(v_out), _ptr(v_tex), _ptr(v_uv), _ptr(scratch),
                                                     scratch.numel(), _stream()), "sgn_cube_texture_bwd_uv_det")
        else:
            _lib.check(L.sgn_cube_texture_bwd_uv(ctx.P, _ptr(uv), _ptr(tex), ctx.R, _ptr(v_out), _ptr(v_tex), _ptr(v_uv), _stream()),
                       "sgn_cube_texture_bwd_uv")
        return v_tex, v_uv, None
