"""Learnable sky cube map on the library's kernels (csrc/sky.cu): the reference's ``EnvLight`` (sgn_splatfacto.py:109-150,
``use_sky_sphere = True`` by default) without nvdiffrast.

    model = SceneGraphRasterModel(background, actors, config, poses_at, sky=CubeMapSky())
    opt = FusedAdam(model.optimizer_params(), extra={"sky": (model.env_map.base, 0.005)})   # sgn_config.py:72-75

``CubeMapSky.base`` is the reference's parameter (``env_map.base`` [6, R, R, 3], initialised to 0.5), so checkpoints load
either way.  ``forward(camera, train)`` returns the [H, W, 3] sky; in training the per-pixel jitter is drawn with two
``torch.rand`` calls of [H, W] on the current CUDA generator (u's first), as ``EnvLight.get_world_directions`` draws it, so a
seeded run consumes the generator exactly as the reference does.  The gradient for ``base`` uses float atomics: it is not
bit-reproducible, with or without ``RenderSettings.deterministic``."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
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
                want_dirs: bool = False):
    """(sky [H, W, 3], dirs [H, W, 3] or None) through sgn_sky_fwd."""
    R = _check_tex(tex)
    tex = tex.contiguous()
    sky = torch.empty(cs.height, cs.width, 3, device=tex.device)
    dirs = torch.empty_like(sky) if want_dirs else None
    _lib.check(_lib.load().sgn_sky_fwd(C.byref(cs), _ptr(ju), _ptr(jv), _ptr(tex), R, _ptr(sky), _ptr(dirs), _stream()), "sgn_sky_fwd")
    return sky, dirs


def sky_backward(cs: _lib.CameraStruct, R: int, ju, jv, v_sky: torch.Tensor, device) -> torch.Tensor:
    v_tex = torch.zeros(6, R, R, 3, device=device)
    _lib.check(_lib.load().sgn_sky_bwd(C.byref(cs), _ptr(ju), _ptr(jv), R, _ptr(v_sky.contiguous()), _ptr(v_tex), _stream()),
               "sgn_sky_bwd")
    return v_tex


class _CubeMapSky(torch.autograd.Function):
    @staticmethod
    def forward(ctx, base: torch.Tensor, cs: _lib.CameraStruct, ju, jv):
        sky, _ = sky_forward(cs, base.detach(), ju, jv)
        ctx.cs, ctx.R, ctx.device = cs, int(base.shape[1]), base.device
        ctx.save_for_backward(*(t for t in (ju, jv) if t is not None))
        return sky

    @staticmethod
    def backward(ctx, v_sky):
        saved = ctx.saved_tensors
        ju, jv = (saved[0], saved[1]) if saved else (None, None)
        v_tex = sky_backward(ctx.cs, ctx.R, ju, jv, v_sky, ctx.device) if ctx.needs_input_grad[0] else None
        return v_tex, None, None, None


class CubeMapSky(torch.nn.Module):
    """Drop-in replacement of the reference's ``EnvLight`` on this library's kernels (see the module docstring)."""

    def __init__(self, resolution: int = 1024):
        super().__init__()
        self.base = torch.nn.Parameter(0.5 * torch.ones(6, resolution, resolution, 3))

    def jitter(self, camera: Camera):
        """The two training draws of EnvLight.get_world_directions: torch.rand_like(u), then torch.rand_like(v), [H, W]."""
        ju = torch.rand(camera.height, camera.width, device=self.base.device)
        jv = torch.rand(camera.height, camera.width, device=self.base.device)
        return ju, jv

    def forward(self, camera: Camera, train: bool = False) -> torch.Tensor:
        ju, jv = self.jitter(camera) if train else (None, None)
        return _CubeMapSky.apply(self.base, camera_struct(camera, RenderSettings()), ju, jv)


def cube_texture(tex: torch.Tensor, uv: torch.Tensor) -> torch.Tensor:
    """The sampler on given directions: tex [6, R, R, 3], uv [..., 3] float32 CUDA -> [..., 3], differentiable in tex."""
    return _CubeTexture.apply(tex, uv)


class _CubeTexture(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tex, uv):
        R = _check_tex(tex)
        uv = uv.detach().contiguous()
        if not (uv.is_cuda and uv.dtype == torch.float32 and uv.shape[-1] == 3):
            raise _lib.SgnError(f"uv must be a CUDA float32 [..., 3] tensor, got {tuple(uv.shape)} {uv.dtype} on {uv.device}")
        out = torch.empty_like(uv)
        P = uv.numel() // 3
        _lib.check(_lib.load().sgn_cube_texture_fwd(P, _ptr(uv), _ptr(tex.detach().contiguous()), R, _ptr(out), _stream()),
                   "sgn_cube_texture_fwd")
        ctx.save_for_backward(uv)
        ctx.R, ctx.P = R, P
        return out

    @staticmethod
    def backward(ctx, v_out):
        (uv,) = ctx.saved_tensors
        v_tex = None
        if ctx.needs_input_grad[0]:
            v_tex = torch.zeros(6, ctx.R, ctx.R, 3, device=uv.device)
            _lib.check(_lib.load().sgn_cube_texture_bwd(ctx.P, _ptr(uv), ctx.R, _ptr(v_out.contiguous()), _ptr(v_tex), _stream()),
                       "sgn_cube_texture_bwd")
        return v_tex, None
