"""nvdiffrast-compatible ``texture`` for the calls the reference makes (Level-1 drop-in backed by csrc/sky.cu).

The reference uses one nvdiffrast function (street_gaussians_ns/sgn_splatfacto.py:22, 147):

    import nvdiffrast.torch as dr
    light = dr.texture(self.base[None, ...], l, filter_mode='linear', boundary_mode='cube')

with ``base`` [6, R, R, 3] and ``l`` [1, H, W, 3] (or [1, 1, P, 3]).  ``texture`` serves exactly those call shapes, with the
gradient for the texture; anything else -- mip filtering, other boundary modes, a channel count other than 3, a batch other
than 1 -- raises ``NotImplementedError``.  ``install()`` registers this package as ``nvdiffrast`` and ``nvdiffrast.torch``
in ``sys.modules``, so the reference's model source runs unmodified.

Directions that require a gradient (``l`` depends on a ``camera_to_worlds`` that trains, as under nerfstudio's camera
optimizer) raise as well, unless the shim is installed with ``install(uv_grad=True)``: then the registered ``texture``
returns nvdiffrast's uv gradient for them too (sky.cube_texture, sgn_cube_texture_bwd_uv).
"""
import functools
import sys
import types

import torch

from ..sky import cube_texture


def texture(tex: torch.Tensor, uv: torch.Tensor, uv_da=None, mip_level_bias=None, mip=None, filter_mode: str = "auto",
            boundary_mode: str = "wrap", max_mip_level=None, *, uv_grad: bool = False) -> torch.Tensor:
    """``uv_grad``: accept a ``uv`` that requires a gradient and return its gradient (``install(uv_grad=True)`` sets it)."""
    if filter_mode != "linear":
        raise NotImplementedError(f"nvdiffrast_compat.texture: filter_mode={filter_mode!r} (only 'linear' is implemented)")
    if boundary_mode != "cube":
        raise NotImplementedError(f"nvdiffrast_compat.texture: boundary_mode={boundary_mode!r} (only 'cube' is implemented)")
    if uv_da is not None or mip_level_bias is not None or mip is not None or max_mip_level is not None:
        raise NotImplementedError("nvdiffrast_compat.texture: mip-mapping is not implemented")
    if tex.dim() != 5 or tex.shape[0] != 1 or tex.shape[1] != 6 or tex.shape[2] != tex.shape[3] or tex.shape[4] != 3:
        raise NotImplementedError(f"nvdiffrast_compat.texture: tex must be [1, 6, R, R, 3], got {tuple(tex.shape)}")
    if uv.dim() != 4 or uv.shape[0] != 1 or uv.shape[3] != 3:
        raise NotImplementedError(f"nvdiffrast_compat.texture: uv must be [1, H, W, 3], got {tuple(uv.shape)}")
    if uv.requires_grad and not uv_grad:
        raise NotImplementedError("nvdiffrast_compat.texture: no gradient for uv (install(uv_grad=True) provides it)")
    return cube_texture(tex[0], uv)


def install(name: str = "nvdiffrast", uv_grad: bool = False) -> None:
    """Make ``import nvdiffrast.torch as dr`` resolve to this shim; ``uv_grad``: its ``texture`` is differentiable in uv."""
    pkg, sub = types.ModuleType(name), types.ModuleType(name + ".torch")
    sub.texture = pkg.texture = functools.partial(texture, uv_grad=True) if uv_grad else texture
    pkg.torch = sub
    sys.modules[name], sys.modules[name + ".torch"] = pkg, sub
