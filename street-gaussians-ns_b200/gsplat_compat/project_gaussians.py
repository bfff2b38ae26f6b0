"""gsplat.project_gaussians.project_gaussians (call site street_gaussians_ns/sgn_splatfacto.py:860-873)."""
import ctypes as C
from typing import Tuple

import torch
from torch.autograd import Function

from .. import _lib
from ._common import camera_struct, need_cuda, ptr, stream


def project_gaussians(means3d, scales, glob_scale: float, quats, viewmat, fx: float, fy: float, cx: float, cy: float,
                      img_height: int, img_width: int, block_width: int, clip_thresh: float = 0.01) -> Tuple:
    """-> (xys[N,2], depths[N], radii[N] int32, conics[N,3], compensation[N], num_tiles_hit[N] int32, cov3d[N,6]).
    Differentiable w.r.t. means3d, scales and quats (through xys, depths, conics and compensation: the antialiased
    mode's ``opacities * comp[:, None]`` trains the geometry through comp, as gsplat's does)."""
    assert block_width > 1 and block_width <= 16, "block_width must be between 2 and 16"
    assert (quats.norm(dim=-1) - 1 < 1e-6).all(), "quats must be normalized"
    return _ProjectGaussians.apply(means3d.contiguous(), scales.contiguous(), glob_scale, quats.contiguous(), viewmat,
                                   fx, fy, cx, cy, img_height, img_width, block_width, clip_thresh)


class _ProjectGaussians(Function):
    @staticmethod
    def forward(ctx, means3d, scales, glob_scale, quats, viewmat, fx, fy, cx, cy, img_height, img_width, block_width,
                clip_thresh):
        L = _lib.load()
        means3d, scales, quats = need_cuda(means3d, "means3d"), need_cuda(scales, "scales"), need_cuda(quats, "quats")
        N = means3d.shape[0]
        if means3d.shape != (N, 3) or scales.shape != (N, 3) or quats.shape != (N, 4):
            raise ValueError("means3d/scales must be (N,3) and quats (N,4)")
        dev = means3d.device
        cs = camera_struct(viewmat, fx, fy, cx, cy, img_height, img_width, block_width, clip_thresh)
        xys = torch.empty(N, 2, device=dev)
        depths = torch.empty(N, device=dev)
        radii = torch.empty(N, device=dev, dtype=torch.int32)
        conics = torch.empty(N, 3, device=dev)
        comp = torch.empty(N, device=dev)
        tiles = torch.empty(N, device=dev, dtype=torch.int32)
        cov3d = torch.empty(N, 6, device=dev)
        _lib.check(L.sgn_l1_project_fwd(N, ptr(means3d), ptr(scales), float(glob_scale), ptr(quats), C.byref(cs), ptr(xys),
                                        ptr(depths), ptr(radii), ptr(conics), ptr(comp), ptr(tiles), ptr(cov3d), stream()),
                   "sgn_l1_project_fwd")
        ctx.cs, ctx.glob_scale = cs, float(glob_scale)
        ctx.save_for_backward(means3d, scales, quats, radii)
        ctx.mark_non_differentiable(radii, tiles)
        ctx.set_materialize_grads(False)
        return xys, depths, radii, conics, comp, tiles, cov3d

    @staticmethod
    def backward(ctx, v_xys, v_depths, v_radii, v_conics, v_comp, v_tiles, v_cov3d):
        L = _lib.load()
        means3d, scales, quats, radii = ctx.saved_tensors
        N = means3d.shape[0]
        c = lambda t: None if t is None else t.contiguous()
        v_xys, v_depths, v_conics = c(v_xys), c(v_depths), c(v_conics)
        v_means, v_scales, v_quats = torch.empty_like(means3d), torch.empty_like(scales), torch.empty_like(quats)
        if v_comp is None:
            _lib.check(L.sgn_l1_project_bwd(N, ptr(means3d), ptr(scales), ctx.glob_scale, ptr(quats), C.byref(ctx.cs), ptr(radii),
                                            ptr(v_xys), ptr(v_depths), ptr(v_conics), ptr(v_means), ptr(v_scales), ptr(v_quats),
                                            stream()), "sgn_l1_project_bwd")
        else:  # compensation was used (the antialiased mode): its cotangent reaches the geometry through cov2d
            v_comp = v_comp.contiguous()
            _lib.check(L.sgn_l1_project_bwd_comp(N, ptr(means3d), ptr(scales), ctx.glob_scale, ptr(quats), C.byref(ctx.cs),
                                                 ptr(radii), ptr(v_xys), ptr(v_depths), ptr(v_conics), ptr(v_comp), ptr(v_means),
                                                 ptr(v_scales), ptr(v_quats), stream()), "sgn_l1_project_bwd_comp")
        return (v_means, v_scales, None, v_quats) + (None,) * 9
