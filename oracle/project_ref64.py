"""Float64 statement of the projection stage (compose + EWA projection + SH / Fourier colour + sigmoid + tile AABB + touch
test), forward and backward.  TEST INFRASTRUCTURE -- never imported by the product.

Written from the specification, not from csrc/project.cu or oracle/sgn_oracle.c:
  * compose / pre-ops (the lines cited in include/sgn_raster.h): world mean R m + t, quaternion q_box * q (Hamilton, w first),
    Fourier DC sum_f dc_f idft_f, scale exp(log s), quaternion normalised;
  * gsplat project_gaussians (SURVEY Appendix A.1-A.4, the sgn_exact.cuh header): view point p = W[:, :3] m + W[:, 3],
    near-plane clip z <= clip_thresh, J at the FOV-clamped (tx, ty) = z * clamp(p / z, +-lim), cov2d = J W S W^T J^T + 0.3 I,
    conic = inverse, radius = ceil(3 sqrt(lambda_max)) with the discriminant floored at 0.1, xy = p (f / (z + 1e-6)) + c,
    tile AABB by truncation, visible iff the AABB is not empty;
  * colour (Appendix A.7, sgn_splatfacto.py:933-949): SH of degree sh_degree_to_use over the first (deg_use+1)^2 coefficients,
    view direction (world mean - camera position) DETACHED, + 0.5 clamped at 0; at sh_degree 0 a sigmoid of the DC colour;
    sigmoid opacity;
  * touch test (sgn_touch.cuh header): a tile of the AABB matters iff min sigma over the rectangle spanned by its pixel centres
    (clipped to the image) is <= tau = ln(255 o).

``forward`` returns every record field, radii, tile_bbox, num_tiles_hit, the aux bits, and for every decision its relative
distance from the threshold (``margins``).  ``backward`` is torch float64 autograd of the same forward for given v_records,
deliberately independent of the hand-derived VJP.  With ``dtype=torch.float32`` (and the spec exp, oracle_torch.expf_spec) the
same code gives an fp32 evaluation whose distance from the float64 one is the per-case fp32 noise scale of the bars.
``l1_project`` / ``l1_project_bwd`` / ``l1_sh`` state gsplat's project_gaussians and spherical_harmonics on plain arrays.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np
import torch

from oracle.oracle_torch import expf_spec

AUX_OBJECT = 8
AUX_VISIBLE = 16
MARGIN_NAMES = ("near", "fovx", "fovy", "disc", "ceil", "tmin_x", "tmin_y", "tmax_x", "tmax_y", "area", "pre")

_Y0 = 0.28209479177387814
_Y1 = 0.4886025119029199
_Y2 = (1.0925484305920792, 0.31539156525252005, 0.5462742152960396)
_Y3 = (0.5900435899266435, 2.890611442640554, 0.4570457994644658, 0.3731763325901154, 1.445305721320277)


@dataclass
class Settings:
    sh_degree: int = 3
    sh_degree_to_use: Optional[int] = None
    block_width: int = 16
    clip_thresh: float = 0.01

    @property
    def deg_use(self) -> int:
        return self.sh_degree if self.sh_degree_to_use is None else self.sh_degree_to_use


def sh_basis(deg: int, d: torch.Tensor) -> torch.Tensor:
    """Real SH basis of gsplat (Appendix A.7) up to degree ``deg`` at directions d[N,3] -> [N,16] (zeros above deg)."""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    Y = [torch.full_like(x, _Y0)] + [torch.zeros_like(x)] * 15
    if deg >= 1:
        Y[1], Y[2], Y[3] = -_Y1 * y, _Y1 * z, -_Y1 * x
    if deg >= 2:
        Y[4] = _Y2[0] * x * y
        Y[5] = -_Y2[0] * y * z
        Y[6] = _Y2[1] * (2 * z * z - x * x - y * y)
        Y[7] = -_Y2[0] * x * z
        Y[8] = _Y2[2] * (x * x - y * y)
    if deg >= 3:
        Y[9] = -_Y3[0] * y * (3 * x * x - y * y)
        Y[10] = _Y3[1] * x * y * z
        Y[11] = -_Y3[2] * y * (4 * z * z - x * x - y * y)
        Y[12] = _Y3[3] * z * (2 * z * z - 3 * x * x - 3 * y * y)
        Y[13] = -_Y3[2] * x * (4 * z * z - x * x - y * y)
        Y[14] = _Y3[4] * z * (x * x - y * y)
        Y[15] = -_Y3[0] * x * (x * x - 3 * y * y)
    return torch.stack(Y, -1)


def _rotmat(q):
    w, x, y, z = q.unbind(-1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1).reshape(-1, 3, 3)


def _near_int_margin(v: np.ndarray, lo: int, hi: int) -> np.ndarray:
    """Relative distance of v from the nearest integer threshold in [lo, hi] (trunc-then-clamp changes only there)."""
    k = np.clip(np.round(v), lo, hi)
    return np.abs(v - k) / np.maximum(np.abs(v), 1.0)


def project_core(mw, qr, s, cam, bw: int, clip: float, dtype) -> Dict:
    """gsplat project_gaussians on world means mw[N,3], quaternions qr[N,4] (un-normalised) and linear scales s[N,3]."""
    W = torch.tensor(np.asarray(cam.viewmat(), np.float64), dtype=dtype)
    fx, fy, cx, cy = cam.fx, cam.fy, cam.cx, cam.cy
    limx, limy = cam.fov_limits()
    N = mw.shape[0]
    p = mw @ W[:, :3].T + W[:, 3]
    z = p[:, 2]
    zn = z.detach().double().numpy()
    unclipped = zn > clip
    uc = torch.from_numpy(unclipped)
    zs = torch.where(uc, z, torch.ones_like(z))
    qn = qr / torch.sqrt((qr * qr).sum(-1, keepdim=True))
    M = _rotmat(qn) * s[:, None, :]
    S = M @ M.transpose(1, 2)
    ux, uy = p[:, 0] / zs, p[:, 1] / zs
    uxn, uyn = ux.detach().double().numpy(), uy.detach().double().numpy()
    clampx = np.where(uxn > limx, 1, np.where(uxn < -limx, -1, 0)) * unclipped
    clampy = np.where(uyn > limy, 1, np.where(uyn < -limy, -1, 0)) * unclipped
    tx = zs * torch.where(torch.from_numpy(clampx != 0), torch.from_numpy(clampx * limx).to(dtype), ux)
    ty = zs * torch.where(torch.from_numpy(clampy != 0), torch.from_numpy(clampy * limy).to(dtype), uy)
    zero = torch.zeros_like(zs)
    J = torch.stack([fx / zs, zero, -fx * tx / (zs * zs), zero, fy / zs, -fy * ty / (zs * zs)], -1).reshape(N, 2, 3)
    T = J @ W[:, :3]
    cov = T @ S @ T.transpose(1, 2)
    a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = a * c - b * b
    detn = det.detach().double().numpy()
    ok = unclipped & (detn != 0)
    okt = torch.from_numpy(ok)
    dets = torch.where(okt, det, torch.ones_like(det))
    conic = torch.stack([c / dets, -b / dets, a / dets], -1) * okt[:, None]
    an, bn, cn = (t.detach().double().numpy() for t in (a, b, c))
    bm = 0.5 * (an + cn)
    d2 = bm * bm - detn
    lam = bm + np.sqrt(np.maximum(0.1, d2))
    r = 3.0 * np.sqrt(np.maximum(lam, 0.0))
    radius = np.where(ok, np.ceil(r), 0).astype(np.int64)
    rw = 1.0 / (zs + 1e-6)
    xy = torch.stack([p[:, 0] * rw * fx + cx, p[:, 1] * rw * fy + cy], -1)
    xyn = xy.detach().double().numpy()
    tiles = np.array([(cam.width + bw - 1) // bw, (cam.height + bw - 1) // bw])
    tc, tr = xyn / bw, (radius / bw)[:, None]
    lo_raw, hi_raw = tc - tr, tc + tr + 1.0
    tmin = np.minimum(np.maximum(np.trunc(lo_raw), 0), tiles).astype(np.int64)
    tmax = np.minimum(np.maximum(np.trunc(hi_raw), 0), tiles).astype(np.int64)
    area = (tmax[:, 0] - tmin[:, 0]) * (tmax[:, 1] - tmin[:, 1])
    vis = ok & (area > 0)
    inf = np.full(N, np.inf)
    mg = dict(near=np.abs(zn - clip) / max(clip, 1e-30))
    mg["fovx"] = np.where(unclipped, np.abs(np.abs(uxn) - limx) / limx, inf)
    mg["fovy"] = np.where(unclipped, np.abs(np.abs(uyn) - limy) / limy, inf)
    mg["disc"] = np.where(ok, np.abs(d2 - 0.1) / np.maximum(np.abs(d2), 0.1), inf)
    mg["ceil"] = np.where(ok, np.abs(r - np.round(r)) / np.maximum(r, 1.0), inf)
    for k, (v, ax) in {"tmin_x": (lo_raw, 0), "tmin_y": (lo_raw, 1), "tmax_x": (hi_raw, 0), "tmax_y": (hi_raw, 1)}.items():
        mg[k] = np.where(ok, _near_int_margin(v[:, ax], 1, tiles[ax]), inf)
    # area > 0 is decided by the four truncations above: its margin is the smallest of them
    mg["area"] = np.where(ok, np.minimum.reduce([mg[k] for k in ("tmin_x", "tmin_y", "tmax_x", "tmax_y")]), inf)
    vt = torch.from_numpy(vis)
    return dict(p=p, z=z, xy=xy * vt[:, None], conic=conic, S=S, a=a, b=b, c=c, radius=np.where(vis, radius, 0),
                tmin=np.where(ok[:, None], tmin, 0), tmax=np.where(ok[:, None], tmax, 0), vis=vis, unclipped=unclipped,
                clampx=clampx, clampy=clampy, margins=mg)


def _leaves(seg, dtype, grad):
    return {k: getattr(seg.params, k).detach().cpu().double().to(dtype).clone().requires_grad_(grad)
            for k in ("means", "scales", "quats", "features_dc", "features_rest", "opacities")}


def forward(frame, st: Settings, dtype=torch.float64, grad: bool = False) -> Dict:
    """The fused projection of every segment of ``frame`` (rows concatenated in segment order)."""
    cam = frame.camera
    spec_exp = dtype == torch.float32
    leaves, mws, qrs, lss, fdcs, rests, opl, cls = [], [], [], [], [], [], [], []
    for sg in frame.segments:
        lf = _leaves(sg, dtype, grad)
        leaves.append(lf)
        F = lf["features_dc"].shape[1]
        idft = torch.tensor(sg.idft_f32()[:F].astype(np.float64), dtype=dtype)
        fdcs.append((lf["features_dc"] * idft[None, :, None]).sum(1))
        if sg.has_pose:
            R, t, q = (torch.tensor(x.astype(np.float64), dtype=dtype) for x in sg.pose_f32())
            mws.append(lf["means"] @ R.reshape(3, 3).T + t)
            bw_, bx, by, bz = lf["quats"].unbind(-1)
            aw, ax, ay, az = q
            qrs.append(torch.stack([aw * bw_ - ax * bx - ay * by - az * bz, aw * bx + ax * bw_ + ay * bz - az * by,
                                    aw * by - ax * bz + ay * bw_ + az * bx, aw * bz + ax * by - ay * bx + az * bw_], -1))
        else:
            mws.append(lf["means"])
            qrs.append(lf["quats"])
        lss.append(lf["scales"])
        rests.append(lf["features_rest"])
        opl.append(lf["opacities"][:, 0])
        cls.append(np.full(sg.params.num_points, sg.cls, np.int64))
    mw, qr, ls = torch.cat(mws), torch.cat(qrs), torch.cat(lss)
    fdc, rest, logit = torch.cat(fdcs), torch.cat(rests), torch.cat(opl)
    cls = np.concatenate(cls) if cls else np.zeros(0, np.int64)
    N = mw.shape[0]
    s = expf_spec(ls) if spec_exp else torch.exp(ls)
    pr = project_core(mw, qr, s, cam, st.block_width, st.clip_thresh, dtype)
    vis = pr["vis"]
    vt = torch.from_numpy(vis)
    # colour
    aux = np.where(cls == 1, AUX_OBJECT, 0) | np.where(vis, AUX_VISIBLE, 0)
    pre_margin = np.full(N, np.inf)
    if st.sh_degree > 0:
        cp = torch.tensor(cam.cam_pos().astype(np.float64), dtype=dtype)
        d = mw.detach() - cp
        d = torch.where(vt[:, None], d, torch.ones_like(d))  # a clipped row may sit on the camera centre
        d = d / torch.sqrt((d * d).sum(-1, keepdim=True))
        Y = sh_basis(st.deg_use, d)
        Kuse = (st.deg_use + 1) ** 2
        terms = Y[:, :1, None] * fdc[:, None, :]
        if Kuse > 1:
            terms = torch.cat([terms, Y[:, 1:Kuse, None] * rest[:, :Kuse - 1]], 1)
        pre = terms.sum(1) + 0.5
        pn = pre.detach().double().numpy()
        pass_ = pn >= 0
        rgb = torch.where(torch.from_numpy(pass_), pre, torch.zeros_like(pre))
        scale = np.abs(terms.detach().double().numpy()).sum(1) + 0.5
        pre_margin = np.where(vis, (np.abs(pn) / scale).min(1), np.inf)
        aux = aux | np.where(vis, (pass_ * np.array([1, 2, 4])).sum(1), 0)
    else:
        pn = None
        rgb = torch.sigmoid(fdc)
        aux = aux | np.where(vis, 7, 0)
    opac = torch.sigmoid(logit)
    pr["margins"]["pre"] = pre_margin
    # the 10 differentiable record components; invisible rows hold constants (their colour is never read downstream)
    rec = torch.cat([pr["xy"], pr["conic"] * vt[:, None], (opac * vt)[:, None], rgb * vt[:, None], (pr["z"] * vt)[:, None]], 1)
    recn = np.zeros((N, 12))
    recn[:, :10] = rec.detach().double().numpy()
    recn[:, 2:5] = pr["conic"].detach().double().numpy()  # written for every unclipped row (gsplat writes conics first)
    mg = pr["margins"]
    margin = np.minimum.reduce([mg[k] for k in MARGIN_NAMES]) if N else np.zeros(0)
    return dict(leaves=leaves, rec=rec, records=recn, radii=pr["radius"], tmin=pr["tmin"], tmax=pr["tmax"],
                num_tiles_hit=np.where(vis, (pr["tmax"][:, 0] - pr["tmin"][:, 0]) * (pr["tmax"][:, 1] - pr["tmin"][:, 1]), 0),
                vis=vis, unclipped=pr["unclipped"], aux=aux, cls=cls, clampx=pr["clampx"], clampy=pr["clampy"], pre=pn,
                margins=mg, margin=margin, conic_all=pr["conic"].detach().double().numpy())


def backward(frame, st: Settings, v_records: np.ndarray, dtype=torch.float64) -> List[Dict[str, np.ndarray]]:
    """Gradients of sum(records[:, :10] * v_records[:, :10]) w.r.t. the six parameter tensors of every segment."""
    fw = forward(frame, st, dtype, grad=True)
    v = torch.tensor(np.asarray(v_records, np.float64)[:, :10], dtype=dtype)
    loss = (fw["rec"] * v).sum()
    out = []
    flat = [t for lf in fw["leaves"] for t in lf.values()]
    gs = torch.autograd.grad(loss, flat, allow_unused=True) if flat and loss.requires_grad else [None] * len(flat)
    k = 0
    for lf in fw["leaves"]:
        d = {}
        for name, t in lf.items():
            g = gs[k]
            d[name] = np.zeros(t.shape) if g is None else g.double().numpy()
            k += 1
        out.append(d)
    return out


def touch_min_sigma(xy, conic, opac, tmin, tmax, width, height, bw):
    """For every tile of the AABB [tmin, tmax): (tile x, tile y, min sigma - tau, |terms| at the minimiser), float64, over the
    rectangle spanned by the tile's pixel centres clipped to the image; tau = ln(255 o).  Inputs of one Gaussian."""
    a, b, c = (float(v) for v in conic)
    gx, gy = float(xy[0]), float(xy[1])
    tau = np.log(255.0 * float(opac)) if opac > 0 else -np.inf
    tys, txs = np.meshgrid(np.arange(tmin[1], tmax[1]), np.arange(tmin[0], tmax[0]), indexing="ij")
    txs, tys = txs.reshape(-1), tys.reshape(-1)
    x0 = txs * bw + 0.5 - gx
    x1 = np.minimum(txs * bw + bw, width) - 0.5 - gx
    y0 = tys * bw + 0.5 - gy
    y1 = np.minimum(tys * bw + bw, height) - 0.5 - gy

    def q(dx, dy):
        return 0.5 * a * dx * dx + 0.5 * c * dy * dy + b * dx * dy, 0.5 * abs(a) * dx * dx + 0.5 * abs(c) * dy * dy + abs(b * dx * dy)

    # the minimiser of a convex quadratic over a box: the centre if inside, else on one of the four edges
    best = np.full(txs.shape, np.inf)
    mag = np.zeros(txs.shape)
    inside = (x0 <= 0) & (x1 >= 0) & (y0 <= 0) & (y1 >= 0)
    best[inside] = 0.0
    for xe in (x0, x1):
        dy = np.clip(-b * xe / c, y0, y1)
        v, m = q(xe, dy)
        upd = v < best
        best, mag = np.where(upd, v, best), np.where(upd, m, mag)
    for ye in (y0, y1):
        dx = np.clip(-b * ye / a, x0, x1)
        v, m = q(dx, ye)
        upd = v < best
        best, mag = np.where(upd, v, best), np.where(upd, m, mag)
    return txs, tys, best - tau, mag


# ------------------------------------------------------------------------------------------------------------------
# Level-1: gsplat 0.1.x project_gaussians / spherical_harmonics on plain arrays
# ------------------------------------------------------------------------------------------------------------------
def l1_project(means, scales, glob_scale, quats, cam, bw=16, clip=0.01, dtype=torch.float64, grad=False):
    """project_gaussians(means3d, scales, glob_scale, quats, viewmat, fx, fy, cx, cy, H, W, block_width, clip_thresh):
    xys, depths, radii, conics, compensation, num_tiles_hit, cov3d (cov3d written whenever the Gaussian is not clipped)."""
    m, s, q = (torch.tensor(np.asarray(x, np.float64), dtype=dtype).requires_grad_(grad) for x in (means, scales, quats))
    pr = project_core(m, q, s * glob_scale, cam, bw, clip, dtype)
    vis = pr["vis"]
    vt = torch.from_numpy(vis)
    det_orig = (pr["a"] - 0.3) * (pr["c"] - 0.3) - pr["b"] ** 2
    det_blur = pr["a"] * pr["c"] - pr["b"] ** 2
    comp = np.where(vis, np.sqrt(np.maximum(0.0, (det_orig / det_blur).detach().double().numpy())), 0.0)
    iu = [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]
    cov3d = pr["S"][:, iu[0], iu[1]].detach().double().numpy() * pr["unclipped"][:, None]
    return dict(leaves=(m, s, q), xys=pr["xy"], depths=pr["z"] * vt, conics=pr["conic"], radii=pr["radius"],
                num_tiles_hit=np.where(vis, (pr["tmax"][:, 0] - pr["tmin"][:, 0]) * (pr["tmax"][:, 1] - pr["tmin"][:, 1]), 0),
                compensation=comp, cov3d=cov3d, vis=vis, unclipped=pr["unclipped"], margins=pr["margins"],
                margin=np.minimum.reduce([pr["margins"][k] for k in MARGIN_NAMES if k != "pre"]))


def l1_project_bwd(means, scales, glob_scale, quats, cam, v_xys, v_depths, v_conics, bw=16, clip=0.01):
    """(v_means, v_scales, v_quats) of sum(xys v_xys + depths v_depths + conics v_conics); None cotangent = zeros."""
    fw = l1_project(means, scales, glob_scale, quats, cam, bw, clip, grad=True)
    loss = 0.0
    for out, v in ((fw["xys"], v_xys), (fw["depths"], v_depths), (fw["conics"], v_conics)):
        if v is not None:
            loss = loss + (out * torch.tensor(np.asarray(v, np.float64).reshape(out.shape))).sum()
    if not torch.is_tensor(loss):
        return tuple(np.zeros(np.shape(x)) for x in (means, scales, quats))
    gs = torch.autograd.grad(loss, fw["leaves"], allow_unused=True)
    return tuple(np.zeros(np.shape(x)) if g is None else g.numpy() for g, x in zip(gs, (means, scales, quats)))


def l1_sh(degree: int, viewdirs: np.ndarray, coeffs: np.ndarray, v_colors: Optional[np.ndarray] = None):
    """spherical_harmonics(degree, viewdirs[N,3], coeffs[N,K,3]): colors = sum_{k < Kuse} Y_k c_k, Kuse = min((deg+1)^2, K);
    v_coeffs[:, k] = Y_k v_colors for k < Kuse, 0 above."""
    K = coeffs.shape[1]
    Kuse = min((degree + 1) ** 2, K)
    Y = sh_basis(degree, torch.tensor(np.asarray(viewdirs, np.float64))).numpy()
    colors = (Y[:, :Kuse, None] * np.asarray(coeffs, np.float64)[:, :Kuse]).sum(1)
    v_coeffs = None
    if v_colors is not None:
        v_coeffs = np.zeros(coeffs.shape)
        v_coeffs[:, :Kuse] = Y[:, :Kuse, None] * np.asarray(v_colors, np.float64)[:, None, :]
    return colors, v_coeffs
