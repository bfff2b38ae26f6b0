"""Mip-Splatting's 3D smoothing filter (Yu et al., "Mip-Splatting: Alias-free 3D Gaussian Splatting", CVPR 2024, eq. 7):
per-Gaussian filter sizes from the training cameras, computed on the device (sgn_filter3d, csrc/filter3d.cu).

Every Gaussian is convolved with an isotropic 3D Gaussian of standard deviation sigma_i = sqrt(variance) / nu_i, where
nu_i = max over the training views that sample it of max(fx, fy) / z is the highest rate at which any training camera saw
it.  A view samples a row when its camera-space depth exceeds ``near`` and its projection lies inside the image with a 15 %
margin.  Rows no view samples get the largest sigma.  The projection then renders each row with scales
sqrt(s^2 + sigma^2) and its opacity times coef = prod_k sqrt(s_k^2 / (s_k^2 + sigma^2)) (include/sgn_raster.h,
sgn_camera.filter_3d), so that views sampling the scene more finely than any training camera (closer, zoomed in, higher
resolution) do not show a Gaussian's unconstrained high-frequency shape.

The host builds two small tables and uploads each in one copy, once per set of cameras (they are kept on the model for the
recomputes during training): the views' intrinsics, and for every (view, sub-model) the object->camera transform -- the view matrix composed with the sub-model's annotated box at the view's
timestamp (``poses_at``; box corrections are not applied) -- with a presence flag.  An actor is present in a view when it has
a box at the view's timestamp and at least one Gaussian, as a render of that view lists it.
"""
from __future__ import annotations

import ctypes as C
import hashlib
from typing import List, Sequence

import numpy as np
import torch

from . import _lib

CHUNK_ROWS = 128  # rows per block of the sweep (csrc/filter3d.cu FT_CHUNK)


def view_table(cameras: Sequence) -> np.ndarray:
    """sgn_filter_view rows of ``cameras`` (fx, fy, cx, cy, width, height)."""
    out = (_lib.FilterView * len(cameras))()
    for k, cam in enumerate(cameras):
        out[k].fx, out[k].fy, out[k].cx, out[k].cy = cam.fx, cam.fy, cam.cx, cam.cy
        out[k].width, out[k].height = cam.width, cam.height
    return np.frombuffer(out, np.uint8).copy()


XFORM_DTYPE = np.dtype([("M", "<f8", (12,)), ("present", "<i4"), ("pad", "<i4")])  # numpy mirror of sgn_filter_xform


def transform_table(model, cameras: Sequence, names: List[str]) -> np.ndarray:
    """sgn_filter_xform rows [V, nsub]: per (view, sub-model) the object->camera transform M = [W_3x3 R | W_3x3 c + w]
    (row-major 3x4, float64 from the float32 view matrix and the float64 box) and whether the sub-model is in the view.  The
    background (``names[0]``) is in every view, with M = W."""
    V, S = len(cameras), len(names)
    index = {n: i for i, n in enumerate(names)}
    tab = np.zeros((V, S), XFORM_DTYPE)
    rows = [model.all_models[n].num_points for n in names]
    by_time = {}
    for v, cam in enumerate(cameras):
        W = np.asarray(cam.viewmat(), np.float64).reshape(3, 4)
        tab["M"][v, 0] = W.reshape(-1)
        tab["present"][v, 0] = 1
        poses = by_time.get(cam.time)
        if poses is None:
            poses = by_time[cam.time] = [(index[model.get_object_model_name(p.track_id)], np.asarray(p.rot, np.float64).reshape(3, 3),
                                          np.asarray(p.center, np.float64).reshape(3)) for p in model.poses_at(cam.time)]
        for m, R, c in poses:
            if rows[m] == 0:
                continue
            tab["M"][v, m] = np.concatenate([W[:, :3] @ R, (W[:, :3] @ c + W[:, 3])[:, None]], 1).reshape(-1)
            tab["present"][v, m] = 1
    return tab


def _camera_digest(cameras: Sequence) -> bytes:
    h = hashlib.sha1()
    for c in cameras:
        h.update(c.c2w.tobytes())
        h.update(np.array([c.fx, c.fy, c.cx, c.cy, c.width, c.height, c.time], np.float64).tobytes())
    return h.digest()


def _device_tables(model, cameras: Sequence, names: List[str], counts: np.ndarray, dev):
    """The view and transform tables on the device, kept on the model for the next call with the same cameras (by content),
    the same sub-models and the same empty ones: a recompute during training then uploads nothing.  The boxes are taken to
    be fixed annotations (``poses_at`` is read when the tables are built)."""
    key = (_camera_digest(cameras), tuple(names), tuple(bool(n) for n in counts), str(dev))
    hit = model.__dict__.get("_filter_tables")
    if hit is None or hit[0] != key:
        views = torch.from_numpy(view_table(cameras)).to(dev, non_blocking=True)
        xforms = torch.from_numpy(transform_table(model, cameras, names).view(np.uint8).reshape(-1)).to(dev, non_blocking=True)
        hit = model.__dict__["_filter_tables"] = (key, views, xforms)
    return hit[1], hit[2]


def compute(model, cameras: Sequence, variance: float, near: float) -> int:
    """Fills every sub-model's ``filter_3d`` buffer from ``cameras`` (sgn_filter3d).  Returns the number of rows some view
    samples; 0 means no view samples any row, and every sigma is then 0."""
    L = _lib.load()
    names = list(model.all_models._modules)
    subs = [model.all_models[n] for n in names]
    dev = model.device
    counts = np.array([s.num_points for s in subs], np.int64)
    chunks = (counts + CHUNK_ROWS - 1) // CHUNK_ROWS
    chunk0 = np.concatenate([[0], np.cumsum(chunks)[:-1]])
    st = (_lib.FilterSub * len(subs))()
    for k, s in enumerate(subs):
        f = s.filter_3d
        assert f is not None and f.is_cuda and f.dtype == torch.float32 and f.is_contiguous() and f.numel() == counts[k]
        st[k].means = s.gauss_params["means"].data_ptr()
        st[k].out = f.data_ptr()
        st[k].count, st[k].chunk0 = int(counts[k]), int(chunk0[k])
    subs_dev = torch.from_numpy(np.frombuffer(st, np.uint8).copy()).to(dev, non_blocking=True)
    V = len(cameras)
    views_dev = xforms_dev = None
    if V:
        views_dev, xforms_dev = _device_tables(model, cameras, names, counts, dev)
    stats = torch.empty(2, device=dev, dtype=torch.int32)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(L.sgn_filter3d(C.c_void_p(subs_dev.data_ptr()), len(subs), int(chunks.sum()),
                              None if views_dev is None else C.c_void_p(views_dev.data_ptr()), V,
                              None if xforms_dev is None else C.c_void_p(xforms_dev.data_ptr()), float(variance), float(near),
                              C.c_void_p(stats.data_ptr()), stream), "sgn_filter3d")
    return int(stats[0].item())
