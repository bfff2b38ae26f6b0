"""Inria-layout PLY export / import of one sub-model's Gaussians (SURVEY.md 8f rank 4): the on-disk format on the far
side of the path.  Restates ``save_gs_model`` of the reference exporter (street_gaussians_ns/scripts/exporter.py:59-129):
float32 vertex properties, in this order,

    x y z  nx ny nz (zeros)  f_dc_0..2  f_rest_0..44  opacity  scale_0..2  rot_0..3

with ``f_dc`` = features_dc[:, 0, :] (the first Fourier coefficient only: ``shs_0``, sgn_splatfacto.py:341-343),
``f_rest`` = features_rest transposed to channel-major ("to match the sh order in Inria version", exporter.py:78-81),
opacity as logit, scales as log, rotation un-normalised wxyz; rows with any non-finite attribute are dropped
(exporter.py:103-116).  plyfile is not needed: the binary little-endian PLY it would write is produced directly.

A sub-model with semantic logits [n, C] (``SceneGraphConfig.semantic_classes``) appends ``semantic_0..C-1`` after ``rot_3``;
``read_semantic`` reads them back.  Files without semantics are byte for byte what they were before.

A model with the 3D smoothing filter (``SceneGraphConfig.filter_3d``) exports either way Mip-Splatting does:
``filter_3d="bake"`` folds the filter into the parameters -- scales log(sqrt(exp(s)^2 + sigma^2)) and opacity
logit(sigmoid(o) * coef), coef = prod_k sqrt(exp(s_k)^2 / (exp(s_k)^2 + sigma^2)) -- so that a viewer without the filter
renders what the model renders with it; ``filter_3d="column"`` writes the raw parameters plus a ``filter_3D`` property,
which ``read_filter_3d`` reads back.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from .scene import GaussianSet


def property_names(n_rest: int, n_semantic: int = 0) -> List[str]:
    return (["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(3)] + [f"f_rest_{i}" for i in range(n_rest)]
            + ["opacity"] + [f"scale_{i}" for i in range(3)] + [f"rot_{i}" for i in range(4)]
            + [f"semantic_{i}" for i in range(n_semantic)])


def bake_filter_3d(params: GaussianSet, filter_3d: torch.Tensor) -> GaussianSet:
    """The parameters with the 3D smoothing filter folded in (Mip-Splatting's fused export), evaluated in float64 and rounded
    once to float32: scales log(s') with s' = sqrt(s^2 + sigma^2), opacity logit(sigmoid(o) * coef) with coef =
    prod_k sqrt(s_k^2 / (s_k^2 + sigma^2)), s = exp(scales).  Means, rotations and colours are unchanged."""
    with torch.no_grad():
        ls = params.scales.detach().double()
        sig2 = filter_3d.detach().double().reshape(-1, 1).to(ls.device) ** 2
        s2 = torch.exp(2.0 * ls)
        v = s2 + sig2
        r = torch.where(v > 0, s2 / torch.where(v > 0, v, torch.ones_like(v)), torch.ones_like(v))
        coef = torch.sqrt(r).prod(1, keepdim=True)
        o = torch.sigmoid(params.opacities.detach().double()) * coef
        logit = torch.log(o) - torch.log1p(-o)
        scales = torch.where(v > 0, 0.5 * torch.log(torch.where(v > 0, v, torch.ones_like(v))), ls)
        return GaussianSet(params.means, scales.float().contiguous(), params.quats, params.features_dc, params.features_rest,
                           logit.float().contiguous())


def to_columns(params: GaussianSet, semantic: Optional[torch.Tensor] = None,
               filter_3d: Optional[torch.Tensor] = None) -> Tuple[List[str], np.ndarray]:
    """[n, n_props] float32 table in the exporter's column order (+ the semantic logits [n, C], when given, + the 3D filter
    sizes as ``filter_3D``, when given), finite rows only."""
    with torch.no_grad():
        means = params.means.detach().cpu().numpy().astype(np.float32)
        n = means.shape[0]
        dc = params.features_dc.detach()[:, 0, :].contiguous().cpu().numpy()
        rest = params.features_rest.detach().transpose(1, 2).contiguous().cpu().numpy().reshape(n, -1)
        cols = [means, np.zeros_like(means), dc, rest, params.opacities.detach().cpu().numpy().reshape(n, 1),
                params.scales.detach().cpu().numpy(), params.quats.detach().cpu().numpy()]
        n_sem = 0
        if semantic is not None:
            cols.append(semantic.detach().cpu().numpy().reshape(n, -1))
            n_sem = cols[-1].shape[1]
        if filter_3d is not None:
            cols.append(filter_3d.detach().cpu().numpy().reshape(n, 1))
    table = np.concatenate([c.astype(np.float32).reshape(n, -1) for c in cols], axis=1)
    table = table[np.isfinite(table).all(axis=1)]
    return property_names(rest.shape[1], n_sem) + (["filter_3D"] if filter_3d is not None else []), table


def write_ply(path, params: GaussianSet, semantic: Optional[torch.Tensor] = None, filter_3d: Optional[torch.Tensor] = None) -> int:
    """Writes ``point_cloud_<name>.ply`` for one sub-model; returns the number of exported Gaussians.  ``semantic``: the
    sub-model's semantic logits [n, C], written as ``semantic_0..C-1`` after ``rot_3`` (None: no such columns).
    ``filter_3d``: the 3D filter sizes [n], written as the last property ``filter_3D`` (None: no such column)."""
    names, table = to_columns(params, semantic, filter_3d)
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % table.shape[0]
    header += "".join(f"property float {k}\n" for k in names) + "end_header\n"
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(np.ascontiguousarray(table, dtype="<f4").tobytes())
    return int(table.shape[0])


def read_ply_columns(path) -> Dict[str, np.ndarray]:
    """Binary little-endian PLY with scalar vertex properties -> {name: [n] array}."""
    types = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1",
             "char": "i1", "int8": "i1", "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2",
             "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4"}
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, n, props, in_vertex = None, None, [], False
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: truncated PLY header")
            tok = line.decode("ascii").split()
            if not tok or tok[0] == "comment":
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                in_vertex = tok[1] == "vertex"
                if in_vertex:
                    n = int(tok[2])
                elif n is not None and props:
                    pass  # elements after the vertex element are ignored
            elif tok[0] == "property" and in_vertex:
                if tok[1] == "list":
                    raise ValueError(f"{path}: list properties on vertices are not supported")
                props.append((tok[2], types[tok[1]]))
            elif tok[0] == "end_header":
                break
        if fmt != "binary_little_endian":
            raise ValueError(f"{path}: only binary_little_endian PLY is supported (got {fmt})")
        if n is None:
            raise ValueError(f"{path}: no vertex element")
        dt = np.dtype(props)
        data = np.frombuffer(f.read(n * dt.itemsize), dtype=dt, count=n)
    return {k: np.asarray(data[k]) for k, _ in props}


def read_ply(path, device="cpu") -> GaussianSet:
    """Inverse of ``write_ply``: a GaussianSet with F = 1 Fourier coefficient (the file holds no others)."""
    c = read_ply_columns(path)
    n = c["x"].shape[0]
    n_rest = sum(1 for k in c if k.startswith("f_rest_"))
    if n_rest % 3:
        raise ValueError(f"{path}: {n_rest} f_rest properties is not a multiple of 3")

    def stack(keys):
        return torch.from_numpy(np.stack([c[k].astype(np.float32) for k in keys], axis=1))

    rest = stack([f"f_rest_{i}" for i in range(n_rest)]).reshape(n, 3, n_rest // 3).transpose(1, 2).contiguous()
    return GaussianSet(stack(["x", "y", "z"]), stack([f"scale_{i}" for i in range(3)]), stack([f"rot_{i}" for i in range(4)]),
                       stack([f"f_dc_{i}" for i in range(3)]).reshape(n, 1, 3), rest, stack(["opacity"])).to(device)


def read_semantic(path, device="cpu") -> Optional[torch.Tensor]:
    """The ``semantic_0..C-1`` columns of a ``write_ply`` file as float32 [n, C], or None when the file has none."""
    c = read_ply_columns(path)
    C = sum(1 for k in c if k.startswith("semantic_"))
    if C == 0:
        return None
    return torch.from_numpy(np.stack([c[f"semantic_{i}"].astype(np.float32) for i in range(C)], axis=1)).to(device)


def read_filter_3d(path, device="cpu") -> Optional[torch.Tensor]:
    """The ``filter_3D`` column of a ``write_ply(..., filter_3d=...)`` file as float32 [n], or None when the file has none."""
    c = read_ply_columns(path)
    if "filter_3D" not in c:
        return None
    return torch.from_numpy(c["filter_3D"].astype(np.float32)).to(device)


def export_model(model, output_dir, filter_3d: Optional[str] = None) -> Dict[str, int]:
    """exporter.py:131-137: one ``point_cloud_<sub-model>.ply`` per entry of ``all_models`` (with its semantic logits, when
    the model has them).  ``filter_3d`` (a model with ``SceneGraphConfig.filter_3d``): None writes the raw parameters alone,
    "bake" the parameters with the filter folded in (``bake_filter_3d``), "column" the raw parameters plus ``filter_3D``."""
    import os
    if filter_3d not in (None, "bake", "column"):
        raise ValueError(f"filter_3d must be None, 'bake' or 'column' (got {filter_3d!r})")
    os.makedirs(output_dir, exist_ok=True)
    out = {}
    for k, sub in model.all_models.items():
        params, column = sub.as_set(), None
        if filter_3d is not None:
            f = getattr(sub, "filter_3d", None)
            if f is None:
                raise ValueError(f"sub-model {k} has no 3D filter (SceneGraphConfig.filter_3d is off)")
            if filter_3d == "bake":
                params = bake_filter_3d(params, f)
            else:
                column = f
        out[k] = write_ply(os.path.join(output_dir, f"point_cloud_{k}.ply"), params, getattr(sub, "semantic_logits", None), column)
    return out
