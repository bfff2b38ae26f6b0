"""Generates tests/golden/reference_sky.npz: the lookup directions ``l`` that THE REFERENCE'S OWN ``EnvLight``
(sgn_splatfacto.py:109-150: ``__init__``, ``get_world_directions``, ``forward``) hands to nvdiffrast's ``dr.texture``, on the
CPU, for a few small cameras in eval and in training, with the jitter draws it made.

What is not the reference's code here:
  * device arguments ("cuda") are redirected to the CPU;
  * ``kornia.utils.create_meshgrid(H, W, normalized_coordinates=False)`` is restated in one line (pixel x, y grid);
  * ``dr.texture`` is a stand-in that records its ``l`` argument (and returns zeros of the right shape);
  * ``torch.rand_like`` is wrapped to record its draws (u's first, then v's).

Per case ``k``: c2w_k [3,4], intr_k = (fx, fy, cx, cy), size_k = (W, H), train_k, ju_k / jv_k [H,W] (train only), l_k [H,W,3].

    SGN_REFERENCE_ROOT=<checkout of street-gaussians-ns> python tests/golden/make_golden_reference_sky.py
"""
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import reference_loader as rl  # noqa: E402

OUT = os.path.join(HERE, "reference_sky.npz")


def _rot(yaw, pitch, roll):
    cy, sy, cp, sp, cr, sr = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch), math.cos(roll), math.sin(roll)
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rx = np.array([[1, 0, 0], [0, cp, -sp], [0, sp, cp]])
    Rz = np.array([[cr, -sr, 0], [sr, cr, 0], [0, 0, 1]])
    return Ry @ Rx @ Rz


# (W, H, fx, fy, cx, cy, yaw, pitch, roll, train)
CASES = [
    (61, 47, 55.0, 57.5, 30.25, 23.75, 0.0, 0.0, 0.0, False),
    (61, 47, 55.0, 57.5, 30.25, 23.75, 0.0, 0.0, 0.0, True),
    (61, 47, 40.0, 40.0, 31.0, 22.0, math.radians(50), math.radians(-10), 0.05, False),
    (61, 47, 40.0, 40.0, 31.0, 22.0, math.radians(-100), math.radians(20), -0.1, True),
    (33, 29, 20.0, 21.0, 16.5, 14.5, 0.3, math.radians(89), 0.2, True),
    (33, 29, 20.0, 21.0, 16.5, 14.5, 1.1, math.radians(-80), 0.0, False),
]


def main():
    base, _ = rl.load()
    recorded = {}

    def texture(tex, uv, filter_mode=None, boundary_mode=None, **kw):
        assert filter_mode == "linear" and boundary_mode == "cube"
        recorded["l"] = uv.detach().clone()
        return torch.zeros(*uv.shape[:-1], tex.shape[-1])

    base.dr = types.SimpleNamespace(texture=texture)
    base.kornia = types.SimpleNamespace(utils=types.SimpleNamespace(create_meshgrid=lambda H, W, normalized_coordinates=False, device=None:
        torch.stack(torch.meshgrid(torch.arange(W, dtype=torch.float32), torch.arange(H, dtype=torch.float32), indexing="xy"), -1)[None]))
    real_tensor, real_rand_like = torch.tensor, torch.rand_like
    draws = []

    def tensor(*a, device=None, **k):
        return real_tensor(*a, **k)

    def rand_like(x, *a, **k):
        r = real_rand_like(x, *a, **k)
        draws.append(r.clone())
        return r

    torch.tensor, torch.rand_like = tensor, rand_like
    try:
        env = base.EnvLight(resolution=2)
        out = {}
        for k, (W, H, fx, fy, cx, cy, yaw, pitch, roll, train) in enumerate(CASES):
            R = _rot(yaw, pitch, roll)
            c2w = np.concatenate([R, np.array([[1.5], [-0.25], [3.0]])], 1).astype(np.float32)
            cam = types.SimpleNamespace(width=real_tensor([W]), height=real_tensor([H]), fx=real_tensor([fx], dtype=torch.float32),
                                        fy=real_tensor([fy], dtype=torch.float32), cx=real_tensor([cx], dtype=torch.float32),
                                        cy=real_tensor([cy], dtype=torch.float32), camera_to_worlds=torch.from_numpy(c2w)[None])
            torch.manual_seed(100 + k)
            draws.clear()
            light = env(cam, train=train)
            assert light.shape == (H, W, 3)
            out[f"c2w_{k}"] = c2w
            out[f"intr_{k}"] = np.array([fx, fy, cx, cy], np.float32)
            out[f"size_{k}"] = np.array([W, H], np.int64)
            out[f"train_{k}"] = np.array(train)
            assert len(draws) == (2 if train else 0)
            if train:
                out[f"ju_{k}"], out[f"jv_{k}"] = draws[0].numpy(), draws[1].numpy()
            out[f"l_{k}"] = recorded["l"].reshape(H, W, 3).numpy()
        out["num_cases"] = np.array(len(CASES))
    finally:
        torch.tensor, torch.rand_like = real_tensor, real_rand_like
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, {k: v.shape for k, v in out.items() if k.startswith("l_")})


if __name__ == "__main__":
    main()
