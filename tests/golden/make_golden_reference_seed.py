"""Generates tests/golden/reference_seed.npz: the six ``gauss_params`` that THE REFERENCE'S OWN
``SplatfactoModel.populate_modules`` (sgn_splatfacto.py:253-300) builds on the CPU under a fixed seed, and the distances its
``k_nearest_sklearn`` (:439-457, sklearn's NearestNeighbors) returned for them.

What is not the reference's code here (tests/golden/reference_loader.py explains how its model code runs here):
  * ``Tensor.cuda`` is the identity while it runs (the ``.cuda()`` of :274);
  * the model is built with ``__new__``: ``use_sky_sphere`` off, sub-model index 0 (so no torchmetrics), and a camera
    optimizer whose ``setup`` returns None.

Clouds: ``bg_xyz`` (street-like: a ground slab, sparse volume, two far outliers, exact duplicates -- one point five times, so
its scale is -inf) with uint8 ``bg_rgb``; ``act_xyz`` (an actor-sized box) with float ``act_rgb`` in 0..255.
Per case ``c``: ``c_seed``, ``c_cfg`` = (random_init, sh_degree, fourier_dim, num_random, cloud: 0 bg / 1 actor), the six
``c_<param>`` and ``c_sk_dist`` (float32 [N, 3], as k_nearest_sklearn returns them).

    SGN_REFERENCE_ROOT=<checkout of street-gaussians-ns> python tests/golden/make_golden_reference_seed.py
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import reference_loader as rl  # noqa: E402

OUT = os.path.join(HERE, "reference_seed.npz")
PARAMS = ("means", "scales", "quats", "features_dc", "features_rest", "opacities")
# (name, random_init, sh_degree, fourier_dim, num_random, cloud, seed)
CASES = [
    ("bg_sh3_f1_u8", False, 3, 1, 0, 0, 11),
    ("bg_sh0_f1_u8", False, 0, 1, 0, 0, 12),
    ("act_sh3_f5_float", False, 3, 5, 0, 1, 13),
    ("act_sh0_f5_float", False, 0, 5, 0, 1, 14),
    ("random_sh3_f5", True, 3, 5, 1500, 0, 15),
]


def clouds():
    rng = np.random.RandomState(5)
    ground = np.stack([rng.uniform(-40, 40, 1400), rng.uniform(-1.7, -1.5, 1400), rng.uniform(-90, -1.5, 1400)], 1)
    volume = np.stack([rng.uniform(-40, 40, 500), rng.uniform(-6, 14, 500), rng.uniform(-90, -1.5, 500)], 1)
    outliers = np.array([[3000.0, 20.0, -500.0], [-2500.0, 400.0, 800.0]])
    bg = np.concatenate([ground, volume, outliers]).astype(np.float32)
    bg = np.concatenate([bg, bg[[7, 7, 7, 7, 100, 100, 1500]]])  # duplicates: row 7 five times over
    bg = bg[rng.permutation(bg.shape[0])]
    bg_rgb = rng.randint(0, 256, (bg.shape[0], 3)).astype(np.uint8)
    act = ((rng.rand(1200, 3) - 0.5) * np.array([1.9, 1.7, 4.6])).astype(np.float32)
    act = np.concatenate([act, act[[3, 3, 40]]])
    act_rgb = (rng.rand(act.shape[0], 3) * 255).astype(np.float32)
    act_rgb[:5] = [0.0, 255.0, 0.0]  # the logit branch's eps clamp at both ends
    return bg, bg_rgb, act, act_rgb


def main():
    base, _ = rl.load()
    bg, bg_rgb, act, act_rgb = clouds()
    out = {"bg_xyz": bg, "bg_rgb": bg_rgb, "act_xyz": act, "act_rgb": act_rgb, "cases": np.array([c[0] for c in CASES])}
    real_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        for name, random_init, sh, F, num_random, cloud, seed in CASES:
            cfg = base.SplatfactoModelConfig()
            cfg.random_init, cfg.sh_degree, cfg.fourier_features_dim, cfg.use_sky_sphere = random_init, sh, F, False
            cfg.background_color = "random"
            cfg.camera_optimizer = types.SimpleNamespace(setup=lambda **k: None)
            if num_random:
                cfg.num_random = num_random
            m = base.SplatfactoModel.__new__(base.SplatfactoModel)
            torch.nn.Module.__init__(m)
            m.config, m.num_train_data, m._model_idx_in_scene_graph = cfg, 0, 0
            xyz, rgb = (bg, bg_rgb) if cloud == 0 else (act, act_rgb)
            m.seed_points = (torch.from_numpy(xyz), torch.from_numpy(rgb))
            recorded = {}
            real_knn = m.k_nearest_sklearn

            def knn(x, k, real_knn=real_knn, recorded=recorded):
                d, i = real_knn(x, k)
                recorded["d"] = d
                return d, i

            m.k_nearest_sklearn = knn
            torch.manual_seed(seed)
            m.populate_modules()
            out[f"{name}_seed"] = np.array(seed)
            out[f"{name}_cfg"] = np.array([int(random_init), sh, F, num_random, cloud])
            for p in PARAMS:
                out[f"{name}_{p}"] = m.gauss_params[p].detach().numpy().astype(np.float32)
            out[f"{name}_sk_dist"] = recorded["d"]
    finally:
        torch.Tensor.cuda = real_cuda
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
