"""Initialisation from seed points on the GPU: populate.py against the reference's own populate_modules
(tests/golden/reference_seed.npz), and SceneGraphRasterModel.from_points against the reference's draw order, then one
training step of the built model."""
import math
import os

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from street_gaussians_ns_b200 import populate
from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
from street_gaussians_ns_b200.scene import PARAM_NAMES

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_seed.npz"))
CASES = [str(c) for c in GOLDEN["cases"]]


def ulp_diff(a, b):
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


@pytest.mark.parametrize("case", CASES)
def test_populate_matches_the_reference(case):
    random_init, sh, F, num_random, cloud = (int(v) for v in GOLDEN[f"{case}_cfg"])
    torch.manual_seed(int(GOLDEN[f"{case}_seed"]))
    if random_init:
        gs = populate.random_gaussians(num_random, 10.0, sh, F, device=DEV)
    else:
        pre = "bg" if cloud == 0 else "act"
        gs = populate.gaussians_from_points(torch.from_numpy(GOLDEN[f"{pre}_xyz"]), torch.from_numpy(GOLDEN[f"{pre}_rgb"]), sh, F,
                                            device=DEV)
    got = {p: getattr(gs, p).cpu().numpy() for p in PARAM_NAMES}
    assert all(getattr(gs, p).device == DEV for p in PARAM_NAMES)
    for p in ("means", "quats", "opacities", "features_rest"):
        assert np.array_equal(got[p], GOLDEN[f"{case}_{p}"]), p
    dc, ref_dc = got["features_dc"], GOLDEN[f"{case}_features_dc"]
    fin = np.isfinite(ref_dc)
    assert np.array_equal(dc[~fin], ref_dc[~fin]) and ulp_diff(dc[fin], ref_dc[fin]).max() <= 1
    s, ref_s = got["scales"], GOLDEN[f"{case}_scales"]
    assert np.array_equal(np.isneginf(s), np.isneginf(ref_s))
    fin = np.isfinite(ref_s)
    assert np.abs(s[fin] - ref_s[fin]).max() <= 4e-6


def restated_reference(seed, background, actors, sh, F):
    """The reference's draws on the CPU, in its order (scene graph :50-52, then populate_modules per sub-model): what the
    quats and colours of every sub-model must be."""
    torch.manual_seed(seed)
    torch.rand(50000, 3)
    u, v, w = torch.rand(50000), torch.rand(50000), torch.rand(50000)
    torch.rand(50000, 3)
    out = {}
    names = ["background"] + [f"object_{t}" for t in actors]
    clouds = [background] + list(actors.values())
    for name, (xyz, rgb) in zip(names, clouds):
        n = xyz.shape[0]
        u, v, w = torch.rand(n), torch.rand(n), torch.rand(n)
        quats = torch.stack([torch.sqrt(1 - u) * torch.sin(2 * math.pi * v), torch.sqrt(1 - u) * torch.cos(2 * math.pi * v),
                             torch.sqrt(u) * torch.sin(2 * math.pi * w), torch.sqrt(u) * torch.cos(2 * math.pi * w)], -1)
        dc = torch.zeros(n, 1 if name == "background" else F, 3)
        dc[:, 0] = (rgb / 255 - 0.5) / 0.28209479177387814
        out[name] = (xyz, quats, dc, (sh + 1) ** 2 - 1)
    return out


@pytest.fixture(scope="module")
def seeded():
    bg_xyz = syn.street_points(30000, seed=3)
    bg_rgb = torch.randint(0, 256, (30000, 3), generator=torch.Generator().manual_seed(4), dtype=torch.uint8)
    actors = {}
    for a in range(3):
        xyz = syn.actor_points(2000, seed=10 + a)
        actors[str(a)] = (xyz, torch.rand(2000, 3, generator=torch.Generator().manual_seed(20 + a)) * 255)
    cfg = SceneGraphConfig(use_sky_sphere=False, ssim_lambda=0.0)
    torch.manual_seed(1234)
    model = SceneGraphRasterModel.from_points((bg_xyz, bg_rgb), actors, config=cfg, device=DEV)
    return model, bg_xyz, bg_rgb, actors, cfg


def test_from_points_follows_the_reference_draw_order(seeded):
    model, bg_xyz, bg_rgb, actors, cfg = seeded
    ref = restated_reference(1234, (bg_xyz, bg_rgb), actors, cfg.sh_degree, cfg.fourier_features_dim)
    assert list(model.all_models.keys()) == list(ref.keys())
    for name, (xyz, quats, dc, n_rest) in ref.items():
        gp = model.all_models[name].gauss_params
        assert torch.equal(gp["means"].detach().cpu(), xyz.float())
        assert torch.equal(gp["quats"].detach().cpu(), quats), name
        assert torch.equal(gp["features_dc"].detach().cpu(), dc), name
        assert gp["features_rest"].shape == (xyz.shape[0], n_rest, 3)
        assert bool(torch.isfinite(gp["scales"]).all())


def test_from_points_without_replay_and_random_background():
    torch.manual_seed(9)
    a = SceneGraphRasterModel.from_points(None, {}, config=SceneGraphConfig(use_sky_sphere=False), replay_scene_graph_init=False,
                                          device=DEV)
    torch.manual_seed(9)
    b = populate.random_gaussians(50000, 10.0, 3, 1, device=DEV)
    for p in PARAM_NAMES:
        assert torch.equal(a.all_models["background"].gauss_params[p].detach(), getattr(b, p)), p
    torch.manual_seed(9)
    c = SceneGraphRasterModel.from_points(None, {}, config=SceneGraphConfig(use_sky_sphere=False), device=DEV)
    assert not torch.equal(c.all_models["background"].gauss_params["quats"].detach(), getattr(b, "quats"))


def test_uint8_and_float_rgb_give_the_same_colours():
    g = torch.Generator().manual_seed(11)
    xyz = torch.rand(500, 3, generator=g)
    rgb = torch.randint(0, 256, (500, 3), generator=g, dtype=torch.uint8)
    a = populate.gaussians_from_points(xyz, rgb, 3, 1, generator=torch.Generator().manual_seed(1), device=DEV)
    b = populate.gaussians_from_points(xyz, rgb.float(), 3, 1, generator=torch.Generator().manual_seed(1), device=DEV)
    for p in PARAM_NAMES:
        assert torch.equal(getattr(a, p), getattr(b, p)), p


def test_built_model_trains_one_step(seeded):
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.training import TrainStep
    model, _, _, actors, _ = seeded
    poses = [ActorPose(t, np.eye(3), np.array([1.5 * (i - 1), -0.8, -12.0]), 21, list(range(85))) for i, t in enumerate(actors)]
    model.poses_at = lambda t: poses
    model.train()
    cam = syn.make_camera(320, 240, c2w=np.array([[1.0, 0, 0, 0], [0, 1.0, 0, 0], [0, 0, 1.0, 5.0]]), time=21.0)
    before = {n: model.all_models[n].gauss_params["means"].detach().clone() for n in model.all_models.keys()}
    opt = FusedAdam(model.optimizer_params())
    step = TrainStep(model, opt, refine_every=0)
    gt = torch.rand(240, 320, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    out = step(100, cam, {"image": gt})
    torch.cuda.synchronize()
    assert model.visible_model_names == ["background"] + [f"object_{t}" for t in actors]
    arena = model._holder.grad_arena
    assert bool(torch.isfinite(arena).all()) and float(arena.abs().max()) > 0
    for name in model.all_models.keys():
        gp = model.all_models[name].gauss_params
        assert all(bool(torch.isfinite(gp[p]).all()) for p in PARAM_NAMES), name
        assert not torch.equal(gp["means"].detach(), before[name]), name
    for v in out.values():
        if torch.is_tensor(v) and v.is_floating_point():
            assert bool(torch.isfinite(v).all())
