"""The sky cube map kernels (csrc/sky.cu) against the float64 oracle (oracle/sky_ref64.py), the reference's own EnvLight
directions (tests/golden/reference_sky.npz) and nvdiffrast's own kernels built from the reference checkout
(oracle/_ref/libnvdr_texture.so; that comparison skips only when the binary is absent), plus the model-level wiring:
sky.CubeMapSky, TrainStep with the sky in FusedAdam, and the Level-1 nvdiffrast_compat shim.

Bars come from fp32 noise in the texel coordinate: forward |d| <= 4 R 2^-24 (largest difference of the four taps) + 1e-7
on lookups whose texel coordinate the oracle puts at least 1e-4 texel from a floor boundary (and 1 / (2|c|) in the normal
fp32 range), and identical face / texel indices where the oracle puts the coordinate at least max(1e-4, 4 R 2^-24) texel
from a floor boundary; gradient per texel within the oracle's fp32 summation bound and, over the tensor, <= 1e-5 relative L2 or the
relative size of the texel-coordinate noise term of that bound where it is larger (at R = 1024), with the cotangent of the
other lookups set to zero."""
import os

import numpy as np
import pytest
import torch

from oracle import nvdr_texture
from oracle import sky_ref64 as ref
from tests import sky_cases as cases

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
EPS = 2.0 ** -24
STATS = []


def _sky():
    from street_gaussians_ns_b200 import sky
    return sky


def _fwd_bar(tex, lk, idx, R):
    t = tex.reshape(-1, 3).astype(np.float64)
    vals = t[np.maximum(idx, 0)]  # [..., 4, 3]
    spread = np.where((idx >= 0)[..., None], vals, np.nan)
    adj = np.nan_to_num(np.nanmax(spread, -2) - np.nanmin(spread, -2))
    return 4 * R * EPS * adj + 1e-7


def check_forward(name, R, uv, tex, got):
    lk = ref.lookup(uv, R)
    want, _, idx = ref.sample_torch(torch.from_numpy(tex.astype(np.float64)), uv, R)
    want = want.numpy()
    ok = ~lk["fragile"]
    err = np.abs(got - want)
    bar = _fwd_bar(tex, lk, idx, R)
    assert np.all(np.isfinite(got))
    bad = ok[..., None] & (err > bar)
    assert not bad.any(), (name, float(err[bad].max()), int(bad.sum()))
    assert np.all(got[~lk["valid"]] == 0)
    return float((err / bar)[ok].max()) if ok.any() else 0.0


def check_gradient(name, R, uv, v, got):
    lk = ref.lookup(uv, R)
    v = np.where(lk["fragile"][..., None], 0.0, v)
    want = ref.grad((6, R, R, 3), uv, v, R).reshape(-1, 3)
    bound, coord = ref.grad_bound(uv, v, R, parts=True)
    g = got.reshape(-1, 3).astype(np.float64)
    err = np.abs(g - want)
    assert np.all(err <= bound), (name, float((err / bound).max()))
    rel = float(np.linalg.norm(g - want) / max(np.linalg.norm(want), 1e-30))
    # 1e-5, or the relative size of the texel-coordinate noise itself where that is larger (R = 1024: s R - 1/2 is rounded
    # in fp32, as in the sampler this stands in for, so the bilinear weights carry ~R 2^-24 absolute error)
    rel_bar = max(1e-5, float(np.linalg.norm(coord) / max(np.linalg.norm(want), 1e-30)))
    assert rel <= rel_bar, (name, rel, rel_bar)
    return rel


INDEX_FLIPS = []


def index_texture(R):
    """Texel (face, j, i) holds (i, j, face): for a lookup whose four taps lie on one face the bilinear result is exactly the
    kernel's texel coordinates (u, v) = (i0 + fu, j0 + fv) and its face, so floor(u), floor(v) are its tap indices."""
    j, i = np.meshgrid(np.arange(R, dtype=np.float32), np.arange(R, dtype=np.float32), indexing="ij")
    f = np.arange(6, dtype=np.float32)[:, None, None]
    return np.stack(np.broadcast_arrays(i[None], j[None], f), -1).astype(np.float32)


def check_indices(name, R, lk, out):
    """Identical face and texel indices wherever the oracle puts both texel coordinates at least max(1e-4, 4 R 2^-24) texel
    from a floor boundary (the second term is the fp32 noise of the texel coordinate, larger than 1e-4 at R = 1024; the lookups
    in between are counted and reported), for lookups whose taps do not leave the face."""
    inside = lk["valid"] & (lk["i0"] >= 0) & (lk["j0"] >= 0) & (lk["i0"] + 1 < R) & (lk["j0"] + 1 < R) & ~lk["extreme"]
    differs = (np.floor(out[..., 0]) != lk["i0"]) | (np.floor(out[..., 1]) != lk["j0"]) | (out[..., 2] != lk["face"])
    thr = max(1e-4, 4 * R * EPS)
    bad = inside & (lk["floor"] >= thr) & differs
    assert not bad.any(), (name, int(bad.sum()))
    INDEX_FLIPS.append((name, int((inside & (lk["floor"] >= 1e-4) & differs).sum()), int((inside & (lk["floor"] >= 1e-4)).sum())))


def _nvdiffrast_grad_error(R, uv, v, g_nv):
    """Relative L2 of nvdiffrast's texture gradient against the same float64 oracle, reported next to the kernel's.  Its
    coalesced atomics (a per-warp shared-memory partial sum, no warp synchronisation between zeroing, adding and flushing it)
    lose or double contributions where lanes of a warp hit the same texel (tens of per cent at R = 1), so it is not held to a
    bar; the kernel's gradient is held to the oracle's (check_gradient)."""
    want = ref.grad((6, R, R, 3), uv, v, R).reshape(-1, 3)
    return float(np.linalg.norm(g_nv.reshape(-1, 3).astype(np.float64) - want) / max(np.linalg.norm(want), 1e-30))


def _check_against_nvdiffrast(name, R, tex, lk, got, nv):
    """Forward against nvdiffrast: both are held to the fp32 bar around the oracle, so they may differ by twice that bar, on the
    lookups the oracle does not call fragile (on those two fp32 statements may round a texel coordinate across a floor
    boundary differently); returns the number of bit-equal lookups."""
    bar = 2 * _fwd_bar(tex, lk, ref.taps(lk, R), R)
    bad = ~lk["fragile"][..., None] & (np.abs(got - nv) > bar)
    assert not bad.any(), (name, int(bad.sum()))
    return int(np.all(got == nv, -1).sum())


UV_CASES = cases.uv_cases()


@pytest.mark.parametrize("kind", cases.TEXTURES)
@pytest.mark.parametrize("case", UV_CASES, ids=[c[0] for c in UV_CASES])
def test_uv_path_against_oracle_and_nvdiffrast(case, kind):
    sky = _sky()
    name, R, uv = case
    tex = cases.texture(kind, R)
    tex_d, uv_d = torch.from_numpy(tex).to(DEV), torch.from_numpy(uv).to(DEV)
    out = sky.cube_texture(tex_d, uv_d)
    got = out.cpu().numpy()
    ratio = check_forward(name, R, uv, tex, got)
    # zero / NaN / infinite directions are not fragile in the oracle: they sample exactly 0
    v = np.random.default_rng(3).normal(size=uv.shape).astype(np.float32)
    lk = ref.lookup(uv, R)
    v_eff = np.where(lk["fragile"][..., None], 0.0, v).astype(np.float32)
    tex_p = tex_d.clone().requires_grad_(True)
    sky.cube_texture(tex_p, uv_d).backward(torch.from_numpy(v_eff).to(DEV))
    rel = check_gradient(name, R, uv, v_eff, tex_p.grad.cpu().numpy())
    if kind == cases.TEXTURES[0]:
        check_indices(name, R, lk, sky.cube_texture(torch.from_numpy(index_texture(R)).to(DEV), uv_d).cpu().numpy())
    if not nvdr_texture.available():
        pytest.skip("oracle/_ref/libnvdr_texture.so is absent (no reference checkout at build time)")
    same = _check_against_nvdiffrast(name, R, tex, lk, got, nvdr_texture.texture(tex_d, uv_d).cpu().numpy())
    g_nv = nvdr_texture.texture_grad(tex_d, uv_d, torch.from_numpy(v_eff).to(DEV)).cpu().numpy()
    STATS.append((name, kind, same, uv.shape[0], ratio, rel, _nvdiffrast_grad_error(R, uv, v_eff, g_nv)))


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "reference_sky.npz"))


def test_directions_match_the_reference_envlight(golden):
    from street_gaussians_ns_b200.raster import RenderSettings, camera_struct
    from street_gaussians_ns_b200.scene import Camera
    sky = _sky()
    for k in range(int(golden["num_cases"])):
        W, H = (int(x) for x in golden[f"size_{k}"])
        fx, fy, cx, cy = (float(x) for x in golden[f"intr_{k}"])
        cam = Camera(c2w=golden[f"c2w_{k}"], fx=fx, fy=fy, cx=cx, cy=cy, width=W, height=H)
        train = bool(golden[f"train_{k}"])
        ju = torch.from_numpy(golden[f"ju_{k}"]).to(DEV) if train else None
        jv = torch.from_numpy(golden[f"jv_{k}"]).to(DEV) if train else None
        tex = torch.rand(6, 8, 8, 3, device=DEV)
        _, dirs = sky.sky_forward(camera_struct(cam, RenderSettings()), tex, ju, jv, want_dirs=True)
        np.testing.assert_allclose(dirs.cpu().numpy(), golden[f"l_{k}"], rtol=0, atol=4 * 2.0 ** -24 * 4)


RIG = cases.rig_cameras()


@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
@pytest.mark.parametrize("cam", RIG, ids=[c[0] for c in RIG])
def test_full_size_cameras(cam, train):
    from street_gaussians_ns_b200.raster import RenderSettings, camera_struct
    sky = _sky()
    name, camera = cam
    R = 1024
    kind = "random" if name in ("yaw0", "up", "yaw-100") else "smooth"
    tex = cases.texture(kind, R)
    tex_d = torch.from_numpy(tex).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(11)
    H, W = camera.height, camera.width
    ju = torch.rand(H, W, device=DEV, generator=g) if train else None
    jv = torch.rand(H, W, device=DEV, generator=g) if train else None
    cs = camera_struct(camera, RenderSettings())
    out, dirs = sky.sky_forward(cs, tex_d, ju, jv, want_dirs=True)
    l = dirs.cpu().numpy()
    # directions: the float64 statement on the same jitter (a few fp32 ulps of a unit vector)
    want_l = ref.directions(ref.c2w_from_viewmat(camera.viewmat()), camera.fx, camera.fy, camera.cx, camera.cy, W, H,
                            None if ju is None else ju.cpu().numpy(), None if jv is None else jv.cpu().numpy())
    np.testing.assert_allclose(l, want_l, rtol=0, atol=8 * 2.0 ** -24)
    ratio = check_forward(name, R, l, tex, out.cpu().numpy())
    v = torch.randn(H, W, 3, device=DEV, generator=g)
    lk = ref.lookup(l, R)
    v = v * torch.from_numpy(~lk["fragile"]).to(DEV)[..., None]
    v_tex = sky.sky_backward(cs, R, ju, jv, v, DEV)
    rel = check_gradient(name, R, l, v.cpu().numpy(), v_tex.cpu().numpy())
    check_indices(name, R, lk, sky.sky_forward(cs, torch.from_numpy(index_texture(R)).to(DEV), ju, jv)[0].cpu().numpy())
    if not nvdr_texture.available():
        pytest.skip("oracle/_ref/libnvdr_texture.so is absent")
    same = _check_against_nvdiffrast(name, R, tex, lk, out.cpu().numpy(), nvdr_texture.texture(tex_d, dirs).cpu().numpy())
    g_nv = nvdr_texture.texture_grad(tex_d, dirs, v).cpu().numpy()
    STATS.append((f"{name}_{'train' if train else 'eval'}", kind, same, H * W, ratio, rel,
                  _nvdiffrast_grad_error(R, l, v.cpu().numpy(), g_nv)))


def test_report_bit_equal_fraction():
    flips, n = sum(f[1] for f in INDEX_FLIPS), sum(f[2] for f in INDEX_FLIPS)
    print(f"texel indices: {flips}/{n} unwrapped lookups at least 1e-4 texel from a floor boundary differ from the oracle")
    if not STATS:
        pytest.skip("no nvdiffrast comparison ran")
    eq = sum(s[2] for s in STATS)
    n = sum(s[3] for s in STATS)
    worst_f = max(s[4] for s in STATS)
    worst_g = max(s[5] for s in STATS)
    worst_nv = max(s[6] for s in STATS)
    lines = [f"{s[0]:32s} {s[1]:8s} bit-equal {s[2]}/{s[3]}  fwd err/bar {s[4]:.3f}  grad relL2 {s[5]:.2e}  nvdiffrast grad relL2 {s[6]:.2e}"
             for s in STATS]
    msg = (f"sky vs nvdiffrast: {eq}/{n} lookups bit-equal ({eq / n:.6f}); worst fwd err/bar {worst_f:.3f}; worst grad rel L2 "
           f"{worst_g:.2e} (nvdiffrast's own against the oracle: up to {worst_nv:.2e})")
    out = os.environ.get("SGN_SKY_REPORT")
    if out:
        with open(out, "w") as f:
            f.write("\n".join(lines + [f"index flips at >= 1e-4 texel: {flips}/{n}", msg]) + "\n")
    print(msg)


# ---- model level ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scene():
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
    from street_gaussians_ns_b200.sky import CubeMapSky
    fr = syn.make_frame(n_background=20000, n_actors=4, n_per_actor=1500, width=320, height=240, seed=3,
                        actor_shift=np.array([1.0, 0.0, -1.0]))
    bg = fr.segments[0].params.to(DEV)
    actors = {s.name.replace("object_", ""): s.params.to(DEV) for s in fr.segments[1:]}
    poses = [ActorPose(s.name.replace("object_", ""), s.rot, s.center, 21, list(range(85))) for s in fr.segments[1:]]

    def make(seed=0):
        torch.manual_seed(seed)
        env = CubeMapSky(16)
        with torch.no_grad():
            env.base.copy_(torch.rand(6, 16, 16, 3))
        m = SceneGraphRasterModel(bg, actors, SceneGraphConfig(ssim_lambda=0.0), poses_at=lambda t: poses, sky=env).to(DEV)
        m.step = 30000
        return m
    return fr, make


def test_model_sky_output_rgb_and_gradient(scene):
    from street_gaussians_ns_b200 import raster
    fr, make = scene
    model = make()
    model.train()
    cam = fr.camera
    H, W = cam.height, cam.width
    state = torch.cuda.get_rng_state(DEV)
    out = model.get_outputs(cam)
    after = torch.cuda.get_rng_state(DEV)
    torch.cuda.set_rng_state(state, DEV)
    ju, jv = torch.rand(H, W, device=DEV), torch.rand(H, W, device=DEV)
    assert torch.equal(torch.cuda.get_rng_state(DEV), after)  # exactly two [H,W] draws, as EnvLight makes
    sky_mod, dirs = _sky().sky_forward(raster.camera_struct(cam, raster.RenderSettings()), model.env_map.base.detach(), ju, jv,
                                       want_dirs=True)
    assert torch.equal(out["sky"], sky_mod)
    w = torch.rand(H, W, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    (out["rgb"] * w).sum().backward()
    # the same render given that sky as a tensor: rgb and the blend's v_sky
    sky_t = sky_mod.clone().requires_grad_(True)
    frame = model._frame(cam)
    out2, _ = raster.render_frame(frame, model._settings(class_streams=True), sky=sky_t)
    assert torch.equal(out["rgb"], out2["rgb"])
    (out2["rgb"] * w).sum().backward()
    l = dirs.cpu().numpy()
    v = sky_t.grad.cpu().numpy()
    lk = ref.lookup(l, 16)
    v = np.where(lk["fragile"][..., None], 0.0, v)
    want = ref.grad((6, 16, 16, 3), l, v, 16).reshape(-1, 3)
    got = model.env_map.base.grad.cpu().numpy().reshape(-1, 3).astype(np.float64)
    if lk["fragile"].any():  # recompute the module's gradient on the same cotangent without the fragile lookups
        got = _sky().sky_backward(raster.camera_struct(cam, raster.RenderSettings()), 16, ju, jv,
                                  torch.from_numpy(v.astype(np.float32)).to(DEV), DEV).cpu().numpy().reshape(-1, 3)
    assert np.all(np.abs(got - want) <= ref.grad_bound(l, v, 16))


def test_state_dict_round_trip_and_eval(scene):
    fr, make = scene
    a, b = make(0), make(1)
    assert not torch.equal(a.env_map.base, b.env_map.base)
    sd = a.state_dict()
    assert "env_map.base" in sd and sd["env_map.base"].shape == (6, 16, 16, 3)
    b.load_state_dict(sd)
    assert torch.equal(a.env_map.base, b.env_map.base)
    a.eval()
    with torch.no_grad():
        out = a.get_outputs(fr.camera)
        assert torch.equal(out["sky"], a.env_map(fr.camera, False))


def test_train_step_moves_the_sky_like_torch_adam(scene):
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.training import TrainStep
    fr, make = scene
    model = make(2)
    model.train()
    base = model.env_map.base
    before = base.detach().clone()
    opt = FusedAdam(model.optimizer_params(), extra={"sky": (base, 0.005)})
    step_fn = TrainStep(model, opt, refine_every=0)
    gt = torch.rand(fr.camera.height, fr.camera.width, 3, device=DEV)
    step_fn(30000, fr.camera, {"image": gt})
    torch.cuda.synchronize()
    grad = base.grad.detach().clone()
    assert float(grad.abs().max()) > 0
    ref_p = before.clone().requires_grad_(True)
    ref_p.grad = grad
    torch.optim.Adam([ref_p], lr=0.005, eps=1e-15).step()
    assert not torch.equal(base.detach(), before)
    assert torch.allclose(base.detach(), ref_p.detach(), rtol=1e-6, atol=1e-6)


def test_nvdiffrast_compat_matches_cube_map_sky(scene):
    from street_gaussians_ns_b200 import nvdiffrast_compat, raster
    fr, make = scene
    model = make(3)
    cam = fr.camera
    with torch.no_grad():
        sky_mod, dirs = _sky().sky_forward(raster.camera_struct(cam, raster.RenderSettings()), model.env_map.base, None, None,
                                           want_dirs=True)
    nvdiffrast_compat.install()
    import nvdiffrast.torch as dr
    base = model.env_map.base
    light = dr.texture(base[None, ...], dirs[None], filter_mode="linear", boundary_mode="cube")
    assert light.shape == (1, cam.height, cam.width, 3)
    assert torch.equal(light[0], sky_mod)
    flat = dr.texture(base[None, ...], dirs.reshape(1, 1, -1, 3), filter_mode="linear", boundary_mode="cube")
    assert torch.equal(flat.view(cam.height, cam.width, 3), sky_mod)
    flat.sum().backward()
    assert base.grad is not None and float(base.grad.sum()) == pytest.approx(cam.height * cam.width * 3, rel=1e-4)
    for kw in (dict(filter_mode="linear-mipmap-linear", boundary_mode="cube"), dict(filter_mode="linear", boundary_mode="wrap"),
               dict(filter_mode="linear", boundary_mode="cube", max_mip_level=0)):
        with pytest.raises(NotImplementedError):
            dr.texture(base[None, ...], dirs[None], **kw)
    with pytest.raises(NotImplementedError):
        dr.texture(torch.zeros(1, 6, 4, 4, 4, device=DEV), dirs[None], filter_mode="linear", boundary_mode="cube")
    with pytest.raises(NotImplementedError):
        dr.texture(base[None, ...], dirs[None].clone().requires_grad_(True), filter_mode="linear", boundary_mode="cube")
