"""The sky lookup's gradient for its direction on the GPU (csrc/sky.cu cube_dir_grad: sgn_cube_texture_bwd_uv[_det],
sgn_sky_bwd_view_rot / sgn_sky_bwd_det_view_rot) and its chain to the camera rotation.

  * uv gradient against nvdiffrast's own TextureGradKernelCubeLinear (oracle/_ref/libnvdr_texture.so; skipped only when the
    binary is absent) and against the float64 statement (tests/sky_grad_cases.py) within its fp32 bound, on every face,
    wrapped edges and corners, ties, zero / NaN / infinite directions, zero cotangents, R = 1, 2, 16, 1024 and the camera's
    own directions in eval and training; lookups the oracle calls fragile (a texel coordinate within 1e-4 texel of a floor
    boundary) get a zero cotangent in the comparison, as in tests/test_gpu_sky.py;
  * the texture gradient beside it: bit-identical to the texture-only entry points in deterministic mode, within 1e-5
    relative L2 with float atomics; CubeMapSky() without the switch runs today's launches;
  * v_view at 1920 x 1280, R = 1024, jittered, against float64 within a bound from the float64 sums of |terms|;
    bit-reproducible in both modes; translation entries exactly 0;
  * the chain into CameraPoseOptimizer.pose_adjustment (float64 autograd and finite differences), the model's camera share
    (projection plus a rotation-only sky share), a camera pulled back further with the switch on, and the Level-1 shim with
    install(uv_grad=True)."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from oracle import nvdr_texture
from oracle import sky_ref64 as ref
from street_gaussians_ns_b200 import _lib, raster
from street_gaussians_ns_b200 import sky as skym
from street_gaussians_ns_b200.camera_pose import CameraPoseOptimizer
from street_gaussians_ns_b200.raster import RenderSettings, camera_struct
from street_gaussians_ns_b200.scene import Camera
from street_gaussians_ns_b200.sky import CubeMapSky
from tests import camera_cases as cc
from tests import sky_cases
from tests import sky_grad_cases as sg

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
STATS = {}


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def nvdr_grad_uv(tex, uv, dy):
    """nvdiffrast's gradUV for uv [P, 3] (its gradTex goes to a scratch tensor)."""
    uv, dy = uv.contiguous(), dy.contiguous()
    g = torch.zeros_like(tex)
    guv = torch.empty_like(uv)
    rc = nvdr_texture.lib().nvdr_cube_linear_grad(_ptr(tex), tex.shape[1], _ptr(uv), 1, uv.shape[0], _ptr(dy), _ptr(g), _ptr(guv),
                                                  _stream())
    assert rc == 0
    return guv


def bwd_uv(tex, uv, v, det=False, want_tex=True):
    L = _lib.load()
    R = tex.shape[1]
    P = uv.shape[0]
    v_tex = torch.zeros_like(tex) if want_tex else None
    v_uv = torch.full_like(uv, float("nan"))  # every row must be written
    if det:
        s = skym._det_scratch(R, DEV)
        _lib.check(L.sgn_cube_texture_bwd_uv_det(P, _ptr(uv), _ptr(tex), R, _ptr(v), _ptr(v_tex), _ptr(v_uv), _ptr(s), s.numel(), _stream()),
                   "sgn_cube_texture_bwd_uv_det")
    else:
        _lib.check(L.sgn_cube_texture_bwd_uv(P, _ptr(uv), _ptr(tex), R, _ptr(v), _ptr(v_tex), _ptr(v_uv), _stream()), "sgn_cube_texture_bwd_uv")
    return v_tex, v_uv


def _uv_cases():
    out = []
    for name, R, uv in sky_cases.uv_cases():
        if R in (1, 2, 16, 1024):
            out.append((name, R, uv))
    return out


def _check_uv(name, R, uv, tex, v):
    """The kernel's uv gradient against float64 (within the fp32 bound) and nvdiffrast (bit-equal share, bar on the rest)."""
    uv_d, tex_d = torch.from_numpy(uv).to(DEV), torch.from_numpy(tex).to(DEV)
    lk = ref.lookup(uv.astype(np.float64), R)
    v = np.where(lk["fragile"][..., None], 0.0, v).astype(np.float32)
    v_d = torch.from_numpy(v).to(DEV)
    _, got = bwd_uv(tex_d, uv_d, v_d)
    got = got.cpu().numpy().astype(np.float64)
    assert np.all(np.isfinite(got)), name
    want = sg.grad_uv(tex.astype(np.float64), uv.astype(np.float64), v.astype(np.float64), R)
    bound = sg.grad_uv_bound(tex.astype(np.float64), uv.astype(np.float64), v.astype(np.float64), R)
    err = np.abs(got - want)
    assert np.all(err <= bound), (name, float((err / bound).max()), int((err > bound).sum()))
    assert np.all(got[~lk["valid"]] == 0) and np.all(got[(v == 0).all(-1)] == 0)
    if nvdr_texture.available():
        nv = nvdr_grad_uv(tex_d, uv_d, v_d).cpu().numpy().astype(np.float64)
        same = (got == nv).all(-1)
        STATS[name] = (int(same.sum()), len(same))
        assert np.all(np.abs(got - nv) <= 2 * bound), (name, float((np.abs(got - nv) / bound).max()))
    return got


@pytest.mark.parametrize("case", _uv_cases(), ids=lambda c: c[0])
def test_uv_gradient_against_float64_and_nvdiffrast(case):
    name, R, uv = case
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    tex = sky_cases.texture("random", R, seed=4)
    v = rng.normal(size=uv.shape)
    v[::5] = 0  # all-zero cotangents
    _check_uv(name, R, uv, tex, v)


@pytest.mark.parametrize("train", [False, True], ids=["eval", "jittered"])
def test_uv_gradient_on_camera_directions(train):
    R = 1024
    cam = syn.make_camera(480, 320)
    sky = CubeMapSky(resolution=R).to(DEV)
    with torch.no_grad():
        sky.base.copy_(torch.from_numpy(sky_cases.texture("random", R, seed=9)))
    torch.manual_seed(5)
    ju, jv = sky.jitter(cam) if train else (None, None)
    _, dirs = skym.sky_forward(camera_struct(cam, RenderSettings()), sky.base.detach(), ju, jv, want_dirs=True)
    uv = dirs.reshape(-1, 3).cpu().numpy()
    v = np.random.default_rng(2).normal(size=uv.shape)
    _check_uv(f"camera_{'jittered' if train else 'eval'}", R, uv, sky.base.detach().cpu().numpy(), v)


def test_report_bit_equal_share():
    if not STATS:
        pytest.skip("nvdiffrast's binary is absent")
    same = sum(s for s, _ in STATS.values())
    n = sum(t for _, t in STATS.values())
    print(f"\nuv gradient bit-equal to nvdiffrast on {same}/{n} lookups ({100.0 * same / n:.2f} %)")
    for k, (s, t) in STATS.items():
        print(f"  {k}: {s}/{t}")


@pytest.mark.parametrize("R", [2, 16, 1024])
def test_texture_gradient_unchanged_beside_the_uv_gradient(R):
    L = _lib.load()
    rng = np.random.default_rng(R)
    uv = np.concatenate([sky_cases.edge_bands(R, rng), rng.normal(size=(20000, 3))]).astype(np.float32)
    uv_d = torch.from_numpy(uv).to(DEV)
    tex = torch.from_numpy(sky_cases.texture("random", R)).to(DEV)
    v = torch.from_numpy(rng.normal(size=uv.shape).astype(np.float32)).to(DEV)
    P = uv.shape[0]
    det_old = torch.zeros_like(tex)
    s = skym._det_scratch(R, DEV)
    _lib.check(L.sgn_cube_texture_bwd_det(P, _ptr(uv_d), R, _ptr(v), _ptr(det_old), _ptr(s), s.numel(), _stream()), "det")
    det_new, vuv_det = bwd_uv(tex, uv_d, v, det=True)
    assert torch.equal(det_old, det_new)
    flt_old = torch.zeros_like(tex)
    _lib.check(L.sgn_cube_texture_bwd(P, _ptr(uv_d), R, _ptr(v), _ptr(flt_old), _stream()), "float")
    flt_new, vuv = bwd_uv(tex, uv_d, v)
    assert float((flt_new - flt_old).norm() / flt_old.norm()) <= 1e-5
    assert torch.equal(vuv, vuv_det)
    _, vuv2 = bwd_uv(tex, uv_d, v, want_tex=False)
    assert torch.equal(vuv, vuv2)


def _big_case(seed=0, W=1920, H=1280, R=1024):
    cam = sky_cases.rig_cameras(W, H)[1][1]
    tex = torch.from_numpy(sky_cases.texture("random", R, seed=seed)).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    ju = torch.rand(H, W, device=DEV, generator=g)
    jv = torch.rand(H, W, device=DEV, generator=g)
    v = torch.randn(H, W, 3, device=DEV, generator=g)
    cs = camera_struct(cam, RenderSettings())
    view = torch.tensor(list(cs.viewmat)[:12] + list(cs.cam_pos), device=DEV, dtype=torch.float32)
    return cam, tex, ju, jv, v, view


def test_view_cotangent_config3_against_float64_and_reproducible():
    cam, tex, ju, jv, v, view = _big_case()
    cs = camera_struct(cam, RenderSettings())
    R = tex.shape[1]
    runs = {}
    for det in (False, True):
        a = skym.sky_backward_rot(cs, tex, ju, jv, v, view, True, det)
        b = skym.sky_backward_rot(cs, tex, ju, jv, v, view, True, det)
        assert torch.equal(a[1], b[1])
        assert torch.all(a[1][[3, 7, 11, 12, 13, 14]] == 0)
        runs[det] = a
    assert torch.equal(runs[False][1], runs[True][1])  # the direction gradient does not depend on the texture-gradient mode
    # the texture gradient beside it is today's
    s = skym._det_scratch(R, DEV)
    old = skym.sky_backward(cs, R, ju, jv, v, DEV, True, view)
    assert torch.equal(old, runs[True][0])
    old_f = skym.sky_backward(cs, R, ju, jv, v, DEV, False, view)
    assert float((old_f - runs[False][0]).norm() / old_f.norm()) <= 1e-5
    # float64, on the kernel's own directions (the same face and texel decisions); fragile lookups carry no cotangent there
    _, dirs = skym.sky_forward(cs, tex, ju, jv, want_dirs=True, view=view)
    l = dirs.cpu().numpy().astype(np.float64)
    lk = ref.lookup(l, R)
    vm = v * torch.from_numpy(~lk["fragile"]).to(DEV)[..., None]
    got = skym.sky_backward_rot(cs, tex, ju, jv, vm, view, False)[1][:12].cpu().numpy().astype(np.float64)
    vm_np = vm.cpu().numpy().astype(np.float64)
    vmat = view[:12].cpu().numpy().astype(np.float64).reshape(3, 4)
    want, terms, noise = sg.grad_view(vmat, (cam.fx, cam.fy, cam.cx, cam.cy, cam.width, cam.height), tex.cpu().numpy().astype(np.float64),
                                      vm_np, R, ju.cpu().numpy(), jv.cpu().numpy(), l=l, parts=True)
    n = cam.width * cam.height
    # per term: the lookup's own fp32 bound plus a few roundings of the chain; the sum: a fixed-order fp32 reduction over n
    bound = noise + 2.0 ** -24 * (8 + np.log2(n) + 40) * terms + 1e-30
    err = np.abs(got - want)
    print(f"\nv_view |err| / bound max {float((err / bound).max()):.3g}; |err| / sum|terms| max {float((err / (terms + 1e-30)).max()):.3g}")
    assert np.all(err <= bound), (err, bound)


def test_chain_into_pose_adjustment_matches_float64():
    W, H, R = 160, 96, 16
    cam = syn.make_camera(W, H)
    cam.index = 0
    co = CameraPoseOptimizer(1).to(DEV)
    with torch.no_grad():
        co.pose_adjustment[0] = torch.tensor([0.1, 0.0, -0.2, 0.05, -0.1, 0.08])
    sky = CubeMapSky(resolution=R, view_grad=True).to(DEV)
    with torch.no_grad():
        sky.base.copy_(torch.from_numpy(sky_cases.texture("random", R, seed=2)))
    w = torch.randn(H, W, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    view = co.view(cam)
    # the kernel's own directions: the oracle takes the same decisions there; fragile lookups get no cotangent
    l = skym.sky_forward(camera_struct(cam, RenderSettings()), sky.base.detach(), None, None, want_dirs=True, view=view.detach())[1]
    l = l.cpu().numpy().astype(np.float64)
    w = w * torch.from_numpy(~ref.lookup(l, R)["fragile"]).to(DEV)[..., None]
    out = sky(cam, False, view=view)
    (out * w).sum().backward()
    got = co.pose_adjustment.grad[0].cpu().double()
    # float64: the oracle's view cotangent at the kernel's view, composed with autograd of camera_cases' view
    vv = sg.grad_view(view.detach()[:12].cpu().numpy().astype(np.float64).reshape(3, 4), (cam.fx, cam.fy, cam.cx, cam.cy, W, H),
                      sky.base.detach().cpu().numpy().astype(np.float64), w.cpu().numpy().astype(np.float64), R, l=l)
    x = co.pose_adjustment.detach()[0].cpu().double().requires_grad_(True)
    v64 = cc.view_of(cam.c2w, x)
    (want,) = torch.autograd.grad(v64[:12], x, grad_outputs=torch.from_numpy(vv))
    assert float((got - want).norm() / want.norm()) <= 1e-4, (got, want)
    assert float(sky.base.grad.abs().sum()) > 0


def test_chain_against_float64_finite_differences_on_a_smooth_texture():
    W, H, R = 64, 48, 32
    cam = syn.make_camera(W, H)
    cam.index = 0
    tex = sky_cases.texture("smooth", R).astype(np.float64)
    co = CameraPoseOptimizer(1).to(DEV)
    with torch.no_grad():
        co.pose_adjustment[0] = torch.tensor([0.0, 0.0, 0.0, 0.03, -0.02, 0.05])
    sky = CubeMapSky(resolution=R, view_grad=True).to(DEV)
    with torch.no_grad():
        sky.base.copy_(torch.from_numpy(tex.astype(np.float32)))
    wnp = np.random.default_rng(4).normal(size=(H, W, 3))
    sky(cam, False, view=co.view(cam)).mul(torch.from_numpy(wnp.astype(np.float32)).to(DEV)).sum().backward()
    got = co.pose_adjustment.grad[0, 3:].cpu().double().numpy()
    x0 = co.pose_adjustment.detach()[0].cpu().double()

    def loss(x):
        vm = cc.view_of(cam.c2w, x)[:12].numpy().reshape(3, 4)
        l = ref.directions(ref.c2w_from_viewmat(vm), cam.fx, cam.fy, cam.cx, cam.cy, W, H)
        return float((ref.sample(tex, l, R) * wnp).sum())

    h = 1e-6
    fd = np.array([(loss(x0 + h * e) - loss(x0 - h * e)) / (2 * h) for e in torch.eye(6, dtype=torch.float64)[3:]])
    assert np.linalg.norm(got - fd) <= 2e-2 * np.linalg.norm(fd), (got, fd)


def test_default_sky_is_unchanged():
    """CubeMapSky() and CubeMapSky(view_grad=True) with a view that requires no gradient launch the same kernels and give
    the same bits; without the switch the view gets no gradient."""
    L = _lib.load()
    cam = syn.make_camera(160, 96)
    cam.index = 0
    co = CameraPoseOptimizer(1).to(DEV)
    res = []
    for flag in (False, True):
        sky = CubeMapSky(resolution=16, deterministic=True, view_grad=flag).to(DEV)
        with torch.no_grad():
            sky.base.copy_(torch.from_numpy(sky_cases.texture("random", 16, seed=1)))
        view = co.view(cam)
        n0 = L.sgn_launch_count()
        out = sky(cam, False, view=view if not flag else view.detach())
        out.sum().backward()
        torch.cuda.synchronize()
        res.append((L.sgn_launch_count() - n0, out.detach(), sky.base.grad.clone()))
        assert co.pose_adjustment.grad is None
    assert res[0][0] == res[1][0] and torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][2], res[1][2])


def _sky_model(fr, co, sky):
    from street_gaussians_ns_b200.model import SceneGraphConfig, SceneGraphRasterModel
    m = SceneGraphRasterModel(fr.segments[0].params.to(DEV), {}, SceneGraphConfig(use_sky_sphere=True, ssim_lambda=0.2), sky=sky,
                              camera_optimizer=co).to(DEV)
    m.train()
    return m


def test_model_camera_share_is_projection_plus_sky():
    fr = syn.make_frame(n_background=3000, n_actors=0, n_per_actor=0, width=320, height=240, seed=3)
    co = CameraPoseOptimizer(2)
    sky = CubeMapSky(resolution=32, view_grad=True)
    m = _sky_model(fr, co, sky)
    with torch.no_grad():
        co.pose_adjustment.normal_(0, 0.01)
        m.env_map.base.copy_(torch.from_numpy(sky_cases.texture("random", 32, seed=3)))
    cam = fr.camera
    cam.index = 1
    torch.manual_seed(0)
    out = m.get_outputs(cam)
    gt = (torch.rand(240, 320, 3, generator=torch.Generator().manual_seed(2)) * 0.5 + 0.25).to(DEV)
    losses = m.get_loss_dict(out, {"image": gt})
    sum(v for k, v in losses.items() if k != "camera_opt_regularizer").backward()
    g = co.pose_adjustment.grad.clone()
    assert float(g[0].abs().max()) == 0
    # replay the sky's backward on the same cotangent: the model's sky output is out["sky"] when published, else recompute
    v_proj = m._holder.v_view
    assert v_proj is not None
    view = co.view(cam)
    total = g[1]
    (proj_share,) = torch.autograd.grad(view, co.pose_adjustment, grad_outputs=torch.cat([v_proj, torch.zeros(3, device=DEV)]))
    sky_share = total - proj_share[1]
    assert float(sky_share.abs().max()) > 0  # the sky pulls on the rotation
    assert float(sky_share[:3].abs().max()) <= 1e-6 * float(total.abs().max()) + 1e-12  # ... and only on the rotation


def test_it_trains_the_rotation_further():
    W, H, R = 256, 160, 64
    fr = syn.make_frame(n_background=400, n_actors=0, n_per_actor=0, width=W, height=H, seed=5)
    cam = fr.camera
    cam.index = 0
    texture = torch.from_numpy(sky_cases.texture("smooth", R)).to(DEV) * 0.5 + torch.from_numpy(sky_cases.texture("random", R, seed=6)).to(DEV) * 0.1
    with torch.no_grad():
        target_sky = CubeMapSky(resolution=R).to(DEV)
        target_sky.base.copy_(texture)
        mt = _sky_model(fr, None, target_sky)
        mt.eval()
        target = mt.get_outputs(cam)["rgb"].detach()
    errs = {}
    for flag in (False, True):
        co = CameraPoseOptimizer(1)
        sky = CubeMapSky(resolution=R, view_grad=flag)
        m = _sky_model(fr, co, sky)
        with torch.no_grad():
            m.env_map.base.copy_(texture)
            co.pose_adjustment[0, 3:] = torch.tensor([0.02, -0.015, 0.01], device=DEV)
        start = float(co.pose_adjustment.detach()[0, 3:].norm())
        opt = torch.optim.Adam([co.pose_adjustment], lr=1e-3)
        for _ in range(60):
            opt.zero_grad()
            torch.manual_seed(0)
            out = m.get_outputs(cam)
            acc = float(out["accumulation"].detach().mean())
            ((out["rgb"] - target).abs().mean()).backward()
            opt.step()
        errs[flag] = float(co.pose_adjustment[0, 3:].norm()) / start
    print(f"\nrotation error left after 60 steps: switch off {errs[False]:.3f}, on {errs[True]:.3f} (coverage {acc:.2f})")
    assert acc < 0.9
    assert errs[True] < 0.8 * errs[False], errs


def test_level1_envlight_restatement_matches_cube_map_sky():
    import sys
    from street_gaussians_ns_b200 import nvdiffrast_compat
    saved = {k: sys.modules.get(k) for k in ("nvdiffrast", "nvdiffrast.torch")}
    try:
        nvdiffrast_compat.install()
        import nvdiffrast.torch as dr
        W, H, R = 1920, 1280, 1024
        cam, tex, ju, jv, v, view = _big_case(seed=1)
        # lookups the oracle calls fragile on the kernel's directions take no cotangent (there torch's own roundings of the
        # direction may cross a texel boundary the kernel's did not)
        cs = camera_struct(cam, RenderSettings())
        dirs = skym.sky_forward(cs, tex, ju, jv, want_dirs=True, view=view)[1]
        v = v * torch.from_numpy(~ref.lookup(dirs.cpu().numpy().astype(np.float64), R)["fragile"]).to(DEV)[..., None]
        c2w = torch.from_numpy(np.asarray(cam.c2w, np.float32)).to(DEV).requires_grad_(True)
        base = tex.clone().requires_grad_(True)

        def envlight(dr):
            # EnvLight.get_world_directions + forward (sgn_splatfacto.py:118-147) in torch fp32
            yy, xx = torch.meshgrid(torch.arange(H, device=DEV, dtype=torch.float32), torch.arange(W, device=DEV, dtype=torch.float32),
                                    indexing="ij")
            d = torch.stack([(xx - cam.cx + ju) / cam.fx, (yy - cam.cy + jv) / cam.fy, torch.ones_like(xx)], -1)
            d = torch.nn.functional.normalize(d, dim=-1)
            d = (c2w[:3, :3] @ d.reshape(-1, 3).T).T.reshape(H, W, 3)
            to_opengl = torch.tensor([[1, 0, 0], [0, 0, 1], [0, -1, 0]], dtype=torch.float32, device=DEV)
            l = (to_opengl @ d.reshape(-1, 3).T).T.reshape(1, H, W, 3)
            return dr.texture(base[None], l.contiguous(), filter_mode="linear", boundary_mode="cube")[0]

        with pytest.raises(NotImplementedError):
            envlight(dr)
        nvdiffrast_compat.install(uv_grad=True)
        import nvdiffrast.torch as dr
        (envlight(dr) * v).sum().backward()
        got = c2w.grad[:3, :3].double().cpu()
        # CubeMapSky(view_grad=True)'s v_view, mapped to c2w: v_R[i][j] = s_j v_view[4j+i]
        vv = skym.sky_backward_rot(cs, tex, ju, jv, v, view, False)[1][:12].double().cpu().reshape(3, 4)
        want = torch.stack([torch.stack([vv[j, i] * (1 if j == 0 else -1) for j in range(3)]) for i in range(3)])
        rel = float((got - want).norm() / want.norm())
        print(f"\nLevel-1 c2w rotation gradient vs CubeMapSky: relative L2 {rel:.3g}")
        assert rel <= 1e-3
    finally:
        for k, mod in saved.items():
            if mod is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = mod
