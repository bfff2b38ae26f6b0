"""Deterministic sky backward (sgn_sky_bwd_det / sgn_cube_texture_bwd_det, csrc/sky.cu): every addend rounded once to 64-bit
fixed point and added as an integer, so the gradient is bit-identical whatever the order of the lookups.

  * order independence: permuted lookup rows (uv with its cotangent) land in other blocks and other shared boxes and give
    the same bits, on face centres, edge and corner bands, R = 1 ... 1024, tiles whose texel box exceeds the deterministic
    box (the global path) and zero cotangents;
  * the camera form equals the uv form on the directions sgn_sky_fwd returns for the same jitter;
  * accuracy against the float64 oracle (oracle/sky_ref64.py): per texel within the oracle's fp32 bound plus half a grid
    unit per addend, over the tensor within the relative L2 bar of tests/test_gpu_sky.py, and against the float path;
  * a training step with the reference's defaults (SSIM 0.2, the learnable sky in FusedAdam, a refinement) under
    raster.DETERMINISTIC repeats bit for bit, and CubeMapSky(deterministic=True) does without the switch;
  * nvdiffrast_compat.texture under the switch gives sky.cube_texture's deterministic gradient;
  * argument errors (null, misaligned or undersized scratch) launch nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import sky_ref64 as ref
from tests import sky_cases as cases

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
REPORT = []


def L():
    from street_gaussians_ns_b200 import _lib
    return _lib.load()


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _scratch(R):
    return torch.empty(L().sgn_sky_det_scratch_bytes(R), dtype=torch.uint8, device=DEV)


def _scale(scratch, R):
    """The grid the call used: the float behind the int64 sums."""
    return float(scratch[18 * R * R * 8:18 * R * R * 8 + 4].view(torch.float32).item())


def uv_det(uv, v, R, v_tex=None):
    """(v_tex, scale) of sgn_cube_texture_bwd_det; uv [P, 3] / v [P, 3] CUDA float32."""
    v_tex = torch.zeros(6, R, R, 3, device=DEV) if v_tex is None else v_tex
    s = _scratch(R)
    rc = L().sgn_cube_texture_bwd_det(uv.shape[0], _p(uv), R, _p(v), _p(v_tex), _p(s), s.numel(), _stream())
    assert rc == 0, L().sgn_last_error()
    return v_tex, _scale(s, R)


def uv_float(uv, v, R):
    v_tex = torch.zeros(6, R, R, 3, device=DEV)
    assert L().sgn_cube_texture_bwd(uv.shape[0], _p(uv), R, _p(v), _p(v_tex), _stream()) == 0, L().sgn_last_error()
    return v_tex


def cam_det(cs, ju, jv, R, v):
    v_tex = torch.zeros(6, R, R, 3, device=DEV)
    s = _scratch(R)
    rc = L().sgn_sky_bwd_det(C.byref(cs), _p(ju), _p(jv), R, _p(v), _p(v_tex), _p(s), s.numel(), _stream())
    assert rc == 0, L().sgn_last_error()
    return v_tex, _scale(s, R)


def _face_block(face, R, lo, hi, n, rng):
    """n directions on ``face`` whose texel coordinates lie in [lo, hi) on both axes."""
    u = lo + (hi - lo) * rng.random(n)
    w = lo + (hi - lo) * rng.random(n)
    return cases._face_dirs(face, (u + 0.5) / R, (w + 0.5) / R)


def order_cases():
    """(name, R, uv [P, 3] float32, v [P, 3] float32), each with P > 2048 so that a permutation moves rows across blocks."""
    out = []
    for R in cases.RESOLUTIONS:
        rng = np.random.default_rng(2000 + R)
        base = {"face_centres": cases.face_centres(R, rng), "edge_corner_bands": cases.edge_bands(R, rng),
                "random": rng.normal(size=(1024, 3))}
        for name, d in base.items():
            d = np.concatenate([d] * (-(-3000 // d.shape[0])))[:3000 + R % 7]
            out.append((f"{name}_R{R}", R, d))
    rng = np.random.default_rng(7)
    R = 1024
    # one face, texel boxes of 40 x 40 (over SKY_DET_BOX_TEXELS, inside the float box) and of the whole face
    out.append(("box_40x40_R1024", R, np.concatenate([_face_block(4, R, 100, 138, 3072, rng)])))
    out.append(("box_whole_face_R1024", R, _face_block(1, R, 1, R - 2, 4096, rng)))
    # every block starts on a face whose box is small, followed by lookups of other faces and of wide boxes
    mix = [np.concatenate([_face_block(f, R, 500, 510, 512, rng), _face_block((f + 1) % 6, R, 0, R - 1, 256, rng),
                           rng.normal(size=(256, 3))]) for f in range(6)]
    out.append(("mixed_R1024", R, np.concatenate(mix)))
    res = []
    for name, R, uv in out:
        rng = np.random.default_rng(len(res))
        uv = np.asarray(uv, np.float32)
        v = rng.normal(size=uv.shape).astype(np.float32)
        res.append((name, R, uv, v))
        if name.startswith("edge_corner_bands"):  # zero cotangents: all of them, and a random half of the rows
            res.append((name + "_zero", R, uv, np.zeros_like(v)))
            res.append((name + "_half_zero", R, uv, np.where(rng.random((uv.shape[0], 1)) < 0.5, 0.0, v).astype(np.float32)))
    return res


ORDER = order_cases()


@pytest.mark.parametrize("case", ORDER, ids=[c[0] for c in ORDER])
def test_permuted_lookups_give_the_same_bits(case):
    name, R, uv, v = case
    uv_d, v_d = torch.from_numpy(uv).to(DEV), torch.from_numpy(v).to(DEV)
    g0, scale = uv_det(uv_d, v_d, R)
    assert torch.equal(g0, uv_det(uv_d, v_d, R)[0])
    gen = torch.Generator(device="cpu").manual_seed(R)
    for _ in range(3):
        perm = torch.randperm(uv.shape[0], generator=gen).to(DEV)
        g1, s1 = uv_det(uv_d[perm].contiguous(), v_d[perm].contiguous(), R)
        assert s1 == scale
        assert torch.equal(g0, g1), (name, int((g0 != g1).sum()))
    m = float(np.abs(v).max())
    assert scale == (2.0 ** (32 - np.ceil(np.log2(m))) if m > 0 else 2.0 ** 32), (name, scale, m)
    if not v.any():
        assert not g0.any()


def _addends_per_texel(uv, R):
    """Number of lookups that add to each texel (each gives it at most one addend)."""
    idx = ref.taps(ref.lookup(uv, R), R).reshape(-1, 4)
    n = np.zeros(6 * R * R, np.int64)
    for k in range(4):
        ok = idx[:, k] >= 0
        n += np.bincount(idx[ok, k], minlength=n.size)
    return n


def check_det_gradient(name, R, uv, v, got, scale, got_float):
    """Per texel: the oracle's fp32 bound plus half a grid unit per addend; over the tensor: test_gpu_sky.check_gradient's
    relative L2 bar; against the float path on the same input: relative L2 <= 1e-5, or that bar where it is larger."""
    lk = ref.lookup(uv, R)
    v = np.where(lk["fragile"][..., None], 0.0, v)
    want = ref.grad((6, R, R, 3), uv, v, R).reshape(-1, 3)
    bound, coord = ref.grad_bound(uv, v, R, parts=True)
    grid = _addends_per_texel(uv, R)[:, None] * (0.5 / scale)
    g = got.reshape(-1, 3).astype(np.float64)
    err = np.abs(g - want)
    assert np.all(err <= bound + grid), (name, float((err / (bound + grid)).max()))
    nw = max(np.linalg.norm(want), 1e-30)
    rel = float(np.linalg.norm(g - want) / nw)
    rel_bar = max(1e-5, float(np.linalg.norm(coord) / nw))
    assert rel <= rel_bar, (name, rel, rel_bar)
    gf = got_float.reshape(-1, 3).astype(np.float64)
    rel_f = float(np.linalg.norm(g - gf) / max(np.linalg.norm(gf), 1e-30))
    assert rel_f <= rel_bar, (name, rel_f, rel_bar)
    REPORT.append((name, float((err / (bound + grid)).max()), rel, rel_bar, rel_f))


UV_CASES = cases.uv_cases()


@pytest.mark.parametrize("case", UV_CASES, ids=[c[0] for c in UV_CASES])
def test_uv_gradient_against_oracle(case):
    name, R, uv = case
    lk = ref.lookup(uv, R)
    v = np.random.default_rng(3).normal(size=uv.shape).astype(np.float32)
    v = np.where(lk["fragile"][..., None], 0.0, v).astype(np.float32)
    uv_d, v_d = torch.from_numpy(uv).to(DEV), torch.from_numpy(v).to(DEV)
    got, scale = uv_det(uv_d, v_d, R)
    check_det_gradient(name, R, uv, v, got.cpu().numpy(), scale, uv_float(uv_d, v_d, R).cpu().numpy())
    # "adds into v_tex": on a prefilled gradient the result is the prefill plus the gradient, one fp32 addition
    pre = torch.randn(6, R, R, 3, device=DEV)
    assert torch.equal(uv_det(uv_d, v_d, R, pre.clone())[0], pre + got)


RIG = cases.rig_cameras()


@pytest.mark.parametrize("cam", [c for c in RIG if c[0] in ("yaw0", "yaw50", "up")], ids=lambda c: c[0])
def test_camera_form_equals_uv_form_and_oracle(cam):
    from street_gaussians_ns_b200 import sky
    from street_gaussians_ns_b200.raster import RenderSettings, camera_struct
    name, camera = cam
    R = 1024
    H, W = camera.height, camera.width
    g = torch.Generator(device=DEV).manual_seed(13)
    ju, jv = torch.rand(H, W, device=DEV, generator=g), torch.rand(H, W, device=DEV, generator=g)
    cs = camera_struct(camera, RenderSettings())
    _, dirs = sky.sky_forward(cs, torch.zeros(6, R, R, 3, device=DEV), ju, jv, want_dirs=True)
    l = dirs.cpu().numpy()
    lk = ref.lookup(l, R)
    v = torch.randn(H, W, 3, device=DEV, generator=g) * torch.from_numpy(~lk["fragile"]).to(DEV)[..., None]
    got, scale = cam_det(cs, ju, jv, R, v)
    via_uv, scale_uv = uv_det(dirs.reshape(-1, 3), v.reshape(-1, 3), R)
    assert scale == scale_uv
    assert torch.equal(got, via_uv), (name, int((got != via_uv).sum()))
    assert torch.equal(got, cam_det(cs, ju, jv, R, v)[0])
    flt = sky.sky_backward(cs, R, ju, jv, v, DEV, deterministic=False)
    assert torch.equal(sky.sky_backward(cs, R, ju, jv, v, DEV, deterministic=True), got)
    check_det_gradient(name, R, l, v.cpu().numpy(), got.cpu().numpy(), scale, flt.cpu().numpy())


def test_report():
    if not REPORT:
        pytest.skip("no accuracy case ran")
    worst = max(REPORT, key=lambda r: r[1])
    print(f"deterministic sky gradient: worst per-texel err/bound {worst[1]:.3f} ({worst[0]}); worst relative L2 against the "
          f"oracle {max(r[2] for r in REPORT):.2e}; worst against the float path {max(r[4] for r in REPORT):.2e}")


# ---- argument errors --------------------------------------------------------------------------------------------------
def test_argument_errors_launch_nothing():
    from street_gaussians_ns_b200.raster import RenderSettings, camera_struct
    import street_gaussians_ns_b200.synthetic as syn
    R = 8
    need = L().sgn_sky_det_scratch_bytes(R)
    assert need == 18 * R * R * 8 + 16
    assert L().sgn_sky_det_scratch_bytes(0) == 0 and L().sgn_sky_det_scratch_bytes(1024) == 18 * 1024 * 1024 * 8 + 16
    cs = camera_struct(syn.make_camera(64, 48), RenderSettings())
    uv = torch.randn(100, 3, device=DEV)
    v = torch.randn(100, 3, device=DEV)
    v_sky = torch.randn(48, 64, 3, device=DEV)
    ju, jv = torch.rand(48, 64, device=DEV), torch.rand(48, 64, device=DEV)
    s = torch.empty(need + 8, dtype=torch.uint8, device=DEV)
    v_tex = torch.full((6, R, R, 3), 7.0, device=DEV)
    torch.cuda.synchronize()
    before = L().sgn_launch_count()

    def sky_det(scr, nbytes, vt=v_tex, r=R, jitter=(ju, jv)):
        return L().sgn_sky_bwd_det(C.byref(cs), _p(jitter[0]), _p(jitter[1]), r, _p(v_sky), _p(vt), scr, nbytes, _stream())

    def tex_det(scr, nbytes, vt=v_tex, r=R):
        return L().sgn_cube_texture_bwd_det(100, _p(uv), r, _p(v), _p(vt), scr, nbytes, _stream())

    for call in (sky_det, tex_det):
        assert call(None, need) == -1 and b"null scratch" in L().sgn_last_error()
        assert call(_p(s), need - 1) == -1 and b"sgn_sky_det_scratch_bytes" in L().sgn_last_error()
        assert call(C.c_void_p(s.data_ptr() + 4), need) == -1 and b"aligned" in L().sgn_last_error()
        assert call(_p(s), need, vt=None) == -1
        assert call(_p(s), need, r=0) == -1
    assert sky_det(_p(s), need, jitter=(ju, None)) == -1
    # a scratch sized for a smaller map
    assert tex_det(_p(s), L().sgn_sky_det_scratch_bytes(R - 1)) == -1
    assert L().sgn_launch_count() == before, "an argument error launched a kernel"
    torch.cuda.synchronize()
    assert bool((v_tex == 7.0).all())
    # empty uv array: nothing to add, nothing launched
    assert L().sgn_cube_texture_bwd_det(0, _p(uv), R, _p(v), _p(v_tex), _p(s), need, _stream()) == 0
    assert L().sgn_launch_count() == before
    # the smallest valid scratch is enough
    assert tex_det(_p(s), need) == 0 and sky_det(_p(s), need) == 0
    torch.cuda.synchronize()


# ---- Level 1 ----------------------------------------------------------------------------------------------------------
def test_nvdiffrast_compat_follows_the_switch(monkeypatch):
    from street_gaussians_ns_b200 import nvdiffrast_compat, raster, sky
    import street_gaussians_ns_b200.synthetic as syn
    cam = syn.make_camera(320, 240)
    R = 16
    base = torch.rand(6, R, R, 3, device=DEV).requires_grad_(True)
    with torch.no_grad():
        _, dirs = sky.sky_forward(raster.camera_struct(cam, raster.RenderSettings()), base, None, None, want_dirs=True)
    w = torch.randn(1, cam.height, cam.width, 3, device=DEV)
    want, _ = uv_det(dirs.reshape(-1, 3), w.reshape(-1, 3).contiguous(), R)
    nvdiffrast_compat.install()
    import nvdiffrast.torch as dr
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    grads = []
    for _ in range(2):
        base.grad = None
        (dr.texture(base[None, ...], dirs[None], filter_mode="linear", boundary_mode="cube") * w).sum().backward()
        grads.append(base.grad.clone())
    base.grad = None
    (sky.cube_texture(base, dirs, deterministic=True) * w[0]).sum().backward()
    assert torch.equal(grads[0], want) and torch.equal(grads[1], want) and torch.equal(base.grad, want)


# ---- model level ------------------------------------------------------------------------------------------------------
def _run(steps, det_module, seed=0):
    """A fresh model (synthetic scene, CubeMapSky, SSIM 0.2), FusedAdam with the sky, TrainStep with a refinement at step
    700; returns every parameter, the Adam moments and the sky's gradient after ``steps``."""
    import street_gaussians_ns_b200.synthetic as syn
    from street_gaussians_ns_b200 import refine
    from street_gaussians_ns_b200.model import ActorPose, SceneGraphConfig, SceneGraphRasterModel
    from street_gaussians_ns_b200.optim import FusedAdam
    from street_gaussians_ns_b200.sky import CubeMapSky
    from street_gaussians_ns_b200.training import TrainStep
    fr = syn.make_frame(n_background=20000, n_actors=3, n_per_actor=1500, width=320, height=240, seed=3,
                        actor_shift=np.array([1.0, 0.0, -1.0]))
    bg = fr.segments[0].params.to(DEV)
    actors = {s.name.replace("object_", ""): s.params.to(DEV) for s in fr.segments[1:]}
    poses = [ActorPose(s.name.replace("object_", ""), s.rot, s.center, 21, list(range(85))) for s in fr.segments[1:]]
    rs = refine.RefineSettings(densify_grad_thresh=2e-5, densify_size_thresh=0.05, cull_alpha_thresh=0.05)
    cfg = SceneGraphConfig(ssim_lambda=0.2, refine=rs, object_refine=rs, num_train_data=5)
    torch.manual_seed(seed)
    env = CubeMapSky(16, deterministic=det_module)
    with torch.no_grad():
        env.base.copy_(torch.rand(6, 16, 16, 3))
    model = SceneGraphRasterModel(bg, actors, cfg, poses_at=lambda t: poses, sky=env).to(DEV)
    model.train()
    opt = FusedAdam(model.optimizer_params(), extra={"sky": (model.env_map.base, 0.005)})
    step_fn = TrainStep(model, opt, refine_every=100)
    gt = (torch.rand(240, 320, 3, generator=torch.Generator().manual_seed(2)) * 0.5 + 0.25).to(DEV)
    counts = []
    for step in steps:
        step_fn(step, fr.camera, {"image": gt})
        counts.append([sub.num_points for sub in model.all_models.values()])
    torch.cuda.synchronize()
    state = {f"{n}.{k}": p.detach().clone() for n, sub in model.all_models.items() for k, p in sub.gauss_params.items()}
    state["env_map.base"] = model.env_map.base.detach().clone()
    state["env_map.base.grad"] = model.env_map.base.grad.clone()
    m, v = opt.moment_views(opt.extra_index["sky"])
    state["env_map.exp_avg"], state["env_map.exp_avg_sq"] = m.clone(), v.clone()
    state["exp_avg"], state["exp_avg_sq"] = opt.exp_avg.clone(), opt.exp_avg_sq.clone()
    return state, counts


def _assert_same(a, b):
    assert a.keys() == b.keys()
    diff = [k for k in a if not torch.equal(a[k], b[k])]
    assert not diff, diff


def test_training_steps_repeat_bit_for_bit(monkeypatch):
    from street_gaussians_ns_b200 import raster
    monkeypatch.setattr(raster, "DETERMINISTIC", True)
    steps = list(range(696, 704))
    a, counts = _run(steps, None)
    assert counts[3] != counts[4], counts  # the refinement at step 700 changed the row counts
    b, _ = _run(steps, None)
    _assert_same(a, b)
    assert float(a["env_map.base.grad"].abs().max()) > 0


def test_module_flag_without_the_switch(monkeypatch):
    """CubeMapSky(deterministic=True) with the switch off: the same jittered render and cotangent twice give the same bits,
    those of sgn_sky_bwd_det on that jitter; the default module takes the float path."""
    from street_gaussians_ns_b200 import raster
    from street_gaussians_ns_b200.sky import CubeMapSky
    import street_gaussians_ns_b200.synthetic as syn
    monkeypatch.setattr(raster, "DETERMINISTIC", False)
    cam = syn.make_camera(320, 240)
    R = 64
    w = torch.randn(cam.height, cam.width, 3, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    grads = {}
    for det in (True, None):
        env = CubeMapSky(R, deterministic=det).to(DEV)
        for k in range(2):
            env.base.grad = None
            torch.manual_seed(9)
            (env(cam, True) * w).sum().backward()
            grads[det, k] = env.base.grad.clone()
    torch.manual_seed(9)
    ju, jv = env.jitter(cam)
    want, _ = cam_det(raster.camera_struct(cam, raster.RenderSettings()), ju, jv, R, w)
    assert torch.equal(grads[True, 0], want) and torch.equal(grads[True, 1], want)
    flt = grads[None, 0].double()
    rel = float(torch.linalg.vector_norm(want.double() - flt) / torch.linalg.vector_norm(flt))
    assert 0 < float(flt.abs().max()) and rel <= 1e-5, rel
