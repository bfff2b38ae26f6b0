"""Named cases for the sky cube map kernels (tests/test_gpu_sky.py): lookup directions fed through the uv path, full-size
cameras of the config-4 rig, and textures.  Everything is generated from seeds on the host (float32)."""
import math

import numpy as np

from oracle import sky_ref64 as ref

RESOLUTIONS = (1, 2, 3, 16, 1024)


def _face_dirs(face, s, t):
    B = ref.BASIS[face].astype(np.float64)
    a, b = 2 * np.asarray(s) - 1, 2 * np.asarray(t) - 1
    return B[0] + a[..., None] * B[1] + b[..., None] * B[2]


def face_centres(R, rng):
    d = [_face_dirs(f, np.array([0.5]), np.array([0.5]))[0] * (1 + rng.random()) for f in range(6)]
    jit = [_face_dirs(f, 0.5 + (rng.random(20) - 0.5) * 0.2, 0.5 + (rng.random(20) - 0.5) * 0.2) for f in range(6)]
    return np.concatenate([np.array(d)] + jit)


def edge_bands(R, rng, n=64):
    """Directions inside the half-texel band along every border of every face (so every one of the 12 edges, from both of
    its faces) and in the half-texel squares at the 4 corners of every face (every one of the 8 cube corners, from its 3
    faces).  At R = 1 every lookup is a corner."""
    h = 0.5 / R
    out = []
    for f in range(6):
        band = h * rng.random(n)
        along = rng.random(n)
        out += [_face_dirs(f, band, along), _face_dirs(f, 1 - band, along), _face_dirs(f, along, band), _face_dirs(f, along, 1 - band)]
        for cs in (0, 1):
            for ct in (0, 1):
                u, v = h * rng.random(n // 4), h * rng.random(n // 4)
                out.append(_face_dirs(f, np.abs(cs - u), np.abs(ct - v)))
    return np.concatenate(out)


def exact_ties():
    """|x| = |y|, |x| = |z|, |y| = |z| and all equal, every sign combination, exactly representable."""
    base = [(1, 1, 0.25), (1, 0.5, 1), (0.75, 1, 1), (1, 1, 1), (2, 2, 0), (0, 3, 3), (0.5, 0, 0.5), (1, 1, 0.9999), (1, 0.9999, 1)]
    out = []
    for x, y, z in base:
        for sx in (-1, 1):
            for sy in (-1, 1):
                for sz in (-1, 1):
                    out.append((sx * x, sy * y, sz * z))
    return np.array(out, np.float64)


def degenerate():
    """Zero, NaN and infinite directions (they sample 0, no gradient) and extreme but finite magnitudes."""
    nan, inf = float("nan"), float("inf")
    return np.array([(0, 0, 0), (-0.0, 0, -0.0), (nan, 1, 0), (1, nan, 1), (0, 0, nan), (inf, 0, 0), (1, -inf, 2),
                     (3e38, 1e38, -2e38), (1e-38, 2e-39, -5e-39), (1e-45, 0, 0), (0, 1e-44, 3e-45), (1e30, 1e30, 1e-30),
                     (1e20, -1e20, 1e20), (2e-30, 1e-30, 1e-30)], np.float64)


def uv_cases():
    """(name, R, uv [P, 3] float32)."""
    cases = []
    for R in RESOLUTIONS:
        rng = np.random.default_rng(1000 + R)
        cases.append((f"face_centres_R{R}", R, face_centres(R, rng)))
        cases.append((f"edge_corner_bands_R{R}", R, edge_bands(R, rng)))
        cases.append((f"ties_R{R}", R, exact_ties()))
        cases.append((f"degenerate_R{R}", R, degenerate()))
        cases.append((f"random_R{R}", R, rng.normal(size=(4096, 3))))
    return [(n, R, np.asarray(uv, np.float32)) for n, R, uv in cases]


def texture(kind, R, seed=0):
    rng = np.random.default_rng(seed + R)
    if kind == "random":
        return rng.random((6, R, R, 3)).astype(np.float32)
    if kind == "constant":
        return np.full((6, R, R, 3), 0.5, np.float32)
    # smooth: a linear function of the texel centre's direction
    j, i = np.meshgrid(np.arange(R), np.arange(R), indexing="ij")
    d = np.stack([_face_dirs(f, (i + 0.5) / R, (j + 0.5) / R) for f in range(6)])
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    v = d @ np.array([0.3, -0.6, 0.45]) + 0.5
    return np.stack([v, 1 - v, 0.5 * v], -1).astype(np.float32)


TEXTURES = ("random", "smooth", "constant")


def rig_cameras(width=1920, height=1280):
    """(name, Camera): the five config-4 rig yaws (0, +-50, +-100 degrees) and the camera turned straight up and down."""
    import street_gaussians_ns_b200.synthetic as syn
    out = []
    for yaw in (0.0, 50.0, -50.0, 100.0, -100.0):
        y = math.radians(yaw)
        c, s = math.cos(y), math.sin(y)
        R = np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
        out.append((f"yaw{int(yaw)}", syn.make_camera(width, height, c2w=np.concatenate([R, np.array([[0.0], [0.0], [-3.0]])], 1))))
    for name, p in (("up", math.pi / 2), ("down", -math.pi / 2)):
        c, s = math.cos(p), math.sin(p)
        R = np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])
        out.append((name, syn.make_camera(width, height, c2w=np.concatenate([R, np.zeros((3, 1))], 1))))
    return out
