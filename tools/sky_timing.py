"""Sky cube map timing at 1920 x 1280, R = 1024, training mode (jittered directions), and the privatisation count.

    python tools/sky_timing.py               # on the GPU: native forward / backward against the reference's sky path
    python tools/sky_timing.py --count-only  # on the CPU: share of backward contributions that bypass shared memory

GPU part (CUDA events, five alternations of the two paths, each a mean over --iters calls):
  * native: sgn_sky_fwd (directions generated in the kernel) and sgn_sky_bwd (into a freshly zeroed gradient);
  * reference: EnvLight's torch direction ops (get_world_directions + to_opengl, restated below) and nvdiffrast's own
    cube-linear kernels from oracle/_ref/libnvdr_texture.so (forward; gradient into zeros_like(tex), with the gradUV buffer
    it writes).
The jitter draws (two torch.rand [H, W]) are timed on both sides.

CPU part: the backward privatises per 32 x 32 pixel tile onto the face of the tile's first pixel; a lookup goes straight to
global atomics when it is on another face, wraps an edge or corner, or when its tile's texel box exceeds the shared
capacity.  The count uses the float64 oracle on the eval directions of the five config-4 rig cameras."""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TILE, BOX_TEXELS = 32, 2048  # csrc/sky.cu: SKY_TILE, SKY_BOX_TEXELS


def rig(width=1920, height=1280):
    import street_gaussians_ns_b200.synthetic as syn
    cams = []
    for yaw in (0.0, 50.0, -50.0, 100.0, -100.0):
        y = math.radians(yaw)
        c, s = math.cos(y), math.sin(y)
        R = np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
        cams.append((f"yaw{int(yaw)}", syn.make_camera(width, height, c2w=np.concatenate([R, np.zeros((3, 1))], 1))))
    return cams


def fallback_share(R=1024):
    from oracle import sky_ref64 as ref
    out = {}
    for name, cam in rig():
        H, W = cam.height, cam.width
        l = ref.directions(ref.c2w_from_viewmat(cam.viewmat()), cam.fx, cam.fy, cam.cx, cam.cy, W, H).astype(np.float32)
        lk = ref.lookup(l, R)
        face, i0, j0 = lk["face"], lk["i0"], lk["j0"]
        wrapped = (i0 < 0) | (j0 < 0) | (i0 + 1 >= R) | (j0 + 1 >= R) | ~lk["valid"]
        glob = 0
        tiles_priv = tiles = 0
        for y0 in range(0, H, TILE):
            for x0 in range(0, W, TILE):
                f, iw, jw, wr = (a[y0:y0 + TILE, x0:x0 + TILE] for a in (face, i0, j0, wrapped))
                tiles += 1
                dom = -1 if wr[0, 0] else f[0, 0]
                on = (f == dom) & ~wr
                if dom >= 0 and on.any():
                    bw = iw[on].max() - iw[on].min() + 2
                    bh = jw[on].max() - jw[on].min() + 2
                    if bw * bh <= BOX_TEXELS:
                        tiles_priv += 1
                        glob += int((~on).sum())
                        continue
                glob += f.size
        out[name] = {"global_share": glob / (H * W), "tiles_privatised": tiles_priv / tiles}
    return out


def timing(iters=50, alternations=5, R=1024, W=1920, H=1280):
    import torch
    import torch.nn.functional as F
    from oracle import nvdr_texture
    from street_gaussians_ns_b200 import sky
    from street_gaussians_ns_b200.raster import RenderSettings, camera_struct
    assert torch.cuda.is_available(), "needs a CUDA device"
    assert nvdr_texture.available(), "oracle/_ref/libnvdr_texture.so is missing: build it from a reference checkout first"
    dev = torch.device("cuda", 0)
    cam = rig(W, H)[0][1]
    cs = camera_struct(cam, RenderSettings())
    tex = torch.rand(6, R, R, 3, device=dev)
    v_sky = torch.randn(H, W, 3, device=dev)
    c2w = torch.from_numpy(cam.c2w).to(dev)
    to_opengl = torch.tensor([[1, 0, 0], [0, 0, 1], [0, -1, 0]], dtype=torch.float32, device=dev)
    gy, gx = torch.meshgrid(torch.arange(H, dtype=torch.float32, device=dev), torch.arange(W, dtype=torch.float32, device=dev),
                            indexing="ij")

    def ref_dirs():  # EnvLight.get_world_directions(train=True) + forward's to_opengl (sgn_splatfacto.py:118-146)
        d = torch.stack([(gx - cam.cx + torch.rand_like(gx)) / cam.fx, (gy - cam.cy + torch.rand_like(gy)) / cam.fy, torch.ones_like(gx)], 0)
        d = F.normalize(d, dim=0)
        d = (c2w[:3, :3] @ d.reshape(3, -1)).reshape(3, H, W).permute(1, 2, 0)
        return (d.reshape(-1, 3) @ to_opengl.T).reshape(H, W, 3).contiguous()

    def native_fwd():
        ju, jv = torch.rand(H, W, device=dev), torch.rand(H, W, device=dev)
        return sky.sky_forward(cs, tex, ju, jv)[0], (ju, jv)

    def native_bwd(state):
        return sky.sky_backward(cs, R, state[0], state[1], v_sky, dev)

    def ref_fwd():
        l = ref_dirs()
        return nvdr_texture.texture(tex, l), l

    def ref_bwd(l):
        return nvdr_texture.texture_grad(tex, l, v_sky)

    def time_pair(fwd, bwd):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        state = fwd()[1]
        bwd(state)
        torch.cuda.synchronize()
        tf = tb = 0.0
        for _ in range(iters):
            e[0].record()
            state = fwd()[1]
            e[1].record()
            bwd(state)
            e[2].record()
            torch.cuda.synchronize()
            tf += e[0].elapsed_time(e[1])
            tb += e[1].elapsed_time(e[2])
        return tf / iters, tb / iters

    rows = []
    for a in range(alternations):
        nf, nb = time_pair(native_fwd, native_bwd)
        rf, rb = time_pair(ref_fwd, ref_bwd)
        rows.append({"native_fwd_ms": nf, "native_bwd_ms": nb, "reference_fwd_ms": rf, "reference_bwd_ms": rb})
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    med = {k: float(np.median([r[k] for r in rows])) for k in rows[0]}
    return {"gpu": smi, "size": [W, H], "R": R, "iters": iters, "alternations": rows, "median": med,
            "bytes_lower_bound_MB": {"fwd": (H * W * 3 * 4 + 2 * H * W * 4) / 1e6,
                                     "bwd": (H * W * 3 * 4 + 2 * H * W * 4 + 2 * 6 * R * R * 3 * 4) / 1e6}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--count-only", action="store_true")
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    res = {"fallback": fallback_share()} if args.count_only else timing(args.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
