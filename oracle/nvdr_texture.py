"""nvdiffrast's own cube-map texture kernels as a reference binary (test infrastructure, never the product path).

``build()`` compiles the reference checkout's vendored ``nvdiffrast/common/texture.cu`` (with its ``common.cpp``, which
chooses the plugin's launch shapes) together with oracle/nvdr_texture_launcher.cu into ``oracle/_ref/libnvdr_texture.so``
for sm_90a.  The checkout is ``$SGN_REFERENCE_ROOT``, else ``../reference`` beside the repository; without it nothing is
built and an existing binary is left as it is.  The GPU tests load the binary when it is present (``available()``) and
skip the comparison when it is not."""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libnvdr_texture.so")
LAUNCHER = os.path.join(_HERE, "nvdr_texture_launcher.cu")


def reference_root() -> str:
    return os.environ.get("SGN_REFERENCE_ROOT") or os.path.join(os.path.dirname(os.path.dirname(_HERE)), "reference")


def _common_dir() -> str:
    return os.path.join(reference_root(), "dependencies", "nvdiffrast", "nvdiffrast", "common")


def build(force: bool = False) -> str | None:
    """Returns the library path, or None when the checkout is absent (an existing binary is kept)."""
    common = _common_dir()
    src, launch_shapes = os.path.join(common, "texture.cu"), os.path.join(common, "common.cpp")
    if not (os.path.exists(src) and os.path.exists(launch_shapes)):
        return LIB_PATH if os.path.exists(LIB_PATH) else None
    newest = max(os.path.getmtime(f) for f in (src, launch_shapes, LAUNCHER, os.path.abspath(__file__)))
    if not force and os.path.exists(LIB_PATH) and os.path.getmtime(LIB_PATH) >= newest:
        return LIB_PATH
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    os.makedirs(os.path.dirname(LIB_PATH), exist_ok=True)
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-DNVDR_TORCH", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
           "-shared", "-I", common, LAUNCHER, launch_shapes, "-o", LIB_PATH]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building the nvdiffrast reference binary failed:\n" + r.stdout + r.stderr)
    return LIB_PATH


def available() -> bool:
    return os.path.exists(LIB_PATH)


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB_PATH)
        vp, i32 = C.c_void_p, C.c_int
        L.nvdr_cube_linear_fwd.argtypes = [vp, i32, vp, i32, i32, vp, vp]
        L.nvdr_cube_linear_grad.argtypes = [vp, i32, vp, i32, i32, vp, vp, vp, vp]
        L.nvdr_cube_linear_fwd.restype = L.nvdr_cube_linear_grad.restype = C.c_int
        _lib = L
    return _lib


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def texture(tex, uv):
    """nvdiffrast's forward: tex [6,R,R,3], uv [H,W,3] (or [P,3]) CUDA float32 -> [..., 3]."""
    import torch
    uv = uv.contiguous()
    H, W = (uv.shape[0], uv.shape[1]) if uv.dim() == 3 else (1, uv.shape[0])
    out = torch.empty_like(uv)
    rc = lib().nvdr_cube_linear_fwd(C.c_void_p(tex.data_ptr()), tex.shape[1], C.c_void_p(uv.data_ptr()), H, W,
                                    C.c_void_p(out.data_ptr()), _stream())
    assert rc == 0, rc
    return out


def texture_grad(tex, uv, dy):
    """nvdiffrast's gradient for the texture (the uv gradient it also computes is discarded)."""
    import torch
    uv, dy = uv.contiguous(), dy.contiguous()
    H, W = (uv.shape[0], uv.shape[1]) if uv.dim() == 3 else (1, uv.shape[0])
    g = torch.zeros_like(tex)
    guv = torch.empty_like(uv)
    rc = lib().nvdr_cube_linear_grad(C.c_void_p(tex.data_ptr()), tex.shape[1], C.c_void_p(uv.data_ptr()), H, W,
                                     C.c_void_p(dy.data_ptr()), C.c_void_p(g.data_ptr()), C.c_void_p(guv.data_ptr()), _stream())
    assert rc == 0, rc
    return g
