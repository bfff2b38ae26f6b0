"""Builds libsgn_raster.so IN-TREE with nvcc for sm_90a (H100) (no torch headers: the library is a
plain C-ABI shared object, see include/sgn_raster.h)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsgn_raster.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xptxas", "-v", "--expt-relaxed-constexpr"]

# per-file extra flags.  project.cu: the exact section is built from never-contracted intrinsics (sgn_exact.cuh: xf), the
# colour / gradient code around it may use FMAs
SOURCES = {
    "project.cu": [],
    "binning.cu": [],
    "binning_local.cu": [],
    "blend.cu": ["--use_fast_math"],
    "loss.cu": [],
    "ssim.cu": [],  # IEEE divisions (no fast math); contraction allowed
    "metrics.cu": [],  # IEEE expf / division; the squared differences use explicit _rn intrinsics
    "sky.cu": [],  # IEEE divisions / square root and denormals, as the directions and the sampler it stands in for use
    "densify.cu": ["--fmad=false"],
    "adam.cu": ["--fmad=false"],  # keep torch.optim.Adam's rounding sequence (no contraction)
    "refine.cu": ["--fmad=false"],
    "collective.cu": [],  # the refinement rules mirror torch's separately rounded elementwise kernels
    "camera.cu": [],  # IEEE sinf / cosf / sqrtf (no fast math)
    "knn.cu": [],  # distances through explicit _rn intrinsics: the box bound must not exceed a point's distance
    "depth.cu": [],  # the lidar projection is the projection's xf arithmetic; IEEE log / division in the metrics
    "semantic.cu": [],  # IEEE expf / logf / division in the cross-entropy; the carry only copies
    "scale_reg.cu": [],  # IEEE expf; the gradient chain through explicit _rn intrinsics, as torch autograd rounds it
    "filter3d.cu": ["--fmad=false"],  # fp64 sampling tests rounded per operation, as the float64 statement evaluates them
    "bilagrid.cu": [],  # IEEE division; the grid coordinates and the gray through explicit _rn intrinsics
}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libsgn_raster.so cannot be built")


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [
        os.path.join(os.path.dirname(HERE), "include", "sgn_raster.h"), os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)

    def compile_one(item):
        src, extra = item
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc, *ARCH, *COMMON, *extra, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = r.stdout + r.stderr
        with open(obj + ".log", "w") as f:
            f.write(" ".join(cmd) + "\n" + log)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{log}")
        if verbose:
            print(log)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES.items()))
    cmd = [nvcc, *ARCH, "-shared", "-o", LIB, *objs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
