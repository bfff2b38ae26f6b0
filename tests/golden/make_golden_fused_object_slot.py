"""Writes fused_object_slot.npz: the object slot (final_T[1], final_idx[1]) of the blend forward's saved state on the scenes
of tests/test_gpu_fused_objects.py, as the separate objects-only pass (acc_fwd_kernel on the object sub-lists) computed it
before that accumulation was folded into the main traversal.  Needs a GPU and a built checkout of that earlier commit:

    SGN_GOLDEN_PACKAGE_ROOT=<checkout> python tests/golden/make_golden_fused_object_slot.py [out.npz]
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.environ["SGN_GOLDEN_PACKAGE_ROOT"]))
spec = importlib.util.spec_from_file_location("fused_objects", os.path.join(os.path.dirname(HERE), "test_gpu_fused_objects.py"))
mod = importlib.util.module_from_spec(spec)
spec.loader.exec_module(mod)

out = {}
for name, kw in mod.SCENES.items():
    fr = mod.to_cuda(mod.syn.make_frame(**kw))
    st, _ = mod.forward_state(fr, mod.raster.RenderSettings())
    out[name + "_T"] = st["final_T"][1].cpu().numpy()
    out[name + "_idx"] = st["final_idx"][1].cpu().numpy()
path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "fused_object_slot.npz")
np.savez_compressed(path, **out)
print("wrote", path, {k: v.shape for k, v in out.items()})
