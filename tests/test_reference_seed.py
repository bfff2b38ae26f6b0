"""CPU checks against tests/golden/reference_seed.npz (the reference's own populate_modules under a fixed seed): the kNN
oracle reproduces sklearn's distances, and populate.py's host logic -- draws, colours, opacities, shapes -- reproduces every
parameter, with the kNN scales taken from the oracle here (the GPU tests run the kernel)."""
import os

import numpy as np
import pytest
import torch

from oracle.knn_ref64 import knn_ref64
from street_gaussians_ns_b200 import populate

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_seed.npz"))
CASES = [str(c) for c in GOLDEN["cases"]]
PARAMS = ("means", "scales", "quats", "features_dc", "features_rest", "opacities")


def oracle_log_scales(points, k=3):
    d, _ = knn_ref64(points.cpu().numpy(), k)
    d = torch.from_numpy(d.astype(np.float32))
    return torch.log(d.mean(dim=-1, keepdim=True).repeat(1, 3))


def build(case):
    random_init, sh, F, num_random, cloud = (int(v) for v in GOLDEN[f"{case}_cfg"])
    torch.manual_seed(int(GOLDEN[f"{case}_seed"]))
    if random_init:
        return populate.random_gaussians(num_random, 10.0, sh, F, device="cpu")
    pre = "bg" if cloud == 0 else "act"
    return populate.gaussians_from_points(torch.from_numpy(GOLDEN[f"{pre}_xyz"]), torch.from_numpy(GOLDEN[f"{pre}_rgb"]), sh, F,
                                          device="cpu")


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_sklearn_distances(case):
    random_init, _, _, _, cloud = (int(v) for v in GOLDEN[f"{case}_cfg"])
    xyz = GOLDEN[f"{case}_means"] if random_init else GOLDEN["bg_xyz" if cloud == 0 else "act_xyz"]
    d, _ = knn_ref64(xyz, 3)
    assert np.allclose(d.astype(np.float32), GOLDEN[f"{case}_sk_dist"], rtol=1e-6, atol=1e-12)


@pytest.mark.parametrize("case", CASES)
def test_host_logic_reproduces_populate_modules(case, monkeypatch):
    monkeypatch.setattr(populate, "knn_log_scales", oracle_log_scales)
    gs = build(case)
    for p in PARAMS:
        got, ref = getattr(gs, p).numpy(), GOLDEN[f"{case}_{p}"]
        assert got.shape == ref.shape and got.dtype == np.float32, p
        if p == "scales":
            assert np.array_equal(np.isneginf(got), np.isneginf(ref))
            fin = np.isfinite(ref)
            assert np.abs(got[fin] - ref[fin]).max() <= 4e-6
        else:
            assert np.array_equal(got, ref, equal_nan=True), p


def test_golden_has_the_directed_cases():
    assert np.isneginf(GOLDEN["bg_sh3_f1_u8_scales"]).any()  # a point with four exact duplicates
    assert GOLDEN["bg_rgb"].dtype == np.uint8 and GOLDEN["act_rgb"].dtype == np.float32
    assert np.isinf(GOLDEN["act_sh0_f5_float_features_dc"]).any()  # logit at rgb = 255 (1 - 1e-10 rounds to 1 in fp32)
