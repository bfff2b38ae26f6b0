"""CPU checks of the trainable box corrections: ``box_pose.BoxPoseOptimizer`` against vectors of the reference's own
``BBoxOptimizer.apply_to_bbox`` (tests/golden/reference_bbox.npz), its autograd against finite differences, the float64
pose-cotangent reference the GPU tests compare with (tests/pose_cases.py) against finite differences of the float64 render,
and the model-side plumbing that needs no device."""
import os

import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from oracle import oracle_c
from street_gaussians_ns_b200.box_pose import BoxPoseOptimizer
from street_gaussians_ns_b200.model import ActorPose
from street_gaussians_ns_b200.pose_table import PoseTable, quaternion_matrix
from tests import pose_cases as pz

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_bbox.npz")


def _module(d, dtype=torch.float32):
    F, B = d["delta_yaw"].shape
    m = BoxPoseOptimizer(F, [str(t) for t in d["tracks"]], {int(ts): i for i, ts in enumerate(d["timestamps"])}, mode="simple")
    with torch.no_grad():
        m.delta_center.copy_(torch.from_numpy(d["delta_center"]))
        m.delta_yaw.copy_(torch.from_numpy(d["delta_yaw"]))
    return m.to(dtype)


def test_poses_reproduce_the_reference():
    d = np.load(GOLD)
    out = _module(d).poses(d["frame_ids"], d["box_ids"], d["rot0"], d["center0"])
    assert out.dtype == torch.float32 and tuple(out.shape) == (len(d["frame_ids"]), 16)
    out = out.detach()
    got = out.numpy().astype(np.float64)
    np.testing.assert_allclose(got[:, 0:9].reshape(-1, 3, 3), d["rot"].astype(np.float32), atol=1e-6, rtol=0)
    np.testing.assert_allclose(got[:, 9:12], d["center"].astype(np.float32), atol=1e-6 * 32, rtol=0)  # centres reach 30: 1e-6 relative
    np.testing.assert_allclose(got[:, 12:16], d["q"].astype(np.float32), atol=1e-6, rtol=0)
    assert np.all(got[:, 12] >= 0) and np.all(d["q"][:, 0] >= 0)
    # the yaw parameter turns the box by TWICE its value about the box's own z axis
    k = 0
    turn = d["rot0"][k].T @ d["rot"][k]
    a = 2.0 * float(d["delta_yaw"][d["frame_ids"][k], d["box_ids"][k]])
    np.testing.assert_allclose(turn, [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]], atol=1e-6)
    # a box without an annotated frame passes through untouched
    skip = np.nonzero(d["frame_ids"] < 0)[0]
    assert len(skip) == 1
    assert np.array_equal(out[skip[0], 0:9].numpy(), d["rot0"][skip[0]].reshape(9).astype(np.float32))
    assert np.array_equal(out[skip[0], 9:12].numpy(), d["center0"][skip[0]].astype(np.float32))


def test_mode_off_hands_the_annotation_on():
    d = np.load(GOLD)
    m = BoxPoseOptimizer(4, ["a", "b", "c"], {}, mode="off")
    assert list(m.parameters()) == []
    out = m.poses(d["frame_ids"], d["box_ids"], d["rot0"], d["center0"]).numpy()
    from street_gaussians_ns_b200.scene import quaternions_from_matrices
    want = np.concatenate([d["rot0"].reshape(-1, 9), d["center0"], quaternions_from_matrices(d["rot0"])], 1).astype(np.float32)
    assert out.tobytes() == want.tobytes()  # the casts the segment table applies to an annotated box
    with pytest.raises(ValueError):
        BoxPoseOptimizer(4, ["a"], {}, mode="SE3")


def test_state_dict_has_the_reference_names():
    m = BoxPoseOptimizer(5, ["a", "b"], {}, mode="simple")
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {"delta_center": (5, 2, 3), "delta_yaw": (5, 2)}
    assert float(m.delta_center.detach().abs().sum()) == 0 and float(m.delta_yaw.detach().abs().sum()) == 0


def test_autograd_matches_finite_differences():
    d = np.load(GOLD)
    m = _module(d, torch.float64)
    st = m.stage(d["frame_ids"], d["box_ids"], d["rot0"], d["center0"])
    w = torch.rand(len(d["frame_ids"]), 16, generator=torch.Generator().manual_seed(2), dtype=torch.float64)

    def loss():
        # forward() ends in the float32 cast of the kernel's input; differences are taken before it
        return (m.poses_f64(st) * w).sum()

    L = loss()
    L.backward()
    eps = 1e-6
    live = [(int(f), int(b)) for f, b in zip(d["frame_ids"], d["box_ids"]) if f >= 0]
    for p, g in ((m.delta_center, m.delta_center.grad), (m.delta_yaw, m.delta_yaw.grad)):
        for f, b in live:
            for idx in ([(f, b, c) for c in range(3)] if p.dim() == 3 else [(f, b)]):
                vals = []
                for sgn in (1, -1):
                    with torch.no_grad():
                        p[idx] += sgn * eps
                        vals.append(float(loss()))
                        p[idx] -= sgn * eps
                fd = (vals[0] - vals[1]) / (2 * eps)
                assert abs(fd - float(g[idx])) <= 1e-7 * max(1.0, abs(fd)), (idx, fd, float(g[idx]))
        touched = torch.zeros_like(g, dtype=torch.bool)
        for f, b in live:
            touched[f, b] = True
        assert float(g[~touched].abs().sum()) == 0  # rows of other (frame, box) pairs and of the passed-through box


def test_pose_reference_matches_finite_differences_of_the_render():
    """Central differences of the float64 render in R, t and q_box of an actor validate the autograd reference itself."""
    fr = syn.make_frame(5, 1, n_per_actor=4, width=32, height=32, seed=5)
    with torch.no_grad():
        fr.segments[0].params.means.copy_(torch.tensor(
            [[0.02, 0.01, -3.0], [-0.03, 0.02, -3.5], [0.01, -0.02, -4.0], [0.0, 0.0, -2.5], [0.03, 0.03, -5.0]]))
        fr.segments[0].params.scales.fill_(np.log(0.02))
        fr.segments[0].params.opacities.fill_(0.3)
        fr.segments[1].params.means.mul_(0.02)
        # the view direction of the SH colour is taken from detached means (sgn_splatfacto.py:934): autograd leaves
        # d(colour)/d(pose) out on purpose; without higher SH orders finite differences see the same function
        fr.segments[0].params.features_rest.zero_()
        fr.segments[1].params.features_rest.zero_()
        fr.segments[1].params.scales.copy_(torch.log(torch.tensor([[0.02, 0.01, 0.015]])).expand(4, 3))
        fr.segments[1].params.opacities.fill_(0.2)
    fr.segments[1].center = np.array([0.01, 0.0, -3.2])
    fw = oracle_c.Oracle(fr).forward()
    assert (fw.radii > 0).all()
    g = torch.Generator().manual_seed(1)
    w_img, w_a, w_o = torch.rand(32, 32, 4, generator=g).double(), torch.rand(32, 32, generator=g).double(), torch.rand(32, 32, generator=g).double()
    base = pz.frame_poses(fr).astype(np.float64)
    leaf = pz.pose_leaves(base)
    L = pz.render_loss(fr, leaf, fw.sorted_ids, fw.tile_bins, w_img, w_a, w_o)
    (grad,) = torch.autograd.grad(L, leaf)
    assert all(float(x.abs().max()) > 0 for x in (grad[0, 0:9], grad[0, 9:12], grad[0, 12:16]))
    eps = 1e-6
    for j in range(16):
        vals = []
        for sgn in (1, -1):
            p = base.copy()
            p[0, j] += sgn * eps
            with torch.no_grad():
                vals.append(float(pz.render_loss(fr, torch.tensor(p), fw.sorted_ids, fw.tile_bins, w_img, w_a, w_o)))
        fd = (vals[0] - vals[1]) / (2 * eps)
        assert abs(fd - float(grad[0, j])) <= 1e-5 * max(1.0, abs(fd)), (j, fd, float(grad[0, j]))


def test_record_reference_agrees_with_the_render_reference_shape():
    """The record-level reference (what the GPU tests use) differentiates the same composition: on a hand-built frame its
    cotangents for random record cotangents match finite differences."""
    case = pz.get("actors_and_background")
    v = np.random.default_rng(3).uniform(-1, 1, (case.fwd["records"].shape[0], 12))
    base = pz.frame_poses(case.frame).astype(np.float64)
    got = pz.v_pose_ref(case.frame, case.st, v, base)
    assert got.shape == (4, 16) and np.all(got[3] == 0) and np.abs(got[:3]).min(1).max() > 0  # the empty actor: zeros
    eps = 1e-6
    rng = np.random.default_rng(4)
    for _ in range(12):
        a, j = int(rng.integers(0, 3)), int(rng.integers(0, 16))
        vals = []
        for sgn in (1, -1):
            p = base.copy()
            p[a, j] += sgn * eps
            with torch.no_grad():
                vals.append(float(pz.record_loss(case.frame, case.st, v, torch.tensor(p))[0]))
        fd = (vals[0] - vals[1]) / (2 * eps)
        assert abs(fd - got[a, j]) <= 2e-5 * max(1.0, abs(fd)), (a, j, fd, got[a, j])


def test_hand_built_cases_cover_what_they_name():
    c = pz.get("off_screen")
    n = [s.params.num_points for s in c.frame.segments]
    assert not c.fwd["vis"][n[0] + n[1]:].any() and c.fwd["vis"][:n[0] + n[1]].any()
    c = pz.get("clip_plane")
    assert 100 <= int((~c.fwd["unclipped"]).sum()) <= 160 and c.fwd["vis"].sum() > 50
    c = pz.get("actors_and_background")
    assert [s.params.num_points for s in c.frame.segments] == [300, 300, 50, 128, 0]


def test_pose_table_fills_frame_id_and_indices():
    def obj(gid, x):
        return dict(type="car", is_moving=True, gid=gid, translation=[x, 0.0, 0.0], rotation=[1.0, 0.0, 0.0, 0.0], size=[4.0, 2.0, 1.5])
    frames = [dict(timestamp=1000 + 100 * i, objects=[obj("a", float(i)), obj("b", 5.0 + i)]) for i in range(3)]
    tab = PoseTable(frames)
    fmap = tab.frame_idx_map()
    assert list(fmap.values()) == [0, 1, 2]
    bo = BoxPoseOptimizer(len(tab), tab.unique_track_ids, fmap, mode="simple")
    at = tab.poses_at(int(tab.all_names[1]))
    assert [p.frame_id for p in at] == [int(tab.all_names[1])] * 2
    assert bo.indices(at) == ([1, 1], [0, 1])
    between = tab.poses_at((int(tab.all_names[1]) + int(tab.all_names[2])) // 2)
    assert len(between) == 2 and all(p.frame == -1 and p.frame_id is None for p in between)
    assert bo.indices(between) == ([-1, -1], [-1, -1])
    legacy = ActorPose("a", np.eye(3), np.zeros(3), 1, [0, 1, 2])  # no frame_id: not corrected
    assert legacy.frame_id is None and bo.indices([legacy]) == ([-1], [-1])
    assert np.allclose(quaternion_matrix([1, 0, 0, 0])[:3, :3], np.eye(3))
