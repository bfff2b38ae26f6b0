"""The host binning reference (oracle/bin_ref64.py) checked on the CPU: with the touch filter off its lists are the C
oracle's gsplat lists on the parity scenes; its touch decisions are those of project_ref64 on the projection cases; and the
hand-built cases (tests/bin_cases.py) drive the paths they were built for."""
import numpy as np
import pytest

import street_gaussians_ns_b200.synthetic as syn
from oracle import bin_ref64 as ref
from oracle import oracle_c
from oracle import project_ref64 as pref
from tests import bin_cases as bc
from tests import project_cases as pc
from tests.test_blend_ref64 import PARITY_SCENES


@pytest.mark.parametrize("name", list(PARITY_SCENES))
def test_lists_without_touch_filter_equal_c_oracle(name):
    fr = syn.make_frame(**PARITY_SCENES[name])
    orc = oracle_c.Oracle(fr)
    pr = orc.project()
    M, ids, bins = orc.bin_sort(pr)
    N = orc.N
    rec = np.zeros((N, 12), np.float32)
    rec[:, 0:2], rec[:, 2:5], rec[:, 5], rec[:, 9] = pr["xys"], pr["conics"], pr["opac"], pr["depths"]
    rec[:, 10] = (np.where(orc.cls == 1, ref.AUX_OBJECT, 0).astype(np.int32)).view(np.float32)
    h = ref.rows(rec, pr["radii"], pr["tile_bbox"], pr["num_tiles_hit"], np.zeros(N, np.uint32))
    cam = fr.camera
    tile, row = ref.entries(h, cam.width, cam.height, 16, touch_filter=False)
    want_ids, want_bins = ref.lists(h, len(bins), *ref.list_order(h, tile, row))
    assert len(want_ids) == M > 0
    np.testing.assert_array_equal(want_ids & 0x7FFFFFFF, ids)
    np.testing.assert_array_equal(want_ids < 0, orc.cls[ids] == 1)
    cnt = bins[:, 1] - bins[:, 0]
    nz = cnt > 0
    np.testing.assert_array_equal(want_bins[nz], bins[nz])  # the oracle gives an empty tile its offset, the product (0, 0)
    assert np.all(want_bins[~nz] == 0)
    # the scan: depth order of the visible rows, the invisible ones behind them
    sc = ref.scan(h)
    vis = pr["radii"] > 0
    assert np.all(vis[sc["rows"][:vis.sum()]]) and sc["total"] == M


@pytest.mark.parametrize("name", ["touch_bw16", "touch_bw2", "edges_333x177_bw2", "edges_17x3_bw16", "shapes"])
def test_touch_decisions_match_projection_reference(name):
    """On the projection's float64 forward (records rounded to float32 as the kernels store them): every decided tile of
    bin_ref64's touch test is project_ref64's min sigma <= tau, and touch_counts agrees wherever no tile is in the band."""
    case = pc.get(name)
    fw = case.fwd
    cam, bw = case.frame.camera, case.st.block_width
    rec = fw["records"].astype(np.float32)
    bbox = np.concatenate([fw["tmin"], fw["tmax"]], 1)
    h = ref.rows(rec, fw["radii"], bbox, np.zeros(len(rec), np.int64), np.zeros(len(rec), np.uint32))
    decided = 0
    for g, (tiles, must, may) in ref.touch(h, cam.width, cam.height, bw).items():
        _, _, d, mag = pref.touch_min_sigma(rec[g, 0:2].astype(np.float64), rec[g, 2:5].astype(np.float64), float(rec[g, 5]),
                                            fw["tmin"][g], fw["tmax"][g], cam.width, cam.height, bw)
        np.testing.assert_array_equal(must, d <= 0)
        np.testing.assert_array_equal(may, d <= ref.TOUCH_A + ref.TOUCH_R * mag)
        x0, y0, x1, y1 = bbox[g]
        assert np.array_equal(tiles, (np.arange(y0, y1)[:, None] * ((cam.width + bw - 1) // bw) + np.arange(x0, x1)).reshape(-1))
        decided += int(np.array_equal(must, may))
    assert decided > 0.5 * len(np.nonzero(fw["vis"])[0])


def test_cases_drive_their_paths():
    p = {n: bc.get(n).paths() for n in bc.CASES}
    for n, v in p.items():
        print(n, v)
    assert len(bc.SHAPES) == 119
    assert p["mask_shapes"]["small"] >= 5 * 119
    assert bc.get("warp_sums").notes["warp_sums"] == [32, 33, 1024, 32, 1]
    for n in ("big_runs_1920x1280_bw16", "big_runs_400x300_bw2"):
        c = bc.get(n)
        area = ref.areas(c.h())
        vis = c.radii > 0
        assert p[n]["warp"] >= 10 and p[n]["cta"] >= 4 and p[n]["small"] >= 20, n
        for a in (33, 64, 1024, 1025, c.tiles):
            assert np.any(vis & (area == a) & (c.touched > 0)), (n, a)
        assert np.any(vis & (area > 32) & (c.touched == 0)), n            # opacity below 1/255
        reached = vis & (area > 32) & (c.touched > 0)
        assert np.any(reached & (c.touched < area)), n                    # sparse reached sets
        assert c.geometric
    c = bc.get("big_runs_1920x1280_bw16")
    assert c.bw == 16 and (c.width, c.height) == (1920, 1280)
    h = bc.get("ties").h()
    vis = h["radii"] > 0
    assert np.bincount(h["depth"][vis].astype(np.int64)).max() >= 200
    assert p["ties"]["both"] > 100 and (~vis).sum() >= 50
    assert p["empty"]["M"] == 0 and p["single"]["M"] == 1
    assert p["classes_bw2"]["tiles"] > 14000 and p["classes_bw2"]["longest"] > 512
    assert min(p["classes_bw2"][k] for k in ("bg_only", "obj_only", "both")) > 1000
    for n, t in (("tiles_1", 1), ("tiles_15", 15), ("tiles_16", 16), ("tiles_17", 17), ("tiles_65535", 65535), ("tiles_65536", 65536)):
        r = bc.get(n).ref()
        assert p[n]["tiles"] == t and r["bins"][t - 1, 1] > r["bins"][t - 1, 0] and r["bins"][0, 1] > 0, n
    lens = bc.get("local_1024_1025_8192_1").ref()["bins"]
    assert (lens[:, 1] - lens[:, 0]).tolist() == [1024, 1025, 8192, 1]
    assert p["local_8193"]["longest"] == 8193
