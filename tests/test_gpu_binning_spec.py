"""The per-tile lists and their class sub-lists checked against their specification (not against an earlier build):

* every tile's ids are strictly increasing in (depth bits, row), and each payload carries its row's object-class bit;
* the (tile, row) pairs are exactly those the projection's tile_bbox + touch_mask decode to; rows whose AABB exceeds the mask
  (more than 32 tiles) list tiles_touched distinct tiles of their AABB;
* tile_bins are the contiguous ranges of the tiles in tile order, (0, 0) for an empty tile;
* each class sub-list is the stable partition of its tile's list, and cls_bins are the exclusive scans of the class counts
  (an empty tile gets the scanned offset, with zero length).

On small scenes and at config 3, in the synchronous mode and in the capped mode without the count's read-back, including a
capacity the frame overflows: the truncated lists are the first `capacity` entries of the depth-ordered entry sequence."""
import numpy as np
import pytest
import torch

import street_gaussians_ns_b200.synthetic as syn
from street_gaussians_ns_b200 import raster
from street_gaussians_ns_b200.scene import Frame, Segment
from oracle.bin_ref64 import COOP_AREA, check_lists, emission_prefix, expected_pairs, list_order

pytestmark = pytest.mark.gpu

SCENES = {
    "actors_in_front": lambda: syn.make_frame(n_background=60000, n_actors=4, n_per_actor=3000, width=128, height=96, seed=12,
                                              actor_shift=np.array([0.0, 0.0, 4.0])),
    "long_lists": lambda: syn.make_frame(n_background=300000, n_actors=3, n_per_actor=6000, width=64, height=48, seed=5,
                                         actor_shift=np.array([1.0, 0.0, 2.0])),
    "wide": lambda: syn.make_frame(n_background=40000, n_actors=6, n_per_actor=2000, width=640, height=360, seed=9),
    "config3": lambda: syn.config_frame(3),
}


def project(fr):
    frc = Frame(fr.camera, [Segment(s.params.to("cuda:0"), s.cls, s.rot, s.center, s.idft, s.name) for s in fr.segments])
    settings = raster.RenderSettings()
    params = [seg.params.tensors() for seg in frc.segments]
    cs = raster.camera_struct(frc.camera, settings)
    table = raster.SegmentTable(frc, params, torch.device("cuda", 0))
    return cs, raster.project_fwd(table, cs, torch.device("cuda", 0))


def host_rows(proj):
    rec = proj.records.cpu().numpy()
    return dict(depth=rec[:, 9].view(np.uint32).astype(np.uint64), obj=(rec[:, 10].view(np.int32) & 0x8) != 0,
                radii=proj.radii.cpu().numpy(), bbox=proj.bbox.cpu().numpy().view(np.uint16).astype(np.int64),
                touched=proj.tiles_touched.cpu().numpy().astype(np.int64), mask=proj.touch_mask.cpu().numpy().view(np.uint32))


def spec_entries(h, tiles_x, lists_tile, lists_row):
    """All entries in list order: the small AABBs from their masks, the big ones as listed (checked against tiles_touched)."""
    st, sr, area = expected_pairs(h, tiles_x)
    big = np.isin(lists_row, np.nonzero((h["radii"] > 0) & (area > COOP_AREA))[0])
    bt, br = lists_tile[big], lists_row[big]
    bb = h["bbox"][br]
    tx, ty = bt % tiles_x, bt // tiles_x
    assert np.all((tx >= bb[:, 0]) & (tx < bb[:, 2]) & (ty >= bb[:, 1]) & (ty < bb[:, 3]))
    assert len(np.unique(bt.astype(np.int64) * (1 << 32) + br)) == len(bt)
    big_rows = np.nonzero((h["radii"] > 0) & (area > COOP_AREA))[0]
    assert np.array_equal(np.bincount(br, minlength=len(area))[big_rows], h["touched"][big_rows])
    small = (h["radii"] > 0) & (area <= COOP_AREA)
    popc = np.unpackbits(h["mask"][small].view(np.uint8)).reshape(-1, 32).sum(1)
    assert np.array_equal(h["touched"][small], popc)
    tile = np.concatenate([st, bt])
    row = np.concatenate([sr, br])
    return tile, row


@pytest.fixture(scope="module", params=list(SCENES))
def scene(request):
    cs, proj = project(SCENES[request.param]())
    return request.param, cs, proj, host_rows(proj)


def run(cs, proj, async_binning):
    M, ids, bins = raster.bin_and_sort(cs, proj.records, proj.radii, proj=proj, async_binning=async_binning)
    cls_ids, cls_bins = raster.class_lists(cs, M, ids, bins)
    torch.cuda.synchronize()
    return M, ids.cpu().numpy(), bins.cpu().numpy(), cls_ids.cpu().numpy(), cls_bins.cpu().numpy()


def test_lists_match_specification(scene):
    name, cs, proj, h = scene
    tiles_x = (cs.width + cs.block_width - 1) // cs.block_width
    tiles = tiles_x * ((cs.height + cs.block_width - 1) // cs.block_width)
    M, ids, bins, cls_ids, cls_bins = run(cs, proj, async_binning=False)
    assert M == int(h["touched"][h["radii"] > 0].sum())
    tile_of = np.repeat(np.arange(tiles), bins[:, 1] - bins[:, 0])
    want = list_order(h, *spec_entries(h, tiles_x, tile_of, ids[:M] & 0x7FFFFFFF))
    check_lists(h, tiles_x, tiles, ids, bins, cls_ids, cls_bins, want)

    # capped mode, no read-back: the first frame learns the count, the second runs without it
    raster._ASYNC_STATE.clear()
    run(cs, proj, async_binning=True)
    Mc, ids_c, bins_c, cls_c, cls_bins_c = run(cs, proj, async_binning=True)
    assert isinstance(Mc, raster.LazyCount) and int(Mc) == M and len(ids_c) > M
    check_lists(h, tiles_x, tiles, ids_c, bins_c, cls_c, cls_bins_c, want)
    assert np.array_equal(ids_c[:M], ids[:M]) and np.array_equal(bins_c, bins)

    # a capacity the frame overflows: the lists hold the first `capacity` entries of the depth-ordered sequence
    st = raster._ASYNC_STATE[str(torch.device("cuda", 0))]
    raster._async_poll(st)
    st["max_m"] = max(1, M // 3)
    granule, raster.ASYNC_GRANULE = raster.ASYNC_GRANULE, 256
    try:
        Mo, ids_o, bins_o, cls_o, cls_bins_o = run(cs, proj, async_binning=True)
    finally:
        raster.ASYNC_GRANULE = granule
        raster._ASYNC_STATE.clear()
    cap = Mo.capacity
    assert Mo.raw() == M and int(Mo) == cap < M
    kept = list_order(h, *emission_prefix(h, *want, cap))
    check_lists(h, tiles_x, tiles, ids_o, bins_o, cls_o, cls_bins_o, kept)
