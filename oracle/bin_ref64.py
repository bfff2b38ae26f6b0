"""Host statement of the binning stage (csrc/binning.cu, csrc/binning_local.cu), in numpy.  TEST INFRASTRUCTURE -- never
imported by the product.  Every output is an integer, so the kernels are compared with it exactly.

Written from the contract (the binning.cu / binning_local.cu headers, include/sgn_raster.h), not from the kernels:
  * scan (sgn_bin_scan): the rows in order of their key -- the depth bits for a visible row (radii > 0), 0xffffffff for an
    invisible one -- stable in the row index; the payload is row | object << 31 for a visible row and the bare row for an
    invisible one; cum is the inclusive scan of tiles_touched in that order (every row's value, invisible ones included),
    total its last value (0 for N = 0);
  * tiles of a row: an AABB of at most 32 tiles lists the tiles of the set bits of its touch mask (bit k = AABB tile k,
    row-major); a larger one lists the AABB tiles the touch test reaches (project_ref64.touch_min_sigma: min sigma over the
    tile's pixel-centre rectangle <= tau = ln(255 o); a degenerate conic keeps every tile).  The decision is exact when no
    tile lies in the band between "must keep" (d <= 0) and "may keep" (d <= TOUCH_A + TOUCH_R |terms|): the case builders
    move opacities until that holds;
  * emission sequence: the runs in scan order, tiles ascending inside a run; the capped form keeps its first `cap` entries;
  * lists: the entries in (tile, depth bits, row) order; tile_bins the contiguous range of every tile, (0, 0) when empty;
  * class sub-lists: the stable partition of every tile's list into background (class 0) and object (class 1) entries.
    sgn_bin_class_lists places class c of tile t at the exclusive scan of the class-c counts over the tiles; the local
    variant places it at the tile's own offset tile_bins[t, 0] ((0, 0) for an empty tile).
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np

from oracle import project_ref64 as pref

COOP_AREA = 32     # AABBs up to this many tiles carry a touch mask
HUGE_AREA = 1024   # emit_big_kernel: runs of larger AABBs are taken by a whole CTA, the others by one warp
TOUCH_A, TOUCH_R = 2e-3, 1e-5  # the "may keep" band of the touch test (as in the projection's directed tests)
AUX_OBJECT = 8


def rows(records, radii, bbox, touched, mask) -> Dict[str, np.ndarray]:
    """Host view of the binning inputs: records [N,12] float32, radii, tile_bbox [N,4] (x0, y0, x1, y1), tiles_touched,
    touch_mask."""
    rec = np.ascontiguousarray(records, np.float32)
    return dict(rec=rec, depth=rec[:, 9].view(np.uint32).astype(np.uint64), obj=(rec[:, 10].view(np.int32) & AUX_OBJECT) != 0,
                radii=np.asarray(radii).astype(np.int64), bbox=np.asarray(bbox).astype(np.int64),
                touched=np.asarray(touched).astype(np.int64), mask=np.asarray(mask).astype(np.uint32))


def areas(h):
    bb = h["bbox"]
    return (bb[:, 2] - bb[:, 0]) * (bb[:, 3] - bb[:, 1])


def payload(h, row):
    return (row.astype(np.uint32) | (h["obj"][row].astype(np.uint32) << np.uint32(31))).view(np.int32)


# ------------------------------------------------------------------------------------------------------------------
# touch test
# ------------------------------------------------------------------------------------------------------------------
def degenerate(rec_row) -> bool:
    a, b, c = (float(v) for v in rec_row[2:5])
    return not (a > 0 and c > 0 and a * c - b * b > 0)


def touch_row(rec_row, bb, width, height, bw):
    """(tiles of the AABB in row-major order, must keep, may keep) of one visible row."""
    x0, y0, x1, y1 = (int(v) for v in bb)
    tiles_x = (width + bw - 1) // bw
    tys, txs = np.meshgrid(np.arange(y0, y1), np.arange(x0, x1), indexing="ij")
    tiles = (tys * tiles_x + txs).reshape(-1)
    if degenerate(rec_row):
        keep = np.ones(len(tiles), bool)
        return tiles, keep, keep
    _, _, d, mag = pref.touch_min_sigma(rec_row[0:2].astype(np.float64), rec_row[2:5].astype(np.float64), float(rec_row[5]),
                                        (x0, y0), (x1, y1), width, height, bw)
    return tiles, d <= 0, d <= TOUCH_A + TOUCH_R * mag


def touch(h, width, height, bw, sel=None):
    """{row: (tiles, must, may)} for the visible rows (or the rows of `sel`)."""
    idx = np.nonzero(h["radii"] > 0)[0] if sel is None else np.asarray(sel)
    return {int(g): touch_row(h["rec"][g], h["bbox"][g], width, height, bw) for g in idx}


def touch_counts(h, width, height, bw):
    """tiles_touched and touch_mask as the projection / sgn_bin_count must produce them (rows with a tile in the band
    raise: their decision is not exact)."""
    N = len(h["radii"])
    touched = np.zeros(N, np.int64)
    mask = np.zeros(N, np.uint32)
    for g, (tiles, must, may) in touch(h, width, height, bw).items():
        assert np.array_equal(must, may), f"row {g}: an AABB tile lies in the touch band"
        touched[g] = must.sum()
        if len(tiles) <= COOP_AREA:
            mask[g] = np.uint32(int((must.astype(np.int64) << np.arange(len(must))).sum()))
    return touched, mask


# ------------------------------------------------------------------------------------------------------------------
# scan, entries, lists
# ------------------------------------------------------------------------------------------------------------------
def scan(h):
    """sgn_bin_scan: order (payloads in scan order), cum, total, and the scan order's rows and ranks."""
    vis = h["radii"] > 0
    key = np.where(vis, h["depth"], np.uint64(0xFFFFFFFF))
    order_rows = np.argsort(key, kind="stable")
    pl = np.where(vis[order_rows], payload(h, order_rows), order_rows.astype(np.int32))
    cum = np.cumsum(h["touched"][order_rows])
    rank = np.empty(len(order_rows), np.int64)
    rank[order_rows] = np.arange(len(order_rows))
    return dict(order=pl.astype(np.int32), cum=cum.astype(np.int64), total=int(cum[-1]) if len(cum) else 0, rows=order_rows,
                rank=rank)


def expected_pairs(h, tiles_x):
    """(tile, row) of every entry the masks decode to (AABBs of at most 32 tiles)."""
    bb, mask = h["bbox"], h["mask"].astype(np.int64)
    w, area = bb[:, 2] - bb[:, 0], (bb[:, 2] - bb[:, 0]) * (bb[:, 3] - bb[:, 1])
    small = np.nonzero((h["radii"] > 0) & (area <= COOP_AREA) & (mask != 0))[0]
    tiles, rows_ = [], []
    for b in range(32):
        r = small[((mask[small] >> b) & 1).astype(bool)]
        assert np.all(b < area[r])
        tiles.append((bb[r, 1] + b // w[r]) * tiles_x + bb[r, 0] + b % w[r])
        rows_.append(r)
    return np.concatenate(tiles), np.concatenate(rows_), area


def entries(h, width, height, bw, touch_filter=True):
    """(tile, row) of every entry, in no particular order.  touch_filter=False lists every tile of every AABB (gsplat's
    lists, which the C oracle builds)."""
    tiles_x = (width + bw - 1) // bw
    vis = h["radii"] > 0
    area = areas(h)
    if not touch_filter:
        rr = np.nonzero(vis & (area > 0))[0]
        bb = h["bbox"][rr]
        w = bb[:, 2] - bb[:, 0]
        row = np.repeat(rr, area[rr])
        k = np.arange(len(row)) - np.repeat(np.cumsum(area[rr]) - area[rr], area[rr])
        wr = np.repeat(w, area[rr])
        tile = (np.repeat(bb[:, 1], area[rr]) + k // wr) * tiles_x + np.repeat(bb[:, 0], area[rr]) + k % wr
        return tile.astype(np.int64), row.astype(np.int64)
    st, sr, _ = expected_pairs(h, tiles_x)
    bt, br = [st], [sr]
    for g, (tiles, must, may) in touch(h, width, height, bw, np.nonzero(vis & (area > COOP_AREA))[0]).items():
        assert np.array_equal(must, may), f"row {g}: an AABB tile lies in the touch band"
        bt.append(tiles[must])
        br.append(np.full(int(must.sum()), g, np.int64))
    tile, row = np.concatenate(bt).astype(np.int64), np.concatenate(br).astype(np.int64)
    # the input contract: tiles_touched counts a visible row's entries
    assert np.array_equal(np.bincount(row, minlength=len(vis))[vis], h["touched"][vis]), "tiles_touched != the listed tiles"
    return tile, row


def list_order(h, tile, row):
    """Sort (tile, row) pairs by (tile, depth bits, row)."""
    o = np.lexsort((row, h["depth"][row], tile))
    return tile[o], row[o]


def emission_prefix(h, tile, row, n):
    """The first n entries of the depth-ordered entry sequence: runs in (depth bits, row) order, tiles ascending in a run."""
    o = np.lexsort((tile, row, h["depth"][row]))[:n]
    return tile[o], row[o]


def lists(h, tiles, tile, row):
    """(sorted_ids, tile_bins) of entries already in list order."""
    cnt = np.bincount(tile, minlength=tiles).astype(np.int64)
    start = np.cumsum(cnt) - cnt
    bins = np.stack([np.where(cnt > 0, start, 0), np.where(cnt > 0, start + cnt, 0)], 1)
    return payload(h, row), bins


def class_lists(ids, bins, stride, variant="default"):
    """(cls_ids [2, stride], defined [2, stride], cls_bins [2, tiles, 2]) of the lists (ids, bins); `defined` marks the slots
    the contract fixes (the others are unspecified)."""
    tiles = len(bins)
    tile_of = np.repeat(np.arange(tiles), bins[:, 1] - bins[:, 0])
    M = len(tile_of)
    ids = ids[:M]
    cls_ids = np.zeros((2, stride), np.int32)
    defined = np.zeros((2, stride), bool)
    cls_bins = np.zeros((2, tiles, 2), np.int64)
    for c, sel in ((0, ids >= 0), (1, ids < 0)):
        n_c = np.bincount(tile_of[sel], minlength=tiles)
        if variant == "default":
            lo = np.cumsum(n_c) - n_c
            pos = np.arange(int(n_c.sum()))
        else:
            lo = bins[:, 0]
            # entry j of tile t's class-c sub-list sits at tile_bins[t, 0] + j
            first = np.cumsum(n_c) - n_c
            pos = lo[tile_of[sel]] + np.arange(int(n_c.sum())) - first[tile_of[sel]]
        cls_bins[c, :, 0], cls_bins[c, :, 1] = lo, lo + n_c
        cls_ids[c, pos] = ids[sel]
        defined[c, pos] = True
    return cls_ids, defined, cls_bins


def reference(h, width, height, bw, cap: Optional[int] = None):
    """Every output of the binning stage for the rows h; with `cap`, the capped form's (sorted_ids has `cap` slots, the
    ones past min(M, cap) hold the padding payload 0)."""
    tiles_x, tiles_y = (width + bw - 1) // bw, (height + bw - 1) // bw
    tiles = tiles_x * tiles_y
    sc = scan(h)
    tile, row = entries(h, width, height, bw)
    M = len(tile)
    assert M == sc["total"]
    keep = M if cap is None else min(M, cap)
    tile, row = list_order(h, *emission_prefix(h, tile, row, keep))
    ids, bins = lists(h, tiles, tile, row)
    stride = max(M, 1) if cap is None else cap
    full = np.zeros(stride, np.int32)
    full[:keep] = ids
    return dict(scan=sc, M=M, kept=keep, tile=tile, row=row, ids=full, bins=bins, tiles=tiles, tiles_x=tiles_x,
                overflow=cap is not None and M > cap)


def check_lists(h, tiles_x, tiles, ids, tile_bins, cls_ids, cls_bins, want_entries):
    """want_entries: (tile, row) of every listed entry, in list order (tile, depth bits, row)."""
    M = len(want_entries[0])
    ids = ids[:M]
    row = ids & 0x7FFFFFFF
    tile_of = np.repeat(np.arange(tiles), tile_bins[:, 1] - tile_bins[:, 0])
    # tile_bins: contiguous in tile order, (0, 0) when empty
    cnt = tile_bins[:, 1] - tile_bins[:, 0]
    assert np.all(cnt >= 0) and cnt.sum() == M
    nz = cnt > 0
    assert np.array_equal(tile_bins[nz, 0], (np.cumsum(cnt) - cnt)[nz])
    assert np.all(tile_bins[~nz] == 0)
    # the entries are the specified (tile, row) pairs, in the specified order
    assert np.array_equal(tile_of, want_entries[0])
    assert np.array_equal(row, want_entries[1])
    assert np.array_equal(ids < 0, h["obj"][row])
    key = (h["depth"][row] << np.uint64(32)) | row.astype(np.uint64)
    same = tile_of[1:] == tile_of[:-1]
    assert np.all(key[1:][same] > key[:-1][same]), "a tile's ids are not strictly increasing in (depth bits, row)"
    # class sub-lists: stable partition, offsets are exclusive scans of the class counts
    is_obj = ids < 0
    for c, sel in ((0, ~is_obj), (1, is_obj)):
        n_c = np.bincount(tile_of[sel], minlength=tiles)
        scan_ = np.cumsum(n_c) - n_c
        assert np.array_equal(cls_bins[c, :, 0], scan_), c
        assert np.array_equal(cls_bins[c, :, 1], scan_ + n_c), c
        assert np.array_equal(cls_ids[c, :int(n_c.sum())], ids[sel]), c  # per tile in order, tiles in order: the stable partition
