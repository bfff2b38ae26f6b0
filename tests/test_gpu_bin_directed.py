"""The binning kernels on hand-built rows (tests/bin_cases.py) against the host statement of the stage
(oracle/bin_ref64.py).  Every output is an integer, so every comparison is exact.

  * sgn_bin_scan: the payloads in depth order (invisible rows last, bare row), the inclusive scan and the total;
  * sgn_bin_sort: sorted ids and tile_bins; sgn_bin_class_lists: class ids and cls_bins (exclusive scans of the class counts);
  * sgn_bin_sort_capped: with room to spare on every case (the padding key above the last tile), and cut at 1, at the end of
    a small run, inside a small, a warp-path and a CTA-path run, at M - 1, M, M + 1 and far above M: the truncated prefix,
    the class lists at the capacity's stride, the overflow flag (set exactly when M > capacity, otherwise left alone) and
    the padding payload 0 past min(M, capacity);
  * sgn_bin_count: tiles_touched row by row and touch_mask bit by bit on the cases built from real conics, and bit-identical
    to project_fwd on the projection's touch cases;
  * the local variant (binning_local.cu) on the same cases, class sub-lists at the tile's own offset, tiles of 1024, 1025
    and 8192 entries; a tile of 8193 makes it decline, and bin_and_sort falls back to the device-wide path;
  * argument errors of the binning ABI: status and message;
  * a camera of 65536 tiles (the capped form has no 16-bit key left for its padding): bin_and_sort renders it in both
    modes, as it does 65535 tiles.

The kernels are called through the ABI with zero-filled outputs and scratch, so a slot a kernel fails to write reads 0
(a valid tile key) rather than whatever the allocator held.

Observed on an H100 80GB HBM3 (700 W power limit), 43 tests in 9.4 s.  Before this file, bin_and_sort in the capped mode
raised on a camera of exactly 65536 tiles (the padding sentinel needs a 17th key bit); it now falls back to the synchronous
form there.  Nine one-token changes each fail at least one test here: nth_set_bit's `k >= c` -> `k > c` (18 tests), the
CTA path's warp prefix `k < warp` -> `k <= warp` (4), the warp path's position + 1 (5), the overflow flag's `>` -> `>=` (2),
bin_edges_kernel's last end M -> M - 1 (19), the invisible rows' depth key 0xffffffff -> 0 (13), the class look-back's
`lane <= stop` -> `lane < stop` (15), the local sort's padding key -> 0 (13), local_sort_kernel's `n > HI` -> `n >= HI` (1).
test_gpu_binning_spec.py, the parity binning test and the experimental local-vs-default tests catch four of the seven
that leave no slot of the key buffer unwritten (nth_set_bit, the last bin end, the look-back, the local padding) and miss
the overflow flag, the invisible key and the local size class; the two position mutants were not run against them, since
those tests allocate the key scratch uninitialised.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from street_gaussians_ns_b200 import _lib, raster
from street_gaussians_ns_b200.scene import Frame, Segment
from oracle import bin_ref64 as ref
from tests import bin_cases as bc
from tests import project_cases as pc

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
ERR_INVALID, ERR_WORKSPACE = -1, -3


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _z(n, dtype=torch.int32):
    return torch.zeros(n, dtype=dtype, device=DEV)


def camera(width, height, bw):
    cs = _lib.CameraStruct()
    cs.width, cs.height, cs.block_width = width, height, bw
    return cs


def inputs(case):
    return dict(cs=camera(case.width, case.height, case.bw), N=case.N,
                rec=torch.from_numpy(case.records.copy()).to(DEV), radii=torch.from_numpy(case.radii.astype(np.int32)).to(DEV),
                bbox=torch.from_numpy(case.bbox.astype(np.uint16).view(np.int16).copy()).to(DEV),
                touched=torch.from_numpy(case.touched.astype(np.int32)).to(DEV),
                mask=torch.from_numpy(case.mask.astype(np.uint32).view(np.int32).copy()).to(DEV))


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def run_scan(L, d):
    N = d["N"]
    order, cum, total = _z(max(N, 1)), _z(max(N, 1)), _z(1, torch.int64)
    sb = L.sgn_bin_scan_scratch_bytes(N)
    scratch = _z(sb, torch.uint8)
    _lib.check(L.sgn_bin_scan(N, _p(d["rec"]), _p(d["radii"]), _p(d["touched"]), _p(order), _p(cum), _p(total), _p(scratch), sb,
                              None), "sgn_bin_scan")
    return order, cum, total


def run_sort(L, case, d, scan, M, cap=None):
    """sgn_bin_sort (cap None) or sgn_bin_sort_capped: (sorted_ids, tile_bins, overflow flag or None)."""
    n = max(M, 1) if cap is None else cap
    ids, bins = _z(n), _z((case.tiles, 2))
    sb = L.sgn_bin_sort_scratch_bytes(n if cap is not None else M)
    scratch = _z(sb, torch.uint8)
    args = (_p(d["rec"]), _p(d["radii"]), _p(d["bbox"]), _p(d["mask"]), _p(scan[0]), _p(scan[1]), _p(ids), _p(bins), _p(scratch), sb, None)
    if cap is None:
        _lib.check(L.sgn_bin_sort(d["N"], M, C.byref(d["cs"]), *args), "sgn_bin_sort")
        return ids, bins, None
    overflow = torch.full((1,), 7, dtype=torch.int32, device=DEV)  # 7: "not written"
    _lib.check(L.sgn_bin_sort_capped(d["N"], cap, _p(scan[2]), _p(overflow), C.byref(d["cs"]), *args), "sgn_bin_sort_capped")
    return ids, bins, overflow


def run_classes(L, d, ids, bins):
    stride, tiles = ids.shape[0], bins.shape[0]
    cls_ids, cls_bins = _z((2, stride)), _z((2, tiles, 2))
    sb = L.sgn_bin_class_scratch_bytes(tiles)
    scratch = _z(sb, torch.uint8)
    _lib.check(L.sgn_bin_class_lists(C.byref(d["cs"]), stride, _p(ids), _p(bins), _p(cls_ids), _p(cls_bins), _p(scratch), sb, None),
               "sgn_bin_class_lists")
    return cls_ids, cls_bins


def check_scan(case, order, cum, total):
    sc = case.ref()["scan"]
    N = case.N
    np.testing.assert_array_equal(host(order)[:N], sc["order"], err_msg=f"{case.name}: order")
    np.testing.assert_array_equal(host(cum)[:N], sc["cum"], err_msg=f"{case.name}: cum")
    assert int(host(total)[0]) == sc["total"]


def check_lists(case, r, ids, bins, cls=None, variant="default", tag=""):
    what = f"{case.name}{tag}"
    ids_h, bins_h = host(ids), host(bins)
    M = r["kept"]
    got_tile = np.repeat(np.arange(case.tiles), np.maximum(bins_h[:, 1] - bins_h[:, 0], 0))
    if not np.array_equal(ids_h[:M], r["ids"][:M]):
        bad = int(np.nonzero(ids_h[:M] != r["ids"][:M])[0][0])
        raise AssertionError(f"{what}: sorted id {bad} of {M} is {ids_h[bad]} (row {ids_h[bad] & 0x7FFFFFFF}), expected "
                             f"{r['ids'][bad]} (row {r['row'][bad]}, tile {r['tile'][bad]})")
    np.testing.assert_array_equal(ids_h[M:], r["ids"][M:], err_msg=f"{what}: padding past the kept entries")
    if not np.array_equal(bins_h, r["bins"]):
        t = int(np.nonzero((bins_h != r["bins"]).any(1))[0][0])
        raise AssertionError(f"{what}: tile_bins[{t}] = {bins_h[t]}, expected {r['bins'][t]}")
    assert len(got_tile) == M
    if cls is not None:
        ci, cb = host(cls[0]), host(cls[1])
        want_ids, defined, want_bins = ref.class_lists(r["ids"], r["bins"], ci.shape[1], variant)
        for c in range(2):
            if not np.array_equal(cb[c], want_bins[c]):
                t = int(np.nonzero((cb[c] != want_bins[c]).any(1))[0][0])
                raise AssertionError(f"{what}: cls_bins[{c}][{t}] = {cb[c, t]}, expected {want_bins[c, t]}")
            np.testing.assert_array_equal(ci[c][defined[c]], want_ids[c][defined[c]], err_msg=f"{what}: class {c} ids")


@pytest.mark.parametrize("name", bc.LIST_CASES)
def test_lists_against_reference(name):
    """Scan, lists and class lists; then the capped form with room to spare (the padding key sorts behind the last tile)."""
    L = _lib.load()
    case = bc.get(name)
    d = inputs(case)
    r = case.ref()
    print(f"[{name}] {case.paths()}")
    scan = run_scan(L, d)
    check_scan(case, *scan)
    ids, bins, _ = run_sort(L, case, d, scan, r["M"])
    check_lists(case, r, ids, bins, run_classes(L, d, ids, bins))
    if case.tiles < 65536:
        cap = r["M"] + 300
        rc = case.ref(cap)
        ids, bins, ovf = run_sort(L, case, d, scan, r["M"], cap)
        check_lists(case, rc, ids, bins, run_classes(L, d, ids, bins), tag=f" [capacity {cap}]")
        assert int(host(ovf)[0]) == 7, f"{name}: the overflow flag was written although M <= capacity"


def _cuts(case):
    """Capacities at the edges of the runs of each emit path."""
    h = case.h()
    r = case.ref()
    sc = r["scan"]
    rows_, cum = sc["rows"], sc["cum"]
    start = np.concatenate([[0], cum[:-1]])
    n = cum - start
    area = ref.areas(h)[rows_]
    vis = h["radii"][rows_] > 0
    M = r["M"]
    small = np.nonzero(vis & (area <= ref.COOP_AREA) & (n >= 2) & (start > 0))[0]
    warp = np.nonzero(vis & (area > ref.COOP_AREA) & (area <= ref.HUGE_AREA) & (n > 34))[0]
    cta = np.nonzero(vis & (area > ref.HUGE_AREA) & (n > 300))[0]
    assert len(small) and len(warp) and len(cta), f"{case.name}: a run class to cut is missing"
    i, j, k = small[len(small) // 2], warp[len(warp) // 2], cta[0]
    cuts = {"1": 1, "small_end": int(cum[i]), "inside_small": int(start[i] + 1), "inside_warp": int(start[j] + 33),
            "inside_cta": int(start[k] + 300), "M-1": M - 1, "M": M, "M+1": M + 1, "far_above": 4 * M + 3}
    return cuts


@pytest.mark.parametrize("name", ["big_runs_1920x1280_bw16", "big_runs_400x300_bw2"])
def test_capacity_cuts(name):
    L = _lib.load()
    case = bc.get(name)
    d = inputs(case)
    M = case.ref()["M"]
    scan = run_scan(L, d)
    for label, cap in _cuts(case).items():
        r = case.ref(cap)
        ids, bins, ovf = run_sort(L, case, d, scan, M, cap)
        check_lists(case, r, ids, bins, run_classes(L, d, ids, bins), tag=f" [cut {label} = {cap} of {M}]")
        assert int(host(ovf)[0]) == (1 if M > cap else 7), f"{name}: overflow flag at capacity {cap} of {M}"


# ------------------------------------------------------------------------------------------------------------------
# the count kernel
# ------------------------------------------------------------------------------------------------------------------
def run_count(L, d):
    touched, mask = _z(max(d["N"], 1)), _z(max(d["N"], 1))
    _lib.check(L.sgn_bin_count(d["N"], C.byref(d["cs"]), _p(d["rec"]), _p(d["radii"]), _p(d["bbox"]), _p(touched), _p(mask), None),
               "sgn_bin_count")
    return host(touched)[:d["N"]], host(mask)[:d["N"]].view(np.uint32)


@pytest.mark.parametrize("name", [n for n in bc.LIST_CASES if n.startswith(("big_runs", "empty"))])
def test_count_kernel_against_reference(name):
    L = _lib.load()
    case = bc.get(name)
    assert case.geometric
    touched, mask = run_count(L, inputs(case))
    vis = case.radii > 0
    for g in np.nonzero(touched != case.touched)[0][:1]:
        raise AssertionError(f"{name}: row {g} (AABB {case.bbox[g].tolist()}) counts {touched[g]} tiles, expected {case.touched[g]}")
    want = np.where(vis, case.mask, 0).astype(np.uint32)
    for g in np.nonzero(mask != want)[0][:1]:
        diff = int(mask[g] ^ want[g])
        raise AssertionError(f"{name}: row {g}: touch mask {mask[g]:#010x}, expected {want[g]:#010x} (bits {diff:#010x})")


@pytest.mark.parametrize("name", ["touch_bw16", "touch_bw2"])
def test_count_kernel_equals_projection(name):
    L = _lib.load()
    case = pc.get(name)
    frc = Frame(case.frame.camera, [Segment(s.params.to("cuda"), s.cls, s.rot, s.center, s.idft) for s in case.frame.segments])
    st = case.st
    cs = raster.camera_struct(frc.camera, raster.RenderSettings(sh_degree=st.sh_degree, sh_degree_to_use=st.deg_use,
                                                               block_width=st.block_width, clip_thresh=st.clip_thresh))
    table = raster.SegmentTable(frc, [s.params.tensors() for s in frc.segments], DEV)
    pr = raster.project_fwd(table, cs, DEV)
    d = dict(cs=cs, N=table.N, rec=pr.records, radii=pr.radii, bbox=pr.bbox)
    touched, mask = run_count(L, d)
    assert touched.tobytes() == host(pr.tiles_touched).tobytes(), f"{name}: tiles_touched differs from project_fwd"
    assert mask.tobytes() == host(pr.touch_mask).view(np.uint32).tobytes(), f"{name}: touch_mask differs from project_fwd"
    assert (touched > 0).sum() > 20


# ------------------------------------------------------------------------------------------------------------------
# the local variant
# ------------------------------------------------------------------------------------------------------------------
def run_local(L, case, d, M, longest):
    tiles = case.tiles
    ids, bins, cls_ids, cls_bins = _z(max(M, 1)), _z((tiles, 2)), _z((2, max(M, 1))), _z((2, tiles, 2))
    sb = L.sgn_bin_local_scratch_bytes(M, tiles)
    scratch = _z(sb, torch.uint8)
    _lib.check(L.sgn_bin_local_sort(d["N"], M, longest, C.byref(d["cs"]), _p(d["rec"]), _p(d["radii"]), _p(d["bbox"]), _p(d["mask"]),
                                    _p(d["counts"][0]), _p(d["counts"][1]), _p(ids), _p(bins), _p(cls_ids), _p(cls_bins),
                                    _p(scratch), sb, None), "sgn_bin_local_sort")
    return ids, bins, (cls_ids, cls_bins)


def run_local_count(L, case, d):
    counts, info = _z((2, case.tiles)), _z(2, torch.int64)
    sb = L.sgn_bin_local_scratch_bytes(0, case.tiles)
    scratch = _z(sb, torch.uint8)
    _lib.check(L.sgn_bin_local_count(d["N"], C.byref(d["cs"]), _p(d["rec"]), _p(d["radii"]), _p(d["bbox"]), _p(d["mask"]),
                                     _p(counts[0]), _p(counts[1]), _p(info), _p(scratch), sb, None), "sgn_bin_local_count")
    d["counts"] = counts
    return host(counts), host(info)


@pytest.mark.parametrize("name", bc.LIST_CASES)
def test_local_variant_against_reference(name):
    L = _lib.load()
    case = bc.get(name)
    r = case.ref()
    d = inputs(case)
    counts, info = run_local_count(L, case, d)
    cnt = r["bins"][:, 1] - r["bins"][:, 0]
    np.testing.assert_array_equal(counts[0], cnt, err_msg=f"{name}: tile counts")
    np.testing.assert_array_equal(counts[1], np.cumsum(cnt) - cnt, err_msg=f"{name}: tile starts")
    assert tuple(info) == (r["M"], int(cnt.max(initial=0))), f"{name}: (M, longest) = {tuple(info)}"
    ids, bins, cls = run_local(L, case, d, r["M"], int(info[1]))
    check_lists(case, r, ids, bins, cls, variant="local", tag=" [local]")


def _projected(case):
    d = inputs(case)
    proj = raster.Projected(d["rec"], d["radii"], d["touched"], d["bbox"], d["touched"], d["mask"])
    return d, proj


def test_local_variant_declines_a_long_list(monkeypatch):
    """8193 entries in one tile: _bin_local returns None, and bin_and_sort builds the lists on the device-wide path."""
    case = bc.get("local_8193")
    d, proj = _projected(case)
    assert raster._bin_local(d["cs"], d["rec"], d["radii"], proj) is None
    monkeypatch.setattr(raster, "BIN_LOCAL", True)
    M, ids, bins = raster.bin_and_sort(d["cs"], d["rec"], d["radii"], proj=proj, async_binning=False)
    r = case.ref()
    assert M == r["M"]
    check_lists(case, r, ids, bins, raster.class_lists(d["cs"], M, ids, bins), tag=" [fallback]")


# ------------------------------------------------------------------------------------------------------------------
# the 65536-tile camera through bin_and_sort
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("async_binning", [False, True])
@pytest.mark.parametrize("name", ["tiles_65535", "tiles_65536"])
def test_tile_limit_camera(name, async_binning, monkeypatch):
    monkeypatch.setattr(raster, "BIN_LOCAL", False)
    case = bc.get(name)
    d, proj = _projected(case)
    r = case.ref()
    raster._ASYNC_STATE.clear()
    try:
        for frame in range(2 if async_binning else 1):  # the first frame of the capped mode learns the count
            M, ids, bins = raster.bin_and_sort(d["cs"], d["rec"], d["radii"], proj=proj, async_binning=async_binning)
            assert int(M) == r["M"]
            check_lists(case, r, ids[:r["M"]], bins, tag=f" [async {async_binning}, frame {frame}]")
        if async_binning:
            assert isinstance(M, raster.LazyCount) == (case.tiles < 65536)
    finally:
        raster._ASYNC_STATE.clear()


# ------------------------------------------------------------------------------------------------------------------
# argument errors
# ------------------------------------------------------------------------------------------------------------------
def _expect(rc, code, text):
    msg = _lib.load().sgn_last_error().decode("utf-8", "replace")
    assert rc == code and text in msg, f"status {rc}, message {msg!r}; expected {code} and {text!r}"


def test_argument_errors():
    L = _lib.load()
    case = bc.get("tiles_65536")
    d = inputs(case)
    cs, N, M = d["cs"], d["N"], case.ref()["M"]
    scan = run_scan(L, d)
    order, cum, total = scan
    ids, bins = _z(M), _z((case.tiles, 2))
    sb = L.sgn_bin_sort_scratch_bytes(M)
    scratch = _z(sb, torch.uint8)
    rec, radii, bbox, mask = _p(d["rec"]), _p(d["radii"]), _p(d["bbox"]), _p(d["mask"])
    S = (_p(order), _p(cum), _p(ids), _p(bins))

    # scan
    ssb = L.sgn_bin_scan_scratch_bytes(N)
    sscr = _z(ssb, torch.uint8)
    _expect(L.sgn_bin_scan(N, rec, radii, _p(d["touched"]), _p(order), _p(cum), _p(total), _p(sscr), ssb - 1, None), ERR_WORKSPACE,
            "sgn_bin_scan: scratch too small")
    _expect(L.sgn_bin_scan(N, None, radii, _p(d["touched"]), _p(order), _p(cum), _p(total), _p(sscr), ssb, None), ERR_INVALID,
            "sgn_bin_scan: null pointer")
    # count
    _expect(L.sgn_bin_count(N, C.byref(cs), rec, None, bbox, _p(ids), _p(ids), None), ERR_INVALID, "sgn_bin_count: null pointer")
    # sort
    big = camera(514, 512, 2)  # 257 x 256 tiles
    _expect(L.sgn_bin_sort(N, M, C.byref(big), rec, radii, bbox, mask, *S, _p(scratch), sb, None), ERR_INVALID,
            "more than 65536 tiles")
    for bad_m in (-1, 1 << 31):
        _expect(L.sgn_bin_sort(N, bad_m, C.byref(cs), rec, radii, bbox, mask, *S, _p(scratch), sb, None), ERR_INVALID,
                "out of the int32 range")
    _expect(L.sgn_bin_sort(N, M, C.byref(cs), rec, radii, bbox, mask, *S, _p(scratch), sb - 1, None), ERR_WORKSPACE,
            "sgn_bin_sort: scratch too small")
    _expect(L.sgn_bin_sort(N, M, C.byref(cs), None, radii, bbox, mask, *S, _p(scratch), sb, None), ERR_INVALID,
            "sgn_bin_sort: null pointer")
    _expect(L.sgn_bin_sort(N, M, C.byref(cs), rec, radii, bbox, mask, S[0], S[1], None, S[3], _p(scratch), sb, None), ERR_INVALID,
            "sorted_ids is null")
    # capped form
    ovf = _z(1)
    _expect(L.sgn_bin_sort_capped(N, M, _p(total), _p(ovf), C.byref(cs), rec, radii, bbox, mask, *S, _p(scratch), sb, None),
            ERR_INVALID, "leave no 16-bit key for the padding")
    _expect(L.sgn_bin_sort_capped(N, 0, _p(total), _p(ovf), C.byref(cs), rec, radii, bbox, mask, *S, _p(scratch), sb, None),
            ERR_INVALID, "a positive capacity")
    _expect(L.sgn_bin_sort_capped(N, M, None, _p(ovf), C.byref(cs), rec, radii, bbox, mask, *S, _p(scratch), sb, None),
            ERR_INVALID, "needs the device-side entry count")
    _expect(L.sgn_bin_sort_capped(N, M, _p(total), None, C.byref(cs), rec, radii, bbox, mask, *S, _p(scratch), sb, None),
            ERR_INVALID, "overflow flag is null")
    # class lists
    csb = L.sgn_bin_class_scratch_bytes(case.tiles)
    cscr, cls_ids, cls_bins = _z(csb, torch.uint8), _z((2, M)), _z((2, case.tiles, 2))
    _expect(L.sgn_bin_class_lists(C.byref(cs), M, _p(ids), _p(bins), _p(cls_ids), _p(cls_bins), _p(cscr), csb - 1, None), ERR_WORKSPACE,
            "sgn_bin_class_lists: scratch too small")
    _expect(L.sgn_bin_class_lists(C.byref(cs), 1 << 31, _p(ids), _p(bins), _p(cls_ids), _p(cls_bins), _p(cscr), csb, None), ERR_INVALID,
            "out of the int32 range")
    _expect(L.sgn_bin_class_lists(C.byref(cs), M, _p(ids), _p(bins), None, _p(cls_bins), _p(cscr), csb, None), ERR_INVALID,
            "sgn_bin_class_lists: null pointer")
    # local variant
    counts, info = _z((2, case.tiles)), _z(2, torch.int64)
    lsb = L.sgn_bin_local_scratch_bytes(0, case.tiles)
    lscr = _z(lsb, torch.uint8)
    cnt = (_p(counts[0]), _p(counts[1]))
    _expect(L.sgn_bin_local_count(N, C.byref(cs), rec, radii, bbox, mask, *cnt, _p(info), _p(lscr), lsb - 1, None), ERR_WORKSPACE,
            "sgn_bin_local_count: scratch too small")
    _expect(L.sgn_bin_local_count(N, C.byref(cs), rec, radii, bbox, None, *cnt, _p(info), _p(lscr), lsb, None), ERR_INVALID,
            "sgn_bin_local_count: null pointer")
    lsb2 = L.sgn_bin_local_scratch_bytes(M, case.tiles)
    lscr2 = _z(lsb2, torch.uint8)
    cap = L.sgn_bin_local_cap()
    assert cap == 8192

    def local_sort(m, longest, sbytes, cls=(cls_ids, cls_bins), records=rec):
        return L.sgn_bin_local_sort(N, m, longest, C.byref(cs), records, radii, bbox, mask, *cnt, _p(ids), _p(bins), _p(cls[0]),
                                    _p(cls[1]), _p(lscr2), sbytes, None)
    _expect(local_sort(M, cap + 1, lsb2), ERR_INVALID, "more than the 8192 a CTA sorts in shared memory")
    _expect(local_sort(-1, 1, lsb2), ERR_INVALID, "sgn_bin_local_sort: M=-1 out of range")
    _expect(local_sort(M, 1, lsb2 - 1), ERR_WORKSPACE, "sgn_bin_local_sort: scratch too small")
    _expect(local_sort(M, 1, lsb2, records=None), ERR_INVALID, "sgn_bin_local_sort: null pointer")
    _expect(local_sort(M, 1, lsb2, cls=(cls_ids, None)), ERR_INVALID, "cls_ids and cls_bins go together")
    torch.cuda.synchronize()
