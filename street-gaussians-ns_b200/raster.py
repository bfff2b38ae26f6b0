"""Host side of the fused rasterizer: stages the segment table, calls the C-ABI kernels of
libsgn_raster.so on the current torch CUDA stream, and wires them into autograd.

``render_frame`` is what ``SplatfactoSceneGraphModel.get_outputs`` reduces to
(street_gaussians_ns/sgn_splatfacto_scene_graph.py:305-374 + street_gaussians_ns/sgn_splatfacto.py:793-1001):
one compose+project launch, one binning pass, ONE blend traversal for rgb / accumulation / depth /
object_acc / background_acc (the reference runs four sorts + four traversals).

PyTorch is plumbing here (allocation, streams, autograd bookkeeping); all arithmetic is in the
CUDA library.  There is no CPU fallback.
"""
from __future__ import annotations

import copy
import ctypes as C
import os
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from . import scene as scene_mod
from .scene import PARAM_NAMES, Camera, Frame


@dataclass
class RenderSettings:
    sh_degree: int = 3
    sh_degree_to_use: Optional[int] = None  # None -> sh_degree
    block_width: int = 16
    clip_thresh: float = 0.01
    alpha_clamp_fwd: float = 0.999  # gsplat rasterize_forward
    alpha_clamp_bwd: float = 0.99   # gsplat rasterize_backward (SURVEY.md Appendix A.6)
    class_streams: bool = True      # object_acc / background_acc (scene graph :364-366)
    training: bool = True           # eval adds rgb.clamp(0,1) (sgn_splatfacto.py:974-975)
    # bit-reproducible gradients: the backward accumulates per-Gaussian gradients in 64-bit fixed point instead of with
    # float atomics (whose summation order varies from run to run).  None -> the SGN_DETERMINISTIC environment variable
    deterministic: Optional[bool] = None
    # no host read-back of the intersection count inside a frame (gsplat's ``cum_tiles_hit[-1].item()``): buffers and launches
    # are bounded by a capacity learnt from earlier frames, the count stays on the device, the host runs ahead of the GPU.
    # A frame whose count exceeds the capacity renders truncated lists; it is detected with the NEXT frame (warning,
    # ``raster.ASYNC_STATS``), the capacity grows.  None -> the SGN_ASYNC_BIN environment variable.  Off: exact, one sync.
    async_binning: Optional[bool] = None
    # "classic" or "antialiased" (the reference's rasterize_mode, sgn_splatfacto.py:214-223): antialiased scales every
    # visible Gaussian's opacity by comp = sqrt(det(cov2d) / det(cov2d + 0.3 I)), so that the 0.3 px^2 blur of the EWA
    # projection does not inflate sub-pixel Gaussians -- gsplat's antialiased mode.  Every stream that blends the records
    # (rgb, accumulation, depth, the class streams, the extra channels, the sky composite) follows, forward and backward
    rasterize_mode: str = "classic"
    # gsplat's absgrad (AbsGS): the backward also accumulates the absolute screen-space gradient, sum over pixels of
    # |d out_p / d xy| per row (sgn_blend_bwd_absgrad), into ``holder.v_absxy`` [N,2], from the main stream's outputs
    # (rgb, accumulation, depth) only.  A background_acc cotangent is then refused.  Off: holder.v_absxy is None
    absgrad: bool = False


class StageTimer:
    """Optional CUDA-event timing of each C-ABI stage on the launching stream (bench.py / tools)."""

    def __init__(self):
        self.events: Dict[str, list] = {}

    def record(self, name: str):
        ev = torch.cuda.Event(enable_timing=True)
        ev.record(torch.cuda.current_stream())
        self.events.setdefault(name, []).append(ev)

    def mean_ms(self) -> Dict[str, float]:
        out = {}
        for name in {k[:-6] for k in self.events if k.endswith(":start")}:
            st, en = self.events[name + ":start"], self.events[name + ":end"]
            out[name] = sum(a.elapsed_time(b) for a, b in zip(st, en)) / max(len(st), 1)
        return out


TIMER: Optional[StageTimer] = None


class _timed:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if TIMER is not None:
            TIMER.record(self.name + ":start")

    def __exit__(self, *a):
        if TIMER is not None:
            TIMER.record(self.name + ":end")
        return False


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def camera_struct(cam: Camera, s: RenderSettings) -> _lib.CameraStruct:
    cs = _lib.CameraStruct()
    vm = cam.viewmat().reshape(-1)
    for i in range(12):
        cs.viewmat[i] = float(vm[i])
    cs.fx, cs.fy, cs.cx, cs.cy = cam.fx, cam.fy, cam.cx, cam.cy
    cs.width, cs.height = cam.width, cam.height
    cp = cam.cam_pos()
    for i in range(3):
        cs.cam_pos[i] = float(cp[i])
    cs.limx, cs.limy = cam.fov_limits()
    cs.clip_thresh = s.clip_thresh
    cs.block_width = s.block_width
    cs.sh_degree = s.sh_degree
    cs.sh_degree_to_use = s.sh_degree if s.sh_degree_to_use is None else s.sh_degree_to_use
    cs.antialiased = rasterize_mode_flag(s.rasterize_mode)
    return cs


RASTERIZE_MODES = ("classic", "antialiased")


def rasterize_mode_flag(mode: str) -> int:
    '''sgn_camera.antialiased for a rasterize_mode name; any other name raises ValueError.'''
    if mode not in RASTERIZE_MODES:
        raise ValueError(f"Unknown rasterize_mode: {mode}")
    return int(mode == "antialiased")


def _check_param(t: torch.Tensor, name: str, device) -> None:
    if not (t.is_cuda and t.device == device):
        raise _lib.SgnError(f"{name} must live on {device} (got {t.device}); the rasterizer has no CPU path")
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise _lib.SgnError(f"{name} must be contiguous float32")
    if t.data_ptr() % 16 != 0:
        raise _lib.SgnError(f"{name} must be 16-byte aligned")


CHUNK_ROWS = 128  # rows per thread block of the per-Gaussian kernels (project.cu)

SEG_DTYPE = np.dtype([
    ("row0", "<i4"), ("count", "<i4"), ("F", "<i4"), ("cls", "<i4"), ("has_pose", "<i4"), ("chunk0", "<i4"),
    ("R", "<f4", (9,)), ("t", "<f4", (3,)), ("q", "<f4", (4,)), ("idft", "<f4", (8,)),
    ("means", "<u8"), ("scales", "<u8"), ("quats", "<u8"), ("features_dc", "<u8"), ("features_rest", "<u8"),
    ("opacities", "<u8")])
assert SEG_DTYPE.itemsize == C.sizeof(_lib.Segment), "numpy mirror of sgn_segment is out of sync"

_STATIC_CACHE: Dict[tuple, dict] = {}


class SegmentTable:
    """Host array of sgn_segment (numpy mirror of the C struct) + its device copy.

    The per-model part (pointers, row offsets, shapes; validated once) is cached on the parameter
    storage addresses; per frame only the poses and the IDFT bases are rewritten."""

    def __init__(self, frame: Frame, params: List[List[torch.Tensor]], device, upload: bool = True):
        pre = getattr(frame, "_prebuilt", None)
        if pre is not None and pre.dev is not None and pre.dev.device == device:
            # a row block of the device-resident (frame, actor) table (model.prepare_frames): nothing to build, nothing to copy
            self.host, self.N, self.num_chunks, self.nseg, self.static, self.dev = pre.host, pre.N, pre.num_chunks, pre.nseg, pre.static, pre.dev
            self.filter_dev = filter_table(frame, self.static, device)
            return
        n = len(frame.segments)
        # the per-model part is cached on the parameter storage addresses -- or on a key the model vouches for
        # (model._frame: (model id, parameter epoch, visible sub-models): spares ~200 data_ptr() calls per frame)
        key = getattr(frame, "_static_key", None)
        st = _STATIC_CACHE.get(key) if key is not None else None
        if st is None:
            ptrs = tuple(t.data_ptr() for ps in params for t in ps)
            if key is None:
                key = (ptrs, tuple(ps[0].shape[0] for ps in params), tuple(ps[3].shape[1] for ps in params),
                       tuple(ps[4].shape[1] for ps in params), str(device))
                st = _STATIC_CACHE.get(key)
        if st is None:
            for i, ps in enumerate(params):
                for t, nm in zip(ps, PARAM_NAMES):
                    _check_param(t, f"segment {i} {nm}", device)
            host = np.zeros(n, SEG_DTYPE)
            counts = np.array([ps[0].shape[0] for ps in params], np.int64)
            host["count"] = counts
            host["row0"] = np.concatenate([[0], np.cumsum(counts)[:-1]])
            chunks = (counts + CHUNK_ROWS - 1) // CHUNK_ROWS
            host["chunk0"] = np.concatenate([[0], np.cumsum(chunks)[:-1]])
            host["F"] = [ps[3].shape[1] for ps in params]
            P = np.array(ptrs, np.uint64).reshape(n, 6)
            for c, nm in enumerate(PARAM_NAMES):
                host[nm] = P[:, c]
            sizes = [[(t.numel() + 3) // 4 * 4 for t in ps] for ps in params]
            st = dict(host=host, N=int(counts.sum()), num_chunks=int(chunks.sum()), sizes=sizes, shapes=[[tuple(t.shape) for t in ps] for ps in params])
            if len(_STATIC_CACHE) > 64:
                _STATIC_CACHE.clear()
            _STATIC_CACHE[key] = st
        dyn = getattr(frame, "_dyn_table", None)
        if dyn is None or dyn[0] is not st:
            host = st["host"].copy()
            segs = frame.segments
            host["cls"] = [s.cls for s in segs]
            posed = [i for i, s in enumerate(segs) if s.has_pose]
            host["has_pose"] = 0
            host["R"] = np.eye(3, dtype=np.float32).reshape(-1)
            host["q"] = (1.0, 0.0, 0.0, 0.0)
            if posed:
                # object2world_gs (scene graph :404-417): float64 box pose -> float32; the quaternion of every box of the
                # frame from ONE batched eigen-decomposition (nerfstudio quaternion_from_matrix, restated in scene.py)
                R64 = np.stack([np.asarray(segs[i].rot, np.float64) for i in posed])
                host["has_pose"][posed] = 1
                host["R"][posed] = R64.reshape(-1, 9).astype(np.float32)
                host["t"][posed] = np.stack([np.asarray(segs[i].center, np.float64) for i in posed]).astype(np.float32)
                host["q"][posed] = scene_mod.quaternions_from_matrices(R64).astype(np.float32)
            padded = {}  # the actors of a frame share a handful of basis arrays (scene.idft_basis caches per (time, dim))
            for i, seg in enumerate(segs):
                k = (id(seg.idft), seg.params.features_dc.shape[1])
                b = padded.get(k)
                if b is None:
                    b = padded[k] = seg.idft_f32()
                host["idft"][i] = b
            try:
                frame._dyn_table = (st, host)  # poses of a Frame object do not change: reuse on re-render
            except Exception:
                pass
        else:
            host = dyn[1]
        self.host = host
        self.N = st["N"]
        self.num_chunks = st["num_chunks"]
        self.nseg = n
        self.static = st
        self.dev = torch.from_numpy(host.view(np.uint8).reshape(-1)).to(device, non_blocking=True) if upload else None
        self.filter_dev = filter_table(frame, st, device)
        slot = getattr(frame, "_table_slot", None)
        if slot is not None and upload:  # the model keeps a timestamp's rows (validated by content, model._frame)
            slot["table"] = self


def filter_table(frame: Frame, static: dict, device) -> Optional[torch.Tensor]:
    """The device array of per-segment 3D filter pointers (sgn_camera.filter_3d) of ``frame``'s segments, or None when no
    segment carries a filter.  Cached with the segment rows' static part, on the filter tensors' addresses."""
    fl = [s.filter_3d for s in frame.segments]
    if all(f is None for f in fl):
        return None
    if any(f is None for f in fl):
        raise _lib.SgnError("only some segments of the frame carry a 3D filter: give every segment one, or none")
    key = tuple(f.data_ptr() for f in fl)
    cache = static.setdefault("filter_tables", {})
    hit = cache.get(key)
    if hit is None:
        for i, (f, seg) in enumerate(zip(fl, frame.segments)):
            n = seg.params.num_points
            if not (f.is_cuda and f.device == device and f.dtype == torch.float32 and f.is_contiguous() and tuple(f.shape) == (n,)):
                raise _lib.SgnError(f"segment {i} filter_3d must be a contiguous float32 [{n}] tensor on {device}; got {f.dtype} "
                                    f"{tuple(f.shape)} on {f.device}")
        if len(cache) > 16:
            cache.clear()
        hit = cache[key] = torch.from_numpy(np.array(key, np.uint64).view(np.uint8)).to(device, non_blocking=True)
    return hit


def with_filter(cs: _lib.CameraStruct, table: "SegmentTable") -> _lib.CameraStruct:
    """``cs`` for a projection call over ``table``: a copy that points at the table's 3D filter array, or ``cs`` itself when
    the table has none (the field stays as the caller set it, NULL by default)."""
    fd = getattr(table, "filter_dev", None)
    if fd is None:
        return cs
    out = _lib.CameraStruct.from_buffer_copy(cs)
    out.filter_3d = fd.data_ptr()
    return out


def _grads_table(arena: torch.Tensor, static: dict, device) -> torch.Tensor:
    """sgn_segment_grads rows: pointers into the flat gradient arena (offsets are static per model)."""
    off = static.get("grad_offsets")
    if off is None:
        flat = np.array([x for ss in static["sizes"] for x in ss], np.uint64)
        off = static["grad_offsets"] = (np.concatenate([[0], np.cumsum(flat)[:-1]]) * 4).astype(np.uint64)
    tab = (np.uint64(arena.data_ptr()) + off).view(np.uint8)
    return torch.from_numpy(tab).to(device, non_blocking=True)


SEG_FLOATS = SEG_DTYPE.itemsize // 4
POSE_OFFSET = SEG_DTYPE.fields["R"][1] // 4  # R[9], t[3], q[4] are contiguous floats of a row
assert SEG_DTYPE.fields["t"][1] == 4 * (POSE_OFFSET + 9) and SEG_DTYPE.fields["q"][1] == 4 * (POSE_OFFSET + 12)


def posed_rows(table: SegmentTable):
    """Indices of the table's segments that carry a pose, as a slice when they are adjacent (background first, then the
    actors: the usual frame) and as a list otherwise."""
    idx = np.nonzero(table.host["has_pose"])[0]
    if idx.size and idx[-1] - idx[0] + 1 == idx.size:
        return slice(int(idx[0]), int(idx[-1]) + 1), int(idx.size)
    return [int(i) for i in idx], int(idx.size)


def with_poses(table: SegmentTable, pose: torch.Tensor) -> SegmentTable:
    """A copy of ``table`` whose device rows carry ``pose`` [n_posed, 16] (R 9 row-major, t 3, q 4; float32, in the order of
    the posed segments) instead of the poses it was built with.  The rows ``table`` holds -- which may be a timestamp's
    resident rows (model.prepare_frames) -- are not written: one device copy of nseg x 168 bytes, one assignment."""
    rows, n = posed_rows(table)
    if not (pose.is_cuda and pose.device == table.dev.device and pose.dtype == torch.float32 and tuple(pose.shape) == (n, _lib.POSE_FLOATS)):
        raise _lib.SgnError(f"pose must be a float32 [{n}, {_lib.POSE_FLOATS}] tensor on {table.dev.device} (one row per posed segment); "
                            f"got {pose.dtype} {tuple(pose.shape)} on {pose.device}")
    out = copy.copy(table)
    out.dev = table.dev.clone()
    out.dev.view(torch.float32).view(table.nseg, SEG_FLOATS)[rows, POSE_OFFSET:POSE_OFFSET + _lib.POSE_FLOATS] = pose.detach()
    return out


# --------------------------------------------------------------------------------------------------
# stage wrappers (also used directly by tests and bench.py)
# --------------------------------------------------------------------------------------------------
class Projected:
    """Outputs of the fused compose+project+SH kernel (also iterable as the legacy 4-tuple)."""

    def __init__(self, records, radii, tiles_hit, bbox, tiles_touched, touch_mask):
        self.records, self.radii, self.tiles_hit, self.bbox = records, radii, tiles_hit, bbox
        self.tiles_touched, self.touch_mask = tiles_touched, touch_mask

    def __iter__(self):
        return iter((self.records, self.radii, self.tiles_hit, self.bbox))


def check_view(view: torch.Tensor, device) -> torch.Tensor:
    """A device view (viewmat 12 row-major, cam_pos 3): float32 [15] on ``device``; returns it detached and contiguous."""
    if not (view.is_cuda and view.device == device and view.dtype == torch.float32 and tuple(view.shape) == (VIEW_LEN,)):
        raise _lib.SgnError(f"view must be a float32 [{VIEW_LEN}] tensor on {device} (viewmat 3x4 row-major, then cam_pos); "
                            f"got {view.dtype} {tuple(view.shape)} on {view.device}")
    return view.detach().contiguous()


VIEW_LEN = _lib.VIEW_FLOATS + 3


def project_fwd(table: SegmentTable, cs: _lib.CameraStruct, device, view: Optional[torch.Tensor] = None) -> Projected:
    """``view``: a device view (check_view) in place of the camera's (sgn_project_fwd_view)."""
    L = _lib.load()
    N = table.N
    cs = with_filter(cs, table)
    records = torch.empty(N, _lib.RECORD_FLOATS, device=device, dtype=torch.float32)
    ints = torch.empty(4, max(N, 1), device=device, dtype=torch.int32)  # radii, num_tiles_hit, tiles_touched, touch_mask
    bbox = torch.empty(N, 4, device=device, dtype=torch.int16)
    with _timed("project_fwd"):
        if view is not None:
            _lib.check(L.sgn_project_fwd_view(_ptr(table.dev), table.nseg, N, table.num_chunks, C.byref(cs), _ptr(view), _ptr(records),
                                              _ptr(ints[0]), _ptr(ints[1]), _ptr(bbox), _ptr(ints[2]), _ptr(ints[3]), _stream()),
                       "sgn_project_fwd_view")
        else:
            _lib.check(L.sgn_project_fwd(_ptr(table.dev), table.nseg, N, table.num_chunks, C.byref(cs), _ptr(records), _ptr(ints[0]),
                                         _ptr(ints[1]), _ptr(bbox), _ptr(ints[2]), _ptr(ints[3]), _stream()), "sgn_project_fwd")
    return Projected(records, ints[0][:N], ints[1][:N], bbox, ints[2][:N], ints[3][:N])


BIN_LOCAL = os.environ.get("SGN_BIN_LOCAL", "0") == "1"  # experimental: per-tile shared-memory sort (csrc/binning_local.cu)


def _bin_local(cs: _lib.CameraStruct, records, radii, proj: Projected):
    """The experimental binning variant: tile histogram + scatter + a sort inside every tile.  Same outputs as the
    device-wide path; returns None when a tile's list is too long for the shared-memory sort (the caller falls back)."""
    L = _lib.load()
    device = records.device
    N = records.shape[0]
    bw = cs.block_width
    tiles = ((cs.width + bw - 1) // bw) * ((cs.height + bw - 1) // bw)
    counts = torch.empty(2, tiles, device=device, dtype=torch.int32)  # per tile: entries, start
    info = torch.empty(2, device=device, dtype=torch.int64)           # M, longest list
    sb = L.sgn_bin_local_scratch_bytes(0, tiles)
    scratch = torch.empty(sb, device=device, dtype=torch.uint8)
    with _timed("bin_scan"):
        _lib.check(L.sgn_bin_local_count(N, C.byref(cs), _ptr(records), _ptr(radii), _ptr(proj.bbox), _ptr(proj.touch_mask),
                                         _ptr(counts[0]), _ptr(counts[1]), _ptr(info), _ptr(scratch), sb, _stream()), "sgn_bin_local_count")
    M, longest = (int(x) for x in info.tolist())
    if longest > L.sgn_bin_local_cap():
        return None
    tile_bins = torch.empty(tiles, 2, device=device, dtype=torch.int32)
    sorted_ids = torch.empty(max(M, 1), device=device, dtype=torch.int32)
    cls_ids = torch.empty(2, max(M, 1), device=device, dtype=torch.int32)   # the class sub-lists come out of the same pass
    cls_bins = torch.empty(2, tiles, 2, device=device, dtype=torch.int32)
    sb2 = L.sgn_bin_local_scratch_bytes(M, tiles)
    scratch2 = torch.empty(sb2, device=device, dtype=torch.uint8)
    with _timed("bin_sort"):
        _lib.check(L.sgn_bin_local_sort(N, M, longest, C.byref(cs), _ptr(records), _ptr(radii), _ptr(proj.bbox), _ptr(proj.touch_mask),
                                        _ptr(counts[0]), _ptr(counts[1]), _ptr(sorted_ids), _ptr(tile_bins), _ptr(cls_ids), _ptr(cls_bins),
                                        _ptr(scratch2), sb2, _stream()), "sgn_bin_local_sort")
    global _LOCAL_CLASSES
    _LOCAL_CLASSES = (sorted_ids, cls_ids, cls_bins)
    return M, sorted_ids, tile_bins


_LOCAL_CLASSES = None  # (sorted_ids, cls_ids, cls_bins) of the last _bin_local call: class_lists() hands them out instead of recomputing


ASYNC_BIN = os.environ.get("SGN_ASYNC_BIN", "0") == "1"
ASYNC_HEADROOM = float(os.environ.get("SGN_ASYNC_BIN_HEADROOM", "1.2"))
ASYNC_GRANULE = 65536  # capacities are multiples of this many entries
ASYNC_STATS = {"frames": 0, "overflows": 0, "sync_frames": 0}
_ASYNC_STATE: Dict[str, dict] = {}


class LazyCount:
    """The intersection count of a frame rendered without the read-back: an int once somebody asks (that waits for the copy)."""

    def __init__(self, event, pinned, capacity: int, device_count=None):
        self.event, self.pinned, self.capacity, self._value = event, pinned, capacity, None
        self.device_count = device_count  # the int64[1] tensor on the device (for device-side decisions, e.g. "nothing in view")

    def ready(self) -> bool:
        return self._value is not None or self.event.query()

    def raw(self) -> int:
        if self._value is None:
            self.event.synchronize()
            self._value = int(self.pinned[0])
        return self._value

    def __int__(self) -> int:
        return min(self.raw(), self.capacity)

    __index__ = __int__

    def __eq__(self, other):
        return int(self) == other

    def __lt__(self, other):
        return int(self) < other

    def __le__(self, other):
        return int(self) <= other

    def __gt__(self, other):
        return int(self) > other

    def __ge__(self, other):
        return int(self) >= other

    def __hash__(self):
        return hash(int(self))

    def __repr__(self):
        return f"LazyCount({int(self)})"


def _async_state(device) -> dict:
    st = _ASYNC_STATE.get(str(device))
    if st is None:
        st = _ASYNC_STATE[str(device)] = {"max_m": 0, "pending": [], "overflow": torch.zeros(1, dtype=torch.int32, device=device),
                                          "pinned": [torch.zeros(1, dtype=torch.int64).pin_memory() for _ in range(64)], "slot": 0}
    return st


def async_learn(device, count: int) -> None:
    """Tell the capacity logic about an intersection count observed elsewhere (e.g. a look at the widest cameras in exact mode
    before a training run switches the read-back off)."""
    st = _async_state(device)
    st["max_m"] = max(st["max_m"], int(count))


def _async_poll(st: dict) -> None:
    """Counts of earlier frames that have arrived: the capacity follows the largest one; an overflow is reported."""
    keep = []
    for lc in st["pending"]:
        if lc.ready():
            m = lc.raw()
            st["max_m"] = max(st["max_m"], m)
            if m > lc.capacity:
                ASYNC_STATS["overflows"] += 1
                import warnings
                warnings.warn(f"async binning: a frame had {m} intersections, capacity {lc.capacity}: its lists were truncated "
                              "(the capacity has been raised; SGN_ASYNC_BIN=0 renders exactly)")
        else:
            keep.append(lc)
    st["pending"] = keep[-32:]


def bin_and_sort(cs: _lib.CameraStruct, records, radii, tiles_hit=None, bbox=None, proj: Optional[Projected] = None,
                 async_binning: Optional[bool] = None):
    """Returns (M, sorted_ids[M], tile_bins[tiles,2]).  One host sync to read M (as gsplat does) -- or, with
    ``async_binning``, none: M is then a LazyCount and sorted_ids has the capacity's length.
    Pass ``proj`` (from project_fwd) or plain records/radii/bbox (the touched-tile count is then computed here)."""
    L = _lib.load()
    device = records.device
    N = records.shape[0]
    use_async = ASYNC_BIN if async_binning is None else async_binning
    if BIN_LOCAL and proj is not None:
        res = _bin_local(cs, records, radii, proj)
        if res is not None:
            return res
    if proj is not None:
        bbox, touched, mask = proj.bbox, proj.tiles_touched, proj.touch_mask
    else:
        touched = torch.empty(max(N, 1), device=device, dtype=torch.int32)
        mask = torch.empty(max(N, 1), device=device, dtype=torch.int32)
        with _timed("bin_count"):
            _lib.check(L.sgn_bin_count(N, C.byref(cs), _ptr(records), _ptr(radii), _ptr(bbox), _ptr(touched), _ptr(mask),
                                       _stream()), "sgn_bin_count")
    oc = torch.empty(2, max(N, 1), device=device, dtype=torch.int32)  # order, cum
    total = torch.empty(1, device=device, dtype=torch.int64)
    sb = L.sgn_bin_scan_scratch_bytes(N)
    scratch = torch.empty(sb, device=device, dtype=torch.uint8)
    with _timed("bin_scan"):
        _lib.check(L.sgn_bin_scan(N, _ptr(records), _ptr(radii), _ptr(touched), _ptr(oc[0]), _ptr(oc[1]), _ptr(total),
                                  _ptr(scratch), sb, _stream()), "sgn_bin_scan")
    bw = cs.block_width
    tiles = ((cs.width + bw - 1) // bw) * ((cs.height + bw - 1) // bw)
    tile_bins = torch.empty(tiles, 2, device=device, dtype=torch.int32)
    # the capped form keys its padding as one more tile: a camera of 65536 tiles leaves it no 16-bit key, so such a frame
    # reads the count back like the synchronous form
    if use_async and N > 0 and tiles < 65536:
        st = _async_state(device)
        _async_poll(st)
        if st["max_m"] > 0:  # a capacity is known: no read-back in this frame
            cap = int((int(st["max_m"] * ASYNC_HEADROOM) + ASYNC_GRANULE - 1) // ASYNC_GRANULE * ASYNC_GRANULE)
            pin = st["pinned"][st["slot"] % len(st["pinned"])]
            st["slot"] += 1
            pin.copy_(total, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            lazy = LazyCount(ev, pin, cap, total)
            st["pending"].append(lazy)
            ASYNC_STATS["frames"] += 1
            sorted_ids = torch.empty(cap, device=device, dtype=torch.int32)
            sb2 = L.sgn_bin_sort_scratch_bytes(cap)
            scratch2 = torch.empty(sb2, device=device, dtype=torch.uint8)
            with _timed("bin_sort"):
                _lib.check(L.sgn_bin_sort_capped(N, cap, _ptr(total), _ptr(st["overflow"]), C.byref(cs), _ptr(records), _ptr(radii),
                                                 _ptr(bbox), _ptr(mask), _ptr(oc[0]), _ptr(oc[1]), _ptr(sorted_ids), _ptr(tile_bins),
                                                 _ptr(scratch2), sb2, _stream()), "sgn_bin_sort_capped")
            return lazy, sorted_ids, tile_bins
        ASYNC_STATS["sync_frames"] += 1  # first frame on this device: learn the count the exact way
    M = int(total.item())
    if use_async and N > 0:
        _async_state(device)["max_m"] = max(_async_state(device)["max_m"], M)
    sorted_ids = torch.empty(max(M, 1), device=device, dtype=torch.int32)
    sb2 = L.sgn_bin_sort_scratch_bytes(M)
    scratch2 = torch.empty(sb2, device=device, dtype=torch.uint8)
    with _timed("bin_sort"):
        _lib.check(L.sgn_bin_sort(N, M, C.byref(cs), _ptr(records), _ptr(radii), _ptr(bbox), _ptr(mask), _ptr(oc[0]), _ptr(oc[1]),
                                  _ptr(sorted_ids), _ptr(tile_bins), _ptr(scratch2), sb2, _stream()), "sgn_bin_sort")
    return M, sorted_ids, tile_bins


ID_MASK = 0x7FFFFFFF  # sorted payload: bits 0-30 Gaussian row, bit 31 object class


def class_lists(cs: _lib.CameraStruct, M: int, sorted_ids, tile_bins):
    """Per-tile class sub-lists (stable partition of the sorted list into background / object entries).
    Returns (cls_ids[2,M], cls_bins[2,tiles,2])."""
    global _LOCAL_CLASSES
    if _LOCAL_CLASSES is not None and _LOCAL_CLASSES[0] is sorted_ids:  # built together with the lists (experimental local binning)
        _, cls_ids, cls_bins = _LOCAL_CLASSES
        _LOCAL_CLASSES = None
        return cls_ids, cls_bins
    L = _lib.load()
    device = sorted_ids.device
    tiles = tile_bins.shape[0]
    M = sorted_ids.shape[0]  # the sub-lists' stride: the list buffer's length (== max(M, 1), or the capacity without the read-back)
    obj_ids = torch.empty(2, max(M, 1), device=device, dtype=torch.int32)
    obj_bins = torch.empty(2, tiles, 2, device=device, dtype=torch.int32)
    sb = L.sgn_bin_class_scratch_bytes(tiles)
    scratch = torch.empty(sb, device=device, dtype=torch.uint8)
    with _timed("class_lists"):
        _lib.check(L.sgn_bin_class_lists(C.byref(cs), max(M, 1), _ptr(sorted_ids), _ptr(tile_bins), _ptr(obj_ids), _ptr(obj_bins),
                                         _ptr(scratch), sb, _stream()), "sgn_bin_class_lists")
    return obj_ids, obj_bins


HEAVY_FIRST = os.environ.get("SGN_HEAVY_FIRST", "1") != "0"
# paired row-slot bodies in the main forward, scalar ones in the backward (with the objects-only gradient folded in, the
# scalar backward body is the faster one on an H100; DESIGN.md §5), no row skipping in the main kernels
DEFAULT_TUNING = 4


def blend_opts(s: RenderSettings, has_sky: bool) -> _lib.BlendOpts:
    bo = _lib.BlendOpts()
    bo.alpha_clamp_fwd, bo.alpha_clamp_bwd = s.alpha_clamp_fwd, s.alpha_clamp_bwd
    bo.class_streams, bo.has_sky, bo.eval_clamp = int(s.class_streams), int(has_sky), int(not s.training)
    bo.split_fwd_main = int(os.environ.get("SGN_SPLIT_FWD_MAIN", "0"))
    bo.split_fwd_acc = int(os.environ.get("SGN_SPLIT_FWD_ACC", "0"))
    bo.split_bwd_main = int(os.environ.get("SGN_SPLIT_BWD_MAIN", "0"))
    bo.split_bwd_acc = int(os.environ.get("SGN_SPLIT_BWD_ACC", "0"))
    # SGN_TUNE_* bits (include/sgn_raster.h): 1 fwd row skip, 4 fwd paired row slots, 8 bwd paired row slots, 16 no row skip in the
    # accumulation-only kernels, 32 fwd TMA staging
    bo.tuning = int(os.environ.get("SGN_TUNING", str(DEFAULT_TUNING)))
    return bo


def blend_fwd(cs, bo, records, sorted_ids, tile_bins, sky: Optional[torch.Tensor], obj_ids=None, obj_bins=None):
    L = _lib.load()
    device = records.device
    H, W = cs.height, cs.width
    S = 3 if bo.class_streams else 1
    out = dict(
        rgb=torch.empty(H, W, 3, device=device), accumulation=torch.empty(H, W, 1, device=device),
        depth=torch.empty(H, W, 1, device=device), raw=torch.empty(H, W, 4, device=device),
        final_T=torch.empty(S, H, W, device=device), final_idx=torch.empty(S, H, W, device=device, dtype=torch.int32),
        tile_depth=torch.empty(3, tile_bins.shape[0], device=device, dtype=torch.int32))
    if bo.class_streams:
        out["object_acc"] = torch.empty(H, W, 1, device=device)
        out["background_acc"] = torch.empty(H, W, 1, device=device)
    fo = _lib.BlendFwdOut()
    fo.rgb, fo.accumulation, fo.depth = out["rgb"].data_ptr(), out["accumulation"].data_ptr(), out["depth"].data_ptr()
    fo.object_acc = out["object_acc"].data_ptr() if bo.class_streams else None
    fo.background_acc = out["background_acc"].data_ptr() if bo.class_streams else None
    fo.raw, fo.final_T, fo.final_idx = out["raw"].data_ptr(), out["final_T"].data_ptr(), out["final_idx"].data_ptr()
    fo.tile_depth = out["tile_depth"].data_ptr()
    fo.staged = None
    if bo.tuning & 32:  # SGN_TUNE_FWD_TMA (experiment): scratch for the materialised staged entries, 48 B per list entry
        out["staged"] = torch.empty(max(sorted_ids.shape[0], 1) * _lib.RECORD_FLOATS, device=device, dtype=torch.float32)
        fo.staged = out["staged"].data_ptr()
    if HEAVY_FIRST:  # scratch for the heavy-first work lists (scheduling only), reused by the backward
        out["sched"] = torch.empty(L.sgn_blend_sched_ints(tile_bins.shape[0]), device=device, dtype=torch.int32)
        fo.sched = out["sched"].data_ptr()
    with _timed("blend_fwd"):
        _lib.check(L.sgn_blend_fwd(C.byref(cs), C.byref(bo), _ptr(records), _ptr(sorted_ids), _ptr(tile_bins),
                                   max(sorted_ids.shape[0], 1), _ptr(obj_ids), _ptr(obj_bins), _ptr(sky), C.byref(fo), _stream()),
                   "sgn_blend_fwd")
    return out


DETERMINISTIC = os.environ.get("SGN_DETERMINISTIC", "0") == "1"


def blend_bwd(cs, bo, records, sorted_ids, tile_bins, saved: Dict[str, torch.Tensor], sky, v: Dict[str, Optional[torch.Tensor]],
              want_v_sky: bool, obj_ids=None, obj_bins=None, deterministic: Optional[bool] = None, absgrad: bool = False):
    """Returns (v_records[N,12], v_sky or None); with ``absgrad``, (v_records, v_sky, v_absxy[N,2]) from
    sgn_blend_bwd_absgrad (the same v_records and v_sky, plus the main stream's absolute screen-space gradient)."""
    L = _lib.load()
    device = records.device
    bi = _lib.BlendBwdIn()
    det = DETERMINISTIC if deterministic is None else deterministic
    N = records.shape[0]
    fixed_absxy = None
    if det:  # fixed-point accumulators (zeroed) + one float of scratch; v_records is then written, not accumulated into
        v_records = torch.empty_like(records)
        v_fixed = torch.zeros(N, _lib.RECORD_FLOATS, device=device, dtype=torch.int64)
        fixed_scale = torch.empty(1, device=device, dtype=torch.float32)
        bi.v_fixed, bi.fixed_scale, bi.num_gaussians = v_fixed.data_ptr(), fixed_scale.data_ptr(), N
        if absgrad:
            v_absxy = torch.empty(N, 2, device=device, dtype=torch.float32)
            fixed_absxy = torch.zeros(N, 2, device=device, dtype=torch.int64)
    else:
        v_records = torch.zeros_like(records)
        bi.v_fixed = bi.fixed_scale = None
        bi.num_gaussians = N
        if absgrad:
            v_absxy = torch.zeros(N, 2, device=device, dtype=torch.float32)

    def c(t):
        return None if t is None else t.contiguous()

    keep = {k: c(t) for k, t in v.items()}
    bi.v_rgb = keep["rgb"].data_ptr() if keep.get("rgb") is not None else None
    bi.v_accumulation = keep["accumulation"].data_ptr() if keep.get("accumulation") is not None else None
    bi.v_depth = keep["depth"].data_ptr() if keep.get("depth") is not None else None
    bi.v_object_acc = keep["object_acc"].data_ptr() if keep.get("object_acc") is not None else None
    bi.v_background_acc = keep["background_acc"].data_ptr() if keep.get("background_acc") is not None else None
    bi.raw, bi.final_T, bi.final_idx = saved["raw"].data_ptr(), saved["final_T"].data_ptr(), saved["final_idx"].data_ptr()
    bi.tile_depth = saved["tile_depth"].data_ptr()
    bi.sched = saved["sched"].data_ptr() if "sched" in saved else None
    bi.sky = sky.data_ptr() if sky is not None else None
    v_sky = torch.zeros(cs.height, cs.width, 3, device=device) if (want_v_sky and sky is not None) else None
    bi.v_sky = v_sky.data_ptr() if v_sky is not None else None
    if absgrad:
        with _timed("blend_bwd"):
            _lib.check(L.sgn_blend_bwd_absgrad(C.byref(cs), C.byref(bo), _ptr(records), _ptr(sorted_ids), _ptr(tile_bins),
                                               max(sorted_ids.shape[0], 1), _ptr(obj_ids), _ptr(obj_bins), C.byref(bi), _ptr(v_records),
                                               _ptr(v_absxy), _ptr(fixed_absxy), _stream()), "sgn_blend_bwd_absgrad")
        return v_records, v_sky, v_absxy
    with _timed("blend_bwd"):
        _lib.check(L.sgn_blend_bwd(C.byref(cs), C.byref(bo), _ptr(records), _ptr(sorted_ids), _ptr(tile_bins),
                                   max(sorted_ids.shape[0], 1), _ptr(obj_ids), _ptr(obj_bins), C.byref(bi), _ptr(v_records), _stream()),
                   "sgn_blend_bwd")
    return v_records, v_sky


def arena_layout(static: dict):
    """(padded sizes, shapes, numels) of the flat gradient arena, in segment-major parameter order."""
    if static.get("flat_sizes") is None:
        static["flat_sizes"] = [x for ss in static["sizes"] for x in ss]
        static["flat_shapes"] = [x for ss in static["shapes"] for x in ss]
        static["flat_numel"] = [int(np.prod(x)) for x in static["flat_shapes"]]
    return static["flat_sizes"], static["flat_shapes"], static["flat_numel"]


def arena_views(arena: torch.Tensor, static: dict) -> List[torch.Tensor]:
    sizes, shapes, numels = arena_layout(static)
    chunks = arena.split_with_sizes(sizes)
    return [c[:n].view(shp) if n != c.shape[0] else c.view(shp) for c, n, shp in zip(chunks, numels, shapes)]


def _arena_grads_table(arena: torch.Tensor, static: dict, device, out_offsets: Optional[np.ndarray] = None) -> torch.Tensor:
    """The sgn_segment_grads rows of a frame into ``arena``: back to back in the frame's layout, or at ``out_offsets``
    (floats, one per parameter tensor, multiples of 4) inside a larger arena."""
    flat_sizes, _, _ = arena_layout(static)
    if out_offsets is None:
        assert arena.numel() == sum(flat_sizes)
        return _grads_table(arena, static, device)
    assert len(out_offsets) == len(flat_sizes)
    off = np.asarray(out_offsets, np.int64)
    assert (off % 4 == 0).all() and int((off + np.asarray(flat_sizes, np.int64)).max()) <= arena.numel()
    return torch.from_numpy((np.uint64(arena.data_ptr()) + (off * 4).astype(np.uint64)).view(np.uint8)).to(device, non_blocking=True)


def scale_reg_fwd(table: SegmentTable, max_ratio: float) -> torch.Tensor:
    """The scale regularisation over the frame's rows, 0.1 * mean(max(amax(s) / amin(s), max_ratio) - max_ratio) with
    s = exp(scales): a 0-d float32 tensor on the device, no read-back (sgn_scale_reg_fwd)."""
    L = _lib.load()
    device = table.dev.device
    out = torch.empty((), device=device, dtype=torch.float32)
    sb = L.sgn_scale_reg_scratch_bytes()
    scratch = torch.empty(sb, device=device, dtype=torch.uint8)
    with _timed("scale_reg_fwd"):
        _lib.check(L.sgn_scale_reg_fwd(_ptr(table.dev), table.nseg, table.N, table.num_chunks, float(max_ratio), _ptr(out), _ptr(scratch),
                                       sb, _stream()), "sgn_scale_reg_fwd")
    return out


def scale_reg_bwd(table: SegmentTable, arena: torch.Tensor, max_ratio: float, v_out: torch.Tensor,
                  out_offsets: Optional[np.ndarray] = None) -> None:
    """ADDS the scale regularisation's gradient times ``v_out`` (a float32 device scalar) into the scales slices of the
    gradient arena (laid out as project_bwd's, ``out_offsets`` likewise); sgn_scale_reg_bwd."""
    L = _lib.load()
    v_out = v_out.detach().reshape(()).to(torch.float32).contiguous()
    gt = _arena_grads_table(arena, table.static, arena.device, out_offsets)
    with _timed("scale_reg_bwd"):
        _lib.check(L.sgn_scale_reg_bwd(_ptr(table.dev), _ptr(gt), table.nseg, table.N, table.num_chunks, float(max_ratio), _ptr(v_out),
                                       _stream()), "sgn_scale_reg_bwd")


def mcmc_reg_fwd(table: SegmentTable, w_opacity: float, w_scale: float) -> torch.Tensor:
    """MCMC's regularisers over the frame's rows, [w_opacity * mean(sigmoid(opacities)), w_scale * mean(exp(scales))]: a float32
    pair on the device, no read-back (sgn_mcmc_reg_fwd)."""
    L = _lib.load()
    device = table.dev.device
    out = torch.empty(2, device=device, dtype=torch.float32)
    sb = L.sgn_mcmc_reg_scratch_bytes()
    scratch = torch.empty(sb, device=device, dtype=torch.uint8)
    with _timed("mcmc_reg_fwd"):
        _lib.check(L.sgn_mcmc_reg_fwd(_ptr(table.dev), table.nseg, table.N, table.num_chunks, float(w_opacity), float(w_scale), _ptr(out),
                                      _ptr(scratch), sb, _stream()), "sgn_mcmc_reg_fwd")
    return out


def mcmc_reg_bwd(table: SegmentTable, arena: torch.Tensor, w_opacity: float, w_scale: float, v_opacity: Optional[torch.Tensor],
                 v_scale: Optional[torch.Tensor], out_offsets: Optional[np.ndarray] = None) -> None:
    """ADDS the gradients of the two MCMC regularisers times their cotangents (float32 device scalars, None = no cotangent) into
    the opacities and scales slices of the gradient arena (laid out as project_bwd's); sgn_mcmc_reg_bwd."""
    L = _lib.load()
    vo = None if v_opacity is None else v_opacity.detach().reshape(()).to(torch.float32).contiguous()
    vs = None if v_scale is None else v_scale.detach().reshape(()).to(torch.float32).contiguous()
    gt = _arena_grads_table(arena, table.static, arena.device, out_offsets)
    with _timed("mcmc_reg_bwd"):
        _lib.check(L.sgn_mcmc_reg_bwd(_ptr(table.dev), _ptr(gt), table.nseg, table.N, table.num_chunks, float(w_opacity), float(w_scale),
                                      _ptr(vo), _ptr(vs), _stream()), "sgn_mcmc_reg_bwd")


class ParamTerm:
    """A loss term of the Gaussian parameters alone, evaluated over the frame's rows through its segment table, as outputs of the
    render node (``render_frame(terms=...)``).  It is an output of the node rather than a function of its own because project_bwd
    OVERWRITES the gradient arena: as an output, the render's backward waits for the term's cotangents and adds its gradient into
    the arena after project_bwd, before the arena is handed on.  ``names``: the outputs, in order; ``kinds``: the PARAM_NAMES
    positions its gradient reaches."""

    names: Tuple[str, ...] = ()
    kinds: Tuple[int, ...] = ()

    def forward(self, table: SegmentTable) -> List[torch.Tensor]:
        raise NotImplementedError

    def backward(self, table: SegmentTable, arena: torch.Tensor, v: Sequence[Optional[torch.Tensor]],
                 out_offsets: Optional[np.ndarray] = None) -> None:
        raise NotImplementedError


class ScaleRegTerm(ParamTerm):
    """nerfstudio's scale regularisation (scale_reg_fwd / scale_reg_bwd)."""

    names, kinds = ("scale_reg",), (1,)

    def __init__(self, max_ratio: float):
        self.max_ratio = max_ratio

    def forward(self, table):
        return [scale_reg_fwd(table, self.max_ratio)]

    def backward(self, table, arena, v, out_offsets=None):
        scale_reg_bwd(table, arena, self.max_ratio, v[0], out_offsets)


class MCMCRegTerm(ParamTerm):
    """MCMC's opacity and scale regularisers (mcmc_reg_fwd / mcmc_reg_bwd), two scalar outputs."""

    names, kinds = ("mcmc_opacity_reg", "mcmc_scale_reg"), (1, 5)

    def __init__(self, w_opacity: float, w_scale: float):
        self.w_opacity, self.w_scale = w_opacity, w_scale

    def forward(self, table):
        out = mcmc_reg_fwd(table, self.w_opacity, self.w_scale)
        return [out[0], out[1]]

    def backward(self, table, arena, v, out_offsets=None):
        mcmc_reg_bwd(table, arena, self.w_opacity, self.w_scale, v[0], v[1], out_offsets)


_TERM_NAMES = ScaleRegTerm.names + MCMCRegTerm.names


def _terms_of(scale_reg: Optional[float], terms: Sequence[ParamTerm]) -> Tuple[ParamTerm, ...]:
    return tuple(terms) + ((ScaleRegTerm(scale_reg),) if scale_reg is not None else ())


def _split_term_cotangents(terms: Sequence[ParamTerm], v: Sequence[Optional[torch.Tensor]]) -> List[List[Optional[torch.Tensor]]]:
    out, i = [], 0
    for t in terms:
        out.append(list(v[i:i + len(t.names)]))
        i += len(t.names)
    return out


def _zero_arena(static: dict, device, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The gradient arena of a backward with no image-space cotangent: ``out`` zeroed (all of it, also the slices of sub-models
    outside the frame when ``out`` has the layout of the whole model), or a new zero arena in the frame's layout."""
    if out is None:
        flat_sizes, _, _ = arena_layout(static)
        return torch.zeros(sum(flat_sizes), device=device, dtype=torch.float32)
    return out.zero_()


def project_bwd(table: SegmentTable, params: List[List[torch.Tensor]], cs, records, radii, v_records, make_views: bool = True,
                out: Optional[torch.Tensor] = None, out_offsets: Optional[np.ndarray] = None, chunk_ranges=None, after_range=None,
                v_pose: Optional[torch.Tensor] = None, view: Optional[torch.Tensor] = None, v_view: Optional[torch.Tensor] = None):
    """Dense parameter gradients, one flat arena (a single allocation, 16-byte aligned slices; ``out`` reuses one).
    ``out_offsets`` (floats, one per parameter tensor of the frame, multiples of 4) places the slices inside a larger
    ``out`` -- the data-parallel arena that has the layout of ALL sub-models (model._FullArenaSink).
    ``v_pose`` [nseg, 16] float32: also filled with the cotangents of the segments' poses (R 9, t 3, q 4; zero rows for
    segments without one) -- sgn_project_bwd_pose for every range, then sgn_pose_grad_reduce.  The arena is the same bits.
    ``view``: the device view the forward projected with (check_view); ``v_view`` [12] float32 is then filled with its
    cotangent -- sgn_project_bwd_view for every range (with the pose sums too when ``v_pose`` is given), then
    sgn_view_grad_reduce.  The arena is the same bits as sgn_project_bwd_range's with that view."""
    assert (view is None) == (v_view is None), "view and v_view go together"
    L = _lib.load()
    cs = with_filter(cs, table)
    device = records.device
    st = table.static
    flat_sizes, _, _ = arena_layout(st)
    arena = out if out is not None else torch.empty(sum(flat_sizes), device=device, dtype=torch.float32)
    assert arena.dtype == torch.float32 and arena.is_contiguous()
    if out_offsets is not None:
        assert out is not None and not make_views
    gt = _arena_grads_table(arena, st, device, out_offsets)
    flat = arena_views(arena, st) if make_views else None
    if chunk_ranges is None:
        chunk_ranges = [(0, table.num_chunks)]
    partials = None
    if v_pose is not None:
        assert v_pose.shape == (table.nseg, _lib.POSE_FLOATS) and v_pose.dtype == torch.float32 and v_pose.is_contiguous() and v_pose.device == device
        partials = torch.empty(max(table.num_chunks, 1), _lib.POSE_FLOATS, device=device, dtype=torch.float32)
    view_partials = None
    if v_view is not None:
        assert v_view.shape == (_lib.VIEW_FLOATS,) and v_view.dtype == torch.float32 and v_view.is_contiguous() and v_view.device == device
        view_partials = torch.empty(max(table.num_chunks, 1), _lib.VIEW_FLOATS, device=device, dtype=torch.float32)
    with _timed("project_bwd"):
        # range by range (data parallel): ``after_range(k)`` is called once range k's launch is enqueued -- the exchange of
        # that range's slices starts there and overlaps the production of the next range (dp.SymmetricExchange)
        for k, (c0, c1) in enumerate(chunk_ranges):
            if view_partials is not None:
                _lib.check(L.sgn_project_bwd_view(_ptr(table.dev), _ptr(gt), table.nseg, table.N, table.num_chunks, C.byref(cs),
                                                  _ptr(view), _ptr(records), _ptr(radii), _ptr(v_records), int(c0), int(c1),
                                                  _ptr(partials), _ptr(view_partials), _stream()), "sgn_project_bwd_view")
            elif partials is not None:
                _lib.check(L.sgn_project_bwd_pose(_ptr(table.dev), _ptr(gt), table.nseg, table.N, table.num_chunks, C.byref(cs),
                                                  _ptr(records), _ptr(radii), _ptr(v_records), int(c0), int(c1), _ptr(partials),
                                                  _stream()), "sgn_project_bwd_pose")
            else:
                _lib.check(L.sgn_project_bwd_range(_ptr(table.dev), _ptr(gt), table.nseg, table.N, table.num_chunks, C.byref(cs),
                                                   _ptr(records), _ptr(radii), _ptr(v_records), int(c0), int(c1), _stream()),
                           "sgn_project_bwd_range")
            if after_range is not None:
                after_range(k)
        if partials is not None:
            _lib.check(L.sgn_pose_grad_reduce(_ptr(table.dev), table.nseg, table.num_chunks, _ptr(partials), _ptr(v_pose), _stream()),
                       "sgn_pose_grad_reduce")
        if view_partials is not None:
            _lib.check(L.sgn_view_grad_reduce(table.num_chunks, _ptr(view_partials), _ptr(v_view), _stream()), "sgn_view_grad_reduce")
    return flat, arena


# --------------------------------------------------------------------------------------------------
# autograd
# --------------------------------------------------------------------------------------------------
class _Holder:
    """Per-call state the model surface reads back (side-effect attributes, SURVEY.md 8a a15)."""

    def __init__(self):
        self.xys = self.depths = self.radii = self.conics = self.num_tiles_hit = None
        self.records = None
        self.v_records = None
        self.v_absxy = None  # [N,2] absolute screen-space gradient after a backward with RenderSettings.absgrad, else None
        self.grad_arena = None
        self.param_grads = None
        self.v_sky = None
        self.v_pose = None  # [nseg, 16] after a backward through a render whose ``pose`` required grad
        self.v_view = None  # [12] after a backward through a render whose ``view`` required grad
        self.M = 0
        self.tile_bins = self.tile_depth = None
        self.table = None  # the frame's SegmentTable: its device rows are what sgn_metrics reads the parameters through
        self.post_backward = None
        # model path: an object with target(static) -> arena-or-None and publish(arena, static); the parameter
        # gradients are then delivered through it instead of through 6 x segments autograd leaves
        self.grad_sink = None
        # the last backward had no image-space cotangent (only parameter terms', e.g. the scale regularisation's): the blend and
        # projection were skipped, and the arena holds zeros but for the tensors ``term_kinds`` names (PARAM_NAMES positions)
        self.params_only = False
        self.term_kinds: List[int] = []


IMAGE_NAMES = ("rgb", "accumulation", "depth", "object_acc", "background_acc")


def _output_names(settings: RenderSettings, extra: Optional[torch.Tensor], terms: Sequence[ParamTerm]) -> List[str]:
    """The names of a frame's outputs in the order the render node returns them: the images (the two class streams only with
    ``class_streams``), ``extra`` with extra channels, then each term's outputs."""
    names = list(IMAGE_NAMES if settings.class_streams else IMAGE_NAMES[:3])
    if extra is not None:
        names.append("extra")
    return names + [n for t in terms for n in t.names]


class _FramePass(SimpleNamespace):
    """One frame's forward as its backward reads it: the launch structs (cs, bo), the table and parameters, the projection's
    records / radii / tiles_hit, the tile lists and class sub-lists, the blend buffers the backward replays (``saved``, not
    the images), sky, view, extra and terms.  ``outputs``: the forward's outputs in ``_output_names`` order, for the caller
    to hand out."""

    def fill(self, h: _Holder) -> None:
        """The side-effect attributes of ``h`` that the forward sets."""
        h.records, h.radii, h.num_tiles_hit, h.M, h.table = self.records, self.radii, self.tiles_hit, self.M, self.table
        h.xys, h.conics, h.depths = self.records[:, 0:2], self.records[:, 2:5], self.records[:, 9]


def _forward(frame: Frame, settings: RenderSettings, params: List[List[torch.Tensor]], sky: Optional[torch.Tensor],
             extra: Optional[torch.Tensor], pose: Optional[torch.Tensor], view: Optional[torch.Tensor], terms: Sequence[ParamTerm],
             after_project=None) -> _FramePass:
    """The forward of one frame, the one place its stages are called: project, bin, class sub-lists, blend, the extra
    channels, the terms.  ``after_project(radii)`` runs between the projection and the binning."""
    device = params[0][0].device
    K = (settings.sh_degree + 1) ** 2
    for ps in params:
        if ps[4].shape[1] != K - 1:
            raise _lib.SgnError(f"features_rest has {ps[4].shape[1]} coefficients, sh_degree={settings.sh_degree} needs {K - 1}")
    cs = camera_struct(frame.camera, settings)
    if sky is not None:
        sky = sky.contiguous()
        assert sky.shape == (cs.height, cs.width, 3)
    bo = blend_opts(settings, sky is not None)
    table = SegmentTable(frame, params, device)
    if pose is not None:
        table = with_poses(table, pose)
    if view is not None:
        view = check_view(view, device)
    proj = project_fwd(table, cs, device, view)
    records, radii, tiles_hit, _ = proj
    if after_project is not None:  # data parallel: the rows this replica sees are published early (dp.SymmetricExchange)
        after_project(radii)
    M, sorted_ids, tile_bins = bin_and_sort(cs, records, radii, proj=proj, async_binning=settings.async_binning)
    cls_ids = cls_bins = None
    if settings.class_streams:
        cls_ids, cls_bins = class_lists(cs, M, sorted_ids, tile_bins)
    out = blend_fwd(cs, bo, records, sorted_ids, tile_bins, sky, cls_ids, cls_bins)
    outputs = [out[k] for k in IMAGE_NAMES if k in out]
    if extra is not None:  # generic per-Gaussian channels composited with the main render's weights, 8 per traversal
        assert extra.dim() == 2 and extra.shape[0] == records.shape[0] and extra.dtype == torch.float32 and extra.is_cuda
        extra = extra.contiguous().detach()
        outputs.append(blend_extra_fwd(cs, bo, records, sorted_ids, tile_bins, out["final_T"], out["final_idx"], extra))
    for t in terms:  # terms of the parameters alone (the scale regularisation, ...), from the frame's table
        outputs += t.forward(table)
    # "sched", the heavy-first work lists' scratch, is saved too: the backward rebuilds its schedule in it
    saved = {k: out[k] for k in ("raw", "final_T", "final_idx", "tile_depth", "sched") if k in out}
    return _FramePass(settings=settings, cs=cs, bo=bo, table=table, params=params, records=records, radii=radii, tiles_hit=tiles_hit,
                      M=M, sorted_ids=sorted_ids, tile_bins=tile_bins, cls_ids=cls_ids, cls_bins=cls_bins, saved=saved, sky=sky,
                      view=view, extra=extra, terms=terms, outputs=outputs)


def _backward(st: _FramePass, v: Dict[str, Optional[torch.Tensor]], v_extra_img: Optional[torch.Tensor],
              v_terms: Sequence[Sequence[Optional[torch.Tensor]]], want_v_sky: bool, want_v_pose: bool,
              out: Optional[torch.Tensor] = None, out_offsets: Optional[np.ndarray] = None, make_views: bool = False,
              chunk_ranges=None, after_range=None) -> SimpleNamespace:
    """The backward of one frame, the one place its stages are called: blend, extra channels, projection, then the terms'
    gradients added into the arena.  ``v``: the image cotangents by name; ``v_terms``: one list per term; the arena
    arguments are project_bwd's.  Returns v_records, v_sky, v_absxy (with ``settings.absgrad``), v_extra, arena, views (with
    ``make_views``), v_pose ([nseg, 16] with ``want_v_pose``), v_view (the view's [15] cotangent when the forward had a
    view), params_only and term_kinds; a params-only backward has no v_pose or v_view."""
    # the terms' gradients are added after project_bwd: with ranges, the exchange of a range may already be reading the arena
    assert not st.terms or (chunk_ranges is None and after_range is None), "parameter terms do not combine with ranged exchange"
    s, table, device = st.settings, st.table, st.records.device
    due = [(t, vt) for t, vt in zip(st.terms, v_terms) if any(x is not None for x in vt)]
    # only parameter terms have a cotangent (nothing in view, or a backward of the terms alone): every image-space gradient is
    # zero, so the blend and the projection are skipped and the arena starts from zeros
    params_only = bool(st.terms) and v_extra_img is None and all(t is None for t in v.values())
    v_sky = v_absxy = v_extra = v_pose = v_view = None
    if params_only:
        v_records = torch.zeros_like(st.records)
        if s.absgrad:
            v_absxy = torch.zeros(st.records.shape[0], 2, device=device, dtype=torch.float32)
        arena = _zero_arena(table.static, device, out)
        views = arena_views(arena, table.static) if make_views else None
    else:
        res = blend_bwd(st.cs, st.bo, st.records, st.sorted_ids, st.tile_bins, st.saved, st.sky, v, want_v_sky, st.cls_ids,
                        st.cls_bins, deterministic=s.deterministic, absgrad=s.absgrad)
        v_records, v_sky = res[:2]
        if s.absgrad:
            v_absxy = res[2]
        if v_extra_img is not None:  # adds the extra channels' share of the geometry gradients to v_records before project_bwd
            v_extra = blend_extra_bwd(st.cs, st.bo, st.records, st.sorted_ids, st.tile_bins, st.saved["final_T"],
                                      st.saved["final_idx"], st.extra, v_extra_img, v_records, deterministic=s.deterministic)
        if want_v_pose:
            v_pose = torch.empty(table.nseg, _lib.POSE_FLOATS, device=device, dtype=torch.float32)
        # a render with a device view differentiates with that view and yields its cotangent (cam_pos, detached like the SH
        # view direction, gets 0)
        if st.view is not None:
            v_view = torch.zeros(VIEW_LEN, device=device, dtype=torch.float32)
        views, arena = project_bwd(table, st.params, st.cs, st.records, st.radii, v_records, make_views=make_views, out=out,
                                   out_offsets=out_offsets, chunk_ranges=chunk_ranges, after_range=after_range, v_pose=v_pose,
                                   view=st.view, v_view=None if v_view is None else v_view[:_lib.VIEW_FLOATS])
    for t, vt in due:  # project_bwd overwrote the arena: the terms' gradients are added after it
        t.backward(table, arena, vt, out_offsets)
    return SimpleNamespace(v_records=v_records, v_sky=v_sky, v_absxy=v_absxy, v_extra=v_extra, arena=arena, views=views, v_pose=v_pose,
                           v_view=v_view, params_only=params_only, term_kinds=sorted({k for t, _ in due for k in t.kinds}))


class _SceneGraphRasterize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, frame: Frame, settings: RenderSettings, holder: _Holder, sky: Optional[torch.Tensor],
                extra: Optional[torch.Tensor], pose: Optional[torch.Tensor], view: Optional[torch.Tensor], terms: Tuple[ParamTerm, ...],
                *flat):
        # unused outputs must reach backward as None, not as zero tensors: the kernels specialise on
        # which cotangents exist (depth / background_acc have none in training)
        ctx.set_materialize_grads(False)
        nseg = len(frame.segments)
        if holder.grad_sink is not None:  # flat = (anchor,): only there so that autograd calls backward
            assert len(flat) == 1
            params = [list(seg.params.tensors()) for seg in frame.segments]
        else:
            assert len(flat) == 6 * nseg
            params = [list(flat[6 * i: 6 * i + 6]) for i in range(nseg)]
        st = _forward(frame, settings, params, sky, extra, pose, view, terms)
        st.fill(holder)
        outs, st.outputs = st.outputs, None  # until the backward the node keeps the blend buffers, not the images
        ctx.st, ctx.holder = st, holder
        return tuple(outs)

    @staticmethod
    def backward(ctx, *v):
        st, h = ctx.st, ctx.holder
        _, _, _, want_v_sky, _, want_v_pose, want_v_view = ctx.needs_input_grad[:7]
        names = _output_names(st.settings, st.extra, ())
        vd = dict(zip(names, v))
        v_extra_img = vd.pop("extra", None)
        sink = h.grad_sink
        target = offsets = chunk_ranges = after_range = None
        if sink is not None:
            target = sink.target(st.table.static, st.records.device)
            if target is not None:
                offsets = sink.grad_offsets(st.table.static)  # None: the frame's own layout
                plan = getattr(sink, "exchange_plan", None)  # data parallel: the arena is produced and exchanged range by range
                if plan is not None:
                    chunk_ranges, after_range = plan(st.table)
        g = _backward(st, vd, v_extra_img, _split_term_cotangents(st.terms, v[len(names):]), want_v_sky, want_v_pose, out=target,
                      out_offsets=offsets, make_views=sink is None, chunk_ranges=chunk_ranges, after_range=after_range)
        if sink is not None:
            sink.publish(g.arena, st.table.static)
        h.params_only, h.term_kinds = g.params_only, g.term_kinds
        h.v_records, h.grad_arena, h.v_pose, h.v_absxy = g.v_records, g.arena, g.v_pose, g.v_absxy
        h.v_view = None if g.v_view is None else g.v_view[:_lib.VIEW_FLOATS]
        # the reference reads ``self.xys.grad`` after backward (densification statistics,
        # sgn_splatfacto.py:520-524): xys is a view of the record array, its gradient a view of v_records
        h.xys.grad = g.v_records[:, 0:2]
        if h.post_backward is not None:
            h.post_backward(h)
        g_pose = None if g.v_pose is None else g.v_pose[posed_rows(st.table)[0]]
        flat = (None,) if sink is not None else g.views
        return (None, None, None, g.v_sky, g.v_extra, g_pose, g.v_view if want_v_view else None, None, *flat)


def forward_backward(frame: Frame, settings: RenderSettings, cotangents: Dict[str, Optional[torch.Tensor]],
                     sky: Optional[torch.Tensor] = None, want_param_grads: bool = False, grad_out: Optional[torch.Tensor] = None,
                     chunk_ranges=None, after_range=None, after_project=None, scale_reg: Optional[float] = None,
                     terms: Sequence[ParamTerm] = ()):
    """One frame, forward AND backward, straight through the C-ABI stages (no autograd graph).

    ``cotangents`` maps output names (rgb, accumulation, depth, object_acc, background_acc, and scale_reg with ``scale_reg``) to
    their cotangent tensors (missing / None = no gradient from that output).  ``scale_reg`` (max_ratio, None = off): the outputs
    also hold the scale regularisation (see ``render_frame``); its cotangent, a device scalar, adds the term's gradient to the
    arena after project_bwd.  ``terms`` (raster.ParamTerm): further terms of the parameters alone, likewise.  Returns (outputs, holder);
    ``holder.grad_arena`` is the flat dense gradient arena (what the data-parallel all-reduce and a
    fused optimizer consume), ``holder.v_records[:, 0:2]`` the pixel-space mean gradients the
    densification statistics read.  With ``want_param_grads`` the per-parameter views are returned in
    ``holder.param_grads``.  The same forward and backward as ``render_frame`` + ``backward()``, with the sky's gradient
    (``holder.v_sky``) always computed.
    ``grad_out``: a persistent arena to write into (data parallel: a symmetric allocation); ``chunk_ranges`` / ``after_range``:
    see ``project_bwd``; ``after_project(radii)``: called between the projection and the binning."""
    terms = _terms_of(scale_reg, terms)
    st = _forward(frame, settings, [seg.params.tensors() for seg in frame.segments], sky, None, None, None, terms, after_project)
    named = {n for t in terms for n in t.names}
    for n in _TERM_NAMES:
        assert cotangents.get(n) is None or n in named, f"a {n} cotangent needs its term (scale_reg= / terms=)"
    g = _backward(st, {k: cotangents.get(k) for k in IMAGE_NAMES}, None, [[cotangents.get(n) for n in t.names] for t in terms],
                  sky is not None, False, out=grad_out, make_views=want_param_grads, chunk_ranges=chunk_ranges, after_range=after_range)
    holder = _Holder()
    st.fill(holder)
    holder.v_records, holder.grad_arena, holder.v_sky, holder.v_absxy = g.v_records, g.arena, g.v_sky, g.v_absxy
    holder.param_grads = g.views
    holder.tile_bins, holder.tile_depth = st.tile_bins, st.saved["tile_depth"]  # diagnostics (tools/depth_stats.py)
    return dict(zip(_output_names(settings, None, terms), st.outputs)), holder


def blend_extra_fwd(cs, bo, records, sorted_ids, tile_bins, final_T, final_idx, extra: torch.Tensor) -> torch.Tensor:
    """extra[N,C] composited with the main render's weights -> [H,W,C] (sgn_blend_extra_fwd)."""
    L = _lib.load()
    Cn = extra.shape[1]
    out = torch.empty(cs.height, cs.width, Cn, device=records.device, dtype=torch.float32)
    with _timed("blend_extra_fwd"):
        _lib.check(L.sgn_blend_extra_fwd(C.byref(cs), C.byref(bo), _ptr(records), _ptr(sorted_ids), _ptr(tile_bins), _ptr(final_T),
                                         _ptr(final_idx), _ptr(extra), Cn, _ptr(out), _stream()), "sgn_blend_extra_fwd")
    return out


def blend_extra_bwd(cs, bo, records, sorted_ids, tile_bins, final_T, final_idx, extra, v_out, v_records,
                    deterministic: Optional[bool] = None) -> torch.Tensor:
    """Returns v_extra[N,C]; adds the geometry part (xy, conic, opacity) to ``v_records`` in place.  ``deterministic``
    (default: SGN_DETERMINISTIC): fixed-point accumulation, bit-identical from run to run (sgn_blend_extra_bwd_det)."""
    L = _lib.load()
    v_extra = torch.zeros_like(extra)
    v_out = v_out.contiguous()
    det = DETERMINISTIC if deterministic is None else deterministic
    with _timed("blend_extra_bwd"):
        if det:
            N, Cn = extra.shape
            fx_geom = torch.zeros(N, 6, device=records.device, dtype=torch.int64)
            fx_extra = torch.zeros(N, Cn, device=records.device, dtype=torch.int64)
            fx_scale = torch.empty(2, device=records.device, dtype=torch.float32)
            _lib.check(L.sgn_blend_extra_bwd_det(C.byref(cs), C.byref(bo), _ptr(records), _ptr(sorted_ids), _ptr(tile_bins),
                                                 _ptr(final_T), _ptr(final_idx), _ptr(extra), Cn, N, _ptr(v_out), _ptr(v_extra),
                                                 _ptr(v_records), _ptr(fx_geom), _ptr(fx_extra), _ptr(fx_scale), _stream()),
                       "sgn_blend_extra_bwd_det")
        else:
            _lib.check(L.sgn_blend_extra_bwd(C.byref(cs), C.byref(bo), _ptr(records), _ptr(sorted_ids), _ptr(tile_bins), _ptr(final_T),
                                             _ptr(final_idx), _ptr(extra), extra.shape[1], _ptr(v_out), _ptr(v_extra), _ptr(v_records),
                                             _stream()), "sgn_blend_extra_bwd")
    return v_extra


def render_frame(frame: Frame, settings: Optional[RenderSettings] = None, sky: Optional[torch.Tensor] = None,
                 grad_sink=None, anchor: Optional[torch.Tensor] = None, extra: Optional[torch.Tensor] = None,
                 pose: Optional[torch.Tensor] = None, view: Optional[torch.Tensor] = None, scale_reg: Optional[float] = None,
                 terms: Sequence[ParamTerm] = ()):
    """Render one camera.  Returns (outputs dict, holder).  Segment parameters must be CUDA tensors.

    ``scale_reg`` (max_ratio; None = off, and the call sequence is unchanged): ``out["scale_reg"]`` is nerfstudio's scale
    regularisation over the frame's rows, 0.1 * mean(max(amax(s) / amin(s), max_ratio) - max_ratio) with s = exp(scales), a
    0-d device tensor (sgn_scale_reg_fwd).  It is an output of the render node rather than a function of its own because
    project_bwd OVERWRITES the gradient arena: as an output, the render's backward waits for the term's cotangent and adds
    its gradient (sgn_scale_reg_bwd) into the arena after project_bwd, before the arena is handed on.  When the term is the
    only output with a cotangent (nothing in view, or a backward of the term alone) the blend and projection backward are
    skipped and the arena holds zeros plus the term's gradient.

    ``terms`` (raster.ParamTerm, e.g. ``MCMCRegTerm``): further terms of the parameters alone, computed and differentiated the
    same way; ``out`` holds each term's outputs under its names.  Without terms and ``scale_reg`` the call sequence is unchanged.

    ``view`` [15] (float32, on the device): the world->camera view to project with -- viewmat 3x4 row-major, then cam_pos
    (the SH view directions' origin) -- in place of the one ``frame.camera`` gives; intrinsics and image size still come
    from the camera.  It is read on the device (sgn_project_fwd_view), so a view computed there (camera_pose) costs no
    read-back.  Differentiable: when it requires grad, backward returns its cotangent -- viewmat's 12 floats from the
    projection backward (sgn_project_bwd_view + sgn_view_grad_reduce, no atomics: the same bits on every run over the same
    image cotangents), zeros for cam_pos, whose SH direction is treated as constant -- and composes with ``pose``: both come
    out of the same launches.  Without ``view`` the call sequence is unchanged.

    ``pose`` [n_posed, 16] (float32, on the device; one row per posed segment in the frame's order: R 9 row-major, t 3,
    q 4 -- the unit quaternion of R with w >= 0, as ``object2world_gs`` hands it on): the object->world poses to render
    with, in place of the ones the frame's segments carry.  Differentiable: when it requires grad, backward reduces its
    cotangent inside the projection backward (sgn_project_bwd_pose + sgn_pose_grad_reduce; no atomics, so the gradient
    is the same bits on every run over the same image cotangents in deterministic mode).  R enters through the means and
    q through the covariances only, exactly as the kernels use them; nothing ties the two together here, that is the
    caller's parametrisation (box_pose.BoxPoseOptimizer).  Without ``pose`` the call sequence is unchanged.

    ``extra`` [N, C] (rows in the frame's concatenated order, float32): generic per-Gaussian channels -- e.g. semantic
    logits -- composited with the weights of the main render into ``out["extra"]`` [H, W, C], 8 channels per traversal,
    differentiable w.r.t. ``extra`` and the Gaussian parameters.

    With ``grad_sink`` (+ ``anchor``, a 1-element leaf that requires grad) the parameter gradients are handed
    to the sink after backward instead of flowing through one autograd leaf per parameter tensor."""
    settings = settings or RenderSettings()
    holder = _Holder()
    holder.grad_sink = grad_sink
    flat = [anchor] if grad_sink is not None else [t for seg in frame.segments for t in seg.params.tensors()]
    terms = _terms_of(scale_reg, terms)
    outs = _SceneGraphRasterize.apply(frame, settings, holder, sky, extra, pose, view, terms, *flat)
    out = dict(zip(_output_names(settings, extra, terms), outs))
    if sky is not None:
        out["sky"] = sky
    return out, holder
