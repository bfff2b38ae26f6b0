"""Fused multi-tensor Adam over the flat gradient arena (SURVEY.md 8f rank 1).

Drop-in for the nine ``torch.optim.Adam`` instances nerfstudio builds from
street_gaussians_ns/sgn_config.py:71-108 for the Gaussian parameter groups: same update rule (dense, eps 1e-15,
betas (0.9, 0.999)), one kernel launch for all ~200 tensors.  Moments live in two flat arenas laid out like the
gradient arena of a frame in which every sub-model is visible (raster.project_bwd), so a training step is
``forward_backward -> (all-reduce arena) -> FusedAdam.step(arena)``.

Two torch.optim.Adam behaviours the scene graph depends on are kept:

* a parameter without a gradient is skipped -- no moment decay, no step count.  The gradient arena of a frame only
  holds the sub-models visible in it (an actor is in view for a fraction of the frames), so ``step`` takes the
  list of sub-models the arena covers and every tensor keeps its own step count, as torch keeps ``state["step"]``;
* the refinement step replaces parameters and edits their moments (sgn_splatfacto.py:459-511): ``rebuild`` moves the
  optimizer onto the new tensors (refine.py fills the new moment arenas).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .scene import PARAM_NAMES

# street_gaussians_ns/sgn_config.py:84-107
REFERENCE_LRS: Dict[str, float] = {
    "means": 1.6e-4, "scales": 0.005, "quats": 0.001, "features_dc": 0.0025, "features_rest": 0.0025 / 20,
    "opacities": 0.05,
}

ADAM_DTYPE = np.dtype([("param", "<u8"), ("arena_offset", "<i8"), ("grad_offset", "<i8"), ("numel", "<i8"), ("chunk0", "<i4"),
                       ("beta1", "<f4"), ("beta2", "<f4"), ("eps", "<f4"), ("step_size", "<f4"),
                       ("sqrt_bc2", "<f4"), ("one_minus_beta1", "<f4"), ("one_minus_beta2", "<f4")])
assert ADAM_DTYPE.itemsize == C.sizeof(_lib.AdamTensor) == 64
# sgn_adam_rows: the row table of the selective step, parallel to the sgn_adam_tensor rows (flag_row0 = -1: dense)
ADAM_ROWS_DTYPE = np.dtype([("flag_row0", "<i8"), ("row_width", "<i4"), ("pad", "<i4")])
assert ADAM_ROWS_DTYPE.itemsize == C.sizeof(_lib.AdamRows) == 16


def padded(numel: int) -> int:
    """Arena slices are 16-byte aligned: every tensor occupies a multiple of 4 floats."""
    return (numel + 3) // 4 * 4


def arena_capacity(elems: int) -> int:
    """Moment arenas are allocated on a geometric grid of sizes (eight per octave, >= 2 % above the request): a refinement
    changes the model by a few per cent, so the arenas of the new layout almost always have the SAME capacity as the ones
    they replace and come out of the caching allocator's pool instead of cudaMalloc -- which, with peer access enabled
    (data parallel), maps every new allocation into all peers."""
    want = max(int(elems * 1.02), 1024)
    octave = 1 << (want.bit_length() - 1)
    for k in range(8, 17):
        if octave * k // 8 >= want:
            return octave * k // 8
    return octave * 2


class FusedAdam:
    """``params``: per sub-model (segment), the six parameter tensors in PARAM_NAMES order (the order of the gradient arena)."""

    def __init__(self, params: Sequence[Sequence[torch.Tensor]], lrs: Dict[str, float] = None, betas=(0.9, 0.999),
                 eps: float = 1e-15, chunk_elems: Optional[int] = None, extra: Optional[Dict[str, Tuple[torch.Tensor, float]]] = None,
                 reserve_spare: bool = False, rows: Optional[Dict[str, Tuple[Sequence[torch.Tensor], float]]] = None):
        """``extra``: further tensors stepped by the same launch, name -> (tensor, lr): the reference's other Adam groups on
        the step -- the sky cube map ``env_map.base`` [6, res, res, 3] (sgn_splatfacto.py:114-116; group ``sky`` of
        sgn_config.py:71-108).  Their gradients are not part of the rasterizer's arena (the sky gradient comes out of
        nvdiffrast's backward): pass them to ``step(..., extra_grads={name: grad})``; a tensor without a gradient in a step is
        skipped like any parameter whose ``.grad`` is None.

        ``rows``: groups of per-row tensors, name -> (one tensor per sub-model, lr), stepped by the same launch: the per-Gaussian
        semantic logits (group ``semantic``; the reference config names no optimizer for it, so the rate is the caller's).
        Unlike ``extra`` they change shape at a refinement (``rebuild(params, rows=...)``).  Their moments sit behind the extra
        tensors'; their gradients, like the extra tensors', are addressed relative to the gradient arena: pass them to
        ``step(..., row_grads={name: [grad or None per sub-model]})``.  None: the tables and arenas are those without them."""
        self._chunk = chunk_elems if chunk_elems is not None else _lib.load().sgn_adam_chunk_elems()
        self.lrs = dict(REFERENCE_LRS if lrs is None else lrs)
        self.betas, self.eps = betas, eps
        self._extra = dict(extra or {})
        self._rows = {name: (list(ts), lr) for name, (ts, lr) in (rows or {}).items()}
        self.step_count = 0  # calls of step(); the bias correction uses the per-tensor counts below
        self._install(params)
        if self.device.type == "cuda" and chunk_elems is not None and chunk_elems != _lib.load().sgn_adam_chunk_elems():
            # every block of the kernel steps sgn_adam_chunk_elems() elements: a table cut at another chunk size would
            # leave elements unstepped or step them twice (``chunk_elems`` is for host stand-ins of the kernel)
            raise ValueError(f"FusedAdam on CUDA: chunk_elems={chunk_elems}, the kernel's chunk is "
                             f"{_lib.load().sgn_adam_chunk_elems()}")
        self.exp_avg, self.exp_avg_sq = self._new_moments(), self._new_moments()
        if reserve_spare:
            # a refinement needs the old and the new arenas at the same time: put a second pair into the caching allocator's
            # pool now, so that the first refinement does not call cudaMalloc in the middle of training either
            spare = [torch.empty(arena_capacity(self.moment_elems), device=self.device) for _ in range(2)]
            del spare
        self.steps = np.zeros(len(self._params), np.int64)  # torch.optim.Adam keeps state["step"] per parameter

    def _new_moments(self) -> torch.Tensor:
        """A zeroed moment arena of the current layout: the first ``moment_elems`` floats of an allocation of grid capacity."""
        return torch.zeros(arena_capacity(self.moment_elems), device=self.device)[:self.moment_elems]

    # ---- layout ---------------------------------------------------------------------------------------------
    def _install(self, params: Sequence[Sequence[torch.Tensor]], rows: Optional[Dict[str, Sequence[torch.Tensor]]] = None) -> None:
        assert all(len(ps) == 6 for ps in params), "six parameter tensors per sub-model, in PARAM_NAMES order"
        for name, ts in (rows or {}).items():
            self._rows[name] = (list(ts), self._rows[name][1])
        flat = [t for ps in params for t in ps]
        self.kinds = [PARAM_NAMES[i % 6] for i in range(len(flat))]
        self.extra_index = {}
        for name, (t, lr) in self._extra.items():  # appended behind the sub-models' tensors: moments at the end of the arenas
            assert t.is_contiguous() and t.dtype == torch.float32 and t.data_ptr() % 16 == 0, name
            self.extra_index[name] = len(flat)
            flat.append(t)
            self.kinds.append("extra:" + name)
            self.lrs["extra:" + name] = lr
        self.row_index = {}
        for name, (ts, lr) in self._rows.items():  # behind the extra tensors: one tensor per sub-model
            assert len(ts) == len(params), f"row group {name}: {len(ts)} tensors for {len(params)} sub-models"
            self.row_index[name] = len(flat)
            for t in ts:
                assert t.is_contiguous() and t.dtype == torch.float32 and t.data_ptr() % 16 == 0, name
                flat.append(t)
                self.kinds.append("row:" + name)
            self.lrs["row:" + name] = lr
        self.device = flat[0].device
        self.sizes = np.array([padded(t.numel()) for t in flat], np.int64)
        self.offsets = np.concatenate([[0], np.cumsum(self.sizes)[:-1]]).astype(np.int64)
        self.chunks = np.array([(t.numel() + self._chunk - 1) // self._chunk for t in flat], np.int64)
        tab = np.zeros(len(flat), ADAM_DTYPE)
        tab["param"] = [t.data_ptr() for t in flat]
        tab["arena_offset"] = tab["grad_offset"] = self.offsets
        tab["numel"] = [t.numel() for t in flat]
        tab["chunk0"] = np.concatenate([[0], np.cumsum(self.chunks)[:-1]])
        b1, b2 = self.betas
        tab["beta1"], tab["beta2"], tab["eps"] = b1, b2, self.eps
        tab["one_minus_beta1"], tab["one_minus_beta2"] = 1.0 - b1, 1.0 - b2  # double, then rounded (torch)
        self.table = tab
        self.num_chunks = int(self.chunks.sum())
        self.num_segments = len(params)
        self.arena_elems = int(self.sizes[:6 * len(params)].sum())  # the gradient arena of the rasterizer (all sub-models)
        self.moment_elems = int(self.sizes.sum())                   # + the extra tensors' moments behind it
        self._params = flat  # keep the tensors (and their storage) alive
        self._extra_ptrs = {t.data_ptr() for t, _ in self._extra.values()}
        self._extra_ptrs |= {t.data_ptr() for ts, _ in self._rows.values() for t in ts}  # addressed relative to the arena too
        self._lr_vec = np.array([self.lrs[k] for k in self.kinds], np.float64)
        # per tensor, for the selective step: the sub-model whose rows it holds (-1: an extra tensor) and its row width
        self._sub_of = np.array([i // 6 if i < 6 * len(params) else -1 for i in range(len(flat))], np.int64)
        for name, i0 in self.row_index.items():
            self._sub_of[i0:i0 + len(params)] = np.arange(len(params))
        self._width = np.array([t.numel() // t.shape[0] if t.dim() and t.shape[0] else 1 for t in flat], np.int64)

    def extra_tensors(self) -> Dict[str, torch.Tensor]:
        """The further tensors this optimizer steps (``extra``), by name."""
        return {name: t for name, (t, _) in self._extra.items()}

    def row_tensors(self) -> Dict[str, List[torch.Tensor]]:
        """The per-row groups this optimizer steps (``rows``), by name: one tensor per sub-model."""
        return {name: list(ts) for name, (ts, _) in self._rows.items()}

    def row_moment_views(self, name: str, sub: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """exp_avg / exp_avg_sq of sub-model ``sub``'s tensor of row group ``name``."""
        return self.moment_views(self.row_index[name] + sub)

    def set_lr(self, kind: str, lr: float) -> None:
        """Schedulers (e.g. the exponential decay of the means lr, sgn_config.py:85-90) update rates here."""
        self.lrs[kind] = lr
        self._lr_vec = np.array([self.lrs[k] for k in self.kinds], np.float64)

    def moment_views(self, tensor_index: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """exp_avg / exp_avg_sq of one tensor, shaped like the parameter (views of the arenas)."""
        t = self._params[tensor_index]
        o = int(self.offsets[tensor_index])
        return self.exp_avg[o:o + t.numel()].view(t.shape), self.exp_avg_sq[o:o + t.numel()].view(t.shape)

    # ---- the step -------------------------------------------------------------------------------------------
    def step_table(self, present: Optional[Sequence[int]] = None, full_layout: bool = False, grad_arena: Optional[torch.Tensor] = None,
                   extra_grads: Optional[Dict[str, torch.Tensor]] = None,
                   row_grads: Optional[Dict[str, Sequence[Optional[torch.Tensor]]]] = None,
                   kinds: Optional[Sequence[int]] = None, visible: bool = False,
                   row_flag_row0: Optional[Dict[str, Sequence[int]]] = None):
        """Advance the step counts of the tensors that have a gradient and return their sgn_adam_tensor rows.
        ``present``: indices of the sub-models that have a gradient this step (None = all).  The gradient arena
        either holds exactly those, back to back in that order (a frame's arena, the default), or has the optimizer's
        own layout with the absent sub-models' slices unused (``full_layout``: the data-parallel arena, model.py).
        ``kinds``: which of a present sub-model's six tensors (PARAM_NAMES positions) have a gradient (None = all six); the
        arena keeps its layout, the other tensors are skipped -- moments, step counts and values untouched, as torch.optim.Adam
        skips a parameter whose ``grad`` is None.

        ``visible``: return ``(tab, rows)``, with the parallel sgn_adam_rows table of the selective step.  The flags are in the
        frame's row order -- the present sub-models back to back, in ``present``'s order (None: all, in the optimizer's order)
        -- so a present sub-model's tensors, and its tensors of the row groups, start at the sum of the row counts of the present
        sub-models before it; the extra tensors are dense (flag_row0 = -1).  ``row_flag_row0``: name of a row group -> per
        sub-model the flag byte of its row 0, in place of the frame's (a mask kept across frames, training.py); a row-group
        tensor with a gradient whose sub-model is not present needs one."""
        extras = []
        if self.extra_index:  # rows of the extra tensors that have a gradient this step
            assert not extra_grads or grad_arena is not None, "extra_grads need grad_arena (their offsets are relative to it)"
            for name, g in (extra_grads or {}).items():
                if g is None:
                    continue
                i = self.extra_index[name]
                assert g.is_contiguous() and g.dtype == torch.float32 and g.numel() == self._params[i].numel()
                delta = g.data_ptr() - grad_arena.data_ptr()
                assert delta % 4 == 0
                extras.append((i, delta // 4))  # the kernel addresses gradients as grad_arena + offset: any float address works
        if self.row_index:  # rows of the per-row groups' tensors that have a gradient this step
            assert not row_grads or grad_arena is not None, "row_grads need grad_arena (their offsets are relative to it)"
            for name, gs in (row_grads or {}).items():
                assert len(gs) == self.num_segments, (name, len(gs))
                for s, g in enumerate(gs):
                    if g is None:
                        continue
                    i = self.row_index[name] + s
                    assert g.is_contiguous() and g.dtype == torch.float32 and g.numel() == self._params[i].numel(), (name, s)
                    delta = g.data_ptr() - grad_arena.data_ptr()
                    assert delta % 4 == 0
                    extras.append((i, delta // 4))
        if present is None and not self.extra_index and not self.row_index and kinds is None:
            idx = slice(None)
            tab = self.table  # grad_offset == arena_offset, chunk0 as installed
        else:
            present = list(range(self.num_segments)) if present is None else list(present)
            assert len(set(present)) == len(present) and all(0 <= s < self.num_segments for s in present), present
            idx = (np.asarray(present, np.int64)[:, None] * 6 + np.arange(6)[None, :]).reshape(-1)
            goff = self.table["grad_offset"][idx]
            if not full_layout and len(present) < self.num_segments:
                goff = np.concatenate([[0], np.cumsum(self.sizes[idx])[:-1]])
            if kinds is not None:  # the arena's layout holds all six tensors: offsets first, then the selection
                assert all(0 <= k < 6 for k in kinds), kinds
                keep = np.isin(idx % 6, np.asarray(list(kinds), np.int64))
                idx, goff = idx[keep], goff[keep]
            n_own = len(idx)
            idx = np.concatenate([idx, np.asarray([i for i, _ in extras], np.int64)]) if extras else idx
            tab = self.table[idx]
            ch = self.chunks[idx]
            tab["grad_offset"][:n_own] = goff
            for r, (_, off) in enumerate(extras):
                tab["grad_offset"][n_own + r] = off
            tab["chunk0"] = np.concatenate([[0], np.cumsum(ch)[:-1]]) if len(idx) else []

        self.steps[idx] += 1
        st = self.steps[idx].astype(np.float64)
        b1, b2 = self.betas
        tab["step_size"] = self._lr_vec[idx] / (1.0 - b1 ** st)   # lr / bias_correction1, in double like torch
        tab["sqrt_bc2"] = np.sqrt(1.0 - b2 ** st)
        if not visible:
            assert row_flag_row0 is None, "row_flag_row0 belongs to the selective step (visible=True)"
            return tab
        return tab, self._flag_rows(tab, idx, present, row_flag_row0)

    def _flag_rows(self, tab: np.ndarray, idx, present: Optional[Sequence[int]],
                   row_flag_row0: Optional[Dict[str, Sequence[int]]]) -> np.ndarray:
        """The sgn_adam_rows table of ``tab`` (whose rows are the optimizer's tensors ``idx``), see step_table."""
        tidx = np.arange(len(self._params), dtype=np.int64)[idx]
        pres = list(range(self.num_segments)) if present is None else list(present)
        frame_row0 = np.full(self.num_segments, -1, np.int64)
        if pres:
            n = np.array([self._params[6 * s].shape[0] for s in pres], np.int64)
            frame_row0[pres] = np.concatenate([[0], np.cumsum(n)[:-1]])
        sub = self._sub_of[tidx]
        f0 = np.where(sub >= 0, frame_row0[np.maximum(sub, 0)], -1)
        for name, r0s in (row_flag_row0 or {}).items():
            i0 = self.row_index[name]
            sel = (tidx >= i0) & (tidx < i0 + self.num_segments)
            r0s = np.asarray(r0s, np.int64)
            assert r0s.shape == (self.num_segments,) and np.all(r0s >= 0), (name, r0s)
            f0[sel] = r0s[tidx[sel] - i0]
        if np.any((sub >= 0) & (f0 < 0)):
            raise ValueError("visible: a row-group tensor of a sub-model that is not in the frame needs row_flag_row0")
        # the kernel indexes a tensor in 32 bits
        assert int(tab["numel"].max(initial=0)) < 2 ** 31
        rows = np.zeros(len(tab), ADAM_ROWS_DTYPE)
        rows["flag_row0"], rows["row_width"] = f0, self._width[tidx]
        return rows

    def step(self, grad_arena: torch.Tensor, present: Optional[Sequence[int]] = None, full_layout: bool = False,
             extra_grads: Optional[Dict[str, torch.Tensor]] = None,
             row_grads: Optional[Dict[str, Sequence[Optional[torch.Tensor]]]] = None, kinds: Optional[Sequence[int]] = None,
             visible: Optional[torch.Tensor] = None, row_flag_row0: Optional[Dict[str, Sequence[int]]] = None) -> None:
        """``visible``: the selective step (gsplat's visible_adam): uint8 [frame rows], one byte per row of the frame in its
        row order (``sgn_visible_flags`` of the frame's radii); a present sub-model's rows whose byte is 0 keep their
        parameters and moments, bit for bit.  The step counts advance as in the dense step.  ``row_flag_row0``: see
        step_table.  None: the dense step (``sgn_adam_step``)."""
        self.step_count += 1
        # the launch is asynchronous: keep the gradient tensors alive until the next step
        self._keep = extra_grads if row_grads is None else (extra_grads, row_grads)
        if visible is None:
            self.launch(self.step_table(present, full_layout, grad_arena, extra_grads, row_grads, kinds), grad_arena)
            return
        self._keep = (self._keep, visible)
        tab, rows = self.step_table(present, full_layout, grad_arena, extra_grads, row_grads, kinds, visible=True,
                                    row_flag_row0=row_flag_row0)
        self.launch(tab, grad_arena, rows=rows, visible=visible)

    def launch(self, tab: np.ndarray, grad_arena: torch.Tensor, rows: Optional[np.ndarray] = None,
               visible: Optional[torch.Tensor] = None) -> None:
        """One ``sgn_adam_step`` over the rows of ``tab`` (from step_table, possibly cut by rows_in_range); with ``rows`` and
        ``visible`` one ``sgn_adam_step_visible``."""
        assert grad_arena.is_cuda, "FusedAdam runs on the CUDA library only"
        if len(tab) == 0:
            return
        # rows of the extra tensors and the row groups (always last) address their gradient relative to the arena, wherever it
        # lives
        outside = self.extra_index or self.row_index
        inside = tab[: len(tab) - sum(1 for k in tab["param"] if int(k) in self._extra_ptrs)] if outside else tab
        if len(inside):
            need = int((inside["grad_offset"] + inside["numel"]).max())
            assert grad_arena.numel() >= need, (grad_arena.numel(), need)
        num_chunks = int(tab["chunk0"][-1] + (int(tab["numel"][-1]) + self._chunk - 1) // self._chunk)
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        L = _lib.load()
        if rows is not None:
            assert visible is not None and visible.is_cuda and visible.dtype == torch.uint8 and visible.is_contiguous()
            assert len(rows) == len(tab)
            masked = rows["flag_row0"] >= 0
            if masked.any():  # every row of a masked tensor has its byte
                last = rows["flag_row0"][masked] + (tab["numel"][masked] + rows["row_width"][masked] - 1) // rows["row_width"][masked]
                assert int(last.max()) <= visible.numel(), (int(last.max()), visible.numel())
            # one upload: the tensor table, then the row table (16-byte aligned behind it)
            raw = np.concatenate([np.ascontiguousarray(tab).view(np.uint8).reshape(-1), np.ascontiguousarray(rows).view(np.uint8).reshape(-1)])
            dev = torch.from_numpy(raw).to(self.device, non_blocking=True)
            _lib.check(L.sgn_adam_step_visible(C.c_void_p(dev.data_ptr()), C.c_void_p(dev.data_ptr() + tab.nbytes), len(tab), num_chunks,
                                               C.c_void_p(grad_arena.data_ptr()), C.c_void_p(self.exp_avg.data_ptr()),
                                               C.c_void_p(self.exp_avg_sq.data_ptr()), C.c_void_p(visible.data_ptr()), stream),
                       "sgn_adam_step_visible")
            return
        dev_tab = torch.from_numpy(np.ascontiguousarray(tab).view(np.uint8).reshape(-1)).to(self.device, non_blocking=True)
        _lib.check(L.sgn_adam_step(C.c_void_p(dev_tab.data_ptr()), len(tab), num_chunks,
                                   C.c_void_p(grad_arena.data_ptr()), C.c_void_p(self.exp_avg.data_ptr()),
                                   C.c_void_p(self.exp_avg_sq.data_ptr()), stream), "sgn_adam_step")

    def rows_in_range(self, tab: np.ndarray, lo: int, hi: int) -> np.ndarray:
        """The part of a step's table that falls into floats [lo, hi) of the arena (full layout: gradient and
        moment offsets coincide): tensors are cut at the range's ends, so that a step can be issued range by range
        while the all-reduce of the next range is still in flight (dp.allreduce_and_step).  ``lo`` / ``hi`` must be
        multiples of 4 floats (16-byte slices)."""
        assert lo % 4 == 0 and hi % 4 == 0 and np.array_equal(tab["grad_offset"], tab["arena_offset"])
        a = np.maximum(tab["arena_offset"], lo)
        b = np.minimum(tab["arena_offset"] + tab["numel"], hi)
        keep = a < b
        out = tab[keep].copy()
        a, b = a[keep], b[keep]
        out["param"] = out["param"] + ((a - out["arena_offset"]) * 4).astype(np.uint64)
        out["arena_offset"] = out["grad_offset"] = a
        out["numel"] = b - a
        ch = (out["numel"] + self._chunk - 1) // self._chunk
        out["chunk0"] = np.concatenate([[0], np.cumsum(ch)[:-1]]) if len(out) else []
        return out

    def rows_in_slices(self, tab: np.ndarray, slices) -> np.ndarray:
        """The part of a step's table inside a LIST of arena slices [(offset, length, ...)] (full layout): what one exchanged
        range of the data-parallel step covers -- the six tensors' rows [r0, r1) of the background, or everything behind it."""
        parts = [self.rows_in_range(tab, int(sl[0]), int(sl[0]) + int(sl[1])) for sl in slices]
        parts = [p for p in parts if len(p)]
        if not parts:
            return tab[:0]
        out = np.concatenate(parts)
        ch = (out["numel"] + self._chunk - 1) // self._chunk
        out["chunk0"] = np.concatenate([[0], np.cumsum(ch)[:-1]])
        return out

    # ---- refinement (sgn_splatfacto.py:459-511) ---------------------------------------------------------------
    def rebuild(self, params: Sequence[Sequence[torch.Tensor]], rows: Optional[Dict[str, Sequence[torch.Tensor]]] = None
                ) -> Tuple[torch.Tensor, torch.Tensor, np.ndarray]:
        """Move the optimizer onto new parameter tensors (same sub-models, new row counts).  Allocates new, ZEROED
        moment arenas for the new layout and returns the OLD ``(exp_avg, exp_avg_sq, offsets)`` so that the caller
        (refine.py) can carry the surviving rows' moments over; step counts are kept (the reference moves
        ``param_state`` -- including ``step`` -- to the new parameter).  ``rows``: the row groups' new tensors, name -> one per
        sub-model (None: unchanged).  A row-group tensor that is still the same storage keeps its moments; a new one starts at
        zero here and the caller carries its rows (semantic.refine_carry)."""
        assert len(params) == self.num_segments
        old = (self.exp_avg, self.exp_avg_sq, self.offsets.copy())
        before = {i: (t.data_ptr(), t.numel()) for name, i0 in self.row_index.items() for i, t in
                  enumerate(self._params[i0:i0 + self.num_segments], i0)}
        self._install(params, rows)
        self.exp_avg, self.exp_avg_sq = self._new_moments(), self._new_moments()
        same = [i for i in self.extra_index.values()]  # the extra tensors do not change in a refinement: their moments move along
        same += [i for i, key in before.items() if key == (self._params[i].data_ptr(), self._params[i].numel())]
        for i in same:
            a, b, n = int(old[2][i]), int(self.offsets[i]), int(self.sizes[i])
            self.exp_avg[b:b + n].copy_(old[0][a:a + n])
            self.exp_avg_sq[b:b + n].copy_(old[1][a:a + n])
        return old

    def rebuild_pointers(self, params: Sequence[Sequence[torch.Tensor]], rows: Optional[Dict[str, Sequence[torch.Tensor]]] = None) -> None:
        """The layout is unchanged but the tensors were re-wrapped (``nn.Parameter(t)`` shares storage): refresh the
        pointer column and the keep-alive list (and the row groups' tensors, when given)."""
        flat = [t for ps in params for t in ps]
        n = len(flat)
        assert [t.numel() for t in flat] == [int(x) for x in self.table["numel"][:n]]
        self.table["param"][:n] = [t.data_ptr() for t in flat]
        self._params = flat + self._params[n:]
        for name, ts in (rows or {}).items():
            i0 = self.row_index[name]
            assert [t.numel() for t in ts] == [int(x) for x in self.table["numel"][i0:i0 + len(ts)]]
            self.table["param"][i0:i0 + len(ts)] = [t.data_ptr() for t in ts]
            self._params[i0:i0 + len(ts)] = list(ts)
            self._rows[name] = (list(ts), self._rows[name][1])
