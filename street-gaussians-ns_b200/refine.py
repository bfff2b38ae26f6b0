"""Refinement of the Gaussian sets: split / duplicate / cull / opacity reset (SURVEY.md 8f rank 3, second half).

Host side of csrc/refine.cu.  Mirrors what every sub-model's ``refinement_after`` callback does every
``refine_every`` steps (street_gaussians_ns/sgn_splatfacto.py:550-646 with cull_gaussians :648-672, split_gaussians
:674-710, dup_gaussians :712-720) including the surgery on the Adam state (dup_in_optim / remove_from_optim
:459-511), with the same configuration names.  Per sub-model the reference issues ~120 torch statements and eight
``.item()`` syncs; here it is ``sgn_refine_decide`` -> one prefix sum + ONE read-back of four counts ->
``sgn_refine_apply``, which writes the new parameter tensors and the new Adam moments directly (for FusedAdam:
into the new moment arenas, no intermediate copies).

All arithmetic runs in the CUDA library; there is no CPU path (tensors must be CUDA tensors).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .scene import PARAM_NAMES


@dataclass
class RefineSettings:
    """The refinement fields of ``SplatfactoModelConfig`` (sgn_splatfacto.py:158-194; defaults are the ones the scene
    graph's sub-model configs end up with, sgn_config.py:49-65: cull_alpha_thresh 0.02 for the background / 0.005
    for objects, cull_scale_thresh 0.2, stop_split_at 25000 -- pass per sub-model settings where they differ)."""

    warmup_length: int = 500
    refine_every: int = 100
    reset_alpha_every: int = 30
    stop_split_at: int = 25000
    stop_screen_size_at: int = 4000
    densify_grad_thresh: float = 0.0002
    densify_size_thresh: float = 0.01
    n_split_samples: int = 2
    split_screen_size: float = 0.05
    cull_alpha_thresh: float = 0.02
    cull_scale_thresh: float = 0.2
    cull_screen_size: float = 0.15
    continue_cull_post_densification: bool = True
    # the split / duplicate threshold with SceneGraphConfig.absgrad, against the absolute screen-space gradient (normalised
    # alike, * 0.5 * max(H, W)): AbsGS's published value.  No measurement on street data backs it: tune it on the data (set
    # it on the instance).  A plain attribute, not a field: the fields are the reference's SplatfactoModelConfig's
    densify_absgrad_thresh = 0.0008


SIZE_FAC = 1.6  # split_gaussians (:694)


def phase(s: RefineSettings, step: int, num_train_data: int) -> Tuple[bool, bool, bool]:
    """(densify, cull_only, reset_opacity) for a refinement call at ``step`` (:552-566, :620-621, :629)."""
    if step <= s.warmup_length:
        return False, False, False
    reset_interval = s.reset_alpha_every * s.refine_every
    densify = step < s.stop_split_at and step % reset_interval > num_train_data + s.refine_every
    cull_only = (not densify) and step >= s.stop_split_at and s.continue_cull_post_densification
    reset = step < s.stop_split_at and step % reset_interval == s.refine_every
    return densify, cull_only, reset


def opacity_reset_logit(s: RefineSettings) -> float:
    """``torch.logit(torch.tensor(cull_alpha_thresh * 2.0)).item()`` (:631-635): the logit evaluated in fp32."""
    return float(torch.logit(torch.tensor(s.cull_alpha_thresh * 2.0)).item())


def make_config(s: RefineSettings, step: int, last_size: Tuple[int, int], densify: bool, absgrad: bool = False) -> _lib.RefineConfig:
    """``absgrad``: the statistics are absolute screen-space gradients, thresholded at ``densify_absgrad_thresh``."""
    cfg = _lib.RefineConfig()
    cfg.densify = int(densify)
    cfg.n_split_samples = s.n_split_samples
    cfg.use_screen_size = int(step < s.stop_screen_size_at)
    cfg.cull_big = int(step > s.refine_every * s.reset_alpha_every)
    cfg.max_size = float(max(last_size[0], last_size[1]))
    cfg.densify_grad_thresh = s.densify_absgrad_thresh if absgrad else s.densify_grad_thresh
    cfg.densify_size_thresh = s.densify_size_thresh
    cfg.split_screen_size = s.split_screen_size
    cfg.cull_alpha_thresh, cfg.cull_scale_thresh, cfg.cull_screen_size = s.cull_alpha_thresh, s.cull_scale_thresh, s.cull_screen_size
    cfg.inv_size_fac = float(np.float32(1.0) / np.float32(SIZE_FAC))  # ATen: a / scalar == a * (1.f / (float)scalar)
    return cfg


def _backend():
    return _lib.load()


def _require_cuda(t: torch.Tensor, what: str) -> None:
    if not t.is_cuda:
        raise _lib.SgnError(f"{what} must be a CUDA tensor: the refinement kernels have no CPU path")


def _p(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream(t: torch.Tensor):
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream) if t.is_cuda else None


_RECORD_MASKS: Dict[torch.device, torch.Tensor] = {}


class Plan:
    """Decision for one sub-model: flag byte per row, prefix sums, the four totals and the split samples."""

    def __init__(self, n: int, cfg: _lib.RefineConfig, flags: torch.Tensor, scan: torch.Tensor, totals: List[int],
                 samples: Optional[torch.Tensor]):
        self.n, self.cfg, self.flags, self.scan, self.totals, self.samples = n, cfg, flags, scan, totals, samples

    @property
    def out_rows(self) -> int:
        return self.totals[0] + self.cfg.n_split_samples * self.totals[1] + self.totals[2]

    @property
    def changed(self) -> bool:
        """False when every row survives and nothing is added: the tensors can stay as they are."""
        return not (self.totals[0] == self.n and self.totals[1] == 0 and self.totals[2] == 0)

    def record_counts(self) -> torch.Tensor:
        """Seven flag-pattern counts as a device tensor (three launches, nothing read back): rows with HIGH_GRAD, SPLIT, DUP,
        TOOBIG, ALPHA, ALPHA and SPLIT, ALPHA and DUP set."""
        masks = _RECORD_MASKS.get(self.flags.device)
        if masks is None:  # uploaded once per device: a pageable host-to-device copy per sub-model would wait for the stream each time
            masks = _RECORD_MASKS[self.flags.device] = torch.tensor(
                [_lib.RF_HIGH_GRAD, _lib.RF_SPLIT, _lib.RF_DUP, _lib.RF_TOOBIG, _lib.RF_ALPHA, _lib.RF_ALPHA | _lib.RF_SPLIT,
                 _lib.RF_ALPHA | _lib.RF_DUP], dtype=torch.uint8).to(self.flags.device)
        return ((self.flags.view(-1, 1) & masks) == masks).sum(0)

    def record_from(self, counts: Sequence[int]) -> Dict[str, int]:
        """The counters the reference logs in ``refine_record_dict`` (:572-588, :655, :668) from ``record_counts()`` read
        back by the caller (one read-back for all sub-models of a refinement)."""
        high, split, dup, toobig, alpha, alpha_split, alpha_dup = (int(x) for x in counts)
        # cull_gaussians sees 1 + n_split_samples * split + dup rows per source row; the alpha mark of a source row counts for all of them
        out = {"refine_culls_alpha_count": alpha + self.cfg.n_split_samples * alpha_split + alpha_dup}
        if self.cfg.densify:
            out.update(high_grads_count=high, refine_splits_count=split, refine_dups_count=dup)
        if self.cfg.cull_big:
            out["refine_culls_toobigs_count"] = toobig  # old rows only (the flag byte does not keep it for new rows)
        return out

    def record(self) -> Dict[str, int]:
        return self.record_from(self.record_counts().tolist())


def decide_submodel(scales: torch.Tensor, opacities: torch.Tensor, xys_grad_norm: Optional[torch.Tensor],
                    vis_counts: Optional[torch.Tensor], max_2dsize: Optional[torch.Tensor], cfg: _lib.RefineConfig):
    """``sgn_refine_decide`` + the prefix sums of its four mark rows; nothing is read back.  Returns (flags, scan)."""
    L = _backend()
    n = int(scales.shape[0])
    dev = scales.device
    for t, nm in ((scales, "scales"), (opacities, "opacities"), (xys_grad_norm, "xys_grad_norm"), (vis_counts, "vis_counts"),
                  (max_2dsize, "max_2Dsize")):
        if t is not None:
            _require_cuda(t, nm)
            assert t.dtype == torch.float32 and t.is_contiguous() and t.shape[0] == n, (nm, t.dtype, tuple(t.shape), n)
    flags = torch.empty(n, dtype=torch.uint8, device=dev)
    marks = torch.empty((4, n), dtype=torch.int32, device=dev)
    _lib.check(L.sgn_refine_decide(n, C.byref(cfg), _p(scales), _p(opacities), _p(xys_grad_norm), _p(vis_counts), _p(max_2dsize),
                                   _p(flags), _p(marks), _stream(scales)), "sgn_refine_decide")
    return flags, torch.cumsum(marks, dim=1, dtype=torch.int32)


def read_totals(scans: Sequence[torch.Tensor]) -> List[List[int]]:
    """The four totals (survivors, surviving split rows, surviving duplicates, split rows) of every scan: ONE read-back
    for any number of sub-models (the reference syncs eight times per sub-model)."""
    live = [s for s in scans if s.shape[1] > 0]
    vals = torch.stack([s[:, -1] for s in live]).tolist() if live else []
    it = iter(vals)
    return [[int(x) for x in next(it)] if s.shape[1] > 0 else [0, 0, 0, 0] for s in scans]


def finish_plan(flags: torch.Tensor, scan: torch.Tensor, totals: List[int], cfg: _lib.RefineConfig,
                generator: Optional[torch.Generator] = None) -> Plan:
    """Draws the split samples as the reference draws them -- ``torch.randn((samps * n_splits, 3), device=...)`` (:680) --
    so equal seeds give equal draws (data-parallel replicas seed identically and take identical decisions, SURVEY.md 8e)."""
    samples = None
    if cfg.densify:
        samples = torch.randn((cfg.n_split_samples * totals[3], 3), device=flags.device, generator=generator)
    return Plan(int(flags.shape[0]), cfg, flags, scan, totals, samples)


def plan_submodel(scales: torch.Tensor, opacities: torch.Tensor, xys_grad_norm: Optional[torch.Tensor],
                  vis_counts: Optional[torch.Tensor], max_2dsize: Optional[torch.Tensor], cfg: _lib.RefineConfig,
                  generator: Optional[torch.Generator] = None) -> Plan:
    """decide -> prefix sums -> the one host read-back -> split samples, for one sub-model."""
    flags, scan = decide_submodel(scales, opacities, xys_grad_norm, vis_counts, max_2dsize, cfg)
    return finish_plan(flags, scan, read_totals([scan])[0], cfg, generator)


def apply_plan(plan: Plan, src: Sequence[torch.Tensor], dst: Sequence[torch.Tensor],
               src_moments: Optional[Sequence[Tuple[torch.Tensor, torch.Tensor]]] = None,
               dst_moments: Optional[Sequence[Tuple[torch.Tensor, torch.Tensor]]] = None) -> None:
    """``sgn_refine_apply``: ``src`` / ``dst`` are the six parameter tensors in PARAM_NAMES order (dst rows =
    ``plan.out_rows``); the moments are (exp_avg, exp_avg_sq) pairs shaped like the parameters, or None."""
    L = _backend()
    assert len(src) == len(dst) == 6
    t = _lib.RefineTensors()
    for k, (a, b) in enumerate(zip(src, dst)):
        _require_cuda(a, PARAM_NAMES[k])
        assert a.dtype == b.dtype == torch.float32 and a.is_contiguous() and b.is_contiguous()
        assert a.shape[0] == plan.n and b.shape[0] == plan.out_rows and a.shape[1:] == b.shape[1:], (PARAM_NAMES[k], a.shape, b.shape)
        t.src[k], t.dst[k] = a.data_ptr(), b.data_ptr()
        t.width[k] = int(np.prod(a.shape[1:]))
    if src_moments is not None:
        assert dst_moments is not None and len(src_moments) == len(dst_moments) == 6
        for k, ((m0, v0), (m1, v1)) in enumerate(zip(src_moments, dst_moments)):
            for x, rows in ((m0, plan.n), (v0, plan.n), (m1, plan.out_rows), (v1, plan.out_rows)):
                assert x.dtype == torch.float32 and x.is_contiguous() and x.shape[0] == rows and x.shape[1:] == src[k].shape[1:]
            t.src_m[k], t.src_v[k], t.dst_m[k], t.dst_v[k] = m0.data_ptr(), v0.data_ptr(), m1.data_ptr(), v1.data_ptr()
    totals = (C.c_int32 * 4)(*plan.totals)
    _lib.check(L.sgn_refine_apply(plan.n, C.byref(plan.cfg), C.byref(t), _p(plan.flags), _p(plan.scan), totals,
                                  _p(plan.samples), _stream(src[0])), "sgn_refine_apply")


def refine_tensors(params: Sequence[torch.Tensor], moments: Optional[Sequence[Tuple[torch.Tensor, torch.Tensor]]],
                   stats: Tuple[Optional[torch.Tensor], Optional[torch.Tensor], Optional[torch.Tensor]], settings: RefineSettings,
                   step: int, last_size: Tuple[int, int], num_train_data: int, generator: Optional[torch.Generator] = None):
    """Functional form for one sub-model: returns ``(new_params, new_moments, plan)``; tensors that need no change
    are returned as they are.  ``stats`` = (xys_grad_norm, vis_counts, max_2Dsize) as sgn_densify_stats left them.
    The opacity reset (:629-642) is applied last, to the survivors, as in the reference."""
    densify, cull_only, reset = phase(settings, step, num_train_data)
    params, plan = list(params), None
    if stats[0] is None:  # no statistics since the last refinement: the reference returns before anything (:554-555)
        return params, moments, None
    if densify or cull_only:
        cfg = make_config(settings, step, last_size, densify)
        plan = plan_submodel(params[1], params[5], stats[0] if densify else None, stats[1] if densify else None,
                             stats[2] if cfg.use_screen_size else None, cfg, generator)
        if plan.changed:
            new = [torch.empty((plan.out_rows,) + tuple(t.shape[1:]), device=t.device, dtype=t.dtype) for t in params]
            new_m = None
            if moments is not None:
                new_m = [(torch.empty_like(a), torch.empty_like(a)) for a in new]
            apply_plan(plan, params, new, moments, new_m)
            params, moments = new, new_m
    if reset:
        params, moments = reset_opacities(params, moments, settings)
    return params, moments, plan


def reset_opacities(params: List[torch.Tensor], moments, settings: RefineSettings):
    """Clamp the opacity logits to logit(2 * cull_alpha_thresh) and zero their Adam moments (:629-642)."""
    params = list(params)
    params[5] = torch.clamp(params[5], max=opacity_reset_logit(settings))
    if moments is not None:
        moments = list(moments)
        moments[5] = (torch.zeros_like(moments[5][0]), torch.zeros_like(moments[5][1]))
    return params, moments
