"""Densification by MCMC: gsplat's ``MCMCStrategy`` ("3D Gaussian Splatting as Markov Chain Monte Carlo", Kheradmand et al.,
NeurIPS 2024), as an alternative to the reference's split / duplicate / cull policy (refine.py).

Per sub-model, every ``refine_every`` steps strictly inside (``refine_start``, ``refine_stop``):

1. relocate: the dead rows (opacity <= ``min_opacity``) become copies of live rows drawn in proportion to opacity, and the
   drawn rows' opacity and scale are rescaled so that the copies together render like the original (``compute_relocation``);
   the drawn rows' Adam moments are zeroed;
2. add: ``min(cap_max, int(1.05 n)) - n`` rows drawn over all rows in proportion to opacity are rescaled likewise and appended,
   with zero moments.

Every training step moves each row by a noise of covariance-shaped size that only near-transparent rows feel (``inject_noise``).
The host side here is a few launches per sub-model (csrc/mcmc.cu) and no read-back: the number of dead rows stays on the device,
the number of added rows follows from the row count.  Draws come from Philox keyed by (seed, step, sub-model, purpose, index).

Deliberate differences from gsplat: the update rule runs in fp64 (its alternating sum loses accuracy in fp32 as the count
grows and the opacity nears 1), and the regularisers average over the frame's rows (raster.MCMCRegTerm), not all rows.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib


@dataclass
class MCMCSettings:
    """One sub-model's MCMC settings; the defaults are gsplat's ``MCMCStrategy``."""

    cap_max: int = 1_000_000
    noise_lr: float = 5e5
    min_opacity: float = 0.005
    refine_start: int = 500
    refine_stop: int = 25_000
    refine_every: int = 100


def in_window(s: MCMCSettings, step: int) -> bool:
    """gsplat's window, strict at both ends."""
    return s.refine_start < step < s.refine_stop


def due(s: MCMCSettings, step: int) -> bool:
    return in_window(s, step) and s.refine_every > 0 and step % s.refine_every == 0


def num_added(n: int, s: MCMCSettings) -> int:
    """``max(0, min(cap_max, int(1.05 * n)) - n)``, in Python doubles as gsplat computes it."""
    return max(0, min(int(s.cap_max), int(1.05 * n)) - n)


def _p(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check_rows(t: torch.Tensor, rows: int, what: str) -> int:
    if not t.is_cuda:
        raise _lib.SgnError(f"{what} must be a CUDA tensor: the MCMC kernels have no CPU path")
    assert t.dtype == torch.float32 and t.is_contiguous() and t.shape[0] == rows, (what, t.dtype, tuple(t.shape), rows)
    return t.numel() // rows if rows > 0 else 1


def tensor_table(ts: Sequence[torch.Tensor], rows: int) -> _lib.MCMCTensors:
    """The row-major tensors [rows, ...] of one sub-model as an sgn_mcmc_tensors (at most 16)."""
    assert len(ts) <= _lib.MCMC_MAX_TENSORS, len(ts)
    tab = _lib.MCMCTensors()
    for k, t in enumerate(ts):
        tab.width[k] = max(1, _check_rows(t, rows, f"tensor {k}"))
        tab.data[k] = t.data_ptr()
    tab.count = len(ts)
    return tab


def sample(opacities: torch.Tensor, min_opacity: float, exclude_dead: bool, max_draws: int, seed: int, step: int, sub: int,
           purpose: int, num_draws: Optional[torch.Tensor] = None, uniforms: Optional[torch.Tensor] = None,
           want_dead: bool = False, draw_dead: bool = False) -> Dict[str, torch.Tensor]:
    """``sgn_mcmc_sample`` over one sub-model's opacity logits [n, 1]: ``draws`` [max_draws] (int32; the first ``*num_draws`` are
    drawn when ``num_draws`` (a device int32) is given), ``counts`` [n], ``total`` (device float64), and with ``want_dead`` the
    compacted ``dead_rows`` [n] and ``num_dead`` (device int32); ``draw_dead`` (with ``want_dead``): as many draws as dead rows.
    ``uniforms`` [max_draws] float64 in [0, 1) replace Philox."""
    L = _lib.load()
    n = int(opacities.shape[0])
    _check_rows(opacities, n, "opacities")
    dev = opacities.device
    out = {"draws": torch.empty(max(max_draws, 0), dtype=torch.int32, device=dev),
           "counts": torch.empty(n, dtype=torch.int32, device=dev),
           "total": torch.empty((), dtype=torch.float64, device=dev)}
    if want_dead:
        out["dead_rows"] = torch.empty(n, dtype=torch.int32, device=dev)
        out["num_dead"] = torch.empty((), dtype=torch.int32, device=dev)
    if uniforms is not None:
        assert uniforms.dtype == torch.float64 and uniforms.is_contiguous() and uniforms.numel() >= max_draws and uniforms.device == dev
    if draw_dead:
        assert want_dead and num_draws is None
        num_draws = out["num_dead"]  # written by the same call before its draws
    if num_draws is not None:
        assert num_draws.dtype == torch.int32 and num_draws.device == dev
    sb = L.sgn_mcmc_sample_scratch_bytes(n)
    scratch = torch.empty(sb, dtype=torch.uint8, device=dev)
    _lib.check(L.sgn_mcmc_sample(_p(opacities), n, float(min_opacity), int(exclude_dead), int(max_draws), _p(num_draws),
                                 C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), int(step), int(sub), int(purpose), _p(uniforms),
                                 _p(out["draws"]), _p(out["counts"]), _p(out.get("dead_rows")), _p(out.get("num_dead")), _p(out["total"]),
                                 _p(scratch), sb, _stream()), "sgn_mcmc_sample")
    return out


def update_rows(opacities: torch.Tensor, scales: torch.Tensor, counts: torch.Tensor, min_opacity: float,
                zero: Sequence[torch.Tensor] = ()) -> None:
    """``sgn_mcmc_relocate``: the update rule in place on every row drawn ``counts[i] > 0`` times, and that row of every tensor of
    ``zero`` (the Adam moments) set to 0."""
    L = _lib.load()
    n = int(opacities.shape[0])
    _check_rows(opacities, n, "opacities")
    _check_rows(scales, n, "scales")
    assert counts.dtype == torch.int32 and counts.numel() == n
    tab = tensor_table(zero, n) if zero else None
    _lib.check(L.sgn_mcmc_relocate(_p(opacities), _p(scales), n, _p(counts), float(min_opacity), C.byref(tab) if tab is not None else None,
                                   _stream()), "sgn_mcmc_relocate")


def copy_rows(tensors: Sequence[torch.Tensor], src_rows: torch.Tensor, max_rows: int, dst_rows: Optional[torch.Tensor] = None,
              dst_row0: int = 0, num_rows: Optional[torch.Tensor] = None) -> None:
    """``sgn_mcmc_copy_rows``: row ``dst_rows[j]`` (or ``dst_row0 + j``) <- row ``src_rows[j]`` of every tensor, for j below
    ``max_rows`` (and below the device count ``num_rows`` when given); a negative source is skipped."""
    L = _lib.load()
    if not tensors or max_rows <= 0:
        return
    rows = int(tensors[0].shape[0])
    tab = tensor_table(tensors, rows)
    _lib.check(L.sgn_mcmc_copy_rows(C.byref(tab), _p(dst_rows), int(dst_row0), _p(src_rows), int(max_rows), _p(num_rows), _stream()),
               "sgn_mcmc_copy_rows")


def relocate(params: Sequence[torch.Tensor], carried: Sequence[torch.Tensor], moments: Sequence[torch.Tensor], s: MCMCSettings,
             seed: int, step: int, sub: int, uniforms: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Phase 1 on one sub-model, in place: ``params`` the six tensors in PARAM_NAMES order, ``carried`` further per-row tensors
    copied with them (the semantic logits, the 3D filter sizes), ``moments`` the Adam moments zeroed at the drawn rows.  Returns
    the number of relocated rows as a device int32 (0 when no row is live), read back by nobody here."""
    opac, scales = params[5], params[1]
    n = int(opac.shape[0])
    if n == 0:
        return torch.zeros((), dtype=torch.int32, device=opac.device)
    # as many draws as dead rows, a count that stays on the device: draw j goes to dead row j
    r = sample(opac, s.min_opacity, True, n, seed, step, sub, _lib.MCMC_RELOCATE, uniforms=uniforms, want_dead=True, draw_dead=True)
    update_rows(opac, scales, r["counts"], s.min_opacity, moments)
    copy_rows(list(params) + list(carried), r["draws"], n, dst_rows=r["dead_rows"], num_rows=r["num_dead"])
    return torch.where(r["total"] > 0, r["num_dead"], torch.zeros_like(r["num_dead"]))


def draw_added(params: Sequence[torch.Tensor], count: int, s: MCMCSettings, seed: int, step: int, sub: int,
               uniforms: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Phase 2's draws on one sub-model: ``count`` rows over all rows in proportion to opacity, with the update rule applied in
    place to the drawn rows (their moments are kept).  Returns the draws [count] (int32, device): the caller appends copies of
    those rows in that order (``copy_rows(..., dst_row0=n)``) into tensors grown by ``count`` rows."""
    opac, scales = params[5], params[1]
    r = sample(opac, s.min_opacity, False, count, seed, step, sub, _lib.MCMC_ADD, uniforms=uniforms)
    update_rows(opac, scales, r["counts"], s.min_opacity)
    return r["draws"]


class NoiseTable:
    """The device table of ``sgn_mcmc_noise`` over a list of sub-models, rebuilt only when a pointer, a row count or a noise_lr
    changes (a refinement)."""

    def __init__(self):
        self._key = None
        self.dev = None
        self.num_chunks = self.rows = 0

    def get(self, subs: Sequence[Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, float]], device) -> torch.Tensor:
        key = tuple((m.data_ptr(), int(m.shape[0]), float(sc)) for m, _, _, _, sc in subs) + tuple(
            (s.data_ptr(), q.data_ptr(), o.data_ptr()) for _, s, q, o, _ in subs)
        if key != self._key:
            tab = (_lib.MCMCSub * len(subs))()
            chunk0 = row0 = 0
            for k, (m, s, q, o, sc) in enumerate(subs):
                n = int(m.shape[0])
                for t, w, nm in ((m, 3, "means"), (s, 3, "scales"), (q, 4, "quats"), (o, 1, "opacities")):
                    assert _check_rows(t, n, nm) == w or n == 0, (nm, tuple(t.shape))
                e = tab[k]
                e.means, e.scales, e.quats, e.opacities = m.data_ptr(), s.data_ptr(), q.data_ptr(), o.data_ptr()
                e.count, e.chunk0, e.row0, e.index, e.noise_lr = n, chunk0, row0, k, float(sc)
                chunk0 += (n + 127) // 128
                row0 += n
            self.dev = torch.frombuffer(bytearray(bytes(tab)), dtype=torch.uint8).to(device, non_blocking=True)
            self.num_chunks, self.rows, self._key = chunk0, row0, key
        return self.dev


def inject_noise(table: NoiseTable, subs: Sequence[Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, float]], lr: float,
                 seed: int, step: int, normals: Optional[torch.Tensor] = None, rebuild: bool = True) -> None:
    """``sgn_mcmc_noise`` over every row of ``subs`` = [(means, scales, quats, opacities, noise_lr)], one launch, with ``lr`` the
    means' learning rate of this step.
    ``normals`` [rows, 3] (float32, the sub-models' rows back to back) replace the Philox draws.  ``rebuild=False``: the caller
    knows ``table`` was built over these ``subs`` (its key is not recomputed)."""
    L = _lib.load()
    if not subs:
        return
    dev_tab = table.get(subs, subs[0][0].device) if rebuild else table.dev
    if normals is not None:
        _check_rows(normals, table.rows, "normals")
    _lib.check(L.sgn_mcmc_noise(_p(dev_tab), len(subs), table.num_chunks, float(lr), C.c_uint64(int(seed) & 0xFFFFFFFFFFFFFFFF), int(step),
                                _p(normals), _stream()), "sgn_mcmc_noise")


def moment_tensors(pairs: Sequence[Optional[Tuple[torch.Tensor, torch.Tensor]]]) -> List[torch.Tensor]:
    return [t for p in pairs if p is not None for t in p]
