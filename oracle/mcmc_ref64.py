"""Float64 statement of densification by MCMC (gsplat's MCMCStrategy, "3D Gaussian Splatting as Markov Chain Monte Carlo",
Kheradmand et al., NeurIPS 2024) as the library implements it (csrc/mcmc.cu, mcmc.py): the relocation update rule
(gsplat's ``compute_relocation``), the relocate and add row / moment semantics on explicit draws, the opacity-weighted sampler
on explicit uniforms, the position noise on explicit normals and the two regularisers.

Inputs are the float32 parameters; o = sigmoid(logit) and s = exp(log_scale) are taken in float32 (as the kernels read them) and
everything after that in float64.
"""
from __future__ import annotations

from math import comb, sqrt
from typing import Dict, List, Sequence, Tuple

import numpy as np

N_MAX = 51
EPS_CLAMP = 1.0 - 2.0 ** -23  # the largest opacity gsplat's clamp keeps (1 - torch.finfo(float32).eps)


def sigmoid32(x: np.ndarray) -> np.ndarray:
    """torch.sigmoid in float32: 1 / (1 + exp(-x))."""
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore"):
        return (np.float32(1.0) / (np.float32(1.0) + np.exp(-x))).astype(np.float32)


def denom_closed(op: float, N: int) -> float:
    """sum_{k=1..N} (-1)^(k-1) C(N,k) o'^k / sqrt(k)."""
    return float(sum((-1) ** (k - 1) * comb(N, k) * op ** k / sqrt(k) for k in range(1, N + 1)))


def denom_double_sum(op: float, N: int) -> float:
    """gsplat's form: sum_{i=1..N} sum_{k=0..i-1} C(i-1,k) (-1)^k o'^(k+1) / sqrt(k+1)."""
    return float(sum(comb(i - 1, k) * (-1) ** k * op ** (k + 1) / sqrt(k + 1) for i in range(1, N + 1) for k in range(i)))


def relocation(o: float, s: np.ndarray, count: int, min_opacity: float) -> Tuple[float, np.ndarray, float]:
    """The update rule for a row drawn ``count`` times (N = min(count + 1, 51)): (clamped o_new, s_new, unclamped o')."""
    N = min(int(count) + 1, N_MAX)
    op = 1.0 - (1.0 - float(o)) ** (1.0 / N)
    ratio = float(o) / denom_closed(op, N)
    o_new = min(max(op, float(np.float32(min_opacity))), EPS_CLAMP)
    return o_new, ratio * np.asarray(s, np.float64), op


def relocation_params(logit: float, log_scale: np.ndarray, count: int, min_opacity: float, sigmoid=sigmoid32) -> Tuple[float, np.ndarray]:
    """The stored (logit, log_scale) of a drawn row in float64: logit(o_new) and log(s_new) from the float32 o and s.  The clamp
    is applied to o' rounded to float32, as the kernel clamps.  ``sigmoid``: the float32 sigmoid to take o with (a device's
    expf may differ from the host's by an ulp, which the logit of an opacity near 1 amplifies)."""
    return relocation_params_o(sigmoid(np.float32(logit)), np.exp(np.asarray(log_scale, np.float32)), count, min_opacity)


def relocation_params_o(o: np.float32, s: np.ndarray, count: int, min_opacity: float) -> Tuple[float, np.ndarray]:
    """``relocation_params`` from the float32 opacity and scales themselves."""
    o = float(np.float32(o))
    s = np.asarray(s, np.float32).astype(np.float64)
    _, s_new, op = relocation(o, s, count, min_opacity)
    o_new = float(min(max(np.float32(op), np.float32(min_opacity)), np.float32(EPS_CLAMP)))
    return float(np.log(o_new / (1.0 - o_new))), np.log(s_new)


def draws_from_uniforms(weights: np.ndarray, u: np.ndarray) -> np.ndarray:
    """First row whose float64 prefix sum exceeds u * total."""
    p = np.cumsum(np.asarray(weights, np.float64))
    return np.searchsorted(p, np.asarray(u, np.float64) * p[-1], side="right")


def acceptable_draws(weights: np.ndarray, u: np.ndarray, rel: float = 1e-12) -> List[set]:
    """Per draw, the rows that may be taken: the statement's row, and where u * total lies within ``rel`` (relative to the total)
    of a prefix-sum boundary, the positive-weight rows on either side of it."""
    w = np.asarray(weights, np.float64)
    p = np.cumsum(w)
    T = p[-1]
    out = []
    for t in np.asarray(u, np.float64) * T:
        ok = {int(np.searchsorted(p, t, side="right"))}
        for r in np.searchsorted(p, [t - rel * T, t + rel * T], side="right"):
            ok.add(int(r))
        ok = {min(r, len(w) - 1) for r in ok}
        out.append({r for r in ok if w[r] > 0})
    return out


def dead_rows(opacity_logits: np.ndarray, min_opacity: float, sigmoid=sigmoid32) -> np.ndarray:
    return np.nonzero(sigmoid(np.asarray(opacity_logits, np.float32).reshape(-1)) <= np.float32(min_opacity))[0]


def relocate(rows: Dict[str, np.ndarray], moments: Dict[str, Tuple[np.ndarray, np.ndarray]], draws: Sequence[int],
             min_opacity: float, sigmoid=sigmoid32) -> Tuple[Dict[str, np.ndarray], Dict[str, Tuple[np.ndarray, np.ndarray]]]:
    """Phase 1 with explicit draws (``draws[j]`` the source of the j-th dead row in ascending order).  ``rows``: every per-row
    tensor by name ("opacities" [n,1] logits and "scales" [n,3] logs among them); ``moments``: name -> (exp_avg, exp_avg_sq) of
    the tensors the optimizer holds.  Returns new dicts (float64 for the two updated tensors)."""
    rows = {k: np.array(v, np.float64) for k, v in rows.items()}
    moments = {k: (np.array(m, np.float64), np.array(v, np.float64)) for k, (m, v) in moments.items()}
    dead = dead_rows(rows["opacities"], min_opacity, sigmoid)
    draws = np.asarray(draws, np.int64)
    assert len(draws) == len(dead)
    if len(dead) == 0:
        return rows, moments
    counts = np.bincount(draws, minlength=rows["opacities"].shape[0])
    for r in np.nonzero(counts)[0]:
        lo, ls = relocation_params(np.float32(rows["opacities"][r, 0]), rows["scales"][r].astype(np.float32), counts[r], min_opacity,
                                   sigmoid)
        rows["opacities"][r, 0], rows["scales"][r] = lo, ls
        for m, v in moments.values():
            m[r] = 0.0
            v[r] = 0.0
    for d, src in zip(dead, draws):
        for t in rows.values():
            t[d] = t[src]
    return rows, moments


def add(rows: Dict[str, np.ndarray], moments: Dict[str, Tuple[np.ndarray, np.ndarray]], draws: Sequence[int],
        min_opacity: float, sigmoid=sigmoid32) -> Tuple[Dict[str, np.ndarray], Dict[str, Tuple[np.ndarray, np.ndarray]]]:
    """Phase 2 with explicit draws: the update rule on the drawn rows (counts from these draws; moments kept), then copies of
    the drawn rows appended in draw order with zero moments."""
    rows = {k: np.array(v, np.float64) for k, v in rows.items()}
    draws = np.asarray(draws, np.int64)
    counts = np.bincount(draws, minlength=rows["opacities"].shape[0])
    for r in np.nonzero(counts)[0]:
        lo, ls = relocation_params(np.float32(rows["opacities"][r, 0]), rows["scales"][r].astype(np.float32), counts[r], min_opacity,
                                   sigmoid)
        rows["opacities"][r, 0], rows["scales"][r] = lo, ls
    rows = {k: np.concatenate([t, t[draws]]) for k, t in rows.items()}
    moments = {k: tuple(np.concatenate([np.asarray(x, np.float64), np.zeros((len(draws),) + np.asarray(x).shape[1:])]) for x in mv)
               for k, mv in moments.items()}
    return rows, moments


def quat_to_rot(q: np.ndarray) -> np.ndarray:
    q = np.asarray(q, np.float64)
    q = q / np.maximum(np.linalg.norm(q, axis=-1, keepdims=True), 1e-12)
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.stack([
        np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
        np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def noise_delta(scales: np.ndarray, quats: np.ndarray, opacity_logits: np.ndarray, eps: np.ndarray, scale: float) -> np.ndarray:
    """gsplat's inject_noise_to_position: Sigma (eps * gate(1 - o) * scale) with Sigma = R diag(s^2) R^T, in float64 from the
    float32 o and s."""
    o = sigmoid32(np.asarray(opacity_logits).reshape(-1)).astype(np.float64)
    gate = 1.0 / (1.0 + np.exp(-100.0 * ((1.0 - o) - 0.995)))
    s = np.exp(np.asarray(scales, np.float32)).astype(np.float64)
    R = quat_to_rot(quats)
    cov = R @ (s[:, :, None] ** 2 * np.swapaxes(R, -1, -2))
    t = np.asarray(eps, np.float64) * (gate * scale)[:, None]
    return np.einsum("nij,nj->ni", cov, t)


def regularisers(opacity_logits: np.ndarray, scales: np.ndarray, w_opacity: float, w_scale: float) -> Tuple[float, float]:
    o = sigmoid32(np.asarray(opacity_logits).reshape(-1)).astype(np.float64)
    s = np.exp(np.asarray(scales, np.float32)).astype(np.float64)
    return w_opacity * o.mean(), w_scale * s.mean()


def regulariser_grads(opacity_logits: np.ndarray, scales: np.ndarray, w_opacity: float, w_scale: float,
                      sigmoid=sigmoid32) -> Tuple[np.ndarray, np.ndarray]:
    """d / d logit of w_o mean(o) and d / d log_scale of w_s mean(s)."""
    o = sigmoid(np.asarray(opacity_logits, np.float32).reshape(-1, 1)).astype(np.float64)
    s = np.exp(np.asarray(scales, np.float32)).astype(np.float64)
    n = o.shape[0]
    return w_opacity / n * o * (1 - o), w_scale / (3 * n) * s
