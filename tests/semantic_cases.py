"""Float64 statement of the semantic term (csrc/semantic.cu, semantic.py): the cross-entropy loss over the valid pixels, its
cotangent, the confusion matrix of eval with the metrics derived from it, and the row map of the refinement carry.

Valid pixel: 0 <= label < C and (no mask or mask != 0).  loss = w * sum_valid (logsumexp(S[p]) - S[p, label]) / n_valid, 0 when
n_valid = 0; v = g * w / n_valid * (softmax(S[p]) - onehot(label)) on the valid pixels, 0 elsewhere.  Argmax ties go to the
lowest class.  The carry: output rows [survivors | split samples, sample-major | duplicates], each a copy of its source row;
survivors keep their moments, new rows start at zero (what the refinement does to features_dc)."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

RF_SPLIT, RF_DUP, RF_KEEP_ORIG, RF_KEEP_SPLIT, RF_KEEP_DUP = 0x01, 0x02, 0x04, 0x08, 0x10


def valid_ref(labels: np.ndarray, C: int, mask: Optional[np.ndarray] = None) -> np.ndarray:
    lab = np.asarray(labels).reshape(-1).astype(np.int64)
    ok = (lab >= 0) & (lab < C)
    if mask is not None:
        ok &= np.asarray(mask).reshape(-1) != 0
    return ok


def loss_ref64(logits: np.ndarray, labels: np.ndarray, mask: Optional[np.ndarray] = None, weight: float = 1.0) -> Tuple[float, int]:
    """(loss, n_valid) in float64."""
    C = logits.shape[-1]
    S = np.asarray(logits, np.float64).reshape(-1, C)
    ok = valid_ref(labels, C, mask)
    n = int(ok.sum())
    if n == 0:
        return 0.0, 0
    s, lab = S[ok], np.asarray(labels).reshape(-1)[ok].astype(np.int64)
    m = s.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(s - m).sum(axis=1))
    return float(weight * (lse - s[np.arange(n), lab]).sum() / n), n


def grad_ref64(logits: np.ndarray, labels: np.ndarray, mask: Optional[np.ndarray] = None, weight: float = 1.0,
               grad_loss: float = 1.0) -> np.ndarray:
    """d loss / d logits, shaped like ``logits``."""
    C = logits.shape[-1]
    S = np.asarray(logits, np.float64).reshape(-1, C)
    ok = valid_ref(labels, C, mask)
    v = np.zeros_like(S)
    n = int(ok.sum())
    if n:
        s = S[ok]
        e = np.exp(s - s.max(axis=1, keepdims=True))
        p = e / e.sum(axis=1, keepdims=True)
        p[np.arange(n), np.asarray(labels).reshape(-1)[ok].astype(np.int64)] -= 1.0
        v[ok] = grad_loss * weight / n * p
    return v.reshape(logits.shape)


def confusion_ref64(logits: np.ndarray, labels: np.ndarray, mask: Optional[np.ndarray] = None) -> np.ndarray:
    """[C, C] int64: entry (label, argmax) counts the valid pixels (np.argmax takes the first maximum)."""
    C = logits.shape[-1]
    S = np.asarray(logits).reshape(-1, C)
    ok = valid_ref(labels, C, mask)
    conf = np.zeros((C, C), np.int64)
    np.add.at(conf, (np.asarray(labels).reshape(-1)[ok].astype(np.int64), S[ok].argmax(axis=1)), 1)
    return conf


def metrics_ref64(conf: np.ndarray) -> Tuple[float, float]:
    """(pixel accuracy, mean IoU over the classes whose union is > 0); NaN where undefined."""
    conf = np.asarray(conf, np.float64)
    tp = np.diag(conf)
    union = conf.sum(0) + conf.sum(1) - tp
    seen = union > 0
    acc = tp.sum() / conf.sum() if conf.sum() > 0 else float("nan")
    miou = float((tp[seen] / union[seen]).mean()) if seen.any() else float("nan")
    return float(acc), miou


def carry_rows_ref(flags: np.ndarray, n_split_samples: int) -> Tuple[np.ndarray, np.ndarray]:
    """(source row of every output row, whether it keeps its source's moments) for the refinement's flag bytes."""
    f = np.asarray(flags).astype(np.int64)
    rows = np.arange(f.shape[0])
    keep = rows[(f & RF_KEEP_ORIG) != 0]
    split = rows[(f & RF_KEEP_SPLIT) != 0]
    dup = rows[(f & RF_KEEP_DUP) != 0]
    src = np.concatenate([keep] + [split] * n_split_samples + [dup]).astype(np.int64)
    kept = np.concatenate([np.ones(keep.shape[0], bool), np.zeros(src.shape[0] - keep.shape[0], bool)])
    return src, kept


def carry_ref(src: np.ndarray, flags: np.ndarray, n_split_samples: int, moments: Optional[Tuple[np.ndarray, np.ndarray]] = None):
    """The carried tensor (and moments) for ``flags``."""
    rows, kept = carry_rows_ref(flags, n_split_samples)
    out = np.asarray(src)[rows]
    if moments is None:
        return out, None
    m, v = (np.where(kept.reshape((-1,) + (1,) * (out.ndim - 1)), np.asarray(x)[rows], 0.0).astype(np.asarray(x).dtype) for x in moments)
    return out, (m, v)
