"""Oracle of the threshold search (test infrastructure only, like oracle/similarity.py).

The reference saves the whole score matrix (diff_retrieval.py:402, :414) and thresholds it (:454).  The oracle's
contract, which dcr_sim_range reproduces: score(q, g) = the float64 dot product of the float32 inputs, rounded to
float32; a pair is reported when that fp32 score is >= the fp32 threshold (never when it is NaN); rows in CSR form with
gallery indices ascending.
"""
from __future__ import annotations

import numpy as np


def dense_scores(q: np.ndarray, g: np.ndarray) -> np.ndarray:
    """float32 [Q, G]: float64 matmul of the float32 inputs, rounded to float32."""
    return (np.asarray(q, dtype=np.float32).astype(np.float64) @ np.asarray(g, dtype=np.float32).astype(np.float64).T
            ).astype(np.float32)


def sim_range(q: np.ndarray, g: np.ndarray, threshold: float, chunk: int = 256):
    """(offsets i64[Q+1], indices i64[P], scores f32[P]) of every pair with fp32 score >= threshold."""
    q = np.asarray(q, dtype=np.float32)
    g = np.asarray(g, dtype=np.float32)
    assert q.ndim == 2 and g.ndim == 2 and q.shape[1] == g.shape[1]
    t = np.float32(threshold)
    offsets = np.zeros(q.shape[0] + 1, dtype=np.int64)
    idx, vals = [], []
    for s in range(0, q.shape[0], chunk):
        S = dense_scores(q[s:s + chunk], g)
        for r in range(S.shape[0]):
            cols = np.nonzero(S[r] >= t)[0]            # NaN >= t is False
            idx.append(cols.astype(np.int64))
            vals.append(S[r, cols])
            offsets[s + r + 1] = offsets[s + r] + cols.size
    cat = (lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dtype=dt))
    return offsets, cat(idx, np.int64), cat(vals, np.float32)
