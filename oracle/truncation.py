"""fp64 restatement of the fused sampler's top-k / top-p truncation (include/paella_b200.h,
pb200_paella_sample_tokens_params_trunc): the kept set of a row of scaled logits s and the Gumbel-max winner over it, given
the Exp(1) draws q of that row (oracle/philox.py).  Every function takes numpy arrays of one row or of rows [n, NL]."""
import numpy as np


def kept_set(s: np.ndarray, k: int = 0, p: float = 1.0) -> np.ndarray:
    """bool mask of the kept labels.  top-k (k >= 1): s >= the k-th largest s, equal values counted separately (boundary ties
    kept; k >= NL keeps all).  top-p (0 < p < 1): over the top-k set, w = exp(s - max s); tau_p = the largest kept s_j with
    sum_{s_i >= s_j, kept} w_i >= p * sum_kept w; kept s >= tau_p.  k = 0 and p = 1 are off."""
    s = np.asarray(s, dtype=np.float64)
    if s.ndim == 2:
        return np.stack([kept_set(r, k, p) for r in s])
    keep = np.ones(s.shape, dtype=bool)
    if 0 < k < s.size:
        keep = s >= np.sort(s)[::-1][k - 1]
    if 0.0 < p < 1.0:
        w = np.where(keep, np.exp(s - s.max()), 0.0)
        # mass at or above each kept value: sum of w over s_i >= s_j
        order = np.argsort(-s, kind="stable")
        ss, ws = s[order], w[order]
        cum = np.cumsum(ws)
        last = np.searchsorted(-ss, -ss, side="right") - 1          # the last index of each value's tie group
        mass_at = cum[last]
        ok = keep[order] & (mass_at >= p * w.sum())
        tau = ss[ok].max()
        keep &= s >= tau
    return keep


def truncated_winner(s: np.ndarray, q: np.ndarray, k: int = 0, p: float = 1.0) -> np.ndarray:
    """argmax over the kept labels of s - log q (the first maximum), per row."""
    s, q = np.atleast_2d(np.asarray(s, np.float64)), np.atleast_2d(np.asarray(q, np.float64))
    score = np.where(kept_set(s, k, p), s - np.log(q), -np.inf)
    return score.argmax(1)


def boundary_distance(s: np.ndarray, k: int = 0, p: float = 1.0):
    """For one row: (tau_k, the smallest relative distance |mass_at(s_j) - p sum w| / sum w over the kept set's values), the
    quantities a margin audit compares with the kernel's fixed-point bound.  tau_k is None when top-k is off, the distance
    inf when top-p is."""
    s = np.asarray(s, np.float64)
    tau_k = np.sort(s)[::-1][k - 1] if 0 < k < s.size else None
    if not 0.0 < p < 1.0:
        return tau_k, np.inf
    keep = s >= tau_k if tau_k is not None else np.ones(s.shape, bool)
    w = np.where(keep, np.exp(s - s.max()), 0.0)
    vals = np.unique(s[keep])
    mass = np.array([w[s >= v].sum() for v in vals])
    return tau_k, float(np.abs(mass - p * w.sum()).min() / w.sum())
