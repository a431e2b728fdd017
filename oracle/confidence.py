"""Confidence-guided renoising restated in numpy: which tokens a renoising step replaces (paella_b200.utils module docstring).

For one sample with drawn tokens x [N], logits l [N, num_labels] (the operand the step's sampler consumed, through the
out_mapper), temperature T, next noise level t, choice temperature tau and the uniforms u [N] add_noise would draw:

    c_j  = log_softmax(l_j * (1/T))[x_j]           the product rounded once to fp32, the log-softmax in fp64
    n    = floor(fp32(t * N))                       N = the number of tokens in the sample's region (all of them without one)
    g_j  = -log(-log(u_j))                          fp32; u = 0 gives -inf
    k_j  = c_j + fp32(tau * t) * g_j                fp32, each operation rounded
    the n candidates with the smallest keys are renoised, ties to the lower index; a NaN key ranks below every other key.

Keys compare as their order-preserving 32-bit patterns (``order_keys``), so -0 ranks below +0.  A row with tau < 0 is add_noise's
own rule (u <= t), and a row with t < 0 keeps its tokens.  Only numpy and the logits / uniforms given to it are used here.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np


def token_logprob(logits: np.ndarray, inv_t: float, tokens: np.ndarray) -> np.ndarray:
    """c_j: logits [N, K] (fp32 or fp64 values of the fp32 accumulation), fp32 1/T, tokens int [N] -> float64 [N]."""
    s = (np.asarray(logits, dtype=np.float32) * np.float32(inv_t)).astype(np.float64)
    m = s.max(1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(s - m).sum(1))
    return s[np.arange(s.shape[0]), np.asarray(tokens, dtype=np.int64)] - lse


def gumbel(u: np.ndarray) -> np.ndarray:
    """g = -log(-log(u)) in fp32 (u = 0 -> -inf)."""
    u = np.asarray(u, dtype=np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return -np.log(-np.log(u)).astype(np.float32)


def keys(c: np.ndarray, u: np.ndarray, tau: float, t: float) -> np.ndarray:
    """fp32 keys c + fp32(tau * t) * g(u)."""
    tt = np.float32(np.float32(tau) * np.float32(t))
    with np.errstate(invalid="ignore", over="ignore"):
        return (np.asarray(c, dtype=np.float32) + (tt * gumbel(u)).astype(np.float32)).astype(np.float32)


def order_keys(k: np.ndarray) -> np.ndarray:
    """uint32 patterns in the order of the fp32 keys: negative values inverted, others with the sign bit set; NaN -> 0."""
    b = np.asarray(k, dtype=np.float32).view(np.uint32)
    out = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)
    return np.where(np.isnan(k), np.uint32(0), out).astype(np.uint32)


def renoise_count(t: float, n_tokens: int) -> int:
    """n = floor(fp32(t * N)), clamped to [0, N]; 0 for t < 0."""
    if t < 0:
        return 0
    return int(min(max(np.floor(np.float32(t) * np.float32(n_tokens)), 0), n_tokens))


def select(c: np.ndarray, u: np.ndarray, tau: float, t: float, region: Optional[np.ndarray] = None) -> np.ndarray:
    """bool [N]: the tokens a step renoises (region: bool [N] of the candidates, or None for all)."""
    c = np.asarray(c).reshape(-1)
    u = np.asarray(u, dtype=np.float32).reshape(-1)
    cand = np.ones(c.shape[0], dtype=bool) if region is None else np.asarray(region, dtype=bool).reshape(-1)
    if tau < 0:
        return cand & (u <= np.float32(t))
    n = renoise_count(t, int(cand.sum()))
    idx = np.flatnonzero(cand)
    ok = order_keys(keys(c[idx], u[idx], tau, t))
    order = np.lexsort((idx, ok))           # by key, then by index
    m = np.zeros(c.shape[0], dtype=bool)
    m[idx[order[:n]]] = True
    return m


def renoise(x: np.ndarray, random_x: np.ndarray, c: np.ndarray, u: np.ndarray, tau: float, t: float,
            src: Optional[np.ndarray] = None, region: Optional[np.ndarray] = None) -> Tuple[np.ndarray, np.ndarray]:
    """(out, mask) for one sample: random_x where renoised, x elsewhere in the region, src outside it."""
    m = select(c, u, tau, t, region)
    out = np.where(m, np.asarray(random_x).reshape(-1), np.asarray(x).reshape(-1))
    if region is not None:
        out = np.where(np.asarray(region, dtype=bool).reshape(-1), out, np.asarray(src).reshape(-1))
    return out, m
