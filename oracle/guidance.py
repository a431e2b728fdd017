"""Guidance prompts in fp64 torch: the K-way guided mix over the oracle's forwards.

On a guided step with scale cfg a sample's logits are l_u + cfg * [(l_c - l_u) + sum_j w_j (l_j - l_u)], where l_c is its
conditional forward, l_u its unconditional forward and l_j the conditional forward under term j's inputs.  Each term row is an
ordinary conditional forward (paella_oracle.paella_forward, pinned to the reference by tests/golden/paella_tiny.npz); only the mix
is new, and it is restated here in float64.  The coefficients (cfg, 1 - cfg (1 + sum w), cfg w_j) sum to 1, so the same mix of the
out_mapper's input features gives the same logits: the out_mapper is linear after its LayerNorm.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch
from torch import Tensor

from . import paella_oracle as po


def coefficients(cfg: float, weights: Sequence[float]) -> List[float]:
    """(a_c, a_u, a_1 ..) in float64: cfg, 1 - cfg (1 + sum w), cfg w_j."""
    return [float(cfg), 1.0 - float(cfg) * (1.0 + float(sum(weights)))] + [float(cfg) * float(w) for w in weights]


def mix(cond: Tensor, uncond: Tensor, terms: Sequence[Tensor], cfg: float, weights: Sequence[float]) -> Tensor:
    """The guided mix in float64: uncond + cfg * ((cond - uncond) + sum_j w_j (terms[j] - uncond)).  Works on logits and on the
    features before the out_mapper alike."""
    c, u = cond.double(), uncond.double()
    inner = c - u
    for t, w in zip(terms, weights):
        inner = inner + float(w) * (t.double() - u)
    return u + float(cfg) * inner


def guided_logits(sd: Dict[str, Tensor], cfg: po.PaellaConfig, x: Tensor, r: Tensor, cond: dict, uncond: dict,
                  terms: Sequence[dict], scale: float, weights: Sequence[float]) -> Tensor:
    """float64 logits [B, num_labels, H, W] of one guided step of B samples that share their terms: the oracle's forwards of x
    under ``cond``, ``uncond`` and each term's batch-1 inputs (broadcast to the batch), mixed in float64."""
    B = x.shape[0]

    def fwd(g):
        rep = {k: (v.expand(B, *v.shape[1:]) if torch.is_tensor(v) and v.shape[0] == 1 else v) for k, v in g.items()}
        return po.paella_forward(sd, cfg, x, r, rep["byt5"], rep.get("clip"), rep.get("clip_image"))
    return mix(fwd(cond), fwd(uncond), [fwd(t) for t in terms], scale, weights)
