"""Token scoring in fp64 torch on the oracle's forward: train.py's per-token objective (src/train.py:36,64,71).

For logits l [B, num_labels, H, W] and target codes y [B, H, W], per token:

    lse    = log sum_j exp(l_j)
    nll    = lse - l_y                                  nn.CrossEntropyLoss(reduction='none')
    loss   = (1 - eps) nll + eps (lse - mean_j l_j)     nn.CrossEntropyLoss(label_smoothing=eps, reduction='none')
    argmax = the lowest j with l_j = max l              pred.argmax(1)

A guided sample is scored on the notebook's guided logits l_c cfg + l_u (1 - cfg), l_u being the forward under the
unconditional inputs.  The logits come from paella_oracle.paella_forward (pinned to the reference by tests/golden/paella_tiny.npz)
and everything after them is restated here in float64.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import Tensor

from . import paella_oracle as po


def token_scores(logits: Tensor, targets: Tensor, eps: float = 0.0) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """(nll, smooth, loss, argmax) in float64 (argmax int64) from logits [B, K, H, W] and targets [B, H, W]; smooth is
    lse - mean_j l_j and loss (1 - eps) nll + eps smooth."""
    l = logits.double()
    lse = torch.logsumexp(l, 1)
    nll = lse - l.gather(1, targets.long()[:, None]).squeeze(1)
    smooth = lse - l.mean(1)
    return nll, smooth, (1.0 - eps) * nll + eps * smooth, l.argmax(1)


def score_logits(sd, cfg: po.PaellaConfig, x: Tensor, r: Tensor, cond: dict, uncond: Optional[dict] = None,
                 scale: Optional[float] = None) -> Tensor:
    """float64 logits [B, num_labels, H, W] the scores are taken on: the oracle's forward of x under ``cond``, or with ``scale``
    the guided mix l_c scale + l_u (1 - scale) with the forward under ``uncond``."""
    def fwd(g):
        return po.paella_forward(sd, cfg, x, r, g["byt5"], g.get("clip"), g.get("clip_image")).double()
    lc = fwd(cond)
    if scale is None:
        return lc
    return lc * float(scale) + fwd(uncond) * (1.0 - float(scale))
