"""Prompt-to-prompt injection on the oracle's forward: sample b replays sample a's attention probabilities.

For sample b with source a, every AttnBlock computes, per head,

    O_b = (softmax(scale * Q_a [K_a,self ; K_a,cond]^T) * w_b) [V_b,self ; V_b,cond]

where Q_a and K_a are sample a's own projections in the same forward, w_b is sample b's attn_weights (post-softmax, not
renormalised, on the last len(w_b) keys; all ones without) and V_b sample b's own values.  Everything else is paella_oracle
unchanged: its attention_core is called as it is, on the injected rows with q and k replaced by the source row's, in float64.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
from torch import Tensor

from . import paella_oracle as po


def injected_core(src: Sequence[Optional[int]], weights: Sequence[Optional[Tensor]]):
    """An attention_core for a batch whose sample b reads q and k from sample src[b] (None: its own) and is weighted by
    weights[b] (None: unweighted), computed per sample in float64 and returned in q's dtype."""
    attention_core = po.attention_core

    def core(q, k, v, nhead, aw=None):
        out = []
        for b in range(q.shape[0]):
            a = src[b] if src[b] is not None else b
            out.append(attention_core(q[a:a + 1].double(), k[a:a + 1].double(), v[b:b + 1].double(), nhead, weights[b]))
        return torch.cat(out).to(q.dtype)
    return core


def paella_forward_injected(sd, cfg: po.PaellaConfig, x: Tensor, r: Tensor, byt5: Tensor, clip=None, clip_image=None,
                            src: Optional[Sequence[Optional[int]]] = None, attn_weights: Optional[Sequence[Optional[Tensor]]] = None,
                            mm=po.mm_fp32) -> Tensor:
    """Logits [B, num_labels, H, W] of one forward where sample b < B with src[b] not None attends with sample src[b]'s
    probabilities, and ``attn_weights`` gives each sample its own weight vector (None: unweighted)."""
    B = x.shape[0]
    src = list(src) if src is not None else [None] * B
    weights = list(attn_weights) if attn_weights is not None else [None] * B
    core = po.attention_core
    po.attention_core = injected_core(src, weights)
    try:
        return po.paella_forward(sd, cfg, x, r, byt5, clip, clip_image, None, mm)
    finally:
        po.attention_core = core
