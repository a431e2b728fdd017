"""Attention maps in fp64 torch on the fp32 oracle: per-token cross-attention heat maps of the denoiser's AttnBlocks.

For sample b, conditioning key s (gen_c_embeddings order) and latent token (y, x), one forward's map is

    (1 / n_attn) * sum over every AttnBlock of (1 / nhead) * sum over heads of P[pos(y, x), n_self + s]

where P is the softmax over [self keys ; conditioning keys] times the attn_weights (post-softmax, not renormalised) -- what the
reference's CustomMultiheadAttention returns with need_weights=True -- and pos(y, x) the block position whose
(patch_size * 2^level)-token footprint holds the token (nearest-neighbour upsampling).  A sampling call averages the maps of its
steps' conditional forwards.  Everything else is paella_oracle unchanged: its attention_core is called as it is, and the
probabilities are recomputed beside it from the same q and k.
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch import Tensor

from . import paella_oracle as po


def attention_probs(q: Tensor, k: Tensor, nhead: int, attn_weights: Optional[Tensor] = None) -> Tensor:
    """q [B, Nq, E], k [B, Nk, E] -> P [B, nhead, Nq, Nk]: attention_core's softmax times its weights on the last n keys."""
    B, Nq, E = q.shape
    Nk = k.shape[1]
    hd = E // nhead
    qh = q.view(B, Nq, nhead, hd).permute(0, 2, 1, 3)
    kh = k.view(B, Nk, nhead, hd).permute(0, 2, 1, 3)
    p = torch.softmax((qh @ kh.transpose(-2, -1)) / (hd ** 0.5), dim=-1)
    if attn_weights is not None:
        w = torch.ones(Nk, dtype=p.dtype)
        w[-attn_weights.shape[0]:] = attn_weights.to(p.dtype)
        p = p * w
    return p


def aggregate(probs: List[Tensor], S: int, hw) -> Tensor:
    """The map [B, S, H, W] of one forward from its AttnBlocks' P [B, nhead, P_l, P_l (self) + S] (self-attention on), in order."""
    H, W = hw
    out = None
    for p in probs:
        B, _, P, Nk = p.shape
        g = int(round(P ** 0.5))
        stride = H // g
        m = p.mean(dim=1)[:, :, Nk - S:]                                  # [B, P, S]: the heads' mean on the conditioning keys
        m = m.transpose(1, 2).reshape(B, S, H // stride, W // stride)
        m = m.repeat_interleave(stride, dim=2).repeat_interleave(stride, dim=3)
        out = m if out is None else out + m
    return out / len(probs)


def paella_maps(sd, cfg: po.PaellaConfig, x: Tensor, r: Tensor, byt5: Tensor, clip=None, clip_image=None,
                attn_weights=None, mm=po.mm_fp32):
    """(features [B, H, W, c_out], maps [B, S, H, W] float64) of one forward (square token grids): the oracle's fp32 forward,
    with each AttnBlock's probabilities and their aggregation in fp64."""
    probs: List[Tensor] = []
    core = po.attention_core

    def recording_core(q, k, v, nhead, aw=None):
        probs.append(attention_probs(q.double(), k.double(), nhead, aw))
        return core(q, k, v, nhead, aw)
    po.attention_core = recording_core
    try:
        feats = po.paella_features(sd, cfg, x, r, byt5, clip, clip_image, attn_weights, mm)
    finally:
        po.attention_core = core
    S = po.c_embeddings(sd, cfg, byt5, clip, clip_image, mm).shape[1]
    return feats, aggregate(probs, S, x.shape[1:])
