"""Perturbed-attention guidance on the oracle's forward, and its guided mix.

Sample b's perturbed forward is its conditional forward where, in every AttnBlock listed for it (plan order, the order
paella_oracle.iter_blocks visits them) and every head, each query p computes

    P   = softmax(scale * q_p [K_self ; K_cond]^T) * w_b
    O_p = (sum_{j in self} P_pj) V_self,p + sum_{k in cond} P_pk V_cond,k

w_b being sample b's attn_weights (post-softmax, not renormalised, on the last len(w_b) keys; all ones without).  The image's own
tokens' probability mass goes to the query's own value; the probabilities on the conditioning are unchanged.  Everything else is
paella_oracle unchanged, in float64 for the perturbed attention.  The mix of one guided step is

    l = l_u + cfg [(l_c - l_u) + sum_j w_j (l_j - l_u)] + s (l_c - l_p),      unguided (cfg None): l_c + s (l_c - l_p)
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
from torch import Tensor

from . import paella_oracle as po


def perturbed_core(q, k, v, nhead: int, n_self: int, attn_weights: Optional[Tensor] = None) -> Tensor:
    """attention_core with the self part of the map collapsed onto the diagonal, for one sample: q [1,Nq,E], k/v [1,Nk,E] whose
    first n_self keys are the queries' own tokens (n_self = Nq, or 0), in float64."""
    B, Nq, E = q.shape
    Nk = k.shape[1]
    hd = E // nhead
    qh = q.double().view(B, Nq, nhead, hd).permute(0, 2, 1, 3)
    kh = k.double().view(B, Nk, nhead, hd).permute(0, 2, 1, 3)
    vh = v.double().view(B, Nk, nhead, hd).permute(0, 2, 1, 3)
    p = torch.softmax((qh @ kh.transpose(-2, -1)) / (hd ** 0.5), dim=-1)
    if attn_weights is not None:
        w = torch.ones(Nk, dtype=torch.float64)
        w[-attn_weights.shape[0]:] = attn_weights.double()
        p = p * w
    o = p[..., n_self:] @ vh[:, :, n_self:]
    if n_self:
        o = o + p[..., :n_self].sum(-1, keepdim=True) * vh[:, :, :n_self]
    return o.permute(0, 2, 1, 3).reshape(B, Nq, E).to(q.dtype)


def paella_forward_pag(sd, cfg: po.PaellaConfig, x: Tensor, r: Tensor, byt5: Tensor, clip=None, clip_image=None,
                       blocks: Optional[Sequence[Optional[Sequence[int]]]] = None,
                       attn_weights: Optional[Sequence[Optional[Tensor]]] = None, mm=po.mm_fp32) -> Tensor:
    """Logits [B, num_labels, H, W] of one forward where sample b with blocks[b] not None is perturbed in those AttnBlocks, and
    ``attn_weights`` gives each sample its own weight vector (None: unweighted)."""
    B = x.shape[0]
    blocks = [set(bl) if bl is not None else set() for bl in blocks] if blocks is not None else [set()] * B
    weights = list(attn_weights) if attn_weights is not None else [None] * B
    core, block = po.attention_core, po.attn_block
    index = [0]

    def attn_block(x_, c_embed, sd_, pre, nhead, self_attn, aw=None, mm_=po.mm_fp32):
        i = index[0]
        index[0] += 1
        n_self = x_.shape[1] * x_.shape[2] if self_attn else 0

        def core_i(q, k, v, nh, _aw=None):
            out = []
            for b in range(q.shape[0]):
                if i in blocks[b]:
                    out.append(perturbed_core(q[b:b + 1], k[b:b + 1], v[b:b + 1], nh, n_self, weights[b]))
                else:
                    out.append(core(q[b:b + 1].double(), k[b:b + 1].double(), v[b:b + 1].double(), nh, weights[b]).to(q.dtype))
            return torch.cat(out)
        po.attention_core = core_i
        try:
            return block(x_, c_embed, sd_, pre, nhead, self_attn, None, mm_)
        finally:
            po.attention_core = core

    po.attn_block = attn_block
    try:
        return po.paella_forward(sd, cfg, x, r, byt5, clip, clip_image, None, mm)
    finally:
        po.attn_block = block


def pag_mix(l_c: Tensor, l_p: Tensor, scale: float, l_u: Optional[Tensor] = None, cfg: Optional[float] = None,
            terms: Sequence = ()) -> Tensor:
    """The guided logits of one step in float64: l_u + cfg [(l_c - l_u) + sum_j w_j (l_j - l_u)] + s (l_c - l_p), or with cfg
    None l_c + s (l_c - l_p).  ``terms``: (w_j, l_j) pairs."""
    l_c, l_p = l_c.double(), l_p.double()
    if cfg is None:
        return l_c + scale * (l_c - l_p)
    l_u = l_u.double()
    g = l_c - l_u
    for w, l_j in terms:
        g = g + w * (l_j.double() - l_u)
    return l_u + cfg * g + scale * (l_c - l_p)
