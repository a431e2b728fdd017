"""Regional prompts in fp32 torch: the denoiser with per-position conditioning masks in its AttnBlocks.

Sample b carries prompts 0..R_b: prompt 0 is its own conditioning, prompt k >= 1 the inputs of its k-th region.  A token's mask
has bit k (k >= 1) set iff the token lies in region k, and bit 0 iff it lies in no region.  An AttnBlock position at level l
covers a (patch_size * 2^l)-token square footprint and carries the OR of its tokens' masks.  It attends to every self key and,
in one softmax, to the conditioning rows of each prompt whose bit it has: the keys are [self ; prompt 0 ; prompt 1 ; ...] with
a boolean mask, which is the reference's Attention2D with an ``attn_mask`` on its nn.MultiheadAttention.  Everything else is
paella_oracle unchanged; tests/golden/regional_tiny.npz pins it to the reference run that way.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F
from torch import Tensor

from . import paella_oracle as po


def token_masks(regions: Sequence[Sequence[Tensor]], hw) -> Tensor:
    """uint8 [B, H, W] masks from each sample's list of bool [H, W] regions."""
    H, W = hw
    out = torch.zeros(len(regions), H, W, dtype=torch.uint8)
    for b, regs in enumerate(regions):
        for k, r in enumerate(regs, start=1):
            out[b] |= r.to(torch.uint8) << k
        out[b][out[b] == 0] = 1
    return out


def position_masks(masks: Tensor, stride: int) -> Tensor:
    """[B, H, W] token masks -> [B, (H/stride) * (W/stride)] position masks: the OR over each stride x stride footprint."""
    B, H, W = masks.shape
    m = masks.long().view(B, H // stride, stride, W // stride, stride)
    out = torch.zeros(B, H // stride, W // stride, dtype=torch.long)
    for dy in range(stride):
        for dx in range(stride):
            out |= m[:, :, dy, :, dx]
    return out.view(B, -1)


def key_mask(masks: Tensor, stride: int, self_len: int, lens: List[List[int]], total: int) -> Tensor:
    """bool [B, P, self_len + total]: True where position p of sample b may attend to the key.  ``lens[b]``: the conditioning
    rows of sample b's prompts 0..R_b, laid out in order after the self keys; keys past them are padding."""
    pm = position_masks(masks, stride)
    B, P = pm.shape
    allow = torch.zeros(B, P, self_len + total, dtype=torch.bool)
    allow[:, :, :self_len] = True
    for b in range(B):
        off = self_len
        for k, n in enumerate(lens[b]):
            allow[b, :, off:off + n] = ((pm[b] >> k) & 1).bool()[:, None]
            off += n
    return allow


def conditioning(sd, cfg: po.PaellaConfig, prompts: List[List[Dict[str, Tensor]]]):
    """Each sample's prompts' c_embeddings concatenated along the sequence, zero-padded to the longest: ([B, S, c_cond], lens)."""
    seqs, lens = [], []
    for own in prompts:
        es = [po.c_embeddings(sd, cfg, p["byt5"], p.get("clip"), p.get("clip_image"))[0] for p in own]
        seqs.append(torch.cat(es))
        lens.append([e.shape[0] for e in es])
    S = max(s.shape[0] for s in seqs)
    return torch.stack([F.pad(s, (0, 0, 0, S - s.shape[0])) for s in seqs]), lens


def attn_block(x: Tensor, c_embed: Tensor, allow: Tensor, sd, pre: str, nhead: int) -> Tensor:
    """po.attn_block (self_attn) with a boolean key mask [B, P, P + S]."""
    B, H, W, c = x.shape
    kv = po.mm_fp32(F.silu(c_embed), sd[pre + "kv_mapper.1.weight"]) + sd[pre + "kv_mapper.1.bias"]
    xn = po.ln(x).reshape(B, H * W, c)
    kvs = torch.cat([xn, kv], dim=1)
    w_in, b_in = sd[pre + "attention.attn.in_proj_weight"], sd[pre + "attention.attn.in_proj_bias"]
    q = po.mm_fp32(xn, w_in[:c]) + b_in[:c]
    k = po.mm_fp32(kvs, w_in[c:2 * c]) + b_in[c:2 * c]
    v = po.mm_fp32(kvs, w_in[2 * c:]) + b_in[2 * c:]
    hd = c // nhead
    qh, kh, vh = (t.view(B, -1, nhead, hd).permute(0, 2, 1, 3) for t in (q, k, v))
    s = (qh @ kh.transpose(-2, -1)) / (hd ** 0.5)
    s = s.masked_fill(~allow[:, None], float("-inf"))
    o = (torch.softmax(s, dim=-1) @ vh).permute(0, 2, 1, 3).reshape(B, H * W, c)
    o = po.mm_fp32(o, sd[pre + "attention.attn.out_proj.weight"]) + sd[pre + "attention.attn.out_proj.bias"]
    return x + o.view(B, H, W, c)


def paella_forward(sd, cfg: po.PaellaConfig, x: Tensor, r: Tensor, prompts: List[List[Dict[str, Tensor]]], masks: Tensor) -> Tensor:
    """Logits [B, num_labels, H, W] of the regional forward: ``prompts[b]`` = [prompt 0, region 1, ...] as batch-1 conditioning
    dicts, ``masks`` the uint8 [B, H, W] token masks (token_masks).  A self-attending config only, like the default model."""
    if not cfg.self_attn:
        raise ValueError("regional oracle: self_attn=False is not restated")
    r_embed = po.r_embedding(r.float(), cfg.c_r)
    c_embed, lens = conditioning(sd, cfg, prompts)
    h = po.embed_tokens(x, sd, cfg)
    saved: List[Tensor] = []
    L = len(cfg.c_hidden)
    for pre, kind, lvl, c, c_skip in po.iter_blocks(cfg):
        if kind == "save":
            saved.insert(0, h)
        elif kind == "down":
            h = po.down_resample(h, sd[pre + "1.weight"], sd[pre + "1.bias"])
        elif kind == "up":
            h = po.up_resample(h, sd[pre + "1.weight"], sd[pre + "1.bias"])
        elif kind == "C":
            h = po.resblock(h, sd, pre, saved[L - 1 - lvl] if c_skip else None)
        elif kind == "T":
            h = po.timestep_block(h, r_embed, sd, pre)
        elif kind == "A":
            allow = key_mask(masks, cfg.patch_size << lvl, h.shape[1] * h.shape[2], lens, c_embed.shape[1])
            h = attn_block(h, c_embed, allow, sd, pre, cfg.nhead[lvl])
        elif kind == "F":
            h = po.feedforward_block(h, sd, pre)
        else:
            raise ValueError(kind)
    a = po.classifier_features(h, sd, cfg)
    w = sd["out_mapper.1.weight"].reshape(cfg.num_labels, cfg.c_out)
    return po.mm_fp32(a, w).permute(0, 3, 1, 2).contiguous()
