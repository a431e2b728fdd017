"""Seamless tiling in fp32/fp64 torch: the denoiser and the f4 decoder with wrap-around padding on chosen axes.

On a wrapped axis every padded read takes its coordinate modulo the grid size.  That is mod-n indexing, not
F.pad(mode='circular'), so grids smaller than the kernel (the 1x1 and 2x2 deep levels of a small latent) wrap onto
themselves.  On an unwrapped axis each layer keeps its own padding: zeros for the denoiser's depthwise convolutions and the
codec's ConvTranspose2d, replication for the codec ResBlocks' ReplicationPad2d.  Everything else is paella_oracle /
vqgan_oracle unchanged; tests/golden/tiling_tiny.npz pins both to the reference run with circular padding.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

from . import paella_oracle as po
from . import vqgan_oracle as vo

Wrap = Tuple[bool, bool]          # (wrap x, wrap y)
WRAPS = {None: (False, False), "none": (False, False), "x": (True, False), "y": (False, True), "xy": (True, True)}


def pad_axis(x: Tensor, dim: int, p: int, wrap: bool, fill: str = "zeros") -> Tensor:
    """Pad ``p`` positions on both sides of ``dim``: modulo the size when ``wrap``, else zeros or replicated edges."""
    n = x.shape[dim]
    i = torch.arange(-p, n + p, device=x.device)
    if wrap:
        return x.index_select(dim, i % n)
    if fill == "replicate":
        return x.index_select(dim, i.clamp(0, n - 1))
    shape = list(x.shape)
    shape[dim] = p
    z = x.new_zeros(shape)
    return torch.cat([z, x, z], dim)


def pad_nhwc(x: Tensor, p: int, wrap: Wrap, fill: str = "zeros") -> Tensor:
    return pad_axis(pad_axis(x, 1, p, wrap[1], fill), 2, p, wrap[0], fill)


# ------------------------------------------------------------------ denoiser
def dwconv_nhwc(x: Tensor, w: Tensor, b: Tensor, x_skip: Optional[Tensor] = None, wrap: Wrap = (False, False)) -> Tensor:
    """po.dwconv3x3_nhwc (depthwise k x k, [x, skip] channel pairs) with circular padding on the wrapped axes."""
    B, H, W, c = x.shape
    k = w.shape[-1]
    src = x if x_skip is None else torch.cat([x, x_skip], dim=-1)
    srcp = pad_nhwc(src, k // 2, wrap)
    out = torch.zeros(B, H, W, c, dtype=x.dtype, device=x.device) + b
    per = w.shape[1]
    for j in range(per):
        sj = srcp[..., torch.arange(c, device=x.device) * per + j]
        for ky in range(k):
            for kx in range(k):
                out = out + sj[:, ky:ky + H, kx:kx + W, :] * w[:, j, ky, kx]
    return out


def paella_features(sd: Dict[str, Tensor], cfg, x: Tensor, r: Tensor, byt5: Tensor, clip=None, clip_image=None,
                    attn_weights=None, mm: Callable = po.mm_fp32, wrap: Wrap = (False, False)) -> Tensor:
    """po.paella_features with every ResBlock's depthwise convolution wrapping on the axes of ``wrap``."""
    r_embed = po.r_embedding(r.float(), cfg.c_r)
    c_embed = po.c_embeddings(sd, cfg, byt5, clip, clip_image, mm)
    h = po.embed_tokens(x, sd, cfg, mm)
    saved: List[Tensor] = []
    L = len(cfg.c_hidden)
    for pre, kind, lvl, c, c_skip in po.iter_blocks(cfg):
        if kind == "save":
            saved.insert(0, h)
        elif kind == "down":
            h = po.down_resample(h, sd[pre + "1.weight"], sd[pre + "1.bias"], mm)
        elif kind == "up":
            h = po.up_resample(h, sd[pre + "1.weight"], sd[pre + "1.bias"], mm)
        elif kind == "C":
            skip = saved[L - 1 - lvl] if c_skip else None
            d = dwconv_nhwc(h, sd[pre + "depthwise.weight"], sd[pre + "depthwise.bias"], skip, wrap)
            h = h + po.mlp_grn(po.ln(d), sd, pre, mm)
        elif kind == "T":
            h = po.timestep_block(h, r_embed, sd, pre)
        elif kind == "A":
            h = po.attn_block(h, c_embed, sd, pre, cfg.nhead[lvl], cfg.self_attn, attn_weights, mm)
        elif kind == "F":
            h = po.feedforward_block(h, sd, pre, mm)
        else:
            raise ValueError(kind)
    return po.classifier_features(h, sd, cfg, mm)


def paella_forward(sd, cfg, x, r, byt5, clip=None, clip_image=None, attn_weights=None, mm: Callable = po.mm_fp32,
                   wrap: Wrap = (False, False)) -> Tensor:
    """Logits [B, num_labels, H, W] of the tiled denoiser."""
    a = paella_features(sd, cfg, x, r, byt5, clip, clip_image, attn_weights, mm, wrap)
    w = sd["out_mapper.1.weight"].reshape(cfg.num_labels, cfg.c_out)
    return mm(a, w).permute(0, 3, 1, 2).contiguous()


# ------------------------------------------------------------------ decoder
def dwconv3x3_wrap(x: Tensor, w: Tensor, b: Tensor, wrap: Wrap) -> Tensor:
    """vo.dwconv3x3_replicate with circular padding on the wrapped axes (replication on the others)."""
    B, H, W, c = x.shape
    xp = pad_nhwc(x, 1, wrap, "replicate")
    out = torch.zeros_like(x) + b
    for ky in range(3):
        for kx in range(3):
            out = out + xp[:, ky:ky + H, kx:kx + W, :] * w[:, 0, ky, kx]
    return out


def convT_k4s2p1_wrap(x: Tensor, w: Tensor, b: Tensor, wrap: Wrap, mm=vo.mm_fp32) -> Tensor:
    """vo.convT_k4s2p1 with input indices taken modulo the grid on the wrapped axes: the same as
    conv_transpose2d(F.pad(x, (1, 1, 1, 1), mode='circular'), w, b, stride=2)[..., 3:3 + 2h, 3:3 + 2w] when both wrap."""
    B, H, W, C = x.shape
    cout = w.shape[1]
    xp = pad_nhwc(x, 1, wrap)
    out = torch.zeros(B, 2 * H, 2 * W, cout, dtype=x.dtype)
    for py in range(2):
        for px in range(2):
            acc = torch.zeros(B, H, W, cout, dtype=x.dtype) + b
            for ky in range(4):
                if (py + 1 - ky) % 2:
                    continue
                oy = (py + 1 - ky) // 2
                for kx in range(4):
                    if (px + 1 - kx) % 2:
                        continue
                    ox = (px + 1 - kx) // 2
                    acc = acc + mm(xp[:, 1 + oy:1 + oy + H, 1 + ox:1 + ox + W, :], w[:, :, ky, kx].t())
            out[:, py::2, px::2, :] = acc
    return out


def vq_resblock(x: Tensor, sd, pre: str, wrap: Wrap, mm=vo.mm_fp32) -> Tensor:
    g = sd[pre + "gammas"]
    xt = vo.ln(x) * (1 + g[0]) + g[1]
    x = x + dwconv3x3_wrap(xt, sd[pre + "depthwise.1.weight"], sd[pre + "depthwise.1.bias"], wrap) * g[2]
    xt = vo.ln(x) * (1 + g[3]) + g[4]
    h = vo.gelu_erf(mm(xt, sd[pre + "channelwise.0.weight"]) + sd[pre + "channelwise.0.bias"])
    return x + (mm(h, sd[pre + "channelwise.2.weight"]) + sd[pre + "channelwise.2.bias"]) * g[5]


def decode_latents(sd, z: Tensor, n_bottleneck: int = 12, mm=vo.mm_fp32, wrap: Wrap = (False, False)) -> Tensor:
    """vo.decode_latents of the tiled decoder: NHWC latents [B,h,w,c_latent] -> [B,3,4h,4w]."""
    w = sd["up_blocks.0.0.weight"]
    x = mm(z, w.reshape(w.shape[0], -1)) + sd["up_blocks.0.0.bias"]
    j = 1
    for _ in range(n_bottleneck):
        x = vq_resblock(x, sd, f"up_blocks.{j}.", wrap, mm)
        j += 1
    x = convT_k4s2p1_wrap(x, sd[f"up_blocks.{j}.weight"], sd[f"up_blocks.{j}.bias"], wrap, mm)
    j += 1
    x = vq_resblock(x, sd, f"up_blocks.{j}.", wrap, mm)
    w = sd["out_block.0.weight"]
    x = mm(x, w.reshape(w.shape[0], -1)) + sd["out_block.0.bias"]
    return vo.pixel_shuffle2(x).permute(0, 3, 1, 2).contiguous()


def decode_indices(sd, idx: Tensor, n_bottleneck: int = 12, mm=vo.mm_fp32, wrap: Wrap = (False, False)) -> Tensor:
    return decode_latents(sd, sd["vquantizer.codebook.weight"][idx], n_bottleneck, mm, wrap)


def convT_circular_torch(x_nchw: Tensor, w: Tensor, b: Tensor) -> Tensor:
    """The restatement of the wrapped ConvTranspose2d(k4, s2, p1) through torch's own ops (both axes wrap)."""
    h, wd = x_nchw.shape[-2:]
    y = F.conv_transpose2d(F.pad(x_nchw, (1, 1, 1, 1), mode="circular"), w, b, stride=2)
    return y[..., 3:3 + 2 * h, 3:3 + 2 * wd]
