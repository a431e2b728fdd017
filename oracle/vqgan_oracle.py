"""CPU oracle for the f4 VQGAN codec and the vector quantiser.

TEST INFRASTRUCTURE ONLY (see oracle/paella_oracle.py header).

Reference lines restated (``ref`` = dome272/Paella @ e1ab72b):
  ResBlock                 ref/src/vqgan.py:6-42
  VQModel blocks           ref/src/vqgan.py:45-89
  encode / decode / decode_indices   ref/src/vqgan.py:91-107

PARITY UNPINNED for the quantiser itself: ``VectorQuantize`` lives in the
third-party package ``torchtools`` (github.com/pabloppp/pytorch-tools,
requirements.txt:12, unpinned git URL, not vendored, not installable offline).
Its published algorithm is restated here as OUR definition:
  flatten to [N,C]; dist = |c|^2 + |x|^2 - 2 x.c^T  (expanded squared L2, fp32,
  ``addmm(beta=1, alpha=-2)`` order); index = first minimum; z_q = codebook[index].
What the reference call sites pin (ref/src/vqgan.py:71,94,104, notebook cell 3):
  ``VectorQuantize(c_latent, k=codebook_size)``; ``.codebook.weight [k,C]``;
  ``forward(x, dim) -> (z_q, (vq_loss, commit_loss), indices)``;
  ``idx2vq(idx, dim)``.
The conv stacks ARE pinned against the real reference (tests/golden).
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .paella_oracle import gelu_erf, ln, mm_fp32

Tensor = torch.Tensor


# ------------------------------ vector quantiser ---------------------------
def vq_distances(x: Tensor, codebook: Tensor) -> Tensor:
    """[N,C] x [K,C] -> [N,K] expanded squared distances, fp32, fixed op order."""
    c2 = (codebook * codebook).sum(dim=1)            # [K]
    x2 = (x * x).sum(dim=1, keepdim=True)            # [N,1]
    return torch.addmm(c2[None, :] + x2, x, codebook.t(), beta=1.0, alpha=-2.0)


_C_LIB = None


def _c_oracle():
    """oracle/_ref/libvq_oracle.so (built by oracle/Makefile from vq_nearest.c), or None."""
    global _C_LIB
    if _C_LIB is None:
        import ctypes, os
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libvq_oracle.so")
        _C_LIB = ctypes.CDLL(path) if os.path.exists(path) else False
    return _C_LIB


def vq_nearest(x: Tensor, codebook: Tensor) -> Tensor:
    """First-minimum nearest code with the exact fp32 operation order of the CUDA
    kernel: dot/c2/x2 as fmaf chains over j, s = c2 + x2, d = fmaf(-2, dot, s).

    Uses the plain-C oracle (oracle/vq_nearest.c, libm ``fmaf`` = correctly rounded
    fused multiply-add) when it has been built; otherwise an fp64 emulation of the
    same chain (products of fp32 are exact in fp64; a double-rounding difference
    from a true fma needs an exact fp32 tie in the fp64 sum, ~2^-29 per op)."""
    x = x.contiguous().float()
    codebook = codebook.contiguous().float()
    lib = _c_oracle()
    if lib:
        import ctypes
        out = torch.empty(x.shape[0], dtype=torch.int64)
        lib.vq_nearest_f32(ctypes.c_void_p(x.data_ptr()), ctypes.c_int64(x.shape[0]), ctypes.c_int(x.shape[1]),
                           ctypes.c_void_p(codebook.data_ptr()), ctypes.c_int(codebook.shape[0]),
                           ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(0))
        return out
    xd, cd = x.double(), codebook.double()
    dot = torch.zeros(x.shape[0], codebook.shape[0], dtype=torch.float64)
    c2 = torch.zeros(codebook.shape[0], dtype=torch.float64)
    x2 = torch.zeros(x.shape[0], dtype=torch.float64)
    for j in range(x.shape[1]):
        dot = (dot + xd[:, j:j + 1] * cd[None, :, j]).float().double()
        c2 = (c2 + cd[:, j] * cd[:, j]).float().double()
        x2 = (x2 + xd[:, j] * xd[:, j]).float().double()
    s = (c2[None, :] + x2[:, None]).float().double()
    d = (s - 2.0 * dot).float()
    return torch.min(d, dim=1)[1]


def vq_forward(x: Tensor, codebook: Tensor, dim: int = -1):
    """``VectorQuantize.forward`` restatement -> (z_q, (vq_loss, commit_loss), indices)."""
    if dim != -1:
        x = x.movedim(dim, -1)
    shp = x.shape
    flat = x.reshape(-1, shp[-1])
    idx = vq_nearest(flat, codebook)
    zq = codebook[idx].view(shp)
    vq_loss = F.mse_loss(zq, x)
    commit = F.mse_loss(x, zq)
    idx = idx.view(shp[:-1])
    if dim != -1:
        zq = zq.movedim(-1, dim)
    return zq, (vq_loss, commit), idx


def idx2vq(idx: Tensor, codebook: Tensor, dim: int = -1) -> Tensor:
    q = codebook[idx]
    if dim != -1:
        q = q.movedim(-1, dim)
    return q


# ------------------------------ conv stacks (channels-last) -----------------
def dwconv3x3_replicate(x: Tensor, w: Tensor, b: Tensor) -> Tensor:
    """ReplicationPad2d(1) + depthwise 3x3, channels-last.  w [c,1,3,3]."""
    B, H, W, c = x.shape
    xp = F.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="replicate").permute(0, 2, 3, 1)
    out = torch.zeros_like(x) + b
    for ky in range(3):
        for kx in range(3):
            out = out + xp[:, ky:ky + H, kx:kx + W, :] * w[:, 0, ky, kx]
    return out


def vq_resblock(x: Tensor, sd, pre: str, mm=mm_fp32) -> Tensor:
    g = sd[pre + "gammas"]
    xt = ln(x) * (1 + g[0]) + g[1]
    x = x + dwconv3x3_replicate(xt, sd[pre + "depthwise.1.weight"], sd[pre + "depthwise.1.bias"]) * g[2]
    xt = ln(x) * (1 + g[3]) + g[4]
    h = gelu_erf(mm(xt, sd[pre + "channelwise.0.weight"]) + sd[pre + "channelwise.0.bias"])
    return x + (mm(h, sd[pre + "channelwise.2.weight"]) + sd[pre + "channelwise.2.bias"]) * g[5]


def pixel_unshuffle2(x: Tensor) -> Tensor:
    """NHWC PixelUnshuffle(2): out channel = c*4 + dy*2 + dx."""
    B, H, W, C = x.shape
    return x.view(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(B, H // 2, W // 2, C * 4)


def pixel_shuffle2(x: Tensor) -> Tensor:
    B, h, w, C4 = x.shape
    C = C4 // 4
    return x.view(B, h, w, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(B, 2 * h, 2 * w, C)


def conv_k4s2p1(x: Tensor, w: Tensor, b: Tensor, mm=mm_fp32) -> Tensor:
    """Conv2d(k=4,s=2,p=1) channels-last as 16 shifted GEMMs.  w [Cout,Cin,4,4]."""
    B, H, W, C = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    out = torch.zeros(B, H // 2, W // 2, w.shape[0], dtype=x.dtype) + b
    for ky in range(4):
        for kx in range(4):
            out = out + mm(xp[:, ky:ky + H:2, kx:kx + W:2, :], w[:, :, ky, kx])
    return out


def convT_k4s2p1(x: Tensor, w: Tensor, b: Tensor, mm=mm_fp32) -> Tensor:
    """ConvTranspose2d(k=4,s=2,p=1) channels-last as 4 sub-pixel phases of 2x2 taps.
    w [Cin,Cout,4,4].  out[2y+py, 2x+px] = sum over (ky,kx) with matching parity of
    in[(2y+py+1-ky)/2, (2x+px+1-kx)/2] . w[:,:,ky,kx]."""
    B, H, W, C = x.shape
    cout = w.shape[1]
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    out = torch.zeros(B, 2 * H, 2 * W, cout, dtype=x.dtype)
    for py in range(2):
        for px in range(2):
            acc = torch.zeros(B, H, W, cout, dtype=x.dtype) + b
            for ky in range(4):
                if (py + 1 - ky) % 2:
                    continue
                oy = (py + 1 - ky) // 2          # input row = y + oy
                for kx in range(4):
                    if (px + 1 - kx) % 2:
                        continue
                    ox = (px + 1 - kx) // 2
                    acc = acc + mm(xp[:, 1 + oy:1 + oy + H, 1 + ox:1 + ox + W, :], w[:, :, ky, kx].t())
            out[:, py::2, px::2, :] = acc
    return out


def encode_latents(sd: Dict[str, Tensor], img: Tensor, mm=mm_fp32) -> Tensor:
    """in_block + down_blocks: [B,3,H,W] -> pre-quantisation latents [B,h,w,4] (NHWC)."""
    x = pixel_unshuffle2(img.permute(0, 2, 3, 1))
    x = mm(x, sd["in_block.1.weight"].reshape(sd["in_block.1.weight"].shape[0], -1)) + sd["in_block.1.bias"]
    x = vq_resblock(x, sd, "down_blocks.0.", mm)
    x = conv_k4s2p1(x, sd["down_blocks.1.weight"], sd["down_blocks.1.bias"], mm)
    x = vq_resblock(x, sd, "down_blocks.2.", mm)
    w = sd["down_blocks.3.0.weight"]
    x = mm(x, w.reshape(w.shape[0], -1))
    bn = "down_blocks.3.1."
    scale = sd[bn + "weight"] / torch.sqrt(sd[bn + "running_var"] + 1e-5)
    return (x - sd[bn + "running_mean"]) * scale + sd[bn + "bias"]


def encode(sd, img: Tensor, scale_factor: float = 0.3764, mm=mm_fp32):
    """ref/src/vqgan.py:91-95 -> (qe/sf, x/sf, indices, loss); NCHW outputs like the reference."""
    z = encode_latents(sd, img, mm)
    zq, (vl, cl), idx = vq_forward(z, sd["vquantizer.codebook.weight"], dim=-1)
    return (zq.permute(0, 3, 1, 2) / scale_factor, z.permute(0, 3, 1, 2) / scale_factor, idx, vl + cl * 0.25)


def decode_latents(sd, z: Tensor, n_bottleneck: int = 12, mm=mm_fp32) -> Tensor:
    """up_blocks + out_block on NHWC latents [B,h,w,4] -> [B,3,4h,4w]."""
    w = sd["up_blocks.0.0.weight"]
    x = mm(z, w.reshape(w.shape[0], -1)) + sd["up_blocks.0.0.bias"]
    j = 1
    for _ in range(n_bottleneck):
        x = vq_resblock(x, sd, f"up_blocks.{j}.", mm)
        j += 1
    x = convT_k4s2p1(x, sd[f"up_blocks.{j}.weight"], sd[f"up_blocks.{j}.bias"], mm)
    j += 1
    x = vq_resblock(x, sd, f"up_blocks.{j}.", mm)
    w = sd["out_block.0.weight"]
    x = mm(x, w.reshape(w.shape[0], -1)) + sd["out_block.0.bias"]
    return pixel_shuffle2(x).permute(0, 3, 1, 2).contiguous()


def decode(sd, z_nchw: Tensor, scale_factor: float = 0.3764, mm=mm_fp32) -> Tensor:
    return decode_latents(sd, (z_nchw * scale_factor).permute(0, 2, 3, 1), mm=mm)


def decode_indices(sd, idx: Tensor, mm=mm_fp32) -> Tensor:
    return decode_latents(sd, sd["vquantizer.codebook.weight"][idx], mm=mm)
