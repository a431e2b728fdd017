"""Python mirror of the reference denoiser's class surface (ref/src/modules.py, ref/utils/modules.py).

Same class names, constructor kwargs, attribute names and state-dict keys as the reference, so
``load_state_dict(paella_v3.pt)`` and ``paella_inference.ipynb`` work unchanged — but ``forward`` runs the
hand-written sm_90a kernels behind the C ABI (include/paella_b200.h).  The ``torch.nn`` layers created
here are PARAMETER HOLDERS ONLY (they give the reference's key names and initialisation); none of their
``forward`` methods is ever called, and there is no PyTorch or CPU fallback.
"""
from __future__ import annotations

import ctypes
import math
import os
from collections import namedtuple
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
from torch import nn

from . import _lib, ops
from ._lib import PaellaB200Error, check, current_stream, lib, ptr


# ------------------------------------------------------------------------------------------------
# Building blocks — parameter layout AND stand-alone forward of ref/src/modules.py:7-106.
# Inside a Paella the blocks are executed by the fused plan in csrc/paella_model.cu; called on their own
# they compose the same kernels through the block-level C ABI (include/paella_b200.h).  Inference
# semantics (Dropout = identity), fp16 GEMM operands / fp32 accumulation like the model path.
# ------------------------------------------------------------------------------------------------
def _cached(mod: nn.Module, key: str, src: torch.Tensor, make):
    """Derived copy (fp16 cast / repack) of a parameter, rebuilt when the parameter changes."""
    cache = mod.__dict__.setdefault("_pb200_cache", {})
    tag = (src.data_ptr(), src._version, str(src.device))
    hit = cache.get(key)
    if hit is None or hit[0] != tag:
        with torch.no_grad():
            hit = (tag, make(src.detach()))
        cache[key] = hit
    return hit[1]


def _w16(mod, key, w):
    return _cached(mod, key, w, lambda t: t.reshape(t.shape[0], -1).to(torch.float16).contiguous())


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().float().contiguous()


def _to_rows(x: torch.Tensor) -> torch.Tensor:
    """NCHW fp32 -> channels-last rows [B*H*W, C] (a fresh buffer the block may update in place)."""
    if x.dim() != 4:
        raise PaellaB200Error(f"expected an NCHW tensor, got shape {tuple(x.shape)}")
    x = _f32(x)
    B, C, H, W = x.shape
    out = torch.empty(B * H * W, C, dtype=torch.float32, device=x.device)
    check(lib().pb200_nchw_to_nhwc(ptr(x), B, C, H * W, ptr(out), current_stream()), "pb200_nchw_to_nhwc")
    return out


def _to_nchw(rows: torch.Tensor, shape) -> torch.Tensor:
    B, C, H, W = shape
    out = torch.empty(B, C, H, W, dtype=torch.float32, device=rows.device)
    check(lib().pb200_nhwc_to_nchw(ptr(rows), B, C, H * W, ptr(out), current_stream()), "pb200_nhwc_to_nchw")
    return out


def _cast16(x: torch.Tensor, silu: bool = False) -> torch.Tensor:
    x = _f32(x)
    out = torch.empty(x.shape, dtype=torch.float16, device=x.device)
    check(lib().pb200_cast_f16(ptr(x), x.numel(), int(silu), ptr(out), current_stream()), "pb200_cast_f16")
    return out


def _layernorm(rows: torch.Tensor, ln: nn.LayerNorm, half: bool) -> torch.Tensor:
    M, C = rows.shape
    if tuple(ln.normalized_shape) != (C,):
        raise PaellaB200Error(f"LayerNorm over {tuple(ln.normalized_shape)} applied to {C} channels")
    out = torch.empty(M, C, dtype=torch.float16 if half else torch.float32, device=rows.device)
    w = _f32(ln.weight) if ln.weight is not None else None
    b = _f32(ln.bias) if ln.bias is not None else None
    check(lib().pb200_layernorm(ptr(rows), M, C, float(ln.eps), ptr(w), ptr(b), None if half else ptr(out),
                                ptr(out) if half else None, current_stream()), "pb200_layernorm")
    return out


def _mlp_rows(mlp: nn.Sequential, a16: torch.Tensor, resid_rows: torch.Tensor, batch: int) -> torch.Tensor:
    """channelwise = Linear -> GELU -> GRN -> Dropout(eval) -> Linear, added onto resid_rows in place."""
    lin1, grn, lin2 = mlp[0], mlp[2], mlp[4]
    M, c = a16.shape
    n = lin1.out_features
    P = M // batch
    h16 = torch.empty(M, n, dtype=torch.float16, device=a16.device)
    sq = torch.zeros(2, batch, n, dtype=torch.int64, device=a16.device)
    ops.gemm_f16(a16, _w16(lin1, "w16", lin1.weight), _lib.EPI_GELU_F16, h16, bias=_f32(lin1.bias), sqsum=sq[0], rows_per_sample=P)
    mult = torch.empty(batch, n, dtype=torch.float32, device=a16.device)
    check(lib().pb200_grn_f16(ptr(h16), batch, P, n, ptr(sq[0]), ptr(sq[1]), n, ptr(_f32(grn.gamma).view(-1)),
                              ptr(_f32(grn.beta).view(-1)), ptr(mult), current_stream()), "pb200_grn_f16")
    ops.gemm_f16(h16, _w16(lin2, "w16", lin2.weight), _lib.EPI_RESID_F32, resid_rows, bias=_f32(lin2.bias), resid=resid_rows)
    return resid_rows


class Attention2D(nn.Module):
    """ref/src/modules.py:7-19.  ``attn`` holds in_proj_weight/bias and out_proj.* under the reference's keys."""

    def __init__(self, c, nhead, dropout=0.0):
        super().__init__()
        self.attn = torch.nn.MultiheadAttention(c, nhead, dropout=dropout, bias=True, batch_first=True)

    def _core(self, xq16: torch.Tensor, kv16: torch.Tensor, batch: int, self_attn: bool, attn_weights=None) -> torch.Tensor:
        """in-projection + attention core: xq16 [B*P, E] queries (and self keys), kv16 [B*S, E] -> fp16 [B*P, E]."""
        mha = self.attn
        E = mha.embed_dim
        M = xq16.shape[0]
        P = M // batch
        S = kv16.shape[0] // batch if kv16 is not None else 0
        w16 = _w16(mha, "in16", mha.in_proj_weight)
        b32 = _f32(mha.in_proj_bias)
        qkv = torch.empty(M, 3 * E, dtype=torch.float16, device=xq16.device)
        ops.gemm_f16(xq16, w16, _lib.EPI_F16, qkv, bias=b32)
        ckv = None
        if S > 0:
            ckv = torch.empty(batch * S, 2 * E, dtype=torch.float16, device=xq16.device)
            ops.gemm_f16(kv16, w16[E:], _lib.EPI_F16, ckv, bias=b32[E:])
        aw, n_w = None, 0
        if attn_weights is not None:
            aw = _f32(attn_weights).reshape(-1)
            n_w = aw.numel()
        out = torch.empty(M, E, dtype=torch.float16, device=xq16.device)
        check(lib().pb200_attention(ptr(qkv), ptr(ckv), None, ptr(out), batch, P, S, E, mha.num_heads, int(bool(self_attn)),
                                    ptr(aw), n_w, batch, current_stream()), "pb200_attention")
        return out

    def forward(self, x, kv, self_attn=False, **kwargs):
        B, C = x.shape[0], x.shape[1]
        rows16 = _cast16(_to_rows(x))
        kv16 = _cast16(kv).view(-1, C) if kv is not None and kv.numel() > 0 else None
        o16 = self._core(rows16, kv16, B, self_attn, kwargs.get("attn_weights"))
        out = torch.empty(rows16.shape[0], C, dtype=torch.float32, device=x.device)
        ops.gemm_f16(o16, _w16(self.attn, "out16", self.attn.out_proj.weight), _lib.EPI_F32, out, bias=_f32(self.attn.out_proj.bias))
        return _to_nchw(out, x.shape)


class LayerNorm2d(nn.LayerNorm):
    """ref/src/modules.py:22-27 (no parameters when elementwise_affine=False)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)

    def forward(self, x):
        return _to_nchw(_layernorm(_to_rows(x), self, half=False), x.shape)


class GlobalResponseNorm(nn.Module):
    """ref/src/modules.py:30-40 (input NHWC ``[B, H, W, dim]``)."""

    def __init__(self, dim):
        super().__init__()
        self.gamma = nn.Parameter(torch.zeros(1, 1, 1, dim))
        self.beta = nn.Parameter(torch.zeros(1, 1, 1, dim))

    def forward(self, x):
        if x.dim() != 4 or x.shape[-1] != self.gamma.shape[-1]:
            raise PaellaB200Error(f"GlobalResponseNorm({self.gamma.shape[-1]}) got shape {tuple(x.shape)}")
        x = _f32(x)
        B, H, W, N = x.shape
        out = torch.empty_like(x)
        stat = torch.empty(B, N, dtype=torch.float32, device=x.device)
        check(lib().pb200_grn_f32(ptr(x), B, H * W, N, ptr(_f32(self.gamma).view(-1)), ptr(_f32(self.beta).view(-1)), ptr(stat),
                                  ptr(out), current_stream()), "pb200_grn_f32")
        return out


def _mlp_holder(c, dropout):
    return nn.Sequential(nn.Linear(c, c * 4), nn.GELU(), GlobalResponseNorm(c * 4), nn.Dropout(dropout), nn.Linear(c * 4, c))


class ResBlock(nn.Module):
    """ref/src/modules.py:43-62."""

    def __init__(self, c, c_skip=None, kernel_size=3, dropout=0.0):
        super().__init__()
        c_skip = c_skip or 0
        self.depthwise = nn.Conv2d(c + c_skip, c, kernel_size=kernel_size, padding=kernel_size // 2, groups=c)
        self.norm = LayerNorm2d(c, elementwise_affine=False, eps=1e-6)
        self.channelwise = _mlp_holder(c, dropout)

    def forward(self, x, x_skip=None):
        dw = self.depthwise
        c, per, k = dw.out_channels, dw.in_channels // dw.out_channels, dw.kernel_size[0]
        if per not in (1, 2) or dw.in_channels != per * c or (x_skip is not None) != (per == 2):
            raise PaellaB200Error("ResBlock: c_skip must be 0 (no x_skip) or c (with x_skip)")
        if self.norm.elementwise_affine or self.norm.eps != 1e-6:
            raise PaellaB200Error("ResBlock: the fused depthwise+LayerNorm kernel is eps=1e-6 without affine (the reference's setting)")
        B, _, H, W = x.shape
        rows = _to_rows(x)
        skip = _to_rows(x_skip) if x_skip is not None else None
        # [c, per, k, k] -> [k*k][per][c]; with a skip the conv input is cat[x, x_skip], group g reads channels 2g, 2g+1
        wp = _cached(dw, "wp", dw.weight, lambda t: t.float().permute(2, 3, 1, 0).reshape(k * k, per, c).contiguous())
        a16 = torch.empty(B * H * W, c, dtype=torch.float16, device=x.device)
        check(lib().pb200_dwconv_ln(ptr(rows), ptr(skip), ptr(wp), ptr(_f32(dw.bias)), B, H, W, c, k, ptr(a16), current_stream()),
              "pb200_dwconv_ln")
        return _to_nchw(_mlp_rows(self.channelwise, a16, rows, B), x.shape)


class AttnBlock(nn.Module):
    """ref/src/modules.py:65-79 (``attn_weights=`` as in ref/utils/modules.py:76-78)."""

    def __init__(self, c, c_cond, nhead, self_attn=True, dropout=0.0):
        super().__init__()
        self.self_attn = self_attn
        self.norm = LayerNorm2d(c, elementwise_affine=False, eps=1e-6)
        self.attention = Attention2D(c, nhead, dropout)
        self.kv_mapper = nn.Sequential(nn.SiLU(), nn.Linear(c_cond, c))

    def forward(self, x, kv, **kwargs):
        B, C = x.shape[0], x.shape[1]
        rows = _to_rows(x)
        xn16 = _layernorm(rows, self.norm, half=True)
        lin = self.kv_mapper[1]
        kv16 = None
        if kv is not None and kv.numel() > 0:
            s16 = _cast16(kv, silu=True).view(-1, lin.in_features)
            kv16 = torch.empty(s16.shape[0], C, dtype=torch.float16, device=x.device)
            ops.gemm_f16(s16, _w16(lin, "w16", lin.weight), _lib.EPI_F16, kv16, bias=_f32(lin.bias))
        o16 = self.attention._core(xn16, kv16, B, self.self_attn, kwargs.get("attn_weights"))
        mha = self.attention.attn
        ops.gemm_f16(o16, _w16(mha, "out16", mha.out_proj.weight), _lib.EPI_RESID_F32, rows, bias=_f32(mha.out_proj.bias), resid=rows)
        return _to_nchw(rows, x.shape)


class FeedForwardBlock(nn.Module):
    """ref/src/modules.py:82-96."""

    def __init__(self, c, dropout=0.0):
        super().__init__()
        self.norm = LayerNorm2d(c, elementwise_affine=False, eps=1e-6)
        self.channelwise = _mlp_holder(c, dropout)

    def forward(self, x):
        rows = _to_rows(x)
        return _to_nchw(_mlp_rows(self.channelwise, _layernorm(rows, self.norm, half=True), rows, x.shape[0]), x.shape)


class TimestepBlock(nn.Module):
    """ref/src/modules.py:99-106."""

    def __init__(self, c, c_timestep):
        super().__init__()
        self.mapper = nn.Linear(c_timestep, c * 2)

    def forward(self, x, t):
        B, C, H, W = x.shape
        film = torch.empty(B, 2 * C, dtype=torch.float32, device=x.device)
        ops.gemm_f16(_cast16(t).view(B, -1), _w16(self.mapper, "w16", self.mapper.weight), _lib.EPI_F32, film, bias=_f32(self.mapper.bias))
        rows = _to_rows(x)
        check(lib().pb200_film_apply(ptr(rows), B * H * W, C, H * W, ptr(film), 2 * C, 0, current_stream()), "pb200_film_apply")
        return _to_nchw(rows, x.shape)


# ------------------------------------------------------------------------------------------------
# Paella.token_scores: fp32 [B, H, W] negative log-likelihood and label-smoothed loss, int64 [B, H, W] arg-max code
TokenScores = namedtuple("TokenScores", ["nll", "loss", "argmax"])


class ConditioningCache:
    """x- and t-independent conditioning work of one sample() call: c_embed and every AttnBlock's
    cond K/V for ``batch_total`` samples (conditional rows first, then unconditional rows)."""

    def __init__(self, cache: torch.Tensor, batch_total: int, s_max: int, slots: Optional[int] = None,
                 slot_map: Optional[torch.Tensor] = None, extra_slot: int = 0):
        self.cache, self.batch_total, self.s_max = cache, batch_total, s_max
        # a group whose samples all carry the same conditioning (the unconditional half of a CFG batch) occupies ONE
        # slot of the cache; slot_map (int32 [batch_total], None = identity) names the slot each sample attends to
        self.slots = batch_total if slots is None else slots
        self.slot_map = slot_map
        # regional prompts (prepare_conditioning's ``extra``) occupy slots [extra_slot, slots), in the order given
        self.extra_slot = extra_slot


class Paella(nn.Module):
    """Drop-in for ``Paella`` (ref/src/modules.py:109-283, notebook variant ref/utils/modules.py)."""

    def __init__(self, c_in=256, c_out=256, num_labels=8192, c_r=64, patch_size=2, c_cond=1024,
                 c_hidden=[640, 1280, 1280], nhead=[-1, 16, 16], blocks=[6, 16, 6], level_config=['CT', 'CTA', 'CTA'],
                 clip_embd=1024, byt5_embd=1536, clip_seq_len=4, kernel_size=3, dropout=0.1, self_attn=True):
        super().__init__()
        self.c_r, self.c_cond, self.num_labels = c_r, c_cond, num_labels
        self._cfg = dict(c_in=c_in, c_out=c_out, num_labels=num_labels, c_r=c_r, patch_size=patch_size, c_cond=c_cond,
                         c_hidden=list(c_hidden), nhead=list(nhead), blocks=list(blocks), level_config=list(level_config),
                         clip_embd=clip_embd, byt5_embd=byt5_embd, clip_seq_len=clip_seq_len, kernel_size=kernel_size,
                         self_attn=bool(self_attn))
        if not isinstance(dropout, list):
            dropout = [dropout] * len(c_hidden)

        self.byt5_mapper = nn.Linear(byt5_embd, c_cond)
        self.clip_mapper = nn.Linear(clip_embd, c_cond * clip_seq_len)
        self.clip_image_mapper = nn.Linear(clip_embd, c_cond * clip_seq_len)
        self.seq_norm = nn.LayerNorm(c_cond, elementwise_affine=False, eps=1e-6)
        self.in_mapper = nn.Sequential(nn.Embedding(num_labels, c_in), nn.LayerNorm(c_in, elementwise_affine=False, eps=1e-6))
        self.embedding = nn.Sequential(nn.PixelUnshuffle(patch_size),
                                       nn.Conv2d(c_in * (patch_size ** 2), c_hidden[0], kernel_size=1),
                                       LayerNorm2d(c_hidden[0], elementwise_affine=False, eps=1e-6))

        def make(kind, lvl, c_skip=0):
            c = c_hidden[lvl]
            if kind == 'C':
                return ResBlock(c, c_skip, kernel_size=kernel_size, dropout=dropout[lvl])
            if kind == 'A':
                return AttnBlock(c, c_cond, nhead[lvl], self_attn=self_attn, dropout=dropout[lvl])
            if kind == 'F':
                return FeedForwardBlock(c, dropout=dropout[lvl])
            if kind == 'T':
                return TimestepBlock(c, c_r)
            raise Exception(f'Block type {kind} not supported')

        n = len(c_hidden)
        self.down_blocks = nn.ModuleList()
        for i in range(n):
            level = nn.ModuleList()
            if i > 0:
                level.append(nn.Sequential(LayerNorm2d(c_hidden[i - 1], elementwise_affine=False, eps=1e-6),
                                           nn.Conv2d(c_hidden[i - 1], c_hidden[i], kernel_size=2, stride=2)))
            for _ in range(blocks[i]):
                for kind in level_config[i]:
                    level.append(make(kind, i))
            self.down_blocks.append(level)
        self.up_blocks = nn.ModuleList()
        for i in reversed(range(n)):
            level = nn.ModuleList()
            for j in range(blocks[i]):
                for k, kind in enumerate(level_config[i]):
                    level.append(make(kind, i, c_skip=c_hidden[i] if i < n - 1 and j == k == 0 else 0))
            if i > 0:
                level.append(nn.Sequential(LayerNorm2d(c_hidden[i], elementwise_affine=False, eps=1e-6),
                                           nn.ConvTranspose2d(c_hidden[i], c_hidden[i - 1], kernel_size=2, stride=2)))
            self.up_blocks.append(level)
        self.clf = nn.Sequential(LayerNorm2d(c_hidden[0], elementwise_affine=False, eps=1e-6),
                                 nn.Conv2d(c_hidden[0], c_out * (patch_size ** 2), kernel_size=1),
                                 nn.PixelShuffle(patch_size))
        self.out_mapper = nn.Sequential(LayerNorm2d(c_out, elementwise_affine=False, eps=1e-6),
                                        nn.Conv2d(c_out, num_labels, kernel_size=1, bias=False))
        self._reference_init(blocks, num_labels)

        self._handle = None
        self._blob = None
        self._packed_key = None
        self._workspace = None
        self._cond_single = None
        self._batch_invariant = False

    @property
    def batch_invariant(self) -> bool:
        """Batch-invariant forward (default False).  True: every sample's features, logits and tokens are bit-identical
        whatever batch, batch position, CFG pairing or GPU count it runs in -- on any model and latent grid, so every
        "bit for bit" statement of utils.sample*, SamplingEngine and sample_distributed's shards holds on the default model
        too.  It changes how the folded LayerNorm's row statistics are summed (DESIGN.md §3 Numerics), so the results
        differ in the last bits from the default mode.  Set it between calls, not while forwards of this model are being
        enqueued from another thread; TypeError for a non-bool."""
        return self._batch_invariant

    @batch_invariant.setter
    def batch_invariant(self, on: bool) -> None:
        if not isinstance(on, bool):
            raise TypeError(f"batch_invariant must be a bool (got {type(on).__name__})")
        if self._handle is not None:
            check(lib().pb200_paella_set_batch_invariant(self._handle, int(on)), "pb200_paella_set_batch_invariant")
        self._batch_invariant = on

    # -------------------------------------------------------------- initialisation (ref/src/modules.py:189-210)
    def _reference_init(self, blocks, num_labels):
        for mod in self.modules():
            if isinstance(mod, (nn.Conv2d, nn.Linear)):
                nn.init.xavier_uniform_(mod.weight)
                if mod.bias is not None:
                    nn.init.constant_(mod.bias, 0)
        for lin in (self.byt5_mapper, self.clip_mapper, self.clip_image_mapper):
            nn.init.normal_(lin.weight, std=0.02)
        nn.init.xavier_uniform_(self.embedding[1].weight, 0.02)
        nn.init.constant_(self.clf[1].weight, 0)
        nn.init.normal_(self.in_mapper[0].weight, std=np.sqrt(1 / num_labels))
        self.out_mapper[-1].weight.data = self.in_mapper[0].weight.data[:, :, None, None].clone()
        scale = np.sqrt(1 / sum(blocks))
        for level in list(self.down_blocks) + list(self.up_blocks):
            for blk in level:
                if isinstance(blk, (ResBlock, FeedForwardBlock)):
                    blk.channelwise[-1].weight.data *= scale
                elif isinstance(blk, TimestepBlock):
                    nn.init.constant_(blk.mapper.weight, 0)

    # -------------------------------------------------------------- native handle + packed weights
    def __del__(self):
        try:
            if getattr(self, "_handle", None):
                lib().pb200_paella_destroy(self._handle)
        except Exception:
            pass

    def _device(self):
        po = getattr(self, "_packed_only", None)
        return po if po is not None else self.in_mapper[0].weight.device

    def _weights_key(self):
        return (str(self._device()),) + tuple((p.data_ptr(), p._version) for p in self.parameters())

    def pack_weights(self, broadcast_src: Optional[int] = None):
        """Convert the reference-layout fp32 parameters into the library's packed blob (fp16 GEMM weights,
        repacked conv kernels, concatenated FiLM mappers).  With ``broadcast_src`` set and
        ``torch.distributed`` initialised, only that rank converts; the blob is then NCCL-broadcast —
        the single collective of a multi-GPU run (no collective inside the step loop)."""
        dev = self._device()
        if dev.type != "cuda":
            raise PaellaB200Error("Paella runs on CUDA only: move the model with .to('cuda') (no CPU fallback)")
        L = lib()
        if self._handle is None:
            c = self._cfg
            cfg = _lib.PaellaConfig()
            for k in ("c_in", "c_out", "num_labels", "c_r", "patch_size", "c_cond", "clip_embd", "byt5_embd",
                      "clip_seq_len", "kernel_size"):
                setattr(cfg, k, int(c[k]))
            cfg.self_attn = int(c["self_attn"])
            cfg.n_levels = len(c["c_hidden"])
            if cfg.n_levels > _lib.PB200_MAX_LEVELS:
                raise PaellaB200Error("too many levels")
            for i in range(cfg.n_levels):
                cfg.c_hidden[i], cfg.nhead[i], cfg.blocks[i] = c["c_hidden"][i], c["nhead"][i], c["blocks"][i]
                cfg.level_config[i].value = c["level_config"][i].encode()
            h = ctypes.c_void_p()
            check(L.pb200_paella_create(ctypes.byref(cfg), ctypes.byref(h)), "pb200_paella_create")
            self._handle = h
            check(L.pb200_paella_set_batch_invariant(h, int(self._batch_invariant)), "pb200_paella_set_batch_invariant")
        with torch.cuda.device(dev):
            nbytes = L.pb200_paella_weight_bytes(self._handle)
            if self._blob is None or self._blob.numel() != nbytes or self._blob.device != dev:
                self._blob = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
                self._workspace = None
            check(L.pb200_paella_bind_weights(self._handle, ptr(self._blob)), "pb200_paella_bind_weights")
            import torch.distributed as dist
            distributed = broadcast_src is not None and dist.is_available() and dist.is_initialized()
            if not distributed or dist.get_rank() == broadcast_src:
                sd = self.state_dict()
                for i in range(L.pb200_paella_num_params(self._handle)):
                    name = L.pb200_paella_param_name(self._handle, i)
                    t = sd[name.decode()].detach().to(dtype=torch.float32).contiguous()
                    check(L.pb200_paella_load_param(self._handle, name, ptr(t), t.numel(), current_stream()),
                          f"pb200_paella_load_param({name.decode()})")
                torch.cuda.current_stream().synchronize()     # temporaries from .float() must outlive the copies
            if distributed:
                from .parallel import broadcast_blob
                broadcast_blob(self._blob, src=broadcast_src)      # + checksum agreement across ranks (raises on mismatch)
        self._packed_key = self._weights_key()
        self._cond_single = None
        return self

    def _ensure_packed(self):
        if getattr(self, "_packed_only", None) is not None:
            return          # from_packed(): the blob IS the model; the nn parameters are meta placeholders
        if self._handle is None or self._packed_key != self._weights_key():
            self.pack_weights()

    def _apply(self, fn, *a, **k):      # .to()/.cuda()/.half(): repack lazily
        if getattr(self, "_packed_only", None) is not None:
            return self     # a packed-only model lives where from_packed() put it
        self._packed_key = None
        return super()._apply(fn, *a, **k)

    # -------------------------------------------------------------- on-disk packed form (SURVEY.md §8 f3)
    def save_packed(self, path: str):
        """Write the library's packed weight blob (fp16 GEMM weights, repacked conv kernels, fused FiLM table, derived
        row sums) + the constructor config to ``path``: what ``tools/pack_checkpoint.py`` produces from ``paella_v3.pt``
        (nb:178-180).  ``Paella.from_packed`` memory-maps nothing and converts nothing: one H2D copy of 2.0 GB instead of
        materialising 4.0 GB of fp32 parameters and running the pack kernels."""
        from .packed import save_blob
        self._ensure_packed()
        save_blob(path, "paella", dict(self._cfg, dropout=0.0), self._blob)

    @classmethod
    def from_packed(cls, path: str, device="cuda"):
        from .packed import load_blob
        cfg, blob = load_blob(path, "paella", device)
        with torch.device("meta"):
            m = cls(**cfg)
        m.eval().requires_grad_(False)
        L = lib()
        m._packed_only = torch.device(device) if not isinstance(device, torch.device) else device
        if m._packed_only.index is None:
            m._packed_only = torch.device("cuda", torch.cuda.current_device())
        c = m._cfg
        ccfg = _lib.PaellaConfig()
        for k in ("c_in", "c_out", "num_labels", "c_r", "patch_size", "c_cond", "clip_embd", "byt5_embd", "clip_seq_len", "kernel_size"):
            setattr(ccfg, k, int(c[k]))
        ccfg.self_attn = int(c["self_attn"])
        ccfg.n_levels = len(c["c_hidden"])
        for i in range(ccfg.n_levels):
            ccfg.c_hidden[i], ccfg.nhead[i], ccfg.blocks[i] = c["c_hidden"][i], c["nhead"][i], c["blocks"][i]
            ccfg.level_config[i].value = c["level_config"][i].encode()
        h = ctypes.c_void_p()
        check(L.pb200_paella_create(ctypes.byref(ccfg), ctypes.byref(h)), "pb200_paella_create")
        m._handle = h
        if L.pb200_paella_weight_bytes(h) != blob.numel():
            raise PaellaB200Error(f"{path}: packed blob has {blob.numel()} bytes, this build's plan needs {L.pb200_paella_weight_bytes(h)} "
                                  "(packed with a different library version or config)")
        m._blob = blob
        with torch.cuda.device(blob.device):
            check(L.pb200_paella_bind_weights(h, ptr(blob)), "pb200_paella_bind_weights")
        return m

    def _ws(self, nbytes: int) -> torch.Tensor:
        """Scratch for the launches of ONE stream (the library bump-allocates it identically on every call): one buffer per
        CUDA stream the model is driven from, so calls issued on different streams never share scratch."""
        if not isinstance(self._workspace, dict):
            self._workspace = {}
        key = torch.cuda.current_stream(self._device()).cuda_stream
        ws = self._workspace.get(key)
        if ws is None or ws.numel() < nbytes or ws.device != self._device():
            ws = torch.empty(nbytes, dtype=torch.uint8, device=self._device())
            self._workspace[key] = ws
        return ws

    # -------------------------------------------------------------- conditioning
    def prepare_conditioning(self, groups: Sequence[Dict[str, torch.Tensor]], latent_hw=(32, 32),
                             share_uniform: bool = True, extra: Sequence[Dict[str, torch.Tensor]] = (),
                             tail: Sequence[int] = (), lora=None, extra_lora=None, pag_tail: Sequence[int] = ()) -> ConditioningCache:
        """gen_c_embeddings (ref/src/modules.py:223-232) + every AttnBlock's kv_mapper and K/V projection of the
        conditioning rows, for the concatenation of ``groups`` (e.g. [conditional, unconditional]).  A group whose
        samples all carry the same tensors (the usual unconditional group) is projected once and shared.  ``extra``: batch-1
        conditioning dicts (regional and guidance prompts) projected into slots of their own after the groups'
        (cache.extra_slot on), consecutive ones of one sequence layout in one projection.  ``tail``: indices into ``extra``; the
        cache then has len(tail) more samples after the groups', sample k of them attending to extra prompt tail[k] (the term
        rows of features' ``tail_src``).  No other sample's slot_map entry names an extra slot.  ``pag_tail``: samples of the groups;
        the cache then has len(pag_tail) more samples after those, sample k of them attending to sample pag_tail[k]'s own slot (the
        perturbed rows of perturbed-attention guidance).
        ``lora``: None, or per group None or a list of its samples' LoRA entries (ops.lora_entries: None or (adapter, scale)), and
        ``extra_lora``: None or one entry per ``extra`` prompt: each slot is projected under its entry's adapter
        (pb200_paella_prepare_cond_lora), and a group is shared only when its samples also agree on the entry."""
        self._ensure_packed()
        L = lib()
        dev = self._device()
        seq = self._cfg["clip_seq_len"]
        glora = list(lora) if lora is not None else [None] * len(groups)
        xlora = list(extra_lora) if extra_lora is not None else [None] * len(extra)

        def seqlen(g):
            n = (1 if g.get("clip") is not None else 0)
            ci = g.get("clip_image")
            if ci is not None:
                n += len(ci) if isinstance(ci, (list, tuple)) else 1
            return g["byt5"].shape[1] + seq * n
        s_max = max(seqlen(g) for g in list(groups) + list(extra))
        bt = sum(g["byt5"].shape[0] for g in groups)

        def uniform(g):
            """All samples of the group carry identical conditioning (one host sync per tensor, once per sample() call)."""
            if not share_uniform or g["byt5"].shape[0] < 2:
                return False
            ts = [g["byt5"], g.get("clip")]
            ci = g.get("clip_image")
            ts += list(ci) if isinstance(ci, (list, tuple)) else [ci]
            return all(bool((t == t[:1]).all()) for t in ts if t is not None)
        shared = [uniform(g) and (ent is None or all(e == ent[0] for e in ent)) for g, ent in zip(groups, glora)]
        slots = sum(1 if sh else g["byt5"].shape[0] for g, sh in zip(groups, shared))
        extra_slot = slots
        if extra:
            from .engine import cond_layout
            runs, run_lora = [], []      # consecutive extra prompts of one layout: one projection, as groups of batch > 1
            for g, e in zip(extra, xlora):
                if runs and cond_layout(g) == cond_layout(runs[-1][0]):
                    runs[-1].append(g)
                    run_lora[-1].append(e)
                else:
                    runs.append([g])
                    run_lora.append([e])
            glora += [ent if any(e is not None for e in ent) else None for ent in run_lora]
            for run in runs:
                ci = run[0].get("clip_image")
                groups = list(groups) + [{
                    "byt5": torch.cat([g["byt5"] for g in run]),
                    "clip": torch.cat([g["clip"] for g in run]) if run[0].get("clip") is not None else None,
                    "clip_image": None if ci is None else
                    [torch.cat([g["clip_image"][i] for g in run]) for i in range(len(ci))] if isinstance(ci, (list, tuple))
                    else torch.cat([g["clip_image"] for g in run])}]
                shared.append(False)
            slots += len(extra)
        with torch.cuda.device(dev):
            # zero-filled: rows between a slot's own length and s_max are never written by the K/V GEMMs, and the attention
            # kernel multiplies them by exactly-zero probabilities -- they must be finite
            cache = torch.zeros(L.pb200_paella_cond_cache_bytes(self._handle, slots, s_max), dtype=torch.uint8, device=dev)
            ws = self._ws(L.pb200_paella_workspace_bytes(self._handle, max(bt, slots), latent_hw[0], latent_hw[1], s_max))
            off = 0
            keep = []
            slot_of = []
            for g, sh, ent in zip(groups, shared, glora):
                n_g = g["byt5"].shape[0]
                if ent is not None and sh:
                    ent = ent[:1]
                if sh:
                    ci = g.get("clip_image")
                    g = {"byt5": g["byt5"][:1], "clip": g["clip"][:1] if g.get("clip") is not None else None,
                         "clip_image": ([t[:1] for t in ci] if isinstance(ci, (list, tuple)) else ci[:1]) if ci is not None else None}
                    slot_of += [off] * n_g
                else:
                    slot_of += list(range(off, off + n_g))
                byt5 = g["byt5"].to(device=dev, dtype=torch.float32).contiguous()
                B = byt5.shape[0]
                cond = _lib.Cond()
                cond.byt5, cond.byt5_len = ptr(byt5).value, byt5.shape[1]
                clip = g.get("clip")
                if clip is not None:
                    clip = clip.to(device=dev, dtype=torch.float32).contiguous()
                    cond.clip = ptr(clip).value
                ci = g.get("clip_image")
                if ci is not None:
                    ci = torch.stack([t.to(device=dev, dtype=torch.float32) for t in ci]) if isinstance(ci, (list, tuple)) \
                        else ci.to(device=dev, dtype=torch.float32)[None]
                    ci = ci.contiguous()
                    cond.clip_image, cond.n_clip_image = ptr(ci).value, ci.shape[0]
                keep += [byt5, clip, ci]
                if ent is not None and any(e is not None for e in ent):
                    adapters, ids_d, scales_d = ops.lora_rows_to_device(ent, dev)
                    keep += [ids_d, scales_d]
                    check(L.pb200_paella_prepare_cond_lora(self._handle, ctypes.byref(cond), B, off, slots, s_max, ptr(cache), ptr(ws),
                                                           ws.numel(), ops.lora_structs(adapters), len(adapters), ptr(ids_d),
                                                           ptr(scales_d), current_stream()), "pb200_paella_prepare_cond_lora")
                else:
                    check(L.pb200_paella_prepare_cond(self._handle, ctypes.byref(cond), B, off, slots, s_max, ptr(cache), ptr(ws),
                                                      ws.numel(), current_stream()), "pb200_paella_prepare_cond")
                off += B
            identity = slots == bt and not extra and not pag_tail      # (extra slots: slots may equal bt with a shared group)
            slot_map = None if identity else torch.tensor(slot_of[:bt] + [extra_slot + k for k in tail] + [slot_of[b] for b in pag_tail],
                                                          dtype=torch.int32, device=dev)
        return ConditioningCache(cache, bt + len(tail) + len(pag_tail), s_max, slots, slot_map, extra_slot)

    def gen_r_embedding(self, r, max_positions=10000):
        """ref/src/modules.py:212-221 -> [B, c_r]."""
        if max_positions != 10000:
            raise PaellaB200Error("gen_r_embedding: only max_positions=10000 is built (the reference's only value)")
        dev = self._device()
        with torch.cuda.device(dev):
            r = r.to(device=dev, dtype=torch.float32).contiguous()
            out = torch.empty(r.shape[0], self.c_r, dtype=torch.float32, device=dev)
            check(lib().pb200_paella_r_embedding(ptr(r), r.shape[0], self.c_r, ptr(out), current_stream()), "pb200_paella_r_embedding")
        return out

    def gen_c_embeddings(self, byt5, clip, clip_image):
        """ref/src/modules.py:223-232 (+ list-valued clip_image, ref/utils/modules.py:228-235) -> [B, S, c_cond]."""
        self._ensure_packed()
        L, dev = lib(), self._device()
        with torch.cuda.device(dev):
            byt5 = byt5.to(device=dev, dtype=torch.float32).contiguous()
            B = byt5.shape[0]
            cond = _lib.Cond()
            cond.byt5, cond.byt5_len = ptr(byt5).value, byt5.shape[1]
            n = 0
            if clip is not None:
                clip = clip.to(device=dev, dtype=torch.float32).contiguous()
                cond.clip = ptr(clip).value
                n += 1
            ci = clip_image
            if ci is not None:
                ci = torch.stack([t.to(device=dev, dtype=torch.float32) for t in ci]) if isinstance(ci, (list, tuple)) \
                    else ci.to(device=dev, dtype=torch.float32)[None]
                ci = ci.contiguous()
                cond.clip_image, cond.n_clip_image = ptr(ci).value, ci.shape[0]
                n += ci.shape[0]
            S = byt5.shape[1] + self._cfg["clip_seq_len"] * n
            out = torch.empty(B, S, self.c_cond, dtype=torch.float32, device=dev)
            ws = self._ws(L.pb200_paella_workspace_bytes(self._handle, B, 2 * self._cfg["patch_size"] * 2 ** (len(self._cfg["c_hidden"]) - 1),
                                                         2 * self._cfg["patch_size"] * 2 ** (len(self._cfg["c_hidden"]) - 1), S))
            check(L.pb200_paella_c_embeddings(self._handle, ctypes.byref(cond), B, ptr(out), ptr(ws), ws.numel(), current_stream()),
                  "pb200_paella_c_embeddings")
        return out

    # -------------------------------------------------------------- forward pieces
    def features(self, x: torch.Tensor, r: torch.Tensor, cond: ConditioningCache, attn_weights=None,
                 attn_weights_batch: int = 0, cfg_pairs: bool = False, n_pairs: Optional[int] = None,
                 w_len: Optional[torch.Tensor] = None, w_row: Optional[torch.Tensor] = None,
                 wrap: Optional[torch.Tensor] = None, regional=None, tail_src: Optional[torch.Tensor] = None,
                 maps=None, inject: Optional[torch.Tensor] = None, lora=None, perturb: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Everything up to out_mapper's LayerNorm: tokens [Bt,H,W] -> fp32 [Bt*H*W, c_out].

        ``cfg_pairs=True``: x [B,H,W] and r [B] are the classifier-free-guidance batch of ref/src/utils.py:42-45 —
        evaluated under the conditional rows [0,B) and the unconditional rows [B,2B) of ``cond``; the result has 2B
        samples, and the conditioning-independent blocks before the first AttnBlock run once per pair.
        ``n_pairs``: only the first n_pairs samples of x [B,H,W] are guided; the result has B + n_pairs samples, sample
        B + i being sample i under its unconditional rows (n_pairs = B is ``cfg_pairs=True``, 0 is unguided).
        ``attn_weights``: one vector for samples [0, attn_weights_batch), or with ``w_len`` a device float32 table [rows, w_ld]
        of per-sample vectors: sample b < attn_weights_batch reads row ``w_row[b]`` (int32 device [attn_weights_batch]; None:
        row b) and its first ``w_len[row]`` entries (int32 device [rows]; 0 = unweighted), pb200_paella_features_weighted.
        Each length must not exceed the sample's max_attn_weights.
        ``wrap``: seamless tiling, a device uint8 table of one byte per sample of x (ops.tiling_table; bit 0 wraps x, bit 1
        wraps y): the ResBlocks' depthwise convolutions pad circularly on the wrapped axes, and sample B + i of a CFG batch reads
        byte i (pb200_paella_features_tiled).  None launches exactly the untiled kernels.
        ``regional``: regional prompts, (token masks, region_slot, mask_row) on the device: uint8 [rows, H, W] masks (bit k >= 1:
        in region k, bit 0: in none), int32 [rows, R] cache slots of prompts 1..R (-1: none) and int32 [B] rows of the samples
        of x (None: row b); the unconditional rows are never masked (pb200_paella_features_regional).  None launches exactly the
        kernels without it.
        ``tail_src``: an arbitrary tail instead of ``cfg_pairs`` / ``n_pairs``, a device int32 [n_tail] of samples of x: the
        result has B + n_tail samples, sample B + i being sample tail_src[i]'s tokens and r under conditioning row B + i of
        ``cond`` (guidance prompts: the unconditional rows, then the term rows).  Tail rows read their source's wrap byte and are
        never masked nor weighted (pb200_paella_features_tail).
        ``maps``: attention maps, (map_row, map_batch, acc): sample b < map_batch of x adds its AttnBlocks' cross-attention maps to
        accumulator row map_row[b] (a device int32 [map_batch], -1: none; None: row b) of ``acc`` (map_accumulator), so that
        finalize_attention_maps turns it into the map of the forwards summed there (pb200_paella_features_maps).  The features are
        those of the call without it, bit for bit.  None launches exactly the kernels without it.
        ``inject``: prompt-to-prompt injection, a device int32 [n] (n <= B): sample b < n of x with a = inject[b] >= 0 (-1: none)
        attends in every AttnBlock with sample a's attention probabilities and its own values and attn_weights
        (pb200_paella_features_inject).  Sample a and sample b must have the same conditioning length and no regions.  Every
        other row is that of the call without it, bit for bit.  None launches exactly the kernels without it.
        ``lora``: LoRA adapters (lora_device): sample b of x runs every AttnBlock's in_proj and out_proj under its adapter and
        scale, and so does each tail row under its source's (pb200_paella_features_lora).  Rows without an adapter are those of
        the call without it, bit for bit.  None launches exactly the kernels without it.
        ``perturb``: perturbed-attention guidance, a device int64 [n] (n <= rows of the result, tail rows included; ops.pag_table's
        masks, read as uint64): row b < n runs AttnBlock i (plan order) with the self part of its attention collapsed onto the
        diagonal when bit i of perturb[b] is set (pb200_paella_features_pag).  A perturbed row is not regional, injected or a
        source.  With it, ``attn_weights_batch`` may cover tail rows too (a per-sample table whose w_row gives each tail row its
        row; a zero-length row leaves one unweighted).  Rows whose mask is 0 are those of the call without it, bit for bit.
        None launches exactly the kernels without it."""
        self._ensure_packed()
        L = lib()
        dev = self._device()
        Bt, H, W = x.shape
        if tail_src is not None:
            if cfg_pairs or n_pairs is not None or tail_src.dtype != torch.int32 or tail_src.dim() != 1 or tail_src.device != dev \
                    or tail_src.numel() > 65535:
                raise PaellaB200Error(f"features: tail_src must be an int32 vector on {dev} (and not with cfg_pairs or n_pairs)")
            n_pairs = tail_src.numel()
        elif n_pairs is not None:
            if cfg_pairs or not 0 <= n_pairs <= Bt:
                raise PaellaB200Error(f"features: n_pairs={n_pairs} for {Bt} samples (and not with cfg_pairs)")
        else:
            n_pairs = Bt if cfg_pairs else 0
        if wrap is not None and (wrap.dtype != torch.uint8 or wrap.numel() != Bt or wrap.device != dev):
            raise PaellaB200Error(f"features: wrap must be a uint8 table of {Bt} entries on {dev}")
        if inject is not None and (inject.dtype != torch.int32 or inject.dim() != 1 or not 0 < inject.numel() <= Bt
                                   or inject.device != dev or not inject.is_contiguous()):
            raise PaellaB200Error(f"features: inject must be a contiguous int32 vector of at most {Bt} entries on {dev}")
        if perturb is not None and (perturb.dtype != torch.int64 or perturb.dim() != 1 or not 0 < perturb.numel() <= Bt + n_pairs
                                    or perturb.device != dev or not perturb.is_contiguous()):
            raise PaellaB200Error(f"features: perturb must be a contiguous int64 vector of at most {Bt + n_pairs} entries on {dev}")
        Bt += n_pairs
        if Bt != cond.batch_total:
            raise PaellaB200Error(f"batch {Bt} does not match the conditioning cache ({cond.batch_total})")
        with torch.cuda.device(dev):
            x = x.to(device=dev, dtype=torch.int64).contiguous()
            r = r.to(device=dev, dtype=torch.float32).contiguous()
            ws_bytes = L.pb200_paella_workspace_bytes(self._handle, Bt, H, W, cond.s_max)
            if maps is not None:
                map_row, map_batch, acc = maps
                if acc.dtype != torch.float32 or acc.dim() != 3 or not acc.is_contiguous() or acc.device != dev \
                        or acc.shape[2] != self.map_positions((H, W)) or not 0 <= map_batch <= Bt - n_pairs \
                        or (map_row is not None and (map_row.dtype != torch.int32 or map_row.numel() < map_batch)) \
                        or (map_row is None and map_batch > acc.shape[0]):
                    raise PaellaB200Error(f"features: attention maps need a contiguous float32 accumulator [rows, keys, "
                                          f"{self.map_positions((H, W))}] on {dev} and an optional int32 map_row [map_batch]")
                ws_bytes += L.pb200_paella_maps_workspace_bytes(self._handle, acc.shape[0], H, W, cond.s_max)
            ws = self._ws(ws_bytes)
            feats = torch.empty(Bt * H * W, self._cfg["c_out"], dtype=torch.float32, device=dev)
            if w_len is not None:
                if attn_weights is None or attn_weights.dim() != 2 or attn_weights.dtype != torch.float32 or w_len.dtype != torch.int32 \
                        or w_len.numel() != attn_weights.shape[0] or (w_row is not None and w_row.numel() < attn_weights_batch):
                    raise PaellaB200Error("features: a per-sample weight table is float32 [rows, w_ld] with int32 w_len [rows] "
                                          "and an optional int32 w_row [attn_weights_batch]")
                if regional is not None or tail_src is not None or maps is not None or inject is not None or lora is not None \
                        or perturb is not None:
                    self._features_regional(x, r, Bt, n_pairs, H, W, cond, (ptr(attn_weights), 0, attn_weights.shape[1], ptr(w_len),
                                                                            ptr(w_row)), attn_weights_batch, wrap, regional, feats, ws,
                                            tail_src, maps, inject, lora, perturb)
                    return feats
                if wrap is not None:
                    check(L.pb200_paella_features_tiled(self._handle, ptr(x), ptr(r), Bt, n_pairs, H, W, ptr(cond.cache), cond.slots,
                                                        ptr(cond.slot_map), cond.s_max, ptr(attn_weights), 0, attn_weights.shape[1],
                                                        ptr(w_len), ptr(w_row), attn_weights_batch, ptr(wrap), ptr(feats), ptr(ws),
                                                        ws.numel(), current_stream()), "pb200_paella_features_tiled")
                    return feats
                check(L.pb200_paella_features_weighted(self._handle, ptr(x), ptr(r), Bt, n_pairs, H, W, ptr(cond.cache), cond.slots,
                                                       ptr(cond.slot_map), cond.s_max, ptr(attn_weights), 0, attn_weights.shape[1],
                                                       ptr(w_len), ptr(w_row), attn_weights_batch, ptr(feats), ptr(ws), ws.numel(),
                                                       current_stream()), "pb200_paella_features_weighted")
                return feats
            aw = attn_weights.to(device=dev, dtype=torch.float32).contiguous() if attn_weights is not None else None
            if regional is not None or tail_src is not None or maps is not None or inject is not None or lora is not None \
                    or perturb is not None:
                self._features_regional(x, r, Bt, n_pairs, H, W, cond, (ptr(aw), aw.numel() if aw is not None else 0, 0, None, None),
                                        attn_weights_batch, wrap, regional, feats, ws, tail_src, maps, inject, lora, perturb)
                return feats
            if wrap is not None:        # the single weight vector is the weighted call with w_ld = 0 and no w_len
                check(L.pb200_paella_features_tiled(self._handle, ptr(x), ptr(r), Bt, n_pairs, H, W, ptr(cond.cache), cond.slots,
                                                    ptr(cond.slot_map), cond.s_max, ptr(aw), aw.numel() if aw is not None else 0, 0,
                                                    None, None, attn_weights_batch, ptr(wrap), ptr(feats), ptr(ws), ws.numel(),
                                                    current_stream()), "pb200_paella_features_tiled")
                return feats
            check(L.pb200_paella_features_pairs(self._handle, ptr(x), ptr(r), Bt, n_pairs, H, W, ptr(cond.cache), cond.slots,
                                                ptr(cond.slot_map), cond.s_max, ptr(aw),
                                                aw.numel() if aw is not None else 0, attn_weights_batch, ptr(feats), ptr(ws),
                                                ws.numel(), current_stream()), "pb200_paella_features_pairs")
        return feats

    def _features_regional(self, x, r, Bt, n_pairs, H, W, cond, weights, w_batch, wrap, regional, feats, ws, tail_src=None, maps=None,
                           inject=None, lora=None, perturb=None):
        """pb200_paella_features_regional, or with ``tail_src`` pb200_paella_features_tail, or with ``maps``
        pb200_paella_features_maps, or with ``inject`` pb200_paella_features_inject, or with ``lora`` pb200_paella_features_lora, or
        with ``perturb`` pb200_paella_features_pag (``regional`` may then be None)."""
        mask = region_slot = mask_row = None
        if regional is not None:
            mask, region_slot, mask_row = regional
            rows = mask.shape[0]
            if mask.dtype != torch.uint8 or tuple(mask.shape[1:]) != (H, W) or region_slot.dtype != torch.int32 \
                    or region_slot.dim() != 2 or region_slot.shape[0] != rows or not 0 <= region_slot.shape[1] <= ops.MAX_PROMPT_REGIONS \
                    or (mask_row is None and rows < Bt - n_pairs) or (mask_row is not None and mask_row.numel() < Bt - n_pairs):
                raise PaellaB200Error(f"features: regional prompts are uint8 masks [rows, {H}, {W}], int32 region_slot [rows, <= "
                                      f"{ops.MAX_PROMPT_REGIONS}] and an optional int32 mask_row [{Bt - n_pairs}]")
        if w_batch > (Bt if perturb is not None else Bt - n_pairs):
            raise PaellaB200Error(f"features: {w_batch} weighted samples of {Bt - n_pairs}")
        n_regions = region_slot.shape[1] if region_slot is not None else 0
        if perturb is not None:
            structs, n_adapters, ids, scales = lora if lora is not None else (None, 0, None, None)
            if lora is not None and (ids.numel() != Bt - n_pairs or scales.numel() != Bt - n_pairs):
                raise PaellaB200Error(f"features: LoRA tables of {ids.numel()} samples for {Bt - n_pairs}")
            map_row, map_batch, acc = maps if maps is not None else (None, 0, None)
            check(lib().pb200_paella_features_pag(self._handle, ptr(x), ptr(r), Bt, n_pairs, H, W, ptr(cond.cache), cond.slots,
                                                  ptr(cond.slot_map), cond.s_max, *weights, w_batch, ptr(wrap), ptr(mask),
                                                  ptr(mask_row), ptr(region_slot), n_regions, ptr(tail_src), ptr(map_row), map_batch,
                                                  ptr(acc), acc.shape[0] if acc is not None else 0,
                                                  acc.shape[1] if acc is not None else 0, ptr(inject),
                                                  inject.numel() if inject is not None else 0, structs, n_adapters, ptr(ids),
                                                  ptr(scales), ptr(perturb), perturb.numel(), ptr(feats), ptr(ws), ws.numel(),
                                                  current_stream()), "pb200_paella_features_pag")
            return
        if lora is not None:
            structs, n_adapters, ids, scales = lora
            if ids.numel() != Bt - n_pairs or scales.numel() != Bt - n_pairs:
                raise PaellaB200Error(f"features: LoRA tables of {ids.numel()} samples for {Bt - n_pairs}")
            map_row, map_batch, acc = maps if maps is not None else (None, 0, None)
            check(lib().pb200_paella_features_lora(self._handle, ptr(x), ptr(r), Bt, n_pairs, H, W, ptr(cond.cache), cond.slots,
                                                   ptr(cond.slot_map), cond.s_max, *weights, w_batch, ptr(wrap), ptr(mask),
                                                   ptr(mask_row), ptr(region_slot), n_regions, ptr(tail_src), ptr(map_row), map_batch,
                                                   ptr(acc), acc.shape[0] if acc is not None else 0,
                                                   acc.shape[1] if acc is not None else 0, ptr(inject),
                                                   inject.numel() if inject is not None else 0, structs, n_adapters, ptr(ids),
                                                   ptr(scales), ptr(feats), ptr(ws), ws.numel(), current_stream()),
                  "pb200_paella_features_lora")
            return
        if inject is not None:
            map_row, map_batch, acc = maps if maps is not None else (None, 0, None)
            check(lib().pb200_paella_features_inject(self._handle, ptr(x), ptr(r), Bt, n_pairs, H, W, ptr(cond.cache), cond.slots,
                                                     ptr(cond.slot_map), cond.s_max, *weights, w_batch, ptr(wrap), ptr(mask),
                                                     ptr(mask_row), ptr(region_slot), n_regions, ptr(tail_src), ptr(map_row), map_batch,
                                                     ptr(acc), acc.shape[0] if acc is not None else 0,
                                                     acc.shape[1] if acc is not None else 0, ptr(inject), inject.numel(), ptr(feats),
                                                     ptr(ws), ws.numel(), current_stream()), "pb200_paella_features_inject")
            return
        if maps is not None:
            map_row, map_batch, acc = maps
            check(lib().pb200_paella_features_maps(self._handle, ptr(x), ptr(r), Bt, n_pairs, H, W, ptr(cond.cache), cond.slots,
                                                   ptr(cond.slot_map), cond.s_max, *weights, w_batch, ptr(wrap), ptr(mask),
                                                   ptr(mask_row), ptr(region_slot), n_regions, ptr(tail_src), ptr(map_row), map_batch,
                                                   ptr(acc), acc.shape[0], acc.shape[1], ptr(feats), ptr(ws), ws.numel(),
                                                   current_stream()), "pb200_paella_features_maps")
            return
        if tail_src is not None:
            check(lib().pb200_paella_features_tail(self._handle, ptr(x), ptr(r), Bt, n_pairs, H, W, ptr(cond.cache), cond.slots,
                                                   ptr(cond.slot_map), cond.s_max, *weights, w_batch, ptr(wrap), ptr(mask),
                                                   ptr(mask_row), ptr(region_slot), n_regions, ptr(tail_src), ptr(feats), ptr(ws),
                                                   ws.numel(), current_stream()), "pb200_paella_features_tail")
            return
        check(lib().pb200_paella_features_regional(self._handle, ptr(x), ptr(r), Bt, n_pairs, H, W, ptr(cond.cache), cond.slots,
                                                   ptr(cond.slot_map), cond.s_max, *weights, w_batch, ptr(wrap), ptr(mask),
                                                   ptr(mask_row), ptr(region_slot), n_regions, ptr(feats), ptr(ws),
                                                   ws.numel(), current_stream()), "pb200_paella_features_regional")

    def map_positions(self, latent_hw) -> int:
        """Columns of an attention-map accumulator on a ``latent_hw`` token grid: every level's block positions, level 0 first."""
        ps = self._cfg["patch_size"]
        return sum((int(latent_hw[0]) // (ps << l)) * (int(latent_hw[1]) // (ps << l)) for l in range(len(self._cfg["c_hidden"])))

    def map_accumulator(self, rows: int, cond_len: int, latent_hw) -> torch.Tensor:
        """A zeroed attention-map accumulator for features' ``maps``: float32 [rows, cond_len, map_positions] on the model's device."""
        return torch.zeros(rows, cond_len, self.map_positions(latent_hw), dtype=torch.float32, device=self._device())

    def finalize_attention_maps(self, acc: torch.Tensor, latent_hw, cond_len: int, n_steps: int) -> torch.Tensor:
        """Attention maps float32 [rows, cond_len, H, W] from accumulator rows ``acc`` (a contiguous run of map_accumulator rows)
        summed over ``n_steps`` forwards: every level upsampled by nearest neighbour, the levels summed and the result scaled by
        1 / (n_steps * number of AttnBlocks) -- pb200_paella_attention_maps_finalize."""
        self._ensure_packed()
        H, W = int(latent_hw[0]), int(latent_hw[1])
        if acc.dtype != torch.float32 or acc.dim() != 3 or not acc.is_contiguous() or acc.shape[2] != self.map_positions((H, W)) \
                or not 0 <= cond_len <= acc.shape[1]:
            raise PaellaB200Error(f"finalize_attention_maps: a contiguous float32 accumulator [rows, >= {cond_len}, "
                                  f"{self.map_positions((H, W))}] is required")
        with torch.cuda.device(self._device()):
            out = torch.empty(acc.shape[0], cond_len, H, W, dtype=torch.float32, device=self._device())
            check(lib().pb200_paella_attention_maps_finalize(self._handle, ptr(acc), acc.shape[0], acc.shape[1], H, W, cond_len,
                                                             int(n_steps), ptr(out), current_stream()),
                  "pb200_paella_attention_maps_finalize")
        return out

    def guidance_mix(self, feats: torch.Tensor, hw: int, rows: torch.Tensor, coef: torch.Tensor) -> torch.Tensor:
        """Guidance prompts: the K-way guided mix in place on ``feats`` (fp32 [samples * hw, c_out], features' output), one
        launch: composed sample y's row rows[y, 0] becomes the mix of its rows ``rows[y]`` (device int32 [n, 2 + J]: c, u, then
        its term rows, -1 after the last) with the coefficients ``coef[y]`` (device float32 [n, 2 + J],
        ops.guidance_coefficients) -- pb200_paella_guidance_mix.  A sampler then takes row c with params (1, 0, 1/T)."""
        self._ensure_packed()
        if rows.dtype != torch.int32 or coef.dtype != torch.float32 or rows.dim() != 2 or tuple(coef.shape) != tuple(rows.shape) \
                or feats.dtype != torch.float32 or not feats.is_contiguous():
            raise PaellaB200Error("guidance_mix: int32 rows and float32 coef of one shape [n, 2 + J] on contiguous fp32 features")
        with torch.cuda.device(self._device()):
            check(lib().pb200_paella_guidance_mix(self._handle, ptr(feats), hw, ptr(rows), ptr(coef), rows.shape[0], rows.shape[1],
                                                  current_stream()), "pb200_paella_guidance_mix")
        return feats

    def regional_device(self, table, cond: ConditioningCache):
        """The host table of ops.regional_table as features' ``regional`` argument for ``cond``, a cache whose extra slots are the
        table's prompts in order (prepare_conditioning's ``extra``): (uint8 masks [B, H, W], int32 region_slot [B, R]) in one
        asynchronous copy, and mask_row None."""
        masks, prompts = table
        R = max(len(p) for p in prompts)
        slots = torch.full((len(prompts), R), -1, dtype=torch.int32)
        k = cond.extra_slot
        for b, own in enumerate(prompts):
            slots[b, :len(own)] = torch.arange(k, k + len(own), dtype=torch.int32)
            k += len(own)
        mask_d, slot_d = ops.to_device_packed([masks, slots], self._device())
        return mask_d, slot_d, None

    def logits_from_features(self, feats: torch.Tensor, batch: int, h: int, w: int) -> torch.Tensor:
        self._ensure_packed()
        L = lib()
        dev = self._device()
        with torch.cuda.device(dev):
            out = torch.empty(batch, self.num_labels, h, w, dtype=torch.float32, device=dev)
            ws = self._ws(feats.numel() * 2 + 256)
            check(L.pb200_paella_logits(self._handle, ptr(feats), batch, h * w, ptr(out), ptr(ws), ws.numel(),
                                        current_stream()), "pb200_paella_logits")
        return out

    def sample_tokens(self, feats: torch.Tensor, batch: int, h: int, w: int, cfg, temperature, generator=None) -> torch.Tensor:
        """Fused out_mapper + CFG + temperature + multinomial on torch's random stream (ref/src/utils.py:44-50).
        ``generator``: None (the default CUDA generator), one CUDA generator, or a list of ``batch`` of them -- one stream per
        sample, where sample b draws what this call with batch 1 draws on generator b (ops.check_generators).
        ``cfg`` (float or None) and ``temperature`` (float) may also be CPU tensors [batch] of per-sample values; sample b is
        then computed exactly as this call with its own scalars (ops.sampling_params_table).  ``cfg=None`` is no guidance."""
        if torch.is_tensor(cfg) or torch.is_tensor(temperature):
            params = ops.sampling_params_table(cfg, temperature, batch, self._device())
            return self.sample_tokens_params(feats, batch, h, w, cfg is not None, params, generator)
        self._ensure_packed()
        L = lib()
        dev = self._device()
        if ops.per_sample(generator):
            ops.check_generators(generator, batch, dev)
            ops.check_per_sample_numel(h * w * self.num_labels)
            with torch.cuda.device(dev):
                out = torch.empty(batch, h, w, dtype=torch.int64, device=dev)
                ws = self._ws(L.pb200_paella_workspace_bytes(self._handle, batch, h, w, 1))
                table = ops.philox_table(generator, h * w * self.num_labels, dev)
                check(L.pb200_paella_sample_tokens_per_sample(self._handle, ptr(feats), batch, h * w, 1 if cfg is not None else 0,
                                                              float(cfg) if cfg is not None else 0.0, float(temperature), ptr(table),
                                                              ptr(out), ptr(ws), ws.numel(), current_stream()),
                      "pb200_paella_sample_tokens_per_sample")
            return out
        with torch.cuda.device(dev):
            out = torch.empty(batch, h, w, dtype=torch.int64, device=dev)
            ws = self._ws(L.pb200_paella_workspace_bytes(self._handle, batch, h, w, 1))
            n = batch * h * w
            chunks = ops.philox_row_chunks(n, self.num_labels)       # one kernel per 32-bit-indexable piece, like torch
            ops.skip_philox_for_split(chunks, n * self.num_labels, dev, generator)
            flat = out.view(-1)
            for lo, hi in chunks:
                seed, off = ops.take_philox((hi - lo) * self.num_labels, dev, generator)
                if len(chunks) == 1:
                    f = feats
                elif cfg is not None:
                    f = torch.cat([feats[lo:hi], feats[n + lo:n + hi]])
                else:
                    f = feats[lo:hi]
                check(L.pb200_paella_sample_tokens(self._handle, ptr(f), 1, hi - lo, 1 if cfg is not None else 0,
                                                   float(cfg) if cfg is not None else 0.0, float(temperature), seed, off,
                                                   ptr(flat[lo:hi]), ptr(ws), ws.numel(), current_stream()), "pb200_paella_sample_tokens")
        return out

    def sample_tokens_params(self, feats: torch.Tensor, batch: int, h: int, w: int, cfg_on: bool, params: torch.Tensor,
                             generator=None, trunc=None) -> torch.Tensor:
        """sample_tokens with per-sample guidance scale and temperature in one launch over the batch (per random stream):
        ``params`` is a device float32 [batch, 3] of (cfg, 1 - cfg, 1/T) (ops.sampling_params_table); its cfg columns are
        ignored when ``cfg_on`` is False.  Draws on ``generator`` exactly as sample_tokens does.  ``trunc``: None, or the
        device truncation table (int32 k [batch], float32 p [batch]) of ops.truncation_table: sample b's draw keeps its top-k /
        top-p codes (pb200_paella_sample_tokens_params_trunc), on the same random draws."""
        tk, tp = trunc if trunc is not None else (None, None)
        self._ensure_packed()
        L = lib()
        dev = self._device()
        hw = h * w
        with torch.cuda.device(dev):
            out = torch.empty(batch, h, w, dtype=torch.int64, device=dev)
            ws = self._ws(L.pb200_paella_workspace_bytes(self._handle, batch, h, w, 1))
            if ops.per_sample(generator):
                ops.check_generators(generator, batch, dev)
                ops.check_per_sample_numel(hw * self.num_labels)
                table = ops.philox_table(generator, hw * self.num_labels, dev)
                check(L.pb200_paella_sample_tokens_params_trunc(self._handle, ptr(feats), batch, hw, int(cfg_on), ptr(params), 0, 0,
                                                                ptr(table), ptr(tk), ptr(tp), ptr(out), ptr(ws), ws.numel(),
                                                                current_stream()), "pb200_paella_sample_tokens_params_trunc")
                return out
            n = batch * hw
            chunks = ops.philox_row_chunks(n, self.num_labels)       # one kernel per 32-bit-indexable piece, like torch
            flat = out.view(-1)
            for lo, hi in chunks:
                if lo % hw or hi % hw:
                    raise PaellaB200Error("sample_tokens: torch's 32-bit split of this draw falls inside a sample")
            ops.skip_philox_for_split(chunks, n * self.num_labels, dev, generator)
            for lo, hi in chunks:
                seed, off = ops.take_philox((hi - lo) * self.num_labels, dev, generator)
                if len(chunks) == 1:
                    f = feats
                elif cfg_on:
                    f = torch.cat([feats[lo:hi], feats[n + lo:n + hi]])
                else:
                    f = feats[lo:hi]
                sl = slice(lo // hw, hi // hw)
                check(L.pb200_paella_sample_tokens_params_trunc(self._handle, ptr(f), (hi - lo) // hw, hw, int(cfg_on), ptr(params[sl]),
                                                                seed, off, None, ptr(tk[sl] if tk is not None else None),
                                                                ptr(tp[sl] if tp is not None else None), ptr(flat[lo:hi]), ptr(ws),
                                                                ws.numel(), current_stream()), "pb200_paella_sample_tokens_params_trunc")
        return out

    def sample_tokens_pairs(self, feats: torch.Tensor, batch: int, n_pairs: int, h: int, w: int, params: torch.Tensor,
                            seed_offset: torch.Tensor, out: Optional[torch.Tensor] = None, trunc=None) -> torch.Tensor:
        """sample_tokens_params on the features of ``features(..., n_pairs=n_pairs)``: samples b < n_pairs are guided, the rest
        draw on their conditional rows alone, all in one launch on per-sample streams (``seed_offset``: ops.philox_table over
        h * w * num_labels).  ``trunc`` as in sample_tokens_params."""
        tk, tp = trunc if trunc is not None else (None, None)
        self._ensure_packed()
        L = lib()
        dev = self._device()
        with torch.cuda.device(dev):
            if out is None:
                out = torch.empty(batch, h, w, dtype=torch.int64, device=dev)
            ws = self._ws(L.pb200_paella_workspace_bytes(self._handle, batch, h, w, 1))
            check(L.pb200_paella_sample_tokens_pairs_trunc(self._handle, ptr(feats), batch, n_pairs, h * w, ptr(params), ptr(seed_offset),
                                                           None, ptr(tk), ptr(tp), ptr(out), ptr(ws), ws.numel(), current_stream()),
                  "pb200_paella_sample_tokens_pairs_trunc")
        return out

    def resample_workspace_bytes(self, hw: int, chunk: int = ops.RESAMPLE_CHUNK) -> int:
        """Scratch of sample_tokens_modes' argmax and quant samples: fp16 features and fp32 logits of 2 * chunk samples."""
        self._ensure_packed()
        return int(lib().pb200_paella_resample_workspace_bytes(self._handle, chunk, hw))

    def sample_tokens_modes(self, feats: torch.Tensor, batch: int, n_pairs: int, h: int, w: int, params: torch.Tensor,
                            seed_offset: torch.Tensor, modes: Sequence[str], table: torch.Tensor, codebook: Optional[torch.Tensor] = None,
                            out: Optional[torch.Tensor] = None, chunk: int = ops.RESAMPLE_CHUNK, trunc=None) -> torch.Tensor:
        """sample_tokens_pairs with a sampling mode per sample (``modes``: batch names of ops.SAMPLING_MODES; ``table``: their
        ops.mode_table on the device).  The multinomial samples draw in one fused-sampler launch, the others skipped through the
        table's codes (their ``seed_offset`` rows are not read); then each other mode present runs pb200_paella_resample_samples
        over its samples: the out_mapper GEMM to logits, ``chunk`` guided samples at a time, and the argmax or quant kernel,
        which draw nothing.  Sample b's tokens are those of sample_notebook's step in mode b.  ``codebook``: the VQGAN codebook
        fp32 [num_labels, c_latent], for 'quant'.  ``trunc`` (sample_tokens_params) truncates the multinomial samples' draws;
        the argmax and quant samples ignore it."""
        tk, tp = trunc if trunc is not None else (None, None)
        self._ensure_packed()
        L = lib()
        dev = self._device()
        hw = h * w
        count = {md: sum(1 for x in modes if x == md) for md in ops.SAMPLING_MODES}
        if len(modes) != batch or sum(count.values()) != batch:
            raise PaellaB200Error(f"sample_tokens_modes: {len(modes)} modes for {batch} samples (each one of {ops.SAMPLING_MODES})")
        if count["quant"] and (codebook is None or codebook.shape[0] != self.num_labels):
            raise PaellaB200Error("sample_tokens_modes: 'quant' needs the VQGAN codebook [num_labels, c_latent]")
        with torch.cuda.device(dev):
            if out is None:
                out = torch.empty(batch, h, w, dtype=torch.int64, device=dev)
            ws = self._ws(max(L.pb200_paella_workspace_bytes(self._handle, batch, h, w, 1),
                              L.pb200_paella_resample_workspace_bytes(self._handle, chunk, hw) if count["multinomial"] < batch else 0))
            if count["multinomial"]:
                skip = table[:batch] if count["multinomial"] < batch else None
                check(L.pb200_paella_sample_tokens_pairs_trunc(self._handle, ptr(feats), batch, n_pairs, hw, ptr(params), ptr(seed_offset),
                                                               ptr(skip), ptr(tk), ptr(tp), ptr(out), ptr(ws), ws.numel(),
                                                               current_stream()), "pb200_paella_sample_tokens_pairs_trunc")
            off, lists = batch, []
            for code, md in ((1, "argmax"), (2, "quant")):
                lists.append((code, [b for b, x in enumerate(modes) if x == md], off))
                off += count[md]
            cb = codebook.contiguous().float() if count["quant"] else None
            for code, samples, o in lists:
                if not samples:
                    continue
                n_guided = sum(1 for b in samples if b < n_pairs)       # ascending: the guided samples come first
                check(L.pb200_paella_resample_samples(self._handle, ptr(feats), batch, n_pairs, hw, ptr(table[o:o + len(samples)]),
                                                      len(samples), n_guided, ptr(params), code, ptr(cb) if code == 2 else None,
                                                      cb.shape[1] if code == 2 else 0, chunk, ptr(out), ptr(ws), ws.numel(),
                                                      current_stream()), "pb200_paella_resample_samples")
        return out

    @property
    def n_attn_blocks(self) -> int:
        """The number of AttnBlocks, the index space of perturbed-attention guidance's blocks (paella_b200.lora.attn_blocks)."""
        from .lora import attn_blocks
        return len(attn_blocks(self._cfg))

    def pag_default_blocks(self) -> list:
        """The AttnBlocks a PAG entry given as a scale perturbs: those of the deepest level, down and up (ops.pag_default_blocks)."""
        return ops.pag_default_blocks(self._cfg)

    def conditioning_seq_len(self, inputs: Dict[str, torch.Tensor]) -> int:
        """Length of the conditioning sequence of ``inputs`` (byt5 rows + clip_seq_len per clip / clip_image embedding)."""
        n = (1 if inputs.get("clip") is not None else 0)
        ci = inputs.get("clip_image")
        if ci is not None:
            n += len(ci) if isinstance(ci, (list, tuple)) else 1
        return inputs["byt5"].shape[1] + self._cfg["clip_seq_len"] * n

    def max_attn_weights(self, latent_hw, cond_len: int) -> int:
        """The longest ``attn_weights`` vector a sample with ``cond_len`` conditioning rows takes on a ``latent_hw`` token grid:
        the smallest key count it sees in any AttnBlock (that level's positions with self-attention, plus the conditioning).
        The reference fails on a longer vector (ref/utils/alter_attention.py:28)."""
        c = self._cfg
        ps = c["patch_size"]
        keys = [((latent_hw[0] // ps) >> i) * ((latent_hw[1] // ps) >> i) * int(c["self_attn"]) + cond_len
                for i, (kinds, n) in enumerate(zip(c["level_config"], c["blocks"])) if "A" in kinds and n > 0]
        return min(keys) if keys else 2 ** 31 - 1

    def _attn_weights_table(self, attn_weights, batch: int, latent_hw, cond_len: int):
        """Per-sample ``attn_weights`` (a list or tuple, ops.attn_weights_table) -> the device table (w [B, w_ld], lengths
        [B]) in one asynchronous copy; a 1-D tensor or None is returned as is.  ValueError before anything is enqueued."""
        if not isinstance(attn_weights, (list, tuple)):
            return attn_weights, None
        table, lens = ops.attn_weights_table(attn_weights, batch, [self.max_attn_weights(latent_hw, cond_len)] * batch)
        return ops.attn_weights_to_device(table, lens, self._device())

    def write_conditioning(self, cache: ConditioningCache, slot: int, inputs: Dict[str, torch.Tensor], latent_hw, lora=None) -> None:
        """Project the conditioning of B samples (``inputs`` with batch B, one sequence layout) into slots [slot, slot + B)
        of an existing cache, as prepare_conditioning projects a group; each slot's kv_len becomes this sequence's length, so
        rows left over from a longer sequence are never attended to.  ``lora``: None or B entries (None or (adapter, scale)), the
        adapter each slot is projected under.  Host-to-device copies are asynchronous (no stream synchronisation)."""
        self._ensure_packed()
        L = lib()
        dev = self._device()

        def d(v):
            return v.to(device=dev, dtype=torch.float32, non_blocking=True).contiguous()
        with torch.cuda.device(dev):
            cond = _lib.Cond()
            byt5 = d(inputs["byt5"])
            cond.byt5, cond.byt5_len = ptr(byt5).value, byt5.shape[1]
            clip = d(inputs["clip"]) if inputs.get("clip") is not None else None
            cond.clip = ptr(clip).value if clip is not None else None
            ci = inputs.get("clip_image")
            if ci is not None:
                ci = torch.stack([d(v) for v in ci]) if isinstance(ci, (list, tuple)) else d(ci)[None]
                cond.clip_image, cond.n_clip_image = ptr(ci).value, ci.shape[0]
            B = byt5.shape[0]
            ws = self._ws(L.pb200_paella_workspace_bytes(self._handle, B, latent_hw[0], latent_hw[1], cache.s_max))
            if lora is not None and any(e is not None for e in lora):
                adapters, ids_d, scales_d = ops.lora_rows_to_device(lora, dev)
                check(L.pb200_paella_prepare_cond_lora(self._handle, ctypes.byref(cond), B, slot, cache.slots, cache.s_max,
                                                       ptr(cache.cache), ptr(ws), ws.numel(), ops.lora_structs(adapters), len(adapters),
                                                       ptr(ids_d), ptr(scales_d), current_stream()), "pb200_paella_prepare_cond_lora")
                return
            check(L.pb200_paella_prepare_cond(self._handle, ctypes.byref(cond), B, slot, cache.slots, cache.s_max, ptr(cache.cache),
                                              ptr(ws), ws.numel(), current_stream()), "pb200_paella_prepare_cond")

    def forward(self, x, r, byt5, clip=None, clip_image=None, x_cat=None, **kwargs):
        """ref/src/modules.py:263-275 / ref/utils/modules.py:268-282: logits [B, num_labels, H, W] fp32.
        ``attn_weights``: one vector for every sample, or a list or tuple of B entries, each None or a 1-D CPU float tensor
        that weights sample b alone (ValueError for a bad entry, before anything is enqueued).
        ``tiling``: seamless tiling (keyword only): None / 'none', 'x' (left and right edges wrap), 'y' (top and bottom wrap) or
        'xy', one for every sample or a list or tuple of B values.  The ResBlocks' depthwise convolutions then pad circularly,
        as the reference with ``padding_mode='circular'`` on those Conv2d modules does.  ValueError, before anything is
        enqueued, for an unknown value, a list of the wrong length or a tensor.
        ``prompt_regions``: regional prompts (keyword only): None, or a list or tuple of B entries, each None or a list of at most
        7 (inputs, region) pairs -- a batch-1 conditioning dict and a bool [H, W] token mask on the CPU or the model's device
        (ops.regional_table).  Every AttnBlock position then attends to the self keys and to the conditioning of each region its
        footprint touches, and to the sample's own conditioning where its footprint touches no region.  ValueError, before
        anything is enqueued, for a bad entry and for regions on a sample that also has attn_weights.
        ``attention_maps=True`` (keyword only): returns (logits, maps), maps float32 [B, S, H, W] on the model's device: for key s
        of the sample's conditioning sequence (gen_c_embeddings order) and token (y, x), the mean over every AttnBlock and its
        heads of the post-softmax, post-attn_weights probability the block position holding the token gives the key -- what the
        reference's CustomMultiheadAttention returns with need_weights=True.  The logits are those of the call without it, bit
        for bit.  ValueError, before anything is enqueued, for a flag that is not a bool and for maps with prompt_regions.
        ``attention_source``: prompt-to-prompt injection (keyword only): None, or a list or tuple of B entries, each None or the
        int index a of another sample of the call.  Sample b then attends, in every AttnBlock and head, with sample a's attention
        probabilities over [self ; conditioning] keys (from a's queries and keys), times its own attn_weights, applied to its own
        values.  Every other sample's logits are those of the call without it, bit for bit.  ValueError, before anything is
        enqueued, for a bad entry, a source that is itself injected, and prompt_regions on an injected sample or its source
        (ops.attention_source_table).
        ``lora``: LoRA adapters (keyword only; paella_b200.lora.load_lora): None, an adapter or (adapter, scale) for every sample,
        or a list or tuple of B entries, each None, an adapter or (adapter, scale).  Sample b is then the reference model with
        W + scale * (alpha / r) * B A on its adapter's targets (every AttnBlock's in_proj, out_proj and kv_mapper), conditioning
        included.  Samples without an adapter, or at scale 0, get the logits of the call without it, bit for bit.  ValueError,
        before anything is enqueued, for a bad entry or scale and an adapter of another configuration or device (ops.lora_table).
        ``pag_blocks``: perturbed-attention guidance (keyword only): None, or a list or tuple of B entries, each None or a non-empty
        list of AttnBlock indices (plan order, paella_b200.lora.attn_blocks).  Sample b's logits are then its perturbed logits l_p,
        with no mix: in every listed AttnBlock and head, each query's attention mass on the self keys (post-softmax, post
        attn_weights) goes to its own value, and its conditioning probabilities are unchanged.  Every other sample's logits are
        those of the call without it, bit for bit.  With ``attention_maps=True`` a perturbed sample's maps are those of its
        perturbed forward, which are its conditioning probabilities as the plain forward's are (the perturbation changes only
        where the self keys' mass goes), taken at that forward's queries.  ValueError, before anything is enqueued, for a bad
        entry, and PAG on a sample with prompt_regions or on an injected sample or its source (ops.pag_table)."""
        if x_cat is not None:
            x = torch.cat([x, x_cat], dim=1)
        attn_weights = kwargs.pop("attn_weights", None)
        tiling = kwargs.pop("tiling", None)
        prompt_regions = kwargs.pop("prompt_regions", None)
        attention_maps = ops.check_attention_maps(kwargs.pop("attention_maps", False), prompt_regions)
        attention_source = kwargs.pop("attention_source", None)
        lora = kwargs.pop("lora", None)
        pag_blocks = kwargs.pop("pag_blocks", None)
        if kwargs:
            raise TypeError(f"unexpected keyword arguments {sorted(kwargs)}")
        B, H, W = x.shape
        wrap = ops.tiling_table(tiling, B)
        regions = ops.regional_table(prompt_regions, B, (H, W), self._device())
        ops.check_regions_unweighted(regions, attn_weights)
        inject = ops.attention_source_table(attention_source, B, 1, regions, forward=True)
        pag_t = ops.pag_table(pag_blocks, B, self.n_attn_blocks, regions=regions, inject=inject, forward=True)
        lora_t = ops.lora_table(lora, B, self)
        cond_len = self.conditioning_seq_len({"byt5": byt5, "clip": clip, "clip_image": clip_image})
        aw, w_len = self._attn_weights_table(attn_weights, B, (H, W), cond_len)
        regional = None
        if regions is None and lora_t is None:
            cond = self._cond_for_forward(byt5, clip, clip_image, (H, W))
        else:
            entries = ops.lora_entries(lora_t, B)
            cond = self.prepare_conditioning([{"byt5": byt5, "clip": clip, "clip_image": clip_image}], (H, W), share_uniform=False,
                                             extra=[g for own in regions[1] for g in own] if regions is not None else [],
                                             lora=[entries] if lora_t is not None else None,
                                             extra_lora=[entries[b] for b, own in enumerate(regions[1]) for _ in own]
                                             if regions is not None else None)
            regional = self.regional_device(regions, cond) if regions is not None else None
        if wrap is not None:
            wrap = ops.to_device_async(wrap, self._device())
        if inject is not None:
            inject = ops.to_device_async(inject[0], self._device())
        perturb = ops.to_device_async(pag_t[1], self._device()) if pag_t is not None else None
        acc = self.map_accumulator(B, cond_len, (H, W)) if attention_maps else None
        feats = self.features(x, r, cond, aw, B if aw is not None else 0, w_len=w_len, wrap=wrap, regional=regional,
                              maps=(None, B, acc) if attention_maps else None, inject=inject,
                              lora=ops.lora_device(lora_t, self._device()), perturb=perturb)
        logits = self.logits_from_features(feats, B, H, W)
        if attention_maps:
            return logits, self.finalize_attention_maps(acc, (H, W), cond_len, 1)
        return logits

    def token_scores(self, x, r, targets, byt5, clip=None, clip_image=None, *, label_smoothing=0.0, cfg=None,
                     unconditional_inputs=None, attn_weights=None, tiling=None, prompt_regions=None, lora=None) -> TokenScores:
        """How likely the denoiser finds ``targets`` given the noised tokens ``x`` at noise level ``r``: per token the statistics
        of train.py's objective (src/train.py:36,64,71), from one fused out_mapper + log-softmax kernel whose logits never reach
        HBM (pb200_paella_token_scores).  Returns TokenScores(nll, loss, argmax):
          nll     fp32 [B, H, W]  -log_softmax(logits)[target] = logsumexp(l) - l_y;
          loss    fp32 [B, H, W]  (1 - eps) nll + eps (logsumexp(l) - mean_j l_j), which is
                                  nn.CrossEntropyLoss(label_smoothing=eps, reduction='none'); at eps = 0 the nll tensor itself;
          argmax  int64 [B, H, W] the lowest code with the largest logit (pred.argmax(1)).
        ``targets``: int64 [B, H, W] on the model's device; a code outside [0, num_labels) gives a NaN nll and loss in its token
        only.  ``cfg``: None (the conditional logits), a number, or a CPU tensor [B] of per-sample scales: each sample is then
        scored under the guided logits u + cfg (c - u) of the CFG pair batch the sampling loop builds, the distribution sample()
        draws from at temperature 1, with ``unconditional_inputs`` (default: zeros like the conditioning, as in sample_notebook).
        ``attn_weights``, ``tiling`` and ``prompt_regions`` mean what they mean in ``forward`` and apply to the conditional rows;
        ``lora`` means what it means in ``forward`` and applies to the sample's conditional and unconditional rows.
        ValueError, before anything is enqueued, for bad targets, an eps outside [0, 1] and a bad cfg, attn_weights, tiling,
        prompt_regions or lora; TypeError for any other keyword argument."""
        B, H, W = x.shape
        eps = ops.check_label_smoothing(label_smoothing)
        self._check_score_targets(targets, x.shape)
        setup = self._score_setup(B, (H, W), {"byt5": byt5, "clip": clip, "clip_image": clip_image}, unconditional_inputs, cfg,
                                  attn_weights, tiling, prompt_regions, lora)
        return self._score_tokens(setup, x, r, targets, eps)

    def _check_score_targets(self, targets, shape, name: str = "targets") -> None:
        if not torch.is_tensor(targets) or targets.dtype != torch.int64 or targets.device != self._device() \
                or tuple(targets.shape) != tuple(shape):
            got = f"{targets.dtype} {list(targets.shape)} on {targets.device}" if torch.is_tensor(targets) else type(targets).__name__
            raise ValueError(f"{name}: expected int64 codes of shape {list(shape)} on {self._device()} (got {got})")

    def _score_setup(self, batch: int, latent_hw, model_inputs, unconditional_inputs, cfg, attn_weights, tiling, prompt_regions,
                     lora=None):
        """token_scores' per-call state, reused by every forward of utils.score: validates the arguments (ValueError before
        anything is enqueued), then builds the conditioning and the device tables of the conditional rows."""
        H, W = int(latent_hw[0]), int(latent_hw[1])
        params = ops.score_cfg_params(cfg, batch)
        wrap = ops.tiling_table(tiling, batch)
        regions = ops.regional_table(prompt_regions, batch, (H, W), self._device())
        ops.check_regions_unweighted(regions, attn_weights)
        lora_t = ops.lora_table(lora, batch, self)
        cond_len = self.conditioning_seq_len(model_inputs)
        w_table = None
        if isinstance(attn_weights, (list, tuple)):
            w_table = ops.attn_weights_table(attn_weights, batch, [self.max_attn_weights((H, W), cond_len)] * batch)
        if params is not None and unconditional_inputs is None:
            unconditional_inputs = {k: (torch.zeros_like(v) if torch.is_tensor(v) else [torch.zeros_like(t) for t in v])
                                    for k, v in model_inputs.items() if v is not None}
        dev = self._device()
        aw, w_len = attn_weights, None
        if w_table is not None:
            aw, w_len = ops.attn_weights_to_device(*w_table, dev)
        extra = [g for own in regions[1] for g in own] if regions is not None else []
        regional = None
        if params is None and regions is None and lora_t is None:
            cond = self._cond_for_forward(model_inputs["byt5"], model_inputs.get("clip"), model_inputs.get("clip_image"), (H, W))
        else:
            groups = [model_inputs] + ([unconditional_inputs] if params is not None else [])
            entries = ops.lora_entries(lora_t, batch)
            cond = self.prepare_conditioning(groups, (H, W), extra=extra, lora=[entries] * len(groups) if lora_t is not None else None,
                                             extra_lora=[entries[b] for b, own in enumerate(regions[1]) for _ in own]
                                             if regions is not None else None)
            regional = self.regional_device(regions, cond) if regions is not None else None
        return {"batch": batch, "hw": (H, W), "cond": cond, "aw": aw, "w_len": w_len, "regional": regional,
                "lora": ops.lora_device(lora_t, dev),
                "wrap": ops.to_device_async(wrap, dev) if wrap is not None else None,
                "params": ops.to_device_async(params, dev) if params is not None else None}

    def _score_tokens(self, setup, x, r, targets, eps: float) -> TokenScores:
        """One scoring forward on ``_score_setup``'s state: the features of the conditional (and, with cfg, unconditional) rows,
        then pb200_paella_token_scores."""
        B, (H, W) = setup["batch"], setup["hw"]
        if tuple(x.shape) != (B, H, W):
            raise ValueError(f"x of shape {list(x.shape)}; expected {[B, H, W]}")
        params, aw = setup["params"], setup["aw"]
        guided = params is not None
        feats = self.features(x, r, setup["cond"], aw, B if aw is not None else 0, cfg_pairs=guided, w_len=setup["w_len"],
                              wrap=setup["wrap"], regional=setup["regional"], lora=setup.get("lora"))
        L, dev = lib(), self._device()
        with torch.cuda.device(dev):
            nll = torch.empty(B, H, W, dtype=torch.float32, device=dev)
            smooth = torch.empty_like(nll)
            argmax = torch.empty(B, H, W, dtype=torch.int64, device=dev)
            ws = self._ws(L.pb200_paella_token_scores_workspace_bytes(self._handle, B, H * W))
            check(L.pb200_paella_token_scores(self._handle, ptr(feats), B, B if guided else 0, H * W, ptr(params),
                                              ptr(targets.contiguous()), ptr(nll), ptr(smooth), ptr(argmax), ptr(ws), ws.numel(),
                                              current_stream()), "pb200_paella_token_scores")
        return TokenScores(nll, ops.smoothed_loss(nll, smooth, eps), argmax)

    def _cond_for_forward(self, byt5, clip, clip_image, hw):
        """The reference's own loop calls ``model(x, t, **inputs)`` twice per step with the SAME conditioning tensors
        (ref/src/utils.py:42-45): the conditioning cache (44 kv_mapper + K/V GEMMs) is memoised on the identity and version
        of those tensor objects (references are held, so an address cannot be recycled under the memo) and the weights."""
        self._ensure_packed()
        ci = list(clip_image) if isinstance(clip_image, (list, tuple)) else [clip_image]
        ts = [byt5, clip] + ci
        try:
            vers = tuple(None if t is None else t._version for t in ts)
        except RuntimeError:        # inference tensors carry no version counter: no memo
            vers = None
        # a few entries, most recent first: the loop alternates between the conditional and the unconditional inputs
        memos = self._cond_single if isinstance(self._cond_single, list) else []
        if vers is not None:
            for i, memo in enumerate(memos):
                if (memo["hw"] == tuple(hw) and memo["vers"] == vers and len(memo["ts"]) == len(ts)
                        and all(a is b for a, b in zip(memo["ts"], ts)) and memo["key"] == self._packed_key):
                    if i:
                        memos.insert(0, memos.pop(i))
                    return memo["cond"]
        cond = self.prepare_conditioning([{"byt5": byt5, "clip": clip, "clip_image": clip_image}], hw, share_uniform=False)
        if vers is not None:
            memos.insert(0, {"hw": tuple(hw), "vers": vers, "ts": ts, "cond": cond, "key": self._packed_key})
            del memos[4:]
            self._cond_single = memos
        return cond

    def token_logprob(self, feats: torch.Tensor, batch: int, n_pairs: int, hw: int, params: torch.Tensor,
                      tokens: torch.Tensor) -> torch.Tensor:
        """fp32 log_softmax(l * (1/T))[token] per token, shaped like ``tokens`` (int64, batch * hw codes on the device): l the logits
        of the fp16 operand the fused sampler reads from ``feats`` (sample_tokens_pairs' rows: samples b < n_pairs mixed with their
        unconditional rows by ``params`` [batch, 3], the others cast) and 1/T params column 2 (pb200_paella_token_logprob, whose
        logits never reach HBM).  The confidence of confidence-guided renoising (utils module docstring)."""
        self._ensure_packed()
        L = lib()
        dev = self._device()
        with torch.cuda.device(dev):
            out = torch.empty(tokens.shape, dtype=torch.float32, device=dev)
            ws = self._ws(L.pb200_paella_token_scores_workspace_bytes(self._handle, batch, hw))
            check(L.pb200_paella_token_logprob(self._handle, ptr(feats), batch, n_pairs, hw, ptr(params), ptr(tokens.contiguous()),
                                               ptr(out), ptr(ws), ws.numel(), current_stream()), "pb200_paella_token_logprob")
        return out

    def add_noise(self, x, t, mask=None, random_x=None, generator=None, src=None, region=None, confidence=None,
                  choice_temperature=0.0):
        """ref/src/modules.py:277-283 on torch's random stream (``generator``: as in ``sample_tokens``).  ``src`` and ``region``
        (device tensors shaped like x, with mask=None): the tokens outside the region are src's and are never renoised
        (ops.add_noise).  ``confidence`` (fp32 like x, with mask=None: each token's log-probability, token_logprob) renoises each
        sample's floor(t N) least likely tokens instead, ranked by confidence + tau t Gumbel(u) on the uniforms this call draws
        anyway (utils module docstring; ops.renoise_confidence): ``choice_temperature`` is tau, one value >= 0, a list of B entries
        each None (add_noise's rule) or tau, or a device float32 [B] table (ops.confidence_table's encoding).  ``random_x`` (the
        replacement codes, e.g. the loop's initial noise) is required with confidence."""
        if confidence is not None:
            if mask is not None or random_x is None:
                raise ValueError("add_noise: confidence picks the mask itself and needs random_x (the replacement codes)")
            B = x.shape[0]
            if torch.is_tensor(choice_temperature):
                tau = choice_temperature
            else:
                tau = ops.confidence_table(choice_temperature, B, x[0].numel())
                tau = torch.full((B,), -1.0) if tau is None else tau
                tau = ops.to_device_async(tau, x.device)
            return ops.renoise_confidence(x, t, tau, confidence, random_x, generator, src=src, region=region)
        if mask is None:
            return ops.add_noise(x, t, random_x, self.num_labels, generator, src=src, region=region)
        if region is not None:
            raise ValueError("add_noise: region applies to the drawn mask (mask=None); with an explicit mask, pass mask & region")
        if random_x is None:
            random_x = ops.randint(self.num_labels, x.shape, x.device, generator)
        return torch.where(mask.bool(), random_x, x), mask

    def get_loss_weight(self, t, mask, min_val=0.3):    # ref/utils/modules.py:290-291 (training helper)
        return 1 - (1 - mask) * ((1 - t) * (1 - min_val))[:, None, None]
