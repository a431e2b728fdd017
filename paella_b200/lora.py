"""LoRA adapters: per-sample low-rank deltas on every AttnBlock's projections, and host-side merging into a state dict.

Adapter format: a plain state dict keyed by the reference's module paths (``{module}`` below), for each adapted module
  ``{module}.lora_A.weight``  [r, in]
  ``{module}.lora_B.weight``  [out, r]
  ``{module}.alpha``          optional 0-dim tensor, default r;
a sample with the adapter at scale s is the reference model with ``W + s * (alpha / r) * B @ A`` on each adapted module.

``load_lora`` packs an adapter for the per-sample path, which serves three targets of every AttnBlock ``{block}``:
  ``{block}.attention.attn.in_proj``   (q, k and v packed, as in ``in_proj_weight``)  A [r, c]       B [3c, r]
  ``{block}.attention.attn.out_proj``                                                 A [r, c]       B [c, r]
  ``{block}.kv_mapper.1``                                                             A [r, c_cond]  B [c, r]
``merge_lora`` folds any Linear, 1x1-conv or in_proj target into a plain state dict (the single-adapter deployment, and the way
to use adapters that also touch the ResBlock MLPs, TimestepBlocks, embedding, clf or out_mapper).

Packed blob layout (the one definition; pb200_lora_adapter in include/paella_b200.h reads it).  rp = r rounded up to a multiple
of 8.  For each AttnBlock in plan order (down_blocks then up_blocks, module order), for each target the adapter covers, in the
order in_proj, out_proj, kv_mapper, three parts, each starting on a 256-byte boundary:
  A    fp16 [rp][in]    lora_A, rows >= r zero
  B    fp16 [out][rp]   lora_B, columns >= r zero
  aux  fp32 [rp + 1]    the row sums of the fp16 A rows (the QKV GEMM's folded LayerNorm needs them), then alpha / r
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

from . import _lib

MAX_RANK = 64
TARGETS = (("attention.attn.in_proj", 1), ("attention.attn.out_proj", 2), ("kv_mapper.1", 4))     # pb200 target bits
_SUFFIXES = (".lora_A.weight", ".lora_B.weight", ".alpha")


def attn_blocks(cfg: dict) -> List[Tuple[str, int]]:
    """(module path, width) of every AttnBlock of a Paella config, in plan order."""
    out = []
    n = len(cfg["c_hidden"])
    for i in range(n):
        j = 1 if i > 0 else 0
        for _ in range(cfg["blocks"][i]):
            for kind in cfg["level_config"][i]:
                if kind == "A":
                    out.append((f"down_blocks.{i}.{j}", cfg["c_hidden"][i]))
                j += 1
    for ui, i in enumerate(reversed(range(n))):
        j = 0
        for _ in range(cfg["blocks"][i]):
            for kind in cfg["level_config"][i]:
                if kind == "A":
                    out.append((f"up_blocks.{ui}.{j}", cfg["c_hidden"][i]))
                j += 1
    return out


def served_targets(cfg: dict) -> Dict[str, Tuple[int, int, int, int]]:
    """module path -> (AttnBlock index, target bit, in, out) of every target the per-sample path serves."""
    out = {}
    for k, (pre, c) in enumerate(attn_blocks(cfg)):
        out[f"{pre}.attention.attn.in_proj"] = (k, 1, c, 3 * c)
        out[f"{pre}.attention.attn.out_proj"] = (k, 2, c, c)
        out[f"{pre}.kv_mapper.1"] = (k, 4, cfg["c_cond"], c)
    return out


def parse_lora(state_dict) -> Tuple[Dict[str, Tuple[torch.Tensor, torch.Tensor, float]], int]:
    """Validate the format of an adapter state dict -> ({module: (A fp32, B fp32, alpha)}, rank).  ValueError, naming the key, for
    a key that is not ``{module}.lora_A.weight`` / ``.lora_B.weight`` / ``.alpha``, A without B (or B without A), a rank outside
    1..64 or differing between modules, mismatched A/B ranks, and non-finite values."""
    mods: Dict[str, dict] = {}
    for key, v in state_dict.items():
        suffix = next((s for s in _SUFFIXES if key.endswith(s)), None)
        if suffix is None or len(key) == len(suffix):
            raise ValueError(f"lora: unknown key {key!r} (expected {{module}}.lora_A.weight, .lora_B.weight or .alpha)")
        if not torch.is_tensor(v):
            raise ValueError(f"lora: {key!r} is not a tensor")
        if not bool(torch.isfinite(v.detach().double()).all()):
            raise ValueError(f"lora: {key!r} has non-finite values")
        mods.setdefault(key[:-len(suffix)], {})[suffix] = v.detach()
    if not mods:
        raise ValueError("lora: the adapter has no modules")
    out, rank = {}, None
    for mod, parts in mods.items():
        a, b = parts.get(".lora_A.weight"), parts.get(".lora_B.weight")
        if a is None or b is None:
            missing = ".lora_B.weight" if b is None else ".lora_A.weight"
            raise ValueError(f"lora: {mod + missing!r} is missing ({mod!r} needs both lora_A and lora_B)")
        if a.dim() == 4 and a.shape[2:] == (1, 1):
            a = a[:, :, 0, 0]
        if b.dim() == 4 and b.shape[2:] == (1, 1):
            b = b[:, :, 0, 0]
        if a.dim() != 2 or b.dim() != 2 or a.shape[0] != b.shape[1]:
            raise ValueError(f"lora: {mod + '.lora_A.weight'!r} {list(a.shape)} and {mod + '.lora_B.weight'!r} {list(b.shape)} "
                             "are not [r, in] and [out, r]")
        r = a.shape[0]
        if not 1 <= r <= MAX_RANK:
            raise ValueError(f"lora: {mod + '.lora_A.weight'!r} has rank {r} (1..{MAX_RANK})")
        if rank is not None and r != rank:
            raise ValueError(f"lora: {mod + '.lora_A.weight'!r} has rank {r}, other modules {rank} (one rank per adapter)")
        rank = r
        alpha = parts.get(".alpha")
        if alpha is not None and alpha.numel() != 1:
            raise ValueError(f"lora: {mod + '.alpha'!r} must be a 0-dim tensor")
        out[mod] = (a.float().cpu(), b.float().cpu(), float(alpha) if alpha is not None else float(r))
    return out, rank


def _al(n: int) -> int:
    return (n + 255) // 256 * 256


def pack_lora(cfg: dict, modules, rank: int) -> Tuple[torch.Tensor, List[int]]:
    """The packed blob (CPU uint8, the layout of the module docstring) and the per-AttnBlock target bits of parsed modules."""
    served = served_targets(cfg)
    rp = (rank + 7) // 8 * 8
    targets = [0] * len(attn_blocks(cfg))
    for mod in modules:
        k, bit, _, _ = served[mod]
        targets[k] |= bit
    by_block = {(served[m][0], served[m][1]): m for m in modules}
    parts, n = [], 0
    for k in range(len(targets)):
        for _, bit in TARGETS:
            mod = by_block.get((k, bit))
            if mod is None:
                continue
            a, b, alpha = modules[mod]
            _, _, fin, fout = served[mod]
            a16 = torch.zeros(rp, fin, dtype=torch.float16)
            a16[:rank] = a.to(torch.float16)
            b16 = torch.zeros(fout, rp, dtype=torch.float16)
            b16[:, :rank] = b.to(torch.float16)
            aux = torch.zeros(rp + 1, dtype=torch.float32)
            aux[:rp] = a16.double().sum(1).float()
            aux[rp] = alpha / rank
            for t in (a16, b16, aux):
                raw = t.reshape(-1).view(torch.uint8)
                parts.append(raw)
                pad = _al(raw.numel()) - raw.numel()
                if pad:
                    parts.append(torch.zeros(pad, dtype=torch.uint8))
                n += _al(raw.numel())
    blob = torch.cat(parts) if parts else torch.zeros(0, dtype=torch.uint8)
    assert blob.numel() == n
    return blob, targets


def unpack_lora(cfg: dict, blob: torch.Tensor, rank: int, targets: List[int]) -> Dict[str, Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]:
    """Inverse of pack_lora on a CPU blob: {module: (A fp16 [rp, in], B fp16 [out, rp], aux fp32 [rp + 1])}."""
    rp = (rank + 7) // 8 * 8
    blocks = attn_blocks(cfg)
    out, off = {}, 0
    for k, bits in enumerate(targets):
        pre, c = blocks[k]
        for name, bit in TARGETS:
            if not bits & bit:
                continue
            fin = cfg["c_cond"] if bit == 4 else c
            fout = 3 * c if bit == 1 else c
            got = []
            for shape, dt, size in (((rp, fin), torch.float16, 2), ((fout, rp), torch.float16, 2), ((rp + 1,), torch.float32, 4)):
                nb = math.prod(shape) * size
                got.append(blob[off:off + nb].clone().view(dt).view(shape))
                off += _al(nb)
            out[f"{pre}.{name}"] = tuple(got)
    return out


class LoraAdapter:
    """A LoRA adapter packed for the per-sample path of one model configuration, on one device (load_lora).  Pass it as
    ``lora=`` to Paella.forward, token_scores, utils.sample* and utils.score, alone or as (adapter, scale)."""

    def __init__(self, blob: torch.Tensor, rank: int, targets: List[int], config: dict, modules: List[str]):
        self.blob, self.rank, self.targets, self.config, self.modules = blob, rank, list(targets), dict(config), list(modules)
        self.device = blob.device
        self._c = _lib.LoraAdapter()
        self._c.blob = blob.data_ptr()
        self._c.rank = rank
        for k, bits in enumerate(targets):
            self._c.targets[k] = bits

    @property
    def nbytes(self) -> int:
        return self.blob.numel()

    def __repr__(self):
        return f"LoraAdapter(rank={self.rank}, modules={len(self.modules)}, {self.nbytes} bytes on {self.device})"


def load_lora(model, state_dict) -> LoraAdapter:
    """Validate an adapter state dict against ``model``'s configuration and pack it in fp16 on the model's device.
    ValueError, naming the key, for a target the per-sample path does not serve (use merge_lora), an unknown key, a shape that
    does not match the configuration, A without B, a rank outside 1..64 and non-finite values."""
    cfg = model._cfg
    modules, rank = parse_lora(state_dict)
    served = served_targets(cfg)
    known = {k[:-len(".weight")] for k in model.state_dict() if k.endswith(".weight")}
    for mod, (a, b, _) in modules.items():
        if mod not in served:
            if mod in known:
                raise ValueError(f"lora: {mod + '.lora_A.weight'!r}: the per-sample path serves only the AttnBlocks' in_proj, "
                                 f"out_proj and kv_mapper.1; fold {mod!r} into the weights with merge_lora")
            raise ValueError(f"lora: unknown key {mod + '.lora_A.weight'!r}: {mod!r} is not a module of this model")
        _, _, fin, fout = served[mod]
        if tuple(a.shape) != (rank, fin) or tuple(b.shape) != (fout, rank):
            raise ValueError(f"lora: {mod!r}: A {list(a.shape)} and B {list(b.shape)}, expected [{rank}, {fin}] and [{fout}, {rank}]")
    if len(attn_blocks(cfg)) > _lib.PB200_LORA_MAX_ATTN_BLOCKS:
        raise ValueError(f"lora: {len(attn_blocks(cfg))} AttnBlocks (at most {_lib.PB200_LORA_MAX_ATTN_BLOCKS})")
    blob, targets = pack_lora(cfg, modules, rank)
    dev = model._device()
    return LoraAdapter(blob.to(dev), rank, targets, cfg, sorted(modules))


def merge_lora(state_dict, lora_state_dict, scale: float = 1.0) -> dict:
    """A copy of the model state dict ``state_dict`` with the adapter folded in: W + scale * (alpha / r) * B @ A, computed in fp64
    and stored in W's dtype, for every Linear or 1x1-conv target ({module}.weight) and for in_proj ({block}.attention.attn.
    in_proj_weight).  Host-side; load the result with load_state_dict (the model repacks its weights).  ValueError for an
    unknown module, a target that is not a Linear or 1x1 conv, a shape mismatch and everything parse_lora rejects."""
    if isinstance(scale, bool) or not isinstance(scale, (int, float)) or not math.isfinite(scale):
        raise ValueError(f"merge_lora: scale must be a finite real number (got {scale!r})")
    modules, rank = parse_lora(lora_state_dict)
    out = dict(state_dict)
    for mod, (a, b, alpha) in modules.items():
        key = mod + ".weight"
        if mod.endswith(".in_proj") and mod + "_weight" in state_dict:
            key = mod + "_weight"
        if key not in state_dict:
            raise ValueError(f"merge_lora: unknown key {mod + '.lora_A.weight'!r}: no {key!r} in the state dict")
        w = state_dict[key]
        shape = tuple(w.shape)
        if len(shape) == 4 and shape[2:] != (1, 1) or len(shape) not in (2, 4):
            raise ValueError(f"merge_lora: {key!r} {list(shape)} is not a Linear or 1x1-conv weight")
        if (shape[0], shape[1]) != (b.shape[0], a.shape[1]):
            raise ValueError(f"merge_lora: {mod!r}: A {list(a.shape)} and B {list(b.shape)} do not fit {key!r} {list(shape)}")
        delta = (float(scale) * alpha / rank) * (b.double() @ a.double())
        out[key] = (w.detach().cpu().double() + delta.reshape(shape)).to(w.dtype).to(w.device)
    return out
