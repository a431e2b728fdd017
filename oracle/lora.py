"""LoRA merging in fp64 on an oracle (reference-layout) state dict.

An adapter (A [r, in], B [out, r], alpha) on module M at scale s is the reference model with
    W_M' = W_M + s * (alpha / r) * B @ A,
W_M being ``M.weight`` (a Linear, or a 1x1 conv viewed as [out, in]) or, for ``{block}.attention.attn.in_proj``, the packed
``in_proj_weight``.  Nothing else changes, so the oracle of a sample with an adapter is the unmodified oracle forward on the merged
state dict.
"""
from __future__ import annotations

from typing import Dict

import torch
from torch import Tensor


def merge(sd: Dict[str, Tensor], lora_sd: Dict[str, Tensor], scale: float = 1.0) -> Dict[str, Tensor]:
    """A copy of ``sd`` with the adapter ``lora_sd`` ({M}.lora_A.weight, {M}.lora_B.weight, optional {M}.alpha) merged at
    ``scale``: the sum is formed in float64 and stored in each weight's dtype."""
    out = dict(sd)
    mods = sorted({k.rsplit(".lora_", 1)[0] for k in lora_sd if ".lora_" in k})
    for m in mods:
        a = lora_sd[m + ".lora_A.weight"].double()
        b = lora_sd[m + ".lora_B.weight"].double()
        a, b = a.reshape(a.shape[0], -1), b.reshape(b.shape[0], -1)
        r = a.shape[0]
        alpha = float(lora_sd[m + ".alpha"]) if m + ".alpha" in lora_sd else float(r)
        key = m + "_weight" if m.endswith(".in_proj") else m + ".weight"
        w = sd[key]
        out[key] = (w.double() + (scale * alpha / r) * (b @ a).reshape(w.shape)).to(w.dtype)
    return out
