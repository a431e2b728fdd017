#!/usr/bin/env python
"""Generate tests/golden/regional_tiny.npz by running the REAL reference on CPU with regional prompts.

Needs a reference checkout, found and loaded as make_golden.py finds and loads it ($PAELLA_REFERENCE):
    python tests/golden/make_golden_regional.py
The weights and the 8 x 8 inputs are those of the committed paella_tiny.npz.  Each sample's conditioning is its own prompt's
gen_c_embeddings followed by each region prompt's, concatenated along the sequence and zero-padded to the longest sample; each
Attention2D's nn.MultiheadAttention gets the boolean attn_mask of the footprint rule (see oracle/regional.py).  That is the users'
own idiom on unmodified weights: nothing inside the reference modules changes.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import TINY, load_reference     # noqa: E402



def regions(n):
    """Per sample, its list of bool [n, n] regions: sample 0 two overlapping ones with an uncovered area, sample 1 a quadrant
    and an empty region."""
    h = n // 2
    a0 = torch.zeros(n, n, dtype=torch.bool)
    a0[:, :h] = True
    b0 = torch.zeros(n, n, dtype=torch.bool)
    b0[n // 4:3 * n // 4, n // 4:] = True
    a1 = torch.zeros(n, n, dtype=torch.bool)
    a1[:h, :h] = True
    return [[a0, b0], [a1, torch.zeros(n, n, dtype=torch.bool)]]


def allowed(regs, n, stride, lens, S):
    """bool [B, P, P + S]: position p of sample b may attend to every self key and to prompt k's rows (laid out in order
    after the self keys) iff some token of its stride x stride footprint lies in region k (k >= 1), or in no region (k = 0)."""
    g = n // stride
    P = g * g
    out = torch.zeros(len(regs), P, P + S, dtype=torch.bool)
    out[:, :, :P] = True
    for b, rs in enumerate(regs):
        cover = torch.zeros(n, n, dtype=torch.bool)
        for r in rs:
            cover |= r
        tok = [~cover] + list(rs)                       # tokens carrying bit k
        off = P
        for k, t in enumerate(tok):
            pos = t.view(g, stride, g, stride).any(3).any(1).reshape(P)
            out[b, :, off:off + lens[b][k]] = pos[:, None]
            off += lens[b][k]
    return out


class _MaskedMHA(torch.nn.Module):
    """nn.MultiheadAttention called with the boolean attn_mask (True = not allowed) of its query count."""

    def __init__(self, mha, masks):
        super().__init__()
        self.mha, self.masks = mha, masks

    def forward(self, q, k, v, **kw):
        allow = self.masks[q.shape[1]]                                   # [B, P, P + S]
        m = (~allow).repeat_interleave(self.mha.num_heads, dim=0)      # [B * nhead, P, P + S]
        return self.mha(q, k, v, attn_mask=m, **kw)


def regional():
    torch.set_grad_enabled(False)
    _, ref_nb_modules, _, _, _ = load_reference()
    z = np.load(os.path.join(HERE, "paella_tiny.npz"))
    psd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd:")}
    x8, r = torch.from_numpy(z["x"]), torch.from_numpy(z["r"])
    byt5, clip, clip_image = (torch.from_numpy(z[k]) for k in ("byt5", "clip", "clip_image"))
    B = x8.shape[0]
    g = torch.Generator().manual_seed(11)
    out = {}
    # region prompts: sample 0's first with clip, its second byt5 only; sample 1's with clip and clip_image
    rp = [[dict(byt5=torch.randn(1, 3, TINY["byt5_embd"], generator=g), clip=torch.randn(1, TINY["clip_embd"], generator=g)),
           dict(byt5=torch.randn(1, 7, TINY["byt5_embd"], generator=g))],
          [dict(byt5=torch.randn(1, 4, TINY["byt5_embd"], generator=g), clip=torch.randn(1, TINY["clip_embd"], generator=g),
                clip_image=torch.randn(1, TINY["clip_embd"], generator=g)),
           dict(byt5=torch.randn(1, 2, TINY["byt5_embd"], generator=g))]]
    for b, own in enumerate(rp):
        for k, p in enumerate(own):
            for key, v in p.items():
                out[f"rp{b}{k}_{key}"] = v.numpy()
    x16 = torch.randint(0, TINY["num_labels"], (B, 16, 16), generator=g)
    out["x16"] = x16.numpy()
    for n, x in ((8, x8), (16, x16)):
        regs = regions(n)
        for b, rs in enumerate(regs):
            for k, reg in enumerate(rs):
                out[f"reg{n}_{b}{k}"] = reg.numpy()
        torch.manual_seed(0)
        m = ref_nb_modules.Paella(**TINY).eval()
        m.load_state_dict(psd)
        gen = m.gen_c_embeddings
        seqs = [torch.cat([gen(byt5[b:b + 1], clip[b:b + 1], clip_image[b:b + 1])[0]] +
                          [gen(p["byt5"], p.get("clip"), p.get("clip_image"))[0] for p in rp[b]]) for b in range(B)]
        lens = [[gen(byt5[b:b + 1], clip[b:b + 1], clip_image[b:b + 1]).shape[1]] +
                [gen(p["byt5"], p.get("clip"), p.get("clip_image")).shape[1] for p in rp[b]] for b in range(B)]
        S = max(s.shape[0] for s in seqs)
        c_embed = torch.stack([torch.nn.functional.pad(s, (0, 0, 0, S - s.shape[0])) for s in seqs])
        m.gen_c_embeddings = lambda *a: c_embed
        ps = TINY["patch_size"]
        masks_by_p = {(n // (ps << lvl)) ** 2: allowed(regs, n, ps << lvl, lens, S) for lvl in range(len(TINY["c_hidden"]))}
        for mod in m.modules():
            if isinstance(mod, ref_nb_modules.Attention2D):
                mod.attn = _MaskedMHA(mod.attn, masks_by_p)
        out[f"logits_{n}"] = m(x, r, byt5, clip=clip, clip_image=clip_image).numpy()
    np.savez_compressed(os.path.join(HERE, "regional_tiny.npz"), **out)
    print("regional_tiny.npz:", {k: v.shape for k, v in out.items() if k.startswith("logits")})


if __name__ == "__main__":
    regional()
