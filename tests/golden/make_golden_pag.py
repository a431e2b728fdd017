#!/usr/bin/env python
"""Generate tests/golden/pag_tiny.npz: perturbed-attention guidance on the REAL reference denoiser, on CPU.

Needs a reference checkout, found and loaded as make_golden.py finds and loads it ($PAELLA_REFERENCE):
    python tests/golden/make_golden_pag.py
The weights and inputs are those of the committed paella_tiny.npz.  The script installs the reference's CustomMultiheadAttention
with its own replace_attention_layers, the notebook's idiom, then replaces the forward of the listed AttnBlocks' attentions (module
order = plan order) by the perturbed attention: it projects q, k and v with the module's own in_proj weights, takes the per-head
softmax of q k^T / sqrt(head_dim) over [self ; conditioning] keys, multiplies it by the sample's attn_weights on the last keys
(post-softmax, not renormalised), sends the self keys' total probability to the query's own value and the conditioning keys'
probabilities to their values, and applies the module's out_proj.  Sample 0 is perturbed, sample 1 is not.  Cases:
  deep     8 x 8, the deepest level's AttnBlocks (down and up), the default blocks; that level has one position at 8 x 8, where
           the perturbed attention is the plain one
  all      8 x 8, every AttnBlock
  down     8 x 8, AttnBlock 0 alone
  attnw    8 x 8, every AttnBlock, weights longer than the conditioning (w_len > S: they reach into the self keys)
  x16      16 x 16, the deepest level's AttnBlocks
  mix      8 x 8, every AttnBlock: the unconditional logits (zero conditioning) and the mixed logits with CFG (cfg 3, s 2) and without (s 2)
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import TINY, load_reference     # noqa: E402

CFG, SCALE = 3.0, 2.0


def perturbed_forward(mod, index, plan):
    """A CustomMultiheadAttention forward (batch_first) whose rows in plan['rows'] are perturbed when index is in plan['blocks']."""
    def forward(q_in, k_in, v_in, **kwargs):
        E, nh = mod.embed_dim, mod.num_heads
        hd = E // nh
        wq, wk, wv = mod.in_proj_weight.chunk(3, dim=0)
        bq, bk, bv = mod.in_proj_bias.chunk(3, dim=0)

        def heads(t, w, b):
            y = F.linear(t, w, b)
            return y.view(y.shape[0], y.shape[1], nh, hd).transpose(1, 2)
        q, k, v = heads(q_in, wq, bq), heads(k_in, wk, bk), heads(v_in, wv, bv)
        prob = torch.softmax((q @ k.transpose(-2, -1)) / (hd ** 0.5), dim=-1)       # [B, nh, Nq, Nk]
        w = kwargs.get("attn_weights")
        if w is not None:
            prob = prob.clone()
            prob[..., -w.shape[0]:] *= w
        o = prob @ v
        n = q_in.shape[1]                   # Attention2D: kv = cat([x, kv]), the first n keys are the queries' own tokens
        if index in plan["blocks"]:
            for b in plan["rows"]:
                o[b] = prob[b, :, :, n:] @ v[b, :, n:] + prob[b, :, :, :n].sum(-1, keepdim=True) * v[b, :, :n]
        o = o.transpose(1, 2).reshape(q_in.shape[0], n, E)
        return mod.out_proj(o), None
    return forward


def pag():
    torch.set_grad_enabled(False)
    _, ref_nb_modules, ref_alter, _, _ = load_reference()
    z = np.load(os.path.join(HERE, "paella_tiny.npz"))
    psd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd:")}
    x8, r = torch.from_numpy(z["x"]), torch.from_numpy(z["r"])
    byt5, clip, clip_image = (torch.from_numpy(z[k]) for k in ("byt5", "clip", "clip_image"))
    B = x8.shape[0]
    g = torch.Generator().manual_seed(31)
    x16 = torch.randint(0, TINY["num_labels"], (B, 16, 16), generator=g)
    S = byt5.shape[1] + 2 * TINY["clip_seq_len"]
    aw = torch.rand(S + 1, generator=g) + 0.5          # the deepest level at 8 x 8 has 1 self key: the longest vector there

    torch.manual_seed(0)
    m = ref_nb_modules.Paella(**TINY).eval()
    m.load_state_dict(psd)
    ref_alter.replace_attention_layers(m)
    mods = [mod for mod in m.modules() if isinstance(mod, ref_alter.CustomMultiheadAttention)]
    plan = {}
    for i, mod in enumerate(mods):
        mod.forward = perturbed_forward(mod, i, plan)
    n_blocks = len(mods)
    deep = [n_blocks // 2 - 1, n_blocks // 2]          # TINY: one AttnBlock at the deepest level, down and up

    def run(x, cond, blocks, rows=(0,), weights=None):
        plan["blocks"], plan["rows"] = set(blocks), list(rows)
        kw = {"attn_weights": weights} if weights is not None else {}
        return m(x, r, cond["byt5"], clip=cond["clip"], clip_image=cond["clip_image"], **kw).numpy()

    own = dict(byt5=byt5, clip=clip, clip_image=clip_image)
    zero = {k: torch.zeros_like(v) for k, v in own.items()}
    out = {"x16": x16.numpy(), "attn_weights": aw.numpy(), "deep": np.array(deep), "n_blocks": np.array(n_blocks),
           "cfg": np.array(CFG), "scale": np.array(SCALE)}
    out["logits_plain"] = run(x8, own, [])
    out["logits_deep"] = run(x8, own, deep)
    out["logits_all"] = run(x8, own, range(n_blocks))
    out["logits_down"] = run(x8, own, [0])
    out["logits_attnw"] = run(x8, own, range(n_blocks), weights=aw)
    out["logits_attnw_plain"] = run(x8, own, [], weights=aw)
    out["logits_x16"] = run(x16, own, deep)
    out["logits_x16_plain"] = run(x16, own, [])
    lc, lp = torch.from_numpy(out["logits_plain"]).double(), torch.from_numpy(out["logits_all"]).double()
    lu = torch.from_numpy(run(x8, zero, [])).double()
    out["logits_uncond"] = lu.numpy()
    out["mix_cfg"] = (lu + CFG * (lc - lu) + SCALE * (lc - lp)).numpy()
    out["mix_nocfg"] = (lc + SCALE * (lc - lp)).numpy()
    np.savez_compressed(os.path.join(HERE, "pag_tiny.npz"), **out)
    print("pag_tiny.npz:", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    pag()
