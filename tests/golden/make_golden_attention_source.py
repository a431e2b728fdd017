#!/usr/bin/env python
"""Generate tests/golden/attention_source_tiny.npz: prompt-to-prompt injection on the REAL reference denoiser, on CPU.

Needs a reference checkout, found and loaded as make_golden.py finds and loads it ($PAELLA_REFERENCE):
    python tests/golden/make_golden_attention_source.py
The weights and inputs are those of the committed paella_tiny.npz.  The script installs the reference's CustomMultiheadAttention
with its own replace_attention_layers, the notebook's idiom, then replaces each one's forward by a replay: it projects q, k and
v with the module's own in_proj weights, takes the per-head softmax of q k^T / sqrt(head_dim), copies the source row's
probabilities into each edit's row, multiplies the edit's by its own attn_weights on the last keys (post-softmax, not
renormalised), and applies them to the edit's own values and the module's out_proj.  Cases (batch 2, sample 1 the edit of sample
0 unless stated):
  prompt   8 x 8, the two samples on different prompts and tokens
  attnw    8 x 8, the edit on the source's prompt with attn_weights (attention re-weighting)
  x16      16 x 16, different prompts
  self     8 x 8, each sample its own source: the replay of the unpatched forward, stored beside the unpatched logits
"""
import math
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import TINY, load_reference     # noqa: E402


def replay_forward(mod, plan):
    """A CustomMultiheadAttention forward (batch_first) that replays plan['src'][b]'s probabilities in row b."""
    def forward(q_in, k_in, v_in, **kwargs):
        E, nh = mod.embed_dim, mod.num_heads
        hd = E // nh
        wq, wk, wv = mod.in_proj_weight.chunk(3, dim=0)
        bq, bk, bv = mod.in_proj_bias.chunk(3, dim=0)

        def heads(t, w, b):
            y = F.linear(t, w, b)
            return y.view(y.shape[0], y.shape[1], nh, hd).transpose(1, 2)
        q, k, v = heads(q_in, wq, bq), heads(k_in, wk, bk), heads(v_in, wv, bv)
        prob = torch.softmax((q @ k.transpose(-2, -1)) / math.sqrt(hd), dim=-1)       # [B, nh, Nq, Nk]
        prob = prob[torch.tensor(plan["src"])]
        for b, w in enumerate(plan["weights"]):
            if w is not None:
                prob[b, :, :, -w.shape[0]:] *= w
        o = (prob @ v).transpose(1, 2).reshape(q_in.shape[0], q_in.shape[1], E)
        return mod.out_proj(o), None
    return forward


def attention_source():
    torch.set_grad_enabled(False)
    _, ref_nb_modules, ref_alter, _, _ = load_reference()
    z = np.load(os.path.join(HERE, "paella_tiny.npz"))
    psd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd:")}
    x8, r = torch.from_numpy(z["x"]), torch.from_numpy(z["r"])
    byt5, clip, clip_image = (torch.from_numpy(z[k]) for k in ("byt5", "clip", "clip_image"))
    aw = torch.from_numpy(z["attn_weights"])
    B = x8.shape[0]
    g = torch.Generator().manual_seed(29)
    x16 = torch.randint(0, TINY["num_labels"], (B, 16, 16), generator=g)

    torch.manual_seed(0)
    m = ref_nb_modules.Paella(**TINY).eval()
    m.load_state_dict(psd)
    ref_alter.replace_attention_layers(m)
    plan = {}
    patched = [(mod, mod.forward, replay_forward(mod, plan)) for mod in m.modules()
               if isinstance(mod, ref_alter.CustomMultiheadAttention)]

    def run(x, cond, src, weights=(None, None), replay=True):
        plan["src"], plan["weights"] = list(src), list(weights)
        for mod, orig, rep in patched:
            mod.forward = rep if replay else orig
        return m(x, r, cond["byt5"], clip=cond["clip"], clip_image=cond["clip_image"]).numpy()

    own = dict(byt5=byt5, clip=clip, clip_image=clip_image)
    same = {k: v[:1].expand(B, *v.shape[1:]).contiguous() for k, v in own.items()}      # both samples on sample 0's prompt
    out = {"x16": x16.numpy(), "same_byt5": same["byt5"].numpy(), "same_clip": same["clip"].numpy(),
           "same_clip_image": same["clip_image"].numpy()}
    out["logits_prompt"] = run(x8, own, [0, 0])
    out["logits_attnw"] = run(x8, same, [0, 0], (None, aw))
    out["logits_x16"] = run(x16, own, [0, 0])
    out["logits_self"] = run(x8, own, [0, 1])
    out["logits_plain"] = run(x8, own, [0, 1], replay=False)
    np.savez_compressed(os.path.join(HERE, "attention_source_tiny.npz"), **out)
    print("attention_source_tiny.npz:", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    attention_source()
