#!/usr/bin/env python
"""Generate tests/golden/attention_maps_tiny.npz by running the REAL reference on CPU with attention maps.

Needs a reference checkout, found and loaded as make_golden.py finds and loads it ($PAELLA_REFERENCE):
    python tests/golden/make_golden_attention_maps.py
The weights and inputs are those of the committed paella_tiny.npz.  The script installs the reference's CustomMultiheadAttention
with its own replace_attention_layers, the notebook's idiom, and calls each one with need_weights=True (Attention2D passes False,
so the script overrides the keyword and records the returned matrix).  Each forward's matrices [B, nhead, P, P + S] are then
aggregated per the definition of DESIGN.md §3: the heads' mean on the conditioning keys, upsampled to the token grid by nearest
neighbour, averaged over the AttnBlocks.  Cases: the 8 x 8 forward with and without attn_weights, a 16 x 16 forward, and a forward
with two clip_image embeddings.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import TINY, load_reference     # noqa: E402


def maps_of(calls, S, n):
    """[B, S, n, n] from the recorded [B, nhead, P, P + S] matrices, in call order."""
    out = 0
    for a in calls:
        B, _, P, Nk = a.shape
        g = int(round(P ** 0.5))
        m = a.mean(1)[:, :, Nk - S:].transpose(1, 2).reshape(B, S, g, g)
        out = out + m.repeat_interleave(n // g, 2).repeat_interleave(n // g, 3)
    return out / len(calls)


def attention_maps():
    torch.set_grad_enabled(False)
    _, ref_nb_modules, ref_alter, _, _ = load_reference()
    z = np.load(os.path.join(HERE, "paella_tiny.npz"))
    psd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd:")}
    x8, r = torch.from_numpy(z["x"]), torch.from_numpy(z["r"])
    byt5, clip, clip_image = (torch.from_numpy(z[k]) for k in ("byt5", "clip", "clip_image"))
    aw = torch.from_numpy(z["attn_weights"])
    B = x8.shape[0]
    g = torch.Generator().manual_seed(23)
    x16 = torch.randint(0, TINY["num_labels"], (B, 16, 16), generator=g)
    clip_image2 = torch.randn(B, TINY["clip_embd"], generator=g)

    torch.manual_seed(0)
    m = ref_nb_modules.Paella(**TINY).eval()
    m.load_state_dict(psd)
    ref_alter.replace_attention_layers(m)
    calls = []
    for mod in m.modules():
        if isinstance(mod, ref_alter.CustomMultiheadAttention):
            fwd = mod.forward

            def forced(*a, _fwd=fwd, **kw):
                kw["need_weights"] = True
                x, att = _fwd(*a, **kw)
                calls.append(att)
                return x, att
            mod.forward = forced

    out = {"x16": x16.numpy(), "clip_image2": clip_image2.numpy()}
    cases = {
        "plain": (x8, dict(clip=clip, clip_image=clip_image)),
        "attnw": (x8, dict(clip=clip, clip_image=clip_image, attn_weights=aw)),
        "x16": (x16, dict(clip=clip, clip_image=clip_image)),
        "img2": (x8, dict(clip=clip, clip_image=[clip_image, clip_image2])),
    }
    for name, (x, kw) in cases.items():
        calls.clear()
        S = m.gen_c_embeddings(byt5, kw["clip"], kw["clip_image"]).shape[1]
        out[f"logits_{name}"] = m(x, r, byt5, **kw).numpy()
        out[f"maps_{name}"] = maps_of(calls, S, x.shape[1]).numpy()
        out[f"n_attn_{name}"] = np.array(len(calls))
    np.savez_compressed(os.path.join(HERE, "attention_maps_tiny.npz"), **out)
    print("attention_maps_tiny.npz:", {k: v.shape for k, v in out.items() if k.startswith("maps")})


if __name__ == "__main__":
    attention_maps()
