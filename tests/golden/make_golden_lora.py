#!/usr/bin/env python
"""Generate tests/golden/lora_tiny.npz by running the REAL reference on CPU with LoRA-merged weights.

Needs a reference checkout, found and loaded as make_golden.py finds and loads it ($PAELLA_REFERENCE):
    python tests/golden/make_golden_lora.py
The weights are those of the committed paella_tiny.npz.  Two adapters are drawn from a seeded CPU generator, both with non-zero
B (a LoRA initialised the usual way, B = 0, would change nothing and test nothing):
  a  rank 4, alpha = r, on in_proj, out_proj and kv_mapper.1 of every AttnBlock;
  b  rank 16, alpha = 8, on in_proj and kv_mapper.1 of the down AttnBlocks and out_proj of the up ones.
A batch of four samples runs under [a, None, (b, 0.5), (a, 2.0)]: sample i's logits are the reference Paella's forward on the
state dict with W + s (alpha / r) B A merged in (oracle/lora.py's definition, formed here in float64 and stored in fp32), so the
fixture pins the definition to the reference modules.  Also stored: the base model's logits of the same batch.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import ROOT, TINY, load_reference     # noqa: E402

sys.path.insert(0, ROOT)
from oracle.lora import merge      # noqa: E402

ATTN = ["down_blocks.1.3", "down_blocks.1.6", "down_blocks.2.3", "up_blocks.0.2", "up_blocks.1.2", "up_blocks.1.5"]     # every AttnBlock


def adapters(g):
    c, cc = 64, TINY["c_cond"]

    def mod(rank, fin, fout, b_std=0.1):
        return torch.randn(rank, fin, generator=g) / fin ** 0.5, torch.randn(fout, rank, generator=g) * b_std
    a, b = {}, {}
    for pre in ATTN:
        for name, fin, fout in (("attention.attn.in_proj", c, 3 * c), ("attention.attn.out_proj", c, c), ("kv_mapper.1", cc, c)):
            A, B = mod(4, fin, fout)
            a[f"{pre}.{name}.lora_A.weight"], a[f"{pre}.{name}.lora_B.weight"] = A, B
            use = name != "attention.attn.out_proj" if pre.startswith("down") else name == "attention.attn.out_proj"
            if use:
                A, B = mod(16, fin, fout, 0.25)
                b[f"{pre}.{name}.lora_A.weight"], b[f"{pre}.{name}.lora_B.weight"] = A, B
                b[f"{pre}.{name}.alpha"] = torch.tensor(8.0)
    return a, b


def main():
    torch.set_grad_enabled(False)
    _, ref_nb_modules, _, _, _ = load_reference()
    z = np.load(os.path.join(HERE, "paella_tiny.npz"))
    psd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd:")}
    g = torch.Generator().manual_seed(41)
    la, lb = adapters(g)
    B, H, L = 4, 8, 5
    x = torch.randint(0, TINY["num_labels"], (B, H, H), generator=g)
    r = torch.rand(B, generator=g)
    byt5 = torch.randn(B, L, TINY["byt5_embd"], generator=g)
    clip = torch.randn(B, TINY["clip_embd"], generator=g)
    entries = [(la, 1.0), None, (lb, 0.5), (la, 2.0)]
    torch.manual_seed(0)
    m = ref_nb_modules.Paella(**TINY).eval()
    m.load_state_dict(psd)
    attn = sorted(n for n, mod in m.named_modules() if type(mod).__name__ == "AttnBlock")
    assert attn == sorted(ATTN), attn
    base = m(x, r, byt5, clip)
    logits = []
    for i, e in enumerate(entries):
        m.load_state_dict(psd if e is None else merge(psd, e[0], e[1]))
        logits.append(m(x[i:i + 1], r[i:i + 1], byt5[i:i + 1], clip[i:i + 1]))
    out = {"x": x.numpy(), "r": r.numpy(), "byt5": byt5.numpy(), "clip": clip.numpy(), "logits": torch.cat(logits).numpy(),
           "logits_base": base.numpy(), "scales": np.array([1.0, 0.0, 0.5, 2.0], dtype=np.float32),
           "which": np.array([0, -1, 1, 0], dtype=np.int32)}
    out.update({"a:" + k: v.numpy() for k, v in la.items()})
    out.update({"b:" + k: v.numpy() for k, v in lb.items()})
    np.savez_compressed(os.path.join(HERE, "lora_tiny.npz"), **out)
    print("lora_tiny.npz:", len(out), "arrays; max |logits - base| per sample:",
          [float((torch.cat(logits) - base)[i].abs().max()) for i in range(B)])


if __name__ == "__main__":
    main()
