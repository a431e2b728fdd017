#!/usr/bin/env python
"""Generate tests/golden/scores_tiny.npz by running the REAL reference on CPU with train.py's objective.

Needs a reference checkout, found and loaded as make_golden.py finds and loads it ($PAELLA_REFERENCE):
    python tests/golden/make_golden_scores.py
The weights and conditioning are those of the committed paella_tiny.npz.  Clean tokens and their noised versions are drawn here
from a seeded CPU generator and stored, so a test needs no random numbers.  For the reference's denoiser `pred = model(noised,
r, byt5, clip, clip_image)` the fixture holds src/train.py's nn.CrossEntropyLoss(label_smoothing=0.1, reduction='none')(pred,
latents), the same loss at label_smoothing 0 and pred.argmax(1); then the same three for the notebook's guided logits
pred * cfg + uncond * (1 - cfg), uncond being the forward under zero conditioning.
"""
import os
import sys

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import TINY, load_reference     # noqa: E402

CFG = 3.0


def scores():
    torch.set_grad_enabled(False)
    _, ref_nb_modules, _, _, _ = load_reference()
    z = np.load(os.path.join(HERE, "paella_tiny.npz"))
    psd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd:")}
    r = torch.from_numpy(z["r"])
    byt5, clip, clip_image = (torch.from_numpy(z[k]) for k in ("byt5", "clip", "clip_image"))
    B = byt5.shape[0]
    g = torch.Generator().manual_seed(31)
    latents = torch.randint(0, TINY["num_labels"], (B, 8, 8), generator=g)
    mask = torch.rand(B, 8, 8, generator=g) <= r[:, None, None]
    noised = torch.where(mask, torch.randint(0, TINY["num_labels"], (B, 8, 8), generator=g), latents)

    torch.manual_seed(0)
    m = ref_nb_modules.Paella(**TINY).eval()
    m.load_state_dict(psd)
    pred = m(noised, r, byt5, clip, clip_image)
    uncond = m(noised, r, torch.zeros_like(byt5), torch.zeros_like(clip), torch.zeros_like(clip_image))
    guided = pred * CFG + uncond * (1 - CFG)

    out = {"latents": latents.numpy(), "noised": noised.numpy(), "cfg": np.array(CFG)}
    for name, logits in (("cond", pred), ("guided", guided)):
        out[f"loss_smooth_{name}"] = nn.CrossEntropyLoss(label_smoothing=0.1, reduction="none")(logits, latents).numpy()
        out[f"loss_{name}"] = nn.CrossEntropyLoss(reduction="none")(logits, latents).numpy()
        out[f"argmax_{name}"] = logits.argmax(1).numpy()
    np.savez_compressed(os.path.join(HERE, "scores_tiny.npz"), **out)
    print("scores_tiny.npz:", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    scores()
