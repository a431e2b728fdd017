#!/usr/bin/env python
"""Generate tests/golden/confidence_tiny.npz: confidence-guided renoising on the REAL reference's tiny denoiser, on CPU.

Needs a reference checkout, found and loaded as make_golden.py finds and loads it ($PAELLA_REFERENCE):
    python tests/golden/make_golden_confidence.py
The weights, conditioning, tokens and noise levels are those of the committed paella_tiny.npz.  The reference's forward gives the
conditional logits and, under zero conditioning, the unconditional ones; the guided logits are the notebook's
pred * cfg + uncond * (1 - cfg).  Each case then holds, for a temperature T, a choice temperature tau, a noise level t and
optionally a region:
  logp   torch.log_softmax(fp32(logits * (1/T)).double(), 1) at the drawn tokens (float64 [B, H, W]);
  u      the uniforms torch.rand_like draws on a CUDA generator at (SEED, OFFSET) on a 132-SM H100, from oracle/philox.py;
  mask   the tokens renoised: per sample the floor(fp32(t N)) candidates of smallest fp32 key logp + fp32(tau t) (-log(-log u)),
         ties to the lower index, ranked here with torch's stable sort (NaN keys first).
The "ties" case replaces the logits by one row repeated at every token, with two codes drawn, so half the tokens share one key.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from make_golden import TINY, load_reference     # noqa: E402
from oracle import philox                        # noqa: E402

CFG = 3.0
SEED, OFFSET, SM_COUNT = 1234, 8, 132
# name, logits, T, tau, t, region
CASES = [
    ("cond_T1_tau0", "cond", 1.0, 0.0, 0.5, False),
    ("cond_T02_tau2", "cond", 0.2, 2.0, 0.75, False),
    ("cond_T3_tau2", "cond", 3.0, 2.0, 0.3, False),
    ("guided_T1_tau2", "guided", 1.0, 2.0, 0.5, False),
    ("guided_T02_tau0", "guided", 0.2, 0.0, 0.6, False),
    ("guided_T3_tau0_region", "guided", 3.0, 0.0, 0.5, True),
    ("cond_T1_tau2_region", "cond", 1.0, 2.0, 0.9, True),
    ("ties_tau0", "ties", 1.0, 0.0, 0.4, False),
    ("cond_t0", "cond", 1.0, 2.0, 0.0, False),
    ("guided_t1", "guided", 1.0, 2.0, 1.0, False),
]


def select(logp, u, tau, t, region):
    """The renoised tokens of one sample (flat), independently of oracle/confidence.py."""
    g = -torch.log(-torch.log(u))
    k = logp.float() + torch.tensor(tau, dtype=torch.float32) * torch.tensor(t, dtype=torch.float32) * g
    k = torch.where(torch.isnan(k), torch.tensor(-float("inf")), k)      # NaN first (below -inf: stable sort puts index order)
    cand = region.nonzero().flatten()
    n = int(min(torch.floor(torch.tensor(t, dtype=torch.float32) * torch.tensor(float(len(cand)), dtype=torch.float32)), len(cand)))
    order = torch.sort(k[cand], stable=True).indices
    m = torch.zeros_like(region)
    m[cand[order[:n]]] = True
    return m


def main():
    torch.set_grad_enabled(False)
    _, ref_nb_modules, _, _, _ = load_reference()
    z = np.load(os.path.join(HERE, "paella_tiny.npz"))
    psd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd:")}
    x, r = torch.from_numpy(z["x"]), torch.from_numpy(z["r"])
    byt5, clip, clip_image = (torch.from_numpy(z[k]) for k in ("byt5", "clip", "clip_image"))
    B, H, W = x.shape
    torch.manual_seed(0)
    m = ref_nb_modules.Paella(**TINY).eval()
    m.load_state_dict(psd)
    cond = m(x, r, byt5, clip, clip_image)
    uncond = m(x, r, torch.zeros_like(byt5), torch.zeros_like(clip), torch.zeros_like(clip_image))
    logits = {"cond": cond, "guided": cond * CFG + uncond * (1 - CFG)}
    g = torch.Generator().manual_seed(41)
    tokens = torch.randint(0, TINY["num_labels"], (B, H, W), generator=g)
    region = torch.rand(B, H, W, generator=g) < 0.6
    ties_row = cond[:1, :, :1, :1].expand(B, -1, H, W).contiguous()
    ties_tokens = torch.where(torch.rand(B, H, W, generator=g) < 0.5, torch.tensor(5), torch.tensor(9))
    u = torch.from_numpy(philox.rand(B * H * W, SEED, OFFSET, SM_COUNT).reshape(B, H, W))

    out = {"cfg": np.array(CFG), "tokens": tokens.numpy(), "ties_tokens": ties_tokens.numpy(), "region": region.numpy(),
           "logits_cond": cond.numpy(), "logits_guided": logits["guided"].numpy(), "logits_ties": ties_row.numpy(),
           "u": u.numpy(), "seed": np.array(SEED), "offset": np.array(OFFSET), "sm_count": np.array(SM_COUNT),
           "names": np.array([c[0] for c in CASES])}
    for name, which, T, tau, t, use_region in CASES:
        lg = ties_row if which == "ties" else logits[which]
        tk = ties_tokens if which == "ties" else tokens
        inv_t = torch.tensor(1.0 / T, dtype=torch.float32)
        lp = torch.log_softmax((lg * inv_t).double(), 1).gather(1, tk[:, None]).squeeze(1)
        masks = []
        for b in range(B):
            reg = region[b].flatten() if use_region else torch.ones(H * W, dtype=torch.bool)
            masks.append(select(lp[b].flatten(), u[b].flatten(), tau, t, reg).view(H, W))
        out[f"{name}:params"] = np.array([T, tau, t, float(use_region)])
        out[f"{name}:which"] = np.array(which)
        out[f"{name}:logp"] = lp.numpy()
        out[f"{name}:mask"] = torch.stack(masks).numpy()
    np.savez_compressed(os.path.join(HERE, "confidence_tiny.npz"), **out)
    print("confidence_tiny.npz:", len(out), "arrays;", {c[0]: int(out[f"{c[0]}:mask"].sum()) for c in CASES})


if __name__ == "__main__":
    main()
