"""Pin the oracle to the reference at the reference-default size (1.008 B denoiser, f4 VQGAN): the oracle's outputs against
what the unmodified reference computed on the same weights and inputs, stored in tests/golden/default_ref.npz (seeded
samples of the logits and the decoded image, the latents in full; tests/golden/make_golden.py --default writes it).  The weights
are this package's modules initialised like the reference's (same seed, same parameter order) and re-randomised."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_golden as mg
    from paella_b200 import modules, vqgan
    with torch.no_grad():
        inputs = mg.default_inputs(modules, vqgan)
    return inputs, np.load(os.path.join(ROOT, "tests", "golden", "default_ref.npz"))


def test_default_denoiser_forward(golden):
    from oracle import paella_oracle as po
    (m, cond, x, r, _, _, _, (pick, _)), g = golden
    assert sum(p.numel() for p in m.parameters()) == 1008350592
    with torch.no_grad():
        got = po.paella_forward(m.state_dict(), po.PaellaConfig(byt5_embd=2560), x, r, cond["byt5"], cond["clip"], cond["clip_image"])
    assert float(g["logits_std"]) > 0.05          # re-randomised: logits are not identically zero (SURVEY F3)
    torch.testing.assert_close(got.reshape(-1)[torch.from_numpy(pick)], torch.from_numpy(g["logits"]), rtol=1e-3, atol=2e-5)


def test_default_vqgan_conv_stacks(golden):
    from oracle import vqgan_oracle as vo
    (_, _, _, _, vq, img, idx, (_, pick_dec)), g = golden
    sd = vq.state_dict()
    with torch.no_grad():
        torch.testing.assert_close(vo.encode_latents(sd, img).permute(0, 3, 1, 2), torch.from_numpy(g["latents"]), rtol=1e-3, atol=2e-5)
        torch.testing.assert_close(vo.decode_indices(sd, idx).reshape(-1)[torch.from_numpy(pick_dec)], torch.from_numpy(g["decoded"]),
                                   rtol=1e-3, atol=2e-5)
