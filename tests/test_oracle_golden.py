"""Pin the CPU oracle (oracle/) to the golden vectors produced by the real reference
(tests/golden/make_golden.py).  CPU only."""
import numpy as np
import torch

from helpers import load_golden, oracle_cfg, t
from oracle import paella_oracle as po
from oracle import vqgan_oracle as vo

TOL = dict(rtol=2e-4, atol=2e-5)


def test_r_and_c_embeddings():
    cfg, sd, g = load_golden("paella_tiny.npz")
    oc = oracle_cfg(cfg)
    torch.testing.assert_close(po.r_embedding(t(g["r"]), oc.c_r), t(g["r_embed"]), rtol=1e-5, atol=1e-6)
    ce = po.c_embeddings(sd, oc, t(g["byt5"]), t(g["clip"]), t(g["clip_image"]))
    torch.testing.assert_close(ce, t(g["c_embed"]), **TOL)


def test_forward_logits_and_taps():
    cfg, sd, g = load_golden("paella_tiny.npz")
    oc = oracle_cfg(cfg)
    taps = {}
    lg = po.paella_forward(sd, oc, t(g["x"]), t(g["r"]), t(g["byt5"]), t(g["clip"]), t(g["clip_image"]), taps=taps)
    torch.testing.assert_close(lg, t(g["logits"]), **TOL)
    n = 0
    for k, v in g.items():
        if k.startswith("tap:"):
            got = taps[k[4:]].permute(0, 3, 1, 2)
            torch.testing.assert_close(got, t(v), **TOL)
            n += 1
    assert n >= 10


def test_forward_conditioning_variants():
    cfg, sd, g = load_golden("paella_tiny.npz")
    oc = oracle_cfg(cfg)
    a = (t(g["x"]), t(g["r"]), t(g["byt5"]))
    torch.testing.assert_close(po.paella_forward(sd, oc, *a, t(g["clip"])), t(g["logits_noimg"]), **TOL)
    torch.testing.assert_close(po.paella_forward(sd, oc, *a), t(g["logits_byt5only"]), **TOL)


def test_attn_weights_variant():
    cfg, sd, g = load_golden("paella_tiny.npz")
    oc = oracle_cfg(cfg)
    a = (t(g["x"]), t(g["r"]), t(g["byt5"]), t(g["clip"]), t(g["clip_image"]))
    torch.testing.assert_close(po.paella_forward(sd, oc, *a, attn_weights=t(g["attn_weights"])), t(g["logits_attnw"]), **TOL)
    torch.testing.assert_close(po.paella_forward(sd, oc, *a), t(g["logits_custom_mha"]), **TOL)


def test_add_noise():
    cfg, sd, g = load_golden("paella_tiny.npz")
    out, mask = po.add_noise(t(g["x"]), t(g["an_t"]), t(g["an_random_x"]), t(g["an_u"]))
    assert torch.equal(out, t(g["an_out"])) and torch.equal(mask, t(g["an_mask"]))


def test_sample_loop_tokens():
    cfg, sd, _ = load_golden("paella_tiny.npz")
    _, _, s = load_golden("sample_tiny.npz")
    oc = oracle_cfg(cfg)
    byt5, clip = t(s["byt5"]), t(s["clip"])
    draws = {"init": t(s["init"]), "q": [t(q) for q in s["q"]], "u": [t(u) for u in s["u"]]}
    toks = po.sample(sd, oc, {"byt5": byt5, "clip": clip}, tuple(s["init"].shape),
                     {"byt5": torch.zeros_like(byt5), "clip": torch.zeros_like(clip)},
                     steps=int(s["steps"]), renoise_steps=int(s["renoise_steps"]), temperature=(1.0, 0.2),
                     cfg_scale=8.0, draws=draws)
    assert torch.equal(toks, t(s["tokens"]))


def test_vqgan_conv_stacks():
    cfg, sd, g = load_golden("vqgan_tiny.npz")
    lat = vo.encode_latents(sd, t(g["img"]))
    torch.testing.assert_close(lat.permute(0, 3, 1, 2), t(g["latents"]), **TOL)
    nb = cfg["bottleneck_blocks"]
    dec = vo.decode_latents(sd, sd["vquantizer.codebook.weight"][t(g["idx_rand"])], n_bottleneck=nb)
    torch.testing.assert_close(dec, t(g["dec_rand"]), **TOL)
    dec2 = vo.decode_latents(sd, (t(g["qe"]) * 0.3764).permute(0, 2, 3, 1), n_bottleneck=nb)
    torch.testing.assert_close(dec2, t(g["dec"]), **TOL)


def test_vqgan_oracle_fp64_stays_fp64():
    """An fp64 run of the codec oracle is fp64 throughout: both k4s2 convolutions match torch's own fp64 convolutions to
    fp64 rounding (an fp32 intermediate would leave ~1e-7 relative error), and encode / decode return fp64."""
    import torch.nn.functional as F
    cfg, sd, g = load_golden("vqgan_tiny.npz")
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(2, 6, 10, 8, dtype=torch.float64, generator=gen)                          # NHWC
    w = torch.randn(5, 8, 4, 4, dtype=torch.float64, generator=gen)
    b = torch.randn(5, dtype=torch.float64, generator=gen)
    got = vo.conv_k4s2p1(x, w, b)
    want = F.conv2d(x.permute(0, 3, 1, 2), w, b, stride=2, padding=1).permute(0, 2, 3, 1)
    assert got.dtype == torch.float64 and float((got - want).abs().max()) < 1e-12
    wt = torch.randn(8, 5, 4, 4, dtype=torch.float64, generator=gen)
    got = vo.convT_k4s2p1(x, wt, b)
    want = F.conv_transpose2d(x.permute(0, 3, 1, 2), wt, b, stride=2, padding=1).permute(0, 2, 3, 1)
    assert got.dtype == torch.float64 and float((got - want).abs().max()) < 1e-12
    lat = vo.encode_latents(sd64, t(g["img"]).double())
    dec = vo.decode_latents(sd64, sd64["vquantizer.codebook.weight"][t(g["idx_rand"])], n_bottleneck=cfg["bottleneck_blocks"])
    assert lat.dtype == torch.float64 and dec.dtype == torch.float64
    torch.testing.assert_close(lat.permute(0, 3, 1, 2).float(), t(g["latents"]), **TOL)


def test_vq_nearest_definitions_agree():
    """C oracle (exact fmaf) == fp64 emulation == brute force argmin on well-separated data."""
    g = torch.Generator().manual_seed(0)
    cb = torch.randn(512, 4, generator=g)
    x = torch.randn(4096, 4, generator=g)
    a = vo.vq_nearest(x, cb)
    d = ((x[:, None, :].double() - cb[None].double()) ** 2).sum(-1)
    top2 = torch.topk(d, 2, dim=1, largest=False)
    safe = (top2.values[:, 1] - top2.values[:, 0]) > 1e-5
    assert torch.equal(a[safe], top2.indices[safe, 0])
    assert safe.float().mean() > 0.99
    # tie-break: duplicate codes -> lowest index wins
    cb2 = torch.cat([cb[:8], cb[:8]])
    assert int(vo.vq_nearest(cb[:8].clone(), cb2).max()) < 8
    lib = vo._c_oracle()
    if lib:
        saved, vo._C_LIB = vo._C_LIB, False
        try:
            b = vo.vq_nearest(x, cb)
        finally:
            vo._C_LIB = saved
        assert torch.equal(a, b)
