"""GPU parity tests of the denoiser and the sampling loop through the reference-shaped Python API
(paella_b200.modules.Paella / paella_b200.utils.sample) against the golden vectors of the real reference
(tiny config) and against the CPU oracle (reference-default 1.008 B config).

Tolerances: the CUDA path rounds GEMM operands to fp16 (fp32 accumulate, fp32 residual stream).  Emulating
exactly that rounding in the oracle (oracle.paella_oracle.mm_f16_operands) moves the default model's logits
(std 0.18) by 8e-4 max / 1.4e-4 rms; the kernels add fp16 storage of the MLP hidden, q/k/v and softmax
weights.  Bounds below (max-abs / rms): default 1.008 B model (logit std 0.177) 2.5e-3 / 4e-4; tiny golden model 7e-3 / 1.2e-3.
"""
import json
import os

import pytest
import torch

from helpers import load_golden, oracle_cfg, t

pytestmark = pytest.mark.gpu
DEV = "cuda"
MAX_ABS, RMS = 7e-3, 1.2e-3             # tiny golden config
MAX_ABS_D, RMS_D = 2.5e-3, 4e-4         # reference-default config


def _log(name, payload):
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "model_parity.jsonl"), "a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


def _errs(got, want):
    d = (got.float().cpu() - want.float().cpu())
    return float(d.abs().max()), float(d.pow(2).mean().sqrt())


@pytest.fixture(scope="module")
def tiny():
    from paella_b200.modules import Paella
    cfg, sd, g = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m, cfg, sd, g


def test_tiny_forward_matches_reference_golden(tiny):
    m, cfg, sd, g = tiny
    a = dict(byt5=t(g["byt5"]).to(DEV), clip=t(g["clip"]).to(DEV), clip_image=t(g["clip_image"]).to(DEV))
    x, r = t(g["x"]).to(DEV), t(g["r"]).to(DEV)
    out = m(x, r, **a)
    assert out.shape == tuple(g["logits"].shape) and out.dtype == torch.float32
    mx, rms = _errs(out, t(g["logits"]))
    _log("tiny_forward", {"max_abs": mx, "rms": rms})
    assert mx < MAX_ABS and rms < RMS
    mx, rms = _errs(m(x, r, a["byt5"], clip=a["clip"]), t(g["logits_noimg"]))
    assert mx < MAX_ABS and rms < RMS
    mx, rms = _errs(m(x, r, a["byt5"]), t(g["logits_byt5only"]))
    assert mx < MAX_ABS and rms < RMS


def test_tiny_attn_weights_and_list_clip_image(tiny):
    m, cfg, sd, g = tiny
    x, r = t(g["x"]).to(DEV), t(g["r"]).to(DEV)
    byt5, clip, ci = t(g["byt5"]).to(DEV), t(g["clip"]).to(DEV), t(g["clip_image"]).to(DEV)
    out = m(x, r, byt5, clip=clip, clip_image=ci, attn_weights=t(g["attn_weights"]).to(DEV))
    mx, rms = _errs(out, t(g["logits_attnw"]))
    _log("tiny_attn_weights", {"max_abs": mx, "rms": rms})
    assert mx < MAX_ABS and rms < RMS
    # list-valued clip_image with one entry == tensor-valued (ref/utils/modules.py:228-235)
    out2 = m(x, r, byt5, clip=clip, clip_image=[ci])
    mx, _ = _errs(out2, t(g["logits"]))
    assert mx < MAX_ABS


def test_tiny_r_and_c_embeddings_match_reference_golden(tiny):
    """Paella.gen_r_embedding / gen_c_embeddings (ref/src/modules.py:212-232) vs the reference's own outputs."""
    m, cfg, sd, g = tiny
    re = m.gen_r_embedding(t(g["r"]).to(DEV)).cpu()
    assert float((re - t(g["r_embed"])).abs().max()) < 2e-4        # sin/cos of arguments up to 1e4 in fp32
    ce = m.gen_c_embeddings(t(g["byt5"]).to(DEV), t(g["clip"]).to(DEV), t(g["clip_image"]).to(DEV)).cpu()
    assert ce.shape == tuple(g["c_embed"].shape)
    mx, rms = _errs(ce, t(g["c_embed"]))
    _log("tiny_c_embed", {"max_abs": mx, "rms": rms})
    assert mx < 3.5e-3 and rms < 9e-4
    ce2 = m.gen_c_embeddings(t(g["byt5"]).to(DEV), None, [t(g["clip_image"]).to(DEV)] * 2)
    assert ce2.shape == (2, 5 + 8, cfg["c_cond"])


def test_tiny_forward_is_deterministic_and_batch_independent(tiny):
    m, cfg, sd, g = tiny
    x, r = t(g["x"]).to(DEV), t(g["r"]).to(DEV)
    byt5, clip = t(g["byt5"]).to(DEV), t(g["clip"]).to(DEV)
    a = m(x, r, byt5, clip=clip)
    b = m(x, r, byt5, clip=clip)
    assert float((a - b).abs().max()) < 1e-5        # GRN statistics use float atomics: not bit-reproducible
    # sample 1 alone == sample 1 inside the batch (no cross-sample op on the path)
    c = m(x[1:], r[1:], byt5[1:], clip=clip[1:])
    assert float((c - a[1:]).abs().max()) < 1e-4


def test_state_dict_keys_match_reference(tiny):
    m, cfg, sd, g = tiny
    assert set(m.state_dict().keys()) == set(sd.keys())
    for k, v in m.state_dict().items():
        assert tuple(v.shape) == tuple(sd[k].shape), k


def test_cpu_tensors_are_refused():
    from paella_b200 import _lib
    from paella_b200.modules import Paella
    cfg, sd, g = load_golden("paella_tiny.npz")
    m = Paella(**cfg).eval()
    with pytest.raises(_lib.PaellaB200Error):
        m(t(g["x"]), t(g["r"]), t(g["byt5"]))


@pytest.mark.parametrize("NL,B,H", [(8192, 8, 32), (8192, 3, 8), (8200, 2, 16), (64, 2, 8), (8192, 64, 32)])
def test_fused_sampler_matches_torch_multinomial(NL, B, H):
    """out_mapper GEMM + CFG + /T + multinomial in one kernel vs the same expression in torch ops, same seed.
    (8192, B=8/64) = full-grid torch launch policy (stride 37*8192: shared-Philox kernel, partial last block at B=8);
    (8192, 3x8x8) and (64, ...) = small-grid policies (rs = rows); 8200 labels = stride not a multiple of the label
    count -> generic per-element kernel."""
    from paella_b200.modules import Paella
    cfg, sd, g = load_golden("paella_tiny.npz")
    big = dict(cfg)
    big.update(c_in=256, c_out=256, num_labels=NL)
    torch.manual_seed(0)
    m = Paella(**big).to(DEV).eval()
    gen = torch.Generator(device=DEV).manual_seed(3)
    feats = torch.randn(2 * B * H * H, 256, device=DEV, generator=gen)
    W = m.out_mapper[1].weight.detach().view(NL, 256) * 30.0        # spread the logits
    with torch.no_grad():
        m.out_mapper[1].weight.copy_(W.view(NL, 256, 1, 1))
    m.pack_weights()
    n = B * H * H
    cfg_s, T = 8.0, 0.7
    a_mix = (feats[:n] * cfg_s + feats[n:] * (1 - cfg_s)).half().float()
    logits = a_mix @ W.half().float().t()
    p = torch.softmax(logits / T, dim=-1)
    del logits
    torch.manual_seed(42)
    want = torch.multinomial(p, 1)[:, 0].view(B, H, H)
    off_a = torch.cuda.default_generators[0].get_offset()
    torch.manual_seed(42)
    got = m.sample_tokens(feats, B, H, H, cfg_s, T)
    assert torch.cuda.default_generators[0].get_offset() == off_a
    agree = float((got == want).float().mean())
    _log("fused_sampler", {"NL": NL, "B": B, "H": H, "agree": agree, "n": n, "mismatch": int((got != want).sum())})
    assert agree > 0.999
    # no guidance
    del p
    torch.manual_seed(43)
    want2 = torch.multinomial(torch.softmax((feats[:n].half().float() @ W.half().float().t()) / T, dim=-1), 1)[:, 0].view(B, H, H)
    torch.manual_seed(43)
    got2 = m.sample_tokens(feats[:n].contiguous(), B, H, H, None, T)
    assert float((got2 == want2).float().mean()) > 0.999


def test_sample_loop_tiny_vs_oracle_one_step_and_rng_stream(tiny):
    """Each step of sample() from the same state: tokens vs the CPU oracle fed with torch's CUDA draws."""
    from oracle import paella_oracle as po
    from paella_b200 import utils as U
    m, cfg, sd, g = tiny
    oc = oracle_cfg(cfg)
    B, H, K = 2, 8, cfg["num_labels"]
    byt5, clip = t(g["byt5"]), t(g["clip"])
    cond = {"byt5": byt5.to(DEV), "clip": clip.to(DEV)}
    uncond = {"byt5": torch.zeros_like(byt5).to(DEV), "clip": torch.zeros_like(clip).to(DEV)}
    steps, renoise = 4, 3
    # the draws the reference loop would consume on this GPU
    torch.manual_seed(123)
    init = torch.randint(0, K, (B, H, H), device=DEV)
    qs, us = [], []
    for i in range(steps):
        qs.append(torch.empty(B * H * H, K, device=DEV).exponential_(1).cpu())
        if i < renoise:
            us.append(torch.rand(B, H, H, device=DEV).cpu())
    off_ref = torch.cuda.default_generators[0].get_offset()
    want = po.sample(sd, oc, {"byt5": byt5, "clip": clip}, (B, H, H), {"byt5": torch.zeros_like(byt5), "clip": torch.zeros_like(clip)},
                     steps=steps, renoise_steps=renoise, temperature=(1.0, 0.2), cfg_scale=8.0,
                     draws={"init": init.cpu(), "q": qs, "u": us})
    for exact in (True, False):
        torch.manual_seed(123)
        got = U.sample(m, cond, (B, H, H), uncond, steps=steps, renoise_steps=renoise, temperature=(1.0, 0.2), cfg=8.0,
                       exact=exact)
        assert torch.cuda.default_generators[0].get_offset() == off_ref     # consumed the stream like the reference
        agree = float((got.cpu() == want).float().mean())
        _log("sample_tiny", {"exact": exact, "agree": agree})
        assert agree > 0.9          # 128 tokens; fp16-vs-fp32 logits may flip a near-tie which then propagates


@pytest.fixture(scope="module")
def default_model():
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    return m.to(DEV), sd


def test_default_config_forward_vs_oracle(default_model):
    """Reference-default 1.008 B denoiser, 32x32 latents: CUDA logits vs the fp32 CPU oracle."""
    from oracle import paella_oracle as po
    from paella_b200.synth import synthetic_conditioning
    m, sd = default_model
    assert sum(p.numel() for p in m.parameters()) == 1008350592
    cond, _ = synthetic_conditioning(2, 24, with_clip_image=True)
    x = torch.randint(0, 8192, (2, 32, 32), generator=torch.Generator().manual_seed(1))
    r = torch.tensor([0.7, 0.15])
    want = po.paella_forward(sd, po.PaellaConfig(byt5_embd=2560), x, r, cond["byt5"], cond["clip"], cond["clip_image"])
    got = m(x.to(DEV), r.to(DEV), cond["byt5"].to(DEV), clip=cond["clip"].to(DEV), clip_image=cond["clip_image"].to(DEV))
    mx, rms = _errs(got, want)
    top1 = float((got.cpu().argmax(1) == want.argmax(1)).float().mean())
    _log("default_forward", {"max_abs": mx, "rms": rms, "logit_std": float(want.std()), "top1_agree": top1})
    assert mx < MAX_ABS_D and rms < RMS_D
    assert top1 > 0.97


def test_default_config_forward_64x64_vs_oracle(default_model):
    """SURVEY.md §8(d) cfg 4 geometry: 64x64 latents (Nq = 256 and 64 queries, Nk = 392 / 200 keys with clip_image),
    several query tiles per (sample, head) in the attention kernel, 16x16 / 8x8 depthwise grids."""
    from oracle import paella_oracle as po
    from paella_b200.synth import synthetic_conditioning
    m, sd = default_model
    cond, _ = synthetic_conditioning(1, 128, with_clip_image=True)
    x = torch.randint(0, 8192, (1, 64, 64), generator=torch.Generator().manual_seed(2))
    r = torch.tensor([0.45])
    want = po.paella_forward(sd, po.PaellaConfig(byt5_embd=2560), x, r, cond["byt5"], cond["clip"], cond["clip_image"])
    got = m(x.to(DEV), r.to(DEV), cond["byt5"].to(DEV), clip=cond["clip"].to(DEV), clip_image=cond["clip_image"].to(DEV))
    mx, rms = _errs(got, want)
    top1 = float((got.cpu().argmax(1) == want.argmax(1)).float().mean())
    _log("default_forward_64x64", {"max_abs": mx, "rms": rms, "logit_std": float(want.std()), "top1_agree": top1})
    assert mx < MAX_ABS_D and rms < RMS_D
    assert top1 > 0.97


def test_default_config_sample_runs_and_is_seed_deterministic(default_model):
    from paella_b200 import utils as U
    from paella_b200.synth import synthetic_conditioning
    m, _ = default_model
    cond, uncond = synthetic_conditioning(4, 32, device=DEV)
    torch.manual_seed(7)
    a = U.sample(m, cond, (4, 32, 32), uncond, steps=8, renoise_steps=7)
    torch.manual_seed(7)
    b = U.sample(m, cond, (4, 32, 32), uncond, steps=8, renoise_steps=7)
    assert a.shape == (4, 32, 32) and a.dtype == torch.int64
    assert int(a.min()) >= 0 and int(a.max()) < 8192
    same = float((a == b).float().mean())
    _log("default_sample_repeat", {"same": same})
    assert same > 0.999         # bit-identical RNG stream and order-independent (integer) GRN statistics


@pytest.mark.parametrize("which", ["tiny", "default"])
def test_cfg_pairs_prefix_sharing_is_exact(which, tiny, default_model):
    """The CFG batch evaluated with one (tokens, r) per pair (blocks before the first AttnBlock run once) must equal
    the plain 2B-sample forward bit for bit: it is the same arithmetic on the same inputs."""
    from paella_b200.synth import synthetic_conditioning
    m = tiny[0] if which == "tiny" else default_model[0]
    B, L = 3, 16
    kw = dict(byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features)
    cond, uncond = synthetic_conditioning(B, L, device=DEV, **kw)
    cache = m.prepare_conditioning([cond, uncond], (16, 16))
    x = torch.randint(0, m.num_labels, (B, 16, 16), device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    r = torch.tensor([0.9, 0.5, 0.1], device=DEV)
    full = m.features(torch.cat([x, x]), torch.cat([r, r]), cache)
    paired = m.features(x, r, cache, cfg_pairs=True)
    assert paired.shape == full.shape
    assert torch.equal(paired, full)
    assert not torch.equal(full[: full.shape[0] // 2], full[full.shape[0] // 2:])       # the two halves do differ


@pytest.mark.parametrize("which", ["tiny", "default"])
def test_shared_conditioning_slot_matches_per_sample_cache(which, tiny, default_model):
    """An unconditional group with identical rows is projected once and shared through the slot map: same features as
    the cache that stores every sample's K/V (the K/V GEMM runs on 1 x S instead of B x S rows; same per-element sums)."""
    from paella_b200.synth import synthetic_conditioning
    m = tiny[0] if which == "tiny" else default_model[0]
    B, L = 3, 16
    kw = dict(byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features)
    cond, uncond = synthetic_conditioning(B, L, device=DEV, **kw)
    shared = m.prepare_conditioning([cond, uncond], (16, 16))
    plain = m.prepare_conditioning([cond, uncond], (16, 16), share_uniform=False)
    assert shared.slots == B + 1 and shared.slot_map.tolist() == [0, 1, 2, 3, 3, 3]
    assert plain.slots == 2 * B and plain.slot_map is None
    x = torch.randint(0, m.num_labels, (B, 16, 16), device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    r = torch.tensor([0.8, 0.4, 0.2], device=DEV)
    a = m.features(x, r, shared, cfg_pairs=True)
    b = m.features(x, r, plain, cfg_pairs=True)
    mx, rms = _errs(a, b)
    _log("shared_cond_slot", {"which": which, "max_abs": mx, "rms": rms, "equal": bool(torch.equal(a, b))})
    assert mx < 1e-5


def test_notebook_sampler_modes_and_intermediates(tiny):
    """paella_inference.ipynb cell-3 signature: modes multinomial / argmax / quant, sampling_quant_steps, attn_weights,
    init_x, sampling_conditional_steps; returns (sampled, intermediates) with one entry per resample and per renoise."""
    from paella_b200 import utils as U
    from paella_b200.vqgan import VQModel
    m, cfg, sd, g = tiny
    byt5, clip, ci = t(g["byt5"]).to(DEV), t(g["clip"]).to(DEV), t(g["clip_image"]).to(DEV)
    cond = {"byt5": byt5, "clip": clip, "clip_image": ci}
    uncond = {"byt5": torch.zeros_like(byt5), "clip": torch.zeros_like(clip), "clip_image": None}
    vq = VQModel(levels=2, bottleneck_blocks=1, c_hidden=32, c_latent=4, codebook_size=cfg["num_labels"]).to(DEV)
    aw = torch.tensor([1.2, 1.2, 0.4, 0.4, 0.4], device=DEV)
    for mode in ("multinomial", "argmax", "quant"):
        torch.manual_seed(1)
        toks, inter = U.sample_notebook(m, cond, (2, 8, 8), uncond, steps=4, renoise_steps=2, mode=mode, attn_weights=aw, vqmodel=vq)
        assert toks.shape == (2, 8, 8) and len(inter) == 4 + 2
        assert int(toks.min()) >= 0 and int(toks.max()) < cfg["num_labels"]
    torch.manual_seed(2)
    a, _ = U.sample_notebook(m, cond, (2, 8, 8), uncond, steps=4, sampling_quant_steps=2, sampling_conditional_steps=3, vqmodel=vq,
                             init_x=torch.zeros(2, 8, 8, dtype=torch.int64, device=DEV))
    torch.manual_seed(2)
    b, _ = U.sample_notebook(m, cond, (2, 8, 8), uncond, steps=4, sampling_quant_steps=2, sampling_conditional_steps=3, vqmodel=vq,
                             init_x=torch.zeros(2, 8, 8, dtype=torch.int64, device=DEV))
    assert torch.equal(a, b)
    # argmax mode is deterministic and equals the argmax of the guided logits of a plain forward at step 0
    torch.manual_seed(3)
    c, inter = U.sample_notebook(m, cond, (2, 8, 8), uncond, steps=1, renoise_steps=0, mode="argmax", cfg=(3.0, 3.0))
    torch.manual_seed(3)
    from paella_b200 import ops
    x0 = ops.randint(cfg["num_labels"], (2, 8, 8), torch.device(DEV))
    r = torch.ones(2, device=DEV)
    lg = m(x0, r, byt5, clip=clip, clip_image=ci) * 3.0 + m(x0, r, uncond["byt5"], clip=uncond["clip"]) * (1 - 3.0)
    assert float((c == lg.argmax(dim=1)).float().mean()) > 0.98
