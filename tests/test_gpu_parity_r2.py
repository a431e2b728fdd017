"""Round-2 parity tests (VERDICT r1 "next" #1, #6, #9 and ADVICE): everything here compares the CUDA path with an
INDEPENDENT statement of the reference's arithmetic — the fp32 CPU oracle (pinned to the real reference by
tests/test_oracle_golden.py / test_oracle_vs_reference.py), plain torch ops of the published formula, or torch's own CUDA ops.

  * BASELINE config 1: reference-default 1.008 B denoiser, bs=1, 32x32, 8-step CFG sample() vs oracle.sample fed torch's CUDA
    draws — per-step token agreement (teacher-forced on the oracle's trajectory) and a top-2 margin audit of every mismatch
  * mixed-length CFG batch (cond with clip_image / longer byt5, uncond without) vs the oracle run per group
  * VQ indices vs the torchtools form  addmm(|c|^2 + |x|^2, x, c^T, alpha=-2).argmin  with a margin audit
  * torch.autocast-wrapped forward / sample (the notebook wraps everything in autocast, nb:349)
  * init_x / sampling_conditional_steps / per-step cfgs (sample_distributed) vs the oracle, teacher-forced
  * decode fused on the sampler tail: clamp / uint8 writers vs decode_indices(...).clamp(0,1) and save_image's byte conversion
  * packed checkpoints (on-disk blob) incl. {'state_dict': ...} wrapper, DDP 'module.' prefix and extra vquantizer.* EMA keys
  * a pre-packed VQGAN blob bound WITHOUT load_param (the broadcast receiver's situation: host-mirrored gammas)
  * stand-alone vqgan.ResBlock.forward; draws of > 2^29 elements (torch splits them into several kernels)
"""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
MAX_ABS_D = 2.5e-3          # asserted logits tolerance of the default model (tests/test_gpu_model.py)


def _log(name, payload):
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "parity_r2.jsonl"), "a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


@pytest.fixture(scope="module")
def default_model():
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    return m.to(DEV), sd


def _oracle_step(po, sd, oc, tokens, t, cond, uncond, cfg, temp, q):
    """One resample of ref/src/utils.py:42-50 in the oracle: -> (sampled, guided logits [N,K]) ."""
    B = tokens.shape[0]
    r = torch.full((B,), t)
    lc = po.paella_forward(sd, oc, tokens, r, **cond)
    lg = lc * cfg + po.paella_forward(sd, oc, tokens, r, **uncond) * (1 - cfg) if cfg is not None else lc
    K = lg.shape[1]
    flat = lg.permute(0, 2, 3, 1).reshape(-1, K)
    p = flat.div(temp).softmax(dim=-1)
    return torch.argmax(p / q, dim=-1).view(tokens.shape), flat


def _margin_audit(flat_logits, temp, q, want, got):
    """Every disagreement must be a near-tie of the oracle's own Gumbel scores  l_k / T - log q_k  between its choice and
    ours: returns (n_mismatch, worst score gap)."""
    bad = (want.view(-1) != got.view(-1)).nonzero().flatten()
    if bad.numel() == 0:
        return 0, 0.0
    score = flat_logits[bad].double() / temp - torch.log(q[bad].double())
    s_w = score.gather(1, want.view(-1)[bad][:, None])
    s_g = score.gather(1, got.view(-1)[bad][:, None])
    return int(bad.numel()), float((s_w - s_g).max())


def test_cfg1_default_sample_vs_oracle_per_step_with_margin_audit(default_model):
    """BASELINE.json configs[0]: the 'correctness plumbing' case.  Each of the 8 steps is run on the GPU from the ORACLE's state
    (teacher forcing, so one flipped near-tie does not snowball) with torch's CUDA generator positioned where the reference
    loop would have it; tokens must agree >= 99 % per step and every mismatch must be explained by a Gumbel-score gap below
    what the asserted logits tolerance allows: 2 * (|cfg| + |1-cfg|) * MAX_ABS / T.  The free-running sample() from the same
    seed is reported as a rate."""
    from oracle import paella_oracle as po
    from paella_b200 import ops
    from paella_b200 import utils as U
    from paella_b200.synth import synthetic_conditioning
    m, sd = default_model
    oc = po.PaellaConfig(byt5_embd=2560)
    B, H, K, steps, renoise, cfg = 1, 32, 8192, 8, 7, 8.0
    cond, uncond = synthetic_conditioning(B, 128)
    cond_d = {k: v.to(DEV) for k, v in cond.items()}
    uncond_d = {k: v.to(DEV) for k, v in uncond.items()}
    t_list = torch.linspace(1.0, 0.0, steps + 1)
    temps = torch.linspace(1.0, 0.2, steps)
    seed = 20240923

    # the reference loop's draws on THIS GPU, and the generator offset before each of them
    torch.manual_seed(seed)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    init = torch.randint(0, K, (B, H, H), device=DEV)
    offs_q, offs_u, qs, us = [], [], [], []
    for i in range(steps):
        offs_q.append(gen.get_offset())
        qs.append(torch.empty(B * H * H, K, device=DEV).exponential_(1).cpu())
        if i < renoise:
            offs_u.append(gen.get_offset())
            us.append(torch.rand(B, H, H, device=DEV).cpu())
    off_end = gen.get_offset()

    cache = m.prepare_conditioning([cond_d, uncond_d], (H, H))
    state = init.cpu()
    per_step, worst_gap, n_bad = [], 0.0, 0
    with torch.inference_mode():
        for i in range(steps):
            t, temp = float(t_list[i]), float(temps[i])
            want, flat = _oracle_step(po, sd, oc, state, t, cond, uncond, cfg, temp, qs[i])
            # GPU: same state, generator at the offset the reference loop has here
            gen.set_offset(offs_q[i])
            r = torch.full((B,), t, device=DEV)
            feats = m.features(state.to(DEV), r, cache, cfg_pairs=True)
            got = m.sample_tokens(feats, B, H, H, cfg, temp).cpu()
            agree = float((got == want).float().mean())
            nb, gap = _margin_audit(flat, temp, qs[i], want, got)
            bound = 2 * (abs(cfg) + abs(1 - cfg)) * MAX_ABS_D / temp
            per_step.append({"step": i, "T": temp, "agree": agree, "mismatches": nb, "worst_gap": gap, "gap_bound": bound})
            assert agree >= 0.99, per_step[-1]
            assert gap <= bound, per_step[-1]
            worst_gap, n_bad = max(worst_gap, gap), n_bad + nb
            state = want
            if i < renoise:
                state, _ = po.add_noise(state, torch.full((B,), float(t_list[i + 1])), init.cpu(), us[i])
                gen.set_offset(offs_u[i])
                got_n = m.add_noise(want.to(DEV), torch.full((B,), float(t_list[i + 1]), device=DEV), random_x=init)[0]
                assert torch.equal(got_n.cpu(), state)          # renoise is bit-exact given the same tokens
    # free-running: the public sample() from the same seed consumes the generator exactly like the reference loop
    torch.manual_seed(seed)
    free = U.sample(m, cond_d, (B, H, H), uncond_d, steps=steps, renoise_steps=renoise, temperature=(1.0, 0.2), cfg=cfg)
    assert gen.get_offset() == off_end
    final_agree = float((free.cpu() == state).float().mean())
    _log("cfg1_sample_vs_oracle", {"per_step": per_step, "total_mismatches": n_bad, "worst_gap": worst_gap,
                                   "free_running_final_agree": final_agree})
    assert final_agree > 0.5          # chance level is 1/8192; an early near-tie flip legitimately perturbs later steps


def test_mixed_length_cfg_batch_vs_oracle_per_group(default_model):
    """The notebook's CFG batch: conditional rows carry clip_image and a longer byt5 (S = 24 + 8), unconditional rows do not
    (S = 16 + 4) -> one 2B batch with per-sample key lengths and a shared unconditional slot.  Each half vs the oracle run
    on that group alone."""
    from oracle import paella_oracle as po
    m, sd = default_model
    oc = po.PaellaConfig(byt5_embd=2560)
    g = torch.Generator().manual_seed(77)
    B, H = 2, 32
    cond = {"byt5": torch.randn(B, 24, 2560, generator=g), "clip": torch.randn(B, 1024, generator=g),
            "clip_image": torch.randn(B, 1024, generator=g)}
    uncond = {"byt5": torch.zeros(B, 16, 2560), "clip": torch.zeros(B, 1024)}
    x = torch.randint(0, 8192, (B, H, H), generator=g)
    r = torch.tensor([0.8, 0.3])
    want_c = po.paella_forward(sd, oc, x, r, **cond)
    want_u = po.paella_forward(sd, oc, x, r, **uncond)
    cache = m.prepare_conditioning([{k: v.to(DEV) for k, v in cond.items()}, {k: v.to(DEV) for k, v in uncond.items()}], (H, H))
    assert cache.s_max == 32 and cache.slots == B + 1          # the identical unconditional rows share one slot
    feats = m.features(x.to(DEV), r.to(DEV), cache, cfg_pairs=True)
    n = B * H * H
    got_c = m.logits_from_features(feats[:n], B, H, H).cpu()
    got_u = m.logits_from_features(feats[n:], B, H, H).cpu()
    out = {}
    for name, got, want in (("cond", got_c, want_c), ("uncond", got_u, want_u)):
        d = got - want
        out[name] = {"max_abs": float(d.abs().max()), "rms": float(d.pow(2).mean().sqrt())}
        assert out[name]["max_abs"] < MAX_ABS_D and out[name]["rms"] < 4e-4, out
    # and a group whose samples have DIFFERENT conditioning lengths is impossible in the reference API (one tensor per group);
    # different lengths BETWEEN groups is the case above.  Un-shared unconditional rows take the per-sample path:
    plain = m.prepare_conditioning([{k: v.to(DEV) for k, v in cond.items()}, {k: v.to(DEV) for k, v in uncond.items()}], (H, H),
                                   share_uniform=False)
    feats2 = m.features(x.to(DEV), r.to(DEV), plain, cfg_pairs=True)
    out["shared_vs_plain_max_abs"] = float((feats2 - feats).abs().max())
    assert out["shared_vs_plain_max_abs"] < 1e-5
    _log("mixed_length_cfg", out)


def test_vq_indices_vs_torchtools_addmm_form_with_margin_audit():
    """R13: the CUDA nearest-code search vs the quantiser's PUBLISHED form in plain torch ops (oracle.vqgan_oracle.vq_distances:
    addmm(|c|^2 + |x|^2, x, c^T, alpha=-2) -> first minimum), not vs an oracle that copies the kernel's fma order.  The two
    evaluate the same real-valued distance with different fp32 roundings, so exact equality is not implied; every disagreement
    must be a tie within the rounding noise of the expanded form (a sum of ~6 fp32 roundings per entry, two entries):
    |d_a - d_b| <= 4 ulp(|x|^2 + |c|^2)."""
    from oracle import vqgan_oracle as vo
    from paella_b200 import ops
    g = torch.Generator().manual_seed(5)
    cases = {
        "normal": (torch.randn(200000, 4, generator=g), torch.randn(8192, 4, generator=g)),
        "torchtools_init": (torch.randn(100000, 4, generator=g) * 1e-4, (torch.rand(8192, 4, generator=g) * 2 - 1) / 8192),
        "near_ties": None,
    }
    cb = torch.randn(8192, 4, generator=g)
    mid = (cb[torch.randint(0, 8192, (50000,), generator=g)] + cb[torch.randint(0, 8192, (50000,), generator=g)]) / 2
    cases["near_ties"] = (mid + 1e-6 * torch.randn(50000, 4, generator=g), cb)          # points on a bisector: adversarial
    out = {}
    for name, (x, c) in cases.items():
        got = ops.vq_nearest(x.to(DEV), c.to(DEV)).cpu()
        d = vo.vq_distances(x, c)
        want = d.min(dim=1)[1]
        bad = (got != want).nonzero().flatten()
        worst_ulps = 0.0
        if bad.numel():
            gap = (d[bad, got[bad]] - d[bad, want[bad]]).abs()
            scale = (x[bad] ** 2).sum(1) + (c[want[bad]] ** 2).sum(1)
            ulp = torch.maximum(scale, torch.tensor(1e-30)) * 2.0 ** -23
            worst_ulps = float((gap / ulp).max())
        out[name] = {"n": x.shape[0], "mismatch": int(bad.numel()), "agree": 1 - bad.numel() / x.shape[0], "worst_gap_ulps": worst_ulps}
        assert out[name]["agree"] > 0.999, out
        assert worst_ulps <= 4.0, out
    _log("vq_vs_addmm", out)


def test_autocast_wrapped_forward_and_sample(default_model):
    """The notebook runs everything under torch.autocast('cuda') (nb:349).  Our ops take fp32/int64 tensors at the boundary and
    pick their own operand precision, so autocast must change nothing: same logits bit for bit, same tokens, fp32 out; fp16
    conditioning tensors (what an autocast encoder hands over) are accepted."""
    from paella_b200 import utils as U
    from paella_b200.synth import synthetic_conditioning
    m, _ = default_model
    cond, uncond = synthetic_conditioning(2, 16, device=DEV)
    x = torch.randint(0, 8192, (2, 16, 16), device=DEV)
    r = torch.tensor([0.6, 0.2], device=DEV)
    a = m(x, r, cond["byt5"], clip=cond["clip"])
    with torch.autocast("cuda"):
        b = m(x, r, cond["byt5"], clip=cond["clip"])
        c = m(x, r, cond["byt5"].half(), clip=cond["clip"].half())
    assert b.dtype == torch.float32 and torch.equal(a, b)
    assert float((c - a).abs().max()) < 5e-3           # fp16-rounded conditioning INPUTS: a different (legitimate) input
    torch.manual_seed(3)
    t0 = U.sample(m, cond, (2, 16, 16), uncond, steps=3, renoise_steps=2)
    torch.manual_seed(3)
    with torch.autocast("cuda"), torch.inference_mode():
        t1 = U.sample(m, cond, (2, 16, 16), uncond, steps=3, renoise_steps=2)
    assert torch.equal(t0, t1)


def test_forward_memoises_conditioning_for_the_reference_loop(default_model):
    """ref/src/utils.py:42-45 calls model(x, t, **inputs) twice per step with the same tensors: the second call reuses the
    conditioning cache; changing a tensor in place (version bump) or passing a new tensor rebuilds it."""
    m, _ = default_model
    g = torch.Generator(device=DEV).manual_seed(1)
    byt5 = torch.randn(1, 8, 2560, device=DEV, generator=g)
    clip = torch.randn(1, 1024, device=DEV, generator=g)
    x = torch.randint(0, 8192, (1, 16, 16), device=DEV, generator=g)
    r = torch.tensor([0.5], device=DEV)
    a = m(x, r, byt5, clip=clip)
    first = m._cond_single[0]["cond"]
    b = m(x, r, byt5, clip=clip)
    assert m._cond_single[0]["cond"] is first and torch.equal(a, b)
    # the loop alternates conditional / unconditional inputs: both stay memoised
    zb, zc = torch.zeros_like(byt5), torch.zeros_like(clip)
    u0 = m(x, r, zb, clip=zc)
    second = m._cond_single[0]["cond"]
    assert second is not first
    assert torch.equal(m(x, r, byt5, clip=clip), a) and m._cond_single[0]["cond"] is first
    assert torch.equal(m(x, r, zb, clip=zc), u0) and m._cond_single[0]["cond"] is second
    byt5.mul_(2.0)                                    # in-place edit: version counter moves
    c = m(x, r, byt5, clip=clip)
    assert m._cond_single[0]["cond"] is not first and not torch.equal(a, c)
    d = m(x, r, byt5.clone(), clip=clip)              # equal content in a new tensor: rebuilt, same result
    assert torch.equal(c, d)
    assert len(m._cond_single) <= 4


def test_sample_distributed_options_vs_oracle_teacher_forced():
    """§8(f1): init_x, per-step cfgs (linspace), sampling_conditional_steps (later steps unguided) of
    ref/src_distributed/utils.py:97-126 — tiny golden model, every step vs the oracle from the oracle's state."""
    from helpers import load_golden, oracle_cfg, t
    from oracle import paella_oracle as po
    from paella_b200.modules import Paella
    cfg, sd, g = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    oc = oracle_cfg(cfg)
    B, H, K, steps, cond_steps = 2, 8, cfg["num_labels"], 5, 3
    byt5, clip = t(g["byt5"]), t(g["clip"])
    cond = {"byt5": byt5, "clip": clip}
    uncond = {"byt5": torch.zeros_like(byt5), "clip": torch.zeros_like(clip)}
    cond_d, uncond_d = {k: v.to(DEV) for k, v in cond.items()}, {k: v.to(DEV) for k, v in uncond.items()}
    cfgs = torch.linspace(6.0, 2.0, steps).tolist()
    temps = torch.linspace(0.7, 0.3, steps)
    t_list = torch.linspace(1.0, 0.0, steps + 1)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    torch.manual_seed(9)
    init_noise = torch.randint(0, K, (B, H, H), device=DEV)            # the loop draws this even when init_x is given
    init_x = torch.randint(0, K, (B, H, H), generator=torch.Generator().manual_seed(4))
    full = m.prepare_conditioning([cond_d, uncond_d], (H, H))
    only = m.prepare_conditioning([cond_d], (H, H))
    state = init_x.clone()
    agrees = []
    for i in range(steps):
        guided = i < cond_steps
        off = gen.get_offset()
        q = torch.empty(B * H * H, K, device=DEV).exponential_(1).cpu()
        want, flat = _oracle_step(po, sd, oc, state, float(t_list[i]), cond, uncond, cfgs[i] if guided else None, float(temps[i]), q)
        gen.set_offset(off)
        r = torch.full((B,), float(t_list[i]), device=DEV)
        feats = m.features(state.to(DEV), r, full if guided else only, cfg_pairs=guided)
        got = m.sample_tokens(feats, B, H, H, cfgs[i] if guided else None, float(temps[i])).cpu()
        agrees.append(float((got == want).float().mean()))
        nb, gap = _margin_audit(flat, float(temps[i]), q, want, got)
        assert agrees[-1] >= 0.97 and gap < 0.5, (i, agrees, gap)       # 128 tokens per step: one near-tie is 0.8 %
        state = want
        if i < steps - 1:
            u = torch.rand(B, H, H, device=DEV).cpu()
            state, _ = po.add_noise(state, torch.full((B,), float(t_list[i + 1])), init_noise.cpu(), u)
    _log("sample_distributed_options", {"agree_per_step": agrees})
    # and the public entry point runs the same schedule (shape / range / determinism)
    from paella_b200 import utils as U
    torch.manual_seed(9)
    a = U.sample_distributed(m, cond_d, uncond_d, (B, H, H), init_x=init_x.to(DEV), steps=steps, cfg=(6.0, 2.0),
                             sampling_conditional_steps=cond_steps)
    torch.manual_seed(9)
    b = U.sample_distributed(m, cond_d, uncond_d, (B, H, H), init_x=init_x.to(DEV), steps=steps, cfg=(6.0, 2.0),
                             sampling_conditional_steps=cond_steps)
    assert torch.equal(a, b) and a.shape == (B, H, H)


# ---------------------------------------------------------------------------------------------- codec
@pytest.fixture(scope="module")
def f4():
    from paella_b200.synth import rerandomize_
    from paella_b200.vqgan import VQModel
    torch.manual_seed(0)
    m = VQModel().eval()
    rerandomize_(m.state_dict(), seed=4)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    return m.to(DEV), sd


def test_decode_tail_clamp_and_uint8_writers(f4, default_model):
    """§8(f2): decode_indices(x).clamp(0,1) (ref/src_distributed/train.py:168-171) and torchvision save_image's byte conversion
    fused into the decoder's last kernel == the separate torch ops on the unfused output, bit for bit; and
    sample(..., decode=vqmodel) == decode of sample()'s tokens."""
    from paella_b200 import utils as U
    from paella_b200.synth import synthetic_conditioning
    vq, _ = f4
    idx = torch.randint(0, 8192, (3, 32, 32), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    raw = vq.decode_indices(idx)
    assert float(raw.min()) < 0.0 and float(raw.max()) > 1.0           # the clamp does something on this input
    assert torch.equal(vq.decode_indices_clamped(idx), raw.clamp(0, 1))
    u8 = vq.decode_indices_u8(idx)
    want = raw.clamp(0, 1).mul(255).add_(0.5).clamp_(0, 255).permute(0, 2, 3, 1).to(torch.uint8)
    assert u8.shape == (3, 128, 128, 3) and u8.dtype == torch.uint8
    assert torch.equal(u8, want)
    m, _ = default_model
    cond, uncond = synthetic_conditioning(2, 16, device=DEV)
    torch.manual_seed(5)
    toks = U.sample(m, cond, (2, 16, 16), uncond, steps=3, renoise_steps=2)
    for mode, ref in (("uint8", vq.decode_indices_u8(toks)), ("clamp", vq.decode_indices(toks).clamp(0, 1)), ("raw", vq.decode_indices(toks))):
        torch.manual_seed(5)
        img = U.sample(m, cond, (2, 16, 16), uncond, steps=3, renoise_steps=2, decode=vq, decode_output=mode)
        assert torch.equal(img, ref), mode


def test_prepacked_vqgan_blob_without_load_param_matches(f4):
    """ADVICE r1 (high): a handle that only RECEIVES the packed blob (NCCL broadcast receiver, packed file, C-ABI user calling
    bind_weights on a pre-packed blob) never ran load_param, so the host mirror of the ResBlock gammas must be refreshed from
    the blob — otherwise every ResBlock silently runs as identity."""
    import ctypes
    from paella_b200 import _lib
    from paella_b200.vqgan import VQModel
    vq, sd = f4
    vq.pack_weights()
    idx = torch.randint(0, 8192, (2, 16, 16), device=DEV, generator=torch.Generator(device=DEV).manual_seed(8))
    img = torch.rand(2, 3, 64, 64, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
    want_dec, want_idx = vq.decode_indices(idx), vq.encode(img)[2]
    recv = VQModel().to(DEV).eval()            # fresh model: gammas are ZERO in its parameters (reference init)
    L = _lib.lib()
    cfg = _lib.VqganConfig()
    for k in ("levels", "bottleneck_blocks", "c_hidden", "c_latent", "codebook_size"):
        setattr(cfg, k, int(recv._cfg[k]))
    cfg.scale_factor = float(recv.scale_factor)
    h = ctypes.c_void_p()
    _lib.check(L.pb200_vqgan_create(ctypes.byref(cfg), ctypes.byref(h)), "create")
    blob = vq._blob.clone()                    # "received" bytes
    _lib.check(L.pb200_vqgan_bind_weights(h, _lib.ptr(blob)), "bind")
    recv._handle, recv._blob, recv._packed_key = h, blob, recv._weights_key()
    assert torch.equal(recv.decode_indices(idx), want_dec)
    assert torch.equal(recv.encode(img)[2], want_idx)


def test_packed_checkpoint_roundtrip(tmp_path, f4):
    """§8(f3): tools/pack_checkpoint.py on synthetic checkpoints laid out like the real ones — paella_v3.pt = bare state dict
    (here DDP-prefixed), vqgan_f4.pt = {'state_dict': ...} with extra vquantizer.* EMA buffers — then from_packed() must
    reproduce the state-dict-loaded model bit for bit without materialising fp32 parameters."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import pack_checkpoint as pc
    from helpers import load_golden, t
    from paella_b200.modules import Paella
    from paella_b200.vqgan import VQModel
    cfg, sd, g = load_golden("paella_tiny.npz")
    src = str(tmp_path / "paella_tiny.pt")
    torch.save({"module." + k: v for k, v in sd.items()}, src)
    kw = {k: v for k, v in cfg.items()}
    m0 = pc.pack("paella", src, str(tmp_path / "paella_tiny.pb200"), **kw)
    m1 = Paella.from_packed(str(tmp_path / "paella_tiny.pb200"), DEV)
    assert all(p.is_meta for p in m1.parameters())
    x, r = t(g["x"]).to(DEV), t(g["r"]).to(DEV)
    a = dict(byt5=t(g["byt5"]).to(DEV), clip=t(g["clip"]).to(DEV))
    assert torch.equal(m0(x, r, **a), m1(x, r, **a))
    vq, vsd = f4
    ck = {"state_dict": dict(vsd, **{"vquantizer.ema_element_count": torch.ones(8192), "vquantizer.ema_weight_sum": torch.zeros(8192, 4)}),
          "optimizer": {}}
    vsrc = str(tmp_path / "vqgan_f4.pt")
    torch.save(ck, vsrc)
    v0 = pc.pack("vqgan", vsrc, str(tmp_path / "vqgan_f4.pb200"))
    v1 = VQModel.from_packed(str(tmp_path / "vqgan_f4.pb200"), DEV)
    idx = torch.randint(0, 8192, (1, 16, 16), device=DEV)
    assert torch.equal(v0.decode_indices(idx), v1.decode_indices(idx))
    assert torch.equal(vq.decode_indices(idx), v1.decode_indices(idx))
    # a truncated file is refused
    d = torch.load(str(tmp_path / "vqgan_f4.pb200"), weights_only=False)
    d["blob"] = d["blob"][:-256].clone()
    torch.save(d, str(tmp_path / "bad.pb200"))
    from paella_b200._lib import PaellaB200Error
    with pytest.raises(PaellaB200Error):
        VQModel.from_packed(str(tmp_path / "bad.pb200"), DEV)


@pytest.mark.parametrize("c,hw", [(384, 16), (192, 24), (32, 5), (192, 13), (384, 9)])     # 13, 9: partial 2x8 patches, clamped halos
def test_vqgan_resblock_standalone_vs_oracle(c, hw):
    """R15: vqgan.ResBlock.forward on its own (ref/src/vqgan.py:36-42) vs the oracle's restatement."""
    from oracle import vqgan_oracle as vo
    from paella_b200.vqgan import ResBlock
    torch.manual_seed(c)
    blk = ResBlock(c, 4 * c).eval()
    with torch.no_grad():
        blk.gammas.copy_(torch.randn(6) * 0.5)
        for p in blk.parameters():
            if p.dim() == 1 and p.numel() != 6:
                p.normal_(0, 0.1)
    sd = {"b." + k: v.detach().clone() for k, v in blk.state_dict().items()}
    x = torch.randn(2, c, hw, hw, generator=torch.Generator().manual_seed(1))
    want = vo.vq_resblock(x.permute(0, 2, 3, 1).contiguous(), sd, "b.").permute(0, 3, 1, 2)
    got = blk.to(DEV)(x.to(DEV)).cpu()
    d = got - want
    _log("vqgan_resblock", {"c": c, "hw": hw, "max_abs": float(d.abs().max()), "rms": float(d.pow(2).mean().sqrt())})
    assert float(d.abs().max()) < 6e-3 and float(d.pow(2).mean().sqrt()) < 1.2e-3


def test_multinomial_above_2p29_elements_matches_torch_split():
    """torch runs a > 2^29-element fp32 draw as several kernels (TensorIterator 32-bit split), each with its own Philox offset;
    bs=128 at 32x32x8192 = 2^30 elements -> two halves.  pb200 ops mirror the split: same tokens, same final offset."""
    from paella_b200 import ops
    rows, K = 2 * 65536, 8192
    assert ops.philox_row_chunks(rows, K) == [(0, 65536), (65536, 131072)]
    g = torch.Generator(device=DEV).manual_seed(1)
    p = torch.rand(rows, K, device=DEV, generator=g)
    p[:, :8] += 30.0 * torch.rand(rows, 8, device=DEV, generator=g)        # a few dominant entries + a long tail
    torch.manual_seed(11)
    want = torch.multinomial(p, 1)[:, 0]
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    off = gen.get_offset()
    torch.manual_seed(11)
    got = ops.multinomial(p)
    assert gen.get_offset() == off
    mism = int((got != want).sum())
    _log("multinomial_2p30", {"rows": rows, "mismatch": mism})
    assert mism == 0
