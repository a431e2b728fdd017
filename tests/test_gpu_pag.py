"""Perturbed-attention guidance on the GPU.

  1. Kernels: the _perturb instances of both attention kernels (pb200_attention_perturb) against float64 at head dims 16/32/64/96
     (mma.sync) and 80 (wgmma), with perturbed and plain samples in one launch, weights that reach into the self keys, ragged P,
     shared slots and an injected sample beside them; plain samples are bit-identical to pb200_attention_inject, and a perturbed
     sample without conditioning keys returns its own V.
  2. The tiny model against the reference fixture and the oracle; the default model against the oracle at 32 x 32 and 64 x 64.
  3. Sampling: s = 0 and no entries give the tokens of the call without pag, unperturbed samples keep their tokens, batch-1
     equality under per-sample generators on the default model in batch-invariant mode, argmax tokens against the mix of
     separate forwards with and without CFG, and PAG beside guidance prompts, tiling, attn_weights, top-k and argmax/quant modes.
"""
import ctypes

import pytest
import torch

from helpers import load_golden, log_jsonl, oracle_cfg, t

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _p(x):
    return ctypes.c_void_p(x.data_ptr()) if x is not None else None


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


def _rows(d, idx):
    return {k: (v[idx] if torch.is_tensor(v) else v) for k, v in d.items()}


def _conditioning(m, B, L, seed=7):
    from paella_b200.synth import synthetic_conditioning
    return synthetic_conditioning(B, L, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features,
                                  with_clip_image=False, seed=seed, device=DEV)


@pytest.fixture(scope="module")
def tiny():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m


@pytest.fixture(scope="module")
def default_model():
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    m = m.to(DEV)
    m.batch_invariant = True
    return m


# ------------------------------------------------------------------ 1. kernels
KV_SLOT = (3, 1, 3, 0)          # samples 0 and 2 share slot 3
INJ = (-1, -1, -1, 1)           # sample 3 replays sample 1; neither is perturbed
BLOCK = 5
MASKS = (1 << BLOCK, 0, (1 << BLOCK) | 1, 0)     # samples 0 and 2 perturbed in block 5


def _inputs(hd, P, S_lens):
    g = torch.Generator(device=DEV).manual_seed(1000 * P + hd)
    B, H = len(KV_SLOT), 2
    E = H * hd
    S = max(S_lens) + 3 if S_lens else 0
    qkv = (torch.randn(B * P, 3 * E, device=DEV, generator=g) * 0.5).half()
    ckv = (torch.randn(max(1, len(S_lens)), max(S, 1), 2 * E, device=DEV, generator=g) * 0.5).half()
    # weight rows: row 0 reaches into the self keys (w_len = S + P // 2 + 1 > S), row 1 is the conditioning only, row 2 is empty
    w_ld = (min(S_lens) if S_lens else 0) + P
    w = (torch.rand(3, w_ld, device=DEV, generator=g) * 1.5 + 0.25).float()
    w_len = [min(w_ld, (min(S_lens) if S_lens else 0) + P // 2 + 1), min(S_lens) if S_lens else 0, 0]
    return dict(B=B, H=H, E=E, P=P, S=S, lens=list(S_lens), qkv=qkv, ckv=ckv, w=w, w_ld=w_ld, w_len=w_len, w_row=[0, 2, 1, 0])


def _run(c, masks=None, block=BLOCK, inj=INJ):
    from paella_b200 import _lib
    L = _lib.lib()
    B, P, S, E, H = c["B"], c["P"], c["S"], c["E"], c["H"]
    out = torch.full((B * P, E), float("nan"), dtype=torch.float16, device=DEV)
    kv_len = torch.tensor(c["lens"] or [0], dtype=torch.int32, device=DEV)
    kv_slot = torch.tensor(KV_SLOT, dtype=torch.int32, device=DEV) if c["lens"] else None
    w_len = torch.tensor(c["w_len"], dtype=torch.int32, device=DEV)
    w_row = torch.tensor(c["w_row"], dtype=torch.int32, device=DEV)
    inj_d = torch.tensor(inj, dtype=torch.int32, device=DEV) if inj is not None else None
    pm = torch.tensor(masks, dtype=torch.int64, device=DEV) if masks is not None else None
    rc = L.pb200_attention_perturb(_p(c["qkv"]), _p(c["ckv"]) if c["lens"] else None, _p(kv_len) if c["lens"] else None,
                                   _p(kv_slot), len(c["lens"]), _p(out), B, P, S, E, H, 1, _p(c["w"]), 0, c["w_ld"], _p(w_len),
                                   _p(w_row), B, None, None, None, 0, 0, None, None, None, 0, _p(inj_d),
                                   len(inj) if inj is not None else 0, _p(pm), len(masks) if masks is not None else 0, block, None)
    assert rc == 0, L.pb200_last_error() if hasattr(L, "pb200_last_error") else rc
    torch.cuda.synchronize()
    return out


def _want(c, b, kv_slot=KV_SLOT):
    """float64 [P, E] of perturbed sample b."""
    P, E, H = c["P"], c["E"], c["H"]
    hd = E // H
    rows = c["qkv"][b * P:(b + 1) * P].double()
    q, ks, vs = rows[:, :E], rows[:, E:2 * E], rows[:, 2 * E:]
    if c["lens"]:
        n = c["lens"][kv_slot[b]]
        kc, vc = c["ckv"][kv_slot[b], :n, :E].double(), c["ckv"][kv_slot[b], :n, E:].double()
    else:
        kc = vc = torch.zeros(0, E, dtype=torch.float64, device=DEV)
    k, v = torch.cat([ks, kc]), torch.cat([vs, vc])
    row = c["w_row"][b]
    wl = c["w_len"][row]
    out = torch.empty(P, E, dtype=torch.float64, device=DEV)
    for h in range(H):
        sl = slice(h * hd, (h + 1) * hd)
        p = torch.softmax(q[:, sl] @ k[:, sl].t() / hd ** 0.5, dim=-1)
        if wl:
            p[:, -wl:] *= c["w"][row, :wl].double()
        out[:, sl] = p[:, P:] @ v[P:, sl] + p[:, :P].sum(-1, keepdim=True) * vs[:, sl]
    return out


@pytest.mark.parametrize("hd", [16, 32, 64, 80, 96])
@pytest.mark.parametrize("P", [16, 70, 200])
def test_kernel_against_float64(hd, P):
    c = _inputs(hd, P, [67, 129, 1, 64])
    got = _run(c, MASKS)
    plain = _run(c, None)
    for b, m in enumerate(MASKS):
        rows = slice(b * P, (b + 1) * P)
        if (m >> BLOCK) & 1:
            err = float((got[rows].double() - _want(c, b)).abs().max())
            log_jsonl("pag.jsonl", {"test": "kernel", "hd": hd, "P": P, "b": b, "max_abs": err})
            assert err < 4e-3, (hd, P, b, err)
            assert float((plain[rows].double() - _want(c, b)).abs().max()) > 4e-3      # the test sees the perturbation
        else:
            assert torch.equal(got[rows], plain[rows]), (hd, P, b)     # plain and injected samples: bit for bit
    # a block bit that is not set: the whole launch is the plain one
    assert torch.equal(_run(c, MASKS, block=BLOCK + 1), plain)


# five samples: 0 and 2 perturbed; 1 the source of 3 (injected); 4 regional (prompt 0, its region, or both, by query); 1 and 3 map
# rows.  Every combination of the regional, map and inject flags runs the matching _perturb instance.
KV5, INJ5, MAP5 = (3, 1, 3, 0, 0), (-1, -1, -1, 1, -1), (-1, 0, -1, 1, -1)


def _run5(c, reg, maps, inj, pag):
    from paella_b200 import _lib
    L = _lib.lib()
    B, P, S, E, H = 5, c["P"], c["S"], c["E"], c["H"]
    out = torch.full((B * P, E), float("nan"), dtype=torch.float16, device=DEV)
    kv_len = torch.tensor(c["lens"], dtype=torch.int32, device=DEV)
    kv_slot = torch.tensor(KV5, dtype=torch.int32, device=DEV)
    w_len = torch.tensor(c["w_len"], dtype=torch.int32, device=DEV)
    w_row = torch.tensor([0, 2, 1, 0, 2], dtype=torch.int32, device=DEV)
    q_mask = region_slot = scores = lse2 = map_row = inj_d = pm = None
    if reg:
        qm = torch.ones(B, P, dtype=torch.uint8)
        qm[4] = torch.tensor([(1, 3, 2)[i % 3] for i in range(P)], dtype=torch.uint8)
        rs = torch.full((B, 1), -1, dtype=torch.int32)
        rs[4, 0] = 2
        q_mask, region_slot = qm.to(DEV), rs.to(DEV)
    if maps:
        map_row = torch.tensor(MAP5, dtype=torch.int32, device=DEV)
        scores = torch.full((2, H, P, S), float("nan"), device=DEV)
        lse2 = torch.full((2, H, P), float("nan"), device=DEV)
    if inj:
        inj_d = torch.tensor(INJ5, dtype=torch.int32, device=DEV)
    if pag:
        pm = torch.tensor([1 << BLOCK, 0, 1 << BLOCK, 0, 0], dtype=torch.int64, device=DEV)
    rc = L.pb200_attention_perturb(_p(c["qkv"]), _p(c["ckv"]), _p(kv_len), _p(kv_slot), len(c["lens"]), _p(out), B, P, S, E, H, 1,
                                   _p(c["w"]), 0, c["w_ld"], _p(w_len), _p(w_row), B, _p(q_mask), _p(region_slot), None,
                                   1 if reg else 0, B if reg else 0, _p(scores), _p(lse2), _p(map_row), B if maps else 0, _p(inj_d),
                                   B if inj else 0, _p(pm), B if pag else 0, BLOCK, None)
    assert rc == 0
    torch.cuda.synchronize()
    return out, scores, lse2


def _same(a, b):
    return a is None or torch.allclose(a.float(), b.float(), rtol=0, atol=0, equal_nan=True)


@pytest.mark.parametrize("hd", [32, 80])
@pytest.mark.parametrize("P", [16, 70])
@pytest.mark.parametrize("flags", [(r, m, i) for r in (0, 1) for m in (0, 1) for i in (0, 1)],
                         ids=lambda f: "reg%d_maps%d_inj%d" % f)
def test_kernel_beside_regional_map_and_injected_rows(hd, P, flags):
    reg, maps, inj = flags
    g = torch.Generator(device=DEV).manual_seed(7 * P + hd)
    H, E = 2, 2 * hd
    lens = [67, 129, 33, 64]
    S = max(lens) + 3
    w_ld = min(lens) + P
    c = dict(P=P, H=H, E=E, S=S, lens=lens, w_ld=w_ld, w_len=[min(lens) + P // 2 + 1, min(lens), 0],
             qkv=(torch.randn(5 * P, 3 * E, device=DEV, generator=g) * 0.5).half(),
             ckv=(torch.randn(len(lens), S, 2 * E, device=DEV, generator=g) * 0.5).half(),
             w=(torch.rand(3, w_ld, device=DEV, generator=g) * 1.5 + 0.25).float(), w_row=[0, 2, 1, 0, 2])
    got, sc, ls = _run5(c, reg, maps, inj, True)
    plain, sc0, ls0 = _run5(c, reg, maps, inj, False)
    for b in range(5):
        rows = slice(b * P, (b + 1) * P)
        if b in (0, 2):
            err = float((got[rows].double() - _want(c, b, KV5)).abs().max())
            log_jsonl("pag.jsonl", {"test": "kernel_flags", "hd": hd, "P": P, "flags": list(flags), "b": b, "max_abs": err})
            assert err < 4e-3, (flags, b, err)
        else:       # regional, injected, source and map rows: the bits of the instance without PERTURB
            assert torch.equal(got[rows], plain[rows]), (flags, b)
    assert _same(sc, sc0) and _same(ls, ls0), flags


@pytest.mark.parametrize("hd", [32, 80])
def test_zero_conditioning_keys_return_own_v(hd):
    c = _inputs(hd, 70, [])
    c["w_len"] = [0, 0, 0]
    got = _run(c, MASKS, inj=None)
    for b, m in enumerate(MASKS):
        if (m >> BLOCK) & 1:
            v = c["qkv"][b * 70:(b + 1) * 70, 2 * c["E"]:].float()
            assert float((got[b * 70:(b + 1) * 70].float() - v).abs().max()) <= 2e-3 * (1 + float(v.abs().max()))


# ------------------------------------------------------------------ 2. forwards
def test_tiny_forward_matches_fixture_and_oracle(tiny):
    from oracle import pag as op
    from oracle import paella_oracle as po
    cfg, sd, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("pag_tiny.npz")
    r = t(g["r"])
    own = (t(g["byt5"]), t(g["clip"]), t(g["clip_image"]))
    n = int(z["n_blocks"])
    assert tiny.n_attn_blocks == n and tiny.pag_default_blocks() == [int(i) for i in z["deep"]]

    def mm16(a, w):
        return po.mm_f16_operands(a, w).half().float()
    aw = t(z["attn_weights"])
    cases = {"all": (t(g["x"]), list(range(n)), None), "down": (t(g["x"]), [0], None),
             "attnw": (t(g["x"]), list(range(n)), aw), "x16": (t(z["x16"]), [int(i) for i in z["deep"]], None)}
    for name, (x, blocks, w) in cases.items():
        ref = t(z[f"logits_{name}"]).double()
        kw = dict(clip=own[1].to(DEV), clip_image=own[2].to(DEV), attn_weights=w.to(DEV) if w is not None else None)
        with torch.inference_mode():
            got = tiny(x.to(DEV), r.to(DEV), own[0].to(DEV), pag_blocks=[blocks, None], **kw)
            plain = tiny(x.to(DEV), r.to(DEV), own[0].to(DEV), **kw)
        assert torch.equal(got[1], plain[1]), name
        pred = op.paella_forward_pag(sd, oracle_cfg(cfg), x, r, *own, blocks=[blocks, None], attn_weights=[w, w], mm=mm16)
        d16 = float((pred.double() - ref).abs().max())
        err = float((got.cpu().double() - ref).abs().max())
        log_jsonl("pag.jsonl", {"test": "tiny_forward", "case": name, "max_abs": err, "fp16_oracle_max_abs": d16})
        assert err <= 3.0 * d16 + 1e-3, (name, err, d16)
        assert float((plain[0].cpu().double() - ref[0]).abs().max()) > 3.0 * d16 + 1e-3, name


@pytest.mark.parametrize("hw", [32, 64])
def test_default_forward_matches_oracle(default_model, hw):
    from oracle import pag as op
    from oracle import paella_oracle as po
    m = default_model
    cond, _ = _conditioning(m, 2, 16)
    g = torch.Generator().manual_seed(hw)
    x = torch.randint(0, m.num_labels, (2, hw, hw), generator=g)
    r = torch.tensor([0.7, 0.3])
    blocks = m.pag_default_blocks()
    with torch.inference_mode():
        got = m(x.to(DEV), r.to(DEV), cond["byt5"], clip=cond["clip"], pag_blocks=[blocks, None])
        plain = m(x.to(DEV), r.to(DEV), cond["byt5"], clip=cond["clip"])
    assert torch.equal(got[1], plain[1])
    sd = {k: v.detach().float().cpu() for k, v in m.state_dict().items()}
    ocfg = oracle_cfg(dict(m._cfg))
    want = op.paella_forward_pag(sd, ocfg, x[:1], r[:1], cond["byt5"][:1].cpu(), cond["clip"][:1].cpu(), None, blocks=[blocks])
    want_plain = po.paella_forward(sd, ocfg, x[:1], r[:1], cond["byt5"][:1].cpu(), cond["clip"][:1].cpu(), None)
    err = float((got[0].cpu() - want[0]).abs().max())
    moved = float((want[0] - want_plain[0]).abs().max())
    base = float((plain[0].cpu() - want_plain[0]).abs().max())
    log_jsonl("pag.jsonl", {"test": "default_forward", "hw": hw, "max_abs": err, "plain_max_abs": base, "perturbation": moved})
    assert err <= 2.0 * base + 1e-3 and moved > 4 * (2.0 * base + 1e-3), (err, base, moved)


# ------------------------------------------------------------------ 3. sampling
def test_zero_scale_and_no_entries_are_the_call_without(tiny):
    from paella_b200 import utils as U
    H, B = 8, 3
    cond, uncond = _conditioning(tiny, B, 10)
    kw = dict(steps=4, temperature=(1.2, 0.3), cfg=(5.0, 3.0))
    with torch.inference_mode():
        base = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=_gens([1, 2, 3]), **kw)[0]
        zero = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=_gens([1, 2, 3]), pag=[0.0, None, (0, [1])], **kw)[0]
        # (the tiny model's default blocks sit at a level of one position on an 8 x 8 grid, where the perturbation is the identity)
        one = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=_gens([1, 2, 3]), pag=[None, (3.0, [0, 1, 4, 5]), None],
                                **kw)[0]
        s = U.sample(tiny, cond, (B, H, H), uncond, steps=3, renoise_steps=2, generator=_gens([4, 5, 6]))
        s0 = U.sample(tiny, cond, (B, H, H), uncond, steps=3, renoise_steps=2, generator=_gens([4, 5, 6]), pag=[None] * B)
    assert torch.equal(base, zero) and torch.equal(s, s0)
    assert torch.equal(base[0], one[0]) and torch.equal(base[2], one[2]) and not torch.equal(base[1], one[1])


def _mix_check(m, cond, uncond, H, B, pag, cfg):
    """The mixed logits of one guided (or unguided) step from separate forwards."""
    x = torch.randint(0, m.num_labels, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    r = torch.full((B,), 0.6, device=DEV)
    with torch.inference_mode():
        lc = m(x, r, cond["byt5"], clip=cond["clip"])
        lu = m(x, r, uncond["byt5"], clip=uncond["clip"]) if cfg is not None else None
        blocks = [None if e is None else (e[1] if isinstance(e, tuple) else m.pag_default_blocks()) for e in pag]
        lp = m(x, r, cond["byt5"], clip=cond["clip"], pag_blocks=blocks)
    out = []
    for b, e in enumerate(pag):
        s = 0.0 if e is None else (e[0] if isinstance(e, tuple) else e)
        if cfg is None:
            out.append(lc[b] + s * (lc[b] - lp[b]))
        else:
            out.append(lu[b] + cfg * (lc[b] - lu[b]) + s * (lc[b] - lp[b]))
    return torch.stack(out)


@pytest.mark.parametrize("guided", [True, False])
def test_argmax_tokens_follow_the_mixed_logits(tiny, guided):
    """argmax sampling with t_start = t_end (every step sees the same noise level): the first step's tokens are the argmax of the
    mix of separate forwards, where that argmax is unambiguous."""
    from paella_b200 import utils as U
    H, B = 8, 3
    cond, uncond = _conditioning(tiny, B, 10)
    pag = [2.0, None, (1.5, [0, 3, 5])]
    cfg = 4.0 if guided else None
    x = torch.randint(0, tiny.num_labels, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    want = _mix_check(tiny, cond, uncond, H, B, pag, cfg)
    with torch.inference_mode():
        got, _ = U.sample_notebook(tiny, cond, (B, H, H), uncond, init_x=x, steps=1, renoise_steps=0, mode="argmax",
                                   cfg=(cfg, cfg) if guided else None, t_start=0.6, t_end=0.6, pag=pag)
    top2 = want.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-3
    assert bool((got == want.argmax(1))[clear].all()) and float(clear.float().mean()) > 0.9


def test_batch1_equality_under_per_sample_generators(default_model):
    from paella_b200 import utils as U
    m = default_model
    H = 16
    cond, uncond = _conditioning(m, 3, 20)
    kw = dict(steps=3, temperature=(1.0, 0.3), cfg=(4.0, 4.0))
    pag = [2.0, None, (1.0, [0, 1, 40])]
    with torch.inference_mode():
        batch = U.sample_notebook(m, cond, (3, H, H), uncond, generator=_gens([11, 12, 13]), pag=pag, **kw)[0]
        for b in range(3):
            one = U.sample_notebook(m, _rows(cond, slice(b, b + 1)), (1, H, H), _rows(uncond, slice(b, b + 1)),
                                    generator=_gens([11 + b]), pag=[pag[b]], **kw)[0]
            assert torch.equal(one[0], batch[b]), b


def _lora_sd(m):
    """A rank-4 adapter with non-zero B on every target the per-sample path serves."""
    from paella_b200.lora import served_targets
    g = torch.Generator().manual_seed(5)
    sd = {}
    for mod, (_, _, fin, fout) in served_targets(m._cfg).items():
        sd[mod + ".lora_A.weight"] = torch.randn(4, fin, generator=g) / fin ** 0.5
        sd[mod + ".lora_B.weight"] = torch.randn(fout, 4, generator=g) * 0.2
    return sd


def test_combinations_keep_unperturbed_rows(tiny):
    """guidance prompts, LoRA, tiling, attn_weights, top-k, top-p and per-sample modes beside PAG: the unperturbed samples keep their tokens,
    and every generator ends where the call without pag leaves it."""
    from paella_b200 import utils as U
    from paella_b200.vqgan import VQModel
    H, B = 8, 4
    cond, uncond = _conditioning(tiny, B, 10)
    extra, _ = _conditioning(tiny, 1, 10, seed=99)
    cfg_vq, sd_vq, _ = load_golden("vqgan_tiny.npz")
    vq = VQModel(**cfg_vq).to(DEV).eval()
    vq.load_state_dict(sd_vq)
    from paella_b200.lora import load_lora
    lsd = _lora_sd(tiny)
    style = load_lora(tiny, lsd)
    kw = dict(steps=4, temperature=(1.0, 0.4), cfg=(5.0, 5.0), tiling=["x", None, "xy", None], top_k=20,
              top_p=torch.tensor([0.9, 1.0, 0.8, 1.0]), lora=[style, (style, 0.5), None, None],
              attn_weights=[torch.rand(6) + 0.5, None, torch.rand(12) + 0.5, None],
              guidance_prompts=[[(extra, 0.5)], None, None, [(extra, -0.3)]], mode=["multinomial", "argmax", "multinomial", "quant"],
              vqmodel=vq, sampling_conditional_steps=3)
    with torch.inference_mode():
        gens_a, gens_b = _gens([1, 2, 3, 4]), _gens([1, 2, 3, 4])
        base = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=gens_a, **kw)[0]
        got = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=gens_b, pag=[(2.0, [0, 1, 4, 5]), None, (1.0, [1, 2]), None],
                                **kw)[0]
    assert torch.equal(base[1], got[1]) and torch.equal(base[3], got[3])
    assert not torch.equal(base[0], got[0])
    assert [g.get_offset() for g in gens_a] == [g.get_offset() for g in gens_b]


def test_validation_before_any_work(tiny):
    from paella_b200 import utils as U
    H, B = 8, 2
    cond, uncond = _conditioning(tiny, B, 10)
    gens = _gens([1, 2])
    for bad in ([1.0], [True, None], [float("nan"), None], [(1.0, []), None], [(1.0, [99]), None]):
        for fn in (lambda: U.sample(tiny, cond, (B, H, H), uncond, steps=2, renoise_steps=1, generator=gens, pag=bad),
                   lambda: U.sample_distributed(tiny, cond, uncond, (B, H, H), steps=2, generator=gens, pag=bad),
                   lambda: U.sample_notebook(tiny, cond, (B, H, H), uncond, steps=2, generator=gens, pag=bad)):
            with pytest.raises(ValueError):
                fn()
    with pytest.raises(ValueError):
        U.sample(tiny, cond, (B, H, H), uncond, steps=2, renoise_steps=1, generator=gens, pag=[None, 1.0],
                 attention_source=[None, (0, 1)])
    assert [g.get_offset() for g in gens] == [g.get_offset() for g in _gens([1, 2])]
    x = torch.zeros(B, H, H, dtype=torch.int64, device=DEV)
    with pytest.raises(ValueError):
        tiny(x, torch.zeros(B, device=DEV), cond["byt5"], clip=cond["clip"], pag_blocks=[[], None])


def test_pag_beside_regional_and_map_samples(tiny):
    """PAG on one sample, regional prompts or attention maps on another: the other samples' tokens and maps are those of the call
    without pag (the launches run the regional and map _perturb instances)."""
    from paella_b200 import utils as U
    H, B = 8, 3
    cond, uncond = _conditioning(tiny, B, 10)
    extra, _ = _conditioning(tiny, 1, 10, seed=98)
    left = torch.zeros(H, H, dtype=torch.bool)
    left[:, :H // 2] = True
    pag = [None, (2.0, [0, 1, 4, 5]), None]
    kw = dict(steps=3, temperature=(1.1, 0.3), cfg=(4.0, 4.0))
    with torch.inference_mode():
        for extra_kw in (dict(prompt_regions=[[(extra, left)], None, None]), dict(attention_maps=True)):
            base = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=_gens([1, 2, 3]), **kw, **extra_kw)
            got = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=_gens([1, 2, 3]), pag=pag, **kw, **extra_kw)
            for b in (0, 2):
                assert torch.equal(base[0][b], got[0][b]), (list(extra_kw), b)
                if "attention_maps" in extra_kw:
                    assert torch.equal(base[2][b], got[2][b]), b
            assert not torch.equal(base[0][1], got[0][1])
        with pytest.raises(ValueError, match="prompt_regions"):
            U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=_gens([1, 2, 3]), pag=pag,
                              prompt_regions=[None, [(extra, left)], None], **kw)


# ------------------------------------------------------------------ 4. SamplingEngine
def test_engine_equals_batch1_calls(tiny):
    """Requests with PAG -- guided, unguided, with guidance prompts, attn_weights, LoRA, tiling, top-k, attention maps and a
    short sampling_conditional_steps -- arriving staggered beside a plain one in a 3-slot engine equal batch-1 sample_notebook
    calls (sample_distributed's core, which also takes attn_weights), generator offsets included."""
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    from paella_b200.lora import load_lora
    H = 8
    N = 6
    cond, uncond = _conditioning(tiny, N, 12, seed=31)
    tc, _ = _conditioning(tiny, 1, 6, seed=32)
    style = load_lora(tiny, _lora_sd(tiny))
    blocks = [0, 1, 4, 5]
    kinds = [dict(pag=(2.0, blocks)),
             dict(),
             dict(pag=(1.5, blocks), cfg=None),
             dict(pag=(1.0, [1, 4]), guidance_prompts=[(tc, 0.5)], attn_weights=torch.rand(5) + 0.5, tiling="x"),
             dict(pag=(2.5, blocks), lora=(style, 0.7), sampling_conditional_steps=2, top_k=7),
             dict(pag=3.0, attention_maps=True)]
    steps = [3, 4, 3, 2, 4, 3]
    eng = SamplingEngine(tiny, latent_hw=(H, H), max_batch=3, max_cond_len=40, max_guidance_prompts=1)
    assert eng.w_pool.shape[0] == 3       # nothing allocated for PAG before a request uses it
    reqs = []
    for i, kw in enumerate(kinds):
        g = torch.Generator(device=DEV).manual_seed(80 + i)
        reqs.append((eng.submit(_rows(cond, slice(i, i + 1)), _rows(uncond, slice(i, i + 1)), generator=g, steps=steps[i],
                                temperature=(1.2, 0.2), **kw), g, kw))
        if i % 2:
            eng.step()
    eng.run_until_idle()
    assert eng.w_pool.shape[0] == 4
    for i, (q, g, kw) in enumerate(reqs):
        kw = dict(kw)
        for key in ("guidance_prompts", "pag", "lora", "attn_weights"):
            if key in kw:
                kw[key] = [kw[key]]
        if "tiling" in kw:
            kw["tiling"] = [kw["tiling"]]
        kw.setdefault("cfg", (8.0, 8.0))
        maps = kw.pop("attention_maps", False)
        g1 = torch.Generator(device=DEV).manual_seed(80 + i)
        with torch.inference_mode():
            want = U.sample_notebook(tiny, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), steps=steps[i],
                                     temperature=(1.2, 0.2), generator=[g1], attention_maps=maps, **kw)
        assert torch.equal(q.result, want[0]), (i, list(kw))
        if maps:
            assert torch.equal(q.attention_maps, want[2][0]), i
        assert g.get_offset() == g1.get_offset(), i


def test_engine_pag_validation(tiny):
    from paella_b200.engine import SamplingEngine
    H = 8
    eng = SamplingEngine(tiny, latent_hw=(H, H), max_batch=2, max_cond_len=40, max_prompt_regions=1)
    cond, uncond = _conditioning(tiny, 1, 12)
    left = torch.zeros(H, H, dtype=torch.bool)
    left[:, :4] = True
    g = torch.Generator(device=DEV).manual_seed(1)
    off = g.get_offset()
    for bad in ([2.0], True, float("nan"), (1.0, []), (1.0, [1, 1]), (1.0, [99]), (1.0, [0.5]), "x"):
        with pytest.raises(ValueError):
            eng.submit(cond, uncond, generator=g, pag=bad)
    with pytest.raises(ValueError, match="prompt_regions"):
        eng.submit(cond, uncond, generator=g, pag=1.0, prompt_regions=[(cond, left)])
    src = eng.submit(cond, uncond, generator=torch.Generator(device=DEV).manual_seed(2))
    with pytest.raises(ValueError):
        eng.submit(cond, uncond, generator=g, pag=1.0, attention_source=(src, 2))
    psrc = eng.submit(cond, uncond, generator=torch.Generator(device=DEV).manual_seed(3), pag=1.0)
    with pytest.raises(ValueError, match="source"):
        eng.submit(cond, uncond, generator=g, attention_source=(psrc, 2))
    assert g.get_offset() == off
    eng.run_until_idle()
