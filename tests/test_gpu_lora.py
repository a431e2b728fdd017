"""LoRA adapters on the GPU: the segmented shrink + expand kernel against fp64, the tiny and default models against the reference
fixture and the oracle on merged weights, untouched rows, per-sample generators, the CFG pair's unconditional rows, and the
combinations with guidance prompts, regional prompts, attention maps, prompt-to-prompt edits and token scoring.

Tolerances are those of test_gpu_model.py (max-abs / rms): tiny golden model 7e-3 / 1.2e-3, reference-default model 2.5e-3 / 4e-4.
"""
import os

import numpy as np
import pytest
import torch

from helpers import GOLDEN, load_golden, log_jsonl, oracle_cfg, t

pytestmark = pytest.mark.gpu
DEV = "cuda"
MAX_ABS, RMS = 7e-3, 1.2e-3
MAX_ABS_D, RMS_D = 2.5e-3, 4e-4


def _errs(got, want):
    d = got.float().cpu().double() - want.double().cpu()
    return float(d.abs().max()), float(d.pow(2).mean().sqrt())


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


def _fixture():
    z = np.load(os.path.join(GOLDEN, "lora_tiny.npz"))
    la = {k[2:]: torch.from_numpy(z[k].copy()) for k in z.files if k.startswith("a:")}
    lb = {k[2:]: torch.from_numpy(z[k].copy()) for k in z.files if k.startswith("b:")}
    return z, la, lb


@pytest.fixture(scope="module")
def tiny():
    from paella_b200.lora import load_lora
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    z, la, lb = _fixture()
    return m, cfg, sd, load_lora(m, la), load_lora(m, lb), la, lb


def _random_adapter(cfg, rank, seed, b_std, blocks=None):
    from paella_b200.lora import served_targets
    g = torch.Generator().manual_seed(seed)
    out = {}
    for mod, (k, _, fin, fout) in served_targets(cfg).items():
        if blocks is not None and k not in blocks:
            continue
        out[mod + ".lora_A.weight"] = torch.randn(rank, fin, generator=g) / fin ** 0.5
        out[mod + ".lora_B.weight"] = torch.randn(fout, rank, generator=g) * b_std
    return out


# ------------------------------------------------------------------ 1. kernel matrix against fp64
SHAPES = [(32, 64), (64, 192), (1024, 1280), (1280, 3840), (1280, 1280), (64, 64)]
RANKS = [1, 8, 15, 16, 17, 64]
MATRIX = [(r, k, n, ln, f32, False) for (r, (k, n)) in zip(RANKS, SHAPES) for ln in (False, True) for f32 in (False, True)]
# launches holding only the rank under test, so that each instance width (ranks 1-8, 9-16, 17-32, 33-64) runs
MATRIX += [(r, 1280, 3840 if r % 2 else 1280, ln, f32, True) for r in (1, 16, 17, 32, 64) for ln, f32 in ((False, False), (True, True))]


def _operand(rank, K, N, g, alpha):
    rp = (rank + 7) // 8 * 8
    a = torch.zeros(rp, K, dtype=torch.float16)
    a[:rank] = (torch.randn(rank, K, generator=g) / K ** 0.5).half()
    b = torch.zeros(N, rp, dtype=torch.float16)
    b[:, :rank] = (torch.randn(N, rank, generator=g) * 0.3).half()
    aux = torch.zeros(rp + 1, dtype=torch.float32)
    aux[:rp] = a.double().sum(1).float()
    aux[rp] = alpha / rank
    return a.to(DEV), b.to(DEV), aux.to(DEV), rp


@pytest.mark.parametrize("rank, K, N, ln, f32, solo", MATRIX)
def test_kernel_matrix_against_fp64(rank, K, N, ln, f32, solo):
    from paella_b200._lib import PB200_LORA_WORKSPACE_PER_ROW, LoraOperand, check, current_stream, lib, ptr
    g = torch.Generator().manual_seed(rank * 7 + K + N + 2 * ln + f32)
    M, rpe = (77, 1) if rank % 2 else (90, 5)          # ragged row counts; several rows per table entry
    n_e = (M + rpe - 1) // rpe
    ops_ = [_operand(rank, K, N, g, float(rank))] + ([] if solo else [_operand(8, K, N, g, 4.0), _operand(64, K, N, g, 16.0)])
    ids = torch.randint(-1, len(ops_), (n_e,), generator=g, dtype=torch.int32)
    ids[0], ids[-1] = len(ops_) - 1, -1
    scales = torch.rand(n_e, generator=g) * 4 - 2
    scales[1] = 0.0                                       # scale 0: no adapter
    x = torch.randn(M, K, generator=g) + (0.3 if ln else 0.0)
    x16 = x.half()
    st = None
    if ln:       # the folded LayerNorm's fixed-point row statistics of the shifted fp16 rows
        xd = x16.double()
        st = torch.stack([(xd.sum(1) * 2 ** 20).round(), ((xd * xd).sum(1) * 2 ** 16).round()], 1).to(torch.int64)
    y0 = torch.randn(M, N, generator=g)
    y0 = y0 if f32 else y0.half()
    row_e = torch.arange(M) // rpe
    live = (ids[row_e] >= 0) & (scales[row_e] != 0)
    x16[~live] = float("nan")                             # canaries: never read ...
    y0[~live] = float("nan")                              # ... nor written
    xd, yd = x16.to(DEV), y0.to(DEV).clone()
    arr = (LoraOperand * len(ops_))()
    for i, (a, b, aux, rp) in enumerate(ops_):
        arr[i] = LoraOperand(a.data_ptr(), b.data_ptr(), aux.data_ptr(), rp)
    ids_d, sc_d = ids.to(DEV), scales.to(DEV)
    st_d = st.to(DEV) if st is not None else None
    ws = torch.empty(M * PB200_LORA_WORKSPACE_PER_ROW, dtype=torch.uint8, device=DEV)
    check(lib().pb200_lora_shrink_expand(ptr(xd), K, M, K, N, rpe, ptr(ids_d), ptr(sc_d), arr, len(ops_), ptr(st_d), ptr(yd), N, int(f32),
                                         0, 0, ptr(ws), ws.numel(), current_stream()), "pb200_lora_shrink_expand")
    got = yd.cpu()
    # untouched rows, bit for bit (NaN canaries included)
    assert torch.equal(got[~live].view(torch.int16 if not f32 else torch.int32), y0[~live].view(torch.int16 if not f32 else torch.int32))
    want = y0.double().clone()
    for m in torch.nonzero(live).flatten().tolist():
        e = m // rpe
        a, b, aux, rp = ops_[int(ids[e])]
        a, b, aux = a.cpu().double(), b.cpu().double(), aux.cpu().double()
        xr = x16[m].double()
        u = a @ xr
        if ln:
            mean = float(st[m, 0]) / 2 ** 20 / K
            ex2 = float(st[m, 1]) / 2 ** 16 / K
            u = (u - mean * aux[:rp]) / np.sqrt(max(ex2 - mean * mean, 0.0) + 1e-6)
        want[m] += float(scales[e]) * float(aux[rp]) * (b @ u)
    d = (got[live].double() - want[live]).abs()
    delta = (want[live] - y0[live].double()).abs().max()
    bound = (2.0 ** -11 * want[live].abs() if not f32 else 1e-6 * want[live].abs()) + 2e-5 * delta
    log_jsonl("lora.jsonl", {"case": "kernel", "rank": rank, "K": K, "N": N, "ln": ln, "f32": f32, "solo": solo, "max_err": float(d.max()),
                             "max_delta": float(delta)})
    assert float(delta) > 0.05
    assert bool((d <= bound).all()), float((d - bound).max())


def test_kernel_remap_and_rows_without_any_adapter():
    """The conditioning cache's row remap (row (i / S) * s_max + i % S), and a launch where no row has an adapter, which touches
    nothing."""
    from paella_b200._lib import PB200_LORA_WORKSPACE_PER_ROW, LoraOperand, check, current_stream, lib, ptr
    g = torch.Generator().manual_seed(5)
    S, s_max, B, K, N = 3, 5, 4, 64, 128
    a, b, aux, rp = _operand(8, K, N, g, 8.0)
    x = torch.randn(B * S, K, generator=g).half().to(DEV)
    y = torch.randn(B * s_max, N, generator=g).half().to(DEV)
    y0 = y.clone()
    arr = (LoraOperand * 1)(LoraOperand(a.data_ptr(), b.data_ptr(), aux.data_ptr(), rp))
    ws = torch.empty(B * S * PB200_LORA_WORKSPACE_PER_ROW, dtype=torch.uint8, device=DEV)
    ids = torch.tensor([0, -1, 0, 0], dtype=torch.int32, device=DEV)
    sc = torch.tensor([1.0, 1.0, 0.5, 0.0], device=DEV)
    check(lib().pb200_lora_shrink_expand(ptr(x), K, B * S, K, N, S, ptr(ids), ptr(sc), arr, 1, None, ptr(y), N, 0, S, s_max,
                                         ptr(ws), ws.numel(), current_stream()),
          "pb200_lora_shrink_expand")
    got = y.cpu().double().view(B, s_max, N)
    ref = y0.cpu().double().view(B, s_max, N).clone()
    xd = x.cpu().double().view(B, S, K)
    for s_i, s in ((0, 1.0), (2, 0.5)):
        ref[s_i, :S] += s * (xd[s_i] @ a.cpu().double().t()) @ b.cpu().double().t()
    changed = torch.zeros(B, s_max, dtype=torch.bool)
    changed[0, :S] = changed[2, :S] = True
    assert torch.equal(y.cpu().view(B, s_max, N)[~changed], y0.cpu().view(B, s_max, N)[~changed])
    assert float((got - ref).abs().max()) < 2e-3 * float(ref.abs().max())
    ids.fill_(-1)
    y1 = y.clone()
    check(lib().pb200_lora_shrink_expand(ptr(x), K, B * S, K, N, S, ptr(ids), ptr(sc), arr, 1, None, ptr(y), N, 0, S, s_max,
                                         ptr(ws), ws.numel(), current_stream()),
          "pb200_lora_shrink_expand")
    assert torch.equal(y, y1)


# ------------------------------------------------------------------ 2. tiny model against the fixture and the oracle
def test_tiny_forward_against_fixture_and_oracle(tiny):
    from oracle import lora as ol
    from oracle import paella_oracle as po
    m, cfg, sd, a, b, la, lb = tiny
    z, _, _ = _fixture()
    x, r, byt5, clip = (t(z[k]).to(DEV) for k in ("x", "r", "byt5", "clip"))
    got = m(x, r, byt5, clip=clip, lora=[a, None, (b, 0.5), (a, 2.0)])
    base = m(x, r, byt5, clip=clip)
    mx, rms = _errs(got, t(z["logits"]))
    log_jsonl("lora.jsonl", {"case": "tiny_fixture", "max_abs": mx, "rms": rms})
    assert mx < MAX_ABS and rms < RMS
    oc = oracle_cfg(cfg)
    for i, (lsd, s) in enumerate([(la, 1.0), (None, 0.0), (lb, 0.5), (la, 2.0)]):
        msd = sd if lsd is None else ol.merge(sd, lsd, s)
        want = po.paella_forward(msd, oc, *(t(z[k][i:i + 1]) for k in ("x", "r", "byt5", "clip")))
        mx, rms = _errs(got[i:i + 1], want)
        assert mx < MAX_ABS and rms < RMS, (i, mx, rms)
        effect = float((got[i] - base[i]).abs().max())
        log_jsonl("lora.jsonl", {"case": "tiny_oracle", "sample": i, "max_abs": mx, "rms": rms, "effect": effect})
        if lsd is None:
            assert torch.equal(got[i], base[i])
        else:
            assert effect > 20 * MAX_ABS


# ------------------------------------------------------------------ 3. default model against the oracle
@pytest.fixture(scope="module")
def default_model():
    from paella_b200.lora import load_lora
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    m = m.to(DEV)
    lsd = _random_adapter(m._cfg, 16, 11, 0.02)
    return m, sd, lsd, load_lora(m, lsd)


@pytest.mark.parametrize("hw, L", [(32, 24), (64, 128)])
def test_default_forward_vs_oracle(default_model, hw, L):
    from oracle import lora as ol
    from oracle import paella_oracle as po
    from paella_b200.synth import synthetic_conditioning
    m, sd, lsd, ad = default_model
    cond, _ = synthetic_conditioning(1, L, with_clip_image=True)
    x = torch.randint(0, 8192, (1, hw, hw), generator=torch.Generator().manual_seed(hw))
    r = torch.tensor([0.55])
    args = (cond["byt5"], cond["clip"], cond["clip_image"])
    want = po.paella_forward(ol.merge(sd, lsd, 0.8), po.PaellaConfig(byt5_embd=2560), x, r, *args)
    got = m(x.to(DEV), r.to(DEV), *(v.to(DEV) for v in args[:1]), clip=args[1].to(DEV), clip_image=args[2].to(DEV), lora=(ad, 0.8))
    base = m(x.to(DEV), r.to(DEV), args[0].to(DEV), clip=args[1].to(DEV), clip_image=args[2].to(DEV))
    mx, rms = _errs(got, want)
    effect = float((got - base).abs().max())
    top1 = float((got.cpu().argmax(1) == want.argmax(1)).float().mean())
    log_jsonl("lora.jsonl", {"case": "default_oracle", "hw": hw, "max_abs": mx, "rms": rms, "effect": effect, "top1": top1})
    assert mx < MAX_ABS_D and rms < RMS_D
    assert effect > 20 * MAX_ABS_D
    assert top1 > 0.97


# ------------------------------------------------------------------ 4. untouched rows
def test_rows_without_adapter_are_bit_identical(tiny, default_model):
    from paella_b200.synth import synthetic_conditioning
    for m, ad in ((tiny[0], tiny[3]), (default_model[0], default_model[3])):
        kw = dict(byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features)
        cond, _ = synthetic_conditioning(4, 12, device=DEV, **kw)
        x = torch.randint(0, m.num_labels, (4, 16, 16), device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
        r = torch.tensor([0.9, 0.5, 0.3, 0.1], device=DEV)
        plain = m(x, r, cond["byt5"], clip=cond["clip"])
        mixed = m(x, r, cond["byt5"], clip=cond["clip"], lora=[None, (ad, 0.0), ad, None])
        zero = m(x, r, cond["byt5"], clip=cond["clip"], lora=(ad, 0.0))
        assert torch.equal(zero, plain)
        for i in (0, 1, 3):
            assert torch.equal(mixed[i], plain[i])
        assert not torch.equal(mixed[2], plain[2])


# ------------------------------------------------------------------ 5. sample() with per-sample generators; the CFG pair
def _cond(m, B, L, seed=7):
    from paella_b200.synth import synthetic_conditioning
    return synthetic_conditioning(B, L, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features, seed=seed,
                                  device=DEV)


def _rows(d, i):
    return {k: v[i:i + 1] for k, v in d.items()}


def _batch_one_equality(m, entries, H, steps):
    from paella_b200 import utils as U
    B = len(entries)
    cond, uncond = _cond(m, B, 10)
    seeds = [11 + i for i in range(B)]
    ga = _gens(seeds)
    toks = U.sample(m, cond, (B, H, H), uncond, steps=steps, renoise_steps=steps - 1, generator=ga, lora=entries)
    for i in range(B):
        gi = _gens([seeds[i]])
        one = U.sample(m, _rows(cond, i), (1, H, H), _rows(uncond, i), steps=steps, renoise_steps=steps - 1, generator=gi,
                       lora=[entries[i]])
        assert torch.equal(toks[i], one[0]), i
        assert gi[0].get_offset() == ga[i].get_offset()
    return toks


def test_sample_rows_equal_their_batch_one_calls(tiny, default_model):
    m, _, _, a, b, _, _ = tiny
    toks = _batch_one_equality(m, [a, None, (b, 0.5), (a, -1.0)], 8, 3)
    plain = _batch_one_equality(m, [None] * 4, 8, 3)
    assert torch.equal(toks[1], plain[1]) and not torch.equal(toks[0], plain[0])
    md, ad = default_model[0], default_model[3]
    md.batch_invariant = True
    try:
        _batch_one_equality(md, [(ad, 0.7), None, ad], 16, 2)
    finally:
        md.batch_invariant = False


def test_cfg_pair_runs_the_unconditional_rows_under_the_adapter(tiny):
    """A 1-step guided argmax call draws nothing after its start tokens: it must pick the argmax of the hand mix of two lora=
    forwards, the unconditional one under the same adapter."""
    from paella_b200 import utils as U
    m, _, _, a, _, _, _ = tiny
    B, H, cfg = 2, 8, 3.0
    cond, uncond = _cond(m, B, 10)
    x0 = torch.randint(0, m.num_labels, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    toks, _ = U.sample_notebook(m, cond, (B, H, H), uncond, init_x=x0, steps=1, renoise_steps=0, cfg=(cfg, cfg), mode="argmax",
                                lora=a)
    r = torch.ones(B, device=DEV)
    lc = m(x0, r, cond["byt5"], clip=cond["clip"], lora=a)
    lu = m(x0, r, uncond["byt5"], clip=uncond["clip"], lora=a)
    lu_plain = m(x0, r, uncond["byt5"], clip=uncond["clip"])
    right = (lc * cfg + lu * (1 - cfg)).argmax(1)
    wrong = (lc * cfg + lu_plain * (1 - cfg)).argmax(1)
    agree, agree_wrong = float((toks == right).float().mean()), float((toks == wrong).float().mean())
    log_jsonl("lora.jsonl", {"case": "cfg_pair", "agree": agree, "agree_without_uncond_adapter": agree_wrong})
    assert agree >= 0.98 and agree_wrong < agree


# ------------------------------------------------------------------ 6. SamplingEngine
def _one_inputs(m, L, seed, zeros=False):
    g = torch.Generator().manual_seed(seed)
    d = {"byt5": torch.randn(1, L, m.byt5_mapper.in_features, generator=g), "clip": torch.randn(1, m.clip_mapper.in_features, generator=g)}
    return {k: (torch.zeros_like(v) if zeros else v).to(DEV) for k, v in d.items()}


def test_engine_requests_with_and_without_adapters_equal_batch_one(tiny):
    """Requests on different adapters, and without one, share steps; each equals its batch-1 sample_notebook(..., lora=) in tokens,
    intermediates and generator offset, bit for bit (the tiny model is batch-invariant).  Requests use the engine-wide
    unconditional slot or bring their own negative prompt."""
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    m, _, _, a, b, _, _ = tiny
    H = 8
    shared = _one_inputs(m, 6, 99, zeros=True)
    own_neg = _one_inputs(m, 4, 98)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=4, max_cond_len=16, unconditional_inputs=shared)
    specs = [dict(seed=1, L=7, lora=a, uncond=None, steps=4, at=0), dict(seed=2, L=9, lora=None, uncond=None, steps=3, at=0),
             dict(seed=3, L=7, lora=(b, 0.5), uncond=own_neg, steps=4, at=1), dict(seed=4, L=5, lora=(a, 2.0), uncond=None, steps=2, at=1),
             dict(seed=5, L=7, lora=(b, 0.0), uncond=None, steps=3, at=2), dict(seed=6, L=8, lora=b, uncond=own_neg, steps=3, at=3)]
    subs, step = [], 0
    while step <= 3 or eng.busy:
        for i, sp in enumerate(specs):
            if sp["at"] == step:
                g = torch.Generator(device=DEV).manual_seed(sp["seed"])
                inputs = _one_inputs(m, sp["L"], 10 + i)
                subs.append((sp, inputs, g, eng.submit(inputs, sp["uncond"], generator=g, steps=sp["steps"], lora=sp["lora"],
                                                       keep_intermediates=True)))
        eng.step()
        step += 1
    for sp, inputs, g, req in subs:
        assert req.done and req.lora is None           # the adapter is released at retirement
        gr = torch.Generator(device=DEV).manual_seed(sp["seed"])
        toks, inter = U.sample_notebook(m, inputs, (1, H, H), sp["uncond"] if sp["uncond"] is not None else shared, steps=sp["steps"],
                                        generator=[gr], lora=[sp["lora"]])
        assert torch.equal(req.result, toks), sp
        assert len(req.intermediates) == len(inter) and all(torch.equal(p, q) for p, q in zip(req.intermediates, inter))
        assert g.get_offset() == gr.get_offset()


def test_engine_with_more_distinct_adapters_than_one_launch_takes(tiny):
    """36 requests on 36 distinct adapters in an engine of 40 slots: admission holds the requests past the 32 adapters one step's
    launches take until others retire, so every request completes and equals its batch-1 run."""
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    from paella_b200.lora import load_lora
    m, cfg = tiny[0], tiny[1]
    H = 8
    shared = _one_inputs(m, 6, 99, zeros=True)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=40, max_cond_len=16, unconditional_inputs=shared)
    ads = [load_lora(m, _random_adapter(cfg, 4, 100 + i, 0.1)) for i in range(36)]
    subs = []
    for i, a in enumerate(ads):
        g = torch.Generator(device=DEV).manual_seed(200 + i)
        inputs = _one_inputs(m, 7, 300 + i)
        subs.append((i, inputs, g, eng.submit(inputs, generator=g, steps=2, lora=a)))
    first = eng.step()
    assert len(eng._active) + len(first) <= 32 and len(eng._queue) >= 4
    eng.run_until_idle()
    assert all(req.done for _, _, _, req in subs)
    for i, inputs, g, req in (subs[0], subs[-1]):
        gr = torch.Generator(device=DEV).manual_seed(200 + i)
        toks, _ = U.sample_notebook(m, inputs, (1, H, H), shared, steps=2, generator=[gr], lora=[ads[i]])
        assert torch.equal(req.result, toks) and g.get_offset() == gr.get_offset()


# ------------------------------------------------------------------ 7. combinations
def test_guidance_and_regional_prompts_with_lora_match_batch_one(tiny):
    from paella_b200 import utils as U
    m, _, _, a, b, _, _ = tiny
    B, H = 3, 8
    cond, uncond = _cond(m, B, 10)
    tc, _ = _cond(m, 1, 7, seed=9)
    pc, _ = _cond(m, 1, 6, seed=10)
    region = torch.zeros(H, H, dtype=torch.bool)
    region[:, :4] = True
    entries = [a, (b, 0.5), None]
    kws = [dict(guidance_prompts=[[(tc, 1.5)], None, [(tc, -0.5)]]), dict(prompt_regions=[[(pc, region)], None, [(pc, region)]])]
    for kw in kws:
        seeds = [3, 4, 5]
        ga = _gens(seeds)
        toks, inter = U.sample_notebook(m, cond, (B, H, H), uncond, steps=3, generator=ga, lora=entries, **kw)
        plain, _ = U.sample_notebook(m, cond, (B, H, H), uncond, steps=3, generator=_gens(seeds), **kw)
        assert not torch.equal(toks[0], plain[0])
        for i in range(B):
            gi = _gens([seeds[i]])
            one, one_inter = U.sample_notebook(m, _rows(cond, i), (1, H, H), _rows(uncond, i), steps=3, generator=gi,
                                               lora=[entries[i]], **{k: [v[i]] for k, v in kw.items()})
            assert torch.equal(toks[i], one[0]) and all(torch.equal(p[i], q[0]) for p, q in zip(inter, one_inter))
            assert gi[0].get_offset() == ga[i].get_offset()
        assert torch.equal(toks[2], plain[2])


def test_attention_maps_and_source_edit_with_lora(tiny):
    from paella_b200 import utils as U
    m, _, _, a, b, _, _ = tiny
    B, H = 2, 8
    cond, uncond = _cond(m, B, 10)
    seeds = [6, 7]
    toks = U.sample(m, cond, (B, H, H), uncond, steps=3, generator=_gens(seeds), lora=[a, None])
    toks_m, maps = U.sample(m, cond, (B, H, H), uncond, steps=3, generator=_gens(seeds), lora=[a, None], attention_maps=True)
    assert torch.equal(toks, toks_m) and maps.shape[0] == B and bool(torch.isfinite(maps).all())
    _, maps_plain = U.sample(m, cond, (B, H, H), uncond, steps=3, generator=_gens(seeds), attention_maps=True)
    assert torch.equal(maps[1], maps_plain[1]) and not torch.equal(maps[0], maps_plain[0])
    # an edit on another adapter than its source: same seed as the source; the source equals its own solo run
    seeds = [8, 8]
    edit = U.sample(m, cond, (B, H, H), uncond, steps=3, generator=_gens(seeds), lora=[a, (b, 0.5)], attention_source=[None, (0, 2)])
    solo = U.sample(m, _rows(cond, 0), (1, H, H), _rows(uncond, 0), steps=3, generator=_gens([8]), lora=[a])
    assert torch.equal(edit[0], solo[0])
    no_edit = U.sample(m, cond, (B, H, H), uncond, steps=3, generator=_gens(seeds), lora=[a, (b, 0.5)])
    assert torch.equal(no_edit[0], edit[0])


def test_token_scores_with_lora_against_oracle(tiny):
    from oracle import lora as ol
    from oracle import scores as osc
    m, cfg, sd, a, b, la, lb = tiny
    z, _, _ = _fixture()
    x, r, byt5, clip = (t(z[k]) for k in ("x", "r", "byt5", "clip"))
    y = torch.randint(0, cfg["num_labels"], x.shape, generator=torch.Generator().manual_seed(2))
    entries = [(la, 1.0), (None, 0.0), (lb, 0.5), (la, 2.0)]
    s = m.token_scores(x.to(DEV), r.to(DEV), y.to(DEV), byt5.to(DEV), clip.to(DEV), label_smoothing=0.1,
                       lora=[a, None, (b, 0.5), (a, 2.0)])
    for i, (lsd, sc) in enumerate(entries):
        msd = sd if lsd is None else ol.merge(sd, lsd, sc)
        l64 = osc.score_logits(msd, oracle_cfg(cfg), x[i:i + 1], r[i:i + 1], {"byt5": byt5[i:i + 1], "clip": clip[i:i + 1]})
        nll64, _, loss64, _ = osc.token_scores(l64, y[i:i + 1], 0.1)
        e = max(float((s.nll[i].cpu().double() - nll64[0]).abs().max()), float((s.loss[i].cpu().double() - loss64[0]).abs().max()))
        log_jsonl("lora.jsonl", {"case": "token_scores", "sample": i, "err": e})
        assert e < 1.4e-2, (i, e)


# ------------------------------------------------------------------ validation before anything is enqueued
def test_validation_leaves_generators_alone(tiny):
    from paella_b200 import utils as U
    from paella_b200.lora import load_lora
    from paella_b200.modules import Paella
    m, cfg, _, a, _, la, _ = tiny
    cond, uncond = _cond(m, 2, 8)
    other = Paella(**{**cfg, "c_cond": 40}).to(DEV)
    foreign = load_lora(Paella(**cfg), la)                # packed on the CPU model: another device
    for bad in ([a], [a, (a, float("nan"))], [a, "x"], [a, foreign]):
        gens = _gens([1, 2])
        with pytest.raises(ValueError):
            U.sample(m, cond, (2, 8, 8), uncond, steps=2, generator=gens, lora=bad)
        assert [g.get_offset() for g in gens] == [0, 0]
    with pytest.raises(ValueError, match="another model configuration"):
        other(torch.zeros(1, 8, 8, dtype=torch.int64, device=DEV), torch.ones(1, device=DEV),
              torch.zeros(1, 5, cfg["byt5_embd"], device=DEV), lora=a)
