"""Guidance prompts on the GPU.

  1. Tail forward: pb200_paella_features_tail with the map [2, 0, 2], in a batch with tiled and regional rows, gives each tail row
     the features of its source's tokens and r run as an ordinary row with the tail row's K/V slot, bit for bit (tiny model, and the
     default model with batch_invariant = True); tail rows ignore the regional masks and the attention weights.
  2. Mix kernel: within a few fp32 ulps of the fp64 mix; a weight-0 term leaves the row that the cast_kernel<3> CFG mix gives, so
     the sampler draws the same tokens.
  3. Identity: a sample with one weight-0 term draws the tokens of the call without terms, generator offsets included.
  4. Teacher-forced: the fused sampler on composed rows against the oracle's fp64 mixed distribution, on one stream and per-sample
     streams, with and without top-k / top-p; every mismatch is an audited near-tie.
  5. Per sample: a sample_notebook batch mixing composed, plain, inpainting, tiled, regional and argmax rows equals its batch-1
     calls, and a sample_distributed shard equals its rows (tiny model; default model with batch_invariant = True).
  6. Engine: staggered composed, plain, argmax, quant, truncated and region requests equal their batch-1 sample_notebook calls; an
     engine without guidance prompts allocates what it did before.
  7. The plain path: a call without guidance prompts launches no new kernel, and the same kernels as with all-None terms.
  Validation raises ValueError before anything is enqueued or any generator advances.
"""
import numpy as np
import pytest
import torch

from helpers import load_golden, log_jsonl

pytestmark = pytest.mark.gpu
DEV = "cuda"


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
def tiny_vq():
    from paella_b200.vqgan import VQModel
    cfg, sd, _ = load_golden("vqgan_tiny.npz")
    vq = VQModel(**cfg).to(DEV).eval()
    vq.load_state_dict(sd)
    return vq


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


# ------------------------------------------------------------------ 1. the tail forward
def _tail_forward(m, H):
    from paella_b200 import ops
    from paella_b200.modules import ConditioningCache
    B = 3
    cond, _ = _conditioning(m, B, 12)
    ex, _ = _conditioning(m, 4, 9, seed=8)
    extra = [_rows(ex, slice(k, k + 1)) for k in range(4)]      # extra 0: a regional prompt; 1..3: the tail rows' prompts
    src = [2, 0, 2]
    x = torch.randint(0, m.num_labels, (B, H, H), generator=torch.Generator().manual_seed(1)).to(DEV)
    r = torch.tensor([0.7, 0.3, 0.55], device=DEV)
    with torch.inference_mode():
        full = m.prepare_conditioning([cond], (H, H), share_uniform=False, extra=extra, tail=[1, 2, 3])
        assert full.batch_total == B + 3 and full.slot_map.tolist() == [0, 1, 2, 4, 5, 6]
        wrap = torch.tensor([3, 0, 1], dtype=torch.uint8)
        left = torch.zeros(H, H, dtype=torch.bool)
        left[:, :H // 2] = True
        masks, prompts = ops.regional_table([[(extra[0], left)], None, None], B, (H, H))
        tail_d, wrap_d = ops.to_device_packed([torch.tensor(src, dtype=torch.int32), wrap], DEV)
        regional = m.regional_device((masks, prompts), full)
        got = m.features(x, r, full, wrap=wrap_d, regional=regional, tail_src=tail_d)
        # the same rows as ordinary samples: the sources' tokens and r, each under its tail row's K/V slot, untiled sources' bytes
        one = ConditioningCache(full.cache, 3, full.s_max, full.slots, torch.tensor([4, 5, 6], dtype=torch.int32, device=DEV))
        want = m.features(x[src], r[src], one, wrap=wrap[src].to(DEV))
        # the base rows equal the call without a tail
        base = ConditioningCache(full.cache, B, full.s_max, full.slots, torch.tensor([0, 1, 2], dtype=torch.int32, device=DEV),
                                 full.extra_slot)
        want_base = m.features(x, r, base, wrap=wrap_d, regional=regional)
        # attention weights on the base rows leave the tail rows alone
        w = torch.linspace(0.5, 2.0, 5)
        weighted = m.features(x, r, full, w, B, tail_src=tail_d)
        plain_tail = m.features(x, r, full, tail_src=tail_d)
        want_plain = m.features(x[src], r[src], one)
    n = B * H * H
    assert torch.equal(got[n:], want), float((got[n:] - want).abs().max())
    assert torch.equal(got[:n], want_base)
    assert torch.equal(weighted[n:], plain_tail[n:]) and torch.equal(plain_tail[n:], want_plain)
    assert not torch.equal(weighted[:n], plain_tail[:n])        # the weights act on the base rows
    # the regional mask acts on base row 0 only
    assert not torch.equal(got[:H * H], m.features(x, r, base, wrap=wrap_d)[:H * H])


def test_tail_forward_tiny(tiny):
    _tail_forward(tiny, 8)


def test_tail_forward_default_model_batch_invariant(default_model):
    _tail_forward(default_model, 16)


# ------------------------------------------------------------------ 2. the mix kernel
def test_mix_kernel_against_fp64(tiny):
    from oracle import guidance as og
    from paella_b200 import ops
    m = tiny
    c_out, hw = m._cfg["c_out"], 64
    weights = [[0.5, -1.25, 2.0], [], [0.75], [-0.5, 0.25, 1.5, -2.0, 0.1, 0.3, -0.7]]
    comp = [0, 1, 2, 3]
    trows, k = [], 4 + 4
    for ws in weights:
        trows.append(list(range(k, k + len(ws))))
        k += len(ws)
    f0 = torch.randn(k * hw, c_out, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5)) * 3.0
    rows, coef = ops.guidance_mix_table(weights, comp, [4 + b for b in comp], trows, [[7.5, 3.0, 1.0, 4.25]])
    rows_d, coef_d = ops.to_device_packed([rows, coef[0]], DEV)
    f = f0.clone()
    m.guidance_mix(f, hw, rows_d, coef_d)
    torch.cuda.synchronize()
    fs = f0.double().view(-1, hw, c_out).cpu()
    got = f.view(-1, hw, c_out).cpu()
    worst = 0.0
    for y, b in enumerate(comp):
        a = coef[0, y].double()
        idx = rows[y].tolist()
        want = og.mix(fs[b], fs[4 + b], [fs[j] for j in trows[y]], [7.5, 3.0, 1.0, 4.25][y], weights[y])
        mag = a[0].abs() * fs[b].abs() + a[1].abs() * fs[4 + b].abs() + sum(a[2 + j].abs() * fs[t].abs() for j, t in enumerate(idx[2:]) if t >= 0)
        # 2 + J fp32 coefficients and 1 + J fmaf roundings (plus the product u * a_u), each within 2^-24 of the magnitude
        err = ((got[b].double() - want).abs() / (mag * 2.0 ** -24 + 1e-30)).max().item()
        worst = max(worst, err / (2 * (2 + len(weights[y])) + 1))
    log_jsonl("guidance_prompts.jsonl", {"test": "mix_fp64", "max_err_over_bound": worst})
    assert worst <= 1.0, worst
    # untouched rows: every row that is not a composed sample's conditional row
    assert torch.equal(f[4 * hw:], f0[4 * hw:])

    # a weight-0 term: the mixed row, drawn with (1, 0, 1/T), gives the tokens of the CFG mix of cast_kernel<3>
    B = 3
    g = torch.Generator(device=DEV).manual_seed(6)
    feats = torch.randn(3 * B * hw, c_out, device=DEV, generator=g) * 2.0
    cfgs = [4.0, 6.5, 1.5]
    params = ops.sampling_params_table(torch.tensor(cfgs, dtype=torch.float64), 0.8, B, DEV)
    rows, coef = ops.guidance_mix_table([[0.0]] * B, list(range(B)), [B + b for b in range(B)], [[2 * B + b] for b in range(B)], [cfgs])
    rows_d, coef_d = ops.to_device_packed([rows, coef[0]], DEV)
    mixed = feats.clone()
    m.guidance_mix(mixed, hw, rows_d, coef_d)
    one = ops.sampling_params([[1.0]] * B, [[0.8]] * B)[:, 0]
    one[:, 0], one[:, 1] = 1.0, 0.0
    one_d = ops.to_device_async(one, DEV)
    ga, gb = _gens([1, 2, 3]), _gens([1, 2, 3])
    a = m.sample_tokens_params(feats, B, 8, 8, True, params, ga)
    b = m.sample_tokens_params(mixed, B, 8, 8, True, one_d, gb)
    assert torch.equal(a, b)
    assert [x.get_offset() for x in ga] == [x.get_offset() for x in gb]


# ------------------------------------------------------------------ 3. identity
def _identity(m, H, seeds):
    from paella_b200 import utils as U
    B = 3
    cond, uncond = _conditioning(m, B, 12)
    tc, _ = _conditioning(m, 1, 7, seed=9)
    kw = dict(steps=3, temperature=(1.1, 0.3))
    ga, gb = _gens(seeds), _gens(seeds)
    a, ia = U.sample_notebook(m, cond, (B, H, H), uncond, generator=ga, **kw)
    b, ib = U.sample_notebook(m, cond, (B, H, H), uncond, generator=gb, guidance_prompts=[None, [(tc, 0.0)], None], **kw)
    assert torch.equal(a, b) and all(torch.equal(x, y) for x, y in zip(ia, ib))
    assert [g.get_offset() for g in ga] == [g.get_offset() for g in gb]
    # and a term of nonzero weight changes its sample alone
    c, _ = U.sample_notebook(m, cond, (B, H, H), uncond, generator=_gens(seeds), guidance_prompts=[None, [(tc, 1.5)], None], **kw)
    assert torch.equal(c[0], a[0]) and torch.equal(c[2], a[2]) and not torch.equal(c[1], a[1])
    # sample(), scalar cfg, one stream
    torch.manual_seed(3)
    a = U.sample(m, cond, (B, H, H), uncond, steps=3)
    off = torch.cuda.default_generators[0].get_offset()
    torch.manual_seed(3)
    b = U.sample(m, cond, (B, H, H), uncond, steps=3, guidance_prompts=[[(tc, 0.0)]] * B)
    assert torch.equal(a, b) and off == torch.cuda.default_generators[0].get_offset()


def test_identity_tiny(tiny):
    _identity(tiny, 8, [4, 5, 6])
    tiny.batch_invariant = True
    try:
        _identity(tiny, 8, [7, 8, 9])
    finally:
        tiny.batch_invariant = False


def test_identity_default_model_batch_invariant(default_model):
    _identity(default_model, 16, [10, 11, 12])


# ------------------------------------------------------------------ 4. teacher-forced against the fp64 oracle
def _big_model(NL=8192):
    from paella_b200.modules import Paella
    cfg, _, _ = load_golden("paella_tiny.npz")
    big = dict(cfg)
    big.update(c_in=256, c_out=256, num_labels=NL)
    torch.manual_seed(0)
    m = Paella(**big).to(DEV).eval()
    W = m.out_mapper[1].weight.detach().view(NL, 256) * 30.0        # spread the logits
    with torch.no_grad():
        m.out_mapper[1].weight.copy_(W.view(NL, 256, 1, 1))
    m.pack_weights()
    return m


S_REL = 2.0 ** -14         # fp32 GEMM over 256 products, relative to the row's max |s| (as the truncation tests bound it)
MASS_REL = 2.0 ** -16


@pytest.mark.parametrize("trunc", [None, (64, 0.9)])
@pytest.mark.parametrize("streams", ["per_sample", "one"])
def test_sampler_on_composed_rows_against_fp64_oracle(streams, trunc):
    from oracle import guidance as og
    from oracle.truncation import boundary_distance, kept_set, truncated_winner
    from paella_b200 import ops
    m = _big_model()
    NL, c_out, H, hw = m.num_labels, 256, 16, 256
    B = 4
    weights = [[0.5], [0.5, -0.5], [-0.25, 1.0, 0.3], [2.0]]
    T, cfg = 0.7, 3.0
    n_terms = sum(len(w) for w in weights)
    feats = torch.randn((2 * B + n_terms) * hw, c_out, device=DEV, generator=torch.Generator(device=DEV).manual_seed(8)) * 0.5
    f64 = feats.double().view(-1, hw, c_out).cpu()
    trows, k = [], 2 * B
    for ws in weights:
        trows.append(list(range(k, k + len(ws))))
        k += len(ws)
    rows, coef = ops.guidance_mix_table(weights, list(range(B)), [B + b for b in range(B)], trows, [[cfg] * B])
    one = ops.sampling_params([[1.0]] * B, [[T]] * B)[:, 0]
    one[:, 0], one[:, 1] = 1.0, 0.0
    rows_d, coef_d, params_d = ops.to_device_packed([rows, coef[0], one], DEV)
    tr = None
    ks, ps = [0] * B, [1.0] * B
    if trunc is not None:
        ks, ps = [trunc[0]] * B, [trunc[1]] * B
        tr = tuple(ops.to_device_packed([torch.tensor(ks, dtype=torch.int32), torch.tensor(ps, dtype=torch.float32)], DEV))
    mixed = feats.clone()
    m.guidance_mix(mixed, hw, rows_d, coef_d)
    seeds = list(range(900, 900 + B))
    if streams == "per_sample":
        gens = _gens(seeds)
        got = m.sample_tokens_params(mixed, B, H, H, True, params_d, gens, tr).view(B, hw).cpu().numpy()
        qs = []
        for b in range(B):
            g = torch.Generator(device=DEV).manual_seed(seeds[b])
            qs.append(torch.empty(hw, NL, device=DEV).exponential_(1, generator=g).double().cpu().numpy())
            assert g.get_offset() == gens[b].get_offset()
    else:
        g = torch.Generator(device=DEV).manual_seed(77)
        got = m.sample_tokens_params(mixed, B, H, H, True, params_d, g, tr).view(B, hw).cpu().numpy()
        g2 = torch.Generator(device=DEV).manual_seed(77)
        q = torch.empty(B * hw, NL, device=DEV).exponential_(1, generator=g2).double().cpu().numpy()
        assert g.get_offset() == g2.get_offset()
        qs = [q[b * hw:(b + 1) * hw] for b in range(B)]
    W = m.out_mapper[1].weight.detach().view(NL, c_out).half().double().cpu()
    inv_t = float(np.float32(1.0) / np.float32(T))
    agree, total, bad = 0, 0, []
    for b in range(B):
        a64 = og.mix(f64[b], f64[B + b], [f64[j] for j in trows[b]], cfg, weights[b])          # [hw, c_out] fp64
        s = ((a64 @ W.t()) * inv_t).numpy()
        # the kernel's operand is fp16 of the fp32 mix: half an fp16 ulp per element, through |W|
        ds_rows = (((a64.abs() * 2.0 ** -11) @ W.abs().t()).max(1).values * inv_t).numpy() + S_REL * np.abs(s).max(1)
        want = truncated_winner(s, qs[b], ks[b], ps[b])
        agree += int((want == got[b]).sum())
        total += hw
        for j in np.nonzero(want != got[b])[0]:
            sj, ds = s[j], ds_rows[j]
            score = sj - np.log(qs[b][j])
            loose = np.ones(NL, bool)
            tight = np.ones(NL, bool)
            tau_k, _ = boundary_distance(sj, ks[b], 1.0)
            if tau_k is not None:
                loose &= sj >= tau_k - ds
                tight &= sj >= tau_k + ds
            if 0 < ps[b] < 1:
                rel = MASS_REL + 4 * ds
                kl, kh = kept_set(sj, ks[b], max(ps[b] * (1 - rel), 1e-300)), kept_set(sj, ks[b], min(ps[b] * (1 + rel), 1.0))
                lo, hi = sj[kl].min(), sj[kh].min()
                loose &= sj >= min(lo, hi) - ds
                tight &= sj >= max(lo, hi) + ds
            g_, w_ = got[b][j], want[j]
            if not loose[g_]:
                bad.append((b, int(j), "outside the kept set"))
                continue
            best = np.max(np.where(tight, score, -np.inf))
            if score[g_] >= best - (2 * ds + 8 * 2.0 ** -24 * np.abs(score).max()) or not tight[w_] or not tight[g_]:
                continue
            bad.append((b, int(j), "unexplained"))
    log_jsonl("guidance_prompts.jsonl", {"test": "teacher_forced", "streams": streams, "trunc": trunc, "agreement": agree / total,
                                         "unexplained": [str(x) for x in bad[:5]]})
    assert not bad, bad[:5]
    assert agree / total >= 0.99, agree / total


# ------------------------------------------------------------------ 5. per sample
def _mixed_rows_equal_batch1(m, H, steps, seeds):
    from paella_b200 import utils as U
    B = 5
    cond, uncond = _conditioning(m, B, 12)
    tc, _ = _conditioning(m, 4, 6, seed=9)
    tb, _ = _conditioning(m, 1, 10, seed=10)
    left = torch.zeros(H, H, dtype=torch.bool)
    left[:, :H // 2] = True
    terms = [[(_rows(tc, slice(0, 1)), 0.5), (_rows(tb, slice(0, 1)), -0.75)],     # composed: an extra and a negative prompt
             None,                                                                 # plain
             [(_rows(tc, slice(1, 2)), 1.25)],                                     # composed + inpainting + argmax
             [(_rows(tc, slice(2, 3)), -0.5)],                                     # composed + regional + tiled + truncated
             None]                                                                 # tiled
    regions = [None, None, None, [(_rows(tc, slice(3, 4)), left)], None]
    tilings = ["none", "none", "none", "xy", "x"]
    modes = ["multinomial", "multinomial", "argmax", "multinomial", "multinomial"]
    top_k = torch.tensor([0, 0, 0, 7, 0])
    cfg = torch.tensor([[8.0, 6.0], [0.0, 0.0], [4.0, 4.0], [7.0, 2.0], [5.0, 5.0]], dtype=torch.float64)
    init = torch.randint(0, m.num_labels, (B, H, H), generator=torch.Generator().manual_seed(2))
    region = torch.ones(B, H, H, dtype=torch.bool)
    region[2, 1:H - 1, 2:H - 2] = False
    gens = _gens(seeds)
    kw = dict(steps=steps, temperature=(1.2, 0.2))
    got, inter = U.sample_notebook(m, cond, (B, H, H), uncond, init_x=init, region=region, cfg=cfg, generator=gens, tiling=tilings,
                                   top_k=top_k, prompt_regions=regions, guidance_prompts=terms, mode=modes, **kw)
    for i in range(B):
        g1 = _gens([seeds[i]])
        want, inter1 = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), init_x=init[i:i + 1],
                                         region=region[i:i + 1], cfg=cfg[i:i + 1], generator=g1, tiling=tilings[i],
                                         top_k=top_k[i:i + 1], prompt_regions=[regions[i]], guidance_prompts=[terms[i]], mode=modes[i],
                                         **kw)
        assert torch.equal(got[i:i + 1], want), i
        assert all(torch.equal(a[i:i + 1], b) for a, b in zip(inter, inter1)), i
        assert g1[0].get_offset() == gens[i].get_offset(), i
    g2 = _gens(seeds[1:4])
    shard = U.sample_distributed(m, _rows(cond, slice(1, 4)), _rows(uncond, slice(1, 4)), (3, H, H), init_x=init[1:4],
                                 region=region[1:4], cfg=cfg[1:4], generator=g2, tiling=tilings[1:4], top_k=top_k[1:4],
                                 prompt_regions=regions[1:4], guidance_prompts=terms[1:4], **kw)
    want, _ = U.sample_notebook(m, _rows(cond, slice(1, 4)), (3, H, H), _rows(uncond, slice(1, 4)), init_x=init[1:4],
                                region=region[1:4], cfg=cfg[1:4], generator=_gens(seeds[1:4]), tiling=tilings[1:4], top_k=top_k[1:4],
                                prompt_regions=regions[1:4], guidance_prompts=terms[1:4], **kw)
    assert torch.equal(shard, want)
    # the terms change the composed rows and leave the others
    plain, _ = U.sample_notebook(m, cond, (B, H, H), uncond, init_x=init, region=region, cfg=cfg, generator=_gens(seeds), tiling=tilings,
                                 top_k=top_k, prompt_regions=regions, mode=modes, **kw)
    assert not torch.equal(plain[0], got[0]) and torch.equal(plain[1], got[1]) and torch.equal(plain[4], got[4])


def test_tiny_mixed_composed_rows_equal_batch1_calls(tiny):
    _mixed_rows_equal_batch1(tiny, 8, 4, [3, 14, 15, 92, 65])


def test_default_model_batch_invariant_composed_rows(default_model):
    _mixed_rows_equal_batch1(default_model, 16, 3, [8, 80, 800, 8000, 80000])


# ------------------------------------------------------------------ validation
def test_validation_enqueues_nothing(tiny):
    from paella_b200 import utils as U
    cond, uncond = _conditioning(tiny, 2, 12)
    p = _rows(cond, slice(0, 1))
    gens = _gens([1, 2])
    offs = [g.get_offset() for g in gens]
    off0 = torch.cuda.default_generators[0].get_offset()
    bad_values = [[(p, 1.0)], [[(p, 1.0)]], "terms", [[(p, 1.0)] * 8, None], [[(p, float("nan"))], None], [[(cond, 1.0)], None],
                  [[(p,)], None], [[(p, "x")], None]]
    for bad in bad_values:
        for f in (lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=gens, guidance_prompts=bad),
                  lambda: U.sample_notebook(tiny, cond, (2, 8, 8), uncond, steps=2, generator=gens, guidance_prompts=bad),
                  lambda: U.sample_distributed(tiny, cond, uncond, (2, 8, 8), steps=2, generator=gens, guidance_prompts=bad)):
            with pytest.raises(ValueError):
                f()
    ok = [[(p, 1.0)], None]
    for f in (lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=gens, cfg=0, guidance_prompts=ok),
              lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=gens, cfg=torch.tensor([0.0, 3.0]), guidance_prompts=ok),
              lambda: U.sample_notebook(tiny, cond, (2, 8, 8), uncond, steps=2, generator=gens, cfg=None, guidance_prompts=ok),
              lambda: U.sample_distributed(tiny, cond, uncond, (2, 8, 8), steps=2, generator=gens, cfg=None, guidance_prompts=ok),
              lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=gens, exact=True, guidance_prompts=ok),
              lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, exact=True, guidance_prompts=ok)):
        with pytest.raises(ValueError):
            f()
    assert [g.get_offset() for g in gens] == offs and torch.cuda.default_generators[0].get_offset() == off0
    # a per-sample cfg of 0 on a sample without terms is fine
    U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([1, 2]), cfg=torch.tensor([3.0, 0.0]), guidance_prompts=ok)


# ------------------------------------------------------------------ 6. engine
def _engine_equals_batch1(m, H, vq=None):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    N = 7
    cond, uncond = _conditioning(m, N, 12, seed=21)
    tc, _ = _conditioning(m, 8, 6, seed=22)
    t1 = lambda i: _rows(tc, slice(i, i + 1))          # noqa: E731
    region = torch.ones(1, H, H, dtype=torch.bool)
    region[0, 1:H - 1, 2:H - 2] = False
    init = torch.randint(0, m.num_labels, (1, H, H), generator=torch.Generator().manual_seed(5))
    left = torch.zeros(H, H, dtype=torch.bool)
    left[:, :H // 2] = True
    kinds = [dict(guidance_prompts=[(t1(0), 0.5), (t1(1), -0.5)]),
             dict(),
             dict(guidance_prompts=[(t1(2), 1.0)], mode="argmax"),
             dict(guidance_prompts=[(t1(3), 0.75)], mode="quant" if vq is not None else "argmax", sampling_quant_steps=None),
             dict(guidance_prompts=[(t1(4), -0.25)], top_k=5, top_p=0.9, tiling="xy"),
             dict(guidance_prompts=[(t1(5), 0.5)], region=region, init_x=init, sampling_conditional_steps=2),
             dict(guidance_prompts=[(t1(6), 0.5)], prompt_regions=[(t1(7), left)])]
    steps = [3, 4, 2, 3, 4, 3, 3]
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=3, max_cond_len=40, vqmodel=vq, max_prompt_regions=1, max_guidance_prompts=2)
    reqs = []
    for i, kw in enumerate(kinds):
        g = torch.Generator(device=DEV).manual_seed(70 + i)
        reqs.append((eng.submit(_rows(cond, slice(i, i + 1)), _rows(uncond, slice(i, i + 1)), generator=g, steps=steps[i],
                                temperature=(1.2, 0.2), keep_intermediates=True, **kw), g, kw))
        if i % 2:
            eng.step()                # staggered arrivals; max_batch 3 reuses slots and their term K/V slots
    eng.run_until_idle()
    for i, (q, g, kw) in enumerate(reqs):
        kw = dict(kw)
        for key in ("guidance_prompts", "prompt_regions"):
            if key in kw:
                kw[key] = [kw[key]]
        g1 = torch.Generator(device=DEV).manual_seed(70 + i)
        want, inter = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), steps=steps[i],
                                        temperature=(1.2, 0.2), generator=[g1], vqmodel=vq, **kw)
        assert torch.equal(q.result, want), (i, kw.keys())
        assert all(torch.equal(a, b) for a, b in zip(q.intermediates, inter)), i
        assert g.get_offset() == g1.get_offset(), i


def test_engine_composed_requests_equal_batch1_notebook(tiny, tiny_vq):
    _engine_equals_batch1(tiny, 8, tiny_vq)


def test_default_model_engine_composed_requests(default_model):
    _engine_equals_batch1(default_model, 16)


def test_engine_allocation_and_validation(tiny):
    from paella_b200._lib import lib
    from paella_b200.engine import SamplingEngine
    eng = SamplingEngine(tiny, latent_hw=(8, 8), max_batch=3, max_cond_len=40)
    assert eng.cache.cache.numel() == lib().pb200_paella_cond_cache_bytes(tiny._handle, 2 * 3 + 1, 40)
    eng2 = SamplingEngine(tiny, latent_hw=(8, 8), max_batch=3, max_cond_len=40, max_guidance_prompts=2)
    assert eng2.cache.cache.numel() == lib().pb200_paella_cond_cache_bytes(tiny._handle, 2 * 3 + 1 + 2 * 3, 40)
    for bad in (-1, 8, 1.5, True):
        with pytest.raises(ValueError):
            SamplingEngine(tiny, latent_hw=(8, 8), max_batch=2, max_cond_len=60, max_guidance_prompts=bad)
    cond, uncond = _conditioning(tiny, 1, 12)
    long, _ = _conditioning(tiny, 1, 40, seed=3)
    g = torch.Generator(device=DEV).manual_seed(1)
    off = g.get_offset()
    for bad in ([(cond, 1.0)] * 3, (cond, 1.0), [(cond, float("inf"))], [(long, 1.0)], [(cond,)], "x",
                [({"byt5": torch.randn(2, 3, cond["byt5"].shape[2], device=DEV)}, 1.0)]):
        with pytest.raises(ValueError):
            eng2.submit(cond, uncond, generator=g, guidance_prompts=bad)
    with pytest.raises(ValueError):
        eng2.submit(cond, uncond, generator=g, cfg=None, guidance_prompts=[(cond, 1.0)])
    with pytest.raises(ValueError):
        eng.submit(cond, uncond, generator=g, guidance_prompts=[(cond, 1.0)])
    assert not eng.busy and not eng2.busy and g.get_offset() == off


# ------------------------------------------------------------------ 7. the plain path
def _kernel_names(f):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_plain_call_launches_no_new_kernel(tiny):
    from paella_b200 import utils as U
    cond, uncond = _conditioning(tiny, 2, 12)
    tc, _ = _conditioning(tiny, 1, 6, seed=9)
    U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([1, 2]))          # warm-up
    plain = _kernel_names(lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([1, 2])))
    none = _kernel_names(lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([1, 2]), guidance_prompts=[None, None]))
    composed = _kernel_names(lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([1, 2]),
                                              guidance_prompts=[[(tc, 0.5)], None]))
    assert plain == none
    assert not any("guidance_mix" in n or "replicate_rows" in n for n in plain)
    assert any("guidance_mix" in n for n in composed) and any("replicate_rows" in n for n in composed)
    log_jsonl("guidance_prompts.jsonl", {"test": "plain_kernels", "n_plain": len(plain), "n_composed": len(composed)})
