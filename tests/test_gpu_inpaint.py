"""Inpainting and outpainting: ``region`` on sample_distributed, sample_notebook and SamplingEngine.submit.

The contract, per sample, on the sample's generator g (utils module docstring):

    init_noise = torch.randint(0, num_labels, (B, H, W), generator=g)
    sampled = torch.where(region, init_noise, init_x)
    for each step i: sample as without a region, then sampled = torch.where(region, sampled, init_x)   (an intermediate)
        if i < renoise_steps:
            m = (torch.rand(B, H, W, generator=g) <= t_next[:, None, None]) & region
            sampled = model.add_noise(sampled, t_next, mask=m.long(), random_x=init_noise)[0]        (an intermediate)

  * kernel level: the masked add-noise of both kernels against the torch expression (odd H*W, B = 1 and 128, a slot map,
    t < 0 rows, random_x given and drawn)
  * tiny golden model, bit for bit: the restated loop against sample_notebook in every mode and sample_distributed with and
    without exact=True; an all-True region is the call without init_x (tokens and generator offsets); an all-False one
    returns init_x; every intermediate holds init_x outside the region
  * per-sample batching: region, all-True, all-False and outpainting rows with per-sample generators, cfg and temperature;
    row i equals its batch-1 call (tiny model; default model with one forced GEMM tile width in a child process), and a
    teacher-forced Gumbel-margin audit on the default model with the normal planner
  * SamplingEngine: staggered inpainting, outpainting and plain requests, a slot reused by a request without a region; each
    equals its batch-1 call, with no host synchronisation in submit or step
  * host only: validation, token_region, outpaint_canvas
"""
import os
import subprocess
import sys

import pytest
import torch

from helpers import load_golden, log_jsonl

DEV = "cuda"
gpu = pytest.mark.gpu


def _log(payload):
    log_jsonl("inpaint.jsonl", payload)


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


def _inputs(m, B, L, seed=0, zeros=False, device=DEV):
    g = torch.Generator().manual_seed(seed)
    E, C = m.byt5_mapper.in_features, m.clip_mapper.in_features
    d = {"byt5": torch.randn(B, L, E, generator=g), "clip": torch.randn(B, C, generator=g)}
    if zeros:
        d = {k: torch.zeros_like(v) for k, v in d.items()}
    return {k: v.to(device) for k, v in d.items()}


def _row(d, i):
    return {k: v[i:i + 1] for k, v in d.items()}


def _region(B, H, W, seed, p=0.5):
    return torch.rand(B, H, W, generator=torch.Generator().manual_seed(seed)) < p


def _tokens(NL, B, H, W, seed):
    return torch.randint(0, NL, (B, H, W), generator=torch.Generator().manual_seed(seed))


@pytest.fixture(scope="module")
def tiny():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m


def _vq(num_labels):
    from paella_b200.vqgan import VQModel
    torch.manual_seed(0)
    return VQModel(levels=2, bottleneck_blocks=1, c_hidden=32, c_latent=4, codebook_size=num_labels).to(DEV)


def _default_model():
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    return m.to(DEV)


# ------------------------------------------------------------------ host only
def test_token_region_marks_the_whole_token_of_one_masked_pixel():
    from paella_b200 import utils as U
    mask = torch.zeros(2, 16, 24, dtype=torch.bool)
    mask[0, 5, 6] = True                       # token (1, 1)
    mask[1, 15, 23] = True                     # the last pixel: token (3, 5)
    r = U.token_region(mask)
    assert r.shape == (2, 4, 6) and r.dtype == torch.bool
    want = torch.zeros(2, 4, 6, dtype=torch.bool)
    want[0, 1, 1] = want[1, 3, 5] = True
    assert torch.equal(r, want)
    assert torch.equal(U.token_region(torch.ones(8, 4)), torch.ones(2, 1, dtype=torch.bool))
    with pytest.raises(ValueError):
        U.token_region(torch.zeros(1, 6, 8, dtype=torch.bool))        # not whole tokens


@pytest.mark.parametrize("top,left", [(0, 0), (5, 2), (0, 2), (5, 0)])
def test_outpaint_canvas_places_tokens_and_region(top, left):
    from paella_b200 import utils as U
    tok = _tokens(64, 2, 3, 4, 1)
    init_x, region = U.outpaint_canvas(tok, (8, 6), top, left)
    assert init_x.shape == region.shape == (2, 8, 6) and init_x.dtype == torch.int64 and region.dtype == torch.bool
    assert torch.equal(init_x[:, top:top + 3, left:left + 4], tok)
    assert not region[:, top:top + 3, left:left + 4].any()
    assert int(region.sum()) == 2 * (48 - 12) and int((init_x * region).abs().sum()) == 0
    for bad in ((6, 0), (0, 3), (-1, 0)):
        with pytest.raises(ValueError):
            U.outpaint_canvas(tok, (8, 6), *bad)


def test_check_region_rejects_bad_regions():
    from paella_b200 import utils as U
    shape, dev = (2, 4, 5), torch.device("cuda", 0)
    x, r = torch.zeros(shape, dtype=torch.int64), torch.ones(shape, dtype=torch.bool)
    U.check_region(None, None, shape, dev)
    U.check_region(r, x, shape, dev)
    for region, init_x in [(r, None),                                        # no source tokens
                           (r[:, :3], x), (r, x[:1]),                        # wrong shape
                           (r.to(torch.uint8), x), (r, x.float()),           # wrong dtype
                           (r.to("meta"), x), (r, x.to("meta"))]:            # another device
        with pytest.raises(ValueError):
            U.check_region(region, init_x, shape, dev)


# ------------------------------------------------------------------ 1. kernel level
@gpu
@pytest.mark.parametrize("B,H,W", [(1, 7, 9), (128, 27, 27), (3, 5, 7)])
def test_masked_add_noise_equals_torch(B, H, W):
    from paella_b200 import ops
    K = 8192
    x = torch.randint(0, K, (B, H, W), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    rx = torch.randint(0, K, (B, H, W), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    src = torch.randint(0, K, (B, H, W), device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    tt = torch.rand(B, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    tt[1::3] = -1.0                                           # rows that only composite
    region = _region(B, H, W, 4).to(DEV)
    region[0] = True
    if B > 2:
        region[2] = False
    seeds = [500 + 7 * b for b in range(B)]
    for random_x in (rx, None):
        # one generator for the batch
        g, ref = _gens([9, 9])
        out, mask = ops.add_noise(x, tt, random_x, K, g, src=src, region=region)
        u = torch.rand(B, H, W, device=DEV, generator=ref)
        r_ref = rx if random_x is not None else torch.randint(0, K, (B, H, W), device=DEV, generator=ref)
        m_ref = (u <= tt[:, None, None]) & region
        assert torch.equal(mask.bool(), m_ref)
        assert torch.equal(out, torch.where(region, torch.where(m_ref, r_ref, x), src))
        assert g.get_offset() == ref.get_offset()
        # per-sample generators
        gens, refs = _gens(seeds), _gens(seeds)
        out, mask = ops.add_noise(x, tt, random_x, K, gens, src=src, region=region)
        for b in range(B):
            u = torch.rand(1, H, W, device=DEV, generator=refs[b])
            r_ref = rx[b:b + 1] if random_x is not None else torch.randint(0, K, (1, H, W), device=DEV, generator=refs[b])
            m_ref = (u <= tt[b]) & region[b:b + 1]
            assert torch.equal(mask[b:b + 1].bool(), m_ref), b
            assert torch.equal(out[b:b + 1], torch.where(region[b:b + 1], torch.where(m_ref, r_ref, x[b:b + 1]), src[b:b + 1])), b
        assert [q.get_offset() for q in gens] == [q.get_offset() for q in refs]
    # the engine's form: random_x, src, region and out by slot
    slot = torch.randperm(B, generator=torch.Generator().manual_seed(6)).to(torch.int32).to(DEV)
    table = ops.philox_table(_gens(seeds), H * W, DEV)
    pool = torch.full_like(x, -7)
    mask = torch.empty_like(x)
    ops.add_noise_per_sample(x, tt, rx, K, table, pool, mask, slot=slot, src=src, region=region)
    refs = _gens(seeds)
    for b in range(B):
        s = int(slot[b])
        m_ref = (torch.rand(1, H, W, device=DEV, generator=refs[b]) <= tt[b]) & region[s:s + 1]
        assert torch.equal(mask[b:b + 1].bool(), m_ref), b
        assert torch.equal(pool[s:s + 1], torch.where(region[s:s + 1], torch.where(m_ref, rx[s:s + 1], x[b:b + 1]), src[s:s + 1])), b
    # the composite-only launch takes no Philox offset
    neg = torch.full((B,), -1.0, device=DEV)
    assert torch.equal(ops.composite(x, src, region, neg), torch.where(region, x, src))


# ------------------------------------------------------------------ 2. the contract, restated, on the tiny model
def _restated(m, cond, uncond, B, H, W, init_x, region, g, steps=4, renoise_steps=None, temperature=(0.7, 0.3), cfg=(8.0, 8.0),
              mode="multinomial", exact=False, quant_steps=None, codebook=None):
    """The contract loop with the per-step ops the call uses (one CUDA generator g for the batch)."""
    from paella_b200 import ops
    renoise_steps = steps - 1 if renoise_steps is None else renoise_steps
    t_list = torch.linspace(1.0, 0.0, steps + 1)
    temps = torch.linspace(temperature[0], temperature[1], steps)
    cfgs = torch.linspace(cfg[0], cfg[1], steps).tolist()
    init_x, region = init_x.to(DEV), region.to(DEV)
    inter = []
    with torch.inference_mode():
        init_noise = torch.randint(0, m.num_labels, (B, H, W), device=DEV, generator=g)
        sampled = torch.where(region, init_noise, init_x)
        pair = m.prepare_conditioning([cond, uncond], (H, W))
        for i in range(steps):
            md = "quant" if quant_steps is not None and i >= quant_steps else mode
            r = torch.full((B,), float(t_list[i]), device=DEV)
            c, T = float(cfgs[i]), float(temps[i])
            if md == "multinomial" and not exact:
                sampled = m.sample_tokens(m.features(sampled, r, pair, cfg_pairs=True), B, H, W, c, T, g)
            else:
                lc, lu = m(sampled, r, **cond), m(sampled, r, **uncond)
                sampled = ops.resample_quant(lc, lu, c, T, codebook) if md == "quant" else ops.resample_logits(lc, lu, c, T, md, g)
            sampled = torch.where(region, sampled, init_x)
            inter.append(sampled)
            if i < renoise_steps:
                t_next = torch.full((B,), float(t_list[i + 1]), device=DEV)
                mk = (torch.rand(B, H, W, device=DEV, generator=g) <= t_next[:, None, None]) & region
                sampled = m.add_noise(sampled, t_next, mask=mk.long(), random_x=init_noise)[0]
                inter.append(sampled)
    return sampled, inter


CALLS = ["nb-multinomial", "nb-argmax", "nb-quant", "nb-quant_steps", "distributed", "distributed-exact"]


@gpu
@pytest.mark.parametrize("call", CALLS)
def test_tiny_call_equals_restated_contract(call, tiny):
    from paella_b200 import utils as U
    m, B, H = tiny, 2, 8
    cond, uncond = _inputs(m, B, 6, seed=1), _inputs(m, B, 6, zeros=True)
    init_x, region = _tokens(m.num_labels, B, H, H, 2), _region(B, H, H, 3)
    vq = _vq(m.num_labels)
    cb = vq.vquantizer.codebook.weight.data
    mode = {"nb-quant_steps": "multinomial", "distributed": "multinomial", "distributed-exact": "multinomial"}.get(call, call[3:])
    qs = 2 if call == "nb-quant_steps" else None
    g, ref = _gens([11, 11])
    want, want_inter = _restated(m, cond, uncond, B, H, H, init_x, region, ref, mode=mode, exact=call == "distributed-exact",
                                 quant_steps=qs, codebook=cb)
    if call.startswith("distributed"):
        got = U.sample_distributed(m, cond, uncond, (B, H, H), init_x=init_x, steps=4, exact=call == "distributed-exact",
                                   generator=g, region=region)
        inter = None
    else:
        got, inter = U.sample_notebook(m, cond, (B, H, H), uncond, init_x=init_x, steps=4, mode=mode, sampling_quant_steps=qs,
                                       vqmodel=vq, generator=g, region=region)
    assert torch.equal(got, want)
    assert g.get_offset() == ref.get_offset()
    keep = ~region.to(DEV)
    if inter is not None:
        assert len(inter) == len(want_inter)
        for a, b in zip(inter, want_inter):
            assert torch.equal(a, b)
            assert torch.equal(a[keep], init_x.to(DEV)[keep])          # outside the region: init_x at every intermediate
    assert torch.equal(got[keep], init_x.to(DEV)[keep])


@gpu
@pytest.mark.parametrize("call", ["nb-multinomial", "nb-argmax", "distributed", "distributed-exact"])
def test_tiny_all_true_and_all_false_regions(call, tiny):
    from paella_b200 import utils as U
    m, B, H = tiny, 2, 8
    cond, uncond = _inputs(m, B, 5, seed=4), _inputs(m, B, 5, zeros=True)
    init_x = _tokens(m.num_labels, B, H, H, 5).to(DEV)
    exact = call == "distributed-exact"

    def run(g, **kw):
        if call.startswith("distributed"):
            return U.sample_distributed(m, cond, uncond, (B, H, H), steps=3, exact=exact, generator=g, **kw)
        return U.sample_notebook(m, cond, (B, H, H), uncond, steps=3, mode=call[3:], generator=g, **kw)[0]

    for gen in ("one", "per_sample"):
        mk = (lambda: _gens([21])[0]) if gen == "one" else (lambda: _gens([21, 22]))
        offs = lambda g: [q.get_offset() for q in (g if isinstance(g, list) else [g])]     # noqa: E731
        g0, g1, g2 = mk(), mk(), mk()
        plain = run(g0)
        full = run(g1, init_x=init_x, region=torch.ones(B, H, H, dtype=torch.bool))
        assert torch.equal(full, plain) and offs(g1) == offs(g0), gen
        none = run(g2, init_x=init_x, region=torch.zeros(B, H, H, dtype=torch.bool))
        assert torch.equal(none, init_x) and offs(g2) == offs(g0), gen


# ------------------------------------------------------------------ 3. per-sample batching
def _mixed_batch(m, H, W, L=6):
    """Region, all-True, all-False, outpainting and region rows with per-sample cfg and temperature."""
    from paella_b200 import utils as U
    B = 5
    cond, uncond = _inputs(m, B, L, seed=30), _inputs(m, B, L, zeros=True)
    init_x = _tokens(m.num_labels, B, H, W, 31)
    region = _region(B, H, W, 32)
    region[1], region[2] = True, False
    ox, oreg = U.outpaint_canvas(_tokens(m.num_labels, 1, H // 2, W // 2, 33), (H, W), H // 4, 0)
    init_x[3], region[3] = ox[0], oreg[0]
    region[4] = _region(1, H, W, 34, p=0.2)[0]
    cfg = torch.tensor([[8.0, 8.0], [4.0, 2.0], [6.0, 6.0], [9.0, 3.0], [1.5, 5.0]], dtype=torch.float64)
    temp = torch.tensor([[0.7, 0.3], [1.0, 0.2], [0.5, 0.5], [0.9, 0.4], [1.2, 0.6]], dtype=torch.float64)
    return B, cond, uncond, init_x, region, cfg, temp


def _check_rows_equal_batch1(m, H, W, calls, steps=3):
    from paella_b200 import utils as U
    B, cond, uncond, init_x, region, cfg, temp = _mixed_batch(m, H, W)
    seeds = [60 + b for b in range(B)]
    for call in calls:
        exact = call == "distributed-exact"

        def run(sl, gens):
            kw = dict(init_x=init_x[sl], steps=steps, cfg=cfg[sl], temperature=temp[sl], generator=gens, region=region[sl])
            if call.startswith("distributed"):
                return U.sample_distributed(m, {k: v[sl] for k, v in cond.items()}, {k: v[sl] for k, v in uncond.items()},
                                            (sl.stop - sl.start, H, W), exact=exact, **kw)
            return U.sample_notebook(m, {k: v[sl] for k, v in cond.items()}, (sl.stop - sl.start, H, W),
                                     {k: v[sl] for k, v in uncond.items()}, **kw)[0]
        gens = _gens(seeds)
        got = run(slice(0, B), gens)
        for b in range(B):
            g1 = _gens([seeds[b]])
            want = run(slice(b, b + 1), g1)
            assert torch.equal(got[b:b + 1], want), (call, b)
            assert gens[b].get_offset() == g1[0].get_offset(), (call, b)
        keep = ~region.to(DEV)
        assert torch.equal(got[keep], init_x.to(DEV)[keep])


@gpu
def test_tiny_mixed_batch_rows_equal_batch1_calls(tiny):
    _check_rows_equal_batch1(tiny, 8, 8, ["distributed", "distributed-exact", "nb-multinomial"])


@pytest.mark.skipif(not os.environ.get("PB200_INPAINT_CHILD"), reason="run in a child process with PB200_FORCE_BN set")
def test_default_forced_width_child():
    m = _default_model()
    _check_rows_equal_batch1(m, 16, 16, ["distributed"], steps=2)
    _check_engine(m, 16, steps_scale=1)


def _child(test):
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PB200_FORCE_BN="128", PB200_INPAINT_CHILD="1")
    p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join(here, os.path.basename(__file__)),
                        "-k", test], env=env, capture_output=True, text=True, timeout=1200, cwd=os.path.dirname(here))
    assert p.returncode == 0 and "1 passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


@gpu
def test_default_model_with_one_tile_width_equals_batch1():
    _child("test_default_forced_width_child")


@gpu
def test_default_region_step_teacher_forced_margin_audit():
    """Default model, normal tile planner, one guided step of the mixed batch against each row's batch-1 call.  Both start from
    the same tokens (where(region, randint, init_x) on the row's own generator) and draw the same Philox values; only the
    features differ.  Outside the region the tokens are init_x's; inside, every mismatch must be a near-tie of the batch-1
    Gumbel scores, within twice the largest logit difference (over T) plus fp32 rounding."""
    from paella_b200 import utils as U
    m = _default_model()
    H = W = 32
    NL, hw = m.num_labels, H * W
    B, cond, uncond, init_x, region, cfg, temp = _mixed_batch(m, H, W, L=24)
    seeds = [80 + b for b in range(B)]
    w64 = m.out_mapper[1].weight.detach().view(NL, -1).half().double()
    got = U.sample_distributed(m, cond, uncond, (B, H, W), init_x=init_x, steps=1, cfg=cfg, temperature=temp,
                               generator=_gens(seeds), region=region)
    x = torch.stack([torch.where(region[b].to(DEV), torch.randint(0, NL, (H, W), device=DEV, generator=_gens([s])[0]),
                                 init_x[b].to(DEV)) for b, s in enumerate(seeds)])
    r = torch.ones(B, device=DEV)
    with torch.inference_mode():
        fb = m.features(x, r, m.prepare_conditioning([cond, uncond], (H, W)), cfg_pairs=True)
    total, bad, worst = 0, 0, 0.0
    for b in range(B):
        sl = slice(b, b + 1)
        want = U.sample_distributed(m, _row(cond, b), _row(uncond, b), (1, H, W), init_x=init_x[sl], steps=1, cfg=cfg[sl],
                                    temperature=temp[sl], generator=_gens([seeds[b]]), region=region[sl]).view(-1)
        g_i = got[b].view(-1)
        keep = ~region[b].view(-1).to(DEV)
        assert torch.equal(g_i[keep], init_x[b].view(-1).to(DEV)[keep]) and torch.equal(want[keep], g_i[keep]), b
        with torch.inference_mode():
            f1 = m.features(x[sl], r[sl], m.prepare_conditioning([_row(cond, b), _row(uncond, b)], (H, W)), cfg_pairs=True)
        g_q = _gens([seeds[b]])[0]
        torch.randint(0, NL, (1, H, W), device=DEV, generator=g_q)                     # the start draw
        q = torch.empty(hw, NL, device=DEV).exponential_(1, generator=g_q)             # the draws both calls consume
        c, T = float(cfg[b, 0]), float(torch.linspace(float(temp[b, 0]), float(temp[b, 1]), 1)[0])
        mix = lambda f: (f[:hw] * c + f[hw:] * (1 - c)).half().double()                # noqa: E731
        fbi = torch.cat([fb[b * hw:(b + 1) * hw], fb[(B + b) * hw:(B + b + 1) * hw]])
        l1, lb = mix(f1) @ w64.t(), mix(fbi) @ w64.t()
        mism = ((g_i != want) & ~keep).nonzero().flatten()
        total += int((~keep).sum())
        bad += int(mism.numel())
        if mism.numel():
            score = l1[mism] / T - torch.log(q[mism].double())
            gap = score.gather(1, want[mism][:, None]) - score.gather(1, g_i[mism][:, None])
            dl = (lb[mism] - l1[mism]).abs().max(1).values[:, None]
            margin = 2 * dl / T + 8 * 2.0 ** -24 * score.abs().max(1).values[:, None]
            worst = max(worst, float((gap / margin).max()))
    _log({"test": "default_region_margin_audit", "tokens_in_region": total, "mismatch": bad, "worst_gap_over_margin": worst})
    print(f"region margin audit: {bad} of {total} region tokens differ, worst gap/margin {worst:.3f}")
    assert bad <= 0.01 * max(total, 1), (bad, total)
    assert worst <= 1.0, worst


# ------------------------------------------------------------------ 5. SamplingEngine
def _engine_specs(m, H, W):
    from paella_b200 import utils as U
    NL = m.num_labels
    ox, oreg = U.outpaint_canvas(_tokens(NL, 1, H // 2, W, 40), (H, W), H // 2, 0)
    return {
        0: [dict(name="inpaint", seed=1, steps=3, init_x=_tokens(NL, 1, H, W, 41).to(DEV), region=_region(1, H, W, 42), L=5),
            dict(name="outpaint", seed=2, steps=2, cfg=(6.0, 2.0), init_x=ox, region=oreg, L=3, keep=True)],
        1: [dict(name="plain", seed=3, steps=2, cfg=None, L=4)],
        2: [dict(name="init_x_no_region", seed=4, steps=3, init_x=_tokens(NL, 1, H, W, 43).to(DEV), t_start=0.8, L=6),
            dict(name="device_region", seed=5, steps=1, init_x=_tokens(NL, 1, H, W, 44), region=_region(1, H, W, 45).to(DEV), L=2)],
    }


def _check_engine(m, H, W=None, sync_check=False, steps_scale=1):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    W = H if W is None else W
    S = _engine_specs(m, H, W)
    shared = _inputs(m, 1, 4, zeros=True)
    eng = SamplingEngine(m, latent_hw=(H, W), max_batch=2, max_cond_len=12, unconditional_inputs=shared)
    for specs in S.values():
        for sp in specs:
            sp["inputs"] = _inputs(m, 1, sp["L"], seed=100 + sp["seed"])
    torch.cuda.synchronize()
    subs, step = [], 0
    if sync_check:
        torch.cuda.set_sync_debug_mode("error")
    try:
        while step <= max(S) or eng.busy:
            for sp in S.get(step, []):
                kw = {k: sp[k] for k in ("steps", "cfg", "t_start", "init_x", "region") if k in sp}
                g = torch.Generator(device=DEV).manual_seed(sp["seed"])
                subs.append((sp, eng.submit(sp["inputs"], generator=g, keep_intermediates=sp.get("keep", False), **kw), g))
            eng.step()
            step += 1
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for sp, req, g in subs:
        assert req.done, sp["name"]
        kw = {k: sp[k] for k in ("steps", "cfg", "t_start", "init_x", "region") if k in sp}
        g1 = torch.Generator(device=DEV).manual_seed(sp["seed"])
        if sp.get("keep"):
            want, inter = U.sample_notebook(m, sp["inputs"], (1, H, W), shared, mode="multinomial", generator=[g1], **kw)
            assert len(req.intermediates) == len(inter) and all(torch.equal(a, b) for a, b in zip(req.intermediates, inter)), sp["name"]
        else:
            want = U.sample_distributed(m, sp["inputs"], shared, (1, H, W), generator=[g1], **kw)
        assert torch.equal(req.result, want), sp["name"]
        assert g.get_offset() == g1.get_offset(), sp["name"]
        if "region" in sp:
            keep = ~sp["region"].to(DEV)
            assert torch.equal(req.result[keep], sp["init_x"].to(DEV)[keep]), sp["name"]
    return subs


@gpu
def test_tiny_engine_region_requests_equal_batch1(tiny):
    subs = _check_engine(tiny, 8, 16)
    _log({"test": "tiny_engine_regions", "requests": len(subs)})


@gpu
def test_tiny_engine_region_submit_and_step_do_not_synchronise(tiny):
    _check_engine(tiny, 8, sync_check=True)


@gpu
def test_sample_loop_with_region_does_not_synchronise(tiny):
    """The loop of a region call: its tables and region arrive in one asynchronous copy.  (Building the conditioning may
    synchronise once per call, so it runs outside the check.)"""
    from paella_b200 import utils as U
    m, B, H = tiny, 3, 8
    cond, uncond = _inputs(m, B, 5, seed=7), _inputs(m, B, 5, zeros=True)
    init_x, region = _tokens(m.num_labels, B, H, H, 8).to(DEV), _region(B, H, H, 9)
    kw = dict(init_x=init_x, steps=3, cfg=torch.tensor([[8.0, 8.0], [3.0, 1.0], [5.0, 5.0]], dtype=torch.float64), region=region)
    want = U.sample_distributed(m, cond, uncond, (B, H, H), generator=_gens([1, 2, 3]), **kw)
    prep = m.prepare_conditioning

    def prep_unchecked(*a, **k):
        torch.cuda.set_sync_debug_mode(0)
        try:
            return prep(*a, **k)
        finally:
            torch.cuda.set_sync_debug_mode("error")
    m.prepare_conditioning = prep_unchecked
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = U.sample_distributed(m, cond, uncond, (B, H, H), generator=_gens([1, 2, 3]), **kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        del m.prepare_conditioning
    assert torch.equal(got, want)


# ------------------------------------------------------------------ validation
@gpu
def test_region_validation_raises_before_any_draw(tiny):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    m, B, H = tiny, 2, 8
    cond, uncond = _inputs(m, B, 4, seed=1), _inputs(m, B, 4, zeros=True)
    x, r = _tokens(m.num_labels, B, H, H, 1), _region(B, H, H, 2)
    gens = _gens([1, 2])
    g = torch.Generator(device=DEV).manual_seed(3)
    offs = [q.get_offset() for q in gens] + [g.get_offset()]
    bad = [dict(region=r),                                              # no init_x
           dict(init_x=x, region=r[:, :, :H - 1]),                      # wrong shape
           dict(init_x=x, region=r.to(torch.uint8)),                    # not bool
           dict(init_x=x, region=r.to("meta"))]                         # another device
    for kw in bad:
        for gen in (gens, g):
            with pytest.raises(ValueError):
                U.sample_distributed(m, cond, uncond, (B, H, H), steps=2, generator=gen, **kw)
            with pytest.raises(ValueError):
                U.sample_notebook(m, cond, (B, H, H), uncond, steps=2, generator=gen, **kw)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=2, max_cond_len=10)
    ok = _inputs(m, 1, 4, seed=1)
    for kw in (dict(region=r[:1]),                                      # no init_x
               dict(init_x=x[:1], region=r[0]),                         # [H, W], not [1, H, W]
               dict(init_x=x[:1], region=r),                            # [2, H, W]
               dict(init_x=x[:1], region=r[:1].to(torch.uint8))):
        with pytest.raises(ValueError):
            eng.submit(ok, _row(uncond, 0), generator=g, steps=2, **kw)
    assert [q.get_offset() for q in gens] + [g.get_offset()] == offs and not eng._active and not eng._queue
