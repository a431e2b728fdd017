"""Per-sample sampling settings: ``cfg``, ``temperature``, ``t_start`` and ``t_end`` as CPU tensors with one value per sample,
so requests with different settings share one batch.  Sample i must be computed with exactly the scalars a call on its own
settings would use.

  * no change for existing callers: all-equal per-sample tensors give the scalar call's tokens and generator offsets
  * heterogeneous batch, one stream (default model): row i equals row i of a scalar call over the same batch and seed with
    sample i's settings -- the Exp(1) and mask draws depend only on the element index and no op mixes samples
  * heterogeneous batch, per-sample generators: rows equal batch-1 scalar calls (tiny model, bit-exact forward); on the default
    model a teacher-forced Gumbel-margin audit with per-row T
  * op level: the params sampler against scalar launches (per sample slice, or per distinct setting with one stream) on every
    kernel family, and against torch.multinomial; exact and quant resample against the scalar ops and torch
  * a cfg 1.0 row inside a guided batch equals the unguided call
  * validation errors, with no generator advanced; the schedule table on the CPU
  * two GPUs: shards given their slices of the settings and generators
"""
import os
import socket

import numpy as np
import pytest
import torch

from helpers import load_golden, log_jsonl

DEV = "cuda"
F64 = torch.float64


def _log(payload):
    log_jsonl("per_sample_params.jsonl", payload)


def _gens(seeds, device=DEV):
    return [torch.Generator(device=device).manual_seed(s) for s in seeds]


def _default_gen():
    return torch.cuda.default_generators[torch.cuda.current_device()]


def _rows(d, idx):
    return {k: (v[idx] if torch.is_tensor(v) else v) for k, v in d.items()}


@pytest.fixture(scope="module")
def tiny():
    from paella_b200.modules import Paella
    cfg, sd, g = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m, cfg


@pytest.fixture(scope="module")
def default_model():
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    return m.to(DEV)


def _conditioning(m, B, L, seed=7, clip_image=True):
    from paella_b200.synth import synthetic_conditioning
    return synthetic_conditioning(B, L, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features,
                                  with_clip_image=clip_image, seed=seed, device=DEV)


def _vq(num_labels):
    from paella_b200.vqgan import VQModel
    torch.manual_seed(0)
    return VQModel(levels=2, bottleneck_blocks=1, c_hidden=32, c_latent=4, codebook_size=num_labels).to(DEV)


def _run(api, m, cond, uncond, shape, vq, generator, **kw):
    """(tokens, intermediates) of one public entry point; api = 'sample[-exact]', 'distributed[-exact]' or 'nb-<mode>'."""
    from paella_b200 import utils as U
    exact = api.endswith("-exact")
    if api.startswith("sample"):
        kw.pop("init_x", None)
        return U.sample(m, cond, shape, uncond, exact=exact, generator=generator, **kw), []
    if api.startswith("distributed"):
        return U.sample_distributed(m, cond, uncond, shape, exact=exact, generator=generator, **kw), []
    mode = api[3:]
    return U.sample_notebook(m, cond, shape, uncond, vqmodel=vq, generator=generator,
                             mode="multinomial" if mode == "quant_steps" else mode,
                             sampling_quant_steps=2 if mode == "quant_steps" else None, **kw)


# ------------------------------------------------------------------ 0. the schedule table (CPU)
def test_schedule_table_equals_per_sample_linspace():
    """The host table holds, per sample, the torch.linspace values of its own settings, as the fp32 constants the scalar
    entry points derive: (float)cfg, (float)(1.0 - cfg), 1.0f / (float)T."""
    from paella_b200 import utils as U
    B, steps = 3, 5
    temp = torch.tensor([[1.0, 0.2], [0.7, 0.3], [1.3, 1.3]], dtype=F64)
    cfg = torch.tensor([[8.0, 2.0], [1.0, 1.0], [3.3, 4.1]], dtype=F64)
    ts, te = torch.tensor([1.0, 0.55, 0.8], dtype=torch.float32), 0.1
    cfgs = U._cfg_schedule(cfg, B, steps)
    params, r = U.sampling_schedule(B, steps, temp, cfgs, ts, te, per_sample_cfg=True)
    assert params.shape == (steps, B, 3) and params.dtype == torch.float32
    assert r.shape == (steps + 1, B) and r.dtype == torch.float32
    for i in range(B):
        t_i = torch.linspace(float(temp[i, 0]), float(temp[i, 1]), steps)
        c_i = torch.linspace(float(cfg[i, 0]), float(cfg[i, 1]), steps).tolist()
        assert torch.equal(r[:, i], torch.linspace(float(ts[i]), te, steps + 1))
        for s in range(steps):
            want = [np.float32(c_i[s]), np.float32(1.0 - c_i[s]), np.float32(1.0) / np.float32(float(t_i[s]))]
            assert params[s, i].numpy().tobytes() == np.array(want, dtype=np.float32).tobytes(), (i, s)
    # all scalar: no table (the per-call path runs unchanged)
    assert U.sampling_schedule(B, steps, (1.0, 0.2), [8.0] * steps, 1.0, 0.0) is None
    # validation happens on the host, before anything runs
    with pytest.raises(ValueError, match="temperature"):
        U.sampling_schedule(B, steps, torch.tensor([[1.0, 0.0]] * B), None, 1.0, 0.0)
    with pytest.raises(ValueError, match="t_end"):
        U.sampling_schedule(B, steps, (1.0, 0.2), None, 1.0, torch.tensor([0.0, float("nan"), 0.0]))
    with pytest.raises(ValueError, match="shape"):
        U.sampling_schedule(B, steps, (1.0, 0.2), None, torch.zeros(B + 1), 0.0)


# ------------------------------------------------------------------ 1. no change for existing callers
APIS = ["sample", "sample-exact", "distributed", "distributed-exact", "nb-multinomial", "nb-argmax", "nb-quant", "nb-quant_steps"]


@pytest.mark.gpu
@pytest.mark.parametrize("api", APIS)
@pytest.mark.parametrize("which", ["tiny", "default"])
def test_all_equal_per_sample_tensors_give_the_scalar_call(which, api, tiny, default_model):
    m = tiny[0] if which == "tiny" else default_model
    B, H, L = (3, 8, 5) if which == "tiny" else (2, 32, 16)
    cond, uncond = _conditioning(m, B, L, clip_image=False)
    vq = _vq(m.num_labels) if api.startswith("nb") else None
    init_x = torch.randint(0, m.num_labels, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    kw = dict(steps=4, renoise_steps=3, t_end=0.1, init_x=init_x)
    scalar = dict(kw, temperature=(0.9, 0.3), t_start=0.85, cfg=5.5 if api.startswith("sample") else (6.0, 2.5))
    per = dict(kw, temperature=torch.tensor([[0.9, 0.3]] * B, dtype=F64), t_start=torch.full((B,), 0.85, dtype=F64),
               t_end=torch.full((B,), 0.1, dtype=F64),
               cfg=torch.full((B,), 5.5, dtype=F64) if api.startswith("sample") else torch.tensor([[6.0, 2.5]] * B, dtype=F64))
    seeds = [21, 22, 23][:B]
    for per_sample_gens in (False, True):
        gw, gg = (_gens(seeds), _gens(seeds)) if per_sample_gens else (None, None)
        torch.manual_seed(5)
        want, want_i = _run(api, m, cond, uncond, (B, H, H), vq, gw, **scalar)
        off_w = _default_gen().get_offset()
        torch.manual_seed(5)
        got, got_i = _run(api, m, cond, uncond, (B, H, H), vq, gg, **per)
        assert torch.equal(got, want), (api, per_sample_gens)
        assert len(got_i) == len(want_i) and all(torch.equal(a, b) for a, b in zip(got_i, want_i))
        assert _default_gen().get_offset() == off_w
        if per_sample_gens:
            assert [g.get_offset() for g in gg] == [g.get_offset() for g in gw]


# ------------------------------------------------------------------ 2. heterogeneous batch, one stream (default model)
SETS = [((8.0, 2.0), (1.0, 0.3), 1.0), ((4.0, 4.0), (0.7, 0.2), 0.8), ((1.0, 1.0), (1.2, 0.5), 0.6), ((6.0, 3.0), (0.5, 0.5), 0.9)]


@pytest.mark.gpu
@pytest.mark.parametrize("exact", [False, True], ids=["fused", "exact"])
def test_heterogeneous_one_stream_rows_equal_scalar_calls_over_the_batch(exact, default_model):
    from paella_b200 import utils as U
    m = default_model
    B, H = 4, 32
    cond, uncond = _conditioning(m, B, 16, clip_image=False)
    init_x = torch.randint(0, m.num_labels, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(8))
    cfg = torch.tensor([s[0] for s in SETS], dtype=F64)
    temp = torch.tensor([s[1] for s in SETS], dtype=F64)
    t0 = torch.tensor([s[2] for s in SETS], dtype=F64)
    kw = dict(init_x=init_x, steps=4, renoise_steps=3, exact=exact)
    torch.manual_seed(11)
    got = U.sample_distributed(m, cond, uncond, (B, H, H), cfg=cfg, temperature=temp, t_start=t0, **kw)
    off = _default_gen().get_offset()
    for i, (c, T, ts) in enumerate(SETS):
        torch.manual_seed(11)
        want = U.sample_distributed(m, cond, uncond, (B, H, H), cfg=c, temperature=T, t_start=ts, **kw)
        assert torch.equal(got[i], want[i]), f"row {i}"
        assert _default_gen().get_offset() == off
    # sample(): per-sample cfg [B] and temperature [B, 2]
    kw = dict(steps=4, renoise_steps=3, exact=exact)
    torch.manual_seed(12)
    got = U.sample(m, cond, (B, H, H), uncond, cfg=torch.tensor([s[0][0] for s in SETS], dtype=F64), temperature=temp, **kw)
    for i, (c, T, _) in enumerate(SETS):
        torch.manual_seed(12)
        want = U.sample(m, cond, (B, H, H), uncond, cfg=c[0], temperature=T, **kw)
        assert torch.equal(got[i], want[i]), f"sample() row {i}"
    _log({"test": "heterogeneous_one_stream", "exact": exact, "B": B, "H": H})


# ------------------------------------------------------------------ 3. heterogeneous batch, per-sample generators
@pytest.mark.gpu
@pytest.mark.parametrize("api", APIS)
def test_heterogeneous_per_sample_generators_rows_equal_batch1_calls(api, tiny):
    m = tiny[0]
    B, H = 3, 8
    seeds = [40, 41, 42]
    cond, uncond = _conditioning(m, B, 5)
    vq = _vq(m.num_labels) if api.startswith("nb") else None
    init_x = torch.randint(0, m.num_labels, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
    sets = SETS[:B]
    samp = api.startswith("sample")
    per = dict(cfg=torch.tensor([s[0][0] if samp else s[0] for s in sets], dtype=F64),
               temperature=torch.tensor([s[1] for s in sets], dtype=F64), t_start=torch.tensor([s[2] for s in sets], dtype=F64),
               t_end=torch.tensor([0.0, 0.1, 0.05], dtype=F64), steps=4, renoise_steps=3, init_x=init_x)
    got, got_i = _run(api, m, cond, uncond, (B, H, H), vq, _gens(seeds), **per)
    for i, (c, T, ts) in enumerate(sets):
        torch.manual_seed(seeds[i])
        want, want_i = _run(api, m, _rows(cond, slice(i, i + 1)), _rows(uncond, slice(i, i + 1)), (1, H, H), vq, None,
                            cfg=c[0] if samp else c, temperature=T, t_start=ts, t_end=float(per["t_end"][i]), steps=4,
                            renoise_steps=3, init_x=init_x[i:i + 1])
        assert torch.equal(got[i:i + 1], want), f"row {i}"
        assert all(torch.equal(a[i:i + 1], w) for a, w in zip(got_i, want_i))
    # reversing the batch (inputs, settings and generators) reverses the rows
    rev = list(range(B - 1, -1, -1))
    per_rev = {k: (v[rev] if torch.is_tensor(v) else v) for k, v in per.items()}
    got_rev, _ = _run(api, m, _rows(cond, rev), _rows(uncond, rev), (B, H, H), vq, _gens([seeds[i] for i in rev]), **per_rev)
    assert torch.equal(got_rev, got.flip(0))


@pytest.mark.gpu
def test_default_model_per_row_settings_teacher_forced_margin_audit(default_model):
    """Default model, CFG batch of 5 with per-row (cfg, T), per-sample generators: against batch-1 scalar calls from the same
    token state.  The forward is not batch-invariant here (DESIGN.md §3), so mismatches must be near-ties of the batch-1
    Gumbel scores, within twice the largest logit difference over the row's own T, plus fp32 rounding."""
    m = default_model
    B, H, NL = 5, 32, m.num_labels
    n_hw = H * H
    seeds = [31, 4, 159, 26, 5358]
    cfgs, Ts = [8.0, 1.0, 3.0, 5.5, 2.0], [0.6, 1.1, 0.35, 0.9, 0.6]
    cond, uncond = _conditioning(m, B, 24, clip_image=False)
    w64 = m.out_mapper[1].weight.detach().view(NL, -1).half().double()
    total, bad, worst = 0, 0, 0.0
    for step, t_r in enumerate((1.0, 0.6, 0.2)):
        x = torch.randint(0, NL, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(20 + step))
        r = torch.full((B,), t_r, device=DEV)
        with torch.inference_mode():
            fb = m.features(x, r, m.prepare_conditioning([cond, uncond], (H, H)), cfg_pairs=True)
        gens = _gens([s + step for s in seeds])
        got = m.sample_tokens(fb, B, H, H, torch.tensor(cfgs, dtype=F64), torch.tensor(Ts, dtype=F64), gens)
        for i in range(B):
            cfg, T = cfgs[i], Ts[i]
            ci, ui = _rows(cond, slice(i, i + 1)), _rows(uncond, slice(i, i + 1))
            with torch.inference_mode():
                f1 = m.features(x[i:i + 1], r[i:i + 1], m.prepare_conditioning([ci, ui], (H, H)), cfg_pairs=True)
            torch.manual_seed(seeds[i] + step)
            q = torch.empty(n_hw, NL, device=DEV).exponential_(1)
            torch.manual_seed(seeds[i] + step)
            want = m.sample_tokens(f1, 1, H, H, cfg, T).view(-1)
            assert gens[i].get_offset() == _default_gen().get_offset()
            fbi = torch.cat([fb[i * n_hw:(i + 1) * n_hw], fb[(B + i) * n_hw:(B + i + 1) * n_hw]])
            mix = lambda f: (f[:n_hw] * cfg + f[n_hw:] * (1 - cfg)).half().double()      # noqa: E731
            l1, lb = mix(f1) @ w64.t(), mix(fbi) @ w64.t()
            g_i = got[i].view(-1)
            mism = (g_i != want).nonzero().flatten()
            total += n_hw
            bad += int(mism.numel())
            if mism.numel():
                score = l1[mism] / T - torch.log(q[mism].double())
                gap = score.gather(1, want[mism][:, None]) - score.gather(1, g_i[mism][:, None])
                dl = (lb[mism] - l1[mism]).abs().max(1).values[:, None]
                margin = 2 * dl / T + 8 * 2.0 ** -24 * score.abs().max(1).values[:, None]
                worst = max(worst, float((gap / margin).max()))
    _log({"test": "default_per_row_margin_audit", "tokens": total, "mismatch": bad, "worst_gap_over_margin": worst})
    assert bad <= 0.01 * total, (bad, total)
    assert worst <= 1.0, worst


# ------------------------------------------------------------------ 4. op level
# (labels, batch, grid, model): full-grid shared-Philox (rs = 33 on 132 SMs; 32x32 and 27x27 are not multiples of 4 rs), the
# tiny golden model on a small-grid policy (4 rs > H*W), and the generic kernel (stride % 8200 != 0)
FUSED_CASES = [(8192, 5, 32, "big"), (8192, 3, 27, "big"), (64, 5, 8, "tiny"), (8200, 3, 16, "big")]
OP_CFG = [8.0, 1.0, 3.0, 8.0, 5.5]
OP_T = [0.7, 1.3, 0.9, 0.7, 0.45]          # samples 0 and 3 share a setting


def _big_model(NL):
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


@pytest.mark.gpu
@pytest.mark.parametrize("NL,B,H,which", FUSED_CASES, ids=["NL%d-B%d-H%d-%s" % c for c in FUSED_CASES])
def test_fused_params_sampler_equals_scalar_launches(NL, B, H, which, tiny):
    m = tiny[0] if which == "tiny" else _big_model(NL)
    c_out = m.out_mapper[1].weight.shape[1]
    n, hw = B * H * H, H * H
    feats = torch.randn(2 * n, c_out, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    if which == "tiny":
        feats *= 4.0
    w16 = m.out_mapper[1].weight.detach().view(NL, c_out).half().float()
    seeds = [1000 + 17 * b for b in range(B)]
    cfgs, Ts = OP_CFG[:B], OP_T[:B]
    for guided in (True, False):
        f = feats if guided else feats[:n].contiguous()
        cfg_t = torch.tensor(cfgs, dtype=F64) if guided else None
        T_t = torch.tensor(Ts, dtype=F64)
        c_row = torch.tensor(cfgs, device=DEV).repeat_interleave(hw)[:, None]
        a16 = (feats[:n] * c_row + feats[n:] * (1 - c_row)) if guided else feats[:n]
        logits = a16.half().float() @ w16.t()
        t_row = torch.tensor(Ts, device=DEV).repeat_interleave(hw)[:, None]
        # per-sample streams: one scalar launch per sample slice
        gens = _gens(seeds)
        got = m.sample_tokens(f, B, H, H, cfg_t, T_t, gens)
        agree = 0
        for b in range(B):
            fc = feats[b * hw:(b + 1) * hw]
            fb = torch.cat([fc, feats[n + b * hw:n + (b + 1) * hw]]) if guided else fc.contiguous()
            torch.manual_seed(seeds[b])
            want = m.sample_tokens(fb, 1, H, H, cfgs[b] if guided else None, Ts[b])
            assert torch.equal(got[b:b + 1], want), f"per-sample streams, sample {b}, guided {guided}"
            assert gens[b].get_offset() == _default_gen().get_offset()
            torch.manual_seed(seeds[b])
            ref = torch.multinomial(torch.softmax(logits[b * hw:(b + 1) * hw] / Ts[b], dim=-1), 1)[:, 0]
            agree += int((ref == got[b].view(-1)).sum())
        rate_ps = agree / n
        # one stream: one scalar launch over the batch per distinct setting
        torch.manual_seed(99)
        got1 = m.sample_tokens(f, B, H, H, cfg_t, T_t)
        off1 = _default_gen().get_offset()
        for c, T in sorted(set(zip(cfgs, Ts))):
            torch.manual_seed(99)
            want = m.sample_tokens(f, B, H, H, c if guided else None, T)
            assert _default_gen().get_offset() == off1
            for b in range(B):
                if (cfgs[b], Ts[b]) == (c, T):
                    assert torch.equal(got1[b], want[b]), f"one stream, sample {b}, guided {guided}"
        torch.manual_seed(99)
        ref = torch.multinomial(torch.softmax(logits / t_row, dim=-1), 1)[:, 0]
        rate_one = float((ref == got1.view(-1)).float().mean())
        _log({"test": "fused_params", "case": [NL, B, H, which], "guided": guided, "agree_per_sample": rate_ps,
              "agree_one_stream": rate_one})
        assert rate_ps >= 0.999 and rate_one >= 0.999, (rate_ps, rate_one)


@pytest.mark.gpu
@pytest.mark.parametrize("K,H", [(8192, 9), (64, 8)])
def test_resample_ops_with_per_sample_values_match_torch(K, H):
    from paella_b200 import ops
    B = 5
    cfgs, Ts = OP_CFG[:B], OP_T[:B]
    g = torch.Generator(device=DEV).manual_seed(3)
    lc = torch.randn(B, K, H, H, device=DEV, generator=g) * 3
    lu = torch.randn(B, K, H, H, device=DEV, generator=g) * 3
    cb = torch.randn(K, 4, device=DEV, generator=g)
    c32 = torch.tensor(cfgs, dtype=F64)
    c_b = c32.float().to(DEV)[:, None, None, None]                 # (float)cfg
    omc_b = (1.0 - c32).float().to(DEV)[:, None, None, None]       # (float)(1.0 - cfg)
    it_b = (1.0 / torch.tensor(Ts, dtype=F64).float()).to(DEV)[:, None, None, None]
    cfg_t, T_t = torch.tensor(cfgs, dtype=F64), torch.tensor(Ts, dtype=F64)
    for guided in (True, False):
        lg = lc * c_b + lu * omc_b if guided else lc                # the torch expression, per-row cfg
        u = lu if guided else None
        # argmax: bit for bit the torch expression
        assert torch.equal(ops.resample_logits(lc, u, cfg_t, T_t, "argmax"), lg.argmax(1))
        # multinomial, one stream: the scalar op per distinct setting, and torch.multinomial
        torch.manual_seed(17)
        got = ops.resample_logits(lc, u, cfg_t, T_t, "multinomial")
        for b in range(B):
            torch.manual_seed(17)
            want = ops.resample_logits(lc, u, cfgs[b], Ts[b], "multinomial")
            assert torch.equal(got[b], want[b])
        p = torch.softmax(lg * it_b, dim=1).permute(0, 2, 3, 1).reshape(-1, K)
        torch.manual_seed(17)
        rate = float((torch.multinomial(p, 1)[:, 0] == got.view(-1)).float().mean())
        # per-sample generators
        gens = _gens([5, 6, 7, 8, 9])
        got_g = ops.resample_logits(lc, u, cfg_t, T_t, "multinomial", gens)
        for b in range(B):
            torch.manual_seed(5 + b)
            assert torch.equal(got_g[b:b + 1], ops.resample_logits(lc[b:b + 1], u[b:b + 1] if guided else None, cfgs[b], Ts[b]))
            assert gens[b].get_offset() == _default_gen().get_offset()
        # quant: the scalar op per sample, and the torch expression's nearest code
        got_q = ops.resample_quant(lc, u, cfg_t, T_t, cb)
        for b in range(B):
            assert torch.equal(got_q[b:b + 1], ops.resample_quant(lc[b:b + 1], u[b:b + 1] if guided else None, cfgs[b], Ts[b], cb))
        e = torch.softmax(lg * it_b, dim=1).permute(0, 2, 3, 1) @ cb
        d = (e[..., None, :] - cb).pow(2).sum(-1)
        rate_q = float((d.argmin(-1) == got_q).float().mean())
        _log({"test": "resample_ops_params", "K": K, "guided": guided, "agree_multinomial": rate, "agree_quant": rate_q})
        assert rate >= 0.999 and rate_q >= 0.99, (rate, rate_q)


# ------------------------------------------------------------------ 5. unguided rows
@pytest.mark.gpu
@pytest.mark.parametrize("api", ["sample", "sample-exact", "distributed"])
def test_cfg_one_row_in_guided_batch_equals_unguided_call(api, tiny):
    """f*1 + u*0 = f, and the CFG pair's conditional rows equal the unguided forward's rows (tiny model)."""
    from paella_b200 import utils as U
    m = tiny[0]
    B, H = 3, 8
    seeds = [61, 62, 63]
    cond, uncond = _conditioning(m, B, 5, clip_image=False)
    samp = api.startswith("sample")
    cfg = torch.tensor([8.0, 1.0, 3.0], dtype=F64) if samp else torch.tensor([[8.0, 2.0], [1.0, 1.0], [3.0, 3.0]], dtype=F64)
    kw = dict(steps=4, renoise_steps=3)
    got, _ = _run(api, m, cond, uncond, (B, H, H), None, _gens(seeds), cfg=cfg, **kw)
    torch.manual_seed(seeds[1])
    c1 = _rows(cond, slice(1, 2))
    if samp:
        want = U.sample(m, c1, (1, H, H), None, cfg=None, exact=api.endswith("-exact"), **kw)
    else:
        want = U.sample_distributed(m, c1, None, (1, H, H), cfg=None, **kw)
    assert torch.equal(got[1:2], want)


# ------------------------------------------------------------------ 6. validation
@pytest.mark.gpu
def test_per_sample_value_validation_errors_advance_no_generator(tiny):
    from paella_b200 import ops
    from paella_b200 import utils as U
    m = tiny[0]
    B, H = 3, 8
    cond, uncond = _conditioning(m, B, 5, clip_image=False)
    gens = _gens([1, 2, 3])
    nan, inf = float("nan"), float("inf")
    ok_T = torch.tensor([[1.0, 0.2]] * B)
    cases = [
        ("sample", dict(cfg=torch.full((B,), 4.0, device=DEV)), "CPU tensor"),
        ("sample", dict(cfg=torch.full((B + 1,), 4.0)), "shape"),
        ("sample", dict(cfg=torch.tensor([4.0, nan, 4.0])), "finite"),
        ("sample", dict(cfg=torch.tensor([4, 4, 4])), "floating-point"),
        ("sample", dict(temperature=torch.tensor([[1.0, 0.2], [1.0, 0.0], [1.0, 0.2]])), "temperature"),
        ("sample", dict(temperature=torch.tensor([[1.0, 0.2], [-1.0, 0.5], [1.0, 0.2]])), "temperature"),
        ("sample", dict(temperature=torch.tensor([[1.0, inf]] * B)), "finite"),
        ("sample", dict(temperature=torch.tensor([1.0, 0.2, 0.5])), "shape"),
        ("sample", dict(temperature=ok_T, t_start=torch.tensor([1.0, inf, 1.0])), "finite"),
        ("sample", dict(t_end=torch.zeros(2)), "shape"),
        ("sample", dict(t_start=torch.ones(B, device=DEV)), "CPU tensor"),
        ("distributed", dict(cfg=torch.full((B,), 4.0)), "shape"),
        ("distributed", dict(cfg=torch.tensor([[4.0, 2.0], [4.0, nan], [4.0, 2.0]])), "finite"),
        ("nb-multinomial", dict(temperature=torch.tensor([[0.7, 0.3]] * (B - 1))), "shape"),
    ]
    for api, kw, match in cases:
        for g in (None, gens):
            torch.manual_seed(0)
            off = _default_gen().get_offset()
            offs = [x.get_offset() for x in gens]
            with pytest.raises(ValueError, match=match):
                _run(api, m, cond, uncond, (B, H, H), None, g, steps=2, renoise_steps=1, **kw)
            assert _default_gen().get_offset() == off, (api, kw)
            assert [x.get_offset() for x in gens] == offs, (api, kw)
    feats = torch.zeros(2 * B * H * H, m.out_mapper[1].weight.shape[1], device=DEV)
    with pytest.raises(ValueError, match="shape"):
        m.sample_tokens(feats, B, H, H, torch.full((B - 1,), 2.0), 1.0)
    with pytest.raises(ValueError, match="temperature"):
        m.sample_tokens(feats, B, H, H, 2.0, torch.tensor([1.0, 0.0, 1.0]))
    lc = torch.zeros(B, m.num_labels, H, H, device=DEV)
    with pytest.raises(ValueError, match="temperature"):
        ops.resample_logits(lc, None, 0.0, torch.tensor([1.0, -0.5, 1.0]))
    with pytest.raises(ValueError, match="CPU tensor"):
        ops.resample_quant(lc, lc, torch.ones(B, device=DEV), 1.0, torch.zeros(m.num_labels, 4, device=DEV))


# ------------------------------------------------------------------ 7. two GPUs
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


TOTAL, H2, SEEDS2 = 5, 8, [70, 71, 72, 73, 74]
CFG2 = torch.tensor([8.0, 1.0, 4.0, 2.5, 6.0], dtype=F64)
TEMP2 = torch.tensor([[1.0, 0.2], [0.7, 0.7], [1.5, 0.4], [0.9, 0.3], [0.6, 0.2]], dtype=F64)


def _two_gpu_inputs(cfg):
    from paella_b200.synth import synthetic_conditioning
    return synthetic_conditioning(TOTAL, 5, seed=7, byt5_embd=cfg["byt5_embd"], clip_embd=cfg["clip_embd"])


def _worker(rank, world, port, ret):
    import sys
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from helpers import load_golden
    from paella_b200 import parallel as P
    from paella_b200 import utils as U
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).eval()
    m.load_state_dict(sd)
    m = m.to(dev)
    cond, uncond = _two_gpu_inputs(cfg)
    lo, hi = P.shard_range(TOTAL, rank, world)
    gens = [torch.Generator(device=dev).manual_seed(s) for s in SEEDS2[lo:hi]]
    toks = U.sample(m, {k: v[lo:hi].to(dev) for k, v in cond.items()}, (hi - lo, H2, H2),
                    {k: v[lo:hi].to(dev) for k, v in uncond.items()}, steps=3, renoise_steps=2, cfg=CFG2[lo:hi],
                    temperature=TEMP2[lo:hi], generator=gens)
    full = P.gather_tokens(toks, [P.shard_range(TOTAL, r, world)[1] - P.shard_range(TOTAL, r, world)[0] for r in range(world)])
    if rank == 0:
        ret["full"] = full.cpu()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_shards_with_sliced_settings_equal_single_gpu_run(tiny):
    import torch.multiprocessing as mp
    from paella_b200 import utils as U
    m, cfg = tiny
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    cond, uncond = _two_gpu_inputs(cfg)
    want = U.sample(m, {k: v.to(DEV) for k, v in cond.items()}, (TOTAL, H2, H2), {k: v.to(DEV) for k, v in uncond.items()},
                    steps=3, renoise_steps=2, cfg=CFG2, temperature=TEMP2, generator=_gens(SEEDS2))
    assert torch.equal(ret["full"], want.cpu())
