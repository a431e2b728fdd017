"""SamplingEngine: requests admitted and retired at every step, checked against their own batch-1 sample_distributed runs.

  * tiny model, bit for bit (tokens and generator offsets): staggered admission, mixed step counts, guided / unguided /
    ramped cfg, guidance that ends early, per-request t_start / t_end / temperature, init_x, conditioning of different lengths
    with and without clip / clip_image, the shared unconditional slot and per-request negative prompts, a queue longer than
    max_batch, and freed slots reused by shorter sequences (stale K/V rows past kv_len)
  * default model with one forced GEMM tile width (child process), bit for bit
  * op level: features with partial CFG pairs, the partial-pair sampler, one-launch per-sample randint / add_noise
  * retirement decode, no host synchronisation, validation
"""
import os

import pytest
import torch

from helpers import load_golden, log_jsonl

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _log(payload):
    log_jsonl("engine.jsonl", payload)


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


@pytest.fixture(scope="module")
def tiny():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m


def _inputs(m, L, clip=True, clip_image=False, seed=0, zeros=False):
    g = torch.Generator().manual_seed(seed)
    E, C = m.byt5_mapper.in_features, m.clip_mapper.in_features
    d = {"byt5": torch.randn(1, L, E, generator=g)}
    if clip:
        d["clip"] = torch.randn(1, C, generator=g)
    if clip_image:
        d["clip_image"] = torch.randn(1, C, generator=g)
    if zeros:
        d = {k: torch.zeros_like(v) for k, v in d.items()}
    return {k: v.to(DEV) for k, v in d.items()}


def _reference(m, spec, H, W):
    """The request's own batch-1 sample_distributed run: tokens and its generator's final offset."""
    from paella_b200 import utils as U
    g = torch.Generator(device=DEV).manual_seed(spec["seed"])
    kw = {k: spec[k] for k in ("steps", "renoise_steps", "temperature", "cfg", "t_start", "t_end", "sampling_conditional_steps")
          if k in spec}
    out = U.sample_distributed(m, spec["inputs"], spec.get("uncond_ref"), (1, H, W), init_x=spec.get("init_x"), generator=[g], **kw)
    return out, g.get_offset()


def _run_engine(eng, schedule):
    """schedule: {step index: [spec, ...]} -> [(spec, request)], every request run to completion."""
    subs, step = [], 0
    last = max(schedule)
    while step <= last or eng.busy:
        for spec in schedule.get(step, []):
            kw = {k: spec[k] for k in ("steps", "renoise_steps", "temperature", "cfg", "t_start", "t_end",
                                       "sampling_conditional_steps", "init_x") if k in spec}
            g = torch.Generator(device=DEV).manual_seed(spec["seed"])
            subs.append((spec, eng.submit(spec["inputs"], spec.get("uncond"), generator=g, **kw), g))
        eng.step()
        step += 1
    return subs


def _check_against_batch1(m, subs, H, W):
    for spec, req, g in subs:
        assert req.done
        want, off = _reference(m, spec, H, W)
        assert torch.equal(req.result, want), f"request {spec['name']} differs from its batch-1 run"
        assert g.get_offset() == off, f"request {spec['name']}: generator offset {g.get_offset()} != {off}"


def _tiny_schedule(m, H):
    shared = _inputs(m, 6, clip=True, zeros=True)
    neg = lambda L, s: _inputs(m, L, clip=True, seed=s)                      # noqa: E731  a negative prompt
    init_x = torch.randint(0, m.num_labels, (1, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    S = {}
    # the first wave: long conditioning (clip + clip_image: 9 + 8 rows) and few steps, so its slots free early
    S[0] = [dict(name="a", seed=1, steps=3, cfg=(8.0, 8.0), inputs=_inputs(m, 9, True, True, 10), uncond_ref=shared),
            dict(name="b", seed=2, steps=5, cfg=None, inputs=_inputs(m, 12, True, True, 11)),
            dict(name="c", seed=3, steps=8, cfg=(9.0, 2.0), sampling_conditional_steps=4, temperature=(1.1, 0.4),
                 inputs=_inputs(m, 5, False, True, 12), uncond=neg(7, 13), uncond_ref=neg(7, 13)),
            dict(name="d", seed=4, steps=3, cfg=(6.0, 6.0), t_start=0.9, t_end=0.1, renoise_steps=1,
                 inputs=_inputs(m, 11, True, True, 14), uncond_ref=shared)]
    # queued behind a full engine; shorter sequences land in the freed slots
    S[1] = [dict(name="e", seed=5, steps=5, cfg=(7.0, 3.0), init_x=init_x, t_start=0.7, inputs=_inputs(m, 3, False, False, 15),
                 uncond=_inputs(m, 3, False, False, 16, zeros=True), uncond_ref=_inputs(m, 3, False, False, 16, zeros=True)),
            dict(name="f", seed=6, steps=8, cfg=None, temperature=(0.5, 0.5), inputs=_inputs(m, 2, True, False, 17))]
    S[3] = [dict(name="g", seed=7, steps=3, cfg=(5.0, 5.0), sampling_conditional_steps=1, inputs=_inputs(m, 4, True, False, 18),
                 uncond_ref=shared),
            dict(name="h", seed=8, steps=5, cfg=(8.0, 1.0), renoise_steps=6, inputs=_inputs(m, 1, False, False, 19),
                 uncond=neg(2, 20), uncond_ref=neg(2, 20))]
    S[5] = [dict(name="i", seed=9, steps=8, cfg=(4.0, 4.0), t_end=0.2, temperature=(0.9, 0.2),
                 inputs=_inputs(m, 8, True, True, 21), uncond_ref=shared),
            dict(name="j", seed=10, steps=1, cfg=None, inputs=_inputs(m, 2, False, False, 22))]
    return S, shared


def test_tiny_engine_requests_equal_batch1_runs(tiny):
    from paella_b200.engine import SamplingEngine
    m, H = tiny, 8
    S, shared = _tiny_schedule(m, H)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=4, max_cond_len=20, unconditional_inputs=shared)
    subs = _run_engine(eng, S)
    assert not eng.busy and sorted(eng._free) == list(range(4))
    _check_against_batch1(m, subs, H, H)
    _log({"test": "tiny_engine_vs_batch1", "requests": len(subs)})


def test_engine_step_and_submit_do_not_synchronise(tiny):
    from paella_b200.engine import SamplingEngine
    from paella_b200.vqgan import VQModel
    m, H = tiny, 8
    vcfg, vsd, _ = load_golden("vqgan_tiny.npz")
    vq = VQModel(**vcfg).to(DEV).eval()
    vq.load_state_dict(vsd)
    S, shared = _tiny_schedule(m, H)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=3, max_cond_len=20, unconditional_inputs=shared, vqmodel=vq)
    vq.decode_indices_u8(torch.zeros(1, H, H, dtype=torch.int64, device=DEV))      # the codec's one-time set-up
    pinned = {k: v.cpu().pin_memory() for k, v in S[0][1]["inputs"].items()}
    S[0][1] = dict(S[0][1], inputs=pinned)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        subs = []
        for step in range(40):
            for spec in S.get(step, []):
                kw = {k: spec[k] for k in ("steps", "renoise_steps", "temperature", "cfg", "t_start", "t_end",
                                           "sampling_conditional_steps", "init_x") if k in spec}
                subs.append((spec, eng.submit(spec["inputs"], spec.get("uncond"), decode=step % 2 == 0,
                                              generator=torch.Generator(device=DEV).manual_seed(spec["seed"]), **kw)))
            eng.step()
            if step > max(S) and not eng.busy:
                break
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(q.done for _, q in subs)
    # decoded at retirement (with whatever else retired in that step) == decoding the request's tokens alone
    for spec, q in subs:
        if q.decode:
            want, _ = _reference(m, dict(spec, inputs={k: v.to(DEV) for k, v in spec["inputs"].items()}), H, H)
            assert q.result.dtype == torch.uint8 and torch.equal(q.result, vq.decode_indices_u8(want)), spec["name"]


def test_engine_validation_raises_before_any_draw(tiny):
    from paella_b200.engine import SamplingEngine
    m, H = tiny, 8
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=2, max_cond_len=10)
    g = torch.Generator(device=DEV).manual_seed(5)
    off = g.get_offset()
    ok = _inputs(m, 4, True, False, 1)
    unc = _inputs(m, 4, True, False, 1, zeros=True)
    bad = [
        dict(generator=None),
        dict(generator=torch.Generator().manual_seed(1)),                     # a CPU generator
        dict(generator=g, inputs=_inputs(m, 8, True, True, 2)),               # 8 + 8 rows > max_cond_len
        dict(generator=g, uncond=_inputs(m, 9, True, False, 2)),              # 9 + 4 rows > max_cond_len
        dict(generator=g, init_x=torch.zeros(1, H, H + 1, dtype=torch.int64, device=DEV)),
        dict(generator=g, temperature=(0.5, 0.0)),
        dict(generator=g, temperature=(-1.0, 0.3)),
        dict(generator=g, steps=0),
        dict(generator=g, cfg=(8.0, 8.0), uncond=None),                        # no shared unconditional slot either
        dict(generator=g, decode=True),                                        # no vqmodel
    ]
    for case in bad:
        kw = dict(case)
        inputs, uncond = kw.pop("inputs", ok), kw.pop("uncond", unc)
        with pytest.raises(ValueError):
            eng.submit(inputs, uncond, **kw)
    eng.submit(ok, unc, generator=g, steps=2)
    with pytest.raises(ValueError):                                            # the same generator twice in flight
        eng.submit(ok, unc, generator=g, steps=2)
    assert g.get_offset() == off and not eng._active
    with pytest.raises(ValueError):                                            # a per-sample draw above 2^29 elements
        SamplingEngine(m, latent_hw=(2 ** 12, 2 ** 12), max_batch=1, max_cond_len=4)
    eng.run_until_idle()
    assert g.get_offset() != off


# ------------------------------------------------------------------ default model, one forced tile width
@pytest.mark.skipif(not os.environ.get("PB200_FORCE_BN"), reason="run in a child process with PB200_FORCE_BN set")
def test_default_engine_forced_width_child():
    from paella_b200.engine import SamplingEngine
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    m = m.to(DEV)
    H = 32
    shared = _inputs(m, 24, clip=True, zeros=True)
    S = {0: [dict(name="a", seed=1, steps=3, cfg=(8.0, 8.0), inputs=_inputs(m, 24, True, False, 1), uncond_ref=shared),
             dict(name="b", seed=2, steps=2, cfg=None, inputs=_inputs(m, 16, True, False, 2))],
         1: [dict(name="c", seed=3, steps=4, cfg=(7.0, 3.0), sampling_conditional_steps=2, inputs=_inputs(m, 20, True, True, 3),
                  uncond_ref=shared)]}
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=3, max_cond_len=32, unconditional_inputs=shared)
    _check_against_batch1(m, _run_engine(eng, S), H, H)


def test_default_engine_with_one_tile_width_equals_batch1():
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PB200_FORCE_BN="128")
    p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join(here, os.path.basename(__file__)),
                        "-k", "test_default_engine_forced_width_child"], env=env, capture_output=True, text=True, timeout=900,
                       cwd=os.path.dirname(here))
    assert p.returncode == 0 and "1 passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


def test_default_engine_step_teacher_forced_margin_audit():
    """Default model with the normal tile planner, one engine-shaped step: 3 guided and 3 unguided rows (9 forward samples,
    another GEMM tile width than batch 1 or 2), per-row r, cfg and T.  From the same token state each row and its batch-1
    call draw on the same Philox values; only the features differ.  Tokens must agree >= 99 % and every mismatch must be a
    near-tie of the batch-1 Gumbel scores, within twice the largest logit difference (over T) plus fp32 rounding."""
    from paella_b200 import ops
    from paella_b200.modules import ConditioningCache, Paella
    from paella_b200.synth import rerandomize_, synthetic_conditioning
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    m = m.to(DEV)
    Bc, npair, H, NL = 6, 3, 32, m.num_labels
    n_hw = H * H
    cond, uncond = synthetic_conditioning(Bc, 24, seed=7, device=DEV)
    sub = lambda d, s: {k: v[s] for k, v in d.items()}         # noqa: E731
    w64 = m.out_mapper[1].weight.detach().view(NL, -1).half().double()
    cfgs, temps = [8.0, 4.0, 6.5, 0.0, 0.0, 0.0], [0.6, 1.0, 0.8, 0.7, 1.2, 0.5]
    params = ops.sampling_params(cfgs, temps).to(DEV)
    seeds = [41 + 5 * i for i in range(Bc)]
    x = torch.randint(0, NL, (Bc, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(20))
    r = torch.tensor([1.0, 0.8, 0.55, 0.3, 0.9, 0.1], device=DEV)
    with torch.inference_mode():
        full = m.prepare_conditioning([cond, sub(uncond, slice(0, npair))], (H, H), share_uniform=False)
        part = ConditioningCache(full.cache, Bc + npair, full.s_max, full.slots, None)
        fb = m.features(x, r, part, n_pairs=npair)
    got = m.sample_tokens_pairs(fb, Bc, npair, H, H, params, ops.philox_table(_gens(seeds), n_hw * NL, DEV))
    total, bad, worst = 0, 0, 0.0
    for i in range(Bc):
        guided = i < npair
        groups = [sub(cond, slice(i, i + 1))] + ([sub(uncond, slice(i, i + 1))] if guided else [])
        with torch.inference_mode():
            f1 = m.features(x[i:i + 1], r[i:i + 1], m.prepare_conditioning(groups, (H, H)), cfg_pairs=guided)
        g_ref, g_q = _gens([seeds[i], seeds[i]])
        want = m.sample_tokens_params(f1, 1, H, H, guided, params[i:i + 1], [g_ref]).view(-1)
        q = torch.empty(n_hw, NL, device=DEV).exponential_(1, generator=g_q)        # the draws both calls consume
        fbi = torch.cat([fb[i * n_hw:(i + 1) * n_hw], fb[(Bc + i) * n_hw:(Bc + i + 1) * n_hw]]) if guided else fb[i * n_hw:(i + 1) * n_hw]
        c = cfgs[i]
        mix = (lambda f: (f[:n_hw] * c + f[n_hw:] * (1 - c)).half().double()) if guided else (lambda f: f.half().double())
        l1, lb = mix(f1) @ w64.t(), mix(fbi) @ w64.t()
        g_i = got[i].view(-1)
        mism = (g_i != want).nonzero().flatten()
        total += n_hw
        bad += int(mism.numel())
        if mism.numel():
            T = temps[i]
            score = l1[mism] / T - torch.log(q[mism].double())
            gap = score.gather(1, want[mism][:, None]) - score.gather(1, g_i[mism][:, None])
            dl = (lb[mism] - l1[mism]).abs().max(1).values[:, None]
            margin = 2 * dl / T + 8 * 2.0 ** -24 * score.abs().max(1).values[:, None]
            worst = max(worst, float((gap / margin).max()))
    _log({"test": "default_engine_step_margin_audit", "tokens": total, "mismatch": bad, "worst_gap_over_margin": worst})
    print(f"engine-step margin audit: {bad} of {total} tokens differ, worst gap/margin {worst:.3f}")
    assert bad <= 0.01 * total, (bad, total)
    assert worst <= 1.0, worst


# ------------------------------------------------------------------ op level
def test_features_with_partial_pairs_equal_separate_calls(tiny):
    from paella_b200._lib import check, current_stream, lib, ptr
    from paella_b200.modules import ConditioningCache
    m, H = tiny, 8
    Bc, npair = 5, 2
    g = torch.Generator().manual_seed(1)
    cond = {"byt5": torch.randn(Bc, 6, 40, generator=g).to(DEV), "clip": torch.randn(Bc, 24, generator=g).to(DEV)}
    unc = {"byt5": torch.randn(Bc, 6, 40, generator=g).to(DEV), "clip": torch.randn(Bc, 24, generator=g).to(DEV)}
    sub = lambda d, s: {k: v[s] for k, v in d.items()}         # noqa: E731
    x = torch.randint(0, m.num_labels, (Bc, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    r = torch.rand(Bc, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    hw = H * H
    with torch.inference_mode():
        full = m.prepare_conditioning([cond, unc], (H, H), share_uniform=False)          # slots: cond 0..4, uncond 5..9
        slot_map = torch.tensor(list(range(Bc)) + [Bc + i for i in range(npair)], dtype=torch.int32, device=DEV)
        part = ConditioningCache(full.cache, Bc + npair, full.s_max, full.slots, slot_map)
        got = m.features(x, r, part, n_pairs=npair)
        guided = m.features(x[:npair], r[:npair], m.prepare_conditioning([sub(cond, slice(0, npair)), sub(unc, slice(0, npair))],
                                                                        (H, H), share_uniform=False), cfg_pairs=True)
        plain = m.features(x[npair:], r[npair:], m.prepare_conditioning([sub(cond, slice(npair, Bc))], (H, H)))
        assert torch.equal(got[:npair * hw], guided[:npair * hw])
        assert torch.equal(got[Bc * hw:], guided[npair * hw:])
        assert torch.equal(got[npair * hw:Bc * hw], plain)
        # n_pairs in {0, Bc} through the new entry point == the existing one, bit for bit
        L = lib()
        for n_p, cache in ((Bc, full), (0, m.prepare_conditioning([cond], (H, H)))):
            Bt = Bc + n_p
            a = m.features(x, r, cache, n_pairs=n_p)
            ws = m._ws(L.pb200_paella_workspace_bytes(m._handle, Bt, H, H, cache.s_max))
            b = torch.empty_like(a)
            check(L.pb200_paella_features(m._handle, ptr(x), ptr(r), Bt, int(n_p > 0), H, H, ptr(cache.cache), cache.slots,
                                          ptr(cache.slot_map), cache.s_max, None, 0, 0, ptr(b), ptr(ws), ws.numel(),
                                          current_stream()), "pb200_paella_features")
            assert torch.equal(a, b), n_p


def _big_model(NL):
    from paella_b200.modules import Paella
    cfg, _, _ = load_golden("paella_tiny.npz")
    big = dict(cfg)
    big.update(c_in=256, c_out=256, num_labels=NL)
    torch.manual_seed(0)
    m = Paella(**big).to(DEV).eval()
    W = m.out_mapper[1].weight.detach().view(NL, 256) * 30.0
    with torch.no_grad():
        m.out_mapper[1].weight.copy_(W.view(NL, 256, 1, 1))
    m.pack_weights()
    return m


@pytest.mark.parametrize("which,H,Bc", [("tiny", 8, 5), ("big", 32, 4), ("big", 27, 3)])
def test_partial_pair_sampler_equals_two_launches(which, H, Bc, tiny):
    from paella_b200 import ops
    m = tiny if which == "tiny" else _big_model(8192)
    c_out, NL, hw = m.out_mapper[1].weight.shape[1], m.num_labels, H * H
    seeds = [70 + b for b in range(Bc)]
    params = ops.sampling_params([[8.0, 3.0, 1.0, 5.5, 2.0][b] for b in range(Bc)], [[0.7, 1.3, 0.4, 1.0, 0.9][b] for b in range(Bc)])
    params = params.to(DEV)
    for npair in range(Bc + 1):
        feats = torch.randn((Bc + npair) * hw, c_out, device=DEV, generator=torch.Generator(device=DEV).manual_seed(npair)) * 4
        gens, refs = _gens(seeds), _gens(seeds)
        got = m.sample_tokens_pairs(feats, Bc, npair, H, H, params, ops.philox_table(gens, hw * NL, DEV))
        parts = []
        if npair:
            fg = torch.cat([feats[:npair * hw], feats[Bc * hw:]])
            parts.append(m.sample_tokens_params(fg, npair, H, H, True, params[:npair], refs[:npair]))
        if npair < Bc:
            parts.append(m.sample_tokens_params(feats[npair * hw:Bc * hw], Bc - npair, H, H, False, params[npair:], refs[npair:]))
        assert torch.equal(got, torch.cat(parts)), npair
        assert [g.get_offset() for g in gens] == [g.get_offset() for g in refs]


@pytest.mark.parametrize("B,H,W", [(128, 27, 27), (3, 7, 9), (5, 6, 7), (1, 1, 1)])
def test_one_launch_randint_and_add_noise_equal_torch_per_sample(B, H, W):
    from paella_b200 import ops
    K = 8192
    seeds = [1000 + 3 * b for b in range(B)]
    x = torch.randint(0, K, (B, H, W), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    rx = torch.randint(0, K, (B, H, W), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    tt = torch.rand(B, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
    gens, refs = _gens(seeds), _gens(seeds)
    got = ops.randint(K, (B, H, W), DEV, gens)
    for b in range(B):
        assert torch.equal(got[b:b + 1], torch.randint(0, K, (1, H, W), device=DEV, generator=refs[b]))
    for random_x in (rx, None):
        out, mask = ops.add_noise(x, tt, random_x, K, gens)
        for b in range(B):
            u = torch.rand(1, H, W, device=DEV, generator=refs[b])
            m_ref = u <= tt[b]
            r_ref = rx[b:b + 1] if random_x is not None else torch.randint(0, K, (1, H, W), device=DEV, generator=refs[b])
            assert torch.equal(mask[b:b + 1].bool(), m_ref)
            assert torch.equal(out[b:b + 1], torch.where(m_ref, r_ref, x[b:b + 1]))
    assert [g.get_offset() for g in gens] == [g.get_offset() for g in refs]
    # the engine's form: rows placed by a slot map, random_x read by slot, t < 0 keeps the row
    slot = torch.randperm(B, generator=torch.Generator().manual_seed(4)).to(torch.int32).to(DEV)
    t2 = tt.clone()
    t2[::2] = -1.0
    table = ops.philox_table(_gens(seeds), H * W, DEV)
    pool = torch.full_like(x, -7)
    ops.add_noise_per_sample(x, t2, rx, K, table, pool, slot=slot)
    refs = _gens(seeds)
    for b in range(B):
        s = int(slot[b])
        u = torch.rand(1, H, W, device=DEV, generator=refs[b])
        want = torch.where(u <= t2[b], rx[s:s + 1], x[b:b + 1])
        assert torch.equal(pool[s:s + 1], want)
    assert torch.equal(ops.gather_rows(pool, slot, torch.empty_like(x)), pool[slot.long()])
