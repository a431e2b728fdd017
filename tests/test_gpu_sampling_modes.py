"""Per-sample sampling modes ('multinomial', 'argmax', 'quant', and the switch to 'quant' at ``sampling_quant_steps``) in
SamplingEngine and sample_notebook.

  * kernels: the fused sampler's skip table (skipped samples' rows untouched, the others bit-identical to a launch without
    it) in both sampler families, the generic one forced in a child process; pb200_paella_resample_samples on a shuffled
    sample list, guided and unguided, over several chunk sizes, against the whole-batch logits + resample path -- tiny model,
    and the default model with one forced GEMM tile width in a child process
  * engine: a staggered mixed load; every request's tokens, intermediates and generator offset equal its batch-1
    sample_notebook call (tiny model; default model with one forced tile width in a child process)
  * default model, normal planner: a teacher-forced audit of one mixed engine step against batch 1
  * sample_notebook with a mode and quant step per sample: row i equals its batch-1 scalar call
  * validation: submit raises before anything is enqueued and before any generator advances
"""
import os
import random
import subprocess
import sys

import pytest
import torch

from helpers import load_golden, log_jsonl

DEV = "cuda"
gpu = pytest.mark.gpu
CHILD = os.environ.get("PB200_MODES_CHILD")


def _log(payload):
    log_jsonl("sampling_modes.jsonl", payload)


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


def _inputs(m, B, L, seed=0, zeros=False):
    g = torch.Generator().manual_seed(seed)
    E, C = m.byt5_mapper.in_features, m.clip_mapper.in_features
    d = {"byt5": torch.randn(B, L, E, generator=g), "clip": torch.randn(B, C, generator=g)}
    if zeros:
        d = {k: torch.zeros_like(v) for k, v in d.items()}
    return {k: v.to(DEV) for k, v in d.items()}


def _tiny():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m


@pytest.fixture(scope="module")
def tiny():
    return _tiny()


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


def _child(test, env):
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PB200_MODES_CHILD="1", **env)
    p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join(here, os.path.basename(__file__)),
                        "-k", test], env=env, capture_output=True, text=True, timeout=1500, cwd=os.path.dirname(here))
    assert p.returncode == 0 and "1 passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


def _params(B, seed):
    from paella_b200 import ops
    g = torch.Generator().manual_seed(seed)
    cfg = (torch.rand(B, generator=g) * 8 + 1).tolist()
    temp = (torch.rand(B, generator=g) * 1.2 + 0.2).tolist()
    return ops.sampling_params(cfg, temp).to(DEV)


# ------------------------------------------------------------------ kernels
def _check_skip_table(m, H, W, Bc, npair, seed):
    from paella_b200 import ops
    from paella_b200._lib import check, current_stream, lib, ptr
    L, hw, NL = lib(), H * W, m.num_labels
    g = torch.Generator(device=DEV).manual_seed(seed)
    feats = torch.randn((Bc + npair) * hw, m._cfg["c_out"], device=DEV, generator=g)
    params = _params(Bc, seed)
    table = ops.philox_table(_gens(range(seed, seed + Bc)), hw * NL, DEV)
    want = m.sample_tokens_pairs(feats, Bc, npair, H, W, params, table)
    rng = random.Random(seed)
    for trial in range(3):
        skip = torch.tensor([rng.random() < 0.5 for _ in range(Bc)], dtype=torch.int32)
        if trial == 2:
            skip[:] = 1
        out = torch.full((Bc, H, W), -7, dtype=torch.int64, device=DEV)
        ws = m._ws(L.pb200_paella_workspace_bytes(m._handle, Bc, H, W, 1))
        check(L.pb200_paella_sample_tokens_pairs_skip(m._handle, ptr(feats), Bc, npair, hw, ptr(params), ptr(table), ptr(skip.to(DEV)),
                                                      ptr(out), ptr(ws), ws.numel(), current_stream()), "skip")
        for b in range(Bc):
            if skip[b]:
                assert bool((out[b] == -7).all()), (trial, b)
            else:
                assert torch.equal(out[b], want[b]), (trial, b)
        # a NULL table is the launch without one
        out2 = torch.full((Bc, H, W), -7, dtype=torch.int64, device=DEV)
        check(L.pb200_paella_sample_tokens_pairs_skip(m._handle, ptr(feats), Bc, npair, hw, ptr(params), ptr(table), None, ptr(out2),
                                                      ptr(ws), ws.numel(), current_stream()), "skip NULL")
        assert torch.equal(out2, want)


@pytest.mark.skipif(not CHILD, reason="run in a child process with PB200_SAMPLER_GENERIC set")
def test_skip_table_generic_child():
    assert os.environ.get("PB200_SAMPLER_GENERIC")
    _skip_table_cases()


def _skip_table_cases():
    m = _tiny()
    with torch.no_grad():
        for H, W, Bc, npair in ((8, 8, 5, 2), (4, 6, 9, 9), (16, 16, 3, 0)):
            _check_skip_table(m, H, W, Bc, npair, seed=H * 10 + Bc)
        d = _default_model()
        _check_skip_table(d, 32, 32, 6, 3, seed=5)
        _check_skip_table(d, 16, 24, 4, 1, seed=6)


@gpu
def test_skip_table_leaves_skipped_rows_and_matches_unskipped_launch():
    with torch.no_grad():
        _skip_table_cases()


@gpu
def test_skip_table_generic_sampler_family():
    _child("test_skip_table_generic_child", {"PB200_SAMPLER_GENERIC": "1"})


def _resample_samples(m, feats, B, npair, hw, samples, n_guided, params, mode, codebook, chunk, out):
    from paella_b200._lib import check, current_stream, lib, ptr
    L = lib()
    ws = m._ws(L.pb200_paella_resample_workspace_bytes(m._handle, chunk, hw))
    s = torch.tensor(samples, dtype=torch.int32, device=DEV)
    cb = codebook.contiguous().float() if codebook is not None else None
    check(L.pb200_paella_resample_samples(m._handle, ptr(feats), B, npair, hw, ptr(s), len(samples), n_guided, ptr(params), mode, ptr(cb),
                                          cb.shape[1] if cb is not None else 0, chunk, ptr(out), ptr(ws), ws.numel(), current_stream()),
          "resample_samples")


def _check_resample_samples(m, H, W, B, npair, seed, chunks=(1, 2, 3, 8)):
    from paella_b200 import ops
    hw, NL = H * W, m.num_labels
    g = torch.Generator(device=DEV).manual_seed(seed)
    feats = torch.randn((B + npair) * hw, m._cfg["c_out"], device=DEV, generator=g)
    params = _params(B, seed)
    codebook = torch.randn(NL, 4, device=DEV, generator=g)
    lc = m.logits_from_features(feats[:B * hw], B, H, W)
    lu = m.logits_from_features(feats[B * hw:], npair, H, W) if npair else None
    want = {}
    for mode, name in ((1, "argmax"), (2, "quant")):
        parts = []
        if npair:
            parts.append(ops.resample_logits_params(lc[:npair], lu, params[:npair], "argmax") if mode == 1
                         else ops.resample_quant_params(lc[:npair], lu, params[:npair], codebook))
        if npair < B:
            parts.append(ops.resample_logits_params(lc[npair:], None, params[npair:], "argmax") if mode == 1
                         else ops.resample_quant_params(lc[npair:], None, params[npair:], codebook))
        want[mode] = torch.cat(parts)
    rng = random.Random(seed)
    for chunk in chunks:
        for mode in (1, 2):
            listed = [b for b in range(B) if rng.random() < 0.7]
            guided = [b for b in listed if b < npair]
            other = [b for b in listed if b >= npair]
            rng.shuffle(guided)
            rng.shuffle(other)
            out = torch.full((B, H, W), -5, dtype=torch.int64, device=DEV)
            _resample_samples(m, feats, B, npair, hw, guided + other, len(guided), params, mode, codebook if mode == 2 else None, chunk,
                              out)
            for b in range(B):
                if b in listed:
                    assert torch.equal(out[b], want[mode][b]), (chunk, mode, b)
                else:
                    assert bool((out[b] == -5).all()), (chunk, mode, b)


@gpu
def test_resample_samples_equal_whole_batch_path_tiny(tiny):
    with torch.no_grad():
        for H, W, B, npair in ((8, 8, 7, 3), (4, 6, 5, 5), (8, 16, 6, 0)):
            _check_resample_samples(tiny, H, W, B, npair, seed=B * 7 + npair)


@pytest.mark.skipif(not CHILD, reason="run in a child process with PB200_FORCE_BN set")
def test_default_forced_width_child():
    assert os.environ.get("PB200_FORCE_BN")
    m = _default_model()
    with torch.no_grad():
        _check_resample_samples(m, 16, 16, 5, 2, seed=3, chunks=(1, 3))
    _check_engine(m, 16, 16, steps_scale=1)


@gpu
def test_default_model_with_one_tile_width():
    _child("test_default_forced_width_child", {"PB200_FORCE_BN": "128"})


# ------------------------------------------------------------------ engine
def _engine_specs(m, H, W):
    NL = m.num_labels
    g = torch.Generator().manual_seed(50)
    region = torch.rand(1, H, W, generator=g) < 0.5
    init_x = torch.randint(0, NL, (1, H, W), generator=g)
    return {
        0: [dict(name="multinomial-cfg", seed=1, steps=3, L=5),
            dict(name="argmax-cfg", seed=2, steps=2, mode="argmax", L=4),
            dict(name="quant-nocfg", seed=3, steps=3, mode="quant", cfg=None, L=3)],
        1: [dict(name="multinomial-q2", seed=4, steps=4, sampling_quant_steps=2, cfg=(6.0, 2.0), L=6),
            dict(name="argmax-q0-nocfg", seed=5, steps=2, mode="argmax", sampling_quant_steps=0, cfg=None, L=2)],
        2: [dict(name="quant-region", seed=6, steps=3, mode="quant", init_x=init_x, region=region, L=5),
            dict(name="argmax-weights-q2", seed=7, steps=4, mode="argmax", sampling_quant_steps=2, L=5,
                 attn_weights=torch.linspace(0.5, 1.5, 4)),
            dict(name="multinomial-nocfg", seed=8, steps=1, cfg=None, L=4)],
        4: [dict(name="argmax-late", seed=9, steps=2, mode="argmax", t_start=0.8, L=3)],
    }


KEYS = ("steps", "cfg", "t_start", "init_x", "region", "mode", "sampling_quant_steps", "attn_weights")


def _check_engine(m, H, W, steps_scale=1):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    S = _engine_specs(m, H, W)
    vq = _vq(m.num_labels)
    shared = _inputs(m, 1, 4, zeros=True)
    eng = SamplingEngine(m, latent_hw=(H, W), max_batch=4, max_cond_len=12, unconditional_inputs=shared, vqmodel=vq)
    for specs in S.values():
        for sp in specs:
            sp["inputs"] = _inputs(m, 1, sp["L"], seed=100 + sp["seed"])
    subs, step = [], 0
    while step <= max(S) or eng.busy:
        for sp in S.get(step, []):
            kw = {k: sp[k] for k in KEYS if k in sp}
            g = torch.Generator(device=DEV).manual_seed(sp["seed"])
            subs.append((sp, eng.submit(sp["inputs"], generator=g, keep_intermediates=True, **kw), g))
        eng.step()
        step += 1
    for sp, req, g in subs:
        assert req.done, sp["name"]
        kw = {k: sp[k] for k in KEYS if k in sp}
        g1 = torch.Generator(device=DEV).manual_seed(sp["seed"])
        want, inter = U.sample_notebook(m, sp["inputs"], (1, H, W), shared, vqmodel=vq, generator=[g1], **kw)
        assert torch.equal(req.result, want), sp["name"]
        assert len(req.intermediates) == len(inter) and all(torch.equal(a, b) for a, b in zip(req.intermediates, inter)), sp["name"]
        assert g.get_offset() == g1.get_offset(), sp["name"]
    return subs


@gpu
def test_tiny_engine_mixed_modes_equal_batch1(tiny):
    subs = _check_engine(tiny, 8, 8)
    _log({"test": "tiny_engine_mixed_modes", "requests": len(subs)})


@gpu
def test_tiny_engine_mixed_modes_do_not_synchronise(tiny):
    from paella_b200.engine import SamplingEngine
    m, H = tiny, 8
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=3, max_cond_len=8, unconditional_inputs=_inputs(m, 1, 4, zeros=True),
                         vqmodel=_vq(m.num_labels))
    reqs = [(dict(mode=md, sampling_quant_steps=qs), torch.Generator(device=DEV).manual_seed(i))
            for i, (md, qs) in enumerate([("multinomial", 1), ("argmax", None), ("quant", None), ("multinomial", None)])]
    inputs = [_inputs(m, 1, 3, seed=i) for i in range(len(reqs))]
    eng.step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for inp, (kw, g) in zip(inputs, reqs):
            eng.submit(inp, generator=g, steps=3, **kw)
        eng.run_until_idle()
    finally:
        torch.cuda.set_sync_debug_mode(0)


@gpu
def test_submit_validation_raises_before_any_draw(tiny):
    from paella_b200.engine import SamplingEngine
    m, H = tiny, 8
    shared = _inputs(m, 1, 4, zeros=True)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=2, max_cond_len=10, unconditional_inputs=shared)
    eng_vq = SamplingEngine(m, latent_hw=(H, H), max_batch=2, max_cond_len=10, unconditional_inputs=shared, vqmodel=_vq(m.num_labels))
    g = torch.Generator(device=DEV).manual_seed(3)
    off = g.get_offset()
    ok = _inputs(m, 1, 4, seed=1)
    for e, kw in ((eng_vq, dict(mode="sample")), (eng_vq, dict(mode=None)), (eng_vq, dict(sampling_quant_steps=-1)),
                  (eng_vq, dict(sampling_quant_steps=1.0)), (eng_vq, dict(sampling_quant_steps=True)),
                  (eng, dict(mode="quant")), (eng, dict(sampling_quant_steps=1)), (eng, dict(mode="argmax", sampling_quant_steps=0))):
        with pytest.raises(ValueError):
            e.submit(ok, generator=g, steps=2, **kw)
    assert g.get_offset() == off
    assert not eng._active and not eng._queue and not eng_vq._active and not eng_vq._queue
    # quant steps past the last step never use the codebook
    eng.submit(ok, generator=g, steps=2, mode="argmax", sampling_quant_steps=2)
    eng.run_until_idle()


# ------------------------------------------------------------------ default model, normal planner: teacher-forced audit
@gpu
def test_default_mixed_engine_step_teacher_forced_audit():
    """One engine step (steps=1, so no renoise) of guided argmax and quant requests next to multinomial ones, on the default
    model with the normal tile planner, against each request's batch-1 call.  Both start from the same tokens (the request's
    randint) and draw nothing for argmax / quant rows; only the features differ.  A differing argmax token must be within
    twice the largest logit difference of the batch-1 top choice; a differing quant token must be a near-tie of the
    nearest-code distance, within what the difference of the two softmax @ codebook vectors can move it."""
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    m = _default_model()
    vq = _vq(m.num_labels)
    H = W = 32
    NL, hw = m.num_labels, H * W
    shared = _inputs(m, 1, 4, zeros=True)
    specs = [("argmax", 8.0, 81), ("quant", 6.0, 82), ("multinomial", 8.0, 83), ("argmax", 3.0, 84), ("quant", 9.0, 85),
             ("multinomial", 5.0, 86)]
    eng = SamplingEngine(m, latent_hw=(H, W), max_batch=len(specs), max_cond_len=24, unconditional_inputs=shared, vqmodel=vq)
    reqs = []
    for i, (md, c, seed) in enumerate(specs):
        inp = _inputs(m, 1, 16, seed=seed)
        reqs.append((md, c, seed, inp, eng.submit(inp, generator=torch.Generator(device=DEV).manual_seed(seed), steps=1, cfg=(c, c),
                                                  mode=md)))
    eng.run_until_idle()
    w64 = m.out_mapper[1].weight.detach().view(NL, -1).half().double()
    cb = vq.vquantizer.codebook.weight.data.double()
    T = float(torch.linspace(0.7, 0.3, 1)[0])
    x = torch.stack([torch.randint(0, NL, (H, W), device=DEV, generator=_gens([s])[0]) for _, _, s, _, _ in reqs])
    r = torch.ones(len(reqs), device=DEV)
    conds = {k: torch.cat([q[3][k] for q in reqs]) for k in reqs[0][3]}
    unconds = {k: v.expand(len(reqs), *v.shape[1:]).contiguous() for k, v in shared.items()}
    with torch.no_grad():
        fb = m.features(x, r, m.prepare_conditioning([conds, unconds], (H, W)), cfg_pairs=True)
    B = len(reqs)
    stats = {"argmax": [0, 0, 0.0], "quant": [0, 0, 0.0]}
    for b, (md, c, seed, inp, req) in enumerate(reqs):
        want = U.sample_notebook(m, inp, (1, H, W), shared, steps=1, cfg=(c, c), mode=md, vqmodel=vq, generator=_gens([seed]))[0]
        if md == "multinomial":
            continue
        got, want = req.result.view(-1), want.view(-1)
        with torch.no_grad():
            f1 = m.features(x[b:b + 1], r[b:b + 1], m.prepare_conditioning([inp, shared], (H, W)), cfg_pairs=True)
        mix = lambda f: (f[:hw] * c + f[hw:] * (1 - c)).half().double()      # noqa: E731
        fbi = torch.cat([fb[b * hw:(b + 1) * hw], fb[(B + b) * hw:(B + b + 1) * hw]])
        l1, lb = mix(f1) @ w64.t() / T, mix(fbi) @ w64.t() / T
        mism = (got != want).nonzero().flatten()
        st = stats[md]
        st[0] += hw
        st[1] += int(mism.numel())
        if not mism.numel():
            continue
        dl = (lb[mism] - l1[mism]).abs().max(1).values
        if md == "argmax":
            gap = l1[mism].gather(1, want[mism][:, None])[:, 0] - l1[mism].gather(1, got[mism][:, None])[:, 0]
            margin = 2 * dl + 8 * 2.0 ** -24 * l1[mism].abs().max(1).values
        else:
            e1, eb = torch.softmax(l1[mism], 1) @ cb, torch.softmax(lb[mism], 1) @ cb
            d = lambda e, k: ((e - cb[k]) ** 2).sum(1)                       # noqa: E731
            gap = d(e1, got[mism]) - d(e1, want[mism])
            margin = 2 * ((eb - e1).norm(dim=1) * (cb[got[mism]] - cb[want[mism]]).norm(dim=1)) + 1e-5 * (1 + d(e1, want[mism]))
        st[2] = max(st[2], float((gap / margin).max()))
    _log({"test": "default_modes_margin_audit", **{k: dict(tokens=v[0], mismatch=v[1], worst_gap_over_margin=v[2]) for k, v in stats.items()}})
    print(f"modes margin audit: {stats}")
    for md, (total, bad, worst) in stats.items():
        assert bad <= 0.01 * max(total, 1), (md, bad, total)
        assert worst <= 1.0, (md, worst)


# ------------------------------------------------------------------ sample_notebook with per-sample modes
@gpu
def test_sample_notebook_per_sample_modes_rows_equal_batch1(tiny):
    from paella_b200 import utils as U
    m, B, H, W = tiny, 5, 8, 8
    vq = _vq(m.num_labels)
    cond, uncond = _inputs(m, B, 5, seed=11), _inputs(m, B, 5, zeros=True)
    modes = ["multinomial", "argmax", "quant", "argmax", "multinomial"]
    qsteps = [2, None, None, 0, None]
    cfg = torch.tensor([[8.0, 8.0], [4.0, 2.0], [6.0, 6.0], [9.0, 3.0], [1.5, 5.0]], dtype=torch.float64)
    g = torch.Generator().manual_seed(12)
    init_x = torch.randint(0, m.num_labels, (B, H, W), generator=g)
    region = torch.rand(B, H, W, generator=g) < 0.6
    seeds = [40 + b for b in range(B)]
    for kw in (dict(), dict(cfg=cfg), dict(init_x=init_x, region=region, sampling_conditional_steps=2)):
        gens = _gens(seeds)
        got, inter = U.sample_notebook(m, cond, (B, H, W), uncond, steps=4, mode=modes, sampling_quant_steps=qsteps, vqmodel=vq,
                                       generator=gens, **kw)
        for b in range(B):
            g1 = _gens([seeds[b]])
            kb = {k: (v[b:b + 1] if torch.is_tensor(v) else v) for k, v in kw.items()}
            want, inter1 = U.sample_notebook(m, {k: v[b:b + 1] for k, v in cond.items()}, (1, H, W),
                                             {k: v[b:b + 1] for k, v in uncond.items()}, steps=4, mode=modes[b],
                                             sampling_quant_steps=qsteps[b], vqmodel=vq, generator=g1, **kb)
            assert torch.equal(got[b:b + 1], want), (kw.keys(), b)
            assert len(inter) == len(inter1) and all(torch.equal(a[b:b + 1], a1) for a, a1 in zip(inter, inter1)), (kw.keys(), b)
            assert gens[b].get_offset() == g1[0].get_offset(), (kw.keys(), b)


@gpu
def test_sample_notebook_uniform_mode_list_is_the_scalar_call(tiny):
    from paella_b200 import utils as U
    m, B, H = tiny, 3, 8
    vq = _vq(m.num_labels)
    cond, uncond = _inputs(m, B, 5, seed=21), _inputs(m, B, 5, zeros=True)
    for md, qs in (("argmax", 1), ("multinomial", None), ("quant", None)):
        a = U.sample_notebook(m, cond, (B, H, H), uncond, steps=3, mode=md, sampling_quant_steps=qs, vqmodel=vq, generator=_gens([5])[0])
        b = U.sample_notebook(m, cond, (B, H, H), uncond, steps=3, mode=[md] * B, sampling_quant_steps=[qs] * B, vqmodel=vq,
                              generator=_gens([5])[0])
        assert torch.equal(a[0], b[0]) and all(torch.equal(x, y) for x, y in zip(a[1], b[1])), md


@gpu
def test_sample_notebook_mixed_modes_validation_before_any_draw(tiny):
    from paella_b200 import utils as U
    m, B, H = tiny, 2, 8
    cond, uncond = _inputs(m, B, 4, seed=1), _inputs(m, B, 4, zeros=True)
    gens, g = _gens([1, 2]), _gens([3])[0]
    offs = [q.get_offset() for q in gens] + [g.get_offset()]
    vq = _vq(m.num_labels)
    for kw in (dict(mode=["multinomial", "argmax"], generator=g, vqmodel=vq),          # one stream for mixed modes
               dict(mode=["multinomial", "quant"], generator=gens),                     # quant without vqmodel
               dict(mode=["multinomial", "argmax", "argmax"], generator=gens, vqmodel=vq),
               dict(mode=["multinomial", "Argmax"], generator=gens, vqmodel=vq),
               dict(mode="argmax", sampling_quant_steps=[1, -1], generator=gens, vqmodel=vq),
               dict(mode=["multinomial", "argmax"], generator=gens, vqmodel=vq, exact=True)):
        with pytest.raises(ValueError):
            U.sample_notebook(m, cond, (B, H, H), uncond, steps=2, **kw)
    assert [q.get_offset() for q in gens] + [g.get_offset()] == offs
