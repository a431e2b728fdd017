"""Top-k / top-p truncated sampling on the GPU.

  * identity: k = num_labels through the C table runs the truncation kernels with their selection passes and keeps every code,
    so the tokens and generator offsets equal the call without a table, on both kernel families (the generic one in a child
    process with PB200_SAMPLER_GENERIC=1), one stream and per-sample streams
  * teacher-forced against the fp64 oracle (oracle/truncation.py) on the same fp16 operands and the same Exp(1) draws: per case
    agreement, every mismatch explained by a near-tie or a kept-set boundary within the fixed-point and fp32 bound, no token
    outside the kept set beyond that bound, k = 1 the row argmax
    (both families in child processes, one stream and per-sample streams, a mixed per-row table)
  * batch invariance (tiny model, and the default model with batch_invariant = True): row i of a batch with mixed truncation
    equals its batch-1 call
  * engine: a staggered load mixing truncated, untruncated, argmax, quant and region requests equals batch-1 sample_notebook
    calls (tiny model; the default model in batch-invariant mode)
  * validation: nothing enqueued and no generator advanced
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import load_golden, log_jsonl

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _log(payload):
    log_jsonl("truncated_sampling.jsonl", payload)


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


def _rows(d, idx):
    return {k: (v[idx] if torch.is_tensor(v) else v) for k, v in d.items()}


@pytest.fixture(scope="module")
def tiny():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m


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


def _conditioning(m, B, L, seed=7):
    from paella_b200.synth import synthetic_conditioning
    return synthetic_conditioning(B, L, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features,
                                  with_clip_image=False, seed=seed, device=DEV)


def _vq(num_labels):
    from paella_b200.vqgan import VQModel
    torch.manual_seed(0)
    return VQModel(levels=2, bottleneck_blocks=1, c_hidden=32, c_latent=4, codebook_size=num_labels).to(DEV)


def _trunc_d(k, p):
    from paella_b200 import ops
    return tuple(ops.to_device_packed([torch.tensor(k, dtype=torch.int32), torch.tensor(p, dtype=torch.float32)], DEV))


# ------------------------------------------------------------------ 1. identity: k = num_labels through the kernels
def _identity_cases(m, B, H):
    """(tokens equal, offsets equal) for one stream and per-sample streams, guided, with a k = NL table vs no table."""
    from paella_b200 import ops
    NL, c_out, hw = m.num_labels, m.out_mapper[1].weight.shape[1], H * H
    feats = torch.randn(2 * B * hw, c_out, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3)) * 4.0
    params = ops.sampling_params_table(torch.linspace(1.0, 6.0, B, dtype=torch.float64),
                                       torch.linspace(0.4, 1.3, B, dtype=torch.float64), B, DEV)
    trunc = _trunc_d([NL] * B, [1.0] * B)
    out = []
    g = torch.Generator(device=DEV)
    g.manual_seed(11)
    a = m.sample_tokens_params(feats, B, H, H, True, params, g)
    oa = g.get_offset()
    g.manual_seed(11)
    b = m.sample_tokens_params(feats, B, H, H, True, params, g, trunc)
    out.append((bool(torch.equal(a, b)), oa == g.get_offset()))
    ga, gb = _gens(range(40, 40 + B)), _gens(range(40, 40 + B))
    a = m.sample_tokens_params(feats, B, H, H, True, params, ga)
    b = m.sample_tokens_params(feats, B, H, H, True, params, gb, trunc)
    out.append((bool(torch.equal(a, b)), [x.get_offset() for x in ga] == [x.get_offset() for x in gb]))
    # a mixed table with off rows and the k = NL row: the off rows equal the untruncated launch too
    mixed = _trunc_d([0, NL] + [0] * (B - 2), [1.0] * B)
    gc = _gens(range(40, 40 + B))
    c = m.sample_tokens_params(feats, B, H, H, True, params, gc, mixed)
    out.append((bool(torch.equal(a, c)), True))
    torch.cuda.synchronize()
    return out


def _identity_main():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    tiny = Paella(**cfg).to(DEV).eval()
    tiny.load_state_dict(sd)
    res = _identity_cases(tiny, 3, 8) + _identity_cases(_big_model(), 3, 16)
    print("RESULT", all(t and o for t, o in res), res)


def _child(family, call):
    """Run ``call`` of this module in a child process on the given fused-sampler family; returns its RESULT line."""
    env = dict(os.environ)
    if family == "generic":
        env["PB200_SAMPLER_GENERIC"] = "1"
    else:
        env.pop("PB200_SAMPLER_GENERIC", None)
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_truncated_sampling as t; t.%s"
            % (ROOT, os.path.join(ROOT, "tests"), call))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    return [x for x in r.stdout.splitlines() if x.startswith("RESULT")][-1]


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["shared", "generic"])
def test_k_num_labels_through_the_table_is_the_untruncated_draw(family):
    line = _child(family, "_identity_main()")
    _log({"test": "identity", "family": family, "result": line})
    assert line.startswith("RESULT True"), line


# ------------------------------------------------------------------ 2. against the oracle, teacher-forced
ORACLE_CASES = [("k1", 1, 1.0), ("k7", 7, 1.0), ("k64", 64, 1.0), ("k1000", 1000, 1.0), ("p0.5", 0, 0.5), ("p0.9", 0, 0.9),
                ("p0.99", 0, 0.99), ("k64p0.9", 64, 0.9), ("k1000p0.5", 1000, 0.5)]
S_REL = 2.0 ** -14         # bound on |s_fp32 - s_fp64| relative to the row's max |s| (fp32 GEMM over 256 products, margin 4x)
MASS_REL = 2.0 ** -16      # bound on the mass test relative to sum w: expf 2 ulp, 2^-32 quantum per label, s error above


def _audit_row(s, q, k, p, got, want):
    """None if the kernel's token is explained, else a reason.  s fp64 [NL], q fp64 [NL]."""
    from oracle.truncation import boundary_distance, kept_set
    ds = S_REL * np.abs(s).max()
    # the kept set with every boundary label counted in (loose) or out (tight)
    loose = np.ones_like(s, bool)
    tight = np.ones_like(s, bool)
    tau_k, _ = boundary_distance(s, k, 1.0)
    if tau_k is not None:
        loose &= s >= tau_k - ds
        tight &= s >= tau_k + ds
    if 0 < p < 1:
        kl, kh = kept_set(s, k, max(p * (1 - MASS_REL), 1e-300)), kept_set(s, k, min(p * (1 + MASS_REL), 1.0))
        lo_tau, hi_tau = s[kl].min(), s[kh].min()
        loose &= s >= min(lo_tau, hi_tau) - ds
        tight &= s >= max(lo_tau, hi_tau) + ds
    if not loose[got]:
        return "outside the kept set"
    score = s - np.log(q)
    if got == want:
        return None
    best_tight = np.max(np.where(tight, score, -np.inf))
    # a near-tie of the Gumbel scores, or a boundary label that may be in or out
    if score[got] >= best_tight - (2 * ds + 8 * 2.0 ** -24 * np.abs(score).max()) or not tight[want] or not tight[got]:
        return None
    return "unexplained"


def _oracle_main(streams):
    """Teacher-forced oracle check on the 8192-label model, guided, 16x16: every case of ORACLE_CASES as a whole batch, and one
    batch mixing them all with an untruncated row; ``streams`` = 'per_sample' (one generator per sample) or 'one' (one
    generator over the batch: the rows of a Philox call belong to different samples)."""
    from oracle.truncation import truncated_winner
    from paella_b200 import ops
    m = _big_model()
    NL, c_out = m.num_labels, 256
    H, hw = 16, 256
    B = len(ORACLE_CASES) + 1
    feats = torch.randn(2 * B * hw, c_out, device=DEV, generator=torch.Generator(device=DEV).manual_seed(8))
    cfg, T = 3.0, 0.7
    params = ops.sampling_params_table(cfg, T, B, DEV)
    a16 = (feats[:B * hw] * cfg + feats[B * hw:] * (1 - cfg)).half().double()
    w64 = m.out_mapper[1].weight.detach().view(NL, c_out).half().double()
    s_all = ((a16 @ w64.t()) * float(np.float32(1.0) / np.float32(T))).cpu().numpy()
    seeds = list(range(500, 500 + B))
    report, bad = {}, []
    for name, k, p in ORACLE_CASES + [("mixed", None, None)]:
        if name == "mixed":
            ks = [c[1] for c in ORACLE_CASES] + [0]
            ps = [c[2] for c in ORACLE_CASES] + [1.0]
        else:
            ks, ps = [k] * B, [p] * B
        if streams == "per_sample":
            gens = _gens(seeds)
            got = m.sample_tokens_params(feats, B, H, H, True, params, gens, _trunc_d(ks, ps)).view(B, hw).cpu().numpy()
            qs = []
            for b in range(B):
                g = torch.Generator(device=DEV).manual_seed(seeds[b])
                qs.append(torch.empty(hw, NL, device=DEV).exponential_(1, generator=g).double().cpu().numpy())
                assert g.get_offset() == gens[b].get_offset()
        else:
            g = torch.Generator(device=DEV).manual_seed(77)
            got = m.sample_tokens_params(feats, B, H, H, True, params, g, _trunc_d(ks, ps)).view(B, hw).cpu().numpy()
            g2 = torch.Generator(device=DEV).manual_seed(77)
            q = torch.empty(B * hw, NL, device=DEV).exponential_(1, generator=g2).double().cpu().numpy()
            assert g.get_offset() == g2.get_offset()
            qs = [q[b * hw:(b + 1) * hw] for b in range(B)]
        agree, total = 0, 0
        for b in range(B):
            s = s_all[b * hw:(b + 1) * hw]
            want = truncated_winner(s, qs[b], ks[b], ps[b])
            agree += int((want == got[b]).sum())
            total += hw
            for j in range(hw):
                why = _audit_row(s[j], qs[b][j], ks[b], ps[b], got[b][j], want[j])
                if why is not None:
                    bad.append((name, b, j, why))
            if ks[b] == 1:          # the row argmax, up to ties within the fp32 bound
                mx = s.max(1)
                if not (s[np.arange(hw), got[b]] >= mx - S_REL * np.abs(s).max(1)).all():
                    bad.append((name, b, "k=1 token is not the row argmax"))
        report[name] = agree / total
    ok = not bad and min(report.values()) >= 0.99
    print("RESULT", ok, json.dumps({"agreement": report, "unexplained": [str(x) for x in bad[:5]]}))


@pytest.mark.gpu
@pytest.mark.parametrize("streams", ["per_sample", "one"])
@pytest.mark.parametrize("family", ["shared", "generic"])
def test_truncation_against_fp64_oracle_teacher_forced(family, streams):
    line = _child(family, "_oracle_main(%r)" % streams)
    _log({"test": "oracle_teacher_forced", "family": family, "streams": streams, "result": line})
    assert line.startswith("RESULT True"), line


# ------------------------------------------------------------------ 3. batch invariance (tiny model)
@pytest.mark.gpu
def test_mixed_truncation_rows_equal_batch1_calls(tiny):
    from paella_b200 import utils as U
    m = tiny
    B, H = 4, 8
    cond, uncond = _conditioning(m, B, 12)
    ks = torch.tensor([0, 5, 1, 40])
    ps = torch.tensor([0.9, 1.0, 1.0, 0.5], dtype=torch.float64)
    seeds = [3, 14, 15, 92]
    gens = _gens(seeds)
    got, inter = U.sample_notebook(m, cond, (B, H, H), uncond, steps=4, temperature=(1.2, 0.2), generator=gens, top_k=ks, top_p=ps)
    for i in range(B):
        g1 = _gens([seeds[i]])
        want, inter1 = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), steps=4,
                                         temperature=(1.2, 0.2), generator=g1, top_k=int(ks[i]), top_p=float(ps[i]))
        assert torch.equal(got[i:i + 1], want), i
        assert all(torch.equal(a[i:i + 1], b) for a, b in zip(inter, inter1)), i
        assert g1[0].get_offset() == gens[i].get_offset()
    # a shard given top_k[lo:hi] computes rows [lo, hi)
    g2 = _gens(seeds[1:3])
    shard = U.sample_distributed(m, _rows(cond, slice(1, 3)), _rows(uncond, slice(1, 3)), (2, H, H), steps=4,
                                 temperature=(1.2, 0.2), generator=g2, top_k=ks[1:3], top_p=ps[1:3])
    assert torch.equal(shard, got[1:3])
    # truncation changes the draw: k = 1 everywhere differs from the untruncated call somewhere
    a = U.sample(m, cond, (B, H, H), uncond, steps=2, generator=_gens(seeds), top_k=1)
    b = U.sample(m, cond, (B, H, H), uncond, steps=2, generator=_gens(seeds))
    assert not torch.equal(a, b)


# ------------------------------------------------------------------ 4. engine
@pytest.mark.gpu
def test_engine_mixed_truncation_equals_batch1_notebook(tiny):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    m = tiny
    H = 8
    kinds = [dict(top_k=5), dict(), dict(top_p=0.8, top_k=30), dict(mode="argmax"), dict(top_k=1, region=True),
             dict(top_p=0.5), dict(top_k=9, sampling_quant_steps=1), dict(mode="quant", top_p=0.7)]
    steps = [3, 4, 2, 3, 4, 3, 3, 2]
    N = len(kinds)
    cond, uncond = _conditioning(m, N, 12, seed=21)
    vq = _vq(m.num_labels)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=4, max_cond_len=40, vqmodel=vq)
    reqs, calls = [], []
    init = torch.randint(0, m.num_labels, (1, H, H), generator=torch.Generator().manual_seed(1))
    region = torch.zeros(1, H, H, dtype=torch.bool)
    region[:, 2:6, 1:7] = True
    for i, kw in enumerate(kinds):
        kw = dict(kw)
        extra = {}
        if kw.pop("region", False):
            extra = dict(init_x=init, region=region)
        g = torch.Generator(device=DEV).manual_seed(70 + i)
        reqs.append(eng.submit(_rows(cond, slice(i, i + 1)), _rows(uncond, slice(i, i + 1)), generator=g, steps=steps[i],
                               temperature=(1.2, 0.2), keep_intermediates=True, **kw, **extra))
        calls.append((i, kw, extra, g))
        if i % 2:
            eng.step()               # staggered arrivals
    eng.run_until_idle()
    for (i, kw, extra, g), q in zip(calls, reqs):
        g1 = torch.Generator(device=DEV).manual_seed(70 + i)
        want, inter = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), steps=steps[i],
                                        temperature=(1.2, 0.2), generator=[g1], vqmodel=vq, **kw, **extra)
        assert torch.equal(q.result, want), (i, kw)
        assert len(q.intermediates) == len(inter) and all(torch.equal(a, b) for a, b in zip(q.intermediates, inter)), i
        assert g.get_offset() == g1.get_offset(), i


# ------------------------------------------------------------------ 4b. the default model in batch-invariant mode
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


@pytest.mark.gpu
def test_default_model_batch_invariant_truncation_rows_and_engine(default_model):
    """Default 1.008 B model with batch_invariant = True: rows of a batch with mixed truncation equal their batch-1 calls, and
    engine requests (truncated, untruncated, argmax) equal batch-1 sample_notebook calls, tokens and generator offsets."""
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    m = default_model
    B, H, steps = 3, 16, 3
    cond, uncond = _conditioning(m, B, 24, seed=5)
    ks, ps = torch.tensor([64, 0, 1]), torch.tensor([1.0, 0.9, 1.0], dtype=torch.float64)
    seeds = [8, 80, 800]
    gens = _gens(seeds)
    got, _ = U.sample_notebook(m, cond, (B, H, H), uncond, steps=steps, temperature=(1.2, 0.2), generator=gens, top_k=ks, top_p=ps)
    for i in range(B):
        g1 = _gens([seeds[i]])
        want, _ = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), steps=steps,
                                    temperature=(1.2, 0.2), generator=g1, top_k=int(ks[i]), top_p=float(ps[i]))
        assert torch.equal(got[i:i + 1], want), i
        assert g1[0].get_offset() == gens[i].get_offset()
    kinds = [dict(top_k=64), dict(), dict(top_p=0.9, mode="multinomial"), dict(mode="argmax", top_k=5)]
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=2, max_cond_len=40)
    reqs = []
    for i, kw in enumerate(kinds):
        g = torch.Generator(device=DEV).manual_seed(90 + i)
        reqs.append((eng.submit(_rows(cond, slice(i % B, i % B + 1)), _rows(uncond, slice(i % B, i % B + 1)), generator=g,
                                steps=steps - (i % 2), temperature=(1.2, 0.2), **kw), g, kw))
        eng.step()                   # staggered arrivals
    eng.run_until_idle()
    for i, (q, g, kw) in enumerate(reqs):
        g1 = torch.Generator(device=DEV).manual_seed(90 + i)
        want, _ = U.sample_notebook(m, _rows(cond, slice(i % B, i % B + 1)), (1, H, H), _rows(uncond, slice(i % B, i % B + 1)),
                                    steps=steps - (i % 2), temperature=(1.2, 0.2), generator=[g1], **kw)
        assert torch.equal(q.result, want), (i, kw)
        assert g.get_offset() == g1.get_offset(), i


# ------------------------------------------------------------------ 5. validation
@pytest.mark.gpu
def test_validation_enqueues_nothing_and_advances_no_generator(tiny):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    m = tiny
    B, H = 2, 8
    cond, uncond = _conditioning(m, B, 12)
    bad = [dict(top_k=-1), dict(top_k=2.5), dict(top_p=0.0), dict(top_p=1.5), dict(top_p=float("nan")),
           dict(top_k=torch.tensor([1, 2], device=DEV)), dict(top_k=torch.tensor([1, 2, 3])), dict(top_k=3, exact=True)]
    for kw in bad:
        gens = _gens([1, 2])
        before = [g.get_offset() for g in gens]
        for fn in (lambda: U.sample(m, cond, (B, H, H), uncond, steps=2, generator=gens, **kw),
                   lambda: U.sample_notebook(m, cond, (B, H, H), uncond, steps=2, generator=gens, **kw)):
            with pytest.raises(ValueError):
                fn()
            assert [g.get_offset() for g in gens] == before, kw
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=2, max_cond_len=40)
    for kw in (dict(top_k=-3), dict(top_p=2.0), dict(top_k=torch.tensor([4]))):
        g = torch.Generator(device=DEV).manual_seed(5)
        with pytest.raises(ValueError):
            eng.submit(_rows(cond, slice(0, 1)), _rows(uncond, slice(0, 1)), generator=g, steps=2, **kw)
        assert g.get_offset() == 0 and not eng.busy
