"""Per-sample generators: ``generator=[g_0, ..., g_{B-1}]`` gives every sample its own random stream, so row i of a batched
call equals the same call with batch 1 on sample i's inputs after ``torch.manual_seed(seed_i)``.

  * forward batch invariance, measured: features of a sample alone vs inside batches of 2, 5 and 64 at other positions,
    with and without CFG pairs, mixed conditioning lengths.  The tiny model is bit-exact, so its end-to-end checks assert
    ``torch.equal``.  The default model is not: the GEMM tile-width planner picks other widths for larger batches, and the
    features then differ in the last bits (bit-exact again with one forced width, checked below).  Its token rows are
    checked by a teacher-forced Gumbel-margin audit instead
  * op level: per-sample randint / add_noise / exact resample_logits against the torch ops per sample; the fused per-sample
    sampler against one batch-1 launch per sample slice (full-grid, small-grid and generic kernel families, CFG on and
    off, odd B, H*W not a multiple of 4 rs) and against torch.multinomial
  * end to end: sample / sample_distributed / sample_notebook rows vs batch-1 runs, batch reversal, two half-batch calls
  * reference semantics: the CPU oracle fed with per-sample torch draws
  * two GPUs: each rank samples its shard with its slice of the generators
  * validation errors
"""
import os
import socket

import pytest
import torch

from helpers import load_golden, log_jsonl, oracle_cfg, t

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _log(payload):
    log_jsonl("per_sample_generators.jsonl", payload)


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
    return m, cfg, sd, g


@pytest.fixture(scope="module")
def default_model():
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    return m.to(DEV)


def _model(which, tiny, default_model):
    return tiny[0] if which == "tiny" else default_model


def _conditioning(m, B, L, seed=7, clip_image=True):
    """cond with clip_image (longer sequence) and uncond without: mixed conditioning lengths in one CFG batch."""
    from paella_b200.synth import synthetic_conditioning
    cond, uncond = synthetic_conditioning(B, L, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features,
                                          with_clip_image=clip_image, seed=seed, device=DEV)
    return cond, uncond


# ------------------------------------------------------------------ 1. forward batch invariance (measured)
@pytest.mark.parametrize("cfg_pairs", [True, False], ids=["cfg", "nocfg"])
@pytest.mark.parametrize("hw", [32, 64])
@pytest.mark.parametrize("which", ["tiny", "default"])
def test_forward_features_are_batch_invariant(which, hw, cfg_pairs, tiny, default_model):
    """Features of sample i alone == the same sample inside batches of 2, 5 and 64 at other positions, bit for bit."""
    m = _model(which, tiny, default_model)
    N = 64
    cond, uncond = _conditioning(m, N, 16)
    x = torch.randint(0, m.num_labels, (N, hw, hw), device=DEV, generator=torch.Generator(device=DEV).manual_seed(11))
    r = torch.rand(N, device=DEV, generator=torch.Generator(device=DEV).manual_seed(12))
    n_hw = hw * hw

    def run(sel):
        idx = torch.tensor(sel, device=DEV)
        groups = [_rows(cond, idx), _rows(uncond, idx)] if cfg_pairs else [_rows(cond, idx)]
        with torch.inference_mode():
            cache = m.prepare_conditioning(groups, (hw, hw))
            f = m.features(x[idx], r[idx], cache, cfg_pairs=cfg_pairs)
        B = len(sel)
        # per position p: (conditional rows, unconditional rows)
        return [(f[p * n_hw:(p + 1) * n_hw], f[(B + p) * n_hw:(B + p + 1) * n_hw] if cfg_pairs else None) for p in range(B)]

    alone = {}
    worst, n_cmp = 0.0, 0
    for sel in ([1, 0], [3, 0, 4, 1, 2], list(range(N - 1, -1, -1))):
        got = run(sel)
        check = range(len(sel)) if len(sel) <= 5 else [0, 1, 30, 62, 63]
        for p in check:
            s = sel[p]
            if s not in alone:
                alone[s] = run([s])[0]
            for a, b in zip(got[p], alone[s]):
                if a is None:
                    continue
                worst = max(worst, float((a - b).abs().max()))
                n_cmp += 1
    _log({"test": "forward_batch_invariance", "which": which, "hw": hw, "cfg_pairs": cfg_pairs, "compared": n_cmp,
          "max_abs_diff": worst, "force_bn": os.environ.get("PB200_FORCE_BN")})
    if which == "tiny" or os.environ.get("PB200_FORCE_BN"):
        assert worst == 0.0, f"sample features depend on the batch: max |diff| {worst}"
    else:
        assert worst < 1e-2, worst          # measured 2.4e-3: tile-width dependent rounding, not a wrong result


def test_default_forward_is_batch_invariant_with_one_tile_width():
    """The default model's batch dependence comes from the GEMM tile-width choice alone: with one forced width
    (PB200_FORCE_BN, read once per process) the features of every sample are bit-identical in and out of a batch of 64."""
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PB200_FORCE_BN="128")
    sel = "test_forward_features_are_batch_invariant and default and 32"
    p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.join(here, os.path.basename(__file__)),
                        "-k", sel], env=env, capture_output=True, text=True, timeout=900, cwd=os.path.dirname(here))
    assert p.returncode == 0 and "2 passed" in p.stdout, p.stdout[-3000:] + p.stderr[-2000:]


# ------------------------------------------------------------------ 2. op level
def test_per_sample_randint_and_add_noise_match_torch_per_sample():
    from paella_b200 import ops
    B, H, K = 5, 27, 8192
    seeds = [101, 7, 55, 3, 900]
    x = torch.randint(0, K, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    rx = torch.randint(0, K, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(2))
    tt = torch.tensor([0.9, 0.1, 0.5, 0.0, 1.0], device=DEV)
    gens, refs = _gens(seeds), _gens(seeds)
    got = ops.randint(K, (B, H, H), DEV, gens)
    for b in range(B):
        assert torch.equal(got[b:b + 1], torch.randint(0, K, (1, H, H), device=DEV, generator=refs[b]))
    for random_x in (rx, None):
        out, mask = ops.add_noise(x, tt, random_x, K, gens)
        for b in range(B):
            u = torch.rand(1, H, H, device=DEV, generator=refs[b])
            m_ref = u <= tt[b]
            r_ref = rx[b:b + 1] if random_x is not None else torch.randint(0, K, (1, H, H), device=DEV, generator=refs[b])
            assert torch.equal(mask[b:b + 1].bool(), m_ref)
            assert torch.equal(out[b:b + 1], torch.where(m_ref, r_ref, x[b:b + 1]))
    assert [g.get_offset() for g in gens] == [g.get_offset() for g in refs]


@pytest.mark.parametrize("K,H", [(8192, 9), (64, 8)])
def test_per_sample_exact_resample_logits_matches_batch1_and_torch(K, H):
    from paella_b200 import ops
    B, cfg, T = 5, 4.0, 0.7
    seeds = [5, 6, 7, 8, 9]
    g = torch.Generator(device=DEV).manual_seed(3)
    lc = torch.randn(B, K, H, H, device=DEV, generator=g) * 3
    lu = torch.randn(B, K, H, H, device=DEV, generator=g) * 3
    for guided in (True, False):
        gens = _gens(seeds)
        got = ops.resample_logits(lc, lu if guided else None, cfg if guided else 0.0, T, "multinomial", gens)
        agree = 0
        for b in range(B):
            torch.manual_seed(seeds[b])
            want = ops.resample_logits(lc[b:b + 1], lu[b:b + 1] if guided else None, cfg if guided else 0.0, T, "multinomial")
            assert torch.equal(got[b:b + 1], want)
            assert gens[b].get_offset() == _default_gen().get_offset()
            lg = lc[b] * cfg + lu[b] * (1 - cfg) if guided else lc[b]
            p = torch.softmax(lg.div(T).reshape(K, -1).t(), dim=-1)
            torch.manual_seed(seeds[b])
            agree += int((torch.multinomial(p, 1)[:, 0] == got[b].reshape(-1)).sum())
        rate = agree / got.numel()
        _log({"test": "resample_logits_per_sample", "K": K, "H": H, "guided": guided, "agree": rate})
        assert rate >= 0.999


# (labels, batch, grid, model): full-grid shared-Philox (rs = 33 on 132 SMs; 32x32 and 27x27 are not multiples of 4 rs), the
# tiny golden model on a small-grid policy (4 rs > H*W), and the generic kernel (stride % 8200 != 0)
FUSED_CASES = [(8192, 5, 32, "big"), (8192, 3, 27, "big"), (64, 5, 8, "tiny"), (8200, 3, 16, "big")]


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


@pytest.mark.parametrize("NL,B,H,which", FUSED_CASES, ids=["NL%d-B%d-H%d-%s" % c for c in FUSED_CASES])
def test_fused_per_sample_sampler_equals_batch1_launches(NL, B, H, which, tiny):
    m = tiny[0] if which == "tiny" else _big_model(NL)
    c_out = m.out_mapper[1].weight.shape[1]
    n, hw = B * H * H, H * H
    feats = torch.randn(2 * n, c_out, device=DEV, generator=torch.Generator(device=DEV).manual_seed(4))
    if which == "tiny":
        feats *= 4.0
    w16 = m.out_mapper[1].weight.detach().view(NL, c_out).half().float()
    seeds = [1000 + 17 * b for b in range(B)]
    for cfg, T in ((8.0, 0.7), (None, 0.9)):
        f = feats if cfg is not None else feats[:n].contiguous()
        gens = _gens(seeds)
        got = m.sample_tokens(f, B, H, H, cfg, T, gens)
        agree = 0
        for b in range(B):
            fc = feats[b * hw:(b + 1) * hw]
            fb = torch.cat([fc, feats[n + b * hw:n + (b + 1) * hw]]) if cfg is not None else fc.contiguous()
            torch.manual_seed(seeds[b])
            want = m.sample_tokens(fb, 1, H, H, cfg, T)
            assert torch.equal(got[b:b + 1], want), f"sample {b}, cfg {cfg}"
            assert gens[b].get_offset() == _default_gen().get_offset()
            a16 = (fc * cfg + feats[n + b * hw:n + (b + 1) * hw] * (1 - cfg)) if cfg is not None else fc
            torch.manual_seed(seeds[b])
            ref = torch.multinomial(torch.softmax((a16.half().float() @ w16.t()) / T, dim=-1), 1)[:, 0]
            agree += int((ref == got[b].view(-1)).sum())
        rate = agree / n
        _log({"test": "fused_per_sample", "case": [NL, B, H, which], "cfg": cfg, "agree_multinomial": rate})
        assert rate >= 0.999


# ------------------------------------------------------------------ 3. end to end
def _e2e_setup(which, tiny, default_model):
    m = _model(which, tiny, default_model)
    H, L = (8, 5) if which == "tiny" else (32, 24)
    return m, H, L


@pytest.mark.parametrize("exact", [False, True], ids=["fused", "exact"])
@pytest.mark.parametrize("which", ["tiny"])
def test_sample_rows_equal_batch1_runs(which, exact, tiny, default_model):
    from paella_b200 import utils as U
    m, H, L = _e2e_setup(which, tiny, default_model)
    B = 5
    seeds = [31, 4, 159, 26, 5358]
    cond, uncond = _conditioning(m, B, L, clip_image=False)
    kw = dict(steps=4, renoise_steps=3, temperature=(1.0, 0.2), cfg=8.0, exact=exact)
    gens = _gens(seeds)
    got = U.sample(m, cond, (B, H, H), uncond, generator=gens, **kw)
    for i in range(B):
        torch.manual_seed(seeds[i])
        want = U.sample(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), **kw)
        assert torch.equal(got[i:i + 1], want), f"row {i}"
        assert gens[i].get_offset() == _default_gen().get_offset()
    # reversing the batch reverses the rows
    rev = list(range(B - 1, -1, -1))
    got_rev = U.sample(m, _rows(cond, rev), (B, H, H), _rows(uncond, rev), generator=_gens([seeds[i] for i in rev]), **kw)
    assert torch.equal(got_rev, got.flip(0))
    # two half-batch calls with the sliced generator lists (a two-shard run on one GPU)
    gens = _gens(seeds)
    a = U.sample(m, _rows(cond, slice(0, 2)), (2, H, H), _rows(uncond, slice(0, 2)), generator=gens[:2], **kw)
    b = U.sample(m, _rows(cond, slice(2, B)), (B - 2, H, H), _rows(uncond, slice(2, B)), generator=gens[2:], **kw)
    assert torch.equal(torch.cat([a, b]), got)
    # one generator == the default generator seeded the same
    g = torch.Generator(device=DEV).manual_seed(77)
    one = U.sample(m, cond, (B, H, H), uncond, generator=g, **kw)
    torch.manual_seed(77)
    assert torch.equal(one, U.sample(m, cond, (B, H, H), uncond, **kw))
    assert g.get_offset() == _default_gen().get_offset()
    _log({"test": "sample_rows_equal_batch1", "which": which, "exact": exact, "B": B, "H": H})


def test_default_model_rows_vs_batch1_teacher_forced_margin_audit(default_model):
    """Default model, CFG batch of 5 (10 forward samples: another GEMM tile width than batch 1).  From the same token state,
    the batched per-sample call and each batch-1 call draw on the same Philox values; the only difference is the features.
    Tokens must agree >= 99 % and every mismatch must be a near-tie of the batch-1 Gumbel scores, within twice the largest
    logit difference between the two feature sets (over T), plus fp32 rounding of the scores."""
    m = default_model
    B, H, NL = 5, 32, m.num_labels
    n_hw = H * H
    seeds = [31, 4, 159, 26, 5358]
    cond, uncond = _conditioning(m, B, 24, clip_image=False)
    w64 = m.out_mapper[1].weight.detach().view(NL, -1).half().double()
    cfg, T = 8.0, 0.6
    total, bad, worst = 0, 0, 0.0
    for step, t_r in enumerate((1.0, 0.6, 0.2)):
        x = torch.randint(0, NL, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(20 + step))
        r = torch.full((B,), t_r, device=DEV)
        with torch.inference_mode():
            fb = m.features(x, r, m.prepare_conditioning([cond, uncond], (H, H)), cfg_pairs=True)
        gens = _gens([s + step for s in seeds])
        got = m.sample_tokens(fb, B, H, H, cfg, T, gens)
        for i in range(B):
            ci, ui = _rows(cond, slice(i, i + 1)), _rows(uncond, slice(i, i + 1))
            with torch.inference_mode():
                f1 = m.features(x[i:i + 1], r[i:i + 1], m.prepare_conditioning([ci, ui], (H, H)), cfg_pairs=True)
            torch.manual_seed(seeds[i] + step)
            q = torch.empty(n_hw, NL, device=DEV).exponential_(1)        # the draws both calls consume
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
    _log({"test": "default_teacher_forced_margin_audit", "tokens": total, "mismatch": bad, "worst_gap_over_margin": worst})
    assert bad <= 0.01 * total, (bad, total)
    assert worst <= 1.0, worst


def test_sample_distributed_rows_equal_batch1_runs(tiny):
    from paella_b200 import utils as U
    m = tiny[0]
    B, H = 3, 8
    seeds = [2, 3, 5]
    cond, uncond = _conditioning(m, B, 5)
    init_x = torch.randint(0, m.num_labels, (B, H, H), device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
    kw = dict(steps=5, renoise_steps=3, cfg=(6.0, 2.0), sampling_conditional_steps=3)
    got = U.sample_distributed(m, cond, uncond, (B, H, H), init_x=init_x, generator=_gens(seeds), **kw)
    for i in range(B):
        torch.manual_seed(seeds[i])
        want = U.sample_distributed(m, _rows(cond, slice(i, i + 1)), _rows(uncond, slice(i, i + 1)), (1, H, H),
                                    init_x=init_x[i:i + 1], **kw)
        assert torch.equal(got[i:i + 1], want)


@pytest.mark.parametrize("mode", ["multinomial", "argmax", "quant", "quant_steps", "exact"])
def test_sample_notebook_rows_and_intermediates_equal_batch1_runs(mode, tiny):
    from paella_b200 import utils as U
    from paella_b200.vqgan import VQModel
    m, cfg, _, _ = tiny
    B, H = 3, 8
    seeds = [40, 41, 42]
    cond, uncond = _conditioning(m, B, 5)
    uncond = dict(uncond, clip_image=None)
    torch.manual_seed(0)
    vq = VQModel(levels=2, bottleneck_blocks=1, c_hidden=32, c_latent=4, codebook_size=cfg["num_labels"]).to(DEV)
    aw = torch.tensor([1.2, 1.2, 0.4, 0.4, 0.4], device=DEV)
    kw = dict(steps=4, renoise_steps=2, attn_weights=aw, vqmodel=vq,
              mode="multinomial" if mode in ("quant_steps", "exact") else mode,
              sampling_quant_steps=2 if mode == "quant_steps" else None, exact=mode == "exact")
    gens = _gens(seeds)
    got, inter = U.sample_notebook(m, cond, (B, H, H), uncond, generator=gens, **kw)
    for i in range(B):
        torch.manual_seed(seeds[i])
        want, want_inter = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), **kw)
        assert torch.equal(got[i:i + 1], want)
        assert len(inter) == len(want_inter) and all(torch.equal(a[i:i + 1], w) for a, w in zip(inter, want_inter))
        assert gens[i].get_offset() == _default_gen().get_offset()


# ------------------------------------------------------------------ 4. against the reference semantics
def test_sample_tiny_vs_oracle_with_per_sample_draws(tiny):
    """The CPU oracle's sample() fed with each sample's torch draws, taken on its own generator in batch-1 order."""
    from oracle import paella_oracle as po
    from paella_b200 import utils as U
    m, cfg, sd, g = tiny
    oc = oracle_cfg(cfg)
    B, H, K = 2, 8, cfg["num_labels"]
    seeds = [123, 321]
    byt5, clip = t(g["byt5"]), t(g["clip"])
    steps, renoise = 4, 3
    draws = {"init": [], "q": [[] for _ in range(steps)], "u": [[] for _ in range(renoise)]}
    refs = _gens(seeds)
    for b in range(B):
        draws["init"].append(torch.randint(0, K, (1, H, H), device=DEV, generator=refs[b]).cpu())
        for i in range(steps):
            draws["q"][i].append(torch.empty(H * H, K, device=DEV).exponential_(1, generator=refs[b]).cpu())
            if i < renoise:
                draws["u"][i].append(torch.rand(1, H, H, device=DEV, generator=refs[b]).cpu())
    draws = {"init": torch.cat(draws["init"]), "q": [torch.cat(q) for q in draws["q"]], "u": [torch.cat(u) for u in draws["u"]]}
    want = po.sample(sd, oc, {"byt5": byt5, "clip": clip}, (B, H, H), {"byt5": torch.zeros_like(byt5), "clip": torch.zeros_like(clip)},
                     steps=steps, renoise_steps=renoise, temperature=(1.0, 0.2), cfg_scale=8.0, draws=draws)
    cond = {"byt5": byt5.to(DEV), "clip": clip.to(DEV)}
    uncond = {"byt5": torch.zeros_like(byt5).to(DEV), "clip": torch.zeros_like(clip).to(DEV)}
    for exact in (True, False):
        gens = _gens(seeds)
        got = U.sample(m, cond, (B, H, H), uncond, steps=steps, renoise_steps=renoise, temperature=(1.0, 0.2), cfg=8.0,
                       exact=exact, generator=gens)
        assert [x.get_offset() for x in gens] == [x.get_offset() for x in refs]     # consumed each stream like the reference
        agree = float((got.cpu() == want).float().mean())
        _log({"test": "sample_tiny_vs_oracle_per_sample", "exact": exact, "agree": agree})
        assert agree > 0.9          # 128 tokens; fp16-vs-fp32 logits may flip a near-tie which then propagates


# ------------------------------------------------------------------ 5. two GPUs
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


TOTAL, H2, SEEDS2 = 5, 8, [70, 71, 72, 73, 74]


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
                    {k: v[lo:hi].to(dev) for k, v in uncond.items()}, steps=3, renoise_steps=2, generator=gens)
    full = P.gather_tokens(toks, [P.shard_range(TOTAL, r, world)[1] - P.shard_range(TOTAL, r, world)[0] for r in range(world)])
    if rank == 0:
        ret["full"] = full.cpu()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_shards_with_sliced_generators_equal_single_gpu_run(tiny):
    import torch.multiprocessing as mp
    from paella_b200 import utils as U
    m, cfg, _, _ = tiny
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    cond, uncond = _two_gpu_inputs(cfg)
    want = U.sample(m, {k: v.to(DEV) for k, v in cond.items()}, (TOTAL, H2, H2), {k: v.to(DEV) for k, v in uncond.items()},
                    steps=3, renoise_steps=2, generator=_gens(SEEDS2))
    assert torch.equal(ret["full"], want.cpu())


# ------------------------------------------------------------------ 6. validation
def test_generator_list_validation_errors(tiny):
    from paella_b200 import ops
    from paella_b200 import utils as U
    m = tiny[0]
    B, H = 3, 8
    cond, uncond = _conditioning(m, B, 5, clip_image=False)
    call = lambda gens: U.sample(m, cond, (B, H, H), uncond, steps=1, renoise_steps=0, generator=gens)    # noqa: E731
    with pytest.raises(ValueError, match="list of 2 generators for a batch of 3"):
        call(_gens([1, 2]))
    with pytest.raises(ValueError, match="must be a CUDA torch.Generator"):
        call(_gens([1, 2]) + [torch.Generator().manual_seed(3)])
    with pytest.raises(ValueError, match="must be a CUDA torch.Generator"):
        call(_gens([1, 2]) + [3])
    g = torch.Generator(device=DEV).manual_seed(1)
    with pytest.raises(ValueError, match="appears more than once"):
        call([g, torch.Generator(device=DEV).manual_seed(2), g])
    if torch.cuda.device_count() >= 2:
        with pytest.raises(ValueError, match="is on cuda:1"):
            call(_gens([1, 2]) + [torch.Generator(device="cuda:1").manual_seed(3)])
    # a per-sample draw above 2^29 elements (8192 labels: 256 x 257 latents) is refused before anything runs
    with pytest.raises(ValueError, match="exceeds 2\\^29"):
        ops.check_per_sample_numel(256 * 257 * 8192)
    ops.check_per_sample_numel(256 * 256 * 8192)
    with pytest.raises(ValueError, match="exceeds 2\\^29"):
        m.sample_tokens(torch.empty(0, m.out_mapper[1].weight.shape[1], device=DEV), 1, 2 ** 16, 129, None, 1.0, _gens([1]))
    with pytest.raises(ValueError, match="list of 1 generators for a batch of 2"):
        ops.randint(64, (2, 4, 4), DEV, _gens([1]))
