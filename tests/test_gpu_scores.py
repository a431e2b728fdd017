"""Token scoring on the GPU.

  * the kernel through the C entry against fp64 on the same fp16 operands: c_out 16 / 64 / 256, 64 / 200 / 8192 labels, ragged
    row counts; nll and smooth within 2e-4, the arg-max wherever the top-2 gap exceeds the fp32 GEMM's error (margins logged);
    adversarial rows; out-of-range targets; NaN features confined to their sample; the guided pre-mix
  * Paella.token_scores against the oracle and the reference fixture (tiny model), and against fp64 cross entropy of the default
    model's forward logits, guided and not, with tiling, attn_weights and prompt_regions rows
  * batch independence: a sample's scores alone equal its rows in larger batches, bit for bit (tiny model; default model with
    batch_invariant = True)
  * utils.score equals the hand loop of add_noise and token_scores, generators included; equal seeds and prompts give equal
    rows; an all-True region is no region; tokens outside a region are never noised
"""
import math

import pytest
import torch
import torch.nn.functional as F

from helpers import load_golden, log_jsonl, oracle_cfg, t

DEV = "cuda"
G_REL = 2.0 ** -14      # bound on |l_fp32 - l_fp64| relative to the row's max |l| (fp32 accumulation of <= 256 products, 4x margin)


def _log(payload):
    log_jsonl("scores.jsonl", payload)


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


@pytest.fixture(scope="module")
def tiny():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m


def _head_model(c_out, NL, w=None):
    """The tiny model with an out_mapper of c_out inputs and NL labels; ``w`` (fp32 [NL, c_out]) replaces its weight."""
    from paella_b200.modules import Paella
    cfg, _, _ = load_golden("paella_tiny.npz")
    torch.manual_seed(c_out * 7 + NL)
    m = Paella(**dict(cfg, c_in=c_out, c_out=c_out, num_labels=NL)).eval()
    if w is None:
        w = torch.randn(NL, c_out) * (3.0 / math.sqrt(c_out))
    with torch.no_grad():
        m.out_mapper[1].weight.copy_(w.view(NL, c_out, 1, 1))
    return m.to(DEV)


def _c_scores(m, feats, batch, hw, targets, n_pairs=0, params=None):
    """pb200_paella_token_scores on fp32 features [(batch + n_pairs) * hw, c_out] -> (nll, smooth, argmax) of batch * hw rows."""
    from paella_b200._lib import check, current_stream, lib, ptr
    m._ensure_packed()
    L = lib()
    nll = torch.empty(batch * hw, device=DEV)
    smooth = torch.empty_like(nll)
    am = torch.empty(batch * hw, dtype=torch.int64, device=DEV)
    ws = torch.empty(L.pb200_paella_token_scores_workspace_bytes(m._handle, batch, hw), dtype=torch.uint8, device=DEV)
    check(L.pb200_paella_token_scores(m._handle, ptr(feats.contiguous()), batch, n_pairs, hw, ptr(params), ptr(targets.contiguous()),
                                      ptr(nll), ptr(smooth), ptr(am), ptr(ws), ws.numel(), current_stream()), "pb200_paella_token_scores")
    torch.cuda.synchronize()
    return nll, smooth, am


def _ref64(a16, w16, targets):
    """fp64 (logits, nll, smooth) of fp16 operands a16 [R, c] and w16 [NL, c]; targets in range."""
    l = a16.double() @ w16.double().t()
    lse = torch.logsumexp(l, 1)
    return l, lse - l.gather(1, targets[:, None]).squeeze(1), lse - l.mean(1)


def _argmax_audit(l, got, case):
    """got must equal the fp64 first arg-max wherever the top-2 gap exceeds the GEMM error bound; returns the near-tie count."""
    top2 = l.topk(2, dim=1).values
    bound = G_REL * l.abs().amax(1)
    clear = (top2[:, 0] - top2[:, 1]) > 2 * bound
    want = l.argmax(1)
    bad = int((got[clear] != want[clear]).sum())
    assert bad == 0, (case, bad)
    # a near tie must still name one of the tied maxima (within the bound)
    pick = l.gather(1, got[:, None]).squeeze(1)
    assert bool((pick >= top2[:, 0] - 2 * bound).all()), case
    return int((~clear).sum())


# ------------------------------------------------------------------ 1. the kernel against fp64
@pytest.mark.gpu
@pytest.mark.parametrize("c_out", [16, 64, 256])
@pytest.mark.parametrize("NL", [64, 200, 8192])
def test_kernel_matrix_against_fp64(c_out, NL):
    m = _head_model(c_out, NL)
    w16 = m.out_mapper[1].weight.detach().view(NL, c_out).half()
    for rows in (1, 127, 128, 129, 24 * 36 * 3):
        g = torch.Generator().manual_seed(rows + c_out)
        feats = torch.randn(rows, c_out, generator=g).to(DEV)
        y = torch.randint(0, NL, (rows,), generator=g).to(DEV)
        nll, smooth, am = _c_scores(m, feats, 1, rows, y)
        l, nll64, sm64 = _ref64(feats.half(), w16, y)
        e_nll = float((nll.double() - nll64).abs().max())
        e_sm = float((smooth.double() - sm64).abs().max())
        ties = _argmax_audit(l, am, (c_out, NL, rows))
        _log({"case": "matrix", "c_out": c_out, "NL": NL, "rows": rows, "err_nll": e_nll, "err_smooth": e_sm, "near_ties": ties})
        assert e_nll < 2e-4 and e_sm < 2e-4, (rows, e_nll, e_sm)


@pytest.mark.gpu
def test_kernel_adversarial_rows():
    """W = I on 64 labels, so every logit is one exact fp16 feature: all-equal rows (arg-max 0, nll = log 64), one logit 60
    above the rest, and magnitudes around 1e3.  None gives Inf or NaN; the results match fp64 to 2e-4 plus 1e-5 of the row's
    largest |logit| (fp32 rounding of the sum of logits at 1e3)."""
    NL = c = 64
    m = _head_model(c, NL, torch.eye(NL))
    g = torch.Generator().manual_seed(5)
    feats = torch.zeros(6, c)
    feats[1, 17] = 60.0
    feats[2, 0] = -60.0
    feats[3] = 1000.0
    feats[4] = 1000.0 + torch.randn(c, generator=g) * 3
    feats[5] = -1000.0 + torch.randn(c, generator=g) * 3
    feats = feats.half().float().to(DEV)
    y = torch.tensor([5, 17, 3, 63, 9, 40], device=DEV)
    nll, smooth, am = _c_scores(m, feats, 1, 6, y)
    assert bool(torch.isfinite(nll).all() and torch.isfinite(smooth).all()), (nll, smooth)
    l, nll64, sm64 = _ref64(feats.half(), m.out_mapper[1].weight.detach().view(NL, c).half(), y)
    tol = 2e-4 + 1e-5 * l.abs().amax(1)
    assert bool(((nll.double() - nll64).abs() <= tol).all()), (nll, nll64)
    assert bool(((smooth.double() - sm64).abs() <= tol).all()), (smooth, sm64)
    assert abs(float(nll[0]) - math.log(64)) < 2e-6 and int(am[0]) == 0
    assert int(am[1]) == 17 and int(am[3]) == 0 and int(am[2]) == 1
    assert torch.equal(am[4:], l[4:].argmax(1))


@pytest.mark.gpu
def test_out_of_range_targets_and_nan_features_stay_in_their_row():
    m = _head_model(64, 200)
    B, hw = 3, 100
    g = torch.Generator().manual_seed(8)
    feats = torch.randn(B * hw, 64, generator=g).to(DEV)
    y = torch.randint(0, 200, (B * hw,), generator=g).to(DEV)
    ref = _c_scores(m, feats, B, hw, y)
    y_bad = y.clone()
    y_bad[7], y_bad[150] = -1, 200
    got = _c_scores(m, feats, B, hw, y_bad)
    keep = torch.ones(B * hw, dtype=torch.bool, device=DEV)
    keep[[7, 150]] = False
    assert bool(torch.isnan(got[0][~keep]).all())
    assert torch.equal(got[0][keep], ref[0][keep]) and torch.equal(got[1], ref[1]) and torch.equal(got[2], ref[2])
    f_nan = feats.clone()
    f_nan[hw:2 * hw, 3] = float("nan")
    got = _c_scores(m, f_nan, B, hw, y)
    other = torch.ones(B * hw, dtype=torch.bool, device=DEV)
    other[hw:2 * hw] = False
    for a, b in zip(got, ref):
        assert torch.equal(a[other], b[other])
    assert bool(torch.isnan(got[0][~other]).all())


@pytest.mark.gpu
def test_guided_premix_through_the_c_entry():
    """Sample 0 guided with its unconditional rows, sample 1 not: cfg = 1 is the conditional row bit for bit, and cfg = 2.5
    matches fp64 on the fp32 mix rounded to fp16 (to 1e-3: the mix kernel and torch may round a feature to neighbouring
    fp16 values)."""
    NL, c, hw = 8192, 256, 300
    m = _head_model(c, NL)
    w16 = m.out_mapper[1].weight.detach().view(NL, c).half()
    g = torch.Generator().manual_seed(11)
    fc = torch.randn(2 * hw, c, generator=g).to(DEV)
    fu = torch.randn(hw, c, generator=g).to(DEV)
    y = torch.randint(0, NL, (2 * hw,), generator=g).to(DEV)
    plain = _c_scores(m, fc, 2, hw, y)
    for cfg in (1.0, 2.5):
        params = torch.tensor([[cfg, 1.0 - cfg, 1.0], [0.0, 1.0, 1.0]], device=DEV)
        got = _c_scores(m, torch.cat([fc, fu]), 2, hw, y, n_pairs=1, params=params)
        for a, b in zip(got, plain):
            assert torch.equal(a[hw:], b[hw:])
        if cfg == 1.0:
            for a, b in zip(got, plain):
                assert torch.equal(a, b)
        else:
            mix = (fc[:hw] * float(cfg) + fu * float(1.0 - cfg)).half()
            l, nll64, sm64 = _ref64(mix, w16, y[:hw])
            assert float((got[0][:hw].double() - nll64).abs().max()) < 1e-3
            assert float((got[1][:hw].double() - sm64).abs().max()) < 1e-3


# ------------------------------------------------------------------ 2. Paella.token_scores against references
@pytest.mark.gpu
def test_tiny_token_scores_against_oracle_and_fixture(tiny):
    """The tiny model's forward agrees with the oracle to 7e-3 on the logits (smoke); an nll moves by at most twice that, and a
    guided one (cfg 3: 3 l_c - 2 l_u) by at most 10x that."""
    from oracle import scores as osc
    cfg, sd, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("scores_tiny.npz")
    cond = {"byt5": t(g["byt5"]), "clip": t(g["clip"]), "clip_image": t(g["clip_image"])}
    uncond = {k: torch.zeros_like(v) for k, v in cond.items()}
    x, y, r = t(z["noised"]), t(z["latents"]), t(g["r"])
    for name, scale, tol in (("cond", None, 1.4e-2), ("guided", float(z["cfg"]), 7e-2)):
        l64 = osc.score_logits(sd, oracle_cfg(cfg), x, r, cond, uncond, scale)
        for eps in (0.0, 0.1):
            s = tiny.token_scores(x.to(DEV), r.to(DEV), y.to(DEV), *(v.to(DEV) for v in cond.values()), label_smoothing=eps, cfg=scale)
            nll64, _, loss64, am64 = osc.token_scores(l64, y, eps)
            fix = t(z[f"loss_smooth_{name}"] if eps else z[f"loss_{name}"]).double()
            e = [float((s.nll.cpu().double() - nll64).abs().max()), float((s.loss.cpu().double() - loss64).abs().max()),
                 float((s.loss.cpu().double() - fix).abs().max())]
            _log({"case": "tiny", "name": name, "eps": eps, "err_nll": e[0], "err_loss": e[1], "err_fixture": e[2]})
            assert max(e) < tol, (name, eps, e)
            top2 = l64.topk(2, dim=1).values
            clear = (top2[:, 0] - top2[:, 1]) > 2 * tol
            assert torch.equal(s.argmax.cpu()[clear], am64[clear])
            assert torch.equal(s.argmax.cpu()[clear], t(z[f"argmax_{name}"])[clear])


def _default_model():
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    return m.to(DEV)


@pytest.fixture(scope="module")
def default_model():
    return _default_model()


def _conditioning(m, B, L, seed=7):
    from paella_b200.synth import synthetic_conditioning
    return synthetic_conditioning(B, L, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features, seed=seed,
                                  device=DEV)


@pytest.mark.gpu
def test_default_token_scores_against_fp64_cross_entropy(default_model):
    m = default_model
    m.batch_invariant = False
    B, H = 4, 16
    cond, uncond = _conditioning(m, B, 24)
    g = torch.Generator().manual_seed(4)
    x = torch.randint(0, m.num_labels, (B, H, H), generator=g).to(DEV)
    y = torch.randint(0, m.num_labels, (B, H, H), generator=g).to(DEV)
    r = torch.rand(B, generator=g).to(DEV)
    w16 = m.out_mapper[1].weight.detach().view(m.num_labels, -1).half()
    region = torch.zeros(H, H, dtype=torch.bool)
    region[:, :8] = True
    other = {"byt5": torch.randn(1, 24, 2560, generator=g).to(DEV), "clip": torch.randn(1, 1024, generator=g).to(DEV)}
    variants = {
        "plain": {},
        "rows": dict(tiling=["xy", None, None, "x"], attn_weights=[None, torch.linspace(0.5, 1.5, 20), None, None],
                     prompt_regions=[None, None, [(other, region)], None]),
    }
    for vname, kw in variants.items():
        logits = m(x, r, cond["byt5"], cond["clip"], **kw).double()
        for eps in (0.0, 0.1):
            s = m.token_scores(x, r, y, cond["byt5"], cond["clip"], label_smoothing=eps, **kw)
            want = F.cross_entropy(logits, y, reduction="none", label_smoothing=eps)
            e = float((s.loss.double() - want).abs().max())
            _log({"case": "default", "variant": vname, "eps": eps, "err": e})
            assert e < 2e-4, (vname, eps, e)
            _argmax_audit(logits.permute(0, 2, 3, 1).reshape(-1, m.num_labels), s.argmax.reshape(-1), vname)
    # guided, per-sample cfg: fp64 of the out_mapper on the fp32 CFG mix of the pair's features, rounded to fp16
    cfg = torch.tensor([3.0, 1.0, 0.0, 7.5])
    pair = m.prepare_conditioning([cond, uncond], (H, H))
    feats = m.features(x, r, pair, cfg_pairs=True)
    n = B * H * H
    c = cfg.repeat_interleave(H * H)[:, None].to(DEV)
    mix = (feats[:n] * c + feats[n:] * (1.0 - c)).half()
    for eps in (0.0, 0.1):
        s = m.token_scores(x, r, y, cond["byt5"], cond["clip"], label_smoothing=eps, cfg=cfg, unconditional_inputs=uncond)
        l = mix.double() @ w16.double().t()
        want = F.cross_entropy(l, y.reshape(-1), reduction="none", label_smoothing=eps)
        e = float((s.loss.reshape(-1).double() - want).abs().max())
        _log({"case": "default_guided", "eps": eps, "err": e})
        assert e < 1e-3, (eps, e)
        _argmax_audit(l, s.argmax.reshape(-1), "guided")
    # the default unconditional inputs are zeros
    s0 = m.token_scores(x, r, y, cond["byt5"], cond["clip"], cfg=cfg)
    s1 = m.token_scores(x, r, y, cond["byt5"], cond["clip"], cfg=cfg, unconditional_inputs=uncond)
    assert torch.equal(s0.nll, s1.nll)


# ------------------------------------------------------------------ 3. batch independence
def _batch_independence(m, H, L, sizes, cfg_vals):
    from paella_b200.synth import synthetic_conditioning
    big = max(sizes)
    cond, uncond = synthetic_conditioning(big, L, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features, seed=3,
                                          device=DEV)
    g = torch.Generator().manual_seed(6)
    x = torch.randint(0, m.num_labels, (big, H, H), generator=g).to(DEV)
    y = torch.randint(0, m.num_labels, (big, H, H), generator=g).to(DEV)
    r = torch.rand(big, generator=g).to(DEV)
    for cfg in cfg_vals:
        def run(idx):
            c = {k: v[idx] for k, v in cond.items()}
            u = {k: v[idx] for k, v in uncond.items()}
            cf = None if cfg is None else torch.full((len(idx),), cfg)
            return m.token_scores(x[idx], r[idx], y[idx], c["byt5"], c["clip"], label_smoothing=0.1, cfg=cf,
                                  unconditional_inputs=u if cfg is not None else None)
        alone = run([0])
        for n in sizes:
            pos = n - 1 if n > 1 else 0
            idx = list(range(1, n))
            idx.insert(pos, 0)
            got = run(idx)
            for a, b in zip(alone, got):
                assert torch.equal(a[0], b[pos]), (cfg, n)


@pytest.mark.gpu
def test_tiny_batch_independence(tiny):
    _batch_independence(tiny, 8, 5, (2, 5, 64), (None, 4.0))


@pytest.mark.gpu
def test_default_batch_independence_with_batch_invariant_mode(default_model):
    m = default_model
    m.batch_invariant = True
    try:
        _batch_independence(m, 16, 24, (2, 5, 64), (None, 4.0))
    finally:
        m.batch_invariant = False


# ------------------------------------------------------------------ 4. score() equals the hand loop
@pytest.mark.gpu
@pytest.mark.parametrize("guided", [False, True])
def test_score_equals_hand_loop(tiny, guided):
    from paella_b200 import utils as U
    from paella_b200.synth import synthetic_conditioning
    m = tiny
    B, H = 4, 8
    cond, uncond = synthetic_conditioning(B, 5, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features, seed=2,
                                          device=DEV)
    tokens = torch.randint(0, m.num_labels, (B, H, H), generator=torch.Generator().manual_seed(1)).to(DEV)
    levels = [1.0, 0.6, 0.25]
    cfg = torch.tensor([3.0, 1.5, 0.0, 2.0]) if guided else None
    seeds = [10, 11, 12, 13]
    gens = _gens(seeds)
    got = U.score(m, tokens, cond, uncond if guided else None, levels=levels, cfg=cfg, label_smoothing=0.1, generator=gens)
    hand = _gens(seeds)
    nll_sum = None
    for t_k in levels:
        tt = t_k * torch.ones(B, device=DEV)
        noised = m.add_noise(tokens, tt, generator=hand)[0]
        s = m.token_scores(noised, tt, tokens, cond["byt5"], cond["clip"], label_smoothing=0.1, cfg=cfg,
                           unconditional_inputs=uncond if guided else None)
        nll_sum = s.nll.clone() if nll_sum is None else nll_sum + s.nll
    assert torch.equal(got.nll_map, nll_sum / len(levels))
    want = got.nll_map.double().mean((1, 2))
    assert torch.allclose(got.nll.double(), want, rtol=1e-6, atol=0)
    assert all(a.get_offset() == b.get_offset() for a, b in zip(gens, hand))
    assert bool(((got.acc >= 0) & (got.acc <= 1)).all()) and bool(torch.isfinite(got.loss).all())


@pytest.mark.gpu
def test_score_equal_rows_regions_and_common_noise(tiny):
    from paella_b200 import utils as U
    from paella_b200.synth import synthetic_conditioning
    m = tiny
    B, H = 3, 8
    cond, _ = synthetic_conditioning(1, 5, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features, seed=2,
                                     device=DEV)
    cond = {k: v.expand(B, *v.shape[1:]).contiguous() for k, v in cond.items()}
    tok = torch.randint(0, m.num_labels, (1, H, H), generator=torch.Generator().manual_seed(1)).to(DEV).expand(B, H, H).contiguous()
    got = U.score(m, tok, cond, generator=_gens([5, 5, 6]))
    for a in got:
        assert torch.equal(a[0], a[1])
    assert not torch.equal(got.nll_map[0], got.nll_map[2])
    # an all-True region is no region, bit for bit
    full = U.score(m, tok, cond, generator=_gens([5, 5, 6]), region=torch.ones(B, H, H, dtype=torch.bool))
    for a, b in zip(got, full):
        assert torch.equal(a, b)
    # with a region the tokens outside it are never noised, and the means cover the region's tokens only
    region = torch.zeros(B, H, H, dtype=torch.bool)
    region[:, 2:6, 1:7] = True
    seen = []
    add_noise = m.add_noise

    def spy(*a, **k):
        out = add_noise(*a, **k)
        seen.append(out[0])
        return out
    m.add_noise = spy
    try:
        part = U.score(m, tok, cond, generator=_gens([5, 5, 6]), region=region)
    finally:
        del m.add_noise
    rd = region.to(DEV)
    assert seen and all(torch.equal(n[~rd], tok[~rd]) for n in seen)
    want = (part.nll_map.double() * rd).sum((1, 2)) / rd.sum((1, 2))
    assert torch.allclose(part.nll.double(), want, rtol=1e-6, atol=0)
