"""Token scoring without a GPU: the oracle against the reference fixture, the label-smoothed loss composition, argument
validation before any work, score()'s draw order and accumulation, and the SASS of the scoring kernel."""
import collections
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

from helpers import load_golden, oracle_cfg, t

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------ oracle against the reference fixture
def test_oracle_matches_reference_fixture():
    # The reference runs in fp32 and the oracle's forward agrees with it to ~1e-6 relative on logits of magnitude ~2
    # (test_oracle_golden); with cfg = 3 the guided logits are ~5x larger, so 1e-4 absolute on the losses leaves room.
    from oracle import scores as osc
    cfg, sd, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("scores_tiny.npz")
    cond = {"byt5": t(g["byt5"]), "clip": t(g["clip"]), "clip_image": t(g["clip_image"])}
    uncond = {k: torch.zeros_like(v) for k, v in cond.items()}
    x, y, r = t(z["noised"]), t(z["latents"]), t(g["r"])
    for name, scale in (("cond", None), ("guided", float(z["cfg"]))):
        logits = osc.score_logits(sd, oracle_cfg(cfg), x, r, cond, uncond, scale)
        nll, _, loss, argmax = osc.token_scores(logits, y, 0.1)
        assert float((nll - t(z[f"loss_{name}"]).double()).abs().max()) < 1e-4, name
        assert float((loss - t(z[f"loss_smooth_{name}"]).double()).abs().max()) < 1e-4, name
        top2 = logits.topk(2, dim=1).values
        clear = (top2[:, 0] - top2[:, 1]) > 1e-4
        assert torch.equal(argmax[clear], t(z[f"argmax_{name}"])[clear]), name


@pytest.mark.parametrize("eps", [0.0, 0.1, 0.37, 1.0])
def test_loss_composition_is_label_smoothed_cross_entropy(eps):
    """(1 - eps) nll + eps smooth with the kernel's nll = lse - l_y and smooth = lse - mean l is torch's label-smoothed cross
    entropy, in fp64 on synthetic logits (magnitudes up to 30)."""
    from oracle import scores as osc
    from paella_b200 import ops
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(3, 200, 5, 4, generator=g, dtype=torch.float64) * 10
    y = torch.randint(0, 200, (3, 5, 4), generator=g)
    nll, smooth, _, _ = osc.token_scores(logits, y)
    got = ops.smoothed_loss(nll, smooth, eps)
    want = F.cross_entropy(logits, y, reduction="none", label_smoothing=eps)
    assert float((got - want).abs().max()) < 1e-12
    assert float((nll - F.cross_entropy(logits, y, reduction="none")).abs().max()) < 1e-12
    if eps == 0.0:
        assert got is nll


# ------------------------------------------------------------------ validation: ValueError / TypeError before any work
def _sabotaged_tiny():
    """The tiny model on the CPU with every method that enqueues work replaced by a failure: a check must come first."""
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).eval()
    m.load_state_dict(sd)

    def fail(name):
        def f(*a, **k):
            raise AssertionError(f"model.{name} called before the check")
        return f
    for name in ("prepare_conditioning", "_cond_for_forward", "features", "_ws", "regional_device", "add_noise", "_score_tokens"):
        setattr(m, name, fail(name))
    return m


@pytest.fixture
def no_copies(monkeypatch):
    from paella_b200 import ops

    def fail(*a, **k):
        raise AssertionError("a host-to-device copy before the check")
    for name in ("to_device_async", "to_device_packed", "attn_weights_to_device"):
        monkeypatch.setattr(ops, name, fail)


def _args(B=2, H=8):
    _, _, g = load_golden("paella_tiny.npz")
    x = torch.zeros(B, H, H, dtype=torch.int64)
    cond = {"byt5": t(g["byt5"])[:B], "clip": t(g["clip"])[:B]}
    return x, torch.full((B,), 0.5), cond


BAD_TOKEN_SCORES = {
    "targets_int32": dict(targets=torch.zeros(2, 8, 8, dtype=torch.int32)),
    "targets_shape": dict(targets=torch.zeros(2, 8, 4, dtype=torch.int64)),
    "targets_device": dict(targets=torch.zeros(2, 8, 8, dtype=torch.int64, device="meta")),
    "targets_list": dict(targets=[[0]]),
    "eps_negative": dict(label_smoothing=-0.1),
    "eps_above_one": dict(label_smoothing=1.5),
    "eps_nan": dict(label_smoothing=float("nan")),
    "eps_bool": dict(label_smoothing=True),
    "cfg_nan": dict(cfg=float("nan")),
    "cfg_bool": dict(cfg=True),
    "cfg_shape": dict(cfg=torch.ones(3)),
    "cfg_int_tensor": dict(cfg=torch.ones(2, dtype=torch.int64)),
    "tiling_unknown": dict(tiling="z"),
    "tiling_length": dict(tiling=["x"]),
    "attn_weights_length": dict(attn_weights=[None]),
    "attn_weights_too_long": dict(attn_weights=[torch.ones(1000), None]),
    "regions_length": dict(prompt_regions=[None]),
    "regions_shape": dict(prompt_regions=[[({"byt5": torch.zeros(1, 5, 40)}, torch.ones(4, 4, dtype=torch.bool))], None]),
    "regions_weighted": dict(prompt_regions=[[({"byt5": torch.zeros(1, 5, 40)}, torch.ones(8, 8, dtype=torch.bool))], None],
                             attn_weights=torch.ones(3)),
}


@pytest.mark.parametrize("case", sorted(BAD_TOKEN_SCORES))
def test_token_scores_validation_before_any_work(case, no_copies):
    m = _sabotaged_tiny()
    x, r, cond = _args()
    kw = dict(BAD_TOKEN_SCORES[case])
    targets = kw.pop("targets", torch.zeros(2, 8, 8, dtype=torch.int64))
    with pytest.raises(ValueError):
        m.token_scores(x, r, targets, cond["byt5"], cond["clip"], **kw)


def test_token_scores_unknown_keyword_is_a_type_error():
    m = _sabotaged_tiny()
    x, r, cond = _args()
    with pytest.raises(TypeError):
        m.token_scores(x, r, x.clone(), cond["byt5"], cond["clip"], attention_maps=True)
    with pytest.raises(TypeError):
        m.token_scores(x, r, x.clone(), cond["byt5"], cond["clip"], None, 0.1)     # label_smoothing is keyword-only


BAD_SCORE = {
    "tokens_int32": dict(tokens=torch.zeros(2, 8, 8, dtype=torch.int32)),
    "tokens_2d": dict(tokens=torch.zeros(8, 8, dtype=torch.int64)),
    "tokens_device": dict(tokens=torch.zeros(2, 8, 8, dtype=torch.int64, device="meta")),
    "levels_empty": dict(levels=[]),
    "levels_above_one": dict(levels=[0.5, 1.5]),
    "levels_negative": dict(levels=[-0.1]),
    "levels_nan": dict(levels=[float("nan")]),
    "levels_bool": dict(levels=[True]),
    "levels_2d_tensor": dict(levels=torch.ones(2, 2) * 0.5),
    "levels_int_tensor": dict(levels=torch.ones(2, dtype=torch.int64)),
    "levels_scalar": dict(levels=0.5),
    "eps": dict(label_smoothing=2.0),
    "cfg": dict(cfg=torch.ones(5)),
    "generator_length": dict(generator=[torch.Generator()]),
    "region_shape": dict(region=torch.ones(2, 4, 4, dtype=torch.bool)),
    "region_dtype": dict(region=torch.ones(2, 8, 8, dtype=torch.uint8)),
    "tiling": dict(tiling="diagonal"),
    "attn_weights": dict(attn_weights=[None, None, None]),
    "prompt_regions": dict(prompt_regions=[None, None, None]),
}


@pytest.mark.parametrize("case", sorted(BAD_SCORE))
def test_score_validation_before_any_work(case, no_copies):
    from paella_b200 import utils as U
    m = _sabotaged_tiny()
    _, _, cond = _args()
    kw = dict(BAD_SCORE[case])
    tokens = kw.pop("tokens", torch.zeros(2, 8, 8, dtype=torch.int64))
    gens = kw.get("generator")
    before = [g.get_state().clone() for g in gens] if isinstance(gens, list) else None
    with pytest.raises(ValueError):
        U.score(m, tokens, cond, **kw)
    if before is not None:
        assert all(torch.equal(b, g.get_state()) for b, g in zip(before, gens))


# ------------------------------------------------------------------ score(): draw order and accumulation
class _RecordingModel:
    """Stands in for Paella in utils.score: add_noise draws its mask and replacement codes from the generator it is given, and
    the scores are a deterministic function of (noised tokens, r, targets); every call is recorded."""

    num_labels = 16

    def __init__(self):
        self.calls = []

    def _device(self):
        return torch.device("cpu")

    def _check_score_targets(self, targets, shape, name="targets"):
        from paella_b200.modules import Paella
        Paella._check_score_targets(self, targets, shape, name)

    def _score_setup(self, batch, latent_hw, *a):
        self.calls.append(("setup", batch, tuple(latent_hw)))
        return {"batch": batch}

    def add_noise(self, x, t, generator=None, src=None, region=None):
        self.calls.append(("add_noise", t.clone(), generator, region is not None))
        return _hand_add_noise(x, t, generator, region), None

    def _score_tokens(self, setup, x, r, targets, eps):
        from paella_b200.modules import TokenScores
        from paella_b200 import ops
        self.calls.append(("score", x.clone(), r.clone(), eps))
        return _hand_scores(x, r, targets, eps, ops, TokenScores)


def _hand_add_noise(x, t, generator, region=None):
    mask = torch.rand(x.shape, generator=generator) <= t[:, None, None]
    codes = torch.randint(0, 16, x.shape, generator=generator)
    if region is not None:
        mask &= region
    return torch.where(mask, codes, x)


def _hand_scores(x, r, targets, eps, ops, TokenScores):
    nll = (x.float() * 0.37 + r[:, None, None] * 1.3 + targets.float() * 0.01).sin() + 2.0
    smooth = nll * 1.7 + 0.25
    return TokenScores(nll, ops.smoothed_loss(nll, smooth, eps), (x * 3) % 16)


@pytest.mark.parametrize("with_region", [False, True])
def test_score_draw_order_and_accumulation_match_a_hand_loop(with_region):
    from paella_b200 import ops
    from paella_b200 import utils as U
    from paella_b200.modules import TokenScores
    B, H, W = 3, 4, 5
    tokens = torch.randint(0, 16, (B, H, W), generator=torch.Generator().manual_seed(1))
    region = (torch.rand(B, H, W, generator=torch.Generator().manual_seed(2)) < 0.6) if with_region else None
    levels = [1.0, 0.75, 0.3, 0.0]
    m = _RecordingModel()
    g = torch.Generator().manual_seed(9)
    got = U.score(m, tokens, {"byt5": torch.zeros(B, 2, 4)}, levels=levels, label_smoothing=0.1, generator=g, region=region)

    # the hand loop: add_noise then token_scores per level, in level order, on a generator seeded alike
    g2 = torch.Generator().manual_seed(9)
    nll_sum = loss_sum = hits = None
    kinds = [c[0] for c in m.calls]
    assert kinds == ["setup"] + ["add_noise", "score"] * len(levels)
    for k, t_k in enumerate(levels):
        t = t_k * torch.ones(B)
        noised = _hand_add_noise(tokens, t, g2, region)
        _, t_rec, g_rec, reg_rec = m.calls[1 + 2 * k]
        _, x_rec, r_rec, eps_rec = m.calls[2 + 2 * k]
        assert torch.equal(t_rec, t) and g_rec is g and reg_rec == with_region and eps_rec == 0.1
        assert torch.equal(x_rec, noised) and torch.equal(r_rec, t)
        if region is not None:
            assert torch.equal(noised[~region], tokens[~region])
        s = _hand_scores(noised, t, tokens, 0.1, ops, TokenScores)
        hit = (s.argmax == tokens).float()
        if nll_sum is None:
            nll_sum, loss_sum, hits = s.nll.clone(), s.loss.clone(), hit
        else:
            nll_sum += s.nll
            loss_sum += s.loss
            hits += hit
    assert torch.equal(g.get_state(), g2.get_state())
    K = len(levels)
    assert torch.equal(got.nll_map, nll_sum / K)
    w = region.double() if region is not None else torch.ones(B, H, W, dtype=torch.float64)
    for name, mp in (("nll", nll_sum / K), ("loss", loss_sum / K), ("acc", hits / K)):
        want = (mp.double() * w).sum((1, 2)) / w.sum((1, 2))
        assert torch.allclose(getattr(got, name).double(), want, rtol=1e-6, atol=0), name
        assert getattr(got, name).dtype == torch.float32 and getattr(got, name).shape == (B,)


def test_score_default_levels_are_an_8_step_samples():
    from paella_b200 import utils as U
    m = _RecordingModel()
    U.score(m, torch.zeros(1, 2, 2, dtype=torch.int64), {"byt5": torch.zeros(1, 2, 4)}, generator=torch.Generator().manual_seed(0))
    ts = [float(c[1][0]) for c in m.calls if c[0] == "add_noise"]
    assert ts == torch.linspace(1.0, 0.0, 9)[:8].tolist()


# ------------------------------------------------------------------ the scoring kernel's SASS
def test_token_score_kernel_is_wgmma_and_tma_without_uniformisation_loops():
    so = os.path.join(ROOT, "paella_b200", "libpaella_b200.so")
    if shutil.which("cuobjdump") is None or not os.path.exists(so):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, check=True).stdout
    fn, counts = None, collections.Counter()
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            continue
        if fn and "token_score_kernel" in fn:
            m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
            if m:
                counts[m.group(1).split(".")[0]] += 1
                counts["BRA.U.ANY"] += m.group(1).startswith("BRA.U.ANY")
                counts["CALL"] += m.group(1).startswith("CALL")
    assert counts["HGMMA"] > 0 and counts["UTMALDG"] > 0, dict(counts)
    assert counts["HMMA"] == 0 and counts["CALL"] == 0, dict(counts)
    # the TMA issue path is entered through elect.sync: no ELECT ... BRA.U.ANY loop
    assert counts["BRA.U.ANY"] == 0, dict(counts)
