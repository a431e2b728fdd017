"""Confidence-guided renoising on the GPU.

  * pb200_paella_token_logprob against fp64 log-softmax of the kernel's own fp16 operand x fp16 weights x 1/T: c_out 64 / 256,
    8192 labels, hw not a multiple of 128, n_pairs = 0, between and = batch, per-sample T from 0.2 to 5; within (2e-4 + 1e-5 max|l|)
    / T, test_gpu_scores.py's nll bound scaled by 1/T.  At T = 1 it is -nll of pb200_paella_token_scores bit for bit.
  * pb200_renoise_confidence(_per_sample) against oracle/confidence.py on the uniforms oracle/philox.py restates: exactly n renoised
    per sample, ties to the lowest indices (tau = 0 rows bit for bit), regions, t = 0 / 1 / < 0, tau < 0 rows equal to
    pb200_add_noise_region(_per_sample) bit for bit, the slot map, generator offsets equal add_noise's.  Any other disagreement
    must be a key within a few ulp of the threshold (GPU logf against numpy's log): a margin audit.
  * the tiny model's per-step log-probabilities against the reference fixture (tests/golden/confidence_tiny.npz)
  * sampling: no entries launches the same kernels and gives the same tokens; None rows unchanged in a mixed batch; tau = 0
    renoises the least confident tokens; batch-1 equality under per-sample generators (tiny model, and the default model with
    batch_invariant = True); sample_distributed shards; one call mixing every other per-sample feature; the engine.
"""
import math
import types

import numpy as np
import pytest
import torch

from helpers import load_golden, log_jsonl, t

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _log(payload):
    log_jsonl("confidence.jsonl", payload)


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def tiny():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m


# ------------------------------------------------------------------ 1. token log-probabilities
def _head_model(c_out, NL):
    from paella_b200.modules import Paella
    cfg, _, _ = load_golden("paella_tiny.npz")
    torch.manual_seed(c_out * 5 + NL)
    m = Paella(**dict(cfg, c_in=c_out, c_out=c_out, num_labels=NL)).eval()
    with torch.no_grad():
        m.out_mapper[1].weight.copy_((torch.randn(NL, c_out) * (3.0 / math.sqrt(c_out))).view(NL, c_out, 1, 1))
    return m.to(DEV)


def _c_logprob(m, feats, batch, hw, tokens, n_pairs, params):
    """pb200_paella_token_logprob -> (logp fp32 [batch * hw], the fp16 operand it read [batch * hw, c_out])."""
    from paella_b200._lib import check, current_stream, lib, ptr
    m._ensure_packed()
    L = lib()
    out = torch.empty(batch * hw, device=DEV)
    ws = torch.empty(L.pb200_paella_token_scores_workspace_bytes(m._handle, batch, hw), dtype=torch.uint8, device=DEV)
    check(L.pb200_paella_token_logprob(m._handle, ptr(feats.contiguous()), batch, n_pairs, hw, ptr(params), ptr(tokens.contiguous()),
                                       ptr(out), ptr(ws), ws.numel(), current_stream()), "pb200_paella_token_logprob")
    torch.cuda.synchronize()
    a16 = ws[:batch * hw * feats.shape[1] * 2].view(torch.float16).view(batch * hw, feats.shape[1])
    return out, a16.clone()


@pytest.mark.parametrize("c_out,hw", [(64, 300), (256, 300), (256, 1024)])
@pytest.mark.parametrize("n_pairs", [0, 2, 4])
def test_logprob_kernel_against_fp64(c_out, hw, n_pairs):
    NL, B = 8192, 4
    m = _head_model(c_out, NL)
    w16 = m.out_mapper[1].weight.detach().view(NL, c_out).half()
    g = torch.Generator().manual_seed(c_out + hw + n_pairs)
    feats = torch.randn((B + n_pairs) * hw, c_out, generator=g).to(DEV)
    y = torch.randint(0, NL, (B * hw,), generator=g).to(DEV)
    temps = [0.2, 1.0, 2.5, 5.0]
    cfgs = [3.0, 1.5, 0.0, -1.0]
    params = torch.tensor([[c, 1.0 - c, 1.0 / T] for c, T in zip(cfgs, temps)], dtype=torch.float32).to(DEV)
    got, a16 = _c_logprob(m, feats, B, hw, y, n_pairs, params)
    l = a16.double() @ w16.double().t()
    inv_t = params[:, 2].double().repeat_interleave(hw)
    s = l * inv_t[:, None]
    want = s.gather(1, y[:, None]).squeeze(1) - torch.logsumexp(s, 1)
    tol = (2e-4 + 1e-5 * l.abs().amax(1)) * inv_t
    err = (got.double() - want).abs()
    _log({"case": "logprob", "c_out": c_out, "hw": hw, "n_pairs": n_pairs, "max_err_over_tol": float((err / tol).max())})
    assert bool((err <= tol).all()), float((err / tol).max())
    # the unmixed rows' operand is the plain cast; the mixed ones the guided mix of their pair
    assert torch.equal(a16[n_pairs * hw:], feats[n_pairs * hw:B * hw].half())
    if n_pairs:
        mix = feats[:n_pairs * hw] * params[:n_pairs, 0].repeat_interleave(hw)[:, None] + \
            feats[B * hw:] * params[:n_pairs, 1].repeat_interleave(hw)[:, None]
        assert float((a16[:n_pairs * hw].float() - mix).abs().max()) < 2e-3 * float(mix.abs().max())


@pytest.mark.parametrize("n_pairs", [0, 3])
def test_logprob_at_unit_temperature_is_minus_nll_bit_for_bit(n_pairs):
    from paella_b200._lib import check, current_stream, lib, ptr
    NL, c, hw, B = 8192, 256, 200, 3
    m = _head_model(c, NL)
    g = torch.Generator().manual_seed(5)
    feats = torch.randn((B + n_pairs) * hw, c, generator=g).to(DEV)
    y = torch.randint(0, NL, (B * hw,), generator=g).to(DEV)
    params = torch.tensor([[2.0, -1.0, 1.0], [4.0, -3.0, 1.0], [1.0, 0.0, 1.0]], device=DEV)
    got, _ = _c_logprob(m, feats, B, hw, y, n_pairs, params)
    L = lib()
    nll, smooth = torch.empty(B * hw, device=DEV), torch.empty(B * hw, device=DEV)
    am = torch.empty(B * hw, dtype=torch.int64, device=DEV)
    ws = torch.empty(L.pb200_paella_token_scores_workspace_bytes(m._handle, B, hw), dtype=torch.uint8, device=DEV)
    check(L.pb200_paella_token_scores(m._handle, ptr(feats), B, n_pairs, hw, ptr(params), ptr(y), ptr(nll), ptr(smooth), ptr(am),
                                      ptr(ws), ws.numel(), current_stream()), "pb200_paella_token_scores")
    assert torch.equal(got, -nll)


# ------------------------------------------------------------------ 2. the selection + renoise kernel
def _margin_audit(got, want, k_oracle, n, case):
    """got / want bool [N]; a disagreement must be a key within 8 ulp of the n-th smallest oracle key."""
    from oracle import confidence as oc
    assert int(got.sum()) == int(want.sum()) == n, (case, int(got.sum()), int(want.sum()), n)
    diff = np.flatnonzero(got != want)
    if len(diff) == 0:
        return 0
    order = np.lexsort((np.arange(len(k_oracle)), oc.order_keys(k_oracle)))
    thr = np.float32(k_oracle[order[n - 1]])
    ulp = np.spacing(np.abs(thr)).astype(np.float64)
    assert bool((np.abs(k_oracle[diff].astype(np.float64) - float(thr)) <= 8 * ulp).all()), (case, diff, k_oracle[diff], thr)
    return len(diff)


def _setup(B, H, W, seed, ties=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 64, (B, H, W), generator=g)
    rx = torch.randint(0, 64, (B, H, W), generator=g)
    src = torch.randint(0, 64, (B, H, W), generator=g)
    region = torch.rand(B, H, W, generator=g) < 0.7
    logp = -torch.rand(B, H, W, generator=g) * 6
    if ties:        # few distinct values: many equal keys at tau = 0
        logp = -torch.randint(0, 4, (B, H, W), generator=g).float()
    return x, rx, src, region, logp


def _check_rows(out, mask, x, rx, src, region, logp, u, taus, ts, use_region, case):
    from oracle import confidence as oc
    B = x.shape[0]
    audited = 0
    for b in range(B):
        reg = region[b].flatten().numpy() if use_region else None
        m = mask[b].flatten().cpu().numpy().astype(bool)
        if taus[b] < 0:
            continue
        want = oc.select(logp[b].flatten().numpy(), u[b].flatten(), taus[b], ts[b], reg)
        n = oc.renoise_count(ts[b], int(reg.sum()) if reg is not None else x[b].numel())
        if taus[b] == 0 or ts[b] <= 0 or ts[b] >= 1:
            assert np.array_equal(m, want), (case, b)          # keys are logp exactly (tau t = 0), or none / all
        else:
            audited += _margin_audit(m, want, oc.keys(logp[b].flatten().numpy(), u[b].flatten(), taus[b], ts[b]), n, (case, b))
        o, w_out = out[b].flatten().cpu(), torch.where(torch.from_numpy(m), rx[b].flatten(), x[b].flatten())
        if reg is not None:
            w_out = torch.where(torch.from_numpy(reg), w_out, src[b].flatten())
            assert not m[~reg].any()
        assert torch.equal(o, w_out), (case, b)
    return audited


@pytest.mark.parametrize("H,W,ties", [(24, 20, False), (24, 20, True), (64, 64, False), (181, 181, False)])
@pytest.mark.parametrize("use_region", [False, True])
def test_renoise_one_stream_against_oracle(H, W, ties, use_region):
    from oracle import philox
    from paella_b200 import ops
    taus = [0.0, 2.0, -1.0, 0.5, 0.0, 1.0, 3.0]
    ts = [0.5, 0.7, 0.3, 0.35, 1.0, 0.0, -1.0]
    B = len(taus)
    x, rx, src, region, logp = _setup(B, H, W, H + W + int(ties), ties)
    dev = lambda v: v.to(DEV)     # noqa: E731
    g = torch.Generator(device=DEV).manual_seed(77)
    g.set_offset(12)
    g2 = torch.Generator(device=DEV).manual_seed(77)
    g2.set_offset(12)
    seed, off = g.initial_seed(), g.get_offset()
    kw = dict(src=dev(src), region=dev(region)) if use_region else {}
    out, mask = ops.renoise_confidence(dev(x), dev(torch.tensor(ts)), dev(torch.tensor(taus)), dev(logp), dev(rx), g, **kw)
    ref_out, ref_mask = ops.add_noise(dev(x), dev(torch.tensor(ts)), dev(rx), 64, g2, **kw)
    torch.cuda.synchronize()
    assert g.get_offset() == g2.get_offset()
    for b in range(B):                  # tau < 0 rows: add_noise's own rows, bit for bit
        if taus[b] < 0:
            assert torch.equal(out[b], ref_out[b]) and torch.equal(mask[b], ref_mask[b])
    u = philox.rand(B * H * W, seed, off, _sm_count()).reshape(B, H, W)
    audited = _check_rows(out, mask, x, rx, src, region, logp, u, taus, ts, use_region, ("one", H, W, ties, use_region))
    _log({"case": "renoise_one_stream", "H": H, "W": W, "ties": ties, "region": use_region, "audited": audited})


@pytest.mark.parametrize("use_region", [False, True])
def test_renoise_per_sample_with_slot_map_against_oracle(use_region):
    from oracle import philox
    from paella_b200 import ops
    H, W = 32, 24
    taus = [0.0, -1.0, 2.0, 0.25, -1.0]
    ts = [0.6, 0.4, 0.9, 0.1, -1.0]
    B, P = len(taus), 8
    x, rx_pool, src_pool, region_pool, logp = _setup(B, H, W, 3)
    _, rx_pool, src_pool, region_pool, _ = _setup(P, H, W, 4)
    slot = torch.tensor([6, 0, 3, 7, 2], dtype=torch.int32)
    gens, gens2 = _gens(range(10, 10 + B)), _gens(range(10, 10 + B))
    for i, (a, b) in enumerate(zip(gens, gens2)):
        a.set_offset(4 * i)
        b.set_offset(4 * i)
    seeds = [(g.initial_seed(), g.get_offset()) for g in gens]
    table = ops.philox_table(gens, H * W, DEV)
    table2 = ops.philox_table(gens2, H * W, DEV)
    kw = dict(src=src_pool.to(DEV), region=region_pool.to(DEV)) if use_region else {}
    out_pool = torch.full((P, H, W), -7, dtype=torch.int64, device=DEV)
    ref_pool = out_pool.clone()
    mask, ref_mask = torch.empty(B, H, W, dtype=torch.int64, device=DEV), torch.empty(B, H, W, dtype=torch.int64, device=DEV)
    ops.renoise_confidence_per_sample(x.to(DEV), torch.tensor(ts, device=DEV), torch.tensor(taus, device=DEV), logp.to(DEV),
                                      rx_pool.to(DEV), table, out_pool, mask, slot=slot.to(DEV), **kw)
    ops.add_noise_per_sample(x.to(DEV), torch.tensor(ts, device=DEV), rx_pool.to(DEV), 64, table2, ref_pool, ref_mask,
                             slot=slot.to(DEV), **kw)
    torch.cuda.synchronize()
    assert [g.get_offset() for g in gens] == [g.get_offset() for g in gens2]
    untouched = sorted(set(range(P)) - set(slot.tolist()))
    assert bool((out_pool[untouched] == -7).all())
    s = slot.long()
    for b in range(B):
        if taus[b] < 0:
            assert torch.equal(out_pool[s[b]], ref_pool[s[b]]) and torch.equal(mask[b], ref_mask[b])
    u = np.stack([philox.rand(H * W, sd, of, _sm_count()).reshape(H, W) for sd, of in seeds])
    audited = _check_rows(out_pool[s].cpu(), mask, x, rx_pool[s], src_pool[s], region_pool[s], logp, u, taus, ts, use_region,
                          ("per_sample", use_region))
    _log({"case": "renoise_per_sample", "region": use_region, "audited": audited})


def test_renoise_rejects_a_grid_too_large():
    from paella_b200 import ops
    from paella_b200._lib import PaellaB200Error
    x = torch.zeros(1, 32769, dtype=torch.int64, device=DEV)
    with pytest.raises(PaellaB200Error, match="32768"):
        ops.renoise_confidence(x, torch.ones(1, device=DEV), torch.zeros(1, device=DEV), torch.zeros(1, 32769, device=DEV), x)


# ------------------------------------------------------------------ 3. the tiny model against the reference fixture
@pytest.mark.parametrize("which", ["cond", "guided"])
def test_tiny_logprob_and_masks_against_the_fixture(tiny, which):
    """The tiny forward agrees with the reference to 7e-3 on the logits (smoke); a log-probability moves by at most twice that
    over T, a guided one (cfg 3) by at most 10x that over T (test_gpu_scores.py's tiny bounds, scaled by 1/T).  The masks, drawn
    by the kernel on the fixture's (seed, offset) from the fixture's log-probabilities, must match it up to the margin audit."""
    from oracle import confidence as oc
    from paella_b200 import ops
    cfg, _, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("confidence_tiny.npz")
    B, H, W = z["tokens"].shape
    cond = {"byt5": t(g["byt5"]).to(DEV), "clip": t(g["clip"]).to(DEV), "clip_image": t(g["clip_image"]).to(DEV)}
    scale = float(z["cfg"]) if which == "guided" else None
    setup = tiny._score_setup(B, (H, W), cond, None, scale, None, None, None)
    x, r = t(g["x"]).to(DEV), t(g["r"]).to(DEV)
    feats = tiny.features(x, r, setup["cond"], None, 0, cfg_pairs=scale is not None)
    tokens = t(z["tokens"]).to(DEV)
    for name in [str(n) for n in z["names"]]:
        T, tau, t_next, use_region = z[f"{name}:params"].tolist()
        if str(z[f"{name}:which"]) != which:
            continue
        params = torch.tensor([[scale or 0.0, 1.0 - (scale or 0.0), 1.0 / T]] * B, dtype=torch.float32, device=DEV)
        logp = tiny.token_logprob(feats, B, B if scale is not None else 0, H * W, params, tokens)
        err = float((logp.cpu().double() - t(z[f"{name}:logp"])).abs().max())
        tol = (7e-2 if scale is not None else 1.4e-2) / T
        _log({"case": "tiny_fixture", "name": name, "err": err, "tol": tol})
        assert err < tol, (name, err, tol)
        gen = torch.Generator(device=DEV).manual_seed(int(z["seed"]))
        gen.set_offset(int(z["offset"]))
        region = t(z["region"]).to(DEV) if use_region else None
        lp = t(z[f"{name}:logp"]).float().to(DEV)
        kw = dict(src=tokens, region=region) if use_region else {}
        _, mask = ops.renoise_confidence(tokens, torch.full((B,), t_next, device=DEV), torch.full((B,), tau, device=DEV), lp,
                                         torch.zeros_like(tokens), gen, **kw)
        if _sm_count() == int(z["sm_count"]):
            for b in range(B):
                n = oc.renoise_count(t_next, int(z["region"][b].sum()) if use_region else H * W)
                k = oc.keys(z[f"{name}:logp"][b].reshape(-1).astype(np.float32), z["u"][b].reshape(-1), tau, t_next)
                if use_region:
                    k = np.where(z["region"][b].reshape(-1), k, np.float32(np.inf))
                _margin_audit(mask[b].flatten().cpu().numpy().astype(bool), z[f"{name}:mask"][b].reshape(-1), k, n, name)


# ------------------------------------------------------------------ 4. sampling
def _cond(m, B, L=5, seed=0):
    g = torch.Generator().manual_seed(seed)
    E, C = m.byt5_mapper.in_features, m.clip_mapper.in_features
    c = {"byt5": torch.randn(B, L, E, generator=g).to(DEV), "clip": torch.randn(B, C, generator=g).to(DEV)}
    return c, {k: torch.zeros_like(v) for k, v in c.items()}


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "emcpy" not in e.name
             and "emset" not in e.name]
    return out, names


def test_no_entries_launch_the_same_kernels_and_tokens(tiny):
    from paella_b200 import utils as U
    c, u = _cond(tiny, 3)

    def run(conf):
        torch.manual_seed(5)
        return U.sample(tiny, c, (3, 8, 8), u, steps=4, renoise_steps=3, cfg=4.0, confidence_renoise=conf)
    run(None)
    a, na = _kernel_names(lambda: run(None))
    b, nb = _kernel_names(lambda: run([None, None, None]))
    assert torch.equal(a, b) and na == nb and na
    _, nc = _kernel_names(lambda: run([None, 1.0, None]))
    assert any("renoise_confidence" in n for n in nc) and any("token_logprob" in n for n in nc)
    assert not any("renoise_confidence" in n or "token_logprob" in n for n in na)


@pytest.mark.parametrize("per_sample", [False, True])
def test_mixed_batch_leaves_none_rows_unchanged(tiny, per_sample):
    from paella_b200 import utils as U
    c, u = _cond(tiny, 4, seed=1)
    region = torch.rand(4, 8, 8, generator=torch.Generator().manual_seed(2)) < 0.6
    init_x = torch.randint(0, 64, (4, 8, 8), generator=torch.Generator().manual_seed(3))

    def run(conf):
        gens = _gens([1, 2, 3, 4]) if per_sample else None
        if not per_sample:
            torch.manual_seed(9)
        out = U.sample_distributed(tiny, c, u, (4, 8, 8), init_x=init_x, region=region, steps=5, generator=gens,
                                   confidence_renoise=conf)
        offs = [g.get_offset() for g in gens] if per_sample else [torch.cuda.default_generators[0].get_offset()]
        return out, offs
    plain, off_plain = run(None)
    mixed, off_mixed = run([None, 0.0, None, 2.0])
    assert off_plain == off_mixed
    assert torch.equal(plain[0], mixed[0]) and torch.equal(plain[2], mixed[2])
    assert bool((mixed[~region.to(DEV)] == init_x.to(DEV)[~region.to(DEV)]).all())


def test_tau0_renoises_the_least_confident_tokens(tiny):
    from paella_b200 import utils as U
    c, u = _cond(tiny, 3, seed=4)
    rec = []
    orig = tiny.add_noise

    def spy(*a, **k):
        res = orig(*a, **k)
        if k.get("confidence") is not None:
            rec.append((k["confidence"].clone(), res[1].clone()))
        return res
    tiny.add_noise = spy
    try:
        U.sample_notebook(tiny, c, (3, 8, 8), u, steps=6, generator=_gens([4, 5, 6]), confidence_renoise=[0.0, None, 0.0])
    finally:
        del tiny.add_noise
    assert len(rec) == 5
    for logp, mask in rec:
        for b in (0, 2):
            m = mask[b].bool()
            if m.any() and (~m).any():
                assert float(logp[b][m].max()) <= float(logp[b][~m].min())


def _mixed_call(m, B, rows, conf, vq, **over):
    """sample_notebook on rows ``rows`` of a batch mixing every other per-sample feature with confidence renoising."""
    from paella_b200 import utils as U
    c, u = _cond(m, B, seed=11)
    g = torch.Generator().manual_seed(12)
    terms_in = {k: v[:1] * 0.5 for k, v in c.items()}
    init_x = torch.randint(0, 64, (B, 8, 8), generator=g)
    region = torch.rand(B, 8, 8, generator=g) < 0.7
    weights = [torch.rand(4, generator=g) + 0.5 for _ in range(B)]
    per = dict(guidance_prompts=[[(terms_in, 0.5)], None, None, None, None, None][:B], pag=[None, 2.0, None, None, None, None][:B],
               top_k=torch.tensor([0, 0, 8, 0, 0, 3][:B]), tiling=["none", "none", "x", "xy", "y", "none"][:B],
               attn_weights=weights, mode=["multinomial", "multinomial", "multinomial", "argmax", "quant", "multinomial"][:B],
               confidence_renoise=conf)
    per.update(over)
    sel = {}
    for k, v in per.items():
        if torch.is_tensor(v):
            sel[k] = v[rows]
        elif isinstance(v, list):
            sel[k] = [v[i] for i in rows]
        else:
            sel[k] = v
    cc = {k: v[rows] for k, v in c.items()}
    uu = {k: v[rows] for k, v in u.items()}
    gens = _gens([100 + i for i in rows])
    out, inter = U.sample_notebook(m, cc, (len(rows), 8, 8), uu, init_x=init_x[rows], region=region[rows], steps=5, vqmodel=vq,
                                   generator=gens, **sel)
    return out, inter, [gg.get_offset() for gg in gens]


def test_one_call_mixes_every_feature_and_rows_equal_batch1(tiny):
    cb = torch.randn(64, 4, generator=torch.Generator().manual_seed(1)).to(DEV)
    vq = types.SimpleNamespace(vquantizer=types.SimpleNamespace(codebook=types.SimpleNamespace(weight=types.SimpleNamespace(data=cb))))
    B = 6
    conf = [0.0, 2.0, 1.0, 0.5, None, 3.0]
    full, inter, offs = _mixed_call(tiny, B, list(range(B)), conf, vq)
    plain, _, offs_plain = _mixed_call(tiny, B, list(range(B)), None, vq)
    assert offs == offs_plain
    assert torch.equal(full[4], plain[4])
    for b in range(B):
        one, one_inter, one_off = _mixed_call(tiny, B, [b], conf, vq)
        assert torch.equal(full[b:b + 1], one), b
        assert all(torch.equal(a[b:b + 1], o) for a, o in zip(inter, one_inter)), b
        assert one_off == [offs[b]]


def test_sample_distributed_shards_equal_rows(tiny):
    from paella_b200 import utils as U
    B = 5
    c, u = _cond(tiny, B, seed=21)
    conf = [0.0, None, 2.0, 1.0, 0.3]
    temps = torch.tensor([[0.7, 0.3], [1.0, 0.2], [0.5, 0.5], [2.0, 0.4], [0.9, 0.1]])
    full = U.sample_distributed(tiny, c, u, (B, 8, 8), steps=5, temperature=temps, generator=_gens(range(30, 30 + B)),
                                confidence_renoise=conf)
    for lo, hi in ((0, 2), (2, 5)):
        part = U.sample_distributed(tiny, {k: v[lo:hi] for k, v in c.items()}, {k: v[lo:hi] for k, v in u.items()}, (hi - lo, 8, 8),
                                    steps=5, temperature=temps[lo:hi], generator=_gens(range(30 + lo, 30 + hi)),
                                    confidence_renoise=conf[lo:hi])
        assert torch.equal(part, full[lo:hi])


def test_default_model_rows_equal_batch1_in_batch_invariant_mode():
    from paella_b200 import utils as U
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_, synthetic_conditioning
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    m = m.to(DEV)
    m.batch_invariant = True
    B, H = 3, 16
    c, u = synthetic_conditioning(B, 24, byt5_embd=2560, clip_embd=m.clip_mapper.in_features, seed=3, device=DEV)
    conf = [0.0, 2.0, None]
    full = U.sample(m, c, (B, H, H), u, steps=4, renoise_steps=3, cfg=torch.tensor([4.0, 0.0, 6.0]), generator=_gens([1, 2, 3]),
                    confidence_renoise=conf)
    cfgs = [4.0, 0.0, 6.0]
    for b in range(B):
        one = U.sample(m, {k: v[b:b + 1] for k, v in c.items()}, (1, H, H), {k: v[b:b + 1] for k, v in u.items()}, steps=4,
                       renoise_steps=3, cfg=cfgs[b], generator=_gens([b + 1]), confidence_renoise=[conf[b]])
        assert torch.equal(full[b:b + 1], one), b


def test_engine_request_equals_batch1_sample_notebook(tiny):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    c, u = _cond(tiny, 1, seed=41)
    shared = {k: v for k, v in u.items()}
    region = torch.rand(1, 8, 8, generator=torch.Generator().manual_seed(4)) < 0.6
    init_x = torch.randint(0, 64, (1, 8, 8), generator=torch.Generator().manual_seed(5))
    specs = [dict(seed=1, tau=0.0, steps=6), dict(seed=2, tau=None, steps=4), dict(seed=3, tau=2.0, steps=5, region=True),
             dict(seed=4, tau=1.0, steps=3, cfg=None)]
    eng = SamplingEngine(tiny, latent_hw=(8, 8), max_batch=3, max_cond_len=20, unconditional_inputs=shared)
    reqs = []
    for sp in specs:
        g = torch.Generator(device=DEV).manual_seed(sp["seed"])
        kw = dict(init_x=init_x.to(DEV), region=region.to(DEV)) if sp.get("region") else {}
        reqs.append((eng.submit(c, generator=g, steps=sp["steps"], cfg=sp.get("cfg", (4.0, 4.0)), keep_intermediates=True,
                                confidence_renoise=sp["tau"], **kw), g))
    eng.run_until_idle()
    for sp, (q, g) in zip(specs, reqs):
        g1 = torch.Generator(device=DEV).manual_seed(sp["seed"])
        kw = dict(init_x=init_x.to(DEV), region=region.to(DEV)) if sp.get("region") else {}
        out, inter = U.sample_notebook(tiny, c, (1, 8, 8), u, steps=sp["steps"], cfg=sp.get("cfg", (4.0, 4.0)), generator=[g1],
                                       confidence_renoise=[sp["tau"]], **kw)
        assert torch.equal(q.result, out), sp
        assert len(q.intermediates) == len(inter) and all(torch.equal(a, b) for a, b in zip(q.intermediates, inter)), sp
        assert g.get_offset() == g1.get_offset(), sp


def test_validation_raises_before_any_draw(tiny):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    c, u = _cond(tiny, 2)
    gens = _gens([1, 2])
    offs = [g.get_offset() for g in gens]
    for bad in ([1.0], [None, -1.0], True, [math.inf, None]):
        with pytest.raises(ValueError):
            U.sample_notebook(tiny, c, (2, 8, 8), u, generator=gens, confidence_renoise=bad)
    with pytest.raises(ValueError):
        U.sample(tiny, c, (2, 8, 8), u, generator=gens, exact=True, confidence_renoise=0.0)
    assert [g.get_offset() for g in gens] == offs
    eng = SamplingEngine(tiny, latent_hw=(8, 8), max_batch=2, max_cond_len=20, unconditional_inputs={k: v[:1] for k, v in u.items()})
    g = torch.Generator(device=DEV).manual_seed(1)
    for bad in ([1.0], -2.0, False, math.nan):
        with pytest.raises(ValueError):
            eng.submit({k: v[:1] for k, v in c.items()}, generator=g, confidence_renoise=bad)
    assert g.get_offset() == 0 and not eng.busy
