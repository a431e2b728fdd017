"""Attention maps on the GPU.

  1. Kernels: the maps instances of both attention kernels (pb200_attention_maps) against an fp64 softmax of the same fp16 Q/K, at
     head dims 16/32/64/96 (mma.sync), 80 (wgmma) and 80 on the mma.sync kernel (a PB200_ATTN_MMA_SYNC=1 child, as in
     test_gpu_attention_matrix.py): ragged query counts, kv_len < S_max, a slot shared by two samples, a per-sample weight table
     and a skipped sample (map_row -1).  exp2(score - lse2) is each key's probability before the weights; entries past kv_len,
     the skipped sample's row and the unused row are untouched; O equals pb200_attention_slots on the same inputs bit for bit.
  2. Forward: Paella.forward(..., attention_maps=True) on the tiny model against the reference fixture, within a bound derived
     from the oracle with fp16 rounding; the logits equal the call without maps bit for bit.
  3. Sampling: sample, sample_distributed and sample_notebook with maps give the tokens, intermediates and generator offsets of
     the call without them (cfg, per-sample attn_weights, tiling, an inpainting region, argmax / quant rows, guidance prompts);
     sample_notebook's maps equal the mean of Paella.forward's maps over the step inputs recovered from its intermediates.
  4. Batch invariance: each row's maps equal its batch-1 call's bit for bit (tiny model in both modes, default model with
     batch_invariant = True).
  5. Engine: staggered requests with and without maps, different step counts, conditioning lengths and guidance: each
     req.attention_maps equals its batch-1 sample_notebook maps bit for bit, and every request's tokens equal its batch-1 call.
  6. Invariants: maps >= 0, and the keys' sum <= 1 on unweighted samples.
  7. The plain path launches no maps kernel.
"""
import collections
import ctypes
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from helpers import load_golden, log_jsonl, oracle_cfg, t

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


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


# ------------------------------------------------------------------ 1. kernels
P_VALUES = (1, 63, 64, 65, 200)
LENS = (1, 63, 64, 65, 129)            # kv_len of the 5 cache slots, rotated per case
KV_SLOT = (3, 1, 3, 0)                 # samples 0 and 2 share slot 3
MAP_ROW = (2, -1, 0, 1)                # sample 1 is skipped; accumulator row 3 is never named
W_LD, W_LEN, W_ROW = 4, (2, 0, 3), (2, 0, 1)     # samples 0..2 weighted by table rows 2, 0, 1 (row 1 is empty)


def _p(x):
    return ctypes.c_void_p(x.data_ptr()) if x is not None else None


def _kernel_case(hd, P, rot):
    """Runs one case and returns its worst error ratio; raises AssertionError on a failed check."""
    from paella_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device=DEV).manual_seed(100 * P + hd)
    B, H = len(KV_SLOT), 2
    E = H * hd
    lens = [LENS[(j + rot) % len(LENS)] for j in range(len(LENS))]
    S = max(lens) + 3                   # kv_len < S_max for every slot
    qkv = (torch.randn(B * P, 3 * E, device=DEV, generator=g) * 0.5).half()
    ckv = (torch.randn(len(LENS), S, 2 * E, device=DEV, generator=g) * 0.5).half()
    kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    kv_slot = torch.tensor(KV_SLOT, dtype=torch.int32, device=DEV)
    w = (torch.rand(3, W_LD, device=DEV, generator=g) * 1.5 + 0.25).float()
    w_len = torch.tensor(W_LEN, dtype=torch.int32, device=DEV)
    w_row = torch.tensor(W_ROW, dtype=torch.int32, device=DEV)
    map_row = torch.tensor(MAP_ROW, dtype=torch.int32, device=DEV)
    scores = torch.full((4, H, P, S), float("nan"), device=DEV)
    lse2 = torch.full((4, H, P), float("nan"), device=DEV)
    out_m = torch.full((B * P, E), float("nan"), dtype=torch.float16, device=DEV)
    out_p = torch.full_like(out_m, float("nan"))
    args = (_p(qkv), _p(ckv), _p(kv_len), _p(kv_slot), len(LENS), None, B, P, S, E, H, 1, _p(w), 0, W_LD, _p(w_len), _p(w_row), 3)
    a = list(args)
    a[5] = _p(out_m)
    assert L.pb200_attention_maps(*a, _p(scores), _p(lse2), _p(map_row), B, _lib.current_stream()) == 0, L.pb200_last_error()
    a[5] = _p(out_p)
    assert L.pb200_attention_slots(*a, _lib.current_stream()) == 0, L.pb200_last_error()
    torch.cuda.synchronize()
    assert torch.equal(out_m.view(torch.int16), out_p.view(torch.int16)), "O differs from the plain instance"
    worst = 0.0
    for b, mr in enumerate(MAP_ROW):
        if mr < 0:
            continue
        n = lens[KV_SLOT[b]]
        rows = qkv[b * P:(b + 1) * P].double()
        q = rows[:, :E].view(P, H, hd).transpose(0, 1)
        k = torch.cat([rows[:, E:2 * E], ckv[KV_SLOT[b], :n, :E].double()]).view(P + n, H, hd).transpose(0, 1)
        z = q @ k.transpose(-1, -2) / math.sqrt(hd)
        p = torch.softmax(z, -1)[..., P:]
        got = torch.exp2(scores[mr, :, :, :n].double() - lse2[mr, :, :, None].double())
        # fp32 scores of exact fp16 products (relative ~2^-20 of the |q||k| sum) and an fp32 log-sum-exp: the exponent is off by a
        # few 1e-6 at these magnitudes, so p is within 1e-4 relative of the fp64 value (plus a floor for underflowing keys)
        bound = 1e-4 * p + 1e-9
        err = (got - p).abs()
        worst = max(worst, float((err / bound).max()))
        assert bool((err <= bound).all()), (b, float(err.max()))
        assert bool(torch.isnan(scores[mr, :, :, n:]).all()), "entries past kv_len were written"
        assert bool(torch.isfinite(lse2[mr]).all())
    assert bool(torch.isnan(scores[3]).all()) and bool(torch.isnan(lse2[3]).all()), "an unnamed map row was written"
    return worst


KERNEL_CASES = [(hd, P, i) for hd in (16, 32, 64, 80, 96) for i, P in enumerate(P_VALUES)]


@pytest.mark.parametrize("hd,P,rot", KERNEL_CASES, ids=[f"hd{hd}-P{P}" for hd, P, _ in KERNEL_CASES])
def test_maps_kernel_against_fp64(hd, P, rot):
    worst = _kernel_case(hd, P, rot)
    log_jsonl("attention_maps.jsonl", {"test": "kernel", "hd": hd, "P": P, "worst_ratio": worst})


def _child_main():
    """Runs in a PB200_ATTN_MMA_SYNC=1 child: the kernel head_dim 80 runs, then every head_dim-80 case."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _kernel_case(80, 64, 0)
        torch.cuda.synchronize()
    print("KERNELS", json.dumps(sorted({e.name for e in prof.events() if "attention" in e.name})), flush=True)
    for i, P in enumerate(P_VALUES):
        try:
            print("RES", json.dumps({"P": P, "ok": True, "worst": _kernel_case(80, P, i)}), flush=True)
        except Exception as e:
            print("RES", json.dumps({"P": P, "ok": False, "msg": f"{type(e).__name__}: {e}"}), flush=True)


def test_maps_mma_sync_kernel_at_head_dim_80():
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_attention_maps as t; t._child_main()" % (ROOT, HERE)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, PB200_ATTN_MMA_SYNC="1"))
    assert r.returncode == 0, r.stderr[-3000:]
    kernels = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][0][8:])
    assert any("attention_kernel_maps" in k for k in kernels) and not any("wgmma" in k for k in kernels), kernels
    res = [json.loads(ln[4:]) for ln in r.stdout.splitlines() if ln.startswith("RES ")]
    assert len(res) == len(P_VALUES) and all(x["ok"] for x in res), res


# ------------------------------------------------------------------ 2. forward against the reference fixture
def _fixture_cases(dev):
    cfg, sd, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("attention_maps_tiny.npz")
    ci = t(g["clip_image"]).to(dev)
    cases = {"plain": (t(g["x"]), dict(clip_image=ci)),
             "attnw": (t(g["x"]), dict(clip_image=ci, attn_weights=t(g["attn_weights"]))),
             "x16": (t(z["x16"]), dict(clip_image=ci)),
             "img2": (t(g["x"]), dict(clip_image=[ci, t(z["clip_image2"]).to(dev)]))}
    return cfg, sd, g, z, cases


def _cpu(kw):
    return {k: ([x.cpu() for x in v] if isinstance(v, list) else v.cpu()) for k, v in kw.items()}


def test_forward_maps_match_reference_fixture(tiny):
    from oracle import attention_maps as om
    from oracle import paella_oracle as po
    cfg, sd, g, z, cases = _fixture_cases(DEV)
    r, byt5, clip = t(g["r"]), t(g["byt5"]), t(g["clip"])

    def mm16(a, w):         # fp16 operands and fp16 outputs: every rounding of the tensor-core path and more (a bound)
        return po.mm_f16_operands(a, w).half().float()
    for name, (x, kw) in cases.items():
        ref = t(z[f"maps_{name}"]).double()
        with torch.inference_mode():
            logits_m, maps = tiny(x.to(DEV), r.to(DEV), byt5.to(DEV), clip=clip.to(DEV), attention_maps=True, **kw)
            logits = tiny(x.to(DEV), r.to(DEV), byt5.to(DEV), clip=clip.to(DEV), **kw)
        assert torch.equal(logits_m, logits), name
        assert maps.dtype == torch.float32 and maps.device.type == "cuda" and tuple(maps.shape) == tuple(ref.shape)
        _, pred = om.paella_maps(sd, oracle_cfg(cfg), x, r, byt5, clip, mm=mm16, **_cpu(kw))
        d16 = float((pred - ref).abs().max())
        err = float((maps.cpu().double() - ref).abs().max())
        log_jsonl("attention_maps.jsonl", {"test": "forward", "case": name, "max_abs": err, "fp16_oracle_max_abs": d16})
        assert err <= 3.0 * d16 + 1e-5, (name, err, d16)
        # and the bound can see a wrong map: the weights move the maps by far more
        if name == "attnw":
            assert float((t(z["maps_attnw"]) - t(z["maps_plain"])).abs().max()) > 10 * (3.0 * d16 + 1e-5)


# ------------------------------------------------------------------ 3. sampling: nothing else changes
def _check_maps(maps, B, S, H, unweighted):
    assert maps.dtype == torch.float32 and tuple(maps.shape) == (B, S, H, H)
    assert bool((maps >= 0).all()) and bool(torch.isfinite(maps).all())
    for b in unweighted:
        assert float(maps[b].sum(0).max()) <= 1.0 + 1e-5


def test_sampling_with_maps_changes_nothing_else(tiny, tiny_vq):
    from paella_b200 import utils as U
    H, B, steps = 8, 5, 4
    cond, uncond = _conditioning(tiny, B, 12)
    S = 12 + 4
    tc, _ = _conditioning(tiny, 2, 6, seed=9)
    init = torch.randint(0, tiny.num_labels, (B, H, H), generator=torch.Generator().manual_seed(2))
    region = torch.ones(B, H, H, dtype=torch.bool)
    region[2, 1:H - 1, 2:H - 2] = False
    kw = dict(steps=steps, temperature=(1.2, 0.2), init_x=init, region=region,
              cfg=torch.tensor([[8.0, 6.0], [0.0, 0.0], [4.0, 4.0], [7.0, 2.0], [5.0, 5.0]], dtype=torch.float64),
              attn_weights=[torch.linspace(0.5, 2.0, 6), None, None, torch.full((3,), 1.5), None],
              tiling=["none", "xy", "none", "x", "none"], mode=["multinomial", "multinomial", "argmax", "quant", "multinomial"],
              guidance_prompts=[[(_rows(tc, slice(0, 1)), 0.5)], None, None, [(_rows(tc, slice(1, 2)), -0.5)], None],
              vqmodel=tiny_vq)
    seeds = [3, 14, 15, 92, 65]
    gens, gens_m = _gens(seeds), _gens(seeds)
    with torch.inference_mode():
        tok, inter = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=gens, **kw)
        tok_m, inter_m, maps = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=gens_m, attention_maps=True, **kw)
    assert torch.equal(tok, tok_m)
    assert len(inter) == len(inter_m) and all(torch.equal(a, b) for a, b in zip(inter, inter_m))
    assert [x.get_offset() for x in gens] == [x.get_offset() for x in gens_m]
    _check_maps(maps, B, S, H, unweighted=[1, 2, 4])
    # sample and sample_distributed
    dkw = dict(steps=3, temperature=(1.0, 0.3), tiling=["xy", "none", "none", "none", "none"],
               guidance_prompts=[None, [(_rows(tc, slice(0, 1)), 0.75)], None, None, None])
    for fn, args in ((U.sample, (tiny, cond, (B, H, H), uncond)), (U.sample_distributed, (tiny, cond, uncond, (B, H, H)))):
        g1, g2 = _gens(seeds), _gens(seeds)
        extra = dict(cfg=torch.tensor([6.0, 3.0, 0.0, 2.0, 5.0])) if fn is U.sample else dict(region=region, init_x=init)
        with torch.inference_mode():
            a = fn(*args, generator=g1, **dkw, **extra)
            b, mb = fn(*args, generator=g2, attention_maps=True, **dkw, **extra)
        assert torch.equal(a, b), fn.__name__
        assert [x.get_offset() for x in g1] == [x.get_offset() for x in g2]
        _check_maps(mb, B, S, H, unweighted=range(B))
    # the default generator path too
    torch.manual_seed(4)
    a = U.sample(tiny, cond, (B, H, H), uncond, steps=2)
    off = torch.cuda.default_generators[0].get_offset()
    torch.manual_seed(4)
    b, _ = U.sample(tiny, cond, (B, H, H), uncond, steps=2, attention_maps=True)
    assert torch.equal(a, b) and torch.cuda.default_generators[0].get_offset() == off


def test_notebook_maps_are_the_mean_of_forward_maps(tiny):
    from paella_b200 import utils as U
    H, B, steps = 8, 2, 3
    cond, uncond = _conditioning(tiny, B, 9, seed=3)
    init = torch.randint(0, tiny.num_labels, (B, H, H), generator=torch.Generator().manual_seed(6))
    aw = torch.linspace(0.5, 1.5, 5)
    with torch.inference_mode():
        _, inter, maps = U.sample_notebook(tiny, cond, (B, H, H), uncond, init_x=init, steps=steps, cfg=(6.0, 3.0),
                                           attn_weights=aw, generator=_gens([1, 2]), attention_maps=True)
        t_list = torch.linspace(1.0, 0.0, steps + 1)
        acc = 0
        for i in range(steps):
            x = init.to(DEV) if i == 0 else inter[2 * i - 1]
            r = torch.full((B,), float(t_list[i]), dtype=torch.float32, device=DEV)
            _, mi = tiny(x, r, cond["byt5"], clip=cond["clip"], attn_weights=aw, attention_maps=True)
            acc = acc + mi.double()
    want = acc / steps
    err = float((maps.double() - want).abs().max())
    log_jsonl("attention_maps.jsonl", {"test": "notebook_mean", "max_abs": err})
    torch.testing.assert_close(maps.double(), want, rtol=1e-5, atol=1e-8)


# ------------------------------------------------------------------ 4. batch invariance
def _rows_equal_batch1(m, H, steps, seeds):
    from paella_b200 import utils as U
    B = len(seeds)
    cond, uncond = _conditioning(m, B, 10, seed=31)
    tc, _ = _conditioning(m, 1, 5, seed=32)
    cfg = torch.tensor([[7.0, 3.0], [0.0, 0.0], [5.0, 5.0]], dtype=torch.float64)[:B]
    aw = [torch.linspace(0.5, 2.0, 4), None, None][:B]
    tiling = ["x", "none", "xy"][:B]
    terms = [None, None, [(tc, 0.5)]][:B]
    kw = dict(steps=steps, temperature=(1.1, 0.3))
    with torch.inference_mode():
        _, _, maps = U.sample_notebook(m, cond, (B, H, H), uncond, cfg=cfg, attn_weights=aw, tiling=tiling, guidance_prompts=terms,
                                       generator=_gens(seeds), attention_maps=True, **kw)
        for i in range(B):
            _, _, want = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)),
                                           cfg=cfg[i:i + 1], attn_weights=[aw[i]], tiling=tiling[i], guidance_prompts=[terms[i]],
                                           generator=_gens([seeds[i]]), attention_maps=True, **kw)
            assert torch.equal(maps[i:i + 1], want), i


@pytest.mark.parametrize("invariant", [False, True], ids=["default-mode", "batch-invariant"])
def test_tiny_rows_equal_batch1_calls(tiny, invariant):
    old = tiny.batch_invariant
    tiny.batch_invariant = invariant
    try:
        _rows_equal_batch1(tiny, 8, 3, [5, 6, 7])
    finally:
        tiny.batch_invariant = old


def test_default_model_batch_invariant_rows(default_model):
    _rows_equal_batch1(default_model, 16, 2, [8, 80, 800])


# ------------------------------------------------------------------ 5. engine
def _engine_equals_batch1(m, H):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    lens = [12, 7, 12, 9, 7, 12]
    conds = [_conditioning(m, 1, L, seed=40 + i) for i, L in enumerate(lens)]
    tc, _ = _conditioning(m, 2, 6, seed=49)
    kinds = [dict(attention_maps=True, guidance_prompts=[(_rows(tc, slice(0, 1)), 0.5)]),
             dict(),
             dict(attention_maps=True, mode="argmax", tiling="xy"),
             dict(attention_maps=True, attn_weights=torch.linspace(0.5, 2.0, 5), sampling_conditional_steps=1),
             dict(guidance_prompts=[(_rows(tc, slice(1, 2)), -0.5)]),
             dict(attention_maps=True, cfg=None)]
    steps = [3, 4, 2, 3, 4, 2]
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=3, max_cond_len=40, max_guidance_prompts=1)
    assert eng.map_acc is None
    reqs = []
    for i, kw in enumerate(kinds):
        g = torch.Generator(device=DEV).manual_seed(90 + i)
        cond, uncond = conds[i]
        reqs.append((eng.submit(cond, uncond, generator=g, steps=steps[i], temperature=(1.2, 0.2), keep_intermediates=True, **kw),
                     g, kw))
        if i % 2:
            eng.step()                # staggered arrivals; max_batch 3 reuses slots and their accumulators
    eng.run_until_idle()
    for i, (q, g, kw) in enumerate(reqs):
        kw = dict(kw)
        want_maps = kw.pop("attention_maps", False)
        if "guidance_prompts" in kw:
            kw["guidance_prompts"] = [kw["guidance_prompts"]]
        cond, uncond = conds[i]
        g1 = torch.Generator(device=DEV).manual_seed(90 + i)
        out = U.sample_notebook(m, cond, (1, H, H), uncond, steps=steps[i], temperature=(1.2, 0.2), generator=[g1],
                                attention_maps=want_maps, **kw)
        assert torch.equal(q.result, out[0]), i
        assert all(torch.equal(a, b) for a, b in zip(q.intermediates, out[1])), i
        assert g.get_offset() == g1.get_offset(), i
        if want_maps:
            assert q.attention_maps.shape == (lens[i] + 4, H, H)
            assert torch.equal(q.attention_maps, out[2][0]), i
        else:
            assert q.attention_maps is None


def test_engine_maps_equal_batch1_notebook(tiny):
    _engine_equals_batch1(tiny, 8)


def test_default_model_engine_maps(default_model):
    _engine_equals_batch1(default_model, 16)


def test_engine_validation(tiny):
    from paella_b200.engine import SamplingEngine
    eng = SamplingEngine(tiny, latent_hw=(8, 8), max_batch=2, max_cond_len=40, max_prompt_regions=1)
    cond, uncond = _conditioning(tiny, 1, 12)
    g = torch.Generator(device=DEV).manual_seed(1)
    off = g.get_offset()
    left = torch.zeros(8, 8, dtype=torch.bool)
    left[:, :4] = True
    for bad in (dict(attention_maps="yes"), dict(attention_maps=1), dict(attention_maps=True, prompt_regions=[(cond, left)])):
        with pytest.raises(ValueError):
            eng.submit(cond, uncond, generator=g, **bad)
    assert not eng.busy and g.get_offset() == off and eng.map_acc is None
    # a regional request and a maps request share a batch; the maps row equals its batch-1 call
    from paella_b200 import utils as U
    g1, g2 = torch.Generator(device=DEV).manual_seed(3), torch.Generator(device=DEV).manual_seed(4)
    a = eng.submit(cond, uncond, generator=g1, steps=2, attention_maps=True)
    eng.submit(cond, uncond, generator=g2, steps=2, prompt_regions=[(cond, left)])
    eng.run_until_idle()
    _, _, want = U.sample_notebook(tiny, cond, (1, 8, 8), uncond, steps=2, generator=_gens([3]), attention_maps=True)
    assert torch.equal(a.attention_maps, want[0])


# ------------------------------------------------------------------ 7. the plain path
def _kernel_names(f):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_plain_call_launches_no_maps_kernel(tiny):
    from paella_b200 import utils as U
    cond, uncond = _conditioning(tiny, 2, 12)
    # warm-up, the profiler's own included: a first profiled window can miss the launches at its start
    _kernel_names(lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([1, 2])))
    plain = _kernel_names(lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([1, 2])))
    off = _kernel_names(lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([1, 2]), attention_maps=False))
    maps = _kernel_names(lambda: U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([1, 2]), attention_maps=True))
    assert collections.Counter(plain) == collections.Counter(off)
    assert not any("maps" in n for n in plain)
    assert any("attention_maps_accumulate" in n for n in maps) and any("attention_maps_finalize" in n for n in maps)
    assert any("_maps" in n and "attention" in n and "accumulate" not in n and "finalize" not in n for n in maps)
