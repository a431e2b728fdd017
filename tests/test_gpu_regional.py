"""Regional prompts through the denoiser and the sampling functions on the GPU.

  1. Tiny-model logits with regional prompts against the reference fixture (regional_tiny.npz), at 8 x 8 and 16 x 16.
  2. Degenerate regions, bit for bit: one region over the whole grid is the plain call on that region's prompt (default model,
     head_dim 80), and regions that cover no token are the plain call on the base prompt (default and tiny model).
  3. Per sample: each row of a sample_notebook batch mixing regional, plain, inpainting, tiled and truncated rows equals its
     batch-1 call, generator offsets included, and a sample_distributed shard equals its rows (tiny model; default model with
     batch_invariant = True).
  4. Validation raises ValueError before anything is enqueued or any generator advances.
  5. SamplingEngine: with staggered arrivals and slot reuse, each regional, plain or decoded request's result, intermediates and
     generator offset equal its batch-1 sample_notebook call (tiny model; default model with batch_invariant = True); an engine
     without regional prompts allocates the cache it allocated before; its validation enqueues nothing.
"""
import pytest
import torch

from helpers import load_golden, log_jsonl, t

pytestmark = pytest.mark.gpu
DEV = "cuda"


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
def default_model():
    from paella_b200.modules import Paella
    from paella_b200.synth import rerandomize_
    torch.manual_seed(0)
    m = Paella(byt5_embd=2560).eval()
    rerandomize_(m.state_dict(), seed=0)
    m = m.to(DEV)
    m.batch_invariant = True
    return m


# ------------------------------------------------------------------ 1. logits against the reference
def test_tiny_regional_logits_match_reference(tiny):
    _, _, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("regional_tiny.npz")
    r, byt5, clip, ci = (t(g[k]).to(DEV) for k in ("r", "byt5", "clip", "clip_image"))
    rp = [[{key: t(z[f"rp{b}{k}_{key}"]) for key in ("byt5", "clip", "clip_image") if f"rp{b}{k}_{key}" in z} for k in range(2)]
          for b in range(2)]
    for n, x in ((8, t(g["x"])), (16, t(z["x16"]))):
        regions = [[(rp[b][k], t(z[f"reg{n}_{b}{k}"])) for k in range(2)] for b in range(2)]
        got = tiny(x.to(DEV), r, byt5, clip=clip, clip_image=ci, prompt_regions=regions).cpu()
        err = float((got - t(z[f"logits_{n}"])).abs().max())
        log_jsonl("regional.jsonl", {"test": "tiny_logits", "hw": n, "max_abs_ref": err})
        assert err < 7e-3, (n, err)
        plain = tiny(x.to(DEV), r, byt5, clip=clip, clip_image=ci).cpu()
        assert float((plain - t(z[f"logits_{n}"])).abs().max()) > 1e-2      # the regions change the result


# ------------------------------------------------------------------ 2. degenerate regions
def _whole_and_empty(m, H, check_whole):
    from paella_b200 import utils as U
    cond, uncond = _conditioning(m, 2, 12)
    other, _ = _conditioning(m, 2, 9, seed=8)
    x = torch.randint(0, m.num_labels, (2, H, H), generator=torch.Generator().manual_seed(1)).to(DEV)
    r = torch.tensor([0.7, 0.3], device=DEV)
    full = torch.ones(H, H, dtype=torch.bool)
    empty = torch.zeros(H, H, dtype=torch.bool)
    p1 = _rows(other, slice(0, 1))
    # regions covering no token: the base prompt's call
    kw = dict(clip=cond["clip"])
    got = m(x, r, cond["byt5"], prompt_regions=[[(p1, empty)], [(p1, empty), (_rows(other, slice(1, 2)), empty)]], **kw)
    assert torch.equal(got, m(x, r, cond["byt5"], **kw))
    toks = U.sample(m, cond, (2, H, H), uncond, steps=3, generator=_gens([4, 5]), prompt_regions=[[(p1, empty)], None])
    assert torch.equal(toks, U.sample(m, cond, (2, H, H), uncond, steps=3, generator=_gens([4, 5])))
    if not check_whole:
        return
    # one region over the whole grid: the call whose conditioning is that region's prompt
    got = m(x[:1], r[:1], cond["byt5"][:1], clip=cond["clip"][:1], prompt_regions=[[(p1, full)]])
    assert torch.equal(got, m(x[:1], r[:1], p1["byt5"], clip=p1["clip"]))
    toks = U.sample(m, _rows(cond, slice(0, 1)), (1, H, H), _rows(uncond, slice(0, 1)), steps=3, generator=_gens([6]),
                    prompt_regions=[[(p1, full)]])
    assert torch.equal(toks, U.sample(m, p1, (1, H, H), _rows(uncond, slice(0, 1)), steps=3, generator=_gens([6])))


def test_default_model_degenerate_regions_are_plain_calls(default_model):
    _whole_and_empty(default_model, 16, True)


def test_tiny_model_uncovering_regions_are_plain_calls(tiny):
    _whole_and_empty(tiny, 8, False)


# ------------------------------------------------------------------ 3. per sample
def _mixed_rows_equal_batch1(m, H, steps, seeds):
    from paella_b200 import utils as U
    B = 5
    cond, uncond = _conditioning(m, B, 12)
    rc, _ = _conditioning(m, 3, 6, seed=9)
    rb, _ = _conditioning(m, 1, 10, seed=10)
    left = torch.zeros(H, H, dtype=torch.bool)
    left[:, :H // 2] = True
    top = torch.zeros(H, H, dtype=torch.bool)
    top[:H // 2] = True
    regions = [[(_rows(rc, slice(0, 1)), left), (_rows(rb, slice(0, 1)), top)],     # regional, overlapping, rest uncovered
               None,                                                                 # plain
               [(_rows(rc, slice(1, 2)), ~left)],                                    # regional + inpainting
               [(_rows(rc, slice(2, 3)), top)],                                      # regional + tiled + truncated
               None]                                                                 # tiled
    tilings = ["none", "none", "none", "xy", "x"]
    top_k = torch.tensor([0, 0, 0, 7, 0])
    cfg = torch.tensor([[8.0, 6.0], [0.0, 0.0], [4.0, 4.0], [7.0, 2.0], [5.0, 5.0]], dtype=torch.float64)
    init = torch.randint(0, m.num_labels, (B, H, H), generator=torch.Generator().manual_seed(2))
    region = torch.ones(B, H, H, dtype=torch.bool)
    region[2, 1:H - 1, 2:H - 2] = False
    gens = _gens(seeds)
    kw = dict(steps=steps, temperature=(1.2, 0.2))
    got, inter = U.sample_notebook(m, cond, (B, H, H), uncond, init_x=init, region=region, cfg=cfg, generator=gens, tiling=tilings,
                                   top_k=top_k, prompt_regions=regions, **kw)
    for i in range(B):
        g1 = _gens([seeds[i]])
        want, inter1 = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), init_x=init[i:i + 1],
                                         region=region[i:i + 1], cfg=cfg[i:i + 1], generator=g1, tiling=tilings[i],
                                         top_k=top_k[i:i + 1], prompt_regions=[regions[i]], **kw)
        assert torch.equal(got[i:i + 1], want), i
        assert all(torch.equal(a[i:i + 1], b) for a, b in zip(inter, inter1)), i
        assert g1[0].get_offset() == gens[i].get_offset(), i
    g2 = _gens(seeds[1:4])
    shard = U.sample_distributed(m, _rows(cond, slice(1, 4)), _rows(uncond, slice(1, 4)), (3, H, H), init_x=init[1:4],
                                 region=region[1:4], cfg=cfg[1:4], generator=g2, tiling=tilings[1:4], top_k=top_k[1:4],
                                 prompt_regions=regions[1:4], **kw)
    assert torch.equal(shard, got[1:4])
    # the regions change the regional rows
    plain, _ = U.sample_notebook(m, cond, (B, H, H), uncond, init_x=init, region=region, cfg=cfg, generator=_gens(seeds),
                                 tiling=tilings, top_k=top_k, **kw)
    assert not torch.equal(plain[0], got[0]) and torch.equal(plain[1], got[1])


def test_tiny_mixed_regional_rows_equal_batch1_calls(tiny):
    _mixed_rows_equal_batch1(tiny, 8, 4, [3, 14, 15, 92, 65])


def test_default_model_batch_invariant_regional_rows(default_model):
    _mixed_rows_equal_batch1(default_model, 16, 3, [8, 80, 800, 8000, 80000])


# ------------------------------------------------------------------ 4. validation
def test_validation_enqueues_nothing(tiny):
    from paella_b200 import utils as U
    cond, uncond = _conditioning(tiny, 2, 12)
    p = _rows(cond, slice(0, 1))
    ok = torch.ones(8, 8, dtype=torch.bool)
    gens = _gens([1, 2])
    offs = [g.get_offset() for g in gens]
    bad_values = [
        [(p, ok)],                                       # a list of pairs for the batch: ambiguous, refused
        [[(p, ok)]],                                     # wrong length
        "regions",
        [[(p, ok)] * 8, None],                           # more than 7 regions
        [[(p, ok.float())], None],                       # not bool
        [[(p, torch.ones(4, 8, dtype=torch.bool))], None],
        [[(cond, ok)], None],                            # batch-2 inputs
        [[(p,)], None],
    ]
    for bad in bad_values:
        with pytest.raises(ValueError):
            U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=gens, prompt_regions=bad)
        with pytest.raises(ValueError):
            U.sample_notebook(tiny, cond, (2, 8, 8), uncond, steps=2, generator=gens, prompt_regions=bad)
        with pytest.raises(ValueError):
            tiny(torch.zeros(2, 8, 8, dtype=torch.int64, device=DEV), torch.zeros(2, device=DEV), cond["byt5"], prompt_regions=bad)
    with pytest.raises(ValueError):      # regional prompts and attn_weights on one sample
        U.sample_notebook(tiny, cond, (2, 8, 8), uncond, steps=2, generator=gens, prompt_regions=[[(p, ok)], None],
                          attn_weights=[torch.ones(3), None])
    assert [g.get_offset() for g in gens] == offs


# ------------------------------------------------------------------ 5. engine
@pytest.fixture(scope="module")
def tiny_vq():
    from paella_b200.vqgan import VQModel
    cfg, sd, _ = load_golden("vqgan_tiny.npz")
    vq = VQModel(**cfg).to(DEV).eval()
    vq.load_state_dict(sd)
    return vq


def _engine_equals_batch1(m, H, vq=None):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    left = torch.zeros(H, H, dtype=torch.bool)
    left[:, :H // 2] = True
    top = torch.zeros(H, H, dtype=torch.bool)
    top[:H // 2] = True
    N = 6
    cond, uncond = _conditioning(m, N, 12, seed=21)
    rc, _ = _conditioning(m, 4, 6, seed=22)
    rb, _ = _conditioning(m, 1, 10, seed=23)
    kinds = [dict(prompt_regions=[(_rows(rc, slice(0, 1)), left), (_rows(rb, slice(0, 1)), top)]), dict(),
             dict(prompt_regions=[(_rows(rc, slice(1, 2)), ~left)], cfg=None), dict(prompt_regions=[(_rows(rc, slice(2, 3)), top)],
                                                                                  tiling="xy", top_k=5),
             dict(decode=True, prompt_regions=[(_rows(rc, slice(3, 4)), left)]), dict(tiling="x")]
    if vq is None:
        kinds[4].pop("decode")
    steps = [3, 4, 2, 3, 4, 3]
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=3, max_cond_len=40, vqmodel=vq, max_prompt_regions=2)
    reqs = []
    for i, kw in enumerate(kinds):
        g = torch.Generator(device=DEV).manual_seed(70 + i)
        reqs.append((eng.submit(_rows(cond, slice(i, i + 1)), _rows(uncond, slice(i, i + 1)), generator=g, steps=steps[i],
                                temperature=(1.2, 0.2), keep_intermediates=True, **kw), g, kw))
        if i % 2:
            eng.step()                # staggered arrivals; max_batch 3 reuses slots and their regional K/V slots
    eng.run_until_idle()
    for i, (q, g, kw) in enumerate(reqs):
        kw = dict(kw)
        decode = kw.pop("decode", False)
        if "prompt_regions" in kw:
            kw["prompt_regions"] = [kw["prompt_regions"]]
        g1 = torch.Generator(device=DEV).manual_seed(70 + i)
        want, inter = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), steps=steps[i],
                                        temperature=(1.2, 0.2), generator=[g1], **kw)
        if decode:
            want = vq.decode_indices_u8(want, kw.get("tiling"))
        assert torch.equal(q.result, want), (i, kw.keys())
        assert all(torch.equal(a, b) for a, b in zip(q.intermediates, inter)), i
        assert g.get_offset() == g1.get_offset(), i


def test_engine_regional_requests_equal_batch1_notebook(tiny, tiny_vq):
    _engine_equals_batch1(tiny, 8, tiny_vq)


def test_default_model_engine_regional_requests(default_model):
    _engine_equals_batch1(default_model, 16)


def test_engine_without_regions_allocates_as_before(tiny):
    from paella_b200._lib import lib
    from paella_b200.engine import SamplingEngine
    eng = SamplingEngine(tiny, latent_hw=(8, 8), max_batch=3, max_cond_len=40)
    assert eng.cache.cache.numel() == lib().pb200_paella_cond_cache_bytes(tiny._handle, 2 * 3 + 1, 40)
    assert not hasattr(eng, "prompt_mask")
    eng2 = SamplingEngine(tiny, latent_hw=(8, 8), max_batch=3, max_cond_len=40, max_prompt_regions=2)
    assert eng2.cache.cache.numel() == lib().pb200_paella_cond_cache_bytes(tiny._handle, 2 * 3 + 1 + 2 * 3, 40)


def test_engine_validation_enqueues_nothing(tiny):
    from paella_b200.engine import SamplingEngine
    cond, uncond = _conditioning(tiny, 1, 12)
    long, _ = _conditioning(tiny, 1, 40, seed=3)
    ok = torch.ones(8, 8, dtype=torch.bool)
    for bad in (-1, 8, 1.5, True):
        with pytest.raises(ValueError):
            SamplingEngine(tiny, latent_hw=(8, 8), max_batch=2, max_cond_len=60, max_prompt_regions=bad)
    eng = SamplingEngine(tiny, latent_hw=(8, 8), max_batch=2, max_cond_len=40, max_prompt_regions=2)
    g = torch.Generator(device=DEV).manual_seed(1)
    off = g.get_offset()
    bad_values = [
        [(cond, ok)] * 3,                                 # more than max_prompt_regions
        (cond, ok),                                       # a bare pair
        [(cond, ok.float())],
        [(cond, torch.ones(8, 4, dtype=torch.bool))],
        [({"byt5": torch.randn(2, 3, cond["byt5"].shape[2], device=DEV)}, ok)],
        [(long, ok)],                                     # longer than max_cond_len
        "left",
    ]
    for bad in bad_values:
        with pytest.raises(ValueError):
            eng.submit(cond, uncond, generator=g, prompt_regions=bad)
    with pytest.raises(ValueError):
        eng.submit(cond, uncond, generator=g, prompt_regions=[(cond, ok)], attn_weights=torch.ones(3))
    plain = SamplingEngine(tiny, latent_hw=(8, 8), max_batch=2, max_cond_len=40)
    with pytest.raises(ValueError):
        plain.submit(cond, uncond, generator=g, prompt_regions=[(cond, ok)])
    assert not eng.busy and not plain.busy and g.get_offset() == off
