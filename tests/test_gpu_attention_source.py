"""Prompt-to-prompt injection on the GPU.

  1. Kernels: the inject instances of both attention kernels (pb200_attention_inject) at head dims 16/32/64/96 (mma.sync), 80
     (wgmma) and 80 on the mma.sync kernel (a PB200_ATTN_MMA_SYNC=1 child, as in test_gpu_attention_maps.py): ragged query counts,
     kv_len < S_max, a slot shared by an edit and its source, an edit on a slot of its own, a per-sample weight table.  An edit's O
     equals the plain instance's on inputs whose edit rows hold the source's Q and K, bit for bit, and fp64 within a bound; src = b
     is the plain instance bit for bit; injected rows next to regional and maps rows equal the regional-maps instance on the
     rewritten inputs, maps included.
  2. Forward: Paella.forward(..., attention_source=) on the tiny model against the reference fixture; rows that are not
     injected equal the call without it bit for bit, and features(inject=[0, 1]) is the plain forward bit for bit.
  3. Sampling: every k = 0 is the call without attention_source (tokens, intermediates, generator offsets); sources and other
     rows are unchanged bit for bit; an edit on its source's prompt and seed returns the source's tokens for any k.
  4. Batch invariance and composition: a pair placed anywhere in a mixed batch (guidance prompts, tiling, a region, modes,
     truncation, maps), or in a shard, equals the batch-2 call on the pair (tiny model; default model with batch_invariant);
     an engine pair equals the batch-2 sample_notebook call.
  5. A call without injection launches no inject kernel, and k = 0 launches the kernels of the call without attention_source.
"""
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
P_VALUES = (1, 63, 65, 200)
KV_SLOT = (3, 1, 3, 0)                 # samples 0 and 2 share slot 3
INJ = (-1, -1, 0, 1)                   # sample 2 replays sample 0 (same slot), sample 3 sample 1 (slot 0 holds its own values)
W_LD, W_LEN, W_ROW = 4, (2, 0, 3), (2, 0, 1, 0)     # every sample weighted by a table row (row 1 is empty)


def _p(x):
    return ctypes.c_void_p(x.data_ptr()) if x is not None else None


def _inputs(hd, P, rot):
    g = torch.Generator(device=DEV).manual_seed(100 * P + hd)
    B, H = len(KV_SLOT), 2
    E = H * hd
    n_a, n_b = (1, 64, 65, 129)[rot % 4], (63, 129, 1, 64)[rot % 4]
    lens = [n_b, n_b, 70, n_a]              # slot 0 (sample 3) and slot 1 (its source) hold the same count
    S = max(lens) + 3
    qkv = (torch.randn(B * P, 3 * E, device=DEV, generator=g) * 0.5).half()
    ckv = (torch.randn(len(lens), S, 2 * E, device=DEV, generator=g) * 0.5).half()
    w = (torch.rand(3, W_LD, device=DEV, generator=g) * 1.5 + 0.25).float()
    return dict(B=B, H=H, E=E, P=P, S=S, lens=lens, qkv=qkv, ckv=ckv, w=w)


def _rewritten(c, inj):
    """qkv and ckv whose edit rows hold their source's Q and self K, and whose edit slots their source slot's K."""
    qkv, ckv = c["qkv"].clone(), c["ckv"].clone()
    P, E = c["P"], c["E"]
    for b, a in enumerate(inj):
        if a >= 0:
            qkv[b * P:(b + 1) * P, :2 * E] = c["qkv"][a * P:(a + 1) * P, :2 * E]
            ckv[KV_SLOT[b], :, :E] = c["ckv"][KV_SLOT[a], :, :E]
    return qkv, ckv


def _run(c, qkv, ckv, inj=None, regional=None, maps=None):
    """pb200_attention_inject -> out fp16 [B*P, E] (and the maps scores, lse2 when ``maps``)."""
    from paella_b200 import _lib
    L = _lib.lib()
    B, P, S, E, H = c["B"], c["P"], c["S"], c["E"], c["H"]
    out = torch.full((B * P, E), float("nan"), dtype=torch.float16, device=DEV)
    kv_len = torch.tensor(c["lens"], dtype=torch.int32, device=DEV)
    kv_slot = torch.tensor(KV_SLOT, dtype=torch.int32, device=DEV)
    w_len = torch.tensor(W_LEN, dtype=torch.int32, device=DEV)
    w_row = torch.tensor(W_ROW, dtype=torch.int32, device=DEV)
    inj_d = torch.tensor(inj, dtype=torch.int32, device=DEV) if inj is not None else None
    q_mask = region_slot = None
    if regional is not None:
        q_mask, region_slot = regional
    scores = lse2 = map_row = None
    if maps is not None:
        map_row = torch.tensor(maps, dtype=torch.int32, device=DEV)
        scores = torch.full((B, H, P, S), float("nan"), device=DEV)
        lse2 = torch.full((B, H, P), float("nan"), device=DEV)
    rc = L.pb200_attention_inject(_p(qkv), _p(ckv), _p(kv_len), _p(kv_slot), len(c["lens"]), _p(out), B, P, S, E, H, 1, _p(c["w"]), 0,
                                  W_LD, _p(w_len), _p(w_row), B, _p(q_mask), _p(region_slot), None,
                                  region_slot.shape[1] if region_slot is not None else 0, B if q_mask is not None else 0,
                                  _p(scores), _p(lse2), _p(map_row), B if maps is not None else 0, _p(inj_d),
                                  len(inj) if inj is not None else 0, _lib.current_stream())
    assert rc == 0, L.pb200_last_error()
    torch.cuda.synchronize()
    return out, scores, lse2


def _fp64(c, b, a):
    """O of sample b replaying sample a, in fp64: (softmax(scale q_a [k_a]^T) * w_b) [v_b]."""
    P, E, H = c["P"], c["E"], c["H"]
    hd = E // H
    n = c["lens"][KV_SLOT[b]]
    qa, qb = c["qkv"][a * P:(a + 1) * P].double(), c["qkv"][b * P:(b + 1) * P].double()
    q = qa[:, :E].view(P, H, hd).transpose(0, 1)
    k = torch.cat([qa[:, E:2 * E], c["ckv"][KV_SLOT[a], :n, :E].double()]).view(P + n, H, hd).transpose(0, 1)
    v = torch.cat([qb[:, 2 * E:], c["ckv"][KV_SLOT[b], :n, E:].double()]).view(P + n, H, hd).transpose(0, 1)
    p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(hd), -1)
    wl = W_LEN[W_ROW[b]]
    if wl:                                  # the last wl keys; a vector longer than the key list is read from its tail
        p[..., max(0, P + n - wl):] *= c["w"][W_ROW[b], max(0, wl - P - n):wl].double()
    return (p @ v).transpose(0, 1).reshape(P, E), v.abs().max()


def _kernel_case(hd, P, rot):
    """One case; returns its worst error ratio, raises AssertionError on a failed check."""
    c = _inputs(hd, P, rot)
    out, _, _ = _run(c, c["qkv"], c["ckv"], INJ)
    q2, c2 = _rewritten(c, INJ)
    want, _, _ = _run(c, q2, c2)
    assert torch.equal(out.view(torch.int16), want.view(torch.int16)), "edit rows differ from the rewritten plain call"
    plain, _, _ = _run(c, c["qkv"], c["ckv"])
    for b, a in enumerate(INJ):
        if a < 0:
            assert torch.equal(out[b * c["P"]:(b + 1) * c["P"]].view(torch.int16), plain[b * c["P"]:(b + 1) * c["P"]].view(torch.int16))
    same, _, _ = _run(c, c["qkv"], c["ckv"], list(range(c["B"])))
    assert torch.equal(same.view(torch.int16), plain.view(torch.int16)), "src = b differs from the plain instance"
    worst = 0.0
    for b, a in enumerate(INJ):
        ref, vmax = _fp64(c, b, a if a >= 0 else b)
        # fp16 P and O with fp32 accumulation: a few 2^-11 of max |v| times the weights' sum (< 2)
        bound = 4e-3 * float(vmax)
        err = float((out[b * c["P"]:(b + 1) * c["P"]].double() - ref).abs().max())
        worst = max(worst, err / bound)
        assert err <= bound, (b, err, bound)
    return worst


def _mixed_case(hd, P):
    """Injected rows next to a regional row and map rows: the regional-maps inject instance on (qkv, ckv) equals the
    regional-maps instance on the rewritten inputs, O and maps."""
    c = _inputs(hd, P, 1)
    inj = (-1, -1, 0, -1)                   # sample 2 replays sample 0; sample 1 is regional
    mask = torch.ones(c["B"], P, dtype=torch.uint8, device=DEV)
    mask[1, ::3] = 2                        # every third query of sample 1 sees region 1 (slot 2) alone
    mask[1, 1::3] = 3
    region_slot = torch.full((c["B"], 1), -1, dtype=torch.int32, device=DEV)
    region_slot[1, 0] = 2
    maps = (0, -1, 2, 3)
    out, sc, ls = _run(c, c["qkv"], c["ckv"], inj, (mask, region_slot), maps)
    q2, c2 = _rewritten(c, inj)
    want, sc2, ls2 = _run(c, q2, c2, None, (mask, region_slot), maps)
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))
    assert torch.equal(sc.nan_to_num(7.0), sc2.nan_to_num(7.0)) and torch.equal(ls.nan_to_num(7.0), ls2.nan_to_num(7.0))


KERNEL_CASES = [(hd, P, i) for hd in (16, 32, 64, 80, 96) for i, P in enumerate(P_VALUES)]


@pytest.mark.parametrize("hd,P,rot", KERNEL_CASES, ids=[f"hd{hd}-P{P}" for hd, P, _ in KERNEL_CASES])
def test_inject_kernel(hd, P, rot):
    worst = _kernel_case(hd, P, rot)
    log_jsonl("attention_source.jsonl", {"test": "kernel", "hd": hd, "P": P, "worst_ratio": worst})


@pytest.mark.parametrize("hd", (16, 64, 80, 96))
def test_inject_next_to_regional_and_maps_rows(hd):
    for P in (63, 200):
        _mixed_case(hd, P)


def _child_main():
    """Runs in a PB200_ATTN_MMA_SYNC=1 child: every head_dim-80 case on the mma.sync kernel."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _kernel_case(80, 65, 0)
        torch.cuda.synchronize()
    print("KERNELS", json.dumps(sorted({e.name for e in prof.events() if "attention" in e.name})), flush=True)
    for i, P in enumerate(P_VALUES):
        try:
            _kernel_case(80, P, i)
            _mixed_case(80, P)
            print("RES", json.dumps({"P": P, "ok": True}), flush=True)
        except Exception as e:
            print("RES", json.dumps({"P": P, "ok": False, "msg": f"{type(e).__name__}: {e}"}), flush=True)


def test_inject_mma_sync_kernel_at_head_dim_80():
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_attention_source as t; t._child_main()" % (ROOT, HERE)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, PB200_ATTN_MMA_SYNC="1"))
    assert r.returncode == 0, r.stderr[-3000:]
    kernels = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][0][8:])
    assert any("attention_kernel_inject" in k for k in kernels) and not any("wgmma" in k for k in kernels), kernels
    res = [json.loads(ln[4:]) for ln in r.stdout.splitlines() if ln.startswith("RES ")]
    assert len(res) == len(P_VALUES) and all(x["ok"] for x in res), res


# ------------------------------------------------------------------ 2. forward against the reference fixture
def test_forward_matches_reference_fixture(tiny):
    from oracle import attention_source as osrc
    from oracle import paella_oracle as po
    cfg, sd, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("attention_source_tiny.npz")
    own = (t(g["byt5"]), t(g["clip"]), t(g["clip_image"]))
    same = (t(z["same_byt5"]), t(z["same_clip"]), t(z["same_clip_image"]))
    aw = t(g["attn_weights"])
    r = t(g["r"])

    def mm16(a, w):         # fp16 operands and outputs: every rounding of the tensor-core path and more (a bound)
        return po.mm_f16_operands(a, w).half().float()
    cases = {"prompt": (t(g["x"]), own, None), "attnw": (t(g["x"]), same, [None, aw]), "x16": (t(z["x16"]), own, None)}
    for name, (x, cond, w) in cases.items():
        ref = t(z[f"logits_{name}"]).double()
        args = (x.to(DEV), r.to(DEV), cond[0].to(DEV))
        kw = dict(clip=cond[1].to(DEV), clip_image=cond[2].to(DEV), attn_weights=w)
        with torch.inference_mode():
            got = tiny(*args, attention_source=[None, 0], **kw)
            plain = tiny(*args, **kw)
        assert torch.equal(got[0], plain[0]), name            # the source row is untouched
        pred = osrc.paella_forward_injected(sd, oracle_cfg(cfg), x, r, *cond, src=[None, 0], attn_weights=w, mm=mm16)
        d16 = float((pred.double() - ref).abs().max())
        err = float((got.cpu().double() - ref).abs().max())
        log_jsonl("attention_source.jsonl", {"test": "forward", "case": name, "max_abs": err, "fp16_oracle_max_abs": d16})
        assert err <= 3.0 * d16 + 1e-3, (name, err, d16)
        # the bound can see a missing injection: the edit row moves by far more
        assert float((plain[1].cpu().double() - ref[1]).abs().max()) > 10 * (3.0 * d16 + 1e-3), name
    # each sample its own source: the plain forward, bit for bit (features with inject = [0, 1])
    from paella_b200 import ops
    x = t(g["x"]).to(DEV)
    with torch.inference_mode():
        cond = tiny._cond_for_forward(*(v.to(DEV) for v in own), (8, 8))
        f_self = tiny.features(x, r.to(DEV), cond, inject=ops.to_device_async(torch.tensor([0, 1], dtype=torch.int32), DEV))
        f_plain = tiny.features(x, r.to(DEV), cond)
    assert torch.equal(f_self, f_plain)


# ------------------------------------------------------------------ 3. sampling
def test_k0_is_the_call_without_and_other_rows_are_unchanged(tiny):
    from paella_b200 import utils as U
    H, B, steps = 8, 4, 4
    cond, uncond = _conditioning(tiny, B, 10)
    seeds = [3, 3, 15, 92]
    kw = dict(steps=steps, temperature=(1.2, 0.2))
    with torch.inference_mode():
        g0 = _gens(seeds)
        tok0, inter0 = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=g0, **kw)
        g1 = _gens(seeds)
        tok1, inter1 = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=g1, attention_source=[None, (0, 0), None, (2, 0)], **kw)
        g2 = _gens(seeds)
        tok2, inter2 = U.sample_notebook(tiny, cond, (B, H, H), uncond, generator=g2, attention_source=[None, (0, 3), None, None], **kw)
    assert torch.equal(tok0, tok1) and all(torch.equal(a, b) for a, b in zip(inter0, inter1))
    assert [g.get_offset() for g in g0] == [g.get_offset() for g in g1] == [g.get_offset() for g in g2]
    for b in (0, 2, 3):
        assert torch.equal(tok2[b], tok0[b]) and all(torch.equal(a[b], c[b]) for a, c in zip(inter2, inter0))
    assert not torch.equal(tok2[1], tok0[1])


@pytest.mark.parametrize("k", [1, 3, 6])
def test_same_prompt_same_seed_returns_the_source(tiny, k):
    from paella_b200 import utils as U
    H, steps = 8, 6
    cond, uncond = _conditioning(tiny, 1, 9)
    cond2 = {key: torch.cat([v, v]) for key, v in cond.items()}
    uncond2 = {key: torch.cat([v, v]) for key, v in uncond.items()}
    with torch.inference_mode():
        tok = U.sample(tiny, cond2, (2, H, H), uncond2, steps=steps, generator=_gens([11, 11]), attention_source=[None, (0, k)])
    assert torch.equal(tok[0], tok[1])


def _pair_kw(tiny, n_extra):
    """Per-sample settings for [source, edit] and n_extra plain rows, with every feature the pair composes with."""
    tc, _ = _conditioning(tiny, 2, 6, seed=9)
    B = 2 + n_extra
    H = 8
    init = torch.randint(0, tiny.num_labels, (B, H, H), generator=torch.Generator().manual_seed(2))
    region = torch.ones(B, H, H, dtype=torch.bool)
    region[1, 1:5, 2:6] = False
    return dict(steps=5, temperature=torch.tensor([[1.2, 0.2]] * B), init_x=init, region=region,
                cfg=torch.tensor([[6.0, 3.0], [5.0, 5.0]] + [[4.0, 2.0]] * n_extra, dtype=torch.float64),
                tiling=["xy", "x"] + ["none"] * n_extra, mode=["multinomial", "multinomial"] + ["argmax"] * n_extra,
                sampling_quant_steps=[3, None] + [None] * n_extra, top_k=torch.tensor([0, 20] + [0] * n_extra),
                guidance_prompts=[None, [(_rows(tc, slice(0, 1)), 0.5)]] + [None] * n_extra,
                attn_weights=[None, torch.linspace(0.5, 1.5, 4)] + [None] * n_extra)


def _permute(kw, idx):
    out = {}
    for key, v in kw.items():
        if torch.is_tensor(v) and key not in ("steps",):
            out[key] = v[idx]
        elif isinstance(v, list):
            out[key] = [v[i] for i in idx]
        else:
            out[key] = v
    return out


def test_pair_anywhere_in_a_mixed_batch_equals_the_pair_alone(tiny, tiny_vq):
    from paella_b200 import utils as U
    H = 8
    cond, uncond = _conditioning(tiny, 5, 10)
    kw = _pair_kw(tiny, 3)
    seeds = [21, 21, 4, 5, 6]
    # the pair alone, rows [source, edit]; then the pair at rows 3 (source) and 1 (edit) of five
    with torch.inference_mode():
        tok2, inter2, maps2 = U.sample_notebook(tiny, _rows(cond, slice(0, 2)), (2, H, H), _rows(uncond, slice(0, 2)),
                                                generator=_gens(seeds[:2]), vqmodel=tiny_vq, attention_maps=True,
                                                attention_source=[None, (0, 3)], **_permute(kw, [0, 1]))
        idx = [2, 1, 3, 0, 4]              # batch row j holds pair/settings row idx[j]
        ckw = _permute(kw, idx)
        tok5, inter5, maps5 = U.sample_notebook(tiny, _rows(cond, idx), (5, H, H), _rows(uncond, idx),
                                                generator=_gens([seeds[i] for i in idx]), vqmodel=tiny_vq, attention_maps=True,
                                                attention_source=[None, (3, 3), None, None, None], **ckw)
        tok_plain, _ = U.sample_notebook(tiny, _rows(cond, slice(0, 2)), (2, H, H), _rows(uncond, slice(0, 2)),
                                         generator=_gens(seeds[:2]), vqmodel=tiny_vq, **_permute(kw, [0, 1]))
    for pair_row, batch_row in ((0, 3), (1, 1)):
        assert torch.equal(tok2[pair_row], tok5[batch_row])
        assert all(torch.equal(a[pair_row], b[batch_row]) for a, b in zip(inter2, inter5))
        assert torch.equal(maps2[pair_row], maps5[batch_row])
    assert torch.equal(tok_plain[0], tok2[0]) and not torch.equal(tok_plain[1], tok2[1])
    # a shard: rows [2, 4) of a distributed call hold the pair, indices relative to the shard
    skw = dict(steps=4, temperature=(1.0, 0.3), tiling=["none", "none", "xy", "x"])
    full_src = [None, None, None, (2, 2)]
    with torch.inference_mode():
        full = U.sample_distributed(tiny, _rows(cond, slice(0, 4)), _rows(uncond, slice(0, 4)), (4, H, H), generator=_gens([1, 2, 3, 3]),
                                    attention_source=full_src, **skw)
        shard = U.sample_distributed(tiny, _rows(cond, slice(2, 4)), _rows(uncond, slice(2, 4)), (2, H, H), generator=_gens([3, 3]),
                                     attention_source=[None, (0, 2)], **dict(skw, tiling=skw["tiling"][2:]))
    assert torch.equal(full[2:], shard)


def test_default_model_pair_is_batch_invariant(default_model):
    from paella_b200 import utils as U
    m = default_model
    H = 16
    cond, uncond = _conditioning(m, 3, 20)
    kw = dict(steps=2, temperature=(1.0, 0.3))
    with torch.inference_mode():
        alone = U.sample_notebook(m, _rows(cond, slice(0, 2)), (2, H, H), _rows(uncond, slice(0, 2)), generator=_gens([7, 7]),
                                  attention_source=[None, (0, 2)], **kw)[0]
        idx = [2, 1, 0]
        mixed = U.sample_notebook(m, _rows(cond, idx), (3, H, H), _rows(uncond, idx), generator=_gens([9, 7, 7]),
                                  attention_source=[None, (2, 2), None], **kw)[0]
    assert torch.equal(alone[0], mixed[2]) and torch.equal(alone[1], mixed[1])


def test_engine_pair_equals_the_batch2_call(tiny):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    H = 8
    cond, uncond = _conditioning(tiny, 4, 10)
    eng = SamplingEngine(tiny, latent_hw=(H, H), max_batch=4, max_cond_len=32)
    kw = dict(steps=4, temperature=(1.1, 0.3), cfg=(6.0, 4.0))
    with torch.inference_mode():
        other = eng.submit(_rows(cond, slice(2, 3)), _rows(uncond, slice(2, 3)), generator=_gens([5])[0], **dict(kw, steps=3))
        eng.step()
        src = eng.submit(_rows(cond, slice(0, 1)), _rows(uncond, slice(0, 1)), generator=_gens([8])[0], **kw)
        edit = eng.submit(_rows(cond, slice(1, 2)), _rows(uncond, slice(1, 2)), generator=_gens([8])[0], attention_source=(src, 2),
                          keep_intermediates=True, **kw)
        late = eng.submit(_rows(cond, slice(3, 4)), None, generator=_gens([6])[0], cfg=None, steps=2)
        eng.run_until_idle()
        want, inter = U.sample_notebook(tiny, _rows(cond, slice(0, 2)), (2, H, H), _rows(uncond, slice(0, 2)), generator=_gens([8, 8]),
                                        attention_source=[None, (0, 2)], **kw)
    assert torch.equal(src.result[0], want[0]) and torch.equal(edit.result[0], want[1])
    assert all(torch.equal(a[0], b[1]) for a, b in zip(edit.intermediates, inter))
    assert other.done and late.done


# ------------------------------------------------------------------ 5. launches
def _attention_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_launches(tiny):
    from paella_b200 import utils as U
    H = 8
    cond, uncond = _conditioning(tiny, 2, 10)

    def run(src):
        with torch.inference_mode():
            U.sample(tiny, cond, (2, H, H), uncond, steps=3, generator=_gens([1, 1]), attention_source=src)
    run(None)
    plain = _attention_kernels(lambda: run(None))
    k0 = _attention_kernels(lambda: run([None, (0, 0)]))
    inj = _attention_kernels(lambda: run([None, (0, 2)]))
    assert not any("inject" in k for k in plain)
    assert k0 == plain
    assert any("inject" in k for k in inj)
