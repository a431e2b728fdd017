"""Seamless tiling on the GPU.

  1. Kernels: the denoiser's depthwise conv + LayerNorm (pb200_dwconv_ln_tiled) with every wrap code mixed in one launch, in
     process (default dispatch) and in child processes that force the 2x8-patch kernel (PB200_DWCONV_PATCH=1) or the warp kernel
     (PB200_DWCONV_WARP=1): each sample against an fp64 mod-n reference, against its own single-sample launch bit for bit, and
     byte-0 samples against the untiled launch bit for bit.
  2. Decoder: the tiny codec (three-launch ResBlock front) and the default-size codec (fused front) against the circular oracle
     and the reference fixture; decode(roll(tokens, (a, b))) == roll(decode(tokens), (4a, 4b)) bit for bit; every row of a
     mixed batch equals its own decode, and an untiled row the plain decode.
  3. Denoiser: tiled logits of the tiny model against the reference fixture; rolling the tokens by the deepest stride rolls
     the logits.
  4. Per sample and per request: mixed-tiling batches through sample_notebook / sample_distributed equal their batch-1 calls
     (tiny model; default model with batch_invariant = True), and a staggered SamplingEngine load equals batch-1 calls.
  5. No behaviour change: tiling=None and all-'none' calls equal the calls without the argument.
"""
import json
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
CODES = {0: "none", 1: "x", 2: "y", 3: "xy"}


def _log(payload):
    log_jsonl("tiling.jsonl", payload)


def _gens(seeds):
    return [torch.Generator(device=DEV).manual_seed(s) for s in seeds]


def _rows(d, idx):
    return {k: (v[idx] if torch.is_tensor(v) else v) for k, v in d.items()}


# ------------------------------------------------------------------ 1. depthwise conv + LayerNorm kernels
DW_CASES = [(c, h, w, skip, 3) for c in (64, 640, 1280, 2560) for (h, w) in ((1, 1), (2, 2), (3, 5), (7, 9), (32, 32))
            for skip in (False, True)] + [(c, h, w, skip, 5) for c in (64, 640) for (h, w) in ((1, 1), (2, 2), (7, 9))
                                          for skip in (False, True)]
DW_WRAP = [0, 1, 2, 3, 3, 0]          # every code mixed in one launch, two byte-0 samples


def _dw_id(case):
    c, h, w, skip, k = case
    return f"c{c}-{h}x{w}-k{k}-{'skip' if skip else 'noskip'}"


def _dw_launch(x, skip, wp, b, k, wrap):
    from paella_b200._lib import check, current_stream, lib, ptr
    B, h, w, c = x.shape
    out = torch.empty(B * h * w, c, dtype=torch.float16, device=DEV)
    if wrap is None:
        check(lib().pb200_dwconv_ln(ptr(x), ptr(skip), ptr(wp), ptr(b), B, h, w, c, k, ptr(out), current_stream()))
    else:
        check(lib().pb200_dwconv_ln_tiled(ptr(x), ptr(skip), ptr(wp), ptr(b), B, h, w, c, k, ptr(wrap), ptr(out), current_stream()))
    return out.view(B, h, w, c)


def _dw_case(case):
    """Max |error| against fp64, and whether the bit-equality checks hold."""
    from oracle import paella_oracle as po
    from oracle import tiling as ot
    c, h, w, skip, k = case
    g = torch.Generator(device=DEV).manual_seed(c + 7 * h + w + k)
    B, per = len(DW_WRAP), 2 if skip else 1
    x = torch.randn(B, h, w, c, device=DEV, generator=g)
    xs = torch.randn(B, h, w, c, device=DEV, generator=g) if skip else None
    W = torch.randn(c, per, k, k, device=DEV, generator=g) / k
    b = torch.randn(c, device=DEV, generator=g) * 0.2
    wp = W.permute(2, 3, 1, 0).reshape(k * k, per, c).contiguous()
    wrap = torch.tensor(DW_WRAP, dtype=torch.uint8, device=DEV)
    got = _dw_launch(x, xs, wp, b, k, wrap)
    plain = _dw_launch(x, xs, wp, b, k, None)
    err, bits = 0.0, True
    for i, code in enumerate(DW_WRAP):
        flags = (bool(code & 1), bool(code & 2))
        d = ot.dwconv_nhwc(x[i:i + 1].double(), W.double(), b.double(), xs[i:i + 1].double() if skip else None, flags)
        err = max(err, float((got[i:i + 1].double() - po.ln(d)).abs().max()))
        one = _dw_launch(x[i:i + 1].contiguous(), xs[i:i + 1].contiguous() if skip else None, wp, b, k, wrap[i:i + 1])
        bits &= torch.equal(one, got[i:i + 1])
        if code == 0:
            bits &= torch.equal(got[i], plain[i])
    return err, bits


def _dw_child_main():
    for case in DW_CASES:
        try:
            err, bits = _dw_case(case)
            print("RES", json.dumps({"id": _dw_id(case), "ok": True, "err": err, "bits": bits}), flush=True)
        except Exception as e:
            print("RES", json.dumps({"id": _dw_id(case), "ok": False, "msg": f"{type(e).__name__}: {e}"}), flush=True)


_DW_CHILD = {}
DW_KERNELS = {"default": {}, "patch": {"PB200_DWCONV_PATCH": "1"}, "warp": {"PB200_DWCONV_WARP": "1"}}


@pytest.mark.parametrize("kernel", list(DW_KERNELS))
@pytest.mark.parametrize("case", DW_CASES, ids=_dw_id)
def test_dwconv_wrap_against_fp64_and_bits(kernel, case):
    if kernel == "default":
        err, bits = _dw_case(case)
    else:
        if kernel not in _DW_CHILD:
            code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_tiling as t; t._dw_child_main()" % (ROOT, HERE)
            r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **DW_KERNELS[kernel]))
            res = {}
            for line in r.stdout.splitlines():
                if line.startswith("RES "):
                    j = json.loads(line[4:])
                    res[j["id"]] = j
            _DW_CHILD[kernel] = (r.returncode, r.stderr[-3000:], res)
        rc, stderr, res = _DW_CHILD[kernel]
        r = res.get(_dw_id(case))
        assert r is not None, f"child rc {rc}: {stderr}"
        assert r["ok"], r["msg"]
        err, bits = r["err"], r["bits"]
    _log({"test": "dwconv_wrap", "kernel": kernel, "case": _dw_id(case), "max_abs": err, "bits": bits})
    assert bits
    assert err < 1.6e-2, err           # fp16 output of unit-scale LayerNorm values (|y| <= ~5: half an ulp is 2e-3)


# ------------------------------------------------------------------ 2. decoder
@pytest.fixture(scope="module")
def tiny_vq():
    from paella_b200.vqgan import VQModel
    cfg, sd, g = load_golden("vqgan_tiny.npz")
    m = VQModel(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m, cfg, sd


@pytest.fixture(scope="module")
def default_vq():
    from paella_b200.synth import rerandomize_
    from paella_b200.vqgan import VQModel
    torch.manual_seed(0)
    m = VQModel().eval()
    rerandomize_(m.state_dict(), seed=4)
    sd = {k: v.detach().clone().float() for k, v in m.state_dict().items()}
    return m.to(DEV), sd


def _roll_checks(m, idx):
    img = m.decode_indices(idx, tiling="xy")
    for a, b in ((1, 0), (0, 3), (2, 5), (idx.shape[1] - 1, 1)):
        rolled = m.decode_indices(torch.roll(idx, (a, b), (1, 2)), tiling="xy")
        assert torch.equal(rolled, torch.roll(img, (4 * a, 4 * b), (2, 3))), (a, b)
    return img


def _mixed_rows(m, idx):
    codes = ["none", "x", "y", "xy"]
    batch = idx[[i % idx.shape[0] for i in range(4)]]
    got = m.decode_indices_u8(batch, codes)
    for i, name in enumerate(codes):
        assert torch.equal(got[i:i + 1], m.decode_indices_u8(batch[i:i + 1], name)), name
    assert torch.equal(got[0:1], m.decode_indices_u8(batch[0:1]))
    assert torch.equal(m.decode_indices(batch, ["none"] * 4), m.decode_indices(batch))
    assert torch.equal(m.decode_indices(batch, None), m.decode_indices(batch))


def test_tiny_decoder_tiled(tiny_vq):
    from oracle import tiling as ot
    m, cfg, sd = tiny_vq
    _, _, z = load_golden("tiling_tiny.npz")
    idx = t(z["idx"]).to(DEV)
    for name in ("xy", "x"):
        got = m.decode_indices(idx, tiling=name).cpu()
        err = float((got - t(z["dec_" + name])).abs().max())
        err_o = float((got - ot.decode_indices(sd, idx.cpu(), cfg["bottleneck_blocks"], wrap=ot.WRAPS[name])).abs().max())
        _log({"test": "tiny_decode", "tiling": name, "max_abs_ref": err, "max_abs_oracle": err_o})
        assert err < 5e-3 and err_o < 5e-3, (name, err, err_o)
    for shape in ((2, 4, 4), (3, 1, 1), (2, 3, 5)):
        ids = torch.randint(0, cfg["codebook_size"], shape, generator=torch.Generator().manual_seed(sum(shape))).to(DEV)
        _roll_checks(m, ids)
        _mixed_rows(m, ids)


def test_default_decoder_tiled(default_vq):
    from oracle import tiling as ot
    m, sd = default_vq
    idx = torch.randint(0, 8192, (2, 16, 16), generator=torch.Generator().manual_seed(8))
    img = _roll_checks(m, idx.to(DEV))
    want = ot.decode_indices(sd, idx[:1], 12, wrap=(True, True))
    err = float((img[:1].cpu() - want).abs().max())
    _log({"test": "default_decode", "max_abs_oracle": err, "scale": float(want.abs().max())})
    assert err < 2e-2 * max(1.0, float(want.abs().max())), err
    _mixed_rows(m, idx[:, :8, :12].contiguous().to(DEV))
    big = torch.randint(0, 8192, (3, 32, 32), generator=torch.Generator().manual_seed(9)).to(DEV)
    _roll_checks(m, big)


# ------------------------------------------------------------------ 3. denoiser logits
@pytest.fixture(scope="module")
def tiny():
    from paella_b200.modules import Paella
    cfg, sd, _ = load_golden("paella_tiny.npz")
    m = Paella(**cfg).to(DEV).eval()
    m.load_state_dict(sd)
    return m


def test_tiny_denoiser_tiled_logits(tiny):
    from oracle import tiling as ot
    cfg, sd, g = load_golden("paella_tiny.npz")
    _, _, z = load_golden("tiling_tiny.npz")
    args = [t(g[k]).to(DEV) for k in ("x", "r", "byt5", "clip", "clip_image")]
    for name in ("xy", "x", "y"):
        got = tiny(args[0], args[1], args[2], clip=args[3], clip_image=args[4], tiling=name).cpu()
        err = float((got - t(z["logits_" + name])).abs().max())
        _log({"test": "tiny_logits", "tiling": name, "max_abs_ref": err})
        assert err < 7e-3, (name, err)
    # per-sample tiling: each row is its own call
    mixed = tiny(args[0], args[1], args[2], clip=args[3], clip_image=args[4], tiling=["x", "none"])
    assert torch.equal(mixed[:1], tiny(args[0][:1], args[1][:1], args[2][:1], clip=args[3][:1], clip_image=args[4][:1], tiling="x"))
    assert torch.equal(mixed[1:], tiny(args[0][1:], args[1][1:], args[2][1:], clip=args[3][1:], clip_image=args[4][1:]))
    # rolling the tokens by the deepest level's stride (8 tokens) rolls the logits; a 16 x 16 grid against the oracle too
    x16 = torch.randint(0, cfg["num_labels"], (2, 16, 16), generator=torch.Generator().manual_seed(4)).to(DEV)
    base = tiny(x16, args[1], args[2], clip=args[3], tiling="xy")
    want = ot.paella_forward(sd, oracle_cfg(cfg), x16.cpu(), args[1].cpu(), args[2].cpu(), args[3].cpu(), wrap=(True, True))
    assert float((base.cpu() - want).abs().max()) < 7e-3
    for a, b in ((8, 0), (0, 8), (8, 8)):
        rolled = tiny(torch.roll(x16, (a, b), (1, 2)), args[1], args[2], clip=args[3], tiling="xy")
        err = float((rolled - torch.roll(base, (a, b), (2, 3))).abs().max())
        _log({"test": "tiny_roll", "shift": [a, b], "max_abs": err})
        assert err < 7e-3, (a, b, err)


# ------------------------------------------------------------------ 4. per sample and per request
def _conditioning(m, B, L, seed=7):
    from paella_b200.synth import synthetic_conditioning
    return synthetic_conditioning(B, L, byt5_embd=m.byt5_mapper.in_features, clip_embd=m.clip_mapper.in_features,
                                  with_clip_image=False, seed=seed, device=DEV)


def _batch_rows_equal_batch1(m, B, H, steps, tilings, seeds, region_row=None):
    from paella_b200 import utils as U
    cond, uncond = _conditioning(m, B, 12)
    cfg = torch.tensor([[8.0, 6.0], [0.0, 0.0], [4.0, 4.0], [7.0, 2.0]][:B], dtype=torch.float64)
    init = torch.randint(0, m.num_labels, (B, H, H), generator=torch.Generator().manual_seed(2))
    region = torch.ones(B, H, H, dtype=torch.bool)
    if region_row is not None:
        region[region_row, 1:H - 1, 2:H - 2] = False
    gens = _gens(seeds)
    got, inter = U.sample_notebook(m, cond, (B, H, H), uncond, init_x=init, region=region, steps=steps, cfg=cfg,
                                   temperature=(1.2, 0.2), generator=gens, tiling=tilings)
    for i in range(B):
        g1 = _gens([seeds[i]])
        want, inter1 = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)),
                                         init_x=init[i:i + 1], region=region[i:i + 1], steps=steps, cfg=cfg[i:i + 1],
                                         temperature=(1.2, 0.2), generator=g1, tiling=tilings[i])
        assert torch.equal(got[i:i + 1], want), i
        assert all(torch.equal(a[i:i + 1], b) for a, b in zip(inter, inter1)), i
        assert g1[0].get_offset() == gens[i].get_offset(), i
    g2 = _gens(seeds[1:3])
    shard = U.sample_distributed(m, _rows(cond, slice(1, 3)), _rows(uncond, slice(1, 3)), (2, H, H), init_x=init[1:3],
                                 region=region[1:3], steps=steps, cfg=cfg[1:3], temperature=(1.2, 0.2), generator=g2,
                                 tiling=tilings[1:3])
    assert torch.equal(shard, got[1:3])
    return cond, uncond


def test_mixed_tiling_rows_equal_batch1_calls(tiny):
    from paella_b200 import utils as U
    cond, uncond = _batch_rows_equal_batch1(tiny, 4, 8, 4, ["none", "x", "y", "xy"], [3, 14, 15, 92], region_row=2)
    # tiling changes the tokens, and an untiled call is the call without the argument
    a = U.sample(tiny, cond, (4, 8, 8), uncond, steps=2, generator=_gens([1, 2, 3, 4]), tiling="xy")
    b = U.sample(tiny, cond, (4, 8, 8), uncond, steps=2, generator=_gens([1, 2, 3, 4]))
    c = U.sample(tiny, cond, (4, 8, 8), uncond, steps=2, generator=_gens([1, 2, 3, 4]), tiling=["none"] * 4)
    assert not torch.equal(a, b) and torch.equal(b, c)
    torch.manual_seed(5)
    d = U.sample(tiny, cond, (4, 8, 8), uncond, steps=2, tiling=None)
    torch.manual_seed(5)
    assert torch.equal(d, U.sample(tiny, cond, (4, 8, 8), uncond, steps=2))


def test_sample_decode_uses_each_rows_tiling(tiny, tiny_vq):
    from paella_b200 import utils as U
    vq = tiny_vq[0]
    cond, uncond = _conditioning(tiny, 2, 12)
    tilings = ["xy", "none"]
    toks = U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([5, 6]), tiling=tilings)
    imgs = U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=_gens([5, 6]), tiling=tilings, decode=vq)
    assert torch.equal(imgs, vq.decode_indices_u8(toks, tilings))


def test_engine_mixed_tiling_equals_batch1_notebook(tiny, tiny_vq):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    m, vq = tiny, tiny_vq[0]
    H = 8
    kinds = [dict(tiling="xy"), dict(), dict(tiling="x", cfg=None), dict(tiling="y", top_k=5), dict(tiling="xy", cfg=None),
             dict(tiling="x", decode=True)]
    steps = [3, 4, 2, 3, 4, 3]
    N = len(kinds)
    cond, uncond = _conditioning(m, N, 12, seed=21)
    eng = SamplingEngine(m, latent_hw=(H, H), max_batch=3, max_cond_len=40, vqmodel=vq)
    reqs = []
    for i, kw in enumerate(kinds):
        g = torch.Generator(device=DEV).manual_seed(70 + i)
        reqs.append((eng.submit(_rows(cond, slice(i, i + 1)), _rows(uncond, slice(i, i + 1)), generator=g, steps=steps[i],
                                temperature=(1.2, 0.2), keep_intermediates=True, **kw), g, kw))
        if i % 2:
            eng.step()                # staggered arrivals; max_batch 3 reuses slots
    eng.run_until_idle()
    for i, (q, g, kw) in enumerate(reqs):
        kw = dict(kw)
        decode = kw.pop("decode", False)
        g1 = torch.Generator(device=DEV).manual_seed(70 + i)
        want, inter = U.sample_notebook(m, _rows(cond, slice(i, i + 1)), (1, H, H), _rows(uncond, slice(i, i + 1)), steps=steps[i],
                                        temperature=(1.2, 0.2), generator=[g1], **kw)
        if decode:
            want = vq.decode_indices_u8(want, kw.get("tiling"))
        assert torch.equal(q.result, want), (i, kw)
        assert all(torch.equal(a, b) for a, b in zip(q.intermediates, inter)), i
        assert g.get_offset() == g1.get_offset(), i


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


def test_default_model_batch_invariant_tiling_rows(default_model):
    _batch_rows_equal_batch1(default_model, 4, 16, 3, ["xy", "none", "x", "y"], [8, 80, 800, 8000], region_row=1)


def test_validation_enqueues_nothing(tiny):
    from paella_b200 import utils as U
    from paella_b200.engine import SamplingEngine
    cond, uncond = _conditioning(tiny, 2, 12)
    gens = _gens([1, 2])
    offs = [g.get_offset() for g in gens]
    for bad in ("xz", ["x"], torch.tensor([1, 1])):
        with pytest.raises(ValueError):
            U.sample(tiny, cond, (2, 8, 8), uncond, steps=2, generator=gens, tiling=bad)
        with pytest.raises(ValueError):
            tiny(torch.zeros(2, 8, 8, dtype=torch.int64, device=DEV), torch.zeros(2, device=DEV), cond["byt5"], tiling=bad)
    assert [g.get_offset() for g in gens] == offs
    eng = SamplingEngine(tiny, latent_hw=(8, 8), max_batch=2, max_cond_len=40)
    for bad in ("q", ["x"], torch.tensor([1])):
        with pytest.raises(ValueError):
            eng.submit(_rows(cond, slice(0, 1)), _rows(uncond, slice(0, 1)), generator=gens[0], tiling=bad)
    assert not eng.busy
