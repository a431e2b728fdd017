"""GPU parity of the reference's building-block classes called ON THEIR OWN (ref/src/modules.py:7-106):
paella_b200.modules.{ResBlock, AttnBlock, Attention2D, FeedForwardBlock, TimestepBlock, LayerNorm2d,
GlobalResponseNorm}.forward against the CPU oracle's restatement of the same blocks (fp32), same weights.

Tolerance: fp16 GEMM operands / fp16 storage of the MLP hidden and q,k,v (as in the model path) on O(1)
activations: 2e-2 max-abs, 4e-3 rms; the GEMM-free blocks (LayerNorm2d, GlobalResponseNorm) 1e-5.
"""
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _log(name, payload):
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "block_parity.jsonl"), "a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


def _errs(got, want):
    d = got.float().cpu() - want.float().cpu()
    return float(d.abs().max()), float(d.pow(2).mean().sqrt())


def _randomise(mod, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in mod.named_parameters():
            if n.endswith("gamma") or n.endswith("beta") or "bias" in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2)
            else:
                p.copy_(torch.randn(p.shape, generator=g) / (p[0].numel() ** 0.5))
    return mod


def _sd(mod, pre):
    return {pre + k: v.detach().float().cpu() for k, v in mod.state_dict().items()}


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def _nchw(x):
    return x.permute(0, 3, 1, 2).contiguous()


@pytest.mark.parametrize("c,skip,hw,B", [(64, False, 8, 3), (64, True, 8, 2), (1280, True, 8, 2), (640, False, 16, 2), (96, False, 5, 2)])
def test_resblock_standalone(c, skip, hw, B):
    from oracle import paella_oracle as po
    from paella_b200.modules import ResBlock
    blk = _randomise(ResBlock(c, c if skip else None), 1).eval()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B, c, hw, hw, generator=g)
    xs = torch.randn(B, c, hw, hw, generator=g) if skip else None
    want = _nchw(po.resblock(_nhwc(x), _sd(blk, "b."), "b.", _nhwc(xs) if skip else None))
    blk = blk.to(DEV)
    got = blk(x.to(DEV), xs.to(DEV) if skip else None)
    assert got.shape == x.shape and got.dtype == torch.float32
    mx, rms = _errs(got, want)
    _log("resblock", {"c": c, "skip": skip, "hw": hw, "max_abs": mx, "rms": rms})
    assert mx < 6e-3 and rms < 1.2e-3, (mx, rms)


def test_feedforward_standalone():
    from oracle import paella_oracle as po
    from paella_b200.modules import FeedForwardBlock
    blk = _randomise(FeedForwardBlock(128), 3).eval()
    x = torch.randn(2, 128, 8, 8, generator=torch.Generator().manual_seed(4))
    want = _nchw(po.feedforward_block(_nhwc(x), _sd(blk, "b."), "b."))
    got = blk.to(DEV)(x.to(DEV))
    mx, rms = _errs(got, want)
    _log("feedforward", {"max_abs": mx, "rms": rms})
    assert mx < 6e-3 and rms < 1.2e-3, (mx, rms)


def test_timestep_standalone():
    from oracle import paella_oracle as po
    from paella_b200.modules import TimestepBlock
    blk = _randomise(TimestepBlock(96, 64), 5).eval()
    g = torch.Generator().manual_seed(6)
    x, t = torch.randn(3, 96, 6, 6, generator=g), torch.randn(3, 64, generator=g)
    want = _nchw(po.timestep_block(_nhwc(x), t, _sd(blk, "b."), "b."))
    got = blk.to(DEV)(x.to(DEV), t.to(DEV))
    mx, rms = _errs(got, want)
    _log("timestep", {"max_abs": mx, "rms": rms})
    assert mx < 6e-3 and rms < 1.2e-3, (mx, rms)


@pytest.mark.parametrize("c,nhead,hw,S,self_attn,weighted", [(64, 4, 4, 9, True, False), (1280, 16, 8, 132, True, False),
                                                              (1280, 16, 4, 132, True, True), (128, 4, 8, 20, False, False)])
def test_attnblock_standalone(c, nhead, hw, S, self_attn, weighted):
    from oracle import paella_oracle as po
    from paella_b200.modules import AttnBlock
    c_cond = 96
    blk = _randomise(AttnBlock(c, c_cond, nhead, self_attn=self_attn), 7).eval()
    g = torch.Generator().manual_seed(8)
    x, kv = torch.randn(2, c, hw, hw, generator=g), torch.randn(2, S, c_cond, generator=g)
    aw = torch.rand(5, generator=g) * 2 if weighted else None
    want = _nchw(po.attn_block(_nhwc(x), kv, _sd(blk, "b."), "b.", nhead, self_attn, attn_weights=aw))
    blk = blk.to(DEV)
    got = blk(x.to(DEV), kv.to(DEV), **({"attn_weights": aw.to(DEV)} if weighted else {}))
    mx, rms = _errs(got, want)
    _log("attnblock", {"c": c, "hw": hw, "S": S, "self_attn": self_attn, "weighted": weighted, "max_abs": mx, "rms": rms})
    assert mx < 2.5e-3 and rms < 6e-4, (mx, rms)


def test_attention2d_standalone():
    """Attention2D = nn.MultiheadAttention over [self ; kv] tokens, no norm, no residual (ref/src/modules.py:12-19)."""
    from paella_b200.modules import Attention2D
    c, nhead = 128, 4
    blk = _randomise(Attention2D(c, nhead), 9).eval()
    g = torch.Generator().manual_seed(10)
    x, kv = torch.randn(2, c, 4, 4, generator=g) * 0.5, torch.randn(2, 11, c, generator=g) * 0.5
    for self_attn in (False, True):
        with torch.no_grad():       # the holder IS a torch nn.MultiheadAttention: its CPU forward is the reference op
            xt = x.view(2, c, -1).permute(0, 2, 1)
            kvs = torch.cat([xt, kv], dim=1) if self_attn else kv
            want = blk.attn(xt, kvs, kvs, need_weights=False)[0].permute(0, 2, 1).reshape(x.shape)
        got = Attention2D.forward(blk.to(DEV), x.to(DEV), kv.to(DEV), self_attn=self_attn)
        blk = blk.cpu()
        mx, rms = _errs(got, want)
        _log("attention2d", {"self_attn": self_attn, "max_abs": mx, "rms": rms})
        assert mx < 1.4e-3 and rms < 3e-4, (mx, rms)


@pytest.mark.parametrize("affine,eps", [(False, 1e-6), (True, 1e-5)])
def test_layernorm2d_standalone(affine, eps):
    from paella_b200.modules import LayerNorm2d
    ln = LayerNorm2d(48, elementwise_affine=affine, eps=eps)
    if affine:
        _randomise(ln, 11)
    x = torch.randn(2, 48, 5, 7, generator=torch.Generator().manual_seed(12)) * 3 + 1
    with torch.no_grad():
        want = torch.nn.functional.layer_norm(x.permute(0, 2, 3, 1), (48,), ln.weight, ln.bias, eps).permute(0, 3, 1, 2)
    got = ln.to(DEV)(x.to(DEV))
    mx, _ = _errs(got, want)
    assert got.shape == x.shape and mx < 1e-5, mx


def test_grn_standalone():
    from oracle import paella_oracle as po
    from paella_b200.modules import GlobalResponseNorm
    grn = _randomise(GlobalResponseNorm(40), 13)
    x = torch.randn(3, 6, 5, 40, generator=torch.Generator().manual_seed(14))
    want = po.grn(x, grn.gamma.detach().view(-1), grn.beta.detach().view(-1))
    got = grn.to(DEV)(x.to(DEV))
    mx, _ = _errs(got, want)
    assert got.shape == x.shape and mx < 1e-5, mx
