"""Kernels chosen by a dispatcher, each run on every shape whichever variant the dispatcher would pick.

Depthwise conv + LayerNorm (launch_dwconv_ln): ResBlock on its own against the CPU oracle, in-process (default dispatch: the
2x8-patch kernel for c > 640 and w >= 8, the warp kernel otherwise) and in child processes with PB200_DWCONV_PATCH=1 (patch
kernel everywhere) and PB200_DWCONV_WARP=1 (warp kernel everywhere).  Grids with ragged 2x8 patches, channel counts that leave
idle threads, and the c in (1280, 2560] instantiation.

Fused sampler (launch_fused_sampler): the shared-Philox kernel (default) and the generic per-element kernel
(PB200_SAMPLER_GENERIC=1, child process), against torch.multinomial on the same seed, plus a margin audit: every token the
kernel picks scores, in fp64 on the same Exp(1) draws, within an a-priori margin of the row's best Gumbel score.
"""
import json
import math
import os
import subprocess
import sys
import tempfile

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _log(payload):
    from helpers import log_jsonl
    log_jsonl("dispatch_variants.jsonl", payload)


def _child(env, call):
    """Run `call` (an expression over this module, `t`) in a child with `env`; returns the RES lines' JSON."""
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_dispatch_variants as t; %s" % (ROOT, HERE, call)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **env))
    res = {}
    for line in r.stdout.splitlines():
        if line.startswith("RES "):
            j = json.loads(line[4:])
            res[j["id"]] = j
    return r.returncode, r.stderr[-3000:], res


# ------------------------------------------------------------------ depthwise conv through ResBlock
DW_CASES = [(c, h, w, skip) for c in (640, 1280, 2560, 1000) for (h, w) in ((10, 10), (12, 9), (9, 16), (3, 8))
            for skip in (False, True)]
DW_KERNELS = {"default": {}, "patch": {"PB200_DWCONV_PATCH": "1"}, "warp": {"PB200_DWCONV_WARP": "1"}}


def _dw_id(case):
    c, h, w, skip = case
    return f"c{c}-{h}x{w}-{'skip' if skip else 'noskip'}"


def _randomise(mod, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in mod.named_parameters():
            if n.endswith("gamma") or n.endswith("beta") or "bias" in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.2)
            else:
                p.copy_(torch.randn(p.shape, generator=g) / (p[0].numel() ** 0.5))
    return mod


def _dw_inputs(case):
    from paella_b200.modules import ResBlock
    c, h, w, skip = case
    blk = _randomise(ResBlock(c, c if skip else None), c + h).eval()
    g = torch.Generator().manual_seed(h * 31 + w)
    x = torch.randn(2, c, h, w, generator=g)
    xs = torch.randn(2, c, h, w, generator=g) if skip else None
    return blk, x, xs


def _dw_oracle(path):
    """The oracle's ResBlock for every case (NCHW), computed once for all three kernels."""
    from oracle import paella_oracle as po
    want = {}
    for case in DW_CASES:
        blk, x, xs = _dw_inputs(case)
        sd = {"b." + k: v.detach().float() for k, v in blk.state_dict().items()}
        nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous()          # noqa: E731  (h != w: a general NHWC view)
        want[_dw_id(case)] = po.resblock(nhwc(x), sd, "b.", nhwc(xs) if xs is not None else None).permute(0, 3, 1, 2).contiguous()
    torch.save(want, path)


def _dw_run(case, want):
    blk, x, xs = _dw_inputs(case)
    got = blk.to(DEV)(x.to(DEV), xs.to(DEV) if xs is not None else None)
    assert got.shape == x.shape
    d = got.float().cpu() - want
    return float(d.abs().max()), float(d.pow(2).mean().sqrt())


def _dw_child_main(path):
    want = torch.load(path)
    for case in DW_CASES:
        try:
            mx, rms = _dw_run(case, want[_dw_id(case)])
            print("RES", json.dumps({"id": _dw_id(case), "ok": True, "max_abs": mx, "rms": rms}), flush=True)
        except Exception as e:
            print("RES", json.dumps({"id": _dw_id(case), "ok": False, "msg": f"{type(e).__name__}: {e}"}), flush=True)


@pytest.fixture(scope="module")
def dw_oracle():
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "dw_oracle.pt")
        _dw_oracle(path)
        yield path, torch.load(path)


_DW_CHILD = {}


@pytest.mark.parametrize("kernel", list(DW_KERNELS))
@pytest.mark.parametrize("case", DW_CASES, ids=_dw_id)
def test_resblock_dwconv_variant_vs_oracle(kernel, case, dw_oracle):
    path, want = dw_oracle
    if kernel == "default":
        mx, rms = _dw_run(case, want[_dw_id(case)])
    else:
        if kernel not in _DW_CHILD:
            _DW_CHILD[kernel] = _child(DW_KERNELS[kernel], "t._dw_child_main(%r)" % path)
        rc, err, res = _DW_CHILD[kernel]
        r = res.get(_dw_id(case))
        assert r is not None, f"child rc {rc}: {err}"
        assert r["ok"], r["msg"]
        mx, rms = r["max_abs"], r["rms"]
    _log({"test": "resblock_dwconv", "kernel": kernel, "case": _dw_id(case), "max_abs": mx, "rms": rms})
    assert mx < 6e-3 and rms < 1.2e-3, (mx, rms)


# ------------------------------------------------------------------ fused sampler
# (labels, batch, grid): the existing full-grid / small-grid / non-divisible-stride shapes, plus 5 x 27 x 27 = 3645 rows, which
# is not a multiple of 4 rs for any launch policy (odd)
SAMPLER_CASES = [(8192, 8, 32), (8192, 3, 8), (8200, 2, 16), (64, 2, 8), (8192, 64, 32), (8192, 5, 27)]


def _sampler_id(case):
    return "NL%d-B%d-H%d" % case


def _sampler_run(NL, B, H):
    """Agreement with torch.multinomial on the same seed and the fp64 margin audit, with and without guidance."""
    from paella_b200.modules import Paella
    from helpers import load_golden
    cfg, _, _ = load_golden("paella_tiny.npz")
    big = dict(cfg)
    big.update(c_in=256, c_out=256, num_labels=NL)
    torch.manual_seed(0)
    m = Paella(**big).to(DEV).eval()
    gen = torch.Generator(device=DEV).manual_seed(3)
    feats = torch.randn(2 * B * H * H, 256, device=DEV, generator=gen)
    W = m.out_mapper[1].weight.detach().view(NL, 256) * 30.0        # spread the logits
    with torch.no_grad():
        m.out_mapper[1].weight.copy_(W.view(NL, 256, 1, 1))
    m.pack_weights()
    n = B * H * H
    w16 = W.half()
    out = {}
    for guided, (cfg_s, T, seed) in ((True, (8.0, 0.7, 42)), (False, (None, 0.7, 43))):
        a16 = ((feats[:n] * cfg_s + feats[n:] * (1 - cfg_s)) if guided else feats[:n]).half()
        torch.manual_seed(seed)
        want = torch.multinomial(torch.softmax((a16.float() @ w16.float().t()) / T, dim=-1), 1)[:, 0]
        torch.manual_seed(seed)
        q = torch.empty(n, NL, device=DEV).exponential_(1)            # the draws torch.multinomial consumes
        off_a = torch.cuda.default_generators[0].get_offset()
        torch.manual_seed(seed)
        got = m.sample_tokens(feats if guided else feats[:n].contiguous(), B, H, H, cfg_s, T).view(-1)
        assert torch.cuda.default_generators[0].get_offset() == off_a
        agree = float((got == want).float().mean())
        # margin audit in fp64: score = l / T - log q.  The kernel's logit may differ from the fp64 one of the same fp16
        # operands by one fp16 ulp of the mixed operand (its own rounding of the CFG mix) plus fp32 accumulation; its score
        # by fp32 rounding of l / T and of log q.
        worst = 0.0
        a64, w64 = a16.double(), w16.double()
        for r0 in range(0, n, 1024):
            r1 = min(n, r0 + 1024)
            l = a64[r0:r1] @ w64.t()
            s_abs = a64[r0:r1].abs() @ w64.abs().t()
            lq = torch.log(q[r0:r1].double())
            score = l / T - lq
            best = score.max(1).values
            pick = score.gather(1, got[r0:r1, None])[:, 0]
            slack = (2.0 ** -10 + 256 * 2.0 ** -24) * s_abs.max(1).values / T
            margin = 2 * slack + 8 * 2.0 ** -24 * (l.abs().max(1).values / T + lq.abs().max(1).values)
            worst = max(worst, float(((best - pick) / margin).max()))
        out["guided" if guided else "unguided"] = {"agree": agree, "margin_ratio": worst, "mismatch": int((got != want).sum())}
    return out


def _sampler_child_main():
    for case in SAMPLER_CASES:
        try:
            print("RES", json.dumps({"id": _sampler_id(case), "ok": True, "res": _sampler_run(*case)}), flush=True)
        except Exception as e:
            print("RES", json.dumps({"id": _sampler_id(case), "ok": False, "msg": f"{type(e).__name__}: {e}"}), flush=True)


_SAMPLER_CHILD = {}


@pytest.mark.parametrize("kernel", ["default", "generic"])
@pytest.mark.parametrize("case", SAMPLER_CASES, ids=_sampler_id)
def test_fused_sampler_variant_agreement_and_margin(kernel, case):
    if kernel == "default":
        res = _sampler_run(*case)
    else:
        if "generic" not in _SAMPLER_CHILD:
            _SAMPLER_CHILD["generic"] = _child({"PB200_SAMPLER_GENERIC": "1"}, "t._sampler_child_main()")
        rc, err, all_res = _SAMPLER_CHILD["generic"]
        r = all_res.get(_sampler_id(case))
        assert r is not None, f"child rc {rc}: {err}"
        assert r["ok"], r["msg"]
        res = r["res"]
    _log({"test": "fused_sampler", "kernel": kernel, "case": _sampler_id(case), **res})
    for k, v in res.items():
        assert v["agree"] >= 0.999, (k, v)
        assert v["margin_ratio"] <= 1.0, (k, v)       # every pick is a near-tie of the row's best at worst
