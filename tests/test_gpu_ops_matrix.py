"""Every memory-bound denoiser kernel of ops.cu and blocks.cu against an fp64 reference, at every instantiation.

The LayerNorm, depthwise-conv, GRN, FiLM, embedding, cast and layout kernels run on every denoiser step, but the whole-model
fixtures only reach the tiny and default models' shapes, where a later LayerNorm or GEMM can absorb a small error.  Here
each kernel is called on its own through the C ABI (the block-level entries and the executor entries exposed for testing in
include/paella_b200.h).  Each case names the kernel instance it runs, restated in Python from the dispatch conditions in
ops.cu and blocks.cu (_dw_kernel, _grn_rows_per_cta, ...); test_ops_matrix_plan.py checks on the CPU that together the cases
cover every kernel of the two files that the library holds.

Every output lies inside a larger buffer prefilled with a sentinel bit pattern: every logical element must be written,
nothing outside it may change, and a second launch must give the same bits.  Every element is compared with fp64 arithmetic
on the same fp32 / fp16 inputs, within a bound derived for that element from the kernel's operation order:
    U = 2^-24 per fp32 rounding, D_LN = 40 for the depth of any LayerNorm reduction here, half an fp16 ulp per fp16 store.
The casts, pads, gathers, row copies, masks and transposes are exact and are compared bit for bit.

Each family plants a probe: the same reference with one plausible kernel bug (a one-pass variance, eps 1e-5, a dropped tap
or term, zero padding instead of wrap, swapped patch columns, a boundary off by one, ...), and the probe must move some
element by more than its bound.  One row per case goes to ops_matrix.jsonl in $PB200_TEST_LOG_DIR (helpers.log_jsonl), with
the worst error/bound ratio and the probe's ratio.  PB200_DWCONV_PATCH and PB200_DWCONV_WARP are read once per process, so
the depthwise cases also run in one child process per knob.

Out of scope, because other matrices check them: row_stats_kernel and vq_front_patch_kernel (test_gpu_vqgan_matrix.py), and
the attention-map accumulate / finalize kernels (test_gpu_attention_maps.py).
"""
import ctypes
import json
import math
import os
import subprocess
import sys
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# The bounds are a-priori, not calibrated.  Worst error/bound on an H100 80GB HBM3 (700 W power limit), all 341 cases in about
# a minute: 0.98-1.0 wherever the output is fp16 (the half-ulp store term itself: LayerNorms, embedding, depthwise, GRN,
# casts), 0.45 grn_f32, 0.43 film_apply, 0.41 guidance_mix, 0.28 r_embed, 0.13 film_table, 0 for the exact kernels.  The
# weakest probes there moved an element by 5.3x (one-pass variance) and 4.1x (SiLU, cast<3> boundary) its bound.
U = 2.0 ** -24
D_LN = 40
SM_H100 = 132         # the plan test restates the GRN rows-per-CTA rule at the H100's SM count
SENTINELS = {torch.float32: (torch.int32, 0x7FC0DEAD), torch.float16: (torch.int16, 0x7E5A), torch.int64: (torch.int64, 0x5EE55EE55EE55EE5),
             torch.uint8: (torch.uint8, 0xA5)}


def _log(payload):
    from helpers import log_jsonl
    log_jsonl("ops_matrix.jsonl", payload)


def _lib():
    from paella_b200 import _lib
    return _lib


def _rc(fn, *args):
    L = _lib()
    return getattr(L.lib(), fn)(*args)


def _call(fn, *args):
    L = _lib()
    L.check(_rc(fn, *args), fn)


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _st():
    return _lib().current_stream()


def _gen(tag):
    return torch.Generator().manual_seed(zlib.crc32(tag.encode()))


# ------------------------------------------------------------------ outputs with guard bands
class _Out:
    """n dense elements at offset `pre` inside a larger buffer prefilled with a sentinel bit pattern (optionally holding `init`
    in the logical range, for in-place kernels)."""

    def __init__(self, dtype, n, pre=16, init=None):
        itype, self.sent = SENTINELS[dtype]
        self.n, self.pre = n, pre
        self.buf = torch.empty(pre + n + 19, dtype=dtype, device=DEV)
        self.bits = self.buf.view(itype)
        self.bits.fill_(self.sent)
        if init is not None:
            self.buf[pre:pre + n] = init.reshape(-1).to(dtype)

    def ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + self.pre * self.buf.element_size())

    def value(self):
        return self.buf[self.pre:self.pre + self.n]

    def check(self, name, written=True):
        outside = torch.cat([self.bits[:self.pre], self.bits[self.pre + self.n:]])
        n_out = int((outside != self.sent).sum())
        assert n_out == 0, f"{name}: {n_out} elements outside the logical output changed"
        if written:
            n_in = int((self.bits[self.pre:self.pre + self.n] == self.sent).sum())
            assert n_in == 0, f"{name}: {n_in} logical elements were never written"


def _twice(name, dtype, n, launch, pre=16, init=None, written=True):
    """Launch into two sentinel buffers; both must hold the same bits.  Returns the logical output (on the device)."""
    outs = []
    for rep in range(2):
        o = _Out(dtype, n, pre=pre + 8 * rep, init=init)
        launch(o.ptr())
        torch.cuda.synchronize()
        o.check(name, written)
        outs.append(o)
    a, b = (o.bits[o.pre:o.pre + n] for o in outs)
    assert torch.equal(a, b), f"{name}: a second launch gave different bits in {int((a != b).sum())} elements"
    return outs[0].value().clone()


# ------------------------------------------------------------------ fp64 references and bounds
def _ulp16(a):
    e = torch.floor(torch.log2(a.clamp_min(2.0 ** -24))).clamp_min(-14)
    return torch.exp2(e - 10)


def _f16(ref, e):
    """An fp32 value within e of ref, stored as fp16 (round to nearest): within e + half an fp16 ulp."""
    return e + 0.5 * _ulp16(ref.abs() + e)


def _ln64(a, e_in=None, eps=1e-6):
    """fp64 LayerNorm over the last dim of a and the error bound of an fp32 two-pass kernel whose inputs carry e_in:
    the mean's rounding (D_LN U mean|a|) and the input error shift every row's mean and variance (E), which moves y by
    rstd (e_in + E) and rstd itself by E / sigma; the subtraction, product and rstd add (D_LN + 8) U |y|."""
    mean = a.mean(-1, keepdim=True)
    d = a - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    y = d * rstd
    ei = torch.zeros_like(a) if e_in is None else e_in
    E = D_LN * U * a.abs().mean(-1, keepdim=True) + ei.amax(-1, keepdim=True)
    bound = rstd * (ei + E) + y.abs() * (2 * rstd * E + (D_LN + 8) * U) + 2.0 ** -60
    return y, bound


def _ratio(got, ref, bound):
    return float(((got.double() - ref).abs() / bound).max())


def _probe(ref, bound, perturbed):
    return float(((perturbed - ref).abs() / bound).max())


def _report(family, case, kernel, got, ref, bound, probe_ref=None, **extra):
    assert bool(torch.isfinite(got.double()).all()), f"{case}: non-finite output"
    row = dict(family=family, case=case, kernel=kernel, ratio=_ratio(got, ref, bound), **extra)
    if probe_ref is not None:
        row["probe"] = _probe(ref, bound, probe_ref)
    _log(row)
    assert row["ratio"] <= 1.0, row
    if probe_ref is not None:
        assert row["probe"] > 1.0, f"{case}: the probe stays within the bound: {row}"
    return row


# ------------------------------------------------------------------ 1. LayerNorm over rows (ln_rows_kernel<false>)
LN_CASES = [dict(id=f"ln-c{c}-r{r}-{mode}", c=c, rows=r, mode=mode)
            for c in (4, 36, 260, 1284) for r in (13, 37) for mode in ("out16", "out32", "inplace", "affine16", "mean32")]


def _ln_rows_input(tag, rows, c):
    """Rows of four kinds: plain, |mean|/std = 1e3 (a one-pass E[x^2] - E[x]^2 fails), variance ~1e-6 (eps 1e-5 fails) and
    distinct values per column (a layout error moves an element by >= 2^-7)."""
    g = _gen(tag)
    x = torch.randn(rows, c, generator=g, dtype=torch.float64)
    for i in range(rows):
        k = i % 4
        if k == 1:
            x[i] = x[i] + 1e3 * (1 if i % 8 == 1 else -1)
        elif k == 2:
            x[i] = 0.75 + 1e-3 * x[i]
        elif k == 3:
            x[i] = torch.arange(c, dtype=torch.float64) * 2.0 ** -7 + 0.25 * x[i]
    return x.float()


@pytest.mark.parametrize("case", LN_CASES, ids=lambda c: c["id"])
def test_ln_rows(case):
    c, rows, mode = case["c"], case["rows"], case["mode"]
    x = _ln_rows_input(case["id"], rows, c)
    scale, shift = (1.75, -0.375) if mode == "affine16" else (1.0, 0.0)
    xd = x.to(DEV)
    if mode == "inplace":
        got = _twice(case["id"], torch.float32, rows * c,
                     lambda p: _call("pb200_ln_rows", p, rows, c, scale, shift, None, p, None, _st()), init=xd, written=False)
    elif mode in ("out32", "mean32"):
        means = []

        def run(p):
            m = _Out(torch.float32, rows) if mode == "mean32" else None
            _call("pb200_ln_rows", _p(xd), rows, c, scale, shift, None, p, m.ptr() if m else None, _st())
            if m:
                torch.cuda.synchronize()
                m.check("mean_out")
                means.append(m.value().clone())
        got = _twice(case["id"], torch.float32, rows * c, run)
    else:
        got = _twice(case["id"], torch.float16, rows * c,
                     lambda p: _call("pb200_ln_rows", _p(xd), rows, c, scale, shift, p, None, None, _st()))
    x64 = x.double()
    y, e = _ln64(x64)
    ref = y * scale + shift
    bound = abs(scale) * e + 2 * U * (ref.abs() + abs(shift))
    # probes: a one-pass fp32 variance, and eps 1e-5
    xf = x.double().float()
    m1 = xf.mean(-1, keepdim=True)
    v1 = ((xf * xf).mean(-1, keepdim=True) - m1 * m1).clamp_min(0)
    one_pass = ((xf - m1) / torch.sqrt(v1 + 1e-6)).double() * scale + shift
    eps5 = _ln64(x64, eps=1e-5)[0] * scale + shift
    if mode in ("out16", "affine16"):
        bound = _f16(ref, bound)
    got = got.view(rows, c).cpu()
    extra = dict(probe_eps=_probe(ref, bound, eps5))
    if mode == "mean32":
        assert torch.equal(means[0].view(torch.int32), means[1].view(torch.int32)), "mean_out: a second launch gave different bits"
        mg = means[0].cpu().double()
        mr = x64.mean(-1)
        extra["mean_ratio"] = float(((mg - mr).abs() / (D_LN * U * x64.abs().mean(-1) + 2.0 ** -60)).max())
        assert extra["mean_ratio"] <= 1.0, extra
    _report("ln_rows", case["id"], "ln_rows_kernel<0>", got, ref, bound, probe_ref=one_pass, **extra)
    assert extra["probe_eps"] > 1.0, extra


# ------------------------------------------------------------------ 2. LayerNorm + k2s2 im2col (ln_rows_kernel<true>)
PATCHIFY_CASES = [dict(id=f"lnp-b{b}-{h}x{w}-c{c}", b=b, h=h, w=w, c=c)
                  for (b, h, w, c) in ((1, 2, 2, 4), (2, 6, 10, 36), (3, 4, 8, 260), (1, 2, 14, 1284))]


def _patchify_ref(y, b, h, w, c, swap=False):
    """y [b, h, w, c] -> [b*(h/2)*(w/2), 4c], column (dy*2 + dx)*c + ch ((dx*2 + dy) with swap: the probe)."""
    t = y.view(b, h // 2, 2, w // 2, 2, c)
    t = t.permute(0, 1, 3, 4, 2, 5) if swap else t.permute(0, 1, 3, 2, 4, 5)
    return t.reshape(b * (h // 2) * (w // 2), 4 * c)


@pytest.mark.parametrize("case", PATCHIFY_CASES, ids=lambda c: c["id"])
def test_ln_patchify2(case):
    b, h, w, c = case["b"], case["h"], case["w"], case["c"]
    x = _ln_rows_input(case["id"], b * h * w, c)
    xd = x.to(DEV)
    got = _twice(case["id"], torch.float16, b * h * w * c, lambda p: _call("pb200_ln_patchify2", _p(xd), b, h, w, c, p, _st()))
    y, e = _ln64(x.double())
    ref, bound = _patchify_ref(y, b, h, w, c), _patchify_ref(_f16(y, e), b, h, w, c)
    _report("ln_patchify2", case["id"], "ln_rows_kernel<1>", got.view(-1, 4 * c).cpu(), ref, bound,
            probe_ref=_patchify_ref(y, b, h, w, c, swap=True))


# ------------------------------------------------------------------ 3. nn.LayerNorm with eps / affine (ln_affine_kernel)
AFFINE_CASES = [dict(id=f"lna-c{c}-eps{eps:g}-w{int(wt)}b{int(bs)}-{out}", c=c, eps=eps, wt=wt, bs=bs, out=out)
                for c in (5, 36, 130) for eps in (1e-6, 1e-5) for wt, bs in ((False, False), (True, False), (False, True), (True, True))
                for out in ("out16", "out32") if not (c % 4 == 0 and eps == 1e-6 and not wt and not bs)]


def _layernorm_kernel(c, eps, wt, bs):
    """blocks.cu pb200_layernorm: the executor's ln_rows_kernel only for its own LayerNorm2d."""
    return "ln_rows_kernel<0>" if (eps == 1e-6 and not wt and not bs and c % 4 == 0) else "ln_affine_kernel"


@pytest.mark.parametrize("case", AFFINE_CASES, ids=lambda c: c["id"])
def test_ln_affine(case):
    c, eps, rows = case["c"], case["eps"], 21
    g = _gen(case["id"])
    x = _ln_rows_input(case["id"], rows, c)
    wt = (torch.rand(c, generator=g) * 2 - 0.5) if case["wt"] else None
    bs = torch.randn(c, generator=g) if case["bs"] else None
    xd, wd, bd = x.to(DEV), wt.to(DEV) if wt is not None else None, bs.to(DEV) if bs is not None else None
    f16 = case["out"] == "out16"

    def run(p):
        _call("pb200_layernorm", _p(xd), rows, c, eps, _p(wd), _p(bd), None if f16 else p, p if f16 else None, _st())
    got = _twice(case["id"], torch.float16 if f16 else torch.float32, rows * c, run)
    y, e = _ln64(x.double(), eps=eps)
    wv = wt.double() if wt is not None else torch.ones(c, dtype=torch.float64)
    bv = bs.double() if bs is not None else torch.zeros(c, dtype=torch.float64)
    ref = y * wv + bv
    bound = e * wv.abs() + 2 * U * ((y * wv).abs() + ref.abs())
    if f16:
        bound = _f16(ref, bound)
    other = _ln64(x.double(), eps=1e-5 if eps != 1e-5 else 1e-6)[0] * wv + bv
    _report("ln_affine", case["id"], _layernorm_kernel(c, eps, case["wt"], case["bs"]), got.view(rows, c).cpu(), ref, bound,
            probe_ref=other)


# ------------------------------------------------------------------ 4. in_mapper + PixelUnshuffle (embed_tokens_kernel)
EMBED_CASES = [dict(id=f"emb-c{c}-ps{ps}", c=c, ps=ps, b=b, h=h, w=w)
               for (c, ps, b, h, w) in ((16, 1, 2, 3, 5), (5, 1, 1, 4, 7), (3, 2, 2, 4, 6), (5, 2, 1, 6, 2), (4, 2, 3, 2, 4),
                                        (7, 4, 1, 8, 4), (32, 4, 2, 4, 8), (768, 2, 1, 4, 6), (192, 4, 1, 4, 8))]


def _embed_ref(emb64, tok, c, ps, swap=False):
    b, h, w = tok.shape
    rows = emb64[tok.clamp(0, emb64.shape[0] - 1)]                      # [b, h, w, c]
    t = rows.view(b, h // ps, ps, w // ps, ps, c)
    t = t.permute(0, 1, 3, 5, 4, 2) if swap else t.permute(0, 1, 3, 5, 2, 4)
    return t.reshape(b * (h // ps) * (w // ps), c * ps * ps)


@pytest.mark.parametrize("case", EMBED_CASES, ids=lambda c: c["id"])
def test_embed_tokens(case):
    c, ps, b, h, w = case["c"], case["ps"], case["b"], case["h"], case["w"]
    nl = 37
    g = _gen(case["id"])
    emb = torch.randn(nl, c, generator=g) + torch.arange(nl).unsqueeze(1) * 0.5
    tok = torch.randint(0, nl, (b, h, w), generator=g)
    tok.view(-1)[:4] = torch.tensor([-3, nl, nl + 100, -(1 << 40)])[:tok.numel()]      # clamped to [0, nl)
    ed, td = emb.to(DEV), tok.to(DEV)
    n = b * h * w * c
    got = _twice(case["id"], torch.float16, n, lambda p: _call("pb200_embed_tokens", _p(td), _p(ed), nl, c, b, h, w, ps, p, _st()))
    y, e = _ln64(emb.double())
    ref, bound = _embed_ref(y, tok, c, ps), _embed_ref(_f16(y, e), tok, c, ps)
    probe = _embed_ref(y, tok, c, ps, swap=True) if ps > 1 else _embed_ref(y, tok.clamp(0, nl) % nl, c, ps)
    _report("embed_tokens", case["id"], "embed_tokens_kernel", got.view(-1, c * ps * ps).cpu(), ref, bound, probe_ref=probe,
            scalar_stores=(c * ps * ps) % 8 != 0)


def test_embed_tokens_refuses_over_48k():
    """c_in * patch^2 = 3088 > 3072 needs more than 48 KB of shared memory: refused, nothing written."""
    emb = torch.randn(3, 193, device=DEV)
    tok = torch.zeros(1, 4, 4, dtype=torch.int64, device=DEV)
    o = _Out(torch.float16, 193 * 16)
    rc = _rc("pb200_embed_tokens", _p(tok), _p(emb), 3, 193, 1, 4, 4, 4, o.ptr(), _st())
    torch.cuda.synchronize()
    assert rc != 0
    o.check("refused embed", written=False)
    assert bool((o.bits == o.sent).all())
    _log(dict(family="embed_tokens", case="refuse-3088", kernel="embed_tokens_kernel", refused=True))


# ------------------------------------------------------------------ 5. depthwise conv + LayerNorm (dwconv_ln_kernel, dwconv3_ln_patch_kernel)
# (b, h, w, c, k): odd grids, grids smaller than the kernel, channel counts whose c/4 is not a multiple of 32
DW_GEOMS = [(3, 5, 24, 5), (5, 9, 72, 3), (4, 5, 136, 1), (5, 3, 264, 7), (5, 11, 520, 3), (5, 11, 1000, 3), (7, 3, 1000, 5),
            (3, 17, 2056, 3), (3, 5, 2056, 7)]
DW_CASES = [dict(id=f"dw-{h}x{w}-c{c}-k{k}-{'skip' if skip else 'noskip'}-{'wrap' if wrap else 'zero'}", h=h, w=w, c=c, k=k,
                 skip=skip, wrap=wrap)
            for (h, w, c, k) in DW_GEOMS for skip in (False, True) for wrap in (False, True)]
DW_VARIANTS = {"default": {}, "patch": {"PB200_DWCONV_PATCH": "1"}, "warp": {"PB200_DWCONV_WARP": "1"}}
DW_WRAP = [0, 1, 2, 3]           # the wrap bytes of the conditional rows; rows 4, 5 read bytes 0, 1 (n_base = 4)
DW_BATCH = {False: 2, True: 6}


def _dw_kernel(c, k, w, skip, wrap, variant):
    """ops.cu launch_dwconv_ln: the 2x8 patch kernel for k = 3, c <= 2560, c > 640 and w >= 8 (everywhere with
    PB200_DWCONV_PATCH, never with PB200_DWCONV_WARP), MAXT = the next of 64 / 160 / 320 / 640 above c/4 rounded to a warp;
    the warp kernel otherwise, NV = 1 / 5 / 10 / 20 for c <= 128 / 640 / 1280 / 2560."""
    if k == 3 and c <= 2560 and variant != "warp" and (variant == "patch" or (c > 640 and w >= 8)):
        threads = (c // 4 + 31) // 32 * 32
        maxt = 64 if threads <= 64 else 160 if threads <= 160 else 320 if threads <= 320 else 640
        return f"dwconv3_ln_patch_kernel<{int(skip)},{maxt},{int(wrap)}>"
    nv = 1 if c <= 128 else 5 if c <= 640 else 10 if c <= 1280 else 20
    return f"dwconv_ln_kernel<{nv},{int(skip)},{int(wrap)}>"


def _dw_inputs(case):
    g = _gen(case["id"])
    b, h, w, c, k = DW_BATCH[case["wrap"]], case["h"], case["w"], case["c"], case["k"]
    per = 2 if case["skip"] else 1
    # distinct values per channel and position: a wrong tap, channel or padding moves the conv by O(1)
    x = torch.randn(b, h, w, c, generator=g) + torch.linspace(-1, 1, c)
    skip = torch.randn(b, h, w, c, generator=g) - torch.linspace(-1, 1, c) if case["skip"] else None
    wp = torch.randn(k * k, per, c, generator=g) / k
    bias = torch.randn(c, generator=g) * 0.5
    return x, skip, wp, bias


def _dw_ref(case, x, skip, wp, bias, drop_centre=False, no_wrap=False):
    """fp64 depthwise conv (+ bias) with zero or per-sample circular padding, and sum |products| + |bias| per element."""
    b, h, w, c, k = x.shape[0], case["h"], case["w"], case["c"], case["k"]
    pad = k // 2
    if skip is not None:
        cat = torch.cat([x, skip], -1).double()                          # [b, h, w, 2c]
        srcs = [cat[..., 0::2], cat[..., 1::2]]                           # concatenated channels 2g, 2g+1 feed output g
    else:
        srcs = [x.double()]
    acc = bias.double().expand(b, h, w, c).clone()
    s = bias.double().abs().expand(b, h, w, c).clone()
    codes = [DW_WRAP[i] if i < 4 else DW_WRAP[i - 4] for i in range(b)] if case["wrap"] and not no_wrap else [0] * b
    ys, xs = torch.arange(h), torch.arange(w)
    for ky in range(k):
        for kx in range(k):
            if drop_centre and ky == pad and kx == pad:        # the one tap that is never padding
                continue
            for bi in range(b):
                iy, ix = ys + ky - pad, xs + kx - pad
                my = torch.ones(h, dtype=torch.bool) if codes[bi] & 2 else (iy >= 0) & (iy < h)
                mx = torch.ones(w, dtype=torch.bool) if codes[bi] & 1 else (ix >= 0) & (ix < w)
                iy, ix = iy % h, ix % w
                m = (my[:, None] & mx[None, :]).double()[..., None]
                for j, src in enumerate(srcs):
                    v = src[bi][iy][:, ix] * wp[ky * k + kx, j].double() * m
                    acc[bi] += v
                    s[bi] += v.abs()
    return acc, s


def _dw_check(case, variant):
    x, skip, wp, bias = _dw_inputs(case)
    b, h, w, c, k = x.shape[0], case["h"], case["w"], case["c"], case["k"]
    xd, sd, wd, bd = x.to(DEV), skip.to(DEV) if skip is not None else None, wp.to(DEV), bias.to(DEV)
    if case["wrap"]:
        wrap = torch.tensor(DW_WRAP, dtype=torch.uint8, device=DEV)
        run = lambda p: _call("pb200_dwconv_ln_pairs", _p(xd), _p(sd), _p(wd), _p(bd), b, h, w, c, k, _p(wrap), 4, p, _st())  # noqa: E731
    else:
        run = lambda p: _call("pb200_dwconv_ln", _p(xd), _p(sd), _p(wd), _p(bd), b, h, w, c, k, p, _st())  # noqa: E731
    got = _twice(case["id"], torch.float16, b * h * w * c, run).view(-1, c).cpu()
    acc, s = _dw_ref(case, x, skip, wp, bias)
    n_fma = k * k * (2 if skip is not None else 1)
    y, e = _ln64(acc.view(-1, c), e_in=(n_fma + 1) * U * s.view(-1, c))
    bound = _f16(y, e)
    row = dict(family="dwconv_ln", case=case["id"], variant=variant, kernel=_dw_kernel(c, k, w, skip is not None, case["wrap"], variant),
               ratio=_ratio(got, y, bound), probe=_probe(y, bound, _ln64(_dw_ref(case, x, skip, wp, bias, drop_centre=True)[0].view(-1, c))[0]))
    if case["wrap"] and k > 1:
        row["probe_wrap"] = _probe(y, bound, _ln64(_dw_ref(case, x, skip, wp, bias, no_wrap=True)[0].view(-1, c))[0])
    row["finite"] = bool(torch.isfinite(got.double()).all())
    return row


def _dw_assert(row):
    assert row["finite"], row
    assert row["ratio"] <= 1.0, row
    assert row["probe"] > 1.0 and row.get("probe_wrap", 2.0) > 1.0, row


def _dw_child_main(variant):
    for case in DW_CASES:
        try:
            print("RES", json.dumps({"id": case["id"], "ok": True, "row": _dw_check(case, variant)}), flush=True)
        except Exception as e:          # report and go on: one case's failure must not hide the others
            print("RES", json.dumps({"id": case["id"], "ok": False, "msg": f"{type(e).__name__}: {e}"}), flush=True)


_DW_CHILD = {}


def _dw_child(variant):
    if variant not in _DW_CHILD:
        code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_ops_matrix as t; t._dw_child_main(%r)" % (ROOT, HERE, variant)
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, **DW_VARIANTS[variant]))
        res = {}
        for line in r.stdout.splitlines():
            if line.startswith("RES "):
                j = json.loads(line[4:])
                res[j["id"]] = j
        _DW_CHILD[variant] = (r.returncode, r.stderr[-3000:], res)
    return _DW_CHILD[variant]


@pytest.mark.parametrize("variant", list(DW_VARIANTS))
@pytest.mark.parametrize("case", DW_CASES, ids=lambda c: c["id"])
def test_dwconv_ln(case, variant):
    if variant == "default":
        row = _dw_check(case, variant)
    else:
        rc, err, res = _dw_child(variant)
        got = res.get(case["id"])
        assert got is not None, f"case did not report (child rc {rc}): {err}"
        assert got["ok"], got["msg"]
        row = got["row"]
    _log(row)
    _dw_assert(row)


# ------------------------------------------------------------------ 6. GlobalResponseNorm, fp16 in place (grn_scale_kernel + grn_apply_kernel)
GRN_CASES = [dict(id=f"grn-n{n}-p{p}-b3", n=n, p=p, b=3) for n in (8, 2048, 2056, 5120) for p in (1, 7, 8, 15, 16, 17, 64, 100)]
GRN_CASES += [dict(id="grn-n5120-p100-b26", n=5120, p=100, b=26), dict(id="grn-n2056-p64-b66", n=2056, p=64, b=66)]


def _grn_rows_per_cta(b, p, n, sm_count):
    """ops.cu launch_grn_fused: 16 rows per CTA (P when P < 16), 8 when 16 leaves fewer than 4 CTAs per SM."""
    nch = n // 8
    tpb = 256 if nch >= 256 else (nch + 31) // 32 * 32
    rpc = 16 if p >= 16 else p
    if -(-p // rpc) * b * -(-nch // tpb) < 4 * sm_count and rpc > 8:
        rpc = 8
    return rpc, tpb


def _grn_scale_ref(q, gamma, drop_last=False):
    """fp64 scale[b, n] = 1 + gamma[n] * Gx / (mean Gx + 1e-6) from the same 2^-24 fixed-point sums of squares."""
    gx = torch.sqrt(q.double() * 2.0 ** -24)
    mean = (gx[:, :-1].sum(-1, keepdim=True) / gx.shape[1]) if drop_last else gx.mean(-1, keepdim=True)
    nx = gx / (mean + 1e-6)
    return 1 + gamma.double() * nx, gamma.double().abs() * nx


@pytest.mark.parametrize("case", GRN_CASES, ids=lambda c: c["id"])
def test_grn_f16(case):
    b, p, n = case["b"], case["p"], case["n"]
    g = _gen(case["id"])
    h = (torch.randn(b, p, n, generator=g) * 2).half()
    q = (torch.rand(b, n, generator=g, dtype=torch.float64) ** 2 * 1000 * 2 ** 24).to(torch.int64)
    q[:, ::97] = 0
    gamma, beta = torch.randn(n, generator=g), torch.randn(n, generator=g) * 0.5
    zps = n + 3
    hd, qd, gd, bd = h.to(DEV), q.to(DEV), gamma.to(DEV), beta.to(DEV)
    scales, nexts = [], []

    def run(ptr):
        sq_next = _Out(torch.int64, b * zps)
        scale = _Out(torch.float32, b * n)
        _call("pb200_grn_f16", ptr, b, p, n, _p(qd), sq_next.ptr(), zps, _p(gd), _p(bd), scale.ptr(), _st())
        torch.cuda.synchronize()
        sq_next.check("sq_next")
        scale.check("scale_scratch")
        nexts.append(sq_next.value().clone())
        scales.append(scale.value().clone())
    got = _twice(case["id"], torch.float16, b * p * n, run, init=hd, written=False).view(b, p, n).cpu()
    assert bool((nexts[0] == 0).all()), "sq_next: not every one of the batch * zero_per_sample entries was zeroed"
    assert torch.equal(scales[0], scales[1])
    sref, snx = _grn_scale_ref(q, gamma)
    depth = 2 * -(-n // 1024) + 5 + 16 + 2
    e_scale = snx * (depth + 8) * U + U * sref.abs()
    sg = scales[0].view(b, n).cpu()
    probe_scale = _grn_scale_ref(q, gamma, drop_last=True)[0]
    s_ratio, s_probe = _ratio(sg, sref, e_scale), _probe(sref, e_scale, probe_scale)
    h64 = h.double()
    ref = h64 * sref[:, None, :] + beta.double()
    bound = _f16(ref, h64.abs() * e_scale[:, None, :] + U * ((h64 * sref[:, None, :]).abs() + ref.abs()))
    rpc, tpb = _grn_rows_per_cta(b, p, n, torch.cuda.get_device_properties(0).multi_processor_count)
    _report("grn_f16", case["id"], "grn_scale_kernel + grn_apply_kernel", got, ref, bound, scale_ratio=s_ratio, probe_scale=s_probe,
            rows_per_cta=rpc, tpb=tpb)
    assert s_ratio <= 1.0 and s_probe > 1.0, (s_ratio, s_probe)


GRN32_CASES = [dict(id="grn32-b2-p7-n36", b=2, p=7, n=36), dict(id="grn32-b1-p512-n8192", b=1, p=512, n=8192)]


def _grn32_grid(p, n):
    """blocks.cu pb200_grn_f32: P*N / 2048 CTAs per sample, at least 1 and at most 1024."""
    return max(1, min(1024, p * n // 2048))


@pytest.mark.parametrize("case", GRN32_CASES, ids=lambda c: c["id"])
def test_grn_f32(case):
    b, p, n = case["b"], case["p"], case["n"]
    g = _gen(case["id"])
    x = torch.randn(b, p, n, generator=g)
    gamma, beta = torch.randn(n, generator=g), torch.randn(n, generator=g) * 0.5
    xd, gd, bd = x.to(DEV), gamma.to(DEV), beta.to(DEV)
    stat = torch.empty(b, n, device=DEV)
    got = _twice(case["id"], torch.float32, b * p * n,
                 lambda ptr: _call("pb200_grn_f32", _p(xd), b, p, n, _p(gd), _p(bd), _p(stat), ptr, _st())).view(b, p, n).cpu()
    x64 = x.double()

    def ref_of(xs):
        gx = torch.sqrt((xs * xs).sum(1, keepdim=True))
        nx = gx / (gx.mean(-1, keepdim=True) + 1e-6)
        return gamma.double() * (x64 * nx) + beta.double() + x64, nx
    ref, nx = ref_of(x64)
    depth = p / 2 + -(-n // 256) + 5 + 8 + 8
    bound = (gamma.double() * x64 * nx).abs() * depth * U + 2 * U * (ref.abs() + beta.double().abs() + x64.abs())
    _report("grn_f32", case["id"], "grn_f32_stat_kernel + grn_f32_apply_kernel", got, ref, bound, probe_ref=ref_of(x64[:, :-1])[0],
            ctas_per_sample=_grn32_grid(p, n))


# ------------------------------------------------------------------ 7. timestep embedding (r_embed_kernel) and FiLM table
R_EMBED_CASES = [dict(id=f"remb-c{c}", c=c) for c in (4, 5, 64, 65)]


@pytest.mark.parametrize("case", R_EMBED_CASES, ids=lambda c: c["id"])
def test_r_embed(case):
    c_r = case["c"]
    g = _gen(case["id"])
    r = torch.cat([torch.tensor([0.0, 1.0]), torch.rand(7, generator=g)])
    B = r.numel()
    rd = r.to(DEV)
    got = _twice(case["id"], torch.float32, B * c_r, lambda p: _call("pb200_paella_r_embedding", _p(rd), B, c_r, p, _st())).view(B, c_r)
    half = c_r // 2
    j = torch.arange(c_r)
    f = torch.where(j < half, j, j - half).clamp_max(half - 1).double()

    def ref_of(denom):
        ang = r.double()[:, None] * 10000.0 * torch.exp(-math.log(10000.0) / denom * f)[None, :]
        out = torch.where(j[None, :] < half, torch.sin(ang), torch.cos(ang))
        return torch.where(j[None, :] < 2 * half, out, torch.zeros_like(out)), ang
    ref, ang = ref_of(half - 1)
    # the angle's own fp32 error: kneg and f*kneg rounded (2 U |f kneg| through exp), expf (2 ulp), r*1e4 and *freq (2 U)
    kf = math.log(10000.0) / (half - 1) * f
    e_ang = ang.abs() * U * (2 * kf[None, :] + 8)
    bound = e_ang + 4 * U * (ref.abs() + 2.0 ** -126 / U) + 2.0 ** -60
    gc = got.cpu()
    if c_r % 2:
        assert bool((gc[:, -1].view(torch.int32) == 0).all()), "odd c_r: the pad column must be +0"
    # the same formula in fp32 by torch on the device, within 8 ulp (of at least 1/16) where |ang| < 4
    fd = f.float().to(DEV)
    kneg = torch.tensor(-(math.log(10000.0) / (half - 1)), dtype=torch.float32)
    ang32 = (rd[:, None] * 10000.0) * torch.exp(fd * kneg.to(DEV))[None, :]
    t32 = torch.where(j.to(DEV)[None, :] < half, torch.sin(ang32), torch.cos(ang32))
    small = (ang < 4) & (j[None, :] < 2 * half)
    ulp_ratio = float(((got - t32).abs().cpu() / (8 * 2.0 ** -23 * t32.abs().cpu().clamp_min(2.0 ** -4)))[small].max())
    _report("r_embed", case["id"], "r_embed_kernel", gc, ref, bound, probe_ref=ref_of(half)[0], torch_fp32_ulp_ratio=ulp_ratio)
    assert ulp_ratio <= 1.0


FILM_CASES = [dict(id=f"film-b{b}-cr{cr}-t{t}", b=b, cr=cr, t=t) for b in (1, 64, 65, 200) for cr in (32, 64, 65) for t in (100, 300)]


def _film_kernel(c_r):
    """ops.cu launch_film_table: the W-row-in-registers kernel for c_r = 64, the generic one otherwise."""
    return "film_table_kernel<64>" if c_r == 64 else "film_table_generic_kernel"


@pytest.mark.parametrize("case", FILM_CASES, ids=lambda c: c["id"])
def test_film_table(case):
    b, cr, total = case["b"], case["cr"], case["t"]
    g = _gen(case["id"])
    re = torch.randn(b, cr, generator=g) + torch.arange(b)[:, None] * 0.25          # every sample distinct
    W, bias = torch.randn(total, cr, generator=g) / cr ** 0.5, torch.randn(total, generator=g)
    rd, wd, bd = re.to(DEV), W.to(DEV), bias.to(DEV)
    got = _twice(case["id"], torch.float32, b * total,
                 lambda p: _call("pb200_film_table", _p(rd), b, cr, _p(wd), _p(bd), total, p, _st())).view(b, total).cpu()
    r64, W64, b64 = re.double(), W.double(), bias.double()
    ref = r64 @ W64.t() + b64
    bound = (cr + 1) * U * (r64.abs() @ W64.abs().t() + b64.abs())
    probe = r64[:, :-1] @ W64[:, :-1].t() + b64                           # the last r_embed term dropped
    extra = {}
    if b > 64:                                                             # a chunk of 64 samples read from the wrong offset
        shifted = r64.clone()
        shifted[64:] = r64[63:-1]
        extra["probe_chunk"] = _probe(ref, bound, shifted @ W64.t() + b64)
        assert extra["probe_chunk"] > 1.0
    _report("film_table", case["id"], _film_kernel(cr), got, ref, bound, probe_ref=probe, **extra)


def test_film_apply():
    M, N, P, ld, off = 37, 36, 5, 100, 12
    g = _gen("film_apply")
    x = torch.randn(M, N, generator=g)
    film = torch.randn(-(-M // P), ld, generator=g)
    xd, fd = x.to(DEV), film.to(DEV)
    got = _twice("film_apply", torch.float32, M * N, lambda p: _call("pb200_film_apply", p, M, N, P, _p(fd), ld, off, _st()),
                 init=xd, written=False).view(M, N).cpu()
    x64, f64 = x.double(), film.double()

    def ref_of(rows):
        a, s = f64[rows // P, off:off + N], f64[rows // P, off + N:off + 2 * N]
        return x64 * (1 + a) + s, a, s
    rows = torch.arange(M)
    ref, a, s = ref_of(rows)
    bound = 2 * U * ((x64 * (1 + a)).abs() + s.abs() + ref.abs())
    _report("film_apply", "film-m37-p5", "film_apply_kernel", got, ref, bound, probe_ref=ref_of((rows + 1).clamp_max(M - 1))[0])
    for bad_ld, bad_off in ((ld, off + 1), (ld + 2, off)):               # misaligned tables: refused, x untouched
        o = _Out(torch.float32, M * N, init=xd)
        rc = _rc("pb200_film_apply", o.ptr(), M, N, P, _p(fd), bad_ld, bad_off, _st())
        torch.cuda.synchronize()
        assert rc != 0
        o.check("refused film_apply", written=False)
        assert torch.equal(o.value().cpu(), x.view(-1))


# ------------------------------------------------------------------ 8. casts (cast_kernel<0..3>), pad and gather casts
CAST_CASES = [dict(id=f"cast-op{op}-n{n}-{'odd' if mis else 'al'}{'-b' if hb else ''}", op=op, n=n, mis=mis, hb=hb)
              for op in (0, 1, 2, 3) for n in (1024, 1025, 1026, 1027) for mis in (False, True) for hb in ((False, True) if op == 2 else (True,) if op == 3 else (False,))]
CAST_PER = {1024: 10, 1025: 7, 1026: 13, 1027: 6}                          # OP 3: a sample boundary inside a thread's 4 elements


@pytest.mark.parametrize("case", CAST_CASES, ids=lambda c: c["id"])
def test_cast(case):
    op, n = case["op"], case["n"]
    g = _gen(case["id"])
    a = torch.randn(n, generator=g) * 3
    if op == 1:
        a[:3] = torch.tensor([100.0, -100.0, 0.0])
    b = torch.randn(n, generator=g) if case["hb"] else None
    ad, bd = a.to(DEV), b.to(DEV) if b is not None else None
    wa, wb = 1.375, -0.625
    per = CAST_PER[n]
    S = -(-n // per)
    w = torch.stack([torch.rand(S, generator=g) * 2 + 1, -(torch.rand(S, generator=g) * 2 + 1), torch.zeros(S)], 1)
    wd = w.reshape(-1).to(DEV)
    pre = 17 if case["mis"] else 16                                         # out offset by one half: scalar stores

    def run(p):
        if op in (0, 1):
            _call("pb200_cast_f16", _p(ad), n, op, p, _st())
        elif op == 2:
            _call("pb200_mix_cast_f16", _p(ad), _p(bd), wa, wb, n, p, _st())
        else:
            _call("pb200_mix_cast_rows_f16", _p(ad), _p(bd), _p(wd), per, n, p, _st())
    got = _twice(case["id"], torch.float16, n, run, pre=pre).cpu()
    a64 = a.double()
    probe = None
    if op == 0:
        # bit-exact against torch's round-to-nearest-even; the probe rounds toward zero
        h = a.half()
        ref, bound = h.double(), torch.full((n,), 2.0 ** -60, dtype=torch.float64)
        probe = torch.where(h.double().abs() > a64.abs(), torch.nextafter(h, torch.zeros_like(h)), h).double()
    elif op == 1:
        ref = a64 / (1 + torch.exp(-a64))
        bound = _f16(ref, 8 * U * ref.abs() + 2.0 ** -60)
        probe = a64 / (1 + torch.exp(-a64 * 1.001))
    else:
        if op == 2:
            s = torch.zeros(n, dtype=torch.long)
            ca, cb = torch.full((n,), wa, dtype=torch.float64), torch.full((n,), wb, dtype=torch.float64)
        else:
            s = torch.arange(n) // per
            ca, cb = w[s, 0].double(), w[s, 1].double()
        bb = b.double() if b is not None else torch.zeros(n, dtype=torch.float64)
        ref = a64 * ca + bb * cb
        bound = _f16(ref, 2 * U * ((bb * cb).abs() + ref.abs()) + U * (a64 * ca).abs())
        if op == 3:
            sp = ((torch.arange(n) - 1).clamp_min(0)) // per                   # a boundary off by one element
            probe = a64 * w[sp, 0].double() + bb * w[sp, 1].double()
        else:
            probe = a64 * ca * 1.001 + bb * cb
    _report("cast", case["id"], f"cast_kernel<{op}>", got, ref, bound, probe_ref=probe, scalar_stores=case["mis"] or n % 4 != 0)


PAD_CASES = [dict(id=f"pad-{h}x{w}-c{c}", h=h, w=w, c=c) for (h, w, c) in ((3, 5, 8), (1, 4, 4), (5, 1, 12), (1, 1, 4), (6, 7, 36))]


def _pad_ref(x, codes, zero=False):
    b, h, w, c = x.shape
    out = torch.zeros(b, h + 2, w + 2, c, dtype=x.dtype)
    ys, xs = torch.arange(-1, h + 1), torch.arange(-1, w + 1)
    for bi in range(b):
        wc = 0 if zero else codes[bi]
        my = ((ys >= 0) & (ys < h)) | bool(wc & 2)
        mx = ((xs >= 0) & (xs < w)) | bool(wc & 1)
        v = x[bi][ys % h][:, xs % w]
        out[bi] = torch.where((my[:, None] & mx[None, :])[..., None], v, torch.zeros_like(v))
    return out


@pytest.mark.parametrize("case", PAD_CASES, ids=lambda c: c["id"])
def test_pad_cast(case):
    h, w, c = case["h"], case["w"], case["c"]
    codes = [0, 1, 2, 3]
    g = _gen(case["id"])
    x = torch.randn(4, h, w, c, generator=g) * 100
    xd, wr = x.to(DEV), torch.tensor(codes, dtype=torch.uint8, device=DEV)
    n = 4 * (h + 2) * (w + 2) * c
    got = _twice(case["id"], torch.float16, n, lambda p: _call("pb200_pad_cast_f16", _p(xd), 4, h, w, c, _p(wr), p, _st())).cpu()
    want = _pad_ref(x, codes).half().reshape(-1)
    n_diff = int((got.view(torch.int16) != want.view(torch.int16)).sum())
    n_probe = int((_pad_ref(x, codes, zero=True).half().reshape(-1).view(torch.int16) != want.view(torch.int16)).sum())
    _log(dict(family="pad_cast", case=case["id"], kernel="pad_cast_kernel", mismatches=n_diff, probe_mismatches=n_probe))
    assert n_diff == 0 and n_probe > 0


def test_gather_cast():
    batch, per, samples = 4, 1028, [2, 0, 2]
    for n_blocks in (3, 5, 6):
        g = _gen(f"gather{n_blocks}")
        a = torch.randn(2 * batch, per, generator=g) * 50
        ad, sd = a.to(DEV), torch.tensor(samples, dtype=torch.int32, device=DEV)
        got = _twice(f"gather-{n_blocks}", torch.float16, n_blocks * per,
                     lambda p: _call("pb200_gather_cast_f16", _p(ad), _p(sd), len(samples), n_blocks, batch, per, p, _st())).cpu()
        src = [samples[j] if j < len(samples) else batch + samples[j - len(samples)] for j in range(n_blocks)]
        want = a[src].half().reshape(-1)
        n_diff = int((got.view(torch.int16) != want.view(torch.int16)).sum())
        probe = a[[(s + 1) % (2 * batch) for s in src]].half().reshape(-1)              # every block from its neighbour
        n_probe = int((probe.view(torch.int16) != want.view(torch.int16)).sum())
        _log(dict(family="gather_cast", case=f"gather-{n_blocks}", kernel="gather_cast_kernel", mismatches=n_diff, probe_mismatches=n_probe))
        assert n_diff == 0 and n_probe > 0


# ------------------------------------------------------------------ 9. tail rows, guidance mix, layout, regional masks
REPLICATE_CASES = [dict(id=f"rep-per{per}", per=per) for per in (48, 36, 37, 4096)]


def _replicate_kernel(per):
    """ops.cu launch_replicate_rows: the widest word dividing per."""
    return "replicate_rows_kernel<uint4>" if per % 16 == 0 else "replicate_rows_kernel<uint32_t>" if per % 4 == 0 else "replicate_rows_kernel<uint8_t>"


@pytest.mark.parametrize("case", REPLICATE_CASES, ids=lambda c: c["id"])
def test_replicate_rows(case):
    per, n_base, src = case["per"], 3, [1, 1, 0, 2]
    g = _gen(case["id"])
    buf0 = torch.randint(0, 256, ((n_base + len(src)) * per + 64,), generator=g, dtype=torch.uint8)
    want = buf0.clone()
    for y, s in enumerate(src):
        want[(n_base + y) * per:(n_base + y + 1) * per] = buf0[s * per:(s + 1) * per]
    bd, sd = buf0.to(DEV), torch.tensor(src, dtype=torch.int32, device=DEV)
    _call("pb200_replicate_rows", _p(bd), per, n_base, _p(sd), len(src), _st())
    torch.cuda.synchronize()
    once = bd.cpu()
    _call("pb200_replicate_rows", _p(bd), per, n_base, _p(sd), len(src), _st())
    torch.cuda.synchronize()
    n_diff = int((once != want).sum())
    probe = buf0.clone()
    for y, s in enumerate(src):
        probe[(n_base + y) * per:(n_base + y + 1) * per] = buf0[(s + 1) * per:(s + 2) * per]
    _log(dict(family="replicate_rows", case=case["id"], kernel=_replicate_kernel(per), mismatches=n_diff,
              probe_mismatches=int((probe != want).sum())))
    assert n_diff == 0 and torch.equal(bd.cpu(), once) and int((probe != want).sum()) > 0


@pytest.mark.parametrize("ld", [2, 3, 4, 5, 6])
def test_guidance_mix(ld):
    per, S, nc = 1100, 12, 3
    g = _gen(f"gmix{ld}")
    f = torch.randn(S, per, generator=g)
    rows = torch.full((nc, ld), -1, dtype=torch.int32)
    for y in range(nc):
        rows[y, 0], rows[y, 1] = y, nc + y
        for j in range(2, ld):
            rows[y, j] = 6 + (y + j) % 6
        if y == 1 and ld > 3:
            rows[y, 2] = -1                                    # a terminator before ld, with a valid index after it
    coef = torch.randn(nc, ld, generator=g)
    fd, rd, cd = f.to(DEV), rows.to(DEV), coef.to(DEV)
    got = _twice(f"gmix-ld{ld}", torch.float32, S * per, lambda p: _call("pb200_guidance_mix", p, per, _p(rd), _p(cd), nc, ld, _st()),
                 init=fd, written=False).view(S, per).cpu()
    f64 = f.double()
    ref, bound, probe = f64.clone(), torch.full_like(f64, 2.0 ** -60), f64.clone()
    for y in range(nc):
        terms = [(int(rows[y, 0]), float(coef[y, 0])), (int(rows[y, 1]), float(coef[y, 1]))]
        for j in range(2, ld):
            if int(rows[y, j]) < 0:
                break
            terms.append((int(rows[y, j]), float(coef[y, j])))
        t = sum(f64[s] * a for s, a in terms)
        ref[y] = t
        bound[y] = (len(terms) + 1) * U * sum((f64[s] * a).abs() for s, a in terms) + U * t.abs()
        all_terms = terms + [(int(rows[y, j]), float(coef[y, j])) for j in range(len(terms), ld) if int(rows[y, j]) >= 0]
        probe[y] = sum(f64[s] * a for s, a in all_terms) if len(all_terms) > len(terms) else sum(f64[s] * a for s, a in terms[:-1])
    same = int((got[nc:].view(torch.int32) != f[nc:].view(torch.int32)).sum())
    assert same == 0, f"{same} elements of rows other than the composed c rows changed"
    _report("guidance_mix", f"gmix-ld{ld}", "guidance_mix_kernel", got[:nc], ref[:nc], bound[:nc], probe_ref=probe[:nc])


TRANSPOSE_CASES = [(2, 33, 70), (1, 5, 31), (3, 64, 96), (1, 1, 100)]


@pytest.mark.parametrize("bch", TRANSPOSE_CASES, ids=lambda t: "x".join(map(str, t)))
def test_transpose(bch):
    B, C, HW = bch
    g = _gen(f"tr{bch}")
    x = torch.randn(B, C, HW, generator=g)
    xd = x.to(DEV)
    nhwc = _twice("nchw_to_nhwc", torch.float32, B * C * HW, lambda p: _call("pb200_nchw_to_nhwc", _p(xd), B, C, HW, p, _st())).cpu()
    assert torch.equal(nhwc.view(B, HW, C), x.transpose(1, 2))
    yd = nhwc.to(DEV)
    back = _twice("nhwc_to_nchw", torch.float32, B * C * HW, lambda p: _call("pb200_nhwc_to_nchw", _p(yd), B, C, HW, p, _st())).cpu()
    assert torch.equal(back.view(B, C, HW), x)
    probe = int((x.reshape(B, HW, C) != x.transpose(1, 2)).sum())
    _log(dict(family="transpose", case="x".join(map(str, bch)), kernel="transpose_kernel", exact=True, probe_mismatches=probe))
    assert probe > 0 or C == 1 or HW == 1


def test_transpose_refuses_grid():
    """65536 row tiles exceed the grid's y limit: refused, nothing written."""
    C = 32 * 65536
    x = torch.zeros(1, C, 1, device=DEV)
    o = _Out(torch.float32, C)
    rc = _rc("pb200_nchw_to_nhwc", _p(x), 1, C, 1, o.ptr(), _st())
    torch.cuda.synchronize()
    assert rc != 0
    o.check("refused transpose", written=False)
    assert bool((o.bits == o.sent).all())
    _log(dict(family="transpose", case="refuse-grid", kernel="transpose_kernel", refused=True))


REGION_CASES = [dict(id=f"reg-{h}x{w}-p{p}-l{l}-{'rows' if mr else 'null'}", h=h, w=w, patch=p, levels=l, mask_row=mr)
                for (h, w, p, l) in ((8, 12, 1, 3), (10, 12, 2, 2), (6, 10, 2, 1), (16, 8, 1, 2)) for mr in (False, True)]


def _regional_ref(tok, rows, h, w, patch, levels, batch):
    out = []
    for l in range(levels):
        s = patch << l
        gh, gw = h // s, w // s
        lv = torch.zeros(batch, gh * gw, dtype=torch.uint8)
        for b in range(batch):
            t = tok[rows[b]].view(h, w)
            m = torch.zeros(gh, gw, dtype=torch.uint8)
            for dy in range(s):
                for dx in range(s):
                    m |= t[dy:gh * s:s, dx:gw * s:s]
            lv[b] = m.reshape(-1)
        out.append(lv.reshape(-1))
    return torch.cat(out)


@pytest.mark.parametrize("case", REGION_CASES, ids=lambda c: c["id"])
def test_regional_masks(case):
    h, w, patch, levels = case["h"], case["w"], case["patch"], case["levels"]
    batch = 3
    g = _gen(case["id"])
    vals = torch.tensor([0, 1, 2, 4, 8], dtype=torch.uint8)
    tok = vals[torch.randint(0, 5, (4, h * w), generator=g)]
    tok[tok.shape[0] - 1] = 0
    rows = [2, 0, 2] if case["mask_row"] else [0, 1, 2]
    td, rd = tok.to(DEV), torch.tensor(rows, dtype=torch.int32, device=DEV)
    n = sum(batch * (h // (patch << l)) * (w // (patch << l)) for l in range(levels))
    got = _twice(case["id"], torch.uint8, n, lambda p: _call("pb200_regional_masks", _p(td), _p(rd) if case["mask_row"] else None, batch, h, w,
                                                              patch, levels, p, _st())).cpu()
    want = _regional_ref(tok, rows, h, w, patch, levels, batch)
    probe = _regional_ref(tok, [0, 1, 2] if case["mask_row"] else [1, 2, 0], h, w, patch, levels, batch)
    n_diff = int((got != want).sum())
    _log(dict(family="regional_masks", case=case["id"], kernel="regional_masks_kernel", mismatches=n_diff,
              probe_mismatches=int((probe != want).sum())))
    assert n_diff == 0 and int((probe != want).sum()) > 0


# ------------------------------------------------------------------ coverage table
def _coverage():
    """kernel instance -> the cases that run it (restated from the dispatch conditions of ops.cu and blocks.cu)."""
    cov = {}

    def add(k, cid):
        cov.setdefault(k, []).append(cid)
    for c in LN_CASES:
        add("ln_rows_kernel<0>", c["id"])
    for c in PATCHIFY_CASES:
        add("ln_rows_kernel<1>", c["id"])
    for c in AFFINE_CASES:
        add(_layernorm_kernel(c["c"], c["eps"], c["wt"], c["bs"]), c["id"])
    for c in EMBED_CASES:
        add("embed_tokens_kernel", c["id"])
    for c in DW_CASES:
        for v in DW_VARIANTS:
            add(_dw_kernel(c["c"], c["k"], c["w"], c["skip"], c["wrap"], v), f"{c['id']}@{v}")
    for c in GRN_CASES:
        add("grn_scale_kernel", c["id"])
        add("grn_apply_kernel", c["id"])
    for c in GRN32_CASES:
        add("grn_f32_stat_kernel", c["id"])
        add("grn_f32_apply_kernel", c["id"])
    for c in R_EMBED_CASES:
        add("r_embed_kernel", c["id"])
    for c in FILM_CASES:
        add(_film_kernel(c["cr"]), c["id"])
    add("film_apply_kernel", "film_apply")
    for c in CAST_CASES:
        add(f"cast_kernel<{c['op']}>", c["id"])
    for c in PAD_CASES:
        add("pad_cast_kernel", c["id"])
    add("gather_cast_kernel", "gather_cast")
    for c in REPLICATE_CASES:
        add(_replicate_kernel(c["per"]), c["id"])
    add("guidance_mix_kernel", "guidance_mix")
    for t in TRANSPOSE_CASES:
        add("transpose_kernel", "x".join(map(str, t)))
    for c in REGION_CASES:
        add("regional_masks_kernel", c["id"])
    return cov


COVERAGE = _coverage()
OUT_OF_SCOPE = {"row_stats_kernel": "test_gpu_vqgan_matrix.py", "vq_front_patch_kernel": "test_gpu_vqgan_matrix.py",
                "attention_maps_accumulate_kernel": "test_gpu_attention_maps.py", "attention_maps_finalize_kernel": "test_gpu_attention_maps.py"}
