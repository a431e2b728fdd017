"""GPU parity tests for the kernel-level C-ABI entry points (run with -m gpu on an H100).

Random ops are compared BIT-EXACTLY with the torch CUDA ops they replace (same seed, same generator
offset afterwards); the VQ search bit-exactly with the plain-C oracle; the wgmma GEMM against an fp32
torch product of the same fp16 operands.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ops():
    from paella_b200 import ops
    return ops


def _gen():
    return torch.cuda.default_generators[torch.cuda.current_device()]


def _log(name, payload):
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "kernel_parity.jsonl"), "a") as f:
        f.write(json.dumps({"test": name, **payload}) + "\n")


# ------------------------------------------------------------------ RNG streams
@pytest.mark.parametrize("shape", [(7,), (64, 32, 32), (3, 1000, 1001)])
def test_randint_matches_torch(shape):
    ops = _ops()
    torch.manual_seed(1234)
    a = torch.randint(0, 8192, shape, device=DEV)
    off_a = _gen().get_offset()
    torch.manual_seed(1234)
    b = ops.randint(8192, shape, torch.device(DEV))
    assert _gen().get_offset() == off_a
    assert torch.equal(a, b)


@pytest.mark.parametrize("n", [5, 65536, 2_000_003])
def test_rand_matches_torch(n):
    ops = _ops()
    torch.manual_seed(7)
    torch.rand(3, device=DEV)                      # non-zero starting offset
    a = torch.rand(n, device=DEV)
    off_a = _gen().get_offset()
    torch.manual_seed(7)
    torch.rand(3, device=DEV)
    b = ops.rand((n,), torch.device(DEV))
    assert _gen().get_offset() == off_a
    assert torch.equal(a, b)


@pytest.mark.parametrize("rows,k", [(64, 100), (1000, 8192), (16384, 8192)])
def test_multinomial_bit_exact(rows, k):
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(5)
    p = torch.softmax(torch.randn(rows, k, device=DEV, generator=g) * 3.0, dim=-1)
    torch.manual_seed(99)
    a = torch.multinomial(p, 1)[:, 0]
    off_a = _gen().get_offset()
    torch.manual_seed(99)
    b = ops.multinomial(p)
    assert _gen().get_offset() == off_a
    mism = int((a != b).sum())
    _log("multinomial", {"rows": rows, "k": k, "mismatch": mism})
    assert mism == 0


def test_multinomial_ties_and_zeros():
    ops = _ops()
    p = torch.zeros(256, 512, device=DEV)
    p[:, 100] = 0.5
    p[:, 300] = 0.5
    torch.manual_seed(3)
    a = torch.multinomial(p, 1)[:, 0]
    torch.manual_seed(3)
    b = ops.multinomial(p)
    assert torch.equal(a, b)
    assert set(a.tolist()) <= {100, 300}


@pytest.mark.parametrize("B,K,H", [(2, 64, 8), (4, 8192, 32)])
def test_resample_logits_vs_torch_chain(B, K, H):
    """ref/src/utils.py:45-50 executed by torch on the GPU vs the fused exact kernel."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(11)
    lc = torch.randn(B, K, H, H, device=DEV, generator=g) * 2
    lu = torch.randn(B, K, H, H, device=DEV, generator=g) * 2
    cfg, temps = 8.0, torch.linspace(1.0, 0.2, 8)
    for i in (0, 5):
        torch.manual_seed(21 + i)
        logits = lc * cfg + lu * (1 - cfg)
        scores = logits.div(temps[i]).softmax(dim=1)
        s2 = scores.permute(0, 2, 3, 1).reshape(-1, K)
        a = torch.multinomial(s2, 1)[:, 0].view(B, H, H)
        off_a = _gen().get_offset()
        torch.manual_seed(21 + i)
        b = ops.resample_logits(lc, lu, cfg, float(temps[i]), "multinomial")
        assert _gen().get_offset() == off_a
        agree = float((a == b).float().mean())
        _log("resample_logits", {"B": B, "K": K, "H": H, "step": i, "agree": agree})
        # identical up to the softmax denominator's summation order (last-ulp ties only)
        assert agree >= 0.999
        am = ops.resample_logits(lc, lu, cfg, 1.0, "argmax")
        assert torch.equal(am, logits.argmax(dim=1))
    # no guidance
    torch.manual_seed(5)
    a = torch.multinomial(lc.div(temps[3]).softmax(dim=1).permute(0, 2, 3, 1).reshape(-1, K), 1)[:, 0].view(B, H, H)
    torch.manual_seed(5)
    b = ops.resample_logits(lc, None, 0.0, float(temps[3]), "multinomial")
    assert float((a == b).float().mean()) >= 0.999


def test_add_noise_matches_reference_expression():
    ops = _ops()
    B, H, L = 64, 32, 8192
    g = torch.Generator(device=DEV).manual_seed(2)
    x = torch.randint(0, L, (B, H, H), device=DEV, generator=g)
    rx = torch.randint(0, L, (B, H, H), device=DEV, generator=g)
    t = torch.rand(B, device=DEV, generator=g)
    torch.manual_seed(77)
    mask = (torch.rand_like(x.float()) <= t[:, None, None]).long()      # ref/src/modules.py:279
    ref = x * (1 - mask) + rx * mask
    off_a = _gen().get_offset()
    torch.manual_seed(77)
    out, m = ops.add_noise(x, t, rx, L)
    assert _gen().get_offset() == off_a
    assert torch.equal(out, ref) and torch.equal(m, mask)
    # random_x=None: randint_like drawn after the mask
    torch.manual_seed(78)
    mask = (torch.rand_like(x.float()) <= t[:, None, None]).long()
    rx2 = torch.randint_like(x, 0, L)
    ref2 = x * (1 - mask) + rx2 * mask
    off_a = _gen().get_offset()
    torch.manual_seed(78)
    out2, _ = ops.add_noise(x, t, None, L)
    assert _gen().get_offset() == off_a
    assert torch.equal(out2, ref2)


# ------------------------------------------------------------------ vector quantiser
def test_vq_nearest_bit_exact_vs_c_oracle():
    from oracle import vqgan_oracle as vo
    ops = _ops()
    assert vo._c_oracle(), "oracle/_ref/libvq_oracle.so not built"
    g = torch.Generator().manual_seed(0)
    cb = torch.randn(8192, 4, generator=g)
    x = torch.randn(20000, 4, generator=g) * 1.5
    # adversarial: exact duplicates of codes (ties) and midpoints between two codes
    x[:512] = cb[torch.randint(0, 8192, (512,), generator=g)]
    i, j = torch.randint(0, 8192, (2, 512), generator=g)
    x[512:1024] = (cb[i] + cb[j]) * 0.5
    cb[4000:4008] = cb[100:108]                     # duplicated codes: first index must win
    want = vo.vq_nearest(x, cb)
    got = ops.vq_nearest(x.to(DEV), cb.to(DEV)).cpu()
    mism = int((want != got).sum())
    _log("vq_nearest", {"n": x.shape[0], "mismatch": mism})
    assert mism == 0
    q = ops.vq_gather(got.to(DEV), cb.to(DEV)).cpu()
    assert torch.equal(q, cb[got])


def test_vq_nearest_large_roundtrip():
    """Full-size property: quantising exact codebook rows returns a code at distance 0."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(1)
    cb = torch.randn(8192, 4, device=DEV, generator=g)
    idx = torch.randint(0, 8192, (256 * 64 * 64,), device=DEV, generator=g)
    x = cb[idx]
    got = ops.vq_nearest(x, cb)
    assert torch.equal(cb[got], x)


# ------------------------------------------------------------------ wgmma GEMM
def _ref_mm(a, w):
    return a.float() @ w.float().t()


# ragged M / N edges, partial last waves on 132 SMs, every tile width the planner picks
GEMM_SHAPES = [(128, 128, 64), (256, 256, 128), (128, 64, 32), (24, 64, 40), (1000, 640, 1024), (8192, 5120, 1280),
               (2048, 1280, 5120), (32768, 640, 2560), (4100, 3840, 1280), (8192, 1280, 1280), (12032, 512, 256),
               (8100, 1272, 320), (12000, 520, 128)]


@pytest.mark.parametrize("M,N,K", GEMM_SHAPES)
def test_gemm_plain_f32_f16(M, N, K):
    from paella_b200 import _lib
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(M + N + K)
    a = (torch.randn(M, K, device=DEV, generator=g)).half()
    w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).half()
    bias = torch.randn(N, device=DEV, generator=g)
    want = _ref_mm(a, w) + bias
    out = torch.full((M, N), float("nan"), device=DEV)
    ops.gemm_f16(a, w, _lib.EPI_F32, out, bias=bias)
    torch.cuda.synchronize()
    err = float((out - want).abs().max())
    _log("gemm_f32", {"M": M, "N": N, "K": K, "max_abs_err": err, "nan": int(torch.isnan(out).sum())})
    assert err < 2e-4, err
    out16 = torch.zeros(M, N, device=DEV, dtype=torch.float16)
    ops.gemm_f16(a, w, _lib.EPI_F16, out16, bias=None)
    err16 = float((out16.float() - _ref_mm(a, w)).abs().max())
    assert err16 < 4e-3, err16      # half an fp16 ulp of |v| < 8 is 1.95e-3


@pytest.mark.parametrize("M,N,K,P", [(512, 256, 128, 64), (8192, 5120, 1280, 64), (2048, 2560, 640, 16), (300, 128, 64, 100),
                                     (256, 128, 64, 8), (384, 136, 64, 4), (128, 64, 64, 2), (2048, 5120, 1280, 16),
                                     (8192, 1280, 640, 64), (12032, 512, 256, 32)])
def test_gemm_gelu_sqsum(M, N, K, P):
    from paella_b200 import _lib
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(3)
    a = torch.randn(M, K, device=DEV, generator=g).half()
    w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).half()
    bias = torch.randn(N, device=DEV, generator=g) * 0.1
    h = torch.nn.functional.gelu(_ref_mm(a, w) + bias)
    out = torch.zeros(M, N, device=DEV, dtype=torch.float16)
    sq = torch.zeros(M // P, N, device=DEV, dtype=torch.int64)       # 2^-24 fixed point, integer atomics
    ops.gemm_f16(a, w, _lib.EPI_GELU_F16, out, bias=bias, sqsum=sq, rows_per_sample=P)
    err = float((out.float() - h).abs().max())
    want_sq = (h * h).view(M // P, P, N).sum(1)
    rel = float(((sq.double() / 2 ** 24 - want_sq).abs() / (want_sq.abs() + 1e-3)).max())
    _log("gemm_gelu", {"M": M, "N": N, "K": K, "P": P, "max_abs_err": err, "sq_rel": rel})
    assert err < 4e-3 and rel < 1e-4


@pytest.mark.parametrize("M,N,K,P", [(1024, 1280, 5120, 64), (8192, 1280, 1280, 64), (12032, 512, 256, 64)])
def test_gemm_resid_film_inplace(M, N, K, P):
    from paella_b200 import _lib
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(4)
    a = torch.randn(M, K, device=DEV, generator=g).half()
    w = (torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)).half()
    bias = torch.randn(N, device=DEV, generator=g)
    x = torch.randn(M, N, device=DEV, generator=g)
    film = torch.randn(M // P, 7 + 2 * N, device=DEV, generator=g) * 0.1
    fa, fb = film[:, 7:7 + N], film[:, 7 + N:7 + 2 * N]
    y = (_ref_mm(a, w) + bias) * 0.5 + x
    want = (y.view(M // P, P, N) * (1 + fa[:, None]) + fb[:, None]).view(M, N)
    xin = x.clone()
    # film_off must keep 16-byte alignment: use 8
    film8 = torch.zeros(M // P, 8 + 2 * N, device=DEV)
    film8[:, 8:] = film[:, 7:]
    ops.gemm_f16(a, w, _lib.EPI_RESID_F32, xin, bias=bias, resid=xin, alpha=0.5, rows_per_sample=P, film=film8, film_off=8)
    err = float((xin - want).abs().max())
    _log("gemm_resid", {"M": M, "N": N, "K": K, "max_abs_err": err})
    assert err < 1e-4


@pytest.mark.parametrize("M,C,N,P", [(8192, 1280, 3840, 64), (1024, 128, 384, 16), (300, 64, 96, 100)])
def test_gemm_layernorm_folded_across_two_gemms(M, C, N, P):
    """RESID_LN producer (fp32 x, fp16 copy, fixed-point row statistics) + F16_LN consumer:
    consumer(fp16(x)) == LayerNorm(x) @ W^T + b within the fp16-operand tolerance."""
    from paella_b200 import _lib
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(11)
    K1 = 256
    a = torch.randn(M, K1, device=DEV, generator=g).half()
    w1 = (torch.randn(C, K1, device=DEV, generator=g) / math.sqrt(K1)).half()
    b1 = torch.randn(C, device=DEV, generator=g)
    x0 = torch.randn(M, C, device=DEV, generator=g) * 2 + 0.7          # non-zero row means
    film = torch.randn(M // P if M % P == 0 else 1, 2 * C, device=DEV, generator=g) * 0.1
    use_film = M % P == 0
    y = _ref_mm(a, w1) + b1 + x0
    if use_film:
        y = (y.view(M // P, P, C) * (1 + film[:, None, :C]) + film[:, None, C:]).view(M, C)
    x = x0.clone()
    x16 = torch.full((M, C), float("nan"), device=DEV, dtype=torch.float16)
    stat = torch.zeros(M, 2, device=DEV, dtype=torch.int64)
    ops.gemm_f16(a, w1, _lib.EPI_RESID_LN_F32, x, bias=b1, resid=x, rows_per_sample=P if use_film else 0,
                 film=film if use_film else None, out16=x16, ln_stat=stat)
    assert float((x - y).abs().max()) < 5e-3
    assert torch.equal(x16, x.half())
    s_ref, q_ref = x.double().sum(1), (x.double() ** 2).sum(1)
    assert float((stat[:, 0].double() / 2 ** 20 - s_ref).abs().max()) < 1e-2
    assert float(((stat[:, 1].double() / 2 ** 16 - q_ref).abs() / q_ref).max()) < 1e-4
    # consumer
    w2 = (torch.randn(N, C, device=DEV, generator=g) / math.sqrt(C)).half()
    b2 = torch.randn(N, device=DEV, generator=g) * 0.1
    wsum = w2.float().sum(1).contiguous()
    want = torch.nn.functional.layer_norm(x, (C,), eps=1e-6) @ w2.float().t() + b2
    out = torch.full((M, N), float("nan"), device=DEV, dtype=torch.float16)
    ops.gemm_f16(x16, w2, _lib.EPI_F16_LN, out, bias=b2, ln_stat=stat, ln_wsum=wsum)
    err = float((out.float() - want).abs().max())
    rms = float((out.float() - want).pow(2).mean().sqrt())
    _log("gemm_ln_fold", {"M": M, "C": C, "N": N, "max_abs_err": err, "rms": rms})
    assert err < 6e-3 and rms < 9e-4, (err, rms)


@pytest.mark.parametrize("M,C,N,offset", [(8192, 1280, 3840, 40.0), (1024, 128, 384, 300.0)])
def test_gemm_layernorm_fold_with_row_shift_is_offset_invariant(M, C, N, offset):
    """Rows with |mean| / std = 20..150 (a residual stream carrying a large offset): with the per-row shift (here the true
    row mean perturbed by half a std, as if taken from the previous AttnBlock) the folded LayerNorm stays within the SAME
    bound as the zero-mean case; without it the fp16 copy would lose log2(ratio) bits.  Also checks the consumer's
    ln_mean_out = shift + mean' (the next block's shift)."""
    from paella_b200 import _lib
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(12)
    K1 = 256
    a = torch.randn(M, K1, device=DEV, generator=g).half()
    w1 = (torch.randn(C, K1, device=DEV, generator=g) / math.sqrt(K1)).half()
    b1 = torch.randn(C, device=DEV, generator=g)
    x0 = torch.randn(M, C, device=DEV, generator=g) * 2 + offset * (1 + 0.1 * torch.randn(M, 1, device=DEV, generator=g))
    y = _ref_mm(a, w1) + b1 + x0
    shift = (y.mean(1) + torch.randn(M, device=DEV, generator=g)).contiguous()
    x = x0.clone()
    x16 = torch.full((M, C), float("nan"), device=DEV, dtype=torch.float16)
    stat = torch.zeros(M, 2, device=DEV, dtype=torch.int64)
    ops.gemm_f16(a, w1, _lib.EPI_RESID_LN_F32, x, bias=b1, resid=x, out16=x16, ln_stat=stat, ln_shift=shift)
    assert float((x - y).abs().max()) < 1e-3 * max(1.0, offset / 40)          # the fp32 stream itself is NOT shifted
    assert torch.equal(x16, (x - shift[:, None]).half())
    w2 = (torch.randn(N, C, device=DEV, generator=g) / math.sqrt(C)).half()
    b2 = torch.randn(N, device=DEV, generator=g) * 0.1
    wsum = w2.float().sum(1).contiguous()
    want = (torch.nn.functional.layer_norm(x.double(), (C,), eps=1e-6) @ w2.double().t() + b2.double()).float()
    out = torch.full((M, N), float("nan"), device=DEV, dtype=torch.float16)
    mean_out = torch.full((M,), float("nan"), device=DEV)
    ops.gemm_f16(x16, w2, _lib.EPI_F16_LN, out, bias=b2, ln_stat=stat, ln_wsum=wsum, ln_shift=shift, ln_mean_out=mean_out)
    err = float((out.float() - want).abs().max())
    rms = float((out.float() - want).pow(2).mean().sqrt())
    mean_err = float((mean_out.double() - x.double().mean(1)).abs().max())
    _log("gemm_ln_fold_shift", {"M": M, "C": C, "N": N, "offset": offset, "max_abs_err": err, "rms": rms, "mean_err": mean_err})
    assert err < 6e-3 and rms < 9e-4, (err, rms)
    assert mean_err < 1e-3 * max(1.0, offset / 40)


def test_gemm_unpatchify_and_nchw_and_remap():
    from paella_b200 import _lib
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(6)
    B, h, w_, cin, cout = 3, 8, 8, 128, 64
    a = torch.randn(B * h * w_, cin, device=DEV, generator=g).half()
    wt = (torch.randn(4 * cout, cin, device=DEV, generator=g) / math.sqrt(cin)).half()
    bias = torch.randn(4 * cout, device=DEV, generator=g)
    y = (_ref_mm(a, wt) + bias).view(B, h, w_, 2, 2, cout)
    want = y.permute(0, 1, 3, 2, 4, 5).reshape(B, 2 * h, 2 * w_, cout)
    out = torch.zeros(B, 2 * h, 2 * w_, cout, device=DEV)
    ops.gemm_f16(a, wt, _lib.EPI_UNPATCH_F32, out, bias=bias, up=(h, w_, cout))
    assert float((out - want).abs().max()) < 2e-3
    # NCHW
    hw, N = 64, 256
    a2 = torch.randn(B * hw, cin, device=DEV, generator=g).half()
    w2 = (torch.randn(N, cin, device=DEV, generator=g) / math.sqrt(cin)).half()
    out2 = torch.zeros(B, N, hw, device=DEV)
    ops.gemm_f16(a2, w2, _lib.EPI_NCHW_F32, out2, rows_per_sample=hw)
    want2 = _ref_mm(a2, w2).view(B, hw, N).permute(0, 2, 1)
    assert float((out2 - want2).abs().max()) < 2e-3
    # row remap (byt5 rows [B*L] -> sequence rows [B*S])
    L, S = 5, 13
    a3 = torch.randn(B * L, cin, device=DEV, generator=g).half()
    out3 = torch.zeros(B * S, N, device=DEV)
    ops.gemm_f16(a3, w2, _lib.EPI_F32, out3, remap=(L, S))
    want3 = torch.zeros(B, S, N, device=DEV)
    want3[:, :L] = _ref_mm(a3, w2).view(B, L, N)
    assert float((out3.view(B, S, N) - want3).abs().max()) < 2e-3


def test_gemm_repeatable_and_back_to_back():
    """Many launches in a row (mbarrier phases, cached tensor maps) give identical results."""
    from paella_b200 import _lib
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(8)
    a = torch.randn(4096, 1280, device=DEV, generator=g).half()
    w = (torch.randn(1280, 1280, device=DEV, generator=g) / 36).half()
    outs = []
    for _ in range(5):
        o = torch.zeros(4096, 1280, device=DEV)
        ops.gemm_f16(a, w, _lib.EPI_F32, o)
        outs.append(o)
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_resample_quant_vs_torch_expression():
    """Notebook `mode='quant'` (softmax @ codebook -> nearest code) vs the same expression in torch ops."""
    ops = _ops()
    g = torch.Generator(device=DEV).manual_seed(13)
    B, K, H = 3, 8192, 16
    lc = torch.randn(B, K, H, H, device=DEV, generator=g) * 3
    lu = torch.randn(B, K, H, H, device=DEV, generator=g) * 3
    cb = torch.randn(K, 4, device=DEV, generator=g)
    cfg, T = 4.0, 0.6
    logits = lc * cfg + lu * (1 - cfg)
    e = logits.div(T).softmax(dim=1).permute(0, 2, 3, 1) @ cb                    # [B,H,H,4]
    d = torch.cdist(e.reshape(-1, 4).double(), cb.double())
    want = d.argmin(dim=1).view(B, H, H)
    got = ops.resample_quant(lc, lu, cfg, T, cb)
    agree = float((got == want).float().mean())
    _log("resample_quant", {"agree": agree})
    assert agree > 0.995
    got2 = ops.resample_quant(lc, None, 0.0, T, cb)
    want2 = torch.cdist((lc.div(T).softmax(dim=1).permute(0, 2, 3, 1) @ cb).reshape(-1, 4).double(), cb.double()).argmin(1).view(B, H, H)
    assert float((got2 == want2).float().mean()) > 0.995
