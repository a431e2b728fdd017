"""Every instantiation of the wgmma GEMM (csrc/gemm.cu) against an fp64 reference, not only the tile widths the planner picks.

The kernel is instantiated per (BLOCK_N in {64, 128, 256}, epilogue, A mode, a_scale).  PB200_FORCE_BN (read once per process)
pins the width, so each width runs in a child process; the planner's own choice runs in-process.  Every case calls
pb200_gemm_f16 through the C ABI with leading dimensions and base offsets that differ from the dense values, puts every output
inside a larger buffer prefilled with a sentinel bit pattern, and checks:
  * the product and epilogue against fp64 arithmetic on the same fp16 operands, element by element:
        |got - ref| <= gain * (TAU * sum_k |a_ik w_jk| + 8 u32 * |epilogue inputs|) + epilogue rounding + store rounding
    (u32 = 2^-24; store rounding 2^-11 |ref| for fp16 outputs, 2^-24 |ref| for fp32; gain = the epilogue's derivative);
  * that the bound can catch something: dropping the last 16 columns of K, or the last k-block, moves some element by at
    least SENS_MIN times its bound (computed from the fp64 data, so loosening TAU until the test means nothing fails here);
  * bit for bit, that nothing outside the logical outputs changed and that no sentinel is left inside them;
  * the GRN statistic (sqsum), the LayerNorm statistics (ln_stat, ln_mean_out) and the fp16 copy (out16) likewise;
  * a_scale: bit-equality with the same kernel on the pre-scaled A;  GELU + sqsum and RESID_LN: a second launch gives
    bit-identical statistics (integer atomics);
  * the im2col-free conv A modes 1 and 2 through the f4 codec against the CPU oracle (latents 2e-3, decode 1e-3).
One row per case (width, mode, error/bound, sensitivity) is appended to gemm_matrix.jsonl in $PB200_TEST_LOG_DIR (see
helpers.log_jsonl).
"""
import ctypes
import functools
import json
import math
import os
import subprocess
import sys
import tempfile
import zlib

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

# Accumulation error per unit of sum_k |a_ik w_jk|, calibrated on an H100 80GB HBM3 (700 W power limit).  At TAU = 2^-16 the
# fp32-output cases, where the accumulation term dominates the bound, reached 0.10 of it; TAU = 2^-18 keeps a 2.4x margin
# over that.  Observed worst error/bound at TAU = 2^-18: see WORST_OBSERVED (fp16 outputs sit near 1 because their bound is
# mostly the store's own half-ulp rounding, which the kernel meets exactly).
TAU = 2.0 ** -18
WORST_OBSERVED = {"fp32 outputs": 0.136, "fp16 outputs": 0.989}
SENS_MIN = 20.0
U32, U16 = 2.0 ** -24, 2.0 ** -11

MULTI_WAVE_M = 132 * 128 + 37            # 133 row tiles: every CTA walks several units and the stage ring wraps across tiles
WIDTHS = ("plan", 64, 128, 256)
STAGES = {64: 8, 128: 6, 256: 4}         # GemmSmem<BLOCK_N>::STAGES without a_scale (K = 1000 has 16 k-blocks)
MODES = {"F16": 0, "F32": 1, "GELU": 2, "RESID": 3, "UNPATCH": 4, "NCHW": 5, "RESID_LN": 6, "F16_LN": 7}
SENTINEL = {torch.float32: (torch.int32, 0x7FC0DEAD), torch.float16: (torch.int16, 0x7E5A),
            torch.int64: (torch.int64, 0x5EE55EE55EE55EE5)}


def _log(payload):
    from helpers import log_jsonl
    log_jsonl("gemm_matrix.jsonl", payload)


# ------------------------------------------------------------------ the case matrix
def _cases(width):
    """Every epilogue crossed with ragged M / N / K edges, multi-wave M and the epilogue's own options."""
    bn = 128 if width == "plan" else width
    Ns = [8, 24, 40, bn - 8, bn + 8, 3 * bn + 8]                       # N % 32 in {8, 24, 0}
    shapes = ([(129, n, 72) for n in Ns] + [(m, bn + 8, 40) for m in (1, 127, 128, 129, MULTI_WAVE_M)]
              + [(128, 3 * bn + 8, k) for k in (8, 40, 64, 72, 1000)] + [(MULTI_WAVE_M, 3 * bn + 8, 1000)])
    assert (1000 + 63) // 64 > STAGES[bn]
    cases = []

    def add(mode, M, N, K, **kw):
        tag = "-".join(f"{k}{v}" for k, v in sorted(kw.items()) if v not in (None, False))
        cases.append(dict(id=f"{mode}-M{M}-N{N}-K{K}" + (f"-{tag}" if tag else ""), mode=mode, M=M, N=N, K=K, **kw))

    gelu_p = [2, 4, 8, 16, 32, 64, 256, 48, 100]
    film_p = [64, 16, 100, 1]
    for i, (M, N, K) in enumerate(shapes):
        big = M == MULTI_WAVE_M and K == 1000
        add("F16", M, N, K, nobias=i % 2 == 1, remap=(5, 13) if i % 3 == 2 else None)
        add("F32", M, N, K, nobias=i % 2 == 0, remap=(7, 9) if i % 3 == 1 else None)
        add("GELU", M, N, K, P=gelu_p[i % len(gelu_p)], nobias=i % 4 == 3, det=big)
        add("RESID", M, N, K, alias=i % 2 == 0, alpha=[1.0, 0.5, -1.25][i % 3], nobias=i % 4 == 1,
            film=film_p[i % 4] if i % 3 != 0 else None)
        add("RESID_LN", M, N, K, alias=i % 2 == 1, alpha=[1.0, -0.75][i % 2], shift=i % 2 == 0, nobias=i % 5 == 2,
            film=film_p[(i + 1) % 4] if i % 3 != 1 else None, det=big)
        add("F16_LN", M, N, K, shift=i % 2 == 1, meanout=i % 3 != 2, nobias=i % 4 == 2)
    for j, cout in enumerate((8, 24, 64, 320)):
        for M, K in ((129, 72), (MULTI_WAVE_M, 1000) if j % 2 else (1, 8), (128, 40), (127, 128)):
            add("UNPATCH", M, 4 * cout, K, nobias=(M + j) % 2 == 1)
    for hw, B in ((45, 3), (100, 170), (7, 1), (33, 4)):
        for N, K in ((Ns[1], 72), (Ns[4], 1000), (Ns[5], 40), (Ns[0], 64)):
            add("NCHW", B * hw, N, K, P=hw, nobias=N == Ns[4])
    # GlobalResponseNorm folded into A: K % 64 == 0, samples of 16..256 rows, a_scale_ld > K
    for mode in ("RESID", "RESID_LN"):
        for P, M, K in ((16, 1000, 576), (64, 129, 64), (128, 300, 1024), (256, 700, 128), (64, MULTI_WAVE_M, 640)):
            add(mode, M, bn + 8 if P != 128 else 3 * bn + 8, K, ascale=P, alias=P == 64, film=P if P == 16 else None,
                shift=mode == "RESID_LN" and P >= 128)
    if width != "plan":
        cases += [dict(id="CONV-24x36", mode="CONV", geom=(3, 24, 36)), dict(id="CONV-256x200", mode="CONV", geom=(1, 256, 200))]
    ids = [c["id"] for c in cases]
    assert len(ids) == len(set(ids))
    return cases


# ------------------------------------------------------------------ buffers with guard bands
class _Guarded:
    """A flat buffer of `span` logical elements with spare elements before and after, all prefilled with a sentinel."""

    def __init__(self, dtype, span, pre, post):
        self.dtype, self.pre = dtype, pre
        self.buf = torch.empty(pre + span + post, dtype=dtype, device=DEV)
        itype, self.sent = SENTINEL[dtype]
        self.bits = self.buf.view(itype)
        self.bits.fill_(self.sent)

    def ptr(self):
        return self.buf.data_ptr() + self.pre * self.buf.element_size()

    def at(self, idx):
        return self.buf[self.pre + idx]

    def put(self, idx, val):
        self.buf[self.pre + idx] = val.to(self.dtype)

    def check(self, idx, name, written=True):
        inside = torch.zeros(self.buf.numel(), dtype=torch.bool, device=DEV)
        inside[self.pre + idx.reshape(-1)] = True
        n_out = int((self.bits[~inside] != self.sent).sum())
        assert n_out == 0, f"{name}: {n_out} elements outside the logical output changed"
        if written:
            n_in = int((self.bits[inside] == self.sent).sum())
            assert n_in == 0, f"{name}: {n_in} logical elements were never written"


def _rows(M, N, ld):
    return torch.arange(M, device=DEV)[:, None] * ld + torch.arange(N, device=DEV)[None, :]


def _strided(dtype, M, N, ld, seed):
    """[M, N] logical rows of stride ld, two spare rows (plus a few elements) on each side."""
    pre = 2 * ld + 8 * (1 + seed % 3)
    return _Guarded(dtype, M * ld, pre, 2 * ld + 5), _rows(M, N, ld)


def _operand(rows, cols, ld, off, gen, scale=1.0, row_offset=None):
    """fp16 [rows, cols] view with leading dimension ld at a 16-byte-aligned offset; the padding holds NaN, which would
    poison any output that read it."""
    buf = torch.full((off + rows * ld + 64,), float("nan"), dtype=torch.float16, device=DEV)
    v = buf[off:off + rows * ld].view(rows, ld)[:, :cols]
    x = torch.randn(rows, cols, device=DEV, generator=gen) * scale
    if row_offset is not None:
        x = x + row_offset
    v.copy_(x.half())
    return buf, v


# ------------------------------------------------------------------ fp64 reference
def _gelu64(x):
    return 0.5 * x * (1.0 + torch.special.erf(x / math.sqrt(2.0)))


def _epilogue64(s, acc):
    """Reference epilogue on an fp64 accumulator: (value, bound without the accumulation term, gain)."""
    mode = s["mode"]
    bias = s["bias64"]
    x = acc + bias if bias is not None else acc
    mag_in = acc.abs() + (bias.abs() if bias is not None else 0.0)
    if mode in ("F16", "F32", "UNPATCH", "NCHW"):
        return x, 8 * U32 * mag_in, 1.0
    if mode == "GELU":
        # fp32 evaluation of the GELU, plus the erfc approximation (A&S 7.1.26, |error| <= 1.5e-7, scaled by |x|/2)
        return _gelu64(x), 1.13 * 8 * U32 * mag_in + (16 * U32 + 1e-7) * x.abs(), 1.13
    if mode in ("RESID", "RESID_LN"):
        r, alpha = s["resid64"], s["alpha"]
        y = x * alpha + r
        slack = abs(alpha) * 8 * U32 * mag_in + 4 * U32 * ((x * alpha).abs() + r.abs())
        gain = abs(alpha)
        if s["film64"] is not None:
            fa, fb = s["film64"]
            y, slack, gain = y * (1 + fa) + fb, slack * (1 + fa).abs() + 4 * U32 * ((y * (1 + fa)).abs() + fb.abs()), gain * (1 + fa).abs()
        return y, slack, gain
    if mode == "F16_LN":
        mean, rstd, eps_r = s["ln64"]
        core = acc - mean[:, None] * s["wsum64"][None, :]
        y = rstd[:, None] * core
        slack = rstd[:, None] * 8 * U32 * (acc.abs() + (mean[:, None] * s["wsum64"][None, :]).abs()) + eps_r[:, None] * y.abs()
        if bias is not None:
            slack = slack + 4 * U32 * (y.abs() + bias.abs())
            y = y + bias
        return y, slack, rstd[:, None]
    raise AssertionError(mode)


def _reference(s):
    a64, w64 = s["a_eff"].double(), s["w"].double()
    K = a64.shape[1]
    acc = a64 @ w64.t()
    sabs = a64.abs() @ w64.abs().t()
    ref, slack, gain = _epilogue64(s, acc)
    store = (U16 if s["out_dtype"] == torch.float16 else U32) * ref.abs() + 2.0 ** -24
    bound = gain * TAU * sabs + slack + store
    # what the bound can see: the output with the last 16 columns of K (and the last k-block) left out
    sens = math.inf
    cuts = [max(K - 16, 0)] + ([64 * ((K - 1) // 64)] if K > 64 else [])
    for c0 in cuts:
        mut, _, _ = _epilogue64(s, acc - a64[:, c0:] @ w64[:, c0:].t())
        sens = min(sens, float(((mut - ref).abs() / bound).max()))
    pre_bound = gain * TAU * sabs + slack          # before the store's rounding (for the statistics)
    return ref, bound, pre_bound, sens


# ------------------------------------------------------------------ one case
def _launch(s):
    from paella_b200 import _lib
    ep = _lib.GemmEpilogue()
    for k, v in s["ep"].items():
        setattr(ep, k, v)
    _lib.check(_lib.lib().pb200_gemm_f16(ctypes.c_void_p(s["a"].data_ptr()), s["lda"], ctypes.c_void_p(s["w"].data_ptr()), s["ldw"],
                                         s["M"], s["N"], s["K"], ctypes.byref(ep), _lib.current_stream()), "pb200_gemm_f16")
    torch.cuda.synchronize()


def _make(c):
    """Operands, guarded outputs, the epilogue struct and the reference of case c."""
    mode, M, N, K = c["mode"], c["M"], c["N"], c["K"]
    seed = zlib.crc32(c["id"].encode())
    gen = torch.Generator(device=DEV).manual_seed(seed)
    s = dict(mode=mode, M=M, N=N, K=K, id=c["id"])
    s["lda"], s["ldw"] = K + 8 * (1 + seed % 3), K + 8 * (1 + (seed >> 3) % 2)
    row_offset = None
    if mode == "F16_LN":          # un-normalised rows with non-zero means: the folded LayerNorm has work to do
        row_offset = torch.randn(M, 1, device=DEV, generator=gen) * 0.5 + 0.3
    s["a_buf"], s["a"] = _operand(M, K, s["lda"], 8 * (1 + seed % 4), gen, row_offset=row_offset)
    s["w_buf"], s["w"] = _operand(N, K, s["ldw"], 8 * (1 + (seed >> 5) % 3), gen, scale=1.0 / math.sqrt(K))
    s["a_eff"] = s["a"]
    s["alpha"] = c.get("alpha", 1.0)
    ep = dict(mode=MODES[mode], alpha=s["alpha"])
    bias = None if c.get("nobias") else torch.randn(N, device=DEV, generator=gen) * 0.5
    s["bias"], s["bias64"] = bias, (bias.double() if bias is not None else None)
    ep["bias"] = bias.data_ptr() if bias is not None else None
    s["out_dtype"] = torch.float16 if mode in ("F16", "GELU", "F16_LN") else torch.float32
    P = c.get("P") or c.get("film") or c.get("ascale") or 0
    ep["rows_per_sample"] = P
    s["film64"], s["resid64"] = None, None
    guards = {}
    # ---- output index maps (GEMM coordinates [M, N] -> element of the output buffer)
    if mode in ("UNPATCH", "NCHW"):
        if mode == "UNPATCH":
            cout = N // 4
            p = next((d for d in range(2, 64) if M % d == 0), 1)
            h, w_ = p, M // p
            r = torch.arange(M, device=DEV)
            y, x = r // w_, r % w_
            col = torch.arange(N, device=DEV)
            q, co = col // cout, col % cout
            orow = (2 * y[:, None] + (q[None, :] >> 1)) * (2 * w_) + 2 * x[:, None] + (q[None, :] & 1)
            idx = orow * cout + co[None, :]
            ep.update(up_h=h, up_w=w_, up_cout=cout)
        else:
            hw = c["P"]
            r = torch.arange(M, device=DEV)
            idx = ((r // hw)[:, None] * N + torch.arange(N, device=DEV)[None, :]) * hw + (r % hw)[:, None]
        out = _Guarded(torch.float32, M * N, 36, 29)
    else:
        pad = 8 * (1 + seed % 2)
        ldo = N + pad
        if c.get("remap"):
            ri, ro = c["remap"]
            r = torch.arange(M, device=DEV)
            orow = (r // ri) * ro + r % ri
            rows_out = int(orow[-1]) + 1
            out = _Guarded(s["out_dtype"], rows_out * ldo, 2 * ldo + 8, 2 * ldo + 3)
            idx = orow[:, None] * ldo + torch.arange(N, device=DEV)[None, :]
            ep.update(remap_in=ri, remap_out=ro)
        else:
            out, idx = _strided(s["out_dtype"], M, N, ldo, seed)
        ep["ldo"] = ldo
    guards["out"] = (out, idx, True)
    ep["out"] = out.ptr()
    if mode in ("RESID", "RESID_LN"):
        x0 = torch.randn(M, N, device=DEV, generator=gen)
        if c.get("alias"):
            out.put(idx, x0)
            ep.update(resid=out.ptr(), ldr=ep["ldo"])
        else:
            ldr = N + 4 * (1 + seed % 3)
            rb = torch.full((8 + M * ldr + 16,), float("nan"), device=DEV)
            rb[8:8 + M * ldr].view(M, ldr)[:, :N] = x0
            s["resid_buf"] = rb
            ep.update(resid=rb.data_ptr() + 8 * 4, ldr=ldr)
        s["resid64"] = x0.double()
        if c.get("film"):
            Pf = c["film"]
            ns = (M + Pf - 1) // Pf
            off = 4 * (1 + seed % 3)
            fld = off + 2 * N + 4 * (1 + (seed >> 2) % 2)
            film = torch.full((ns, fld), float("nan"), device=DEV)
            film[:, off:off + 2 * N] = torch.randn(ns, 2 * N, device=DEV, generator=gen) * 0.3
            s["film"] = film
            rs = torch.arange(M, device=DEV) // Pf
            s["film64"] = (film[rs, off:off + N].double(), film[rs, off + N:off + 2 * N].double())
            ep.update(film=film.data_ptr(), film_ld=fld, film_off=off)
        if c.get("ascale"):
            Pa = c["ascale"]
            ns = (M + Pa - 1) // Pa
            sld = K + 8 * (1 + seed % 3)
            sb = torch.full((ns * sld + 8,), float("nan"), dtype=torch.float16, device=DEV)
            sv = sb[:ns * sld].view(ns, sld)[:, :K]
            sv.copy_((1.0 + 0.5 * torch.randn(ns, K, device=DEV, generator=gen)).half())
            s["ascale_buf"], s["ascale"] = sb, sv
            rs = torch.arange(M, device=DEV) // Pa
            s["a_eff"] = (s["a"].float() * sv.float()[rs]).half()       # HMUL2: one rounding of the exact product
            ep.update(a_scale=sb.data_ptr(), a_scale_ld=sld)
    if mode == "RESID_LN":
        # out16 is indexed with the fp32 output's ldo
        o16 = _Guarded(torch.float16, M * ep["ldo"], 2 * ep["ldo"] + 16, 2 * ep["ldo"] + 3)
        st = _Guarded(torch.int64, M * 2, 6, 5)
        st_idx = torch.arange(2 * M, device=DEV)
        st.put(st_idx, torch.zeros(2 * M, dtype=torch.int64, device=DEV))
        guards["out16"], guards["ln_stat"] = (o16, idx, True), (st, st_idx, False)
        ep.update(out16=o16.ptr(), ln_stat=st.ptr())
        if c.get("shift"):
            s["shift"] = torch.randn(M, device=DEV, generator=gen) * 2
            ep["ln_shift"] = s["shift"].data_ptr()
    if mode == "GELU":
        ns = (M + P - 1) // P
        sq = _Guarded(torch.int64, ns * N, 10, 7)
        sq_idx = torch.arange(ns * N, device=DEV)
        sq.put(sq_idx, torch.zeros(ns * N, dtype=torch.int64, device=DEV))
        guards["sqsum"] = (sq, sq_idx, False)
        ep["sqsum"] = sq.ptr()
    if mode == "F16_LN":
        a64 = s["a"].double()
        stat = torch.stack([torch.round(a64.sum(1) * 2 ** 20), torch.round((a64 * a64).sum(1) * 2 ** 16)], 1).long()
        s["stat"] = stat
        wsum = s["w"].float().sum(1)
        s["wsum"], s["wsum64"] = wsum, wsum.double()
        mean = stat[:, 0].double() / 2 ** 20 / K
        ex2 = stat[:, 1].double() / 2 ** 16 / K
        var = (ex2 - mean * mean).clamp_min(0)
        rstd = 1.0 / torch.sqrt(var + 1e-6)
        s["ln64"] = (mean, rstd, U32 * (16 + 16 * (ex2 + mean * mean) / (var + 1e-6)))
        ep.update(ln_stat=stat.data_ptr(), ln_wsum=wsum.data_ptr(), ln_c=K)
        if c.get("shift"):
            s["shift"] = torch.randn(M, device=DEV, generator=gen) * 3
            ep["ln_shift"] = s["shift"].data_ptr()
        if c.get("meanout"):
            mo = _Guarded(torch.float32, M, 4, 3)
            guards["ln_mean_out"] = (mo, torch.arange(M, device=DEV), True)
            ep["ln_mean_out"] = mo.ptr()
    s["ep"], s["guards"] = ep, guards
    s["ref"], s["bound"], s["pre_bound"], s["sens"] = _reference(s)
    return s


def _check(s, width):
    """Compare one launched case with its reference; returns the log row."""
    M, N, mode = s["M"], s["N"], s["mode"]
    out, idx, _ = s["guards"]["out"]
    for name, (g, gi, written) in s["guards"].items():
        g.check(gi, name, written)
    got = out.at(idx).double()
    assert bool(torch.isfinite(got).all()), "non-finite output"
    ratio = float(((got - s["ref"]).abs() / s["bound"]).max())
    row = dict(width=width, mode=mode, a_scale=bool(s["ep"].get("a_scale")), amode=0, M=M, N=N, K=s["K"],
               err_over_bound=ratio, sensitivity=s["sens"], case=s["id"])
    if width == "plan":
        row["block_n"] = _plan(M, N, s["K"], 0)
    assert s["sens"] >= SENS_MIN, f"the bound cannot see a dropped k16 slice / k-block (sensitivity {s['sens']:.1f})"
    if mode == "RESID_LN":
        o16, _, _ = s["guards"]["out16"]
        sh = s["shift"][:, None] if "shift" in s else 0.0
        y = out.at(idx)
        assert torch.equal(o16.at(idx), (y - sh).half()), "out16 != fp16(out - shift)"
        st, st_idx, _ = s["guards"]["ln_stat"]
        stat = st.at(st_idx).view(M, 2).double()
        d = y.double() - (s["shift"].double()[:, None] if "shift" in s else 0.0)
        nt = (N + 63) // 64
        es = (stat[:, 0] / 2 ** 20 - d.sum(1)).abs() / (16 * U32 * d.abs().sum(1) + nt * 2.0 ** -21)
        eq = (stat[:, 1] / 2 ** 16 - (d * d).sum(1)).abs() / (17 * U32 * (d * d).sum(1) + nt * 2.0 ** -17)
        row["ln_stat_ratio"] = float(max(es.max(), eq.max()))
        assert row["ln_stat_ratio"] <= 1.0, f"ln_stat off: {row['ln_stat_ratio']}"
    if mode == "GELU":
        sq, sq_idx, _ = s["guards"]["sqsum"]
        P = s["ep"]["rows_per_sample"]
        ns = (M + P - 1) // P
        h, b = s["ref"], s["pre_bound"]
        pad = ns * P - M
        hp = torch.cat([h, h.new_zeros(pad, N)]).view(ns, P, N)
        bp = torch.cat([b, b.new_zeros(pad, N)]).view(ns, P, N)
        want = (hp * hp).sum(1)
        allow = (2 * hp.abs() * bp + bp * bp).sum(1) + 16 * U32 * want + P * 2.0 ** -24
        row["sqsum_ratio"] = float(((sq.at(sq_idx).view(ns, N).double() / 2 ** 24 - want).abs() / allow).max())
        assert row["sqsum_ratio"] <= 1.0, f"sqsum off: {row['sqsum_ratio']}"
    if mode == "F16_LN" and "ln_mean_out" in s["guards"]:
        mo, mi, _ = s["guards"]["ln_mean_out"]
        mean = s["ln64"][0] + (s["shift"].double() if "shift" in s else 0.0)
        err = (mo.at(mi).double() - mean).abs()
        allow = 8 * U32 * (mean.abs() + s["ln64"][0].abs() + 1e-30)
        assert bool((err <= allow).all()), f"ln_mean_out off by {float(err.max())}"
    assert ratio <= 1.0, f"error/bound {ratio:.3g} at element {int(((got - s['ref']).abs() / s['bound']).argmax())}"
    return row


def _relaunch(s, initial, **changes):
    """Launch again from the same pre-launch buffer contents (the aliased residual among them); the buffers' bits after it."""
    for name, (g, _, _) in s["guards"].items():
        g.bits.copy_(initial[name])
    _launch(dict(s, **changes))
    return {name: g.bits.clone() for name, (g, _, _) in s["guards"].items()}


def _run_case(c, width):
    if c["mode"] == "CONV":
        return _run_conv(c, width)
    s = _make(c)
    initial = {name: g.bits.clone() for name, (g, _, _) in s["guards"].items()}
    _launch(s)
    first = {name: g.bits.clone() for name, (g, _, _) in s["guards"].items()}
    row = _check(s, width)
    if c.get("ascale"):
        # the same kernel width on the pre-scaled A: identical MMAs and accumulation order -> identical bits
        a_pre = s["a_eff"].contiguous()
        again = _relaunch(s, initial, a=a_pre, lda=s["K"], ep=dict(s["ep"], a_scale=None, a_scale_ld=0))
        for name in first:
            assert torch.equal(again[name], first[name]), f"a_scale: {name} differs from the kernel on the pre-scaled A"
        row["prescaled_bit_equal"] = True
    if c.get("det"):
        again = _relaunch(s, initial)
        for name in ("sqsum", "ln_stat"):
            if name in first:
                assert torch.equal(again[name], first[name]), f"{name} differs between two launches"
        row["deterministic"] = True
    return row


def _plan(M, N, K, sms=132):
    from paella_b200 import _lib
    bn, two, tail = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.lib().pb200_gemm_plan(M, N, K, sms, ctypes.byref(bn), ctypes.byref(two), ctypes.byref(tail)), "gemm_plan")
    return bn.value


# ------------------------------------------------------------------ conv A modes through the f4 codec
# Decode: the codec tests' 1e-3.  Latents: 2e-3 instead of their 2e-2, which a conv that lost its last 16 K columns would pass
# (it moves the latents by 4.5e-2 at most); measured 6.2e-4 at most on an H100 80GB HBM3 (700 W), at every width.
CONV_LAT_BOUND, CONV_DEC_BOUND = 2e-3, 1e-3


@functools.lru_cache(maxsize=1)
def _f4_state():
    from paella_b200.synth import rerandomize_
    from paella_b200.vqgan import VQModel
    torch.manual_seed(0)
    m = VQModel().eval()
    rerandomize_(m.state_dict(), seed=4)
    return m, {k: v.clone() for k, v in m.state_dict().items()}


def _conv_oracle(path):
    """CPU oracle of both codec geometries, once for every width: latents, indices, the decode of those indices, and how
    far the latents / the decode move when the mode-1 / mode-2 convolution loses its last 16 K columns."""
    from oracle import vqgan_oracle as vo
    _, sd = _f4_state()
    cb = sd["vquantizer.codebook.weight"]
    data = {}
    for B, H, W in ((3, 24, 36), (1, 256, 200)):
        img = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(H * W))
        lat = vo.encode_latents(sd, img)
        idx = vo.vq_nearest(lat.reshape(-1, 4), cb).view(B, H // 4, W // 4)
        dec = vo.decode_indices(sd, idx)
        cut = dict(sd)
        w1 = sd["down_blocks.1.weight"].clone()
        w1[:, -16:, 3, 3] = 0                                          # k-block order: tap-major, channels inside a tap
        cut["down_blocks.1.weight"] = w1
        w2 = sd["up_blocks.13.weight"].clone()
        w2[-16:, :, 2:, 2:] = 0                                        # the last tap of every output phase
        cut["up_blocks.13.weight"] = w2
        lat_sens = float((vo.encode_latents(cut, img) - lat).abs().max()) / CONV_LAT_BOUND
        dec_sens = float((vo.decode_indices(cut, idx) - dec).abs().max()) / CONV_DEC_BOUND
        data[f"{H}x{W}"] = dict(img=img, lat=lat, idx=idx, dec=dec, lat_sens=lat_sens, dec_sens=dec_sens)
    torch.save(data, path)


def _run_conv(c, width):
    m, _ = _f4_state()
    m = m.to(DEV)
    B, H, W = c["geom"]
    d = torch.load(os.environ["PB200_GEMM_MATRIX_ORACLE"])[f"{H}x{W}"]
    _, xs, _, _ = m.encode(d["img"].to(DEV))
    lat = (xs * m.scale_factor).permute(0, 2, 3, 1).cpu()
    dec = m.decode_indices(d["idx"].to(DEV)).cpu()
    lat_r = float((lat - d["lat"]).abs().max()) / CONV_LAT_BOUND
    dec_r = float((dec - d["dec"]).abs().max()) / CONV_DEC_BOUND
    rows = [dict(width=width, mode="F32", a_scale=False, amode=1, M=B * (H // 4) * (W // 4), case=c["id"],
                 err_over_bound=lat_r, sensitivity=d["lat_sens"]),
            dict(width=width, mode="F32", a_scale=False, amode=2, M=B * H * W // 4, case=c["id"],
                 err_over_bound=dec_r, sensitivity=d["dec_sens"])]
    rows[0]["lat_max_abs"], rows[1]["dec_max_abs"] = lat_r * CONV_LAT_BOUND, dec_r * CONV_DEC_BOUND
    for r in rows:
        assert r["sensitivity"] >= SENS_MIN, r
        assert r["err_over_bound"] <= 1.0, r
    return rows[0] | {"dec": rows[1]}


# ------------------------------------------------------------------ drivers
def _child_main(width, probe):
    """Runs in a PB200_FORCE_BN=<width> child: checks the knob is honoured, then every case of the width."""
    M, N, K = probe
    got = _plan(M, N, K, 132)
    print("PLAN", json.dumps({"probe": probe, "block_n": got}), flush=True)
    assert got == width, f"PB200_FORCE_BN={width} ignored: plan({probe}) = {got}"
    for c in _cases(width):
        try:
            row = _run_case(c, width)
            rows = [row] + ([row.pop("dec")] if "dec" in row else [])
            for r in rows:
                _log(r)
            print("RES", json.dumps({"id": c["id"], "ok": True, "row": row}), flush=True)
        except Exception as e:          # report and go on: one case's failure must not hide the others
            print("RES", json.dumps({"id": c["id"], "ok": False, "msg": f"{type(e).__name__}: {e}"}), flush=True)


PROBES = [(64, 1280, 1280), (8192, 1280, 5120), (1000, 640, 1024), (300, 640, 64), (12032, 512, 256), (24, 64, 40)]


@pytest.fixture(scope="module")
def conv_oracle():
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "conv_oracle.pt")
        _conv_oracle(path)
        os.environ["PB200_GEMM_MATRIX_ORACLE"] = path
        yield path
        os.environ.pop("PB200_GEMM_MATRIX_ORACLE", None)


_CHILD = {}


def _child_results(width, oracle_path):
    if width not in _CHILD:
        probe = next(p for p in PROBES if _plan(*p, 132) != width)      # a shape the planner would give another width
        code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_gemm_matrix as t; t._child_main(%d, %r)"
                % (ROOT, HERE, width, probe))
        env = dict(os.environ, PB200_FORCE_BN=str(width), PB200_GEMM_MATRIX_ORACLE=oracle_path)
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env)
        res = {"rc": r.returncode, "stderr": r.stderr[-3000:], "plan": None, "cases": {}}
        for line in r.stdout.splitlines():
            if line.startswith("PLAN "):
                res["plan"] = json.loads(line[5:])
            elif line.startswith("RES "):
                j = json.loads(line[4:])
                res["cases"][j["id"]] = j
        _CHILD[width] = res
    return _CHILD[width]


@pytest.mark.parametrize("width", [w for w in WIDTHS if w != "plan"])
def test_forced_width_is_honoured(width, conv_oracle):
    res = _child_results(width, conv_oracle)
    assert res["plan"] is not None, res["stderr"]
    assert res["plan"]["block_n"] == width, res
    assert res["rc"] == 0, res["stderr"]


@pytest.mark.parametrize("width,case", [(w, c["id"]) for w in WIDTHS for c in _cases(w)])
def test_gemm_instantiation(width, case, conv_oracle):
    if width == "plan":
        c = next(c for c in _cases(width) if c["id"] == case)
        _log(_run_case(c, width))
        return
    res = _child_results(width, conv_oracle)
    got = res["cases"].get(case)
    assert got is not None, f"case did not report (child rc {res['rc']}): {res['stderr']}"
    assert got["ok"], got["msg"]
