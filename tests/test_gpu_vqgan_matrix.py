"""Every VQGAN codec kernel against an fp64 reference, at every latent width, channel width and image geometry the plan accepts.

pb200_vqgan_create takes any c_hidden % 16 == 0 and any c_latent in 1..8, and the codec's kernels dispatch on exactly those
values (paella_b200/csrc/vqgan_model.cu, vq.cu, ops.cu).  COVERAGE below maps each case to the dispatch paths it runs, restated from
those conditions, and test_coverage_table asserts that every path is hit.  Every case calls the C ABI with its outputs
inside a larger buffer prefilled with a sentinel bit pattern, and checks that nothing outside the logical output changed
and no sentinel is left inside it (the uint8 image, whose every value is a legal byte, is written twice over two different
sentinels and must come out the same).

1. Quantiser (pb200_vq_nearest / pb200_vq_gather), C = 1..8, codebooks of 1, 7, 1023, 1024, 1025 and 3000 codes (the edges
   of the 1024-code shared-memory chunks), exact codes, midpoints and duplicated codes: indices bit-exact against the C
   oracle (oracle/vq_nearest.c); the gather exact, including its clamp of negative and >= k indices.
2. Codecs (bottleneck_blocks = 1) through pb200_vqgan_encode / pb200_vqgan_decode_tiled, three runs per geometry:
   * iso_enc / iso_dec: every ResBlock an exact identity (all six gammas zero: x' = fmaf(conv, 0, x), the MLP's RESID
     epilogue fmaf(v, 0, x)), the k4s2 convolution and the ConvTranspose one-hot routings, and dyadic weights and inputs,
     so that in_block, the decoder head, both convolutions and every ResBlock are exact and each element of the latents
     (latent head + BatchNorm) and of the image (out_block) is checked against fp64 with a bound of its own:
         |got - ref| <= TAU * sum |products| + U32 * (the epilogue's operands)
     Any index error in in_block, the routed convolutions or the decoder head moves an element by a multiple of 2^-7.
     Image modes 1 and 2 must equal mode 0's output clamped and converted to bytes by the same torch ops, bit for bit.
   * full: random weights and nonzero gammas against oracle/vqgan_oracle in fp64 with the fp16 operand rounding of the
     kernels (GEMM operands and weights).  The bound of a whole codec is FULL_K times the largest change that fp16
     rounding itself makes (the same oracle without it): the kernels round the same operands, so they may only differ
     where a rounding flips.  Indices bit-exact against the C oracle given the kernel's own latents, at every c_latent.
3. ResBlock front, fused (row_stats + vq_front_patch_kernel, 160 <= c <= 512) against three-launch (ln_rows +
   vq_dw_residual_kernel + ln_rows), through pb200_vqgan_resblock, in-process and in a child with
   PB200_VQ_FRONT_UNFUSED=1 (read once per process).  With gammas[5] = 0 the block returns x' itself, which both fronts
   compute with the same operations in the same order: the two must agree bit for bit.  Each front is checked against fp64
   element by element, x' with the LayerNorm and depthwise bound, the whole block adding one fp16 ulp for every GEMM
   operand whose rounding may differ (a rounding midpoint lies within the operand's own error bound).
4. Seamless tiling: pb200_vqgan_decode_tiled with per-sample wrap codes 0..3 against oracle/tiling in fp64.

Every bound is shown able to catch something: dropping one in_block input tap, one channel, one latent component or one
depthwise tap in the fp64 reference moves some element by at least SENS_MIN times its bound.  One row per case is appended
to vqgan_matrix.jsonl in $PB200_TEST_LOG_DIR (see helpers.log_jsonl).
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

# Accumulation error per unit of sum |products|, and the LayerNorm's error per unit of its normalised value, calibrated on
# an H100 80GB HBM3 (700 W power limit).  At TAU = TAU_LN = 2^-18 the worst error/bound was 0.099 (image), 0.016 (latents),
# 0.074 (x') and 0.33 (whole ResBlock, mostly its possible fp16 flips); 2^-19 keeps at least a 1.5x margin over twice that.
# FULL_K: the whole codecs came within 0.52 of the fp16 rounding effect itself.  WORST_OBSERVED: error/bound at the values
# below, all 171 cases (the file takes about a minute there).
TAU = 2.0 ** -19
TAU_LN = 2.0 ** -19
FULL_K = 1.0
WORST_OBSERVED = {"latents (iso)": 0.032, "image (iso)": 0.195, "whole codec": 0.516, "whole codec, tiled": 0.297,
                  "resblock x'": 0.138, "resblock output": 0.55}
SENS_MIN = 20.0
U32 = 2.0 ** -24
TINY = 2.0 ** -60
SENTINELS = {torch.float32: (torch.int32, (0x7FC0DEAD,)), torch.int64: (torch.int64, (0x5EE55EE55EE55EE5,)),
             torch.uint8: (torch.uint8, (0xA5, 0x5A))}


def _log(payload):
    from helpers import log_jsonl
    log_jsonl("vqgan_matrix.jsonl", payload)


def _lib():
    from paella_b200 import _lib
    return _lib


def _call(fn, *args):
    L = _lib()
    L.check(getattr(L.lib(), fn)(*args), fn)


# ------------------------------------------------------------------ outputs with guard bands
class _Out:
    """n dense elements at a 16-byte-aligned offset inside a larger buffer prefilled with a sentinel bit pattern."""

    def __init__(self, dtype, n, seed=0, sentinel=0):
        itype, sents = SENTINELS[dtype]
        self.n, self.sent = n, sents[sentinel]
        self.pre, post = 16 * (1 + seed % 3), 16 * (1 + (seed >> 2) % 2) + 3
        self.buf = torch.empty(self.pre + n + post, dtype=dtype, device=DEV)
        self.bits = self.buf.view(itype)
        self.bits.fill_(self.sent)

    def ptr(self):
        return ctypes.c_void_p(self.buf.data_ptr() + self.pre * self.buf.element_size())

    def value(self):
        return self.buf[self.pre:self.pre + self.n]

    def check(self, name, unwritten_visible=True):
        outside = torch.cat([self.bits[:self.pre], self.bits[self.pre + self.n:]])
        n_out = int((outside != self.sent).sum())
        assert n_out == 0, f"{name}: {n_out} elements outside the logical output changed"
        if unwritten_visible:
            n_in = int((self.bits[self.pre:self.pre + self.n] == self.sent).sum())
            assert n_in == 0, f"{name}: {n_in} logical elements were never written"


# ------------------------------------------------------------------ fp64 helpers
def _mm64(a, w):
    return a @ w.t()


def _mm16(a, w):
    """The tensor-core GEMMs' operands: both rounded to fp16, products summed exactly (fp64)."""
    return a.half().double() @ w.half().double().t()


def _flip16(v, e):
    """The fp16 operand-rounding term: one fp16 ulp where the kernel's value, within e of v, may round to another fp16 number
    than v does (a rounding midpoint lies within e of v), zero elsewhere (both round to the same number)."""
    r = v.half()
    inf = torch.full_like(r, float("inf"))
    hi, lo = torch.nextafter(r, inf).double(), torch.nextafter(r, -inf).double()
    rd = r.double()
    may = (v + e >= (rd + hi) / 2) | (v - e <= (rd + lo) / 2)
    return torch.where(may, torch.maximum(hi - rd, rd - lo), torch.zeros_like(v))


def _ratio(got, ref, bound):
    return float(((got.double() - ref).abs() / bound).max())


def _sens(ref, bound, *perturbed):
    """How far the bound is from missing a perturbation: min over perturbations of max |perturbed - ref| / bound."""
    return min(float(((p - ref).abs() / bound).max()) for p in perturbed)


# ------------------------------------------------------------------ 1. quantiser
VQ_KS = (1, 7, 1023, 1024, 1025, 3000)
VQ_CASES = [(c, k) for c in range(1, 9) for k in VQ_KS]


def _vq_inputs(c, k):
    seed = zlib.crc32(f"vq{c}-{k}".encode())
    g = torch.Generator().manual_seed(seed)
    n = 512 * (1 + seed % 3) + 37 * c + 11                 # never a multiple of the 512 vectors a CTA takes
    cb = torch.randn(k, c, generator=g)
    x = torch.randn(n, c, generator=g) * 1.5
    q = n // 8
    x[:q] = cb[torch.randint(0, k, (q,), generator=g)]                 # exact codes
    if k >= 2:
        i, j = torch.randint(0, k, (2, q), generator=g)
        x[q:2 * q] = (cb[i] + cb[j]) * 0.5                             # midpoints
    if k >= 16:
        cb[k - 5:k] = cb[3:8]                                          # duplicated codes: the first index must win
        x[2 * q:2 * q + 5] = cb[3:8]
    return x, cb


@pytest.mark.parametrize("c,k", VQ_CASES)
def test_vq_nearest_and_gather(c, k):
    from oracle import vqgan_oracle as vo
    assert vo._c_oracle(), "oracle/_ref/libvq_oracle.so not built"
    x, cb = _vq_inputs(c, k)
    n = x.shape[0]
    want = vo.vq_nearest(x, cb)
    xd, cbd = x.to(DEV), cb.to(DEV)
    idx = _Out(torch.int64, n, seed=c + k)
    _call("pb200_vq_nearest", ctypes.c_void_p(xd.data_ptr()), n, c, ctypes.c_void_p(cbd.data_ptr()), k, idx.ptr(),
          _lib().current_stream())
    torch.cuda.synchronize()
    idx.check("indices")
    got = idx.value().cpu()
    mism = int((got != want).sum())
    # gather: the kernel's indices plus out-of-range ones, which it clamps to [0, k)
    gi = torch.cat([got, torch.tensor([-1, -7, k, k + 5, 1 << 40, -(1 << 40)], dtype=torch.int64)])
    gd = gi.to(DEV)
    out = _Out(torch.float32, gi.numel() * c, seed=c * k)
    _call("pb200_vq_gather", ctypes.c_void_p(gd.data_ptr()), gi.numel(), ctypes.c_void_p(cbd.data_ptr()), k, c, out.ptr(),
          _lib().current_stream())
    torch.cuda.synchronize()
    out.check("gather")
    gather_ok = torch.equal(out.value().cpu().view(-1, c), cb[gi.clamp(0, k - 1)])
    _log(dict(section="quantiser", c=c, k=k, n=n, mismatch=mism, gather_exact=gather_ok))
    assert mism == 0, f"{mism} of {n} indices differ from the C oracle"
    assert gather_ok


# ------------------------------------------------------------------ 2. codec configurations
# (c_hidden, c_latent, codebook size, encode geometries (B, H, W), decode-only latent grids (B, h, w))
CONFIGS = [
    dict(ch=48, cl=3, k=1025, enc=[(2, 4, 4), (1, 8, 512), (3, 20, 28)], dec=[(1, 2, 128)]),
    dict(ch=160, cl=5, k=3000, enc=[(1, 4, 12), (2, 12, 8)], dec=[(3, 5, 7)]),
    dict(ch=192, cl=1, k=7, enc=[(3, 24, 36), (1, 4, 4)], dec=[(1, 2, 128)]),
    dict(ch=544, cl=8, k=1024, enc=[(2, 20, 28)], dec=[(1, 3, 17)]),
    dict(ch=1536, cl=2, k=1023, enc=[(1, 12, 8)], dec=[(2, 2, 5)]),
    dict(ch=1600, cl=4, k=64, enc=[(2, 4, 12)], dec=[(1, 3, 3)]),
]
WRAP_CODES = (3, 0, 1, 2)


def _codec_cases():
    cases = []
    for cfg in CONFIGS:
        name = f"ch{cfg['ch']}-cl{cfg['cl']}"
        for B, H, W in cfg["enc"]:
            for kind in ("iso_enc", "iso_dec", "full"):
                cases.append(dict(cfg, id=f"{name}-{kind}-B{B}-{H}x{W}", kind=kind, B=B, h=H // 4, w=W // 4))
        for B, h, w in cfg["dec"]:
            cases.append(dict(cfg, id=f"{name}-iso_dec-B{B}-{4 * h}x{4 * w}", kind="iso_dec", B=B, h=h, w=w))
        B, h, w = cfg["dec"][0]
        cases.append(dict(cfg, id=f"{name}-tiled-B4-{4 * h}x{4 * w}", kind="tiled", B=4, h=h, w=w))
    return cases


CODEC_CASES = _codec_cases()


def _shapes(ch, cl, k):
    c0, c1 = ch // 2, ch
    s = {"in_block.1.weight": (c0, 12, 1, 1), "in_block.1.bias": (c0,)}

    def res(pre, c):
        s.update({pre + "depthwise.1.weight": (c, 1, 3, 3), pre + "depthwise.1.bias": (c,), pre + "channelwise.0.weight": (4 * c, c),
                  pre + "channelwise.0.bias": (4 * c,), pre + "channelwise.2.weight": (c, 4 * c), pre + "channelwise.2.bias": (c,),
                  pre + "gammas": (6,)})
    res("down_blocks.0.", c0)
    s["down_blocks.1.weight"], s["down_blocks.1.bias"] = (c1, c0, 4, 4), (c1,)
    res("down_blocks.2.", c1)
    s["down_blocks.3.0.weight"] = (cl, c1, 1, 1)
    for n in ("weight", "bias", "running_mean", "running_var"):
        s["down_blocks.3.1." + n] = (cl,)
    s["vquantizer.codebook.weight"] = (k, cl)
    s["up_blocks.0.0.weight"], s["up_blocks.0.0.bias"] = (c1, cl, 1, 1), (c1,)
    res("up_blocks.1.", c1)
    s["up_blocks.2.weight"], s["up_blocks.2.bias"] = (c1, c0, 4, 4), (c0,)
    res("up_blocks.3.", c0)
    s["out_block.0.weight"], s["out_block.0.bias"] = (12, c0, 1, 1), (12,)
    return s


def _random_sd(ch, cl, k, gen):
    """Random codec weights (fp32 values, held in fp64) with nonzero gammas."""
    sd = {}
    for n, shp in _shapes(ch, cl, k).items():
        r = torch.randn(shp, generator=gen)
        if n.endswith("gammas"):
            v = r * 0.5
        elif n.endswith("running_var"):
            v = torch.rand(shp, generator=gen) + 0.5
        elif n.startswith("down_blocks.3.1.weight"):
            v = 1 + 0.2 * r
        elif n == "vquantizer.codebook.weight":
            v = r
        elif n == "out_block.0.bias":
            v = 0.5 + 0.1 * r
        elif len(shp) == 1:
            v = 0.1 * r
        elif "depthwise" in n:
            v = 0.3 * r
        elif n == "up_blocks.2.weight":
            v = r / math.sqrt(4 * shp[0])                  # ConvTranspose: 4 taps per output phase
        elif n == "out_block.0.weight":
            v = 0.3 * r / math.sqrt(shp[1])
        else:
            v = r / math.sqrt(r[0].numel())
        sd[n] = v.float().double()
    return sd


def _dyadic(shp, gen, num, den):
    return torch.randint(-num, num + 1, shp, generator=gen).double() / den


def _iso_sd(ch, cl, k, gen):
    """Identity ResBlocks and one-hot routed convolutions, with dyadic weights where the values stay exact."""
    c0, c1 = ch // 2, ch
    sd = _random_sd(ch, cl, k, gen)
    for n in sd:
        if n.endswith("gammas"):
            sd[n] = torch.zeros(6, dtype=torch.float64)
    # k4s2 conv: output channel co carries input channel co % c0 at input phase p = (ci + 2 (co // c0)) % 4 (tap (1 + p/2,
    # 1 + p%2) reads (2y + p/2, 2x + p%2)): every channel is seen at two phases, every phase for half the channels
    co = torch.arange(c1)
    ci = co % c0
    p = (ci + 2 * (co // c0)) % 4
    w = torch.zeros(c1, c0, 4, 4, dtype=torch.float64)
    w[co, ci, 1 + p // 2, 1 + p % 2] = 1.0
    sd["down_blocks.1.weight"] = w
    sd["down_blocks.1.bias"] = _dyadic((c1,), gen, 8, 8)
    sd["in_block.1.weight"] = _dyadic((c0, 12, 1, 1), gen, 8, 8)
    sd["in_block.1.bias"] = _dyadic((c0,), gen, 8, 8)
    # ConvTranspose: output channel co of phase ph = 2 py + px is input channel (2 co + ph) % c1 through tap (1 + py, 1 + px),
    # the tap of that phase that reads input position (y, x)
    wt = torch.zeros(c1, c0, 4, 4, dtype=torch.float64)
    o = torch.arange(c0)
    for ph in range(4):
        wt[(2 * o + ph) % c1, o, 1 + ph // 2, 1 + ph % 2] = 1.0
    sd["up_blocks.2.weight"] = wt
    sd["up_blocks.2.bias"] = _dyadic((c0,), gen, 8, 8)
    sd["up_blocks.0.0.weight"] = _dyadic((c1, cl, 1, 1), gen, 8, 8)
    sd["up_blocks.0.0.bias"] = _dyadic((c1,), gen, 8, 8)
    return sd


# ---- fp64 codec references (the kernels' rounding points: `mm` for the tensor-core GEMMs; in_block, the latent head, the
# decoder head and out_block are fp32 CUDA-core kernels, fp64 here)
def _bn_scale(sd):
    """BatchNorm's scale as the latent head computes it in fp32: bn_w / sqrtf(var + 1e-5f)."""
    bn = "down_blocks.3.1."
    return (sd[bn + "weight"].float() / torch.sqrt(sd[bn + "running_var"].float() + 1e-5)).double()


def _encode_ref(sd, img, mm):
    """-> latents NHWC, the latent head's pre-BN output v and its input x1."""
    from oracle import vqgan_oracle as vo
    x = vo.pixel_unshuffle2(img.permute(0, 2, 3, 1))
    w = sd["in_block.1.weight"]
    x = _mm64(x, w.reshape(w.shape[0], -1)) + sd["in_block.1.bias"]
    x = vo.vq_resblock(x, sd, "down_blocks.0.", mm)
    x = vo.conv_k4s2p1(x, sd["down_blocks.1.weight"], sd["down_blocks.1.bias"], mm)
    x1 = vo.vq_resblock(x, sd, "down_blocks.2.", mm)
    w = sd["down_blocks.3.0.weight"]
    v = _mm64(x1, w.reshape(w.shape[0], -1))
    bn = "down_blocks.3.1."
    return (v - sd[bn + "running_mean"]) * _bn_scale(sd) + sd[bn + "bias"], v, x1


def _decode_ref(sd, z, mm, wrap=(False, False)):
    """NHWC latents -> (image NCHW, out_block's input NHWC).  oracle/tiling with no wrap is oracle/vqgan_oracle."""
    from oracle import tiling as ot
    from oracle import vqgan_oracle as vo
    w = sd["up_blocks.0.0.weight"]
    x = _mm64(z, w.reshape(w.shape[0], -1)) + sd["up_blocks.0.0.bias"]
    x = ot.vq_resblock(x, sd, "up_blocks.1.", wrap, mm)
    x = ot.convT_k4s2p1_wrap(x, sd["up_blocks.2.weight"], sd["up_blocks.2.bias"], wrap, mm)
    xa = ot.vq_resblock(x, sd, "up_blocks.3.", wrap, mm)
    w = sd["out_block.0.weight"]
    y = _mm64(xa, w.reshape(12, -1)) + sd["out_block.0.bias"]
    return vo.pixel_shuffle2(y).permute(0, 3, 1, 2).contiguous(), xa


def _to_img(y_nhwc12):
    from oracle import vqgan_oracle as vo
    return vo.pixel_shuffle2(y_nhwc12).permute(0, 3, 1, 2).contiguous()


# ---- the codec through the C ABI
class _Codec:
    def __init__(self, ch, cl, k):
        L = _lib()
        cfg = L.VqganConfig(levels=2, bottleneck_blocks=1, c_hidden=ch, c_latent=cl, codebook_size=k, scale_factor=0.3764)
        self.h = ctypes.c_void_p()
        _call("pb200_vqgan_create", ctypes.byref(cfg), ctypes.byref(self.h))
        lib = L.lib()
        self.blob = torch.zeros(lib.pb200_vqgan_weight_bytes(self.h), dtype=torch.uint8, device=DEV)
        _call("pb200_vqgan_bind_weights", self.h, ctypes.c_void_p(self.blob.data_ptr()))
        self.names = [lib.pb200_vqgan_param_name(self.h, i).decode() for i in range(lib.pb200_vqgan_num_params(self.h))]
        self.cl = cl
        assert set(self.names) == set(_shapes(ch, cl, k)), "the plan's parameters are not the codec's state dict"

    def load(self, sd):
        src = []
        for n in self.names:
            t = sd[n].float().contiguous().to(DEV)
            src.append(t)
            _call("pb200_vqgan_load_param", self.h, n.encode(), ctypes.c_void_p(t.data_ptr()), t.numel(), _lib().current_stream())
        _call("pb200_vqgan_sync_params", self.h, _lib().current_stream())
        torch.cuda.synchronize()

    def _ws(self, B, H, W):
        return torch.empty(_lib().lib().pb200_vqgan_workspace_bytes(self.h, B, H, W), dtype=torch.uint8, device=DEV)

    def encode(self, img, seed):
        """-> latents NCHW, quantised NCHW, indices [B,h,w] (each checked for its guard bands)."""
        B, _, H, W = img.shape
        cl, h, w = self.cl, H // 4, W // 4
        lat, q, idx = _Out(torch.float32, B * cl * h * w, seed), _Out(torch.float32, B * cl * h * w, seed + 1), \
            _Out(torch.int64, B * h * w, seed + 2)
        ws = self._ws(B, H, W)
        img = img.to(DEV).float().contiguous()
        _call("pb200_vqgan_encode", self.h, ctypes.c_void_p(img.data_ptr()), B, H, W, lat.ptr(), q.ptr(), idx.ptr(),
              ctypes.c_void_p(ws.data_ptr()), ws.numel(), _lib().current_stream())
        torch.cuda.synchronize()
        for o, name in ((lat, "latents"), (q, "quantised"), (idx, "indices")):
            o.check(name)
        return (lat.value().view(B, cl, h, w).cpu(), q.value().view(B, cl, h, w).cpu(), idx.value().view(B, h, w).cpu())

    def decode(self, B, h, w, mode, seed, latents=None, indices=None, wrap=None):
        """Image of one mode: fp32 NCHW (modes 0, 1) or uint8 NHWC (mode 2, decoded over two sentinels)."""
        lat = latents.to(DEV).float().contiguous() if latents is not None else None
        idx = indices.to(DEV).contiguous() if indices is not None else None
        wr = torch.tensor(wrap, dtype=torch.uint8, device=DEV) if wrap is not None else None
        n = B * 3 * 16 * h * w
        outs = []
        for sentinel in ((0, 1) if mode == 2 else (0,)):
            img = _Out(torch.uint8 if mode == 2 else torch.float32, n, seed, sentinel)
            ws = self._ws(B, 4 * h, 4 * w)
            _call("pb200_vqgan_decode_tiled", self.h, ctypes.c_void_p(idx.data_ptr()) if idx is not None else None,
                  ctypes.c_void_p(lat.data_ptr()) if lat is not None else None, B, h, w, img.ptr(), mode,
                  ctypes.c_void_p(wr.data_ptr()) if wr is not None else None, ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                  _lib().current_stream())
            torch.cuda.synchronize()
            img.check(f"image mode {mode}", unwritten_visible=mode != 2)
            outs.append(img.value().cpu())
        if mode == 2:
            assert torch.equal(outs[0], outs[1]), "uint8 image: some bytes were never written (they differ with the sentinel)"
            return outs[0].view(B, 4 * h, 4 * w, 3)
        return outs[0].view(B, 3, 4 * h, 4 * w)


@functools.lru_cache(maxsize=None)
def _codec(ch, cl, k):
    return _Codec(ch, cl, k)


def _check_modes(cod, B, h, w, seed, img0, **src):
    """Modes 1 and 2 == mode 0 clamped, and converted to bytes as torch does it in fp32."""
    clamped = img0.clamp(0, 1)
    assert torch.equal(cod.decode(B, h, w, 1, seed + 5, **src), clamped), "mode 1 != clamp(mode 0, 0, 1)"
    u8 = clamped.mul(255).add(0.5).clamp(0, 255).permute(0, 2, 3, 1).to(torch.uint8)
    assert torch.equal(cod.decode(B, h, w, 2, seed + 6, **src), u8), "mode 2 != save_image bytes of clamp(mode 0)"


def _run_iso_enc(c, cod, gen, seed):
    ch, cl, k, B, h, w = c["ch"], c["cl"], c["k"], c["B"], c["h"], c["w"]
    from oracle import vqgan_oracle as vo
    sd = _iso_sd(ch, cl, k, gen)
    cod.load(sd)
    img = torch.randint(0, 17, (B, 3, 4 * h, 4 * w), generator=gen).double() / 16
    lat, q, idx = cod.encode(img, seed)
    ref, v, x1 = _encode_ref(sd, img, _mm16)
    W = sd["down_blocks.3.0.weight"].reshape(cl, -1)
    bn = "down_blocks.3.1."
    sc, mean, b = _bn_scale(sd), sd[bn + "running_mean"], sd[bn + "bias"]
    S = x1.abs() @ W.abs().t()
    bound = sc.abs() * (TAU * S + U32 * (v.abs() + mean.abs())) + 2 * U32 * (((v - mean) * sc).abs() + b.abs()) + TINY
    got = lat.permute(0, 2, 3, 1)
    ratio = _ratio(got, ref, bound)
    cut_tap = dict(sd)
    wi = sd["in_block.1.weight"].clone()
    wi[:, 11] = 0
    cut_tap["in_block.1.weight"] = wi
    cut_ch = dict(sd)
    wl = sd["down_blocks.3.0.weight"].clone()
    wl[:, -1] = 0
    cut_ch["down_blocks.3.0.weight"] = wl
    sens = _sens(ref, bound, _encode_ref(cut_tap, img, _mm16)[0], _encode_ref(cut_ch, img, _mm16)[0])
    cb = sd["vquantizer.codebook.weight"].float()
    want_idx = vo.vq_nearest(got.reshape(-1, cl), cb).view(B, h, w)
    assert torch.equal(idx, want_idx), f"{int((idx != want_idx).sum())} indices differ from the C oracle on the kernel's latents"
    assert torch.equal(q.permute(0, 2, 3, 1), cb[idx]), "quantised != codebook[indices]"
    assert sens >= SENS_MIN, f"the latent bound cannot see a dropped in_block tap / latent-head channel ({sens:.1f})"
    assert ratio <= 1.0, f"latents: error/bound {ratio:.3g}"
    return dict(bound="iso_latents", err_over_bound=ratio, sensitivity=sens)


def _run_iso_dec(c, cod, gen, seed):
    ch, cl, k, B, h, w = c["ch"], c["cl"], c["k"], c["B"], c["h"], c["w"]
    sd = _iso_sd(ch, cl, k, gen)
    cod.load(sd)
    z = torch.randint(-4, 5, (B, cl, h, w), generator=gen).double() / 4
    img0 = cod.decode(B, h, w, 0, seed, latents=z)
    zn = z.permute(0, 2, 3, 1)
    ref, xa = _decode_ref(sd, zn, _mm16)
    W, bo = sd["out_block.0.weight"].reshape(12, -1), sd["out_block.0.bias"]
    y = _mm64(xa, W) + bo
    bound = _to_img(TAU * (xa.abs() @ W.abs().t()) + 2 * U32 * (bo.abs() + y.abs())) + TINY
    ratio = _ratio(img0, ref, bound)
    zc = zn.clone()
    zc[..., -1] = 0
    cut_ch = dict(sd)
    wo = sd["out_block.0.weight"].clone()
    wo[:, -1] = 0
    cut_ch["out_block.0.weight"] = wo
    sens = _sens(ref, bound, _decode_ref(sd, zc, _mm16)[0], _decode_ref(cut_ch, zn, _mm16)[0])
    _check_modes(cod, B, h, w, seed, img0, latents=z)
    assert sens >= SENS_MIN, f"the image bound cannot see a dropped latent component / out_block channel ({sens:.1f})"
    assert ratio <= 1.0, f"image: error/bound {ratio:.3g}"
    frac = float(((img0 > 0) & (img0 < 1)).double().mean())
    return dict(bound="iso_image", err_over_bound=ratio, sensitivity=sens, unclamped_fraction=frac)


def _full_bound(ref16, ref64):
    return FULL_K * float((ref16 - ref64).abs().max()) + U32 * float(ref16.abs().max()) + TINY


def _run_full(c, cod, gen, seed):
    ch, cl, k, B, h, w = c["ch"], c["cl"], c["k"], c["B"], c["h"], c["w"]
    from oracle import vqgan_oracle as vo
    sd = _random_sd(ch, cl, k, gen)
    cod.load(sd)
    img = torch.rand(B, 3, 4 * h, 4 * w, generator=gen).float().double()
    lat, q, idx = cod.encode(img, seed)
    got = lat.permute(0, 2, 3, 1)
    ref16, ref64 = _encode_ref(sd, img, _mm16)[0], _encode_ref(sd, img, _mm64)[0]
    lb = _full_bound(ref16, ref64)
    lat_ratio = float((got.double() - ref16).abs().max()) / lb
    cut = dict(sd)
    wi = sd["in_block.1.weight"].clone()
    wi[:, 11] = 0
    cut["in_block.1.weight"] = wi
    lat_sens = float((_encode_ref(cut, img, _mm16)[0] - ref16).abs().max()) / lb
    cb = sd["vquantizer.codebook.weight"].float()
    want_idx = vo.vq_nearest(got.reshape(-1, cl), cb).view(B, h, w)
    assert torch.equal(idx, want_idx), f"{int((idx != want_idx).sum())} indices differ from the C oracle on the kernel's latents"
    assert torch.equal(q.permute(0, 2, 3, 1), cb[idx]), "quantised != codebook[indices]"
    # decode the kernel's indices (the codec's own gather)
    img0 = cod.decode(B, h, w, 0, seed + 9, indices=idx)
    zn = sd["vquantizer.codebook.weight"][idx]
    d16, d64 = _decode_ref(sd, zn, _mm16)[0], _decode_ref(sd, zn, _mm64)[0]
    db = _full_bound(d16, d64)
    dec_ratio = float((img0.double() - d16).abs().max()) / db
    zc = zn.clone()
    zc[..., -1] = 0
    dec_sens = float((_decode_ref(sd, zc, _mm16)[0] - d16).abs().max()) / db
    _check_modes(cod, B, h, w, seed + 9, img0, indices=idx)
    assert min(lat_sens, dec_sens) >= SENS_MIN, f"sensitivity latents {lat_sens:.1f}, image {dec_sens:.1f}"
    assert lat_ratio <= 1.0 and dec_ratio <= 1.0, f"error/bound latents {lat_ratio:.3g}, image {dec_ratio:.3g}"
    return dict(bound="full", err_over_bound=max(lat_ratio, dec_ratio), latents_ratio=lat_ratio, image_ratio=dec_ratio,
                sensitivity=min(lat_sens, dec_sens), latents_max_abs=lat_ratio * lb, image_max_abs=dec_ratio * db)


def _run_tiled(c, cod, gen, seed):
    ch, cl, k, B, h, w = c["ch"], c["cl"], c["k"], c["B"], c["h"], c["w"]
    sd = _random_sd(ch, cl, k, gen)
    cod.load(sd)
    codes = [WRAP_CODES[(i + seed) % 4] for i in range(B)]
    z = torch.randn(B, cl, h, w, generator=gen).float().double()
    img0 = cod.decode(B, h, w, 0, seed, latents=z, wrap=codes)
    zn = z.permute(0, 2, 3, 1)
    ratio, sens = 0.0, math.inf
    for b, code in enumerate(codes):
        wrap = (bool(code & 1), bool(code & 2))
        r16 = _decode_ref(sd, zn[b:b + 1], _mm16, wrap)[0]
        bound = _full_bound(r16, _decode_ref(sd, zn[b:b + 1], _mm64, wrap)[0])
        ratio = max(ratio, float((img0[b:b + 1].double() - r16).abs().max()) / bound)
        zc = zn[b:b + 1].clone()
        zc[..., -1] = 0
        sens = min(sens, float((_decode_ref(sd, zc, _mm16, wrap)[0] - r16).abs().max()) / bound)
    u8 = cod.decode(B, h, w, 2, seed + 3, latents=z, wrap=codes)
    assert torch.equal(u8, img0.clamp(0, 1).mul(255).add(0.5).clamp(0, 255).permute(0, 2, 3, 1).to(torch.uint8))
    assert sens >= SENS_MIN, f"the tiled image bound cannot see a dropped latent component ({sens:.1f})"
    assert ratio <= 1.0, f"tiled image: error/bound {ratio:.3g}"
    return dict(bound="full_tiled", err_over_bound=ratio, sensitivity=sens, wrap=codes)


@pytest.mark.parametrize("case", [c["id"] for c in CODEC_CASES])
def test_codec(case):
    c = next(c for c in CODEC_CASES if c["id"] == case)
    seed = zlib.crc32(case.encode())
    gen = torch.Generator().manual_seed(seed)
    cod = _codec(c["ch"], c["cl"], c["k"])
    run = {"iso_enc": _run_iso_enc, "iso_dec": _run_iso_dec, "full": _run_full, "tiled": _run_tiled}[c["kind"]]
    row = run(c, cod, gen, seed % 1000)
    _log(dict(section="codec", case=case, paths=sorted(p for p, ids in COVERAGE.items() if case in ids), **row))


# ------------------------------------------------------------------ 3. ResBlock front, fused against three-launch
FRONT_CS = (8, 24, 152, 160, 256, 264, 512, 520)
FRONT_HW = ((1, 1), (1, 9), (2, 8), (3, 17), (9, 16))
FRONT_CASES = [dict(id=f"c{c}-B{B}-{h}x{w}", c=c, B=B, h=h, w=w) for c in FRONT_CS for (h, w) in FRONT_HW for B in (1, 3)]


def _front_inputs(fc):
    c, B, h, w = fc["c"], fc["B"], fc["h"], fc["w"]
    g = torch.Generator().manual_seed(zlib.crc32(fc["id"].encode()))
    p = dict(x=(torch.randn(B, h, w, c, generator=g) * 1.5 + torch.randn(B, h, w, 1, generator=g)).double(),
             dw_w=(0.3 * torch.randn(c, 1, 3, 3, generator=g)).double(), dw_b=(0.1 * torch.randn(c, generator=g)).double(),
             w1=(torch.randn(4 * c, c, generator=g) / math.sqrt(c)).half().double(),
             b1=(0.1 * torch.randn(4 * c, generator=g)).double(),
             w2=(torch.randn(c, 4 * c, generator=g) / math.sqrt(4 * c)).half().double(),
             b2=(0.1 * torch.randn(c, generator=g)).double(),
             gam=((0.5 + 0.5 * torch.rand(6, generator=g)) * torch.randn(6, generator=g).sign()).double())
    return p


def _front_launch(p, gam):
    B, h, w, c = p["x"].shape
    x = _Out(torch.float32, B * h * w * c, seed=c + h)
    x.value().copy_(p["x"].float().reshape(-1))
    dev = {k: p[k].to(DEV) for k in ("dw_b", "b1", "b2")}
    w9 = p["dw_w"].reshape(c, 9).t().contiguous().float().to(DEV)
    w1, w2 = p["w1"].half().to(DEV), p["w2"].half().to(DEV)
    f = {k: v.float() for k, v in dev.items()}
    L = _lib()
    ws = torch.empty(L.lib().pb200_vqgan_resblock_workspace_bytes(B, h, w, c), dtype=torch.uint8, device=DEV)
    gh = (ctypes.c_float * 6)(*[float(v) for v in gam])
    vp = lambda t: ctypes.c_void_p(t.data_ptr())
    _call("pb200_vqgan_resblock", x.ptr(), B, h, w, c, vp(w9), vp(f["dw_b"]), vp(w1), vp(f["b1"]), vp(w2), vp(f["b2"]), gh, vp(ws),
          ws.numel(), L.current_stream())
    torch.cuda.synchronize()
    x.check("resblock output")
    return x.value().view(B, h, w, c).cpu()


def _ln(x):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-6), 1.0 / torch.sqrt(var + 1e-6)


def _front_ref(p, gam, dw_w=None):
    """fp64 block with the kernels' fp16 GEMM operands -> (x', its bound, out, its bound)."""
    from oracle import vqgan_oracle as vo
    from oracle.paella_oracle import gelu_erf
    x, dw_w = p["x"], (p["dw_w"] if dw_w is None else dw_w)
    g = [float(v) for v in gam]
    n, _ = _ln(x)
    t = n * (1 + g[0]) + g[1]
    e_t = TAU_LN * ((n.abs() + 1) * abs(1 + g[0]) + abs(g[1]))
    conv = vo.dwconv3x3_replicate(t, dw_w, p["dw_b"])
    s_conv = vo.dwconv3x3_replicate(t.abs(), dw_w.abs(), p["dw_b"].abs())
    e_conv = TAU * s_conv + vo.dwconv3x3_replicate(e_t, dw_w.abs(), torch.zeros_like(p["dw_b"]))
    xp = x + g[2] * conv
    e_xp = abs(g[2]) * e_conv + U32 * (xp.abs() + abs(g[2]) * conv.abs()) + TINY
    n2, rstd2 = _ln(xp)
    a = n2 * (1 + g[3]) + g[4]
    e_a = TAU_LN * ((n2.abs() + 1) * abs(1 + g[3]) + abs(g[4])) + abs(1 + g[3]) * rstd2 * e_xp
    a16 = a.half().double()
    z1 = a16 @ p["w1"].t() + p["b1"]
    e_z1 = TAU * (a16.abs() @ p["w1"].abs().t() + p["b1"].abs()) + _flip16(a, e_a) @ p["w1"].abs().t()
    hh = gelu_erf(z1)
    e_h = 1.13 * e_z1 + (16 * U32 + 1e-7) * z1.abs()
    h16 = hh.half().double()
    z2 = h16 @ p["w2"].t() + p["b2"]
    e_z2 = TAU * (h16.abs() @ p["w2"].abs().t() + p["b2"].abs()) + _flip16(hh, e_h) @ p["w2"].abs().t()
    out = xp + g[5] * z2
    e_out = e_xp + abs(g[5]) * e_z2 + 2 * U32 * (out.abs() + abs(g[5]) * z2.abs()) + TINY
    return xp, e_xp, out, e_out


def _front_case(fc):
    """Both gamma settings of one case: (x' bits with gammas[5] = 0, log row)."""
    p = _front_inputs(fc)
    cut = p["dw_w"].clone()
    cut[:, 0, 2, 2] = 0                                  # the last depthwise tap
    row = {}
    gam0 = p["gam"].clone()
    gam0[5] = 0
    got0 = _front_launch(p, gam0)
    xp, e_xp, _, _ = _front_ref(p, gam0)
    row["x_ratio"] = _ratio(got0, xp, e_xp)
    row["x_sens"] = _sens(xp, e_xp, _front_ref(p, gam0, cut)[0])
    got = _front_launch(p, p["gam"])
    _, _, out, e_out = _front_ref(p, p["gam"])
    row["block_ratio"] = _ratio(got, out, e_out)
    row["block_sens"] = _sens(out, e_out, _front_ref(p, p["gam"], cut)[2])
    assert bool(torch.isfinite(got).all()) and bool(torch.isfinite(got0).all())
    assert min(row["x_sens"], row["block_sens"]) >= SENS_MIN, row
    assert row["x_ratio"] <= 1.0 and row["block_ratio"] <= 1.0, row
    return got0, row


def _front_child_main(path):
    """Runs with PB200_VQ_FRONT_UNFUSED=1: every front case on the three-launch path; x' bits (gammas[5] = 0) to `path`."""
    bits = {}
    for fc in FRONT_CASES:
        try:
            got0, row = _front_case(fc)
            bits[fc["id"]] = got0
            print("RES", json.dumps({"id": fc["id"], "ok": True, "row": row}), flush=True)
        except Exception as e:          # report and go on: one case's failure must not hide the others
            print("RES", json.dumps({"id": fc["id"], "ok": False, "msg": f"{type(e).__name__}: {e}"}), flush=True)
    torch.save(bits, path)


@pytest.fixture(scope="module")
def unfused():
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "unfused.pt")
        code = ("import sys; sys.path[:0] = [%r, %r]; import test_gpu_vqgan_matrix as t; t._front_child_main(%r)"
                % (ROOT, HERE, path))
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True,
                           env=dict(os.environ, PB200_VQ_FRONT_UNFUSED="1"))
        res = {"rc": r.returncode, "stderr": r.stderr[-3000:], "cases": {}, "bits": {}}
        for line in r.stdout.splitlines():
            if line.startswith("RES "):
                j = json.loads(line[4:])
                res["cases"][j["id"]] = j
        if os.path.exists(path):
            res["bits"] = torch.load(path)
        yield res


def _fused(c, h, w):
    """ops.cu vq_front_fused_ok: the fused front takes 160 <= c <= 512."""
    return c % 4 == 0 and 160 <= c <= 512 and h >= 1 and w >= 1


@pytest.mark.parametrize("case", [fc["id"] for fc in FRONT_CASES])
def test_resblock_front(case, unfused):
    fc = next(f for f in FRONT_CASES if f["id"] == case)
    got0, row = _front_case(fc)
    child = unfused["cases"].get(case)
    assert child is not None, f"case did not report (child rc {unfused['rc']}): {unfused['stderr']}"
    fused = _fused(fc["c"], fc["h"], fc["w"])
    _log(dict(section="front", case=case, front="fused" if fused else "three-launch", **row))
    _log(dict(section="front", case=case, front="three-launch (PB200_VQ_FRONT_UNFUSED)", **child.get("row", {})))
    assert child["ok"], child["msg"]
    other = unfused["bits"][case]
    n_diff = int((got0.view(torch.int32) != other.view(torch.int32)).sum())
    assert n_diff == 0, f"x' differs between the {'fused' if fused else 'three-launch'} front and the three-launch one " \
                        f"in {n_diff} elements (max {float((got0 - other).abs().max()):.3g})"


# ------------------------------------------------------------------ coverage table
# Each dispatch path of the codec (the conditions restated from vqgan_model.cu, vq.cu and ops.cu) -> the cases that run it.
def _front_paths(c, h, w):
    if not _fused(c, h, w):
        return {"front three-launch (ln_rows + vq_dw_residual_kernel + ln_rows)"}
    return {"front fused, 64 threads (vq_front_patch_kernel<64,6>)" if (c // 4 + 31) // 32 * 32 <= 64
            else "front fused, 128 threads (vq_front_patch_kernel<128,3>)"}


def _codec_paths(c):
    ch, cl, kind, h, w = c["ch"], c["cl"], c["kind"], c["h"], c["w"]
    c0, c1 = ch // 2, ch
    p = set()
    if kind in ("iso_enc", "full"):
        p |= {f"latent head + gather, c_latent {cl}"} | (_front_paths(c0, 2 * h, 2 * w) | _front_paths(c1, h, w))
        if c0 % 64:
            p.add("conv A mode 1, a 64-channel chunk straddling two positions")
        if w >= 128:
            p.add("conv A mode 1, tile 128 x 1")
    if kind in ("iso_dec", "full", "tiled"):
        p.add("decoder head, generic (vq_dec_head_kernel)" if cl != 4 else "decoder head, c_latent 4 (vq_dec_head4_kernel)")
        p |= _front_paths(c1, h, w) | _front_paths(c0, 2 * h, 2 * w)
        tp = c0 % 32 == 0 and c0 <= 768
        if kind != "tiled":
            p.add("out_block thread per position (vq_out_block_tp_kernel), modes 0-2" if tp
                  else "out_block warp per position (vq_out_block_kernel), modes 0-2")
        if c1 % 64:
            p.add("conv A mode 2, a partial 64-channel chunk")
        if w >= 128:
            p.add("conv A mode 2, tile 128 x 1")
    if kind == "tiled":
        p |= {"tiled decode: " + q for q in _front_paths(c1, h, w) | _front_paths(c0, 2 * h, 2 * w)}
        p.add("tiled decode: pad_cast_kernel + bordered ConvTranspose")
    return p


def _coverage():
    cov = {}
    for c, k in VQ_CASES:
        cov.setdefault(f"vq_nearest_kernel<{c}>", []).append(f"vq-{c}-{k}")
    for c in CODEC_CASES:
        for p in _codec_paths(c):
            cov.setdefault(p, []).append(c["id"])
    for fc in FRONT_CASES:
        for p in _front_paths(fc["c"], fc["h"], fc["w"]):
            cov.setdefault("resblock " + p, []).append(fc["id"])
        if fc["c"] in (160, 256, 512):
            cov.setdefault("resblock front fused at its 160 / 256 / 512 edges", []).append(fc["id"])
    return cov


COVERAGE = _coverage()
REQUIRED_PATHS = ([f"vq_nearest_kernel<{c}>" for c in range(1, 9)]
                  + [f"latent head + gather, c_latent {cl}" for cl in (1, 2, 3, 4, 5, 8)]
                  + ["decoder head, generic (vq_dec_head_kernel)", "decoder head, c_latent 4 (vq_dec_head4_kernel)",
                     "out_block thread per position (vq_out_block_tp_kernel), modes 0-2",
                     "out_block warp per position (vq_out_block_kernel), modes 0-2",
                     "front fused, 64 threads (vq_front_patch_kernel<64,6>)", "front fused, 128 threads (vq_front_patch_kernel<128,3>)",
                     "front three-launch (ln_rows + vq_dw_residual_kernel + ln_rows)",
                     "resblock front fused, 64 threads (vq_front_patch_kernel<64,6>)",
                     "resblock front fused, 128 threads (vq_front_patch_kernel<128,3>)",
                     "resblock front three-launch (ln_rows + vq_dw_residual_kernel + ln_rows)",
                     "resblock front fused at its 160 / 256 / 512 edges",
                     "conv A mode 1, a 64-channel chunk straddling two positions", "conv A mode 2, a partial 64-channel chunk",
                     "conv A mode 1, tile 128 x 1", "conv A mode 2, tile 128 x 1",
                     "tiled decode: front fused, 64 threads (vq_front_patch_kernel<64,6>)",
                     "tiled decode: front fused, 128 threads (vq_front_patch_kernel<128,3>)",
                     "tiled decode: front three-launch (ln_rows + vq_dw_residual_kernel + ln_rows)",
                     "tiled decode: pad_cast_kernel + bordered ConvTranspose"])


def test_coverage_table():
    missing = [p for p in REQUIRED_PATHS if not COVERAGE.get(p)]
    assert not missing, f"no case runs: {missing}"
    # the out_block cases include both dispatch edges: c0 = 768 (shared-memory limit, thread per position) and c0 = 800
    tp = {c["ch"] // 2 for c in CODEC_CASES if c["ch"] // 2 % 32 == 0 and c["ch"] // 2 <= 768}
    assert 768 in tp and any(c["ch"] // 2 == 800 for c in CODEC_CASES)
    _log(dict(section="coverage", rows={p: len(ids) for p, ids in sorted(COVERAGE.items())}))
