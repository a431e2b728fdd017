"""Thin Python wrappers over the C ABI's kernel-level entry points (PyTorch tensors in/out).

Random ops consume the torch CUDA generator exactly like the torch ops they replace: they read
(seed, philox offset) from the generator, run the kernel on that stream, and advance the offset by
what the torch kernel would have consumed (ATen/native/cuda/DistributionTemplates.h:50-62).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import GemmEpilogue, check, current_stream, lib, ptr


# ------------------------------------------------------------------ torch CUDA generator bookkeeping
def _generator(device, generator: Optional[torch.Generator]) -> torch.Generator:
    if generator is not None:
        return generator
    idx = device.index if device.index is not None else torch.cuda.current_device()
    return torch.cuda.default_generators[idx]


def take_philox(numel: int, device, generator: Optional[torch.Generator] = None) -> Tuple[int, int]:
    """(seed, offset) for a distribution kernel over ``numel`` elements; advances the generator."""
    g = _generator(device, generator)
    seed, off = g.initial_seed(), g.get_offset()
    g.set_offset(off + lib().pb200_philox_offset_increment(int(numel)))
    return seed, off


def philox_row_chunks(rows: int, k: int, elem_bytes: int = 4):
    """Row ranges [(lo, hi), ...] over which torch runs ONE distribution kernel each for a contiguous [rows, k] tensor.
    TensorIterator splits an iteration space that is not 32-bit indexable (numel > INT32_MAX or last BYTE offset >
    INT32_MAX, i.e. > 2^29 fp32 elements) into halves, first half first, recursively (ATen TensorIterator::split /
    SplitUntil32Bit, DistributionTemplates.h:132-138); every sub-kernel takes its own Philox offset from the generator --
    and the ROOT call has already taken one for the whole tensor before it notices that it must split (it computes its
    execution policy and calls philox_cuda_state first: a 2^30-element draw advances the offset by
    inc(2^30) + 2 inc(2^29)), see ``skip_philox_for_split``.  bs=64 at 32x32x8192 is exactly 2^29 elements (one kernel);
    larger batches split -- mirrored here so the draws stay bit-identical to torch.multinomial's."""
    lim = 2 ** 31 - 1

    def split(n):
        if n <= lim and 1 + (n - 1) * elem_bytes <= lim:
            return [n]
        half = n // 2
        return split(half) + split(n - half)
    out, lo = [], 0
    for n in split(rows * k):
        if n % k != 0:
            raise _lib.PaellaB200Error(f"a {rows}x{k} draw splits inside a row under torch's 32-bit indexing rule; use a batch whose "
                                       "row count is a power-of-two multiple")
        out.append((lo, lo + n // k))
        lo += n // k
    return out


def skip_philox_for_split(chunks, total_numel: int, device, generator=None) -> None:
    """Consume the offset increment torch's root distribution call takes (and never uses) when the tensor has to be split."""
    if len(chunks) > 1:
        take_philox(total_numel, device, generator)


# ------------------------------------------------------------------ random ops
def randint(num_labels: int, size, device, generator=None) -> torch.Tensor:
    """torch.randint(0, num_labels, size, device=device)  [ref/src/utils.py:37]"""
    out = torch.empty(size, dtype=torch.int64, device=device)
    seed, off = take_philox(out.numel(), out.device, generator)
    check(lib().pb200_randint(ptr(out), out.numel(), num_labels, seed, off, current_stream()), "pb200_randint")
    return out


def rand(size, device, generator=None) -> torch.Tensor:
    out = torch.empty(size, dtype=torch.float32, device=device)
    seed, off = take_philox(out.numel(), out.device, generator)
    check(lib().pb200_rand(ptr(out), out.numel(), seed, off, current_stream()), "pb200_rand")
    return out


def multinomial(p: torch.Tensor, generator=None) -> torch.Tensor:
    """torch.multinomial(p, 1)[:, 0] for fp32 p [rows, k]  [ref/src/utils.py:50]"""
    assert p.dim() == 2 and p.dtype == torch.float32
    p = p.contiguous()
    out = torch.empty(p.shape[0], dtype=torch.int64, device=p.device)
    chunks = philox_row_chunks(p.shape[0], p.shape[1])
    skip_philox_for_split(chunks, p.numel(), p.device, generator)
    for lo, hi in chunks:
        seed, off = take_philox((hi - lo) * p.shape[1], p.device, generator)
        check(lib().pb200_multinomial(ptr(p[lo:hi]), hi - lo, p.shape[1], seed, off, ptr(out[lo:hi]), current_stream()),
              "pb200_multinomial")
    return out


def resample_logits(logits_c: torch.Tensor, logits_u: Optional[torch.Tensor], cfg: float, temperature: float,
                    mode: str = "multinomial", generator=None) -> torch.Tensor:
    """ref/src/utils.py:45-50 on reference-layout logits [B,K,H,W] -> tokens [B,H,W]."""
    B, K = logits_c.shape[:2]
    hw = logits_c[0, 0].numel()
    lc = logits_c.contiguous().float()
    lu = logits_u.contiguous().float() if logits_u is not None else None
    out = torch.empty((B,) + tuple(logits_c.shape[2:]), dtype=torch.int64, device=lc.device)
    m = {"multinomial": 0, "argmax": 1}[mode]
    chunks = philox_row_chunks(B * hw, K) if m == 0 else [(0, B * hw)]
    skip_philox_for_split(chunks, B * hw * K, lc.device, generator)
    for lo, hi in chunks:
        if lo % hw or hi % hw:
            raise _lib.PaellaB200Error("resample_logits: torch's 32-bit split of this draw falls inside a sample")
        b0, b1 = lo // hw, hi // hw
        seed, off = take_philox((hi - lo) * K, lc.device, generator) if m == 0 else (0, 0)
        check(lib().pb200_resample_logits(ptr(lc[b0:b1]), ptr(lu[b0:b1]) if lu is not None else None, b1 - b0, K, hw, float(cfg),
                                          float(temperature), m, seed, off, ptr(out[b0:b1]), current_stream()), "pb200_resample_logits")
    return out


def resample_quant(logits_c: torch.Tensor, logits_u: Optional[torch.Tensor], cfg: float, temperature: float,
                   codebook: torch.Tensor) -> torch.Tensor:
    """Notebook `mode='quant'`: softmax(l/T) @ codebook, then nearest code -> tokens [B,H,W] (no random draw)."""
    B, K = logits_c.shape[:2]
    hw = logits_c[0, 0].numel()
    lc = logits_c.contiguous().float()
    lu = logits_u.contiguous().float() if logits_u is not None else None
    cb = codebook.contiguous().float()
    out = torch.empty((B,) + tuple(logits_c.shape[2:]), dtype=torch.int64, device=lc.device)
    check(lib().pb200_resample_quant(ptr(lc), ptr(lu), B, K, hw, float(cfg), float(temperature), ptr(cb), cb.shape[1], ptr(out),
                                     current_stream()), "pb200_resample_quant")
    return out


def add_noise(x: torch.Tensor, t: torch.Tensor, random_x: Optional[torch.Tensor], num_labels: int, generator=None,
              return_mask: bool = True):
    """Paella.add_noise with mask=None  [ref/src/modules.py:277-283]"""
    x = x.contiguous()
    B = x.shape[0]
    hw = x[0].numel()
    out = torch.empty_like(x)
    mask = torch.empty_like(x) if return_mask else None
    seed, off = take_philox(x.numel(), x.device, generator)
    if random_x is None:
        take_philox(x.numel(), x.device, generator)      # the randint_like draw follows the mask draw
    else:
        random_x = random_x.contiguous()
    check(lib().pb200_add_noise(ptr(x), ptr(random_x), ptr(t.contiguous().float()), B, hw, num_labels, seed, off, ptr(out),
                                ptr(mask), current_stream()), "pb200_add_noise")
    return out, mask


# ------------------------------------------------------------------ vector quantiser
def vq_nearest(x: torch.Tensor, codebook: torch.Tensor) -> torch.Tensor:
    """x fp32 [..., C] -> int64 [...] nearest code."""
    flat = x.contiguous().float().view(-1, x.shape[-1])
    out = torch.empty(flat.shape[0], dtype=torch.int64, device=x.device)
    check(lib().pb200_vq_nearest(ptr(flat), flat.shape[0], flat.shape[1], ptr(codebook.contiguous().float()),
                                 codebook.shape[0], ptr(out), current_stream()), "pb200_vq_nearest")
    return out.view(x.shape[:-1])


def vq_gather(idx: torch.Tensor, codebook: torch.Tensor) -> torch.Tensor:
    idx = idx.contiguous()
    out = torch.empty(idx.shape + (codebook.shape[1],), dtype=torch.float32, device=idx.device)
    check(lib().pb200_vq_gather(ptr(idx), idx.numel(), ptr(codebook.contiguous().float()), codebook.shape[0],
                                codebook.shape[1], ptr(out), current_stream()), "pb200_vq_gather")
    return out


# ------------------------------------------------------------------ GEMM (unit-test surface)
def gemm_f16(a: torch.Tensor, w: torch.Tensor, mode: int, out: torch.Tensor, bias=None, resid=None, alpha: float = 1.0,
             sqsum=None, rows_per_sample: int = 0, film=None, film_off: int = 0, remap=(0, 0), up=(0, 0, 0), out16=None,
             ln_stat=None, ln_wsum=None, ln_shift=None, ln_mean_out=None, a_scale=None) -> torch.Tensor:
    """out = epilogue(a[M,K] @ w[N,K]^T); a, w fp16 contiguous."""
    assert a.dtype == torch.float16 and w.dtype == torch.float16 and a.shape[1] == w.shape[1]
    M, K = a.shape
    N = w.shape[0]
    ep = GemmEpilogue()
    ep.mode = mode
    ep.bias = ptr(bias).value if bias is not None else None
    ep.out = ptr(out).value
    ep.ldo = out.shape[-1] if mode in (_lib.EPI_F16, _lib.EPI_F32, _lib.EPI_GELU_F16, _lib.EPI_RESID_F32, _lib.EPI_RESID_LN_F32,
                                       _lib.EPI_F16_LN) else 0
    ep.out16 = ptr(out16).value if out16 is not None else None
    ep.ln_stat = ptr(ln_stat).value if ln_stat is not None else None
    ep.ln_wsum = ptr(ln_wsum).value if ln_wsum is not None else None
    ep.ln_c = K if mode == _lib.EPI_F16_LN else 0
    ep.ln_shift = ptr(ln_shift).value if ln_shift is not None else None
    ep.ln_mean_out = ptr(ln_mean_out).value if ln_mean_out is not None else None
    ep.a_scale = ptr(a_scale).value if a_scale is not None else None
    ep.a_scale_ld = a_scale.stride(0) if a_scale is not None else 0
    ep.resid = ptr(resid).value if resid is not None else None
    ep.ldr = resid.shape[-1] if resid is not None else 0
    ep.alpha = alpha
    ep.sqsum = ptr(sqsum).value if sqsum is not None else None
    ep.rows_per_sample = rows_per_sample
    ep.film = ptr(film).value if film is not None else None
    ep.film_ld = film.shape[-1] if film is not None else 0
    ep.film_off = film_off
    ep.remap_in, ep.remap_out = remap
    ep.up_h, ep.up_w, ep.up_cout = up
    check(lib().pb200_gemm_f16(ptr(a), a.stride(0), ptr(w), w.stride(0), M, N, K, ep, current_stream()), "pb200_gemm_f16")
    return out
