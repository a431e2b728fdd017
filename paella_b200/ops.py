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


# ------------------------------------------------------------------ per-sample generators
# ``generator`` may be a list of B CUDA generators, one per sample: sample b then draws on its own generator exactly what the
# op run on that sample alone (batch 1) draws, so its result depends only on its own seed, not on its batch.
MAX_PER_SAMPLE_NUMEL = 2 ** 29      # torch splits a larger fp32 draw into two kernels (philox_row_chunks)


def per_sample(generator) -> bool:
    return isinstance(generator, (list, tuple))


def check_generators(generators, batch: int, device) -> None:
    """A per-sample generator list: one distinct CUDA generator per sample, all on ``device``."""
    if len(generators) != batch:
        raise ValueError(f"generator: got a list of {len(generators)} generators for a batch of {batch} (one per sample)")
    device = torch.device(device)
    dev_idx = device.index if device.index is not None else torch.cuda.current_device()
    seen = set()
    for i, g in enumerate(generators):
        if not isinstance(g, torch.Generator) or g.device.type != "cuda":
            where = g.device if isinstance(g, torch.Generator) else type(g).__name__
            raise ValueError(f"generator[{i}] must be a CUDA torch.Generator (got {where})")
        g_idx = g.device.index if g.device.index is not None else torch.cuda.current_device()
        if g_idx != dev_idx:
            raise ValueError(f"generator[{i}] is on cuda:{g_idx}, the model on cuda:{dev_idx}")
        if id(g) in seen:
            raise ValueError(f"generator[{i}] appears more than once in the list; its state would be ambiguous")
        seen.add(id(g))


def check_per_sample_numel(numel: int) -> None:
    if numel > MAX_PER_SAMPLE_NUMEL:
        raise ValueError(f"per-sample generators: one sample's draw of {numel} elements exceeds 2^29, which torch would split "
                         "into two kernels (unsupported); use a smaller latent grid")


def philox_values(generators, numel: int, device) -> list:
    """The (seed, philox offset) pairs, flattened, of one draw of ``numel`` elements per sample as int64 values (the uint64
    seed bit for bit); advances each generator."""
    check_per_sample_numel(numel)
    vals = []
    for g in generators:
        seed, off = take_philox(numel, device, g)
        if off % 4:
            raise ValueError(f"generator offset {off} is not a multiple of 4")
        vals += [seed - 2 ** 64 if seed >= 2 ** 63 else seed, off]
    return vals


def philox_table(generators, numel: int, device) -> torch.Tensor:
    """Device int64 [B, 2] of (seed, philox offset) for one draw of ``numel`` elements per sample; advances each generator.
    Built in pinned memory and copied asynchronously: no host synchronisation, no pageable copy."""
    vals = philox_values(generators, numel, device)
    return torch.tensor(vals, dtype=torch.int64, pin_memory=True).view(-1, 2).to(device, non_blocking=True)


# ------------------------------------------------------------------ per-sample sampling parameters
# ``cfg`` and ``temperature`` may be CPU float tensors with one value per sample.  The kernels then read a device table
# float32 [B, 3] of (cfg, 1 - cfg, 1/T): the fp32 constants the scalar entry points derive from their double arguments,
# (float)cfg, (float)(1.0 - cfg) and 1.0f / (float)T, so sample b is computed exactly as a scalar call on its own values.
def per_sample_values(name: str, value, batch: int, pair: bool = False) -> list:
    """A per-sample argument -- a CPU floating-point tensor [batch] ([batch, 2] for a (start, end) pair) -- as Python floats, each
    the scalar a call on that sample alone takes.  ValueError for a CUDA tensor (reading it would synchronise the stream), a
    wrong shape, or a NaN or inf."""
    if value.device.type != "cpu":
        raise ValueError(f"{name}: per-sample values must be a CPU tensor (got {value.device}; reading it would synchronise the stream)")
    if not value.is_floating_point():
        raise ValueError(f"{name}: per-sample values must be a floating-point tensor (got {value.dtype})")
    want = (batch, 2) if pair else (batch,)
    if tuple(value.shape) != want:
        raise ValueError(f"{name}: per-sample values of shape {list(value.shape)} for a batch of {batch} (expected {list(want)})")
    if not bool(torch.isfinite(value).all()):
        raise ValueError(f"{name}: per-sample values must be finite (got {value.tolist()})")
    return value.tolist()


def check_temperatures(name: str, temps) -> None:
    if not all(t > 0 for t in temps):
        raise ValueError(f"{name}: every temperature must be > 0 (got {list(temps)})")


def sampling_params(cfgs, temperatures) -> torch.Tensor:
    """CPU float32 [..., 3] of (cfg, 1 - cfg, 1/T) from equally shaped nested lists of Python floats (cfg) and of fp32 values
    (T): (float)cfg and (float)(1.0 - cfg) from the doubles, 1/T as an fp32 division, like the scalar entry points."""
    c = torch.tensor(cfgs, dtype=torch.float64)
    t32 = torch.tensor(temperatures, dtype=torch.float64).float()
    return torch.stack([c.float(), (1.0 - c).float(), torch.ones_like(t32) / t32], -1)


def check_attn_weight_vector(name: str, value, max_len: int) -> torch.Tensor:
    """One sample's ``attn_weights``: a 1-D CPU floating-point tensor of finite values, at most ``max_len`` long (the smallest
    key count the sample sees in any AttnBlock; the reference fails on a longer vector).  Returns it as CPU float32.
    ValueError otherwise, like per_sample_values."""
    if not torch.is_tensor(value):
        raise ValueError(f"{name}: expected None or a 1-D CPU float tensor (got {type(value).__name__})")
    if value.device.type != "cpu":
        raise ValueError(f"{name}: per-sample weights must be a CPU tensor (got {value.device}; reading it would synchronise the stream)")
    if not value.is_floating_point() or value.dim() != 1:
        raise ValueError(f"{name}: expected a 1-D floating-point tensor (got {value.dtype} of shape {list(value.shape)})")
    if not bool(torch.isfinite(value).all()):
        raise ValueError(f"{name}: weights must be finite")
    if value.numel() > max_len:
        raise ValueError(f"{name}: {value.numel()} weights, but the sample attends to only {max_len} keys in its smallest AttnBlock")
    return value.float()


def attn_weights_table(entries, batch: int, max_lens) -> Tuple[torch.Tensor, torch.Tensor]:
    """Per-sample ``attn_weights``: a list or tuple of ``batch`` entries, each None (unweighted) or a 1-D CPU float tensor, as
    the host table the attention kernels read: CPU float32 [batch, w_ld] (row b zero-padded past its length) and int32 [batch]
    of the row lengths (0 for None).  ``max_lens[b]`` bounds sample b's length (check_attn_weight_vector).  ValueError for the
    wrong number of entries or a bad entry."""
    if len(entries) != batch:
        raise ValueError(f"attn_weights: got {len(entries)} entries for a batch of {batch} (one per sample, None for unweighted)")
    rows = [None if v is None else check_attn_weight_vector(f"attn_weights[{i}]", v, max_lens[i]) for i, v in enumerate(entries)]
    lens = torch.tensor([0 if v is None else v.numel() for v in rows], dtype=torch.int32)
    table = torch.zeros(batch, max(1, int(lens.max()) if batch else 1), dtype=torch.float32)
    for i, v in enumerate(rows):
        if v is not None:
            table[i, :v.numel()] = v
    return table, lens


def attn_weights_to_device(table: torch.Tensor, lens: torch.Tensor, device) -> Tuple[torch.Tensor, torch.Tensor]:
    """The table of attn_weights_table on the device in one asynchronous copy: (float32 [rows, w_ld], int32 [rows])."""
    buf = to_device_async(torch.cat([table.view(torch.int32).view(-1), lens]), device)
    return buf[:table.numel()].view(torch.float32).view(table.shape), buf[table.numel():]


def to_device_async(host: torch.Tensor, device) -> torch.Tensor:
    """One asynchronous copy from pinned memory: no host synchronisation, no pageable copy."""
    buf = torch.empty(host.shape, dtype=host.dtype, pin_memory=True)
    buf.copy_(host)
    return buf.to(device, non_blocking=True)


def to_device_packed(parts, device) -> list:
    """Several CPU tensors in one asynchronous copy from pinned memory: returns their device copies, each with its own dtype
    and shape, each starting at an 8-byte boundary of one buffer."""
    chunks, offs, n = [], [], 0
    for p in parts:
        pad = -n % 8
        if pad:
            chunks.append(torch.zeros(pad, dtype=torch.uint8))
            n += pad
        offs.append(n)
        chunks.append(p.contiguous().reshape(-1).view(torch.uint8))
        n += p.numel() * p.element_size()
    buf = to_device_async(torch.cat(chunks), device)
    return [buf[o:o + p.numel() * p.element_size()].view(p.dtype).view(p.shape) for o, p in zip(offs, parts)]


def sampling_params_table(cfg, temperature, batch: int, device) -> torch.Tensor:
    """Device float32 [batch, 3] for ``cfg`` (float, None or a CPU tensor [batch]) and ``temperature`` (float or a CPU tensor
    [batch]); a scalar applies to every sample.  ValueError (nothing enqueued) for a bad per-sample value or a T <= 0."""
    cfgs = per_sample_values("cfg", cfg, batch) if torch.is_tensor(cfg) else [float(cfg) if cfg is not None else 0.0] * batch
    temps = per_sample_values("temperature", temperature, batch) if torch.is_tensor(temperature) else [float(temperature)] * batch
    check_temperatures("temperature", temps)
    return to_device_async(sampling_params(cfgs, temps), device)


# ------------------------------------------------------------------ per-sample sampling modes
# The notebook's sampling modes (paella_inference.ipynb cell 3).  'multinomial' draws H*W*num_labels exponentials per step; 'argmax'
# and 'quant' draw nothing.  A step with several modes sends one int32 table to the device: the mode code of every sample, then
# the samples in argmax mode, then the samples in quant mode, each list ascending.
SAMPLING_MODES = ("multinomial", "argmax", "quant")
RESAMPLE_CHUNK = 8      # guided samples per out_mapper GEMM of pb200_paella_resample_samples (bounds its logits scratch)


def check_mode(name: str, mode) -> str:
    if not isinstance(mode, str) or mode not in SAMPLING_MODES:
        raise ValueError(f"{name}={mode!r}: expected one of {', '.join(SAMPLING_MODES)}")
    return mode


def check_quant_steps(name: str, value) -> Optional[int]:
    """``sampling_quant_steps``: None, or a non-negative int (steps i >= value use 'quant')."""
    if value is None:
        return None
    if isinstance(value, bool) or not isinstance(value, int) or value < 0:
        raise ValueError(f"{name}={value!r}: expected None or an int >= 0")
    return value


def mode_at(mode: str, quant_steps: Optional[int], step: int) -> str:
    """The mode of step ``step`` (0-based) of a sample: 'quant' from step ``quant_steps`` on, its own mode before."""
    return "quant" if quant_steps is not None and step >= quant_steps else mode


def mode_table(modes) -> torch.Tensor:
    """CPU int32 table of one step's per-sample modes (see above): [B] codes (SAMPLING_MODES index), then the argmax samples,
    then the quant samples."""
    codes = [SAMPLING_MODES.index(md) for md in modes]
    lists = [b for c in (1, 2) for b, cb in enumerate(codes) if cb == c]
    return torch.tensor(codes + lists, dtype=torch.int32)


# ------------------------------------------------------------------ random ops
def randint(num_labels: int, size, device, generator=None) -> torch.Tensor:
    """torch.randint(0, num_labels, size, device=device)  [ref/src/utils.py:37]"""
    out = torch.empty(size, dtype=torch.int64, device=device)
    if per_sample(generator):
        check_generators(generator, out.shape[0], out.device)
        return randint_per_sample(out, num_labels, philox_table(generator, out[0].numel(), out.device))
    seed, off = take_philox(out.numel(), out.device, generator)
    check(lib().pb200_randint(ptr(out), out.numel(), num_labels, seed, off, current_stream()), "pb200_randint")
    return out


def randint_per_sample(out: torch.Tensor, num_labels: int, table: torch.Tensor, slot: Optional[torch.Tensor] = None,
                       batch: Optional[int] = None) -> torch.Tensor:
    """One launch of per-sample randint draws: sample b draws on (seed, offset) = ``table[b]`` (philox_table) what a batch-1
    randint over ``out[0].numel()`` elements draws, into row b of ``out`` (row ``slot[b]`` with an int32 device slot map)."""
    hw = out[0].numel()
    n = out.shape[0] if batch is None else batch
    check(lib().pb200_randint_per_sample(ptr(out), ptr(slot), n, hw, num_labels, ptr(table), current_stream()),
          "pb200_randint_per_sample")
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


def resample_logits(logits_c: torch.Tensor, logits_u: Optional[torch.Tensor], cfg, temperature, mode: str = "multinomial",
                    generator=None) -> torch.Tensor:
    """ref/src/utils.py:45-50 on reference-layout logits [B,K,H,W] -> tokens [B,H,W].  ``cfg`` and ``temperature`` are floats,
    or CPU tensors [B] of per-sample values (see sampling_params_table)."""
    if torch.is_tensor(cfg) or torch.is_tensor(temperature):
        return resample_logits_params(logits_c, logits_u, sampling_params_table(cfg, temperature, logits_c.shape[0], logits_c.device),
                                      mode, generator)
    return _resample_logits(logits_c, logits_u, (float(cfg), float(temperature)), mode, generator)


def resample_logits_params(logits_c: torch.Tensor, logits_u: Optional[torch.Tensor], params: torch.Tensor,
                           mode: str = "multinomial", generator=None) -> torch.Tensor:
    """resample_logits with per-sample (cfg, 1 - cfg, 1/T): ``params`` device float32 [B, 3] (sampling_params_table), in one
    launch over the batch per random stream."""
    return _resample_logits(logits_c, logits_u, params, mode, generator)


def _resample_logits(logits_c, logits_u, par, mode, generator):
    """``par``: (cfg, temperature) floats, or a device params table [B, 3]."""
    if per_sample(generator) and mode == "multinomial":
        check_generators(generator, logits_c.shape[0], logits_c.device)
        check_per_sample_numel(logits_c[0].numel())
        return torch.cat([_resample_logits(logits_c[b:b + 1], logits_u[b:b + 1] if logits_u is not None else None,
                                           par[b:b + 1] if torch.is_tensor(par) else par, mode, g) for b, g in enumerate(generator)])
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
        lu_p = ptr(lu[b0:b1]) if lu is not None else None
        if torch.is_tensor(par):
            check(lib().pb200_resample_logits_params(ptr(lc[b0:b1]), lu_p, b1 - b0, K, hw, ptr(par[b0:b1]), m, seed, off,
                                                     ptr(out[b0:b1]), current_stream()), "pb200_resample_logits_params")
        else:
            check(lib().pb200_resample_logits(ptr(lc[b0:b1]), lu_p, b1 - b0, K, hw, par[0], par[1], m, seed, off, ptr(out[b0:b1]),
                                              current_stream()), "pb200_resample_logits")
    return out


def resample_quant(logits_c: torch.Tensor, logits_u: Optional[torch.Tensor], cfg, temperature,
                   codebook: torch.Tensor) -> torch.Tensor:
    """Notebook `mode='quant'`: softmax(l/T) @ codebook, then nearest code -> tokens [B,H,W] (no random draw).  ``cfg`` and
    ``temperature`` as in resample_logits."""
    if torch.is_tensor(cfg) or torch.is_tensor(temperature):
        return resample_quant_params(logits_c, logits_u, sampling_params_table(cfg, temperature, logits_c.shape[0], logits_c.device),
                                     codebook)
    return _resample_quant(logits_c, logits_u, (float(cfg), float(temperature)), codebook)


def resample_quant_params(logits_c: torch.Tensor, logits_u: Optional[torch.Tensor], params: torch.Tensor,
                          codebook: torch.Tensor) -> torch.Tensor:
    """resample_quant with per-sample (cfg, 1 - cfg, 1/T) (``params`` as in resample_logits_params), in one launch."""
    return _resample_quant(logits_c, logits_u, params, codebook)


def _resample_quant(logits_c, logits_u, par, codebook):
    B, K = logits_c.shape[:2]
    hw = logits_c[0, 0].numel()
    lc = logits_c.contiguous().float()
    lu = logits_u.contiguous().float() if logits_u is not None else None
    cb = codebook.contiguous().float()
    out = torch.empty((B,) + tuple(logits_c.shape[2:]), dtype=torch.int64, device=lc.device)
    if torch.is_tensor(par):
        check(lib().pb200_resample_quant_params(ptr(lc), ptr(lu), B, K, hw, ptr(par), ptr(cb), cb.shape[1], ptr(out),
                                                current_stream()), "pb200_resample_quant_params")
    else:
        check(lib().pb200_resample_quant(ptr(lc), ptr(lu), B, K, hw, par[0], par[1], ptr(cb), cb.shape[1], ptr(out),
                                         current_stream()), "pb200_resample_quant")
    return out


def _region_u8(region: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """A bool or uint8 device region as the kernels' uint8 bytes (a view, no copy)."""
    if region is None:
        return None
    region = region.contiguous()
    return region.view(torch.uint8) if region.dtype == torch.bool else region


def add_noise(x: torch.Tensor, t: torch.Tensor, random_x: Optional[torch.Tensor], num_labels: int, generator=None,
              return_mask: bool = True, src: Optional[torch.Tensor] = None, region: Optional[torch.Tensor] = None):
    """Paella.add_noise with mask=None  [ref/src/modules.py:277-283].  With ``src`` (int64, like x) and ``region`` (bool or
    uint8, like x): where(region, add_noise(x, t, mask=m & region, random_x), src) for the mask m this call draws -- the
    same draws as without a region; the returned mask is m & region."""
    x = x.contiguous()
    B = x.shape[0]
    hw = x[0].numel()
    out = torch.empty_like(x)
    mask = torch.empty_like(x) if return_mask else None
    src = src.contiguous() if src is not None else None
    region = _region_u8(region)
    if per_sample(generator):
        check_generators(generator, B, x.device)
        check_per_sample_numel(hw)
        table = philox_table(generator, hw, x.device)
        if random_x is None:
            philox_values(generator, hw, x.device)          # the randint_like draw follows the mask draw
        add_noise_per_sample(x, t.contiguous().float(), random_x.contiguous() if random_x is not None else None, num_labels, table,
                             out, mask, src=src, region=region)
        return out, mask
    seed, off = take_philox(x.numel(), x.device, generator)
    if random_x is None:
        take_philox(x.numel(), x.device, generator)      # the randint_like draw follows the mask draw
    else:
        random_x = random_x.contiguous()
    check(lib().pb200_add_noise_region(ptr(x), ptr(random_x), ptr(src), ptr(region), ptr(t.contiguous().float()), B, hw, num_labels,
                                       seed, off, ptr(out), ptr(mask), current_stream()), "pb200_add_noise_region")
    return out, mask


def composite(x: torch.Tensor, src: torch.Tensor, region: torch.Tensor, neg_t: torch.Tensor,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """where(region, x, src) for int64 x, src and a bool / uint8 region of one shape [B, ...]: the add-noise launch with every
    t < 0 (``neg_t``, fp32 [B] on the device), which renoises nothing and so takes no Philox offset from any generator."""
    x = x.contiguous()
    out = torch.empty_like(x) if out is None else out
    check(lib().pb200_add_noise_region(ptr(x), None, ptr(src.contiguous()), ptr(_region_u8(region)), ptr(neg_t), x.shape[0],
                                       x[0].numel(), 1, 0, 0, ptr(out), None, current_stream()), "pb200_add_noise_region")
    return out


def add_noise_per_sample(x: torch.Tensor, t: torch.Tensor, random_x: Optional[torch.Tensor], num_labels: int, table: torch.Tensor,
                         out: torch.Tensor, mask: Optional[torch.Tensor] = None, slot: Optional[torch.Tensor] = None,
                         src: Optional[torch.Tensor] = None, region: Optional[torch.Tensor] = None) -> None:
    """One launch of per-sample add_noise: sample b (x [B, ...], t fp32 [B]) draws its mask on (seed, offset) = ``table[b]`` and
    takes random_x (or, when None, the randint_like drawn at the next offset) where the mask is set; a sample with t < 0 keeps
    its tokens.  ``slot`` (int32 [B]) places sample b's rows of random_x and out at row slot[b] of those buffers.  ``src`` and
    ``region`` (read at the same rows): outside the region the output is src and the mask 0, as in add_noise."""
    B, hw = x.shape[0], x[0].numel()
    check(lib().pb200_add_noise_region_per_sample(ptr(x), ptr(random_x), ptr(src), ptr(_region_u8(region)), ptr(slot), ptr(t), B, hw,
                                                  num_labels, ptr(table), ptr(out), ptr(mask), current_stream()),
          "pb200_add_noise_region_per_sample")


def gather_rows(pool: torch.Tensor, slot: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[b] = pool[slot[b]] (int64 token rows; ``slot`` int32 [out.shape[0]] on the device), in one launch."""
    check(lib().pb200_gather_rows(ptr(pool), ptr(slot), out.shape[0], out[0].numel(), ptr(out), current_stream()), "pb200_gather_rows")
    return out


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
                                       _lib.EPI_F16_LN, _lib.EPI_RESID_LN_INV_F32) else 0
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
